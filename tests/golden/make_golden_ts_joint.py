"""
Generates tests/golden/ts_joint.npz by running the UNMODIFIED reference (dragonfly-opt 0.1.7, source tree in
$DRAGONFLY_REF): Thompson sampling over more candidates than one 4096-candidate device block, where the reference draws
every sample jointly over all candidates (gp_core.py:173-185, general_utils.py:166-232).

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF \
        python -W ignore tests/golden/make_golden_ts_joint.py

ts_joint.npz  a Matern-2.5 GP (d = 6, N = 300) and a second SE GP on the same points;
              draw_samples(4, C) over M = 6000 candidates with the normals it consumed; the diagonal and 200 fixed
              entries of eval(C, 'covar'); asy_ts and the multi-objective lin_ts recommendations at max_evals = 6000
              with acq_opt_method 'rand', each with the gap between the best and the second-best sampled value.
              Seeds are kept only when every gap is at least 1e-5, so that sample errors far below it cannot flip an
              arg-max.
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402
from dragonfly.gp.kernel import SEKernel, MaternKernel  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.opt import multiobjective_gpb_acquisitions as ref_moo  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa

from dragonfly_b200 import synth_data  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__

M = 6000
MIN_GAP = 1e-5


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def second_objective(X):
  return -np.sum((X - 0.4) ** 2, axis=1) + 0.3 * np.sin(5 * X[:, 0])


_RECORD = []


def _recording(module):
  """ Wraps module.maximise_acquisition so that the values of the vectorised objective are recorded; the RNG is
      consumed exactly as without the wrapper. """
  real = module.maximise_acquisition

  def wrapped(acq, anc_data, *args, **kwargs):
    def rec(x):
      v = np.asarray(acq(x)).ravel()
      _RECORD.append(v)
      return v
    return real(rec, anc_data, *args, **kwargs)
  return real, wrapped


def gap(v):
  idx = int(np.argmax(v))
  return float(v[idx] - np.delete(v, idx).max()), idx


def main():
  rs = np.random.RandomState(2026)
  n, d = 300, 6
  X = rs.random_sample((n, d))
  Y1 = synth_data.hartmann6(X)
  Y2 = second_objective(X)
  scale1, bws1, noise1, mean1 = float(Y1.var()), [0.3] * d, 0.01 * float(Y1.var()), float(np.median(Y1))
  scale2, bws2, noise2, mean2 = float(Y2.var()), [0.35] * d, 0.01 * float(Y2.var()), float(np.median(Y2))
  gp1 = GP(X, Y1, MaternKernel(d, 2.5, scale1, bws1), const_mean(mean1), noise1)
  gp2 = GP(X, Y2, SEKernel(d, scale2, bws2), const_mean(mean2), noise2)
  C = rs.random_sample((M, d))
  out = dict(X=X, Y1=Y1, Y2=Y2, C=C, scale1=scale1, bws1=bws1, noise1=noise1, mean1=mean1, scale2=scale2, bws2=bws2,
             noise2=noise2, mean2=mean2)

  # draw_samples(4, C): the normals are the first M x 4 of the seeded stream
  np.random.seed(11)
  out['samples'] = gp1.draw_samples(4, C)
  np.random.seed(11)
  out['U'] = np.random.normal(size=(M, 4))
  out['samples_gap'] = np.array([gap(s)[0] for s in out['samples']])
  mu, covar = gp1.eval(C, 'covar')
  out['mu'] = mu
  out['covar_diag'] = np.diag(covar).copy()
  idx = np.random.RandomState(5).randint(0, M, size=(200, 2))
  out['covar_idx'] = idx
  out['covar_vals'] = covar[idx[:, 0], idx[:, 1]]
  del covar

  dom = EuclideanDomain([[0, 1]] * d)
  weights, refs = np.array([0.6, 0.4]), [0.1, -1.0]

  def anc():
    return Namespace(max_evals=M, t=n, domain=dom, acq_opt_method='rand', handle_parallel='halluc',
                     eval_points_in_progress=[], is_mf=False, obj_weights=weights, reference_point=refs,
                     curr_max_val=float(Y1.max()))

  for name, module, call in [('asy_ts', ref_acq, lambda: ref_acq.asy.ts(gp1, anc())),
                             ('lin_ts', ref_moo, lambda: ref_moo.asy.lin_ts([gp1, gp2], anc()))]:
    real, wrapped = _recording(module)
    module.maximise_acquisition = wrapped
    try:
      seed = 100
      while True:
        del _RECORD[:]
        np.random.seed(seed)
        pt = call()
        g, _ = gap(_RECORD[0])
        if len(_RECORD) == 1 and len(_RECORD[0]) == M and g >= MIN_GAP:
          break
        seed += 1
    finally:
      module.maximise_acquisition = real
    out['%s_seed' % name] = seed
    out['%s_point' % name] = np.asarray(pt)
    out['%s_gap' % name] = g
    out['%s_index' % name] = gap(_RECORD[0])[1]
    print(name, 'seed', seed, 'gap', g)
  out['weights'], out['refs'] = weights, np.array(refs)
  path = os.path.join(HERE, 'ts_joint.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in out.items()})
  print('wrote %s (%.1f KB)' % (path, os.path.getsize(path) / 1024.0))


if __name__ == '__main__':
  main()
