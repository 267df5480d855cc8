"""
Generates tests/golden/moo.npz and tests/golden/incremental.npz by running the UNMODIFIED reference
(dragonfly-opt 0.1.7, source tree in $DRAGONFLY_REF).  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF \
        python -W ignore tests/golden/make_golden_moo.py

moo.npz          two objectives on one 6-D domain, the four multi-objective acquisitions
                 (multiobjective_gpb_acquisitions.py:19-107): per-candidate scalarised scores on a fixed
                 candidate matrix + the end-to-end recommendations under a seeded global RNG.
incremental.npz  GP.add_data_multiple / add_data_single (gp_core.py:135-146): the reference's posterior
                 after appending observations to a built GP (it rebuilds from scratch).
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
from dragonfly.opt import multiobjective_gpb_acquisitions as ref_moo  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa

from dragonfly_b200 import synth_data  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def save(name, **arrs):
  path = os.path.join(HERE, name + '.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrs.items()})
  print('wrote %s (%.1f KB)' % (path, os.path.getsize(path) / 1024.0))


def second_objective(X):
  return -np.sum((X - 0.4) ** 2, axis=1) + 0.3 * np.sin(5 * X[:, 0])


def case_moo():
  n, d, t = 120, 6, 120
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=n, n_cand=1200)
  X, Y1, C = w['X'], w['Y'], w['candidates']
  Y2 = second_objective(X)
  k = w['kernel']
  m1, m2 = float(np.median(Y1)), float(np.median(Y2))
  nv1, nv2 = w['noise_var'], 0.01 * float(Y2.var())
  se_scale, se_bw = float(Y2.var()), [0.35] * d
  gps = [GP(X, Y1, MaternKernel(d, 2.5, k['scale'], k['dim_bandwidths']), const_mean(m1), nv1),
         GP(X, Y2, SEKernel(d, se_scale, se_bw), const_mean(m2), nv2)]
  weights = np.array([0.6, 0.4])
  refs = [0.1, -1.0]
  dom = EuclideanDomain([[0, 1]] * d)

  def anc(max_evals, in_progress=()):
    return Namespace(max_evals=max_evals, t=t, domain=dom, acq_opt_method='rand', handle_parallel='halluc',
                     eval_points_in_progress=list(in_progress), is_mf=False, obj_weights=weights,
                     reference_point=refs)

  out = dict(X=X, Y1=Y1, Y2=Y2, C=C, scale1=k['scale'], bws1=k['dim_bandwidths'], mean1=m1, noise1=nv1,
             scale2=se_scale, bws2=se_bw, mean2=m2, noise2=nv2, weights=weights, refs=refs, t=t,
             beta=ref_moo._get_ucb_beta_th(d, t))
  # per-candidate scores: capture the acquisition closures by replacing the maximiser in the module
  real_max = ref_moo.maximise_acquisition
  ref_moo.maximise_acquisition = lambda acq, anc_data, *a, **kw: acq
  try:
    out['lin_ucb_scores'] = ref_moo.mo_lin_asy_ucb(gps, anc(10))(C)
    out['tch_ucb_scores'] = ref_moo.mo_tch_asy_ucb(gps, anc(10))(C)
  finally:
    ref_moo.maximise_acquisition = real_max
  # end to end (random maximiser, global RNG)
  for name, m_evals in [('lin_ucb', 1500), ('tch_ucb', 1500), ('lin_ts', 300), ('tch_ts', 300)]:
    np.random.seed(9)
    out['e2e_%s_point' % name] = getattr(ref_moo.asy, name)(gps, anc(m_evals))
  Xh = np.random.RandomState(4).random_sample((2, d))
  np.random.seed(9)
  out['e2e_lin_ts_halluc_point'] = ref_moo.asy.lin_ts(gps, anc(300, in_progress=list(Xh)))
  out['Xh'] = Xh
  save('moo', **out)


def case_incremental():
  n0, q = 300, 6
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=n0 + q, n_cand=800)
  X, Y, C = w['X'], w['Y'], w['candidates']
  k = w['kernel']
  gp = GP(X[:n0], Y[:n0], MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']), const_mean(w['mean_const']),
          w['noise_var'])
  gp.add_data_multiple(list(X[n0:n0 + 4]), list(Y[n0:n0 + 4]))
  gp.add_data_single(X[n0 + 4], Y[n0 + 4])
  gp.add_data_single(X[n0 + 5], Y[n0 + 5])
  mu, sd = gp.eval(C, 'std')
  save('incremental', X=X, Y=Y, C=C, n0=n0, scale=k['scale'], bws=k['dim_bandwidths'],
       mean_const=w['mean_const'], noise_var=w['noise_var'], L=gp.L, alpha=gp.alpha,
       lml=gp.compute_log_marginal_likelihood(), mu=mu, sd=sd)


if __name__ == '__main__':
  case_moo()
  case_incremental()
