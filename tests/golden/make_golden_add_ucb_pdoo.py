"""
Generates tests/golden/add_ucb_pdoo.npz by running the UNMODIFIED reference's Add-UCB (dragonfly/opt/gpb_acquisitions.py:
_add_ucb, _add_ucb_for_boca) with the sequential maximisers: acq_opt_method 'pdoo', and 'direct', which falls back to
PDOO without the Fortran DIRECT extension (oper_utils.py:121-137).  Authoring container:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore \\
        tests/golden/make_golden_add_ucb_pdoo.py

An additive GP on N = 300 points in 8 dimensions with three groups of unequal size (3, 1, 4 coordinates).  Cases:
asy_add_ucb at two t (different betas) with 'pdoo' and one with 'direct'; one syn_add_ucb batch of two; one BOCA
add_ucb call on a multi-fidelity GP whose domain kernel is additive.  Per case: every group's query sequence (the points
the reference's one-point objective was called at, in order, and its values), the returned point, and the smallest gap
between two distinct objective values of the case (`margin`: the search compares values, bounds built from them and
their differences; a case is kept only when margin >= 1e-9, so that device rounding cannot reorder it).
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
sys.path.insert(0, HERE)

import dragonfly  # noqa: E402
from dragonfly.gp.kernel import SEKernel, MaternKernel, AdditiveKernel  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.gp.euclidean_gp import EuclideanMFGP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa
from fake_mf_caller import FakeMFCaller  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__

GROUPS = [[0, 1, 2], [3], [4, 5, 6, 7]]
BOCA_GROUPS = [[0, 1], [2, 3]]


def anc(method, max_evals, t, d):
  dom = EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq='add_ucb', max_evals=max_evals, t=t, domain=dom, curr_max_val=0.0,
                   eval_points_in_progress=[], acq_opt_method=method, handle_parallel='halluc', mf_strategy=None,
                   is_mf=False, domain_bounds=np.array(dom.bounds))


class Recorder(object):
  """ Wraps the reference's maximise_acquisition: each call is one group's search; logs its objective calls. """

  def __init__(self):
    self.orig = ref_acq.maximise_acquisition
    self.calls = []

  def __call__(self, acq_fn, anc_data, *args, **kwargs):
    pts, vals = [], []

    def logged(x):
      v = acq_fn(x)
      pts.append(np.array(x, dtype=np.float64).ravel())
      vals.append(float(np.asarray(v).ravel()[0]))
      return v
    pt = self.orig(logged, anc_data, *args, **kwargs)
    self.calls.append((np.array(pts), np.array(vals), np.asarray(pt, dtype=np.float64)))
    return pt


def margin(values):
  u = np.unique(np.concatenate(values))
  return float(np.diff(u).min()) if len(u) > 1 else np.inf


def main():
  rec = Recorder()
  ref_acq.maximise_acquisition = rec
  out = {}
  rs = np.random.RandomState(7)
  n, d = 300, 8
  X = rs.random_sample((n, d))
  Y = np.sin(3 * X).sum(axis=1) + 0.3 * np.cos(5 * X[:, 0] * X[:, 4]) + 0.05 * rs.standard_normal(n)
  scale, noise, m0 = float(Y.var()) / 3, 0.01 * float(Y.var()), float(np.median(Y))
  kern = AdditiveKernel(scale, [MaternKernel(3, 2.5, 1.0, [0.4, 0.5, 0.6]), SEKernel(1, 1.0, [0.3]),
                                MaternKernel(4, 1.5, 1.0, [0.5, 0.45, 0.55, 0.6])], GROUPS)
  gp = GP(X, Y, kern, lambda x: np.array([m0] * len(x)), noise)
  out.update(X=X, Y=Y, scale=scale, noise_var=noise, mean_const=m0)
  cases = [('pdoo_t5', 'pdoo', 600, 5), ('pdoo_t300', 'pdoo', 600, 300), ('direct_t100', 'direct', 450, 100)]
  for name, method, evals, t in cases:
    rec.calls = []
    pt = ref_acq.asy.add_ucb(gp, anc(method, evals, t, d))
    assert len(rec.calls) == len(GROUPS)
    for j, (qp, qv, _) in enumerate(rec.calls):
      out['%s_qpts_%d' % (name, j)], out['%s_qvals_%d' % (name, j)] = qp, qv
    out[name + '_point'] = np.asarray(pt, dtype=np.float64)
    out[name + '_margin'] = margin([c[1] for c in rec.calls])
    out[name + '_args'] = np.array([evals, t])
    print(name, pt, out[name + '_margin'], [len(c[1]) for c in rec.calls])
  # one synchronous batch of two (Add-UCB does not read the evaluations in progress)
  rec.calls = []
  pts = ref_acq.syn.add_ucb(2, gp, anc('pdoo', 450, 40, d))
  out['syn_points'] = np.array(pts)
  out['syn_margin'] = margin([c[1] for c in rec.calls])
  print('syn', out['syn_points'], out['syn_margin'])
  # BOCA's add_ucb on a multi-fidelity GP with an additive domain kernel
  rs = np.random.RandomState(0)
  nm, dx = 150, 4
  Z = rs.random_sample((nm, 1)); Xd = rs.random_sample((nm, dx))
  Ymf = np.sin(3 * Xd).sum(axis=1) * (0.7 + 0.3 * Z[:, 0])
  kF = SEKernel(1, 1.0, [0.7])
  kDa = AdditiveKernel(1.0, [MaternKernel(2, 2.5, 1.0, [0.4, 0.5]), SEKernel(2, 1.0, [0.3, 0.6])], BOCA_GROUPS)
  mscale, mnoise, mm0 = float(Ymf.var()) / 2, 0.01 * float(Ymf.var()), float(np.median(Ymf))
  mfgp = EuclideanMFGP(list(Z), list(Xd), list(Ymf), None, mscale, kF, kDa, lambda x: np.array([mm0] * len(x)),
                       mnoise)
  a = anc('pdoo', 600, nm, dx)
  a.is_mf, a.eval_fidel_points_in_progress = True, []
  a.boca_thresh_coeff, a.y_range, a.boca_max_low_fidel_cost_ratio = 1e-4, float(np.ptp(Ymf)), 0.9
  rec.calls = []
  fid, pt = ref_acq.boca(None, mfgp, a, FakeMFCaller([1.0]))
  for j, (qp, qv, _) in enumerate(rec.calls):
    out['boca_qpts_%d' % j], out['boca_qvals_%d' % j] = qp, qv
  out.update(boca_Z=Z, boca_Xd=Xd, boca_Y=Ymf, boca_scale=mscale, boca_noise_var=mnoise, boca_mean_const=mm0,
             boca_point=np.asarray(pt, dtype=np.float64), boca_fidel=np.asarray(fid, dtype=np.float64),
             boca_margin=margin([c[1] for c in rec.calls]))
  print('boca', pt, fid, out['boca_margin'])
  for k in [k for k in out if k.endswith('margin')]:
    assert out[k] >= 1e-9, (k, out[k])
  np.savez_compressed(os.path.join(HERE, 'add_ucb_pdoo.npz'), **out)


if __name__ == '__main__':
  main()
