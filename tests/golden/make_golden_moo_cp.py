"""
Golden vectors for the multi-objective acquisitions on a mixed Cartesian-product domain, from the UNMODIFIED reference:
the domain, points and first objective of hamming.npz ([Euclidean(2), Integral(1), ProdDiscrete(3 dims),
ProdDiscreteNumeric(1)]), a second objective, and two CPGPs whose kernels differ in scale, bandwidths and Hamming weights.
  1. the per-candidate scalarised UCB scores (mo_lin_asy_ucb, mo_tch_asy_ucb) on hamming.npz's 300 candidates, read
     by capturing the acquisition closure as make_golden_moo.py does;
  2. seeded asy.lin_ucb / asy.tch_ucb with acq_opt_method 'rand', and asy.lin_ts / asy.tch_ts with 'ga' (which the
     reference turns into 'rand' with 4x max_evals) and 'rand', with 0 and 2 evaluations in progress.
For each recommendation: the point (JSON, as in hamming.npz), the index of the winning candidate, the gap between the
best and the second-best scalarised value, and the MT19937 state afterwards.  Seeds are kept only when every gap is at
least 1e-6, so that the 1e-8 variance contract of the device cannot flip a selection.

The values are read by wrapping exd_utils._rand_maximise_vectorised_objective_in_cp_domain: the wrapper calls the
reference's own function with return_history=True and returns what it returns without it.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF:tests/golden python tests/golden/make_golden_moo_cp.py
"""
import json
import os
from argparse import Namespace

import numpy as np
import dragonfly
from dragonfly.gp.kernel import SEKernel, MaternKernel, HammingKernel, CartesianProductKernel
from dragonfly.gp.cartesian_product_gp import CPGP
from dragonfly.exd import exd_utils
from dragonfly.exd.cp_domain_utils import sample_from_cp_domain
from dragonfly.opt import multiobjective_gpb_acquisitions as ref_moo

from make_golden_hamming import jpoint, make_domain, make_kernel, objective, SCALE, NOISE_VAR, LEVELS, NUMERIC_LEVELS

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

MIN_GAP = 1e-6
SCALE2, NOISE_VAR2 = 0.7, 0.01
WEIGHTS, REFS = [0.6, 0.4], [0.1, -1.0]
_RECORD = []
_original = exd_utils._rand_maximise_vectorised_objective_in_cp_domain


def _recording(obj, domain, max_evals, return_history=False):
  max_val, max_pt, history = _original(obj, domain, max_evals, return_history=True)
  vals = np.array([float(np.asarray(v).ravel()[0]) for v in history.query_vals])
  idx = int(np.argmax(vals))
  rest = np.delete(vals, idx)
  _RECORD.append(dict(index=idx, gap=float(vals[idx] - rest.max()), m=len(vals)))
  if return_history:
    return max_val, max_pt, history
  return max_val, max_pt


exd_utils._rand_maximise_vectorised_objective_in_cp_domain = _recording


def make_kernel2():
  return CartesianProductKernel(SCALE2, [SEKernel(2, 1.0, [0.7, 0.5]), MaternKernel(1, 2.5, 1.0, [1.8]),
                                         HammingKernel([0.3, 0.4, 0.3]), MaternKernel(1, 1.5, 1.0, [0.8])])


def objective2(pt):
  e, i, c, n = pt
  return (np.cos(2 * e[1]) - 0.5 * (e[0] - 0.3) ** 2 + 0.05 * i[0] + (0.3 if c[1] == 'x' else -0.2) +
          (0.2 if c[0] in ('a', 'c') else 0.0) - 0.1 * n[0])


def main():
  dom = make_domain()
  np.random.seed(7)                                    # the problem of hamming.npz
  X = sample_from_cp_domain(dom, 160)
  C = sample_from_cp_domain(dom, 300)
  H = sample_from_cp_domain(dom, 3)
  Y = np.array([objective(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  Y2 = np.array([objective2(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  mean_const, mean_const2 = float(np.median(Y)), float(np.median(Y2))
  gps = [CPGP(X, list(Y), make_kernel(), lambda x: np.array([mean_const] * len(x)), NOISE_VAR),
         CPGP(X, list(Y2), make_kernel2(), lambda x: np.array([mean_const2] * len(x)), NOISE_VAR2)]
  out = dict(X=np.array(json.dumps([jpoint(x) for x in X])), C=np.array(json.dumps([jpoint(x) for x in C])),
             H=np.array(json.dumps([jpoint(x) for x in H])), Y=Y, Y2=Y2,
             meta=np.array([SCALE, NOISE_VAR, mean_const]), meta2=np.array([SCALE2, NOISE_VAR2, mean_const2]),
             levels=np.array(json.dumps(LEVELS)), numeric_levels=np.array(json.dumps(NUMERIC_LEVELS)),
             weights=np.array(WEIGHTS), refs=np.array(REFS), t=np.array(len(X)),
             beta=np.array(ref_moo._get_ucb_beta_th(dom.dim, len(X))))

  def anc(method, max_evals, halluc):
    return Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=len(X), handle_parallel='halluc',
                     eval_points_in_progress=H[:halluc], is_mf=False, obj_weights=WEIGHTS, reference_point=REFS)

  # 1. per-candidate scores: the acquisition closures, captured by replacing the maximiser in the module
  real_max = ref_moo.maximise_acquisition
  ref_moo.maximise_acquisition = lambda acq, anc_data, *a, **kw: acq
  try:
    out['lin_ucb_scores'] = ref_moo.mo_lin_asy_ucb(gps, anc('rand', 10, 0))(C)
    out['tch_ucb_scores'] = ref_moo.mo_tch_asy_ucb(gps, anc('rand', 10, 0))(C)
  finally:
    ref_moo.maximise_acquisition = real_max
  # 2. end to end
  runs = []
  cases = [('lin_ucb', 'rand', 2000, 0), ('tch_ucb', 'rand', 2000, 0),
           ('lin_ts', 'ga', 500, 0), ('lin_ts', 'rand', 2000, 0), ('lin_ts', 'ga', 500, 2), ('lin_ts', 'rand', 2000, 2),
           ('tch_ts', 'ga', 500, 0), ('tch_ts', 'rand', 2000, 0), ('tch_ts', 'ga', 500, 2), ('tch_ts', 'rand', 2000, 2)]
  for k, (name, method, max_evals, halluc) in enumerate(cases):
    seed = 500 + 10 * k
    while True:
      del _RECORD[:]
      np.random.seed(seed)
      pt = getattr(ref_moo.asy, name)(gps, anc(method, max_evals, halluc))
      if min(r['gap'] for r in _RECORD) >= MIN_GAP:
        break
      seed += 1
    st = np.random.get_state()
    runs.append(dict(name=name, method=method, max_evals=max_evals, halluc=halluc, seed=seed, point=jpoint(pt),
                     index=_RECORD[0]['index'], gap=_RECORD[0]['gap'], m=_RECORD[0]['m']))
    out['run%d_state' % k] = np.asarray(st[1])
    out['run%d_pos' % k] = np.array(st[2])
    out['run%d_has_gauss' % k] = np.array(st[3])
    out['run%d_cached_gauss' % k] = np.array(st[4])
  out['runs'] = np.array(json.dumps(runs))
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'moo_cp.npz'), **out)
  print(json.dumps([{k: v for k, v in r.items() if k != 'point'} for r in runs]))


if __name__ == '__main__':
  main()
