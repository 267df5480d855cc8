"""
Golden vectors for Thompson sampling on a mixed Cartesian-product domain, from the UNMODIFIED reference: the CPGP and
domain of hamming.npz ([Euclidean(2), Integral(1), ProdDiscrete(3 dims), ProdDiscreteNumeric(1)] under SE / Matern /
Hamming / Matern factors), seeded asy_ts with acq_opt_method 'ga' (which asy_ts turns into 'rand' with 4x max_evals)
and 'rand', with and without hallucinations, and one syn_ts batch of three workers.  For each recommendation: the
point (JSON, as in hamming.npz), the index of the winning candidate, the gap between the best and the second-best
sampled value, and the MT19937 state afterwards.  Seeds are kept only when every gap is at least 1e-6, so that the
1e-8 variance contract of the device cannot flip a selection.

The values are read by wrapping exd_utils._rand_maximise_vectorised_objective_in_cp_domain: the wrapper calls the
reference's own function with return_history=True and returns what it returns without it.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF:tests/golden python tests/golden/make_golden_cp_ts.py
"""
import json
import os
from argparse import Namespace

import numpy as np
import dragonfly
from dragonfly.gp.cartesian_product_gp import CPGP
from dragonfly.exd import exd_utils
from dragonfly.exd.cp_domain_utils import sample_from_cp_domain
from dragonfly.opt import gpb_acquisitions as ref_acq

from make_golden_hamming import jpoint, make_domain, make_kernel, objective, SCALE, NOISE_VAR, LEVELS, NUMERIC_LEVELS

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

MIN_GAP = 1e-6
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


def main():
  dom = make_domain()
  np.random.seed(7)                                    # the problem of hamming.npz
  X = sample_from_cp_domain(dom, 160)
  sample_from_cp_domain(dom, 300)
  H = sample_from_cp_domain(dom, 3)
  Y = np.array([objective(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  mean_const = float(np.median(Y))
  gp = CPGP(X, list(Y), make_kernel(), lambda x: np.array([mean_const] * len(x)), NOISE_VAR)
  out = dict(X=np.array(json.dumps([jpoint(x) for x in X])), H=np.array(json.dumps([jpoint(x) for x in H])), Y=Y,
             meta=np.array([SCALE, NOISE_VAR, mean_const]), levels=np.array(json.dumps(LEVELS)),
             numeric_levels=np.array(json.dumps(NUMERIC_LEVELS)))

  def anc(method, max_evals, halluc):
    return Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=len(X), curr_max_val=float(np.max(Y)),
                     handle_parallel='halluc', eval_points_in_progress=H[:halluc], is_mf=False)

  runs = []
  cases = [('asy', 'ga', 500, 0), ('asy', 'rand', 2000, 0), ('asy', 'ga', 500, 2), ('asy', 'rand', 2000, 2),
           ('syn', 'rand', 1000, 0)]
  for k, (kind, method, max_evals, halluc) in enumerate(cases):
    seed = 300 + 10 * k
    while True:
      del _RECORD[:]
      np.random.seed(seed)
      if kind == 'asy':
        pts = [ref_acq.asy.ts(gp, anc(method, max_evals, halluc))]
      else:
        pts = ref_acq.syn.ts(3, gp, anc(method, max_evals, halluc))
      if min(r['gap'] for r in _RECORD) >= MIN_GAP:
        break
      seed += 1
    st = np.random.get_state()
    runs.append(dict(kind=kind, method=method, max_evals=max_evals, halluc=halluc, seed=seed,
                     points=[jpoint(p) for p in pts], index=[r['index'] for r in _RECORD],
                     gap=[r['gap'] for r in _RECORD], m=[r['m'] for r in _RECORD]))
    out['ts%d_state' % k] = np.asarray(st[1])
    out['ts%d_pos' % k] = np.array(st[2])
    out['ts%d_has_gauss' % k] = np.array(st[3])
    out['ts%d_cached_gauss' % k] = np.array(st[4])
  out['ts_runs'] = np.array(json.dumps(runs))
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cp_ts.npz'), **out)
  print(json.dumps([{k: v for k, v in r.items() if k != 'points'} for r in runs]))


if __name__ == '__main__':
  main()
