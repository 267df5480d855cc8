"""
The `ga` acquisition maximiser on a mixed Cartesian-product domain: bench_mixed's shape ([Euclidean(2), Integral(1),
ProdDiscrete(3 dims, 3/2/5 levels), ProdDiscreteNumeric(1)] under SE x Matern x Hamming x Matern, string categories as in
tests/golden/cp_ga.npz), a CPGP on N = 2000 points, one asy_ei call at budgets of 1 000 and 30 000 evaluations:
  parity  the reference's GA restated (dragonfly_b200/ga.py): the initial pool and every epoch of five mutations scored
          in one fused device call each
  device  candidate_rng 'device': the whole search in one dfb_ga_maximise call (ga_epoch_kernel + the small-batch
          scoring launches per epoch, one synchronisation)
  host    the same search scored the reference's way -- one oracle GP eval per point -- on a small budget, extrapolated
          per evaluation
Prints one JSON line with the median wall time per call (after warm-up), the evaluations per second, the card's name
and its power limit read in the same run.

  python tools/bench_cp_ga.py [--steps 3] [--warmup 1] [--host-budget 200]
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))

from bench_mixed import _card  # noqa: E402  (tools/ is on sys.path when run as a script)

LEVELS, NUMERIC_LEVELS = [['a', 'b', 'c'], ['w', 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--warmup', type=int, default=1)
  ap.add_argument('--n', type=int, default=2000)
  ap.add_argument('--host-budget', type=int, default=200)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import kernel, cartesian_product_gp as cp, gpb_acquisitions as acq, domains, ga, _lib
  from oracle import gp_oracle as O
  import hamming_ref as R
  _lib.load()
  dom = R.make_domain(domains, LEVELS, NUMERIC_LEVELS)
  kern = R.make_kernel(kernel, cp, 1.3)
  parts = acq._cp_parts(dom, kern)
  np.random.seed(0)
  Xr, draws = acq.draw_cp_candidates(parts, args.n)
  X = [acq.point_from_draws(parts, draws, i) for i in range(args.n)]
  Y = np.sin(3 * Xr[:, 0]) + 0.3 * Xr[:, 1] - 0.1 * (Xr[:, 2] - 3) ** 2 + 0.4 * (Xr[:, 3] == 1) + \
      0.2 * np.log(Xr[:, 6]) + 0.05 * np.random.standard_normal(args.n)
  mc = float(np.median(Y))
  gp = cp.CPGP(X, list(Y), kern, lambda x: np.array([mc] * len(x)), 0.02)
  best = float(Y.max())
  result = {}
  for B in (1000, 30000):
    times = {'numpy': [], 'device': []}
    for step in range(args.warmup + args.steps):
      for mode in ('numpy', 'device'):                  # the arms alternate
        anc = Namespace(domain=dom, max_evals=B, acq_opt_method='ga', t=args.n, curr_max_val=best,
                        handle_parallel='halluc', eval_points_in_progress=[], is_mf=False, candidate_rng=mode)
        np.random.seed(step)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        acq.asy.ei(gp, anc)
        t1 = time.perf_counter()
        if step >= args.warmup:
          times[mode].append(t1 - t0)
    for mode, arm in (('numpy', 'parity'), ('device', 'device')):
      s = float(np.median(times[mode]))
      result['%s_%d' % (arm, B)] = dict(s_per_call=round(s, 4), evals_per_s=round((B + 1) / s, 1))
  # host arm: the same search, each point scored on its own through the NumPy oracle
  codes = {}
  ogp = O.OGP(R.encode_points(X, codes), Y, R.oracle_kernel(1.3), lambda x: np.array([mc] * len(x)), 0.02)

  def one_at_a_time(pts):
    out = []
    for p in pts:
      mu, sd = ogp.eval(R.encode_points([p], codes), 'std')
      out.append(O.acq_ei(mu, sd, best)[0])
    return np.array(out)
  np.random.seed(1)
  t0 = time.perf_counter()
  ga.ga_maximise(one_at_a_time, parts, args.host_budget)
  s = (time.perf_counter() - t0) / (args.host_budget + 1)
  for B in (1000, 30000):
    result['host_extrapolated_%d' % B] = dict(s_per_call=round(s * (B + 1), 2), evals_per_s=round(1 / s, 1))
  name, plimit = _card()
  print(json.dumps(dict(bench='cp_ga', n=args.n, steps=args.steps, host_budget=args.host_budget, card=name,
                        power_limit=plimit, arms=result)))


if __name__ == '__main__':
  main()
