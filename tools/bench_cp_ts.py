"""
Thompson sampling on a mixed Cartesian-product domain: the domain, kernel and CPGP of tools/bench_mixed.py
([Euclidean(2), Integral(1), ProdDiscrete(3 dims, 2-5 levels), ProdDiscreteNumeric(1)] under SE x Matern x Hamming x
Matern, N = 2000), asy_ts at 1.2 x 10^5 and 10^6 candidates in both candidate modes, arms alternated:
  parity  candidate_rng 'numpy': the reference's candidates and np.random.normal(size=M) on the host, scored in fused
          device slabs (dfb_score_argmax_ts)
  device  candidate_rng 'device': rows from dfb_fill_mixed_candidates, normals made in the scoring kernel
and a host arm that samples the reference's way -- one 1 x 1 oracle draw_samples per point (exd_utils.py:247-274) -- on
a few hundred points, reported as a rate.  Prints one JSON line with the median wall time per call and candidates/s of
each arm, the card's name and its power limit read in the same run.

  python tools/bench_cp_ts.py [--steps 3] [--warmup 1] [--host-m 300]
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_mixed import _card  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--warmup', type=int, default=1)
  ap.add_argument('--n', type=int, default=2000)
  ap.add_argument('--host-m', type=int, default=300)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import kernel, cartesian_product_gp as cp, gpb_acquisitions as acq, domains, _lib
  from oracle import gp_oracle as O
  import hamming_ref as R
  _lib.load()
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = R.make_domain(domains, levels, numeric_levels)
  kern = R.make_kernel(kernel, cp, 1.3)
  parts = acq._cp_parts(dom, kern)
  np.random.seed(0)
  Xr, draws = acq.draw_cp_candidates(parts, args.n)
  X = [acq.point_from_draws(parts, draws, i) for i in range(args.n)]
  Y = np.sin(3 * Xr[:, 0]) + 0.3 * Xr[:, 1] - 0.1 * (Xr[:, 2] - 3) ** 2 + 0.4 * (Xr[:, 3] == 1) + \
      0.2 * np.log(Xr[:, 6]) + 0.05 * np.random.standard_normal(args.n)
  mc = float(np.median(Y))
  gp = cp.CPGP(X, list(Y), kern, lambda x: np.array([mc] * len(x)), 0.02)
  arms = [(M, mode) for M in (120000, 1000000) for mode in ('numpy', 'device')]
  times = dict((arm, []) for arm in arms)
  for step in range(args.warmup + args.steps):
    for M in (120000, 1000000):
      for mode in (('numpy', 'device') if step % 2 == 0 else ('device', 'numpy')):     # alternate the arms
        anc = Namespace(domain=dom, max_evals=M, acq_opt_method='rand', t=args.n, handle_parallel='halluc',
                        eval_points_in_progress=[], is_mf=False, candidate_rng=mode)
        np.random.seed(step)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        acq.asy.ts(gp, anc)
        t1 = time.perf_counter()
        if step >= args.warmup:
          times[(M, mode)].append(t1 - t0)
  result = {}
  for (M, mode), ts in times.items():
    s = float(np.median(ts))
    result['%s_%d' % ('parity' if mode == 'numpy' else 'device', M)] = dict(s_per_call=round(s, 4),
                                                                           cand_per_s=round(M / s, 1))
  # host arm: the reference's one-point draw_samples (a 1 x 1 covariance, its Cholesky factor, one normal) per point
  codes = {}
  ogp = O.OGP(R.encode_points(X, codes), Y, R.oracle_kernel(1.3), lambda x: np.array([mc] * len(x)), 0.02)
  np.random.seed(1)
  _, hdraws = acq.draw_cp_candidates(parts, args.host_m)
  pts = [acq.point_from_draws(parts, hdraws, i) for i in range(args.host_m)]
  t0 = time.perf_counter()
  vals = []
  for p in pts:
    mu, cov = ogp.eval(R.encode_points([p], codes), 'covar')
    L, _ = O.stable_cholesky(cov)
    vals.append((L.dot(np.random.normal(size=(1, 1))).T + mu).ravel()[0])
  int(np.argmax(vals))
  s = time.perf_counter() - t0
  result['host_one_point_%d' % args.host_m] = dict(s_per_call=round(s, 4), cand_per_s=round(args.host_m / s, 1))
  name, plimit = _card()
  print(json.dumps(dict(bench='cp_ts', n=args.n, steps=args.steps, card=name, power_limit=plimit, arms=result)))


if __name__ == '__main__':
  main()
