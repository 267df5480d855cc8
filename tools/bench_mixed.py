"""
The `rand` acquisition maximiser on a mixed Cartesian-product domain: [Euclidean(2), Integral(1), ProdDiscrete(3 dims,
2-5 levels), ProdDiscreteNumeric(1)] under SE x Matern x Hamming x Matern (the shape of tests/golden/hamming.npz), a CPGP
on N = 2000 points, asy_ei at 10^5 and 10^6 candidates in both candidate modes:
  parity  candidate_rng 'numpy': the reference's draw on the host (sample_from_cp_domain order), scored in fused device
          slabs
  device  candidate_rng 'device': dfb_fill_mixed_candidates, nothing on the host
and a host arm that scores the reference's way -- one oracle GP eval per sampled point (exd_utils.py:247-274) -- for a
small M.  Prints one JSON line with the median wall time per call and candidates/s of each arm, the card's name and its
power limit read in the same run.

  python tools/bench_mixed.py [--steps 3] [--warmup 1] [--host-m 300]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from argparse import Namespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))


def _card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = 'unknown'
  return name, out


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
  best = float(Y.max())
  result = {}
  for M in (100000, 1000000):
    for mode in ('numpy', 'device'):
      times = []
      for step in range(args.warmup + args.steps):
        anc = Namespace(domain=dom, max_evals=M, acq_opt_method='rand', t=args.n, curr_max_val=best,
                        handle_parallel='halluc', eval_points_in_progress=[], is_mf=False, candidate_rng=mode)
        np.random.seed(step)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        acq.asy.ei(gp, anc)
        t1 = time.perf_counter()
        if step >= args.warmup:
          times.append(t1 - t0)
      s = float(np.median(times))
      result['%s_%d' % ('parity' if mode == 'numpy' else 'device', M)] = dict(s_per_call=round(s, 4),
                                                                             cand_per_s=round(M / s, 1))
  # host arm: the reference's one-point-at-a-time scoring, through the NumPy oracle on code rows
  codes = {}
  ogp = O.OGP(R.encode_points(X, codes), Y, R.oracle_kernel(1.3), lambda x: np.array([mc] * len(x)), 0.02)
  np.random.seed(1)
  _, hdraws = acq.draw_cp_candidates(parts, args.host_m)
  pts = [acq.point_from_draws(parts, hdraws, i) for i in range(args.host_m)]
  t0 = time.perf_counter()
  vals = []
  for p in pts:
    mu, sd = ogp.eval(R.encode_points([p], codes), 'std')
    vals.append(O.acq_ei(mu, sd, best)[0])
  int(np.argmax(vals))
  s = time.perf_counter() - t0
  result['host_one_point_%d' % args.host_m] = dict(s_per_call=round(s, 4), cand_per_s=round(args.host_m / s, 1))
  name, plimit = _card()
  print(json.dumps(dict(bench='mixed', n=args.n, steps=args.steps, card=name, power_limit=plimit, arms=result)))


if __name__ == '__main__':
  main()
