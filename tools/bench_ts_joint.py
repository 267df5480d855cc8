"""
One Thompson draw over M candidates (what asy_ts does with its candidates), Matern-2.5, d = 6, three ways:
  joint   the joint device draw (gp.draw_samples(1, C): covariance, factor-only factorisation, L U) for M > 4096;
  blocks  the former independent 4096-candidate blocks, driven directly through post.ts_draws per block;
  oracle  the NumPy oracle's joint draw on the host (M = 8000 only).
The device arms run alternately, median of --reps after one warm-up each (host wall clock around synchronised calls,
profiling off).  Then, in a separate pass with the handle's CUDA-event profiling on (include/dfb200.h:
DFB_PROF_TS_COV / _FACTOR / _PRODUCT), --reps joint draws give the median time of the covariance, the factor-only
factorisation and the L U product, and the factorisation's fp64 rate (Mpad^3 / 3 multiply-adds, 2 flops each).
Prints one JSON line per (N, M) with the card name, power limit and host core count.

    python tools/bench_ts_joint.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dragonfly_b200 import gp_core, kernel  # noqa: E402
from oracle import gp_oracle as O  # noqa: E402


STAGES = dict(cov=11, factor=12, product=13)          # DFB_PROF_TS_COV, _FACTOR, _PRODUCT


def card():
  try:
    out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
    return out.strip().splitlines()[0]
  except Exception:  # pylint: disable=broad-except
    return 'unknown'


def timed(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'this benchmark needs a GPU'
  info = dict(card=card(), host_cores=os.cpu_count())
  for n in (2000, 5000):
    rs = np.random.RandomState(n)
    X = rs.random_sample((n, 6))
    Y = np.sin(3 * X).sum(axis=1)
    gp = gp_core.GP(X, Y, kernel.MaternKernel(6, 2.5, 1.3, [0.4] * 6), gp_core.ConstantMean(0.1), 1e-3 * 1.3)
    post = gp._post
    for M in (4096, 8000, 16384):
      C = rs.random_sample((M, 6))
      U = rs.standard_normal((1, M))
      blk = post.TS_BLOCK

      def joint():
        gp.draw_samples(1, C)

      def blocks():
        for lo in range(0, M, blk):
          post.ts_draws(C[lo:lo + blk], np.ascontiguousarray(U[:, lo:lo + blk]), mean_const=0.1)
      arms = [('joint', joint), ('blocks', blocks)]
      for _, fn in arms:
        fn()                                                 # warm-up (and the joint workspace)
      times = dict((name, []) for name, _ in arms)
      for _ in range(args.reps):
        for name, fn in arms:
          times[name].append(timed(fn))
      row = dict(info, n=n, m=M, chunk=int(post.query('chunk')),
                 **dict(('%s_s' % k, float(np.median(v))) for k, v in times.items()))
      if M > blk:
        stages = dict((name, []) for name in STAGES)
        post.profile_enable(True)
        for name, cls in STAGES.items():
          post.profile_read(cls)                           # start from zero
        for _ in range(args.reps):
          joint()
          for name, cls in STAGES.items():
            ms, _, _ = post.profile_read(cls)
            stages[name].append(ms)
        post.profile_enable(False)
        for name, v in stages.items():
          row['stage_%s_ms' % name] = float(np.median(v))
        mp = -(-M // 128) * 128
        row['factor_tflops'] = 2.0 * mp ** 3 / 3.0 / (row['stage_factor_ms'] * 1e-3) / 1e12
      if M == 8000 and n == 2000:
        ogp = O.OGP(X, Y, O.OMaternKernel(6, 2.5, 1.3, [0.4] * 6), lambda x: np.array([0.1] * len(x)), 1e-3 * 1.3)
        t0 = time.perf_counter()
        ogp.draw_samples_with_normals(C, U.T)
        row['oracle_host_s'] = time.perf_counter() - t0
      print(json.dumps(row), flush=True)


if __name__ == '__main__':
  main()
