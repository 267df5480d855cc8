"""
Acquisitions on a constrained Cartesian-product domain: the domain of golden cp_constrained.npz (float dim 2 + float,
int, discrete strings, discrete numeric) with its compiled constraints (a norm, string equality, a builtin sum with
np.sqrt, int arithmetic; --with-callable adds the fixture's callable, which every accepted row then takes to the host),
a CPGP at N = 2000, asy_ei with the `rand` maximiser at 1.2 x 10^5 and 10^6 candidates, arms alternated:
  parity  candidate_rng 'numpy': the reference's constrained draw, filtered and compacted on the device
  device  candidate_rng 'device': the first M accepted rows of the device's candidate stream
  host    the reference's per-point check (domain.constraints_are_satisfied) timed on a sample, extrapolated to the
          rows the parity draw filtered
Prints one JSON line: median wall time per call of each arm, acceptance rate, undecided rows per 10^6, the share of
the status + compaction kernels in a device-mode call (CUDA events around both on a block of the call's size), and
the card's name and power limit read in the same run.

  python tools/bench_cp_constrained.py [--steps 3] [--warmup 1] [--with-callable]
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_mixed import _card  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--warmup', type=int, default=1)
  ap.add_argument('--n', type=int, default=2000)
  ap.add_argument('--with-callable', action='store_true')
  args = ap.parse_args()
  import torch
  import cp_constrained_ref as F
  import constraint_ref as CR
  from dragonfly_b200 import cartesian_product_gp as cp, gpb_acquisitions as acq, constraints, _lib
  _lib.load()
  cons = F.CONSTRAINTS if args.with_callable else F.PROGRAMS['fixture']
  dom = F.make_domain(cons)
  kern = F.make_kernel(1.2)
  parts = acq._cp_parts(dom, kern)
  np.random.seed(0)
  X = [q for q in _draw_points(acq, parts, dom, args.n)]
  Y = np.array([np.sin(3 * p[0][0]) + 0.3 * p[0][1] - 0.2 * p[0][2] - 0.05 * (p[1][0] - 3) ** 2 for p in X])
  Y = Y + 0.05 * np.random.standard_normal(args.n)
  mc = float(np.median(Y))
  gp = cp.CPGP(X, list(Y), kern, lambda x: np.array([mc] * len(x)), 0.02)
  sizes = (120000, 1000000)
  arms = [(M, mode) for M in sizes for mode in ('numpy', 'device')]
  times = dict((arm, []) for arm in arms)
  for step in range(args.warmup + args.steps):
    for M in sizes:
      for mode in (('numpy', 'device') if step % 2 == 0 else ('device', 'numpy')):     # alternate the arms
        anc = Namespace(domain=dom, max_evals=M, acq_opt_method='rand', t=args.n, handle_parallel='halluc',
                        eval_points_in_progress=[], is_mf=False, candidate_rng=mode, curr_max_val=float(Y.max()))
        np.random.seed(step)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        acq.asy.ei(gp, anc)
        torch.cuda.synchronize()
        if step >= args.warmup:
          times[(M, mode)].append(time.perf_counter() - t0)
  # acceptance, undecided rows and the host's per-point check, on 10^6 parity rows
  filt = constraints.compile_filter(dom, parts)
  np.random.seed(1)
  rows, draws = acq.draw_cp_candidates(parts, 1000000)
  st = CR.status(filt, rows)
  t0 = time.perf_counter()
  acc = sum(dom.constraints_are_satisfied(acq.point_from_draws(parts, draws, i)) for i in range(3000))
  host_us = 1e6 * (time.perf_counter() - t0) / 3000
  # status + compaction kernels on one block of 10^6 rows, CUDA events
  post = gp._device_posterior()
  rows_d = torch.from_numpy(rows).cuda()
  prog = filt.desc()
  for _ in range(2):
    s, _ = post.constraint_status(prog, rows_d)
    post.compact_rows(rows_d, s)
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(5):
    s, _ = post.constraint_status(prog, rows_d)
    post.compact_rows(rows_d, s)
  e1.record()
  torch.cuda.synchronize()
  filter_ms = e0.elapsed_time(e1) / 5
  med = lambda v: float(np.median(v))
  out = dict(metric='asy_ei on a constrained CP domain, N = %d' % args.n, card=_card(),
             constraints=[c if isinstance(c, str) else c.__name__ for c in cons],
             acceptance=float(np.mean(st != constraints.REJECT)), undecided_per_1e6=int(np.sum(st == 2)),
             host_check_us_per_point=host_us, host_accept_rate_sample=acc / 3000.0,
             filter_ms_per_1e6_rows=filter_ms)
  for M in sizes:
    for mode in ('numpy', 'device'):
      out['%s_%d_s' % ('parity' if mode == 'numpy' else 'device', M)] = med(times[(M, mode)])
    # the reference's draw checks about M / acceptance rows, one by one
    out['host_check_only_%d_s_extrapolated' % M] = host_us * 1e-6 * M / max(out['acceptance'], 1e-9)
    out['filter_share_of_device_call_%d' % M] = (filter_ms * 1e-3 * M / 1e6 / max(out['acceptance'], 1e-9)) / \
        out['device_%d_s' % M]
  print(json.dumps(out))


def _draw_points(acq, parts, dom, n):
  pts = []
  while len(pts) < n:
    rows, draws = acq.draw_cp_candidates(parts, 4 * n)
    for i in range(len(rows)):
      pt = acq.point_from_draws(parts, draws, i)
      if dom.constraints_are_satisfied(pt):
        pts.append(pt)
        if len(pts) == n:
          break
  return pts


if __name__ == '__main__':
  main()
