"""
The non-stationary kernels (Poly, ExpDecay) in the fused acquisition arg-max (dfb_score_argmax).  Both run on the
descriptor interpreter (kstar_kernel) and the fp64 DMMA contraction.  Configurations, alternated step by step within the
call:
  A  ExpDecay x SE   multi-fidelity product on [z || x] rows, 1 + 8 dims, N = 4000, 10^6 candidates on the
                     fidel_to_opt slice (z = 1), UCB  (the shape of a BOCA step)
  B  SE x SE         the same with an SE fidelity kernel: the stationary comparison on the same interpreter route
  C  Poly            order 2, d = 6, N = 5000, 10^6 device candidates, EI
Prints one JSON line: per configuration ms per step, candidates/s, the device time of profile classes 0 (K_* stage) and
1 (contraction) from a separate profiled step, and whether the int8 screen ran; plus the card's name and power limit read
in the same run.

  python tools/bench_nonstat.py [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
  ap.add_argument('--steps', type=int, default=5)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--m', type=int, default=1000000)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import kernel, device, _lib
  from oracle import gp_oracle as O
  _lib.load()
  gen = torch.Generator('cuda:0').manual_seed(1)
  # A / B: [z || x] training rows, candidates on the z = 1 slice
  rs = np.random.RandomState(0)
  n_mf, dx = 4000, 8
  Xmf = rs.random_sample((n_mf, 1 + dx))
  Ymf = np.sin(3 * Xmf[:, 1]) * (0.5 + 0.5 * Xmf[:, 0]) + (Xmf[:, 2:] ** 2).sum(axis=1) / dx + \
      0.05 * rs.standard_normal(n_mf)
  Cmf = torch.rand((args.m, 1 + dx), dtype=torch.float64, device='cuda:0', generator=gen)
  Cmf[:, 0] = 1.0
  coords = [[0], list(range(1, 1 + dx))]
  k_dom = lambda: kernel.SEKernel(dx, 1.0, [0.5] * dx)
  k_a = kernel.CoordinateProductKernel(1 + dx, 1.0, [kernel.ExpDecayKernel(1, 1.0, 0.05, [1.5]), k_dom()], coords)
  k_b = kernel.CoordinateProductKernel(1 + dx, 1.0, [kernel.SEKernel(1, 1.0, [0.7]), k_dom()], coords)
  ucb = device.make_acq_desc('ucb', beta=float(O.ucb_beta_th(dx, n_mf)))
  # C: Poly order 2 on 6 dims
  n_p, dp = 5000, 6
  Xp = rs.random_sample((n_p, dp))
  Yp = Xp[:, 0] * Xp[:, 1] - Xp[:, 2] ** 2 + 0.3 * Xp[:, 5] + 0.05 * rs.standard_normal(n_p)
  Cp = torch.rand((args.m, dp), dtype=torch.float64, device='cuda:0', generator=gen)
  k_c = kernel.PolyKernel(dp, 2, 0.5, [0.9, 1.1, 0.8, 1.2, 1.0, 0.7])
  configs = [('A_expdecay_x_se', k_a, Xmf, Ymf, Cmf, ucb),
             ('B_se_x_se', k_b, Xmf, Ymf, Cmf, ucb),
             ('C_poly2', k_c, Xp, Yp, Cp, None)]
  posts = {}
  for name, k, X, Y, C, acq in configs:
    yc = Y - Y.mean()
    post = device.DevicePosterior(len(X) + 8)
    post.set_kernel(kernel.build_descriptor(k))
    post.set_train(X, yc)
    assert post.build(0.01)[0] == 0
    posts[name] = (post, C, acq if acq is not None else device.make_acq_desc('ei', best=float(yc.max())))
  times = {name: [] for name, *_ in configs}
  result = {}
  for step in range(args.warmup + args.steps):
    for name, *_ in configs:                        # alternate the configurations step by step
      post, C, acq = posts[name]
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      _, idx, _ = post.score_argmax(acq, C)         # returns host scalars: the call ends in a synchronise
      t1 = time.perf_counter()
      if step >= args.warmup:
        times[name].append((t1 - t0) * 1e3)
      result.setdefault(name, {})['argmax'] = int(idx)
  for name, *_ in configs:                          # one profiled step per configuration, apart from the timed ones
    post, C, acq = posts[name]
    post.profile_enable(True)
    post.score_argmax(acq, C)
    prof = {c: post.profile_read(c) for c in (0, 1)}
    post.profile_enable(False)
    ms = float(np.median(times[name]))
    result[name].update(ms_per_step=round(ms, 3), cand_per_s=round(args.m / (ms * 1e-3), 1),
                        kstar_ms=round(prof[0][0], 3), contraction_ms=round(prof[1][0], 3),
                        used_i8=int(post.query('last_used_i8')), survivors=int(post.query('last_survivors')))
  name, plimit = _card()
  print(json.dumps(dict(bench='nonstat', m=args.m, steps=args.steps, card=name, power_limit=plimit, configs=result)))


if __name__ == '__main__':
  main()
