"""
ESP kernel vs the plain Matern-2.5 kernel in the fused acquisition arg-max (dfb_score_argmax): N = 5000 training
points, d = 8, 10^6 device candidates, EI.  Configurations, alternated step by step within the call: ESP-SE at orders
2, 4 and 8, and plain Matern-2.5 with option prune 0 and 1.  Prints one JSON line: per configuration ms per step,
candidates/s, the device time of profile classes 0 (K_* stage) and 1 (contraction) per step from a separate profiled
step, and whether the int8 screen ran; plus the card's name and power limit read in the same run.

  python tools/bench_esp.py [--steps 5] [--warmup 2]
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
  ap.add_argument('--n', type=int, default=5000)
  ap.add_argument('--m', type=int, default=1000000)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import kernel, device, _lib
  _lib.load()
  d = 8
  rs = np.random.RandomState(0)
  X = rs.random_sample((args.n, d))
  Y = np.sin(3 * X[:, 0]) + (X ** 2).sum(axis=1) / d + 0.05 * rs.standard_normal(args.n)
  yc = Y - Y.mean()
  Cn = torch.rand((args.m, d), dtype=torch.float64, device='cuda:0', generator=torch.Generator('cuda:0').manual_seed(1))
  acq = device.make_acq_desc('ei', best=float(yc.max()))
  configs = [('esp_se_order%d' % r, kernel.ESPKernelSE(d, 0.2, r, [0.5] * d), 1) for r in (2, 4, 8)] + \
            [('matern25_prune%d' % p, kernel.MaternKernel(d, 2.5, 1.0, [0.5] * d), p) for p in (0, 1)]
  posts = {}
  for name, k, prune in configs:
    post = device.DevicePosterior(args.n + 8)
    post.set_option('prune', prune)
    post.set_kernel(kernel.build_descriptor(k))
    post.set_train(X, yc)
    assert post.build(0.01)[0] == 0
    posts[name] = post
  times = {name: [] for name, _, _ in configs}
  result = {}
  for step in range(args.warmup + args.steps):
    for name, _, _ in configs:                      # alternate the configurations step by step
      post = posts[name]
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      _, idx, _ = post.score_argmax(acq, Cn)        # returns host scalars: the call ends in a synchronise
      t1 = time.perf_counter()
      if step >= args.warmup:
        times[name].append((t1 - t0) * 1e3)
      result.setdefault(name, {})['argmax'] = int(idx)
  for name, _, _ in configs:                        # one profiled step per configuration, apart from the timed ones
    post = posts[name]
    post.profile_enable(True)
    post.score_argmax(acq, Cn)
    prof = {c: post.profile_read(c) for c in (0, 1)}
    post.profile_enable(False)
    ms = float(np.median(times[name]))
    result[name].update(ms_per_step=round(ms, 3), cand_per_s=round(args.m / (ms * 1e-3), 1),
                        kstar_ms=round(prof[0][0], 3), contraction_ms=round(prof[1][0], 3),
                        used_i8=int(post.query('last_used_i8')), survivors=int(post.query('last_survivors')))
  name, plimit = _card()
  print(json.dumps(dict(bench='esp', n=args.n, m=args.m, d=d, acq='ei', steps=args.steps, card=name,
                        power_limit=plimit, configs=result)))


if __name__ == '__main__':
  main()
