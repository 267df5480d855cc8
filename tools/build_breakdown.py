"""Where the time of dfb_build_posterior goes: Matern-5/2 at d = 6, N = 1000, 2000 and 5000, full and LML-only builds.

Per build, from CUDA events on the stream each stage runs on (profiling classes DFB_PROF_BUILD_* of include/dfb200.h):
K(X, X) + init_tall, the chol_diag chain, panel + next (the critical stream), rest (the bulk stream), the tail (W,
alpha, LML sums) and the scoring state (the int8 digit planes of W at N >= 1024, the fp64 TMA maps).  With the
look-ahead schedule the stages overlap, so they do not add up to the build; 'build' is the whole dfb_build_posterior
interval and 'wall' the host time of a synchronised build with profiling off (median of 10).

At N = 5000 (full build) a separate torch.profiler run gives the panel and trailing kernels' busy time (the union of
their kernel intervals; they run on two streams at once), from which the rates below are computed: the tiles' DMMA
flops (2 * 128^3 per 128 x 128 tile) and the trailing tiles' C read + D write (2 * 128 KB per tile, HBM: the tall
matrix does not fit in L2), against the live cuBLAS DGEMM and DMMA issue peaks bench.py measures.

Usage:
  python tools/build_breakdown.py                      # the library DFB200_LIB names (default: the in-tree build)
  python tools/build_breakdown.py --libs A.so B.so     # each library in its own process, alternated, --rounds times
Prints the card name and power limit, one JSON line per run and the tables (medians over rounds)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGES = (('kxx', 5), ('chol', 6), ('panel_next', 7), ('rest', 8), ('tail', 9), ('scoring_state', 10), ('build', 3))
FACTOR_KERNELS = ('factor_update_kernel', 'gemm_tn_kernel')     # the panel / trailing kernels, new and old
SIZES = (1000, 2000, 5000)


def card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = 'unknown'
  return '%s, power limit / max SM clock: %s' % (name, q)


def factor_work(n, with_bottom=True):
  """ (128 x 128 tiles of the panel solves and trailing updates, trailing tiles) of one factorisation. """
  nb = (n + 127) // 128
  panel = trail = 0
  for step in range(nb):
    full = (step + 1 if with_bottom else 0) + 1
    panel += (nb - step - 1) + full
    trail += full * (nb - step - 1) + sum(nb - j for j in range(step + 1, nb))
  return panel + trail, trail


def busy_ms(post, noise, flags):
  """ Union of the panel / trailing kernel intervals of one build (torch.profiler). """
  import torch
  from torch.profiler import profile, ProfilerActivity
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    post.build(noise, 0.0, flags)
    torch.cuda.synchronize()
  iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
              if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in FACTOR_KERNELS))
  total, cur = 0.0, None
  for a, b in iv:
    if cur is None or a > cur[1]:
      if cur is not None:
        total += cur[1] - cur[0]
      cur = [a, b]
    else:
      cur[1] = max(cur[1], b)
  if cur is not None:
    total += cur[1] - cur[0]
  return total * 1e-3, len(iv)       # us -> ms


def measure():
  sys.path.insert(0, ROOT)
  import numpy as np
  import time
  import torch
  from dragonfly_b200 import synth_data, kernel, device, _lib
  out = {'lib': _lib.LIB_PATH, 'card': card()}
  for n in SIZES:
    w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=n, n_cand=16)
    k = w['kernel']
    post = device.DevicePosterior(n)
    post.set_kernel(kernel.build_descriptor(kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])))
    post.set_train(w['X'], w['Y'] - w['mean_const'])
    for name, flags in (('full', _lib.DFB_BUILD_FULL), ('lml_only', _lib.DFB_BUILD_LML_ONLY)):
      for _ in range(3):
        assert post.build(w['noise_var'], 0.0, flags)[0] == 0
      torch.cuda.synchronize()
      ts = []
      for _ in range(10):
        t0 = time.perf_counter()
        post.build(w['noise_var'], 0.0, flags)
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
      post.profile_enable(True)
      for _, cls in STAGES:
        post.profile_read(cls)
      reps = 5
      for _ in range(reps):
        post.build(w['noise_var'], 0.0, flags)
      torch.cuda.synchronize()
      res = {'wall': float(np.median(ts))}
      for stage, cls in STAGES:
        ms, launches, _ = post.profile_read(cls)
        res[stage] = ms / reps
        res[stage + '_launches'] = launches // reps
      post.profile_enable(False)
      out['N%d_%s' % (n, name)] = res
      if n == 5000 and name == 'full':
        ms, launches = busy_ms(post, w['noise_var'], flags)
        tiles, trail = factor_work(n)
        out['factor_kernels_N5000_full'] = {'busy_ms': ms, 'launches': launches, 'gflop': tiles * 2 * 128 ** 3 * 1e-9,
                                            'tflops': tiles * 2 * 128 ** 3 / (ms * 1e-3) * 1e-12,
                                            'trail_hbm_gb': trail * 2 * 128 * 128 * 8 * 1e-9,
                                            'trail_hbm_gbs': trail * 2 * 128 * 128 * 8 / (ms * 1e-3) * 1e-9}
    del post
  import bench
  out['peaks'] = {'cublas_dgemm_tflops': bench.measure_dgemm_peak(torch, torch.device('cuda', 0)),
                  'dmma_issue_tflops': device.measure_peak('f64')}
  return out


def table(runs):
  import numpy as np
  cols = ['kxx', 'chol', 'panel_next', 'rest', 'tail', 'scoring_state', 'build', 'wall']
  lines = ['| N | build | ' + ' | '.join(cols) + ' |', '|---|---|' + '---|' * len(cols)]
  for key in sorted(runs[0].keys()):
    if not key.startswith('N'):
      continue
    n, name = key[1:].split('_', 1)
    vals = [float(np.median([r[key][c] for r in runs])) for c in cols]
    lines.append('| %s | %s | ' % (n, name) + ' | '.join('%.3f' % v for v in vals) + ' |')
  return '\n'.join(lines)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--libs', nargs='*', default=None)
  ap.add_argument('--rounds', type=int, default=2)
  ap.add_argument('--child', action='store_true')
  a = ap.parse_args()
  if a.child or not a.libs:
    print(json.dumps(measure()), flush=True)
    return
  runs = {lib: [] for lib in a.libs}
  for _ in range(a.rounds):
    for lib in a.libs:
      env = dict(os.environ, DFB200_LIB=os.path.abspath(lib))
      r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child'], env=env, capture_output=True,
                         text=True, check=True)
      line = r.stdout.strip().splitlines()[-1]
      print(line, flush=True)
      runs[lib].append(json.loads(line))
  print('card:', runs[a.libs[0]][0]['card'])
  for lib in a.libs:
    print('\n%s (ms per build, median of %d runs)\n%s' % (lib, a.rounds, table(runs[lib])))
    for r in runs[lib]:
      print('panel + trailing kernels, N = 5000 full:', json.dumps(r['factor_kernels_N5000_full']), 'peaks:',
            json.dumps(r['peaks']))


if __name__ == '__main__':
  main()
