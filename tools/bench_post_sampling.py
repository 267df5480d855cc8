"""
post_sampling on the device: what the speculative slice sampler and dfb_lml_batch buy, and where dfb_lml_batch stops
paying (hp_grid.LML_BATCH_MAX_N).  One JSON line per table on stdout; --out FILE also writes the whole result there.

  whole fit     d = 6, Matern with tuned nu, mean and noise (9 continuous hps + nu), num_samples 17 (offset 25),
                burn-in --burn (-1: the reference's default, int(sqrt(10) * 100) = 316), N in --sizes; arms, alternated
                within each repetition:  batch   the sampler with lml_batch_for_hyperparams (dfb_lml_batch below the cap)
                                         single  the sampler with lml_for_hyperparams (one LML-only build per LML)
                                         depth1  speculation depth 1 with lml_batch_for_hyperparams
                columns: ms per fit, LMLs consumed (what the reference computes) and evaluated (plus speculation),
                round trips (batches), LMLs per round trip
  kernel        dfb_lml_batch at B in {1, 8, 32, 132}, N in {64, 128, 256, 512} against B x dfb_build_posterior(
                DFB_BUILD_LML_ONLY) on one handle: CUDA events and host wall time per call, ms per LML
  host          the same sampler with the NumPy oracle's LML, one call at a time, N = 60 and 200, 2 samples, burn --host-burn:
                ms per LML

  python tools/bench_post_sampling.py [--sizes 60,200,500,1000] [--burn -1] [--reps 1] [--host-burn 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def _card():
  import torch
  name = torch.cuda.get_device_name(0)
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = 'unknown'
  return name, out


def _problem(n, d=6, seed=0):
  from dragonfly_b200 import hp_grid
  rs = np.random.RandomState(seed)
  X = rs.random_sample((n, d))
  Y = np.sin(3 * X[:, 0]) + (X ** 2).sum(axis=1) / d + 0.05 * rs.standard_normal(n)
  layout = hp_grid.EuclideanHPLayout(d, 'matern', nu=-1.0, mean_func_type='tune', noise_var_type='tune')
  bounds, dscr = layout.bounds(X, Y, tune_nu=True)
  return X, Y, layout, bounds, dscr


def _fit(X, Y, layout, bounds, dscr, burn, num_samples, lml_batch, depth):
  from dragonfly_b200 import post_sampling
  stats = post_sampling.PostSamplingStats()
  np.random.seed(1)
  t0 = time.perf_counter()
  res = post_sampling.post_sample_hps(X, Y, layout, bounds, dscr, num_samples=num_samples, offset=25, burn=burn,
                                      lml_batch=lml_batch, depth=depth, stats=stats)
  ms = 1e3 * (time.perf_counter() - t0)
  return ms, stats, res


def whole_fit(sizes, burn, reps, num_samples):
  from dragonfly_b200 import hp_grid, post_sampling
  rows = []
  for n in sizes:
    X, Y, layout, bounds, dscr = _problem(n)
    arms = [('batch', hp_grid.lml_batch_for_hyperparams, post_sampling.DEFAULT_DEPTH),
            ('single', hp_grid.lml_for_hyperparams, post_sampling.DEFAULT_DEPTH),
            ('depth1', hp_grid.lml_batch_for_hyperparams, 1)]
    results = {a[0]: [] for a in arms}
    samples = {}
    for _ in range(reps):
      for name, fn, depth in arms:
        src = post_sampling.device_lml_batch(X, Y, layout, batch_fn=fn)
        ms, st, res = _fit(X, Y, layout, bounds, dscr, burn, num_samples, src, depth)
        results[name].append((ms, st))
        samples[name] = (np.array(res[1]), np.array(res[2]))
    same = all(np.array_equal(samples[a][0], samples['batch'][0]) and np.array_equal(samples[a][1], samples['batch'][1])
               for a in samples)
    for name in results:
      ms = [r[0] for r in results[name]]
      st = results[name][-1][1]
      rows.append(dict(n=n, arm=name, ms_per_fit=float(np.median(ms)), ms_all=ms, lml_consumed=st.consumed,
                       lml_evaluated=st.evaluated, round_trips=st.round_trips,
                       lml_per_round_trip=st.evaluated / max(st.round_trips, 1), same_samples_as_batch=same))
      print('  fit N=%5d %-7s %9.1f ms  consumed %6d evaluated %6d round trips %6d (%.2f LML / trip)' % (
          n, name, rows[-1]['ms_per_fit'], st.consumed, st.evaluated, st.round_trips, rows[-1]['lml_per_round_trip']),
          file=sys.stderr)
  return rows


def kernel_alone(Bs=(1, 8, 32, 132), Ns=(64, 128, 256, 512), iters=5):
  import torch
  from dragonfly_b200 import device, kernel, _lib
  rows = []
  d = 6
  for n in Ns:
    rs = np.random.RandomState(n)
    X = rs.random_sample((n, d))
    Y = np.sin(3 * X[:, 0]) + 0.1 * rs.randn(n)
    post = device.DevicePosterior(n)
    stream = torch.cuda.current_stream()
    for B in Bs:
      kerns = [kernel.MaternKernel(d, 2.5, 0.5 + rs.random_sample(), list(0.3 + rs.random_sample(d))) for _ in range(B)]
      descs = [kernel.build_descriptor(k, train_dim=d, cand_dim=d) for k in kerns]
      noise = list(0.01 + 0.01 * rs.random_sample(B))
      mean = list(0.1 * rs.randn(B))

      def singles():
        for i in range(B):
          post.set_train(X, Y - mean[i])
          post.set_kernel(descs[i])
          post.build(noise[i], 0.0, _lib.DFB_BUILD_LML_ONLY)

      def lml_only():
        return post.lml_batch(descs, noise, mean)
      out = {}
      for name, fn in (('lml_batch', lml_only), ('build_posterior_xB', singles)):
        if name == 'lml_batch':
          post.set_train(X, Y)
        fn()                                      # warm-up
        ev = []
        wall = []
        for _ in range(iters):
          s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
          s.record(stream)
          t0 = time.perf_counter()
          fn()
          e.record(stream)
          torch.cuda.synchronize()
          wall.append(1e3 * (time.perf_counter() - t0))
          ev.append(s.elapsed_time(e))
        out[name] = (float(np.median(ev)), float(np.median(wall)))
      rows.append(dict(n=n, B=B, batch_event_ms=out['lml_batch'][0], batch_wall_ms=out['lml_batch'][1],
                       single_event_ms=out['build_posterior_xB'][0], single_wall_ms=out['build_posterior_xB'][1],
                       batch_ms_per_lml=out['lml_batch'][1] / B, single_ms_per_lml=out['build_posterior_xB'][1] / B))
      print('  kernel N=%4d B=%4d  lml_batch %8.3f ms (events %8.3f)   B x build %8.3f ms (events %8.3f)' % (
          n, B, out['lml_batch'][1], out['lml_batch'][0], out['build_posterior_xB'][1], out['build_posterior_xB'][0]),
          file=sys.stderr)
  return rows


def host_arm(sizes=(60, 200), burn=10):
  import post_sampling_ref as R
  rows = []
  for n in sizes:
    X, Y, layout, bounds, dscr = _problem(n)
    ms, st, _ = _fit(X, Y, layout, bounds, dscr, burn, 2, R.oracle_lml_batch(X, Y, layout), 1)
    rows.append(dict(n=n, burn=burn, ms_per_fit=ms, lml=st.evaluated, ms_per_lml=ms / max(st.evaluated, 1)))
    print('  host N=%4d burn %d: %.1f ms, %d LMLs, %.3f ms / LML' % (n, burn, ms, st.evaluated, rows[-1]['ms_per_lml']),
          file=sys.stderr)
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--sizes', default='60,200,500,1000')
  ap.add_argument('--burn', type=int, default=-1)
  ap.add_argument('--num-samples', type=int, default=17)
  ap.add_argument('--reps', type=int, default=1)
  ap.add_argument('--host-burn', type=int, default=10)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  import torch
  assert torch.cuda.is_available(), 'bench_post_sampling.py measures the GPU: no CUDA device visible'
  name, power = _card()
  print('card: %s, power limit %s' % (name, power), file=sys.stderr)
  res = dict(card=name, power_limit=power)
  res['kernel'] = kernel_alone()
  print(json.dumps(dict(table='kernel', card=name, power_limit=power, rows=res['kernel'])))
  res['whole_fit'] = whole_fit([int(s) for s in args.sizes.split(',')], args.burn, args.reps, args.num_samples)
  print(json.dumps(dict(table='whole_fit', burn=args.burn, rows=res['whole_fit'])))
  res['host'] = host_arm(burn=args.host_burn)
  print(json.dumps(dict(table='host', rows=res['host'])))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      json.dump(res, f, indent=1)


if __name__ == '__main__':
  main()
