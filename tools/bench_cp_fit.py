"""
Whole hyper-parameter fits of a Cartesian-product GP on the mixed domain of tools/bench_mixed.py: [Euclidean(2),
Integral(1), ProdDiscrete(3 dims, 2-5 levels), ProdDiscreteNumeric(1)] with CPGPFitter's default kernels (Matern 5/2
numeric parts, three tuned Hamming weights), tuned mean and noise: 13 continuous hps.  Two fits, at N = 60, 200, 500:
  direct  ml_hp_tune_opt 'direct' as PDOO (the CP default for <= 60 hps where Fortran DIRECT is not built), the
          reference's default budget of max(500, 50 x 13) = 650 evaluations;
  post    post_sampling with the slice sampler, one sample, burn-in --burn per hp (the default -1 means
          int(sqrt(13) x 100) = 360 slice samples per hp).
Arms, alternated within each step:
  batched  the device path: dfb_lml_batch_mixed for N <= 512 (one launch per batch), speculation depth 8;
  single   one LML-only dfb_build_posterior per LML (lml_for_hyperparams, one lane), sampler depth 1;
  host     the NumPy oracle per LML, timed over --host-lmls LMLs and multiplied by the LMLs the fit consumed.
Prints one JSON line per table (fit), with the card's name and power limit read in the same run.

  python tools/bench_cp_fit.py [--steps 1] [--burn 50] [--ns 60,200,500]
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


def _problem(n, seed=0):
  from dragonfly_b200 import gpb_acquisitions as acq, domains, kernel, cartesian_product_gp as cp
  import hamming_ref as H
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = H.make_domain(domains, levels, numeric_levels)
  parts = acq._cp_parts(dom, H.make_kernel(kernel, cp, 1.0))
  np.random.seed(seed)
  Xr, draws = acq.draw_cp_candidates(parts, n)
  X = [acq.point_from_draws(parts, draws, i) for i in range(n)]
  Y = np.sin(3 * Xr[:, 0]) + 0.3 * Xr[:, 1] - 0.1 * (Xr[:, 2] - 3) ** 2 + 0.4 * (Xr[:, 3] == 1) + \
      0.2 * np.log(Xr[:, 6]) + 0.05 * np.random.standard_normal(n)
  return X, Y


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=1)
  ap.add_argument('--burn', type=int, default=-1)
  ap.add_argument('--ns', default='60,200,500')
  ap.add_argument('--host-lmls', type=int, default=20)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import hp_grid, post_sampling, _lib
  import cp_fitter_ref as R
  _lib.load()
  lay_parts = R.parts('M')
  name, plimit = _card()
  single_batch = lambda X, Y, hps, layout, nus=None, post=None, device=None: hp_grid.lml_for_hyperparams(
      X, Y, hps, layout, nus=nus, post=post, device=device, lanes=1)
  for fit in ('direct', 'post'):
    table = {}
    for n in [int(v) for v in args.ns.split(',')]:
      X, Y = _problem(n)
      row = {}
      times = {'batched': [], 'single': []}
      consumed = None
      for step in range(args.steps):
        for arm in ('batched', 'single'):
          lay = hp_grid.CartesianProductHPLayout(lay_parts, mean_func_type='tune', noise_var_type='tune')
          bounds, dscr = lay.bounds(X, Y)
          counter = {'n': 0}
          orig = hp_grid.lml_batch_for_hyperparams
          inner = orig if arm == 'batched' else single_batch

          def counted(*a, **k):
            counter['n'] += len(a[2])
            return inner(*a, **k)
          np.random.seed(step)
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          if fit == 'direct':
            hp_grid.lml_batch_for_hyperparams = counted
            try:
              hp_grid.fit_gp(X, Y, lay, bounds, dscr, method='direct', build_gp=lambda c, d, g: None)
            finally:
              hp_grid.lml_batch_for_hyperparams = orig
            lmls = counter['n']
          else:
            stats = post_sampling.PostSamplingStats()
            Xc = lay.encode(X)
            batch_fn = orig if arm == 'batched' else single_batch
            post_sampling.post_sample_hps(X, Y, lay, bounds, dscr, num_samples=1, burn=args.burn,
                                          build_gp=lambda c, d: None, stats=stats, depth=None if arm == 'batched'
                                          else 1, lml_batch=post_sampling.device_lml_batch(Xc, Y, lay, False,
                                                                                           batch_fn=batch_fn))
            lmls = stats.consumed
          torch.cuda.synchronize()
          times[arm].append(time.perf_counter() - t0)
          consumed = lmls if consumed is None else consumed
          row[arm + '_lmls'] = lmls
      for arm in times:
        row[arm + '_s'] = round(float(np.median(times[arm])), 3)
      # host arm: the oracle per LML on a short run, projected onto the LMLs the device fit consumed
      lay = hp_grid.CartesianProductHPLayout(lay_parts, mean_func_type='tune', noise_var_type='tune')
      Xc = lay.encode(X)
      b = lay.bounds(X, Y)[0]
      rs = np.random.RandomState(1)
      hps = b[:, 0] + rs.random_sample((args.host_lmls, len(b))) * (b[:, 1] - b[:, 0])
      t0 = time.perf_counter()
      for h in hps:
        R.oracle_lml(Xc, Y, lay, h, ())
      per = (time.perf_counter() - t0) / args.host_lmls
      row['host_s_per_lml'] = round(per, 5)
      row['host_projected_s'] = round(per * consumed, 1)
      row['speedup_vs_single'] = round(row['single_s'] / row['batched_s'], 2)
      table[str(n)] = row
    print(json.dumps(dict(bench='cp_fit', fit=fit, burn=args.burn, steps=args.steps, card=name, power_limit=plimit,
                          table=table)))


if __name__ == '__main__':
  main()
