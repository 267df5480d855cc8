"""Validation sweep of the int8-slice path's a-priori sigma^2 bound (api.cu: i8_sigma2_bound).

For every (kernel family, N, noise / scale, scale, digit scheme) the SAME posterior (same L, W = L^-1) scores 13056
uniform candidates once with the fp64 DMMA contraction and once with the int8 wgmma digit contraction (guard
switched off with the diagnostic option "i8_unguarded", so that configurations the guard would refuse are measured
too); the record holds max |sigma^2_int8 - sigma^2_fp64|, the library's bound and their ratio.  The run FAILS if any
measured maximum exceeds its bound; this sweep is what the constant 8 in i8_sigma2_bound rests on, so re-run it
whenever the digit schemes or the contraction change.

Usage (on the GPU): python tools/sweep_i8_bound.py [out.json]
"""
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from dragonfly_b200 import gp_core, kernel, synth_data  # noqa: E402

OUT = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), 'i8_bound_sweep.json')
M = 13056


def make_kernel(name, scale):
  if name == 'se':
    return kernel.SEKernel(6, scale, [0.3, 0.35, 0.4, 0.3, 0.5, 0.45]), 6
  if name == 'matern25':
    return kernel.MaternKernel(6, 2.5, scale, 0.3), 6
  if name == 'matern05':
    return kernel.MaternKernel(6, 0.5, scale, 0.4), 6
  if name == 'additive':
    return kernel.AdditiveKernel(scale / 2, [kernel.MaternKernel(3, 2.5, 1.0, 0.5), kernel.SEKernel(3, 1.0, 0.4)],
                                 [[0, 1, 2], [3, 4, 5]]), 6
  if name == 'product':
    return kernel.CoordinateProductKernel(6, scale, [kernel.SEKernel(1, 1.0, [0.7]), kernel.MaternKernel(5, 2.5, 1.0, 0.4)],
                                          [[0], [1, 2, 3, 4, 5]]), 6
  raise ValueError(name)


def main():
  rows, worst = [], 0.0
  t0 = time.time()
  rs = np.random.RandomState(0)
  Xall = rs.random_sample((5000, 6))
  Yall = synth_data.hartmann6(Xall)
  C = torch.from_numpy(np.random.RandomState(1).random_sample((M, 6))).cuda()
  for kname in ['se', 'matern25', 'matern05', 'additive', 'product']:
    for n in [1024, 2000, 3500, 5000]:
      for scale in [1e-2, 1.0, 1e4]:
        for noise_ratio in [1e-2, 1e-4, 1e-6, 1e-8]:
          kern, _ = make_kernel(kname, scale)
          X = Xall[:n]
          Y = Yall[:n] * np.sqrt(scale / Yall.var())
          try:
            gp = gp_core.GP(X, Y, kern, gp_core.ConstantMean(float(np.median(Y))), noise_ratio * scale)
          except Exception as e:  # pylint: disable=broad-except
            rows.append(dict(kernel=kname, n=n, scale=scale, noise_ratio=noise_ratio, error=str(e)[:80]))
            continue
          post = gp._post
          post.set_option('score_impl', 0)
          _, sd0 = post.eval(C, mean_const=0.0)
          var0 = (sd0 ** 2).cpu().numpy()
          post.set_option('i8_unguarded', 1)
          for radix in (0, 1):
            post.set_option('i8_radix', radix)
            post.set_option('score_impl', 1)
            _, sd1 = post.eval(C, mean_const=0.0)
            assert post.query('last_used_i8') == 1.0
            err = float(np.nanmax(np.abs((sd1 ** 2).cpu().numpy() - var0)))
            bound = post.query('i8_sigma2_bound')
            ratio = err / bound
            worst = max(worst, ratio)
            rows.append(dict(kernel=kname, n=n, scale=scale, noise_ratio=noise_ratio, jitter_power=gp.jitter_power,
                             radix=256 if radix else 128, max_abs_dsigma2=err, bound=bound, ratio=ratio,
                             guard_would_allow=bool(bound <= 5e-9)))
          del gp, post
  ok = worst <= 1.0
  allowed = [r for r in rows if r.get('guard_would_allow')]
  out = dict(candidates=M, configurations=len(rows), worst_measured_over_bound=worst,
             margin_of_the_bound=(1.0 / worst if worst > 0 else None),
             worst_abs_error_where_the_guard_allows=max([r['max_abs_dsigma2'] for r in allowed] or [0.0]),
             configurations_the_guard_allows=len(allowed), all_within_bound=ok, seconds=time.time() - t0, rows=rows)
  os.makedirs(os.path.dirname(OUT) or '.', exist_ok=True)
  json.dump(out, open(OUT, 'w'), indent=1)
  print(json.dumps({k: v for k, v in out.items() if k != 'rows'}))
  assert ok, 'a measured int8 sigma^2 error exceeds the a-priori bound'


if __name__ == '__main__':
  main()
