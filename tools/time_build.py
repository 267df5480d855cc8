"""Posterior build time with and without the look-ahead schedule (option "lookahead"), full and LML-only builds,
and a bit-for-bit comparison of what the two schedules produce.  Usage: python tools/time_build.py"""
import os, sys, time, json
import tempfile
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, device, _lib

out = {}
for n in (1000, 2000, 5000):
  w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=n, n_cand=16)
  k = w['kernel']
  desc = kernel.build_descriptor(kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']))
  state = {}
  for la in (0, 1):
    post = device.DevicePosterior(n)
    post.set_option('lookahead', la)
    post.set_kernel(desc)
    post.set_train(w['X'], w['Y'] - w['mean_const'])
    res = {}
    for name, flags in (('full', _lib.DFB_BUILD_FULL), ('lml_only', _lib.DFB_BUILD_LML_ONLY)):
      for _ in range(3):
        info, lml = post.build(w['noise_var'], 0.0, flags)
      torch.cuda.synchronize()
      ts = []
      for _ in range(10):
        t0 = time.perf_counter()
        info, lml = post.build(w['noise_var'], 0.0, flags)
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
      res[name + '_ms_median'] = float(np.median(ts)); res[name + '_ms_min'] = float(min(ts))
      res[name + '_lml'] = lml
      assert info == 0
    info, lml = post.build(w['noise_var'], 0.0, _lib.DFB_BUILD_FULL)
    L, a, _ = post.get_state(want_L=True, want_alpha=True)
    state[la] = (L.cpu().numpy(), a.cpu().numpy(), lml)
    out['N%d_lookahead%d' % (n, la)] = res
    del post
  same = bool((state[0][0] == state[1][0]).all() and (state[0][1] == state[1][1]).all() and state[0][2] == state[1][2])
  out['N%d_bit_identical' % n] = same
  print(n, json.dumps({k2: v for k2, v in out.items() if k2.startswith('N%d' % n)}), flush=True)
  assert same, 'look-ahead schedule changed the numbers'
json.dump(out, open(os.path.join(tempfile.gettempdir(), 'time_build.json'), 'w'), indent=1)
