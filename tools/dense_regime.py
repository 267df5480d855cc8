"""The int8 screen in a dense, low-dimensional regime (C1-like: Branin 2-D, SE, many training points close together, late
BO iterations): how large the fp64 re-score shortlist gets, whether the pass overflows / self-check fails, and what the
step costs against the pure-fp64 path.  Usage: python tools/dense_regime.py"""
import json, os, sys, time
import tempfile
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, gp_core, device

out = {}
for n, tag, spread, noise in [(2000, 'branin2d_se_N2000_tight', 0.02, 0.01), (5000, 'branin2d_se_N5000_tight', 0.02, 0.01),
                              (2000, 'branin2d_se_N2000_loose', 0.06, 0.05), (5000, 'branin2d_se_N5000_loose', 0.06, 0.05)]:
  rs = np.random.RandomState(0)
  # late-iteration data: half of the points clustered around the three Branin optima
  Xu = rs.random_sample((n // 2, 2))
  opt = np.array([[0.124, 0.818], [0.543, 0.152], [0.962, 0.165]])
  Xc = np.clip(opt[rs.randint(0, 3, n - n // 2)] + spread * rs.standard_normal((n - n // 2, 2)), 0, 1)
  X = np.concatenate((Xu, Xc)); Y = synth_data.branin(X)
  Ys = Y / Y.std()
  gp = gp_core.GP(X, Ys, kernel.SEKernel(2, 1.0, [0.2, 0.2]), gp_core.ConstantMean(float(np.median(Ys))), noise)
  C = torch.from_numpy(np.random.RandomState(1).random_sample((1000000, 2))).cuda()
  res = {'jitter_power': gp.jitter_power}
  for name, acq in [('ei', device.make_acq_desc('ei', best=float(Ys.max()))), ('ucb', device.make_acq_desc('ucb', beta=2.5)),
                    ('pi', device.make_acq_desc('pi', best=float(Ys.max())))]:
    r = {}
    for mode, impl in [('auto', 2), ('fp64', 0)]:
      gp._post.set_option('score_impl', impl)
      gp._fused_score(acq, C[:100000]); torch.cuda.synchronize()
      t0 = time.perf_counter(); best, idx, _ = gp._fused_score(acq, C); torch.cuda.synchronize()
      r[mode] = dict(ms=1e3 * (time.perf_counter() - t0), argmax=int(idx), best=float(best), used_i8=gp._post.query('last_used_i8'),
                     shortlist=gp._post.query('last_shortlist'), selfcheck_violations=gp._post.query('last_selfcheck_violations'),
                     selfcheck_ratio=gp._post.query('last_selfcheck_ratio'), bound=gp._post.query('i8_sigma2_bound'))
    r['same_argmax'] = r['auto']['argmax'] == r['fp64']['argmax'] and r['auto']['best'] == r['fp64']['best']
    res[name] = r
  gp._post.set_option('score_impl', 2)
  out[tag] = res
  print(tag, json.dumps(res), flush=True)
json.dump(out, open(os.path.join(tempfile.gettempdir(), 'r02_dense_regime.json'), 'w'), indent=1)
