"""Wall-clock / device-time breakdown of one bench.py step (build + fused score of 10^6 candidates).

The device line splits the score into the contracted rows (kstar, gemm, acq: the seeds and the survivors of the bound
pass) and the bound pass itself (a certified upper bound of mu for every candidate, the seed selection and the
screen)."""
import os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, gp_core, device

n_cand = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=5000, n_cand=1000)
k = w['kernel']
kern = kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])
mean = gp_core.ConstantMean(w['mean_const'])
acq = device.make_acq_desc('ei', best=float(w['Y'].max()))
cd = torch.rand((n_cand, 6), dtype=torch.float64, device='cuda')
sync = torch.cuda.synchronize


def query(post, name):
  try:
    return int(post.query(name))
  except Exception:           # an older library (DFB200_LIB) without this query
    return -1


for prof in (False, False, False, True):
  sync(); t0 = time.perf_counter()
  gp = gp_core.GP(w['X'], w['Y'], kern, mean, w['noise_var'], device=0)
  sync(); t1 = time.perf_counter()
  if prof: gp._post.profile_enable(True)
  best, idx, _ = gp._fused_score(acq, cd)
  sync(); t2 = time.perf_counter()
  line = 'build %.2f ms  score %.2f ms  total %.2f ms' % (1e3 * (t1 - t0), 1e3 * (t2 - t1), 1e3 * (t2 - t0))
  if prof:
    r = [gp._post.profile_read(c) for c in (0, 1, 2, 4)]
    # kstar / gemm / acq: the rows that were contracted (the seeds and the survivors of the bound pass);
    # bound: the upper bound of mu over every candidate, the seed selection and the screen
    line += ' | device: kstar %.2f (%d) gemm %.2f (%d, %d cand) acq %.2f (%d) bound %.2f (%d) sum %.2f' % (
        r[0][0], r[0][1], r[1][0], r[1][1], r[1][2], r[2][0], r[2][1], r[3][0], r[3][1], sum(x[0] for x in r))
    q = lambda name: query(gp._post, name)
    line += ' | shortlist %d seeds %d survivors %d pruned %d contracted %d' % (
        q('last_shortlist'), q('last_seed_rows'), q('last_survivors'), q('last_pruned_candidates'),
        q('last_contracted_rows'))
  print(line)
  del gp

# ---- finer: time each DevicePosterior call inside GP construction -------------------------------------------
import functools
acc = {}
def wrap(name):
  orig = getattr(device.DevicePosterior, name)
  @functools.wraps(orig)
  def f(self, *a, **kw):
    sync(); t = time.perf_counter()
    out = orig(self, *a, **kw)
    sync(); acc.setdefault(name, []).append(1e3 * (time.perf_counter() - t))
    return out
  setattr(device.DevicePosterior, name, f)
for nm in ('__init__', 'set_kernel', 'set_train', 'build', '__del__'):
  wrap(nm)
for _ in range(6):
  sync(); t0 = time.perf_counter()
  gp = gp_core.GP(w['X'], w['Y'], kern, mean, w['noise_var'], device=0)
  sync(); t1 = time.perf_counter()
  acc.setdefault('GP()', []).append(1e3 * (t1 - t0))
  best, idx, _ = gp._fused_score(acq, cd[:6528])
  del gp
for k_, v in acc.items():
  print('%-12s' % k_, ' '.join('%7.2f' % x for x in v))
