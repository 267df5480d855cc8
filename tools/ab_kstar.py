"""A/B of the K_* stage at the headline geometry: kstar_seg in {0,1} -- step time of gp._fused_score over M
candidates, per-class launch times, and the arg-max each variant returns."""
import json, os, sys, time
import tempfile
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, gp_core, device

M = int(sys.argv[1]) if len(sys.argv) > 1 else 1000000
w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=5000, n_cand=16)
gp = gp_core.GP(w['X'], w['Y'], kernel.kernel_from_spec(w['kernel']), gp_core.ConstantMean(w['mean_const']), w['noise_var'])
acq = device.make_acq_desc('ei', best=float(w['Y'].max()))
cd = torch.from_numpy(np.random.RandomState(1000).random_sample((M, 6))).cuda()
out = {}
for seg in (0, 1):
  gp._post.set_option('kstar_seg', seg)
  gp._fused_score(acq, cd[:200000])
  torch.cuda.synchronize()
  ts = []
  for _ in range(3):
    t0 = time.perf_counter(); r = gp._fused_score(acq, cd); torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
  gp._post.profile_enable(True)
  gp._fused_score(acq, cd)
  prof = {n: gp._post.profile_read(c) for n, c in [('kstar', 0), ('gemm', 1), ('acq', 2)]}
  gp._post.profile_enable(False)
  out['seg%d' % seg] = dict(ms=ts, best=float(r[0]), argmax=int(r[1]),
                            kstar_ms_per_launch=prof['kstar'][0] / max(prof['kstar'][1], 1),
                            gemm_ms_per_launch=prof['gemm'][0] / max(prof['gemm'][1], 1),
                            shortlist=gp._post.query('last_shortlist'))
  print('seg%d' % seg, out['seg%d' % seg], flush=True)
# accuracy of the seg path's sigma^2 / mu against fp64 on 4 chunks
sub = cd[:26112]
gp._post.set_option('kstar_seg', 1)
gp._post.set_option('score_impl', 1); mu8, sd8 = gp._post.eval(sub, mean_const=w['mean_const'], want_std=True)
gp._post.set_option('kstar_seg', 0); mu8o, sd8o = gp._post.eval(sub, mean_const=w['mean_const'], want_std=True)
gp._post.set_option('score_impl', 0); mu64, sd64 = gp._post.eval(sub, mean_const=w['mean_const'], want_std=True)
out['accuracy'] = dict(dsig2_seg=float((sd8 ** 2 - sd64 ** 2).abs().max()), dsig2_old=float((sd8o ** 2 - sd64 ** 2).abs().max()),
                       dmu_seg=float((mu8 - mu64).abs().max()), dmu_old=float((mu8o - mu64).abs().max()))
print(out['accuracy'])
json.dump(out, open(os.path.join(tempfile.gettempdir(), 'ab_kstar.json'), 'w'), indent=1)
