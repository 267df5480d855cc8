"""One small scoring call for ncu captures of the K_* kernels (headline geometry, 3 chunks)."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, gp_core, device
w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=5000, n_cand=16)
gp = gp_core.GP(w['X'], w['Y'], kernel.kernel_from_spec(w['kernel']), gp_core.ConstantMean(w['mean_const']), w['noise_var'])
acq = device.make_acq_desc('ei', best=float(w['Y'].max()))
cd = torch.from_numpy(np.random.RandomState(1000).random_sample((3 * 6528, 6))).cuda()
for _ in range(2):
  r = gp._fused_score(acq, cd)
torch.cuda.synchronize()
print(r[:2])
