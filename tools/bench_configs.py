"""Throughput of the other BASELINE.json configs on one GPU (candidates resident in HBM), with the
default (auto) scoring mode and with the int8 path disabled.  Not the headline bench: evidence that
every config of the scope table runs at scale.  Usage: python tools/bench_configs.py [scale]
  scale divides the candidate counts (default 4 -> C2 250k, C3 1M, C4 250k, C5 64k x 256 draws)."""
import os, sys, time, json
import tempfile
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from dragonfly_b200 import synth_data, kernel, gp_core, mf_gp, device
from dragonfly_b200 import gpb_acquisitions as A

scale = int(sys.argv[1]) if len(sys.argv) > 1 else 4
out = {}


def timeit(fn, reps=2):
  fn()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(reps):
    r = fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) / reps, r


def both_modes(run):
  res = {}
  for mode, opt in [('auto', None), ('fp64', 0)]:
    if opt is None:
      device.DEFAULT_OPTIONS.pop('score_impl', None)
    else:
      device.DEFAULT_OPTIONS['score_impl'] = opt
    res[mode] = run()
  device.DEFAULT_OPTIONS.pop('score_impl', None)
  return res


# C2: Hartmann-6, Matern-2.5, N=2000, UCB
def c2():
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_cand=1000000 // scale)
  k = w['kernel']
  gp = gp_core.GP(w['X'], w['Y'], kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                  gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  cd = torch.from_numpy(w['candidates']).cuda()
  acq = device.make_acq_desc('ucb', beta=float(A._get_ucb_beta_th(6, 2000)))
  dt, r = timeit(lambda: gp._fused_score(acq, cd))
  return dict(cands_per_s=len(cd) / dt, argmax=int(r[1]), used_i8=gp._post.query('last_used_i8'))
out['c2_hartmann6_matern_ucb_N2000'] = both_modes(c2)
print('c2', out['c2_hartmann6_matern_ucb_N2000'], flush=True)


# C3: 40-D additive GP, add_ucb, N=5000: 7 groups, candidates per group in the d_j-dim sub-box
def c3():
  w = synth_data.make_workload('c3_additive40_add_ucb', n_cand=16)
  gp = gp_core.GP(w['X'], w['Y'], kernel.kernel_from_spec(w['kernel']), gp_core.ConstantMean(w['mean_const']),
                  w['noise_var'])
  total = 4000000 // scale
  dom = A.EuclideanDomain([[0, 1]] * 40)
  from argparse import Namespace
  anc = Namespace(curr_acq='add_ucb', max_evals=total, t=5000, domain=dom, curr_max_val=float(w['Y'].max()),
                  eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', is_mf=False,
                  domain_bounds=np.array(dom.bounds))
  np.random.seed(0)
  dt, pt = timeit(lambda: A.asy.add_ucb(gp, anc), reps=1)
  return dict(cands_per_s=total / dt, point_head=[float(x) for x in pt[:3]],
              note='end to end asy_add_ucb incl. host candidate generation (NumPy RNG) and H2D')
out['c3_additive40_add_ucb_N5000'] = both_modes(c3)
print('c3', out['c3_additive40_add_ucb_N5000'], flush=True)


# C4: Borehole MF product kernel, N=4000, UCB on the fidel_to_opt slice
def c4():
  w = synth_data.make_workload('c4_borehole_mf_ucb', n_cand=1000000 // scale)
  ks = w['kernel']
  kF = kernel.kernel_from_spec(ks['kernels'][0]); kD = kernel.kernel_from_spec(ks['kernels'][1])
  mfgp = mf_gp.EuclideanMFGP(list(w['X'][:, :1]), list(w['X'][:, 1:]), list(w['Y']), None, ks['scale'], kF, kD,
                             gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  zx = torch.from_numpy(np.concatenate((np.ones((len(w['candidates']), 1)), w['candidates']), axis=1)).cuda()
  acq = device.make_acq_desc('ucb', beta=float(A._get_ucb_beta_th(8, 4000)))
  dt, r = timeit(lambda: mfgp._fused_score(acq, zx))
  return dict(cands_per_s=len(zx) / dt, argmax=int(r[1]), used_i8=mfgp._post.query('last_used_i8'))
out['c4_borehole_mf_ucb_N4000'] = both_modes(c4)
print('c4', out['c4_borehole_mf_ucb_N4000'], flush=True)


# C5: Park1-20, Thompson sampling, 256 joint draws per block of 4096 candidates, N=5000
def c5():
  w = synth_data.make_workload('c5_park1_20_ts', n_cand=(1000000 // scale) // 16)
  k = w['kernel']
  gp = gp_core.GP(w['X'], w['Y'], kernel.MaternKernel(20, 2.5, k['scale'], k['dim_bandwidths']),
                  gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  np.random.seed(2)
  t0 = time.perf_counter()
  samples = gp.draw_samples(256, w['candidates'])
  dt = time.perf_counter() - t0
  return dict(cands_per_s=len(w['candidates']) / dt, draws=256, finite=bool(np.isfinite(samples).all()),
              argmax_head=[int(i) for i in samples.argmax(axis=1)[:4]],
              note='block-exact joint draws (4096-candidate blocks), host normals + H2D/D2H included')
def c5_device_rng():
  w = synth_data.make_workload('c5_park1_20_ts', n_cand=1000000 // scale)
  k = w['kernel']
  gp = gp_core.GP(w['X'], w['Y'], kernel.MaternKernel(20, 2.5, k['scale'], k['dim_bandwidths']),
                  gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  cd = torch.from_numpy(w['candidates']).cuda()
  gp.draw_samples_argmax(256, cd[:4096], seed=2)
  torch.cuda.synchronize(); t0 = time.perf_counter()
  vals, idxs = gp.draw_samples_argmax(256, cd, seed=2)
  torch.cuda.synchronize(); dt = time.perf_counter() - t0
  return dict(cands_per_s=len(cd) / dt, draws=256, candidates=len(cd), seconds=dt, finite=bool(np.isfinite(vals).all()),
              argmax_head=[int(i) for i in idxs[:4]],
              note='GP.draw_samples_argmax: device Philox normals + running per-draw arg-max, nothing but 256 pairs leaves the GPU')
out['c5_park1_20_ts_N5000'] = {'auto': c5(), 'device_rng_argmax': c5_device_rng()}
print('c5', out['c5_park1_20_ts_N5000'], flush=True)

# hp grid: LML-only builds at N=5000
from dragonfly_b200 import hp_grid
w = synth_data.make_workload('headline_hartmann6_matern_ei', n_cand=16)
layout = hp_grid.EuclideanHPLayout(6, 'matern', nu=2.5)
rs = np.random.RandomState(0)
hps = np.concatenate((np.log(w['Y'].var()) + rs.uniform(-6, -3, (12, 1)), np.log(w['Y'].var()) + rs.uniform(-1, 1, (12, 1)),
                      rs.uniform(np.log(0.15), np.log(1.0), (12, 6))), axis=1)
out['hp_grid_N5000'] = {}
for lanes in (1, 2, 3, 4):
  lm, post = hp_grid.lml_for_hyperparams(w['X'], w['Y'], hps[:2 * lanes], layout, lanes=lanes)
  torch.cuda.synchronize()
  t0 = time.perf_counter(); lm, post = hp_grid.lml_for_hyperparams(w['X'], w['Y'], hps, layout, post=post, lanes=lanes); dt = time.perf_counter() - t0
  out['hp_grid_N5000']['lanes%d' % lanes] = dict(lml_per_s=len(hps) / dt, ms_per_lml=1e3 * dt / len(hps), finite=bool(np.isfinite(lm).all()),
                                                 lml_head=[float(v) for v in lm[:3]])
  del post
print('hp', out['hp_grid_N5000'], flush=True)

# multi-objective: 2 objectives on the C2 geometry (N=2000), linear and Tchebychev UCB scalarisations, device candidates
def moo():
  from dragonfly_b200 import multiobjective_gpb_acquisitions as M, _lib
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_cand=1000000 // scale)
  k = w['kernel']
  Y2 = -np.sum((w['X'] - 0.4) ** 2, axis=1)
  gps = [gp_core.GP(w['X'], w['Y'], kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                    gp_core.ConstantMean(w['mean_const']), w['noise_var']),
         gp_core.GP(w['X'], Y2, kernel.SEKernel(6, float(Y2.var()), [0.35] * 6),
                    gp_core.ConstantMean(float(np.median(Y2))), 0.01 * float(Y2.var()))]
  cd = torch.from_numpy(w['candidates']).cuda()
  beta = float(M._get_ucb_beta_th(6, 2000))
  res = {}
  for name, kind in [('lin_ucb', _lib.DFB_MOO_LIN_UCB), ('tch_ucb', _lib.DFB_MOO_TCH_UCB)]:
    def run():
      mus, sds = zip(*[gp.eval(cd, uncert_form='std') for gp in gps])
      return gps[0]._post.moo_score_argmax(kind, list(mus), list(sds), [0.6, 0.4], [0.1, -1.0], beta)
    dt, r = timeit(run)
    res[name] = dict(cands_per_s=len(cd) / dt, argmax=int(r[1]), objectives=2,
                     note='fp64 dfb_eval per objective (exact mu, sigma) + one dfb_moo_score_argmax')
  return res
out['moo_2obj_N2000'] = moo()
print('moo', out['moo_2obj_N2000'], flush=True)


# incremental posterior update at the metric's N: one new observation, and 4 hallucinated points around a scoring call
def incremental():
  w = synth_data.make_workload('headline_hartmann6_matern_ei', n_cand=200000 // scale)
  k = w['kernel']
  X, Y = w['X'], w['Y']
  gp = gp_core.GP(X[:4995], Y[:4995], kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                  gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  res = {}
  ts = []
  for i in range(4995, 5000):
    torch.cuda.synchronize(); t0 = time.perf_counter()
    gp.add_data_single(X[i], Y[i])
    torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
  res['add_data_single_ms'] = [1e3 * t for t in ts]
  dt, _ = timeit(lambda: gp_core.GP(X, Y, gp.kernel, gp.mean_func, w['noise_var']))
  res['full_build_ms'] = 1e3 * dt
  cd = torch.from_numpy(w['candidates']).cuda()
  acq = device.make_acq_desc('ucb', beta=float(A._get_ucb_beta_th(6, 5000)))
  Xh = list(np.random.RandomState(3).random_sample((4, 6)))
  for inc in (True, False):
    gp.incremental_updates = inc
    dt, r = timeit(lambda: gp._fused_score(acq, cd, halluc=Xh))
    res['score_with_4_hallucinations_ms_%s' % ('in_place' if inc else 'fresh_build')] = 1e3 * dt
    res['argmax_%s' % ('in_place' if inc else 'fresh_build')] = int(r[1])
  dt, _ = timeit(lambda: gp._fused_score(acq, cd))
  res['score_without_hallucinations_ms'] = 1e3 * dt
  res['candidates'] = len(cd)
  return res
out['incremental_N5000'] = incremental()
print('inc', out['incremental_N5000'], flush=True)
json.dump(out, open(os.path.join(tempfile.gettempdir(), 'bench_configs.json'), 'w'), indent=1)
