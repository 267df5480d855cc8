"""
Parity tests proper (-m gpu): the CUDA path, called through the C-ABI (ctypes) behind the mirrored
Kernel / GP / gpb_acquisitions surfaces, against
  (1) the committed golden fixtures = outputs of the UNMODIFIED reference (tests/golden/*.npz),
  (2) the NumPy oracle on the same seeded inputs at sizes it finishes in seconds,
  (3) size-independent properties at BASELINE.json's full N.
Tolerances (BASELINE.json north_star): |d mu| <= 1e-10, |d sigma^2| <= 1e-8, arg-max index exact.
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu

MU_TOL = 1e-10
VAR_TOL = 1e-8


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, mf_gp, gpb_acquisitions, domains, device, _lib
  _lib.load()
  return Namespace(kernel=kernel, gp_core=gp_core, mf_gp=mf_gp, acq=gpb_acquisitions,
                   domains=domains, device=device, lib=_lib, torch=torch)


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def anc(B, acq, max_evals, t, d, curr_max, in_progress=(), **kw):
  dom = B.domains.EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq=acq, max_evals=max_evals, t=t, domain=dom, curr_max_val=curr_max,
                   eval_points_in_progress=list(in_progress), acq_opt_method='rand',
                   handle_parallel='halluc', mf_strategy=None, is_mf=False,
                   domain_bounds=np.array(dom.bounds), **kw)


def close(a, b, rtol=0, atol=0):
  np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=atol)


# ---- the reference's own known-answer vectors, on the device -----------------------------------------
def test_kernel_known_answers_on_device(B):
  """ unittest_kernel.py:82-124 restated: closed forms to 1e-10 (Frobenius norm). """
  g = load_golden('known_answers')
  d1, d2 = g['data_1'], g['data_2']
  se = B.kernel.SEKernel(2, 2, [0.1, 1])
  t11 = 2 * np.array([[1, np.exp(-406.25 / 2)], [np.exp(-406.25 / 2), 1]])
  t12 = 2 * np.array([[1, np.exp(-404 / 2)], [np.exp(-406.25 / 2), np.exp(-0.25 / 2)]])
  assert np.linalg.norm(t11 - se(d1)) < 1e-10
  assert np.linalg.norm(t12 - se(d1, d2)) < 1e-10
  close(se(d1, d2), g['se_12'], atol=1e-13)
  for nu in [0.5, 1.5, 2.5]:
    tag = str(nu).replace('.', 'p')
    mk = B.kernel.MaternKernel(2, nu, 2.1, [0.1, 1])
    assert mk.norm_constant == float(g['matern_%s_norm_constant' % tag])
    close(mk(d1), g['matern_%s_11' % tag], atol=1e-13)
    close(mk(d1, d2), g['matern_%s_12' % tag], atol=1e-13)
    close(mk(d2), g['matern_%s_22' % tag], atol=1e-13)


def test_dist_squared_known_answer_through_se(B):
  """ unittest_general_utils.py:26-35: D2 = [[1,4,6],[0,1,3],[2.25,2.25,0.25]] (exact in fp64);
      seen through k = exp(-D2/2) with unit scale and bandwidths. """
  X1 = np.array([[1, 2, 3], [1, 2, 4], [2, 3, 4.5]])
  X2 = np.array([[1, 2, 4], [1, 2, 5], [2, 3, 5]])
  true = np.array([[1, 4, 6], [0, 1, 3], [2.25, 2.25, 0.25]])
  K = B.kernel.SEKernel(3, 1.0, [1.0, 1.0, 1.0])(X1, X2)
  close(K, np.exp(-true / 2), rtol=4e-16)


def test_empty_inputs(B):
  se = B.kernel.SEKernel(2, 1.0, [1.0, 1.0])
  assert se(np.zeros((0, 2)), np.zeros((3, 2))).shape == (0, 3)
  assert se(np.zeros((3, 2)), np.zeros((0, 2))).shape == (3, 0)


# ---- C1: Branin 2-D, SE, N = 50 --------------------------------------------------------------------------
@pytest.fixture(scope='module')
def c1(B):
  g = load_golden('c1_se')
  kern = B.kernel.SEKernel(2, float(g['scale']), g['bws'])
  gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(float(g['mean_const'])), float(g['noise_var']))
  return g, gp


def test_c1_posterior_state(c1):
  g, gp = c1
  close(gp.K_trtr_wo_noise, g['K'], atol=1e-12)
  close(gp.L, g['L'], rtol=1e-9, atol=1e-11)
  close(gp.alpha, g['alpha'], rtol=1e-8, atol=1e-10)
  close(gp.compute_log_marginal_likelihood(), g['lml'], rtol=1e-11)
  assert gp.jitter_power is None


def test_c1_eval(c1):
  g, gp = c1
  mu, sd = gp.eval(g['C'], 'std')
  close(mu, g['mu'], atol=MU_TOL)
  close(sd ** 2, g['sd'] ** 2, atol=VAR_TOL)
  mu0, none = gp.eval(g['C'], 'none')
  assert none is None
  close(mu0, g['mu_none'], atol=MU_TOL)
  with pytest.raises(ValueError):
    gp.eval(g['C'][:4], 'bogus')
  # a single row, a list of rows (gp.X style), and ragged chunk edges
  mu1, sd1 = gp.eval([g['C'][7]], 'std')
  close(mu1, g['mu'][7:8], atol=MU_TOL)
  mu2, sd2 = gp.eval(list(g['C'][:129]), 'std')
  close(mu2, g['mu'][:129], atol=MU_TOL); close(sd2 ** 2, g['sd'][:129] ** 2, atol=VAR_TOL)


def test_c1_device_tensor_candidates(B, c1):
  g, gp = c1
  Cd = B.torch.from_numpy(g['C']).cuda()
  mu, sd = gp.eval(Cd, 'std')
  assert mu.is_cuda and sd.is_cuda
  close(mu.cpu().numpy(), g['mu'], atol=MU_TOL)
  close(sd.cpu().numpy() ** 2, g['sd'] ** 2, atol=VAR_TOL)


@pytest.mark.parametrize('name', ['ucb', 'ei', 'pi', 'ttei'])
def test_c1_acquisition_scores_and_argmax(B, c1, name):
  g, gp = c1
  if name == 'ucb':
    acq = B.device.make_acq_desc('ucb', beta=float(g['beta']))
  elif name == 'ttei':
    ri = int(g['ttei_ref_idx'])
    acq = B.device.make_acq_desc('ttei', ref_mean=float(g['mu'][ri]), ref_std=float(g['sd'][ri]))
  else:
    acq = B.device.make_acq_desc(name, best=float(g['curr_best']))
  best, idx, scores = gp._fused_score(acq, g['C'], want_scores=True)
  assert idx == int(g['argmax_' + name])              # bit-exact arg-max index
  close(scores, g[name], rtol=1e-7, atol=1e-9)
  assert best == scores[idx]
  # device-resident candidates give the same answer
  best_d, idx_d, _ = gp._fused_score(acq, B.torch.from_numpy(g['C']).cuda())
  assert idx_d == idx and best_d == best


@pytest.mark.parametrize('name', ['ei', 'ucb', 'pi'])
def test_c1_end_to_end_acquisition(B, c1, name):
  """ asy_<acq>(gp, anc_data) with the same global seed returns the reference's point exactly. """
  g, gp = c1
  np.random.seed(7)
  pt = getattr(B.acq.asy, name)(gp, anc(B, name, 1500, int(g['t']), 2, float(g['curr_best'])))
  assert (pt == g['e2e_%s_point' % name]).all()


def test_c1_hallucinated(B, c1):
  g, gp = c1
  mu_h, sd_h = gp.eval_with_hallucinated_observations(g['C'][:800], list(g['Xh']), 'std')
  close(mu_h, g['mu_h'], atol=MU_TOL)
  close(sd_h ** 2, g['sd_h'] ** 2, atol=VAR_TOL)
  np.random.seed(7)
  pt = B.acq.asy.ucb(gp, anc(B, 'ucb', 1000, int(g['t']), 2, float(g['curr_best']),
                            in_progress=list(g['Xh'])))
  assert (pt == g['e2e_h_point']).all()


def test_c1_copies_share_the_posterior(c1):
  from copy import copy, deepcopy
  g, gp = c1
  for cp in (copy(gp), deepcopy(gp)):
    mu, _ = cp.eval(g['C'][:32], 'std')
    close(mu, g['mu'][:32], atol=MU_TOL)


def test_c1_chunking_is_invisible(B, c1):
  """ Ragged multi-chunk scoring (chunk = 128 rows) equals single-chunk scoring bit for bit. """
  g, gp = c1
  post = B.device.DevicePosterior(len(g['X']), chunk=128)
  post.set_kernel(B.kernel.build_descriptor(gp.kernel))
  y_c = np.asarray(g['Y']) - float(g['mean_const'])
  post.set_train(g['X'], y_c)
  info, lml = post.build(float(g['noise_var']))
  assert info == 0
  close(lml, g['lml'], rtol=1e-11)
  C = g['C'][:1003]
  mu, sd = post.eval(C, mean_const=float(g['mean_const']))
  mu_ref, sd_ref = gp.eval(C, 'std')
  assert (mu == mu_ref).all() and (sd == sd_ref).all()
  acq = B.device.make_acq_desc('ei', best=float(g['curr_best']))
  b1, i1, _ = post.score_argmax(acq, C, mean_const=float(g['mean_const']))
  b2, i2, _ = gp._fused_score(acq, C)
  assert i1 == i2 and b1 == b2


# ---- Hartmann-6 Matern, N = 300 -------------------------------------------------------------------------------
@pytest.mark.parametrize('nu', [0.5, 1.5, 2.5])
def test_matern_h6(B, nu):
  g = load_golden('matern_h6')
  tag = str(nu).replace('.', 'p')
  kern = B.kernel.MaternKernel(6, nu, float(g['scale']), g['bws'])
  gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(float(g['mean_const'])), float(g['noise_var']))
  close(gp.alpha, g['alpha_' + tag], rtol=1e-8, atol=1e-9)
  close(np.diag(gp.L), g['Ldiag_' + tag], rtol=1e-10)
  close(gp.L[::7, ::5], g['Lsub_' + tag], rtol=1e-8, atol=1e-11)
  close(gp.K_trtr_wo_noise[::7, ::5], g['Ksub_' + tag], atol=1e-13)
  close(gp.compute_log_marginal_likelihood(), g['lml_' + tag], rtol=1e-11)
  close(kern(g['C'][:64], g['X']), g['Kstar_sub_' + tag], atol=1e-13)
  mu, sd = gp.eval(g['C'], 'std')
  close(mu, g['mu_' + tag], atol=MU_TOL)
  close(sd ** 2, g['sd_' + tag] ** 2, atol=VAR_TOL)
  beta = B.acq._get_ucb_beta_th(6, int(g['t']))
  assert beta == float(g['beta'])
  _, i_ucb, s_ucb = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), g['C'], want_scores=True)
  _, i_ei, s_ei = gp._fused_score(B.device.make_acq_desc('ei', best=float(g['curr_best'])), g['C'],
                                  want_scores=True)
  assert i_ucb == int(g['argmax_ucb_' + tag])
  assert i_ei == int(g['argmax_ei_' + tag])
  close(s_ucb, g['ucb_' + tag], atol=1e-8)
  close(s_ei, g['ei_' + tag], rtol=1e-6, atol=1e-10)


# ---- additive GP + Add-UCB ---------------------------------------------------------------------------------------
def test_additive_and_add_ucb(B):
  g = load_golden('additive')
  groups = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
  sub = [B.kernel.MaternKernel(4, 2.5, 1.0, [0.5] * 4), B.kernel.SEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7]),
         B.kernel.MaternKernel(2, 1.5, 1.0, [0.3, 0.45])]
  kern = B.kernel.AdditiveKernel(float(g['scale']), sub, groups)
  gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(float(g['mean_const'])), float(g['noise_var']))
  close(gp.alpha, g['alpha'], rtol=1e-8, atol=1e-9)
  close(gp.K_trtr_wo_noise[::5, ::3], g['Ksub'], atol=1e-12)
  close(gp.compute_log_marginal_likelihood(), g['lml'], rtol=1e-11)
  mu, sd = gp.eval(g['C'], 'std')
  close(mu, g['mu'], atol=MU_TOL); close(sd ** 2, g['sd'] ** 2, atol=VAR_TOL)
  for j in range(3):
    desc = gp._group_test_descriptor(kern, sub[j], groups[j], 10)
    beta_j = B.acq._get_add_ucb_beta_th(len(groups[j]), int(g['t']))
    _, idx, score = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta_j), g['Cj_%d' % j],
                                    test_desc=desc, mean_const=0.0, want_scores=True)
    close(score, g['score_j_%d' % j], atol=1e-8)
    assert idx == int(g['argmax_j_%d' % j])
  # after the per-group calls the GP's own kernel is restored
  mu2, _ = gp.eval(g['C'][:50], 'std')
  close(mu2, g['mu'][:50], atol=MU_TOL)
  np.random.seed(11)
  pt = B.acq.asy.add_ucb(gp, anc(B, 'add_ucb', 900, int(g['t']), 10, float(g['Y'].max())))
  assert (pt == g['e2e_point']).all()


# ---- multi-fidelity product kernel + the fidel_to_opt slice -----------------------------------------------------------
def test_mf_product_kernel_and_fidel_slice(B):
  g = load_golden('mf')
  kF = B.kernel.SEKernel(1, 1.0, [0.7]); kD = B.kernel.MaternKernel(4, 2.5, 1.0, [0.4] * 4)
  mfgp = B.mf_gp.EuclideanMFGP(list(g['Z']), list(g['Xd']), list(g['Y']), None, float(g['scale']), kF, kD,
                               const_mean(float(g['mean_const'])), float(g['noise_var']))
  close(mfgp.alpha, g['alpha'], rtol=1e-8, atol=1e-9)
  close(mfgp.compute_log_marginal_likelihood(), g['lml'], rtol=1e-11)
  mu, sd = mfgp.eval_at_fidel(list(g['Cz']), list(g['Cx']), uncert_form='std')
  close(mu, g['mu'], atol=MU_TOL); close(sd ** 2, g['sd'] ** 2, atol=VAR_TOL)
  boca_gp = B.acq._get_fidel_to_opt_gp(mfgp, g['f2o'])
  mu_f, sd_f = boca_gp.eval(g['Cx'], uncert_form='std')
  close(mu_f, g['mu_f'], atol=MU_TOL); close(sd_f ** 2, g['sd_f'] ** 2, atol=VAR_TOL)
  assert B.acq._get_gp_ucb_dim(boca_gp) == 4
  acq = B.device.make_acq_desc('ucb', beta=float(g['beta']))
  _, idx, score = boca_gp._fused_score(acq, g['Cx'], [], want_scores=True)
  close(score, g['ucb_f'], atol=1e-8)
  assert idx == int(g['argmax_ucb_f'])


# ---- jitter ladder -------------------------------------------------------------------------------------------------------
def test_jitter_ladder(B):
  g = load_golden('jitter')
  kern = B.kernel.SEKernel(3, float(g['scale']), g['bws'])
  import warnings
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(0.0), 0.0)
  assert gp.jitter_power == int(g['power'])
  close(gp.L, g['L'], rtol=1e-6, atol=1e-9)


def test_not_pd_reports_info(B):
  """ A singular matrix with no ladder: the device reports the LAPACK-style pivot index. """
  g = load_golden('jitter')
  post = B.device.DevicePosterior(len(g['X']))
  post.set_kernel(B.kernel.build_descriptor(B.kernel.SEKernel(3, float(g['scale']), g['bws'])))
  post.set_train(g['X'], g['Y'])
  info, lml = post.build(0.0)
  assert info > 0 and lml is None
  with pytest.raises(B.lib.DfbError):
    post.eval(g['C'])


# ---- the hyper-parameter grid objective -------------------------------------------------------------------------------------
def test_lml_grid(B):
  g = load_golden('lml_grid')
  X, Y = g['X'], g['Y']
  post = B.device.DevicePosterior(len(X))
  post.set_train(X, np.asarray(Y) - float(g['mean_const']))
  lmls = []
  for hp in g['hps']:
    kern = B.kernel.MaternKernel(6, 2.5, np.exp(hp[1]), np.exp(hp[2:]))
    post.set_kernel(B.kernel.build_descriptor(kern))
    info, lml = post.build(np.exp(hp[0]), 0.0, B.lib.DFB_BUILD_LML_ONLY)
    assert info == 0
    lmls.append(lml)
  close(lmls, g['lmls'], rtol=1e-10)


# ---- oracle comparison at larger N, and properties at the metric's N ---------------------------------------------------------
def _oracle_gp(w):
  from oracle import gp_oracle as O
  k = w['kernel']
  kern = O.OMaternKernel(k['dim'], k['nu'], k['scale'], k['dim_bandwidths'])
  return O, O.OGP(w['X'], w['Y'], kern, const_mean(w['mean_const']), w['noise_var'])


def test_against_oracle_n2000(B):
  """ BASELINE config 2 geometry (Hartmann-6, Matern-2.5, N = 2000) on a 600-candidate sample. """
  from dragonfly_b200 import synth_data
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_cand=600)
  O, ogp = _oracle_gp(w)
  k = w['kernel']
  gp = B.gp_core.GP(w['X'], w['Y'], B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                    const_mean(w['mean_const']), w['noise_var'])
  close(gp.compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-10)
  close(gp.alpha, ogp.alpha, rtol=1e-7, atol=1e-8)
  mu_o, var_o = O.eval_std_diag(ogp, w['candidates'])
  mu, sd = gp.eval(w['candidates'], 'std')
  close(mu, mu_o, atol=MU_TOL); close(sd ** 2, var_o, atol=VAR_TOL)
  beta = O.ucb_beta_th(6, 2000)
  _, idx, _ = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), w['candidates'])
  assert idx == O.np_argmax_first(O.acq_ucb(mu_o, np.sqrt(var_o), beta))


def test_properties_at_n5000(B):
  """ The metric's N (5000): properties that need no CPU reference --
      (i) at the training inputs mu + noise * alpha reproduces y (K alpha = y_c - noise alpha),
      (ii) 0 <= sigma^2 <= kss, (iii) sigma^2 at a training point is below the noise-limited bound,
      (iv) arg-max returned == arg-max of the returned scores, first index on ties,
      (v) duplicated candidates score identically. """
  from dragonfly_b200 import synth_data
  w = synth_data.make_workload('headline_hartmann6_matern_ei', n_cand=4000)
  k = w['kernel']
  gp = B.gp_core.GP(w['X'], w['Y'], B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                    const_mean(w['mean_const']), w['noise_var'])
  Xs = w['X'][:512]
  mu, sd = gp.eval(Xs, 'std')
  y_c = w['Y'][:512] - w['mean_const']
  close(mu - w['mean_const'] + w['noise_var'] * gp.alpha[:512], y_c, atol=1e-9)
  assert (sd ** 2 <= w['noise_var'] * 1.0000001).all() and (sd ** 2 >= 0).all()
  C = np.concatenate((w['candidates'], w['candidates'][:100]), axis=0)
  acq = B.device.make_acq_desc('ei', best=float(w['Y'].max()))
  best, idx, scores = gp._fused_score(acq, C, want_scores=True)
  assert idx == int(np.argmax(scores)) and best == scores[idx]
  assert (scores[-100:] == scores[:100]).all()
  mu_c, sd_c = gp.eval(C, 'std')
  assert (sd_c ** 2 <= k['scale'] * (1 + 1e-12)).all() and (sd_c ** 2 >= 0).all()


# ---- TTEI, synchronous batches, full covariance, Thompson sampling end to end -----------------------------
@pytest.fixture(scope='module')
def extra_c1(B):
  g = load_golden('extra_c1')
  kern = B.kernel.SEKernel(2, float(g['scale']), g['bws'])
  gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(float(g['mean_const'])), float(g['noise_var']))
  return g, gp


@pytest.mark.parametrize('branch', ['ei', 'tt'])
def test_ttei_end_to_end(B, extra_c1, branch):
  """ asy_ttei: coin flip, EI arg-max as the reference arm, second maximisation (:269-294). """
  g, gp = extra_c1
  np.random.seed(int(g['ttei_%s_seed' % branch]))
  pt = B.acq.asy.ttei(gp, anc(B, 'ttei', 1200, int(g['t']), 2, float(g['curr_best'])))
  assert (pt == g['ttei_%s_point' % branch]).all()


@pytest.mark.parametrize('name', ['ucb', 'ei'])
def test_synchronous_batch(B, extra_c1, name):
  """ syn_<acq>: worker k scores against the GP hallucinated with picks 0..k-1 (:90-115). """
  g, gp = extra_c1
  np.random.seed(21)
  pts = getattr(B.acq.syn, name)(3, gp, anc(B, name, 800, int(g['t']), 2, float(g['curr_best'])))
  assert (np.array(pts) == g['syn_%s_points' % name]).all()


def test_eval_covar(B, extra_c1):
  g, gp = extra_c1
  mu, covar = gp.eval(g['C'][:96], 'covar')
  close(mu, g['covar_mu'], atol=MU_TOL)
  close(covar, g['covar'], atol=VAR_TOL)
  assert covar.shape == (96, 96)
  mu_s, sd = gp.eval(g['C'][:96], 'std')
  close(sd ** 2, np.diag(covar), rtol=1e-11, atol=1e-12)


def test_thompson_end_to_end(B, extra_c1):
  """ asy_ts: one joint posterior draw over all candidates (M x M covariance, stable_cholesky,
      normals from the global RNG), arg-max of the draw -- identical point to the reference. """
  g, gp = extra_c1
  np.random.seed(4)
  pt = B.acq.asy.ts(gp, anc(B, 'ts', 700, int(g['t']), 2, float(g['curr_best'])))
  assert (pt == g['ts_point']).all()
  np.random.seed(4)
  pt = B.acq.asy.ts(gp, anc(B, 'ts', 500, int(g['t']), 2, float(g['curr_best']),
                           in_progress=list(g['C'][:2])))
  assert (pt == g['ts_point_halluc']).all()


def test_thompson_draws_with_supplied_normals(B):
  """ gp.draw_samples against the reference's samples for the same normal matrix (golden ts.npz):
      the global RNG is re-seeded so np.random.normal hands out the recorded U. """
  g = load_golden('ts')
  kern = B.kernel.MaternKernel(20, 2.5, float(g['scale']), g['bws'])
  gp = B.gp_core.GP(g['X'], g['Y'], kern, const_mean(float(g['mean_const'])), float(g['noise_var']))
  np.random.seed(2)
  samples = gp.draw_samples(8, g['C'])
  assert samples.shape == (8, 256)
  close(samples, g['samples'], atol=2e-6)      # L_post of a near-singular covariance: cond * eps
  assert (samples.argmax(axis=1) == g['argmax']).all()
  mu, covar = gp.eval(g['C'], 'covar')
  close(mu, g['mu'], atol=MU_TOL)
  close(np.diag(covar), g['covar_diag'], atol=VAR_TOL)


# ---- BOCA (multi-fidelity selection) ------------------------------------------------------------------------------
def _mf_anc(B, acq, g, coeff, dx=4):
  a = anc(B, acq, 600, 150, dx, float(g['Y'].max()), boca_thresh_coeff=coeff,
          y_range=float(g['Y'].max() - g['Y'].min()), boca_max_low_fidel_cost_ratio=0.9)
  a.is_mf = True
  a.eval_fidel_points_in_progress = []
  return a


def test_boca(B):
  import os, sys
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
  from fake_mf_caller import FakeMFCaller
  g = load_golden('extra_mf')
  kF = B.kernel.SEKernel(1, 1.0, [0.7]); kD = B.kernel.MaternKernel(4, 2.5, 1.0, [0.4] * 4)
  mfgp = B.mf_gp.EuclideanMFGP(list(g['Z']), list(g['Xd']), list(g['Y']), None, float(g['scale']), kF, kD,
                               const_mean(float(g['mean_const'])), float(g['noise_var']))
  caller = FakeMFCaller([1.0])
  for coeff in [1e-4, 0.5]:
    tag = str(coeff).replace('.', 'p').replace('-', 'm')
    np.random.seed(8)
    fid, pt = B.acq.boca(B.acq.asy.ucb, mfgp, _mf_anc(B, 'ucb', g, coeff), caller)
    assert (pt == g['boca_point_%s' % tag]).all()
    assert (np.asarray(fid, dtype=np.float64) == g['boca_fidel_%s' % tag]).all()


def test_add_ucb_for_boca(B):
  import os, sys
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
  from fake_mf_caller import FakeMFCaller
  g = load_golden('extra_mf')
  kF = B.kernel.SEKernel(1, 1.0, [0.7])
  kDa = B.kernel.AdditiveKernel(1.0, [B.kernel.MaternKernel(2, 2.5, 1.0, [0.4, 0.5]),
                                      B.kernel.SEKernel(2, 1.0, [0.3, 0.6])], [[0, 1], [2, 3]])
  mfgp = B.mf_gp.EuclideanMFGP(list(g['Z']), list(g['Xd']), list(g['Y']), None, float(g['scale']) / 2, kF,
                               kDa, const_mean(float(g['mean_const'])), float(g['noise_var']))
  close(mfgp.alpha, g['alpha_add'], rtol=1e-8, atol=1e-9)
  np.random.seed(9)
  fid, pt = B.acq.boca(None, mfgp, _mf_anc(B, 'add_ucb', g, 1e-4), FakeMFCaller([1.0]))
  assert (pt == g['boca_add_point']).all()
  assert (np.asarray(fid, dtype=np.float64) == g['boca_add_fidel']).all()


def test_hp_grid_through_the_fitter_layout(B):
  """ GPFitter's objective (gp_core.py:551-563) for hp vectors laid out as build_gp /
      _child_build_gp unpack them; rand_exp_sampling weights (gp_core.py:443-444). """
  from dragonfly_b200 import hp_grid
  g = load_golden('lml_grid')
  layout = hp_grid.EuclideanHPLayout(6, 'matern', nu=2.5, mean_func_type='median', noise_var_type='tune')
  assert layout.num_hps() == 8
  lmls, post = hp_grid.lml_for_hyperparams(g['X'], g['Y'], g['hps'], layout)
  close(lmls, g['lmls'], rtol=1e-10)
  probs = hp_grid.rand_exp_sampling_probs(lmls)
  want = np.exp(g['lmls'] - g['lmls'].max()); want /= want.sum()
  close(probs, want, rtol=1e-7, atol=1e-12)
  lmls2, _ = hp_grid.sharded_lml_grid(g['X'], g['Y'], g['hps'][:3], layout)   # no process group: local
  close(lmls2, g['lmls'][:3], rtol=1e-10)
  # concurrent lanes (one handle + stream + host thread each) give the very same values as one lane,
  # and the returned posterior re-uses its lanes
  hps = np.concatenate((g['hps'], g['hps'][::-1]), axis=0)
  one, _ = hp_grid.lml_for_hyperparams(g['X'], g['Y'], hps, layout, lanes=1)
  three, post3 = hp_grid.lml_for_hyperparams(g['X'], g['Y'], hps, layout, lanes=3)
  again, post3b = hp_grid.lml_for_hyperparams(g['X'], g['Y'], hps, layout, post=post3, lanes=3)
  assert (one == three).all() and (again == one).all() and post3b is post3 and len(post3._hp_lanes) == 2
  close(one[:len(g['hps'])], g['lmls'], rtol=1e-10)


def test_tma_kernel_matches_cp_async_kernel(B):
  """ The two implementations of the dominant contraction (cp.async ring vs TMA + mbarrier ring)
      contract the same k-ranges in a different lane order: sigma^2 agrees to rounding, arg-max
      identical -- on a ragged multi-chunk shape with several row blocks. """
  from dragonfly_b200 import synth_data
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=700, n_cand=3000)
  k = w['kernel']
  res = []
  for impl in (0, 1):
    post = B.device.DevicePosterior(700, chunk=1024)
    post.set_option('gemm_impl', impl)
    post.set_kernel(B.kernel.build_descriptor(B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])))
    post.set_train(w['X'], w['Y'] - w['mean_const'])
    info, lml = post.build(w['noise_var'])
    assert info == 0
    mu, sd = post.eval(w['candidates'], mean_const=w['mean_const'])
    acq = B.device.make_acq_desc('ucb', beta=2.0)
    res.append((mu, sd, post.score_argmax(acq, w['candidates'], mean_const=w['mean_const'])[:2]))
  assert (res[0][0] == res[1][0]).all()
  close(res[0][1] ** 2, res[1][1] ** 2, atol=1e-13)
  assert res[0][2][1] == res[1][2][1]


# ---- the int8-slice wgmma contraction (score_impl 1 / auto) ------------------------------------------------
def _post_pair(B, kern, X, Y, mean_const, noise_var, chunk=0, i8_impl=None, i8_radix=None):
  posts = []
  for impl in (0, 1):
    post = B.device.DevicePosterior(len(X), chunk=chunk)
    post.set_option('score_impl', impl)
    if i8_impl is not None:      # None: the library default (CTA-pair kernel)
      post.set_option('i8_impl', i8_impl)
    if i8_radix is not None:
      post.set_option('i8_radix', i8_radix)
    post.set_kernel(B.kernel.build_descriptor(kern, train_dim=X.shape[1], cand_dim=X.shape[1]))
    post.set_train(X, np.asarray(Y) - mean_const)
    info, _ = post.build(noise_var)
    assert info == 0
    posts.append(post)
  return posts


def _i8_kernels(B):
  add_groups = [[0, 1, 2], [3, 4, 5]]
  return {
    'se': B.kernel.SEKernel(6, 0.7, [0.3, 0.35, 0.4, 0.3, 0.5, 0.45]),
    'matern05': B.kernel.MaternKernel(6, 0.5, 0.7, 0.4),
    'matern15': B.kernel.MaternKernel(6, 1.5, 0.7, 0.4),
    'matern25': B.kernel.MaternKernel(6, 2.5, 0.7, 0.3),
    'additive': B.kernel.AdditiveKernel(0.35, [B.kernel.MaternKernel(3, 2.5, 1.0, 0.5),
                                               B.kernel.SEKernel(3, 1.0, 0.4)], add_groups),
    'mf_product': B.kernel.CoordinateProductKernel(6, 0.7, [B.kernel.SEKernel(1, 1.0, [0.7]),
                                                             B.kernel.MaternKernel(5, 2.5, 1.0, 0.4)],
                                                   [[0], [1, 2, 3, 4, 5]]),
  }


@pytest.mark.parametrize('i8_impl,i8_radix', [(0, None), (1, None), (2, 0), (2, 1), (2, -1)])
@pytest.mark.parametrize('name', ['se', 'matern05', 'matern15', 'matern25', 'additive', 'mf_product'])
def test_i8_sigma2_within_contract(B, name, i8_impl, i8_radix):
  """ Digit-sliced tensor-core contraction vs fp64 DMMA on the same posterior: mu identical (it never
      leaves fp64), |d sigma^2| far inside the 1e-8 contract and inside the library's own a-priori
      bound, for every kernel family, over several row blocks and ragged chunks; for every i8_impl setting and
      both digit schemes (forced, and as the library picks them). """
  from dragonfly_b200 import synth_data
  rs = np.random.RandomState(3)
  X = rs.random_sample((1100, 6)); Y = synth_data.hartmann6(X)
  C = rs.random_sample((5000, 6))
  kern = _i8_kernels(B)[name]
  fp, i8 = _post_pair(B, kern, X, Y, float(np.median(Y)), 0.01 * 0.7, chunk=2048, i8_impl=i8_impl,
                      i8_radix=i8_radix)
  assert i8.query('i8_ready') == 1.0
  radix256 = i8.query('i8_radix256') == 1.0
  assert radix256 == (i8_radix == 1) or i8_radix == -1
  mu0, sd0 = fp.eval(C, mean_const=1.0)
  mu1, sd1 = i8.eval(C, mean_const=1.0)
  bound = i8.query('i8_sigma2_bound')
  assert fp.query('last_used_i8') == 0.0
  if i8.query('last_used_i8') == 0.0:
    # only a forced radix 256 may be refused (its bound is above half the contract for this kernel): the
    # call then ran in fp64
    assert i8_radix == 1 and bound > 5e-9
    assert (sd0 == sd1).all()
    return
  # mu of the int8 pass comes from the digit-emitting K_* kernel (fused constants, per-segment partial sums): equal
  # to the exact-order fp64 path's to rounding, 100x inside the 1e-10 contract
  close(mu1, mu0, atol=1e-12)
  err = np.abs(sd0 ** 2 - sd1 ** 2).max()
  assert err <= (5e-9 if radix256 else 1e-9), err
  assert err <= bound
  # impl 0, 1 and radix-128 pairs tile the same 21 digit products: the same exact integers, so they agree
  # to the last bits of the fp64 recombination; the radix-256 expansion is a different, coarser one
  if i8_impl >= 1:
    _, ref = _post_pair(B, kern, X, Y, float(np.median(Y)), 0.01 * 0.7, chunk=2048, i8_impl=0)
    _, sd_ref = ref.eval(C, mean_const=1.0)
    close(sd1 ** 2, sd_ref ** 2, atol=2.0 * bound if radix256 else 1e-13)


def test_i8_against_reference_golden(B):
  """ Forced int8 path against the reference itself (golden matern_h6, N = 300). """
  g = load_golden('matern_h6')
  kern = B.kernel.MaternKernel(6, 2.5, float(g['scale']), g['bws'])
  _, i8 = _post_pair(B, kern, g['X'], g['Y'], float(g['mean_const']), float(g['noise_var']))
  mu, sd = i8.eval(g['C'], mean_const=float(g['mean_const']))
  assert i8.query('last_used_i8') == 1.0
  close(mu, g['mu_2p5'], atol=MU_TOL)
  close(sd ** 2, g['sd_2p5'] ** 2, atol=VAR_TOL)


@pytest.mark.parametrize('acq_name', ['ucb', 'ei', 'pi', 'ttei'])
def test_auto_mode_returns_the_fp64_argmax(B, acq_name):
  """ Default mode: int8 pass + exact fp64 re-score of the shortlist == pure fp64 result, bit for bit. """
  from dragonfly_b200 import synth_data
  rs = np.random.RandomState(5)
  X = rs.random_sample((1200, 6)); Y = synth_data.hartmann6(X)
  C = rs.random_sample((30000, 6))
  kern = B.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)
  m0 = float(np.median(Y))
  res = {}
  for impl in (0, 2):
    post = B.device.DevicePosterior(len(X), chunk=4096)
    post.set_option('score_impl', impl)
    post.set_kernel(B.kernel.build_descriptor(kern)); post.set_train(X, Y - m0)
    assert post.build(0.01 * float(Y.var()))[0] == 0
    acq = {'ucb': B.device.make_acq_desc('ucb', beta=3.0),
           'ei': B.device.make_acq_desc('ei', best=float(Y.max())),
           'pi': B.device.make_acq_desc('pi', best=float(Y.max())),
           'ttei': B.device.make_acq_desc('ttei', ref_mean=float(Y.max()) - 0.2, ref_std=0.1)}[acq_name]
    bs, bi, _ = post.score_argmax(acq, C, mean_const=m0)
    res[impl] = (bs, bi, post.query('last_used_i8'), post.query('last_shortlist'))
  assert res[0][2] == 0.0 and res[2][2] == 1.0
  assert 1 <= res[2][3] <= 4096
  assert res[0][1] == res[2][1] and res[0][0] == res[2][0]


def test_auto_mode_guard_and_overflow(B):
  """ (i) an ill-conditioned posterior (tiny noise) exceeds the a-priori int8 bound -> fp64 is used;
      (ii) a candidate set of exact ties overflows the shortlist -> full fp64 pass, first index wins. """
  from dragonfly_b200 import synth_data
  rs = np.random.RandomState(6)
  X = rs.random_sample((1100, 6)); Y = synth_data.hartmann6(X)
  kern = B.kernel.SEKernel(6, float(Y.var()), 0.6)
  post = B.device.DevicePosterior(len(X))
  post.set_kernel(B.kernel.build_descriptor(kern)); post.set_train(X, Y - float(np.median(Y)))
  info, _ = post.build(1e-9 * float(Y.var()), 1e-9 * float(Y.var()))
  assert info == 0
  acq = B.device.make_acq_desc('ucb', beta=2.0)
  C = rs.random_sample((3000, 6))
  post.score_argmax(acq, C)
  assert post.query('last_used_i8') == 0.0
  assert post.query('i8_sigma2_bound') > 1e-9
  post2 = B.device.DevicePosterior(len(X))
  post2.set_kernel(B.kernel.build_descriptor(B.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)))
  post2.set_train(X, Y - float(np.median(Y)))
  assert post2.build(0.01 * float(Y.var()))[0] == 0
  ties = np.repeat(C[:1], 6000, axis=0)
  bs, bi, _ = post2.score_argmax(acq, ties)
  assert post2.query('last_used_i8') == 1.0 and post2.query('last_shortlist') == -1.0
  assert bi == 0


def test_auto_mode_with_group_test_kernel_and_mf(B):
  """ The int8 pass also serves Add-UCB's per-group descriptor (dfb_set_test_kernel) and the MF product
      kernel: default mode == fp64 mode, bit for bit, at N >= 1024. """
  from dragonfly_b200 import synth_data
  rs = np.random.RandomState(11)
  n, d = 1100, 10
  X = rs.random_sample((n, d)); Y = synth_data.tiled(synth_data.park1, 4, X)
  Y = Y / Y.std()       # unit scale: the int8 screen's ABSOLUTE 5e-9 guard (api.cu: I8_BOUND_LIMIT) admits the path
  groups = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
  sub = [B.kernel.MaternKernel(4, 2.5, 1.0, 0.5), B.kernel.SEKernel(4, 1.0, 0.5), B.kernel.MaternKernel(2, 1.5, 1.0, 0.4)]
  kern = B.kernel.AdditiveKernel(float(Y.var()) / 3, sub, groups)
  pts = {}
  for impl in (0, 2):
    B.device.DEFAULT_OPTIONS['score_impl'] = impl
    try:
      gp = B.gp_core.GP(X, Y, kern, const_mean(float(np.median(Y))), 0.01 * float(Y.var()))
      np.random.seed(17)
      pts[impl] = B.acq.asy.add_ucb(gp, anc(B, 'add_ucb', 9000, n, d, float(Y.max())))
      used = gp._post.query('last_used_i8')
      assert used == (1.0 if impl == 2 else 0.0)
    finally:
      B.device.DEFAULT_OPTIONS.pop('score_impl', None)
  assert (pts[0] == pts[2]).all()


def test_thompson_blocks_at_scale(B):
  """ Several 4096-candidate blocks x 64 draws on an N = 1100 posterior: finite, right shape, and the
      first block equals a stand-alone draw with the same normals (blocks are independent). """
  from dragonfly_b200 import synth_data
  rs = np.random.RandomState(12)
  X = rs.random_sample((1100, 6)); Y = synth_data.hartmann6(X)
  gp = B.gp_core.GP(X, Y, B.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3), const_mean(float(np.median(Y))),
                    0.01 * float(Y.var()))
  C = rs.random_sample((9000, 6))
  np.random.seed(3)
  S = gp.draw_samples(64, C)
  assert S.shape == (64, 9000) and np.isfinite(S).all()
  np.random.seed(3)
  U = np.random.normal(size=(9000, 64))
  info, smp, _ = gp._post.ts_draws(C[:4096], np.ascontiguousarray(U[:4096].T), mean_const=gp._mean_const)
  assert info == 0
  close(S[:, :4096], smp.cpu().numpy(), atol=1e-9)
  mu, sd = gp.eval(C[:4096], 'std')
  # the draws scatter around the posterior mean with the posterior standard deviation
  zscore = (S[:, :4096] - mu) / sd
  assert abs(zscore.mean()) < 0.05 and 0.9 < zscore.std() < 1.1
