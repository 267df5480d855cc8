"""
Parity tests (-m gpu) of the incremental posterior update (SURVEY.md 8f rank 1): GP.add_data_multiple
and the hallucinated (N + q)-point posterior of eval_with_hallucinated_observations
(gp_core.py:139-146, 192-220).  The reference re-factorises from scratch in both places; the device
extends the built factorisation in place (dfb_extend_posterior) and must land on the same numbers
as the oracle's full rebuild: |d mu| <= 1e-10, |d sigma^2| <= 1e-8, arg-max index exact, LML rtol 1e-10.
"""
import time
from argparse import Namespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MU_TOL = 1e-10
VAR_TOL = 1e-8


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


def hartmann_case(B, n, n_cand=700, nu=2.5):
  w = B.synth.make_workload('c2_hartmann6_matern_ucb', n_train=n, n_cand=n_cand)
  k = w['kernel']
  mk = lambda: B.kernel.MaternKernel(6, nu, k['scale'], k['dim_bandwidths'])
  ok = lambda: B.O.OMaternKernel(6, nu, k['scale'], k['dim_bandwidths'])
  return w, mk, ok


def check_against_oracle(B, gp, ogp, C, t):
  O = B.O
  close(gp.compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-10)
  close(gp.alpha, ogp.alpha, rtol=1e-7, atol=1e-8)
  close(gp.L, ogp.L, rtol=1e-8, atol=1e-10)
  mu_o, var_o = O.eval_std_diag(ogp, C)
  mu, sd = gp.eval(C, 'std')
  close(mu, mu_o, atol=MU_TOL)
  close(sd ** 2, var_o, atol=VAR_TOL)
  beta = O.ucb_beta_th(6, t)
  _, idx, _ = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), C)
  assert idx == O.np_argmax_first(O.acq_ucb(mu_o, np.sqrt(var_o), beta))


# (n0, q, in_place): 1 row block (no left-looking products), several row blocks, a step that lands exactly on
# the padded size, one that crosses it (-> the reference's full rebuild), and a size where the int8 scoring
# path is active (n >= 1024: the digit planes of W must be re-sliced after the extension).
CASES = [(50, 3, True), (300, 7, True), (380, 4, True), (250, 9, False), (1030, 20, True)]


@pytest.mark.parametrize('n0,q,in_place', CASES)
def test_add_data_multiple_extends_the_factorisation(B, n0, q, in_place):
  w, mk, ok = hartmann_case(B, n0 + q)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  mean = B.gp_core.ConstantMean(m0)
  gp = B.gp_core.GP(X[:n0], Y[:n0], mk(), mean, nv)
  post_before = gp._post
  L_before = gp.L.copy()
  gp.add_data_multiple(list(X[n0:]), list(Y[n0:]))
  assert gp.num_tr_data == n0 + q and len(gp.X) == n0 + q
  assert (gp._post is post_before) == in_place
  ogp = B.O.OGP(X, Y, ok(), const_mean(m0), nv)
  check_against_oracle(B, gp, ogp, w['candidates'], n0 + q)
  # rows of L above the first appended point are untouched by an extension outside the last row block
  lo = (n0 // 128) * 128
  if in_place and lo > 0:
    assert (gp.L[:lo, :lo] == L_before[:lo, :lo]).all()
  # the device's own full rebuild agrees far below the contract
  ref = B.gp_core.GP(X, Y, mk(), mean, nv)
  mu_i, sd_i = gp.eval(w['candidates'], 'std')
  mu_f, sd_f = ref.eval(w['candidates'], 'std')
  close(mu_i, mu_f, atol=1e-11)
  close(sd_i ** 2, sd_f ** 2, atol=1e-10)


def test_add_data_single_repeatedly_and_switch(B):
  """ One observation at a time (the BO loop's pattern), then with the feature switched off. """
  n0, q = 200, 5
  w, mk, ok = hartmann_case(B, n0 + q, nu=1.5)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  gp = B.gp_core.GP(X[:n0], Y[:n0], mk(), B.gp_core.ConstantMean(m0), nv)
  post = gp._post
  for i in range(n0, n0 + q):
    gp.add_data_single(X[i], Y[i])
    assert gp._post is post
  ogp = B.O.OGP(X, Y, ok(), const_mean(m0), nv)
  check_against_oracle(B, gp, ogp, w['candidates'], n0 + q)
  gp2 = B.gp_core.GP(X[:n0], Y[:n0], mk(), B.gp_core.ConstantMean(m0), nv)
  gp2.incremental_updates = False
  post2 = gp2._post
  gp2.add_data_multiple(list(X[n0:]), list(Y[n0:]))
  assert gp2._post is not post2
  check_against_oracle(B, gp2, ogp, w['candidates'], n0 + q)


def test_copies_never_see_an_extension(B):
  """ copy()/deepcopy() share the device posterior (gpb_acquisitions.py:104): adding data to one copy
      must rebuild into a fresh posterior and leave the other untouched. """
  from copy import copy
  n0, q = 150, 4
  w, mk, ok = hartmann_case(B, n0 + q)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  gp = B.gp_core.GP(X[:n0], Y[:n0], mk(), B.gp_core.ConstantMean(m0), nv)
  twin = copy(gp)
  twin.X, twin.Y = list(gp.X), list(gp.Y)
  mu0, sd0 = gp.eval(w['candidates'], 'std')
  twin.add_data_multiple(list(X[n0:]), list(Y[n0:]))
  assert twin._post is not gp._post
  mu1, sd1 = gp.eval(w['candidates'], 'std')
  assert (mu0 == mu1).all() and (sd0 == sd1).all() and gp.num_tr_data == n0
  ogp = B.O.OGP(X, Y, ok(), const_mean(m0), nv)
  check_against_oracle(B, twin, ogp, w['candidates'], n0 + q)


def test_kernel_change_forces_a_rebuild(B):
  n0, q = 150, 4
  w, mk, ok = hartmann_case(B, n0 + q)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  gp = B.gp_core.GP(X[:n0], Y[:n0], mk(), B.gp_core.ConstantMean(m0), nv)
  post = gp._post
  gp.kernel = B.kernel.MaternKernel(6, 2.5, w['kernel']['scale'] * 1.3, [0.4] * 6)
  gp.add_data_multiple(list(X[n0:]), list(Y[n0:]))
  assert gp._post is not post
  ogp = B.O.OGP(X, Y, B.O.OMaternKernel(6, 2.5, w['kernel']['scale'] * 1.3, [0.4] * 6), const_mean(m0), nv)
  check_against_oracle(B, gp, ogp, w['candidates'], n0 + q)


@pytest.mark.parametrize('n0,q', [(300, 3), (1030, 5)])
def test_hallucinations_extend_in_place_and_restore_bit_for_bit(B, n0, q, monkeypatch):
  w, mk, ok = hartmann_case(B, n0, n_cand=900)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  C = w['candidates']
  Xh = list(np.random.RandomState(5).random_sample((q, 6)))
  gp = B.gp_core.GP(X, Y, mk(), B.gp_core.ConstantMean(m0), nv)
  ogp = B.O.OGP(X, Y, ok(), const_mean(m0), nv)
  mu0, sd0 = gp.eval(C, 'std')
  L0, a0 = gp.L.copy(), gp.alpha.copy()
  lml0 = gp.compute_log_marginal_likelihood()
  # the in-place path must be the one that runs: a fresh (N + q) build is a test failure here
  def boom(*a, **k):
    raise AssertionError('fell back to a fresh (N + q)-point build')
  monkeypatch.setattr(gp, '_augmented_posterior', boom)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C, Xh, 'std')
  mu_o, sd_o = ogp.eval_with_hallucinated_observations(C, Xh, 'std')
  close(mu_h, mu_o, atol=MU_TOL)
  close(sd_h ** 2, sd_o ** 2, atol=VAR_TOL)
  assert (mu_h == mu0).all()                # the mean comes from the un-augmented GP (gp_core.py:196)
  assert (sd_h <= sd0 + 1e-12).all()        # conditioning on more points never raises the variance
  # fused acquisition + arg-max against the hallucinated posterior
  beta = B.O.ucb_beta_th(6, n0)
  _, idx, _ = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), C, halluc=Xh)
  assert idx == B.O.np_argmax_first(B.O.acq_ucb(mu_o, sd_o, beta))
  # and everything is back, bit for bit
  gp._cache = {}
  mu1, sd1 = gp.eval(C, 'std')
  assert (mu1 == mu0).all() and (sd1 == sd0).all()
  assert (gp.L == L0).all() and (gp.alpha == a0).all()
  assert gp.compute_log_marginal_likelihood() == lml0 and gp._post.n == n0
  _, idx_plain, _ = gp._fused_score(B.device.make_acq_desc('ucb', beta=beta), C)
  mu_p, var_p = B.O.eval_std_diag(ogp, C)
  assert idx_plain == B.O.np_argmax_first(B.O.acq_ucb(mu_p, np.sqrt(var_p), beta))


def test_hallucinations_that_do_not_fit_build_fresh(B):
  """ 250 + 9 points cross the padded size 256: the reference's fresh (N + q)-point build is used. """
  n0, q = 250, 9
  w, mk, ok = hartmann_case(B, n0, n_cand=500)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  Xh = list(np.random.RandomState(6).random_sample((q, 6)))
  gp = B.gp_core.GP(X, Y, mk(), B.gp_core.ConstantMean(m0), nv)
  ogp = B.O.OGP(X, Y, ok(), const_mean(m0), nv)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(w['candidates'], Xh, 'std')
  mu_o, sd_o = ogp.eval_with_hallucinated_observations(w['candidates'], Xh, 'std')
  close(mu_h, mu_o, atol=MU_TOL)
  close(sd_h ** 2, sd_o ** 2, atol=VAR_TOL)


def test_synchronous_batch_through_the_in_place_path(B):
  """ _get_syn_recommendations_from_asy (gpb_acquisitions.py:90-115): worker k sees k-1 hallucinations;
      with in-place extensions the picks equal those of fresh (N + k)-point builds. """
  n0 = 120
  w, mk, ok = hartmann_case(B, n0, n_cand=10)
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  dom = B.domains.EuclideanDomain([[0, 1]] * 6)

  def run(incremental):
    gp = B.gp_core.GP(X, Y, mk(), B.gp_core.ConstantMean(m0), nv)
    gp.incremental_updates = incremental
    a = Namespace(curr_acq='ucb', max_evals=800, t=n0, domain=dom, curr_max_val=float(Y.max()),
                  eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc',
                  mf_strategy=None, is_mf=False, domain_bounds=np.array(dom.bounds))
    np.random.seed(11)
    return B.acq.syn.ucb(3, gp, a)

  pts_inc, pts_full = run(True), run(False)
  assert len(pts_inc) == 3
  for p, r in zip(pts_inc, pts_full):
    assert (np.asarray(p) == np.asarray(r)).all()


def test_cabi_errors(B):
  n0 = 130
  w, mk, ok = hartmann_case(B, n0, n_cand=10)
  gp = B.gp_core.GP(w['X'], w['Y'], mk(), B.gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  post = gp._post
  assert post.capacity() == 256
  with pytest.raises(B.lib.DfbError):
    post.extend(np.zeros((127, 6)), np.zeros(127))           # 130 + 127 > 256
  with pytest.raises(B.lib.DfbError):
    post.restore(n0)                                          # nothing saved
  info, _ = post.extend(np.random.RandomState(1).random_sample((2, 6)), np.zeros(2),
                        B.lib.DFB_BUILD_NO_ALPHA, save=True)
  assert info == 0
  with pytest.raises(B.lib.DfbError):
    post.extend(np.zeros((1, 6)) + 0.5, np.zeros(1), save=True)   # a saved extension is active
  post.restore(n0)
  # Not positive definite -> info > 0 and, with save=True, the un-extended posterior is back.  With
  # K ~ I (tiny bandwidths) and "noise" -0.9 the matrix 0.1 I is PD, but appending a duplicate of x_0 gives
  # the Schur complement 0.1 - 1 / 0.1 < 0.
  X = w['X'][:100]
  raw = B.device.DevicePosterior(100)
  raw.set_kernel(B.kernel.build_descriptor(B.kernel.SEKernel(6, 1.0, [0.02] * 6)))
  raw.set_train(X, np.zeros(100) + 0.5)
  info, _ = raw.build(-0.9)
  assert info == 0
  mu0, sd0 = raw.eval(w['candidates'], mean_const=0.0)
  info, _ = raw.extend(X[:1], np.zeros(1), B.lib.DFB_BUILD_FULL, save=True)
  assert info > 0 and raw.n == 100
  mu1, sd1 = raw.eval(w['candidates'], mean_const=0.0)
  assert (mu0 == mu1).all() and (sd0 == sd1).all()
  info, _ = raw.extend(X[:1], np.zeros(1), B.lib.DFB_BUILD_FULL)     # no snapshot: posterior is gone
  assert info > 0
  with pytest.raises(B.lib.DfbError):
    raw.eval(w['candidates'], mean_const=0.0)


def test_extension_at_the_metric_n(B):
  """ N = 4993 -> 5000 (the metric's N; 4993 is the first size whose padded size is 5120): the extended
      posterior against the device's own full build, and the wall-clock of both. """
  n0, q = 4993, 7
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_train=n0 + q, n_cand=3000)
  k = w['kernel']
  mk = lambda: B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])
  X, Y, m0, nv = w['X'], w['Y'], w['mean_const'], w['noise_var']
  mean = B.gp_core.ConstantMean(m0)
  gp = B.gp_core.GP(X[:n0], Y[:n0], mk(), mean, nv)
  post = gp._post
  B.torch.cuda.synchronize()
  t0 = time.perf_counter()
  gp.add_data_multiple(list(X[n0:]), list(Y[n0:]))
  B.torch.cuda.synchronize()
  t_ext = time.perf_counter() - t0
  assert gp._post is post
  t0 = time.perf_counter()
  ref = B.gp_core.GP(X, Y, mk(), mean, nv)
  B.torch.cuda.synchronize()
  t_full = time.perf_counter() - t0
  print('N=5000: extend by 7 points %.2f ms, full build %.2f ms' % (1e3 * t_ext, 1e3 * t_full))
  close(gp.compute_log_marginal_likelihood(), ref.compute_log_marginal_likelihood(), rtol=1e-11)
  C = w['candidates']
  mu_i, sd_i = gp.eval(C, 'std')
  mu_f, sd_f = ref.eval(C, 'std')
  close(mu_i, mu_f, atol=MU_TOL)
  close(sd_i ** 2, sd_f ** 2, atol=VAR_TOL)
  acq = B.device.make_acq_desc('ei', best=float(Y.max()))
  b_i, i_i, _ = gp._fused_score(acq, C)
  b_f, i_f, _ = ref._fused_score(acq, C)
  assert i_i == i_f
  # K alpha + noise alpha = y_c at the appended points
  mu_t, _ = gp.eval(X[n0:], 'none')
  close(mu_t - m0 + nv * gp.alpha[n0:], Y[n0:] - m0, atol=1e-9)


def test_add_data_against_the_reference_golden(B):
  """ tests/golden/incremental.npz: the UNMODIFIED reference after add_data_multiple + 2 x add_data_single
      (it rebuilds three times); the device extends in place three times. """
  from conftest import load_golden
  g = load_golden('incremental')
  n0 = int(g['n0'])
  gp = B.gp_core.GP(g['X'][:n0], g['Y'][:n0], B.kernel.MaternKernel(6, 2.5, float(g['scale']), g['bws']),
                    B.gp_core.ConstantMean(float(g['mean_const'])), float(g['noise_var']))
  post = gp._post
  gp.add_data_multiple(list(g['X'][n0:n0 + 4]), list(g['Y'][n0:n0 + 4]))
  gp.add_data_single(g['X'][n0 + 4], g['Y'][n0 + 4])
  gp.add_data_single(g['X'][n0 + 5], g['Y'][n0 + 5])
  assert gp._post is post and gp.num_tr_data == n0 + 6
  close(gp.L, g['L'], rtol=1e-8, atol=1e-10)
  close(gp.alpha, g['alpha'], rtol=1e-7, atol=1e-8)
  close(gp.compute_log_marginal_likelihood(), g['lml'], rtol=1e-10)
  mu, sd = gp.eval(g['C'], 'std')
  close(mu, g['mu'], atol=MU_TOL)
  close(sd ** 2, g['sd'] ** 2, atol=VAR_TOL)
