"""
Poly and ExpDecay kernels on the device (-m gpu): the descriptor interpreter's POLY and EXPDECAY factors against
fixtures recorded from the unmodified reference (golden nonstat.npz, fitter_expdecay.npz) and against the NumPy oracle
(tests/nonstat_ref.py).  Non-stationary kernels score on fp64 DMMA only: neither the int8 screen nor the bound pass
may run for them.
"""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
from oracle import gp_oracle as O
import nonstat_ref as R

pytestmark = pytest.mark.gpu

MU_TOL = 1e-10
VAR_TOL = 1e-8


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, mf_gp, gpb_acquisitions, domains, device, _lib
  _lib.load()
  return Namespace(kernel=kernel, gp_core=gp_core, mf_gp=mf_gp, acq=gpb_acquisitions, domains=domains, device=device,
                   lib=_lib, torch=torch)


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def anc(G, acq, max_evals, t, d, curr_max, **kw):
  dom = G.domains.EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq=acq, max_evals=max_evals, t=t, domain=dom, curr_max_val=curr_max,
                   eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                   is_mf=False, domain_bounds=np.array(dom.bounds), **kw)


def test_kernel_blocks_against_the_reference(G):
  """ Kernel.__call__ on the device: Poly to rtol 1e-13 (the reference's dot products are a dgemm), ExpDecay to 1e-14
      (the last ulps of pow), the Cartesian product of an ExpDecay and a Matern kernel to 1e-13. """
  from dragonfly_b200 import cartesian_product_gp as cp
  g = load_golden('nonstat')
  for d in (1, 2, 4, 8):
    for order in (1, 2, 3, 5):
      k = G.kernel.PolyKernel(d, order, 0.8, g['poly_scal_%d' % d])
      np.testing.assert_allclose(k(g['poly_X1_%d_%d' % (d, order)], g['poly_X2_%d_%d' % (d, order)]),
                                 g['poly_K_%d_%d' % (d, order)], rtol=1e-13, atol=0)
  for i in range(4):
    d, scale, offset = g['ed_meta_%d' % i]
    pw = g['ed_powers_%d' % i]
    k = G.kernel.ExpDecayKernel(int(d), scale, offset, list(pw) if pw.ndim else float(pw))
    np.testing.assert_allclose(k(g['ed_X1_%d' % i], g['ed_X2_%d' % i]), g['ed_K_%d' % i], rtol=1e-14, atol=0)
  kern = cp.CartesianProductKernel(1.4, [G.kernel.ExpDecayKernel(1, 1.0, 0.15, [2.0]),
                                         G.kernel.MaternKernel(3, 2.5, 1.0, [0.5, 0.7, 0.9])])
  np.testing.assert_allclose(kern(g['cp_X1'], g['cp_X2']), g['cp_K'], rtol=1e-13, atol=0)


def _mfgp(G, g, n=None):
  n = len(g['mf_Y']) if n is None else n
  kF = G.kernel.ExpDecayKernel(1, 1.0, float(g['mf_offset']), list(g['mf_powers']))
  kD = G.kernel.MaternKernel(4, 2.5, 1.0, list(g['mf_bws']))
  return G.mf_gp.EuclideanMFGP(list(g['mf_Z'][:n]), list(g['mf_Xd'][:n]), list(g['mf_Y'][:n]), None,
                               float(g['mf_scale']), kF, kD, const_mean(float(g['mf_mean'])), float(g['mf_noise']))


@pytest.fixture(scope='module')
def mf(G):
  g = load_golden('nonstat')
  return g, _mfgp(G, g)


def test_mf_posterior_against_the_reference(G, mf):
  g, gp = mf
  np.testing.assert_allclose(np.asarray(gp.L)[:16], g['mf_L_rows'], rtol=0, atol=1e-8)
  np.testing.assert_allclose(np.asarray(gp.alpha), g['mf_alpha'], rtol=0, atol=1e-8)
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g['mf_lml']), rtol=1e-10)
  for fz in (0.2, 0.6, 1.0):
    tag = ('%g' % fz).replace('.', 'p')
    mu, sd = gp.eval_at_fidel([np.array([fz])] * len(g['mf_Cx']), list(g['mf_Cx']), uncert_form='std')
    np.testing.assert_allclose(mu, g['mf_mu_' + tag], rtol=0, atol=MU_TOL)
    np.testing.assert_allclose(sd ** 2, g['mf_sd_' + tag] ** 2, rtol=0, atol=VAR_TOL)
  mu_h, sd_h = gp.eval_at_fidel_with_hallucinated_observations(
      [np.array([1.0])] * 200, list(g['mf_Cx'][:200]), list(g['mf_Zh']), list(g['mf_Xh']), uncert_form='std')
  np.testing.assert_allclose(mu_h, g['mf_mu_h'], rtol=0, atol=MU_TOL)
  np.testing.assert_allclose(sd_h ** 2, g['mf_sd_h'] ** 2, rtol=0, atol=VAR_TOL)


def test_max_diag_is_the_largest_diagonal_entry(G, mf):
  """ The jitter ladder's scale max(diag(K) + noise I) (general_utils.py:184) depends on the data for these kernels. """
  g, gp = mf
  want = float(np.max(g['mf_Kdiag'] + float(g['mf_noise'])))
  np.testing.assert_allclose(gp._post.max_diag(), want, rtol=1e-14)


@pytest.mark.parametrize('name', ['ucb', 'ei'])
def test_mf_acquisition_points_on_the_fidel_to_opt_slice(G, mf, name):
  g, gp = mf
  np.random.seed(7)
  f2o_gp = G.acq._get_fidel_to_opt_gp(gp, np.array([1.0]))
  pt = getattr(G.acq.asy, name)(f2o_gp, anc(G, name, 1500, int(g['mf_t']), 4, float(g['mf_Y'].max())))
  assert (np.asarray(pt) == g['mf_pt_' + name]).all()


def test_boca_fidelity_and_point(G, mf):
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
  from fake_mf_caller import FakeMFCaller
  g, gp = mf
  Y = g['mf_Y']
  for coeff in (1e-4, 0.5):
    tag = str(coeff).replace('.', 'p').replace('-', 'm')
    np.random.seed(8)
    a = anc(G, 'ucb', 600, int(g['mf_t']), 4, float(Y.max()), boca_thresh_coeff=coeff,
            y_range=float(Y.max() - Y.min()), boca_max_low_fidel_cost_ratio=0.9)
    a.is_mf = True
    a.eval_fidel_points_in_progress = []
    fid, pt = G.acq.boca(G.acq.asy.ucb, gp, a, FakeMFCaller([1.0]))
    assert (np.asarray(pt) == g['mf_boca_point_' + tag]).all()
    assert (np.asarray(fid, dtype=np.float64) == g['mf_boca_fidel_' + tag]).all()


def test_mf_draw_samples_from_the_reference_normals(G, mf):
  g, gp = mf
  np.random.seed(2)                               # the reference's normals come from the same seed
  S = gp.draw_mf_samples(int(g['mf_ts_U'].shape[1]), list(g['mf_Zs']), list(g['mf_Xs']))
  err = np.abs(np.asarray(S) - g['mf_ts_samples']).max()
  assert err <= 1e-8, err


def test_add_data_multiple_equals_a_rebuild(G):
  """ The factorisation extended in place (260 -> 300 points, within the padded size) against a GP built on all 300;
      max_diag follows the appended points. """
  g = load_golden('nonstat')
  gp = _mfgp(G, g, 260)
  assert gp._post.capacity() >= 300
  gp.add_mf_data_multiple(list(g['mf_Z'][260:]), list(g['mf_Xd'][260:]), list(g['mf_Y'][260:]))
  full = _mfgp(G, g)
  C = list(g['mf_Cx'])
  mu_a, sd_a = gp.eval_at_fidel([np.array([0.7])] * len(C), C, uncert_form='std')
  mu_f, sd_f = full.eval_at_fidel([np.array([0.7])] * len(C), C, uncert_form='std')
  assert np.abs(mu_a - mu_f).max() <= MU_TOL and np.abs(sd_a ** 2 - sd_f ** 2).max() <= VAR_TOL
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), full.compute_log_marginal_likelihood(), rtol=1e-10)
  assert gp._post.max_diag() == full._post.max_diag()


def test_poly_gp_against_the_reference(G):
  g = load_golden('nonstat')
  kern = G.kernel.PolyKernel(4, 2, float(g['poly_gp_scale']), g['poly_gp_scal'])
  gp = G.gp_core.GP(g['poly_gp_X'], g['poly_gp_Y'], kern, G.gp_core.ConstantMean(float(g['poly_gp_mean'])),
                    float(g['poly_gp_noise']), device=0)
  np.testing.assert_allclose(np.asarray(gp.L)[:16], g['poly_gp_L_rows'], rtol=0, atol=1e-8)
  np.testing.assert_allclose(np.asarray(gp.alpha), g['poly_gp_alpha'], rtol=0, atol=1e-8)
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g['poly_gp_lml']), rtol=1e-10)
  mu, sd = gp.eval(g['poly_gp_C'], 'std')
  np.testing.assert_allclose(mu, g['poly_gp_mu'], rtol=0, atol=MU_TOL)
  np.testing.assert_allclose(sd ** 2, g['poly_gp_sd'] ** 2, rtol=0, atol=VAR_TOL)
  np.random.seed(11)
  pt = G.acq.asy.ei(gp, anc(G, 'ei', 1500, int(g['poly_gp_t']), 4, float(g['poly_gp_Y'].max())))
  assert (np.asarray(pt) == g['poly_gp_pt_ei']).all()


def _large(G, kind, n=1100, m=30000):
  """ A GP above the int8 threshold (n >= 1024) with its oracle twin, and more candidates than one scoring chunk. """
  rs = np.random.RandomState(21)
  if kind == 'mf':
    X = rs.random_sample((n, 1 + 4))
    Y = np.sin(3 * X[:, 1]) * (0.5 + 0.5 * X[:, 0]) + X[:, 2] * X[:, 3] + 0.02 * rs.standard_normal(n)
    k = G.kernel.CoordinateProductKernel(5, 0.9, [G.kernel.ExpDecayKernel(1, 1.0, 0.05, [1.3]),
                                                  G.kernel.SEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7])], [[0], [1, 2, 3, 4]])
    ok = O.OCoordinateProductKernel(5, 0.9, [R.OExpDecayKernel(1, 1.0, 0.05, [1.3]),
                                             O.OSEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7])], [[0], [1, 2, 3, 4]])
    C = np.concatenate((np.ones((m, 1)), rs.random_sample((m, 4))), axis=1)
  else:
    X = rs.random_sample((n, 6))
    Y = X[:, 0] * X[:, 1] - X[:, 2] ** 2 + 0.3 * X[:, 5] + 0.02 * rs.standard_normal(n)
    scal = [0.9, 1.1, 0.8, 1.2, 1.0, 0.7]
    k, ok = G.kernel.PolyKernel(6, 2, 0.5, scal), R.OPolyKernel(6, 2, 0.5, scal)
    C = rs.random_sample((m, 6))
  mc = float(np.median(Y))
  gp = G.gp_core.GP(X, Y, k, G.gp_core.ConstantMean(mc), 0.01, device=0)
  ogp = O.OGP(X, Y, ok, lambda x: np.array([mc] * len(x)), 0.01)
  return gp, ogp, C


@pytest.mark.parametrize('kind', ['mf', 'poly'])
def test_no_int8_screen_and_no_bound_pass_above_the_int8_threshold(G, kind):
  """ At N = 1100 a stationary kernel would be screened in int8 and pruned by the bound pass; a non-stationary one is
      scored in fp64 and its arg-max is the oracle's, also with score_impl = 1 (which falls back to fp64 for it). """
  gp, ogp, C = _large(G, kind)
  post = gp._post
  d = C.shape[1]
  beta = O.ucb_beta_th(d, 1100)
  mu_o, var_o = O.eval_std_diag(ogp, C)
  want = O.np_argmax_first(O.acq_ucb(mu_o, np.sqrt(var_o), beta))
  for impl in (2, 1):
    post.set_option('score_impl', impl)
    assert post.query('i8_ready') == 0.0
    _, idx, _ = gp._fused_score(G.device.make_acq_desc('ucb', beta=beta), C)
    assert post.query('last_used_i8') == 0.0 and post.query('last_survivors') == 0.0
    assert idx == want, (impl, idx, want)
    mu, sd = gp.eval(C, 'std')
    assert np.abs(mu - mu_o).max() <= MU_TOL and np.abs(sd ** 2 - var_o).max() <= VAR_TOL
    assert post.query('last_used_i8') == 0.0


@pytest.mark.parametrize('kind', ['poly', 'expdecay'])
def test_lml_gradients_are_refused(G, kind):
  """ Neither kernel has a gradient in the reference (Kernel._child_gradient raises): dfb_lml_gradients returns -3. """
  rs = np.random.RandomState(3)
  X, Y = rs.random_sample((200, 2)), rs.random_sample(200)
  k = G.kernel.PolyKernel(2, 2, 1.0, [1.0, 0.5]) if kind == 'poly' else G.kernel.ExpDecayKernel(2, 1.0, 0.1, [1.0, 2.0])
  gp = G.gp_core.GP(X, Y, k, G.gp_core.ConstantMean(0.0), 0.01, device=0)
  import ctypes as C
  out = (C.c_double * 8)()
  assert G.lib.load().dfb_lml_gradients(gp._post.h, out, 8) == -3
  with pytest.raises(NotImplementedError):
    gp._post.lml_gradients(2)


@pytest.mark.parametrize('dom', ['se', 'matern'])
def test_fit_gp_selects_what_the_reference_mf_fitter_selects(G, dom):
  """ hp_grid.fit_gp (LMLs on the device) with the MF layout picks the reference EuclideanMFGPFitter's hps
      (fidel_kernel_type 'expdecay', method 'rand') with the same LML, and rand_exp_sampling its probabilities. """
  from dragonfly_b200 import hp_grid
  g = load_golden('fitter_expdecay')
  X, Y = np.concatenate((g['Z'], g['X']), axis=1), g['Y']
  tag = dom + '_rand'
  lay = hp_grid.EuclideanMFExpDecayHPLayout(1, 3, dom, domain_nu=float(g[tag + '_domain_matern_nu']),
                                            mean_func_type=str(g['mean_func_type']),
                                            noise_var_type=str(g['noise_var_type']))
  np.random.seed(5)
  _, gp, (cts, _) = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], [], method='rand',
                                   max_evals=int(g[tag + '_max_evals']))
  assert (np.array(cts) == g[tag + '_cts']).all()
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-10)
  mu, sd = gp.eval(np.concatenate((g[tag + '_Cz'], g[tag + '_Cx']), axis=1), 'std')
  np.testing.assert_allclose(mu, g[tag + '_mu'], rtol=0, atol=MU_TOL)
  np.testing.assert_allclose(sd ** 2, g[tag + '_sd'] ** 2, rtol=0, atol=VAR_TOL)
  tag = dom + '_rand_exp_sampling'
  np.random.seed(5)
  _, cts, _, _, probs = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], [], method='rand_exp_sampling',
                                       max_evals=int(g[tag + '_max_evals']))
  assert (cts == g[tag + '_cts']).all()
  np.testing.assert_allclose(probs, g[tag + '_probs'], rtol=1e-7, atol=1e-12)
