"""
ESP kernel on the device (-m gpu): kstar_esp_kernel behind Kernel.__call__, the posterior build, dfb_eval, the fused
acquisition arg-max (fp64 and int8 screen), hallucinations / add_data, Thompson draws and the refusal of LML gradients,
against the NumPy restatement of the reference (tests/esp_ref.py) and its extended-precision value.
"""
from argparse import Namespace
import ctypes as C
import math

import numpy as np
import pytest

import esp_ref as E
from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, device, gp_core, _lib
  _lib.load()
  return Namespace(torch=torch, kernel=kernel, device=device, gp_core=gp_core, lib=_lib)


def _kern(G, kind, d, order, scale, bws):
  nus = [(0.5, 1.5, 2.5)[t % 3] for t in range(d)] if kind == 'matern' else None
  k = G.kernel.ESPKernelSE(d, scale, order, bws) if kind == 'se' else \
      G.kernel.ESPKernelMatern(d, nus, scale, order, bws)
  return k, E.oracle_kernel(kind, scale, order, bws, nus), nus


def _data(d, n, m, seed):
  rs = np.random.RandomState(seed)
  X = rs.random_sample((n, d))
  Y = np.sin(3 * X[:, 0]) + (X ** 2).sum(axis=1) / d + 0.05 * rs.standard_normal(n)
  return X, Y, rs.random_sample((m, d))


KCASES = [(kind, d, r) for kind in ('se', 'matern') for d in (1, 2, 4, 8) for r in range(1, d + 1)] + \
         [('se', 20, r) for r in (1, 2, 3, 10, 20)] + [('matern', 20, r) for r in (2, 20)]


@pytest.mark.parametrize('kind,d,order', KCASES)
def test_kernel_call_within_the_bound(G, kind, d, order):
  X, _, Y = _data(d, 150, 70, d * 7 + order)
  bws = list(0.3 + 0.4 * np.random.RandomState(order).random_sample(d)) if d < 20 else [2.0] * d
  k, ok, nus = _kern(G, kind, d, order, 1.3, bws)
  Kd = k(X, Y)
  ex = E.esp_exact(kind, 1.3, order, bws, X, Y, nus)
  b = E.esp_bound(kind, 1.3, order, bws, X, Y, nus)
  ratio = np.max(np.abs(Kd.astype(E.LD) - ex) / b)
  assert ratio < 1.0, ratio
  assert np.all(np.abs(Kd - ok(X, Y)) <= 2 * b)
  Kxx = k(X)                                      # K(X, X): train coordinates on both sides
  assert np.all(np.abs(Kxx - ok(X, X)) <= 2 * E.esp_bound(kind, 1.3, order, bws, X, X, nus))


def _post(G, k, X, Y, noise, chunk=1024, **opts):
  post = G.device.DevicePosterior(len(X) + 8, chunk=chunk)
  for name, v in opts.items():
    post.set_option(name, v)
  post.set_kernel(G.kernel.build_descriptor(k))
  post.set_train(X, Y - np.mean(Y))
  assert post.build(noise)[0] == 0
  return post


PCASES = [('se', 1, 1), ('se', 4, 2), ('matern', 4, 4), ('se', 8, 1), ('se', 8, 4), ('matern', 8, 8), ('se', 20, 2),
          ('se', 20, 3)]


@pytest.mark.parametrize('kind,d,order', PCASES)
def test_posterior_eval_against_the_oracle(G, kind, d, order):
  X, Y, Cn = _data(d, 1100, 3000, 11 * d + order)
  # d = 20: k(x, x) = 1.1 C(20, order) would leave K(X, X) + noise I too ill-conditioned for the 1e-10 mu contract
  scale = 1.1 if d < 20 else 2.0 / math.comb(d, order)
  k, ok, _ = _kern(G, kind, d, order, scale, [0.5] * d)
  mc = float(np.mean(Y))
  ogp = O.OGP(X, Y, ok, lambda x: np.array([mc] * len(x)), 0.01)
  post = _post(G, k, X, Y, 0.01)
  assert abs(post.lml - ogp.compute_log_marginal_likelihood()) <= 1e-9 * abs(ogp.compute_log_marginal_likelihood())
  mu, sd = post.eval(Cn, mean_const=mc)
  mu_o, var_o = O.eval_std_diag(ogp, Cn)
  assert np.abs(mu - mu_o).max() <= 1e-10, np.abs(mu - mu_o).max()
  assert np.abs(sd ** 2 - var_o).max() <= 1e-8, np.abs(sd ** 2 - var_o).max()
  with pytest.raises(NotImplementedError):        # the reference's ESPKernel has no gradient (kernel.py:116-125)
    post.lml_gradients(d)


ACQS = ['ucb', 'ei', 'pi', 'ttei']


def _acq(G, name, Y, d, n):
  if name == 'ucb':
    return G.device.make_acq_desc('ucb', beta=O.ucb_beta_th(d, n)), lambda m, s: O.acq_ucb(m, s, O.ucb_beta_th(d, n))
  if name == 'ttei':
    rm, rsd = float(Y.max()), 0.1
    return G.device.make_acq_desc('ttei', ref_mean=rm, ref_std=rsd), lambda m, s: O.acq_ttei(m, s, rm, rsd)
  best = float(Y.max())
  f = O.acq_ei if name == 'ei' else O.acq_pi
  return G.device.make_acq_desc(name, best=best), lambda m, s: f(m, s, best)


# (kind, d, order, scale): k(x, x) = scale C(d, order) -- small enough for the int8 screen's a-priori bound in the first,
# far too large in the second
SCASES = [('se', 4, 2, 0.2), ('matern', 8, 4, 40.0)]


@pytest.mark.parametrize('kind,d,order,scale', SCASES)
def test_argmax_against_the_oracle(G, kind, d, order, scale):
  X, Y, Cn = _data(d, 1100, 5000, 3 * d + order)
  k, ok, _ = _kern(G, kind, d, order, scale, [0.5] * d)
  mc = float(np.mean(Y))
  ogp = O.OGP(X, Y, ok, lambda x: np.array([mc] * len(x)), 0.01)
  mu_o, var_o = O.eval_std_diag(ogp, Cn)
  used = []
  for impl in (0, 2):
    post = _post(G, k, X, Y, 0.01, score_impl=impl)
    for name in ACQS:
      acq, f = _acq(G, name, Y, d, len(X))
      _, idx, _ = post.score_argmax(acq, Cn, mean_const=mc)
      assert idx == O.np_argmax_first(f(mu_o, np.sqrt(var_o))), (impl, name)
      if impl == 2 and name != 'ttei':
        used.append(post.query('last_used_i8'))
  expect = 1.0 if SCASES.index((kind, d, order, scale)) == 0 else 0.0
  assert set(used) == {expect}, used


def _copy(G, post, name, nbytes):
  t = G.torch.empty((nbytes,), dtype=G.torch.uint8, device=post.device)
  G.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), nbytes), 'dfb_debug_copy')
  return t.cpu().numpy()


def _radix128_values(planes):
  """ The integer 2^42 x that the six radix-128 digits of every entry encode (digit s of column k in plane s // 2, half
      s % 2 of each 64-byte block).  The fused producers split x 2^21 into two 21-bit halves of three digits each while
      slice_i8_kernel peels one rint(128 x) digit at a time: both round x to the same multiple of 2^-42, with digit
      strings that may differ where a digit is +-64 (as for the plain kernels' fused producer), so the value is what
      must match. """
  rows = planes.shape[1]
  p = planes.view(np.int8).reshape(3, rows, -1, 2, 32).astype(np.int64)
  v = np.zeros(p.shape[1:3] + (32,), dtype=np.int64)
  for s in range(6):
    v = v * 128 + p[s // 2, :, :, s % 2, :]
  return v


@pytest.mark.parametrize('radix', [1, 0])
@pytest.mark.parametrize('order', [1, 3, 6, 12])
def test_fused_digits_equal_the_sliced_rows(G, radix, order):
  d = 12
  X, Y, Cn = _data(d, 1100, 700, order)
  k, _, _ = _kern(G, 'se', d, order, 0.5, [0.8] * d)
  out = []
  for fuse in (1, 0):
    post = _post(G, k, X, Y, 0.01, score_impl=1, i8_unguarded=1, i8_radix=radix, i8_fuse=fuse)
    mu, sd = post.eval(Cn, mean_const=0.3)
    assert post.query('last_used_i8') == 1.0
    npad, chunk = int(post.query('npad')), int(post.query('chunk'))
    planes = _copy(G, post, 'Ki8', 6 * chunk * npad).reshape(3, chunk, 2 * npad)
    # the rows of this chunk (m rounded up to 128); radix 256 writes five digits: not the second half of each 64-byte
    # block of plane 3 (the unused sixth slot)
    rows = planes[:, :(len(Cn) + 127) // 128 * 128].copy()
    if radix == 1:
      rows[2].reshape(rows.shape[1], -1, 2, 32)[:, :, 1, :] = 0
    else:
      rows = _radix128_values(rows)
    out.append((mu, sd, rows, post.query('i8_sigma2_bound')))
  assert np.array_equal(out[0][2], out[1][2])
  assert np.array_equal(out[0][0].view(np.int64), out[1][0].view(np.int64))
  if radix == 1:
    assert np.array_equal(out[0][1].view(np.int64), out[1][1].view(np.int64))
  else:
    # the contraction keeps 21 of the 36 radix-128 digit products, so two digit strings of one value give sigma^2
    # within the a-priori bound of each other rather than bit for bit
    assert np.abs(out[0][1] ** 2 - out[1][1] ** 2).max() <= 2 * out[0][3]


def test_prune_stays_off(G):
  d, order = 4, 2
  X, Y, Cn = _data(d, 1100, 5000, 5)
  k, _, _ = _kern(G, 'se', d, order, 0.2, [0.5] * d)
  res = []
  for prune in (1, 0):
    post = _post(G, k, X, Y, 0.01, score_impl=2, prune=prune)
    acq, _ = _acq(G, 'ei', Y, d, len(X))
    s, i, _ = post.score_argmax(acq, Cn, mean_const=float(np.mean(Y)))
    assert post.query('last_survivors') == 0.0 and post.query('last_pruned_candidates') == 0.0
    res.append((np.float64(s).view(np.int64), i))
  assert res[0] == res[1]


def test_extend_restore_and_rebuild(G):
  d, order = 6, 3
  X, Y, Cn = _data(d, 1000, 800, 9)
  k, _, _ = _kern(G, 'matern', d, order, 1.0, [0.6] * d)
  yc = Y - np.mean(Y)
  post = _post(G, k, X[:990], Y[:990], 0.01)
  post.set_train(X[:990], yc[:990])
  assert post.build(0.01)[0] == 0
  mu0, sd0 = post.eval(Cn)
  assert post.extend(X[990:], yc[990:], save=True)[0] == 0           # hallucinated points: extend in place ...
  mu1, sd1 = post.eval(Cn)
  post.restore(990)                                                 # ... and restore bit for bit
  mu2, sd2 = post.eval(Cn)
  assert np.array_equal(mu0.view(np.int64), mu2.view(np.int64)) and np.array_equal(sd0.view(np.int64), sd2.view(np.int64))
  full = G.device.DevicePosterior(len(X) + 8, chunk=1024)
  full.set_kernel(G.kernel.build_descriptor(k))
  full.set_train(X, yc)
  assert full.build(0.01)[0] == 0
  mu_f, sd_f = full.eval(Cn)
  assert np.abs(mu1 - mu_f).max() <= 1e-10 and np.abs(sd1 ** 2 - sd_f ** 2).max() <= 1e-8


def test_thompson_draws_against_the_oracle(G):
  d, order = 5, 2
  X, Y, Cn = _data(d, 400, 300, 13)
  k, ok, _ = _kern(G, 'se', d, order, 1.0, [0.4] * d)
  mc = float(np.mean(Y))
  post = _post(G, k, X, Y, 0.05)
  U = np.random.RandomState(1).standard_normal((Cn.shape[0], 8))
  info, S, _ = post.ts_draws(Cn, U.T.copy(), mean_const=mc)
  assert info == 0
  ogp = O.OGP(X, Y, ok, lambda x: np.array([mc] * len(x)), 0.05)
  ref = ogp.draw_samples_with_normals(Cn, U)
  err = np.abs(S.cpu().numpy() - ref).max()
  print('TS draws vs oracle: max |d sample| = %.3g' % err)
  assert err <= 1e-8, err


def test_gp_gradient_raises_for_d1(G):
  X, Y, _ = _data(1, 200, 10, 2)
  k = G.kernel.ESPKernelSE(1, 1.0, 1, [0.3])
  gp = G.gp_core.GP(X, Y, k, G.gp_core.ConstantMean(float(np.mean(Y))), 0.01, device=0)
  with pytest.raises(NotImplementedError):
    gp.compute_grad_log_marginal_likelihood('scale')


# ---- against the unmodified reference (golden esp.npz, tests/golden/make_golden_esp.py) -----------------------------
G_NUS = (0.5, 1.5, 2.5)


def _golden():
  from conftest import load_golden
  return load_golden('esp')


def test_kernel_call_against_the_reference_blocks(G):
  g = _golden()
  n = 0
  for key in g.files:
    if not key.startswith('K_'):
      continue
    _, kind, d, r = key.split('_')
    d, r = int(d), int(r)
    X1, X2 = g['X1_%d_%d' % (d, r)], g['X2_%d_%d' % (d, r)]
    bws = list(0.3 + 0.5 * np.random.RandomState(100 + d).random_sample(d)) if d < 20 else [2.0] * d
    k, _, nus = _kern(G, kind, d, r, 1.3, bws)
    b = E.esp_bound(kind, 1.3, r, bws, X1, X2, nus)
    assert np.all(np.abs(k(X1, X2) - g[key]) <= 2 * b), key
    n += 1
  assert n == 2 * (1 + 2 + 4 + 8 + 5)


@pytest.fixture(scope='module')
def ggp(G):
  g = _golden()
  d, r = int(g['gp_d']), int(g['gp_order'])
  kern = G.kernel.ESPKernelMatern(d, [G_NUS[t % 3] for t in range(d)], float(g['gp_scale']), r, list(g['gp_bws']))
  gp = G.gp_core.GP(g['gp_X'], g['gp_Y'], kern, G.gp_core.ConstantMean(float(g['gp_mean'])), float(g['gp_noise']),
                    device=0)
  return g, gp


def test_gp_against_the_reference_gp(G, ggp):
  g, gp = ggp
  np.testing.assert_allclose(np.asarray(gp.L)[:16], g['L_rows'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(np.asarray(gp.alpha), g['alpha'], rtol=1e-9, atol=1e-9)
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g['lml']), rtol=1e-11)
  mu, sd = gp.eval(g['gp_C'], 'std')
  np.testing.assert_allclose(mu, g['mu'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(sd ** 2, g['sd'] ** 2, rtol=0, atol=1e-8)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(g['gp_C'][:200], list(g['Xh']), 'std')
  np.testing.assert_allclose(mu_h, g['mu_h'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(sd_h ** 2, g['sd_h'] ** 2, rtol=0, atol=1e-8)


@pytest.mark.parametrize('name', ['ei', 'ucb'])
def test_end_to_end_acquisition_points(G, ggp, name):
  """ asy_ei / asy_ucb(gp, anc_data) under the reference's seed return the reference's point exactly. """
  from dragonfly_b200 import gpb_acquisitions as acq, domains
  g, gp = ggp
  d = int(g['gp_d'])
  dom = domains.EuclideanDomain([[0, 1]] * d)
  anc = Namespace(curr_acq=name, max_evals=1500, t=int(g['t']), domain=dom, curr_max_val=float(g['curr_best']),
                  eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                  is_mf=False, domain_bounds=np.array(dom.bounds))
  np.random.seed(7)
  pt = getattr(acq.asy, name)(gp, anc)
  assert (np.asarray(pt) == g['pt_' + name]).all()


def test_draw_samples_against_the_reference(G, ggp):
  g, gp = ggp
  np.random.seed(2)                               # the reference's normals come from the same seed
  S = gp.draw_samples(int(g['ts_U'].shape[1]), g['gp_C'][:64])
  err = np.abs(np.asarray(S) - g['ts_samples']).max()
  print('draw_samples vs reference: max |d sample| = %.3g' % err)
  assert err <= 1e-8, err


def test_add_data_multiple_and_hallucinated_eval(G):
  """ GP.add_data_multiple (the factorisation extended in place) against a GP built on all points, and a hallucinated
      GP.eval against the oracle's (N + q)-point posterior; the GP is unchanged afterwards. """
  d, order = 6, 3
  X, Y, Cn = _data(d, 1000, 800, 9)
  k, ok, _ = _kern(G, 'matern', d, order, 1.0, [0.6] * d)
  mc = float(np.mean(Y))
  mean = G.gp_core.ConstantMean(mc)
  gp = G.gp_core.GP(X[:980], Y[:980], k, mean, 0.01, device=0)
  mu0, sd0 = gp.eval(Cn, 'std')
  ogp = O.OGP(X[:980], Y[:980], ok, lambda x: np.array([mc] * len(x)), 0.01)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(Cn, list(X[980:990]), 'std')
  mu_ho, var_ho = O.eval_std_diag(ogp, Cn, X[980:990])
  assert np.abs(mu_h - mu_ho).max() <= 1e-10 and np.abs(sd_h ** 2 - var_ho).max() <= 1e-8
  mu1, sd1 = gp.eval(Cn, 'std')
  assert np.array_equal(mu0, mu1) and np.array_equal(sd0, sd1)
  gp.add_data_multiple(list(X[980:]), list(Y[980:]))
  full = G.gp_core.GP(X, Y, k, mean, 0.01, device=0)
  mu_a, sd_a = gp.eval(Cn, 'std')
  mu_f, sd_f = full.eval(Cn, 'std')
  assert np.abs(mu_a - mu_f).max() <= 1e-10 and np.abs(sd_a ** 2 - sd_f ** 2).max() <= 1e-8
  assert abs(gp.compute_log_marginal_likelihood() - full.compute_log_marginal_likelihood()) <= \
      1e-10 * abs(full.compute_log_marginal_likelihood())


# ---- hyper-parameter fitting (hp_grid) ------------------------------------------------------------------------------
def _fitter_golden():
  from conftest import load_golden
  return load_golden('fitter_esp')


def _dscr_vals(g, tag):
  return [list(g[tag + '_dscr_vals_%d' % i]) for i in range(int(g[tag + '_n_dscr']))]


def _layout(kind, g):
  from dragonfly_b200 import hp_grid
  return hp_grid.EuclideanHPLayout(3, 'esp', esp_kernel_type=kind, mean_func_type=str(g['mean_func_type']),
                                   noise_var_type=str(g['noise_var_type']))


def test_lml_for_hyperparams_against_the_oracle(G):
  from dragonfly_b200 import hp_grid
  g = _fitter_golden()
  X, Y = g['X'], g['Y']
  lay = _layout('matern', g)
  b, dv = lay.bounds(X, Y)
  rs = np.random.RandomState(3)
  hps = b[:, 0] + rs.random_sample((12, len(b))) * (b[:, 1] - b[:, 0])
  dscr = [(dv[0][i % 3], dv[1][i % 3]) for i in range(12)]
  l1, _ = hp_grid.lml_for_hyperparams(X, Y, hps, lay, nus=dscr, lanes=1)
  l3, _ = hp_grid.lml_for_hyperparams(X, Y, hps, lay, nus=dscr, lanes=3)
  assert np.array_equal(l1, l3)
  for i, hp in enumerate(hps):
    m, nv, k = lay.unpack(hp, Y, dscr[i])
    ok = E.oracle_kernel('matern', k.hyperparams['scale'], k.hyperparams['order'],
                         [float(c.hyperparams['dim_bandwidths'][0]) for c in k.kernel_list],
                         [c.hyperparams['nu'] for c in k.kernel_list])
    ref = O.OGP(X, Y, ok, lambda x, c=m: np.array([c] * len(x)), nv).compute_log_marginal_likelihood()
    assert abs(l1[i] - ref) <= 1e-10 * max(1.0, abs(ref)), (i, l1[i], ref)


@pytest.mark.parametrize('kind', ['se', 'matern'])
def test_fit_gp_end_to_end(G, kind):
  """ hp_grid.fit_gp on the device against the reference's EuclideanGPFitter with kernel_type 'esp' (fitter_esp.npz):
      the same candidates and selection for rand / rand_exp_sampling; PDOO may branch differently on a 1e-11 LML
      difference and must then end at least as high. """
  from dragonfly_b200 import hp_grid
  g = _fitter_golden()
  X, Y = g['X'], g['Y']
  lay = _layout(kind, g)
  tag = kind + '_rand'
  np.random.seed(5)
  _, gp, (cts, dscr) = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], _dscr_vals(g, tag), method='rand',
                                      max_evals=int(g[tag + '_max_evals']))
  assert (np.array(cts) == g[tag + '_cts']).all() and (np.array(dscr) == g[tag + '_dscr']).all()
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-10)
  mu, sd = gp.eval(g[tag + '_C'], 'std')
  np.testing.assert_allclose(mu, g[tag + '_mu'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(sd ** 2, g[tag + '_sd'] ** 2, rtol=0, atol=1e-8)
  tag = kind + '_rand_exp_sampling'
  np.random.seed(5)
  _, cts, dscr, _, probs = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], _dscr_vals(g, tag),
                                          method='rand_exp_sampling', max_evals=int(g[tag + '_max_evals']))
  assert (cts == g[tag + '_cts']).all() and (np.array(dscr) == g[tag + '_dscr']).all()
  np.testing.assert_allclose(probs, g[tag + '_probs'], rtol=1e-7, atol=1e-12)
  tag = kind + '_pdoo'
  np.random.seed(5)
  _, gp, (cts, dscr) = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], _dscr_vals(g, tag), method='pdoo',
                                      max_evals=int(g[tag + '_max_evals']))
  same = (np.array(cts) == g[tag + '_cts']).all() and (np.array(dscr) == g[tag + '_dscr']).all()
  assert same or gp.compute_log_marginal_likelihood() >= float(g[tag + '_lml']) - 1e-6
