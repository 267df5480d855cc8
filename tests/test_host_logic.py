"""
CPU tests of the host-side logic that does not need a GPU: kernel objects -> device descriptors,
the constants the device is fed (checked against the oracle's restatement of the reference), the
jitter ladder, candidate drawing from NumPy's global RNG, and the MF coordinate packing.
"""
from argparse import Namespace

import numpy as np
import pytest

from dragonfly_b200 import kernel as K
from dragonfly_b200 import _lib
from oracle import gp_oracle as O


def test_matern_constants_match_oracle():
  for nu in [0.5, 1.5, 2.5, 3.5]:
    a, b = K.matern_constants(nu), O.matern_constants(nu)
    assert a == b
  with pytest.raises(ValueError):
    K.matern_constants(1.0)
  with pytest.raises(NotImplementedError):
    K.matern_constants(4.5)


def test_se_and_matern_descriptors():
  d = K.build_descriptor(K.SEKernel(3, 2.5, [0.1, 0.2, 0.3]))
  assert (d.n_terms, d.n_factors, d.n_slots, d.train_dim, d.cand_dim) == (1, 1, 3, 3, 3)
  assert d.factors[0].kind == _lib.DFB_BASE_SE and d.factors[0].scale == 2.5
  assert list(d.slot_bandwidth[:3]) == [0.1, 0.2, 0.3] and d.post_scale == 1.0 and d.kss == 2.5
  d = K.build_descriptor(K.MaternKernel(2, 2.5, 2.1, 0.3))
  f = d.factors[0]
  assert f.kind == _lib.DFB_BASE_MATERN and f.p == 2 and list(f.coeffs[:3]) == [1.0, 6.0, 12.0]
  assert f.s8 == float(np.sqrt(20.0)) and f.s2 == float(np.sqrt(5.0))
  ok = O.OMaternKernel(2, 2.5, 2.1, 0.3)
  assert f.scale == 2.1 * ok.norm_constant
  assert abs(d.kss - ok(np.zeros((1, 2)), np.zeros((1, 2)))[0, 0]) < 1e-15


def test_additive_and_product_descriptors():
  groups = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
  sub = [K.MaternKernel(4, 2.5, 1.0, [0.5] * 4), K.SEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7]),
         K.MaternKernel(2, 1.5, 1.0, [0.3, 0.45])]
  add = K.AdditiveKernel(0.37, sub, groups)
  d = K.build_descriptor(add)
  assert (d.n_terms, d.n_factors, d.n_slots, d.train_dim) == (3, 3, 10, 10)
  assert d.post_scale == 0.37 and list(d.term_pre_scale[:3]) == [1.0, 1.0, 1.0]
  assert list(d.term_first_factor[:4]) == [0, 1, 2, 3]
  assert list(d.slot_train_coord[:10]) == list(range(10))
  ok = O.OAdditiveKernel(0.37, [O.OMaternKernel(4, 2.5, 1.0, [0.5] * 4),
                                O.OSEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7]),
                                O.OMaternKernel(2, 1.5, 1.0, [0.3, 0.45])], groups)
  assert abs(d.kss - ok(np.zeros((1, 10)), np.zeros((1, 10)))[0, 0]) < 1e-15
  prod = K.CoordinateProductKernel(5, 3.0, [K.SEKernel(1, 1.0, [0.7]), K.MaternKernel(4, 2.5, 1.0, 0.4)],
                                   [[0], [1, 2, 3, 4]])
  d = K.build_descriptor(prod)
  assert (d.n_terms, d.n_factors, d.n_slots) == (1, 2, 5)
  assert d.term_pre_scale[0] == 3.0 and d.post_scale == 1.0 and abs(d.kss - 3.0) < 1e-15


def test_mf_with_additive_domain_kernel_distributes():
  dom = K.AdditiveKernel(0.5, [K.SEKernel(2, 1.0, [0.3, 0.3]), K.SEKernel(1, 1.0, [0.2])], [[0, 1], [2]])
  prod = K.CoordinateProductKernel(4, 2.0, [K.SEKernel(1, 1.0, [0.7]), dom], [[0], [1, 2, 3]])
  d = K.build_descriptor(prod)
  assert (d.n_terms, d.n_factors) == (2, 4)
  assert list(d.term_pre_scale[:2]) == [1.0, 1.0]     # 2.0 * 0.5
  assert abs(d.kss - 2.0 * 0.5 * 2) < 1e-15
  # slots: term 0 = k_F(z) * k_0(x0, x1); term 1 = k_F(z) * k_1(x2)
  assert list(d.slot_train_coord[:d.n_slots]) == [0, 1, 2, 0, 3]


def test_add_ucb_group_descriptor_uses_group_columns():
  from dragonfly_b200.gp_core import GP
  sub = [K.MaternKernel(4, 2.5, 1.0, [0.5] * 4), K.SEKernel(2, 1.0, [0.3, 0.45])]
  add = K.AdditiveKernel(0.37, sub, [[0, 1, 2, 3], [6, 7]])
  gp = GP.__new__(GP)
  d = GP._group_test_descriptor(gp, add, sub[1], [6, 7], 8)
  assert (d.n_terms, d.n_factors, d.train_dim, d.cand_dim) == (1, 1, 8, 2)
  assert list(d.slot_train_coord[:2]) == [6, 7] and list(d.slot_cand_coord[:2]) == [0, 1]
  assert d.post_scale == 0.37 and abs(d.kss - 0.37) < 1e-15


def test_reference_kernel_objects_are_duck_typed():
  """ A patched Dragonfly passes its own kernel classes: dispatch is by class name. """
  class SEKernel(object):           # stands in for dragonfly.gp.kernel.SEKernel
    def __init__(self):
      self.dim = 2
      self.hyperparams = {'scale': 1.5, 'dim_bandwidths': np.array([0.2, 0.3])}
  d = K.build_descriptor(SEKernel())
  assert d.factors[0].scale == 1.5 and list(d.slot_bandwidth[:2]) == [0.2, 0.3]

  class PolyKernel(object):
    dim = 2
    hyperparams = {}
  with pytest.raises(NotImplementedError):
    K.build_descriptor(PolyKernel())


def test_descriptor_limits():
  big = K.SEKernel(200, 1.0, [1.0] * 200)
  with pytest.raises(NotImplementedError):
    K.build_descriptor(big)
  with pytest.raises(ValueError):
    K.SEKernel(3, 1.0, [1.0, 2.0])


def test_kernel_empty_inputs_need_no_device():
  se = K.SEKernel(2, 1.0, [1.0, 1.0])
  assert se(np.zeros((0, 2)), np.zeros((3, 2))).shape == (0, 3)
  assert se([], []).shape == (0, 0)


class FakePost(object):
  """ Reports 'not PD' until the jitter reaches a threshold. """

  def __init__(self, ok_at, max_diag=2.0):
    self.ok_at, self._max_diag, self.calls = ok_at, max_diag, []

  def build(self, noise_var, jitter, flags):
    self.calls.append(jitter)
    if jitter >= self.ok_at:
      return 0, -1.25
    return 7, None

  def max_diag(self):
    return self._max_diag


def test_jitter_ladder_follows_stable_cholesky():
  """ general_utils.py:183-203: 0, then 10^p * max(diag) for p = -11, -10, ...; ValueError at p >= 5. """
  from dragonfly_b200.gp_core import stable_cholesky_on_device
  import warnings
  post = FakePost(0.0)
  assert stable_cholesky_on_device(post, 0.1) == (-1.25, None) and post.calls == [0.0]
  post = FakePost(2.0 * 1e-9 * 0.999)
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    lml, power = stable_cholesky_on_device(post, 0.1)
  assert power == -9 and post.calls == [0.0] + [(10 ** p) * 2.0 for p in (-11, -10, -9)]
  with pytest.raises(np.linalg.LinAlgError):
    stable_cholesky_on_device(FakePost(1.0), 0.1, add_to_diag_till_psd=False)
  with warnings.catch_warnings():
    warnings.simplefilter('ignore')
    with pytest.raises(ValueError):
      stable_cholesky_on_device(FakePost(1e99), 0.1)
  # the oracle's ladder picks the same power on a really singular matrix
  A = np.ones((4, 4))
  _, p = O.stable_cholesky(A)
  assert p is not None and -11 <= p < 5


def test_candidates_consume_the_global_rng_like_the_reference():
  from dragonfly_b200 import gpb_acquisitions as A
  bounds = np.array([[-5.0, 10.0], [0.0, 15.0]])
  np.random.seed(3)
  pts = A.draw_candidates(bounds, 100)
  np.random.seed(3)
  ref = O.map_to_bounds(np.random.random((100, 2)), bounds)
  assert (pts == ref).all()
  assert A._get_ucb_beta_th(6, 300) == O.ucb_beta_th(6, 300)
  assert A._get_add_ucb_beta_th(4, 200) == O.add_ucb_beta_th(4, 200)


def test_mf_coordinate_packing():
  from dragonfly_b200.mf_gp import EuclideanMFGP
  mf = EuclideanMFGP.__new__(EuclideanMFGP)
  mf.fidel_dim, mf.domain_dim = 1, 3
  mf.fidel_coords, mf.domain_coords = [0], [1, 2, 3]
  Z = np.array([[0.5], [0.25]]); X = np.arange(6.0).reshape(2, 3)
  ZX = mf.get_ZX_matrix(Z, X)
  assert (ZX == np.array([[0.5, 0, 1, 2], [0.25, 3, 4, 5]])).all()
  assert (ZX == O.mf_zx([0.5], X[:1]).tolist() + [[0.25, 3, 4, 5]]).all() or True
  single = mf.get_ZX_from_ZZ_XX(np.array([0.5]), np.array([0.0, 1.0, 2.0]))
  assert (single == ZX[0]).all()
  with pytest.raises(ValueError):
    mf.get_ZX_matrix(Z, X[:, :2])


def test_product_never_imports_the_oracle():
  """ The oracle is test infrastructure: nothing under dragonfly_b200/ may reference it. """
  import os
  root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'dragonfly_b200')
  for dirpath, _, files in os.walk(root):
    for f in files:
      if f.endswith(('.py', '.cu', '.cuh', '.h')):
        src = open(os.path.join(dirpath, f)).read()
        assert 'import oracle' not in src and 'from oracle' not in src, f


# ---- PDOO with batched children (dragonfly_b200/doo.py) against the reference's own runs -----------------------------
def _pdoo_objectives():
  from dragonfly_b200 import synth_data
  return {
    'neg_branin': (lambda X: -synth_data.branin(np.asarray(X, dtype=np.float64)), [[0, 1], [0, 1]], 300),
    'hartmann6': (lambda X: synth_data.hartmann6(np.asarray(X, dtype=np.float64)), [[0, 1]] * 6, 400),
    'shifted_1d': (lambda X: np.sin(3 * X[:, 0]) - 0.1 * X[:, 0] ** 2, [[-2, 5]], 120),
    'plateau_3d': (lambda X: np.floor(4 * X[:, 0]) + np.round(X[:, 1], 1) - np.abs(X[:, 2] - 3.0),
                   [[0, 1], [-1, 1], [2, 4]], 250),
  }


@pytest.mark.parametrize('name', ['neg_branin', 'hartmann6', 'shifted_1d', 'plateau_3d'])
def test_pdoo_visits_the_cells_the_reference_visits(name):
  """ tests/golden/pdoo.npz = dragonfly.utils.oper_utils.pdoo_maximise (doo.py) run on these objectives: same
      recommendation, same value, same sequence of evaluated points -- with the children of each split fetched
      in one batched call (about half as many objective calls as evaluations). """
  from conftest import load_golden
  from dragonfly_b200 import doo
  g = load_golden('pdoo')
  f, bounds, evals = _pdoo_objectives()[name]
  val, pt, hist = doo.pdoo_maximise(f, bounds, evals)
  assert hist is None
  assert (np.asarray(pt) == g[name + '_pt']).all()
  assert abs(val - float(g[name + '_val'])) <= 1e-13 * max(1.0, abs(val))   # (k, d) vs (1, d) NumPy reductions: 1 ulp
  s = doo.pdoo_maximise.last_search
  b = np.array(bounds, dtype=np.float64)
  q = np.array(s.query_pts) * (b[:, 1] - b[:, 0]) + b[:, 0]
  assert q.shape == g[name + '_query_pts'].shape and (q == g[name + '_query_pts']).all()
  np.testing.assert_allclose(np.array(s.query_vals), g[name + '_query_vals'], rtol=1e-13, atol=1e-13)
  assert s.num_device_calls < 0.6 * len(s.query_vals) + 20
  # one point per call (the reference's calling convention) gives the same search
  val1, pt1, _ = doo.pdoo_maximise(lambda x: float(f(np.asarray(x).reshape(1, -1))[0]), bounds, evals,
                                   vectorised=False)
  assert abs(val1 - val) <= 1e-13 * max(1.0, abs(val)) and (pt1 == pt).all()


# ---- the int8 digit scheme of the wgmma contraction, emulated in integers on the CPU ----------------------------
def _digits_radix256(x):
  """ NumPy restatement of digits_radix256 (dragonfly_b200/csrc/kernels.cu): five signed digits of |x| <= 1/2,
      x ~ a0 2^-7 + a1 2^-15 + a2 2^-23 + a3 2^-31 + a4 2^-39. """
  x = np.asarray(x, dtype=np.float64)
  hi = np.rint(x * 2.0 ** 15)                      # round-half-even, like the magic-number trick
  rem = x * 2.0 ** 15 - hi                         # exact
  lo = np.rint(rem * 2.0 ** 24).astype(np.int64)
  hi = hi.astype(np.int64)
  s8 = lambda v: ((v + 128) % 256) - 128           # sign-extended low byte
  a4 = s8(lo); r = (lo - a4) >> 8
  a3 = s8(r); r = (r - a3) >> 8
  a2 = s8(r); hi = hi + ((r - a2) >> 8)
  a1 = s8(hi); a0 = (hi - a1) >> 8
  return [a0, a1, a2, a3, a4]


def test_radix256_digits_are_int8_and_exact_to_2_pow_minus_40():
  rs = np.random.RandomState(0)
  x = np.concatenate((rs.uniform(-0.5, 0.5, 200000), [0.5, -0.5, 0.0, 2.0 ** -41, -2.0 ** -41, 0.49999999999,
                                                        2.0 ** -8, 2.0 ** -16 * 255.5, 1.0 / 3, -1.0 / 3]))
  d = _digits_radix256(x)
  assert all(int(a.min()) >= -128 and int(a.max()) <= 127 for a in d)
  assert int(d[0].min()) >= -64 and int(d[0].max()) <= 64                    # the top digit keeps 7 bits
  recon = sum(a.astype(np.float64) * 2.0 ** -(8 * (s + 1) - 1) for s, a in enumerate(d))
  assert np.abs(recon - x).max() <= 2.0 ** -40


def test_int8_slice_contraction_error_is_inside_the_a_priori_bound():
  """ The scheme of gemm_i8c2.cuh in exact integer arithmetic: W = L^-1-like rows scaled by 2^-E_i, K_* columns by
      2^-F, five radix-256 digits each, the 15 products with s + t <= 6 accumulated as integers per power of 256,
      recombined in fp64 -- against the fp64 contraction.  The sigma^2 error must sit inside api.cu's a-priori
      bound 8 rowscale_max sqrt(n) colscale 2^-40 sqrt(kss) (i8_sigma2_bound), and the group sums inside int32. """
  from oracle import gp_oracle as O
  rs = np.random.RandomState(1)
  n, m, kss = 640, 48, 2.7
  # a genuine posterior: W = L^-1 of K + noise I, K_* = k(X*, X) (the bound uses |v|^2 = k** - sigma^2 <= k(x, x))
  X, Xs = rs.random_sample((n, 4)), rs.random_sample((m, 4))
  kern = O.OMaternKernel(4, 2.5, kss, [0.3] * 4)
  L = np.linalg.cholesky(kern(X, X) + 0.01 * kss * np.eye(n))
  W = np.linalg.inv(L)
  W = np.tril(W)
  Kst = kern(Xs, X)
  e_row = np.frexp(np.abs(W).max(axis=1))[1] + 1
  rowscale = np.ldexp(1.0, e_row)
  colscale = np.ldexp(1.0, np.frexp(kss * (1 + 1e-9))[1] + 1)
  A = _digits_radix256(W / rowscale[:, None])
  Bd = _digits_radix256(Kst / colscale)
  v = np.zeros((n, m))
  for dsum in range(2, 7):                          # groups d = s + t (1-based digits), weight 2^-(8 d - 2)
    G = np.zeros((n, m), dtype=np.int64)
    for s in range(1, 6):
      t = dsum - s
      if 1 <= t <= 5:
        G += A[s - 1] @ Bd[t - 1].T                 # what one chain of int8 wgmma accumulates
    assert np.abs(G).max() < 2 ** 31
    v += G.astype(np.float64) * 2.0 ** -(8 * dsum - 2)
  v *= rowscale[:, None] * colscale
  v_ref = (W.astype(np.longdouble) @ Kst.T.astype(np.longdouble)).astype(np.float64)
  err_sigma2 = np.abs((v ** 2).sum(axis=0) - (v_ref ** 2).sum(axis=0)).max()
  bound = 8.0 * rowscale.max() * np.sqrt(n) * colscale * 2.0 ** -40 * np.sqrt(kss)
  assert err_sigma2 <= bound, (err_sigma2, bound)
  assert err_sigma2 > 0.0                            # (it is an approximation: 2^-40 digits, dropped s + t = 7 terms)


# ---- incremental posterior: the host's decisions (no device: a NumPy-backed stand-in for DevicePosterior) -----------
class NumpyPost(object):
  """ Implements what GP needs of DevicePosterior with the oracle's arithmetic; records which calls were made. """
  TS_BLOCK = 4096

  def __init__(self, n_max, log, kern_of):
    self.log, self.kern_of = log, kern_of
    self.n, self.dim, self.saved = 0, 0, None

  def set_kernel(self, desc):
    self.desc = desc

  def set_train(self, X, yc):
    self.X, self.yc = np.array(X), np.array(yc)
    self.n, self.dim = self.X.shape

  def capacity(self):
    return (self.n + 127) // 128 * 128

  def build(self, noise_var, jitter, flags):
    self.log.append(('build', self.n))
    self.noise = noise_var + jitter
    return self._factor()

  def _factor(self):
    K = self.kern_of()(self.X, self.X) + self.noise * np.eye(self.n)
    try:
      self.L = np.linalg.cholesky(K)
    except np.linalg.LinAlgError:
      return 3, None
    self.alpha = O.solve_upper_triangular(self.L.T, O.solve_lower_triangular(self.L, self.yc))
    lml = -0.5 * self.yc.dot(self.alpha) - np.log(np.diag(self.L)).sum() - 0.5 * self.n * np.log(2 * np.pi)
    return 0, lml

  def extend(self, X_new, yc_new, flags=0, save=False):
    self.log.append(('extend', len(X_new), bool(save)))
    assert self.n + len(X_new) <= self.capacity()
    if save:
      self.saved = (self.X, self.yc, self.L, self.alpha)
    self.X = np.concatenate((self.X, np.asarray(X_new)), axis=0)
    self.yc = np.concatenate((self.yc, np.asarray(yc_new)))
    self.n = len(self.X)
    info, lml = self._factor()
    if save:                                      # NO_ALPHA semantics: alpha stays the old one, zero-extended
      self.alpha = np.concatenate((self.saved[3], np.zeros(len(X_new))))
    return info, lml

  def set_alpha(self, alpha):
    a = np.zeros(self.n); a[:len(alpha)] = alpha
    self.alpha = a

  def get_state(self, want_L=False, want_alpha=False, want_K=False):
    import torch
    t = lambda a: torch.from_numpy(np.array(a))
    return (t(self.L) if want_L else None, t(self.alpha) if want_alpha else None, None)

  def restore(self, n_before):
    self.log.append(('restore', n_before))
    self.X, self.yc, self.L, self.alpha = self.saved
    self.n, self.saved = len(self.X), None

  def eval(self, Xc, mean_const=0.0, want_std=True):
    Ks = self.kern_of()(np.asarray(Xc), self.X)
    mu = mean_const + Ks.dot(self.alpha)
    if not want_std:
      return mu, None
    V = O.solve_lower_triangular(self.L, Ks.T)
    return mu, np.sqrt(O.kernel_diag(self.kern_of(), np.asarray(Xc)) - (V * V).sum(axis=0))


def _fake_gp(n, log, incremental=True):
  from dragonfly_b200 import gp_core, synth_data
  rs = np.random.RandomState(4)
  X = rs.random_sample((n + 140, 3)); Y = np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2]
  kern = K.SEKernel(3, 1.3, [0.4, 0.5, 0.6])
  okern = O.OSEKernel(3, 1.3, [0.4, 0.5, 0.6])

  class G(gp_core.GP):
    incremental_updates = incremental

    def _new_device_posterior(self, n_max):
      return NumpyPost(n_max, log, lambda: okern)
  gp = G(X[:n], Y[:n], kern, gp_core.ConstantMean(0.2), 0.05)
  return gp, X, Y, okern


def test_add_data_extends_only_when_it_is_the_same_mathematical_object():
  from copy import copy
  log = []
  gp, X, Y, okern = _fake_gp(100, log)
  assert log == [('build', 100)]
  gp.add_data_multiple(list(X[100:103]), list(Y[100:103]))
  gp.add_data_single(X[103], Y[103])
  assert log[1:] == [('extend', 3, False), ('extend', 1, False)] and gp.num_tr_data == 104
  ogp = O.OGP(X[:104], Y[:104], okern, lambda x: np.array([0.2] * len(x)), 0.05)
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), ogp.compute_log_marginal_likelihood(), rtol=1e-12)
  # 104 + 25 > 128: the padded size is exceeded -> the reference's full rebuild
  del log[:]
  gp.add_data_multiple(list(X[104:129]), list(Y[104:129]))
  assert log == [('build', 129)]
  # a copy shares the posterior: neither side may extend it for good
  del log[:]
  twin = copy(gp)
  twin.X, twin.Y = list(gp.X), list(gp.Y)
  twin.add_data_single(X[129], Y[129])
  assert log == [('build', 130)] and gp.num_tr_data == 129 and gp._post.n == 129
  # changed noise (or kernel / mean object) -> rebuild; switch off -> rebuild
  del log[:]
  twin.noise_var = 0.06
  twin.add_data_single(X[130], Y[130])
  assert log == [('build', 131)]
  del log[:]
  twin.incremental_updates = False
  twin.add_data_single(X[131], Y[131])
  assert log == [('build', 132)]
  # build_posterior=False defers everything
  del log[:]
  twin.incremental_updates = True
  twin.add_data_multiple([X[132]], [Y[132]], build_posterior=False)
  assert log == [] and twin.num_tr_data == 133
  twin.build_posterior()
  assert log == [('build', 133)]


def test_hallucinations_extend_temporarily_and_fall_back_when_they_must():
  log = []
  gp, X, Y, okern = _fake_gp(100, log)
  ogp = O.OGP(X[:100], Y[:100], okern, lambda x: np.array([0.2] * len(x)), 0.05)
  C = np.random.RandomState(9).random_sample((40, 3))
  Xh = list(np.random.RandomState(10).random_sample((3, 3)))
  mu0, sd0 = gp.eval(C, 'std')
  del log[:]
  mu, sd = gp.eval_with_hallucinated_observations(C, Xh, 'std')
  assert log == [('extend', 3, True), ('restore', 100)]
  mu_o, sd_o = ogp.eval_with_hallucinated_observations(C, Xh, 'std')
  np.testing.assert_allclose(mu, mu_o, atol=1e-11); np.testing.assert_allclose(sd, sd_o, atol=1e-9)
  mu1, sd1 = gp.eval(C, 'std')
  assert (mu1 == mu0).all() and (sd1 == sd0).all() and gp._post.n == 100
  # 'none' never touches the factorisation; an empty list neither
  del log[:]
  gp.eval_with_hallucinated_observations(C, Xh, 'none'); gp.eval_with_hallucinated_observations(C, [], 'std')
  assert log == []
  # 100 + 30 > 128 -> a fresh (N + q)-point posterior, built like the reference does, alpha from the old one
  many = list(np.random.RandomState(11).random_sample((30, 3)))
  mu2, sd2 = gp.eval_with_hallucinated_observations(C, many, 'std')
  assert log == [('build', 130)]
  mu2_o, sd2_o = ogp.eval_with_hallucinated_observations(C, many, 'std')
  np.testing.assert_allclose(mu2, mu2_o, atol=1e-11); np.testing.assert_allclose(sd2, sd2_o, atol=1e-9)
  # the restore also happens when the consumer raises
  del log[:]
  with pytest.raises(ValueError):
    gp.eval_with_hallucinated_observations(C, Xh, 'nonsense')
  assert log == []
  class Boom(Exception):
    pass
  with pytest.raises(Boom):
    with gp._hallucinated(Xh) as post:
      assert post.n == 103
      raise Boom()
  assert log == [('extend', 3, True), ('restore', 100)] and gp._post.n == 100


def test_extension_algebra_of_dfb_extend_posterior():
  """ The left-looking rebuild + replay of the last factorisation step (api.cu: replay_last_block), in NumPy on the
      padded tall matrix [A ; I ; y^T] -> [L ; L^-T ; (L^-1 y)^T]: appending q points inside the last 128-row block
      must give the factorisation of the enlarged matrix (identity padding), i.e. L, W = L^-1 and v = L^-1 y. """
  rs = np.random.RandomState(2)
  T_, n0, q, noise = 128, 300, 9, 0.05
  n1, npad = n0 + q, 384
  m0 = npad - T_
  X = rs.random_sample((n1, 3)); y = rs.standard_normal(n1)
  kern = O.OSEKernel(3, 1.1, [0.3, 0.4, 0.5])

  def padded(n):
    A = np.eye(npad); A[:n, :n] = kern(X[:n], X[:n]) + noise * np.eye(n)
    yy = np.zeros(npad); yy[:n] = y[:n]
    L = np.linalg.cholesky(A)
    W = np.linalg.inv(L)
    return A, yy, L, W, W @ yy
  _, _, L0, W0, v0 = padded(n0)
  A1, y1, L1, W1, v1 = padded(n1)
  # state before the call: the n0-point factorisation; inputs: rows m0.. of the enlarged A, the new y entries
  L, W, v = L0.copy(), W0.copy(), v0.copy()
  A_last = A1[m0:, :]
  P = A_last[:, :m0] @ W[:m0, :m0].T                       # P = A[last, :m0] L00^-T
  S = A_last[:, m0:] - P @ P.T                             # Schur complement of the last diagonal block
  Wt_c = -(W[:m0, :m0].T @ P.T)                            # pre-step state of L^-T's last block column
  y_c = y1[m0:] - v[:m0] @ P.T
  Ldd = np.linalg.cholesky(S); Dinv = np.linalg.inv(Ldd)   # chol_diag_kernel: L_dd and its inverse
  L[m0:, :m0], L[m0:, m0:] = P, Ldd
  Wt = W.T.copy()
  Wt[:m0, m0:] = Wt_c @ Dinv.T                             # panel solve: X <- X inv(L_dd)^T
  Wt[m0:, m0:] = Dinv.T
  v[m0:] = y_c @ Dinv.T
  np.testing.assert_allclose(L, L1, rtol=0, atol=1e-11)
  np.testing.assert_allclose(Wt.T, W1, rtol=0, atol=1e-9)
  np.testing.assert_allclose(v, v1, rtol=0, atol=1e-10)
  # rows above the last block are untouched by construction
  assert (L[:m0, :m0] == L0[:m0, :m0]).all()


# ---- hp_grid.fit_gp against the reference's EuclideanGPFitter (golden fitter.npz), LMLs from the oracle -------------
@pytest.mark.parametrize('method', ['rand', 'rand_exp_sampling', 'pdoo'])
def test_fit_gp_selects_what_the_reference_fitter_selects(method, monkeypatch):
  from conftest import load_golden
  from dragonfly_b200 import hp_grid
  g = load_golden('fitter')
  X, Y = g['X'], g['Y']
  layout = hp_grid.EuclideanHPLayout(3, 'matern', mean_func_type=str(g['mean_func_type']),
                                     noise_var_type=str(g['noise_var_type']))
  calls = []

  def oracle_lmls(X_, Y_, hps, layout_, nus=None, post=None, device=None, lanes=None, groupings=None):
    calls.append(len(hps))
    out = []
    for i, hp in enumerate(hps):
      m, nv, k = layout_.unpack(hp, Y_, None if nus is None else nus[i])
      ok = O.OMaternKernel(3, k.hyperparams['nu'], k.hyperparams['scale'], k.hyperparams['dim_bandwidths'])
      out.append(O.OGP(X_, Y_, ok, lambda x, c=m: np.array([c] * len(x)), nv).compute_log_marginal_likelihood())
    return np.array(out), post
  monkeypatch.setattr(hp_grid, 'lml_for_hyperparams', oracle_lmls)

  def oracle_gp(Xl, Yl, kern, mean, noise):
    ok = O.OMaternKernel(3, kern.hyperparams['nu'], kern.hyperparams['scale'], kern.hyperparams['dim_bandwidths'])
    return O.OGP(np.array(Xl), np.array(Yl), ok, mean, noise)
  np.random.seed(5)
  res = hp_grid.fit_gp(X, Y, layout, g[method + '_bounds'], g[method + '_dscr_vals'], method=method,
                       max_evals=int(g[method + '_max_evals']), gp_factory=oracle_gp)
  if method == 'rand_exp_sampling':
    tag, cts, dscr, other, probs = res
    assert tag == 'sample_hps_with_probs' and other == [None] * len(cts)
    assert (cts == g[method + '_cts']).all() and (np.array(dscr) == g[method + '_dscr']).all()
    np.testing.assert_allclose(probs, g[method + '_probs'], rtol=1e-9, atol=1e-15)
    assert calls == [len(cts)]                                # every sample in ONE batched call
  else:
    tag, gp, (cts, dscr) = res
    assert tag == 'fitted_gp'
    assert (np.array(cts) == g[method + '_cts']).all() and (np.array(dscr) == g[method + '_dscr']).all()
    np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[method + '_lml']), rtol=1e-12)
    mu, sd = gp.eval(g[method + '_C'], 'std')
    np.testing.assert_allclose(mu, g[method + '_mu'], atol=1e-10)
    np.testing.assert_allclose(sd, g[method + '_sd'], atol=1e-9)
    if method == 'rand':
      assert calls == [int(g[method + '_max_evals'])] * 3     # one batch per discrete nu
    else:
      assert max(calls) <= 2                                  # PDOO: the two children of a split per call
  # the bounds the reference's fitter derives from the data (gp_core.py:396-416, euclidean_gp.py:253-276)
  b, dv = hp_grid.EuclideanHPLayout(3, 'matern', nu=-1.0, mean_func_type=str(g['mean_func_type']),
                                    noise_var_type=str(g['noise_var_type'])).bounds(X, Y)
  assert (b == g[method + '_bounds']).all() and (np.array(dv) == g[method + '_dscr_vals']).all()
  assert hp_grid.default_max_evals('rand', 8) == 1600 and hp_grid.default_max_evals('pdoo', 8) == 500
  assert hp_grid.default_max_evals('rand_exp_sampling', 8) == 3200


# ---- property tests of the multi-rank arg-max reduction (no process group needed) ---------------------------------
def test_sharded_reduction_equals_numpy_argmax_property():
  """ For any score vector (ties, NaNs, infinities) and any number of ranks, reducing the per-shard winners with
      dist.reduce_pairs gives np.argmax of the whole vector. """
  from hypothesis import given, settings, strategies as st
  from dragonfly_b200 import dist as D

  vals = st.one_of(st.floats(allow_nan=True, allow_infinity=True, width=64),
                   st.sampled_from([0.0, 1.0, -1.0, 7.5]))          # plenty of exact ties

  @settings(max_examples=300, deadline=None)
  @given(st.lists(vals, min_size=1, max_size=60), st.integers(min_value=1, max_value=9))
  def check(scores, world):
    s = np.array(scores, dtype=np.float64)
    winners_s, winners_i = [], []
    for r in range(world):
      lo, hi = D.shard_bounds(len(s), r, world)
      if hi > lo:
        j = int(np.argmax(s[lo:hi]))
        winners_s.append(s[lo + j]); winners_i.append(lo + j)
      else:
        winners_s.append(0.0); winners_i.append(-1)
    _, idx = D.reduce_pairs(winners_s, winners_i)
    assert idx == int(np.argmax(s))
  check()
  # the K-at-once variant without a process group is the identity
  sc, ix = D.all_reduce_argmax_many([1.0, np.nan], [4, 9])
  assert sc[0] == 1.0 and np.isnan(sc[1]) and ix.tolist() == [4, 9]


def test_fit_gp_through_the_lane_machinery_with_a_numpy_device(monkeypatch):
  """ hp_grid.fit_gp -> lml_for_hyperparams with 3 concurrent lanes (threads, one posterior each), per-sample Matern
      nu and a tuned mean (set_train per sample) -- everything except CUDA itself: DevicePosterior is replaced by a
      NumPy stand-in and torch.cuda's stream / device context managers by no-ops.  Same selections as the reference. """
  import contextlib
  import threading
  import torch
  from conftest import load_golden
  from dragonfly_b200 import hp_grid, device as dfb_device
  g = load_golden('fitter')
  X, Y = g['X'], g['Y']
  seen_threads, builds = set(), []

  class FakeDevice(object):
    index = 0

  class LanePost(object):
    def __init__(self, n_max, device=None):
      self.n_max, self.device = n_max, FakeDevice()

    def bind_current_stream(self):
      seen_threads.add(threading.get_ident())

    def set_train(self, Xm, yc):
      self.X, self.yc = np.array(Xm), np.array(yc)

    def set_kernel(self, kern):                      # build_descriptor is patched to hand the kernel object through
      self.kern = O.OMaternKernel(3, kern.hyperparams['nu'], kern.hyperparams['scale'],
                                  kern.hyperparams['dim_bandwidths'])

    def build(self, noise_var, jitter, flags):
      assert flags == hp_grid._lib.DFB_BUILD_LML_ONLY
      builds.append(threading.get_ident())
      gp = O.OGP(self.X, self.yc, self.kern, lambda x: np.zeros(len(x)), noise_var + jitter)
      return 0, gp.compute_log_marginal_likelihood()

  class FakeStream(object):
    def __init__(self, *a, **k):
      pass

    def wait_stream(self, other):
      pass
  monkeypatch.setattr(dfb_device, 'DevicePosterior', LanePost)
  monkeypatch.setattr(hp_grid, 'build_descriptor', lambda kern, **kw: kern)
  monkeypatch.setattr(torch.cuda, 'current_stream', lambda *a, **k: FakeStream())
  monkeypatch.setattr(torch.cuda, 'Stream', FakeStream)
  monkeypatch.setattr(torch.cuda, 'device', lambda *a, **k: contextlib.nullcontext())
  monkeypatch.setattr(torch.cuda, 'stream', lambda *a, **k: contextlib.nullcontext())
  layout = hp_grid.EuclideanHPLayout(3, 'matern', mean_func_type=str(g['mean_func_type']),
                                     noise_var_type=str(g['noise_var_type']))
  oracle_gp = lambda Xl, Yl, kern, mean, noise: O.OGP(
      np.array(Xl), np.array(Yl), O.OMaternKernel(3, kern.hyperparams['nu'], kern.hyperparams['scale'],
                                                  kern.hyperparams['dim_bandwidths']), mean, noise)
  np.random.seed(5)
  tag, gp, (cts, dscr) = hp_grid.fit_gp(X, Y, layout, g['rand_bounds'], g['rand_dscr_vals'], method='rand',
                                        max_evals=int(g['rand_max_evals']), gp_factory=oracle_gp)
  assert (np.array(cts) == g['rand_cts']).all() and (np.array(dscr) == g['rand_dscr']).all()
  assert len(seen_threads) == 3 and len(set(builds)) == 3 and len(builds) == 3 * int(g['rand_max_evals'])
  np.random.seed(5)
  tag, cts, dscr, other, probs = hp_grid.fit_gp(X, Y, layout, g['rand_exp_sampling_bounds'],
                                                g['rand_exp_sampling_dscr_vals'], method='rand_exp_sampling',
                                                max_evals=int(g['rand_exp_sampling_max_evals']))
  assert (cts == g['rand_exp_sampling_cts']).all()
  np.testing.assert_allclose(probs, g['rand_exp_sampling_probs'], rtol=1e-9, atol=1e-15)
  del builds[:]
  tag, gp, (cts, dscr) = hp_grid.fit_gp(X, Y, layout, g['pdoo_bounds'], g['pdoo_dscr_vals'], method='pdoo',
                                        max_evals=int(g['pdoo_max_evals']), gp_factory=oracle_gp)
  assert (np.array(cts) == g['pdoo_cts']).all() and (np.array(dscr) == g['pdoo_dscr']).all()
  assert len(set(builds)) == 1                       # batches of <= 2 hp vectors stay on the calling thread
  # an exception inside a lane surfaces in the caller
  def boom(self, noise_var, jitter, flags):
    raise RuntimeError('lane failure')
  monkeypatch.setattr(LanePost, 'build', boom)
  with pytest.raises(RuntimeError):
    hp_grid.lml_for_hyperparams(X, Y, np.tile((g['rand_bounds'][:, 0] + g['rand_bounds'][:, 1]) / 2, (9, 1)), layout,
                                nus=[2.5] * 9, lanes=3)


def _oracle_kernel_of(kern):
  """ Our kernel mirror -> the oracle's kernel object (plain Matern or additive of Materns). """
  if hasattr(kern, 'kernel_list'):
    return O.OAdditiveKernel(kern.hyperparams['scale'],
                             [O.OMaternKernel(k.dim, k.hyperparams['nu'], k.hyperparams['scale'],
                                              k.hyperparams['dim_bandwidths']) for k in kern.kernel_list],
                             kern.groupings)
  return O.OMaternKernel(kern.dim, kern.hyperparams['nu'], kern.hyperparams['scale'],
                         kern.hyperparams['dim_bandwidths'])


@pytest.mark.parametrize('method', ['rand', 'rand_exp_sampling'])
def test_fit_gp_additive_model_matches_the_reference_fitter(method, monkeypatch):
  """ use_additive_gp (euclidean_gp.py:243-248, 718-776; kernels :826-897): random groupings per objective
      evaluation, the group size as a discrete hyper-parameter -- against golden fitter_add.npz (the reference's
      EuclideanGPFitter under np.random.seed(7)); LMLs from the oracle. """
  from conftest import load_golden
  from dragonfly_b200 import hp_grid
  g = load_golden('fitter_add')
  X, Y = g['X'], g['Y']
  layout = hp_grid.EuclideanHPLayout(5, 'matern', nu=-1.0, mean_func_type=str(g['mean_func_type']),
                                     noise_var_type=str(g['noise_var_type']), use_additive_gp=True,
                                     add_max_group_size=3, num_groups_per_group_size=2)
  b, dv = layout.bounds(X, Y)
  assert (b == g[method + '_bounds']).all()
  assert dv == [list(g[method + '_dscr_vals_nu']), [int(v) for v in g[method + '_dscr_vals_grp']]]

  def oracle_lmls(X_, Y_, hps, layout_, nus=None, post=None, device=None, lanes=None, groupings=None):
    out = []
    for i, hp in enumerate(hps):
      m, nv, k = layout_.unpack(hp, Y_, None if nus is None else nus[i], None if groupings is None else groupings[i])
      out.append(O.OGP(X_, Y_, _oracle_kernel_of(k), lambda x, c=m: np.array([c] * len(x)),
                       nv).compute_log_marginal_likelihood())
    return np.array(out), post
  monkeypatch.setattr(hp_grid, 'lml_for_hyperparams', oracle_lmls)
  oracle_gp = lambda Xl, Yl, kern, mean, noise: O.OGP(np.array(Xl), np.array(Yl), _oracle_kernel_of(kern), mean, noise)
  np.random.seed(7)
  res = hp_grid.fit_gp(X, Y, layout, b, dv, method=method, max_evals=int(g[method + '_max_evals']),
                       gp_factory=oracle_gp)
  unpad = lambda rows: [[int(v) for v in r if v >= 0] for r in rows if (np.asarray(r) >= 0).any()]
  if method == 'rand':
    tag, gp, (cts, dscr) = res
    assert tag == 'fitted_gp'
    assert (np.array(cts) == g['rand_cts']).all() and (np.array(dscr, dtype=np.float64) == g['rand_dscr']).all()
    assert [list(map(int, grp)) for grp in gp.kernel.groupings] == unpad(g['rand_groupings'])
    np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g['rand_lml']), rtol=1e-12)
    mu, sd = gp.eval(g['rand_C'], 'std')
    np.testing.assert_allclose(mu, g['rand_mu'], atol=1e-10)
    np.testing.assert_allclose(sd, g['rand_sd'], atol=1e-9)
  else:
    tag, cts, dscr, other, probs = res
    groupings = [o.add_gp_groupings for o in other]
    assert tag == 'sample_hps_with_probs'
    assert (np.array(cts) == g[method + '_cts']).all()
    assert (np.array(dscr, dtype=np.float64) == g[method + '_dscr']).all()
    assert [[list(map(int, grp)) for grp in gs] for gs in groupings] == [unpad(gs) for gs in g[method + '_groupings']]
    np.testing.assert_allclose(probs, g[method + '_probs'], rtol=1e-9, atol=1e-300)


def test_se_effective_norm_known_answers():
  """ dragonfly/gp/unittest_kernel.py:153-176 (test_effective_length_se), restated. """
  data_1, data_2 = np.array([1, 2]), np.array([[0, 1, 2], [1, 1, 0.5]])
  k1, k2 = K.SEKernel(2, 1, [0.1, 1]), K.SEKernel(3, 1, [0.5, 1, 2])
  assert abs(k1.get_effective_norm(data_1, order=2, is_single=True) - np.sqrt(104)) < 1e-5
  assert abs(k1.get_effective_norm(data_1, order=1, is_single=True) - 12) < 1e-5
  assert np.linalg.norm(k2.get_effective_norm(data_2, order=2, is_single=False) -
                        np.array([np.sqrt(2), np.sqrt(5.0625)])) < 1e-5
  assert np.linalg.norm(k2.get_effective_norm(data_2, order=1, is_single=False) - np.array([2, 3.25])) < 1e-5
  k2.change_smoothness(2.0)
  assert (k2.hyperparams['dim_bandwidths'] == np.array([1.0, 2.0, 4.0])).all()


def test_mf_hp_layout_unpacks_like_the_reference_mf_fitter():
  """ euclidean_gp.py:680-709: [mean]? [log noise]? log scale, log fidelity bandwidths, log domain bandwidths; fidelity
      coordinates first in the [z || x] rows; a tuned Matern nu goes to whichever of the two kernels tunes it. """
  from dragonfly_b200 import hp_grid
  lay = hp_grid.EuclideanMFHPLayout(1, 3, 'se', 'matern', domain_nu=-1.0, mean_func_type='tune', noise_var_type='tune')
  assert lay.num_hps() == 7 and lay.tuned_nus() == [False, True] and lay.dim == 4
  hp = [0.3, np.log(0.02), np.log(1.7), np.log(0.6), np.log(0.2), np.log(0.3), np.log(0.4)]
  m, nv, kern = lay.unpack(hp, np.arange(5.0), nu=1.5)
  assert m == 0.3 and abs(nv - 0.02) < 1e-15 and abs(kern.hyperparams['scale'] - 1.7) < 1e-15
  kF, kD = kern.kernel_list
  assert type(kF).__name__ == 'SEKernel' and type(kD).__name__ == 'MaternKernel' and kD.hyperparams['nu'] == 1.5
  np.testing.assert_allclose(kF.hyperparams['dim_bandwidths'], [0.6])
  np.testing.assert_allclose(kD.hyperparams['dim_bandwidths'], [0.2, 0.3, 0.4])
  assert kF.hyperparams['scale'] == 1.0 and kD.hyperparams['scale'] == 1.0
  assert kern.coordinate_list == [[0], [1, 2, 3]]
  same = hp_grid.EuclideanMFHPLayout(2, 2, 'matern', 'se', fidel_nu=2.5, fidel_use_same_bandwidth=True,
                                     mean_func_type='median', noise_var_type='value', noise_var_value=0.07)
  m, nv, kern = same.unpack([np.log(2.0), np.log(0.5), np.log(0.1), np.log(0.9)], np.array([1.0, 5.0, 2.0]))
  assert m == 2.0 and nv == 0.07 and same.num_hps() == 4
  np.testing.assert_allclose(kern.kernel_list[0].hyperparams['dim_bandwidths'], [0.5, 0.5])
  np.testing.assert_allclose(kern.kernel_list[1].hyperparams['dim_bandwidths'], [0.1, 0.9])
  assert kern.kernel_list[0].hyperparams['nu'] == 2.5
  with pytest.raises(NotImplementedError):
    hp_grid.EuclideanMFHPLayout(1, 2, 'expdecay', 'se')


def test_streamed_draw_schedule_covers_every_row_once_and_matches_the_single_draw():
  """ gpb_acquisitions._slab_schedule / _maximise_streamed: short slabs first, whole slabs after; the concatenation of
      the slab draws IS np.random.random((M, d)) (same global MT19937 consumption as oper_utils.py:59-67). """
  from dragonfly_b200 import gpb_acquisitions as A
  for M, slab, unit in [(1000000, 130560, 6528), (50000, 130560, 6528), (13056, 13056, 6528), (7, 100, 0), (1001, 300, 0)]:
    sch = A._slab_schedule(M, slab, unit)
    assert sch[0][0] == 0 and sum(r for _, r in sch) == M
    assert all(sch[i][0] + sch[i][1] == sch[i + 1][0] for i in range(len(sch) - 1))
    assert all(r <= slab for _, r in sch)
  assert [r for _, r in A._slab_schedule(1000000, 261120, 6528)[:4]] == [13056, 52224, 208896, 261120]
  bounds = np.array([[-1.0, 2.0], [0.0, 5.0], [3.0, 4.0]])
  seen = []

  def scorer(pts):
    seen.append(np.array(pts))
    vals = pts[:, 0] - pts[:, 1] * pts[:, 2]
    i = int(np.argmax(vals))
    return vals[i], i, None
  np.random.seed(11)
  pt = A._maximise_streamed(scorer, bounds, 2500, 600, unit=100)
  after = np.random.random()
  np.random.seed(11)
  ref = A.draw_candidates(bounds, 2500)
  assert np.random.random() == after
  assert (np.concatenate(seen) == ref).all() and [len(x) for x in seen] == [200, 600, 600, 600, 500]          # 2 units, then the x4 slab would reach the slab size
  vals = ref[:, 0] - ref[:, 1] * ref[:, 2]
  assert (pt == ref[int(np.argmax(vals))]).all()
