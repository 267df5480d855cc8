"""
The descriptor interpreter (kernels.cu: kernel_rows, behind kstar_kernel, dfb_kernel_matrix and lml_batch_kernel) on
every construct the plain K_* producers do not cover, against the extended-precision reference of tests/interp_ref.py
(where the bounds are derived) and bit for bit across every site that evaluates it (-m gpu).  The catalogue
(interp_ref.catalogue): SE and Matern 1/2 .. 5/2 at d = 9 .. 128, Matern 7/2, additive kernels up to 48 terms, products
up to 48 factors on 128 slots and over an additive child, POLY of order 0 .. 7, EXPDECAY on every numpy_scalar_pow path,
Cartesian products with HAMMING factors; coincident and nearly coincident points, bandwidths that flush and bandwidths
that make K ~ scale; n and m on the 16-row, 32-lane and 128-tile edges.

Bounded checks:
  B1  every entry of dfb_kernel_matrix(Xc, X) lies within the bound;
  B2  mu of dfb_eval (score_impl = 0) lies within kstar_ref.mu_bound, with the device's own alpha and B1's bound;
  B3  k(x*, x*) of dfb_eval (the handle's kssv) lies within the bound of the exact k(x*, x*).
Exact invariants (bit equality, int64 views):
  E1  dfb_kernel_matrix(X, X) is symmetric;
  E2  the K the build factorised is dfb_kernel_matrix(X, X): the top's tiles right of the diagonal tile of T keep it,
      and dfb_get_state's K;
  E3  the fp64 scoring rows of a one-chunk dfb_eval are dfb_kernel_matrix(Xc, X); their padding is exact zeros;
  E4  kssv is the diagonal of dfb_kernel_matrix(Xc, Xc);
  E5  after dfb_extend_posterior, dfb_get_state's K is dfb_kernel_matrix of the extended set; for a non-stationary
      kernel max_diag() is its largest diagonal entry plus the noise;
  E6  dfb_lml_batch (dfb_lml_batch_mixed for HAMMING) gives the LML of dfb_build_posterior(DFB_BUILD_LML_ONLY):
      kernel_rows<1> and kernel_rows<2> agree;
  E7  the Add-UCB test kernel (candidate columns 0 .. d-1 against permuted training columns g) gives the K_* rows of
      dfb_kernel_matrix of the same kernel on (Xc, X[:, g]);
  E8  HAMMING blocks are NumPy's (np.equal(a, b) * w).sum(axis=1), at dims 1 .. 9, 15, 16, 17, 24, 31, 64 and 128.
Measured: the whole file (159 tests) runs in 30 s on one H100 80 GB, 10 s of it the library's first load.
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import interp_ref as IR
import kstar_ref as KR
from dragonfly_b200 import kernel as K
from dragonfly_b200.cartesian_product_gp import CartesianProductKernel

pytestmark = pytest.mark.gpu

TILE = 128
CHUNK = 512
CASES = IR.catalogue(K, CartesianProductKernel)


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  assert np.finfo(np.longdouble).nmant >= 63, 'the reference needs an extended long double'
  from dragonfly_b200 import device, _lib
  _lib.load()
  return Namespace(torch=torch, device=device, lib=_lib)


def _copy(G, post, name, shape):
  t = G.torch.empty(shape, dtype=G.torch.float64, device=post.device)
  G.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), t.numel() * 8), 'dfb_debug_copy')
  return t.cpu().numpy()


def _bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _assert_bits_equal(a, b, what):
  ia, ib = _bits(a), _bits(b)
  assert ia.shape == ib.shape, (what, ia.shape, ib.shape)
  bad = np.argwhere(ia != ib)
  assert len(bad) == 0, (what, 'differs in', len(bad), 'entries; first', tuple(bad[0]),
                         np.asarray(a)[tuple(bad[0])], np.asarray(b)[tuple(bad[0])])


def _assert_within(vals, exact, B, what):
  err = np.abs(np.asarray(vals, dtype=np.float64).astype(np.longdouble) - exact).astype(np.float64)
  assert (err <= B).all(), (what, float(np.max(err / B)), np.unravel_index(np.argmax(err / B), err.shape))


def _noise(case, Kxx):
  """ 5 % of the largest |K_ij| for a PSD kernel; above n max |K_ij| >= ||K||_2 for the ExpDecay kernels with a
      negative power (not PSD), so that every build is positive definite """
  top = float(np.max(np.abs(Kxx)))
  return 0.05 * top if case.psd else 1.01 * case.n * top


def _post(G, n_max):
  post = G.device.DevicePosterior((n_max + TILE - 1) // TILE * TILE, chunk=CHUNK)
  post.set_option('score_impl', 0)
  return post


@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_interpreter(G, case):
  kern, X, Xc, D, n, m = case.kern, case.X, case.Xc, case.D, case.n, case.m
  km = lambda A, B: G.device.kernel_matrix(kern, A, B)
  K_cx, K_xx, K_cc = km(Xc, X), km(X, X), km(Xc, Xc)
  K_ex, B = IR.evaluate(kern, Xc, X)
  # B1, E1
  _assert_within(K_cx, K_ex, B, 'B1')
  _assert_bits_equal(K_xx, K_xx.T, 'E1 K(X, X) symmetric')

  desc = K.build_descriptor(kern, train_dim=D, cand_dim=D)
  stationary = K.is_stationary(desc)
  noise = _noise(case, K_xx)
  y = np.random.RandomState(n + m).standard_normal(n)
  post = _post(G, n)
  post.set_kernel(desc)
  post.set_train(X, y)
  info, _ = post.build(noise)
  assert info == 0
  npad = int(post.query('npad'))
  # E2
  _, alpha, Kst = post.get_state(want_alpha=True, want_K=True)
  alpha = alpha.cpu().numpy()
  _assert_bits_equal(Kst.cpu().numpy(), K_xx, 'E2 dfb_get_state K')
  T = _copy(G, post, 'T', (2 * npad + TILE, npad))
  for I in range(npad // TILE):
    r, c0 = slice(I * TILE, min((I + 1) * TILE, n)), (I + 1) * TILE
    if c0 < n:
      _assert_bits_equal(T[r, c0:n], K_xx[r, c0:n], 'E2 factorised K, row block %d' % I)
  if not stationary:
    assert post.max_diag() == float(np.max(np.diag(K_xx))) + noise, 'max_diag'

  # E3, E4, B2, B3: one chunk of candidates
  mu, _ = post.eval(Xc, mean_const=0.0)
  assert post.query('last_used_i8') == 0.0
  Ks = _copy(G, post, 'Ks', (CHUNK, npad))
  m_rows = (m + TILE - 1) // TILE * TILE
  _assert_bits_equal(Ks[:m, :n], K_cx, 'E3 scoring rows')
  assert (_bits(Ks[:m_rows, n:]) == 0).all() and (_bits(Ks[m:m_rows]) == 0).all(), 'E3 padding'
  kssv = _copy(G, post, 'kssv', (CHUNK,))[:m]
  _assert_bits_equal(kssv, np.diag(K_cc), 'E4 kssv')
  mb = KR.mu_bound(alpha, K_cx, B)
  mu_ex = (K_ex * alpha.astype(np.longdouble)).sum(axis=1)
  _assert_within(mu, mu_ex, mb, 'B2')
  d_ex, d_B = IR.evaluate(kern, Xc, Xc, diag=True)
  _assert_within(kssv, d_ex, d_B, 'B3')

  # E6: the batched LML-only build against the handle's
  info, lml = post.build(noise, 0.0, G.lib.DFB_BUILD_LML_ONLY)
  assert info == 0
  lmls, infos = post.lml_batch([desc], [noise], [0.0], mixed=case.hamming)
  assert infos[0] == 0
  _assert_bits_equal(lmls, np.array([lml]), 'E6 lml_batch')

  # E5: extend by up to 16 points within the padded size
  q = min(16, npad - n)
  if q > 0:
    info, _ = post.build(noise)
    assert info == 0
    Xn = case.Xext[:q]
    info, _ = post.extend(Xn, np.random.RandomState(q).standard_normal(q))
    assert info == 0
    Xall = np.vstack([X, Xn])
    K_all = km(Xall, Xall)
    _assert_bits_equal(post.get_state(want_K=True)[2].cpu().numpy(), K_all, 'E5 extended K')
    if not stationary:
      assert post.max_diag() == float(np.max(np.diag(K_all))) + noise, 'E5 max_diag'


# ---- E7: the Add-UCB test kernel --------------------------------------------------------------------------------------
E7_CASES = [c for c in CASES if not c.hamming and c.D <= 17]


@pytest.mark.parametrize('case', E7_CASES, ids=[c.name for c in E7_CASES])
def test_test_kernel_on_permuted_training_columns(G, case):
  kern, D, n, m = case.kern, case.D, case.n, case.m
  rs = np.random.RandomState(D + n)
  Dw = D + 3
  g = [int(c) for c in rs.permutation(Dw)[:D]]
  Xw = rs.random_sample((n, Dw)) * (case.X.max() - case.X.min()) + case.X.min()
  Xw[:, g] = case.X
  post = _post(G, n)
  post.set_kernel(K.build_descriptor(K.SEKernel(Dw, 1.0, [0.7] * Dw), train_dim=Dw, cand_dim=Dw))
  post.set_train(Xw, rs.standard_normal(n))
  info, _ = post.build(0.05)
  assert info == 0
  post.set_test_kernel(K.build_descriptor(kern, train_dim=Dw, cand_dim=D, train_coords=g, cand_coords=list(range(D))))
  post.eval(case.Xc, mean_const=0.0)
  npad = int(post.query('npad'))
  Ks = _copy(G, post, 'Ks', (CHUNK, npad))[:m, :n]
  _assert_bits_equal(Ks, G.device.kernel_matrix(kern, case.Xc, case.X), 'E7 test-kernel rows')
  K_ex, B = IR.evaluate(kern, case.Xc, Xw, cols2=g)
  _assert_within(Ks, K_ex, B, 'E7 B1')


# ---- E8: HAMMING blocks against NumPy's own sum ---------------------------------------------------------------------------
@pytest.mark.parametrize('d', list(range(1, 10)) + [15, 16, 17, 24, 31, 64, 128])
def test_hamming_blocks_are_numpys_sum(G, d):
  rs = np.random.RandomState(40 + d)
  w = 2.0 ** rs.uniform(-20, 20, size=d)
  n, m = 160, 129
  X = rs.randint(0, 2, size=(n, d)).astype(np.float64)
  Xc = rs.randint(0, 2, size=(m, d)).astype(np.float64)
  Xc[:16] = X[:16]
  got = G.device.kernel_matrix(K.HammingKernel(list(w)), Xc, X)
  want = (np.equal(Xc[:, None, :], X[None, :, :]) * w).sum(axis=2)
  _assert_bits_equal(got, want, 'E8 Hamming d=%d' % d)
