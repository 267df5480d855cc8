"""
The fp64 contraction bounds of tests/contract_ref.py on the CPU: fp64 evaluations in several orders (BLAS, 16-wide
k-slabs as the DMMA ring runs them, and FMA chains through i8_exact.fma_vec) meet every bound with margin, each defect a
broken tiling would produce violates one by a wide factor, and the bounds are tight enough to mean something.
"""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

import contract_ref as CR
import i8_exact as IX
import kstar_ref as KR

T = CR.T
MARGIN = 0.5          # a bound that holds must hold with at least this much to spare
WIDE = 10.0           # a defect must exceed its bound by at least this factor
TIGHT = 1e-10         # bound / |value| on well-conditioned inputs


def test_long_double_is_extended():
  assert np.finfo(np.longdouble).nmant >= 63


class Case(object):
  """ An SE posterior: W = L^-1 with identity padding, the K_* rows of m candidates (zero padding) and k(x, x). """

  def __init__(self, n, m, seed=0, noise=1e-2):
    rs = np.random.RandomState(1000 * n + m + seed)
    self.bw, self.scale = np.array([0.4, 0.5, 0.3]), 1.3
    self.X, self.Xc = rs.random_sample((n, 3)), rs.random_sample((m, 3))
    self.n, self.m = n, m
    self.npad = -(-n // T) * T
    self.mpad = -(-m // T) * T
    K = self.kern(self.X, self.X) + noise * np.eye(n)
    L = np.linalg.cholesky(K)
    self.W = np.eye(self.npad)
    self.W[:n, :n] = np.tril(solve_triangular(L, np.eye(n), lower=True))
    self.Ks = np.zeros((self.mpad, self.npad))
    self.Ks[:m, :n] = self.kern(self.Xc, self.X)
    self.kss = np.full(m, self.scale)

  def kern(self, A, B):
    return KR.kernel_exact('se', 0, self.scale, self.bw, A, B).astype(np.float64)


# ---- fp64 evaluations in several orders --------------------------------------------------------------------------------
def product(A, B, order):
  """ A B^T in fp64: 'blas', 'slab' (16-wide k-slabs added in turn, as the DMMA ring does), 'fma' (one FMA chain). """
  if order == 'blas':
    return A @ B.T
  out = np.zeros((A.shape[0], B.shape[0]))
  if order == 'slab':
    for k0 in range(0, A.shape[1], 16):
      out = out + A[:, k0:k0 + 16] @ B[:, k0:k0 + 16].T
    return out
  for k in range(A.shape[1]):
    out = IX.fma_vec(A[:, k][:, None], B[:, k][None, :], out)
  return out


def partials(W, Ks, order, defect=None):
  """ The score partials (nb x mpad) in fp64, with an optional defect. """
  npad = W.shape[0]
  nb = npad // T
  P = np.zeros((nb, Ks.shape[0]))
  for rb in range(nb):
    kh = CR.k_hi(rb, npad)
    Wr, Kr = W[rb * T:(rb + 1) * T, :kh], Ks[:, :kh]
    if defect == 'drop_slab' and rb == nb - 1:
      Wr, Kr = Wr[:, 16:], Kr[:, 16:]
    if defect == 'short_range' and rb == nb - 1:
      Wr, Kr = Wr[:, :kh - T], Kr[:, :kh - T]
    v = product(Wr, Kr, order)
    P[rb] = (v * v).sum(axis=0)
  if defect == 'block_twice':
    P[-1] = P[-1] + P[0]
  return P


ORDERS = ['blas', 'slab', 'fma']


@pytest.mark.parametrize('order', ORDERS)
@pytest.mark.parametrize('n', [1, 127, 129, 300])
def test_score_partials_meet_the_bound(n, order):
  c = Case(n, 130)
  P = partials(c.W, c.Ks, order)
  Pe, B = CR.score_partials(c.W, c.Ks)
  assert CR._ratio(CR._ld(P) - Pe, B) <= MARGIN


@pytest.mark.parametrize('order', ORDERS)
def test_small_partials_meet_the_bound(order):
  c = Case(200, 9)
  v = product(np.tril(c.W[:200, :200]), c.Ks[:9, :200], order)
  Pe, B = CR.small_partials(c.W, c.Ks, 200, np.arange(9))
  assert CR._ratio(CR._ld(v * v) - Pe, B) <= MARGIN


def test_epilogue_is_the_reference_fold():
  rs = np.random.RandomState(3)
  P = rs.random_sample((5, 40)) * 0.1
  kss = np.full(40, 0.25)
  var, sd = CR.epilogue(P, kss)
  vn = (((P[0] + P[1]) + P[2]) + P[3]) + P[4]
  assert np.array_equal(var, kss - vn)
  assert np.isnan(sd[var < 0]).all() and np.array_equal(sd[var >= 0], np.sqrt(var[var >= 0]))


@pytest.mark.parametrize('tri', [0, 1, 2, 3])
@pytest.mark.parametrize('order', ORDERS)
def test_generic_products_meet_the_bound(tri, order):
  rs = np.random.RandomState(tri)
  A, B, C = rs.standard_normal((256, 384)), rs.standard_normal((384, 384)), rs.standard_normal((256, 384))
  D = np.zeros((256, 384))
  for r in range(2):
    for c in range(3):
      lo, hi = CR.k_range(tri, r + 1, c, 384)
      rs_, cs = slice(r * T, (r + 1) * T), slice(c * T, (c + 1) * T)
      D[rs_, cs] = -1.0 * product(A[rs_, lo:hi], B[cs, lo:hi], order) + C[rs_, cs]
  assert CR.generic_check(A, B, D, alpha=-1.0, C=C, tri=tri, rb0=1) <= MARGIN


@pytest.mark.parametrize('order', ORDERS)
def test_covariance_meets_the_bound(order):
  c = Case(300, 140)
  V = product(c.Ks[:140], c.W, order)
  Cov = c.kern(c.Xc, c.Xc) - product(V, V, order)
  assert CR.covariance_check(Cov, c.Ks[:140], c.W, ('se', 0, c.scale, c.bw, c.Xc)) <= MARGIN


@pytest.mark.parametrize('order', ORDERS)
def test_factor_and_draws_meet_the_bound(order):
  c = Case(300, 200)
  Cov = c.kern(c.Xc, c.Xc) + 1e-3 * np.eye(200)
  A = np.eye(256)
  A[:200, :200] = Cov
  L = np.linalg.cholesky(A)
  assert CR.factor_check(A, L) <= MARGIN
  Ut = np.random.RandomState(1).standard_normal((5, 200))
  mu = np.linspace(-1, 1, 200)
  S = product(Ut, L[:200, :200], order) + mu
  assert CR.draws_check(S, mu, Ut, L[:200, :200]) <= MARGIN


# ---- defects ----------------------------------------------------------------------------------------------------------
def test_dropped_slab_and_short_range_and_block_twice_are_caught():
  c = Case(300, 130)
  Pe, B = CR.score_partials(c.W, c.Ks)
  for defect in ('drop_slab', 'short_range'):
    r = CR._ratio(CR._ld(partials(c.W, c.Ks, 'blas', defect)) - Pe, B)
    assert r >= WIDE, (defect, r)
  # one row block counted twice: sigma^2 from the folded partials against the exact sum
  P = partials(c.W, c.Ks, 'blas', 'block_twice')
  var, _ = CR.epilogue(P[:, :130], c.kss)
  exact = CR._ld(c.kss) - Pe[:, :130].sum(axis=0)
  bnd = B[:, :130].sum(axis=0) + CR.gamma(P.shape[0] + 1) * (np.abs(P[:, :130]).sum(axis=0) + c.kss)
  assert CR._ratio(CR._ld(var) - exact, bnd) >= WIDE


def test_stale_padding_row_of_W_is_caught():
  c = Case(200, 130)
  Wst = c.W.copy()
  Wst[230, :200] = 1e-3                    # a padding row (i >= n) with stale values left of its diagonal
  Pe, B = CR.score_partials(c.W, c.Ks)
  r = CR._ratio(CR._ld(partials(Wst, c.Ks, 'blas')) - Pe, B)
  assert r >= WIDE, r


def test_long_range_and_skipped_tile_are_caught():
  rs = np.random.RandomState(7)
  A, B = rs.standard_normal((384, 384)), rs.standard_normal((384, 384))
  # tri = 1 with a range one tile long over non-zero data (A is full, not triangular)
  D = np.zeros((384, 384))
  for r in range(3):
    for c in range(3):
      lo, hi = CR.k_range(1, r, c, 384)
      hi = min(384, hi + T) if (r, c) == (1, 2) else hi
      D[r * T:(r + 1) * T, c * T:(c + 1) * T] = A[r * T:(r + 1) * T, lo:hi] @ B[c * T:(c + 1) * T, lo:hi].T
  assert CR.generic_check(A, B, D, tri=1) >= WIDE
  # lower_only with one lower tile never written (left at zero)
  D = np.tril(np.ones((3, 3))).repeat(T, 0).repeat(T, 1) * (A @ B.T)
  assert CR.generic_check(A, B, D, lower_only=True) <= MARGIN
  D[2 * T:, T:2 * T] = 0.0
  assert CR.generic_check(A, B, D, lower_only=True) >= WIDE


def test_transposed_covariance_tile_is_caught():
  c = Case(300, 256)
  V = c.Ks[:256] @ c.W.T
  Cov = c.kern(c.Xc, c.Xc) - V @ V.T
  kern = ('se', 0, c.scale, c.bw, c.Xc)
  assert CR.covariance_check(Cov, c.Ks[:256], c.W, kern) <= MARGIN
  Cov[T:, :T] = Cov[T:, :T].T.copy()
  assert CR.covariance_check(Cov, c.Ks[:256], c.W, kern) >= WIDE


def test_bounds_are_tight_on_well_conditioned_inputs():
  c = Case(300, 130, noise=0.5)
  Pe, B = CR.score_partials(c.W, c.Ks[:130])
  assert (B / np.abs(Pe.astype(np.float64)).clip(1e-300)).max() <= TIGHT
  rs = np.random.RandomState(2)
  A, Bm = rs.random_sample((128, 256)), rs.random_sample((128, 256))
  S, bnd = CR._product_tile(A, Bm, 1.0, None, 256)
  assert (bnd / np.abs(S.astype(np.float64))).max() <= TIGHT


# ---- LML gradients -----------------------------------------------------------------------------------------------------------
KINDS = [('se', 0), ('matern', 0), ('matern', 1), ('matern', 2)]


def grad_terms(kind, p, scale, bw, X, Kinv, alpha):
  """ fp64 M and G_p in lml_grad_tile_kernel's form: D2 and d2_q from the norm expansion of the scaled coordinates. """
  n, d = X.shape
  xs = X / bw
  nrm = (xs * xs).sum(axis=1)
  D2 = np.maximum((nrm[None, :] + nrm[:, None]) - 2.0 * (xs @ xs.T), 0.0)
  dsq = [np.maximum((xs[:, q][None, :] ** 2 + xs[:, q][:, None] ** 2) - 2.0 * np.outer(xs[:, q], xs[:, q]), 0.0)
         for q in range(d)]
  M = np.outer(alpha, alpha) - Kinv
  off = ~np.eye(n, dtype=bool)
  if kind == 'se':
    base = scale * np.exp(D2 * -0.5)
    Gs = [base, base * (D2 / bw[0])] + [base * (dsq[q] / bw[q]) for q in range(d)]
  else:
    c = [float(x) for x in KR._matern_consts(p)[0]]
    s8, s2 = np.sqrt(8.0 * (p + 0.5)), np.sqrt(2.0 * (p + 0.5))
    nc = float(KR._matern_consts(p)[4]); gr = float(KR._matern_consts(p)[1])
    dist = np.sqrt(D2)
    mult = s8 * dist
    u = sum(c[t] * mult ** (p - t) for t in range(p + 1))
    up = sum(s8 * (p - t) * c[t] * mult ** (p - t - 1) for t in range(p)) if p else 0.0 * dist
    w = gr * np.exp(-s2 * dist)
    T1 = scale * nc * w * (up - s2 * u)
    with np.errstate(divide='ignore', invalid='ignore'):
      Gs = [scale * nc * (u * w), T1 * (-(dist / bw[0]))] + \
           [np.where(off, T1 * (-1.0 / np.where(off, dist, 1.0)) * (dsq[q] / bw[q]), 0.0) for q in range(d)]
  return M, Gs


def device_sum(M, G, order, defect=None, n=None):
  """ 1/2 sum over the lower tiles with the weights 2 / 1 / 0 of lml_grad_tile_kernel, in one of three orders. """
  nn = M.shape[0]
  wgt = np.tril(np.full((nn, nn), 2.0), -1) + np.eye(nn)
  if defect == 'diag_twice':
    wgt += np.eye(nn)
  t = (wgt * M * G)[np.tril(np.ones((nn, nn), dtype=bool))]
  if order == 'blas':
    s = t.sum()
  elif order == 'slab':
    s = 0.0
    for k in range(0, len(t), 16):
      s = s + t[k:k + 16].sum()
  else:
    s = 0.0
    for x in t:
      s = s + x
  return 0.5 * s


def grad_case(kind, p, n=150, d=3, seed=4):
  rs = np.random.RandomState(seed + n)
  bw, scale = 0.3 + 0.4 * rs.random_sample(d), 1.3
  X = rs.random_sample((n, d))
  K = KR.kernel_exact(kind, p, scale, bw, X, X).astype(np.float64) + 1e-2 * np.eye(n)
  L = np.linalg.cholesky(K)
  npad = -(-n // T) * T
  W = np.eye(npad)
  W[:n, :n] = np.tril(solve_triangular(L, np.eye(n), lower=True))
  alpha = np.zeros(npad)
  alpha[:n] = W[:n, :n].T @ (W[:n, :n] @ np.sin(3 * X).sum(axis=1))
  return bw, scale, X, W, alpha


@pytest.mark.parametrize('kind,p', KINDS)
@pytest.mark.parametrize('order', ORDERS)
def test_lml_gradients_meet_the_bound(kind, p, order):
  bw, scale, X, W, alpha = grad_case(kind, p)
  n = len(X)
  want, bound = CR.lml_gradients(kind, p, scale, bw, X, alpha, W)
  assert np.isfinite(bound).all() and np.isfinite(want.astype(np.float64)).all()
  M, Gs = grad_terms(kind, p, scale, bw, X, W[:n, :n].T @ W[:n, :n], alpha[:n])
  got = [device_sum(M, Gs[0], order), 0.5 * np.trace(M), alpha[:n].sum(), device_sum(M, Gs[1], order)]
  got += [device_sum(M, G, order) for G in Gs[2:]]
  r = float((np.abs(CR._ld(np.array(got)) - want).astype(np.float64) / bound).max())
  assert r <= MARGIN, r
  # and the bound says something: well below the magnitude of the two terms the gradient is a difference of
  mag = np.array([0.5 * (np.abs(M) * np.abs(G)).sum() for G in Gs])
  assert (bound[[0] + list(range(3, 4 + X.shape[1]))] <= 1e-6 * mag).all()


@pytest.mark.parametrize('kind,p', KINDS)
def test_lml_gradient_defects_are_caught(kind, p):
  bw, scale, X, W, alpha = grad_case(kind, p)
  n = len(X)
  want, bound = CR.lml_gradients(kind, p, scale, bw, X, alpha, W)
  M, Gs = grad_terms(kind, p, scale, bw, X, W[:n, :n].T @ W[:n, :n], alpha[:n])
  # the diagonal of a diagonal tile weighted 2, as the entries below it are
  r = abs(CR._ld(device_sum(M, Gs[0], 'blas', 'diag_twice')) - want[0]) / bound[0]
  assert r >= WIDE, r
  # one padding row counted: the padded point (scaled coordinates 0) with its identity row of W and alpha 0
  Xp = np.vstack([X, np.zeros((1, X.shape[1]))])
  Kinv = np.eye(n + 1)
  Kinv[:n, :n] = W[:n, :n].T @ W[:n, :n]
  Mp, Gp = grad_terms(kind, p, scale, bw, Xp, Kinv, np.append(alpha[:n], 0.0))
  r = abs(CR._ld(device_sum(Mp, Gp[0], 'blas')) - want[0]) / bound[0]
  assert r >= WIDE, r
