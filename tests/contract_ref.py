"""
Extended-precision references and componentwise a-posteriori bounds of the fp64 DMMA contractions (gemm.cuh:
gemm_tn_kernel, MODE_SCORE + EPI_SUMSQ and MODE_GENERIC + EPI_STORE; gemm_tma.cuh: score_tma_kernel; kernels.cu:
small_sumsq_kernel, acq_kernel's sigma^2 epilogue) and of the products built on them: the posterior covariance
(api.cu: posterior_covariance), the Thompson draws (dfb_ts_draws) and K^-1 = W^T W of the LML gradients
(dfb_lml_gradients).  Shared by the CPU tests (test_contract_ref.py, against fp64 evaluations in several orders) and the
GPU tests (test_gpu_contract_exact.py, against the device's own operands and outputs read back with dfb_debug_copy).

Notation as in build_ref.py: u = 2^-53, gamma_k = k u / (1 - k u), T = 128, |.| componentwise, products of |.| are
ordinary matrix products.  A sum of k products evaluated in fp64, in any order, with or without FMA (a DMMA k-slab, a
warp shuffle tree, a lane-strided chain), lies within gamma_k of the exact sum times the sum of the absolute products.
No bound uses a condition number: every bound is evaluated from the operands the device actually used.

 1. Score partials.  W = L^-1 (npad x npad, lower triangular, identity padding) and the K_* rows Ks (m x npad, zero
    padding).  Row block rb contracts k < k_hi(rb) = min(npad, T (rb + 1)):
        v_i = sum_{k < k_hi} W_ik Ks_ck,   delta_i = gamma_{k_hi} sum_k |W_ik| |Ks_ck|,   |v^_i - v_i| <= delta_i,
    and the epilogue sums the 128 squares of the block (fma chains, shuffles, one add: depth < 128), so with
    P_rb,c = sum_{i in rb} v_i^2,
        |P^ - P| <= sum_i (2 |v_i| delta_i + delta_i^2) + gamma_128 sum_i (|v_i| + delta_i)^2.
    small_sumsq_kernel writes one partial per row i (per warp, ld 32): the same bound with k_hi = i + 1 and one term.
 2. acq_kernel's epilogue is exact arithmetic on the partials: vn = fold_+(P_0, P_1, ...) in row-block order from 0.0,
    sigma^2 = fl(kss - vn), sd = sqrt(sigma^2) with no clamp (a negative sigma^2 gives NaN).  `epilogue` replays it.
 3. MODE_GENERIC products D = alpha sum_{k in range(rb, cb)} A_ik B_jk + C: range [0, K) for tri 0, [0, T (rb + 1))
    for tri 1, [0, T (cb + 1)) for tri 2, [T max(rb, cb), K) for tri 3 (rb counted from rb0); lower_only tiles with
    cb > rb are not written.  The accumulator is within gamma_depth |alpha| |A| |B|^T of the exact sum (depth = the
    range's length), and the epilogue fl(fl(alpha acc) + C) rounds twice: 2 u (|alpha| |acc| + |C|) (1 + u) more.
 4. Covariance Cov = K** - V V^T, V = fl(Ks W^T) (tri 2, depth <= npad): with E_V = gamma_npad |Ks| |W|^T and
    Va = |V| + E_V >= |V^|, the product V^ V^^T (depth npad) is within E_V Va^T + Va E_V^T + gamma_npad Va Va^T of
    V V^T; K** within kstar_bound of the exact kernel; the epilogue as in 3.
 5. Thompson draws: samples = fl(fl(U^T L^T) + mu) with the device's L (tri 2, depth <= mbp), so
    |samples - mu - U^T L^T| <= gamma_mbp |U^T| |L|^T + u |samples|.  The factor itself is checked with build_ref's
    tall-matrix bound; dfb_ts_draws does not form L^-1, so the bound's D_J = L_JJ^-1 is computed here and its residual
    R_J is taken at chol_diag's own guarantee, 2 gamma_{T+4} |L_JJ| |D_J| (test_build_ref / test_gpu_build_exact
    check that guarantee on the device's D_J).
 6. LML gradients (kernels.cu: lml_grad_tile_kernel, lml_grad_reduce_kernel):
        g_p = 1/2 sum_ij M_ij G_p,ij,   M = alpha alpha^T - W^T W,
    over all n x n pairs, with the device's alpha and W; the device walks the lower tiles with weights 2 (below the
    diagonal), 1 (on it) and 0 (above it and on the padding), which is the same sum since M and G are symmetric.
    Slots: 0 G = K; 1 1/2 tr M; 2 sum alpha (a serial sum, gamma_n sum |alpha|); 3 G = K D2 / bw_0 (SE) or
    T1 (-r / bw_0) (Matern); 4 + q G = K d2_q / bw_q (SE) or T1 (-d2_q / bw_q) / r (Matern), 0 on the diagonal, with
    T1 = dK/dr.  Three sources of error, each bounded from the operands:
     a. The K^-1 product (tri 3, depth <= npad): |Kinv^ - W^T W| <= E = gamma_npad |W|^T |W|, and M^ =
        wgt fl(fl(alpha_i alpha_j) - Kinv^) rounds twice more: |M^ - M| <= dM = E + 2 u (|alpha alpha^T| + |W^T W| +
        E) (1 + u).
     b. G.  D2^ is the kernels' form (|x~|^2 + |y~|^2) - 2 x~.y~ and d2_q^ the same form on one coordinate, so by
        kstar_ref's steps 1-2 |D2^ - D2| <= Delta = gamma_D(d) S and |d2_q^ - d2_q| <= Delta_q = gamma_D(1)
        (a_q^2 + b_q^2); the computed distance lies in [r_lo, r_hi] as in kstar_ref step 3.  Every G is a product
        h g of a positive decreasing h and a non-negative increasing g of these arguments (sign aside):
          SE     slot 3  h = K(D2), g = D2 / bw_0;        slot 4 + q  h = K(D2), g = d2_q / bw_q;
          Matern slot 3  h = |T1| / r, g = r^2 / bw_0 (p = 0: h = |T1|, g = r / bw_0);
                 slot 4 + q  h = |T1| / r, g = d2_q / bw_q;
        with |T1| / r = s2 K / r (p = 0), 3 s exp(-sqrt(3) r) (p = 1), 5/3 s (1 + sqrt(5) r) exp(-sqrt(5) r) (p = 2),
        each decreasing in r.  So |G^ - G| <= (h(lo) - h(hi)) g(hi) + h(lo) (g(hi) - g(lo)) for the propagated
        error, plus the evaluation's own roundings relative to h(lo) g(hi): c_G u with c_G = 16 for SE (exp within
        1.74 u, the scale, the quotient by bw and two products) and, for Matern, c_G = 32 relative to the magnitudes
        the device subtracts (T1 = s w (u' - s2 u) cancels as r -> 0: A(r) = s w (|u'| + s2 |u|), taken at
        w(r_lo) and the polynomials at r_hi, divided by r_lo), times exp(2.0001 u s2 r_hi) for the exponent's
        argument.  Slot 0 takes kstar_bound.  Where r_lo = 0 (coincident or near-coincident points) the Matern 1/2
        bound of the per-dimension slots is infinite: the quotient by the distance has no bound there.
     c. The reduction: a term passes through at most 64 fma steps per thread, a 5-level shuffle tree, 8 warp slots,
        and the serial sum over the nb (nb + 1) / 2 tiles: depth = 80 + nb (nb + 1) / 2.
    Altogether |g^_p - g_p| <= 1/2 sum_ij (dM |G| + (|M| + dM) dG) + 1/2 gamma_depth sum_ij (|M| + dM) (|G| + dG).

Every residual is formed in np.longdouble (u_ld = 2^-64; the tests assert an extended long double).  Bounds are widened
by (depth + 2) 2^-63 of the same magnitudes for the residual's own rounding and the fp64 sums of |.| the bound is made
of, and by an absolute 2^-1000 for fp64's gradual underflow (build_ref.py, last paragraph).
"""
import numpy as np

import build_ref as BR
import kstar_ref as KR

T = BR.T
U = BR.U
U_LD = BR.U_LD
ETA = BR.ETA
LD = np.longdouble
gamma = BR.gamma


def k_hi(rb, npad):
  return min(npad, T * (rb + 1))


def _ld(a):
  return np.asarray(a, dtype=np.float64).astype(LD)


def _ratio(res, bound):
  return BR._ratio(res, bound)


# ---- 1. score partials --------------------------------------------------------------------------------------------------
def score_partials(W, Ks, cols=None):
  """ Exact partials P (nb x len(cols), long double) and their bounds (module docstring, 1).  W: npad x npad, Ks: rows
      of K_* (at least max(cols) + 1 rows, npad columns); cols: the candidate rows to check (all by default). """
  npad = W.shape[0]
  nb = npad // T
  cols = np.arange(Ks.shape[0]) if cols is None else np.asarray(cols)
  K = Ks[cols]
  Kl, aK = _ld(K), np.abs(K)
  P = np.zeros((nb, len(cols)), dtype=LD)
  B = np.zeros((nb, len(cols)))
  for rb in range(nb):
    kh = k_hi(rb, npad)
    Wr = W[rb * T:(rb + 1) * T, :kh]
    v = _ld(Wr) @ Kl[:, :kh].T                                    # (128, c)
    s = (np.abs(Wr) @ aK[:, :kh].T) * (1 + gamma(kh + 1))         # sum |W| |Ks|, widened for its own fp64 rounding
    delta = (gamma(kh) + (kh + 2) * U_LD) * s + ETA
    av = np.abs(v).astype(np.float64)
    P[rb] = (v * v).sum(axis=0)
    B[rb] = ((2 * av * delta + delta * delta).sum(axis=0) +
             (gamma(T) + (T + 2) * U_LD) * ((av + delta) ** 2).sum(axis=0)) * (1 + gamma(T + 2)) + ETA
  return P, B


def small_partials(W, Ks, n, cols):
  """ small_sumsq_kernel: one partial per training row i < n (v_i^2 with k <= i), (n x len(cols)), and the bounds. """
  cols = np.asarray(cols)
  K = Ks[cols, :n]
  v = _ld(np.tril(W[:n, :n])) @ _ld(K).T
  s = (np.abs(np.tril(W[:n, :n])) @ np.abs(K).T) * (1 + gamma(n + 1))
  kh = np.arange(1, n + 1, dtype=np.float64)[:, None]
  delta = (kh * U / (1 - kh * U) + (kh + 2) * U_LD) * s + ETA
  av = np.abs(v).astype(np.float64)
  B = (2 * av * delta + delta * delta + (gamma(2) + 4 * U_LD) * (av + delta) ** 2) * (1 + gamma(4)) + ETA
  return v * v, B


def epilogue(partials, kss):
  """ acq_kernel's sigma^2 and sd from the device's partials (rows: row blocks or warps, in fold order) and kss. """
  vn = np.zeros(partials.shape[1])
  for row in np.asarray(partials, dtype=np.float64):
    vn = vn + row
  var = np.asarray(kss, dtype=np.float64) - vn
  with np.errstate(invalid='ignore'):
    return var, np.sqrt(var)


# ---- 3. MODE_GENERIC products -----------------------------------------------------------------------------------------
def k_range(tri, rb, cb, K):
  if tri == 0:
    return 0, K
  if tri == 1:
    return 0, min(K, T * (rb + 1))
  if tri == 2:
    return 0, min(K, T * (cb + 1))
  return min(K, T * max(rb, cb)), K


def generic_check(A, B, D, alpha=1.0, C=None, tri=0, lower_only=False, rb0=0, K=None):
  """ max |D^ - D| / bound over every written tile of a MODE_GENERIC product (module docstring, 3).  A: (n_rb T) x K
      rows from row block rb0 on, B: (n_cb T) x K, D (and C) the (n_rb T) x (n_cb T) result. """
  K = A.shape[1] if K is None else K
  n_rb, n_cb = A.shape[0] // T, B.shape[0] // T
  worst = 0.0
  for r in range(n_rb):
    rg = r + rb0
    for c in range(n_cb):
      if lower_only and c > rg:
        continue
      lo, hi = k_range(tri, rg, c, K)
      rs, cs = slice(r * T, (r + 1) * T), slice(c * T, (c + 1) * T)
      Cc = None if C is None else C[rs, cs]
      S, bnd = _product_tile(A[rs, lo:hi], B[cs, lo:hi], alpha, Cc, hi - lo)
      worst = max(worst, _ratio(_ld(D[rs, cs]) - S, bnd))
  return worst


def _product_tile(At, Bt, alpha, Ct, depth):
  """ Exact alpha At Bt^T + Ct (long double) and the bound of one tile. """
  S = _ld(At) @ _ld(Bt).T if At.shape[1] else np.zeros((At.shape[0], Bt.shape[0]), dtype=LD)
  aS = (np.abs(At) @ np.abs(Bt).T) * (1 + gamma(depth + 1)) if At.shape[1] else np.zeros(S.shape)
  a = abs(alpha)
  aC = 0.0 if Ct is None else np.abs(Ct)
  acc = np.abs(S).astype(np.float64) + gamma(depth) * aS
  bnd = a * (gamma(depth) + (depth + 2) * U_LD) * aS + 2 * U * (a * acc + aC) * (1 + U) + ETA
  exact = LD(alpha) * S + (0 if Ct is None else _ld(Ct))
  return exact, bnd


# ---- 4. covariance -------------------------------------------------------------------------------------------------------
def covariance_check(Cov, Ks, W, kern):
  """ max |Cov^ - Cov| / bound over the m x m block (module docstring, 4).  Cov: the device's covariance (m x m); Ks:
      its K_* rows (m x npad); W: L^-1 (npad x npad); kern = (kind, p, scale, bw, Xc) of kstar_ref. """
  kind, p, scale, bw, Xc = kern
  npad = W.shape[0]
  V = _ld(Ks) @ _ld(W).T
  EV = (gamma(npad) + (npad + 2) * U_LD) * (np.abs(Ks) @ np.abs(W).T) * (1 + gamma(npad + 1))
  Va = np.abs(V).astype(np.float64) + EV
  Kss = KR.kernel_exact(kind, p, scale, bw, Xc, Xc)
  Bk = KR.kstar_bound(kind, p, scale, bw, Xc, Xc)
  VV = V @ V.T
  exact = Kss - VV
  aVV = (Va @ Va.T) * (1 + gamma(npad + 1))
  bnd = (EV @ Va.T + Va @ EV.T) * (1 + gamma(npad + 1)) + (gamma(npad) + (npad + 2) * U_LD) * aVV + Bk
  bnd = bnd + 2 * U * (aVV + np.abs(Kss).astype(np.float64) + Bk) * (1 + U) + ETA
  return _ratio(_ld(Cov) - exact, bnd)


# ---- 5. Thompson draws ----------------------------------------------------------------------------------------------------
class _FactorBlocks(object):
  """ build_ref.Blocks for a factorisation without its inverse block: D_J = L_JJ^-1 and chol_diag's own bound on
      R_J (module docstring, 5). """

  def __init__(self, L):
    from scipy.linalg import solve_triangular
    npad = L.shape[0]
    self.aD, self.aR, self.ratio = [], [], 0.0
    for J in range(npad // T):
      Lj = L[BR.blk(J), BR.blk(J)]
      Dj = np.tril(solve_triangular(Lj, np.eye(T), lower=True))
      self.aD.append(np.abs(Dj))
      self.aR.append(2 * gamma(T + 4) * (np.abs(Lj) @ np.abs(Dj)) + ETA)


def factor_check(A, L):
  """ max |L^ L^^T - A| / bound over the lower triangle (build_ref's tall-matrix bound, module docstring, 5). """
  npad = L.shape[0]
  rows = np.arange(npad)
  B = BR.tall_bound(L, A, L, _FactorBlocks(L), row_block=rows // T)
  res = BR.factor_residual(L, A, rows)
  return BR._ratio(res, B, np.arange(npad)[None, :] <= rows[:, None])


def draws_check(samples, mu, Ut, L):
  """ max |samples - mu - U^T L^T| / bound (module docstring, 5); samples (S x m), mu (m), Ut (S x m), L (m x m). """
  m = L.shape[0]
  depth = -(-m // T) * T
  exact = _ld(Ut) @ _ld(L).T
  aP = (np.abs(Ut) @ np.abs(L).T) * (1 + gamma(depth + 1))
  bnd = (gamma(depth) + (depth + 2) * U_LD) * aP + U * np.abs(samples) + ETA
  return _ratio(_ld(samples) - _ld(mu)[None, :] - exact, bnd)


# ---- 6. LML gradients ------------------------------------------------------------------------------------------------------
C_G = {'se': 16.0, 'matern': 32.0}


def _h_matern(p, scale, r):
  """ |T1| / r = |dK/dr| / r of the normalised Matern kernel (module docstring, 6b), long double. """
  s = LD(scale)
  with np.errstate(divide='ignore', invalid='ignore'):
    if p == 0:
      return KR._matern_of_r(0, scale, r) / r
  if p == 1:
    return LD(3) * s * np.exp(-np.sqrt(LD(3)) * r)
  return LD(5) / LD(3) * s * (LD(1) + np.sqrt(LD(5)) * r) * np.exp(-np.sqrt(LD(5)) * r)


def matern_dk_dr(p, scale, r):
  """ T1 = dK/dr in the device's form, scale nc gamma_ratio exp(-s2 r) (u' - s2 u) (kernels.cu), long double. """
  coeffs, gamma_ratio, s8, s2, nc = KR._matern_consts(p)
  mult = s8 * r
  u = sum(coeffs[t] * mult ** (p - t) for t in range(p + 1))
  up = sum(s8 * (p - t) * coeffs[t] * mult ** (p - t - 1) for t in range(p))
  return LD(scale) * nc * gamma_ratio * np.exp(-s2 * r) * (up - s2 * u), (up, u)


def _hg(h_lo, h_hi, g_lo, g_hi):
  return (h_lo - h_hi) * g_hi + h_lo * (g_hi - g_lo)


def lml_gradients(kind, p, scale, bw, X, alpha, W, npad=None, with_mag=False):
  """ dfb_lml_gradients' vector in long double from the device's alpha and W and the training points X, and its bound
      (module docstring, 6): (want, bound), both of length 4 + d, and with_mag: also 1/2 sum |M| |G|, the magnitude
      the gradient is a difference of (0.5 |tr M| and sum |alpha| for slots 1 and 2).  Coincident points give the reference's NaN in the
      per-dimension entries of a Matern kernel. """
  n, d = X.shape
  npad = W.shape[0] if npad is None else npad
  nb = npad // T
  bw = np.asarray(bw, dtype=np.float64)
  A = _ld(X) / _ld(bw)
  d2q = [(A[:, q][:, None] - A[:, q][None, :]) ** 2 for q in range(d)]
  sq = [A[:, q] ** 2 for q in range(d)]
  D2 = sum(d2q)
  S = sum(sq)[:, None] + sum(sq)[None, :]
  a = _ld(alpha[:n])
  Wn = _ld(W[:n, :n])
  M = a[:, None] * a[None, :] - Wn.T @ Wn
  aW = np.abs(W[:n, :n])
  E = (gamma(npad) + (npad + 2) * U_LD) * (aW.T @ aW) * (1 + gamma(n + 1))
  aM = np.abs(M).astype(np.float64)
  dM = E + 2 * U * (np.abs(a[:, None] * a[None, :]).astype(np.float64) + aM + E) * (1 + U) + ETA
  K = KR.kernel_exact(kind, p, scale, bw, X, X)
  off = ~np.eye(n, dtype=bool)
  delta = LD(KR.gamma_d(d)) * S
  dlo, dhi = np.maximum(D2 - delta, LD(0)), D2 + delta
  gq = [(np.maximum(d2q[q] - LD(KR.gamma_d(1)) * (sq[q][:, None] + sq[q][None, :]), LD(0)) / LD(bw[q]),
         (d2q[q] + LD(KR.gamma_d(1)) * (sq[q][:, None] + sq[q][None, :])) / LD(bw[q])) for q in range(d)]
  with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
    if kind == 'se':
      Gs = [K, K * D2 / LD(bw[0])] + [K * d2q[q] / LD(bw[q]) for q in range(d)]
      h_lo, h_hi = KR._se_of_d2(scale, dlo), KR._se_of_d2(scale, dhi)
      hg = [(h_lo, h_hi, dlo / LD(bw[0]), dhi / LD(bw[0]))] + [(h_lo, h_hi) + gq[q] for q in range(d)]
      ev = [LD(C_G['se'] * U) * h_lo * g_hi for (h_lo, _, _, g_hi) in hg]
    else:
      r = np.sqrt(D2)
      T1, _ = matern_dk_dr(p, scale, r)
      Gs = [K, T1 * (-(r / LD(bw[0])))] + [np.where(off, T1 * (-(d2q[q] / LD(bw[q])) / r), 0) for q in range(d)]
      u2 = LD(2 * U)
      r_lo, r_hi = np.sqrt(dlo) * (LD(1) - u2), np.sqrt(dhi) * (LD(1) + u2)
      h_lo, h_hi = _h_matern(p, scale, r_lo), _h_matern(p, scale, r_hi)
      if p == 0:                                     # slot 3 as (s2 K) r: s2 K / r alone is unbounded on the diagonal
        s2_ = KR._matern_consts(0)[3]
        h3 = (s2_ * KR._matern_of_r(0, scale, r_lo), s2_ * KR._matern_of_r(0, scale, r_hi), r_lo / LD(bw[0]),
              r_hi / LD(bw[0]))
      else:
        h3 = (h_lo, h_hi, r_lo * r_lo / LD(bw[0]), r_hi * r_hi / LD(bw[0]))
      hg = [h3] + [(h_lo, h_hi) + gq[q] for q in range(d)]
      coeffs, gamma_ratio, s8, s2, nc = KR._matern_consts(p)
      _, (up_hi, u_hi) = matern_dk_dr(p, scale, r_hi)
      A_max = LD(scale) * nc * gamma_ratio * np.exp(-s2 * r_lo) * (np.abs(up_hi) + s2 * np.abs(u_hi))
      arg = np.expm1(LD(2.0001 * U) * s2 * r_hi)
      c = LD(C_G['matern'] * U) + arg
      ev = [c * A_max * r_hi / LD(bw[0])] + [c * A_max / r_lo * g_hi for (_, _, _, g_hi) in hg[1:]]
    dG = [KR.kstar_bound(kind, p, scale, bw, X, X)]
    for (hl, hh, gl, gh), e in zip(hg, ev):
      b = (_hg(hl, hh, gl, gh) + e + LD(2.0 ** -60) * hl * gh).astype(np.float64) + ETA
      dG.append(np.where(np.isnan(b), np.inf, b))
    for q in range(d):
      dG[2 + q][~off] = 0.0                          # the diagonal of a per-dimension gradient is exactly 0 on both sides
  depth = 80 + nb * (nb + 1) // 2
  want, bound, mag = [], [], []
  with np.errstate(invalid='ignore', over='ignore'):
    for k, (G, B) in enumerate(zip(Gs, dG)):
      aG = np.abs(G).astype(np.float64)
      w = LD(0.5) * (M * G).sum()
      b = 0.5 * ((dM * aG + (aM + dM) * B).sum() + gamma(depth) * ((aM + dM) * (aG + B)).sum())
      want.append(w)
      bound.append(b)
      mag.append(0.5 * float((aM * aG).sum()))
      if k == 0:
        mag += [0.5 * float(np.diag(aM).sum()), float(np.abs(a).sum())]
        tr = np.diag(aM).sum()
        want += [LD(0.5) * np.trace(M), a.sum()]
        bound += [0.5 * (np.diag(dM).sum() + gamma(max(depth, n + 1)) * (tr + np.diag(dM).sum())),
                  gamma(n + 1) * float(np.abs(a).sum())]
  bound = np.array(bound) * (1 + 1e-12) + (n * n + 2) * U_LD * np.abs(np.array(want, dtype=np.float64)) + ETA
  out = (np.array(want, dtype=LD), np.where(np.isnan(bound), np.inf, bound))
  return out + (np.array(mag),) if with_mag else out
