"""
Extended-precision reference and componentwise a-posteriori error bounds of the posterior build: the blocked
right-looking factorisation of the tall matrix [A ; I ; y_c^T] in 128-wide tiles (api.cu: factorise_tall; kernels.cu:
chol_diag_kernel, transpose_kernel, alpha_kernel, lml_reduce_kernel; gemm.cuh: MODE_PANEL, MODE_TRAIL).  Shared by the
CPU tests (test_build_ref.py, against the NumPy emulation `emulate` below) and the GPU tests (test_gpu_build_exact.py,
against the device's own outputs read back with dfb_debug_copy).

Every bound is evaluated from the outputs being checked -- L^ (top of the tall matrix), X^ = L^-T (its middle, whose
transpose is W^), v^ = (L^-1 y_c)^T (its y row), alpha^ and the LML -- and from A, the matrix that was actually
factorised: the device's K (dfb_get_state) with fl(K_ii + fl(noise + jitter)) on the diagonal, identity on the padding.
No bound uses cond(A): where the algorithm's explicit inverses enter, they enter through their measured residuals.
All matrices are npad x npad (npad = 128 ceil(n / 128)), padding included, so a wrong padding entry breaks a bound too.

Notation: u = 2^-53, gamma_k = k u / (1 - k u), T = 128, blocks J = 0 .. nb-1 of T rows / columns, |.| and <= are
componentwise, products of |.| are ordinary matrix products.  Any sum of k products or k terms evaluated in fp64, in any
order and with or without FMA, lies within gamma_k of the exact sum times the sum of the absolute terms; a DMMA
contraction of depth K is such a sum.

The algorithm.  Step J: chol_diag factorises the diagonal tile A~_JJ into L^_JJ and writes D^_J, an approximation of
L^_JJ^-1 obtained by the same elimination on [A~_JJ ; I] (not by inverting L^_JJ).  MODE_PANEL replaces every active
tile of column block J (top rows below it, X rows 0 .. J, the y row) by fl(A~_rJ D^_J^T): a product, not a triangular
solve.  MODE_TRAIL updates every active tile (r, j), j > J: A~_rj <- fl(A~_rj - fl(P_rJ P_jJ^T)), depth T.

 1. Rows of the tall matrix.  Let x^_r be a final row (of L^, X^ or the y row), a_r the same row of [A ; I ; y_c^T]
    and A~_rJ its block J just before the panel of step J.  Summing the trailing updates of steps s < J,
        A~_rJ = a_rJ - sum_{s<J} x^_rs L^_Js^T + E,   |E| <= gamma_{T+J+2} M_rJ,
        M_rJ = |a_rJ| + sum_{s<J} |x^_rs| |L^_Js|^T
    (depth T per product, one rounding of each subtraction relative to a partial sum bounded by (1 + gamma) M).
    The panel gives x^_rJ = A~_rJ D^_J^T + F, |F| <= gamma_T |A~_rJ| |D^_J|^T, so with R_J = L^_JJ D^_J - I,
        x^_rJ L^_JJ^T - A~_rJ = A~_rJ R_J^T + F L^_JJ^T,
    and altogether, with Mh = (1 + gamma_{T+J+2}) M_rJ >= |A~_rJ|,
        |sum_{s<=J} x^_rs L^_Js^T - a_rJ| <= gamma_{T+J+2} M_rJ + Mh |R_J|^T + gamma_T (Mh |D^_J|^T) |L^_JJ|^T.   (B)
    R_J is measured in long double from the outputs; |R_J| is widened by (T + 2) u_ld |L^_JJ| |D^_J| for its own
    rounding.  The last term is the price of the explicit inverse: (Mh |D^_J|^T) |L^_JJ|^T is evaluated, not assumed.
 2. Factor, |L^ L^^T - A| (lower triangle).  Rows r of block J at columns of block J (the diagonal tile) come from
    chol_diag instead of a panel: its fma recurrence, the correctly rounded square root and the reciprocal it scales by
    (one Newton step, under 2u) give |L^_JJ L^_JJ^T - A~_JJ| <= gamma_{T+4} |L^_JJ| |L^_JJ|^T, so there
        bound = gamma_{T+J+2} M_rJ + gamma_{T+4} |L^_rJ| |L^_JJ|^T.
    Below the diagonal tile, (B) with x^ = L^, a = A.
 3. Inverse, |L^ W^ - I| = |X^ L^^T - I|^T.  (B) with x^ = X^, a = I.  The diagonal tiles of W^ ARE the D^_J, bit for
    bit: the X tile (J, J) is an exact identity until step J (no earlier trailing update touches X rows of block J) and
    the panel's products with an identity tile have one non-zero term each.  test_build_ref.py checks this on the
    emulation; the bound reads D^_J from W^.  That makes (B) trivially true on the diagonal tiles of X^, so D^_J is
    checked on its own: chol_diag computes the rows of D^_J^T by the same elimination as the rows of L^_JJ, whence
        |R_J| = |L^_JJ D^_J - I| <= gamma_{T+4} |L^_JJ| |D^_J|.
    A stale or wrong D^_J fails there; every use of it in (B) then carries its measured R_J.  (The residual of the
    right inverse is the one the algorithm controls; a componentwise bound on W^ L^ - I would need cond(L).)
 4. y row, |L^ v^ - y_c|: (B) with x^ = v^^T, a = y_c^T.
 5. alpha = W^T v (alpha_kernel: one warp per entry, lane-strided fma chains of at most npad / 32 terms and a 5-level
    shuffle tree): |alpha^ - W^^T v^| <= gamma_{npad/32+5} |W^|^T |v^|.
 6. LML = -quad / 2 - sum_i log L^_ii - n log(2 pi) / 2 with quad = y_c . alpha^ (DFB_BUILD_FULL) or |v^|^2 (the
    others).  lml_reduce_kernel sums element i on thread i mod 1024 (chains of ceil(n / 1024) terms) and then through two
    5-level shuffle trees: depth ceil(n / 1024) + 10, so |quad^ - quad| <= gamma_depth sum |terms|, and the log sum,
    each log within 1 ulp, is within gamma_{depth+2} sum |log L^_ii|.  The host's combination adds gamma_6 of the
    magnitudes.  The exact values are recomputed from the device's own L^_ii, alpha^ and v^ with mpmath.
 7. Extension (dfb_extend_posterior, api.cu: replay_last_block): rows of the last block are rebuilt by left-looking
    products of depth m0 = npad - T split over at most 8 slices and a fixed-order slice sum (depth <= m0 + 9), then
    chol_diag and the panel of step nb-1 run once.  For X rows and the y row at the last column block, (B) holds with
    gamma_{m0+9} in place of gamma_{T+J+2}.  The last block of the top is P = fl(A_r,:m0 W^00^T) (F: gamma_{m0+9}
    |A_r| |W^00|^T), so below its diagonal tile
        |P L^00^T - A_r,:m0| <= |A_r,:m0| |L^00 W^00 - I|^T + gamma_{m0+9} (|A_r,:m0| |W^00|^T) |L^00|^T,
    with L^00 W^00 - I measured, and its diagonal tile has gamma_{m0+9} (|A_dd| + |P| |P|^T) + gamma_{T+4} |L^dd| |L^dd|^T.

Residuals are computed in np.longdouble (64-bit significand on x86-64, unit roundoff u_ld = 2^-64; the tests assert it).
Each bound is widened by (npad + 2) 2^-63 (|x^| |L^|^T + |a|) for the residual's own rounding, and by an absolute
2^-1000 for fp64's gradual underflow, which the relative model above leaves out: kernel entries such as exp(-500) have
products below 2^-1022 that fp64 rounds absolutely (by at most 2^-1075 each, or flushes) while the long-double residual
still resolves them.
"""
import math

import mpmath
import numpy as np
from scipy.linalg import solve_triangular

T = 128
U = 2.0 ** -53
U_LD = 2.0 ** -63
ETA = 2.0 ** -1000        # absolute allowance for fp64's underflow range (module docstring)
LD = np.longdouble


def gamma(k):
  return k * U / (1.0 - k * U)


def n_blocks(npad):
  assert npad % T == 0
  return npad // T


def blk(J):
  return slice(J * T, (J + 1) * T)


def pad_matrix(K, noise_plus_jitter, npad):
  """ A = K + fl(noise + jitter) I on the n x n part, identity on the padding (init_tall_kernel). """
  n = K.shape[0]
  A = np.zeros((npad, npad))
  A[:n, :n] = K
  idx = np.arange(n)
  A[idx, idx] = K[idx, idx] + np.float64(noise_plus_jitter)
  A[np.arange(n, npad), np.arange(n, npad)] = 1.0
  return A


def pad_vector(y, npad):
  out = np.zeros(npad)
  out[:len(y)] = y
  return out


# ---- the measured residuals of the explicit inverses ---------------------------------------------------------------------
class Blocks(object):
  """ |D^_J| (W^'s diagonal tiles), |R_J| = |L^_JJ D^_J - I| (long double, widened by its own rounding) and the
      largest |R_J| / (gamma_{T+4} |L^_JJ| |D^_J|): chol_diag's own bound on its inverse (module docstring, 3). """

  def __init__(self, L, W):
    npad = L.shape[0]
    self.aD, self.aR, self.ratio = [], [], 0.0
    for J in range(n_blocks(npad)):
      Lj, Dj = L[blk(J), blk(J)], W[blk(J), blk(J)]
      R = Lj.astype(LD) @ Dj.astype(LD) - np.eye(T, dtype=LD)
      LDj = np.abs(Lj) @ np.abs(Dj)
      self.aD.append(np.abs(Dj))
      self.aR.append(np.abs(R).astype(np.float64) + (T + 2) * U_LD * LDj + ETA)
      self.ratio = max(self.ratio, _ratio(R, gamma(T + 4) * LDj + (T + 2) * U_LD * LDj + ETA))


def tall_bound(Xr, Ar, L, blocks, row_block=None, replay=None):
  """ Componentwise bound on |Xr L^T - Ar| for final rows Xr (k x npad) of the tall matrix and their initial content Ar.
      row_block: for rows of the top (Xr = L^ rows), the block of each row -- its diagonal tile takes the chol_diag
      bound and tiles right of it are irrelevant (set to 0).  replay: None, or (A, Rinv00, W) of an extension: the last
      column block takes the replay's accumulation depth and the top rows of the last block the left-looking bound
      (module docstring, 7). """
  k, npad = Xr.shape
  nb = n_blocks(npad)
  aX, aA, aL = np.abs(Xr), np.abs(Ar), np.abs(L)
  B = np.zeros((k, npad))
  m0 = npad - T
  for J in range(nb):
    cs, p = blk(J), J * T
    M = aA[:, cs] + aX[:, :p] @ aL[cs, :p].T
    g1 = gamma(m0 + 9) if (replay is not None and J == nb - 1) else gamma(T + J + 2)
    Mh = (1.0 + g1) * M
    B[:, cs] = g1 * M + Mh @ blocks.aR[J].T + gamma(T) * ((Mh @ blocks.aD[J].T) @ aL[cs, cs].T)
    if row_block is not None:
      on = row_block == J
      B[on, cs] = g1 * M[on] + gamma(T + 4) * (aX[on, cs] @ aL[cs, cs].T)
      B[row_block < J, cs] = 0.0
      if replay is not None and J < nb - 1:
        A, Rinv00, W = replay
        last = row_block == nb - 1
        aAr = np.abs(A[last, :m0])
        B[last, cs] = aAr @ np.abs(Rinv00[cs, :m0]).T + gamma(m0 + 9) * ((aAr @ np.abs(W[:m0, :m0]).T) @ aL[cs, :m0].T)
  return B + (npad + 2) * U_LD * (aX @ aL.T + aA) + ETA


def alpha_bound(W, v):
  npad = W.shape[0]
  return gamma(npad // 32 + 5) * (np.abs(W).T @ np.abs(v)) + (npad + 2) * U_LD * (np.abs(W).T @ np.abs(v)) + ETA


# ---- long-double residuals --------------------------------------------------------------------------------------------
def factor_residual(L, A, rows):
  """ (L^ L^^T - A)[rows] in long double, columns <= the row's block end (the rest is not part of L). """
  npad = L.shape[0]
  out = np.zeros((len(rows), npad), dtype=LD)
  rb = rows // T
  for I in np.unique(rb):
    sel = np.nonzero(rb == I)[0]
    e = (I + 1) * T
    out[sel, :e] = L[rows[sel], :e].astype(LD) @ L[:e, :e].astype(LD).T - A[rows[sel], :e]
  return out


def inverse_residual(L, W, rows):
  """ (X^ L^^T - I)[rows] = (L^ W^ - I)^T[rows] in long double; X^ = W^^T is upper triangular (checked bit for bit), so
      columns left of a row's block are exactly zero. """
  npad = L.shape[0]
  X = W.T
  out = np.zeros((len(rows), npad), dtype=LD)
  rb = rows // T
  for I in np.unique(rb):
    sel = np.nonzero(rb == I)[0]
    b = I * T
    out[sel, b:] = X[rows[sel], b:].astype(LD) @ L[b:, b:].astype(LD).T
  out[np.arange(len(rows)), rows] -= 1
  return out


def full_inverse_residual(L, W):
  """ L^ W^ - I, long double, whole matrix (the extension bound needs it). """
  return L.astype(LD) @ W.astype(LD) - np.eye(L.shape[0], dtype=LD)


def yrow_residual(L, v, y):
  return (v.astype(LD) @ L.astype(LD).T - y)[None, :]


def alpha_residual(W, v, alpha):
  return alpha.astype(LD) - W.astype(LD).T @ v.astype(LD)


# ---- the LML -----------------------------------------------------------------------------------------------------------
def lml_check(lml_dev, L_diag, a, b, n):
  """ (|lml_dev - exact|, bound) with quad = a . b over n entries and exact = -quad / 2 - sum log L_ii - n log(2 pi) / 2
      recomputed at 200 bits from the device's own values (module docstring, 6). """
  with mpmath.workprec(200):
    quad = mpmath.fsum(mpmath.mpf(float(x)) * mpmath.mpf(float(z)) for x, z in zip(a[:n], b[:n]))
    logs = [mpmath.log(mpmath.mpf(float(x))) for x in L_diag[:n]]
    s = mpmath.fsum(logs)
    exact = -quad / 2 - s - mpmath.mpf(n) / 2 * mpmath.log(2 * mpmath.pi)
    err = abs(mpmath.mpf(float(lml_dev)) - exact)
    sum_abs_q = float(mpmath.fsum(abs(mpmath.mpf(float(x)) * mpmath.mpf(float(z))) for x, z in zip(a[:n], b[:n])))
    sum_abs_l = float(mpmath.fsum(abs(t) for t in logs))
    depth = -(-n // 1024) + 10
    const = n / 2.0 * math.log(2 * math.pi)
    bound = (0.5 * gamma(depth) * sum_abs_q + gamma(depth + 2) * sum_abs_l +
             gamma(6) * (0.5 * abs(float(quad)) + abs(float(s)) + const))
    return float(err), bound


# ---- everything at once ---------------------------------------------------------------------------------------------
def check_build(A, y, L, W, v, alpha=None, lml=None, lml_quad='v', n=None, rows=None, replay=False):
  """ Ratios max(|residual| / bound) per checked output (0 where both are 0; inf where only the bound is 0).
      A, y: what was factorised (npad-padded); L (npad x npad lower), W, v, alpha: the outputs; lml: the returned LML,
      lml_quad 'alpha' (DFB_BUILD_FULL: y_c . alpha) or 'v' (|v|^2); rows: the rows of L and X^ to check (all by
      default); replay: the outputs are those of an extension (module docstring, 7). """
  npad = L.shape[0]
  n = npad if n is None else n
  rows = np.arange(npad) if rows is None else np.asarray(rows)
  blocks = Blocks(L, W)
  rep = (A, full_inverse_residual(L, W)[:npad - T, :npad - T].astype(np.float64), W) if replay else None
  out = {'D': blocks.ratio}
  B = tall_bound(L[rows], A[rows], L, blocks, row_block=rows // T, replay=rep)
  res = factor_residual(L, A, rows)
  low = np.arange(npad)[None, :] <= rows[:, None]
  out['L'] = _ratio(res, B, low)
  I = np.eye(npad)
  B = tall_bound(W.T[rows], I[rows], L, blocks, replay=rep)
  out['W'] = _ratio(inverse_residual(L, W, rows), B)
  B = tall_bound(v[None, :], y[None, :], L, blocks, replay=rep)
  out['v'] = _ratio(yrow_residual(L, v, y), B)
  if alpha is not None:
    out['alpha'] = _ratio(alpha_residual(W, v, alpha), alpha_bound(W, v))
  if lml is not None:
    a, b = (y, alpha) if lml_quad == 'alpha' else (v, v)
    err, bound = lml_check(lml, np.diag(L), a, b, n)
    out['lml'] = err / bound
  return out


def _ratio(res, bound, mask=None):
  r = np.abs(np.asarray(res, dtype=LD))
  b = np.asarray(bound, dtype=np.float64)
  if mask is not None:
    r = np.where(mask, r, 0)
  with np.errstate(divide='ignore', invalid='ignore'):
    q = np.where(r == 0, 0.0, (r / b).astype(np.float64))
  return float(q.max()) if q.size else 0.0


# ---- NumPy emulation of the blocked algorithm ------------------------------------------------------------------------
def emulate(A, y, defect=None, at=1):
  """ The device's blocked algorithm on the host: same tiling, explicit D_k, NumPy's own summation order.  Returns
      (L, W, v, alpha, lml_full, lml_v) on npad x npad.  `defect` injects one of the errors the bounds must catch:
      'drop_slab' (one 16-wide k-slab of one trailing tile left out), 'tile_twice' (one trailing tile applied twice),
      'stale_D' (the panel of step `at` multiplies by D_{at-1}); `at` is the step. """
  npad = A.shape[0]
  nb = n_blocks(npad)
  Tm = np.zeros((2 * npad + T, npad))
  Tm[:npad] = A
  Tm[npad:2 * npad] = np.eye(npad)
  Tm[2 * npad] = y
  Ds = []
  for k in range(nb):
    ks = blk(k)
    Lkk = np.linalg.cholesky(Tm[ks, ks])
    D = np.tril(solve_triangular(Lkk, np.eye(T), lower=True))
    Ds.append(D)
    if defect == 'stale_D' and k == at:
      D = Ds[k - 1]
    Tm[ks, ks] = Lkk
    active = list(range(k + 1, nb)) + list(range(nb, nb + k + 1)) + [2 * nb]
    for rb in active:
      Tm[blk(rb), ks] = Tm[blk(rb), ks] @ D.T
    for j in range(k + 1, nb):
      for rb in active:
        if rb < nb and j > rb:
          continue
        P, Pj = Tm[blk(rb), ks], Tm[blk(j), ks]
        if defect == 'drop_slab' and (k, rb, j) == (at - 1, nb - 1, at):
          upd = P[:, 16:] @ Pj[:, 16:].T
        else:
          upd = P @ Pj.T
        Tm[blk(rb), blk(j)] -= upd
        if defect == 'tile_twice' and (k, rb, j) == (at - 1, nb - 1, at):
          Tm[blk(rb), blk(j)] -= upd
  L = np.tril(Tm[:npad])
  X = Tm[npad:2 * npad]
  W = np.ascontiguousarray(X.T)
  v = Tm[2 * npad].copy()
  # alpha_kernel's order: lane i mod 32 chains the products of row j, then a 5-level tree over the lanes
  lanes = (X * v[None, :]).reshape(npad, -1, 32)
  acc = np.zeros((npad, 32))
  for c in range(lanes.shape[1]):
    acc = acc + lanes[:, c, :]
  while acc.shape[1] > 1:
    h = acc.shape[1] // 2
    acc = acc[:, :h] + acc[:, h:]
  alpha = acc[:, 0]
  return L, W, v, alpha


def emulate_lml(L, v, y, alpha, n):
  """ lml_reduce_kernel's sums and the host formula (api.cu: lml), in lml_reduce's order: 1024 strided chains, then two
      5-level trees.  Returns (lml from y . alpha, lml from |v|^2). """
  def tree(t):
    m = -(-max(n, 1) // 1024) * 1024
    z = np.zeros(m)
    z[:n] = t[:n]
    z = z.reshape(-1, 1024)
    acc = np.zeros(1024)
    for row in z:
      acc = acc + row
    while len(acc) > 1:
      h = len(acc) // 2
      acc = acc[:h] + acc[h:]
    return acc[0]
  logdet = tree(np.log(np.diag(L)))
  const = 0.5 * n * np.log(2.0 * np.pi)
  return (-0.5 * tree(y * alpha) - logdet - const, -0.5 * tree(v * v) - logdet - const)
