"""
Extended-precision reference of the plain SE / Matern kernel values that the K_* kernels compute
(dragonfly_b200/csrc/kernels.cu: kstar_kernel, kstar_fast_kernel, cand_prep_kernel + kstar_seg_kernel), and a
per-entry forward-error bound that every fp64 evaluation of the kernels' form must meet.  Shared by the CPU tests
(test_kstar_ref.py) and the GPU tests (test_gpu_kstar_variants.py).

kernel_exact works in np.longdouble (64-bit significand on x86-64, unit roundoff 2^-64): it forms D^2 from the
DIFFERENCES (x - y) / bw, so it carries no cancellation of its own, and its own rounding error (a few 2^-64 relative)
is 2^-11 below the fp64 unit roundoff u = 2^-53 that the bound is written in.

kstar_bound, the derivation.  Notation: a = x / bw and b = y / bw exactly (vectors of d coordinates), x~ = fl(x / bw)
and y~ = fl(y / bw) the scaled coordinates every kernel stores, S = |a|^2 + |b|^2, D^2 = |a - b|^2 the exact squared
distance, gamma_k = k u / (1 - k u).

 1. Coordinate roundings.  x~_q - y~_q = (a_q - b_q) + e_q with |e_q| <= u (|a_q| + |b_q|), so
        | |x~ - y~|^2 - D^2 | = | sum_q e_q (2 (a_q - b_q) + e_q) | <= u (2 + u) sum_q (|a_q| + |b_q|)^2
                              <= 2 u (2 + u) S.
 2. The kernels' form D^2~ = (|y~|^2 + |x~|^2) - 2 x~.y~, evaluated in any order, with or without FMA:
    s_x = fl(|x~|^2) and t = fl(x~.y~) are sums of d products, so |s_x - |x~|^2| <= gamma_d |x~|^2 and
    |t - x~.y~| <= gamma_d sum_q |x~_q y~_q| <= gamma_d (|x~|^2 + |y~|^2) / 2 (one rounding per product and at most
    d - 1 per partial sum on any summation tree; an FMA only removes roundings).  The add s_y + s_x rounds once
    (u (1 + gamma_d) S~, S~ = |x~|^2 + |y~|^2 <= (1 + u)^2 S) and the final subtraction (or the FMA that replaces it)
    rounds once more, relative to a result of at most 2 S~ (1 + 2 gamma_d).  Altogether
        |D^2^ - |x~ - y~|^2| <= (2 gamma_d + 3 u) S~ + O(u^2 d S).
    Steps 1 and 2 together, with every O(u^2) term absorbed into one more u (d <= 128):
        |D^2^ - D^2| <= Delta = gamma_D S,  gamma_D = (2 d + 8) u.
    Clipping at 0 (fmax(d2, 0), or the kernels' flush of d2 < 2^-960 to distance 0) only moves D^2^ towards D^2 >= 0.
 3. SE, K = s exp(-D^2 / 2): K is monotone in D^2, so |K(D^2^) - K(D^2)| <= max over the two ends of
    [D^2 - Delta, D^2 + Delta] of |K(end) - K(D^2)| (= integral of |K'| <= max |K'| Delta; the left end is the larger).
    Matern, K = s P(r) exp(-sqrt(2 nu) r) / P(0) with r = sqrt(D^2): K is monotone decreasing in r, and the
    computed distance lies in [r_lo, r_hi] = [sqrt(max(D^2 - Delta, 0)) (1 - 2u), sqrt(D^2 + Delta) (1 + 2u)]:
    |sqrt(a) - sqrt(b)| = |a - b| / (sqrt(a) + sqrt(b)) <= min(|a - b| / sqrt(b), sqrt(|a - b|)) -- the second form
    is what bounds Matern-1/2 at coincident points, where D^2 = 0 and D^2^ is pure rounding residue -- and the sqrt
    itself is within one ulp (2u relative: the correctly rounded sqrt, or kstar_seg's reciprocal-square-root
    sequence without the Markstein step).  Again max |K(end) - K(r)| over the two ends.
 4. The remaining roundings are relative to the computed value, taken at its largest, K(left end):
    c_v u |K| with c_v = 8 for SE (exp <= 0.87 ulp = 1.74 u, exp_nonpos.h; scale, pre- and post-scale products, or
    the fused constant of kstar_seg and its product: at most 5 roundings) and c_v = 24 for Matern (exp; the
    constants Gamma(p+1)/Gamma(2p+1), norm_constant and the scale product, 4 roundings; the polynomial in
    mm = sqrt(8 nu) r: 8 u relative for p <= 2 since every coefficient is a positive integer; the products with the
    exponential and the scales, or kstar_seg's fused constant, 5 roundings).  Matern-7/2 (p = 3, only the descriptor
    interpreter evaluates it) forms mm ** 3 with pow: mm carries 2 roundings (fl(sqrt(8 nu)) and the product), pow
    adds at most 2 ulp = 4 u (CUDA documents 2 ulp; NumPy's libm pow is within 1 ulp), so mm ** 3 is within 10 u,
    its coefficient product 11 u, and the three adds of positive terms make the polynomial 14 u instead of 8 u:
    c_v = 24 + 6 = 30, taken as 32.  The exponent argument of Matern,
    -fl(sqrt(2 nu)) r^, carries 2u of relative error, which multiplies K by at most exp(2.0001 u sqrt(2 nu) r_hi).
    An absolute 1e-290 |s| covers the exponential's flush to zero below -707 and subnormal intermediates.

mu_bound: mu = mean + sum_j alpha_j K_j with the device's own alpha; |mu^ - mu| <= sum_j |alpha_j| B_j (the kernel
values) + gamma_n sum_j |alpha_j K^_j| (n products and the sum, in any order, warp shuffles and segment partials
included) + u |mu^| for the add of a non-zero mean.
"""
import math

import numpy as np

U = 2.0 ** -53
LD = np.longdouble
# the kinds of the plain K_* producers (and of the bound pass built on them): Matern p <= 2
KINDS = {'se': ('se', 0), 'matern12': ('matern', 0), 'matern32': ('matern', 1), 'matern52': ('matern', 2)}
# the kinds the descriptor interpreter evaluates as well: Matern-7/2 (p = 3) too
INTERP_KINDS = dict(KINDS, matern72=('matern', 3))
C_V = {'se': 8.0, 'matern': 24.0}
C_V_MATERN_POW = 32.0          # Matern with p >= 3: the polynomial's leading power comes from pow


def c_v(kind, p):
  """ The multiple of u |K| of step 4 (module docstring). """
  if kind == 'matern' and p >= 3:
    return C_V_MATERN_POW
  return C_V[kind]


def gamma_d(d):
  """ The multiple of u in |D^2^ - D^2| <= gamma_D (|x/bw|^2 + |y/bw|^2) (module docstring, steps 1-2). """
  return (2 * int(d) + 8) * U


def _scaled(Z, bw):
  return np.asarray(Z, dtype=np.float64).astype(LD) / np.asarray(bw, dtype=np.float64).astype(LD)


def pair(a, b, diag=False):
  """ Column vectors a (m,) and b (n,) as operands of an entrywise operation: (m, n) outer form, or (m,) entries
      (a_i, b_i) when diag (m = n: the diagonal of the (m, n) form without the rest). """
  if diag:
    return a, b
  return a[:, None], b[None, :]


def _d2_and_s(Xc, X, bw, diag=False):
  """ Exact (longdouble) D^2 from the scaled differences and S = |a|^2 + |b|^2, both (m, n) (or (m,) when diag). """
  A, B = _scaled(Xc, bw), _scaled(X, bw)
  d2 = LD(0)
  for q in range(A.shape[1]):
    a, b = pair(A[:, q], B[:, q], diag)
    diff = a - b
    d2 = d2 + diff * diff
  return d2, sum(pair((A * A).sum(axis=1), (B * B).sum(axis=1), diag))


def _matern_consts(p):
  """ oracle/gp_oracle.py matern_constants, in longdouble: coefficients (p+i)! / (i! (p-i)!), sqrt(8 nu),
      sqrt(2 nu), Gamma(p+1) / Gamma(2p+1) and norm_constant = 1 / (unnormalised value at 0). """
  nu = LD(p) + LD(0.5)
  coeffs = [LD(math.factorial(p + i) // (math.factorial(i) * math.factorial(p - i))) for i in range(p + 1)]
  gamma_ratio = LD(math.factorial(p)) / LD(math.factorial(2 * p))
  s8, s2 = np.sqrt(LD(8) * nu), np.sqrt(LD(2) * nu)
  norm_constant = LD(1) / (coeffs[p] * gamma_ratio)
  return coeffs, gamma_ratio, s8, s2, norm_constant


def _matern_of_r(p, scale, r):
  coeffs, gamma_ratio, s8, s2, norm_constant = _matern_consts(p)
  mm = s8 * r
  u = np.zeros(np.shape(r), dtype=LD)
  for i in range(p + 1):
    u = u + coeffs[i] * mm ** (p - i)
  return LD(scale) * norm_constant * u * gamma_ratio * np.exp(-s2 * r)


def _se_of_d2(scale, d2):
  return LD(scale) * np.exp(-d2 / LD(2))


def kernel_exact(kind, p, scale, bw, Xc, X, diag=False):
  """ k(Xc_i, X_j) in longdouble, (m, n) (or k(Xc_i, X_i), (m,), when diag).  kind 'se' or 'matern' (nu = p + 1/2);
      scale = k(x, x), the product of every scale factor of the kernel (for a Matern kernel, hyperparams['scale']); bw
      the d bandwidths. """
  d2, _ = _d2_and_s(Xc, X, bw, diag)
  if kind == 'se':
    return _se_of_d2(scale, d2)
  return _matern_of_r(p, scale, np.sqrt(d2))


def kstar_bound(kind, p, scale, bw, Xc, X, diag=False):
  """ Per-entry bound on |K^ - K| for any fp64 evaluation of the kernels' form (module docstring), (m, n) float64
      (or (m,) when diag). """
  d2, s = _d2_and_s(Xc, X, bw, diag)
  d = np.shape(bw)[0] if np.ndim(bw) else np.shape(Xc)[1]
  delta = LD(gamma_d(d)) * s
  u2 = LD(2 * U)
  if kind == 'se':
    k = _se_of_d2(scale, d2)
    k_lo, k_hi = _se_of_d2(scale, d2 - delta), _se_of_d2(scale, d2 + delta)
    prop = np.maximum(np.abs(k_lo - k), np.abs(k - k_hi))
    eval_err = LD(c_v(kind, p) * U) * np.abs(k_lo)
  else:
    r = np.sqrt(d2)
    r_lo = np.sqrt(np.maximum(d2 - delta, LD(0))) * (LD(1) - u2)
    r_hi = np.sqrt(d2 + delta) * (LD(1) + u2)
    k = _matern_of_r(p, scale, r)
    k_lo, k_hi = _matern_of_r(p, scale, r_lo), _matern_of_r(p, scale, r_hi)
    prop = np.maximum(np.abs(k_lo - k), np.abs(k - k_hi))
    s2 = _matern_consts(p)[3]
    arg = np.expm1(LD(2.0001 * U) * s2 * r_hi)
    eval_err = (LD(c_v(kind, p) * U) + arg) * np.abs(k_lo)
  # longdouble rounding of the reference itself (2^-60 |K|) and the absolute floor
  b = prop + eval_err + LD(2.0 ** -60) * np.abs(k_lo) + LD(1e-290) * abs(LD(scale))
  return b.astype(np.float64)


def mu_bound(alpha, K_hat, B, mean_const=0.0):
  """ Bound on |mu^ - (mean + sum_j alpha_j K_j)| per row: K_hat (m, n) the computed kernel values (or any values
      within B of the exact ones: the bound is relative to them), B their per-entry bounds, alpha the n weights. """
  alpha = np.abs(np.asarray(alpha, dtype=np.float64))
  n = alpha.shape[0]
  g_n = (n + 2) * U / (1.0 - (n + 2) * U)
  aK = np.abs(np.asarray(K_hat, dtype=np.float64)[:, :n]) @ alpha
  aB = np.asarray(B, dtype=np.float64)[:, :n] @ alpha
  out = aB + g_n * aK + 2.0 ** -1000
  if mean_const != 0.0:
    out = out + U * (abs(mean_const) + aK + aB)
  return out * (1.0 + 1e-12)          # the two fp64 dot products above: n u < 1e-12 relative
