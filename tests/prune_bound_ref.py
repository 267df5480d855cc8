"""
Reference of the single-precision screen of dfb_score_argmax's bound pass (dragonfly_b200/csrc/kernels.cu:
prune_bound_kernel, pb_coeffs): the derivation of its bound mu_bar >= mu, the same coefficients, and a NumPy
emulation of the kernel's fp32 operation sequence.  Shared by test_prune_f32_bound.py (CPU) and
test_gpu_prune_f32.py (device).

Notation: u = 2^-24 (fp32 unit roundoff), u64 = 2^-53, x~ = x / bw and y~_j the scaled fp64 coordinates every K_*
producer uses, c the centre (midpoint of the training set's bounding box), X = |x~ - c|, Y_j = |y~_j - c|,
R = max_j Y_j, r_j = |x~ - y~_j| the exact distance, eps_a = EPS_APPROX the relative error assumed for
ex2.approx.ftz.f32 and rsqrt.approx.ftz.f32 (2^-20, at least 4x what the PTX ISA states and what
test_gpu_prune_f32.py measures over every input the kernel gives them), gamma_k = k u / (1 - k u).

 1. Coordinates.  x_bar = fp32(fl64(x~ - c)): |x_bar_q - (x~_q - c_q)| <= u' |x~_q - c_q|, u' = u (1 + 2^-28), and
    likewise y_bar.  So a_q = x_bar_q - y_bar_q = t_q + e_q (t = x~ - y~) with |e| <= u' (X + Y_j) (Minkowski).
 2. The fp32 difference rounds once more: rho = |fl(a)| lies within (1 + u) u' (X + Y_j) + u r of r.
 3. d2 = sum of D squares by an fma chain, every term >= 0: d2 = rho^2 (1 + theta), |theta| <= gamma_D.
 4. Matern: r^ = fl(d2 rsqrt(max(d2, 2^-120))) = rho sqrt(1 + theta) (1 + eps_a) (1 + u): relative error
    eps_r <= 1.01 ((D/2 + 1) u + eps_a); d2 below 2^-120 (or flushed) gives r^ <= 2^-60, r <= 2^-59.
    SE uses d2 itself; its virtual distance q = sqrt(d2) has eps_r without eps_a.
    Together |r^ - r| <= Delta_j = A (X + Y_j) + B r^ + 2^-58, A = 1.01 u, B = 1.01 (u + eps_r): the 1.01 absorbs
    every product of two of these small quantities (all below 2^-18).
 5. Kernel value.  Matern (nu = p + 1/2, p <= 2): k(r) = s P(s8 r) exp(-c r) with positive polynomial coefficients,
    decreasing, and |k'(r)| = s e^(-c r) (c P - s8 P') <= c k(r), c = sqrt(2 nu).  So
        |k(r^) - k(r)| <= c Delta_j max(k(r), k(r^)) <= c Delta_j k(r^) e^(c Delta_j).
    The computed k^ = fl(poly(r^) ex2(fl(r^ ka))): the constants rounded to fp32 (u each), two fma and one product
    (3u), ex2 (eps_a) -- within eps_a + 8u of k(r^) -- and the exponent's argument r^ ka carries 2u relative, which
    multiplies k by at most exp(2.02 u c r^).
        |k^ - k(r)| <= (1 + tau) k^ [eps_a + 8u + c (A (X + R) + 2^-58) + c (B + 2.02 u) r^],   tau = 2^-6,
    valid while c A (X + R) <= 2^-9 (checked per candidate; beyond it mu_bar = +inf): every candidate with k^ > 0
    has ex2's argument >= -126, so r^ <= 88 / c and c Delta_j <= 2^-8, and e^x - 1 <= x (1 + 2^-7) there.
    SE: k(q) = s exp(-q^2 / 2), |k'(q)| = q k(q): |k(q) - k(r)| <= Delta_j (q + Delta_j) k(q) e^(...), with
    Delta_j (q + Delta_j) <= A (X + Y) (1 + q^2) / 2 + (B + 2 B^2) q^2 + 2 A^2 (X + Y)^2 + 2^-57 (1 + q^2); the argument
    fl(d2 ka) carries 2u, i.e. q^2 u of k; ex2, the constant and the product eps_a + 3u.  Checked: A (X + R) <= 2^-13
    (k^ > 0 means q <= 13.3).
 6. mu.  alpha_j rounded to fp32 (u |alpha_j| k^_j), sum_j alpha_j k^_j in fp32 blocks of 32 by fma (gamma_32 of
    sum |alpha k^|), the block sums exact in fp64 and added there (gamma_{n/32}, inside the n u64 term below).
 7. The fp64 producers' own error (tests/kstar_ref.py: kstar_bound, mu_bound): Delta64 = (2D + 8) u64 S,
    S = |x~|^2 + max_j |y~_j|^2 (uncentred).  SE and Matern p >= 1 are smooth in d2 (|dk / d d2| <= 1.5 k):
    1.5 Delta64 relative; Matern-1/2: sqrt(Delta64) + 2 u64 (the distance's rounding near coincident points); c_v u64
    = 24 u64 of evaluation (32 u64 taken), gamma_n u64 of their sum, the mean's add (4 u64 (|mean| + |mu|)), and
    2^-60 of kstar_bound's own longdouble term.
 8. Assembly.  T0 = sum |alpha_j| k^_j and T1 = sum |alpha_j| k^_j r^_j (SE: ... k^_j d2_j) are fp32 sums of
    non-negative terms (products rounded: (1 + 2u), sums: 1 / (1 - (n + 2) u)):
        E = M (K0 T0 + K1 T1) + eta + 4 u64 (|mean| + |mu|),   M = (1 + 4u) / (1 - (n + 2) u) (1 + tau)
    with K0, K1 of `coefficients` (every relative term above, K0 the ones of T0, K1 those of T1).
    eta = (sum |alpha| (k(x, x) + 1) + n + 1) 2^-100 covers what flushes to zero: an ex2 argument below -126 means
    k <= s 2^-112 (Matern: x^2 e^-x at x >= 86) or s 2^-125 (SE), and fp32 results below 2^-126.
    mu_bar = fl(mean + mu) + E, then + 2^-50 |mu_bar| for the two fp64 adds.
"""
import math

import numpy as np

EPS_APPROX = 2.0 ** -20          # kernels.cu: PB_EPS_APPROX
DOC_APPROX = 2.0 ** -22          # the size of the PTX ISA's stated maxima: the emulation's adversarial perturbation
BLK = 32                         # kernels.cu: PB_BLK
U = 2.0 ** -24
U64 = 2.0 ** -53
F32 = np.float32
LOG2E = 1.4426950408889634


def coefficients(kind, p, d, c, XR, S64):
  """ (K0, K1) of the bound for one candidate (kernels.cu: pb_coeffs), or None where mu_bar = +inf. """
  eps_r = 1.01 * ((d / 2.0 + 1.0) * U + (0.0 if kind == 'se' else EPS_APPROX))
  A, B = 1.01 * U, 1.01 * (U + eps_r)
  gam = BLK * U / (1.0 - BLK * U)
  sum32 = U + 1.01 * gam
  d64 = (2.0 * d + 8.0) * U64 * S64
  f64 = 32.0 * U64 + 2.0 ** -60
  f64 += (math.sqrt(d64) + 2.0 * U64) if (kind == 'matern' and p == 0) else 1.5 * d64
  if not XR <= 2.0 ** 60:
    return None
  a = A * XR
  if kind == 'se':
    if not a <= 2.0 ** -13:
      return None
    return (EPS_APPROX + 3.0 * U + a / 2.0 + 2.0 * a * a + 2.0 ** -57 + sum32 + f64,
            a / 2.0 + B + 2.0 * B * B + 1.01 * U + 2.0 ** -57)
  if not c * a <= 2.0 ** -9:
    return None
  return (EPS_APPROX + 8.0 * U + c * (a + 2.0 ** -58) + sum32 + f64, c * (B + 2.02 * U) + 4.0 * U64 * c)


def _matern_consts(p):
  nu = p + 0.5
  coeffs = [math.factorial(p + i) // (math.factorial(i) * math.factorial(p - i)) for i in range(p + 1)]
  gamma_ratio = math.factorial(p) / math.factorial(2 * p)
  return coeffs, gamma_ratio, math.sqrt(8.0 * nu), math.sqrt(2.0 * nu)


def _fma32(a, b, c):
  """ fp32 fused multiply-add (a * b is exact in fp64; the fp64 add and the cast round twice -- an emulation). """
  return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def _flush(x):
  return np.where(np.abs(x) < F32(2.0 ** -126), F32(0.0), x).astype(F32)


def _approx(exact, delta):
  """ The correctly rounded fp32 value of an fp64 `exact`, moved by the relative error `delta`. """
  return (exact * (1.0 + delta)).astype(F32)


def emulate(kind, p, scale, bw, Xc, X, alpha, mean_const=0.0, delta_ex2=0.0, delta_rsqrt=0.0):
  """ The kernel's fp32 sequence for candidates Xc (m, d) against training points X (n, d) with weights alpha;
      ex2 / rsqrt results perturbed by the given relative errors.  Returns (mu32, E): mu_bar = mu32 + E (E = inf where
      the bound refuses). """
  bw = np.asarray(bw, dtype=np.float64)
  xs = np.asarray(Xc, dtype=np.float64) / bw
  ys = np.asarray(X, dtype=np.float64) / bw
  n, d = ys.shape
  cen = 0.5 * ys.min(axis=0) + 0.5 * ys.max(axis=0)
  xb = (xs - cen).astype(F32)
  yb = (ys - cen).astype(F32)
  a32 = np.asarray(alpha, dtype=np.float64).astype(F32)
  if kind == 'se':
    ka, p0, p1, p2, c = F32(-0.5 * LOG2E), F32(scale), F32(0), F32(0), 0.0
  else:
    coeffs, gr, s8, s2 = _matern_consts(p)
    cm = scale * gr
    c, ka = s2, F32(-s2 * LOG2E)
    pc = [cm * coeffs[i] * s8 ** (p - i) for i in range(p + 1)] + [0.0, 0.0]
    p0, p1, p2 = F32(pc[0]), F32(pc[1]), F32(pc[2])
  m = xb.shape[0]
  mu64 = np.zeros(m)
  t0 = np.zeros(m, dtype=F32)
  t1 = np.zeros(m, dtype=F32)
  acc = np.zeros(m, dtype=F32)
  with np.errstate(over='ignore', invalid='ignore', divide='ignore'):
    for j in range(n):
      d2 = np.zeros(m, dtype=F32)
      for q in range(d):
        df = (xb[:, q] - yb[j, q]).astype(F32)
        d2 = _flush(_fma32(df, df, d2))
      if kind == 'se':
        arg = _flush((d2 * ka).astype(F32))
        e = np.where(arg >= -126.0, _approx(np.exp2(arg.astype(np.float64)), delta_ex2), F32(0.0))
        kv = _flush((p0 * e).astype(F32))
        rr = d2
      else:
        y = _approx(1.0 / np.sqrt(np.maximum(d2, F32(2.0 ** -120)).astype(np.float64)), delta_rsqrt)
        rr = _flush((d2 * y).astype(F32))
        arg = _flush((rr * ka).astype(F32))
        e = np.where(arg >= -126.0, _approx(np.exp2(arg.astype(np.float64)), delta_ex2), F32(0.0))
        if p == 0:
          poly = np.full(m, p0, dtype=F32)
        elif p == 1:
          poly = _fma32(np.full(m, p0, dtype=F32), rr, np.full(m, p1, dtype=F32))
        else:
          poly = _fma32(_fma32(np.full(m, p0, dtype=F32), rr, np.full(m, p1, dtype=F32)), rr, np.full(m, p2, dtype=F32))
        kv = _flush((poly * e).astype(F32))
      acc = _flush(_fma32(np.full(m, a32[j], dtype=F32), kv, acc))
      w = _flush((np.abs(a32[j]) * kv).astype(F32))
      t0 = (t0 + w).astype(F32)
      t1 = _flush(_fma32(w, rr, t1))
      if j % BLK == BLK - 1 or j == n - 1:
        mu64 += acc.astype(np.float64)
        acc = np.zeros(m, dtype=F32)
  X_ = np.sqrt(((xs - cen) ** 2).sum(axis=1)) * (1.0 + 2.0 ** -40)
  R_ = math.sqrt(float(((ys - cen) ** 2).sum(axis=1).max())) * (1.0 + 2.0 ** -40)
  S64 = ((xs * xs).sum(axis=1) + float((ys * ys).sum(axis=1).max())) * (1.0 + 2.0 ** -40)
  A1 = float(np.abs(alpha).sum()) * (1.0 + 2.0 ** -40)
  M = (1.0 + 4.0 * U) / (1.0 - (n + 2) * U) * (1.0 + 2.0 ** -6)
  eta = (A1 * (scale + 1.0) + n + 1.0) * 2.0 ** -100
  E = np.empty(m)
  for i in range(m):
    k = coefficients(kind, p, d, c, X_[i] + R_, S64[i])
    if k is None or not np.isfinite(X_[i]):
      E[i] = np.inf
      continue
    K0, K1 = k
    E[i] = M * ((K0 + (n + 40) * U64) * float(t0[i]) + K1 * float(t1[i])) + eta + \
        4.0 * U64 * (abs(mean_const) + abs(mu64[i]))
  mu = mean_const + mu64
  return mu, E
