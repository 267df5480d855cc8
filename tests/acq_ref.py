"""
Reference of the acquisition epilogue (kernels.cu: acq_kernel, acq_score, norm_cdf_ref, norm_pdf_ref, ei_for_norm_diff,
i8_score_err, collect_shortlist_kernel, selfcheck_kernel, better) for tests/test_acq_ref.py and
tests/test_gpu_acq_exact.py.

Three layers:
  * exact values -- Phi, phi, UCB, EI, PI, TTEI and the TS marginal draw in mpmath (80 digits) on the device's own fp64
    inputs: mu, sd (or the partial sums vn and k**: sd = sqrt(fl(k** - ((vn_0 + vn_1) + ...)))), best, beta, ref_mean,
    ref_std, z.  Every input is a double and the arithmetic on it is exact;
  * a NumPy restatement of the device's operation sequence (+, *, / and sqrt are IEEE round-to-nearest on both sides,
    so it agrees with the device bit for bit wherever no elementary function enters: UCB, TS, sd; erf / erfc / exp
    are passed in, which lets the tests push them by whole ulps);
  * forward-error bounds of that sequence against the exact value, parameterised by the largest ulp errors of erf,
    erfc and exp (ULP_CUDA for the device, ULP_CEPHES for SciPy's ndtr and NumPy's exp, the reference's functions).

The bounds are running-error bounds (Higham, Accuracy and Stability of Numerical Algorithms, 3.3): every rounding of
an IEEE operation is bounded by half the spacing of its result, taken from the restated intermediate values, so
subnormal and underflowing intermediates are covered without a special case; an elementary function's error is k ulps
of its result.  Errors are carried to first order with the derivatives of Phi, phi and g(z) = z Phi(z) + phi(z)
(g' = Phi, Phi' = phi, |phi'| = |z| phi) bounded over the interval the argument may lie in, and the total is widened by
1e-6 relative plus one subnormal unit.  EI's bound is thus relative to the magnitudes sd (|z| Phi(z) + phi(z)), not to
the result: for z << 0 the sum cancels and the relative error of the score grows like z^2.
"""
import math

import mpmath as mp
import numpy as np
from scipy import special

mp.mp.dps = 80

U = 2.0 ** -53                    # unit roundoff of fp64
TINY = 2.0 ** -1074               # the smallest subnormal
SQRT1_2 = 0.70710678118654752440  # the device's constants, as doubles
SQRT2PI = 2.50662827463100050242
SAFE = 1.0 + 1e-6                 # covers the second-order terms the bounds drop

UCB, EI, PI, TTEI, TS = 1, 2, 3, 4, 5          # DFB_ACQ_*
KINDS = {'ucb': UCB, 'ei': EI, 'pi': PI, 'ttei': TTEI, 'ts': TS}

# Largest errors in ulps of the result.  Device: the double-precision table of the CUDA C++ Programming Guide
# (appendix "Mathematical Functions"): erf 2, erfc 5, exp 1 -- documented, not measured here.  Reference: SciPy's
# cephes ndtr calls cephes erf / erfc, and norm.pdf NumPy's exp; cephes documents its accuracy only as sampled relative
# errors (erf 3.7e-16, erfc 5.7e-14), so the values below come from measurement against mpmath on the grids of
# tests/test_acq_ref.py (erfc: up to 2 x^2 + 4 ulps at x, the rounding of exp(-x^2) in its tail, taken as a bound of
# k + 2 x^2 with k = 8) and are checked there.
# 'sqrt2pi': the divisor of phi -- the device's literal is sqrt(2 pi) correctly rounded, SciPy's norm.pdf divides by
# np.sqrt(2 * np.pi), one ulp below it.
ULP_CUDA = {'erf': 2.0, 'erfc': 5.0, 'exp': 1.0, 'erfc_x2': 0.0, 'sqrt2pi': SQRT2PI}
# 'erfc_zero': the argument above which erfc returns 0 (cephes: x^2 > MAXLOG = 709.78), where its value is still a
# subnormal number up to ~1e-310.
ULP_CUDA['erfc_zero'] = np.inf
ULP_CEPHES = {'erf': 4.0, 'erfc': 8.0, 'exp': 4.0, 'erfc_x2': 2.0, 'sqrt2pi': float(np.sqrt(2 * np.pi)),
              'erfc_zero': math.sqrt(7.09782712893383973096e2)}

_C_ERR = float(abs(mp.mpf(SQRT1_2) - 1 / mp.sqrt(2)))              # |fl(1/sqrt 2) - 1/sqrt 2|


def _c2_err(c):
  """ |1 / c - 1 / sqrt(2 pi)| for the double c """
  return float(abs(1 / mp.mpf(c) - 1 / mp.sqrt(2 * mp.pi)))


def _f(x):
  return np.asarray(x, dtype=np.float64)


# ---- the device's operation sequence in NumPy ----------------------------------------------------------------------
def _rounded(f):
  """ f correctly rounded to fp64, elementwise (mpmath; NaN and infinities as the IEEE functions give them). """
  def g(x):
    x = _f(x)
    out = np.empty(x.shape)
    for i, v in np.ndenumerate(x):
      out[i] = float(f(mp.mpf(float(v)))) if not np.isnan(v) else np.nan
    return out
  return g


cr_erf, cr_erfc, cr_exp = _rounded(mp.erf), _rounded(mp.erfc), _rounded(mp.exp)


class Fns(object):
  """ The elementary functions of a restatement: erf, erfc, exp (vectorised, float64); by default correctly rounded. """

  def __init__(self, erf=cr_erf, erfc=cr_erfc, exp=cr_exp):
    self.erf, self.erfc, self.exp = erf, erfc, exp


EXACT_FNS = Fns()


def norm_cdf(z, fns=EXACT_FNS):
  """ kernels.cu: norm_cdf_ref (cephes ndtr's split at |x| = 1/sqrt 2). """
  z = _f(z)
  with np.errstate(all='ignore'):
    x = z * SQRT1_2
    ax = np.abs(x)
    lo = 0.5 + 0.5 * fns.erf(x)
    hi = 0.5 * fns.erfc(ax)
    hi = np.where(x > 0, 1.0 - hi, hi)
    y = np.where(ax < SQRT1_2, lo, hi)
  return np.where(np.isnan(z), z, y)


def norm_pdf(z, fns=EXACT_FNS):
  """ kernels.cu: norm_pdf_ref, exp((z z) (-0.5)) / fl(sqrt(2 pi)). """
  z = _f(z)
  with np.errstate(all='ignore'):
    return fns.exp((z * z) * -0.5) / SQRT2PI


def ei_term(z, fns=EXACT_FNS):
  """ kernels.cu: ei_for_norm_diff, fl(fl(z Phi(z)) + phi(z)). """
  z = _f(z)
  with np.errstate(all='ignore'):
    return z * norm_cdf(z, fns) + norm_pdf(z, fns)


def sigma(partial, kss):
  """ acq_kernel's sd from the partial sums (rows of partial, summed in row order) and k**: sqrt(fl(k** - vn)). """
  kss = _f(kss)
  vn = np.zeros_like(kss)
  with np.errstate(all='ignore'):
    for row in _f(partial).reshape(-1, kss.shape[0]) if np.size(partial) else ():
      vn = vn + row
    return np.sqrt(kss - vn)


def acq(kind, mean, sd, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0, z=None, fns=EXACT_FNS):
  """ kernels.cu: acq_score (and acq_kernel's TS draw fl(fl(sd z) + mean)) in the device's operation order. """
  mean, sd = _f(mean), _f(sd)
  with np.errstate(all='ignore'):
    if kind == UCB:
      return mean + beta * sd
    if kind == EI:
      return sd * ei_term((mean - best) / sd, fns)
    if kind == PI:
      return norm_cdf((mean - best) / sd, fns)
    if kind == TTEI:
      comb = np.sqrt(ref_std * ref_std + sd * sd)
      return comb * ei_term((mean - ref_mean) / comb, fns)
    if kind == TS:
      return sd * _f(z) + mean
  raise ValueError(kind)


def _ulp(v):
  """ ulp(v) of the real v: the spacing of the binade |v| lies in (2^-1074 below the normal range). """
  a = abs(v)
  t = float(a)
  if mp.mpf(t) > a:
    t = float(np.nextafter(t, 0.0))
  return float(np.spacing(t))


def _pushed(f, k):
  """ f moved k ulps away from its exact value (k < 0: downwards), rounded toward the exact value: the farthest a
  function within |k| ulps may be (NaN and infinite values as the IEEE functions give them). """
  def g(x):
    x = _f(x)
    out = np.empty(x.shape)
    for i, v in np.ndenumerate(x):
      if np.isnan(v):
        out[i] = np.nan
        continue
      ex = f(mp.mpf(float(v)))
      if mp.isinf(ex):
        out[i] = float(ex)
        continue
      lim = abs(k) * mp.mpf(_ulp(ex))
      t = float(ex + (lim if k > 0 else -lim))
      if abs(mp.mpf(t) - ex) > lim:
        t = float(np.nextafter(t, float(ex)))
      out[i] = t
    return out
  return g


def pushed_fns(k_erf, k_erfc, k_exp):
  """ erf, erfc and exp moved by k ulps each from their exact values: a device within its documented errors, pushed
  adversarially. """
  return Fns(_pushed(mp.erf, k_erf), _pushed(mp.erfc, k_erfc), _pushed(mp.exp, k_exp))


def beyond_fns(sign, ulp=ULP_CUDA, base=ULP_CEPHES):
  """ Fast and cruder than pushed_fns, for large grids: SciPy's erf / erfc and NumPy's exp moved by sign (the device's
  k ulps + their own error bound `base`) ulps -- at least as far in that direction as a device within `ulp` may be,
  except where cephes erfc flushes to 0 (values below 1e-309). """
  def mv(f, n):
    def g(x):
      with np.errstate(all='ignore'):
        y = f(x)
        return y + sign * n(_f(x)) * np.spacing(np.abs(y))
    return g
  return Fns(mv(special.erf, lambda x: ulp['erf'] + base['erf']),
             mv(special.erfc, lambda x: ulp['erfc'] + base['erfc'] + base['erfc_x2'] * x * x),
             mv(np.exp, lambda x: ulp['exp'] + base['exp']))


# ---- exact values ---------------------------------------------------------------------------------------------------
def _m(x):
  return mp.mpf(float(x))


def exact_cdf(z):
  return mp.ncdf(z)


def exact_pdf(z):
  return mp.npdf(z)


def exact_g(z):
  return z * mp.ncdf(z) + mp.npdf(z)


def exact(kind, mean, sd, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0, z=None):
  """ The exact acquisition of one candidate on its fp64 inputs (mpf); sd > 0 (TTEI: the combined std > 0). """
  mean, sd = _m(mean), _m(sd)
  if kind == UCB:
    return mean + _m(beta) * sd
  if kind == EI:
    return sd * exact_g((mean - _m(best)) / sd)
  if kind == PI:
    return exact_cdf((mean - _m(best)) / sd)
  if kind == TTEI:
    comb = mp.sqrt(_m(ref_std) ** 2 + sd ** 2)
    return comb * exact_g((mean - _m(ref_mean)) / comb)
  if kind == TS:
    return sd * _m(z) + mean
  raise ValueError(kind)


def errors(kind, scores, mean, sd, **kw):
  """ |scores - exact| per candidate as float64, the difference taken in mpmath; NaN where a score is not finite. """
  s = _f(scores).ravel()
  mean, sd = np.broadcast_to(_f(mean), s.shape), np.broadcast_to(_f(sd), s.shape)
  zz = np.broadcast_to(_f(kw.pop('z', 0.0)), s.shape)
  out = np.full(s.shape, np.nan)
  for i in np.flatnonzero(np.isfinite(s)):
    out[i] = float(abs(mp.mpf(float(s[i])) - exact(kind, mean[i], sd[i], z=zz[i], **kw)))
  return out


# ---- forward-error bounds -------------------------------------------------------------------------------------------
def _sp(v):
  """ An upper bound of the spacing of every double within a relative 2^-40 of |v|: bounds one ulp of a result that a
  few ulps of error or a restatement with other elementary functions may have moved across a binade. """
  with np.errstate(all='ignore'):
    return np.spacing(np.abs(_f(v)) * (1.0 + 2.0 ** -40))


def _hs(v):
  return 0.5 * _sp(v)


def _phi(t):
  with np.errstate(all='ignore'):
    return np.exp(-0.5 * _f(t) * _f(t)) / math.sqrt(2 * math.pi) * (1 + 1e-12)


def _phi_near(t, w):
  """ sup of phi over [t - w, t + w]. """
  return _phi(np.maximum(np.abs(t) - w, 0.0))


def _Phi_up(t):
  """ an upper bound of Phi(t) """
  return np.minimum(special.ndtr(_f(t)) * (1 + 1e-10) + TINY, 1.0)


def cdf_bound(z, ulp):
  """ |norm_cdf(z) - Phi(z)| for the double z: the device evaluation at its own argument. """
  z = _f(z)
  with np.errstate(all='ignore'):
    x = z * SQRT1_2
    ex = _hs(x) + np.abs(z) * _C_ERR                           # |x - z / sqrt 2|
    ax = np.abs(x)
    e = special.erf(x)
    e_lo = 0.5 * ulp['erf'] * _sp(e) + _hs(0.5 + 0.5 * e)
    ec = np.where(ax > 26.0, cr_erfc(np.where(ax > 26.0, ax, 0.0)), special.erfc(ax))     # scipy's flushes to 0
    h = 0.5 * ec
    e_hi = 0.5 * (ulp['erfc'] + ulp['erfc_x2'] * ax * ax) * _sp(ec) + 0.5 * TINY + np.where(x > 0, _hs(1.0 - h), 0.0)
    e_hi = e_hi + np.where(ax > ulp['erfc_zero'], h, 0.0)
    e_eval = np.where(ax < SQRT1_2, e_lo, e_hi)
    # 0.5 + 0.5 erf(x) = 0.5 erfc(-x) = Phi(sqrt 2 x)
    # + whole subnormal units: the terms above are rounded themselves where they are subnormal
    floor = (ulp['erf'] + ulp['erfc'] + 2.0) * TINY
    return e_eval + math.sqrt(2.0) * ex * _phi_near(z, math.sqrt(2.0) * ex) + floor


def pdf_bound(z, ulp):
  """ |norm_pdf(z) - phi(z)| for the double z. """
  z = _f(z)
  with np.errstate(all='ignore'):
    s = z * z
    w = s * -0.5
    ew = _hs(w) + 0.5 * _hs(s)                                 # |w + z^2 / 2|
    p = np.exp(w)
    e_p = ulp['exp'] * _sp(p) + np.exp(w + ew) * ew
    c = ulp['sqrt2pi']
    r = p / c
    return _hs(r) + e_p / c + p * _c2_err(c) + (ulp['exp'] + 2.0) * TINY


def g_bound(z, ulp):
  """ |ei_term(z) - g(z)| for the double z, and the magnitude |z| Phi(z) + phi(z) it is measured against. """
  z = _f(z)
  with np.errstate(all='ignore'):
    cdf, pdf = special.ndtr(z), _phi(z)
    t = z * cdf
    g = t + pdf
    err = _hs(g) + _hs(t) + np.abs(z) * cdf_bound(z, ulp) + pdf_bound(z, ulp)
    return err, np.abs(z) * cdf + pdf


def bound(kind, mean, sd, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0, z=None, ulp=ULP_CUDA):
  """ An upper bound of |acq(...) - exact(...)| for the fp64 inputs, with the elementary functions within `ulp`.  Where
  the restated score is not finite the bound is NaN (those positions are compared by classification). """
  mean, sd = _f(mean), _f(sd)
  with np.errstate(all='ignore'):
    if kind == UCB:
      t = beta * sd
      e = _hs(mean + t) + _hs(t)
    elif kind == TS:
      t = sd * _f(z)
      e = _hs(t + mean) + _hs(t)
    elif kind in (EI, PI):
      d = mean - best
      zc = d / sd
      ez = _hs(zc) + _hs(d) / sd                               # |zc - (mean - best) / sd|
      if kind == PI:
        e = cdf_bound(zc, ulp) + _phi_near(zc, ez) * ez
      else:
        eg, _ = g_bound(zc, ulp)
        g = ei_term(zc)
        e = _hs(sd * g) + sd * (eg + _Phi_up(zc + ez) * ez)
    elif kind == TTEI:
      a, b = ref_std * ref_std, sd * sd
      q = a + b
      comb = np.sqrt(q)
      eq = _hs(q) + _hs(a) + _hs(b)
      ecomb = _hs(comb) + np.minimum(eq / comb, np.sqrt(eq))   # |comb - sqrt(ref_std^2 + sd^2)|
      d = mean - ref_mean
      zc = d / comb
      rel = ecomb / (comb - ecomb)
      ez = _hs(zc) + _hs(d) / comb + (np.abs(zc) + _hs(d) / comb) * rel
      ez = np.where(comb > ecomb, ez, np.inf)
      eg, _ = g_bound(zc, ulp)
      g = ei_term(zc)
      gerr = eg + _Phi_up(zc + ez) * ez
      e = _hs(comb * g) + comb * gerr + ecomb * (np.abs(g) + gerr)
    else:
      raise ValueError(kind)
    s = acq(kind, mean, sd, beta, best, ref_mean, ref_std, z)
    return np.where(np.isfinite(s), e * SAFE + TINY, np.nan)


def magnitude(kind, mean, sd, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0, z=None):
  """ The term magnitudes a bound is measured against: |mean| + |beta sd| (UCB), |mean| + |sd z| (TS),
  sd (|z| Phi + phi) (EI), comb (|z| Phi + phi) (TTEI), Phi(z) + |z| phi(z) (PI). """
  mean, sd = _f(mean), _f(sd)
  with np.errstate(all='ignore'):
    if kind == UCB:
      return np.abs(mean) + np.abs(beta * sd)
    if kind == TS:
      return np.abs(mean) + np.abs(sd * _f(z))
    if kind == EI:
      return sd * g_bound((mean - best) / sd, ULP_CUDA)[1]
    if kind == TTEI:
      comb = np.sqrt(ref_std * ref_std + sd * sd)
      return comb * g_bound((mean - ref_mean) / comb, ULP_CUDA)[1]
    if kind == PI:
      zc = (mean - best) / sd
      return special.ndtr(zc) + np.abs(zc) * _phi(zc)
  raise ValueError(kind)


# ---- the int8 pass's rules ------------------------------------------------------------------------------------------
SENS = {UCB: None, EI: 0.4, TTEI: 0.4, PI: 0.25, TS: None}      # api.cu: score_argmax_impl (UCB |beta|, TS |z_i|)


def sens_of(kind, beta=0.0):
  return abs(beta) if kind == UCB else SENS[kind]


def score_err(kind, sd, b2, sens):
  """ kernels.cu: i8_score_err -- the allowance E of a candidate with int8 sd, or -1 (always re-scored) when
  sd <= sqrt(b2) or NaN.  sens: a scalar or (TS) the per-candidate |z_i|. """
  sd = _f(sd)
  with np.errstate(all='ignore'):
    root = np.sqrt(b2)
    e = b2 / sd
    if kind == PI:
      lo = sd - e
      val = np.where(lo > 0.0, np.fmin(1.0, sens * e / lo), 1.0)
    else:
      val = sens * e
    return np.where(sd > root, val, -1.0)


def lower_bounds(s, e):
  """ acq_kernel's lb: s - E for a candidate with E >= 0 and a score that is not NaN, else -inf. """
  with np.errstate(all='ignore'):
    return np.where((e >= 0.0) & ~np.isnan(s), s - e, -np.inf)


def keep(s, e, best_lb, pad):
  """ collect_shortlist_kernel's rule: isnan(s) || E < 0 || s + E >= best_lb - pad. """
  with np.errstate(all='ignore'):
    return np.isnan(s) | (e < 0.0) | (s + e >= best_lb - pad)


def selfcheck(s8, e, s64):
  """ selfcheck_kernel's count: candidates with E >= 0 and NaN s64 or |s8 - s64| > E + slack (selfcheck_slack). """
  s8, e, s64 = _f(s8), _f(e), _f(s64)
  with np.errstate(all='ignore'):
    d = np.abs(s8 - s64)
    return int(((e >= 0.0) & (np.isnan(s64) | (d > e + selfcheck_slack(s8, s64)))).sum())


def selfcheck_slack(s8, s64):
  """ The rounding slack of the self-check: 2^-48 (|s8| + |s64|), 32 u of each score (see selfcheck_kernel). """
  with np.errstate(all='ignore'):
    return 2.0 ** -48 * (np.abs(_f(s8)) + np.abs(_f(s64)))


def argmax(scores):
  """ better()'s order over a whole vector: the first NaN, else the first maximum (np.argmax).  -1 for m = 0. """
  s = _f(scores)
  if s.size == 0:
    return -1
  nan = np.flatnonzero(np.isnan(s))
  return int(nan[0]) if nan.size else int(np.argmax(s))


def running_best_lb(s, e, chunk, init=-np.inf):
  """ best_lb after each chunk of a collecting pass: the running max of init and the lower bounds. """
  lb = lower_bounds(s, e)
  out, cur = [], init
  for c0 in range(0, len(s), chunk):
    seg = lb[c0:c0 + chunk]
    cur = max(cur, float(seg.max())) if seg.size else cur
    out.append(cur)
  return out


def shortlist(s, e, chunk, pad, init=-np.inf):
  """ The indices collect_shortlist_kernel appends over a collecting pass: per chunk, the keep rule against best_lb
  after that chunk. """
  lbs = running_best_lb(s, e, chunk, init)
  idx = []
  for c, c0 in enumerate(range(0, len(s), chunk)):
    k = keep(s[c0:c0 + chunk], e[c0:c0 + chunk], lbs[c], pad)
    idx.extend((c0 + np.flatnonzero(k)).tolist())
  return np.array(idx, dtype=np.int64)


# ---- the exact supremum behind the allowance ------------------------------------------------------------------------
def allowance_sup(kind, sd8, b2, mean=0.0, best=0.0, beta=0.0, ref_mean=0.0, ref_std=0.0, z=None):
  """ sup |S(sd64) - S(sd8)| over every sd64 > 0 with sd64^2 in [sd8^2 - b2, sd8^2 + b2], in mpmath.  Every kind is
  monotone in sd at a fixed mean (UCB, TS: linear; EI: dS/dsd = phi(z) > 0; TTEI: phi(z) sd / comb > 0; PI:
  -z phi(z) / sd, of the fixed sign of -(mean - best)), so the supremum is at an end of the interval -- at its lower
  end the limit sd64 -> 0 when sd8^2 <= b2. """
  sd8m, b2m = _m(sd8), _m(b2)
  lo2 = sd8m ** 2 - b2m
  hi = mp.sqrt(sd8m ** 2 + b2m)
  d = _m(mean) - (_m(ref_mean) if kind == TTEI else _m(best))

  def S(sd):
    if kind == TS:
      return sd * _m(z) + _m(mean)
    if kind == UCB:
      return _m(mean) + _m(beta) * sd
    if kind == EI:
      return sd * exact_g(d / sd) if sd > 0 else max(d, mp.mpf(0))
    if kind == PI:
      if sd > 0:
        return exact_cdf(d / sd)
      return mp.mpf(1) if d > 0 else (mp.mpf('0.5') if d == 0 else mp.mpf(0))
    comb = mp.sqrt(_m(ref_std) ** 2 + sd ** 2)
    return comb * exact_g(d / comb) if comb > 0 else max(d, mp.mpf(0))

  s8 = S(sd8m)
  lo = mp.sqrt(lo2) if lo2 > 0 else mp.mpf(0)
  return max(abs(S(lo) - s8), abs(S(hi) - s8))
