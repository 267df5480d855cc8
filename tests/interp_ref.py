"""
Extended-precision reference of the kernels the descriptor interpreter evaluates (dragonfly_b200/csrc/kernels.cu:
kernel_rows, behind kstar_kernel, dfb_kernel_matrix and lml_batch_kernel), and a per-entry forward-error bound that
every fp64 evaluation of the interpreter's form must meet.  Shared by the CPU tests (test_interp_ref.py) and the GPU
tests (test_gpu_interp_exact.py).

The exact value is computed from the KERNEL OBJECTS (SEKernel, MaternKernel, PolyKernel, ExpDecayKernel, HammingKernel,
AdditiveKernel, CoordinateProductKernel and its CartesianProductKernel), never from the descriptor: an additive kernel
is scale * sum of its children on their groups, a product scale * prod of its children on their coordinates, in
np.longdouble (64-bit significand, unit roundoff 2^-64, 2^-11 below the fp64 u = 2^-53 the bound is written in).  So a
wrong slot offset, pre- or post-scale or coordinate map in kernel.build_descriptor / _expand shows up as a value outside
the bound, like a wrong operation on the device.

The bound, one step per construct.  gamma_k = k u / (1 - k u); |.| of a vector is taken entrywise.

 SE / Matern factor (any p <= 3): tests/kstar_ref.py kstar_bound on the factor's own columns and bandwidths, with the
    factor's own scale (the product scale * norm_constant of a Matern factor is one of the roundings c_v counts).
 POLY factor, v = s ((x w).(y w) + 1) ** p.  Exact a_q = x_q w_q, c_q = y_q w_q, P = sum_q |a_q c_q|, b = a.c + 1.
    The staged x~ = fl(x w), y~ = fl(y w) round once each: |x~_q y~_q - a_q c_q| <= (2u + u^2) |a_q c_q|.  The FMA
    chain over the d slots rounds once per step: gamma_d sum_q |x~_q y~_q|.  The + 1 rounds once, relative to the
    computed sum.  Altogether
        |b^ - b| <= delta = gamma_(d+3) P + u (|b| + gamma_(d+3) P),
    absolute, so the cancellation at x~.y~ ~ -1 is bounded too.  The power: p in {0, 1} is exact, p = 2 (b * b)
    rounds once, p >= 3 is pow (<= 2 ulp = 4u on CUDA; NumPy's libm pow is tighter); propagated with
    |(b + e)^p - b^p| <= p |e| (|b| + |e|)^(p-1).  The scale product rounds once:
        B = s [p delta (|b| + delta)^(p-1) + (c_p + u + c_p u) (|b| + delta)^p],  c_p = 0, 0, u, 4u for p = 0, 1, 2, >= 3.
 EXPDECAY factor, v = s prod_q (1 + x_q + y_q) ** (-p_q) + o, on coordinates where w_q = 1 + x_q + y_q > 0.  Per slot:
    fl(x + y) and fl(1 + .) give |w^ - w| <= u |x + y| + u (|w| + u |x + y|), relative rho_q = that / w.  The power's
    input error is then at most expm1(|p| * -log1p(-rho_q)) relative; the power itself is exact for p in {1, 0}, one
    rounding for 2 (w * w), 0.5 (the correctly rounded sqrt) and -1 (1 / w), else pow's 4u.  The reciprocal and the
    product with the accumulator round once each.  With A = |s| prod_q w_q^(-p_q) and E = prod_q (1 + e_q) - 1 over the
    per-slot relative errors e_q of those four steps, the + o rounds once more:
        B = A E + u (A (1 + E) + |o|).
 HAMMING factor, v = sum_q w_q [x_q == y_q]: every term is exactly 0 or w_q, so the only error is the d - 1 adds of
    numpy_add_reduce: B = gamma_(d-1) sum_q |w_q| [x_q == y_q].  Alone, the device's value is checked bit for bit against
    NumPy's own (np.equal(a, b) * w).sum(axis=1) instead (test_gpu_interp_exact E8).
 Products and sums.  The interpreter distributes every product over its additive children into terms
    k = post_scale * sum_t pre_scale_t * prod_(f in t) v_f (kernel._expand), pre_scale_t the host product of the scales
    between the root and the term.  A term of F factors with exact values v_f, bounds B_f and scales S_t (list of n_t
    numbers, exact) is off by at most
        E_t = |S_t| (prod_f (|v_f| + B_f) - prod_f |v_f|) + gamma_(n_t + F) |S_t| prod_f (|v_f| + B_f)
    (n_t - 1 roundings on the host, F on the device).  The term sum starts from 0 and rounds once per term, in order:
    sum_t E_t + gamma_T sum_t (|S_t| prod_f (|v_f| + B_f) + E_t).  The post-scale product rounds once more.
 An absolute floor of 1e-290 times the product of the scales covers the flush to zero below -707 and subnormals, and
 2^-60 |k| the longdouble rounding of the reference itself.
"""
import math

import numpy as np

import kstar_ref as KR

U = KR.U
LD = np.longdouble
FLOOR = 1e-290


def gamma(k):
  k = max(int(k), 0)
  return k * U / (1.0 - k * U)


def kind_of(kern):
  names = [c.__name__ for c in type(kern).__mro__]
  for n in ('SEKernel', 'MaternKernel', 'PolyKernel', 'ExpDecayKernel', 'HammingKernel', 'AdditiveKernel',
            'CoordinateProductKernel'):
    if n in names:
      return n
  raise NotImplementedError(type(kern).__name__)


def _cols(X, cols):
  return np.asarray(X, dtype=np.float64)[:, list(cols)]


# ---- leaves: (exact value, bound) on columns `cols` of X1 and X2 ------------------------------------------------------
def _leaf_se_matern(kern, A, B, diag):
  bw = np.asarray(kern.hyperparams['dim_bandwidths'], dtype=np.float64).reshape(-1)
  scale = float(kern.hyperparams['scale'])
  if kind_of(kern) == 'SEKernel':
    kind, p = 'se', 0
  else:
    kind, p = 'matern', int(kern.hyperparams['nu'])
  return KR.kernel_exact(kind, p, scale, bw, A, B, diag), KR.kstar_bound(kind, p, scale, bw, A, B, diag)


def poly_exact(scale, order, w, A, B, diag):
  """ scale ((A w).(B w) + 1) ** order in longdouble, and P = sum_q |a_q c_q|. """
  w = np.asarray(w, dtype=np.float64).astype(LD)
  dot, P = LD(0), LD(0)
  for q in range(A.shape[1]):
    a, c = KR.pair(A[:, q].astype(LD) * w[q], B[:, q].astype(LD) * w[q], diag)
    dot = dot + a * c
    P = P + np.abs(a * c)
  b = dot + LD(1)
  return LD(scale) * b ** int(order), b, P


def _leaf_poly(kern, A, B, diag):
  scale, order = float(kern.hyperparams['scale']), int(kern.hyperparams['order'])
  val, b, P = poly_exact(scale, order, kern.hyperparams['dim_scalings'], A, B, diag)
  g = LD(gamma(A.shape[1] + 3))
  ab = np.abs(b)
  delta = g * P + LD(U) * (ab + g * P)
  c_p = {0: 0.0, 1: 0.0, 2: U}.get(order, 4 * U)
  top = (ab + delta) ** order
  prop = LD(order) * delta * (ab + delta) ** max(order - 1, 0) if order >= 1 else LD(0) * ab
  bound = abs(LD(scale)) * (prop + LD(c_p + U + c_p * U) * top)
  return val, bound


def expdecay_exact(scale, offset, powers, A, B, diag):
  acc = LD(scale)
  for q in range(A.shape[1]):
    a, c = KR.pair(A[:, q].astype(LD), B[:, q].astype(LD), diag)
    acc = acc * (LD(1) + a + c) ** (-LD(powers[q]))
  return acc + LD(offset), acc


def _pow_rounding(p):
  if p in (1.0, 0.0):
    return 0.0
  if p in (2.0, 0.5, -1.0):
    return U
  return 4 * U


def _leaf_expdecay(kern, A, B, diag):
  hp = kern.hyperparams
  powers = [float(v) for v in np.asarray(hp['powers'], dtype=np.float64).reshape(-1)]
  scale, offset = float(hp['scale']), float(hp['offset'])
  val, acc = expdecay_exact(scale, offset, powers, A, B, diag)
  one_plus_E = LD(1)
  for q in range(A.shape[1]):
    a, c = KR.pair(A[:, q].astype(LD), B[:, q].astype(LD), diag)
    z = np.abs(a + c)
    w = LD(1) + a + c
    assert (w > 0).all(), 'ExpDecay needs 1 + x + y > 0'
    rho = (LD(U) * z + LD(U) * (w + LD(U) * z)) / w
    e_in = np.expm1(LD(abs(powers[q])) * -np.log1p(-rho))
    e_q = (LD(1) + e_in) * (LD(1) + LD(_pow_rounding(powers[q]))) * (LD(1) + LD(U)) ** 2 - LD(1)
    one_plus_E = one_plus_E * (LD(1) + e_q)
  A_abs = np.abs(acc)
  E = one_plus_E - LD(1)
  return val, A_abs * E + LD(U) * (A_abs * one_plus_E + abs(LD(offset)))


def _leaf_hamming(kern, A, B, diag):
  w = np.asarray(kern.hyperparams['dim_weights'], dtype=np.float64).reshape(-1)
  val = LD(0)
  for q in range(A.shape[1]):
    a, c = KR.pair(A[:, q], B[:, q], diag)
    val = val + np.where(a == c, LD(w[q]), LD(0))
  # every weight is >= 0 (dfb_set_kernel refuses others), so val = sum |w_q| [x_q == y_q]
  return val, LD(gamma(A.shape[1] - 1)) * np.abs(val)


_LEAVES = {'SEKernel': _leaf_se_matern, 'MaternKernel': _leaf_se_matern, 'PolyKernel': _leaf_poly,
           'ExpDecayKernel': _leaf_expdecay, 'HammingKernel': _leaf_hamming}


# ---- composition -------------------------------------------------------------------------------------------------------
def _node(kern, X1, X2, cols1, cols2, diag):
  """ (exact value, terms) of `kern` on columns cols1 of X1 and cols2 of X2.  A term is (scales, [(v_f, B_f), ...]):
      the node is the sum of its terms, a term the product of its scales and factor values. """
  kind = kind_of(kern)
  if kind in _LEAVES:
    v, b = _LEAVES[kind](kern, _cols(X1, cols1), _cols(X2, cols2), diag)
    return v, [([], [(v, b)])]
  scale = float(kern.hyperparams['scale'])
  if kind == 'AdditiveKernel':
    total, terms = LD(0), []
    for sub, grp in zip(kern.kernel_list, kern.groupings):
      v, sub_terms = _node(sub, X1, X2, [cols1[g] for g in grp], [cols2[g] for g in grp], diag)
      total = total + v
      terms += sub_terms
    return LD(scale) * total, [(sc + [scale], fs) for sc, fs in terms]
  # CoordinateProductKernel (and CartesianProductKernel)
  total, terms = LD(scale), [([scale], [])]
  for sub, crd in zip(kern.kernel_list, kern.coordinate_list):
    v, sub_terms = _node(sub, X1, X2, [cols1[c] for c in crd], [cols2[c] for c in crd], diag)
    total = total * v
    terms = [(sa + sb, fa + fb) for sa, fa in terms for sb, fb in sub_terms]
  return total, terms


def _bound(post, terms):
  err_sum, abs_sum, floor = LD(0), LD(0), 0.0
  for scales, facs in terms:
    s = abs(LD(float(np.prod(np.abs(scales))))) if scales else LD(1)
    exact_abs, upper = LD(1), LD(1)
    for v, b in facs:
      exact_abs = exact_abs * np.abs(v)
      upper = upper * (np.abs(v) + b)
    e_t = s * (upper - exact_abs) + LD(gamma(len(scales) + len(facs))) * s * upper
    err_sum = err_sum + e_t
    abs_sum = abs_sum + s * upper + e_t
    floor = max(floor, float(s))
  err = err_sum + LD(gamma(len(terms))) * abs_sum
  p = abs(LD(post))
  return p * err + LD(U) * p * (abs_sum + err), floor * float(p)


def evaluate(kern, X1, X2, diag=False, cols1=None, cols2=None):
  """ (k exact in longdouble, per-entry bound in float64) of k(X1_i, X2_j), (m, n), or of k(X1_i, X2_i), (m,), when
      diag.  cols1 / cols2: the columns of X1 / X2 the kernel's coordinates 0 .. dim-1 read (default: the first dim). """
  dim = int(kern.dim)
  cols1 = list(range(dim)) if cols1 is None else list(cols1)
  cols2 = list(range(dim)) if cols2 is None else list(cols2)
  if kind_of(kern) == 'AdditiveKernel':
    post = float(kern.hyperparams['scale'])
    total, terms = LD(0), []
    for sub, grp in zip(kern.kernel_list, kern.groupings):
      v, sub_terms = _node(sub, X1, X2, [cols1[g] for g in grp], [cols2[g] for g in grp], diag)
      total = total + v
      terms += sub_terms
    val = LD(post) * total
  else:
    post = 1.0
    val, terms = _node(kern, X1, X2, cols1, cols2, diag)
  err, floor = _bound(post, terms)
  b = err + LD(2.0 ** -60) * np.abs(val) + LD(FLOOR * max(floor, 1.0))
  return val, np.asarray(b, dtype=np.float64)


# ---- the fp64 NumPy oracles of the same kernel objects -----------------------------------------------------------------
def oracle_of(kern):
  """ The oracle kernel (oracle/gp_oracle.py, tests/nonstat_ref.py, tests/hamming_ref.py) of a kernel object. """
  from oracle import gp_oracle as O
  import hamming_ref as H
  import nonstat_ref as N
  kind, hp = kind_of(kern), kern.hyperparams
  if kind == 'SEKernel':
    return O.OSEKernel(kern.dim, hp['scale'], np.asarray(hp['dim_bandwidths']).reshape(-1))
  if kind == 'MaternKernel':
    return O.OMaternKernel(kern.dim, hp['nu'], hp['scale'], np.asarray(hp['dim_bandwidths']).reshape(-1))
  if kind == 'PolyKernel':
    return N.OPolyKernel(kern.dim, hp['order'], hp['scale'], hp['dim_scalings'])
  if kind == 'ExpDecayKernel':
    return N.OExpDecayKernel(kern.dim, hp['scale'], hp['offset'], list(hp['powers']))
  if kind == 'HammingKernel':
    return H.OHammingKernel(hp['dim_weights'])
  if kind == 'AdditiveKernel':
    return O.OAdditiveKernel(hp['scale'], [oracle_of(k) for k in kern.kernel_list], kern.groupings)
  return O.OCoordinateProductKernel(kern.dim, hp['scale'], [oracle_of(k) for k in kern.kernel_list],
                                    kern.coordinate_list)


def numpy_add_reduce(vals):
  """ kernels.cu numpy_add_reduce restated on the host: NumPy's pairwise_sum order for n <= 128 -- sequential from 0
      below 8 terms, else eight interleaved accumulators combined as ((r0+r1)+(r2+r3)) + ((r4+r5)+(r6+r7)) and a
      sequential tail. """
  v = [float(x) for x in vals]
  n = len(v)
  if n < 8:
    res = 0.0
    for x in v:
      res = res + x
    return res
  r = v[:8]
  i = 8
  while i < n - (n % 8):
    for q in range(8):
      r[q] = r[q] + v[i + q]
    i += 8
  res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
  for x in v[i:]:
    res = res + x
  return res


# ---- the catalogue -----------------------------------------------------------------------------------------------------
class Case(object):
  """ One kernel object on D columns with training points X (n, D) and candidates Xc (m, D).  construct: the group
      the worst ratios are reported by; psd: whether K + a small noise is positive definite; hamming: whether a factor
      is HAMMING (the columns in cat_cols hold category codes). """

  def __init__(self, name, construct, kern, D, n, m, seed, lo=0.0, hi=1.0, cat_cols=(), psd=True):
    self.name, self.construct, self.kern, self.D = name, construct, kern, int(D)
    self.n, self.m, self.psd = n, m, psd
    self.cat_cols = list(cat_cols)
    self.hamming = bool(self.cat_cols)
    rs = np.random.RandomState(seed)
    self.X, self.Xc = points(rs, D, n, m, lo, hi, self.cat_cols)
    self.Xext = points(rs, D, 16, 0, lo, hi, self.cat_cols)[0]


def points(rs, D, n, m, lo, hi, cat_cols=()):
  """ n training points uniform in [lo, hi)^D; m candidates: m / 4 copies of training points, m / 4 training points
      moved by 1e-9 .. 1e-3 along a random direction, the rest uniform.  Category columns hold codes 0 .. 2 and are
      not moved. """
  cont = np.array([c not in cat_cols for c in range(D)])
  def draw(k):
    Z = lo + (hi - lo) * rs.random_sample((k, D))
    Z[:, ~cont] = rs.randint(0, 3, size=(k, int((~cont).sum())))
    return Z
  X = draw(n)
  Xc = draw(m)
  k = m // 4
  Xc[:k] = X[np.arange(k) % n]
  if cont.any():
    v = rs.standard_normal((k, D)) * cont
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    eps = 10.0 ** -rs.randint(3, 10, size=(k, 1))
    Xc[k:2 * k] = X[np.arange(k, 2 * k) % n] + eps * v
  return X, Xc


# n and m on the 16-row (KSTAR_CANDS), 32-lane and 128-tile edges
NS = (129, 160, 255, 256, 257, 224, 143, 200)
MS = (112, 128, 129, 143, 256, 272, 288, 300, 100, 161)


def catalogue(K, CP, small=False):
  """ The kernels of the interpreter's check, from the kernel module K and CartesianProductKernel CP.  small: CPU-sized
      point sets. """
  out = []
  rs = np.random.RandomState(2026)
  def add(name, construct, kern, D, **kw):
    i = len(out)
    n, m = (48, 56) if small else (NS[i % len(NS)], MS[(3 * i) % len(MS)])
    out.append(Case(name, construct, kern, D, n, m, seed=1000 + i, **kw))
  def bws(d, lo=0.2, hi=0.8):
    return list(lo + (hi - lo) * rs.random_sample(d))
  def stat(kname, d, bw, scale=1.3):
    kind, p = KR.INTERP_KINDS[kname]
    return K.SEKernel(d, scale, bw) if kind == 'se' else K.MaternKernel(d, p + 0.5, scale, bw)
  # SE / Matern above the plain producers' d <= 8, up to the 128 slots
  for kname in ('se', 'matern12', 'matern32', 'matern52'):
    for d in (9, 15, 16, 17, 32, 128):
      scl = math.sqrt(d / 8.0)
      out_kern = stat(kname, d, bws(d, 0.2 * scl, 0.8 * scl))
      add('%s-d%d' % (kname, d), kname, out_kern, d)
  for d in (1, 2, 8, 9):
    add('matern72-d%d' % d, 'matern72', stat('matern72', d, bws(d)), d)
  # bandwidths that flush every non-coincident pair, and ones that make K ~ scale
  add('se-flush-d16', 'se', stat('se', 16, bws(16, 0.004, 0.01)), 16)
  add('matern12-flush-d9', 'matern12', stat('matern12', 9, bws(9, 1e-4, 2e-4)), 9)
  add('se-wide-d17', 'se', stat('se', 17, bws(17, 1e3, 1e4)), 17)
  add('matern52-wide-d32', 'matern52', stat('matern52', 32, bws(32, 1e3, 1e4)), 32)
  # additive kernels
  add('add-2groups', 'additive',
      K.AdditiveKernel(0.35, [K.MaternKernel(3, 2.5, 1.1, bws(3)), K.SEKernel(2, 0.7, bws(2))], [[0, 3, 4], [1, 2]]), 5)
  kids, groups, c = [], [], 0
  for g in range(48):
    dg = 2 if g % 3 else 1
    kids.append(stat(('se', 'matern12', 'matern32', 'matern52', 'matern72')[g % 5], dg, bws(dg, 0.3, 1.2),
                     scale=0.5 + 0.02 * g))
    groups.append(list(range(c, c + dg)))
    c += dg
  add('add-48terms', 'additive', K.AdditiveKernel(0.9, kids, groups), c)
  add('add-overlap', 'additive',
      K.AdditiveKernel(1.7, [K.SEKernel(3, 0.6, bws(3)), K.MaternKernel(3, 1.5, 0.8, bws(3)),
                             K.MaternKernel(2, 0.5, 0.4, bws(2))], [[0, 1, 2], [1, 2, 3], [3, 0]]), 4)
  # products
  kids, coords, c = [], [], 0
  for f in range(48):
    df = 6 if f % 3 == 0 else 1                 # 16 six-slot and 32 one-slot factors: 48 factors, 128 slots
    kids.append(stat(('se', 'matern32', 'matern52', 'matern12')[f % 4], df, bws(df, 1.0 * math.sqrt(df), 3.0 * math.sqrt(df)),
                     scale=0.9 + 0.01 * f))
    coords.append(list(range(c, c + df)))
    c += df
  add('prod-48factors-128slots', 'product', K.CoordinateProductKernel(c, 1.1, kids, coords), c)
  add('mf-se-matern', 'product',
      K.CoordinateProductKernel(4, 0.7, [K.SEKernel(1, 1.0, [0.7]), K.MaternKernel(3, 2.5, 1.0, bws(3))],
                                [[0], [1, 2, 3]]), 4)
  add('mf-expdecay-matern', 'product',
      K.CoordinateProductKernel(4, 1.3, [K.ExpDecayKernel(2, 0.8, 0.1, [1.0, 2.0]), K.MaternKernel(2, 1.5, 1.0, bws(2))],
                                [[0, 1], [2, 3]]), 4)
  add('prod-over-additive', 'product',
      K.CoordinateProductKernel(5, 0.6, [K.SEKernel(2, 1.2, bws(2)),
                                         K.AdditiveKernel(0.45, [K.MaternKernel(1, 2.5, 1.0, bws(1)),
                                                                 K.SEKernel(1, 0.9, bws(1)),
                                                                 K.MaternKernel(1, 0.5, 1.3, bws(1))],
                                                          [[0], [1], [2]])],
                                [[0, 1], [2, 3, 4]]), 5)
  # POLY: coordinates of both signs, so that x~.y~ + 1 crosses 0
  for order in (0, 1, 2, 3, 7):
    for d in (1, 4, 9, 17):
      w = list((0.6 + 0.8 * rs.random_sample(d)) / math.sqrt(d))
      add('poly%d-d%d' % (order, d), 'poly', K.PolyKernel(d, order, 0.8, w), d, lo=-1.5, hi=1.5)
  # EXPDECAY: every numpy_scalar_pow path, offset 0 and > 0
  powers = (1.0, 2.0, 0.5, -1.0, 0.0, 1.3, 3.0)
  for i, p in enumerate(powers):
    for d in (1, 2):
      pw = [p] if d == 1 else [p, powers[(i + 3) % len(powers)]]
      offset = 0.0 if (i + d) % 2 else 0.25
      add('expdecay-p%g-d%d-o%g' % (p, d, offset), 'expdecay', K.ExpDecayKernel(d, 1.2, offset, pw), d,
          psd=min(pw) >= 0)
  pw9 = list(powers) + [2.0, 0.5]
  for offset in (0.0, 0.3):
    add('expdecay-d9-o%g' % offset, 'expdecay', K.ExpDecayKernel(9, 0.9, offset, pw9), 9, psd=False)
  # Cartesian products of SE / Matern x Hamming x ExpDecay
  for i, dh in enumerate((1, 9, 16, 17)):
    wts = list(2.0 ** rs.uniform(-6, 6, size=dh))
    first = K.SEKernel(2, 1.0, bws(2)) if i % 2 == 0 else K.MaternKernel(2, (0.5, 1.5, 2.5, 3.5)[i], 1.0, bws(2))
    kern = CP(0.8, [first, K.HammingKernel(wts), K.ExpDecayKernel(1, 1.0, 0.2, [1.5])])
    add('cp-hamming%d' % dh, 'cartesian', kern, 2 + dh + 1, cat_cols=list(range(2, 2 + dh)))
  return out
