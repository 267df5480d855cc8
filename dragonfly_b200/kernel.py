"""
Host-side mirror of dragonfly/gp/kernel.py for the kernels on the hot path: SEKernel, MaternKernel,
PolyKernel, ExpDecayKernel, AdditiveKernel, CoordinateProductKernel, ESPKernel (same constructor arguments,
`hyperparams` dict, `dim`, `kernel_list` / `groupings` / `coordinate_list`, `is_guaranteed_psd`, `__call__`), plus the
translation of such kernel objects -- these classes OR the reference's own, duck-typed by class name
so that a patched Dragonfly install needs no changes -- into the POD `dfb_kernel_desc` that
libdfb200's CUDA kernels evaluate (include/dfb200.h).

`Kernel.__call__(X1, X2)` (kernel.py:72-83) runs on the GPU through dfb_kernel_matrix.  ESPKernel /
ESPKernelSE / ESPKernelMatern (kernel.py:671-744) map to the descriptor's ESP form (esp_order > 0).  PolyKernel and
ExpDecayKernel (kernel.py:331-433) map to the non-stationary factor kinds POLY and EXPDECAY; a descriptor with one of
them carries kss = NaN, because k(x, x) depends on x.  HammingKernel (kernel.py:436-457) maps to the HAMMING factor on
category codes (CategoryCodes); it keeps a descriptor stationary.  Kernel types outside the hot-path scope (NN kernels,
an ESP kernel nested in another, Poly / ExpDecay / Hamming as ESP children, a Poly kernel of non-integer order) raise
NotImplementedError: there is no CPU fallback.
"""
import math

import numpy as np

from . import _lib


# ---------------------------------------------------------------------------------------------
# The Kernel surface (kernel.py:59-129)
# ---------------------------------------------------------------------------------------------
class Kernel(object):
  """ kernel.py:59-129 """

  def __init__(self):
    super(Kernel, self).__init__()
    self.hyperparams = {}

  def is_guaranteed_psd(self):
    raise NotImplementedError('Implement in a child class.')

  def __call__(self, X1, X2=None):
    return self.evaluate(X1, X2)

  def evaluate(self, X1, X2=None):
    """ n1 x n2 Gram matrix; zeros((n1, n2)) if either side is empty (kernel.py:76-83). """
    X2 = X1 if X2 is None else X2
    if len(X1) == 0 or len(X2) == 0:
      return np.zeros((len(X1), len(X2)))
    return self._child_evaluate(X1, X2)

  def _child_evaluate(self, X1, X2):
    from .device import kernel_matrix      # late import: device.py needs torch + the library
    return kernel_matrix(self, X1, X2)

  def set_hyperparams(self, **kwargs):
    self.hyperparams = kwargs

  def add_hyperparams(self, **kwargs):
    for key, value in kwargs.items():
      self.hyperparams[key] = value

  def __str__(self):
    return '%s:: %s' % (type(self), str(self.hyperparams))


class SEKernel(Kernel):
  """ kernel.py:130-181: scale * exp(-||(x - y) / bw||^2 / 2). """

  def __init__(self, dim, scale=None, dim_bandwidths=None):
    super(SEKernel, self).__init__()
    self.dim = dim
    self.set_se_hyperparams(scale, dim_bandwidths)

  def is_guaranteed_psd(self):
    return True

  def set_dim_bandwidths(self, dim_bandwidths):
    if dim_bandwidths is not None:
      if len(dim_bandwidths) != self.dim:
        raise ValueError('Dimension of dim_bandwidths should be the same as dimension.')
      dim_bandwidths = np.array(dim_bandwidths).T
    self.add_hyperparams(dim_bandwidths=dim_bandwidths)

  def set_single_bandwidth(self, bandwidth):
    self.set_dim_bandwidths(None if bandwidth is None else [bandwidth] * self.dim)

  def set_scale(self, scale):
    self.add_hyperparams(scale=scale)

  def set_se_hyperparams(self, scale, dim_bandwidths):
    self.set_scale(scale)
    if hasattr(dim_bandwidths, '__len__'):
      self.set_dim_bandwidths(dim_bandwidths)
    else:
      self.set_single_bandwidth(dim_bandwidths)

  def change_smoothness(self, factor):
    self.hyperparams['dim_bandwidths'] *= factor

  # host-side metadata helpers of the reference's SEKernel (kernel.py:179-190): no kernel evaluation involved
  def get_scaled_repr(self, X):
    return X / self.hyperparams['dim_bandwidths']

  def get_effective_norm(self, X, order=None, is_single=True):
    scaled_X = self.get_scaled_repr(X)
    if is_single:
      return np.linalg.norm(scaled_X, ord=order)
    return np.array([np.linalg.norm(sx, ord=order) for sx in scaled_X])

  def __str__(self):
    return 'SE: sc:%0.4f avg-bw: %0.4f' % (self.hyperparams['scale'],
                                           np.mean(self.hyperparams['dim_bandwidths']))


def matern_constants(nu):
  """ The scalar constants of the half-integer Matern kernel formed exactly as the reference forms
      them (set_matern_hyperparams kernel.py:242-253, _eval_kernel_values_unnormalised :259-270). """
  if nu % 1 != 0.5:
    raise ValueError('Matern kernel: nu has to be p + 0.5 where p is an integer.')
  p = int(nu)
  if p > _lib.DFB_MAX_MATERN_P:
    raise NotImplementedError('Matern nu=%s: only nu <= %d.5 is supported on device.' % (
        nu, _lib.DFB_MAX_MATERN_P))
  coeffs = [math.factorial(p + i) / (math.factorial(i) * math.factorial(p - i))
            for i in range(p + 1)]
  gamma_ratio = math.gamma(p + 1) / math.gamma(2 * p + 1)
  s8 = float(np.sqrt(8 * nu))
  s2 = float(np.sqrt(2 * nu))
  u0 = 0
  for i in range(p + 1):
    u0 += coeffs[i] * (s8 * 0) ** (p - i)
  u0 *= (gamma_ratio * np.exp(-s2 * 0))
  return dict(p=p, s8=s8, s2=s2, coeffs=[float(c) for c in coeffs],
              gamma_ratio=float(gamma_ratio), norm_constant=float(1.0 / u0))


class MaternKernel(Kernel):
  """ kernel.py:224-299: half-integer Matern, nu = p + 1/2. """

  def __init__(self, dim, nu=None, scale=None, dim_bandwidths=None):
    super(MaternKernel, self).__init__()
    self.dim = dim
    self.p = None
    self.norm_constant = None
    self.set_matern_hyperparams(nu, scale, dim_bandwidths)

  def is_guaranteed_psd(self):
    return True

  def set_matern_hyperparams(self, nu, scale, dim_bandwidths):
    consts = matern_constants(nu)
    self.add_hyperparams(nu=nu)
    self.add_hyperparams(scale=scale)
    dim_bandwidths = dim_bandwidths if hasattr(dim_bandwidths, '__len__') else \
                     [dim_bandwidths] * self.dim
    self.add_hyperparams(dim_bandwidths=np.array(dim_bandwidths).T)
    self.p = consts['p']
    self.norm_constant = consts['norm_constant']

  def __str__(self):
    return 'Matern: nu=%0.1f sc:%0.4f avg-bw: %0.4f' % (
        self.hyperparams['nu'], self.hyperparams['scale'],
        np.mean(self.hyperparams['dim_bandwidths']))


class PolyKernel(Kernel):
  """ kernel.py:331-392: scale * ((x * dim_scalings) . (y * dim_scalings) + 1) ** order. """

  def __init__(self, dim, order, scale, dim_scalings=None):
    super(PolyKernel, self).__init__()
    self.dim = dim
    self.set_poly_hyperparams(order, scale, dim_scalings)

  def is_guaranteed_psd(self):
    return True

  def set_order(self, order):
    self.add_hyperparams(order=order)

  def set_scale(self, scale):
    self.add_hyperparams(scale=scale)

  def set_dim_scalings(self, dim_scalings):
    if dim_scalings is not None:
      if len(dim_scalings) != self.dim:
        raise ValueError('Dimension of dim_scalings should be dim.')
      dim_scalings = np.array(dim_scalings)
    self.add_hyperparams(dim_scalings=dim_scalings)

  def set_single_scaling(self, scaling):
    self.set_dim_scalings(None if scaling is None else [scaling] * self.dim)

  def set_poly_hyperparams(self, order, scale, dim_scalings):
    self.set_order(order)
    self.set_scale(scale)
    if hasattr(dim_scalings, '__len__'):
      self.set_dim_scalings(dim_scalings)
    else:
      self.set_single_scaling(dim_scalings)

  def __str__(self):
    return 'Poly: d=%d, scale=%0.2f, %s' % (self.hyperparams['order'], self.hyperparams['scale'],
                                            ','.join(['%0.2f' % (e) for e in self.hyperparams['dim_scalings']]))


class ExpDecayKernel(Kernel):
  """ kernel.py:395-433: the freeze-thaw kernel of Swersky et al.,
      scale * prod_i 1 / (1 + x_i + y_i) ** powers[i] + offset, on raw coordinates. """

  def __init__(self, dim, scale=None, offset=None, powers=None):
    super(ExpDecayKernel, self).__init__()
    self.dim = dim
    if not hasattr(powers, '__iter__'):
      powers = [powers] * dim
    self.set_hyperparams(scale=scale, offset=offset, powers=powers)

  def is_guaranteed_psd(self):
    return True

  def __str__(self):
    return 'ExpDec: sc=%0.3f, offset=%0.3f, pow=%s' % (self.hyperparams['scale'], self.hyperparams['offset'],
                                                       str(list(self.hyperparams['powers'])))


class CategoryCodes(object):
  """ The value -> code table of one Hamming kernel: categories are compared on the device as small non-negative integer
      codes (fp64 columns).  Two values get the same code exactly when Python's == calls them equal -- what the
      reference's np.equal on object arrays does (general_utils.py:139-142) -- so a dict keyed by the value is the
      table.  It only grows: training rows, candidates and hallucinations all use one table.  NaN is refused (NaN != NaN
      would make k(x, x) depend on x), and so is an unhashable category. """

  def __init__(self):
    self.codes = {}

  def encode(self, value):
    try:
      is_nan = bool(value != value)
    except Exception:  # pylint: disable=broad-except
      is_nan = False
    if is_nan:
      raise ValueError('Hamming kernel: a NaN category is not equal to itself (k(x, x) would depend on x).')
    try:
      code = self.codes.get(value)
    except TypeError:
      raise ValueError('Hamming kernel: category %r is not hashable.' % (value,))
    if code is None:
      code = len(self.codes)
      self.codes[value] = code
    return code

  def encode_rows(self, X):
    """ A list of category rows -> (n, d) float64 matrix of codes. """
    rows = [[self.encode(v) for v in row] for row in X]
    return np.array(rows, dtype=np.float64).reshape(len(rows), -1)


def category_codes(kern):
  """ The CategoryCodes table of a Hamming kernel -- ours or the reference's object (attached on first use). """
  table = getattr(kern, 'category_codes', None)
  if not isinstance(table, CategoryCodes):
    table = CategoryCodes()
    kern.category_codes = table
  return table


def hamming_weights(kern):
  """ dim_weights of a Hamming kernel as float64 (an int weight array compares and sums to the same values). """
  return np.asarray(kern.hyperparams['dim_weights'], dtype=np.float64).reshape(-1)


class HammingKernel(Kernel):
  """ kernel.py:436-457: sum_q w_q [x_q == y_q] over categorical coordinates (pairwise_hamming_kernel,
      general_utils.py:113-146).  An int dim_weights d means d uniform weights 1/d.  No scale hyper-parameter. """

  def __init__(self, dim_weights):
    super(HammingKernel, self).__init__()
    if isinstance(dim_weights, (int, float)):
      dim_weights = np.ones((dim_weights,)) / float(dim_weights)
    dim_weights = np.array(dim_weights)
    self.set_hyperparams(dim_weights=dim_weights)
    self.category_codes = CategoryCodes()

  @property
  def dim(self):
    return len(self.hyperparams['dim_weights'])

  def is_guaranteed_psd(self):
    return True

  def _child_evaluate(self, X1, X2):
    from .device import kernel_matrix
    table = category_codes(self)
    return kernel_matrix(self, table.encode_rows(X1), table.encode_rows(X2))

  def __str__(self):
    return 'Hamming: wts=%s' % (str(list(self.hyperparams['dim_weights'])))


def kernel_dim(kern):
  """ Number of coordinates a kernel acts on; the reference's HammingKernel has no `dim`: its weights count them. """
  if _kind_of(kern) == 'HammingKernel':
    return len(kern.hyperparams['dim_weights'])
  return int(kern.dim)


class AdditiveKernel(Kernel):
  """ kernel.py:461-500: scale * sum_g k_g(x[g], y[g]) over non-overlapping groups. """

  def __init__(self, scale, kernel_list, groupings):
    if len(kernel_list) != len(groupings):
      raise ValueError('number of kernels do not correspond to number of groups.')
    super(AdditiveKernel, self).__init__()
    self.kernel_list = kernel_list
    self.groupings = groupings
    self.add_hyperparams(scale=scale)
    self.dim = sum([kern.dim for kern in self.kernel_list])

  def is_guaranteed_psd(self):
    return all([kern.is_guaranteed_psd() for kern in self.kernel_list])

  def __str__(self):
    return 'ADD scale=%0.2f, ' % (self.hyperparams['scale']) + ', '.join(
        ['%s(%s)' % (g, k) for (g, k) in zip(self.groupings, self.kernel_list)])


class CoordinateProductKernel(Kernel):
  """ kernel.py:541-590: scale * prod_i k_i(x[c_i], y[c_i]); the multi-fidelity kernel is the
      product of a fidelity-space and a domain kernel (euclidean_gp.py:369-374). """

  def __init__(self, dim, scale, kernel_list=None, coordinate_list=None):
    super(CoordinateProductKernel, self).__init__()
    self.dim = dim
    self.add_hyperparams(scale=scale)
    self.kernel_list = kernel_list
    self.coordinate_list = coordinate_list

  def set_kernel_list(self, kernel_list):
    self.kernel_list = kernel_list

  def set_new_kernel(self, kernel_idx, new_kernel):
    self.kernel_list[kernel_idx] = new_kernel

  def set_kernel_hyperparams(self, kernel_idx, **kwargs):
    self.kernel_list[kernel_idx].set_hyperparams(**kwargs)

  def is_guaranteed_psd(self):
    return all([kern.is_guaranteed_psd() for kern in self.kernel_list])

  def __str__(self):
    return 'CoordProd scale=%0.2f, ' % (self.hyperparams['scale']) + ', '.join(
        ['%s(%s)' % (g, k) for (g, k) in zip(self.coordinate_list, self.kernel_list)])


class ESPKernel(Kernel):
  """ kernel.py:671-726: the ESP kernel of Kandasamy & Yu (2016), scale * e_order(k_1(x_1, y_1), ..., k_d(x_d, y_d)),
      e_order the elementary symmetric polynomial of the d one-dimensional child kernels. """

  def __init__(self, scale, order, kernel_list):
    super(ESPKernel, self).__init__()
    self.dim = len(kernel_list)
    self.kernel_list = kernel_list
    self.add_hyperparams(scale=scale, order=order)
    if self.dim < 0:
      raise ValueError("dim cannot not be negative")
    if order > self.dim:
      raise ValueError("order must be less than or equal to dim")
    if order < 1:
      raise ValueError("order must be an integer between 1 and dim")

  def is_guaranteed_psd(self):
    return all([kern.is_guaranteed_psd() for kern in self.kernel_list])


class ESPKernelSE(ESPKernel):
  """ kernel.py:729-735: one 1-D SE child of scale 1 per dimension. """

  def __init__(self, dim, scale, order, dim_bandwidths):
    kernel_list = [SEKernel(1, 1.0, float(np.asarray(dim_bandwidths[i]).item())) for i in range(dim)]
    super(ESPKernelSE, self).__init__(scale, order, kernel_list)


class ESPKernelMatern(ESPKernel):
  """ kernel.py:738-744: one 1-D Matern child of scale 1 per dimension, nu[i] per dimension. """

  def __init__(self, dim, nu, scale, order, dim_bandwidths):
    kernel_list = [MaternKernel(1, nu[i], 1.0, float(np.asarray(dim_bandwidths[i]).item())) for i in range(dim)]
    super(ESPKernelMatern, self).__init__(scale, order, kernel_list)


def kernel_from_spec(spec):
  """ Builds a kernel object from the nested-dict form used by synth_data.make_workload. """
  t = spec['type']
  if t == 'se':
    return SEKernel(spec['dim'], spec['scale'], spec['dim_bandwidths'])
  if t == 'matern':
    return MaternKernel(spec['dim'], spec['nu'], spec['scale'], spec['dim_bandwidths'])
  if t == 'additive':
    return AdditiveKernel(spec['scale'], [kernel_from_spec(s) for s in spec['kernels']],
                          spec['groupings'])
  if t == 'coordinate_product':
    return CoordinateProductKernel(spec['dim'], spec['scale'],
                                   [kernel_from_spec(s) for s in spec['kernels']],
                                   spec['coordinate_list'])
  raise ValueError('unknown kernel spec type %s' % (t))


# ---------------------------------------------------------------------------------------------
# Kernel object -> canonical sum-of-products form -> dfb_kernel_desc
# ---------------------------------------------------------------------------------------------
class _Factor(object):
  __slots__ = ('kind', 'p', 'scale', 's8', 's2', 'gamma_ratio', 'coeffs', 'train_coords',
               'cand_coords', 'bandwidths')


def _kind_of(kern):
  """ Duck-typed dispatch on the class name so the reference's own kernel objects work too. """
  names = [c.__name__ for c in type(kern).__mro__]
  for n in ('SEKernel', 'MaternKernel', 'PolyKernel', 'ExpDecayKernel', 'HammingKernel', 'AdditiveKernel',
            'CoordinateProductKernel', 'ESPKernel'):
    if n in names:
      return n
  raise NotImplementedError(
      'Kernel type %s is outside the GPU hot-path scope (supported: SEKernel, MaternKernel, PolyKernel, ExpDecayKernel, '
      'HammingKernel, AdditiveKernel, CoordinateProductKernel, ESPKernel); there is no CPU fallback.'
      % (type(kern).__name__))


def _nonstationary_factor(kern, kind, train_coords, cand_coords):
  """ PolyKernel -> one POLY factor (p = order, slot values = dim_scalings); ExpDecayKernel -> one EXPDECAY factor
      (s2 = offset, slot values = powers).  include/dfb200.h, "kernel descriptor". """
  need = ('order', 'scale', 'dim_scalings') if kind == 'PolyKernel' else ('scale', 'offset', 'powers')
  missing = [key for key in need if key not in getattr(kern, 'hyperparams', {})]
  if missing:
    # not the reference's object: a duck-typed class name without the hyper-parameters that define the kernel
    raise NotImplementedError('%s object without hyper-parameter(s) %s has no device form; there is no CPU fallback.'
                              % (kind, ', '.join(missing)))
  f = _Factor()
  f.train_coords = [int(c) for c in train_coords]
  f.cand_coords = [int(c) for c in cand_coords]
  f.s8, f.gamma_ratio, f.coeffs = 0.0, 0.0, []
  f.scale = float(kern.hyperparams['scale'])
  if kind == 'PolyKernel':
    order = kern.hyperparams['order']
    if float(order) != int(order) or int(order) < 0:
      raise NotImplementedError('PolyKernel of order %s: only non-negative integer orders run on the device.' % (order,))
    if kern.hyperparams['dim_scalings'] is None:
      raise ValueError('PolyKernel needs dim_scalings.')
    vals = np.asarray(kern.hyperparams['dim_scalings'], dtype=np.float64).reshape(-1)
    f.kind, f.p, f.s2 = _lib.DFB_BASE_POLY, int(order), 0.0
  else:
    vals = np.asarray(kern.hyperparams['powers'], dtype=np.float64).reshape(-1)
    f.kind, f.p, f.s2 = _lib.DFB_BASE_EXPDECAY, 0, float(kern.hyperparams['offset'])
  if len(vals) != len(train_coords):
    raise ValueError('%s has %d dim_scalings / powers for %d coordinates' % (kind, len(vals), len(train_coords)))
  f.bandwidths = [float(v) for v in vals]
  return f


def _expand(kern, train_coords, cand_coords):
  """ Returns (post_scale, [(pre_scale, [factor, ...]), ...]) for `kern` applied to the given
      columns of the training / candidate matrices. """
  kind = _kind_of(kern)
  if kind in ('SEKernel', 'MaternKernel'):
    bws = np.asarray(kern.hyperparams['dim_bandwidths'], dtype=np.float64).reshape(-1)
    if len(bws) != len(train_coords):
      raise ValueError('kernel has %d bandwidths for %d coordinates' % (len(bws), len(train_coords)))
    f = _Factor()
    f.train_coords = [int(c) for c in train_coords]
    f.cand_coords = [int(c) for c in cand_coords]
    f.bandwidths = [float(b) for b in bws]
    if kind == 'SEKernel':
      f.kind = _lib.DFB_BASE_SE
      f.p, f.s8, f.s2, f.gamma_ratio, f.coeffs = 0, 0.0, 0.0, 0.0, []
      f.scale = float(kern.hyperparams['scale'])
    else:
      consts = matern_constants(kern.hyperparams['nu'])
      f.kind = _lib.DFB_BASE_MATERN
      f.p, f.s8, f.s2 = consts['p'], consts['s8'], consts['s2']
      f.gamma_ratio, f.coeffs = consts['gamma_ratio'], consts['coeffs']
      # K = hyperparams['scale'] * norm_constant * unnorm: the first product is formed on the host
      f.scale = float(kern.hyperparams['scale'] * consts['norm_constant'])
    return 1.0, [(1.0, [f])]
  if kind in ('PolyKernel', 'ExpDecayKernel'):
    # one factor value each: ExpDecay's offset stays inside its factor, so a product multiplies ((scale k_F) k_D)
    # in CoordinateProductKernel._child_evaluate's order (kernel.py:573-584)
    return 1.0, [(1.0, [_nonstationary_factor(kern, kind, train_coords, cand_coords)])]
  if kind == 'HammingKernel':
    # the columns hold category codes (CategoryCodes); the weights ride in the slots, the scale is not read
    wts = hamming_weights(kern)
    if len(wts) != len(train_coords):
      raise ValueError('HammingKernel has %d dim_weights for %d coordinates' % (len(wts), len(train_coords)))
    f = _Factor()
    f.train_coords = [int(c) for c in train_coords]
    f.cand_coords = [int(c) for c in cand_coords]
    f.kind, f.p, f.scale, f.s8, f.s2, f.gamma_ratio, f.coeffs = _lib.DFB_BASE_HAMMING, 0, 1.0, 0.0, 0.0, 0.0, []
    f.bandwidths = [float(w) for w in wts]
    return 1.0, [(1.0, [f])]
  if kind == 'ESPKernel':
    raise NotImplementedError('An ESP kernel inside an additive or product kernel is outside the GPU hot-path scope.')
  if kind == 'AdditiveKernel':
    terms = []
    for sub, grp in zip(kern.kernel_list, kern.groupings):
      post, sub_terms = _expand(sub, [train_coords[g] for g in grp], [cand_coords[g] for g in grp])
      for pre, facs in sub_terms:
        terms.append((pre * post if post != 1.0 else pre, facs))
    return float(kern.hyperparams['scale']), terms
  # CoordinateProductKernel: distribute the product over the (usually single-term) children
  terms = [(float(kern.hyperparams['scale']), [])]
  for sub, crd in zip(kern.kernel_list, kern.coordinate_list):
    post, sub_terms = _expand(sub, [train_coords[c] for c in crd], [cand_coords[c] for c in crd])
    new_terms = []
    for pre_a, facs_a in terms:
      for pre_b, facs_b in sub_terms:
        scale_b = pre_b * post
        new_terms.append((pre_a * scale_b if scale_b != 1.0 else pre_a, facs_a + facs_b))
    terms = new_terms
  return 1.0, terms


def _base_at_zero(f):
  """ Base-kernel value at distance 0 in the device's operation order. """
  if f.kind == _lib.DFB_BASE_SE:
    return f.scale * np.exp(-0.0)
  if f.kind == _lib.DFB_BASE_HAMMING:
    # every coordinate equal: (np.equal(x, x) * wts).sum(), NumPy's pairwise order
    return float(np.add.reduce(np.asarray(f.bandwidths, dtype=np.float64)))
  u = 0.0
  for i in range(f.p + 1):
    e = f.p - i
    u = u + f.coeffs[i] * (1.0 if e == 0 else 0.0)
  u = u * (f.gamma_ratio * np.exp(-0.0))
  return f.scale * u


def esp_combine(values, order):
  """ e_order(values) in the reference's operation order (ESPKernel._child_evaluate, kernel.py:710-726), for scalars or
      NumPy arrays: power sums p_i = ((0 + v_1^i) + v_2^i) + ... (^1 = v, ^2 = v * v, ^i>=3 = pow), then Newton-Girard
      e_m = (sum_{i=1..m} ((-1)^(i-1) e_{m-i}) p_i) / m. """
  p = [None] + [0.0 * values[0] for _ in range(order)]
  for i in range(1, order + 1):
    for v in values:
      p[i] = p[i] + (v if i == 1 else (v * v if i == 2 else v ** i))
  e = [1.0 + 0.0 * values[0]] + [None] * order
  for m in range(1, order + 1):
    acc = 0.0 * values[0]
    for i in range(1, m + 1):
      acc = acc + (((-1) ** (i - 1)) * e[m - i]) * p[i]
    e[m] = acc / m
  return e[order]


def _expand_esp(kern, train_coords, cand_coords):
  """ ESPKernel -> (scale, one term per 1-D child) for the ESP form of the descriptor (esp_order > 0). """
  if len(kern.kernel_list) != len(train_coords):
    raise ValueError('ESP kernel has %d children for %d coordinates' % (len(kern.kernel_list), len(train_coords)))
  terms = []
  for t, sub in enumerate(kern.kernel_list):
    if _kind_of(sub) not in ('SEKernel', 'MaternKernel') or int(sub.dim) != 1:
      raise NotImplementedError('ESP children must be 1-D SE or Matern kernels on device (got %s).'
                                % (type(sub).__name__))
    _, sub_terms = _expand(sub, [train_coords[t]], [cand_coords[t]])
    terms += sub_terms
  return float(kern.hyperparams['scale']), terms


def build_descriptor(kern, train_dim=None, cand_coords=None, train_coords=None, cand_dim=None):
  """ kern -> _lib.KernelDesc.  By default train and candidate matrices share the column layout
      (kernel applied to columns 0..dim-1).  Add-UCB passes train_coords = the group's columns of
      the training matrix and cand_coords = 0..d_j-1 (gpb_acquisitions.py:160-168). """
  dim = int(kern.dim)
  if train_coords is None:
    train_coords = list(range(dim))
  if cand_coords is None:
    cand_coords = list(range(dim))
  if train_dim is None:
    train_dim = max(train_coords) + 1
  if cand_dim is None:
    cand_dim = max(cand_coords) + 1
  esp_order = 0
  if _kind_of(kern) == 'ESPKernel':
    esp_order = int(kern.hyperparams['order'])
    post, terms = _expand_esp(kern, train_coords, cand_coords)
  else:
    post, terms = _expand(kern, train_coords, cand_coords)
  n_factors = sum(len(facs) for _, facs in terms)
  n_slots = sum(len(f.bandwidths) for _, facs in terms for f in facs)
  if len(terms) > _lib.DFB_MAX_TERMS or n_factors > _lib.DFB_MAX_FACTORS or \
     n_slots > _lib.DFB_MAX_SLOTS:
    raise NotImplementedError('kernel too large for the device descriptor: %d terms, %d factors, '
                              '%d slots' % (len(terms), n_factors, n_slots))
  d = _lib.KernelDesc()
  d.n_terms, d.n_factors, d.n_slots = len(terms), n_factors, n_slots
  d.train_dim, d.cand_dim = int(train_dim), int(cand_dim)
  d.post_scale = float(post)
  fi, si = 0, 0
  total = 0.0
  for ti, (pre, facs) in enumerate(terms):
    d.term_first_factor[ti] = fi
    d.term_pre_scale[ti] = float(pre)
    prod = float(pre)
    for f in facs:
      fd = d.factors[fi]
      fd.kind, fd.p, fd.n_dims, fd.slot_off = f.kind, f.p, len(f.bandwidths), si
      fd.scale, fd.s8, fd.s2, fd.gamma_ratio = f.scale, f.s8, f.s2, f.gamma_ratio
      for i, cval in enumerate(f.coeffs):
        fd.coeffs[i] = cval
      for q in range(len(f.bandwidths)):
        d.slot_train_coord[si] = f.train_coords[q]
        d.slot_cand_coord[si] = f.cand_coords[q]
        d.slot_bandwidth[si] = f.bandwidths[q]
        si += 1
      prod = prod * (_base_at_zero(f) if f.kind in _STATIONARY_KINDS else np.nan)
      fi += 1
    total = total + prod
  d.term_first_factor[len(terms)] = fi
  # NaN for a non-stationary kernel (a POLY or EXPDECAY factor): no k(x, x) holds for every x
  d.kss = float(post * total) if is_stationary(d) else float('nan')
  if esp_order:
    # stationary: k(x, x) = scale * e_order(child values at distance 0)
    d.esp_order = esp_order
    d.kss = float(post * esp_combine([_base_at_zero(facs[0]) for _, facs in terms], esp_order))
  check_esp_descriptor(d)
  return d


_STATIONARY_KINDS = (_lib.DFB_BASE_SE, _lib.DFB_BASE_MATERN, _lib.DFB_BASE_HAMMING)


def is_stationary(d):
  """ Whether k(x, x) is the same for every x: no factor of the descriptor is POLY or EXPDECAY (api.cu and common.cuh:
      kernel_stationary). """
  return all(d.factors[f].kind in _STATIONARY_KINDS for f in range(d.n_factors))


def check_esp_descriptor(d):
  """ The ESP rules of dfb_set_kernel's descriptor check (api.cu: check_desc), raised as ValueError before the
      descriptor reaches the device: 0 <= esp_order <= n_terms, and for esp_order > 0 every term one 1-slot factor with
      pre_scale 1. """
  if d.esp_order < 0 or d.esp_order > d.n_terms:
    raise ValueError('ESP order %d outside 0 .. n_terms = %d' % (d.esp_order, d.n_terms))
  if d.esp_order > 0:
    for t in range(d.n_terms):
      f = d.term_first_factor[t]
      if d.term_first_factor[t + 1] != f + 1 or d.factors[f].n_dims != 1 or d.term_pre_scale[t] != 1.0:
        raise ValueError('ESP term %d is not one 1-slot factor with pre_scale 1' % (t))
