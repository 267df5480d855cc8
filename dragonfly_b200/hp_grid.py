"""
The hyper-parameter "grid" objective of GPFitter on the device (SURVEY.md 8 row a23):

  GPFitter._tuning_objective (gp_core.py:551-563)  = LML of the GP built from one hp vector
  GPFitter.build_gp (gp_core.py:501-543)           : [mean const if mean_func_type == 'tune'],
                                                     [log noise if noise_var_type == 'tune'], child hps
  EuclideanGPFitter._child_build_gp (euclidean_gp.py:325-339) /
  get_euclidean_integral_gp_kernel_with_scale (:808-900): log scale, log bandwidth (x d or x 1),
                                                     discrete nu for Matern
  _rand_exp_sampling_wrap (gp_core.py:439-445)     : probs = exp(lml - max lml), normalised

Each objective evaluation is one DFB_BUILD_LML_ONLY factorisation (K build + blocked Cholesky with
the y row riding along; no L^-1, no alpha).  The samples are independent, so under torch.distributed
they shard across ranks with one all-gather of the LML values at the end (NCCL on GPUs, gloo in the
CPU tests of the sharding logic).
"""
import numpy as np

from . import _lib
from .kernel import SEKernel, MaternKernel, ExpDecayKernel, AdditiveKernel, CoordinateProductKernel, ESPKernelSE, \
    ESPKernelMatern, HammingKernel, CategoryCodes, build_descriptor
from .gp_core import stable_cholesky_on_device


class EuclideanHPLayout(object):
  """ How a continuous hp vector maps to (mean const, noise var, kernel) for an SE / Matern / ESP GP.
      ESP (kernel_type 'esp', euclidean_gp.py:283-299, 249-251, 816-892): log scale and d log bandwidths whatever
      use_same_bandwidth says; discrete hps [nu]? (esp_kernel_type 'matern' with esp_matern_nu < 0) then [order]?
      (esp_order == -1), handed to unpack as one tuple per sample. """

  def __init__(self, dim, kernel_type='matern', nu=2.5, use_same_bandwidth=False,
               mean_func_type='median', mean_func_const=0.0, noise_var_type='tune',
               noise_var_label=0.05, noise_var_value=0.1, use_additive_gp=False, add_max_group_size=6,
               num_groups_per_group_size=-1, esp_kernel_type='se', esp_order=-1, esp_matern_nu=-1.0):
    if kernel_type not in ('se', 'matern', 'esp'):
      raise NotImplementedError('kernel_type %s is outside the GPU hot-path scope.' % (kernel_type))
    if kernel_type == 'esp':
      if esp_kernel_type not in ('se', 'matern'):
        raise NotImplementedError('esp_kernel_type %s is not implemented (euclidean_gp.py:285-286).'
                                  % (esp_kernel_type))
      if use_additive_gp:
        raise NotImplementedError('use_additive_gp with an ESP kernel is outside the device path.')
    self.esp_kernel_type, self.esp_order, self.esp_matern_nu = esp_kernel_type, esp_order, esp_matern_nu
    self.dim, self.kernel_type, self.nu = dim, kernel_type, nu
    self.use_same_bandwidth = use_same_bandwidth
    self.mean_func_type, self.mean_func_const = mean_func_type, mean_func_const
    self.noise_var_type = noise_var_type
    self.noise_var_label, self.noise_var_value = noise_var_label, noise_var_value
    # additive models (euclidean_gp.py:50-60, 243-248): the group size is one more discrete hyper-parameter and
    # every objective evaluation carries a random grouping of the coordinates
    self.use_additive_gp = use_additive_gp
    self.add_max_group_size = min(add_max_group_size, dim)
    self.num_groups_per_group_size = num_groups_per_group_size

  def num_hps(self):
    n = 1 + (1 if self.use_same_bandwidth and self.kernel_type != 'esp' else self.dim)
    n += 1 if self.mean_func_type == 'tune' else 0
    n += 1 if self.noise_var_type == 'tune' else 0
    return n

  def _mean_noise_bounds(self, Y):
    """ (Y_var, [mean bounds]? [log noise bounds]?) as GPFitter._set_up sets them up (gp_core.py:336-338, 396-416). """
    Y = np.asarray(Y, dtype=np.float64)
    Y_var = Y.std() ** 2 + 0.0001 if len(Y) > 0 else 0.0001
    out = []
    if self.mean_func_type == 'tune':
      Y_std = np.sqrt(Y_var)
      Y_median = np.median(Y) if len(Y) > 0 else 0.0
      Y_half_range = 0.5 * (max(Y) - min(Y)) if len(Y) > 0 else 1.0
      Y_width = 0.5 * (Y_half_range + Y_std)
      out.append([Y_median - 3 * Y_width, Y_median + 3 * Y_width])
    if self.noise_var_type == 'tune':
      out.append([np.log(0.005 * Y_var), np.log(0.2 * Y_var)])
    return Y_var, out

  def bounds(self, X, Y, tune_nu=None):
    """ (cts_hp_bounds, dscr_hp_vals) the way the reference's fitter sets them up from the data
        (gp_core.py:336-338, 396-416; euclidean_gp.py:253-276): mean value (if tuned), log noise (if tuned),
        log scale, log bandwidth(s); discrete [0.5, 1.5, 2.5] for a Matern kernel whose nu is tuned
        (options.matern_nu < 0; default here: tuned iff self.nu is None or negative). """
    X = np.asarray(X, dtype=np.float64)
    Y_var, out = self._mean_noise_bounds(Y)
    out.append([np.log(0.1 * Y_var), np.log(10 * Y_var)])
    X_std_norm = np.linalg.norm(X, 'fro') + 1e-4
    single = [np.log(0.01 * X_std_norm), np.log(10 * X_std_norm)]
    out += [single] * (1 if self.use_same_bandwidth and self.kernel_type != 'esp' else self.dim)
    if self.kernel_type == 'esp':
      dscr = [[0.5, 1.5, 2.5]] if (self.esp_kernel_type == 'matern' and self.esp_matern_nu < 0) else []
      if self.esp_order == -1:
        dscr.append(list(range(1, max(self.dim, self.esp_order) + 1)))
      return np.array(out), dscr
    if tune_nu is None:
      tune_nu = self.kernel_type == 'matern' and (self.nu is None or self.nu < 0)
    dscr = [[0.5, 1.5, 2.5]] if (self.kernel_type == 'matern' and tune_nu) else []
    if self.use_additive_gp:
      dscr.append([x + 1 for x in range(self.add_max_group_size)])
    return np.array(out), dscr

  def _mean_and_noise(self, hp, Y):
    """ Pops the mean value / log noise from the front of `hp` when they are tuned (gp_core.py:509-538). """
    if self.mean_func_type == 'mean':
      mean_const = np.mean(Y)
    elif self.mean_func_type == 'median':
      mean_const = np.median(Y)
    elif self.mean_func_type == 'upper_bound':
      mean_const = np.mean(Y) + 3 * np.std(Y)
    elif self.mean_func_type == 'const':
      mean_const = self.mean_func_const
    elif self.mean_func_type == 'tune':
      mean_const = hp.pop(0)
    else:
      mean_const = 0
    if self.noise_var_type == 'tune':
      noise_var = np.exp(hp.pop(0))
    elif self.noise_var_type == 'label':
      noise_var = self.noise_var_label * (Y.std() ** 2)
    else:
      noise_var = self.noise_var_value
    return mean_const, noise_var

  def unpack(self, hp, Y, nu=None, groupings=None):
    """ gp_core.py:509-538 + euclidean_gp.py:801-861 """
    hp = list(np.asarray(hp, dtype=np.float64))
    Y = np.asarray(Y, dtype=np.float64)
    mean_const, noise_var = self._mean_and_noise(hp, Y)
    scale = np.exp(hp.pop(0))
    if self.kernel_type == 'esp':
      return float(mean_const), float(noise_var), self._esp_kernel(scale, hp, nu)
    if self.use_same_bandwidth:
      bws = [np.exp(hp.pop(0))] * self.dim
    else:
      bws = [np.exp(hp.pop(0)) for _ in range(self.dim)]
    assert len(hp) == 0
    nu = self.nu if nu is None else nu
    if groupings is not None:
      # get_euclidean_integral_gp_kernel_with_scale (euclidean_gp.py:826-831, 850-861, 895-897): group kernels
      # with scale 1 on their own bandwidths, the outer scale on the sum
      groups = [[int(i) for i in grp] for grp in groupings]
      make = (lambda grp: SEKernel(len(grp), 1.0, [bws[i] for i in grp])) if self.kernel_type == 'se' else \
             (lambda grp: MaternKernel(len(grp), nu, 1.0, [bws[i] for i in grp]))
      kern = AdditiveKernel(scale, [make(grp) for grp in groups], groups)
    elif self.kernel_type == 'se':
      kern = SEKernel(self.dim, scale, bws)
    else:
      kern = MaternKernel(self.dim, nu, scale, bws)
    return float(mean_const), float(noise_var), kern

  def _esp_kernel(self, scale, hp, dscr):
    """ get_euclidean_integral_gp_kernel_with_scale for kernel_type 'esp' (euclidean_gp.py:816-824, 841-847,
        878-892): the order is the last discrete hp unless fixed, nu (the same for every dimension) the first. """
    bws = [np.exp(h) for h in hp[:self.dim]]
    assert len(hp) == self.dim
    dscr = [] if dscr is None else list(dscr)
    if self.esp_order > 0:
      order = self.esp_order
    else:
      order, dscr = dscr[-1], dscr[:-1]
    if self.esp_kernel_type == 'se':
      return ESPKernelSE(self.dim, scale, int(order), bws)
    nu = self.esp_matern_nu if self.esp_matern_nu > 0 else dscr[0]
    return ESPKernelMatern(self.dim, [nu] * self.dim, scale, int(order), bws)


class EuclideanMFHPLayout(EuclideanHPLayout):
  """ Hyper-parameter vector of the reference's EuclideanMFGPFitter (euclidean_gp.py:432-483, 680-709) with SE / Matern
      fidelity and domain kernels: [mean const]? [log noise]? log scale, log fidelity bandwidth(s), log domain
      bandwidth(s); at most one tuned Matern nu (fidelity or domain) as the discrete hp.  The GP lives on [z || x] rows
      with the product kernel scale * k_F(z, z') * k_D(x, x') (fidelity and domain kernels with scale 1).  An ExpDecay
      fidelity kernel has no bandwidths: EuclideanMFExpDecayHPLayout below. """
  FIDEL_KERNEL_TYPES = ('se', 'matern')

  def __init__(self, fidel_dim, domain_dim, fidel_kernel_type='se', domain_kernel_type='se', fidel_nu=2.5,
               domain_nu=2.5, fidel_use_same_bandwidth=False, domain_use_same_bandwidth=False, **kwargs):
    for kt, allowed in ((fidel_kernel_type, self.FIDEL_KERNEL_TYPES), (domain_kernel_type, ('se', 'matern'))):
      if kt not in allowed:
        raise NotImplementedError('kernel_type %s is outside the GPU hot-path scope of %s.' % (kt, type(self).__name__))
    super(EuclideanMFHPLayout, self).__init__(fidel_dim + domain_dim, 'se', **kwargs)
    self.fidel_dim, self.domain_dim = fidel_dim, domain_dim
    self.fidel_kernel_type, self.domain_kernel_type = fidel_kernel_type, domain_kernel_type
    self.fidel_nu, self.domain_nu = fidel_nu, domain_nu
    self.fidel_use_same_bandwidth = fidel_use_same_bandwidth
    self.domain_use_same_bandwidth = domain_use_same_bandwidth
    if self.use_additive_gp:
      raise NotImplementedError('Additive domain kernels in the MF fitter are outside the device path.')

  def tuned_nus(self):
    return [self.fidel_kernel_type == 'matern' and self.fidel_nu < 0,
            self.domain_kernel_type == 'matern' and self.domain_nu < 0]

  def _num_fidel_hps(self):
    return 1 if self.fidel_use_same_bandwidth else self.fidel_dim

  def num_hps(self):
    n = 1 + self._num_fidel_hps()
    n += 1 if self.domain_use_same_bandwidth else self.domain_dim
    n += 1 if self.mean_func_type == 'tune' else 0
    n += 1 if self.noise_var_type == 'tune' else 0
    return n

  def bounds(self, X, Y, tune_nu=None):
    raise NotImplementedError('Use the bounds of the reference EuclideanMFGPFitter (fitter.cts_hp_bounds).')

  @staticmethod
  def _bandwidths(hp, n, same):
    return [np.exp(hp.pop(0))] * n if same else [np.exp(hp.pop(0)) for _ in range(n)]

  def _fidel_kernel(self, hp, nu):
    """ Pops the fidelity kernel's hps from the front of `hp` (after the scale) and returns the kernel (scale 1). """
    bws = self._bandwidths(hp, self.fidel_dim, self.fidel_use_same_bandwidth)
    if self.fidel_kernel_type == 'se':
      return SEKernel(self.fidel_dim, 1.0, bws)
    return MaternKernel(self.fidel_dim, nu, 1.0, bws)

  def unpack(self, hp, Y, nu=None, groupings=None):
    """ gp_core.py:509-538 + euclidean_gp.py:680-709 """
    hp = list(np.asarray(hp, dtype=np.float64))
    Y = np.asarray(Y, dtype=np.float64)
    mean_const, noise_var = self._mean_and_noise(hp, Y)
    scale = np.exp(hp.pop(0))
    f_tuned, d_tuned = self.tuned_nus()
    assert not (f_tuned and d_tuned), 'at most one tuned Matern nu on the device path'
    k_f = self._fidel_kernel(hp, nu if f_tuned else self.fidel_nu)
    d_bws = self._bandwidths(hp, self.domain_dim, self.domain_use_same_bandwidth)
    assert len(hp) == 0
    d_nu = nu if d_tuned else self.domain_nu
    k_d = SEKernel(self.domain_dim, 1.0, d_bws) if self.domain_kernel_type == 'se' else \
        MaternKernel(self.domain_dim, d_nu, 1.0, d_bws)
    fidel_coords = list(range(self.fidel_dim))
    domain_coords = list(range(self.fidel_dim, self.fidel_dim + self.domain_dim))
    kern = CoordinateProductKernel(self.dim, scale, [k_f, k_d], [fidel_coords, domain_coords])
    return float(mean_const), float(noise_var), kern


class EuclideanMFExpDecayHPLayout(EuclideanMFHPLayout):
  """ EuclideanMFGPFitter with fidel_kernel_type 'expdecay' (the freeze-thaw fidelity kernel): the fidelity part of the
      hp vector is [log offset, log power x fidel_dim] (_fidel_expdecay_kernel_setup, euclidean_gp.py:521-541), unpacked
      into ExpDecayKernel(fidel_dim, 1.0, exp(offset), exp(powers)) (get_euclidean_integral_gp_kernel_with_scale,
      :871-877); fidel_use_same_bandwidth plays no part, as in the reference.  The domain kernel is SE or Matern. """
  FIDEL_KERNEL_TYPES = ('expdecay',)

  def __init__(self, fidel_dim, domain_dim, domain_kernel_type='se', domain_nu=2.5, domain_use_same_bandwidth=False,
               **kwargs):
    super(EuclideanMFExpDecayHPLayout, self).__init__(fidel_dim, domain_dim, 'expdecay', domain_kernel_type,
                                                      domain_nu=domain_nu,
                                                      domain_use_same_bandwidth=domain_use_same_bandwidth, **kwargs)

  def _num_fidel_hps(self):
    return 1 + self.fidel_dim

  def _fidel_kernel(self, hp, nu):
    offset = np.exp(hp.pop(0))
    powers = np.exp(np.array([hp.pop(0) for _ in range(self.fidel_dim)]))
    return ExpDecayKernel(self.fidel_dim, 1.0, offset, powers)


class CPPart(object):
  """ One part of a Cartesian-product domain as CPGPFitter sees it: the domain type ('euclidean', 'integral',
      'prod_discrete_numeric' or 'prod_discrete'), its dimension, the resolved kernel type ('se' / 'matern' for the
      numeric parts, 'hamming' for prod_discrete), the Matern nu option as given (a float < 0: tuned; 'default': 2.5;
      > 0: fixed) and the part's same-bandwidth / same-weight flag. """

  NUMERIC = ('euclidean', 'integral', 'prod_discrete_numeric')

  def __init__(self, dom_type, dim, kernel_type, nu='default', same=False):
    self.dom_type, self.dim, self.kernel_type, self.nu, self.same = dom_type, int(dim), kernel_type, nu, bool(same)

  def nu_tuned(self):
    """ _set_up_hyperparams_for_domain adds a discrete nu only for a float option < 0 (cartesian_product_gp.py:532). """
    return self.kernel_type == 'matern' and isinstance(self.nu, float) and self.nu < 0

  def fixed_nu(self):
    """ The nu a Matern part is built with when it is not tuned; None when that is not a number. """
    if isinstance(self.nu, str):
      return 2.5 if self.nu == 'default' else None
    return self.nu if isinstance(self.nu, (int, float)) and not isinstance(self.nu, bool) else None


class CartesianProductHPLayout(EuclideanHPLayout):
  """ Hyper-parameter vector of the reference's CPGPFitter (cartesian_product_gp.py:325-391, 504-678, 817-945):
      [mean const]? [log noise]? log kernel scale, then per part in domain order
        euclidean / integral / prod_discrete_numeric (se, matern): one log bandwidth per dimension;
        prod_discrete (hamming): none (dim 1 or same weights: 1 / dim each), one linear weight w in [0, 1]
                                  (dim 2: [w, 1 - w]) or dim linear weights normalised by their sum (dim > 2);
      one discrete nu in [0.5, 1.5, 2.5] per Matern part whose nu option is a float < 0, in part order.  unpack takes the
      tuple of discrete hps and returns CartesianProductKernel(scale, [part kernels with scale 1]); its Hamming
      children carry this layout's CategoryCodes tables, so the rows of encode() and every kernel of a batch share one
      encoding.  Options the reference itself cannot build with (use_same_bandwidth, an integer or zero Matern nu) and
      parts outside the device path raise NotImplementedError. """

  def __init__(self, parts, mean_func_type='median', mean_func_const=0.0, noise_var_type='tune', noise_var_label=0.05,
               noise_var_value=0.1):
    parts = [p if isinstance(p, CPPart) else CPPart(*p) for p in parts]
    for p in parts:
      if p.dom_type in CPPart.NUMERIC:
        if p.kernel_type not in ('se', 'matern'):
          raise NotImplementedError('kernel_type %s on a %s part is outside the device path.'
                                    % (p.kernel_type, p.dom_type))
        if p.same:
          raise NotImplementedError('use_same_bandwidth on a Cartesian-product part: the reference raises in '
                                    '_set_up_dim_bandwidths.')
        if p.kernel_type == 'matern' and not p.nu_tuned() and not (p.fixed_nu() is not None and p.fixed_nu() > 0):
          raise NotImplementedError('Matern nu option %r: the reference pops a discrete hp it never set up.' % (p.nu,))
      elif p.dom_type == 'prod_discrete':
        if p.kernel_type != 'hamming':
          raise NotImplementedError('kernel_type %s on a prod_discrete part.' % (p.kernel_type))
      else:
        raise NotImplementedError('%s parts are outside the device path.' % (p.dom_type))
    dim = sum(p.dim for p in parts)
    super(CartesianProductHPLayout, self).__init__(dim, 'se', mean_func_type=mean_func_type,
                                                   mean_func_const=mean_func_const, noise_var_type=noise_var_type,
                                                   noise_var_label=noise_var_label, noise_var_value=noise_var_value)
    self.kernel_type = 'cartesian_product'
    self.parts = parts
    self.codes = [CategoryCodes() if p.dom_type == 'prod_discrete' else None for p in parts]

  @staticmethod
  def _num_part_hps(p):
    if p.dom_type != 'prod_discrete':
      return p.dim
    if p.same or p.dim == 1:
      return 0
    return 1 if p.dim == 2 else p.dim

  def num_hps(self):
    n = 1 + sum(self._num_part_hps(p) for p in self.parts)
    n += 1 if self.mean_func_type == 'tune' else 0
    n += 1 if self.noise_var_type == 'tune' else 0
    return n

  def num_dscr(self):
    return sum(p.nu_tuned() for p in self.parts)

  def bounds(self, X, Y, tune_nu=None):
    """ (cts_hp_bounds, dscr_hp_vals) of CPGPFitter._child_set_up on list-of-parts points X. """
    cts, dscr, _ = self.bounds_and_order(X, Y)
    return cts, dscr

  def bounds_and_order(self, X, Y):
    """ (cts_hp_bounds, dscr_hp_vals, param_order) as CPGPFitter sets them up (gp_core.py:323-350,
        cartesian_product_gp.py:371-377, 504-678). """
    Y_var, cts = self._mean_noise_bounds(Y)
    order = ([['noise_mean', 'cts']] if self.mean_func_type == 'tune' else []) + \
        ([['noise_var', 'cts']] if self.noise_var_type == 'tune' else [])
    order.append(['kernel_scale', 'cts'])
    cts.append([np.log(0.03 * Y_var), np.log(30 * Y_var)])
    dscr = []
    for idx, p in enumerate(self.parts):
      ident = 'dom-%d-%s' % (idx, p.dom_type)
      if p.dom_type == 'prod_discrete':
        if p.same or p.dim == 1:
          continue
        if p.dim == 2:
          cts.append([0, 1])
          order.append([ident + '-hamming_wt-2D', 'cts'])
        else:
          cts.extend([[0, 1]] * p.dim)
          order.extend([['%s-hamming_wts-%d' % (ident, i), 'cts'] for i in range(p.dim)])
        continue
      if p.nu_tuned():
        dscr.append([0.5, 1.5, 2.5])
        order.append(['%s-matern_nu' % (ident), 'dscr'])
      if len(X) > 0:
        part_X = np.array([x[idx] for x in X])
        diffs = part_X - part_X.mean(axis=0)
        norms = [np.linalg.norm(diffs[:, i]) + 1e-4 for i in range(p.dim)]
      else:
        norms = [1.0] * p.dim
      cts.extend([[np.log(0.01 * s), np.log(100 * s)] for s in norms])
      order.extend([['%s-dom_bandwidths-%d' % (ident, i), 'cts'] for i in range(p.dim)])
    return np.array(cts), dscr, order

  def encode(self, X):
    """ list-of-parts points -> (n, dim) float64 rows, the parts side by side and every category replaced by its code in
        the part's table (CartesianProductKernel / flatten_parts layout). """
    rows = []
    for x in X:
      cols = []
      for part, table in zip(x, self.codes):
        if table is None:
          cols.append(np.atleast_1d(np.asarray(part, dtype=np.float64)).reshape(-1))
        else:
          cols.append(np.array([table.encode(v) for v in part], dtype=np.float64))
      rows.append(np.concatenate(cols))
    return np.ascontiguousarray(np.array(rows, dtype=np.float64).reshape(len(rows), self.dim))

  def unpack(self, hp, Y, nu=None, groupings=None):
    """ gp_core.py:509-538 + CPGPFitter._child_build_gp / _build_kernel_for_domain (cartesian_product_gp.py:379-391,
        817-945).  `nu`: the tuple of discrete hps, one per tuned Matern part in part order. """
    from .cartesian_product_gp import CartesianProductKernel
    assert groupings is None
    hp = list(np.asarray(hp, dtype=np.float64))
    Y = np.asarray(Y, dtype=np.float64)
    mean_const, noise_var = self._mean_and_noise(hp, Y)
    dscr = [] if nu is None else list(nu)
    scale = np.exp(hp[0])
    hp = np.array(hp[1:])
    kernels = []
    for p, table in zip(self.parts, self.codes):
      if p.dom_type == 'prod_discrete':
        if p.dim == 1 or p.same:
          wts = np.ones((p.dim,)) / float(p.dim)
        elif p.dim == 2:
          wts = np.array([hp[0], 1 - hp[0]])
          hp = hp[1:]
        else:
          unnorm = np.array(hp[0:p.dim])
          total = unnorm.sum()
          wts = unnorm / total if total > 0 else np.ones((p.dim,)) / float(p.dim)
          hp = hp[p.dim:]
        kern = HammingKernel(wts)
        kern.category_codes = table
      else:
        bws = np.exp(hp[0:p.dim])
        hp = hp[p.dim:]
        if p.kernel_type == 'se':
          kern = SEKernel(p.dim, 1.0, bws)
        else:
          if p.nu_tuned():
            part_nu, dscr = dscr[0], dscr[1:]
          else:
            part_nu = p.fixed_nu()
          kern = MaternKernel(p.dim, part_nu, 1.0, bws)
      kernels.append(kern)
    assert len(hp) == 0 and len(dscr) == 0
    return float(mean_const), float(noise_var), CartesianProductKernel(scale, kernels)


# One LML-only build at N = 5000 is a 40-step dependency chain (chol_diag -> panel -> next column) that leaves most
# of the GPU idle (7.7 ms for 42 GFLOP); the hp samples are independent, so `lanes` of them are built
# concurrently -- one DevicePosterior (handle + workspace) per lane, each on its own CUDA stream, driven from its
# own host thread (ctypes releases the GIL during the C call).  Sample i goes to lane i % lanes; every LML is
# computed by the same kernels whatever the lane count, so the values do not depend on it.
DEFAULT_LANES = 3


def _lane_worker(lane_post, stream, X, Y, hps, idxs, layout, nus, out, groupings=None):
  import torch
  with torch.cuda.device(lane_post.device), torch.cuda.stream(stream):
    lane_post.bind_current_stream()
    last_mean = None
    for i in idxs:
      mean_const, noise_var, kern = layout.unpack(hps[i], Y, None if nus is None else nus[i],
                                                  None if groupings is None else groupings[i])
      if last_mean is None or mean_const != last_mean:
        lane_post.set_train(X, Y - mean_const)
        last_mean = mean_const
      lane_post.set_kernel(build_descriptor(kern, train_dim=X.shape[1], cand_dim=X.shape[1]))
      out[i], _ = stable_cholesky_on_device(lane_post, noise_var, flags=_lib.DFB_BUILD_LML_ONLY)


def lml_for_hyperparams(X, Y, hps, layout, nus=None, post=None, device=None, lanes=None, groupings=None):
  """ LML of the GP built from each hp vector (rows of `hps`); `nus` optionally gives the discrete
      Matern nu per sample.  Returns (lmls, post) -- `post` can be passed back in to reuse the
      device workspaces (it carries the extra lanes). """
  import threading
  import torch
  from .device import DevicePosterior
  X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
  Y = np.asarray(Y, dtype=np.float64)
  if post is None or post.n_max < len(X):
    post = DevicePosterior(len(X), device=device)
  lmls = np.empty(len(hps))
  if lanes is None:
    lanes = DEFAULT_LANES if len(hps) >= 2 * DEFAULT_LANES else 1
  lanes = max(1, min(int(lanes), len(hps)))
  if lanes == 1:
    _lane_worker(post, torch.cuda.current_stream(post.device), X, Y, hps, range(len(hps)), layout, nus, lmls,
                 groupings)
    return lmls, post
  extra = getattr(post, '_hp_lanes', [])
  while len(extra) < lanes - 1:
    extra.append((DevicePosterior(len(X), device=post.device.index), torch.cuda.Stream(post.device)))
  post._hp_lanes = extra
  main_stream = torch.cuda.current_stream(post.device)
  workers, errors = [], []

  def guarded(*a):
    try:
      _lane_worker(*a)
    except BaseException as e:  # pylint: disable=broad-except
      errors.append(e)
  for j in range(1, lanes):
    lane_post, stream = extra[j - 1]
    stream.wait_stream(main_stream)
    t = threading.Thread(target=guarded, args=(lane_post, stream, X, Y, hps, range(j, len(hps), lanes), layout,
                                               nus, lmls, groupings))
    t.start()
    workers.append(t)
  guarded(post, main_stream, X, Y, hps, range(0, len(hps), lanes), layout, nus, lmls, groupings)
  for t in workers:
    t.join()
  for j in range(1, lanes):
    main_stream.wait_stream(extra[j - 1][1])
  if errors:
    raise errors[0]
  return lmls, post


# Largest training set dfb_lml_batch serves (DESIGN.md 4.3, 10): one CTA factorises a whole item, so its time grows
# as N^3 on one SM while lml_for_hyperparams spreads each build over the GPU.
LML_BATCH_MAX_N = 512


def lml_batch_for_hyperparams(X, Y, hps, layout, nus=None, post=None, device=None):
  """ What lml_for_hyperparams returns, with every LML of a plain (not ESP, not additive) layout on N <= LML_BATCH_MAX_N
      points from ONE dfb_lml_batch call (dfb_lml_batch_mixed for a CartesianProductHPLayout, whose kernels have Hamming
      factors; X is then its encode()d rows).  Items that are not positive definite are rebuilt one at a time through
      stable_cholesky_on_device (its jitter ladder), as lml_for_hyperparams builds them.  Returns (lmls, post). """
  from .device import DevicePosterior
  X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
  Y = np.asarray(Y, dtype=np.float64)
  if (len(X) > LML_BATCH_MAX_N or getattr(layout, 'kernel_type', None) == 'esp' or
      getattr(layout, 'use_additive_gp', False)):
    return lml_for_hyperparams(X, Y, hps, layout, nus=nus, post=post, device=device)
  if post is None or post.n_max < len(X):
    post = DevicePosterior(len(X), device=device)
  key = (X.shape, X.tobytes(), Y.tobytes())
  if getattr(post, '_lml_batch_train', None) != key:
    post.set_train(X, Y)                          # raw Y: the kernel forms Y - mean_const per item
    post._lml_batch_train = key
  descs, noise, means = [], [], []
  for i, hp in enumerate(hps):
    mean_const, noise_var, kern = layout.unpack(hp, Y, None if nus is None else nus[i])
    descs.append(build_descriptor(kern, train_dim=X.shape[1], cand_dim=X.shape[1]))
    noise.append(noise_var)
    means.append(mean_const)
  if not descs:
    return np.empty(0), post
  lmls, infos = post.lml_batch(descs, noise, means, mixed=isinstance(layout, CartesianProductHPLayout))
  bad = np.nonzero(infos != 0)[0]
  for i in bad:
    post.set_train(X, Y - means[i])
    post.set_kernel(descs[i])
    lmls[i], _ = stable_cholesky_on_device(post, noise[i], flags=_lib.DFB_BUILD_LML_ONLY)
  if len(bad):
    post._lml_batch_train = None
  return lmls, post


def default_max_evals(method, num_hps):
  """ gp_core.py:456-462 """
  if method in ('direct', 'pdoo'):
    return int(min(1e4, max(500, num_hps * 50)))
  if method == 'rand':
    return int(min(1e4, max(500, num_hps * 200)))
  if method == 'rand_exp_sampling':
    return int(min(1e5, max(500, num_hps * 400)))
  raise ValueError('Unknown ml_hp_tune_opt method %s.' % (method))


def fit_gp(X, Y, layout, cts_hp_bounds, dscr_hp_vals=(), method='rand_exp_sampling', max_evals=None,
           device=None, gp_factory=None, build_gp=None):
  """ GPFitter.fit_gp for hp_tune_criterion == 'ml' (gp_core.py:783-808) with the marginal likelihood of every
      hyper-parameter vector evaluated on the device, in batches instead of one _tuning_objective call at a time
      (gp_core.py:551-563):
        'rand'               random_maximise over the continuous hps for every combination of the discrete ones
                             (oper_utils.py:69-80, gp_core.py:787-799): all max_evals candidates of a combination are
                             one lml_for_hyperparams call (concurrent build lanes);
        'pdoo' / 'direct'    pdoo_maximise (oper_utils.py:257-271; 'direct' is PDOO wherever the reference's Fortran
                             DIRECT is not built) through dragonfly_b200.doo: both children of a split in one call;
        'rand_exp_sampling'  random_sample_cts_dscr + exp(lml - max) weights (oper_utils.py:362-371,
                             gp_core.py:439-445): one call for all samples.
      The global NumPy RNG is consumed exactly like the reference does, so a seeded run picks the same
      hyper-parameters.  `cts_hp_bounds` / `dscr_hp_vals` are the fitter's (euclidean_gp.py:222-320); the discrete
      hps are the Matern nu (and for additive models the group size), or for an ESP layout [nu]? [order]?.  Returns what the reference returns:
        ('fitted_gp', gp, (cts_hps, dscr_hps))   or   ('sample_hps_with_probs', cts, dscr, [None] * n, probs). """
  from itertools import product as itertools_product
  from .gp_core import GP, ConstantMean
  from .gpb_acquisitions import map_to_bounds, _reference_fortran_direct_available
  cp = isinstance(layout, CartesianProductHPLayout)
  if cp:
    X_parts = list(X)                                # CPGPFitter's list-of-parts points
    X = layout.encode(X_parts)
  X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
  Y = np.asarray(Y, dtype=np.float64)
  bounds = np.asarray(cts_hp_bounds, dtype=np.float64)
  dscr_hp_vals = [list(v) for v in dscr_hp_vals]
  additive = bool(getattr(layout, 'use_additive_gp', False))
  esp = getattr(layout, 'kernel_type', None) == 'esp'
  if not cp and len(dscr_hp_vals) > (2 if additive or esp else 1):
    raise NotImplementedError('Discrete hyper-parameters on the device path: the Matern nu and, for additive '
                              'models, the group size.')
  has_nu = len(dscr_hp_vals) == (2 if additive else 1)       # [nu]? then [group size]? (euclidean_gp.py:226-248)

  def kernel_dscr(dscr):
    """ What unpack / lml_for_hyperparams take per sample: nu (SE / Matern), the tuple [nu]? [order]? (ESP), or the
        tuple of every tuned Matern nu (Cartesian product). """
    if cp:
      return tuple(dscr)
    if esp:
      return tuple(dscr) if len(dscr) else None
    return dscr[0] if has_nu else None
  dim = layout.dim
  if max_evals is None:
    max_evals = default_max_evals(method, len(bounds) + len(dscr_hp_vals))
  n_evals = int(max_evals)
  state = {'post': None}

  def lmls_of(hps, nus, groupings=None):
    if cp:                                           # one dfb_lml_batch_mixed launch per batch up to LML_BATCH_MAX_N
      vals, state['post'] = lml_batch_for_hyperparams(X, Y, hps, layout, nus=nus, post=state['post'], device=device)
      return vals
    vals, state['post'] = lml_for_hyperparams(X, Y, hps, layout, nus=nus, post=state['post'], device=device,
                                              groupings=groupings)
    return vals

  def build(cts, dscr, groupings=None):
    if build_gp is not None:                         # e.g. the reference fitter's own build_gp (fit_gp_on_fitter)
      return build_gp(cts, dscr, groupings)
    mean_const, noise_var, kern = layout.unpack(cts, Y, kernel_dscr(dscr), groupings)
    if cp:
      from .cartesian_product_gp import CPGP
      make = CPGP if gp_factory is None else gp_factory
      return make(X_parts, list(Y), kern, ConstantMean(mean_const), noise_var)
    make = GP if gp_factory is None else gp_factory
    return make(list(X), list(Y), kern, ConstantMean(mean_const), noise_var)

  def random_grouping(group_size):
    rand_perm = list(np.random.permutation(dim))               # euclidean_gp.py:733-735, 760-761
    return [rand_perm[i:i + group_size] for i in range(0, dim, group_size)]

  if method == 'rand_exp_sampling':
    if additive:
      # sample_cts_dscr_hps_for_rand_exp_sampling_in_add_model (euclidean_gp.py:749-776): per sample a group size, a
      # random grouping, the discrete hps (group size overwritten), the continuous hps -- in that RNG order; the
      # weights are exp(lml) / sum WITHOUT subtracting the maximum, as written there
      cts, dscr, groupings = [], [], []
      for _ in range(n_evals):
        group_size = np.random.choice(dscr_hp_vals[-1])
        groupings.append(random_grouping(group_size))
        cur = [np.random.choice(categ) for categ in dscr_hp_vals]
        cur[-1] = group_size
        dscr.append(cur)
        cts.append(map_to_bounds(np.random.random((len(bounds),)), bounds))
      vals = lmls_of(np.array(cts), [d[0] for d in dscr] if has_nu else None, groupings)
      probs = np.exp(vals)
      from argparse import Namespace
      other = [Namespace(add_gp_groupings=grp) for grp in groupings]      # as the reference returns them (:762)
      return 'sample_hps_with_probs', cts, dscr, other, probs / probs.sum()
    cts = map_to_bounds(np.random.random((n_evals, len(bounds))), bounds)
    dscr = [[np.random.choice(categ) for categ in dscr_hp_vals] for _ in range(n_evals)]
    vals = lmls_of(cts, [kernel_dscr(d) for d in dscr] if dscr_hp_vals else None)
    return 'sample_hps_with_probs', cts, dscr, [None] * n_evals, rand_exp_sampling_probs(vals)
  if method == 'direct' and _reference_fortran_direct_available():
    raise NotImplementedError('Fortran DIRECT is a sequential host optimiser; use pdoo / rand / rand_exp_sampling.')
  if method not in ('rand', 'pdoo', 'direct'):
    raise ValueError('Unknown ml_hp_tune_opt method %s.' % (method))

  def optimise_cts(nu, evals, groupings=None):
    """ cts_hp_optimise (gp_core.py:463-472) for one setting of the discrete hps (and one grouping). """
    rep = (lambda k: None) if groupings is None else (lambda k: [groupings] * k)
    if method == 'rand':
      pts = map_to_bounds(np.random.random((int(evals), len(bounds))), bounds)
      vals = lmls_of(pts, None if nu is None else [nu] * len(pts), rep(len(pts)))
      idx = int(np.argmax(vals))
      return vals[idx], pts[idx]
    from .doo import pdoo_maximise
    val, pt, _ = pdoo_maximise(lambda P: lmls_of(P, None if nu is None else [nu] * len(P), rep(len(P))), bounds,
                               evals)
    return val, pt

  best_val, best_cts, best_dscr, best_groupings = -np.inf, None, None, None
  for dscr in itertools_product(*dscr_hp_vals):
    nu = kernel_dscr(dscr)
    if not additive:
      opt_val, opt_pt, opt_groupings = optimise_cts(nu, max_evals) + (None,)
    else:
      # optimise_cts_hps_for_given_dscr_hps_in_add_model (euclidean_gp.py:718-746)
      group_size = dscr[-1]
      n_groupings = layout.num_groups_per_group_size
      if n_groupings < 0:
        n_groupings = 1 if group_size == 1 else max(5, min(2 * dim, 25))
      opt_val, opt_pt, opt_groupings = -np.inf, None, None
      for _ in range(n_groupings):
        groupings = random_grouping(group_size)
        val, pt = optimise_cts(nu, int(max(500, max_evals / n_groupings)), groupings)
        if val > opt_val:
          opt_val, opt_pt, opt_groupings = val, pt, groupings
    if opt_val > best_val:
      best_val, best_cts, best_dscr, best_groupings = opt_val, list(opt_pt), list(dscr), opt_groupings
  return 'fitted_gp', build(best_cts, best_dscr, best_groupings), (best_cts, best_dscr)


# ---- drop-in for GPFitter.fit_gp on a Dragonfly EuclideanGPFitter (INTEGRATION.md 2e) --------------------------------
def layout_from_fitter(fitter):
  """ The EuclideanHPLayout equivalent to a reference EuclideanGPFitter's options (euclidean_gp.py:205-248,
      gp_core.py:509-538), or None when the fitter tunes something the device path does not cover. """
  opt = fitter.options
  if getattr(opt, 'mean_func', None) is not None:
    return None
  common = dict(mean_func_type=opt.mean_func_type, mean_func_const=getattr(opt, 'mean_func_const', 0.0),
                noise_var_type=opt.noise_var_type, noise_var_label=getattr(opt, 'noise_var_label', 0.05),
                noise_var_value=getattr(opt, 'noise_var_value', 0.1))
  if hasattr(fitter, 'domain_kernel_ordering') or hasattr(fitter, 'fidel_space'):
    return _cp_layout_from_fitter(fitter, common)
  if hasattr(fitter, 'fidel_dim') and hasattr(opt, 'fidel_kernel_type'):
    # EuclideanMFGPFitter (euclidean_gp.py:418-716); a 'poly' fidelity or domain kernel stays with the reference,
    # whose fitter raises NotImplementedError for it (:515-519, 587-591, 619-621)
    if (opt.fidel_kernel_type not in ('se', 'matern', 'expdecay') or opt.domain_kernel_type not in ('se', 'matern') or
        getattr(opt, 'domain_use_additive_gp', False)):
      return None
    domain = dict(domain_nu=getattr(opt, 'domain_matern_nu', 2.5),
                  domain_use_same_bandwidth=bool(getattr(opt, 'domain_use_same_bandwidth', False)), **common)
    if opt.fidel_kernel_type == 'expdecay':
      return EuclideanMFExpDecayHPLayout(fitter.fidel_dim, fitter.domain_dim, opt.domain_kernel_type, **domain)
    layout = EuclideanMFHPLayout(
        fitter.fidel_dim, fitter.domain_dim, opt.fidel_kernel_type, opt.domain_kernel_type,
        fidel_nu=getattr(opt, 'fidel_matern_nu', 2.5),
        fidel_use_same_bandwidth=bool(getattr(opt, 'fidel_use_same_bandwidth', False)), **domain)
    return None if sum(layout.tuned_nus()) > 1 else layout
  kernel_type = getattr(fitter, 'kernel_type', getattr(opt, 'kernel_type', None))
  additive = bool(getattr(opt, 'use_additive_gp', False))
  if kernel_type == 'esp':
    # EuclideanGPFitter._esp_kernel_set_up (euclidean_gp.py:283-299); ESP together with use_additive_gp falls through
    if additive or getattr(opt, 'esp_kernel_type', 'se') not in ('se', 'matern'):
      return None
    return EuclideanHPLayout(fitter.dim, 'esp', esp_kernel_type=getattr(opt, 'esp_kernel_type', 'se'),
                             esp_order=int(getattr(opt, 'esp_order', -1)),
                             esp_matern_nu=getattr(opt, 'esp_matern_nu', -1.0), **common)
  if kernel_type not in ('se', 'matern'):
    return None
  return EuclideanHPLayout(
      fitter.dim, kernel_type, nu=getattr(opt, 'matern_nu', 2.5),
      use_same_bandwidth=bool(getattr(opt, 'use_same_bandwidth', False)),
      mean_func_type=opt.mean_func_type, mean_func_const=getattr(opt, 'mean_func_const', 0.0),
      noise_var_type=opt.noise_var_type, noise_var_label=getattr(opt, 'noise_var_label', 0.05),
      noise_var_value=getattr(opt, 'noise_var_value', 0.1), use_additive_gp=additive,
      add_max_group_size=getattr(fitter, 'add_max_group_size', getattr(opt, 'add_max_group_size', 6)),
      num_groups_per_group_size=getattr(opt, 'num_groups_per_group_size', -1))


_CP_OPTION_CODES = {'euclidean': 'euc', 'integral': 'int', 'prod_discrete_numeric': 'disc_num', 'prod_discrete': 'disc'}
_CP_DEFAULT_KERNELS = {'euclidean': 'matern', 'integral': 'matern', 'prod_discrete_numeric': 'matern',
                       'prod_discrete': 'hamming'}


def _cp_layout_from_fitter(fitter, common):
  """ The CartesianProductHPLayout of a reference CPGPFitter: its domain's parts (fitter.domain.list_of_domains), their
      kernel types from fitter.domain_kernel_ordering, or the dom_*_kernel_type options when an entry is empty, 'default'
      resolved by part type (_get_kernel_type_from_options, get_default_kernel_type, cartesian_product_gp.py:188-203,
      622-634), and the dom_* options of each part.  None for a CPMFGPFitter, precomputed distance lists, additive
      parts, and anything CartesianProductHPLayout refuses: those fits stay with the reference. """
  opt = fitter.options
  domain = getattr(fitter, 'domain', None)
  ordering = getattr(fitter, 'domain_kernel_ordering', None)
  if (hasattr(fitter, 'fidel_space') or domain is None or ordering is None or
      not hasattr(domain, 'list_of_domains') or len(ordering) != len(domain.list_of_domains)):
    return None
  if any(d is not None for d in (getattr(fitter, 'domain_lists_of_dists', None) or [])):
    return None
  parts = []
  for dom, kernel_type in zip(domain.list_of_domains, ordering):
    dom_type = dom.get_type()
    code = _CP_OPTION_CODES.get(dom_type)
    if code is None:
      return None
    if kernel_type == '' or kernel_type is None:
      kernel_type = getattr(opt, 'dom_%s_kernel_type' % code, None)
    if kernel_type == 'default':
      kernel_type = _CP_DEFAULT_KERNELS[dom_type]
    if dom_type == 'prod_discrete':
      parts.append(CPPart(dom_type, dom.get_dim(), kernel_type, same=getattr(opt, 'dom_disc_hamming_use_same_weight',
                                                                             False)))
      continue
    if code in ('euc', 'int') and getattr(opt, 'dom_%s_use_additive_gp' % code, False):
      return None
    parts.append(CPPart(dom_type, dom.get_dim(), kernel_type, nu=getattr(opt, 'dom_%s_matern_nu' % code, 'default'),
                        same=getattr(opt, 'dom_%s_use_same_bandwidth' % code, False)))
  try:
    return CartesianProductHPLayout(parts, **common)
  except NotImplementedError:
    return None


def post_sampling_covers(layout):
  """ The layouts whose 'post_sampling' fits run on the device (post_sampling.post_sample_hps): SE / Matern, not
      additive; the MF product of SE / Matern fidelity and domain kernels; Cartesian products of SE / Matern and Hamming
      parts without a tuned nu.  ESP and ExpDecay stay with the reference, and so do CP fitters with a tuned nu: the
      reference's sampler takes hp i as discrete when param_order[i] says so (gp_core.py:689-697), and CPGPFitter lists a
      part's nu before that part's bandwidths, so its fit fails or samples bandwidths as categories. """
  if type(layout) is EuclideanHPLayout:
    return layout.kernel_type in ('se', 'matern') and not layout.use_additive_gp
  if type(layout) is CartesianProductHPLayout:
    return layout.num_dscr() == 0
  return type(layout) is EuclideanMFHPLayout


def _fitter_data(fitter, layout):
  """ The rows the fitter's GPs are built on: [z || x] for an MF fitter, the list-of-parts points for a CP fitter (the
      layout encodes them). """
  if isinstance(layout, CartesianProductHPLayout):
    return list(fitter.X), np.array(fitter.Y)
  if isinstance(layout, EuclideanMFHPLayout):
    X_mat = np.concatenate((np.asarray(fitter.ZZ, dtype=np.float64).reshape(len(fitter.YY), -1),
                            np.asarray(fitter.XX, dtype=np.float64).reshape(len(fitter.YY), -1)), axis=1)
    return X_mat, np.array(fitter.YY)
  return np.array(fitter.X), np.array(fitter.Y)


def fit_gp_on_fitter(fitter, reference_fit_gp, num_samples=1, hp_tune_criterion=None):
  """ GPFitter.fit_gp (gp_core.py:783-821) for a reference EuclideanGPFitter instance: hp_tune_criterion 'ml' with
      ml_hp_tune_opt rand / rand_exp_sampling / pdoo / direct-without-Fortran runs fit_gp above (every batch of
      _tuning_objective evaluations as one lml_for_hyperparams call; same global-RNG consumption, same selection,
      the final GP built by the fitter's own build_gp); 'post_sampling' with the slice sampler on a layout that
      post_sampling_covers runs post_sampling.post_sample_hps; everything else is handed to `reference_fit_gp`. """
  from argparse import Namespace
  from .gpb_acquisitions import _reference_fortran_direct_available
  crit = fitter.options.hp_tune_criterion if hp_tune_criterion is None else hp_tune_criterion
  method = getattr(fitter, 'ml_hp_tune_opt_method', None)
  if crit == 'post_sampling':
    layout = layout_from_fitter(fitter)
    if getattr(fitter.options, 'post_hp_tune_method', None) != 'slice' or not post_sampling_covers(layout):
      return reference_fit_gp(fitter, num_samples, hp_tune_criterion)
    from .post_sampling import post_sample_hps
    X_mat, Y_vec = _fitter_data(fitter, layout)
    return post_sample_hps(X_mat, Y_vec, layout, fitter.cts_hp_bounds, fitter.dscr_hp_vals, num_samples=num_samples,
                           offset=fitter.options.post_hp_tune_offset, burn=fitter.options.post_hp_tune_burn,
                           build_gp=lambda cts, dscr: fitter.build_gp(cts, dscr, other_gp_params=None))
  layout = layout_from_fitter(fitter) if crit == 'ml' else None
  if (layout is None or method not in ('rand', 'rand_exp_sampling', 'pdoo', 'direct') or
      (method == 'direct' and _reference_fortran_direct_available())):
    return reference_fit_gp(fitter, num_samples, hp_tune_criterion)
  other = lambda grp: None if grp is None else Namespace(add_gp_groupings=grp)
  X_mat, Y_vec = _fitter_data(fitter, layout)
  return fit_gp(X_mat, Y_vec, layout, fitter.cts_hp_bounds, fitter.dscr_hp_vals,
                method=method, max_evals=fitter.hp_tune_max_evals,
                build_gp=lambda cts, dscr, grp: fitter.build_gp(cts, dscr, other_gp_params=other(grp)))


def bind_fit_gp(fitter_class):
  """ Re-binds fit_gp on a reference GPFitter class (dragonfly.gp.gp_core.GPFitter); returns the original. """
  original = fitter_class.fit_gp

  def fit_gp_b200(self, num_samples=1, hp_tune_criterion=None):
    return fit_gp_on_fitter(self, original, num_samples, hp_tune_criterion)
  fitter_class.fit_gp = fit_gp_b200
  return original


def rand_exp_sampling_probs(lml_vals):
  """ gp_core.py:443-444 """
  lml_vals = np.asarray(lml_vals, dtype=np.float64)
  probs = np.exp(lml_vals - max(lml_vals))
  return probs / probs.sum()


def sharded_lml_grid(X, Y, hps, layout, nus=None, device=None, group=None):
  """ Rank r evaluates hps[lo:hi]; one all-gather of the fp64 LML values.  Every rank returns the
      full vector and the rand_exp_sampling probabilities. """
  import torch
  import torch.distributed as dist
  from .dist import shard_bounds
  hps = np.asarray(hps, dtype=np.float64)
  H = len(hps)
  if not (dist.is_available() and dist.is_initialized()):
    lmls, _ = lml_for_hyperparams(X, Y, hps, layout, nus, device=device)
    return lmls, rand_exp_sampling_probs(lmls)
  rank, world = dist.get_rank(group), dist.get_world_size(group)
  lo, hi = shard_bounds(H, rank, world)
  mine, _ = lml_for_hyperparams(X, Y, hps[lo:hi], layout, None if nus is None else nus[lo:hi],
                                device=device) if hi > lo else (np.empty(0), None)
  return gather_shards(mine, H, group=group, device=device)


def gather_shards(mine, total, group=None, device=None):
  """ All-gather of variable-length fp64 shards (padded to the largest shard). """
  import torch
  import torch.distributed as dist
  from .dist import shard_bounds
  world = dist.get_world_size(group)
  backend = dist.get_backend(group)
  dev = torch.device('cpu') if backend == 'gloo' else (
      torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device('cuda', device))
  cap = max(shard_bounds(total, r, world)[1] - shard_bounds(total, r, world)[0] for r in range(world))
  buf = torch.zeros(max(cap, 1), dtype=torch.float64, device=dev)
  buf[:len(mine)] = torch.from_numpy(np.asarray(mine, dtype=np.float64)).to(dev)
  out = [torch.empty_like(buf) for _ in range(world)]
  dist.all_gather(out, buf, group=group)
  parts = []
  for r in range(world):
    lo, hi = shard_bounds(total, r, world)
    parts.append(out[r][:hi - lo].cpu().numpy())
  lmls = np.concatenate(parts) if parts else np.empty(0)
  return lmls, rand_exp_sampling_probs(lmls)
