"""
Drop-in for dragonfly.gp.gp_core.GP (gp_core.py:86-304) whose numeric bodies run on an H100 through
libdfb200: same constructor, methods, option meaning, public attributes (X, Y lists, num_tr_data,
kernel, noise_var, mean_func, L, alpha, K_trtr_wo_noise) and error behaviour.

What stays on the host, as in the reference: the Python `mean_func` callable (evaluated on the
training inputs for centring; constant means -- what GPFitter.build_gp always produces,
gp_core.py:527-530 -- are folded into the device call, anything else is added on the host), and the
jitter ladder of stable_cholesky (general_utils.py:166-204), which re-submits the factorisation with
10^p * max(diag) added until the device reports success.
"""
import sys
from contextlib import contextmanager
from warnings import warn

import numpy as np

from . import _lib
from .kernel import build_descriptor


def _check_feature_label_lengths_and_format(X, Y):
  """ gp_core.py:71-75.  (The reference concatenates str + int here, so a length mismatch
      surfaces as TypeError there; we raise the ValueError it meant to.) """
  if len(X) != len(Y):
    raise ValueError('Length of X (%d) and Y (%d) do not match.' % (len(X), len(Y)))


def _as_2d(X):
  arr = np.asarray(X, dtype=np.float64)
  if arr.ndim == 1:
    arr = arr.reshape(1, -1)
  return np.ascontiguousarray(arr)


def _constant_mean_value(mean_func, X_train):
  """ (c, trusted).  A mean function that ADVERTISES its constant (`const_value`: ConstantMean below, what the
      fitter path builds) is folded into the device call as is: trusted.  Any other callable -- e.g. the plain
      lambda of the reference's GPFitter.build_gp (gp_core.py:527-530) -- is a candidate constant only if it is
      constant on the actual training inputs, and is then RE-CHECKED on the actual candidates of every call
      (GP._mean_const_for) before the constant is used; it is never inferred from probe points. """
  if hasattr(mean_func, 'const_value'):
    return float(mean_func.const_value), True
  try:
    vals = np.asarray(mean_func(X_train), dtype=np.float64).reshape(-1)
  except Exception:  # pylint: disable=broad-except
    return None, False
  if vals.shape[0] == len(X_train) and vals.shape[0] > 0 and np.all(vals == vals[0]):
    return float(vals[0]), False
  return None, False


def _owners_of(post):
  """ The WeakSet of GP objects that use a device posterior (created on first use). """
  import weakref
  owners = getattr(post, '_owners', None)
  if owners is None:
    owners = weakref.WeakSet()
    post._owners = owners
  return owners


# Scoring chunk (candidate rows per device pass) of new posteriors; 0 = the library default (~256 MB of K_* rows).
DEFAULT_CHUNK = [0]


class ConstantMean(object):
  """ lambda x: np.array([c] * len(x)) with the constant advertised (gp_core.py:527-530). """

  def __init__(self, value):
    self.const_value = float(value)

  def __call__(self, x):
    return np.array([self.const_value] * len(x))


def stable_cholesky_on_device(post, noise_var, add_to_diag_till_psd=True, flags=_lib.DFB_BUILD_FULL):
  """ general_utils.py:166-204 with np.linalg.cholesky replaced by the device factorisation:
      try jitter 0, then 10^p * max(diag M) for p = -11, -10, ...; ValueError once p reaches 5.
      Returns (lml, jitter_power or None). """
  info, lml = post.build(noise_var, 0.0, flags)
  if info == 0:
    return lml, None
  if not add_to_diag_till_psd:
    raise np.linalg.LinAlgError('Matrix is not positive definite (pivot %d).' % (info - 1))
  max_M = post.max_diag()
  diag_noise_power = -11
  printed_warning = False
  while True:
    diag_noise = (10 ** diag_noise_power) * max_M
    info, lml = post.build(noise_var, diag_noise, flags)
    if info == 0:
      return lml, diag_noise_power
    if diag_noise_power > -9 and not printed_warning:
      warn(('Could not compute Cholesky decomposition despite adding %0.4f to the diagonal. '
            'This is likely because the M is not positive semi-definite.') % (diag_noise))
      printed_warning = True
    diag_noise_power += 1
    if diag_noise_power >= 5:
      raise ValueError(('Could not compute Cholesky decomposition despite adding %0.4f to the '
                        'diagonal. This is likely because the M is not positive semi-definite or '
                        'has infinities/nans.') % (diag_noise))


# What INTEGRATION.md's recipe copies onto the reference's own dragonfly.gp.gp_core.GP (setattr by name): the
# public methods the device path replaces plus the private helpers they call.
# Kept by the reference class: its constructor / set-up, data bookkeeping and printing.
_REBIND_KEEPS_REFERENCE = ('__init__', '_set_up', '_write_message', 'set_data', 'add_data_single', '__str__',
                           '_child_str', '_get_training_kernel_matrix')


def _rebind_methods():
  """ Every plain method / class attribute of the device-backed GP except the ones the reference keeps: derived from
      the class itself so that the recipe cannot fall behind the implementation. """
  names = []
  for name, val in vars(GP).items():
    if name in _REBIND_KEEPS_REFERENCE or name in REBIND_PROPERTIES or isinstance(val, property):
      continue
    if callable(val) or name == 'incremental_updates':
      names.append(name)
  return names


REBIND_PROPERTIES = ['L', 'alpha', 'K_trtr_wo_noise']


class _FusedSession(object):
  """ See GP._fused_session. """

  def __init__(self, gp, post, acq, mean_const):
    self.gp, self.post, self.acq, self.mean_const = gp, post, acq, mean_const

  def _slab(self, pts):
    """ (candidate matrix, mean constant) of one slab; raises if the mean is not a constant on the candidates. """
    mc = self.gp._mean_const_for(pts) if self.mean_const is None else self.mean_const
    if mc is None:
      raise NotImplementedError('Fused acquisition scoring needs a mean function that is constant on the '
                                'candidates (what GPFitter.build_gp produces, gp_core.py:527-530).')
    return self.gp._test_matrix(pts), mc

  def score(self, pts, want_scores=False):
    """ dfb_score_argmax over one slab: (best_score, best_index within the slab, scores or None). """
    return self.post.score_argmax(self.acq, *self._slab(pts), want_scores=want_scores)

  def score_ts(self, pts, z=None, seed=0, row0=0, want_scores=False):
    """ dfb_score_argmax_ts over one slab: one marginal posterior draw per candidate (the session's acq is not used),
        with the normals z (same memory space as pts) or the device's counter-based normals of (seed, row0 + row).
        Returns (best_score, best_index within the slab, scores or None, count of variances that are not > 0). """
    return self.post.score_argmax_ts(*self._slab(pts), z=z, seed=seed, row0=row0, want_scores=want_scores)

  def slab_rows(self, target):
    """ Rows per streamed slab: a whole number of the handle's scoring chunks (no ragged chunk inside a slab). """
    chunk = int(self.post.query('chunk'))
    return max(1, int(target) // chunk) * chunk


class GP(object):
  """ Base class for Gaussian processes -- device-backed mirror of gp_core.py:86-304. """
  # pylint: disable=attribute-defined-outside-init

  def __init__(self, X, Y, kernel, mean_func, noise_var, build_posterior=True,
               reporter=None, handle_non_psd_kernels='guaranteed_psd', device=None):
    super(GP, self).__init__()
    _check_feature_label_lengths_and_format(X, Y)
    self._device = device
    self._post = None
    self._cache = {}
    self.set_data(X, Y, build_posterior=False)
    self.kernel = kernel
    self.mean_func = mean_func
    self.noise_var = noise_var
    self.reporter = reporter
    self.handle_non_psd_kernels = handle_non_psd_kernels
    self.num_tr_data = len(self.Y)
    self.jitter_power = None
    self._set_up()
    if build_posterior:
      self.build_posterior()

  def _set_up(self):
    """ gp_core.py:113-118 """
    if not self.kernel.is_guaranteed_psd():
      assert self.handle_non_psd_kernels in ['project_first', 'try_before_project']

  def _write_message(self, msg):
    if self.reporter is not None and hasattr(self.reporter, 'write'):
      self.reporter.write(msg)
    else:
      sys.stdout.write(msg)

  # -- data ---------------------------------------------------------------------------------------
  def set_data(self, X, Y, build_posterior=True):
    """ gp_core.py:127-133 """
    self.X = list(X)
    self.Y = list(Y)
    self.num_tr_data = len(self.Y)
    if build_posterior:
      self.build_posterior()

  def add_data_single(self, x_new, y_new, *args, **kwargs):
    self.add_data_multiple([x_new], [y_new], *args, **kwargs)

  # The reference re-factorises from scratch on every new observation (gp_core.py:139-146).  Here the
  # built posterior is extended in place (dfb_extend_posterior: only the last row block of L changes,
  # O(N^2) instead of O(N^3)) whenever that is exactly the same mathematical object; set to False to
  # force the reference's full rebuild.
  incremental_updates = True

  def add_data_multiple(self, X_new, Y_new, build_posterior=True):
    """ gp_core.py:139-146 """
    _check_feature_label_lengths_and_format(X_new, Y_new)
    X_new, Y_new = list(X_new), list(Y_new)
    self.X.extend(X_new)
    self.Y.extend(Y_new)
    self.num_tr_data = len(self.Y)
    if build_posterior:
      if not self._extend_posterior(len(Y_new)):
        self.build_posterior()

  def _posterior_token(self):
    """ What the built device posterior depends on besides the data: the kernel's hyper-parameters BY VALUE (the
        bytes of its device descriptor, so an in-place set_hyperparams / change_smoothness invalidates the
        posterior), the mean function, the noise and the PSD handling. """
    try:
      dim = self._post.dim if getattr(self, '_post', None) is not None else self._train_matrix().shape[1]
      kern_fp = bytes(build_descriptor(self.kernel, train_dim=dim, cand_dim=dim))
    except Exception:  # pylint: disable=broad-except
      kern_fp = id(self.kernel)
    return (kern_fp, id(self.mean_func), getattr(self.mean_func, 'const_value', None), float(self.noise_var),
            self.handle_non_psd_kernels)

  def _post_is_shared(self):
    """ True while another live GP object (a copy() / deepcopy() of this one) uses the same device posterior. """
    post = getattr(self, '_post', None)
    if post is None:
      return False
    owners = _owners_of(post)
    return len([o for o in owners if o is not self and getattr(o, '_post', None) is post]) > 0

  def _rows_as_train_matrix(self, rows):
    """ `rows` (a list in the format of self.X) as rows of the matrix the kernel sees. """
    saved_X = self.X
    try:
      self.X = list(rows)
      return self._train_matrix()
    finally:
      self.X = saved_X

  def _can_extend_in_place(self, q):
    post = getattr(self, '_post', None)
    return (self.incremental_updates and post is not None and q >= 1 and
            getattr(self, 'jitter_power', None) is None and
            getattr(self, '_post_token', None) == self._posterior_token() and
            post.n + q <= post.capacity())

  def _extend_posterior(self, q):
    """ The last q entries of self.X / self.Y are new: extend the device posterior in place.
        Returns False when a full build_posterior() is needed instead (posterior shared with a copy
        of this GP, a jitter ladder in play, kernel / noise / mean changed since the build, padded
        size exceeded, or the extended matrix not positive definite at jitter 0). """
    post = getattr(self, '_post', None)
    if (not self._can_extend_in_place(q) or self._post_is_shared() or
        post.n + q != self.num_tr_data):
      return False
    y_new = (np.asarray(self.Y[-q:], dtype=np.float64) -
             np.asarray(self.mean_func(self.X[-q:]), dtype=np.float64))
    info, lml = post.extend(self._rows_as_train_matrix(self.X[-q:]), y_new, _lib.DFB_BUILD_FULL)
    if info != 0:
      self._post = None        # the factorisation was overwritten: rebuild (with the jitter ladder)
      return False
    self._cache = {}
    self._y_centred = np.concatenate((self._y_centred, y_new))
    self._lml = lml
    return True

  # -- posterior ------------------------------------------------------------------------------------
  def _train_matrix(self):
    """ The training inputs as the (n, d) matrix the kernel sees.  Child classes with structured
        inputs (multi-fidelity [z || x] rows) override this. """
    return _as_2d(self.X)

  def _get_training_kernel_matrix(self):
    """ gp_core.py:149-153: K(X, X) without noise, evaluated on the device (Kernel.__call__ -> dfb_kernel_matrix).
        build_posterior does not need it -- the device forms K inside dfb_build_posterior -- but subclasses and
        callers of the reference may. """
    X_mat = self._train_matrix()
    return self.kernel(X_mat, X_mat)

  def _new_device_posterior(self, n_max):
    from .device import DevicePosterior
    return DevicePosterior(n_max, device=getattr(self, '_device', None), chunk=DEFAULT_CHUNK[0])

  def _build_on_device(self, X_mat, y_centred, flags):
    if self.handle_non_psd_kernels not in ('guaranteed_psd', 'try_before_project', 'project_first'):
      raise ValueError('Unknown option for handle_non_psd_kernels: %s' % (
          self.handle_non_psd_kernels))
    if self.handle_non_psd_kernels == 'project_first':
      raise NotImplementedError('project_first needs an eigen-decomposition; every kernel on the '
                                'GPU hot path is guaranteed PSD (no CPU fallback).')
    post = self._new_device_posterior(len(X_mat))
    post.set_kernel(build_descriptor(self.kernel, train_dim=X_mat.shape[1], cand_dim=X_mat.shape[1]))
    post.set_train(X_mat, y_centred)
    ladder = (self.handle_non_psd_kernels == 'guaranteed_psd')
    try:
      lml, power = stable_cholesky_on_device(post, self.noise_var, add_to_diag_till_psd=ladder,
                                             flags=flags)
    except np.linalg.LinAlgError:
      raise NotImplementedError('try_before_project fell through to project_first, which needs '
                                'an eigen-decomposition (out of the GPU hot-path scope).')
    return post, lml, power

  def build_posterior(self):
    """ gp_core.py:155-163: K, L = chol(K + noise I), alpha -- all on the device. """
    self._cache = {}
    if self.num_tr_data == 0:
      self._post = None
      self._cache = {'L': np.zeros((0, 0)), 'alpha': np.zeros((0,)), 'K': np.zeros((0, 0))}
      self._lml = -0.0
      return
    X_mat = self._train_matrix()
    y_centred = np.asarray(self.Y, dtype=np.float64) - np.asarray(self.mean_func(self.X))
    self._y_centred = y_centred
    self._post, self._lml, self.jitter_power = self._build_on_device(X_mat, y_centred,
                                                                     _lib.DFB_BUILD_FULL)
    _owners_of(self._post).add(self)
    self._post_token = self._posterior_token()
    self._mean_const, self._mean_trusted = _constant_mean_value(self.mean_func, self.X)

  def _state(self, name):
    if not hasattr(self, '_cache'):
      self._cache = {}
    if name not in self._cache:
      if getattr(self, '_post', None) is None:
        raise RuntimeError('Posterior has not been built.')
      L, a, K = self._post.get_state(want_L=(name == 'L'), want_alpha=(name == 'alpha'),
                                     want_K=(name == 'K'))
      t = {'L': L, 'alpha': a, 'K': K}[name]
      self._cache[name] = t.cpu().numpy()
    return self._cache[name]

  # gp.L / gp.alpha are read directly by _add_ucb (gpb_acquisitions.py:169-171) and
  # gp.K_trtr_wo_noise by gp_core.py:203: lazily copied back as NumPy arrays.
  @property
  def L(self):
    return None if (getattr(self, '_post', None) is None and
                    'L' not in getattr(self, '_cache', {})) else self._state('L')

  @L.setter
  def L(self, value):
    if value is not None:
      if not hasattr(self, '_cache'):
        self._cache = {}
      self._cache['L'] = value

  @property
  def alpha(self):
    return None if (getattr(self, '_post', None) is None and
                    'alpha' not in getattr(self, '_cache', {})) else self._state('alpha')

  @alpha.setter
  def alpha(self, value):
    if value is not None:
      if not hasattr(self, '_cache'):
        self._cache = {}
      self._cache['alpha'] = value

  @property
  def K_trtr_wo_noise(self):
    return None if (getattr(self, '_post', None) is None and
                    'K' not in getattr(self, '_cache', {})) else self._state('K')

  @K_trtr_wo_noise.setter
  def K_trtr_wo_noise(self, value):
    if value is not None:
      if not hasattr(self, '_cache'):
        self._cache = {}
      self._cache['K'] = value

  def compute_log_marginal_likelihood(self):
    """ gp_core.py:222-227 (evaluated on the device during build_posterior). """
    if self._post is None and self.num_tr_data > 0:
      raise RuntimeError('Posterior has not been built.')
    return self._lml

  def compute_grad_log_marginal_likelihood(self, param, *args):
    """ gp_core.py:229-240: 1/2 tr((alpha alpha^T - K^-1) dK/dparam) for param in 'noise_var', 'noise_mean' and the
        kernel's own 'scale', 'same_dim_bandwidths' and (any other name, param_num) = bandwidth of one dimension
        (kernel.py:202-217, 301-322).  One device call (dfb_lml_gradients) yields the gradients w.r.t. ALL of them
        -- K^-1 from one triangular product of L^-T with itself, dK/dparam re-derived entry by entry, never
        stored -- and is cached for the posterior, so looping over the parameters as the reference's samplers do
        (gp_core.py:571) costs one pass.  The reference indexes dim_bandwidths[0, j], which only works for kernels
        that were given a (d, 1) bandwidth column; the values here are those it returns in that case. """
    if self._post is None or self.num_tr_data == 0:
      raise RuntimeError('Posterior has not been built.')
    if param == 'noise_mean':
      return float(self._lml_gradient_vector()[2])
    if param == 'noise_var':
      return float(self.noise_var * self._lml_gradient_vector()[1])
    if param == 'scale':
      return float(self._lml_gradient_vector()[0])
    if param == 'same_dim_bandwidths':
      return float(self._lml_gradient_vector()[3])
    param_num = args[0] if len(args) > 0 else None
    if param_num is None or not 0 <= int(param_num) < self.kernel.dim:
      raise IndexError('param_num %s is not a dimension of the kernel.' % (param_num,))
    return float(self._lml_gradient_vector()[4 + int(param_num)])

  def _lml_gradient_vector(self):
    if getattr(self, '_cache', None) is None:
      self._cache = {}
    key = ('lml_grad', id(self._post), self._post.n)
    if self._cache.get('lml_grad_key') != key:
      self._cache['lml_grad'] = self._post.lml_gradients(self.kernel.dim)
      self._cache['lml_grad_key'] = key
    return self._cache['lml_grad']

  # -- prediction --------------------------------------------------------------------------------------
  def _test_matrix(self, X_test):
    import torch
    if isinstance(X_test, torch.Tensor):
      return X_test
    return _as_2d(X_test)

  def _mean_const_for(self, X_test):
    """ The constant to fold into the device call for these candidates, or None.  An advertised constant is used as
        is; an inferred one only after mean_func has been evaluated on the ACTUAL candidates (what the reference
        does anyway, gp_core.py:172) and found equal to it everywhere. """
    import torch
    c = getattr(self, '_mean_const', None)
    if c is None or getattr(self, '_mean_trusted', False):
      return c
    if isinstance(X_test, torch.Tensor):
      # a Python callable can only see host rows: the check costs one device->host copy of the candidates
      # (advertise the constant with ConstantMean to avoid it)
      X_test = X_test.detach().cpu().numpy()
    try:
      vals = np.asarray(self.mean_func(X_test), dtype=np.float64).reshape(-1)
    except Exception:  # pylint: disable=broad-except
      return None
    return c if (vals.shape[0] == len(X_test) and np.all(vals == c)) else None

  def _eval_on(self, post, X_test, want_std):
    import torch
    Xm = self._test_matrix(X_test)
    mc = self._mean_const_for(X_test)
    if mc is not None:
      return post.eval(Xm, mean_const=mc, want_std=want_std)
    mu, sd = post.eval(Xm, mean_const=0.0, want_std=want_std)
    if isinstance(Xm, torch.Tensor):
      # non-constant Python mean on device candidates: evaluated on a host copy of the rows (gp_core.py:172)
      mvals = np.asarray(self.mean_func(Xm.detach().cpu().numpy()), dtype=np.float64).reshape(-1)
      return torch.from_numpy(mvals).to(mu.device) + mu, sd
    return np.asarray(self.mean_func(X_test)) + mu, sd

  def eval(self, X_test, uncert_form='none'):
    """ gp_core.py:165-190.  'std' never forms the M x M covariance. """
    if uncert_form not in ('none', 'std', 'covar'):
      raise ValueError('uncert_form should be none, covar or std.')
    if len(X_test) == 0:
      return np.zeros((0,)), (None if uncert_form == 'none' else np.zeros((0,)))
    if self.num_tr_data == 0:
      raise NotImplementedError('eval with no training data is outside the device path.')
    if uncert_form == 'covar':
      return self._eval_covar_on(self._post, X_test)
    return self._eval_on(self._post, X_test, uncert_form == 'std')

  def _eval_covar_on(self, post, X_test):
    """ The full M x M posterior covariance (gp_core.py:179-185) -- one device block, so M is
        bounded (DevicePosterior.TS_BLOCK); 'std' is the path for large M. """
    Xm = self._test_matrix(X_test)
    if len(Xm) > post.TS_BLOCK:
      raise NotImplementedError('uncert_form="covar" materialises an M x M matrix; M = %d exceeds '
                                'the device block of %d.' % (len(Xm), post.TS_BLOCK))
    mc = self._mean_const_for(X_test)
    if mc is not None:
      return post.eval_covar(Xm, mean_const=mc)
    mu, cov = post.eval_covar(Xm, mean_const=0.0)
    return np.asarray(self.mean_func(X_test)) + mu, cov

  def _augmented_posterior(self, X_halluc):
    """ gp_core.py:200-206: the GP with the pending points appended, variance only.  alpha is the
        un-augmented alpha zero-extended, so mu = K_*aug alpha_aug == K_* alpha exactly. """
    X_aug = list(self.X) + list(X_halluc)
    saved_X = self.X
    try:
      self.X = X_aug
      X_mat = self._train_matrix()
    finally:
      self.X = saved_X
    y_aug = np.concatenate((self._y_centred, np.zeros(len(X_halluc))))
    post, _, _ = self._build_on_device(X_mat, y_aug, _lib.DFB_BUILD_NO_ALPHA)
    post.set_alpha(self.alpha)
    return post

  @contextmanager
  def _hallucinated(self, X_halluc):
    """ The device posterior with the pending points appended (variance from the augmented GP, mean
        from the un-augmented one: gp_core.py:200-217).  When the q points fit the padded size, the
        built posterior is extended in place (dfb_extend_posterior | DFB_EXTEND_SAVE, alpha
        zero-extended) and restored bit for bit on exit; otherwise -- or if the extended matrix needs
        the jitter ladder -- a fresh (N + q)-point posterior is built like the reference does. """
    q = len(X_halluc)
    post = getattr(self, '_post', None)
    if q == 0:
      yield post
      return
    if self._can_extend_in_place(q) and not getattr(post, '_ext_active', False):
      n0 = post.n
      info, _ = post.extend(self._rows_as_train_matrix(X_halluc), np.zeros(q), _lib.DFB_BUILD_NO_ALPHA,
                            save=True)
      if info == 0:
        post._ext_active = True
        try:
          yield post        # alpha was left untouched: its tail beyond n0 is zero
        finally:
          post.restore(n0)
          post._ext_active = False
        return
    yield self._augmented_posterior(X_halluc)

  def eval_with_hallucinated_observations(self, X_test, X_halluc, uncert_form='none'):
    """ gp_core.py:192-220 """
    if uncert_form not in ('none', 'std', 'covar'):
      raise ValueError('uncert_form should be none, covar or std.')
    if uncert_form == 'none' or len(X_halluc) == 0:
      return self.eval(X_test, uncert_form)
    with self._hallucinated(X_halluc) as post:
      if uncert_form == 'covar':
        return self._eval_covar_on(post, X_test)
      return self._eval_on(post, X_test, True)

  # -- fused acquisition scoring (the body of gpb_acquisitions' objectives + np.argmax) -----------
  def _device_posterior(self, halluc=None):
    if halluc is None or len(halluc) == 0:
      return self._post
    return self._augmented_posterior(halluc)

  @contextmanager
  def _fused_session(self, acq, halluc=None, test_desc=None, mean_const=None):
    """ One acquisition-maximisation session on the device posterior: the evaluations in progress are appended
        ONCE (in place when possible, gp_core.py:200-217) and the group's test kernel bound once, however many
        slabs of candidates are then scored through `session.score(pts)` (gpb_acquisitions._fused_maximise streams
        the candidates in slabs so that drawing them overlaps with scoring them). """
    with self._hallucinated([] if halluc is None else halluc) as post:
      if test_desc is not None:
        post.set_test_kernel(test_desc)
      try:
        yield _FusedSession(self, post, acq, mean_const)
      finally:
        if test_desc is not None:
          post.set_test_kernel(None)

  def _fused_score(self, acq, pts, halluc=None, test_desc=None, mean_const=None,
                   want_scores=False):
    """ One dfb_score_argmax call: returns (best_score, best_index, scores or None). """
    with self._fused_session(acq, halluc, test_desc, mean_const) as session:
      return session.score(pts, want_scores=want_scores)

  def _group_test_descriptor(self, add_kernel, kernel_j, group_j, train_dim):
    """ K_*j = scale * k_j(X*_j, X[:, g_j]) (gpb_acquisitions.py:166-170): candidates have d_j
        columns, the training matrix keeps all of its columns. """
    from .kernel import AdditiveKernel
    d_j = len(group_j)
    single = AdditiveKernel(add_kernel.hyperparams['scale'], [kernel_j], [list(range(d_j))])
    return build_descriptor(single, train_dim=train_dim, cand_dim=d_j,
                            train_coords=[int(g) for g in group_j], cand_coords=list(range(d_j)))

  # -- sampling (gp_core.py:250-261) --------------------------------------------------------------------
  def _draw_samples_on(self, post, num_samples, X_test, cols=None):
    """ draw_gaussian_samples (general_utils.py:224-232) per block of <= TS_BLOCK candidates:
        L = stable_cholesky(covar) with the same jitter ladder, U = np.random.normal(size=(M, S))
        drawn ONCE from the global RNG exactly like the reference, samples = (L U)^T + mu.
        DEVIATION from the reference for M > TS_BLOCK (min(4096, the handle's scoring chunk)): blocks are
        sampled INDEPENDENTLY of each other -- the reference's single joint draw needs the M x M covariance
        (8 TB at M = 10^6) -- so cross-block correlations are dropped and the sample matrix is not the one
        the reference's RNG stream would give (DESIGN.md 7).  Exact, and seed-identical, for M <= TS_BLOCK. """
    Xm = self._test_matrix(X_test)
    mean_c = self._mean_const_for(X_test)
    if mean_c is None:
      raise NotImplementedError('Thompson sampling on device needs a constant mean function.')
    M = len(Xm)
    U = np.random.normal(size=(M, int(num_samples)))
    out = np.empty((int(num_samples), M))
    if cols is not None:
      # multi-GPU sharding by whole blocks (gpb_acquisitions._draw_one_sample): foreign blocks stay -inf
      assert cols[0] % post.TS_BLOCK == 0
      out.fill(-np.inf)
    for lo in range(0, M, post.TS_BLOCK):
      hi = min(M, lo + post.TS_BLOCK)
      if cols is not None and not (cols[0] <= lo < cols[1]):
        continue
      xb = Xm[lo:hi]
      for s_lo in range(0, int(num_samples), 256):
        s_hi = min(int(num_samples), s_lo + 256)
        Ut = np.ascontiguousarray(U[lo:hi, s_lo:s_hi].T)
        info, smp, max_diag = post.ts_draws(xb, Ut, mean_const=mean_c, jitter=0.0)
        power = -11
        while info != 0:
          jitter = (10 ** power) * max_diag
          info, smp, _ = post.ts_draws(xb, Ut, mean_const=mean_c, jitter=jitter)
          if info != 0:
            power += 1
            if power >= 5:
              raise ValueError('Could not compute Cholesky decomposition despite adding %0.4f to '
                               'the diagonal.' % (jitter))
        out[s_lo:s_hi, lo:hi] = smp.cpu().numpy()
    return out

  def draw_samples_argmax(self, num_samples, X_test, seed=0, X_halluc=None, return_values=True):
    """ Thompson sampling at scale (BASELINE config 5: 256 draws x 10^6 candidates): the arg-max of each of
        `num_samples` joint posterior draws over X_test -- what asy_ts does with each draw
        (gpb_acquisitions.py:119-127) -- without ever moving normals or samples through the host.  Same
        algorithm as draw_samples (gp_core.py:250-254, general_utils.py:224-232; exact within 4096-candidate
        blocks, DESIGN.md 7), but the standard normals come from the device's counter-based generator
        (dfb_fill_rng: a candidate's normals depend only on (seed, its global row, draw index)) instead of
        np.random.normal, and a running per-draw arg-max (dfb_ts_argmax) replaces the (S, M) sample matrix.
        Under torch.distributed the blocks are shared out over the ranks and joined with one all-gather of S
        16-byte pairs.  Returns (values (S,), indices (S,)) as NumPy arrays. """
    import torch
    from . import dist as dfb_dist
    from .gpb_acquisitions import _shard_info
    mean_c = self._mean_const_for(X_test)
    if mean_c is None:
      raise NotImplementedError('Thompson sampling on device needs a constant mean function (advertised through '
                                '`const_value` for device-tensor candidates).')
    S = int(num_samples)
    with self._hallucinated([] if X_halluc is None else X_halluc) as post:
      Xm = self._test_matrix(X_test)
      M = len(Xm)
      blk = post.TS_BLOCK
      n_blocks = (M + blk - 1) // blk
      rank, world, coll_dev = _shard_info()
      b_lo, b_hi = dfb_dist.shard_bounds(n_blocks, rank, world) if world > 1 else (0, n_blocks)
      best = torch.zeros((S,), dtype=torch.float64, device=post.device)
      index = torch.full((S,), -1, dtype=torch.int64, device=post.device)
      first = True
      for b in range(b_lo, b_hi):
        lo, hi = b * blk, min(M, (b + 1) * blk)
        xb = Xm[lo:hi]
        for s_lo in range(0, S, 256):
          s_hi = min(S, s_lo + 256)
          Ut = post.fill_rng(seed, lo, S, hi - lo)[s_lo:s_hi] if S > 256 else post.fill_rng(seed, lo, S, hi - lo)
          info, smp, max_diag = post.ts_draws(xb, Ut, mean_const=mean_c, jitter=0.0)
          power = -11
          while info != 0:                                    # stable_cholesky's ladder, per block
            jitter = (10 ** power) * max_diag
            info, smp, _ = post.ts_draws(xb, Ut, mean_const=mean_c, jitter=jitter)
            if info != 0:
              power += 1
              if power >= 5:
                raise ValueError('Could not compute Cholesky decomposition despite adding %0.4f to '
                                 'the diagonal.' % (jitter))
          post.ts_argmax(smp, lo, best[s_lo:s_hi], index[s_lo:s_hi], reset=first)
        first = False
      vals, idxs = best.cpu().numpy(), index.cpu().numpy()
    if world > 1:
      vals, idxs = dfb_dist.all_reduce_argmax_many(vals, idxs, device=coll_dev)
    return (vals, idxs) if return_values else idxs

  def draw_samples(self, num_samples, X_test=None, mean_vals=None, covar=None, cols=None):
    """ gp_core.py:250-254 (`cols`: multi-GPU block range, see _draw_samples_on) """
    if X_test is None:
      raise NotImplementedError('draw_samples from a caller-supplied (mean, covar) is host-side '
                                'NumPy in the reference and outside the device path.')
    return self._draw_samples_on(self._post, num_samples, X_test, cols=cols)

  def draw_samples_with_hallucinated_observations(self, num_samples, X_test, X_halluc, cols=None):
    """ gp_core.py:256-261 """
    if len(X_halluc) == 0:
      return self.draw_samples(num_samples, X_test, cols=cols)
    with self._hallucinated(X_halluc) as post:
      return self._draw_samples_on(post, num_samples, X_test, cols=cols)

  def __str__(self):
    return '%s, noise-var=%0.3f (n=%d)' % (self._child_str(), self.noise_var, len(self.Y))

  def _child_str(self):
    return 'H100-GP %s' % (str(self.kernel))

  # Copies share the device posterior; while another live copy uses it a posterior is never extended for good
  # (add_data on either copy rebuilds into a fresh one), only temporarily for hallucinations (restored on exit).
  # Sharing is tracked with a WeakSet of owners on the DevicePosterior, so it ends with the copy's lifetime (the
  # syn_* wrappers copy the GP on every call, gpb_acquisitions.py:104).
  def __copy__(self):
    cls = self.__class__
    new = cls.__new__(cls)
    new.__dict__.update(self.__dict__)
    if getattr(self, '_post', None) is not None:
      _owners_of(self._post).add(new)    # weak: the share ends when the copy is garbage-collected
    return new

  def __deepcopy__(self, memo):
    import copy as _copy
    cls = self.__class__
    new = cls.__new__(cls)
    memo[id(self)] = new
    for k, v in self.__dict__.items():
      if k == '_post':
        new.__dict__[k] = v
      elif k == '_post_token':
        new.__dict__[k] = None     # ids of the deep-copied kernel / mean differ: first add_data rebuilds
      else:
        new.__dict__[k] = _copy.deepcopy(v, memo)
    if getattr(self, '_post', None) is not None:
      _owners_of(self._post).add(new)
    return new


REBIND_METHODS = _rebind_methods()
