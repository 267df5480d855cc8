"""
CPU oracle (NumPy/SciPy restatement) of Dragonfly's GP-BO inner loop.  TEST INFRASTRUCTURE ONLY --
see oracle/__init__.py for who may import this.  All arithmetic is IEEE fp64, evaluated in the same
operation order as the reference so that differences to the reference are BLAS-summation-order only.

Reference paths are relative to the reference source tree (dragonfly-opt 0.1.7).
"""
import math
import numpy as np
from scipy.linalg import solve_triangular
from scipy.special import ndtr


# ---------------------------------------------------------------------------------------------
# L0: linear-algebra utilities                                   dragonfly/utils/general_utils.py
# ---------------------------------------------------------------------------------------------
def dist_squared(X1, X2):
  """ ||x1_i||^2 + ||x2_j||^2 - 2 x1_i.x2_j, clipped at 0.   general_utils.py:58-70 """
  X1 = np.asarray(X1, dtype=np.float64)
  X2 = np.asarray(X2, dtype=np.float64)
  if X1.shape[1] != X2.shape[1]:
    raise ValueError('Second dimension of X1 and X2 should be equal.')
  sq1 = (X1 ** 2).sum(axis=1)
  sq2 = (X2 ** 2).sum(axis=1)
  ret = (sq2[None, :] + sq1[:, None]) - 2 * X1.dot(X2.T)
  return np.clip(ret, 0.0, np.inf)


def stable_cholesky(M, add_to_diag_till_psd=True):
  """ Lower Cholesky factor with the reference's jitter ladder.   general_utils.py:166-204
      On failure retries with M + 10^p * max(diag M) * I for p = -11, -10, ...; raises ValueError
      once p reaches 5.  Returns (L, jitter_power_used or None). """
  if M.size == 0:
    return M, None
  try:
    return np.linalg.cholesky(M), None
  except np.linalg.LinAlgError:
    if not add_to_diag_till_psd:
      raise
  max_diag = np.diag(M).max()
  power = -11
  while True:
    jitter = (10 ** power) * max_diag
    try:
      return np.linalg.cholesky(M + jitter * np.eye(M.shape[0])), power
    except np.linalg.LinAlgError:
      power += 1
    if power >= 5:
      raise ValueError('Could not compute Cholesky decomposition despite adding %0.4f to the '
                       'diagonal.' % (jitter))


def solve_lower_triangular(A, b):
  """ general_utils.py:208-217 (SciPy dtrtrs; empty-input special case). """
  if A.size == 0 and b.shape[0] == 0:
    return np.zeros(b.shape)
  return solve_triangular(A, b, lower=True)


def solve_upper_triangular(A, b):
  """ general_utils.py:208-221 """
  if A.size == 0 and b.shape[0] == 0:
    return np.zeros(b.shape)
  return solve_triangular(A, b, lower=False)


def project_symmetric_to_psd_cone(M, epsilon=0):
  """ general_utils.py:150-163 (symmetric branch). """
  eigvals, eigvecs = np.linalg.eigh(M)
  return (eigvecs * np.clip(eigvals, epsilon, np.inf)).dot(eigvecs.T)


def draw_gaussian_samples_with_normals(mu, K, U):
  """ general_utils.py:224-232 with the N(0,1) matrix U (num_pts x num_samples) supplied by the
      caller instead of np.random.normal, so a device implementation can be fed the same draws. """
  L, _ = stable_cholesky(K)
  return L.dot(U).T + mu


def map_to_bounds(pts, bounds):
  """ general_utils.py:25-27 """
  bounds = np.asarray(bounds, dtype=np.float64)
  return pts * (bounds[:, 1] - bounds[:, 0]) + bounds[:, 0]


# ---------------------------------------------------------------------------------------------
# L1: kernels                                                          dragonfly/gp/kernel.py
# ---------------------------------------------------------------------------------------------
class OKernel(object):
  """ Kernel protocol: kernel.py:59-83 (zeros((n1,n2)) when either side is empty). """
  dim = None

  def __call__(self, X1, X2=None):
    X2 = X1 if X2 is None else X2
    if len(X1) == 0 or len(X2) == 0:
      return np.zeros((len(X1), len(X2)))
    return self._evaluate(np.asarray(X1, dtype=np.float64), np.asarray(X2, dtype=np.float64))

  def is_guaranteed_psd(self):
    return True


class OSEKernel(OKernel):
  """ scale * exp(-D2(X1/bw, X2/bw)/2).   kernel.py:130-181 """

  def __init__(self, dim, scale, dim_bandwidths):
    self.dim = dim
    bws = dim_bandwidths if hasattr(dim_bandwidths, '__len__') else [dim_bandwidths] * dim
    if len(bws) != dim:
      raise ValueError('Dimension of dim_bandwidths should be the same as dimension.')
    self.hyperparams = {'scale': scale, 'dim_bandwidths': np.array(bws, dtype=np.float64)}

  def _evaluate(self, X1, X2):
    bw = self.hyperparams['dim_bandwidths']
    d2 = dist_squared(X1 / bw, X2 / bw)
    return self.hyperparams['scale'] * np.exp(-d2 / 2)

  def gradient(self, param, X1, X2=None, param_num=None):
    """ dK/d(param), kernel.py:116-121, 202-217.  The reference indexes the bandwidth vector as
        hyperparams['dim_bandwidths'][0, j], which only works when the kernel was given its bandwidths as a
        (d, 1) column (set_dim_bandwidths transposes it to (1, d)); that is the configuration the goldens of
        tests/golden/make_golden_grad.py pin.  Here bw[j] is the same number. """
    X2 = X1 if X2 is None else X2
    if len(X1) == 0 or len(X2) == 0:
      return np.zeros((len(X1), len(X2)))
    X1 = np.asarray(X1, dtype=np.float64); X2 = np.asarray(X2, dtype=np.float64)
    bw = self.hyperparams['dim_bandwidths']
    s1, s2 = X1 / bw, X2 / bw
    d2 = dist_squared(s1, s2)
    if param == 'scale':
      return self.hyperparams['scale'] * np.exp(-d2 / 2)
    if param == 'same_dim_bandwidths':
      return self.hyperparams['scale'] * np.multiply(d2 / bw[0], np.exp(-d2 / 2))
    dim_sq = dist_squared(s1[:, [param_num]], s2[:, [param_num]]) / bw[param_num]
    return self.hyperparams['scale'] * np.multiply(dim_sq, np.exp(-d2 / 2))


def matern_constants(nu):
  """ The scalar constants of the half-integer Matern kernel exactly as the reference forms them
      (kernel.py:242-253, 259-270): p, sqrt(8 nu), sqrt(2 nu), coeff_i, Gamma(p+1)/Gamma(2p+1),
      norm_constant = 1 / (unnormalised value at 0). """
  if nu % 1 != 0.5:
    raise ValueError('Matern kernel: nu has to be p + 0.5 where p is an integer.')
  p = int(nu)
  coeffs = [math.factorial(p + i) / (math.factorial(i) * math.factorial(p - i))
            for i in range(p + 1)]
  gamma_ratio = math.gamma(p + 1) / math.gamma(2 * p + 1)
  s8 = np.sqrt(8 * nu)
  s2 = np.sqrt(2 * nu)
  # unnormalised value at dist = 0, same accumulation order as kernel.py:262-269
  u0 = 0
  for i in range(p + 1):
    u0 += coeffs[i] * (s8 * 0) ** (p - i)
  u0 *= (gamma_ratio * np.exp(-s2 * 0))
  return dict(p=p, s8=float(s8), s2=float(s2), coeffs=[float(c) for c in coeffs],
              gamma_ratio=float(gamma_ratio), norm_constant=float(1.0 / u0))


class OMaternKernel(OKernel):
  """ Half-integer Matern.   kernel.py:224-299 """

  def __init__(self, dim, nu, scale, dim_bandwidths):
    self.dim = dim
    bws = dim_bandwidths if hasattr(dim_bandwidths, '__len__') else [dim_bandwidths] * dim
    self.hyperparams = {'nu': nu, 'scale': scale,
                        'dim_bandwidths': np.array(bws, dtype=np.float64)}
    self.consts = matern_constants(nu)
    self.p = self.consts['p']
    self.norm_constant = self.consts['norm_constant']

  def _unnormalised(self, dist):
    c = self.consts
    out = np.zeros(dist.shape)
    for i in range(self.p + 1):
      out += c['coeffs'][i] * (c['s8'] * dist) ** (self.p - i)
    out *= (c['gamma_ratio'] * np.exp(-c['s2'] * dist))
    return out

  def _evaluate(self, X1, X2):
    bw = self.hyperparams['dim_bandwidths']
    dist = np.sqrt(dist_squared(X1 / bw, X2 / bw))
    return self.hyperparams['scale'] * self.norm_constant * self._unnormalised(dist)

  def _grad_unnormalised(self, dist, dist_dv):
    """ kernel.py:272-290 """
    c = self.consts
    u = np.zeros(dist.shape)
    u_dv = np.zeros(dist_dv.shape)
    for i in range(self.p + 1):
      mult = c['s8'] * dist
      u += c['coeffs'][i] * mult ** (self.p - i)
      if self.p - i > 0:
        u_dv += c['s8'] * (self.p - i) * c['coeffs'][i] * (mult ** (self.p - i - 1)) * dist_dv
    u_dv *= (c['gamma_ratio'] * np.exp(-c['s2'] * dist))
    u *= (c['gamma_ratio'] * np.exp(-c['s2'] * dist) * (-c['s2'] * dist_dv))
    return u + u_dv

  def gradient(self, param, X1, X2=None, param_num=None):
    """ dK/d(param), kernel.py:116-121, 301-322 (see OSEKernel.gradient for the bandwidth indexing). """
    X2 = X1 if X2 is None else X2
    if len(X1) == 0 or len(X2) == 0:
      return np.zeros((len(X1), len(X2)))
    X1 = np.asarray(X1, dtype=np.float64); X2 = np.asarray(X2, dtype=np.float64)
    bw = self.hyperparams['dim_bandwidths']
    s1, s2 = X1 / bw, X2 / bw
    dist = np.sqrt(dist_squared(s1, s2))
    sc = self.hyperparams['scale'] * self.norm_constant
    if param == 'scale':
      return sc * self._unnormalised(dist)
    if param == 'same_dim_bandwidths':
      return sc * self._grad_unnormalised(dist, -(dist / bw[0]))
    np.fill_diagonal(dist, 1.0)
    dist_dv = 1 / dist
    np.fill_diagonal(dist, 0.0)
    dim_sq = dist_squared(s1[:, [param_num]], s2[:, [param_num]])
    dist_dv *= -(dim_sq / bw[param_num])
    return sc * self._grad_unnormalised(dist, dist_dv)


class OAdditiveKernel(OKernel):
  """ scale * sum_g k_g(X1[:, g], X2[:, g]).   kernel.py:461-494 """

  def __init__(self, scale, kernel_list, groupings):
    if len(kernel_list) != len(groupings):
      raise ValueError('number of kernels do not correspond to number of groups.')
    self.kernel_list = kernel_list
    self.groupings = groupings
    self.hyperparams = {'scale': scale}
    self.dim = sum(k.dim for k in kernel_list)

  def _evaluate(self, X1, X2):
    out = np.zeros((X1.shape[0], X2.shape[0]))
    for kern, grp in zip(self.kernel_list, self.groupings):
      out += kern(X1[:, grp], X2[:, grp])
    return self.hyperparams['scale'] * out


class OCoordinateProductKernel(OKernel):
  """ scale * prod_i k_i(X1[:, c_i], X2[:, c_i]).   kernel.py:541-584
      The multi-fidelity kernel is k_F on fidelity coords x k_D on domain coords
      (euclidean_gp.py:369-374). """

  def __init__(self, dim, scale, kernel_list, coordinate_list):
    self.dim = dim
    self.hyperparams = {'scale': scale}
    self.kernel_list = kernel_list
    self.coordinate_list = coordinate_list

  def _evaluate(self, X1, X2):
    out = self.hyperparams['scale'] * np.ones((X1.shape[0], X2.shape[0]))
    for kern, crd in zip(self.kernel_list, self.coordinate_list):
      out *= kern(X1[:, crd], X2[:, crd])
    return out


# ---------------------------------------------------------------------------------------------
# L1: GP posterior                                                    dragonfly/gp/gp_core.py
# ---------------------------------------------------------------------------------------------
def get_cholesky_decomp(K_wo_noise, noise_var, handle_non_psd_kernels='guaranteed_psd'):
  """ gp_core.py:827-847.  Returns (L, jitter_power). """
  n = K_wo_noise.shape[0]
  if handle_non_psd_kernels == 'try_before_project':
    try:
      return stable_cholesky(K_wo_noise + noise_var * np.eye(n), add_to_diag_till_psd=False)
    except np.linalg.LinAlgError:
      return get_cholesky_decomp(K_wo_noise, noise_var, 'project_first')
  elif handle_non_psd_kernels == 'project_first':
    return get_cholesky_decomp(project_symmetric_to_psd_cone(K_wo_noise), noise_var,
                               'guaranteed_psd')
  elif handle_non_psd_kernels == 'guaranteed_psd':
    return stable_cholesky(K_wo_noise + noise_var * np.eye(n))
  raise ValueError('Unknown option for handle_non_psd_kernels: %s' % (handle_non_psd_kernels))


class OGP(object):
  """ gp_core.py:86-261.  mean_func is a Python callable, as in the reference. """

  def __init__(self, X, Y, kernel, mean_func, noise_var, build_posterior=True,
               handle_non_psd_kernels='guaranteed_psd'):
    if len(X) != len(Y):
      raise ValueError('Length of X and Y do not match.')
    self.kernel = kernel
    self.mean_func = mean_func
    self.noise_var = noise_var
    self.handle_non_psd_kernels = handle_non_psd_kernels
    self.L = None
    self.alpha = None
    self.K_trtr_wo_noise = None
    self.jitter_power = None
    self.set_data(X, Y, build_posterior)

  def set_data(self, X, Y, build_posterior=True):        # gp_core.py:127-133
    self.X = list(X)
    self.Y = list(Y)
    self.num_tr_data = len(self.Y)
    if build_posterior:
      self.build_posterior()

  def add_data_multiple(self, X_new, Y_new, build_posterior=True):   # gp_core.py:139-146
    self.X.extend(X_new)
    self.Y.extend(Y_new)
    self.num_tr_data = len(self.Y)
    if build_posterior:
      self.build_posterior()

  def build_posterior(self):                              # gp_core.py:155-163
    K = self.kernel(self.X, self.X)
    self.K_trtr_wo_noise = K
    self.L, self.jitter_power = get_cholesky_decomp(K, self.noise_var,
                                                    self.handle_non_psd_kernels)
    Yc = np.asarray(self.Y) - self.mean_func(self.X)
    self.alpha = solve_upper_triangular(self.L.T, solve_lower_triangular(self.L, Yc))

  def compute_log_marginal_likelihood(self):              # gp_core.py:222-227
    Yc = np.asarray(self.Y) - self.mean_func(self.X)
    return (-0.5 * Yc.T.dot(self.alpha) - np.log(np.diag(self.L)).sum()
            - 0.5 * self.num_tr_data * np.log(2 * np.pi))

  def compute_grad_log_marginal_likelihood(self, param, *args):    # gp_core.py:229-240
    alpha = np.expand_dims(self.alpha, axis=0)
    if param == 'noise_var':
      grad_m = self.noise_var * np.identity(len(self.X))
    elif param == 'noise_mean':
      return np.matmul(alpha, np.ones((len(self.Y), 1))).item()
    else:
      grad_m = self.kernel.gradient(param, self.X, self.X, *args)
    grad_m = np.matmul(alpha.T, np.matmul(alpha, grad_m)) - \
             solve_upper_triangular(self.L.T, solve_lower_triangular(self.L, grad_m))
    return 0.5 * np.trace(grad_m)

  def eval(self, X_test, uncert_form='none'):             # gp_core.py:165-190
    """ NOTE: like the reference this materialises K(X_test, X_test) and V^T V in full. """
    K_tetr = self.kernel(X_test, self.X)
    mu = self.mean_func(X_test) + K_tetr.dot(self.alpha)
    if uncert_form == 'none':
      return mu, None
    K_tete = self.kernel(X_test, X_test)
    V = solve_lower_triangular(self.L, K_tetr.T)
    covar = K_tete - V.T.dot(V)
    if not self.kernel.is_guaranteed_psd():               # gp_core.py:849-857
      covar = project_symmetric_to_psd_cone(covar, epsilon=0.05 * self.noise_var)
    if uncert_form == 'covar':
      return mu, covar
    elif uncert_form == 'std':
      return mu, np.sqrt(np.diag(covar))
    raise ValueError('uncert_form should be none, covar or std.')

  def eval_with_hallucinated_observations(self, X_test, X_halluc, uncert_form='none'):
    """ gp_core.py:192-220: mean from the plain GP, uncertainty from the GP augmented with the
        pending points (fresh (N+q) Cholesky). """
    mu, _ = self.eval(X_test, 'none')
    if uncert_form == 'none':
      return mu, None
    X_aug = list(self.X) + list(X_halluc)
    K_haha = self.kernel(X_halluc, X_halluc)
    K_trha = self.kernel(self.X, X_halluc)
    K_aug = np.vstack((np.hstack((self.K_trtr_wo_noise, K_trha)),
                       np.hstack((K_trha.T, K_haha))))
    L_aug, _ = get_cholesky_decomp(K_aug, self.noise_var, self.handle_non_psd_kernels)
    K_tete = self.kernel(X_test, X_test)
    K_tetr = self.kernel(X_test, X_aug)
    V = solve_lower_triangular(L_aug, K_tetr.T)
    covar = K_tete - V.T.dot(V)
    if uncert_form == 'covar':
      return mu, covar
    elif uncert_form == 'std':
      return mu, np.sqrt(np.diag(covar))
    raise ValueError('uncert_form should be none, covar or std.')

  def draw_samples_with_normals(self, X_test, U, X_halluc=None):
    """ gp_core.py:250-261 with the normal matrix U (M x S) supplied. Returns (S, M). """
    if X_halluc is None or len(X_halluc) == 0:
      mu, covar = self.eval(X_test, 'covar')
    else:
      mu, covar = self.eval_with_hallucinated_observations(X_test, X_halluc, 'covar')
    return draw_gaussian_samples_with_normals(mu, covar, U)


# Diagonal-only evaluation: mathematically what 'std' returns, without the M x M temporaries.
# Used by the tests at sizes where the faithful eval() above cannot allocate K(X*, X*).
def eval_std_diag(gp, X_test, X_halluc=None):
  X_test = np.asarray(X_test, dtype=np.float64)
  K_tetr = gp.kernel(X_test, gp.X)
  mu = gp.mean_func(X_test) + K_tetr.dot(gp.alpha)
  if X_halluc is not None and len(X_halluc) > 0:
    X_aug = list(gp.X) + list(X_halluc)
    K_haha = gp.kernel(X_halluc, X_halluc)
    K_trha = gp.kernel(gp.X, X_halluc)
    K_aug = np.vstack((np.hstack((gp.K_trtr_wo_noise, K_trha)), np.hstack((K_trha.T, K_haha))))
    L, _ = get_cholesky_decomp(K_aug, gp.noise_var, gp.handle_non_psd_kernels)
    K_tetr = gp.kernel(X_test, X_aug)
  else:
    L = gp.L
  V = solve_lower_triangular(L, K_tetr.T)
  kss = kernel_diag(gp.kernel, X_test)
  var = kss - (V * V).sum(axis=0)
  return mu, var


def kernel_diag(kern, X, block=256):
  """ diag K(X, X) through the same kernel code path, block by block. """
  X = np.asarray(X, dtype=np.float64)
  out = np.empty(len(X))
  for s in range(0, len(X), block):
    out[s:s + block] = np.diag(kern(X[s:s + block], X[s:s + block]))
  return out


# ---------------------------------------------------------------------------------------------
# L2: acquisitions + the `rand` maximiser                  dragonfly/opt/gpb_acquisitions.py
# ---------------------------------------------------------------------------------------------
def ucb_beta_th(dim, t):
  """ gpb_acquisitions.py:211-213 """
  return np.sqrt(0.5 * dim * np.log(2 * dim * t + 1))


def add_ucb_beta_th(dim, t):
  """ gpb_acquisitions.py:135-137 """
  return np.sqrt(0.2 * dim * np.log(2 * dim * t + 1))


def norm_cdf(z):
  """ scipy.stats.norm.cdf == scipy.special.ndtr (gpb_acquisitions.py:238,249). """
  return ndtr(z)


def norm_pdf(z):
  """ scipy.stats.norm.pdf: exp(-z^2/2)/sqrt(2 pi). """
  return np.exp(-z ** 2 / 2.0) / np.sqrt(2 * np.pi)


def acq_ucb(mu, sigma, beta_th):
  """ gpb_acquisitions.py:219-222 """
  return mu + beta_th * sigma


def acq_pi(mu, sigma, curr_best):
  """ gpb_acquisitions.py:235-238 """
  return norm_cdf((mu - curr_best) / sigma)


def acq_ei(mu, sigma, curr_best):
  """ gpb_acquisitions.py:247-260 """
  z = (mu - curr_best) / sigma
  return sigma * (z * norm_cdf(z) + norm_pdf(z))


def acq_ttei(mu, sigma, ref_mean, ref_std):
  """ gpb_acquisitions.py:274-279 """
  comb = np.sqrt(ref_std ** 2 + sigma ** 2)
  z = (mu - ref_mean) / comb
  return comb * (z * norm_cdf(z) + norm_pdf(z))


def np_argmax_first(vals):
  """ oper_utils.py:73: np.argmax -> first index of the maximum; NaN counts as the maximum. """
  return int(np.argmax(vals))


def random_maximise_on_points(obj, pts):
  """ oper_utils.py:59-80 with the candidate matrix supplied (rand_pts = map_to_bounds(U)). """
  vals = obj(pts)
  idx = np_argmax_first(vals)
  return vals[idx], pts[idx], idx, vals


def chunked_scores(gp, X_cand, acq, chunk=2000, X_halluc=None, **acq_args):
  """ The CPU-baseline driver (SURVEY 8d): score candidates in chunks through the FAITHFUL
      gp.eval(chunk, 'std') (which builds the chunk x chunk covariance exactly like
      gp_core.py:179-187) and keep a running first-index arg-max.  Returns (best_val, best_idx,
      scores). """
  X_cand = np.asarray(X_cand, dtype=np.float64)
  scores = np.empty(len(X_cand))
  for s in range(0, len(X_cand), chunk):
    xs = X_cand[s:s + chunk]
    if X_halluc is not None and len(X_halluc) > 0:
      mu, sd = gp.eval_with_hallucinated_observations(xs, X_halluc, 'std')
    else:
      mu, sd = gp.eval(xs, 'std')
    if acq == 'ucb':
      scores[s:s + chunk] = acq_ucb(mu, sd, acq_args['beta_th'])
    elif acq == 'ei':
      scores[s:s + chunk] = acq_ei(mu, sd, acq_args['curr_best'])
    elif acq == 'pi':
      scores[s:s + chunk] = acq_pi(mu, sd, acq_args['curr_best'])
    elif acq == 'ttei':
      scores[s:s + chunk] = acq_ttei(mu, sd, acq_args['ref_mean'], acq_args['ref_std'])
    else:
      raise ValueError('unknown acquisition %s' % (acq))
  idx = np_argmax_first(scores)
  return scores[idx], idx, scores


def add_ucb_group_scores(gp, add_kernel, group_idx, X_test_j, t, mean_val_j=0.0):
  """ One group of Add-UCB: gpb_acquisitions.py:160-176.  K_*j = scale * k_j(X*_j, X[:, g_j]);
      the FULL additive-GP L and alpha are reused. """
  grp = add_kernel.groupings[group_idx]
  kern_j = add_kernel.kernel_list[group_idx]
  scale = add_kernel.hyperparams['scale']
  X_train_j = np.asarray(gp.X)[:, grp]
  beta_j = add_ucb_beta_th(len(grp), t)
  K_tetr_j = scale * kern_j(X_test_j, X_train_j)
  mu_j = K_tetr_j.dot(gp.alpha) + mean_val_j
  K_tete_j = scale * kern_j(X_test_j, X_test_j)
  V_j = solve_lower_triangular(gp.L, K_tetr_j.T)
  covar_j = K_tete_j - V_j.T.dot(V_j)
  sd_j = np.sqrt(np.diag(covar_j))
  return mu_j + beta_j * sd_j, mu_j, sd_j


def add_ucb_on_points(gp, add_kernel, group_points, t):
  """ gpb_acquisitions.py:139-189 with the per-group candidate matrices supplied.  Returns the
      scattered d-vector and the per-group arg-max indices. """
  ret = np.zeros((sum(len(g) for g in add_kernel.groupings),))
  idxs = []
  for j, (grp, pts) in enumerate(zip(add_kernel.groupings, group_points)):
    scores, _, _ = add_ucb_group_scores(gp, add_kernel, j, pts, t)
    idx = np_argmax_first(scores)
    idxs.append(idx)
    ret[grp] = pts[idx]
  return ret, idxs


def mf_zx(fidel, X):
  """ euclidean_gp.py:387-403 for the default coordinate order: rows [z || x] with the same
      fidelity prefix on every candidate row (gpb_acquisitions.py:314-332). """
  X = np.asarray(X, dtype=np.float64)
  Z = np.repeat(np.asarray(fidel, dtype=np.float64).reshape(1, -1), len(X), axis=0)
  return np.concatenate((Z, X), axis=1)


def rand_exp_sampling_probs(lmls):
  """ gp_core.py:806-810: weights proportional to exp(LML - max LML). """
  lmls = np.asarray(lmls, dtype=np.float64)
  w = np.exp(lmls - lmls.max())
  return w / w.sum()


# ---------------------------------------------------------------------------------------------
# Multi-objective scalarisations                dragonfly/opt/multiobjective_gpb_acquisitions.py
# ---------------------------------------------------------------------------------------------
def moo_ucb_beta_th(dim, time_step):
  """ multiobjective_gpb_acquisitions.py:73-75 """
  return np.sqrt(0.2 * dim * np.log(2 * dim * time_step + 1))


def moo_lin_ucb(mus, sds, weights, beta_th):
  """ :79-91 -- mu_tot + beta_th sqrt(sigma2_tot), accumulated objective by objective. """
  mu_tot = 0.0
  sigma2_tot = 0.0
  for mu, sigma, weight in zip(mus, sds, weights):
    mu_tot += mu * weight
    sigma2_tot += sigma * sigma * weight**2
  return mu_tot + beta_th * np.sqrt(sigma2_tot)


def moo_tch_ucb(mus, sds, weights, refs, beta_th):
  """ :94-107 -- the reference unpacks eval(..., 'std') into `mu, sigma2` and takes np.sqrt of it:
      the square root of the STANDARD DEVIATION enters the UCB.  Restated as written. """
  ret = np.asarray([np.inf for _ in range(len(mus[0]))])
  for mu, sigma2, weight, ref in zip(mus, sds, weights, refs):
    ucb = mu + beta_th * np.sqrt(sigma2) - ref
    ret = np.minimum(ret, ucb / weight)
  return ret


def moo_lin_vals(samples, weights):
  """ :31-39 (lin_ts): s = sum_k sample_k * w_k """
  s = 0.0
  for sample, weight in zip(samples, weights):
    s += sample * weight
  return s


def moo_tch_vals(samples, weights, refs):
  """ :56-65 (tch_ts): s = min_k (sample_k - ref_k) / w_k """
  s = np.full((len(samples[0]), ), np.inf)
  for sample, weight, ref in zip(samples, weights, refs):
    s = np.minimum(s, (sample - ref) / weight)
  return s
