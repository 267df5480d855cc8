"""
Device-backed mirror of the Cartesian-product GP: dragonfly/gp/kernel.py:504-538 (CartesianProductKernel) and
dragonfly/gp/cartesian_product_gp.py:207-248 (CPGP).

A CPGP point is a list of per-domain parts, x = [x^(0), x^(1), ...]; its kernel is scale * prod_j k_j(x^(j), y^(j))
(kernel.py:524-533; CPGP._get_training_kernel_matrix builds the same product, cartesian_product_gp.py:238-248).  With SE /
Matern factors that is exactly the coordinate-product form the device descriptor already evaluates (the multi-fidelity
kernel's form, SURVEY a5): the parts are laid side by side in one row and factor j reads its own columns.  Nothing else
changes -- build, eval, hallucinations, LML, the acquisition operators all come from gp_core.GP.

Parts served: Euclidean, integral and prod_discrete_numeric parts under SE / Matern (their values are the columns), and
prod_discrete parts under HammingKernel (kernel.py:436-457): each categorical value becomes the code its Hamming child's
CategoryCodes table gives it, and the device's HAMMING factor compares codes.  The table is the child's, so the training
rows, candidates, hallucinations and kernel(X1, X2) all see one encoding.

Out of scope (SURVEY 2): factors evaluated from precomputed distance lists (`domain_lists_of_dists`: the OTMANN distances
of neural-network domains, kernel.evaluate_from_dists) -- they raise.

`handle_non_psd_kernels`: the reference's CPGP defaults to 'project_first' (an eigen-projection of K onto the PSD cone
before the Cholesky, gp_core.py:839-842) because its NN factors are not PSD.  Every factor served here is, so the
projection is the identity up to rounding (its eigen-clip moves K by ~1e-14, measured against the reference in
tests/golden/cpgp.npz) and the build is the guaranteed-PSD one.
"""
import numpy as np

from .gp_core import GP
from .kernel import CoordinateProductKernel, category_codes, kernel_dim, _kind_of


def _part_encoders(kernel):
  """ Per part: the CategoryCodes table of its Hamming factor, or None for a numeric part.  None without a kernel. """
  kernel_list = getattr(kernel, 'kernel_list', None) if kernel is not None else None
  if kernel_list is None:
    return None
  return [category_codes(k) if _kind_of(k) == 'HammingKernel' else None for k in kernel_list]


def flatten_parts(X, kernel=None):
  """ list of points, each a list of per-domain parts -> (n, sum d_j) matrix with the parts side by side.  With a
      CartesianProductKernel, the parts of its Hamming factors are laid out as category codes. """
  if len(X) == 0:
    return np.zeros((0, 0))
  enc = _part_encoders(kernel)
  if enc is None or all(e is None for e in enc):
    return np.ascontiguousarray(np.array([np.concatenate([np.atleast_1d(np.asarray(part, dtype=np.float64)).reshape(-1)
                                                            for part in x]) for x in X]))
  rows = []
  for x in X:
    cols = []
    for part, e in zip(x, enc):
      if e is None:
        cols.append(np.atleast_1d(np.asarray(part, dtype=np.float64)).reshape(-1))
      else:
        cols.append(np.array([e.encode(v) for v in part], dtype=np.float64))
    rows.append(np.concatenate(cols))
  return np.ascontiguousarray(np.array(rows))


class CartesianProductKernel(CoordinateProductKernel):
  """ kernel.py:504-538.  kernel_list[j] acts on part j of every point. """

  def __init__(self, scale, kernel_list):
    dims = [kernel_dim(k) for k in kernel_list]
    starts = np.concatenate(([0], np.cumsum(dims))).astype(int)
    coords = [list(range(starts[j], starts[j + 1])) for j in range(len(dims))]
    super(CartesianProductKernel, self).__init__(int(starts[-1]), scale, list(kernel_list), coords)
    self.num_kernels = len(kernel_list)

  def _child_evaluate(self, X1, X2):
    return super(CartesianProductKernel, self)._child_evaluate(_as_rows(X1, self), _as_rows(X2, self))

  def __str__(self):
    return 'DomProd scale=%0.2f, ' % (self.hyperparams['scale']) + ', '.join([str(k) for k in self.kernel_list])


def _as_rows(X, kernel=None):
  """ Points in CPGP's list-of-parts format, or an already flat (n, d) matrix / CUDA tensor (categories already coded). """
  try:
    import torch
    if isinstance(X, torch.Tensor):
      return X
  except ImportError:
    pass
  if isinstance(X, np.ndarray) and X.ndim == 2 and X.dtype != object:
    return X
  return flatten_parts(X, kernel)


class CPGP(GP):
  """ cartesian_product_gp.py:207-248 for Euclidean-type and Hamming factors. """

  def __init__(self, X, Y, kernel, mean_func, noise_var, domain_lists_of_dists=None, build_posterior=True,
               reporter=None, handle_non_psd_kernels='project_first', **kwargs):
    if domain_lists_of_dists is None:
      domain_lists_of_dists = [None] * kernel.num_kernels
    if any(d is not None for d in domain_lists_of_dists):
      raise NotImplementedError('factors evaluated from precomputed distance lists (kernel.evaluate_from_dists: the '
                                'neural-network domains) are outside the GPU hot-path scope.')
    self.domain_lists_of_dists = domain_lists_of_dists
    if handle_non_psd_kernels in ('project_first', 'try_before_project'):
      if not kernel.is_guaranteed_psd():
        raise NotImplementedError('a non-PSD factor needs the eigen-projection of the reference (gp_core.py:839-842).')
      handle_non_psd_kernels = 'guaranteed_psd'          # the projection of a PSD matrix is the identity
    super(CPGP, self).__init__(X, Y, kernel, mean_func, noise_var, build_posterior, reporter, handle_non_psd_kernels,
                               **kwargs)

  def set_domain_lists_of_dists(self, domain_lists_of_dists):
    if any(d is not None for d in domain_lists_of_dists):
      raise NotImplementedError('precomputed distance lists are outside the GPU hot-path scope.')
    self.domain_lists_of_dists = domain_lists_of_dists

  def _train_matrix(self):
    return flatten_parts(self.X, self.kernel)

  def _test_matrix(self, X_test):
    return _as_rows(X_test, self.kernel)

  def _get_training_kernel_matrix(self):
    return self.kernel(self.X, self.X)

  def _child_str(self):
    mean_str = 'mu[#0]=%0.4f, ' % (self.mean_func([self.X[0]])[0]) if len(self.X) > 0 else ''
    return mean_str + str(self.kernel)
