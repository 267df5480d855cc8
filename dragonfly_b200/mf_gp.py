"""
Device-backed mirrors of the multi-fidelity GP wrappers: dragonfly/gp/mf_gp.py:26-99 (MFGP) and
dragonfly/gp/euclidean_gp.py:134-150, 347-415 (EuclideanGP, EuclideanMFGP).  These are thin: they
only arrange the (fidelity, domain) coordinates into the [z || x] rows the product kernel
scale * k_F(z, z') * k_D(x, x') sees (euclidean_gp.py:369-374, 387-403); all numerics are in GP.
"""
import numpy as np

from . import kernel as gp_kernel
from .gp_core import GP


class EuclideanGP(GP):
  """ euclidean_gp.py:134-150: kernel may be an object or one of 'se' / 'matern' / 'poly' / 'esp'. """

  def __init__(self, X, Y, kernel, mean_func, noise_var, kernel_hyperparams=None,
               build_posterior=True, reporter=None, **kwargs):
    if isinstance(kernel, str):
      kernel = self._get_kernel_from_type(kernel, kernel_hyperparams)
    super(EuclideanGP, self).__init__(X, Y, kernel, mean_func, noise_var, build_posterior,
                                      reporter, **kwargs)

  @classmethod
  def _get_kernel_from_type(cls, kernel_type, kernel_hyperparams):
    if kernel_type in ['se']:
      return gp_kernel.SEKernel(kernel_hyperparams['dim'], kernel_hyperparams['scale'],
                                kernel_hyperparams['dim_bandwidths'])
    elif kernel_type in ['matern']:
      return gp_kernel.MaternKernel(kernel_hyperparams['dim'], kernel_hyperparams['nu'],
                                    kernel_hyperparams['scale'],
                                    kernel_hyperparams['dim_bandwidths'])
    elif kernel_type in ['poly']:         # euclidean_gp.py:160-163
      return gp_kernel.PolyKernel(kernel_hyperparams['dim'], kernel_hyperparams['order'],
                                  kernel_hyperparams['scale'], kernel_hyperparams['dim_scalings'])
    elif kernel_type in ['esp']:          # euclidean_gp.py:168-171
      return gp_kernel.ESPKernelSE(kernel_hyperparams['dim'], kernel_hyperparams['scale'],
                                   kernel_hyperparams['order'], kernel_hyperparams['dim_bandwidths'])
    raise NotImplementedError('kernel_type %s is outside the GPU hot-path scope.' % (kernel_type))


def get_ZX_from_ZZ_XX(ZZ, XX):
  """ mf_gp.py:18-23 """
  if hasattr(ZZ, '__iter__') and len(ZZ) == len(XX):
    return [(z, x) for (z, x) in zip(ZZ, XX)]
  return (ZZ, XX)


class EuclideanMFGP(GP):
  """ An MFGP for Euclidean fidelity and domain spaces (euclidean_gp.py:347-415). """

  def __init__(self, ZZ, XX, YY, mf_kernel, kernel_scale, fidel_kernel, domain_kernel, mean_func,
               noise_var, *args, **kwargs):
    if len(ZZ) != 0:
      self.fidel_dim = len(ZZ[0])
      self.domain_dim = len(XX[0])
    if fidel_kernel is not None and domain_kernel is not None:
      self.fidel_kernel = fidel_kernel
      self.domain_kernel = domain_kernel
      self.fidel_dim = fidel_kernel.dim
      self.domain_dim = domain_kernel.dim
    elif 'fidel_dim' in kwargs and 'domain_dim' in kwargs:
      self.fidel_dim = kwargs.pop('fidel_dim')
      self.domain_dim = kwargs.pop('domain_dim')
    else:
      raise Exception('Specify fidel_dim and domain_dim.')
    self.fidel_coords = list(range(self.fidel_dim))
    self.domain_coords = list(range(self.fidel_dim, self.fidel_dim + self.domain_dim))
    if mf_kernel is None:
      mf_kernel = gp_kernel.CoordinateProductKernel(self.fidel_dim + self.domain_dim, kernel_scale,
                                                    [fidel_kernel, domain_kernel],
                                                    [self.fidel_coords, self.domain_coords])
    self.ZZ = list(ZZ)
    self.XX = list(XX)
    self.YY = list(YY)
    ZX = self.get_ZX_from_ZZ_XX(ZZ, XX)
    super(EuclideanMFGP, self).__init__(ZX, YY, mf_kernel, mean_func, noise_var, *args, **kwargs)

  def _test_fidel_domain_dims(self, test_fidel_dim, test_domain_dim):
    if test_fidel_dim != self.fidel_dim or test_domain_dim != self.domain_dim:
      raise ValueError('ZZ, XX dimensions should be (%d, %d). Given (%d, %d)' % (
          self.fidel_dim, self.domain_dim, test_fidel_dim, test_domain_dim))

  def get_ZX_matrix(self, ZZ, XX):
    """ (n, fidel_dim + domain_dim) matrix of [z || x] rows in kernel coordinate order. """
    ZZ = np.asarray(ZZ, dtype=np.float64)
    XX = np.asarray(XX, dtype=np.float64)
    self._test_fidel_domain_dims(ZZ.shape[1], XX.shape[1])
    ordering = np.argsort(self.fidel_coords + self.domain_coords)
    return np.concatenate((ZZ, XX), axis=1)[:, ordering]

  def get_ZX_from_ZZ_XX(self, ZZ, XX):
    """ euclidean_gp.py:387-403 """
    ordering = np.argsort(self.fidel_coords + self.domain_coords)
    if hasattr(ZZ, '__iter__') and len(ZZ) == 0:
      return []
    elif hasattr(ZZ[0], '__iter__'):
      return list(self.get_ZX_matrix(ZZ, XX))
    self._test_fidel_domain_dims(len(ZZ), len(XX))
    return np.concatenate((ZZ, XX))[ordering]

  def eval_at_fidel(self, ZZ_test, XX_test, *args, **kwargs):
    """ mf_gp.py:56-60 """
    return self.eval(self.get_ZX_matrix(ZZ_test, XX_test), *args, **kwargs)

  def eval_at_fidel_with_hallucinated_observations(self, ZZ_test, XX_test, ZZ_halluc, XX_halluc,
                                                   *args, **kwargs):
    """ mf_gp.py:62-67 """
    return self.eval_with_hallucinated_observations(
        self.get_ZX_matrix(ZZ_test, XX_test), self.get_ZX_from_ZZ_XX(ZZ_halluc, XX_halluc),
        *args, **kwargs)

  def set_mf_data(self, ZZ, XX, YY, build_posterior=True):
    """ mf_gp.py:69-75 """
    self.ZZ = list(ZZ)
    self.XX = list(XX)
    self.YY = list(YY)
    super(EuclideanMFGP, self).set_data(self.get_ZX_from_ZZ_XX(ZZ, XX), YY, build_posterior)

  def add_mf_data_multiple(self, ZZ_new, XX_new, YY_new, *args, **kwargs):
    """ mf_gp.py:77-82 """
    ZX_new = self.get_ZX_from_ZZ_XX(ZZ_new, XX_new)
    self.ZZ.extend(ZZ_new)
    self.XX.extend(XX_new)
    self.add_data_multiple(ZX_new, YY_new, *args, **kwargs)

  def add_mf_data_single(self, zz_new, xx_new, yy_new, *args, **kwargs):
    self.add_mf_data_multiple([zz_new], [xx_new], [yy_new], *args, **kwargs)

  def draw_mf_samples(self, num_samples, ZZ_test=None, XX_test=None, *args, **kwargs):
    """ mf_gp.py:88-91 """
    ZX_test = None if ZZ_test is None else self.get_ZX_matrix(ZZ_test, XX_test)
    return self.draw_samples(num_samples, ZX_test, *args, **kwargs)

  def get_fidel_kernel(self):
    return self.fidel_kernel

  def get_domain_kernel(self):
    return self.domain_kernel

  def get_domain_pts(self, data_idxs=None):
    data_idxs = data_idxs if data_idxs is not None else range(self.num_tr_data)
    return [self.XX[i] for i in data_idxs]

  def get_fidel_pts(self, data_idxs=None):
    data_idxs = data_idxs if data_idxs is not None else range(self.num_tr_data)
    return [self.ZZ[i] for i in data_idxs]
