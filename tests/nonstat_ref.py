"""
NumPy restatement of the reference's non-stationary kernels (dragonfly/gp/kernel.py:331-433) as oracle kernels: they
plug into oracle.gp_oracle's OGP / OCoordinateProductKernel like the oracle's own OSEKernel and OMaternKernel.  Used
only by the tests.
"""
import numpy as np

from oracle.gp_oracle import OKernel


class OPolyKernel(OKernel):
  """ scale * ((X1 * s) . (X2 * s)^T + 1) ** order   kernel.py:381-386 """

  def __init__(self, dim, order, scale, dim_scalings):
    self.dim = dim
    scal = dim_scalings if hasattr(dim_scalings, '__len__') else [dim_scalings] * dim
    self.hyperparams = {'order': order, 'scale': scale, 'dim_scalings': np.array(scal, dtype=np.float64)}

  def _evaluate(self, X1, X2):
    s = self.hyperparams['dim_scalings']
    return self.hyperparams['scale'] * (((X1 * s).dot((X2 * s).T) + 1) ** self.hyperparams['order'])


class OExpDecayKernel(OKernel):
  """ scale * prod_i 1 / (1 + x_i + y_i) ** powers[i] + offset   kernel.py:415-426 """

  def __init__(self, dim, scale, offset, powers):
    self.dim = dim
    if not hasattr(powers, '__iter__'):
      powers = [powers] * dim
    self.hyperparams = {'scale': scale, 'offset': offset, 'powers': powers}

  def _evaluate(self, X1, X2):
    ret = self.hyperparams['scale'] * np.ones((X1.shape[0], X2.shape[0]))
    for i in range(self.dim):
      ret *= 1 / (1 + np.add.outer(X1[:, i], X2[:, i])) ** self.hyperparams['powers'][i]
    ret += self.hyperparams['offset']
    return ret
