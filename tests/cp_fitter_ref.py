"""
The CP fitter goldens (tests/golden/cp_fitter.npz, make_golden_cp_fitter.py) as inputs of dragonfly_b200.hp_grid /
post_sampling, and the NumPy oracle's LML of a CartesianProductHPLayout's hp vector on its encoded rows.  Shared by
test_cp_fitter_host.py and test_gpu_cp_fitter.py.
"""
import json

import numpy as np

from dragonfly_b200 import hp_grid
from dragonfly_b200.kernel import SEKernel, MaternKernel, HammingKernel
from oracle import gp_oracle as O
import hamming_ref as H

CONFIGS = ('M', 'T')
ML_METHODS = ('rand', 'rand_exp_sampling', 'pdoo', 'direct')


def parts(tag):
  if tag == 'M':
    return [('euclidean', 2, 'matern'), ('integral', 1, 'matern'), ('prod_discrete', 3, 'hamming'),
            ('prod_discrete_numeric', 1, 'matern')]
  return [('euclidean', 2, 'matern', -1.0), ('prod_discrete', 2, 'hamming'), ('integral', 1, 'matern', -1.0)]


def layout(tag):
  return hp_grid.CartesianProductHPLayout(parts(tag), mean_func_type='tune', noise_var_type='tune')


def points(g, tag):
  return [H.jpoint(p) for p in json.loads(str(g[tag + '_points']))]


def oracle_kernel(kern):
  """ a CartesianProductKernel of SE / Matern / Hamming children -> the oracle's coordinate-product kernel """
  kids = []
  for k in kern.kernel_list:
    hp = k.hyperparams
    if isinstance(k, HammingKernel):
      kids.append(H.OHammingKernel(hp['dim_weights']))
    elif isinstance(k, MaternKernel):
      kids.append(O.OMaternKernel(k.dim, hp['nu'], hp['scale'], hp['dim_bandwidths']))
    else:
      assert isinstance(k, SEKernel)
      kids.append(O.OSEKernel(k.dim, hp['scale'], hp['dim_bandwidths']))
  return O.OCoordinateProductKernel(kern.dim, kern.hyperparams['scale'], kids, kern.coordinate_list)


def oracle_lml(X, Y, lay, cts, dscr):
  """ X: the layout's encoded rows """
  mean_const, noise_var, kern = lay.unpack(cts, Y, tuple(dscr))
  gp = O.OGP(X, Y, oracle_kernel(kern), lambda x: np.array([mean_const] * len(x)), noise_var)
  return gp.compute_log_marginal_likelihood()


def oracle_lml_batch(X, Y, lay):
  """ the post_sampling lml_batch(cts_rows, dscr_rows) of the oracle """
  return lambda cts_rows, dscr_rows: np.array([oracle_lml(X, Y, lay, c, d) for c, d in zip(cts_rows, dscr_rows)])


def dscr_vals(g, tag):
  return [list(v) for v in g[tag + '_dscr_vals']]
