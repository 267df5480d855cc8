"""
The post_sampling goldens (tests/golden/post_sampling.npz, make_golden_post_sampling.py) as inputs of
dragonfly_b200.post_sampling.post_sample_hps, and the NumPy oracle's LML of a layout's hp vector.  Shared by
test_post_sampling_host.py and test_gpu_post_sampling.py.
"""
import numpy as np

from dragonfly_b200 import hp_grid
from dragonfly_b200.kernel import SEKernel, MaternKernel, CoordinateProductKernel
from oracle import gp_oracle as O

CONFIGS = ('A', 'B', 'C')


def oracle_kernel(kern):
  hp = kern.hyperparams
  if isinstance(kern, SEKernel):
    return O.OSEKernel(kern.dim, hp['scale'], hp['dim_bandwidths'])
  if isinstance(kern, MaternKernel):
    return O.OMaternKernel(kern.dim, hp['nu'], hp['scale'], hp['dim_bandwidths'])
  assert isinstance(kern, CoordinateProductKernel)
  return O.OCoordinateProductKernel(kern.dim, hp['scale'], [oracle_kernel(k) for k in kern.kernel_list],
                                    kern.coordinate_list)


def oracle_lml(X, Y, layout, cts, dscr):
  mean_const, noise_var, kern = layout.unpack(cts, Y, dscr[0] if len(dscr) else None)
  gp = O.OGP(X, Y, oracle_kernel(kern), lambda x: np.array([mean_const] * len(x)), noise_var)
  return gp.compute_log_marginal_likelihood()


def oracle_lml_batch(X, Y, layout):
  return lambda cts_rows, dscr_rows: np.array([oracle_lml(X, Y, layout, c, d) for c, d in zip(cts_rows, dscr_rows)])


def config(g, tag):
  """ (X, Y, layout, bounds, dscr_vals, kwargs of post_sample_hps) of golden configuration `tag`. """
  common = dict(mean_func_type=str(g[tag + '_mean_func_type']), noise_var_type=str(g[tag + '_noise_var_type']))
  Y = g[tag + '_Y']
  if tag == 'A':
    X, layout = g['A_X'], hp_grid.EuclideanHPLayout(3, 'matern', nu=-1.0, **common)
  elif tag == 'B':
    X, layout = g['B_X'], hp_grid.EuclideanHPLayout(2, 'se', **common)
  else:
    X = np.concatenate((g['C_Z'], g['C_X']), axis=1)
    layout = hp_grid.EuclideanMFHPLayout(1, 2, 'se', 'matern', domain_nu=2.5, **common)
  dscr_vals = [list(v) for v in g[tag + '_dscr_vals']]
  kw = dict(num_samples=int(g[tag + '_num_samples']), offset=int(g[tag + '_offset']), burn=int(g[tag + '_burn']))
  return X, Y, layout, g[tag + '_bounds'], dscr_vals, kw


def num_slice_samples(g, tag):
  """ Slice samples the fit draws: (burn + total samples) per continuous hp. """
  n_cts, n_dscr = len(g[tag + '_bounds']), len(g[tag + '_dscr_vals'])
  burn = int(g[tag + '_burn'])
  if burn == -1:
    burn = int(np.sqrt(n_cts + n_dscr) * 100)
  total = (int(g[tag + '_num_samples']) - 1) * int(g[tag + '_offset']) + 1
  return n_cts * (burn + total)
