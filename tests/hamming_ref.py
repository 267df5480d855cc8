"""
NumPy restatement of the reference's HammingKernel (dragonfly/gp/kernel.py:436-457, pairwise_hamming_kernel,
general_utils.py:113-146) as an oracle kernel on category codes: it plugs into oracle.gp_oracle's OGP /
OCoordinateProductKernel like the oracle's own OSEKernel and OMaternKernel.  Also the decoding of the JSON points of
tests/golden/hamming.npz and the golden problem's domain and kernels.  Used only by the tests.
"""
import json

import numpy as np

from oracle import gp_oracle as O


class OHammingKernel(O.OKernel):
  """ (np.equal(x, y) * wts).sum() for every pair of rows of codes -- codes are equal exactly when the categories are,
      and every term is 0 or w_q, summed over the last (contiguous) axis in NumPy's pairwise order like the reference. """

  def __init__(self, dim_weights):
    if isinstance(dim_weights, (int, float)):
      dim_weights = np.ones((dim_weights,)) / float(dim_weights)
    self.hyperparams = {'dim_weights': np.array(dim_weights, dtype=np.float64)}
    self.dim = len(self.hyperparams['dim_weights'])

  def _evaluate(self, X1, X2):
    eq = np.equal(X1[:, None, :], X2[None, :, :])
    return np.ascontiguousarray(eq * self.hyperparams['dim_weights']).sum(axis=2)


_TYPES = {'str_': np.str_, 'int64': np.int64, 'float64': np.float64, 'bool_': np.bool_, 'bool': bool, 'str': str,
          'int': int, 'float': float}


def jvalue(v):
  """ [value, type name] of the golden's JSON -> the value with its type """
  return _TYPES[v[1]](v[0])


def jpoint(p):
  """ a golden JSON point -> list of parts, each a list of typed scalars """
  return [[jvalue(v) for v in part] for part in p]


def jencode(pt):
  """ a list-of-parts point -> the golden's JSON form (make_golden_hamming.jpoint): an ndarray part as [[x, dtype], ..],
      a list part as [[value, type name], ..] """
  def _v(v):
    return [v.item(), type(v).__name__] if isinstance(v, np.generic) else [v, type(v).__name__]
  return [[[x, part.dtype.name] for x in part.tolist()] if isinstance(part, np.ndarray) else [_v(v) for v in part]
          for part in pt]


def golden_points(g, key):
  return [jpoint(p) for p in json.loads(str(g[key]))]


def golden_problem(g):
  """ (levels, numeric_levels, scale, noise_var, mean_const) of golden 2 """
  scale, noise_var, mean_const = [float(v) for v in g['meta']]
  return json.loads(str(g['levels'])), json.loads(str(g['numeric_levels'])), scale, noise_var, mean_const


def make_domain(domains, levels, numeric_levels):
  """ the golden's domain from a module of domain mirrors (dragonfly_b200.domains) """
  return domains.CartesianProductDomain([domains.EuclideanDomain([[0, 1], [-1, 2]]), domains.IntegralDomain([[0, 6]]),
                                         domains.ProdDiscreteDomain(levels),
                                         domains.ProdDiscreteNumericDomain(numeric_levels)])


def make_kernel(kernel, cp, scale):
  """ the golden's CartesianProductKernel from dragonfly_b200.kernel / cartesian_product_gp """
  return cp.CartesianProductKernel(scale, [kernel.SEKernel(2, 1.0, [0.4, 0.9]), kernel.MaternKernel(1, 2.5, 1.0, [2.5]),
                                           kernel.HammingKernel([0.5, 0.2, 0.3]),
                                           kernel.MaternKernel(1, 1.5, 1.0, [1.2])])


def oracle_kernel(scale):
  """ the same kernel as an oracle kernel on rows [e0, e1, i, c0, c1, c2, n] (categories as codes) """
  return O.OCoordinateProductKernel(7, scale, [O.OSEKernel(2, 1.0, [0.4, 0.9]), O.OMaternKernel(1, 2.5, 1.0, [2.5]),
                                               OHammingKernel([0.5, 0.2, 0.3]), O.OMaternKernel(1, 1.5, 1.0, [1.2])],
                                    [[0, 1], [2], [3, 4, 5], [6]])


def encode_points(points, codes):
  """ list-of-parts points -> rows [e0, e1, i, c0, c1, c2, n] with the categories coded by `codes` (value -> code
      dict shared across calls, Python == semantics like CategoryCodes) """
  rows = []
  for e, i, c, n in points:
    cc = []
    for v in c:
      if v not in codes:
        codes[v] = len(codes)
      cc.append(codes[v])
    rows.append(list(np.asarray(e, dtype=np.float64)) + [float(i[0])] + [float(x) for x in cc] + [float(n[0])])
  return np.array(rows, dtype=np.float64)
