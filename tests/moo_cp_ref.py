"""
NumPy oracle of the multi-objective acquisitions on a Cartesian-product domain with the `rand` maximiser: the reference
scores its sampled points one at a time, each objective's UCB from gp.eval([x], 'std') or its own 1 x 1 posterior draw
fl(fl(sqrt(sigma^2) z) + mu) with the normals consumed candidate-major, objective-minor.  Built on oracle.gp_oracle and
tests/hamming_ref.py, for the problem of tests/golden/moo_cp.npz.  Used only by the tests.
"""
import json

import numpy as np

from oracle import gp_oracle as O
import hamming_ref as R

TS_NAMES = ('lin_ts', 'tch_ts')


def golden_problem(g):
  """ (levels, numeric_levels, X points, [Y, Y2], [(scale, noise_var, mean_const) per objective], H points) """
  levels, numeric_levels = json.loads(str(g['levels'])), json.loads(str(g['numeric_levels']))
  metas = [tuple(float(v) for v in g[key]) for key in ('meta', 'meta2')]
  return levels, numeric_levels, R.golden_points(g, 'X'), [np.asarray(g['Y']), np.asarray(g['Y2'])], metas, \
      R.golden_points(g, 'H')


def make_kernel2(kernel, cp, scale):
  """ the second objective's CartesianProductKernel (make_golden_moo_cp.make_kernel2) from dragonfly_b200's classes """
  return cp.CartesianProductKernel(scale, [kernel.SEKernel(2, 1.0, [0.7, 0.5]), kernel.MaternKernel(1, 2.5, 1.0, [1.8]),
                                           kernel.HammingKernel([0.3, 0.4, 0.3]),
                                           kernel.MaternKernel(1, 1.5, 1.0, [0.8])])


def oracle_kernel2(scale):
  return O.OCoordinateProductKernel(7, scale, [O.OSEKernel(2, 1.0, [0.7, 0.5]), O.OMaternKernel(1, 2.5, 1.0, [1.8]),
                                               R.OHammingKernel([0.3, 0.4, 0.3]), O.OMaternKernel(1, 1.5, 1.0, [0.8])],
                                    [[0, 1], [2], [3, 4, 5], [6]])


def oracle_gps(g, codes):
  _, _, X, Ys, metas, _ = golden_problem(g)
  rows = R.encode_points(X, codes)
  return [O.OGP(rows, Y, okern(scale), (lambda c: (lambda x: np.array([c] * len(x))))(mean_const), noise_var)
          for Y, (scale, noise_var, mean_const), okern in zip(Ys, metas, (R.oracle_kernel, oracle_kernel2))]


def scalarise(name, mus, sds_or_vals, weights, refs, beta):
  """ the reference's scalarisation (:19-107) of per-objective vectors: (mu, sd) for UCB, the sampled values for TS """
  if name == 'lin_ucb':
    return O.moo_lin_ucb(mus, sds_or_vals, weights, beta)
  if name == 'tch_ucb':
    return O.moo_tch_ucb(mus, sds_or_vals, weights, refs, beta)
  if name == 'lin_ts':
    return O.moo_lin_vals(sds_or_vals, weights)
  return O.moo_tch_vals(sds_or_vals, weights, refs)


def oracle_scores(ogps, name, C_rows, weights, refs, beta, z=None, H_rows=None):
  """ per-candidate scalarised values: UCB from each GP's (mu, sd), TS from fl(fl(sqrt(sigma^2_k) z_k) + mu_k) with
      sigma^2_k of GP k augmented with H_rows (variance only) """
  mus, vals = [], []
  for k, ogp in enumerate(ogps):
    mu, var = O.eval_std_diag(ogp, C_rows, H_rows if name in TS_NAMES else None)
    mus.append(mu)
    vals.append(np.sqrt(var) * z[:, k] + mu if name in TS_NAMES else np.sqrt(var))
  return scalarise(name, mus, vals, weights, refs, beta)


def oracle_run(ogps, acq, parts, name, M, halluc_pts, codes, weights, refs, beta):
  """ one call after the TS 'rand' / 4x rewrite: the reference's candidates (draw_cp_candidates), then for TS
      np.random.normal(size=(M, K)), then np.argmax.  Returns (point, index, scores). """
  _, draws = acq.draw_cp_candidates(parts, M)
  z = np.random.normal(size=(M, len(ogps))) if name in TS_NAMES else None
  pts = [acq.point_from_draws(parts, draws, i) for i in range(M)]
  C = R.encode_points(pts, codes)
  H = R.encode_points(halluc_pts, codes) if len(halluc_pts) > 0 else None
  s = oracle_scores(ogps, name, C, weights, refs, beta, z, H)
  i = O.np_argmax_first(s)
  return pts[i], i, s


def runs(g):
  return json.loads(str(g['runs']))


def run_size(run):
  return run['max_evals'] * (4 if run['name'] in TS_NAMES and run['method'] != 'rand' else 1)


def check_state(g, k):
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['run%d_state' % k])
  assert st[2] == int(g['run%d_pos' % k])
  assert st[3] == int(g['run%d_has_gauss' % k])
  assert st[4] == float(g['run%d_cached_gauss' % k])
