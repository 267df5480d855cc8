"""
NumPy oracle of Thompson sampling on a Cartesian-product domain (asy_ts with the `rand` maximiser): the reference draws
one 1 x 1 posterior sample per candidate, sqrt(sigma^2) z + mu with one normal each, in candidate order.  Built on
oracle.gp_oracle and tests/hamming_ref.py, for the problem of tests/golden/cp_ts.npz.  Used only by the tests.
"""
import json

import numpy as np

from oracle import gp_oracle as O
import hamming_ref as R


def golden_problem(g):
  """ (levels, numeric_levels, scale, noise_var, mean_const, X points, Y, H points) of cp_ts.npz """
  levels, numeric_levels, scale, noise_var, mean_const = R.golden_problem(g)
  return levels, numeric_levels, scale, noise_var, mean_const, R.golden_points(g, 'X'), np.asarray(g['Y']), \
      R.golden_points(g, 'H')


def oracle_gp(g, codes):
  _, _, scale, noise_var, mean_const, X, Y, _ = golden_problem(g)
  return O.OGP(R.encode_points(X, codes), Y, R.oracle_kernel(scale), lambda x: np.array([mean_const] * len(x)),
               noise_var)


def marginal_scores(ogp, C_rows, z, H_rows=None):
  """ fl(fl(sqrt(sigma^2) z) + mu): mu from the GP, sigma^2 from the GP augmented with H_rows (variance only) """
  mu, var = O.eval_std_diag(ogp, C_rows, H_rows)
  return np.sqrt(var) * z + mu, mu, var


def oracle_asy_ts(ogp, acq, parts, max_evals, halluc_pts, codes):
  """ asy_ts after the 'rand' / 4x rewrite: the reference's candidates (draw_cp_candidates), then
      np.random.normal(size=M), then the np.argmax of the marginal draws.  Returns (point, index, scores). """
  M = int(max_evals)
  _, draws = acq.draw_cp_candidates(parts, M)
  z = np.random.normal(size=M)
  pts = [acq.point_from_draws(parts, draws, i) for i in range(M)]
  C = R.encode_points(pts, codes)
  H = R.encode_points(halluc_pts, codes) if len(halluc_pts) > 0 else None
  s, _, _ = marginal_scores(ogp, C, z, H)
  i = O.np_argmax_first(s)
  return pts[i], i, s


def run_golden_case(g, k, acq, parts, ogp, codes, asy_ts=None):
  """ Replays run k of cp_ts.npz from its seed: through asy_ts(max_evals, halluc points) when given, else through the
      oracle.  Returns (points, indices or None). """
  run = json.loads(str(g['ts_runs']))[k]
  H = R.golden_points(g, 'H')
  M = run['max_evals'] * (4 if run['method'] != 'rand' else 1)
  np.random.seed(run['seed'])
  workers = 3 if run['kind'] == 'syn' else 1
  pts, idx = [], []
  for w in range(workers):
    halluc = H[:run['halluc']] if run['kind'] == 'asy' else pts[:w]
    if asy_ts is not None:
      pts.append(asy_ts(run['method'], run['max_evals'], halluc))
    else:
      p, i, _ = oracle_asy_ts(ogp, acq, parts, M, halluc, codes)
      pts.append(p)
      idx.append(i)
  return pts, (idx if asy_ts is None else None)


def check_state(g, k):
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['ts%d_state' % k])
  assert st[2] == int(g['ts%d_pos' % k])
  assert st[3] == int(g['ts%d_has_gauss' % k])
  assert st[4] == float(g['ts%d_cached_gauss' % k])
