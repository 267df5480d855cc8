"""
NumPy oracle of the `ga` acquisition maximiser on a Cartesian-product domain, for the problem of tests/golden/cp_ga.npz:
the parity restatement (dragonfly_b200.ga) driven by oracle.gp_oracle's values, and the acquisition operators around it
(asy_* / syn_ei / mo_lin_ucb) replayed call by call.  Used only by the tests.
"""
import json

import numpy as np

from oracle import gp_oracle as O
import hamming_ref as R
import moo_cp_ref as MR

from dragonfly_b200 import domains
from dragonfly_b200 import ga
from dragonfly_b200 import gpb_acquisitions as acq


def golden_problem(g):
  """ (domain, parts, X points, H points) of cp_ga.npz """
  levels, numeric_levels = json.loads(str(g['levels'])), json.loads(str(g['numeric_levels']))
  dom = R.make_domain(domains, levels, numeric_levels)
  return dom, acq._cp_parts(dom), R.golden_points(g, 'X'), R.golden_points(g, 'H')


def oracle_gps(g, codes):
  _, _, X, _ = golden_problem(g)
  rows = R.encode_points(X, codes)
  gps = []
  for key, yk, okern in (('meta', 'Y', R.oracle_kernel), ('meta2', 'Y2', MR.oracle_kernel2)):
    scale, noise_var, mean_const = [float(v) for v in g[key]]
    gps.append(O.OGP(rows, np.asarray(g[yk]), okern(scale), (lambda c: (lambda x: np.array([c] * len(x))))(mean_const),
                     noise_var))
  return gps


def runs(g):
  return json.loads(str(g['runs']))


def golden_log(g, k):
  """ run k's query log: per GA call the list of points, and all values in order """
  return [[R.jpoint(p) for p in call] for call in json.loads(str(g['run%d_log' % k]))], np.asarray(g['run%d_vals' % k])


class Scorer(object):
  """ The acquisition values of list-of-parts points under the oracle GPs: kind 'ucb' / 'ei' / 'pi' / 'ttei' /
      'mo_lin_ucb', variance from the GP augmented with halluc (mean from the GP itself). """

  def __init__(self, g, ogps, codes, kind, halluc=(), ref=None):
    self.g, self.ogps, self.codes, self.kind, self.ref = g, ogps, codes, kind, ref
    self.H = R.encode_points(list(halluc), codes) if len(halluc) > 0 else None

  def mu_sd(self, ogp, pts):
    mu, var = O.eval_std_diag(ogp, R.encode_points(pts, self.codes), self.H if self.kind != 'mo_lin_ucb' else None)
    return mu, np.sqrt(var)

  def __call__(self, pts):
    if self.kind == 'mo_lin_ucb':
      mus, sds = zip(*[self.mu_sd(ogp, pts) for ogp in self.ogps])
      return O.moo_lin_ucb(list(mus), list(sds), list(self.g['weights']), float(self.g['mo_beta']))
    mu, sd = self.mu_sd(self.ogps[0], pts)
    if self.kind == 'ucb':
      return O.acq_ucb(mu, sd, float(self.g['beta']))
    if self.kind == 'ei':
      return O.acq_ei(mu, sd, float(self.g['curr_max']))
    if self.kind == 'pi':
      return O.acq_pi(mu, sd, float(self.g['curr_max']))
    return O.acq_ttei(mu, sd, self.ref[0], self.ref[1])


def replay(g, k, maximise=None):
  """ Replays run k from its seed.  maximise(kind, halluc, method, max_evals, ref) -> point runs one GA call; the default
      is the parity restatement scored by the oracle.  Returns (points returned, per GA call (points, values) logged by
      the default maximiser). """
  run = runs(g)[k]
  codes = {}
  ogps = oracle_gps(g, codes)
  _, parts, _, H = golden_problem(g)
  logs = []

  def oracle_maximise(kind, halluc, method, max_evals, ref=None):
    log = []
    pt = ga.maximise(Scorer(g, ogps, codes, kind, halluc, ref), parts, method, max_evals, log)
    logs.append(([p for b in log for p in b[0]], np.concatenate([b[1] for b in log])))
    return pt
  call = maximise or oracle_maximise
  name, method, B = run['name'], run['method'], run['max_evals']
  halluc = H[:run['halluc']]
  np.random.seed(run['seed'])
  if name == 'syn_ei':
    pts = []
    for _ in range(2):
      pts.append(call('ei', list(pts), method, B))
  elif name == 'ttei':                     # asy_ttei (gpb_acquisitions.py:282-294)
    if np.random.random() < 0.5:
      pts = [call('ei', halluc, method, B)]
    else:
      ei_pt = call('ei', halluc, method, B // 2)
      mu, sd = Scorer(g, ogps, codes, 'ei', halluc).mu_sd(ogps[0], [ei_pt])
      pts = [call('ttei', halluc, method, B // 2, (float(mu[0]), float(sd[0])))]
  else:
    pts = [call(name, halluc, method, B)]
  return pts, logs


def check_state(g, k):
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['run%d_state' % k])
  assert st[2] == int(g['run%d_pos' % k])
  assert st[3] == int(g['run%d_has_gauss' % k])
  assert st[4] == float(g['run%d_cached_gauss' % k])


# ---- the device GA (dfb_ga_maximise) ------------------------------------------------------------------------------
def philox_rng(seed):
  """ The counter-based streams of the device GA from oracle/philox.py: uniform(S, row) / normal(S, row) are elements
      (0 .. S-1, row) of dfb_fill_rng(seed, ..., DFB_RNG_UNIFORM / DFB_RNG_NORMAL). """
  from oracle import philox
  return (lambda S, row: philox.fill(seed, row, S, 1, 1)[:, 0]), (lambda S, row: philox.fill(seed, row, S, 1, 0)[:, 0])


def device_ga(score_rows, desc, seed, n_pool, n_total, uniform, normal, epochs=None):
  """ NumPy restatement of dfb_ga_maximise (include/dfb200.h) on level rows: score_rows(rows) -> values.  Returns
      (rows, values, smallest selection margin -- the distance of a parent or numeric-level uniform from a CDF boundary,
      relative to the CDF's total).  epochs: stop after that many epochs. """
  d = desc.d
  U = np.array([uniform(d, r) for r in range(n_pool)]).reshape(n_pool, d)
  rows = np.empty((n_total, d))
  for c in range(d):
    lo, hi, kind = desc.lo[c], desc.hi[c], desc.kind[c]
    if kind == 2:
      L = desc.n_levels[c]
      rows[:n_pool, c] = np.minimum(np.floor(U[:, c] * L), L - 1)
    else:
      v = U[:, c] * (hi - lo) + lo
      rows[:n_pool, c] = np.trunc(v) if kind == 1 else v
  vals = list(np.asarray(score_rows(rows[:n_pool]), dtype=np.float64))
  margin, r0, e = np.inf, n_pool, 0
  while r0 < n_total and (epochs is None or e < epochs):
    c = min(5, n_total - r0)
    v = np.asarray(vals[:r0])
    n = r0
    mean = v.sum() / n
    std = np.sqrt(((v - mean) ** 2).sum() / n)
    ex = np.exp((v - mean) / (2.0 * (std + 0.0001)))
    cdf = np.cumsum(ex)
    bad = not (np.all(np.isfinite(ex)) and np.isfinite(cdf[-1]) and cdf[-1] > 0)
    for j in range(c):
      row = r0 + j
      u = uniform(2 * d + 1, row)
      z = normal(d, row)
      if bad:
        par = min(int(u[0] * n), n - 1)
      else:
        t = u[0] * cdf[-1]
        par = min(int(np.searchsorted(cdf, t, side='right')), n - 1)
        margin = min(margin, np.abs(cdf - t).min() / cdf[-1])
      x = rows[par].copy()
      for p in range(desc.n_parts):
        c0, c1, kind = desc.part_c0[p], desc.part_c1[p], desc.part_kind[p]
        if kind in (0, 1):
          for k in range(c0, c1):
            sigma = (desc.hi[k] - desc.lo[k]) / 10.0
            xv = min(max(x[k] + sigma * z[k], desc.lo[k]), desc.hi[k])
            x[k] = np.rint(xv) if kind == 1 else xv
        elif kind == 2:
          w = c1 - c0
          q = c0 + min(int(u[1 + c0] * w), w - 1)
          L = desc.n_levels[q]
          k = min(int(u[1 + d + c0] * (L - 1)), L - 2)
          x[q] = k if k < x[q] else k + 1
        else:
          for k in range(c0, c1):
            L = desc.n_levels[k]
            lv = np.array([desc.lut[desc.val_off[k] + l] for l in range(L)])
            wts = np.exp(-np.abs(lv - lv[int(x[k])]))
            cdf_k = np.cumsum(0.8 * (wts / wts.sum()) + 0.2 / L)
            cdf_k = cdf_k / cdf_k[-1]
            x[k] = float(min(int(np.searchsorted(cdf_k, u[1 + k], side='right')), L - 1))
            margin = min(margin, np.abs(cdf_k - u[1 + k]).min())
      rows[row] = x
    vals.extend(np.asarray(score_rows(rows[r0:r0 + c]), dtype=np.float64))
    r0 += c
    e += 1
  return rows[:r0], np.asarray(vals), margin
