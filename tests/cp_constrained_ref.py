"""
The constrained fixture's domain (golden cp_constrained.npz, make_golden_cp_constrained.py) as a mirror domain, the
programs the filter tests run, and the host pieces that reproduce the fixture's draws with the NumPy oracle of the
status kernel (constraint_ref.py) in place of the device.
"""
import json
import os
import sys

import numpy as np

import constraint_ref as CR
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
from constraint_fns import z_or_n  # noqa: E402  (tests/golden/constraint_fns.py, shared with the generator)
from dragonfly_b200 import domains, gpb_acquisitions as acq, kernel as K, cartesian_product_gp as cp
from dragonfly_b200.constraints import compile_filter, ACCEPT

CONSTRAINTS = ['np.linalg.norm(x[0:2]) + z <= 1.5', "c != 'b' or n > 2", 'sum(x) + np.sqrt(abs(z)) * w <= 3.5',
               'n * 2 - 3 <= 7 or x[0] < 0.5', z_or_n]
TIGHT = CONSTRAINTS + ['z <= -0.8']
ORDERINGS = dict(raw_name_ordering=['x', 'z', 'n', 'c', 'w'], index_ordering=[[0, 1], [2], [3], [4]],
                 dim_ordering=[[2, ''], [''], [''], ['']])
# programs of the filter tests: each a list of constraints on the fixture's domain
PROGRAMS = {
    'fixture': CONSTRAINTS[:4],
    'exact': ['x[0] + x[1] * z - n / 3 <= 0.25', 'x[-1] * x[-1] + z * z < 1.0 or n >= 4', 'min(z, x[0]) <= max(n, 2)',
              'sum(x[0:2]) - abs(-z) != 0.5', '(n + 1) ** 2 - n * 3 <= 20', 'not (c == \'a\' and w > 1.0)'],
    'approx': ['np.exp(z) + np.log(1 + x[0]) <= 2.5', 'np.sum(x) + z ** 3 >= 0.1', 'np.linalg.norm(x) <= z + 1.0',
               'np.sqrt(x[0] + z) > 0.4 or c == \'c\''],
}


def make_domain(constraints=CONSTRAINTS):
  cons = None if constraints is None else [{'name': 'dc%02d' % k, 'constraint': c} for k, c in enumerate(constraints)]
  return domains.CartesianProductDomain(
      [domains.EuclideanDomain([[0, 1], [0, 1], [-1, 2]]), domains.IntegralDomain([[0, 6]]),
       domains.ProdDiscreteDomain([['a', 'b', 'c']]), domains.ProdDiscreteNumericDomain([[0.5, 1.0, 2.0, 4.0]])],
      domain_constraints=cons, **ORDERINGS)


def make_kernel(scale=1.0):
  return cp.CartesianProductKernel(scale, [K.SEKernel(3, 1.0, [0.4, 0.9, 1.1]), K.MaternKernel(1, 2.5, 1.0, [2.5]),
                                           K.HammingKernel([1.0]), K.MaternKernel(1, 1.5, 1.0, [1.2])])


def jval(v):
  if isinstance(v, (np.ndarray, list, tuple)):
    return [jval(e) for e in v]
  if isinstance(v, (np.integer, int)) and not isinstance(v, bool):
    return int(v)
  if isinstance(v, (np.floating, float)):
    return float(v)
  return str(v)


def oracle_keep_round(parts, filt):
  """ keep_round of gpb_acquisitions.constrained_rand_draw with the oracle's status and the host's settlement. """
  def keep_round(rows, draws, need):
    X = acq._level_rows(draws)
    st = filt.settle(CR.status(filt, X), lambda i: acq.point_from_draws(parts, draws, i))
    sel = np.flatnonzero(st == ACCEPT)[:need]
    return [d[sel] for d in draws], len(sel)
  return keep_round


def run_case(g, k):
  """ The fixture's case k on the host: (points, count) with the global RNG seeded as recorded. """
  run = json.loads(str(g['runs']))[k]
  dom = make_domain(CONSTRAINTS if run['which'] == 'all' else TIGHT)
  parts = acq._cp_parts(dom, make_kernel())
  filt = compile_filter(dom, parts, levels=True)
  np.random.seed(run['seed'])
  chunks = []
  if run['kind'] == 'sample':
    total = acq.constrained_sample(parts, run['M'], oracle_keep_round(parts, filt), chunks)
  else:
    chunks, total = acq.constrained_rand_draw(parts, run['M'], oracle_keep_round(parts, filt))
  draws = [np.concatenate([c[j] for c in chunks]) for j in range(len(parts))] if chunks else None
  pts = [acq.point_from_draws(parts, draws, i) for i in range(total)]
  return pts, total, run


def check_state(g, k):
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['state%d' % k])
  assert st[2] == int(g['pos%d' % k])
  assert [st[3], st[4]] == list(g['gauss%d' % k])


def decode(p):
  """ a fixture point (jval) -> the list-of-parts point """
  return [np.array(p[0], dtype=np.float64), np.array(p[1], dtype=np.int64), [np.str_(v) for v in p[2]],
          [np.float64(v) for v in p[3]]]


def golden_gps(g):
  """ (gp, gp2, H) of the fixture's acquisitions, as dragonfly_b200 CPGPs (the device needs a CUDA build) """
  scale, noise_var, mc, mc2 = [float(v) for v in g['meta']]
  X = [decode(p) for p in json.loads(str(g['X']))]
  H = [decode(p) for p in json.loads(str(g['H']))]
  gp = cp.CPGP(X, list(g['Y']), make_kernel(scale), lambda x: np.array([mc] * len(x)), noise_var)
  gp2 = cp.CPGP(X, list(g['Y2']), make_kernel(scale), lambda x: np.array([mc2] * len(x)), noise_var)
  return gp, gp2, H


def check_acq_state(g, k):
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['acq%d_state' % k])
  assert st[2] == int(g['acq%d_pos' % k])
  assert [st[3], st[4]] == list(g['acq%d_gauss' % k])
