"""
Constrained Cartesian-product domains on the host (no GPU): the mirror domain's raw points and constraint checks, the
compiler's column map and residue routing, the certified statuses of the NumPy oracle of the device filter against the
domain's own evaluator, and the constrained draw against the unmodified reference (golden cp_constrained.npz).
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import constraint_ref as CR
import cp_constrained_ref as F

from dragonfly_b200 import domains, gpb_acquisitions as acq
from dragonfly_b200.constraints import compile_filter, column_map, ACCEPT, REJECT, UNDECIDED


def _setup(constraints=F.CONSTRAINTS, levels=True):
  dom = F.make_domain(constraints)
  parts = acq._cp_parts(dom, F.make_kernel())
  return dom, parts, compile_filter(dom, parts, levels=levels)


def _random_rows(parts, m, seed):
  np.random.seed(seed)
  _, draws = acq.draw_cp_candidates(parts, m)
  return acq._level_rows(draws), draws


def test_orderings_match_the_reference():
  g = load_golden('cp_constrained')
  import json
  assert json.loads(str(g['orderings'])) == F.ORDERINGS
  assert json.loads(str(g['types'])) == [d.get_type() for d in F.make_domain().list_of_domains]


def test_probe_column_map_equals_get_raw_point():
  dom, parts, _ = _setup()
  cmap = column_map(dom, parts)
  assert {k: (v.cols, v.vector, v.kind) for k, v in cmap.items()} == {
      'x': ([0, 1], True, 'euclidean'), 'z': ([2], False, 'euclidean'), 'n': ([3], False, 'integral'),
      'c': ([4], False, 'prod_discrete'), 'w': ([5], False, 'prod_discrete_numeric')}
  rows, draws = _random_rows(parts, 20, 3)
  for i in range(20):
    raw = dom.get_raw_point(acq.point_from_draws(parts, draws, i))
    assert list(raw[0]) == list(rows[i, 0:2]) and raw[1] == rows[i, 2] and raw[2] == rows[i, 3]
    assert raw[3] == np.array(['a', 'b', 'c'])[int(rows[i, 4])] and raw[4] == [0.5, 1.0, 2.0, 4.0][int(rows[i, 5])]


def test_residue_routing():
  _, _, f = _setup(F.CONSTRAINTS + ['math.sqrt(z) > 0', 'x * 2 <= 1', 'n and z', 'undefined_name < 1',
                                   'np.cos(z) < 1', 'dc2.py'.replace('.py', '') + ' > 0'])
  assert f.n_compiled == 4
  assert f.residue == [4, 5, 6, 7, 8, 9, 10]


def test_mirror_constraint_checks_bool_results():
  dom = F.make_domain(['z + 1'])
  with pytest.raises(ValueError):
    dom.constraints_are_satisfied([np.array([0.1, 0.2, 0.3]), np.array([1]), ['a'], [0.5]])
  assert not F.make_domain(None).has_constraints()


@pytest.mark.parametrize('name', sorted(F.PROGRAMS))
def test_decided_statuses_agree_with_the_domain(name):
  dom, parts, f = _setup(F.PROGRAMS[name])
  assert f.n_compiled == len(F.PROGRAMS[name]) and not f.residue
  m = 20000 if name != 'fixture' else 100000
  rows, draws = _random_rows(parts, m, 5)
  st = CR.status(f, rows)
  if name in ('exact', 'fixture'):
    assert not np.any(st == UNDECIDED)
  check = np.random.RandomState(0).choice(m, 4000, replace=False) if m > 4000 else np.arange(m)
  for i in check:
    if st[i] != UNDECIDED:
      assert (st[i] == ACCEPT) == dom.constraints_are_satisfied(acq.point_from_draws(parts, draws, i)), i


@pytest.mark.parametrize('name', sorted(F.PROGRAMS))
def test_rows_on_and_near_the_constraint_surface(name):
  """ Rows exactly on a linear surface and 1 ulp either side: decided rows still agree with the domain. """
  dom, parts, f = _setup(F.PROGRAMS[name])
  rows, draws = _random_rows(parts, 3000, 9)
  rows[:1000, 0] = 0.25 - rows[:1000, 1] * rows[:1000, 2] + rows[:1000, 3] / 3     # 'exact'[0] on its surface
  rows[1000:2000, 0] = np.nextafter(rows[:1000, 0], 2.0)
  rows[2000:, 2] = 1.5 - np.sqrt(rows[2000:, 0] ** 2 + rows[2000:, 1] ** 2)          # 'fixture'[0] on its surface
  st = CR.status(f, rows)
  for i in range(0, 3000, 7):
    if st[i] == UNDECIDED or not (0 <= rows[i, 0] <= 1 and -1 <= rows[i, 2] <= 2):
      continue
    pt = [rows[i, 0:3].copy(), draws[1][i], [np.array(['a', 'b', 'c'])[int(rows[i, 4])]],
          [np.array([0.5, 1.0, 2.0, 4.0])[int(rows[i, 5])]]]
    assert (st[i] == ACCEPT) == dom.constraints_are_satisfied(pt), (name, i)


def test_hamming_keyed_tables_match_level_keyed():
  _, parts_l, fl = _setup(levels=True)
  _, parts_c, fc = _setup(levels=False)
  rows, draws = _random_rows(parts_l, 5000, 13)
  coded = acq.draw_cp_candidates
  np.random.seed(13)
  crow, _ = coded(parts_c, 5000)
  np.testing.assert_array_equal(CR.status(fl, rows), CR.status(fc, crow))


@pytest.mark.parametrize('k', range(5))
def test_constrained_draw_reproduces_the_reference(k):
  g = load_golden('cp_constrained')
  pts, total, run = F.run_case(g, k)
  assert total == run['count']
  assert [F.jval(p) for p in pts] == run['points']
  F.check_state(g, k)


def test_fixture_covers_the_rules():
  import json
  runs = json.loads(str(load_golden('cp_constrained')['runs']))
  assert any(r['count'] > r['M'] for r in runs)                # the maximiser keeps more than M
  assert any(r['kind'] == 'sample' and r['count'] < r['M'] for r in runs)     # ten rounds did not fill M


def test_nothing_accepted_warns_and_raises():
  dom, parts, f = _setup(['z > 5'])
  np.random.seed(0)
  with pytest.warns(UserWarning), pytest.raises(ValueError):
    acq.constrained_rand_draw(parts, 3, F.oracle_keep_round(parts, f))


def test_host_ga_runs_and_device_ga_is_refused():
  a = Namespace(domain=F.make_domain(), max_evals=30, acq_opt_method='ga', t=5, handle_parallel='halluc',
                eval_points_in_progress=[], is_mf=False)
  np.random.seed(2)
  pt = acq._cp_other_maximiser(lambda pts: np.array([float(p[0][1]) for p in pts]), a)
  assert a.domain.constraints_are_satisfied(pt)

  class _GP(object):
    kernel = F.make_kernel()
  a.candidate_rng = 'device'
  with pytest.raises(NotImplementedError):
    acq._cp_other_maximiser(lambda pts: np.zeros(len(pts)), a, _GP(), object())


def test_ga_pool_reproduces_the_reference():
  import json
  from dragonfly_b200 import ga
  g = load_golden('cp_constrained')
  dom = F.make_domain()
  parts = acq._cp_parts(dom, F.make_kernel())
  np.random.seed(31)
  pool = ga.draw_constrained_pool(parts, dom, 17)
  assert [F.jval(p) for p in pool] == json.loads(str(g['pool']))
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['pool_state'])
  assert st[2] == int(g['pool_pos'])


def test_ga_mutations_are_filtered_by_the_constraints():
  from dragonfly_b200 import ga
  dom = F.make_domain()
  parts = acq._cp_parts(dom, F.make_kernel())
  np.random.seed(4)
  pool = ga.draw_constrained_pool(parts, dom, 20)
  vals = np.arange(len(pool), dtype=np.float64)
  for _ in range(20):
    for pt in ga.mutation_epoch(parts, pool, vals, dom):
      assert ga.is_a_member(parts, pt) and dom.constraints_are_satisfied(pt)
  val, pt = ga.ga_maximise(lambda pts: np.array([float(p[0][0]) for p in pts]), parts, 40, domain=dom)
  assert dom.constraints_are_satisfied(pt)


def test_settlement_stops_at_need():
  dom, parts, f = _setup(F.CONSTRAINTS)          # the callable is residue: every accepted row goes to the host
  assert f.residue == [4]
  rows, draws = _random_rows(parts, 2000, 17)
  calls = []

  def point_of(i):
    calls.append(i)
    return acq.point_from_draws(parts, draws, i)
  full = f.settle(CR.status(f, rows), lambda i: acq.point_from_draws(parts, draws, i))
  part = f.settle(CR.status(f, rows), point_of, need=5)
  first = np.flatnonzero(full == ACCEPT)[:5]
  np.testing.assert_array_equal(np.flatnonzero(part == ACCEPT), first)
  assert max(calls) == first[-1]


def test_impure_and_placeholder_subexpressions_stay_exact():
  st0 = np.random.get_state()[1].copy()
  _, _, f = _setup(["z < np.random.rand()", "c == 'a' or z < np.random.random()"])
  assert f.residue == [0, 1]
  np.testing.assert_array_equal(np.random.get_state()[1], st0)   # nothing drawn at compile time
  _, parts, f = _setup(['w ** 2 >= 1 or z > 5'])
  rows, _ = _random_rows(parts, 10, 1)
  rows[:, 5] = np.nan                            # no level: the lookup is unknown, and so is its power
  assert np.all(CR.status(f, rows) == UNDECIDED)


def test_op_codes_and_layout_match_the_header():
  import ctypes as C
  import os
  import re
  from dragonfly_b200 import _lib
  from dragonfly_b200.constraints import OPS
  src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'dfb200.h')).read()
  ops = dict((k.lower(), int(v)) for k, v in re.findall(r'#define\s+DFB_CONS_OP_([A-Z]+)\s+(\d+)', src))
  assert ops == {name: k for k, name in enumerate(OPS)}
  consts = dict((k, int(v)) for k, v in re.findall(r'#define\s+(DFB_CONS_[A-Z_]+)\s+(\d+)\b', src))
  assert consts['DFB_CONS_N_OPS'] == len(OPS)
  for name in ('DFB_CONS_MAX_OPS', 'DFB_CONS_MAX_STACK', 'DFB_CONS_MAX_TAB', 'DFB_CONS_MAX_VEC', 'DFB_CONS_REJECT',
               'DFB_CONS_ACCEPT', 'DFB_CONS_UNDECIDED'):
    assert getattr(_lib, name) == consts[name], name
  n, t = consts['DFB_CONS_MAX_OPS'], consts['DFB_CONS_MAX_TAB']
  assert C.sizeof(_lib.ConsProg) == 16 + 3 * 4 * n + 8 * n + 2 * 8 * t
