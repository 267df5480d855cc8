"""
The `ga` acquisition maximiser of Cartesian-product domains on the host (no GPU): the parity restatement
(dragonfly_b200.ga) scored by the NumPy oracle against the unmodified reference (golden cp_ga.npz), the latin-hc initial
pool's use of the MT19937 stream, the routing of 'ga' / 'ga-pdoo' / 'ga-direct', and the reference's exceptions.
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import cp_ga_ref as T
import hamming_ref as R

from dragonfly_b200 import domains
from dragonfly_b200 import ga
from dragonfly_b200 import kernel as K
from dragonfly_b200 import cartesian_product_gp as cp
from dragonfly_b200 import gpb_acquisitions as acq


# ---- the restatement against the reference ---------------------------------------------------------------------
def test_golden_selections_are_clear():
  g = load_golden('cp_ga')
  names = [(r['name'], r['method'], r['halluc']) for r in T.runs(g)]
  assert names == [('ucb', 'ga', 0), ('ucb', 'ga', 2), ('ei', 'ga', 0), ('ei', 'ga', 2), ('pi', 'ga', 0), ('pi', 'ga', 2),
                   ('ttei', 'ga', 0), ('ttei', 'ga', 2), ('syn_ei', 'ga', 0), ('ei', 'ga-pdoo', 0),
                   ('mo_lin_ucb', 'ga', 0)]
  for r in T.runs(g):
    assert r['margin'] >= 1e-9
    assert all(c == (r['max_evals'] // (2 if r['name'] == 'ttei' and len(r['calls']) == 2 else 1)) + 1
               for c in r['calls'])


@pytest.mark.parametrize('k', range(11))
def test_oracle_restatement_reproduces_the_reference(k):
  g = load_golden('cp_ga')
  run = T.runs(g)[k]
  pts, logs = T.replay(g, k)
  ref_calls, ref_vals = T.golden_log(g, k)
  assert [len(c) for c in ref_calls] == [len(p) for p, _ in logs] == run['calls']
  for (pts_k, _), ref_k in zip(logs, ref_calls):
    assert [R.jencode(p) for p in pts_k] == [R.jencode(p) for p in ref_k]      # every point, in order, with its types
  np.testing.assert_allclose(np.concatenate([v for _, v in logs]), ref_vals, rtol=0, atol=1e-9)
  assert [R.jencode(p) for p in pts] == run['points']
  T.check_state(g, k)


# ---- the latin-hc initial pool ---------------------------------------------------------------------------------
def _ref_latin_hc_indices(dim, num_samples):
  """ oper_utils.py:286-296 as written """
  index_set = [list(range(num_samples))] * dim
  lhs_indices = []
  for i in range(num_samples):
    curr_idx_idx = np.random.randint(num_samples - i, size=dim)
    curr_idx = [index_set[j][curr_idx_idx[j]] for j in range(dim)]
    index_set = [index_set[j][:curr_idx_idx[j]] + index_set[j][curr_idx_idx[j] + 1:] for j in range(dim)]
    lhs_indices.append(curr_idx)
  return lhs_indices


@pytest.mark.parametrize('dim,n', [(1, 2), (2, 5), (3, 22), (1, 750)])
def test_latin_hc_consumes_the_stream_like_the_reference(dim, n):
  np.random.seed(5)
  ref_idx = _ref_latin_hc_indices(dim, n)
  ref_u = np.random.random((n, dim))
  after_ref = np.random.get_state()
  np.random.seed(5)
  pts = ga.latin_hc_sampling(dim, n)
  after = np.random.get_state()
  lower = np.linspace(0, 1, n + 1)[:n]
  ref = np.array([[lower[i] for i in row] for row in ref_idx]) + (lower[1] - lower[0]) * ref_u
  np.testing.assert_array_equal(pts, ref)
  np.testing.assert_array_equal(after[1], after_ref[1])
  assert after[2:] == after_ref[2:]
  assert sorted(np.floor(pts[:, 0] * n).astype(int)) == list(range(n))


def test_initial_pool_points_have_the_reference_types():
  dom = R.make_domain(domains, [['a', 'b'], ['c'], ['d', 'e', 'f']], [[0.5, 1.0, 2.0, 4.0]])
  np.random.seed(3)
  pool = ga.draw_cp_initial_pool(acq._cp_parts(dom), 7)
  assert len(pool) == 7
  for e, i, c, n in pool:
    assert e.dtype == np.float64 and i.dtype == np.int64 and isinstance(c[0], np.str_) and isinstance(n[0], np.float64)
    assert ga.is_a_member(acq._cp_parts(dom), [e, i, c, n])


# ---- routing ---------------------------------------------------------------------------------------------------
def _anc(method, max_evals=40, **kw):
  dom = R.make_domain(domains, [['a', 'b', 'c'], ['w', 'x'], ['p', 'q']], [[0.5, 1.0, 2.0]])
  a = Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=5, handle_parallel='halluc',
                eval_points_in_progress=[], is_mf=False)
  a.__dict__.update(kw)
  return a


def _score(pts):
  return np.array([np.sin(3 * p[0][0]) + 0.1 * p[1][0] + (p[2][0] == 'b') + 0.1 * p[3][0] for p in pts])


@pytest.mark.parametrize('method', ['ga', 'ga-pdoo', 'ga-direct', 'GA'])
def test_routing_runs_the_restatement(method, monkeypatch):
  a = _anc(method)
  before = dict(vars(a))
  seen = []
  real = ga.maximise
  monkeypatch.setattr(ga, 'maximise', lambda score, parts, m, B, log=None: seen.append((m, B)) or real(score, parts,
                                                                                                      m, B))
  monkeypatch.setattr(acq, '_reference_fortran_direct_available', lambda: False)
  np.random.seed(0)
  pt = acq._cp_other_maximiser(_score, a)
  assert seen == [(method.lower(), 40)] and vars(a) == before                # the caller's anc_data is not touched
  assert ga.is_a_member(acq._cp_parts(a.domain), pt)
  np.random.seed(0)
  assert R.jencode(real(_score, acq._cp_parts(a.domain), method, 40)) == R.jencode(pt)


def test_follow_up_keeps_the_larger_value():
  parts = acq._cp_parts(_anc('ga').domain)
  np.random.seed(1)
  val, pt = ga.ga_maximise(_score, parts, 40)
  np.random.seed(1)
  state = np.random.get_state()
  pt2 = ga.maximise(_score, parts, 'ga-pdoo', 40)
  assert _score([pt2])[0] >= val
  assert [list(x) for x in pt2[1:]] == [list(x) for x in pt[1:]]      # only the Euclidean part moves
  np.random.set_state(state)
  assert R.jencode(ga.maximise(_score, parts, 'ga', 40)) == R.jencode(pt)


class _FakeGP(object):

  def __init__(self):
    self.kernel = cp.CartesianProductKernel(1.0, [K.SEKernel(2, 1.0, [1.0, 1.0]), K.MaternKernel(1, 2.5, 1.0, [1.0]),
                                                  K.HammingKernel(2), K.MaternKernel(1, 1.5, 1.0, [1.0])])


def test_refusals(monkeypatch):
  class Constrained(domains.CartesianProductDomain):
    def has_constraints(self):
      return True
  a = _anc('ga')
  a.domain = Constrained(list(a.domain.list_of_domains))
  with pytest.raises(NotImplementedError):
    acq._cp_other_maximiser(_score, a)
  with pytest.raises(NotImplementedError):
    acq._cp_other_maximiser(_score, _anc('ga-rand'))
  monkeypatch.setattr(acq, '_shard_info', lambda: (0, 2, None))
  with pytest.raises(NotImplementedError):
    acq._cp_other_maximiser(_score, _anc('ga'))
  with pytest.raises(NotImplementedError):
    acq._cp_other_maximiser(_score, _anc('ga'), _FakeGP(), object())


# ---- the reference's exceptions --------------------------------------------------------------------------------
def test_promoted_category_fails_the_membership_assertion():
  """ [1, 'x'] draws '1', which is not a member of the domain: the reference asserts at its first evaluation """
  dom = R.make_domain(domains, [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]])
  parts = acq._cp_parts(dom)
  np.random.seed(0)
  pool = ga.draw_cp_initial_pool(parts, 7)                 # budget 100: init_capital 7.5, pools of 7
  assert [pt[2][1] for pt in pool].count(np.str_('1')) > 0
  np.random.seed(0)
  scored = []
  with pytest.raises(AssertionError):
    ga.ga_maximise(lambda pts: scored.append(pts) or _score(pts), parts, 100)
  assert scored == []


def test_device_oracle_rows_are_members_and_repeat():
  kern = cp.CartesianProductKernel(1.0, [K.SEKernel(2, 1.0, [1.0, 1.0]), K.MaternKernel(1, 2.5, 1.0, [1.0]),
                                         K.HammingKernel(3), K.MaternKernel(1, 1.5, 1.0, [1.0])])
  parts = acq._cp_parts(_anc('ga').domain, kern)
  desc = ga.device_desc(parts)
  score = lambda rows: _score([acq._cp_point_from_device_row(parts, r) for r in rows])
  _, n_pool, n_total = ga.ga_budget(parts, 60)
  outs = [T.device_ga(score, desc, 1234, n_pool, n_total, *T.philox_rng(1234)) for _ in range(2)]
  rows, vals, _ = outs[0]
  np.testing.assert_array_equal(rows, outs[1][0])
  assert rows.shape == (n_total, desc.d) and len(vals) == n_total
  for r in rows:
    assert ga.is_a_member(parts, acq._cp_point_from_device_row(parts, r))


def test_mutation_exceptions():
  parts = acq._cp_parts(R.make_domain(domains, [['a'], [1, 'x'], ['p']], [[0.5]]))
  pd = parts[2]
  np.random.seed(0)
  with pytest.raises(ValueError):                   # np.random.choice([]) on a coordinate with one level
    for _ in range(20):
      ga.mutate_part(pd, [np.str_('a'), np.str_('x'), np.str_('p')])
  with pytest.raises(ValueError):                   # list.remove of the promoted '1'
    for _ in range(20):
      ga.mutate_part(pd, [np.str_('a'), np.str_('1'), np.str_('p')])


def test_fifty_one_failed_tries(monkeypatch):
  parts = acq._cp_parts(_anc('ga').domain)
  monkeypatch.setattr(ga, 'is_a_member', lambda parts, pt: False)
  np.random.seed(0)
  pool = ga.draw_cp_initial_pool(parts, 6)
  with pytest.raises(ValueError, match='despite 51 tries'):
    ga.mutation_epoch(parts, pool, _score(pool))
