"""
Thompson sampling on Cartesian-product domains on the host (no GPU): the one-call normal draw that replaces the
reference's one draw per candidate, the NumPy oracle of the marginal draw against the unmodified reference (golden
cp_ts.npz), and the routing and refusals of asy_ts.
"""
import json
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import cp_ts_ref as T
import hamming_ref as R

from dragonfly_b200 import domains
from dragonfly_b200 import kernel as K
from dragonfly_b200 import cartesian_product_gp as cp
from dragonfly_b200 import gpb_acquisitions as acq


# ---- np.random.normal(size=M) == M calls of normal(size=(1, 1)) ------------------------------------------------
@pytest.mark.parametrize('M', [1, 2, 7, 1000, 1001])
@pytest.mark.parametrize('cached', [False, True])
def test_one_normal_call_equals_one_call_per_candidate(M, cached):
  np.random.seed(123)
  if cached:
    np.random.normal()                        # leaves the second normal of a pair cached
  assert np.random.get_state()[3] == (1 if cached else 0)
  start = np.random.get_state()
  many = np.array([np.random.normal(size=(1, 1))[0, 0] for _ in range(M)])
  after_many = np.random.get_state()
  np.random.set_state(start)
  one = np.random.normal(size=M)
  after_one = np.random.get_state()
  np.testing.assert_array_equal(one, many)
  np.testing.assert_array_equal(after_one[1], after_many[1])
  assert after_one[2:] == after_many[2:]


# ---- the oracle against the reference --------------------------------------------------------------------------
def _golden_setup(g):
  levels, numeric_levels, scale, _, _, _, _, _ = T.golden_problem(g)
  dom = R.make_domain(domains, levels, numeric_levels)
  parts = acq._cp_parts(dom, R.make_kernel(K, cp, scale))
  codes = {}
  return dom, parts, T.oracle_gp(g, codes), codes


def test_golden_selections_are_clear():
  g = load_golden('cp_ts')
  runs = json.loads(str(g['ts_runs']))
  assert [(r['kind'], r['method'], r['halluc']) for r in runs] == [
      ('asy', 'ga', 0), ('asy', 'rand', 0), ('asy', 'ga', 2), ('asy', 'rand', 2), ('syn', 'rand', 0)]
  for r in runs:
    assert min(r['gap']) >= 1e-6
    assert r['m'] == [r['max_evals'] * (4 if r['method'] != 'rand' else 1)] * len(r['m'])


@pytest.mark.parametrize('k', range(5))
def test_oracle_reproduces_the_reference(k):
  g = load_golden('cp_ts')
  run = json.loads(str(g['ts_runs']))[k]
  _, parts, ogp, codes = _golden_setup(g)
  pts, idx = T.run_golden_case(g, k, acq, parts, ogp, codes)
  assert [R.jencode(p) for p in pts] == run['points']
  assert idx == run['index']
  T.check_state(g, k)


# ---- routing and refusals --------------------------------------------------------------------------------------
def _cp_anc(method='ga', max_evals=10, **kw):
  dom = domains.CartesianProductDomain([domains.EuclideanDomain([[0, 1]]), domains.ProdDiscreteDomain([['a', 'b']])])
  a = Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=5, handle_parallel='halluc',
                eval_points_in_progress=[], is_mf=False)
  a.__dict__.update(kw)
  return a


class _FakeGP(object):
  kernel = cp.CartesianProductKernel(1.0, [K.SEKernel(1, 1.0, [1.0]), K.HammingKernel(1)])


def test_cp_domain_routes_to_the_marginal_draw(monkeypatch):
  seen = []
  monkeypatch.setattr(acq, '_cp_ts', lambda gp, a: seen.append((a.acq_opt_method, a.max_evals)) or 'pt')
  a = _cp_anc('ga', 10)
  assert acq.asy_ts(_FakeGP(), a) == 'pt'
  assert acq.asy.ts is acq.asy_ts
  assert acq.asy_ts(_FakeGP(), _cp_anc('rand', 10)) == 'pt'
  assert seen == [('rand', 40), ('rand', 10)]
  assert (a.acq_opt_method, a.max_evals) == ('ga', 10)            # the caller's anc_data is not touched
  assert acq.syn_ts(2, _FakeGP(), _cp_anc('rand', 7)) == ['pt', 'pt']
  assert seen[-2:] == [('rand', 7), ('rand', 7)]


def test_euclidean_ts_is_not_routed(monkeypatch):
  monkeypatch.setattr(acq, '_cp_ts', lambda gp, a: pytest.fail('routed a Euclidean domain'))
  monkeypatch.setattr(acq, '_draw_one_sample', lambda gp, pts, halluc: np.arange(len(pts), dtype=np.float64))
  a = Namespace(domain=domains.EuclideanDomain([[0, 1], [0, 2]]), max_evals=5, acq_opt_method='rand',
                handle_parallel='halluc', eval_points_in_progress=[], is_mf=False)
  np.random.seed(0)
  pt = acq.asy_ts(object(), a)
  np.random.seed(0)
  np.testing.assert_array_equal(pt, acq.draw_candidates([[0, 1], [0, 2]], 5)[4])


def test_refusals(monkeypatch):
  with pytest.raises(NotImplementedError):                      # multi-fidelity
    acq.asy_ts(_FakeGP(), _cp_anc(is_mf=True, eval_fidel_points_in_progress=[]))
  class MFGP(_FakeGP):
    fidel_space_kernel = None
  with pytest.raises(NotImplementedError):
    acq.asy_ts(MFGP(), _cp_anc())
  class Constrained(domains.CartesianProductDomain):
    def has_constraints(self):
      return True
  a = _cp_anc()
  a.domain = Constrained(list(a.domain.list_of_domains))
  with pytest.raises(NotImplementedError):                      # constrained domain
    acq.asy_ts(_FakeGP(), a)
  monkeypatch.setattr(acq, '_shard_info', lambda: (0, 2, None))
  with pytest.raises(NotImplementedError):                      # more than one rank
    acq.asy_ts(_FakeGP(), _cp_anc())
  monkeypatch.setattr(acq, '_shard_info', lambda: (0, 1, None))
  with pytest.raises(ValueError):
    acq.asy_ts(_FakeGP(), _cp_anc(candidate_rng='philox'))
