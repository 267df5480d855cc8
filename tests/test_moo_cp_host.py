"""
The multi-objective acquisitions on Cartesian-product domains on the host (no GPU): the (M, K) normal draw that replaces
the reference's one draw per candidate and objective, the NumPy oracle against the unmodified reference (golden
moo_cp.npz), and the routing and refusals of mo_*_asy_ucb / mo_*_asy_ts.
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import moo_cp_ref as T
import hamming_ref as R

from dragonfly_b200 import _lib
from dragonfly_b200 import domains
from dragonfly_b200 import kernel as K
from dragonfly_b200 import cartesian_product_gp as cp
from dragonfly_b200 import gpb_acquisitions as acq
from dragonfly_b200 import multiobjective_gpb_acquisitions as moo


# ---- np.random.normal(size=(M, K)) == M x K calls of normal(size=(1, 1)), candidate-major ------------------------
@pytest.mark.parametrize('M', [1, 2, 7, 1001])
@pytest.mark.parametrize('n_obj', [1, 2, 3])
@pytest.mark.parametrize('cached', [False, True])
def test_one_normal_call_equals_one_call_per_candidate_and_objective(M, n_obj, cached):
  np.random.seed(321)
  if cached:
    np.random.normal()                        # leaves the second normal of a pair cached
  assert np.random.get_state()[3] == (1 if cached else 0)
  start = np.random.get_state()
  many = np.array([[np.random.normal(size=(1, 1))[0, 0] for _ in range(n_obj)] for _ in range(M)])
  after_many = np.random.get_state()
  np.random.set_state(start)
  one = np.random.normal(size=(M, n_obj))
  after_one = np.random.get_state()
  np.testing.assert_array_equal(one, many)
  np.testing.assert_array_equal(after_one[1], after_many[1])
  assert after_one[2:] == after_many[2:]


# ---- the oracle against the reference --------------------------------------------------------------------------
def _golden_setup(g):
  levels, numeric_levels, _, _, metas, H = T.golden_problem(g)
  dom = R.make_domain(domains, levels, numeric_levels)
  parts = acq._cp_parts(dom, R.make_kernel(K, cp, metas[0][0]))
  codes = {}
  return dom, parts, T.oracle_gps(g, codes), codes, H


def test_golden_selections_are_clear():
  g = load_golden('moo_cp')
  runs = T.runs(g)
  assert [(r['name'], r['method'], r['halluc']) for r in runs] == [
      ('lin_ucb', 'rand', 0), ('tch_ucb', 'rand', 0),
      ('lin_ts', 'ga', 0), ('lin_ts', 'rand', 0), ('lin_ts', 'ga', 2), ('lin_ts', 'rand', 2),
      ('tch_ts', 'ga', 0), ('tch_ts', 'rand', 0), ('tch_ts', 'ga', 2), ('tch_ts', 'rand', 2)]
  for r in runs:
    assert r['gap'] >= 1e-6
    assert r['m'] == T.run_size(r)


def test_oracle_ucb_scores_match_the_reference():
  g = load_golden('moo_cp')
  dom, _, ogps, codes, _ = _golden_setup(g)
  assert moo._get_ucb_beta_th(dom.dim, int(g['t'])) == float(g['beta'])
  C = R.encode_points(R.golden_points(g, 'C'), codes)
  for name in ('lin_ucb', 'tch_ucb'):
    s = T.oracle_scores(ogps, name, C, list(g['weights']), list(g['refs']), float(g['beta']))
    np.testing.assert_allclose(s, g[name + '_scores'], rtol=0, atol=1e-9)
    assert int(np.argmax(s)) == int(np.argmax(g[name + '_scores']))


@pytest.mark.parametrize('k', range(10))
def test_oracle_reproduces_the_reference(k):
  g = load_golden('moo_cp')
  run = T.runs(g)[k]
  _, parts, ogps, codes, H = _golden_setup(g)
  np.random.seed(run['seed'])
  pt, idx, _ = T.oracle_run(ogps, acq, parts, run['name'], T.run_size(run), H[:run['halluc']], codes,
                            list(g['weights']), list(g['refs']), float(g['beta']))
  assert R.jencode(pt) == run['point']
  assert idx == run['index']
  T.check_state(g, k)


# ---- routing and refusals --------------------------------------------------------------------------------------
def _cp_anc(method='ga', max_evals=10, **kw):
  dom = domains.CartesianProductDomain([domains.EuclideanDomain([[0, 1]]), domains.ProdDiscreteDomain([['a', 'b']])])
  a = Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=5, handle_parallel='halluc',
                eval_points_in_progress=[], is_mf=False, obj_weights=[0.5, 0.5], reference_point=[0.0, 0.0])
  a.__dict__.update(kw)
  return a


class _FakeGP(object):

  def __init__(self):
    self.kernel = cp.CartesianProductKernel(1.0, [K.SEKernel(1, 1.0, [1.0]), K.HammingKernel(1)])


LIN_UCB, TCH_UCB, LIN_VAL, TCH_VAL = _lib.DFB_MOO_LIN_UCB, _lib.DFB_MOO_TCH_UCB, _lib.DFB_MOO_LIN_VAL, _lib.DFB_MOO_TCH_VAL


def test_cp_domain_routes_to_the_device_maximiser(monkeypatch):
  seen = []
  monkeypatch.setattr(moo, '_mo_cp', lambda kind, gps, a, w, refs, beta=0.0:
                      seen.append((kind, a.acq_opt_method, a.max_evals, refs, beta)) or 'pt')
  gps = [_FakeGP(), _FakeGP()]
  a = _cp_anc('ga', 10)
  assert moo.asy.lin_ts(gps, a) == 'pt' and moo.asy.tch_ts(gps, _cp_anc('rand', 10)) == 'pt'
  assert (a.acq_opt_method, a.max_evals) == ('ga', 10)            # the caller's anc_data is not touched
  assert moo.asy.lin_ucb(gps, _cp_anc('rand', 7)) == 'pt' and moo.asy.tch_ucb(gps, _cp_anc('rand', 7)) == 'pt'
  beta = moo._get_ucb_beta_th(2, 5)
  assert seen == [(LIN_VAL, 'rand', 40, None, 0.0), (TCH_VAL, 'rand', 10, [0.0, 0.0], 0.0),
                  (LIN_UCB, 'rand', 7, None, beta), (TCH_UCB, 'rand', 7, [0.0, 0.0], beta)]
  for name in ('lin_ts', 'tch_ts', 'lin_ucb', 'tch_ucb'):
    assert getattr(moo.seq, name) is getattr(moo.asy, name)
  assert not vars(moo.syn)


def test_other_ucb_maximisers_score_list_of_parts_points(monkeypatch):
  seen = []
  def other(acq_fn, a):
    seen.append(a.acq_opt_method)
    return acq_fn
  monkeypatch.setattr(moo, '_cp_other_maximiser', other)
  monkeypatch.setattr(moo, '_mo_cp', lambda *args, **kw: pytest.fail("'rand' only"))
  scored = []
  monkeypatch.setattr(moo, '_mo_cp_ucb_scores', lambda kind, gps, pts, w, refs, beta: scored.append((kind, pts)))
  gps = [_FakeGP(), _FakeGP()]
  for method in ('pdoo', 'direct', 'ga'):
    fn = moo.asy.tch_ucb(gps, _cp_anc(method))
    fn([[np.array([0.5]), ['a']]])
  assert seen == ['pdoo', 'direct', 'ga']
  assert [s[0] for s in scored] == [TCH_UCB] * 3 and scored[0][1] == [[np.array([0.5]), ['a']]]


def test_euclidean_domains_are_not_routed(monkeypatch):
  monkeypatch.setattr(moo, '_mo_cp', lambda *args, **kw: pytest.fail('routed a Euclidean domain'))
  monkeypatch.setattr(moo, '_draw_one_sample', lambda gp, pts, halluc: np.arange(len(pts), dtype=np.float64))

  class _Post(object):
    def moo_score_argmax(self, kind, a_list, b_list, weights, refs=None, beta=0.0, want_scores=False):
      return float(a_list[0][-1]), len(a_list[0]) - 1, None

  class _GP(object):
    _post = _Post()
  a = Namespace(domain=domains.EuclideanDomain([[0, 1], [0, 2]]), max_evals=5, acq_opt_method='rand',
                handle_parallel='halluc', eval_points_in_progress=[], is_mf=False, obj_weights=[1.0, 1.0],
                reference_point=[0.0, 0.0])
  np.random.seed(0)
  pt = moo.asy.lin_ts([_GP(), _GP()], a)
  np.random.seed(0)
  np.testing.assert_array_equal(pt, acq.draw_candidates([[0, 1], [0, 2]], 5)[4])


def test_refusals(monkeypatch):
  gps = [_FakeGP(), _FakeGP()]
  for name in ('lin_ts', 'lin_ucb'):
    fn = getattr(moo.asy, name)
    with pytest.raises(NotImplementedError):                    # n_obj outside 1 .. DFB_MOO_MAX_OBJ
      fn([], _cp_anc('rand'))
    with pytest.raises(NotImplementedError):
      fn([_FakeGP() for _ in range(_lib.DFB_MOO_MAX_OBJ + 1)], _cp_anc('rand'))
    with pytest.raises(NotImplementedError):                    # multi-fidelity
      fn(gps, _cp_anc('rand', is_mf=True, eval_fidel_points_in_progress=[]))
    class MFGP(_FakeGP):
      fidel_space_kernel = None
    with pytest.raises(NotImplementedError):
      fn([_FakeGP(), MFGP()], _cp_anc('rand'))
    class Constrained(domains.CartesianProductDomain):
      def has_constraints(self):
        return True
    a = _cp_anc('rand')
    a.domain = Constrained(list(a.domain.list_of_domains))
    with pytest.raises(NotImplementedError):                    # constrained domain
      fn(gps, a)
    bad = _FakeGP()
    bad.kernel = cp.CartesianProductKernel(1.0, [K.SEKernel(1, 1.0, [1.0]), K.SEKernel(1, 1.0, [1.0])])
    with pytest.raises(NotImplementedError):                    # a prod_discrete part without a Hamming factor
      fn([_FakeGP(), bad], _cp_anc('rand'))
    monkeypatch.setattr(moo, '_shard_info', lambda: (0, 2, None))
    with pytest.raises(NotImplementedError):                    # more than one rank
      fn(gps, _cp_anc('rand'))
    monkeypatch.setattr(moo, '_shard_info', lambda: (0, 1, None))
