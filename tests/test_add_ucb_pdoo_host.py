"""
Add-UCB with the sequential maximisers on the host side (no GPU): the lock-step PDOO driver of dragonfly_b200/doo.py
against independent per-group searches, scored by the NumPy oracle, and the routing of _add_ucb_groups by
acq_opt_method.
"""
from argparse import Namespace

import numpy as np
import pytest

from dragonfly_b200 import doo
from dragonfly_b200 import gpb_acquisitions as A
from dragonfly_b200.domains import EuclideanDomain
from oracle import gp_oracle as O

GROUPS = [[0, 1, 2], [3], [4, 5, 6, 7]]


def _oracle_gp(n=120, seed=3):
  rs = np.random.RandomState(seed)
  X = rs.random_sample((n, 8))
  Y = np.sin(3 * X).sum(axis=1) + 0.1 * rs.standard_normal(n)
  kern = O.OAdditiveKernel(0.4, [O.OMaternKernel(3, 2.5, 1.0, [0.4, 0.5, 0.6]), O.OSEKernel(1, 1.0, [0.3]),
                                 O.OMaternKernel(4, 1.5, 1.0, [0.5] * 4)], GROUPS)
  gp = O.OGP(X, Y, kern, lambda x: np.zeros(len(x)), 0.01)
  return gp, kern


def _anc(method, max_evals=300, t=40):
  dom = EuclideanDomain([[0, 1]] * 8)
  return Namespace(curr_acq='add_ucb', max_evals=max_evals, t=t, domain=dom, acq_opt_method=method,
                   domain_bounds=np.array(dom.bounds), handle_parallel='halluc', eval_points_in_progress=[],
                   is_mf=False)


@pytest.mark.parametrize('t', [5, 400])
def test_lockstep_searches_match_independent_searches(t):
  gp, kern = _oracle_gp()
  bounds = [np.array([[0.0, 1.0]] * len(g)) for g in GROUPS]
  bounds[1] = np.array([[-0.5, 2.0]])
  evals = 400 // len(GROUPS)
  calls = []

  def score(requests):
    calls.append([len(X) for _, X in requests])
    return [O.add_ucb_group_scores(gp, kern, j, X, t)[0] for j, X in requests]
  found = doo.pdoo_maximise_lockstep(score, bounds, evals)
  rounds = doo.pdoo_maximise_lockstep.last_rounds
  assert rounds == len(calls)
  assert all(n <= doo.PDOOSearch.PREFETCH_GROUP for c in calls for n in c)
  alone_calls = 0
  for j, (val, pt) in enumerate(found):
    val1, pt1, _ = doo.pdoo_maximise(lambda X: O.add_ucb_group_scores(gp, kern, j, X, t)[0], bounds[j], evals)
    alone = doo.pdoo_maximise.last_search
    s = doo.pdoo_maximise_lockstep.last_searches[j]
    assert val == val1 and (pt == pt1).all()
    assert len(s.query_pts) == len(alone.query_pts)
    assert all((a == b).all() for a, b in zip(s.query_pts, alone.query_pts))
    assert s.query_vals == alone.query_vals
    assert s.num_device_calls == alone.num_device_calls
    alone_calls += alone.num_device_calls
  # one call per round for all groups together, instead of one per group and round
  assert rounds == max(s.num_device_calls for s in doo.pdoo_maximise_lockstep.last_searches)
  assert rounds < alone_calls


def _route(method, monkeypatch, fortran=False):
  """ Runs _add_ucb_groups with recording fakes; returns (maximise_group calls, score_groups requests, delegations). """
  monkeypatch.setattr(A, '_reference_fortran_direct_available', lambda: fortran)
  gp, kern = _oracle_gp(n=60)
  rand_calls, requests, delegated = [], [], []

  def maximise_group(j, acq, anc_j):
    rand_calls.append((j, acq.beta, anc_j.max_evals))
    return np.full(len(GROUPS[j]), 0.5)

  def score_groups(reqs, betas):
    requests.append([(j, np.array(X)) for j, X in reqs])
    return [O.add_ucb_group_scores(gp, kern, j, X, 40)[0] for j, X in reqs]

  def fake_delegate(acq_fn, anc_j, deterministic=True):
    x = np.full((1, anc_j.domain.get_dim()), 0.25)
    delegated.append((anc_j.max_evals, acq_fn(x)))
    return x[0]
  monkeypatch.setattr(A, '_delegate_to_reference_maximiser', fake_delegate)
  pt = A._add_ucb_groups(_anc(method), GROUPS, maximise_group, score_groups)
  assert pt.shape == (8,)
  return rand_calls, requests, delegated


@pytest.mark.parametrize('method', ['pdoo', 'direct'])
def test_pdoo_and_direct_without_fortran_take_the_lockstep_search(method, monkeypatch):
  rand_calls, requests, delegated = _route(method, monkeypatch)
  assert not rand_calls and not delegated
  assert len(requests) == doo.pdoo_maximise_lockstep.last_rounds > 1
  assert {j for r in requests for j, _ in r} == {0, 1, 2}
  assert all(len(X) <= doo.PDOOSearch.PREFETCH_GROUP for r in requests for _, X in r)


def test_direct_with_fortran_delegates_each_group_with_one_point_rows(monkeypatch):
  rand_calls, requests, delegated = _route('direct', monkeypatch, fortran=True)
  assert not rand_calls
  assert len(delegated) == len(GROUPS) and all(e == 300 // len(GROUPS) for e, _ in delegated)
  assert [r[0][0] for r in requests] == [0, 1, 2]
  assert all(len(r) == 1 and r[0][1].shape == (1, len(GROUPS[r[0][0]])) for r in requests)
  assert all(np.shape(v) == (1,) for _, v in delegated)


def test_rand_still_takes_the_fused_maximiser(monkeypatch):
  rand_calls, requests, delegated = _route('rand', monkeypatch)
  assert not requests and not delegated
  assert [j for j, _, _ in rand_calls] == [0, 1, 2]
  assert [b for _, b, _ in rand_calls] == [A._get_add_ucb_beta_th(len(g), 40) for g in GROUPS]
  assert all(e == 100 for _, _, e in rand_calls)


# ---- the reference's own Add-UCB runs with 'pdoo' / 'direct' (tests/golden/add_ucb_pdoo.npz) -------------------------
def golden_oracle_gp(g):
  """ The additive GP of tests/golden/make_golden_add_ucb_pdoo.py in the NumPy oracle. """
  kern = O.OAdditiveKernel(float(g['scale']), [O.OMaternKernel(3, 2.5, 1.0, [0.4, 0.5, 0.6]), O.OSEKernel(1, 1.0, [0.3]),
                                               O.OMaternKernel(4, 1.5, 1.0, [0.5, 0.45, 0.55, 0.6])], GROUPS)
  m0 = float(g['mean_const'])
  return O.OGP(g['X'], g['Y'], kern, lambda x: np.array([m0] * len(x)), float(g['noise_var'])), kern


@pytest.mark.parametrize('case', ['pdoo_t5', 'pdoo_t300', 'direct_t100'])
def test_lockstep_driver_reproduces_the_reference_query_logs(case, monkeypatch):
  from conftest import load_golden
  g = load_golden('add_ucb_pdoo')
  assert float(g[case + '_margin']) >= 1e-9
  gp, kern = golden_oracle_gp(g)
  evals, t = [int(v) for v in g[case + '_args']]
  monkeypatch.setattr(A, '_reference_fortran_direct_available', lambda: False)
  pt = A._add_ucb_groups(_anc(case.split('_')[0], evals, t), GROUPS, None,
                         lambda reqs, betas: [O.add_ucb_group_scores(gp, kern, j, X, t)[0] for j, X in reqs])
  assert (pt == g[case + '_point']).all()
  for j, s in enumerate(doo.pdoo_maximise_lockstep.last_searches):
    qp, qv = g['%s_qpts_%d' % (case, j)], g['%s_qvals_%d' % (case, j)]
    k = len(s.query_vals)                     # recorded up to the budget, as the reference's history is
    assert k == min(len(qv), evals // len(GROUPS) + 1)
    assert (np.array(s.query_pts) == qp[:k]).all()
    np.testing.assert_allclose(s.query_vals, qv[:k], rtol=0, atol=1e-12)


# ---- more groups than one dfb_score_groups call takes ------------------------------------------------------------------
class _LimitedPost(object):
  """ Stands in for DevicePosterior.score_groups: checks the entry's limits, scores row r as a function of its
      group's columns and beta, and records the calls. """

  def __init__(self):
    self.calls = []

  def score_groups(self, descs, betas, X, groups):
    from dragonfly_b200 import _lib
    assert len(descs) <= _lib.DFB_MAX_GROUPS and len(betas) == len(descs)
    assert sum(d.n_slots for d in descs) <= _lib.DFB_MAX_SLOTS
    assert sum(d.n_factors for d in descs) <= _lib.DFB_MAX_FACTORS
    assert set(groups.tolist()) == set(range(len(descs)))          # only the groups present, remapped
    self.calls.append(len(descs))
    return np.array([np.sin(3 * X[r, :descs[g].cand_dim]).sum() + betas[g] * descs[g].cand_dim
                     for r, g in enumerate(groups)])


def _descs(n_groups, dims, dz=0):
  from dragonfly_b200 import kernel as K
  out = []
  for j in range(n_groups):
    parts = [K.SEKernel(dims, 1.0, [0.3] * dims)]
    coords = [list(range(dz, dz + dims))]
    if dz:
      parts.insert(0, K.SEKernel(dz, 1.0, [0.7] * dz))
      coords.insert(0, list(range(dz)))
    out.append(K.build_descriptor(K.CoordinateProductKernel(dz + dims, 1.0, parts, coords), train_dim=dz + dims,
                                  cand_dim=dz + dims))
  return out


@pytest.mark.parametrize('n_groups, dz, per_call', [(60, 0, 48), (30, 1, 24)])
def test_rounds_with_more_groups_than_one_call_takes_are_split(n_groups, dz, per_call, monkeypatch):
  """ 60 one-coordinate groups (> DFB_MAX_GROUPS), and 30 fidelity x domain groups of 2 factors each (BOCA: > 48
      factors): every round is split into calls within the limits, and the values are those of one group per call. """
  monkeypatch.setattr(A, '_reference_fortran_direct_available', lambda: False)
  descs = _descs(n_groups, 1, dz)
  assert all(d.n_factors == 1 + (dz > 0) for d in descs)
  groupings = [[j] for j in range(n_groups)]
  dom = EuclideanDomain([[0, 1]] * n_groups)
  anc = Namespace(curr_acq='add_ucb', max_evals=30 * n_groups, t=40, domain=dom, acq_opt_method='pdoo',
                  domain_bounds=np.array(dom.bounds))
  post = _LimitedPost()
  prefix = np.full(dz, 1.0) if dz else None
  pt = A._add_ucb_groups(anc, groupings, None, A._group_scorer(post, descs, prefix=prefix))
  assert pt.shape == (n_groups,)
  assert max(post.calls) == per_call and len(post.calls) > doo.pdoo_maximise_lockstep.last_rounds
  # the same point with every group alone in its call
  alone = _LimitedPost()
  single = A._group_scorer(alone, descs, prefix=prefix)
  pt1 = A._add_ucb_groups(anc, groupings, None,
                          lambda reqs, betas: [single([r], betas)[0] for r in reqs])
  assert (pt1 == pt).all() and max(alone.calls) == 1
