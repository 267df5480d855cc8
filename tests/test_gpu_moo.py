"""
Parity tests (-m gpu) of the multi-objective acquisitions (SURVEY.md 8f rank 3;
dragonfly/opt/multiobjective_gpb_acquisitions.py:19-125) against tests/golden/moo.npz -- scores and
recommendations of the UNMODIFIED reference -- and against the NumPy oracle on other inputs.
Scores: the scalarisation adds no error of its own, so the (mu, sigma^2) contract carries over
(|d score| <= 1e-9 here); recommendations (arg-max under a seeded RNG) must be identical.
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, domains, device, _lib
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  from oracle import gp_oracle as O
  _lib.load()
  return Namespace(kernel=kernel, gp_core=gp_core, domains=domains, device=device, lib=_lib, torch=torch,
                   moo=moo, O=O)


@pytest.fixture(scope='module')
def case(B):
  g = load_golden('moo')
  gps = [B.gp_core.GP(g['X'], g['Y1'], B.kernel.MaternKernel(6, 2.5, float(g['scale1']), g['bws1']),
                      B.gp_core.ConstantMean(float(g['mean1'])), float(g['noise1'])),
         B.gp_core.GP(g['X'], g['Y2'], B.kernel.SEKernel(6, float(g['scale2']), g['bws2']),
                      B.gp_core.ConstantMean(float(g['mean2'])), float(g['noise2']))]
  return g, gps


def anc(B, g, max_evals, in_progress=(), method='rand'):
  return Namespace(max_evals=max_evals, t=int(g['t']), domain=B.domains.EuclideanDomain([[0, 1]] * 6),
                   acq_opt_method=method, handle_parallel='halluc', eval_points_in_progress=list(in_progress),
                   is_mf=False, obj_weights=g['weights'], reference_point=list(g['refs']))


def test_scalarised_ucb_scores_match_the_reference(B, case):
  g, gps = case
  beta = B.moo._get_ucb_beta_th(6, int(g['t']))
  assert beta == float(g['beta'])
  for kind, key in [(B.lib.DFB_MOO_LIN_UCB, 'lin_ucb_scores'), (B.lib.DFB_MOO_TCH_UCB, 'tch_ucb_scores')]:
    sc = B.moo._mo_ucb_scores(kind, gps, g['C'], list(g['weights']), list(g['refs']), beta)
    np.testing.assert_allclose(sc, g[key], rtol=0, atol=1e-9)
    assert int(np.argmax(sc)) == int(np.argmax(g[key]))


@pytest.mark.parametrize('name', ['lin_ucb', 'tch_ucb', 'lin_ts', 'tch_ts'])
def test_recommendations_match_the_reference(B, case, name):
  g, gps = case
  np.random.seed(9)
  pt = getattr(B.moo.asy, name)(gps, anc(B, g, 1500 if 'ucb' in name else 300))
  assert (pt == g['e2e_%s_point' % name]).all()
  np.random.seed(9)
  pt_seq = getattr(B.moo.seq, name)(gps, anc(B, g, 1500 if 'ucb' in name else 300))
  assert (pt_seq == pt).all()


def test_ts_with_evaluations_in_progress(B, case):
  g, gps = case
  np.random.seed(9)
  pt = B.moo.asy.lin_ts(gps, anc(B, g, 300, in_progress=list(g['Xh'])))
  assert (pt == g['e2e_lin_ts_halluc_point']).all()


def test_combine_kernel_against_oracle_with_edge_values(B, case):
  """ dfb_moo_score_argmax alone on synthetic vectors: three objectives, NaN / inf entries, ties, more
      candidates than one scoring chunk -- np.minimum's NaN propagation and np.argmax's NaN-first /
      first-index-on-ties order. """
  g, gps = case
  post = gps[0]._post
  rs = np.random.RandomState(3)
  m = 40000
  mus = [rs.randn(m) for _ in range(3)]
  sds = [np.abs(rs.randn(m)) + 0.1 for _ in range(3)]
  w, refs, beta = [0.5, 0.3, 0.2], [0.1, -0.2, 0.05], 1.7
  O = B.O
  want = {B.lib.DFB_MOO_LIN_UCB: O.moo_lin_ucb(mus, sds, w, beta),
          B.lib.DFB_MOO_TCH_UCB: O.moo_tch_ucb(mus, sds, w, refs, beta),
          B.lib.DFB_MOO_LIN_VAL: O.moo_lin_vals(mus, w),
          B.lib.DFB_MOO_TCH_VAL: O.moo_tch_vals(mus, w, refs)}
  for kind, ref in want.items():
    ucb = kind in (B.lib.DFB_MOO_LIN_UCB, B.lib.DFB_MOO_TCH_UCB)
    best, idx, sc = post.moo_score_argmax(kind, mus, sds if ucb else None, w, refs, beta, want_scores=True)
    sc = sc.cpu().numpy()
    assert (sc == ref).all()                      # same operations in the same order: bit-identical
    assert idx == int(np.argmax(ref)) and best == ref[idx]
  # ties -> first index; NaN -> counts as the maximum, first NaN wins
  v = [np.zeros(1000), np.zeros(1000)]
  v[0][[17, 400]] = 2.0
  _, idx, _ = post.moo_score_argmax(B.lib.DFB_MOO_LIN_VAL, v, None, [1.0, 1.0])
  assert idx == 17
  v[1][[333, 900]] = np.nan
  for kind in (B.lib.DFB_MOO_LIN_VAL, B.lib.DFB_MOO_TCH_VAL):
    best, idx, sc = post.moo_score_argmax(kind, v, None, [1.0, 1.0], [0.0, 0.0], want_scores=True)
    assert idx == 333 and np.isnan(best) and np.isnan(sc.cpu().numpy()[[333, 900]]).all()
  with pytest.raises(B.lib.DfbError):
    post.moo_score_argmax(7, v, None, [1.0, 1.0])
  with pytest.raises(B.lib.DfbError):
    post.moo_score_argmax(B.lib.DFB_MOO_LIN_UCB, v, None, [1.0, 1.0])     # UCB kinds need the sd vectors


def test_three_objectives_at_n2000_against_oracle(B):
  """ Larger posterior (int8 path available but dfb_eval stays fp64), three objectives, oracle (mu, sigma). """
  from dragonfly_b200 import synth_data
  O = B.O
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=1500, n_cand=500)
  X, C = w['X'], w['candidates']
  Ys = [w['Y'], -np.sum((X - 0.3) ** 2, axis=1), np.cos(3 * X[:, 1]) + X[:, 2]]
  k = w['kernel']
  gps, ogps = [], []
  for Y in Ys:
    m0, nv = float(np.median(Y)), 0.01 * float(Y.var())
    gps.append(B.gp_core.GP(X, Y, B.kernel.MaternKernel(6, 2.5, float(Y.var()), k['dim_bandwidths']),
                            B.gp_core.ConstantMean(m0), nv))
    ogps.append(O.OGP(X, Y, O.OMaternKernel(6, 2.5, float(Y.var()), k['dim_bandwidths']),
                      (lambda c: (lambda x: np.array([c] * len(x))))(m0), nv))
  weights, refs = [0.5, 0.3, 0.2], [0.0, -1.5, 0.2]
  beta = O.moo_ucb_beta_th(6, 1500)
  mus, vars_ = zip(*[O.eval_std_diag(og, C) for og in ogps])
  sds = [np.sqrt(v) for v in vars_]
  lin = O.moo_lin_ucb(mus, sds, weights, beta)
  tch = O.moo_tch_ucb(mus, sds, weights, refs, beta)
  got_lin = B.moo._mo_ucb_scores(B.lib.DFB_MOO_LIN_UCB, gps, C, weights, refs, beta)
  got_tch = B.moo._mo_ucb_scores(B.lib.DFB_MOO_TCH_UCB, gps, C, weights, refs, beta)
  np.testing.assert_allclose(got_lin, lin, rtol=0, atol=1e-8)
  np.testing.assert_allclose(got_tch, tch, rtol=0, atol=1e-7)
  assert int(np.argmax(got_lin)) == int(np.argmax(lin)) and int(np.argmax(got_tch)) == int(np.argmax(tch))
