"""
The `ga` acquisition maximiser of Cartesian-product domains on the device (-m gpu): the public acquisitions (asy_* /
syn_ei / mo_lin_asy_ucb with acq_opt_method 'ga' / 'ga-pdoo') on device CPGPs against the unmodified reference (golden
cp_ga.npz) -- every queried point in order, its value within the device contract, the returned points and the MT19937
states -- plus a 30 000-evaluation budget and repeatability.
"""
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
import cp_ga_ref as T
import moo_cp_ref as MR
import hamming_ref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, cartesian_product_gp, gpb_acquisitions, domains, ga, _lib
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  _lib.load()
  return Namespace(kernel=kernel, cp=cartesian_product_gp, acq=gpb_acquisitions, domains=domains, ga=ga, moo=moo, lib=_lib)


@pytest.fixture(scope='module')
def g():
  return load_golden('cp_ga')


def _golden_gps(G, g):
  dom, _, X, H = T.golden_problem(g)
  gps = []
  for key, yk, make in (('meta', 'Y', R.make_kernel), ('meta2', 'Y2', MR.make_kernel2)):
    scale, noise_var, mean_const = [float(v) for v in g[key]]
    gps.append(G.cp.CPGP(X, list(np.asarray(g[yk])), make(G.kernel, G.cp, scale),
                         (lambda c: (lambda x: np.array([c] * len(x))))(mean_const), noise_var))
  return gps, dom, H


def _anc(g, dom, method, max_evals, halluc):
  return Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=int(g['t']), handle_parallel='halluc',
                   eval_points_in_progress=list(halluc), is_mf=False, curr_max_val=float(g['curr_max']),
                   obj_weights=list(g['weights']), reference_point=list(g['refs']))


def _call(G, g, gps, dom, H, run):
  name, method, B = run['name'], run['method'], run['max_evals']
  if name == 'syn_ei':
    return G.acq.syn.ei(2, gps[0], _anc(g, dom, method, B, []))
  if name == 'mo_lin_ucb':
    return [G.moo.asy.lin_ucb(gps, _anc(g, dom, method, B, []))]
  return [getattr(G.acq.asy, name)(gps[0], _anc(g, dom, method, B, H[:run['halluc']]))]


@pytest.mark.parametrize('k', range(11))
def test_golden_query_logs_points_and_rng_states(G, g, k, monkeypatch):
  gps, dom, H = _golden_gps(G, g)
  run = T.runs(g)[k]
  logs = []
  real = G.ga.ga_maximise

  def logged(score, parts, max_evals, log=None):
    logs.append([])
    return real(score, parts, max_evals, logs[-1])
  monkeypatch.setattr(G.ga, 'ga_maximise', logged)
  np.random.seed(run['seed'])
  pts = _call(G, g, gps, dom, H, run)
  assert [R.jencode(p) for p in pts] == run['points']
  T.check_state(g, k)
  ref_calls, ref_vals = T.golden_log(g, k)
  assert [sum(len(b[0]) for b in log) for log in logs] == run['calls']
  for log, ref in zip(logs, ref_calls):
    assert [R.jencode(p) for b in log for p in b[0]] == [R.jencode(p) for p in ref]
  vals = np.concatenate([b[1] for log in logs for b in log])
  np.testing.assert_allclose(vals, ref_vals, rtol=1e-7, atol=1e-7)


def test_epochs_are_scored_in_batches(G, g, monkeypatch):
  """ one device call for the initial pool and one per epoch of five """
  gps, dom, _ = _golden_gps(G, g)
  sizes = []
  real = G.ga.ga_maximise
  monkeypatch.setattr(G.ga, 'ga_maximise', lambda score, parts, B, log=None: real(
      lambda pts: sizes.append(len(pts)) or score(pts), parts, B, log))
  np.random.seed(4)
  G.acq.asy.ei(gps[0], _anc(g, dom, 'ga', 1000, []))
  assert sizes[0] == 35 and sum(sizes) == 1001 and all(s <= 5 for s in sizes[1:])
  assert len(sizes) >= 1 + (1001 - 35) // 5


def test_large_budget_completes_and_repeats(G, g):
  gps, dom, H = _golden_gps(G, g)
  out = []
  for _ in range(2):
    np.random.seed(21)
    pt = G.acq.asy.ei(gps[0], _anc(g, dom, 'ga', 30000, H[:2]))
    out.append((R.jencode(pt), np.random.get_state()[2]))
  assert out[0] == out[1]
  assert G.ga.is_a_member(G.acq._cp_parts(dom), pt)


def test_logged_points_mu_and_variance_within_the_contract(G, g):
  """ the acquisition values above carry the contract through EI / PI / UCB; here mu and sigma^2 of the logged points
      themselves, device against the oracle: |d mu| <= 1e-10, |d sigma^2| <= 1e-8 """
  from oracle import gp_oracle as O
  gps, dom, H = _golden_gps(G, g)
  codes = {}
  ogp = T.oracle_gps(g, codes)[0]
  for k in (0, 1):
    run = T.runs(g)[k]
    pts = T.golden_log(g, k)[0][0]
    halluc = H[:run['halluc']]
    mu_o, var_o = O.eval_std_diag(ogp, R.encode_points(pts, codes),
                                  R.encode_points(halluc, codes) if len(halluc) else None)
    mu, sd = gps[0].eval_with_hallucinated_observations(pts, halluc, 'std') if len(halluc) else gps[0].eval(pts, 'std')
    np.testing.assert_allclose(mu, mu_o, rtol=0, atol=1e-10)
    np.testing.assert_allclose(np.asarray(sd) ** 2, var_o, rtol=0, atol=1e-8)


# ---- device mode: dfb_ga_maximise against the NumPy oracle fed with the same Philox streams ------------------------
def _device_oracle(G, g, gps, parts, seed, B, halluc, epochs=None):
  codes = {}
  ogps = T.oracle_gps(g, codes)
  score = T.Scorer(g, ogps, codes, 'ei', halluc)
  post = gps[0]._post
  uniform = lambda S, row: post.fill_rng(seed, row, S, 1, G.lib.DFB_RNG_UNIFORM).cpu().numpy()[:, 0]
  normal = lambda S, row: post.fill_rng(seed, row, S, 1, G.lib.DFB_RNG_NORMAL).cpu().numpy()[:, 0]
  _, n_pool, n_total = G.ga.ga_budget(parts, B)
  rows, vals, margin = T.device_ga(lambda rs: score([G.acq._cp_point_from_device_row(parts, r) for r in rs]),
                                   G.ga.device_desc(parts), seed, n_pool, n_total, uniform, normal, epochs)
  return rows, vals, margin, n_pool, n_total


def _seed_of(k):
  np.random.seed(k)
  return (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))


@pytest.mark.parametrize('halluc', [0, 2])
def test_device_mode_rows_values_and_point_match_the_oracle(G, g, halluc):
  gps, dom, H = _golden_gps(G, g)
  parts = G.acq._cp_parts(dom, gps[0].kernel)
  B = 200
  for k in range(40, 80):                        # a seed whose every selection is clear of the 1e-10 / 1e-8 contract
    rows_o, vals_o, margin, n_pool, n_total = _device_oracle(G, g, gps, parts, _seed_of(k), B, H[:halluc])
    if margin >= 1e-9:
      break
  assert margin >= 1e-9
  seed = _seed_of(k)
  from dragonfly_b200.device import make_acq_desc
  acq = make_acq_desc('ei', best=float(g['curr_max']))
  with gps[0]._fused_session(acq, H[:halluc]) as sess:
    val, idx, row, rows, vals = sess.post.ga_maximise(acq, float(g['meta'][2]), G.ga.device_desc(parts), seed, n_pool,
                                                      n_total)
  rows, vals = rows.cpu().numpy(), vals.cpu().numpy()
  np.testing.assert_array_equal(rows, rows_o)                     # every row, the mutated ones too, bit for bit
  np.testing.assert_allclose(vals, vals_o, rtol=0, atol=1e-8)
  assert idx == int(np.argmax(vals_o)) and np.array_equal(row, rows_o[idx])
  np.random.seed(k)
  pt = G.acq.asy.ei(gps[0], Namespace(**dict(vars(_anc(g, dom, 'ga', B, H[:halluc])), candidate_rng='device')))
  assert R.jencode(pt) == R.jencode(G.acq._cp_point_from_device_row(parts, rows_o[int(np.argmax(vals_o))]))


def test_device_mode_large_budget_repeats(G, g):
  gps, dom, H = _golden_gps(G, g)
  out = []
  for _ in range(2):
    np.random.seed(5)
    a = Namespace(**dict(vars(_anc(g, dom, 'ga-pdoo', 30000, H[:2])), candidate_rng='device'))
    pt = G.acq.asy.ei(gps[0], a)
    out.append(R.jencode(pt))
  assert out[0] == out[1]
  assert G.ga.is_a_member(G.acq._cp_parts(dom), pt)
