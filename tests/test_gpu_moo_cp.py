"""
The multi-objective acquisitions on Cartesian-product domains on the device (-m gpu): dfb_moo_score_argmax_ts bit for
bit against the NumPy scalarisation of fl(fl(sd z) + mu) from dfb_eval, against dfb_score_argmax_ts for one objective,
its counter-based normals against dfb_fill_rng, and mo_*_asy_ucb / mo_*_asy_ts against the unmodified reference (golden
moo_cp.npz) and the NumPy oracle (tests/moo_cp_ref.py).
"""
from argparse import Namespace
from copy import copy

import numpy as np
import pytest

from conftest import load_golden
from oracle import gp_oracle as O
import moo_cp_ref as T
import hamming_ref as R

pytestmark = pytest.mark.gpu

SEED = 0x2468_ACE0_1357_9BDF


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, cartesian_product_gp, gpb_acquisitions, domains, device, _lib
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  _lib.load()
  return Namespace(kernel=kernel, cp=cartesian_product_gp, acq=gpb_acquisitions, domains=domains, device=device,
                   lib=_lib, torch=torch, moo=moo)


@pytest.fixture(scope='module')
def g():
  return load_golden('moo_cp')


def _host(v):
  return v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)


# ---- dfb_moo_score_argmax_ts on synthetic posteriors -------------------------------------------------------------
def _mixed_posteriors(G, n, m, seed, n_obj):
  """ n_obj device posteriors on one mixed training set (golden kernels with different scales), m candidate rows """
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = R.make_domain(G.domains, levels, numeric_levels)
  parts = G.acq._cp_parts(dom, R.make_kernel(G.kernel, G.cp, 1.0))
  np.random.seed(seed)
  X, _ = G.acq.draw_cp_candidates(parts, n)
  C, _ = G.acq.draw_cp_candidates(parts, m)
  Ys = [np.sin(3 * X[:, 0]) + 0.3 * X[:, 1] - 0.1 * (X[:, 2] - 3) ** 2 + 0.4 * (X[:, 3] == 1),
        np.cos(2 * X[:, 1]) - 0.5 * X[:, 0] ** 2 + 0.2 * np.log(X[:, 6]),
        0.1 * X[:, 2] + 0.3 * (X[:, 4] == 0) - 0.2 * X[:, 0] * X[:, 1]][:n_obj]
  posts, ogps = [], []
  for k, Y in enumerate(Ys):
    Y = Y + 0.05 * np.random.standard_normal(n)
    scale, mc = 0.8 + 0.3 * k, float(np.mean(Y))
    post = G.device.DevicePosterior(n + 8, chunk=1024)
    post.set_option('score_impl', 0)
    post.set_kernel(G.kernel.build_descriptor(R.make_kernel(G.kernel, G.cp, scale), train_dim=7, cand_dim=7))
    post.set_train(X, Y - mc)
    assert post.build(0.01)[0] == 0
    post.mc = mc
    posts.append(post)
    ogps.append(O.OGP(X, Y, R.oracle_kernel(scale), (lambda c: (lambda x: np.array([c] * len(x))))(mc), 0.01))
  return posts, ogps, C


def _eval_all(G, posts, C):
  Cd = G.torch.from_numpy(C).cuda()
  mus, sds = zip(*[p.eval(Cd, mean_const=p.mc) for p in posts])
  return list(mus), list(sds)


def _vals(name, mus, sds, z, w, refs):
  v = [_host(s) * z[:, k] + _host(mu) for k, (mu, s) in enumerate(zip(mus, sds))]     # one product, one sum: no FMA
  return O.moo_lin_vals(v, w) if name == 'lin' else O.moo_tch_vals(v, w, refs)


def test_ts_scores_bit_for_bit_and_counter_normals_are_fill_rng(G):
  posts, _, C = _mixed_posteriors(G, 600, 20000, 1, 3)           # 20000 rows: several chunks of 1024
  mus, sds = _eval_all(G, posts, C)
  w, refs = [0.5, 0.3, 0.2], [0.1, -0.4, 0.05]
  np.random.seed(2)
  z = np.random.normal(size=(len(C), 3))
  kinds = [('lin', G.lib.DFB_MOO_LIN_VAL), ('tch', G.lib.DFB_MOO_TCH_VAL)]
  for row0 in (0, 777, (1 << 33) + 5):
    zp = _host(posts[0].fill_rng(SEED, row0, 3, len(C)))        # row k: objective k's normals
    for name, kind in kinds:
      for zz, kw in [(z, dict(z=z)), (z, dict(z=G.torch.from_numpy(z).cuda())), (zp.T, dict(seed=SEED, row0=row0))]:
        want = _vals(name, mus, sds, zz, w, refs)
        bs, bi, sc, nonpos = posts[0].moo_score_argmax_ts(kind, mus, sds, w, refs, want_scores=True, **kw)
        np.testing.assert_array_equal(_host(sc), want, err_msg=name)
        assert bi == O.np_argmax_first(want) and bs == want[bi] and nonpos == 0, name
    # a candidate's normals depend on (seed, its global row, objective) only
    _, _, sc, _ = posts[0].moo_score_argmax_ts(kinds[0][1], mus, sds, w, seed=SEED, row0=row0, want_scores=True)
    _, _, sc2, _ = posts[0].moo_score_argmax_ts(kinds[0][1], [v[5000:] for v in mus], [v[5000:] for v in sds], w,
                                                seed=SEED, row0=row0 + 5000, want_scores=True)
    np.testing.assert_array_equal(_host(sc2), _host(sc)[5000:])


def test_one_objective_equals_score_argmax_ts(G):
  posts, _, C = _mixed_posteriors(G, 700, 6000, 5, 1)
  post = posts[0]
  mus, sds = _eval_all(G, posts, C)
  np.random.seed(6)
  z = np.random.normal(size=len(C))
  for kw_moo, kw_ts in [(dict(z=z.reshape(-1, 1)), dict(z=z)), (dict(seed=SEED, row0=123), dict(seed=SEED, row0=123))]:
    _, i1, s1, n1 = post.moo_score_argmax_ts(G.lib.DFB_MOO_LIN_VAL, mus, sds, [1.0], want_scores=True, **kw_moo)
    _, i0, s0, n0 = post.score_argmax_ts(C, mean_const=post.mc, want_scores=True, **kw_ts)
    np.testing.assert_array_equal(_host(s1), _host(s0))
    assert (i1, n1) == (i0, n0) == (i0, 0)


def test_three_objectives_at_n1100_against_the_oracle(G):
  posts, ogps, C = _mixed_posteriors(G, 1100, 3000, 7, 3)
  mus, sds = _eval_all(G, posts, C)
  w, refs = [0.5, 0.3, 0.2], [0.1, -0.4, 0.05]
  mo, vo = zip(*[O.eval_std_diag(og, C) for og in ogps])
  np.random.seed(8)
  z = np.random.normal(size=(len(C), 3))
  beta = O.moo_ucb_beta_th(7, 1100)
  for name, kind in [('lin', G.lib.DFB_MOO_LIN_VAL), ('tch', G.lib.DFB_MOO_TCH_VAL)]:
    want = _vals(name, mo, [np.sqrt(v) for v in vo], z, w, refs)
    _, bi, sc, nonpos = posts[0].moo_score_argmax_ts(kind, mus, sds, w, refs, z=z, want_scores=True)
    assert np.abs(_host(sc) - want).max() <= 1e-6 and bi == O.np_argmax_first(want) and nonpos == 0
  for kind, want in [(G.lib.DFB_MOO_LIN_UCB, O.moo_lin_ucb(mo, [np.sqrt(v) for v in vo], w, beta)),
                     (G.lib.DFB_MOO_TCH_UCB, O.moo_tch_ucb(mo, [np.sqrt(v) for v in vo], w, refs, beta))]:
    _, bi, sc = posts[0].moo_score_argmax(kind, mus, sds, w, refs, beta, want_scores=True)
    assert np.abs(_host(sc) - want).max() <= 1e-6 and bi == O.np_argmax_first(want)


def test_bad_arguments_are_refused(G):
  posts, _, C = _mixed_posteriors(G, 200, 100, 4, 2)
  mus, sds = _eval_all(G, posts, C)
  for kind in (G.lib.DFB_MOO_LIN_UCB, G.lib.DFB_MOO_TCH_UCB, 7):
    with pytest.raises(G.lib.DfbError):
      posts[0].moo_score_argmax_ts(kind, mus, sds, [1.0, 1.0])
  with pytest.raises(G.lib.DfbError):
    posts[0].moo_score_argmax_ts(G.lib.DFB_MOO_LIN_VAL, mus, sds, [1.0, 1.0], row0=-1)


# ---- the acquisitions against the reference ----------------------------------------------------------------------
def _golden_gps(G, g, code_orders=None):
  """ the golden's two CPGPs; code_orders[k]: category levels to encode into objective k's Hamming table first """
  levels, numeric_levels, X, Ys, metas, H = T.golden_problem(g)
  gps = []
  for k, (Y, (scale, noise_var, mean_const)) in enumerate(zip(Ys, metas)):
    kern = (R.make_kernel if k == 0 else T.make_kernel2)(G.kernel, G.cp, scale)
    for v in (code_orders or {}).get(k, []):
      G.kernel.category_codes(kern.kernel_list[2]).encode(v)
    gps.append(G.cp.CPGP(X, list(Y), kern, (lambda c: (lambda x: np.array([c] * len(x))))(mean_const), noise_var))
  return gps, R.make_domain(G.domains, levels, numeric_levels), H


def _anc(g, dom, method, max_evals, halluc, **kw):
  a = Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=int(g['t']), handle_parallel='halluc',
                eval_points_in_progress=halluc, is_mf=False, obj_weights=list(g['weights']),
                reference_point=list(g['refs']))
  a.__dict__.update(kw)
  return a


def test_ucb_scores_match_the_reference(G, g):
  gps, dom, _ = _golden_gps(G, g)
  beta = G.moo._get_ucb_beta_th(dom.dim, int(g['t']))
  assert beta == float(g['beta'])
  C = R.golden_points(g, 'C')
  for name, kind in [('lin_ucb', G.lib.DFB_MOO_LIN_UCB), ('tch_ucb', G.lib.DFB_MOO_TCH_UCB)]:
    sc = G.moo._mo_cp_ucb_scores(kind, gps, C, list(g['weights']), list(g['refs']), beta)
    np.testing.assert_allclose(sc, g[name + '_scores'], rtol=0, atol=1e-9)
    assert int(np.argmax(sc)) == int(np.argmax(g[name + '_scores']))


def _run_golden(G, g, gps, dom, H):
  for k, run in enumerate(T.runs(g)):
    np.random.seed(run['seed'])
    pt = getattr(G.moo.asy, run['name'])(gps, _anc(g, dom, run['method'], run['max_evals'], H[:run['halluc']]))
    assert R.jencode(pt) == run['point'], run
    T.check_state(g, k)


def test_golden_points_and_rng_states(G, g):
  gps, dom, H = _golden_gps(G, g)
  _run_golden(G, g, gps, dom, H)


def test_disagreeing_code_tables(G, g):
  levels = T.golden_problem(g)[0]
  gps, dom, H = _golden_gps(G, g, code_orders={1: [v for loi in levels for v in reversed(loi)][::-1]})
  parts = [G.acq._cp_parts(dom, gp.kernel) for gp in gps]
  luts = [G.acq._cp_device_layout(p)[3] for p in parts]
  assert any(a is not None and not np.array_equal(a, b) for a, b in zip(luts[0], luts[1]))
  _run_golden(G, g, gps, dom, H)


def test_two_objectives_sharing_one_posterior(G, g):
  """ hallucinations on two GP objects with one device posterior: the second is augmented out of place """
  gps, dom, H = _golden_gps(G, g)
  twin = [gps[0], copy(gps[0])]
  assert twin[1]._post is twin[0]._post
  fresh = [gps[0], _golden_gps(G, g)[0][0]]
  out = []
  for pair in (twin, fresh):
    np.random.seed(44)
    out.append((R.jencode(G.moo.asy.tch_ts(pair, _anc(g, dom, 'rand', 3000, H[:2]))), np.random.get_state()[2]))
  assert out[0] == out[1]


def test_device_candidate_mode(G, g):
  gps, dom, _ = _golden_gps(G, g)
  M = 40000
  w, refs = list(g['weights']), list(g['refs'])
  for name, kind in [('lin_ts', G.lib.DFB_MOO_LIN_VAL), ('tch_ts', G.lib.DFB_MOO_TCH_VAL)]:
    np.random.seed(9)
    pt = getattr(G.moo.asy, name)(gps, _anc(g, dom, 'ga', M // 4, [], candidate_rng='device'))
    after = np.random.get_state()
    np.random.seed(9)
    pt2 = getattr(G.moo.asy, name)(gps, _anc(g, dom, 'ga', M // 4, [], candidate_rng='device'))
    assert R.jencode(pt2) == R.jencode(pt)
    np.random.seed(9)
    seed = (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))
    np.testing.assert_array_equal(np.random.get_state()[1], after[1])   # no host RNG beyond the seed
    parts = G.acq._cp_parts(dom, gps[0].kernel)
    post = gps[0]._device_posterior()
    kinds, bounds, n_levels, _ = G.acq._cp_device_layout(parts)
    raw = post.fill_mixed_candidates(seed, 0, M, kinds, bounds, n_levels).cpu().numpy()
    pts = [G.acq._cp_point_from_device_row(parts, r) for r in raw]
    mus, sds = zip(*[gp.eval(pts, 'std') for gp in gps])
    z = _host(post.fill_rng(seed, 0, 2, M)).T
    want = _vals(name[:3], mus, sds, z, w, refs)
    assert R.jencode(pt) == R.jencode(pts[O.np_argmax_first(want)])


def test_nan_candidate_raises_value_error(G, g, monkeypatch):
  gps, dom, _ = _golden_gps(G, g)
  real = G.acq.draw_cp_candidates
  def with_nan(parts, M):
    rows, draws = real(parts, M)
    draws[0][M // 2, 0] = np.nan
    return rows, draws
  monkeypatch.setattr(G.acq, 'draw_cp_candidates', with_nan)
  for name in ('lin_ts', 'tch_ts'):
    np.random.seed(1)
    with pytest.raises(ValueError):
      getattr(G.moo.asy, name)(gps, _anc(g, dom, 'rand', 2000, []))


def test_multi_rank_still_raises(G, g, monkeypatch):
  gps, dom, _ = _golden_gps(G, g)
  monkeypatch.setattr(G.moo, '_shard_info', lambda: (0, 2, None))
  for name in ('lin_ts', 'tch_ts', 'lin_ucb', 'tch_ucb'):
    with pytest.raises(NotImplementedError):
      getattr(G.moo.asy, name)(gps, _anc(g, dom, 'rand', 100, []))
