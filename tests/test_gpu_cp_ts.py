"""
Thompson sampling on Cartesian-product domains on the device (-m gpu): dfb_score_argmax_ts bit for bit against
fl(fl(sd z) + mu) from dfb_eval in every memory space, its int8 screen and bound-pass switch against the fp64 path at
the tile edges, its counter-based normals against dfb_fill_rng, and asy_ts / syn_ts against the unmodified reference
(golden cp_ts.npz) and the NumPy oracle (tests/cp_ts_ref.py).
"""
import json
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
from oracle import gp_oracle as O
import cp_ts_ref as T
import hamming_ref as R

pytestmark = pytest.mark.gpu

SEED = 0x1234_5678_9ABC_DEF1


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, cartesian_product_gp, gpb_acquisitions, domains, device, _lib
  _lib.load()
  return Namespace(kernel=kernel, cp=cartesian_product_gp, acq=gpb_acquisitions, domains=domains, device=device,
                   lib=_lib, torch=torch)


@pytest.fixture(scope='module')
def g():
  return load_golden('cp_ts')


def _mixed_problem(G, n, m, seed):
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = R.make_domain(G.domains, levels, numeric_levels)
  kern = R.make_kernel(G.kernel, G.cp, 0.8)
  parts = G.acq._cp_parts(dom, kern)
  np.random.seed(seed)
  X, _ = G.acq.draw_cp_candidates(parts, n)
  C, _ = G.acq.draw_cp_candidates(parts, m)
  Y = np.sin(3 * X[:, 0]) + 0.3 * X[:, 1] - 0.1 * (X[:, 2] - 3) ** 2 + 0.4 * (X[:, 3] == 1) + 0.2 * np.log(X[:, 6])
  Y = Y + 0.05 * np.random.standard_normal(n)
  return kern, X, Y, C


def _posterior(G, kern, X, Y, mc, impl, chunk=1024):
  post = G.device.DevicePosterior(len(X) + 8, chunk=chunk)
  post.set_option('score_impl', impl)
  post.set_kernel(G.kernel.build_descriptor(kern, train_dim=7, cand_dim=7))
  post.set_train(X, Y - mc)
  assert post.build(0.01)[0] == 0
  return post


def _host(v):
  return v.cpu().numpy() if hasattr(v, 'cpu') else np.asarray(v)


def _spaces(G, C, z):
  """ (name, candidates, normals) in pageable host, page-locked host and device memory """
  torch = G.torch
  Cp = torch.from_numpy(C).pin_memory()
  zp = torch.from_numpy(z).pin_memory()
  return [('pageable', C, z), ('pinned', Cp.numpy(), zp.numpy()),
          ('device', torch.from_numpy(C).cuda(), torch.from_numpy(z).cuda())]


def test_scores_bit_for_bit_in_every_memory_space(G):
  kern, X, Y, C = _mixed_problem(G, 1100, 20000, 1)     # 20000 rows: several chunks, two page-locked staging halves
  mc = float(np.mean(Y))
  post = _posterior(G, kern, X, Y, mc, 0)
  mu, sd = post.eval(C, mean_const=mc)
  np.random.seed(2)
  z = np.random.normal(size=len(C))
  want = sd * z + mu                                     # NumPy: one product, then one sum, no FMA
  zp = _host(post.fill_rng(SEED, 777, 1, len(C)))[0]
  want_p = sd * zp + mu
  for name, Cs, zs in _spaces(G, C, z):
    bs, bi, sc, nonpos = post.score_argmax_ts(Cs, mean_const=mc, z=zs, want_scores=True)
    np.testing.assert_array_equal(_host(sc), want, err_msg=name)
    assert bi == O.np_argmax_first(want) and bs == want[bi] and nonpos == 0, name
    bs, bi, sc, nonpos = post.score_argmax_ts(Cs, mean_const=mc, seed=SEED, row0=777, want_scores=True)
    np.testing.assert_array_equal(_host(sc), want_p, err_msg=name)
    assert bi == O.np_argmax_first(want_p) and bs == want_p[bi] and nonpos == 0, name


def test_counter_normals_are_fill_rng(G):
  kern, X, Y, C = _mixed_problem(G, 300, 5000, 3)
  mc = float(np.mean(Y))
  post = _posterior(G, kern, X, Y, mc, 0)
  mu, sd = post.eval(C, mean_const=mc)
  for seed, row0 in [(0, 0), (SEED, 0), (SEED, (1 << 33) + 5)]:
    z = _host(post.fill_rng(seed, row0, 1, len(C)))[0]
    _, _, sc, _ = post.score_argmax_ts(C, mean_const=mc, seed=seed, row0=row0, want_scores=True)
    np.testing.assert_array_equal(sc, sd * z + mu)
    # a candidate's normal depends on (seed, its global row) only: a slab from row r sees the same normals
    _, _, sc2, _ = post.score_argmax_ts(C[1000:], mean_const=mc, seed=seed, row0=row0 + 1000, want_scores=True)
    np.testing.assert_array_equal(sc2, sc[1000:])


@pytest.mark.parametrize('n', [1024, 1100, 1152])
def test_int8_screen_equals_fp64_and_the_oracle(G, n):
  kern, X, Y, C = _mixed_problem(G, n, 6000, n)
  mc = float(np.mean(Y))
  ogp = O.OGP(X, Y, R.oracle_kernel(0.8), lambda x: np.array([mc] * len(x)), 0.01)
  mu_o, var_o = O.eval_std_diag(ogp, C)
  np.random.seed(n)
  z = np.random.normal(size=len(C))
  exact = _posterior(G, kern, X, Y, mc, 0)
  fast = _posterior(G, kern, X, Y, mc, 2)
  zp = _host(exact.fill_rng(SEED, 0, 1, len(C)))[0]
  for kw, zz in [(dict(z=z), z), (dict(seed=SEED, row0=0), zp)]:
    s0, i0, _, n0 = exact.score_argmax_ts(C, mean_const=mc, **kw)
    assert i0 == O.np_argmax_first(np.sqrt(var_o) * zz + mu_o)
    for prune in (0, 1):
      fast.set_option('prune', prune)
      s1, i1, _, n1 = fast.score_argmax_ts(C, mean_const=mc, **kw)
      assert fast.query('last_used_i8') == 1.0
      assert fast.query('last_selfcheck_violations') == 0.0
      assert 0 < fast.query('last_shortlist') < len(C)
      assert fast.query('last_survivors') == 0.0                 # no bound pass for this kind
      assert (s1, i1, n1) == (s0, i0, n0) == (s0, i0, 0), (kw, prune)


def _golden_gp(G, g):
  levels, numeric_levels, scale, noise_var, mean_const, X, Y, H = T.golden_problem(g)
  gp = G.cp.CPGP(X, list(Y), R.make_kernel(G.kernel, G.cp, scale), lambda x: np.array([mean_const] * len(x)),
                 noise_var)
  return gp, R.make_domain(G.domains, levels, numeric_levels), H


def _anc(gp, dom, method, max_evals, halluc, **kw):
  a = Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=len(gp.X), curr_max_val=float(np.max(gp.Y)),
                handle_parallel='halluc', eval_points_in_progress=halluc, is_mf=False)
  a.__dict__.update(kw)
  return a


@pytest.mark.parametrize('impl', [0, 2])
def test_golden_points_and_rng_states(G, g, impl, monkeypatch):
  monkeypatch.setitem(G.device.DEFAULT_OPTIONS, 'score_impl', impl)
  gp, dom, H = _golden_gp(G, g)
  for k, run in enumerate(json.loads(str(g['ts_runs']))):
    np.random.seed(run['seed'])
    if run['kind'] == 'syn':
      pts = G.acq.syn.ts(3, gp, _anc(gp, dom, run['method'], run['max_evals'], H[:run['halluc']]))
    else:
      pts = [G.acq.asy.ts(gp, _anc(gp, dom, run['method'], run['max_evals'], H[:run['halluc']]))]
    assert [R.jencode(p) for p in pts] == run['points'], (impl, run)
    T.check_state(g, k)


def test_hallucinated_scores_follow_the_augmented_posterior(G, g):
  gp, dom, H = _golden_gp(G, g)
  parts = G.acq._cp_parts(dom, gp.kernel)
  np.random.seed(5)
  rows, draws = G.acq.draw_cp_candidates(parts, 3000)
  z = np.random.normal(size=3000)
  codes = {}
  ogp = T.oracle_gp(g, codes)
  C = R.encode_points([G.acq.point_from_draws(parts, draws, i) for i in range(3000)], codes)
  s_o, _, _ = T.marginal_scores(ogp, C, z, R.encode_points(H, codes))
  s_plain, _, _ = T.marginal_scores(ogp, C, z)
  with gp._fused_session(None, H) as sess:
    bs, bi, sc, nonpos = sess.score_ts(rows, z=z, want_scores=True)
  assert nonpos == 0 and bi == O.np_argmax_first(s_o) and bs == sc[bi]
  assert np.abs(sc - s_o).max() <= 1e-6
  assert np.abs(s_plain - s_o).max() > 1e-3                   # the hallucinations do change the draw


def test_device_candidate_mode(G, g):
  gp, dom, _ = _golden_gp(G, g)
  np.random.seed(9)
  pt = G.acq.asy.ts(gp, _anc(gp, dom, 'ga', 5000, [], candidate_rng='device'))
  after = np.random.get_state()
  parts = G.acq._cp_parts(dom, gp.kernel)
  np.random.seed(9)
  seed = (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))
  np.testing.assert_array_equal(np.random.get_state()[1], after[1])   # no host RNG beyond the seed
  post = gp._device_posterior()
  kinds, bounds, n_levels, _ = G.acq._cp_device_layout(parts)
  raw = post.fill_mixed_candidates(seed, 0, 20000, kinds, bounds, n_levels).cpu().numpy()
  pts = [G.acq._cp_point_from_device_row(parts, r) for r in raw]
  mu, sd = gp.eval(pts, 'std')
  z = _host(post.fill_rng(seed, 0, 1, 20000))[0]
  assert R.jencode(pt) == R.jencode(pts[O.np_argmax_first(sd * z + mu)])


def test_nan_candidate_raises_value_error(G, g, monkeypatch):
  gp, dom, _ = _golden_gp(G, g)
  real = G.acq.draw_cp_candidates
  def with_nan(parts, M):
    rows, draws = real(parts, M)
    rows[M // 2, 0] = np.nan
    return rows, draws
  monkeypatch.setattr(G.acq, 'draw_cp_candidates', with_nan)
  for impl in (0, 2):
    monkeypatch.setitem(G.device.DEFAULT_OPTIONS, 'score_impl', impl)
    gp2, _, _ = _golden_gp(G, g)
    np.random.seed(1)
    with pytest.raises(ValueError):
      G.acq.asy.ts(gp2, _anc(gp2, dom, 'rand', 2000, []))


def test_multi_rank_still_raises(G, g, monkeypatch):
  gp, dom, _ = _golden_gp(G, g)
  monkeypatch.setattr(G.acq, '_shard_info', lambda: (0, 2, None))
  with pytest.raises(NotImplementedError):
    G.acq.asy.ts(gp, _anc(gp, dom, 'rand', 100, []))


def test_bad_arguments_are_refused(G):
  kern, X, Y, C = _mixed_problem(G, 200, 100, 4)
  post = _posterior(G, kern, X, Y, 0.0, 0)
  with pytest.raises(G.lib.DfbError):
    post.score_argmax_ts(C, row0=-1)
  acq = G.device.make_acq_desc('ucb')
  acq.kind = G.lib.DFB_ACQ_TS_MARGINAL                          # the kind needs normals: not through dfb_score_argmax
  with pytest.raises(G.lib.DfbError):
    post.score_argmax(acq, C)
