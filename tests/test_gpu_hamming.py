"""
Categorical and mixed Cartesian-product domains on the device (-m gpu): the descriptor interpreter's HAMMING factor
against the unmodified reference (golden hamming.npz) and the NumPy oracle (tests/hamming_ref.py), the fused `rand`
maximiser on CP domains against the reference's seeded acquisitions, and dfb_fill_mixed_candidates.
"""
import json
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
from oracle import gp_oracle as O
import hamming_ref as R

pytestmark = pytest.mark.gpu

MU_TOL = 1e-10
VAR_TOL = 1e-8


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
  return load_golden('hamming')


def _golden_gp(G, g):
  levels, numeric_levels, scale, noise_var, mean_const = R.golden_problem(g)
  kern = R.make_kernel(G.kernel, G.cp, scale)
  X = R.golden_points(g, 'X')
  gp = G.cp.CPGP(X, list(g['Y']), kern, lambda x: np.array([mean_const] * len(x)), noise_var)
  return gp, R.make_domain(G.domains, levels, numeric_levels)


def test_hamming_blocks_bit_for_bit(G, g):
  for ci, m in enumerate(json.loads(str(g['hk_meta']))):
    X1 = [[R.jvalue(v) for v in r] for r in m['X1']]
    X2 = [[R.jvalue(v) for v in r] for r in m['X2']]
    k = G.kernel.HammingKernel(m['dim'] if m['weights'] is None else m['weights'])
    np.testing.assert_array_equal(k(X1, X2), g['hk%d_K' % ci])
    np.testing.assert_array_equal(k(X1, X1), g['hk%d_Kss' % ci])


def test_cpgp_against_the_reference(G, g):
  gp, _ = _golden_gp(G, g)
  X = R.golden_points(g, 'X')
  np.testing.assert_allclose(gp.kernel(X[:16], X), g['K'], rtol=0, atol=1e-13)
  assert abs(gp.compute_log_marginal_likelihood() - float(g['lml'])) <= 1e-9 * abs(float(g['lml']))
  C, H = R.golden_points(g, 'C'), R.golden_points(g, 'H')
  mu, sd = gp.eval(C, 'std')
  assert np.max(np.abs(mu - g['mu'])) <= MU_TOL
  assert np.max(np.abs(sd ** 2 - g['sd'] ** 2)) <= VAR_TOL
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:100], H, 'std')
  assert np.max(np.abs(mu_h - g['mu_h'])) <= MU_TOL
  assert np.max(np.abs(sd_h ** 2 - g['sd_h'] ** 2)) <= VAR_TOL


def test_seeded_acquisitions_match_the_reference(G, g):
  gp, dom = _golden_gp(G, g)
  H = R.golden_points(g, 'H')
  for k, run in enumerate(json.loads(str(g['acq_runs']))):
    np.random.seed(run['seed'])
    anc = Namespace(domain=dom, max_evals=2000, acq_opt_method='rand', t=len(gp.X), curr_max_val=float(np.max(g['Y'])),
                    handle_parallel='halluc', eval_points_in_progress=H[:run['halluc']], is_mf=False)
    pt = getattr(G.acq.asy, run['name'])(gp, anc)
    st = np.random.get_state()
    assert R.jencode(pt) == run['point'], run
    np.testing.assert_array_equal(st[1], g['acq%d_state' % k])
    assert st[2] == int(g['acq%d_pos' % k])


def _mixed_problem(G, n, m, seed):
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = R.make_domain(G.domains, levels, numeric_levels)
  kern = R.make_kernel(G.kernel, G.cp, 0.8)
  parts = G.acq._cp_parts(dom, kern)
  np.random.seed(seed)
  X, Xd = G.acq.draw_cp_candidates(parts, n)
  C, _ = G.acq.draw_cp_candidates(parts, m)
  Y = np.sin(3 * X[:, 0]) + 0.3 * X[:, 1] - 0.1 * (X[:, 2] - 3) ** 2 + 0.4 * (X[:, 3] == 1) + 0.2 * np.log(X[:, 6])
  Y = Y + 0.05 * np.random.standard_normal(n)
  return kern, X, Y, C


@pytest.mark.parametrize('n', [1100, 1024, 1152])
def test_argmax_against_the_oracle_at_tile_edges(G, n):
  kern, X, Y, C = _mixed_problem(G, n, 6000, n)
  mc = float(np.mean(Y))
  ok = R.oracle_kernel(0.8)
  ogp = O.OGP(X, Y, ok, lambda x: np.array([mc] * len(x)), 0.01)
  mu_o, var_o = O.eval_std_diag(ogp, C)
  best = float(Y.max())
  for impl in (0, 2):
    post = G.device.DevicePosterior(n + 8, chunk=1024)
    post.set_option('score_impl', impl)
    post.set_kernel(G.kernel.build_descriptor(kern, train_dim=7, cand_dim=7))
    post.set_train(X, Y - mc)
    assert post.build(0.01)[0] == 0
    mu, sd = post.eval(C, mean_const=mc)
    assert np.abs(mu - mu_o).max() <= MU_TOL
    assert np.abs(sd ** 2 - var_o).max() <= VAR_TOL
    for name, acq, f in [('ei', G.device.make_acq_desc('ei', best=best), lambda m, s: O.acq_ei(m, s, best)),
                         ('ucb', G.device.make_acq_desc('ucb', beta=2.0), lambda m, s: O.acq_ucb(m, s, 2.0)),
                         ('pi', G.device.make_acq_desc('pi', best=best), lambda m, s: O.acq_pi(m, s, best))]:
      _, idx, _ = post.score_argmax(acq, C, mean_const=mc)
      assert idx == O.np_argmax_first(f(mu_o, np.sqrt(var_o))), (impl, name)


def test_duplicate_candidates_resolve_to_the_first_index(G):
  kern, X, Y, C = _mixed_problem(G, 1100, 3000, 5)
  mc = float(np.mean(Y))
  for impl in (0, 2):
    post = G.device.DevicePosterior(1108, chunk=1024)
    post.set_option('score_impl', impl)
    post.set_kernel(G.kernel.build_descriptor(kern, train_dim=7, cand_dim=7))
    post.set_train(X, Y - mc)
    assert post.build(0.01)[0] == 0
    acq = G.device.make_acq_desc('ei', best=float(Y.max()))
    _, i0, _ = post.score_argmax(acq, C, mean_const=mc)
    D = C.copy()
    for pos in (2999, 2500, 1023, 1024, i0 + 1):        # copies of the winner across chunk edges, after it
      if i0 < pos < 3000:
        D[pos] = C[i0]
    D2 = np.concatenate([D, D])
    s1, i1, sc = post.score_argmax(acq, D2, mean_const=mc, want_scores=True)
    assert i1 == i0
    sc = np.asarray(sc.cpu().numpy() if hasattr(sc, 'cpu') else sc)
    same = np.all(D2 == C[i0], axis=1)
    assert len(set(sc[same].tolist())) == 1              # identical rows score bit-identically wherever they fall


def test_hallucinations_restore_bit_for_bit(G, g):
  gp, dom = _golden_gp(G, g)
  C, H = R.golden_points(g, 'C'), R.golden_points(g, 'H')
  mu0, sd0 = gp.eval(C, 'std')
  np.random.seed(4)
  anc = Namespace(domain=dom, max_evals=3000, acq_opt_method='rand', t=len(gp.X), curr_max_val=float(np.max(g['Y'])),
                  handle_parallel='halluc', eval_points_in_progress=H, is_mf=False)
  G.acq.asy.ei(gp, anc)
  mu1, sd1 = gp.eval(C, 'std')
  np.testing.assert_array_equal(mu0, mu1)
  np.testing.assert_array_equal(sd0, sd1)


def test_device_candidate_mode(G, g):
  gp, dom = _golden_gp(G, g)
  np.random.seed(9)
  anc = Namespace(domain=dom, max_evals=20000, acq_opt_method='rand', t=len(gp.X), curr_max_val=float(np.max(g['Y'])),
                  handle_parallel='halluc', eval_points_in_progress=[], is_mf=False, candidate_rng='device')
  pt = G.acq.asy.ei(gp, anc)
  assert 0 <= pt[0][0] <= 1 and -1 <= pt[0][1] <= 2 and pt[1].dtype.kind == 'i' and 0 <= pt[1][0] <= 6
  levels, numeric_levels, _, _, _ = R.golden_problem(g)
  assert all(pt[2][q] in np.array(levels[q]) for q in range(3)) and pt[3][0] in numeric_levels[0]
  # the winner is the oracle's arg-max over the rows the device generated
  parts = G.acq._cp_parts(dom, gp.kernel)
  np.random.seed(9)
  seed = (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))
  post = gp._device_posterior()
  kinds, bounds, n_levels, _ = G.acq._cp_device_layout(parts)
  raw = post.fill_mixed_candidates(seed, 0, 20000, kinds, bounds, n_levels).cpu().numpy()
  pts = [G.acq._cp_point_from_device_row(parts, r) for r in raw]
  mu, sd = gp.eval(pts, 'std')
  best = float(np.max(g['Y']))
  assert R.jencode(pt) == R.jencode(pts[O.np_argmax_first(O.acq_ei(mu, sd, best))])


def test_fill_mixed_candidates(G):
  post = G.device.DevicePosterior(256)
  L = G.lib
  bounds = [[0.0, 1.0], [-2.0, 3.5], [1.0, 7.0], [-5.0, 5.0], [0.0, 0.0], [0.0, 0.0], [0.0, 0.0]]
  real = post.fill_candidates(77, 0, 5000, bounds[:4]).cpu().numpy()
  allreal = post.fill_mixed_candidates(77, 0, 5000, [L.DFB_CAND_REAL] * 4, bounds[:4], [0] * 4).cpu().numpy()
  np.testing.assert_array_equal(allreal, real)
  kinds = [L.DFB_CAND_REAL, L.DFB_CAND_REAL, L.DFB_CAND_INTEGER, L.DFB_CAND_INTEGER, L.DFB_CAND_CATEGORICAL,
           L.DFB_CAND_CATEGORICAL, L.DFB_CAND_CATEGORICAL]
  levels = [0, 0, 0, 0, 1, 3, 1000]
  mixed = post.fill_mixed_candidates(77, 0, 5000, kinds, bounds, levels).cpu().numpy()
  ref7 = post.fill_candidates(77, 0, 5000, bounds[:4] + [[0.0, 1.0]] * 3).cpu().numpy()
  np.testing.assert_array_equal(mixed[:, :2], ref7[:, :2])
  np.testing.assert_array_equal(mixed[:, 2:4], np.trunc(ref7[:, 2:4]))
  for c, n in zip((4, 5, 6), (1, 3, 1000)):
    col = mixed[:, c]
    assert np.all(col == np.floor(col)) and col.min() >= 0 and col.max() <= n - 1
    np.testing.assert_array_equal(col, np.minimum(np.floor(ref7[:, c] * n), n - 1))
  assert len(np.unique(mixed[:, 6])) > 900
  shard = post.fill_mixed_candidates(77, 1234, 777, kinds, bounds, levels).cpu().numpy()
  np.testing.assert_array_equal(shard, mixed[1234:1234 + 777])
  with pytest.raises(G.lib.DfbError):
    post.fill_mixed_candidates(77, 0, 10, [L.DFB_CAND_CATEGORICAL], [[0, 0]], [0])


def test_lml_batch_and_gradients_refuse_hamming(G):
  kern, X, Y, _ = _mixed_problem(G, 200, 10, 3)
  post = G.device.DevicePosterior(208)
  desc = G.kernel.build_descriptor(kern, train_dim=7, cand_dim=7)
  post.set_kernel(desc)
  post.set_train(X, Y)
  assert post.build(0.01)[0] == 0
  with pytest.raises(G.lib.DfbError):
    post.lml_batch([desc], [0.01], [0.0])
  with pytest.raises(NotImplementedError):
    post.lml_gradients(7)
