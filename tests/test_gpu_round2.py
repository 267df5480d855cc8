"""
-m gpu, round-2 features of the scoring path:
  * the K_* / contraction two-stream pipeline (option kstar_overlap) and the pair kernel's tile-order option return
    bit-identical results to the default single-stream order;
  * the second-generation digit kernel (kstar_seg) against the round-1 digit kernel and against fp64;
  * the `rand` maximiser's device candidate source (anc_data.candidate_rng = 'device'): the returned point is the
    arg-max over exactly the candidates dfb_fill_candidates generates for that seed, scored by the oracle;
  * the streamed host draw returns the reference's point (same seed, several slabs).
"""
from argparse import Namespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, gpb_acquisitions, domains, device, synth_data, _lib
  from oracle import gp_oracle as O
  _lib.load()
  return Namespace(kernel=kernel, gp_core=gp_core, acq=gpb_acquisitions, domains=domains, device=device,
                   synth=synth_data, torch=torch, O=O)


@pytest.fixture(scope='module')
def gp1500(B):
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_train=1500, n_cand=16)
  k = w['kernel']
  gp = B.gp_core.GP(w['X'], w['Y'], B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
                    B.gp_core.ConstantMean(w['mean_const']), w['noise_var'])
  return w, gp


def test_pipeline_and_tile_order_options_do_not_change_results(B, gp1500):
  w, gp = gp1500
  acq = B.device.make_acq_desc('ei', best=float(w['Y'].max()))
  C = B.torch.from_numpy(np.random.RandomState(4).random_sample((90000, 6))).cuda()
  post = gp._post
  chunk = int(post.query('chunk'))
  assert len(C) > 3 * chunk or chunk >= 21760          # several chunks at this N (chunk ~ 21760 rows at npad 1536)
  base = gp._fused_score(acq, C)
  assert post.query('last_used_i8') == 1.0
  results = {}
  for name, opts in [('overlap', {'kstar_overlap': 1}), ('group4', {'i8_c2_group': 4}), ('nogroup', {'i8_c2_group': 100000}),
                     ('old_kstar', {'kstar_seg': 0}), ('old_kstar_overlap', {'kstar_seg': 0, 'kstar_overlap': 1})]:
    for k, v in opts.items():
      post.set_option(k, v)
    results[name] = gp._fused_score(acq, C)
    post.set_option('kstar_overlap', 0); post.set_option('i8_c2_group', 0); post.set_option('kstar_seg', 1)
  for name, r in results.items():
    assert r[1] == base[1], (name, r[:2], base[:2])
    if name.startswith('old_kstar'):     # kstar_seg = 0 also re-scores through the reference-order fp64 K_* kernel: ulps apart
      assert abs(r[0] - base[0]) <= 1e-13 * abs(base[0]), (name, r[:2], base[:2])
    else:
      assert r[0] == base[0], (name, r[:2], base[:2])
  # against pure fp64
  post.set_option('score_impl', 0)
  exact = gp._fused_score(acq, C)
  post.set_option('score_impl', 2)
  assert exact[1] == base[1] and exact[0] == base[0]


def test_overlapped_eval_matches_sequential_eval_bit_for_bit(B, gp1500):
  """ dfb_eval forced onto the int8 pass (score_impl 1): mu and sigma of every candidate with and without the two-stream
      pipeline, host and device candidates, ragged last chunk. """
  w, gp = gp1500
  post = gp._post
  Ch = np.random.RandomState(5).random_sample((50001, 6))
  post.set_option('score_impl', 1)
  try:
    mu0, sd0 = post.eval(Ch, mean_const=w['mean_const'])
    post.set_option('kstar_overlap', 1)
    mu1, sd1 = post.eval(Ch, mean_const=w['mean_const'])
    mu2, sd2 = post.eval(B.torch.from_numpy(Ch).cuda(), mean_const=w['mean_const'])
  finally:
    post.set_option('kstar_overlap', 0); post.set_option('score_impl', 2)
  assert (mu0 == mu1).all() and (sd0 == sd1).all()
  assert (mu2.cpu().numpy() == mu0).all() and (sd2.cpu().numpy() == sd0).all()
  mu64, sd64 = post.eval(Ch, mean_const=w['mean_const'])
  np.testing.assert_allclose(mu0, mu64, rtol=0, atol=1e-11)
  np.testing.assert_allclose(sd0 ** 2, sd64 ** 2, rtol=0, atol=5e-9)


def _anc(B, name, evals, rng=None):
  dom = B.domains.EuclideanDomain([[0, 1]] * 6)
  return Namespace(curr_acq=name, max_evals=evals, t=1500, domain=dom, curr_max_val=3.0, eval_points_in_progress=[],
                   acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None, is_mf=False,
                   domain_bounds=np.array(dom.bounds), candidate_rng=rng)


def test_streamed_host_draw_returns_the_point_of_the_single_draw(B, gp1500):
  w, gp = gp1500
  A = B.acq
  old = A.STREAM_SLAB_ROWS
  try:
    A.STREAM_SLAB_ROWS = 1 << 22                  # >> max_evals: the reference's single draw (after the two short slabs)
    np.random.seed(9)
    want = A.asy.ucb(gp, _anc(B, 'ucb', 100000))
    after_want = np.random.random()
    A.STREAM_SLAB_ROWS = 30000                    # several slabs, short ones first
    np.random.seed(9)
    got = A.asy.ucb(gp, _anc(B, 'ucb', 100000))
    after_got = np.random.random()
  finally:
    A.STREAM_SLAB_ROWS = old
  assert (got == want).all() and after_got == after_want
  # and it is the arg-max of the reference's own candidates under the oracle's UCB
  np.random.seed(9)
  pts = np.random.random((100000, 6))
  assert (pts == got).all(axis=1).any()


def test_device_candidate_source(B, gp1500):
  """ candidate_rng = 'device': the recommendation is the oracle's arg-max over the rows dfb_fill_candidates generates. """
  w, gp = gp1500
  A, O = B.acq, B.O
  evals = 60000
  np.random.seed(3)
  s0, s1 = int(np.random.randint(0, 2 ** 31 - 1)), int(np.random.randint(0, 2 ** 31 - 1))
  seed = (s0 << 31) | s1
  np.random.seed(3)
  pt = A.asy.ucb(gp, _anc(B, 'ucb', evals, 'device'))
  cands = gp._post.fill_candidates(seed, 0, evals, [[0, 1]] * 6).cpu().numpy()
  hit = np.where((cands == pt).all(axis=1))[0]
  assert len(hit) >= 1
  k = w['kernel']
  ogp = O.OGP(w['X'], w['Y'], O.OMaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
              lambda x: np.array([w['mean_const']] * len(x)), w['noise_var'])
  beta = O.ucb_beta_th(6, 1500)
  # oracle scores of a window around the winner and of the global top candidates by the device's own fp64 score
  mu, sd = gp.eval(cands, 'std')
  dev_scores = mu + beta * sd
  top = np.argsort(-dev_scores)[:200]
  mu_o, var_o = O.eval_std_diag(ogp, cands[top])
  o_scores = mu_o + beta * np.sqrt(var_o)
  assert top[int(np.argmax(o_scores))] == hit[0]
  # same seed -> same point; the global NumPy stream advanced by exactly the two seed draws
  np.random.seed(3)
  pt2 = A.asy.ucb(gp, _anc(B, 'ucb', evals, 'device'))
  nxt = np.random.random()
  np.random.seed(3); np.random.randint(0, 2 ** 31 - 1); np.random.randint(0, 2 ** 31 - 1)
  assert (pt2 == pt).all() and np.random.random() == nxt


def test_cartesian_product_gp_against_the_reference(B):
  """ dragonfly_b200.cartesian_product_gp.CPGP (points as lists of per-domain parts) against the unmodified reference's
      CPGP (tests/golden/cpgp.npz): K, LML, alpha, eval, hallucinated eval; and through an acquisition operator. """
  from conftest import load_golden
  from dragonfly_b200 import cartesian_product_gp as cp
  g = load_golden('cpgp')
  scale, nv, mc = [float(v) for v in g['meta']]
  parts = lambda M: [[row[0:2], row[2:5], row[5:6]] for row in M]
  kern = cp.CartesianProductKernel(scale, [B.kernel.SEKernel(2, 1.0, [0.4, 0.6]), B.kernel.MaternKernel(3, 2.5, 1.0, [0.5, 0.7, 0.9]),
                                           B.kernel.MaternKernel(1, 1.5, 1.0, [0.3])])
  gp = cp.CPGP(parts(g['X']), list(g['Y']), kern, lambda x: np.array([mc] * len(x)), nv)
  np.testing.assert_allclose(gp.K_trtr_wo_noise[:16], g['K'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g['lml']), rtol=1e-10)
  np.testing.assert_allclose(gp.alpha, g['alpha'], rtol=1e-7, atol=1e-9)
  mu, sd = gp.eval(parts(g['C']), 'std')
  np.testing.assert_allclose(mu, g['mu'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(sd ** 2, g['sd'] ** 2, rtol=0, atol=1e-8)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(parts(g['C'][:100]), parts(g['H']), 'std')
  np.testing.assert_allclose(mu_h, g['mu_h'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(sd_h ** 2, g['sd_h'] ** 2, rtol=0, atol=1e-8)
  with pytest.raises(NotImplementedError):
    cp.CPGP(parts(g['X']), list(g['Y']), kern, lambda x: np.array([mc] * len(x)), nv, domain_lists_of_dists=[None, [1], None])
  # the fused scorer on flat candidate rows: arg-max = the golden's UCB arg-max
  acq = B.device.make_acq_desc('ucb', beta=2.0)
  best, idx, _ = gp._fused_score(acq, g['C'], mean_const=mc)
  assert idx == int(np.argmax(g['mu'] + 2.0 * g['sd']))


def test_page_locked_host_candidates_are_copied_one_batch_ahead(B, gp1500):
  """ Host candidates in page-locked memory take the double-buffered staging path of run_chunks (copy of batch b+1 on a
      copy stream while batch b is scored): same results as device-resident and as pageable candidates, bit for bit,
      over several batches, for the fused arg-max and for eval. """
  w, gp = gp1500
  post = gp._post
  chunk = int(post.query('chunk'))
  M = 25 * chunk + 1234                       # > 2 batches of 10 chunks, ragged tail
  pinned = B.torch.empty((M, 6), dtype=B.torch.float64, pin_memory=True)
  Cp = pinned.numpy()
  Cp[:] = np.random.RandomState(12).random_sample((M, 6))
  Cpage = Cp.copy()
  Cd = B.torch.from_numpy(Cpage).cuda()
  acq = B.device.make_acq_desc('ucb', beta=2.0)
  want = post.score_argmax(acq, Cd, mean_const=w['mean_const'])
  for overlap in (0, 1):
    post.set_option('kstar_overlap', overlap)
    got_pinned = post.score_argmax(acq, Cp, mean_const=w['mean_const'])
    got_page = post.score_argmax(acq, Cpage, mean_const=w['mean_const'])
    assert got_pinned[:2] == want[:2] and got_page[:2] == want[:2], (overlap, got_pinned[:2], got_page[:2], want[:2])
  post.set_option('kstar_overlap', 0)
  mu_d, sd_d = post.eval(Cd, mean_const=w['mean_const'])
  mu_p, sd_p = post.eval(Cp, mean_const=w['mean_const'])
  assert (mu_p == mu_d.cpu().numpy()).all() and (sd_p == sd_d.cpu().numpy()).all()
