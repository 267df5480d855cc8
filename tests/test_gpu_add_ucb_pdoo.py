"""
Add-UCB with the PDOO maximiser on the device (-m gpu): dfb_score_groups against the per-group row-streaming
evaluation (bit for bit) and the NumPy oracle; asy.add_ucb / BOCA's add_ucb with 'pdoo' and 'direct' against the same
lock-step search scored one group at a time, and against the reference's own points (tests/golden/add_ucb_pdoo.npz),
in one process and on two ranks.
"""
import os
from argparse import Namespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GROUPS = [[0, 1, 2], [3], [4, 5, 6, 7]]


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available()
  from dragonfly_b200 import kernel, gp_core, mf_gp, gpb_acquisitions, domains, doo
  from oracle import gp_oracle as O
  return Namespace(kernel=kernel, gp_core=gp_core, mf_gp=mf_gp, acq=gpb_acquisitions, domains=domains, doo=doo, O=O)


def _gp(B, n, groups=GROUPS, seed=0):
  rs = np.random.RandomState(seed)
  d = 8
  X = rs.random_sample((n, d))
  Y = np.sin(3 * X).sum(axis=1) + 0.05 * rs.standard_normal(n)
  kinds = [('matern', 2.5), ('se', None), ('matern', 1.5), ('se', None)]
  sub, osub = [], []
  for j, g in enumerate(groups):
    kind, nu = kinds[j % len(kinds)]
    bws = [0.3 + 0.05 * q for q in range(len(g))]
    if kind == 'se':
      sub.append(B.kernel.SEKernel(len(g), 1.0, bws)); osub.append(B.O.OSEKernel(len(g), 1.0, bws))
    else:
      sub.append(B.kernel.MaternKernel(len(g), nu, 1.0, bws)); osub.append(B.O.OMaternKernel(len(g), nu, 1.0, bws))
  scale = float(Y.var()) / len(groups)
  kern = B.kernel.AdditiveKernel(scale, sub, groups)
  gp = B.gp_core.GP(X, Y, kern, B.gp_core.ConstantMean(0.0), 0.01 * float(Y.var()))
  okern = B.O.OAdditiveKernel(scale, osub, groups)
  ogp = B.O.OGP(X, Y, okern, lambda x: np.zeros(len(x)), 0.01 * float(Y.var()))
  descs = [gp._group_test_descriptor(kern, sub[j], groups[j], d) for j in range(len(groups))]
  return gp, ogp, okern, descs


def _per_group(gp, desc, X, beta):
  """ The existing per-group path: dfb_eval of the rows (<= 32 at a time) with the group's test kernel bound. """
  with gp._fused_session(None, [], test_desc=desc, mean_const=0.0) as sess:
    mus, sds = [], []
    for r0 in range(0, len(X), 32):
      mu, sd = sess.post.eval(X[r0:r0 + 32], 0.0)
      mus.append(mu); sds.append(sd)
  mu, sd = np.concatenate(mus), np.concatenate(sds)
  return mu + beta * sd, mu, sd


@pytest.mark.parametrize('n', [1024, 1100, 1152])
def test_score_groups_is_the_per_group_evaluation_bit_for_bit(B, n):
  gp, ogp, okern, descs = _gp(B, n)
  post = gp._device_posterior()
  t = 300
  betas = [B.acq._get_add_ucb_beta_th(len(g), t) for g in GROUPS]
  rs = np.random.RandomState(n)
  for m in [1, 31, 32, 33, 200]:
    for present in ([0], [2, 1], [0, 1, 2]):
      groups = np.array(present)[rs.randint(0, len(present), m)].astype(np.int32)
      X = rs.random_sample((m, 4)) * 1.2 - 0.1
      scores = post.score_groups(descs, betas, X, groups)
      for j in set(groups.tolist()):
        rows = np.where(groups == j)[0]
        Xj = X[rows, :len(GROUPS[j])]
        ref, mu, sd = _per_group(gp, descs[j], Xj, betas[j])
        assert (scores[rows] == ref).all(), (n, m, j)
        _, mu_o, sd_o = B.O.add_ucb_group_scores(ogp, okern, j, Xj, t)
        assert np.abs(mu - mu_o).max() <= 1e-10 and np.abs(sd ** 2 - sd_o ** 2).max() <= 1e-8
  # a row's score does not depend on the other rows of the call
  X = rs.random_sample((40, 4))
  groups = (np.arange(40) % 3).astype(np.int32)
  full = post.score_groups(descs, betas, X, groups)
  assert (post.score_groups(descs, betas, X[7:8], groups[7:8])[0] == full[7])
  # a bound test kernel stays bound
  with gp._fused_session(None, [], test_desc=descs[2], mean_const=0.0) as sess:
    before = sess.post.eval(X[:3, :4], 0.0)
    post.score_groups(descs, betas, X, groups)
    after = sess.post.eval(X[:3, :4], 0.0)
  assert (before[0] == after[0]).all() and (before[1] == after[1]).all()


def test_group_sizes_one_to_d(B):
  groups = [[0], [1, 2], [3, 4, 5], [6, 7]]
  gp, ogp, okern, descs = _gp(B, 300, groups=groups, seed=4)
  betas = [B.acq._get_add_ucb_beta_th(len(g), 50) for g in groups]
  rs = np.random.RandomState(5)
  X = rs.random_sample((70, 3))
  g = rs.randint(0, 4, 70).astype(np.int32)
  scores = gp._device_posterior().score_groups(descs, betas, X, g)
  for j in range(4):
    rows = np.where(g == j)[0]
    assert (scores[rows] == _per_group(gp, descs[j], X[rows, :len(groups[j])], betas[j])[0]).all()
  # one group of all d coordinates
  gp8, _, _, descs8 = _gp(B, 300, groups=[list(range(8))], seed=6)
  X8 = rs.random_sample((33, 8))
  s8 = gp8._device_posterior().score_groups(descs8, [0.7], X8, np.zeros(33, dtype=np.int32))
  assert (s8 == _per_group(gp8, descs8[0], X8, 0.7)[0]).all()


def _anc(B, method, max_evals, t, d=8):
  dom = B.domains.EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq='add_ucb', max_evals=max_evals, t=t, domain=dom, curr_max_val=0.0,
                   eval_points_in_progress=[], acq_opt_method=method, handle_parallel='halluc', mf_strategy=None,
                   is_mf=False, domain_bounds=np.array(dom.bounds))


def _per_group_lockstep(B, gp, descs, groups, anc):
  """ The same lock-step search, each group's points scored through its own session (one call per group and round). """
  betas = [B.acq._get_add_ucb_beta_th(len(g), anc.t) for g in groups]

  def score(requests):
    return [_per_group(gp, descs[j], X, betas[j])[0] for j, X in requests]
  found = B.doo.pdoo_maximise_lockstep(score, [np.asarray(anc.domain_bounds)[g] for g in groups],
                                       anc.max_evals // len(groups))
  ret = np.zeros(sum(len(g) for g in groups))
  for (_, pt), g in zip(found, groups):
    ret[g] = pt
  return ret


@pytest.mark.parametrize('method', ['pdoo', 'direct'])
def test_asy_add_ucb_takes_one_device_call_per_round(B, method):
  gp, _, _, descs = _gp(B, 1100, seed=2)
  post = gp._device_posterior()
  calls = []
  real = post.score_groups

  def counted(*a, **k):
    calls.append(len(a[2]))
    return real(*a, **k)
  post.score_groups = counted
  try:
    for t in [10, 1100]:
      calls.clear()
      pt = B.acq.asy.add_ucb(gp, _anc(B, method, 900, t))
      assert len(calls) == B.doo.pdoo_maximise_lockstep.last_rounds
      assert (pt == _per_group_lockstep(B, gp, descs, GROUPS, _anc(B, method, 900, t))).all()
    picks = B.acq.syn.add_ucb(2, gp, _anc(B, method, 600, 50))
    assert len(picks) == 2 and all(p.shape == (8,) for p in picks)
  finally:
    del post.score_groups


def test_boca_add_ucb_with_pdoo(B):
  import os
  import sys
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
  from fake_mf_caller import FakeMFCaller
  rs = np.random.RandomState(9)
  n = 200
  Z, Xd = rs.random_sample((n, 1)), rs.random_sample((n, 4))
  Y = np.sin(3 * Xd).sum(axis=1) * (0.8 + 0.2 * Z[:, 0])
  kF = B.kernel.SEKernel(1, 1.0, [0.7])
  kDa = B.kernel.AdditiveKernel(1.0, [B.kernel.MaternKernel(2, 2.5, 1.0, [0.4, 0.5]),
                                      B.kernel.SEKernel(2, 1.0, [0.3, 0.6])], [[0, 1], [2, 3]])
  mfgp = B.mf_gp.EuclideanMFGP(list(Z), list(Xd), list(Y), None, float(Y.var()) / 2, kF, kDa,
                               B.gp_core.ConstantMean(float(np.median(Y))), 0.01 * float(Y.var()))
  anc = _anc(B, 'pdoo', 600, 150, d=4)
  anc.is_mf, anc.eval_fidel_points_in_progress = True, []
  anc.boca_thresh_coeff, anc.y_range, anc.boca_max_low_fidel_cost_ratio = 1e-4, float(np.ptp(Y)), 0.9
  np.random.seed(9)
  _, pt = B.acq.boca(None, mfgp, anc, FakeMFCaller([1.0]))
  rounds = B.doo.pdoo_maximise_lockstep.last_rounds
  assert pt.shape == (4,) and rounds > 1
  # the per-group objective of the fidel_to_opt slice, scored through dfb_eval on [z || x_j]
  from dragonfly_b200.kernel import CoordinateProductKernel, build_descriptor
  train_dim = mfgp._train_matrix().shape[1]
  groups = kDa.groupings
  ref = np.zeros(4)
  betas = [B.acq._get_add_ucb_beta_th(len(g), anc.t) for g in groups]
  descs = []
  for j, g in enumerate(groups):
    prod = CoordinateProductKernel(1 + len(g), mfgp.kernel.hyperparams['scale'], [mfgp.fidel_kernel, kDa.kernel_list[j]],
                                   [[0], list(range(1, 1 + len(g)))])
    descs.append(build_descriptor(prod, train_dim=train_dim, cand_dim=1 + len(g),
                                  train_coords=[mfgp.fidel_coords[0]] + [mfgp.domain_coords[int(q)] for q in g],
                                  cand_coords=list(range(1 + len(g)))))

  def score(requests):
    return [_per_group(mfgp, descs[j], np.concatenate((np.ones((len(X), 1)), X), axis=1), betas[j])[0]
            for j, X in requests]
  found = B.doo.pdoo_maximise_lockstep(score, [np.asarray(anc.domain_bounds)[g] for g in groups], 600 // 2)
  for (_, p), g in zip(found, groups):
    ref[g] = p
  assert (pt == ref).all()


# ---- the reference's own runs (tests/golden/add_ucb_pdoo.npz, tests/golden/make_golden_add_ucb_pdoo.py) ---------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'add_ucb_pdoo.npz')


def _golden_gp(g):
  from dragonfly_b200 import kernel, gp_core
  kern = kernel.AdditiveKernel(float(g['scale']), [kernel.MaternKernel(3, 2.5, 1.0, [0.4, 0.5, 0.6]),
                                                   kernel.SEKernel(1, 1.0, [0.3]),
                                                   kernel.MaternKernel(4, 1.5, 1.0, [0.5, 0.45, 0.55, 0.6])], GROUPS)
  return gp_core.GP(g['X'], g['Y'], kern, gp_core.ConstantMean(float(g['mean_const'])), float(g['noise_var']))


def _golden_points():
  """ asy.add_ucb on the golden GP for every asy case: {case: point}. """
  from dragonfly_b200 import domains
  from dragonfly_b200 import gpb_acquisitions as A
  g = np.load(GOLDEN)
  gp = _golden_gp(g)
  out = {}
  for case in ['pdoo_t5', 'pdoo_t300', 'direct_t100']:
    evals, t = [int(v) for v in g[case + '_args']]
    dom = domains.EuclideanDomain([[0, 1]] * 8)
    anc = Namespace(curr_acq='add_ucb', max_evals=evals, t=t, domain=dom, curr_max_val=0.0, eval_points_in_progress=[],
                    acq_opt_method=case.split('_')[0], handle_parallel='halluc', mf_strategy=None, is_mf=False,
                    domain_bounds=np.array(dom.bounds))
    out[case] = A.asy.add_ucb(gp, anc)
  return out


def test_golden_points_of_the_reference(B):
  g = np.load(GOLDEN)
  for case, pt in _golden_points().items():
    assert (pt == g[case + '_point']).all(), (case, pt, g[case + '_point'])
  gp = _golden_gp(g)
  picks = B.acq.syn.add_ucb(2, gp, _anc(B, 'pdoo', 450, 40))
  assert (np.array(picks) == g['syn_points']).all()


def test_golden_boca_add_ucb_with_pdoo(B):
  import sys
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
  from fake_mf_caller import FakeMFCaller
  g = np.load(GOLDEN)
  kF = B.kernel.SEKernel(1, 1.0, [0.7])
  kDa = B.kernel.AdditiveKernel(1.0, [B.kernel.MaternKernel(2, 2.5, 1.0, [0.4, 0.5]),
                                      B.kernel.SEKernel(2, 1.0, [0.3, 0.6])], [[0, 1], [2, 3]])
  Y = g['boca_Y']
  mfgp = B.mf_gp.EuclideanMFGP(list(g['boca_Z']), list(g['boca_Xd']), list(Y), None, float(g['boca_scale']), kF, kDa,
                               B.gp_core.ConstantMean(float(g['boca_mean_const'])), float(g['boca_noise_var']))
  anc = _anc(B, 'pdoo', 600, len(Y), d=4)
  anc.is_mf, anc.eval_fidel_points_in_progress = True, []
  anc.boca_thresh_coeff, anc.y_range, anc.boca_max_low_fidel_cost_ratio = 1e-4, float(np.ptp(Y)), 0.9
  fid, pt = B.acq.boca(None, mfgp, anc, FakeMFCaller([1.0]))
  assert (pt == g['boca_point']).all()
  assert (np.asarray(fid, dtype=np.float64) == g['boca_fidel']).all()


def _two_rank_worker(rank, world, port, out_dir):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  import sys
  sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
  import torch
  import torch.distributed as dist
  torch.cuda.set_device(0)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  np.savez(os.path.join(out_dir, 'rank%d.npz' % rank), **_golden_points())
  dist.barrier()
  dist.destroy_process_group()


def test_two_ranks_return_the_single_process_point(tmp_path):
  """ Every rank runs the whole search (no collective): two ranks on cuda:0 over gloo return the single-process
      points, which are the reference's. """
  import torch.multiprocessing as mp
  port = 37500 + (os.getpid() % 2000)
  mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
  want = _golden_points()
  g = np.load(GOLDEN)
  for r in range(2):
    got = np.load(os.path.join(str(tmp_path), 'rank%d.npz' % r))
    for case, pt in want.items():
      assert (got[case] == pt).all() and (pt == g[case + '_point']).all(), (case, r)
