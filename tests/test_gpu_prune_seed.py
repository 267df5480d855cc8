"""
The seeds of dfb_score_argmax's bound pass (option "prune_seed_rows", api.cu: run_bound_pass, kernels.cu:
seed_*_kernel) (-m gpu).

The rows with the largest bounds ub are contracted first, and the screen compares every other row against the
maximum they give.  Any seed set gives the same arg-max, so prune = 1 must return the (score, index) of prune = 0 and
of score_impl = 0, bit for bit, at every K: at the headline, with the winner inside and outside the seeds, exact ties
at the threshold, NaN rows and PI rows without a bound, every ub equal, K beyond the rows, UCB with negative scores, a
hallucinated posterior, every candidate memory space across staging batches and device rows beyond one screen
launch.  The device's seeds are those of the NumPy restatement (prune_seed_ref.py) of the stored bounds.
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import prune_seed_ref as S

pytestmark = pytest.mark.gpu

CHUNK = 1024
N_SMALL = 1100


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, device, synth_data, _lib
  _lib.load()
  return Namespace(torch=torch, kernel=kernel, device=device, synth=synth_data, lib=_lib)


def _bits(x):
  return np.array([x], dtype=np.float64).view(np.int64)[0]


def _post(B, X, Y, kern, noise, chunk, score_impl, prune=1):
  post = B.device.DevicePosterior(len(X) + 8, chunk=chunk)
  post.set_option('score_impl', score_impl)
  post.set_option('prune', prune)
  post.set_kernel(B.kernel.build_descriptor(kern))
  post.set_train(X, Y)
  assert post.build(noise)[0] == 0
  return post


def _debug(B, post, name, dtype, cap_name):
  n = int(post.query(cap_name))
  t = B.torch.empty((n,), dtype=dtype, device='cuda')
  B.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), n * t.element_size()),
              'dfb_debug_copy')
  return t.cpu().numpy()


class Trio(object):
  """ prune = 1 (K settable), prune = 0 and pure fp64 on the same posterior. """

  def __init__(self, pruned, full, fp64):
    self.pruned, self.full, self.fp64 = pruned, full, fp64
    self.posts = (pruned, full, fp64)

  def score(self, acq, C_, K, mean_const=0.0, B=None, check_seeds=False):
    self.pruned.set_option('prune_seed_rows', K)
    res = [p.score_argmax(acq, C_, mean_const=mean_const)[:2] for p in self.posts]
    (s1, i1), (s0, i0), (s64, i64) = res
    assert i1 == i0 == i64, res
    assert _bits(s1) == _bits(s0) == _bits(s64), res
    p = self.pruned
    assert p.query('last_used_i8') == 1.0 and p.query('last_selfcheck_violations') == 0.0
    q = {k: int(p.query(k)) for k in ('last_survivors', 'last_pruned_candidates', 'last_seed_rows',
                                      'last_contracted_rows')}
    m, chunk = len(C_), int(p.query('chunk'))
    assert q['last_survivors'] + q['last_pruned_candidates'] == m - chunk or q['last_pruned_candidates'] == 0
    seeds = ub = None
    if check_seeds:                       # device candidates within one screen launch: every row's bound is stored
      assert m <= p.query('keep_cap')
      ub = _debug(B, p, 'prune_ub', B.torch.float64, 'keep_cap')[:m]
      seeds = _debug(B, p, 'seed_idx', B.torch.int64, 'seed_cap')[:q['last_seed_rows']]
      assert (seeds == S.select_seeds(ub, K)).all()
    return Namespace(s=s1, i=i1, seeds=seeds, ub=ub, **q)


def _acq(B, name, Y, **kw):
  if name == 'ei':
    return B.device.make_acq_desc('ei', best=kw.get('best', float(Y.max())))
  if name == 'pi':
    return B.device.make_acq_desc('pi', best=kw.get('best', float(Y.max())))
  return B.device.make_acq_desc('ucb', beta=kw.get('beta', 3.0))


@pytest.fixture(scope='module')
def small(B):
  rs = np.random.RandomState(31)
  X = rs.random_sample((N_SMALL, 6))
  Y = B.synth.hartmann6(X)
  Y = Y - float(np.median(Y))
  kern = B.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)
  noise = 0.01 * float(Y.var())
  trio = Trio(*[_post(B, X, Y, kern, noise, CHUNK, impl, prune) for impl, prune in ((2, 1), (2, 0), (0, 1))])
  return Namespace(X=X, Y=Y, trio=trio, rs=rs)


def _dev(B, C_):
  return B.torch.from_numpy(np.ascontiguousarray(C_)).cuda()


# ---- the headline shape ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def headline(B):
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_cand=16)
  k = w['kernel']
  kern = B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])
  Yc = w['Y'] - w['mean_const']
  trio = Trio(*[_post(B, w['X'], Yc, kern, w['noise_var'], 0, impl, prune) for impl, prune in ((2, 1), (2, 0), (0, 1))])
  host = np.random.RandomState(1000).random_sample((1000000, 6))           # bench.py's rank-0 candidates
  return Namespace(w=w, trio=trio, C=_dev(B, host))


@pytest.mark.parametrize('K', [128, 512, 2048])
def test_headline(B, headline, K):
  w = headline.w
  r = headline.trio.score(_acq(B, 'ei', w['Y']), headline.C, K, mean_const=w['mean_const'], B=B, check_seeds=True)
  print('headline K %d: seeds %d, survivors %d, pruned %d, contracted %d' % (
      K, r.last_seed_rows, r.last_survivors, r.last_pruned_candidates, r.last_contracted_rows))
  assert K <= r.last_seed_rows <= 2 * K
  assert 0 < r.last_contracted_rows < 0.01 * len(headline.C)


# ---- edges ----------------------------------------------------------------------------------------------------------
def test_winner_inside_and_outside_the_seeds(B, small):
  """ The best training points have the largest mean, so the largest bounds, but sigma ~ 0: as the only seeds they
      lose to a candidate outside the seeds; with many seeds the winner is one of them. """
  Ch = small.rs.random_sample((5 * CHUNK + 3, 6))
  top = np.argsort(small.Y)[-5:]
  Ch[[40, 2 * CHUNK + 1, 3 * CHUNK, 4 * CHUNK + 9, 5 * CHUNK]] = small.X[top]
  C_ = _dev(B, Ch)
  acq = _acq(B, 'ei', small.Y)
  where = {}
  for K in (1, 2048):
    r = small.trio.score(acq, C_, K, B=B, check_seeds=True)
    where[K] = r.i in set(r.seeds.tolist())
  assert where == {1: False, 2048: True}


def test_exact_ties_straddling_the_threshold(B, small):
  Ch = small.rs.random_sample((4 * CHUNK + 21, 6))
  acq = _acq(B, 'ei', small.Y)
  r = small.trio.score(acq, _dev(B, Ch), 8, B=B, check_seeds=True)
  top = int(np.argmax(r.ub))
  pos = small.rs.choice(np.delete(np.arange(len(Ch)), top), 40, replace=False)
  Ch[pos] = Ch[top]                               # 41 exact copies of the largest bound at K = 8: cut at 2K in row order
  r = small.trio.score(acq, _dev(B, Ch), 8, B=B, check_seeds=True)
  assert r.last_seed_rows == 16 and (r.seeds == np.sort(np.append(pos, top))[:16]).all()


def test_nan_rows_and_pi_rows_without_a_bound(B, small):
  Ch = small.rs.random_sample((4 * CHUNK + 9, 6))
  Ch[[3, 2 * CHUNK + 7], 1] = np.nan
  for name, kw in (('ei', {}), ('ucb', {}), ('pi', {}), ('pi', {'best': float(np.median(small.Y))})):
    r = small.trio.score(_acq(B, name, small.Y, **kw), _dev(B, Ch), 64, B=B, check_seeds=True)
    assert {3, 2 * CHUNK + 7} <= set(r.seeds.tolist()) and r.i == 3 and np.isnan(r.s)
  r = small.trio.score(_acq(B, 'pi', small.Y, best=float(np.median(small.Y))),
                       _dev(B, small.rs.random_sample((4 * CHUNK + 9, 6))), 64, B=B, check_seeds=True)


def test_every_ub_equal(B, small):
  C_ = _dev(B, 3.0 + small.rs.random_sample((7 * CHUNK + 5, 6)))
  r = small.trio.score(_acq(B, 'ucb', small.Y, beta=50.0), C_, 256, B=B, check_seeds=True)
  assert (r.seeds == np.arange(512)).all()
  assert r.last_survivors > 4 * CHUNK and r.last_pruned_candidates == 0


@pytest.mark.parametrize('K', [100, 1124, 4096])
def test_k_at_or_beyond_the_rows(B, small, K):
  C_ = _dev(B, small.rs.random_sample((CHUNK + 100, 6)))
  r = small.trio.score(_acq(B, 'ei', small.Y), C_, K, B=B, check_seeds=True)
  if K >= CHUNK + 100:
    assert r.last_seed_rows == CHUNK + 100 and r.last_survivors == 100 and r.last_pruned_candidates == 0


def test_ucb_with_negative_scores(B, small):
  C_ = _dev(B, small.rs.random_sample((4 * CHUNK + 1, 6)))
  r = small.trio.score(_acq(B, 'ucb', small.Y, beta=1.0), C_, 64, mean_const=-1000.0, B=B, check_seeds=True)
  assert r.s < 0 and r.last_pruned_candidates > 0


def test_hallucinated_posterior(B, small):
  Xh = small.rs.random_sample((5, 6))
  for p in small.trio.posts:
    _, alpha, _ = p.get_state(want_alpha=True)
    assert p.extend(Xh, np.zeros(5), save=True)[0] == 0
    p.set_alpha(alpha)
  try:
    Ch = small.rs.random_sample((4 * CHUNK + 11, 6))
    Ch[2 * CHUNK:2 * CHUNK + 5] = Xh
    for name in ('ei', 'ucb', 'pi'):
      small.trio.score(_acq(B, name, small.Y), _dev(B, Ch), 64, B=B, check_seeds=True)
  finally:
    for p in small.trio.posts:
      p.restore(N_SMALL)


# 45 chunks: at d = 6 a staging batch is 21 chunks, so pageable candidates cross three batches, page-locked ones five
# halves; the seeds come from the first batch (half), whose buffer is refilled later.
@pytest.mark.parametrize('space', ['pageable', 'pinned', 'device'])
def test_candidate_memory_spaces(B, small, space):
  m = 45 * CHUNK + 5
  host = small.rs.random_sample((m, 6))
  if space == 'pageable':
    C_ = host
  else:
    t = B.torch.empty((m, 6), dtype=B.torch.float64, pin_memory=True)
    t.numpy()[:] = host
    C_ = t.numpy() if space == 'pinned' else t.cuda()
  for name in ('ei', 'ucb', 'pi'):
    for K in (16, 512):
      r = small.trio.score(_acq(B, name, small.Y), C_, K, B=B, check_seeds=(space == 'device'))
      assert r.last_pruned_candidates > 0


def test_device_rows_beyond_one_screen_launch(B, small):
  keep_cap = int(small.trio.pruned.query('keep_cap'))
  Ch = small.rs.random_sample((keep_cap + 3 * CHUNK + 7, 6))
  Ch[keep_cap + 100] = small.X[int(np.argmax(small.Y))] + 1e-3      # a strong candidate in the second launch
  C_ = _dev(B, Ch)
  r = small.trio.score(_acq(B, 'ei', small.Y), C_, 256)
  assert r.last_pruned_candidates > 0
  ub = _debug(B, small.trio.pruned, 'prune_ub', B.torch.float64, 'keep_cap')
  seeds = _debug(B, small.trio.pruned, 'seed_idx', B.torch.int64, 'seed_cap')[:r.last_seed_rows]
  assert (seeds == S.select_seeds(ub, 256)).all()                   # from the first launch's rows only
