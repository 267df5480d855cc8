"""
The bound pass of dfb_score_argmax (option "prune", api.cu: run_chunks_pruned, run_bound_pass) (-m gpu).

After chunk 0 is scored, the candidates of the later chunks get mu alone and are dropped when acq(mu, sqrt(k**)) lies
below a certain lower bound of the fp64 maximum.  The arg-max must not notice: prune = 1 returns the same (score,
index), bit for bit, as prune = 0 (every candidate through the int8 contraction) and as score_impl = 0 (everything in
fp64 DMMA), here at the headline shape and at the edges of the scheme -- exact ties across chunks, a NaN candidate in
a late chunk, candidates on training points, an unreachable incumbent, a large UCB beta, a survivor list that
overflows, m around the chunk size, every candidate memory space and a hallucinated posterior.  The mu-only variant of
the segment kernel is checked bit for bit against the digit and fp64-row variants at every (kind, d <= 8).
"""
from argparse import Namespace

import numpy as np
import pytest

import kstar_ref as R

pytestmark = pytest.mark.gpu

CHUNK = 1024
N_SMALL = 1100          # >= 1024: the int8 screen is the default there


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, device, synth_data, _lib
  _lib.load()
  return Namespace(torch=torch, kernel=kernel, device=device, synth=synth_data)


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


class Trio(object):
  """ The same posterior three times: auto mode with prune = 1 and = 0, and pure fp64. """

  def __init__(self, B, X, Y, kern, noise, chunk=CHUNK):
    self.B = B
    self.pruned = _post(B, X, Y, kern, noise, chunk, 2, 1)
    self.full = _post(B, X, Y, kern, noise, chunk, 2, 0)
    self.fp64 = _post(B, X, Y, kern, noise, chunk, 0, 1)
    self.posts = (self.pruned, self.full, self.fp64)

  def score(self, acq, C, mean_const=0.0):
    """ Asserts the three results agree bit for bit; returns (score, index, survivors, pruned). """
    res = [p.score_argmax(acq, C, mean_const=mean_const)[:2] for p in self.posts]
    for p in self.posts[:2]:
      assert p.query('last_used_i8') == 1.0
    assert self.full.query('last_survivors') == 0.0 and self.full.query('last_pruned_candidates') == 0.0
    (s1, i1), (s0, i0), (s64, i64) = res
    assert i1 == i0 == i64, res
    assert _bits(s1) == _bits(s0) == _bits(s64), res
    assert self.pruned.query('last_selfcheck_violations') == 0.0
    return s1, i1, self.pruned.query('last_survivors'), self.pruned.query('last_pruned_candidates')


def _acq(B, name, Y, **kw):
  if name == 'ei':
    return B.device.make_acq_desc('ei', best=kw.get('best', float(Y.max())))
  if name == 'pi':
    return B.device.make_acq_desc('pi', best=kw.get('best', float(Y.max())))
  return B.device.make_acq_desc('ucb', beta=kw.get('beta', 3.0))


@pytest.fixture(scope='module')
def small(B):
  rs = np.random.RandomState(21)
  X = rs.random_sample((N_SMALL, 6))
  Y = B.synth.hartmann6(X)
  Y = Y - float(np.median(Y))
  kern = B.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)
  return Namespace(X=X, Y=Y, trio=Trio(B, X, Y, kern, 0.01 * float(Y.var())), rs=rs)


# ---- the headline shape ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def headline(B):
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_cand=16)
  k = w['kernel']
  kern = B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])
  Yc = w['Y'] - w['mean_const']
  posts = [_post(B, w['X'], Yc, kern, w['noise_var'], 0, impl, prune) for impl, prune in ((2, 1), (2, 0), (0, 1))]
  trio = Trio.__new__(Trio)
  trio.B, trio.pruned, trio.full, trio.fp64 = B, posts[0], posts[1], posts[2]
  trio.posts = tuple(posts)
  host = np.random.RandomState(1000).random_sample((1000000, 6))           # bench.py's rank-0 candidates
  return Namespace(w=w, trio=trio, C=B.torch.from_numpy(host).cuda())


@pytest.mark.parametrize('acq_name', ['ei', 'ucb', 'pi'])
def test_headline(B, headline, acq_name):
  w = headline.w
  acq = (B.device.make_acq_desc('ucb', beta=float(np.sqrt(0.2 * 6 * np.log(2 * 6 * 5000 + 1))))
         if acq_name == 'ucb' else _acq(B, acq_name, w['Y']))
  s, i, surv, pruned = headline.trio.score(acq, headline.C, mean_const=w['mean_const'])
  m = len(headline.C)
  chunk = headline.trio.pruned.query('chunk')
  print('headline %s: survivors %d, pruned %d of %d' % (acq_name, surv, pruned, m))
  assert 0 <= surv < 0.01 * m
  assert surv + pruned == m - chunk
  assert 1 <= headline.trio.pruned.query('last_shortlist') <= 64


# ---- edges ----------------------------------------------------------------------------------------------------------
def test_exact_ties_split_across_chunks(B, small):
  C = small.rs.random_sample((6 * CHUNK + 77, 6))
  acq = _acq(B, 'ei', small.Y)
  _, i, _, _ = small.trio.score(acq, C)
  positions = (CHUNK + 13, 3 * CHUNK + 2, 5 * CHUNK + 70)
  assert i not in positions
  for pos in positions:                                         # three copies of the winner, none in the seed chunk
    C[pos] = C[i]
  C[i] = small.rs.random_sample(6) * 0.01 + 2.0                 # far from the data: no longer a contender
  s, i2, surv, pruned = small.trio.score(acq, C)
  assert i2 == CHUNK + 13 and pruned > 0


def test_nan_candidate_in_a_late_chunk_wins(B, small):
  C = small.rs.random_sample((5 * CHUNK + 9, 6))
  C[4 * CHUNK + 500, 2] = np.nan
  for name in ('ei', 'ucb', 'pi'):
    s, i, _, pruned = small.trio.score(_acq(B, name, small.Y), C)
    assert i == 4 * CHUNK + 500 and np.isnan(s) and pruned > 0


def test_candidates_on_training_points(B, small):
  C = small.rs.random_sample((4 * CHUNK, 6))
  C[CHUNK:CHUNK + 600] = small.X[:600]
  C[3 * CHUNK + 1] = small.X[int(np.argmax(small.Y))]
  for name in ('ei', 'ucb', 'pi'):
    small.trio.score(_acq(B, name, small.Y), C)


def test_unreachable_incumbent(B, small):
  C = small.rs.random_sample((4 * CHUNK + 3, 6))
  for name in ('ei', 'pi'):
    for above in (0.5, 50.0):          # small but positive scores; scores that underflow to exact zeros everywhere
      small.trio.score(_acq(B, name, small.Y, best=float(small.Y.max()) + above), C)


def test_large_ucb_beta(B, small):
  C = small.rs.random_sample((3 * CHUNK + 100, 6))
  _, _, surv, pruned = small.trio.score(_acq(B, 'ucb', small.Y, beta=50.0), C)
  assert surv + pruned == len(C) - CHUNK


def test_survivor_list_overflow(B, small):
  """ Candidates far from the data all have sigma = sqrt(k**) to the last bit and a large UCB beta puts them at the
      top: every one of them survives, the list (4 chunks) overflows and chunks 1.. are contracted as without the
      screen. """
  C = 3.0 + small.rs.random_sample((7 * CHUNK + 5, 6))
  _, _, surv, pruned = small.trio.score(_acq(B, 'ucb', small.Y, beta=50.0), C)
  assert surv > 4 * CHUNK and pruned == 0


@pytest.mark.parametrize('m', [CHUNK, CHUNK + 1])
def test_m_around_the_chunk(B, small, m):
  C = small.rs.random_sample((m, 6))
  for name in ('ei', 'ucb', 'pi'):
    _, _, surv, pruned = small.trio.score(_acq(B, name, small.Y), C)
    if m == CHUNK:
      assert surv == 0 and pruned == 0
    else:
      assert surv + pruned == 1


SPACES = ['pageable', 'pinned', 'device']


# 12 chunks: > half the staging buffer, the double-buffered copy of page-locked candidates.  45 chunks: at d = 6 a staging
# batch is 21 chunks, so the bound pass of pageable candidates crosses three batches, page-locked ones five halves.
@pytest.mark.parametrize('space,m', [(s, 12 * CHUNK + 5) for s in SPACES] + [(s, 45 * CHUNK + 5) for s in SPACES],
                         ids=SPACES + [s + '-45chunks' for s in SPACES])
def test_candidate_memory_spaces(B, small, space, m):
  host = small.rs.random_sample((m, 6))
  if space == 'pageable':
    C = host
  else:
    t = B.torch.empty((m, 6), dtype=B.torch.float64, pin_memory=True)
    t.numpy()[:] = host
    C = t.numpy() if space == 'pinned' else t.cuda()
  for name in ('ei', 'ucb', 'pi'):
    _, _, _, pruned = small.trio.score(_acq(B, name, small.Y), C)
    assert pruned > 0


def test_hallucinated_posterior(B, small):
  """ Evaluations in progress: the posterior extended by hallucinated points (their noise + jitter on the diagonal),
      the mean of the un-augmented one (eval_with_hallucinated_observations). """
  Xh = small.rs.random_sample((5, 6))
  for p in small.trio.posts:
    _, alpha, _ = p.get_state(want_alpha=True)
    assert p.extend(Xh, np.zeros(5), save=True)[0] == 0
    p.set_alpha(alpha)
  try:
    C = small.rs.random_sample((4 * CHUNK + 11, 6))
    C[2 * CHUNK:2 * CHUNK + 5] = Xh
    for name in ('ei', 'ucb', 'pi'):
      small.trio.score(_acq(B, name, small.Y), C)
  finally:
    for p in small.trio.posts:
      p.restore(N_SMALL)


def test_off_for_ttei_scores_and_negative_beta(B, small):
  C = small.rs.random_sample((3 * CHUNK, 6))
  p = small.trio.pruned
  for acq in (B.device.make_acq_desc('ttei', ref_mean=float(small.Y.max()) - 0.2, ref_std=0.1),
              B.device.make_acq_desc('ucb', beta=-1.0)):
    small.trio.score(acq, C)
    assert p.query('last_survivors') == 0 and p.query('last_pruned_candidates') == 0
  p.set_option('score_impl', 1)                  # a score vector is asked for: every candidate is contracted
  try:
    p.score_argmax(_acq(B, 'ei', small.Y), C, want_scores=True)
    assert p.query('last_pruned_candidates') == 0
  finally:
    p.set_option('score_impl', 2)


# ---- the mu-only segment kernel ------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', list(range(1, 9)))
@pytest.mark.parametrize('kname', list(R.KINDS))
def test_mu_only_variant_is_bit_identical(B, kname, d):
  """ mu of the mu-only kernel (mean-only dfb_eval) == mu of the digit kernel (score_impl 1, radix 256) == mu of the
      fp64-row kernel (score_impl 0), bit for bit. """
  kind, p = R.KINDS[kname]
  rs = np.random.RandomState(40 + d)
  X = rs.random_sample((300, d)); Y = np.sin(3.0 * X).sum(axis=1)
  C = rs.random_sample((700, d)); C[:50] = X[:50]
  bw = list(0.2 + 0.6 * rs.random_sample(d))
  kern = B.kernel.SEKernel(d, 1.3, bw) if kind == 'se' else B.kernel.MaternKernel(d, p + 0.5, 1.3, bw)
  post = _post(B, X, Y, kern, 0.013, 256, 0)
  mu64, _ = post.eval(C, mean_const=0.25)
  mu_only, sd = post.eval(C, mean_const=0.25, want_std=False)
  assert sd is None
  for k, v in (('score_impl', 1), ('i8_radix', 1), ('i8_unguarded', 1)):
    post.set_option(k, v)
  mu8, _ = post.eval(C, mean_const=0.25)
  assert post.query('last_used_i8') == 1.0 and post.query('i8_radix256') == 1.0
  assert (mu_only.view(np.int64) == mu8.view(np.int64)).all()
  assert (mu_only.view(np.int64) == mu64.view(np.int64)).all()
