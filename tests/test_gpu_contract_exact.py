"""
The fp64 DMMA contractions (gemm.cuh, gemm_tma.cuh, small_sumsq_kernel) and the products built on them against the
extended-precision bounds of tests/contract_ref.py, and bit for bit against themselves (-m gpu).

  C1. Score partials: both gemm_impl values and the small path (m <= 32) at the tile edges of n and m and three chunk
      sizes, SE and Matern 1/2, 3/2, 5/2, well- and ill-conditioned (clustered points, noise 1e-10 of the scale, where
      sigma^2 is almost all cancellation).  Every partial read back meets its bound, and sd equals acq_kernel's
      epilogue replayed on the host from the device's partials and k(x*, x*), bit for bit.  Chunks before the last are
      checked through C2: each is scored again on its own, and must give the same bits.
  C2. Per gemm_impl, a candidate's mu, sd and score do not depend on its column or chunk, the chunk size,
      tma_cb_group, the rest of the batch, where the candidates live (host, page-locked, device) or repetition.  The
      two kernels contract k in different lane orders, so across gemm_impl only the bound of C1 is required.
  C3. dfb_eval_covar: the covariance meets the covariance bound on every tile; its padding is exact zero.
  C4. dfb_ts_draws: the lower tiles of ts_Cov are those of dfb_eval_covar, bit for bit; the factor in ts_T meets the
      factorisation bound for fl(Cov + jitter) with identity padding; samples - mu meet the L U product bound; a TS
      workspace filled with NaN bytes before the call gives the same bits (every integer field of the TS workspace is
      cleared by the call, so this checks values only).
  C5. dfb_lml_gradients at the tile edges of n, SE and Matern 1/2, 3/2, 5/2, d = 1, 3, 8: the K^-1 = W^T W tiles (one
      stripe, read from Ks) meet the tri = 3 product bound, the gradient vector meets its bound (contract_ref, 6), and
      it is bit-identical across chunk sizes that give 1, 2 and nb stripes.  Training points 1e-9 of a bandwidth apart
      give finite gradients within their bound; coincident points give NaN exactly where the oracle's
      Kernel.gradient does.
  C6. C1, C3 and C5 on a pooled workspace just used by a larger, different problem, and on a zero-filled one: the same
      bits.
Each check prints its largest residual / bound ratio ("RATIO" lines).
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import contract_ref as CR

pytestmark = pytest.mark.gpu

T = CR.T
NU = {'se': None, 'matern12': 0.5, 'matern32': 1.5, 'matern52': 2.5}
KIND = {'se': ('se', 0), 'matern12': ('matern', 0), 'matern32': ('matern', 1), 'matern52': ('matern', 2)}
SCALE = 1.3


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  assert np.finfo(np.longdouble).nmant >= 63, 'the residuals need an extended long double'
  from dragonfly_b200 import device, kernel, _lib
  _lib.load()
  return Namespace(torch=torch, device=device, kernel=kernel, lib=_lib, cache={})


def _copy(G, post, name, count):
  t = G.torch.empty((count,), dtype=G.torch.float64, device=post.device)
  G.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), t.numel() * 8), 'dfb_debug_copy')
  return t.cpu().numpy()


def bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def assert_same(a, b, what):
  a, b = np.asarray(a), np.asarray(b)
  assert a.shape == b.shape, (what, a.shape, b.shape)
  bad = np.argwhere(bits(a) != bits(b))
  assert len(bad) == 0, (what, 'differs in', len(bad), 'entries; first', tuple(bad[0]), a[tuple(bad[0])],
                         b[tuple(bad[0])])


def report(tag, r):
  print('RATIO %-48s %s' % (tag, ' '.join('%s=%.3g' % (k, v) for k, v in sorted(r.items()))))
  assert max(r.values()) <= 1.0, (tag, r)


class Post(object):
  """ One built posterior: kernel kname in d dimensions, n training points, scoring chunk `chunk` (0: default). """

  def __init__(self, G, kname, n, d=3, chunk=0, kind='well', seed=0, n_max=None):
    self.G, self.kname, self.d, self.n = G, kname, d, n
    rs = np.random.RandomState(seed + 31 * n + d)
    self.bw = 0.3 + 0.4 * rs.random_sample(d)
    if kind == 'clustered':
      self.X = rs.random_sample((5, d))[rs.randint(0, 5, n)] + 1e-4 * rs.random_sample((n, d))
      self.noise = 1e-10 * SCALE
    else:
      self.X = rs.random_sample((n, d))
      self.noise = 1e-3 * SCALE
    self.y = np.sin(3 * self.X).sum(axis=1)
    k = G.kernel
    kern = k.SEKernel(d, SCALE, list(self.bw)) if NU[kname] is None else k.MaternKernel(d, NU[kname], SCALE, list(self.bw))
    self.post = G.device.DevicePosterior(n_max or n, chunk=chunk)
    self.post.set_kernel(k.build_descriptor(kern, train_dim=d, cand_dim=d))
    self.post.set_train(self.X, self.y)
    info, _ = self.post.build(self.noise)
    assert info == 0
    self.npad = int(self.post.query('npad'))
    self.chunk = int(self.post.query('chunk'))
    self.nb = self.npad // T
    self.W = _copy(G, self.post, 'W', self.npad * self.npad).reshape(self.npad, self.npad)

  def opt(self, **kw):
    for k, v in kw.items():
      self.post.set_option(k, v)

  def cands(self, m, seed=1):
    return np.random.RandomState(seed + m).random_sample((m, self.d))

  def kern_ref(self, Xc):
    kind, p = KIND[self.kname]
    return (kind, p, SCALE, self.bw, Xc)


def posterior(G, kname, n, d=3, chunk=0, kind='well'):
  key = (kname, n, d, chunk, kind)
  if key not in G.cache:
    G.cache[key] = Post(G, kname, n, d, chunk, kind)
  return G.cache[key]


def sample_cols(mc, seed, k=24):
  edges = [0, 1, 7, 8, 9, 31, 32, 33, 126, 127, 128, 129, mc - 2, mc - 1]
  rs = np.random.RandomState(seed)
  extra = rs.choice(mc, min(mc, k), replace=False)
  return np.unique([c for c in edges if 0 <= c < mc] + list(extra))


# ---- C1: partials and the exact epilogue ----------------------------------------------------------------------------------
def score_check(P, Xc, impl, small, tag):
  """ Scores Xc (host), checks the last chunk's partials against their bound and every sd of that chunk against the
      replayed epilogue; returns (mu, sd). """
  G = P.G
  P.opt(gemm_impl=impl, small_eval=1 if small else 0, score_impl=0)
  mu, sd = P.post.eval(Xc)
  m = len(Xc)
  c0 = (m - 1) // P.chunk * P.chunk
  mc = m - c0
  part = _copy(G, P.post, 'partial', P.nb * P.chunk)
  kss = _copy(G, P.post, 'kssv', P.chunk)[:mc]
  Ks = _copy(G, P.post, 'Ks', P.chunk * P.npad).reshape(P.chunk, P.npad)
  m_rows = -(-mc // T) * T
  assert (Ks[:mc, P.n:] == 0).all() and (Ks[mc:m_rows] == 0).all(), 'K_* padding is not exact zero'
  use_small = small and m <= 32 and (P.n + 7) // 8 * 8 * 32 <= P.nb * P.chunk
  if use_small:
    rows = (P.n + 7) // 8 * 8
    parts = part[:rows * 32].reshape(rows, 32)[:, :mc]
    assert (parts[P.n:] == 0).all()
    Pe, B = CR.small_partials(P.W, Ks, P.n, np.arange(mc))
    r = CR._ratio(CR._ld(parts[:P.n]) - Pe, B)
  else:
    parts = part.reshape(P.nb, P.chunk)[:, :mc]
    cols = sample_cols(mc, m)
    Pe, B = CR.score_partials(P.W, Ks, cols)
    r = CR._ratio(CR._ld(parts[:, cols]) - Pe, B)
  _, sd_host = CR.epilogue(parts, kss)
  assert_same(sd[c0:], sd_host, tag + ' sd vs the replayed epilogue')
  report(tag, {'partial': r})
  return mu, sd


N_EDGES = [1, 2, 15, 16, 17, 127, 128, 129, 255, 256, 257, 383, 385, 1100]


@pytest.mark.parametrize('impl', [0, 1])
@pytest.mark.parametrize('n', N_EDGES + [2600 + int(np.random.RandomState(2600).randint(-60, 60))])
def test_c1_partials_at_n_tile_edges(G, n, impl):
  P = posterior(G, 'se', n)
  score_check(P, P.cands(300), impl, False, 'C1 se n=%d m=300 impl=%d' % (n, impl))


def m_list(chunk):
  return sorted({1, 7, 8, 9, 32, 33, 127, 128, 129, chunk - 1, chunk, chunk + 1, 2 * chunk + 77})


@pytest.mark.parametrize('impl', [0, 1])
@pytest.mark.parametrize('chunk', [128, 256, 0])
def test_c1_c2_partials_at_m_tile_edges_and_chunks(G, chunk, impl):
  """ Every m of the list; for m > chunk each earlier chunk is scored on its own and must give the same bits (C2). """
  P = posterior(G, 'matern52', 257, chunk=chunk)
  for m in m_list(P.chunk):
    Xc = P.cands(m, seed=5)
    mu, sd = score_check(P, Xc, impl, False, 'C1 m=%d chunk=%d impl=%d' % (m, P.chunk, impl))
    for c0 in range(0, m - P.chunk, P.chunk):
      mu1, sd1 = score_check(P, Xc[c0:c0 + P.chunk], impl, False, 'C2 chunk %d of m=%d' % (c0 // P.chunk, m))
      assert_same(mu[c0:c0 + P.chunk], mu1, 'mu by chunk')
      assert_same(sd[c0:c0 + P.chunk], sd1, 'sd by chunk')


@pytest.mark.parametrize('n', [1, 2, 127, 128, 129, 1100])
def test_c1_small_path(G, n):
  P = posterior(G, 'se', n)
  for m in (1, 7, 8, 9, 32):
    Xc = P.cands(m, seed=9)
    mu, sd = score_check(P, Xc, 1, True, 'C1 small n=%d m=%d' % (n, m))
    for impl in (0, 1):                      # the tile kernels meet their own bound on the same candidates
      score_check(P, Xc, impl, False, 'C1 tile n=%d m=%d impl=%d' % (n, m, impl))


@pytest.mark.parametrize('kname', ['se', 'matern12', 'matern32', 'matern52'])
@pytest.mark.parametrize('impl', [0, 1])
def test_c1_kernels(G, kname, impl):
  P = posterior(G, kname, 257)
  score_check(P, P.cands(300), impl, False, 'C1 %s n=257 impl=%d' % (kname, impl))


@pytest.mark.parametrize('kname,n', [('se', 300), ('matern12', 513), ('matern52', 1100)])
def test_c1_ill_conditioned(G, kname, n):
  P = posterior(G, kname, n, kind='clustered')
  Xc = np.concatenate([P.X[:40] + 1e-6, P.cands(260)])       # near training points: sigma^2 is mostly cancellation
  for impl in (0, 1):
    score_check(P, Xc, impl, False, 'C1 ill %s n=%d impl=%d' % (kname, n, impl))


# ---- C2: invariances --------------------------------------------------------------------------------------------------
def scores(P, Xc, acq):
  mu, sd = P.post.eval(Xc)
  _, _, sc = P.post.score_argmax(acq, Xc, want_scores=True)
  to = lambda a: a.cpu().numpy() if hasattr(a, 'cpu') else np.asarray(a)
  return to(mu), to(sd), to(sc)


@pytest.mark.parametrize('impl', [0, 1])
def test_c2_bit_invariances(G, impl):
  acq = G.device.make_acq_desc('ucb', beta=2.0)
  m = 700
  base = None
  for chunk in (128, 256, 1024):
    P = posterior(G, 'matern32', 385, chunk=chunk)
    Xc = P.cands(m, seed=3)
    P.opt(gemm_impl=impl, small_eval=1, score_impl=0)
    ref = scores(P, Xc, acq)
    if base is None:
      base = ref
    for a, b, w in zip(ref, base, ('mu', 'sd', 'score')):
      assert_same(a, b, '%s: chunk %d vs 128' % (w, chunk))
    perm = np.random.RandomState(chunk).permutation(m)
    for a, b, w in zip(scores(P, Xc[perm], acq), ref, ('mu', 'sd', 'score')):
      assert_same(a, b[perm], '%s: permuted columns' % w)
    sub = np.arange(0, m, 3)
    for a, b, w in zip(scores(P, Xc[sub], acq), ref, ('mu', 'sd', 'score')):
      assert_same(a, b[sub], '%s: a sub-batch' % w)
    pinned = G.torch.empty((m, P.d), dtype=G.torch.float64).pin_memory()
    pinned.copy_(G.torch.from_numpy(Xc))
    for Xv, where in ((pinned.numpy(), 'page-locked'), (G.torch.from_numpy(Xc).cuda(), 'device'), (Xc, 'repeat')):
      for a, b, w in zip(scores(P, Xv, acq), ref, ('mu', 'sd', 'score')):
        assert_same(a, b, '%s: %s' % (w, where))
    if impl == 1:
      for grp in (1, 2, 3):
        P.opt(tma_cb_group=grp)
        for a, b, w in zip(scores(P, Xc, acq), ref, ('mu', 'sd', 'score')):
          assert_same(a, b, '%s: tma_cb_group %d' % (w, grp))
      P.opt(tma_cb_group=1 << 20)
  # the posterior itself does not depend on the chunk
  assert_same(posterior(G, 'matern32', 385, chunk=128).W, posterior(G, 'matern32', 385, chunk=1024).W, 'W by chunk')


# ---- C3: covariance ------------------------------------------------------------------------------------------------------
def covar_check(P, m, tag, seed=11):
  G = P.G
  Xc = P.cands(m, seed=seed)
  mu, cov = P.post.eval_covar(Xc)
  mbp = -(-m // T) * T
  Ks = _copy(G, P.post, 'Ks', P.chunk * P.npad).reshape(P.chunk, P.npad)
  tsc = _copy(G, P.post, 'ts_Cov', _ts_len(P))
  full = tsc[:mbp * mbp].reshape(mbp, mbp)
  assert_same(full[:m, :m], cov, tag + ' eval_covar output vs ts_Cov')
  assert (full[m:] == 0).all() and (full[:, m:] == 0).all(), tag + ' covariance padding is not exact zero'
  r = CR.covariance_check(cov, Ks[:m], P.W, P.kern_ref(Xc))
  report(tag, {'cov': r})
  return mu, cov, full


def _ts_len(P):
  mbp = -(-P.post._ts_mb // T) * T
  return mbp * mbp


@pytest.mark.parametrize('n', [128, 257])
@pytest.mark.parametrize('m', [1, 127, 128, 129, 300, 640])
def test_c3_covariance(G, m, n):
  P = posterior(G, 'matern52', n)
  covar_check(P, m, 'C3 m=%d n=%d' % (m, n))


# ---- C4: Thompson draws -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('m', [129, 300])
def test_c4_ts_draws(G, m):
  P = posterior(G, 'se', 257)
  mu, cov, full = covar_check(P, m, 'C4 covariance m=%d' % m, seed=13)
  mbp = -(-m // T) * T
  S = 5
  Ut = np.random.RandomState(m).standard_normal((S, m))
  jitter = 1e-6 * float(np.diag(cov).max())
  outs = []
  for fill in (None, 0xFF):
    if fill is not None:
      P.post._ts_workspace.fill_(fill)          # every double of the TS workspace is a NaN
    info, smp, _ = P.post.ts_draws(P.cands(m, seed=13), Ut, jitter=jitter)
    assert info == 0
    q = -(-P.post._ts_mb // T) * T
    tT = _copy(G, P.post, 'ts_T', (2 * q + T) * q)[:(2 * mbp + T) * mbp].reshape(2 * mbp + T, mbp)
    tc = _copy(G, P.post, 'ts_Cov', _ts_len(P))[:mbp * mbp].reshape(mbp, mbp)
    outs.append((smp.cpu().numpy(), np.tril(tT[:mbp]), tc))
  for smp, L, tc in outs:
    for I in range(mbp // T):
      for J in range(I + 1):
        s, t = slice(I * T, (I + 1) * T), slice(J * T, (J + 1) * T)
        assert_same(tc[s, t], full[s, t], 'ts_Cov lower tile (%d, %d) vs eval_covar' % (I, J))
  assert_same(outs[0][0], outs[1][0], 'samples after a NaN-filled TS workspace')
  assert_same(outs[0][1], outs[1][1], 'factor after a NaN-filled TS workspace')
  smp, L, _ = outs[0]
  A = np.eye(mbp)
  A[:m, :m] = full[:m, :m]
  idx = np.arange(m)
  A[idx, idx] = full[idx, idx] + np.float64(jitter)
  r = {'factor': CR.factor_check(A, L), 'samples': CR.draws_check(smp, mu, Ut, L[:m, :m])}
  report('C4 ts_draws m=%d' % m, r)


# ---- C5: LML gradients ---------------------------------------------------------------------------------------------------
def kinv_and_grad(G, kname, n, d, chunk, check=True):
  P = Post(G, kname, n, d=d, chunk=chunk, seed=d)
  g = P.post.lml_gradients(d)
  r = {}
  if check:
    assert P.chunk >= P.npad
    Ks = _copy(G, P.post, 'Ks', P.chunk * P.npad).reshape(P.chunk, P.npad)[:P.npad]
    Tm = _copy(G, P.post, 'T', (2 * P.npad + T) * P.npad).reshape(2 * P.npad + T, P.npad)
    Wt = Tm[P.npad:2 * P.npad]
    r['kinv'] = CR.generic_check(Wt, Wt, Ks, tri=3, lower_only=True)
    r['grad'] = grad_ratio(G, P, g)
  return P, g, r


def grad_ratio(G, P, g):
  """ The gradient vector against its bound (contract_ref, 6), from the device's alpha, W and training points. """
  alpha = _copy(G, P.post, 'alpha', P.npad)
  W = _copy(G, P.post, 'W', P.npad * P.npad).reshape(P.npad, P.npad)
  kind, p = KIND[P.kname]
  want, bound = CR.lml_gradients(kind, p, SCALE, P.bw, P.X, alpha, W)
  return float((np.abs(CR._ld(g) - want).astype(np.float64) / bound).max())


@pytest.mark.parametrize('kname,d', [('se', 3), ('matern12', 1), ('matern32', 8), ('matern52', 3)])
@pytest.mark.parametrize('n', [1, 2, 127, 128, 129, 257, 1100])
def test_c5_kinv_tiles_gradients_and_stripes(G, n, kname, d):
  npad = -(-n // T) * T
  nb = npad // T
  P, g1, r = kinv_and_grad(G, kname, n, d, max(npad, 256))
  report('C5 %s d=%d n=%d' % (kname, d, n), r)
  assert np.isfinite(g1).all()
  for chunk in sorted({-(-nb // 2) * T, T}):
    _, g, _ = kinv_and_grad(G, kname, n, d, chunk, check=False)
    assert_same(g, g1, 'gradients with chunk %d vs one stripe' % chunk)


@pytest.mark.parametrize('kname,d', [('se', 8), ('matern12', 3), ('matern32', 1), ('matern52', 8)])
def test_c5_gradients_other_dimensions(G, kname, d):
  P, g, r = kinv_and_grad(G, kname, 257, d, 384)
  report('C5 %s d=%d n=257' % (kname, d), r)


# ---- C6: stale and zeroed workspaces -----------------------------------------------------------------------------------------
def c6_run(G, dirty_ptr=None):
  """ C1, C3 and C5 on a fresh handle of n_max 640 (the pool key of the dirtying problem): their results.  dirty_ptr:
      the workspace the handle must have been given. """
  P = Post(G, 'matern32', 385, chunk=512, n_max=640, seed=77)
  if dirty_ptr is not None:
    assert P.post.workspace.data_ptr() == dirty_ptr, 'the pool did not hand the dirty workspace back'
  out = list(score_check(P, P.cands(900, seed=2), 1, False, 'C6 score'))
  out += list(covar_check(P, 300, 'C6 covariance')[:2])
  out.append(P.post.lml_gradients(P.d))
  del P
  return out


def test_c6_stale_and_zeroed_workspaces(G, monkeypatch):
  # a larger, different problem on a workspace of the same size: another kernel, the int8 path, gradients, draws
  dirty = Post(G, 'se', 640, d=6, chunk=512, seed=99)
  dirty.opt(score_impl=1)
  dirty.post.score_argmax(G.device.make_acq_desc('ucb', beta=2.0), dirty.cands(5000), want_scores=True)
  dirty.post.lml_gradients(6)
  dirty.post.ts_draws(dirty.cands(256), np.ones((3, 256)), jitter=1e-6)
  ptr = dirty.post.workspace.data_ptr()
  del dirty
  stale = c6_run(G, ptr)
  torch = G.torch
  monkeypatch.setattr(G.device, '_take_workspace',
                      lambda key, dev: torch.zeros(key[1] + 256, dtype=torch.uint8, device=dev))
  zeroed = c6_run(G)
  for a, b, w in zip(stale, zeroed, ('mu', 'sd', 'covariance mu', 'covariance', 'gradients')):
    assert_same(np.asarray(a), np.asarray(b), w + ': stale vs zeroed workspace')


# ---- C5: near-duplicate and coincident training points ---------------------------------------------------------------------
@pytest.mark.parametrize('kname', ['se', 'matern12', 'matern32', 'matern52'])
def test_c5_near_duplicates_give_finite_gradients(G, kname):
  """ Pairs of training points 1e-9 of a bandwidth apart, where the computed distance may flush to 0: the gradients are
      finite and meet their bound.  For Matern 1/2 the bound of the per-dimension entries is infinite at such pairs
      (contract_ref, 6b), so those entries are also held to the tolerance of test_gpu_grad.py: 1e-9 of the magnitude
      the gradient is a difference of, against the long-double gradient. """
  n, d = 257, 3
  P = Post(G, kname, n, d=d, seed=41)
  rs = np.random.RandomState(41)
  X = P.X.copy()
  v = rs.standard_normal((40, d))
  v /= np.linalg.norm(v, axis=1, keepdims=True)
  X[1:80:2] = X[0:80:2] + 1e-9 * P.bw * v
  P.X = X
  P.post.set_train(X, P.y)
  assert P.post.build(P.noise)[0] == 0
  g = P.post.lml_gradients(d)
  assert np.isfinite(g).all(), g
  W = _copy(G, P.post, 'W', P.npad * P.npad).reshape(P.npad, P.npad)
  alpha = _copy(G, P.post, 'alpha', P.npad)
  kind, p = KIND[kname]
  want, bound, mag = CR.lml_gradients(kind, p, SCALE, P.bw, X, alpha, W, with_mag=True)
  err = np.abs(CR._ld(g) - want).astype(np.float64)
  report('C5 near-duplicates %s' % kname, {'grad': float((err / bound).max())})
  assert (err <= 1e-9 * mag).all(), (err, mag)


@pytest.mark.parametrize('kname,d', [('matern12', 1), ('matern32', 3), ('matern52', 3), ('se', 3)])
def test_c5_coincident_points_give_the_oracles_nans(G, kname, d):
  """ Coincident training points on a dyadic grid (every distance exact): NaN exactly where OMaternKernel.gradient
      divides 0 by 0, finite elsewhere. """
  from oracle import gp_oracle as O
  n = 129
  rs = np.random.RandomState(d)
  X = rs.randint(0, 8, (n, d)) / 8.0
  X[1] = X[0]
  bw = [0.5] * d
  y = np.sin(3 * X).sum(axis=1)
  nu = NU[kname]
  k = G.kernel
  kern = k.SEKernel(d, SCALE, bw) if nu is None else k.MaternKernel(d, nu, SCALE, bw)
  post = G.device.DevicePosterior(n)
  post.set_kernel(k.build_descriptor(kern, train_dim=d, cand_dim=d))
  post.set_train(X, y)
  noise = 0.05
  assert post.build(noise)[0] == 0
  g = post.lml_gradients(d)
  okern = O.OSEKernel(d, SCALE, bw) if nu is None else O.OMaternKernel(d, nu, SCALE, bw)
  # the oracle's GP solves refuse NaN, so its gradient is NaN exactly where Kernel.gradient's matrix has one
  params = [('scale', ()), ('same_dim_bandwidths', ())] + [('dim_bandwidths', (q,)) for q in range(d)]
  with np.errstate(all='ignore'):
    nan = [bool(np.isnan(okern.gradient(pn, X, X, *a)).any()) for pn, a in params]
  want = np.array([np.nan if nan[0] else 0.0, 0.0, 0.0] + [np.nan if x else 0.0 for x in nan[1:]])
  assert np.array_equal(np.isnan(g), np.isnan(want)), (g, want)
  assert np.isnan(want).any() == (nu is not None)
