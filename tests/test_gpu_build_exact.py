"""
The posterior build (api.cu: factorise_tall and posterior_tail) against the componentwise a-posteriori bounds of
tests/build_ref.py, and bit for bit against itself across its schedules (-m gpu).

  B1. L, W = L^-1, the y row v = (L^-1 y_c)^T, alpha and the LML of every build flag meet their bounds, at the tile
      edges n = 1 .. 1100 and sampled at n = 5000, for SE, Matern 1/2, 3/2, 5/2, an additive kernel, the multi-fidelity
      product and an ExpDecay kernel, well- and ill-conditioned (clustered points, noise 1e-10 of the scale, a jitter).
  B2. The padding of L, W, alpha and v is exact identity or zero; W is exactly the transpose of the L^-T block and
      exactly lower triangular; an LML-only build leaves the same L and v bits as a full one.
  B3. The look-ahead schedule and the single-stream one give the same bits (nb = 4, 5, 8, 40); so do repeated builds on
      one handle and a build on a caller stream.
  B4. `info` of a non-positive or NaN pivot is LAPACK's, and the handle builds correctly afterwards.
  B5. The factor left by dfb_extend_posterior meets the bounds of its replay.
Each test prints the largest residual / bound ratio per output ("RATIO" lines).  The outputs are read back whole with
dfb_debug_copy ("T", "W", "alpha"); A is the device's own K (dfb_get_state) with fl(K_ii + fl(noise + jitter)).
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import build_ref as BR

pytestmark = pytest.mark.gpu

FULL, LML_ONLY, NO_ALPHA = 0, 1, 2
REPEATS = 3                    # builds of one matrix compared with each other


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  assert np.finfo(np.longdouble).nmant >= 63, 'the residuals need an extended long double'
  from dragonfly_b200 import device, kernel, _lib
  _lib.load()
  return Namespace(torch=torch, device=device, kernel=kernel, lib=_lib)


def kernels(G):
  k = G.kernel
  return {
    'se': (k.SEKernel(4, 1.3, [0.3, 0.5, 0.4, 0.6]), 4),
    'matern12': (k.MaternKernel(4, 0.5, 1.3, 0.4), 4),
    'matern32': (k.MaternKernel(4, 1.5, 1.3, 0.4), 4),
    'matern52': (k.MaternKernel(4, 2.5, 1.3, 0.4), 4),
    'additive': (k.AdditiveKernel(0.35, [k.MaternKernel(2, 2.5, 1.0, 0.5), k.SEKernel(2, 1.0, 0.4)],
                                  [[0, 1], [2, 3]]), 4),
    'mf_product': (k.CoordinateProductKernel(4, 0.7, [k.SEKernel(1, 1.0, [0.7]), k.MaternKernel(3, 2.5, 1.0, 0.4)],
                                             [[0], [1, 2, 3]]), 4),
    'expdecay': (k.ExpDecayKernel(2, 1.0, 0.1, [1.0, 2.0]), 2),
  }


def points(kind, n, d, seed):
  rs = np.random.RandomState(seed)
  if kind == 'clustered':                 # a few tight clusters: nearly equal rows, K numerically singular
    return rs.random_sample((5, d))[rs.randint(0, 5, n)] + 1e-4 * rs.random_sample((n, d))
  return rs.random_sample((n, d))


def _ptr(t):
  return C.c_void_p(t.data_ptr())


def _copy(G, post, name, shape):
  t = G.torch.empty(shape, dtype=G.torch.float64, device=post.device)
  G.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), _ptr(t), t.numel() * 8), 'dfb_debug_copy')
  return t.cpu().numpy()


def bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def same_bits(a, b):
  return a.shape == b.shape and np.array_equal(bits(a), bits(b))


class Case(object):
  """ One handle with a kernel and a training set (X, y_c); read() returns the outputs of its last build. """

  def __init__(self, G, kern, d, X, y, n_max=None):
    self.G, self.X, self.y = G, X, np.asarray(y, dtype=np.float64)
    self.post = G.device.DevicePosterior(n_max or len(X), chunk=256)
    self.post.set_kernel(G.kernel.build_descriptor(kern, train_dim=d, cand_dim=d))
    self.post.set_train(X, self.y)
    self.npad = int(self.post.query('npad'))

  def build(self, noise, jitter=0.0, flags=FULL):
    self.n_built = self.post.n
    return self.post.build(noise, jitter, flags)

  def read(self, noise_plus_jitter, lml, with_w=True):
    G, npad, n = self.G, self.npad, self.post.n
    Tm = _copy(G, self.post, 'T', (2 * npad + BR.T, npad))
    W = _copy(G, self.post, 'W', (npad, npad)) if with_w else None
    alpha = _copy(G, self.post, 'alpha', (npad,))
    _, _, K = self.post.get_state(want_K=True)
    K = K.cpu().numpy()
    # the K of dfb_get_state is the one the build factorised: the top's tiles right of the diagonal keep it (over the
    # points of the full build; an extension rebuilds the last row block only)
    nb_ = self.n_built
    for I in range(npad // BR.T):
      r = slice(I * BR.T, min((I + 1) * BR.T, nb_))
      c0 = (I + 1) * BR.T
      if c0 < nb_:
        assert same_bits(Tm[r, c0:nb_], K[r, c0:nb_]), 'dfb_get_state K differs from the factorised K (row block %d)' % I
    return Namespace(T=Tm, L=np.tril(Tm[:npad]), X=Tm[npad:2 * npad], v=Tm[2 * npad].copy(), W=W, alpha=alpha,
                     A=BR.pad_matrix(K, noise_plus_jitter, npad), y=BR.pad_vector(self.y[:n], npad), lml=lml, n=n,
                     npad=npad)


def make_case(G, kname, n, kind='well', seed=0, n_max=None):
  kern, d = kernels(G)[kname]
  X = points(kind, n, d, seed + 7 * n)
  y = np.random.RandomState(seed + 1).standard_normal(n)
  return Case(G, kern, d, X, y, n_max=n_max)


def report(tag, r):
  print('RATIO %-40s %s' % (tag, ' '.join('%s=%.3g' % (k, v) for k, v in sorted(r.items()))))


def check_b1(o, flags, tag, rows=None, W=None, replay=False):
  W = o.W if W is None else W
  if flags == FULL:
    r = BR.check_build(o.A, o.y, o.L, W, o.v, alpha=o.alpha, lml=o.lml, lml_quad='alpha', n=o.n, rows=rows,
                       replay=replay)
  else:
    r = BR.check_build(o.A, o.y, o.L, W, o.v, lml=o.lml, lml_quad='v', n=o.n, rows=rows, replay=replay)
  report(tag, r)
  assert max(r.values()) <= 1.0, (tag, r)
  return r


def check_b2(o):
  n, npad = o.n, o.npad
  L, X, W = o.L, o.X, o.W
  eye = np.eye(npad)
  assert same_bits(L[n:], eye[n:]), 'padding rows of L are not exact identity rows'
  for I in range(npad // BR.T):          # above the diagonal inside the diagonal tiles: exact zeros
    s = BR.blk(I)
    assert (np.triu(o.T[s, s], 1) == 0).all()
  assert (o.v[n:] == 0).all() and (o.T[2 * npad + 1:] == 0).all(), 'y row padding / rows 1.. of its block'
  assert (o.alpha[n:] == 0).all(), 'alpha padding'
  if W is not None:
    assert same_bits(W, np.ascontiguousarray(X.T)), 'W is not exactly the transpose of the L^-T block'
    assert (np.triu(W, 1) == 0).all(), 'W has non-zeros above its diagonal'
    assert (W[n:, :n] == 0).all() and same_bits(W[n:, n:], eye[n:, n:]), 'padding of W'


# ---- B1 + B2 ------------------------------------------------------------------------------------------------------------
SIZES = [1, 2, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1100]


@pytest.mark.parametrize('n', SIZES)
def test_se_bounds_and_structure_at_tile_edges(G, n):
  c = make_case(G, 'se', n)
  noise = 1e-3 * 1.3
  info, lml = c.build(noise)
  assert info == 0
  o = c.read(noise, lml)
  check_b2(o)
  check_b1(o, FULL, 'se n=%d FULL' % n)


@pytest.mark.parametrize('kname', ['se', 'matern12', 'matern32', 'matern52', 'additive', 'mf_product', 'expdecay'])
def test_kernels_bounds_and_structure(G, kname):
  n = 513
  c = make_case(G, kname, n, seed=3)
  noise = 1e-2
  info, lml = c.build(noise)
  assert info == 0
  o = c.read(noise, lml)
  check_b2(o)
  check_b1(o, FULL, '%s n=%d FULL' % (kname, n))


@pytest.mark.parametrize('kname,n', [('se', 300), ('se', 1100), ('matern12', 513), ('matern52', 1100),
                                     ('additive', 513)])
def test_ill_conditioned_bounds(G, kname, n):
  """ Clustered points and noise 1e-10 of the scale: forward errors are useless here, the bounds are not. """
  c = make_case(G, kname, n, kind='clustered', seed=5)
  noise = 1e-10                           # every kernel here has scale ~1
  info, lml = c.build(noise)
  assert info == 0
  o = c.read(noise, lml)
  check_b2(o)
  check_b1(o, FULL, '%s n=%d ill' % (kname, n))


def test_jitter_build_bounds(G):
  """ A build the jitter ladder would make: clustered points, tiny noise, jitter 1e-8 of max(diag K). """
  c = make_case(G, 'matern32', 640, kind='clustered', seed=9)
  noise = 1e-10
  c.build(noise)
  jitter = 1e-8 * c.post.max_diag()
  info, lml = c.build(noise, jitter)
  assert info == 0
  o = c.read(np.float64(noise) + np.float64(jitter), lml)
  check_b2(o)
  check_b1(o, FULL, 'matern32 n=640 jitter')


@pytest.mark.parametrize('n', [257, 1100])
def test_flags_no_alpha_and_lml_only(G, n):
  c = make_case(G, 'matern52', n, seed=11)
  noise = 1e-3
  info, lml = c.build(noise, flags=FULL)
  full = c.read(noise, lml)
  info, lml = c.build(noise, flags=NO_ALPHA)
  assert info == 0
  o = c.read(noise, lml)
  check_b2(Namespace(**dict(vars(o), alpha=np.zeros(o.npad))))
  assert same_bits(o.T[:o.npad], full.T[:o.npad]) and same_bits(o.W, full.W)
  check_b1(o, NO_ALPHA, 'matern52 n=%d NO_ALPHA' % n)
  info, lml = c.build(noise, flags=LML_ONLY)
  assert info == 0
  o = c.read(noise, lml, with_w=False)
  # the same L bits and y row as the full build; its D_J (W's diagonal tiles) are therefore the full build's
  assert same_bits(o.T[:o.npad], full.T[:o.npad]) and same_bits(o.v, full.v)
  check_b1(o, LML_ONLY, 'matern52 n=%d LML_ONLY' % n, W=full.W)


def test_n5000_sampled_rows(G):
  """ Every row at a block boundary and a seeded sample of others, all columns of each. """
  n = 5000
  c = make_case(G, 'se', n, seed=13)
  noise = 1e-4
  info, lml = c.build(noise)
  assert info == 0
  o = c.read(noise, lml)
  check_b2(o)
  b = np.arange(BR.T, o.npad, BR.T)
  rows = np.unique(np.concatenate([[0], b - 1, b, np.random.RandomState(5000).choice(o.npad, 16, replace=False)]))
  check_b1(o, FULL, 'se n=5000 FULL sampled', rows=rows)


# ---- B3: schedules ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('nb', [4, 5, 8, 40])
def test_lookahead_is_bit_identical(G, nb):
  n = nb * BR.T - 37
  c = make_case(G, 'matern52', n, seed=17)
  outs = []
  for la in (1, 0):
    c.post.set_option('lookahead', la)
    info, lml = c.build(1e-3)
    assert info == 0
    outs.append(c.read(1e-3, lml))
  c.post.set_option('lookahead', 1)
  a, b = outs
  assert same_bits(a.T, b.T) and same_bits(a.W, b.W) and same_bits(a.alpha, b.alpha) and a.lml == b.lml


@pytest.mark.parametrize('n', [700, 2600])
def test_repeated_builds_and_caller_stream_are_bit_identical(G, n):
  c = make_case(G, 'se', n, seed=19)
  outs = []
  for _ in range(REPEATS):
    info, lml = c.build(1e-3)
    assert info == 0
    outs.append(c.read(1e-3, lml))
  torch = G.torch
  s = torch.cuda.Stream(device=c.post.device)
  G.lib.check(c.post.lib.dfb_set_stream(c.post.h, C.c_void_p(s.cuda_stream)), 'dfb_set_stream')
  try:
    info, lml = c.build(1e-3)
    s.synchronize()
    assert info == 0
    outs.append(c.read(1e-3, lml))
  finally:
    c.post.bind_current_stream()
  for o in outs[1:]:
    assert same_bits(o.T, outs[0].T) and same_bits(o.W, outs[0].W) and same_bits(o.alpha, outs[0].alpha)
    assert o.lml == outs[0].lml


# ---- B4: info -------------------------------------------------------------------------------------------------------------
def _info_case(G, n, bad, nan=False):
  """ A handle whose matrix has its first non-positive (or NaN) pivots at the global indices `bad`, the noise that makes
      it so, and A itself (K from dfb_kernel_matrix). """
  rs = np.random.RandomState(100 + n + sum(bad))
  if nan:
    kern, d = G.kernel.ExpDecayKernel(1, 1.0, 0.1, [1.5]), 1
    X = rs.random_sample((n, d))
    X[bad[0]] = np.nan
    noise = 1e-2
  else:
    # SE with a short bandwidth in 6 dimensions: K is close to scale * I; a point equal to its predecessor makes K
    # singular there, and noise -0.02 scale turns that pivot to about -0.04 scale while every earlier one stays near
    # 0.98 scale
    kern, d = G.kernel.SEKernel(6, 1.0, 0.03), 6
    X = rs.random_sample((n, d))
    for j in bad:
      if j > 0:
        X[j] = X[j - 1]
    noise = -1.1 if bad[0] == 0 else -0.02
  c = Case(G, kern, d, X, rs.standard_normal(n))
  A = G.device.kernel_matrix(kern, X, X)
  A[np.diag_indices(n)] += np.float64(noise)
  return c, A, noise


def lapack_info(A):
  """ LAPACK's dpotrf info: the first pivot that is not positive, NaN included (the reference dpotrf tests DISNAN;
      SciPy's optimised one does not, so a NaN diagonal entry is located directly, behind a positive definite leading
      block). """
  from scipy.linalg.lapack import dpotrf
  nan = np.argwhere(np.isnan(np.diag(A)))
  if len(nan):
    j = int(nan[0][0])
    assert dpotrf(A[:j, :j], lower=1)[1] == 0
    return j + 1
  return dpotrf(A, lower=1)[1]


def _good_build_after(c, tag):
  """ The same handle after a failed build, a positive noise: the build succeeds and meets B1 and B2. """
  if np.isnan(c.X).any():
    c.X = np.nan_to_num(c.X, nan=0.5)
    c.post.set_train(c.X, c.y)
  info, lml = c.build(0.5)
  assert info == 0
  o = c.read(0.5, lml)
  check_b2(o)
  check_b1(o, FULL, tag)


@pytest.mark.parametrize('n', [300, 600])
@pytest.mark.parametrize('j', [0, 1, 127, 128, 129, -1])
def test_info_matches_lapack(G, n, j):
  j = n - 1 if j < 0 else j
  c, A, noise = _info_case(G, n, [j])
  want = lapack_info(A)
  assert want == j + 1, 'the construction did not place the first bad pivot at %d (LAPACK: %d)' % (j, want)
  info, _ = c.build(noise)
  assert info == want
  _good_build_after(c, 'after info=%d n=%d' % (info, n))


def test_info_nan_and_two_bad_pivots(G):
  n = 300
  c, A, noise = _info_case(G, n, [200], nan=True)
  want = lapack_info(A)
  info, _ = c.build(noise)
  assert info == want == 201
  _good_build_after(c, 'after NaN n=%d' % n)
  c, A, noise = _info_case(G, n, [129, 290])
  want = lapack_info(A)
  info, _ = c.build(noise)
  assert info == want == 130
  _good_build_after(c, 'after two bad pivots n=%d' % n)


# ---- B5: extension --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n0,q', [(300, 84), (300, 1), (1000, 24)])
def test_extended_factor_meets_the_replay_bounds(G, n0, q):
  kern, d = kernels(G)['matern52']
  n = n0 + q
  X = points('well', n, d, 23 + n)
  y = np.random.RandomState(n).standard_normal(n)
  c = Case(G, kern, d, X[:n0], y[:n0], n_max=n)
  noise = 1e-3
  info, _ = c.build(noise)
  assert info == 0
  info, lml = c.post.extend(X[n0:], y[n0:], flags=FULL)
  assert info == 0
  c.y = y
  o = c.read(noise, lml)
  check_b2(o)
  check_b1(o, FULL, 'extend %d+%d' % (n0, q), replay=True)
