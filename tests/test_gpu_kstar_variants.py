"""
Every K_* kernel variant of the plain SE / Matern kernels, at every compiled dimension d = 1 .. 8 (-m gpu).

The K_* producer is picked at run time by the options, kernel kind and d (kernels.cu: route_kstar); each path below is
forced through the handle's options and read back with dfb_debug_copy:
  P1  kstar_kernel (the descriptor interpreter)        kstar_fast = 0
  P2  kstar_fast_kernel, fp64 rows                      kstar_rows64 = 0
  P3  cand_prep + kstar_seg_kernel<ROWS64>, fp64 rows   score_impl = 0 (the default fp64 build of dfb_eval)
  P4  cand_prep + kstar_seg_kernel, digit planes        score_impl = 1, i8_radix = 1, i8_unguarded = 1
  P5  kstar_fast_kernel<I8OUT>, radix 256               P4 + kstar_seg = 0
  P6  kstar_fast_kernel<I8OUT>, radix 128               score_impl = 1, i8_radix = 0, i8_unguarded = 1

Exact invariants (bit equality, int64 views):
  E1  Ks(P1) == Ks(P2), padding rows and columns (exact zeros) included: the same operation sequence;
  E2  sd(P1) == sd(P2): the same K_*, k(x*, x*) and contraction;
  E3  the planes of P5 are i8_exact.digits_radix256(Ks(P2) 2^-F); those of P6 are kstar_fast's own radix-128
      expansion of the same values (i8_exact.digits_radix128_split), which reconstructs to the same integer as the
      slice_i8 expansion;
  E4  the planes of P4 are the digits of Ks(P3) 2^-F, and mu(P4) == mu(P3): both kstar_seg variants form the kernel
      value and the mu partials with the same expressions;
  E5  the posterior built with kstar_fast = 1 and = 0 (K(X, X) by kstar_fast_kernel or the interpreter): L, alpha and
      the LML are identical.
Bounded checks against the longdouble reference (tests/kstar_ref.py, where the bounds are derived):
  B1  the fp64 rows of P1, P2, P3 and K(X, X) lie within kstar_bound;
  B2  mu of P1 .. P4 lies within mu_bound, with the device's own alpha;
  B3  Matern-1/2 at (candidate, training point) pairs that coincide or lie within 1e-9 .. 1e-3 of each other: P3
      within 4 ulp of P1 (kstar_seg keeps the reference's rounding order of D^2 there; only its fused scale constant
      and its sqrt without the Markstein step differ).
Measured: the whole file (180 tests) runs in about 55 s on one H100 80 GB.
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import i8_exact as IX
import kstar_ref as R

pytestmark = pytest.mark.gpu

KNAMES = list(R.KINDS)
N_MAIN, M_MAIN, CHUNK_MAIN = 129, 700, 1024
CHUNK_SMALL = 256
PATHS = ('P1', 'P2', 'P3', 'P4', 'P5', 'P6')
ROW_PATHS = ('P1', 'P2', 'P3')
N_NEAR = 64                  # candidate rows 0 .. 63: on training points, 64 .. 127: within 1e-9 .. 1e-3 of them


@pytest.fixture(scope='module')
def D():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import device, kernel, _lib
  _lib.load()
  return Namespace(torch=torch, device=device, kernel=kernel, lib=_lib)


def _copy(D, post, name, shape, dtype):
  t = D.torch.empty(shape, dtype=dtype, device=post.device)
  D.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), t.numel() * t.element_size()),
              'dfb_debug_copy')
  return t.cpu().numpy()


def _bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _assert_bits_equal(a, b, what):
  ia, ib = _bits(a), _bits(b)
  assert ia.shape == ib.shape, (what, ia.shape, ib.shape)
  bad = np.argwhere(ia != ib)
  assert len(bad) == 0, (what, 'differs in', len(bad), 'entries; first', tuple(bad[0]),
                         np.asarray(a)[tuple(bad[0])], np.asarray(b)[tuple(bad[0])])


class Case(object):
  """ One kernel (kind, d, scale, bandwidths), data and candidates. """

  def __init__(self, kname, d, n, m, seed, scale=1.3, post_scale=None):
    self.kname, self.d, self.n, self.m = kname, d, n, m
    self.kind, self.p = R.KINDS[kname]
    rs = np.random.RandomState(seed)
    self.bw = 0.2 + 0.6 * rs.random_sample(d)
    self.scale, self.post_scale = scale, post_scale
    self.X = rs.random_sample((n, d))
    self.Y = np.sin(3.0 * self.X).sum(axis=1) + 0.3
    cand = rs.random_sample((m, d))
    k = min(N_NEAR, m)
    cand[:k] = self.X[np.arange(k) % n]
    k2 = min(2 * N_NEAR, m)
    if k2 > k:
      v = rs.standard_normal((k2 - k, d))
      v /= np.linalg.norm(v, axis=1, keepdims=True)
      eps = 10.0 ** -rs.randint(3, 10, size=(k2 - k, 1))
      cand[k:k2] = self.X[np.arange(k, k2) % n] + eps * v
    self.Cand = cand

  def kernel(self, D):
    kd = D.kernel
    if self.kind == 'se':
      k = kd.SEKernel(self.d, self.scale, list(self.bw))
    else:
      k = kd.MaternKernel(self.d, self.p + 0.5, self.scale, list(self.bw))
    if self.post_scale is not None:
      k = kd.AdditiveKernel(self.post_scale, [k], [list(range(self.d))])
    return k

  def total_scale(self):
    s = np.longdouble(self.scale)
    return s * np.longdouble(self.post_scale) if self.post_scale is not None else s

  def exact(self, Xc, X):
    return R.kernel_exact(self.kind, self.p, self.total_scale(), self.bw, Xc, X)

  def bound(self, Xc, X):
    return R.kstar_bound(self.kind, self.p, self.total_scale(), self.bw, Xc, X)


# path -> options set before its eval (applied in this order on one built posterior)
PATH_OPTIONS = [
  ('P3', {'score_impl': 0}),
  ('P2', {'kstar_rows64': 0}),
  ('P1', {'kstar_fast': 0}),
  ('P4', {'kstar_fast': 1, 'kstar_rows64': 1, 'score_impl': 1, 'i8_radix': 1, 'i8_unguarded': 1}),
  ('P5', {'kstar_seg': 0}),
  ('P6', {'kstar_seg': 1, 'i8_radix': 0}),
]


def _build(D, desc, X, y, chunk, n_max, kstar_fast=1):
  post = D.device.DevicePosterior(n_max, chunk=chunk)
  post.set_option('kstar_fast', kstar_fast)
  post.set_kernel(desc)
  post.set_train(X, y)
  info, lml = post.build(0.01 * float(desc.kss))
  assert info == 0
  return post, lml


def run_paths(D, case, chunk, Xtrain=None, desc=None, test_desc=None, paths=PATHS):
  """ Builds the posterior once and evaluates the candidates through each path.  Returns a Namespace with the
      handle's alpha, npad, chunk geometry and per path mu, sd, and Ks (P1-P3) or the digit planes (P4-P6) of the
      last chunk. """
  Xtr = case.X if Xtrain is None else Xtrain
  desc = D.kernel.build_descriptor(case.kernel(D), train_dim=case.d, cand_dim=case.d) if desc is None else desc
  post, lml = _build(D, desc, Xtr, case.Y, chunk, max(case.n, 1))
  if test_desc is not None:
    post.set_test_kernel(test_desc)
  _, alpha, _ = post.get_state(want_alpha=True)
  npad, ch = int(post.query('npad')), int(post.query('chunk'))
  c0 = (case.m - 1) // ch * ch                     # first row of the last chunk
  mc = case.m - c0
  m_rows = (mc + 127) // 128 * 128
  res = Namespace(alpha=alpha.cpu().numpy(), npad=npad, chunk=ch, c0=c0, mc=mc, m_rows=m_rows, lml=lml,
                  kss=float((test_desc or desc).kss), post=post, desc=desc, out={})
  for name, opts in PATH_OPTIONS:
    for k, v in opts.items():
      post.set_option(k, v)
    if name not in paths:
      continue
    mu, sd = post.eval(case.Cand, mean_const=0.0)
    r = Namespace(mu=mu, sd=sd)
    if name in ROW_PATHS:
      assert post.query('last_used_i8') == 0.0
      r.Ks = _copy(D, post, 'Ks', (ch, npad), D.torch.float64)[:m_rows]
    else:
      assert post.query('last_used_i8') == 1.0, name
      radix256 = post.query('i8_radix256') == 1.0
      assert radix256 == (name != 'P6'), name
      r.planes = _copy(D, post, 'Ki8', (3, ch, 2 * npad), D.torch.int8)[:, :m_rows]
    res.out[name] = r
  return res


def check_paths(case, res, Xtrain=None, check_near=True):
  """ E1-E4, B1-B3 on the results of run_paths. """
  Xtr = case.X if Xtrain is None else Xtrain
  n, out = case.n, res.out
  last = case.Cand[res.c0:]
  K_ex = case.exact(case.Cand, Xtr)
  B = case.bound(case.Cand, Xtr)
  K_ex64 = K_ex.astype(np.float64)
  mb = R.mu_bound(res.alpha, K_ex64, B)
  mu_ex = (K_ex * res.alpha.astype(np.longdouble)).sum(axis=1)
  sl = slice(res.c0, res.c0 + res.mc)

  # B1 and the padding of the fp64 rows (exact zeros)
  for name in ROW_PATHS:
    if name not in out:
      continue
    Ks = out[name].Ks
    assert (_bits(Ks[res.mc:]) == 0).all() and (_bits(Ks[:, n:]) == 0).all(), (name, 'padding')
    err = np.abs(Ks[:res.mc, :n].astype(np.longdouble) - K_ex[sl]).astype(np.float64)
    assert (err <= B[sl]).all(), (name, 'B1', float(np.max(err / B[sl])),
                                  np.unravel_index(np.argmax(err / B[sl]), err.shape))
  # B2
  for name in ('P1', 'P2', 'P3', 'P4'):
    if name not in out:
      continue
    err = np.abs(out[name].mu.astype(np.longdouble) - mu_ex).astype(np.float64)
    assert (err <= mb).all(), (name, 'B2', float(np.max(err / mb)), int(np.argmax(err / mb)))
  # E1, E2
  if 'P1' in out and 'P2' in out:
    _assert_bits_equal(out['P1'].Ks, out['P2'].Ks, 'E1 Ks(P1) == Ks(P2)')
    _assert_bits_equal(out['P1'].sd, out['P2'].sd, 'E2 sd(P1) == sd(P2)')
  inv_f = 1.0 / IX.col_scale(res.kss)
  # E3
  if 'P2' in out:
    x = out['P2'].Ks * inv_f
    for name, want in (('P5', IX.digits_radix256(x) if 'P5' in out else None),
                       ('P6', IX.digits_radix128_split(x) if 'P6' in out else None)):
      if want is None:
        continue
      got = IX.unpack_planes(out[name].planes, len(want))
      for s in range(len(want)):
        bad = np.argwhere(got[s] != want[s])
        assert len(bad) == 0, ('E3', name, 'digit', s, 'differs in', len(bad), 'entries; first', tuple(bad[0]))
      if name == 'P6':
        assert np.array_equal(IX.reconstruct(got, False), IX.reconstruct(IX.digits_radix128(x), False))
  # E4
  if 'P3' in out and 'P4' in out:
    want = IX.digits_radix256(out['P3'].Ks * inv_f)
    got = IX.unpack_planes(out['P4'].planes, 5)
    for s in range(5):
      bad = np.argwhere(got[s] != want[s])
      assert len(bad) == 0, ('E4 digit', s, 'differs in', len(bad), 'entries; first', tuple(bad[0]))
    _assert_bits_equal(out['P4'].mu, out['P3'].mu, 'E4 mu(P4) == mu(P3)')
  # B3
  if check_near and case.kname == 'matern12' and 'P1' in out and 'P3' in out and res.c0 == 0:
    # the (candidate, training point) pairs that coincide or nearly do; elsewhere one ulp of the distance is worth
    # sqrt(2 nu) r ulp of exp(-sqrt(2 nu) r), and B1 is the check
    rows = np.arange(min(2 * N_NEAR, case.m))
    a, b = out['P1'].Ks[rows, rows % n], out['P3'].Ks[rows, rows % n]
    ulps = np.abs(a - b) / np.spacing(np.abs(a))
    assert (ulps <= 4).all(), ('B3', float(ulps.max()), int(np.argmax(ulps)))


def check_build_variants(D, case, res):
  """ E5 and B1 of K(X, X): the posterior with kstar_fast = 1 (res.post) and a second one built with kstar_fast = 0. """
  post1 = res.post
  post1.set_option('kstar_fast', 1)
  L1, a1, K1 = post1.get_state(want_L=True, want_alpha=True, want_K=True)
  post0, lml0 = _build(D, res.desc, case.X, case.Y, res.chunk, max(case.n, 1), kstar_fast=0)
  L0, a0, K0 = post0.get_state(want_L=True, want_alpha=True, want_K=True)
  _assert_bits_equal(L1.cpu().numpy(), L0.cpu().numpy(), 'E5 L')
  _assert_bits_equal(a1.cpu().numpy(), a0.cpu().numpy(), 'E5 alpha')
  _assert_bits_equal(np.array([res.lml]), np.array([lml0]), 'E5 lml')
  K_ex = case.exact(case.X, case.X)
  B = case.bound(case.X, case.X)
  for K in (K1.cpu().numpy(), K0.cpu().numpy()):
    err = np.abs(K.astype(np.longdouble) - K_ex).astype(np.float64)
    assert (err <= B).all(), ('B1 K(X, X)', float(np.max(err / B)))
  _assert_bits_equal(K1.cpu().numpy(), K0.cpu().numpy(), 'E5 K(X, X)')


# ---- every (kind, d) at a ragged shape ----------------------------------------------------------------------------------
@pytest.mark.parametrize('d', list(range(1, 9)))
@pytest.mark.parametrize('kname', KNAMES)
def test_every_variant_at_every_dimension(D, kname, d):
  case = Case(kname, d, N_MAIN, M_MAIN, seed=10 * d + KNAMES.index(kname))
  res = run_paths(D, case, CHUNK_MAIN)
  assert res.c0 == 0
  check_paths(case, res)
  check_build_variants(D, case, res)


# ---- shapes -------------------------------------------------------------------------------------------------------------
# N = 1 .. 1100 at m = 700 (N = 320: the last 64-point segment of kstar_seg is all padding; N >= 1024: the int8 path is
# the scoring default); m = 1, 31 (the small_sumsq contraction), 33, 127, the chunk, and 2 chunks + 1 row (only mu and
# sd are whole there: Ks and the planes hold the last, 1-row chunk) at N = 129
SHAPES = [(n, M_MAIN, CHUNK_MAIN) for n in (1, 127, 128, 320, 1100)] + \
         [(N_MAIN, m, CHUNK_SMALL) for m in (1, 31, 33, 127, CHUNK_SMALL, 2 * CHUNK_SMALL + 1)]


@pytest.mark.parametrize('shape', SHAPES, ids=['n%d-m%d' % s[:2] for s in SHAPES])
@pytest.mark.parametrize('d', [1, 7, 8])
@pytest.mark.parametrize('kname', KNAMES)
def test_shapes(D, kname, d, shape):
  n, m, chunk = shape
  case = Case(kname, d, n, m, seed=1000 + 10 * d + KNAMES.index(kname) + n + 7 * m)
  res = run_paths(D, case, chunk)
  check_paths(case, res)
  if m == M_MAIN:
    check_build_variants(D, case, res)


# ---- coordinate maps: Add-UCB group descriptors --------------------------------------------------------------------------
@pytest.mark.parametrize('kname', KNAMES)
def test_group_descriptors_on_a_column_subset(D, kname):
  """ The test kernel of one Add-UCB group (gp_core: build_descriptor(..., train_coords=group, cand_coords=0..g-1)) on a
      permuted, non-contiguous subset of a 12-column training matrix, group sizes 1 .. 8; post_scale != 1. """
  rs = np.random.RandomState(77 + KNAMES.index(kname))
  X12 = rs.random_sample((N_MAIN, 12))
  full = D.kernel.SEKernel(12, 1.0, [0.9] * 12)
  desc_tr = D.kernel.build_descriptor(full, train_dim=12, cand_dim=12)
  for g in range(1, 9):
    cols = [int(c) for c in rs.permutation(12)[:g]]
    case = Case(kname, g, N_MAIN, 300, seed=500 + g, scale=0.8, post_scale=1.7)
    case.X = X12[:, cols]                          # what the group kernel sees of the training matrix
    case.Cand[:2 * N_NEAR] = case.X[np.arange(2 * N_NEAR) % N_MAIN] + \
        np.where(np.arange(2 * N_NEAR)[:, None] < N_NEAR, 0.0, 1e-6)
    case.Y = np.sin(3.0 * X12).sum(axis=1)
    test_desc = D.kernel.build_descriptor(case.kernel(D), train_dim=12, cand_dim=g, train_coords=cols,
                                          cand_coords=list(range(g)))
    res = run_paths(D, case, CHUNK_MAIN, Xtrain=X12, desc=desc_tr, test_desc=test_desc, paths=ROW_PATHS)
    check_paths(case, res, check_near=False)


# ---- the interpreter above d = 8 -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', [9, 16, 17])
@pytest.mark.parametrize('kname', KNAMES)
def test_interpreter_above_eight_dimensions(D, kname, d):
  """ numpy_sumsq's eight-accumulator branch with a tail (9, 17) and without (16): every path falls back to
      kstar_kernel there. """
  case = Case(kname, d, N_MAIN, M_MAIN, seed=300 + d + KNAMES.index(kname))
  res = run_paths(D, case, CHUNK_MAIN, paths=('P1', 'P3'))
  check_paths(case, res, check_near=False)
  _assert_bits_equal(res.out['P1'].Ks, res.out['P3'].Ks, 'd > 8: one kernel')
  check_build_variants(D, case, res)
