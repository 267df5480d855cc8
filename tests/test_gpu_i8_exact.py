"""
The int8 scoring contraction (gemm_i8.cuh: score_i8_kernel) and its digit producers (kernels.cu: kstar_seg_kernel,
kstar_fast_kernel<..., I8OUT>, slice_i8_kernel), checked BIT FOR BIT against the exact restatement of tests/i8_exact.py
(-m gpu).

Before its epilogue the kernel does exact integer arithmetic, and the epilogue is a fixed sequence of fp64 operations,
so `partial` is a deterministic function of the digit planes, the row scales and the column scale.  A tolerance on
sigma^2 cannot see the low digit groups (group 6 of radix 256 weighs 2^-46 against 2^-14 for the top one); these
tests fail on a single wrong integer:
  A. the kernel on synthetic planes (dfb_debug_score_i8): both schemes, K blocks from fewer than the ring's stages to
     many times round it, tile groupings with a narrower last group, garbage above W's diagonal blocks, a guarded
     output buffer, the shortlist-overflow gate;
  B. int32 headroom at the largest K that admits radix 256;
  C. the production digit planes of every producer, read back with dfb_debug_copy after one dfb_eval;
  D. the production `partial` of the same runs.
Group sums are computed by torch.matmul in fp64 on the device: exact, since every partial sum is an integer below 2^53.
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import i8_exact as IX

pytestmark = pytest.mark.gpu

SHORTLIST_CAP = 4096          # kernels.cuh: the abort gate's cap
R256_MAX_NPAD = 24576         # api.cu prepare_i8: the largest npad that admits radix 256


@pytest.fixture(scope='module')
def D():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import device, kernel, synth_data, _lib
  _lib.load()
  post = device.DevicePosterior(256, chunk=128)       # a handle to launch the kernel on; no posterior needed
  return Namespace(torch=torch, device=device, kernel=kernel, synth=synth_data, lib=_lib, post=post)


def _ptr(t):
  return C.c_void_p(t.data_ptr()) if t is not None else None


def _score(D, radix256, A, B, n_rb, n_cb, rowscale, colscale, out, ld, abort=None):
  D.lib.check(D.post.lib.dfb_debug_score_i8(D.post.h, int(radix256), _ptr(A), _ptr(B), int(n_rb), int(n_cb),
                                            _ptr(rowscale), float(colscale), _ptr(abort), _ptr(out), int(ld)),
              'dfb_debug_score_i8')


def _copy(D, post, name, shape, dtype):
  t = D.torch.empty(shape, dtype=dtype, device=post.device)
  D.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), _ptr(t), t.numel() * t.element_size()), 'dfb_debug_copy')
  return t


def _pack_dev(D, dg):
  """ Device twin of IX.pack_planes: digits (rows x cols int tensors) -> int8 planes (3, rows, 2 cols). """
  rows, cols = dg[0].shape
  planes = D.torch.zeros((3, rows, 2 * cols), dtype=D.torch.int8, device=dg[0].device)
  view = planes.view(3, rows, cols // IX.KB, 2, IX.KB)
  for s, a in enumerate(dg):
    view[s // 2, :, :, s % 2, :] = a.to(D.torch.int8).view(rows, cols // IX.KB, IX.KB)
  return planes


def _unpack_dev(D, planes, n):
  """ Device twin of IX.unpack_planes, as fp64 tensors (the operands of the exact fp64 group sums). """
  _, rows, cols2 = planes.shape
  cols = cols2 // 2
  view = planes.view(3, rows, cols // IX.KB, 2, IX.KB)
  return [view[s // 2, :, :, s % 2, :].reshape(rows, cols).to(D.torch.float64) for s in range(n)]


def _keep_dev(D, rows, K, device):
  torch = D.torch
  limit = torch.clamp((torch.arange(rows, device=device) // IX.TILE + 1) * IX.TILE, max=K)
  return torch.arange(K, device=device)[None, :] < limit[:, None]


def _partial_dev(D, A, Bd, rowscale, colscale, radix256):
  """ IX.partial_reference with the W digits masked and both GEMMs of every group on the device. """
  keep = _keep_dev(D, A[0].shape[0], A[0].shape[1], A[0].device)
  Am = [a * keep for a in A]
  return IX.partial_reference(Am, Bd, np.asarray(rowscale), colscale, radix256, matmul=lambda a, b: a @ b.T)


def _bits_equal(a, b):
  a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
  return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def _row_scales_pattern(rows):
  # 2^-3 .. 2^3, different for rows r and r + 8 (the two rows of a thread), r + 16 (next warp) and r + 64 (the other
  # consumer warpgroup)
  r = np.arange(rows)
  return np.ldexp(1.0, (r + 3 * (r // 8)) % 7 - 3)


# ---- A. the kernel on synthetic planes ---------------------------------------------------------------------------------
@pytest.mark.parametrize('radix256', [True, False])
@pytest.mark.parametrize('n_rb', [1, 2, 3, 7, 48])
def test_kernel_on_synthetic_planes_is_bit_exact(D, radix256, n_rb):
  torch = D.torch
  dev = D.post.device
  gen = torch.Generator(device=dev)
  gen.manual_seed(1000 * n_rb + radix256)
  nd, bn = IX.n_digits(radix256), IX.tile_n(radix256)
  n_cb = 13                                   # groups of 8 and 3 leave a narrower last group, 1 / 13 / 100000 none
  K, rows_b = n_rb * IX.TILE, n_cb * bn

  def rand_digits(rows, top):
    lo, hi = (-64, 65) if (top or not radix256) else (-128, 128)
    return torch.randint(lo, hi, (rows, K), generator=gen, device=dev, dtype=torch.int16)

  keep = _keep_dev(D, K, K, dev)
  A = []
  for s in range(nd):
    a = rand_digits(K, s == 0)
    A.append(torch.where(keep | (a != 0), a, torch.ones_like(a)))     # non-zero garbage above the diagonal blocks
  Bd = [rand_digits(rows_b, s == 0) for s in range(nd)]
  Ap, Bp = _pack_dev(D, A), _pack_dev(D, Bd)
  rowscale = _row_scales_pattern(K)
  colscale = 2.0 ** -3
  ref = _partial_dev(D, [a.to(torch.float64) for a in A], [b.to(torch.float64) for b in Bd], rowscale, colscale,
                     radix256)
  assert np.isfinite(ref).all() and (ref > 0).all()
  rs_dev = torch.from_numpy(rowscale).to(dev)
  ld = rows_b + 40
  outs = []
  for group in (0, 1, 3, 8, n_cb, 100000):
    D.post.set_option('i8_c2_group', group)
    out = torch.full((n_rb + 1, ld), float('nan'), dtype=torch.float64, device=dev)
    _score(D, radix256, Ap, Bp, n_rb, n_cb, rs_dev, colscale, out, ld)
    o = out.cpu().numpy()
    assert _bits_equal(o[:n_rb, :rows_b], ref), (group, np.abs(o[:n_rb, :rows_b] - ref).max())
    assert np.isnan(o[:n_rb, rows_b:]).all() and np.isnan(o[n_rb:]).all(), group
    outs.append(o[:n_rb, :rows_b])
  assert all(_bits_equal(o, outs[0]) for o in outs)
  D.post.set_option('i8_c2_group', 0)
  # the abort gate: a launch behind an overflowed shortlist writes nothing; at the cap it runs normally
  for count, writes in ((SHORTLIST_CAP + 1, False), (SHORTLIST_CAP, True)):
    abort = torch.tensor([count], dtype=torch.int32, device=dev)
    out = torch.full((n_rb + 1, ld), float('nan'), dtype=torch.float64, device=dev)
    _score(D, radix256, Ap, Bp, n_rb, n_cb, rs_dev, colscale, out, ld, abort=abort)
    o = out.cpu().numpy()
    if writes:
      assert _bits_equal(o[:n_rb, :rows_b], ref) and np.isnan(o[:n_rb, rows_b:]).all() and np.isnan(o[n_rb:]).all()
    else:
      assert np.isnan(o).all()


# ---- B. int32 headroom ---------------------------------------------------------------------------------------------------
def test_int32_headroom_at_the_radix256_limit(D):
  """ Uniform extreme digits at K = 24576: group 6 reaches K (2 64 128 + 3 128^2) = 1,610,612,736 < 2^31 in the last
      row block; the mixed-sign operands (B digits 64, 127, 127, 127, 127) reach -K (64 127 + 128 64 + 3 128 127) =
      -1,599,602,688.  Against the closed form pushed through the same epilogue. """
  torch = D.torch
  dev = D.post.device
  K = R256_MAX_NPAD
  n_rb, n_cb, bn = K // IX.TILE, 1, IX.tile_n(True)
  a_dig = [-64, -128, -128, -128, -128]

  def uniform_planes(rows, dig):
    planes = torch.zeros((3, rows, 2 * K), dtype=torch.int8, device=dev)
    view = planes.view(3, rows, K // IX.KB, 2, IX.KB)
    for s, val in enumerate(dig):
      view[s // 2, :, :, s % 2, :] = val
    return planes

  Ap = uniform_planes(K, a_dig)                       # 3.6 GB
  try:
    rowscale = _row_scales_pattern(K)
    rs_dev = torch.from_numpy(rowscale).to(dev)
    k_eff = np.minimum(K, (np.arange(K) // IX.TILE + 1) * IX.TILE).astype(np.float64)
    for b_dig in ([-64, -128, -128, -128, -128], [64, 127, 127, 127, 127]):
      Bp = uniform_planes(n_cb * bn, b_dig)
      G = {}
      for d, _ in IX.groups(True):
        c_d = sum(a_dig[s - 1] * b_dig[d - s - 1] for s in range(1, 6) if 1 <= d - s <= 5)
        G[d] = np.repeat((k_eff * c_d)[:, None], n_cb * bn, axis=1)
      g6 = G[6][-1, 0]
      assert abs(g6) < 2.0 ** 31
      assert g6 == (1610612736 if b_dig[0] < 0 else -K * (64 * 127 + 128 * 64 + 3 * 128 * 127))
      ref = IX.epilogue(G, rowscale, 1.0, True)
      out = torch.full((n_rb, n_cb * bn), float('nan'), dtype=torch.float64, device=dev)
      _score(D, True, Ap, Bp, n_rb, n_cb, rs_dev, 1.0, out, n_cb * bn)
      o = out.cpu().numpy()
      assert _bits_equal(o, ref), (b_dig, np.nanmax(np.abs(o - ref)))
      del Bp
  finally:
    del Ap
    torch.cuda.empty_cache()


# ---- C / D. the production digit planes and `partial` --------------------------------------------------------------------
def _kernels(D):
  k = D.kernel
  return {
    'matern25': k.MaternKernel(6, 2.5, 0.7, 0.3),
    'additive': k.AdditiveKernel(0.35, [k.MaternKernel(3, 2.5, 1.0, 0.5), k.SEKernel(3, 1.0, 0.4)],
                                 [[0, 1, 2], [3, 4, 5]]),
    'mf_product': k.CoordinateProductKernel(6, 0.7, [k.SEKernel(1, 1.0, [0.7]), k.MaternKernel(5, 2.5, 1.0, 0.4)],
                                            [[0], [1, 2, 3, 4, 5]]),
  }


# producer -> (kernel, options, digit scheme (None: as the library picks it), digits emitted by the K_* kernel)
PRODUCERS = {
  'kstar_seg': ('matern25', {'i8_radix': 1}, True, True),
  'kstar_fast_r256': ('matern25', {'i8_radix': 1, 'kstar_seg': 0}, True, True),
  'kstar_fast_r128': ('matern25', {'i8_radix': 0}, False, True),
  'slice_r256': ('matern25', {'i8_radix': 1, 'i8_fuse': 0}, True, False),
  'slice_r128': ('matern25', {'i8_radix': 0, 'i8_fuse': 0}, False, False),
  'slice_additive': ('additive', {}, None, False),
  'slice_mf_product': ('mf_product', {}, None, False),
}
M_CAND = 700                  # not a multiple of 128; 12 radix-256 tiles: a narrower last group of the default 8


def _check_digits_rowwise(planes, x, radix256, step=1024):
  """ Unpacked planes == the restatement of x, block of rows by block of rows (bounded host memory). """
  nd = IX.n_digits(radix256)
  for r0 in range(0, x.shape[0], step):
    got = IX.unpack_planes(planes[:, r0:r0 + step], nd)
    want = IX.digits(x[r0:r0 + step], radix256)
    for s in range(nd):
      bad = np.argwhere(got[s] != want[s])
      assert len(bad) == 0, ('digit', s, 'first mismatch at', (bad[0][0] + r0, bad[0][1]), len(bad))


@pytest.mark.parametrize('n', [300, 1100, 5000])
@pytest.mark.parametrize('producer', list(PRODUCERS))
def test_production_digit_planes_and_partial_are_bit_exact(D, producer, n):
  torch = D.torch
  kname, opts, want_r256, fused = PRODUCERS[producer]
  kern = _kernels(D)[kname]
  rs = np.random.RandomState(n)
  X = rs.random_sample((n, 6)); Y = D.synth.hartmann6(X)
  Cand = rs.random_sample((M_CAND, 6))
  post = D.device.DevicePosterior(n, chunk=1024)
  post.set_option('score_impl', 1)
  post.set_option('i8_unguarded', 1)          # the int8 path whatever its a-priori bound: these tests are exact
  for name, value in opts.items():
    post.set_option(name, value)
  desc = D.kernel.build_descriptor(kern, train_dim=6, cand_dim=6)
  post.set_kernel(desc)
  post.set_train(X, Y - float(np.median(Y)))
  assert post.build(0.01 * 0.7)[0] == 0
  mu_i8, _ = post.eval(Cand, mean_const=1.0)
  assert post.query('last_used_i8') == 1.0
  radix256 = post.query('i8_radix256') == 1.0
  if want_r256 is not None:
    assert radix256 == want_r256
  nd = IX.n_digits(radix256)
  npad, chunk = int(post.query('npad')), int(post.query('chunk'))
  nb, m_rows = npad // IX.TILE, (M_CAND + 127) // 128 * 128
  assert m_rows <= chunk
  W = _copy(D, post, 'W', (npad, npad), torch.float64)
  Wi8 = _copy(D, post, 'Wi8', (3, npad, 2 * npad), torch.int8)
  rowscale = _copy(D, post, 'rowscale', (npad,), torch.float64).cpu().numpy()
  Ki8 = _copy(D, post, 'Ki8', (3, chunk, 2 * npad), torch.int8)[:, :m_rows].contiguous()
  partial = np.ascontiguousarray(_copy(D, post, 'partial', (nb, chunk), torch.float64).cpu().numpy()[:, :m_rows])
  with pytest.raises(D.lib.DfbError):
    _copy(D, post, 'partial', (nb * chunk + 1,), torch.float64)          # the size must match
  colscale = IX.col_scale(desc.kss)

  # W digits: the restatement of the copied fp64 W; rowscale = 2^(e + 1) of each row's max
  W_h = W.cpu().numpy()
  Wi8_h = Wi8.cpu().numpy()
  assert _bits_equal(rowscale, IX.row_scales(W_h))
  _check_digits_rowwise(Wi8_h, W_h * (1.0 / rowscale)[:, None], radix256)
  Wd = IX.unpack_planes(Wi8_h, nd)
  off_diag = ~np.eye(npad - n, dtype=bool)
  for s in range(nd):
    assert (Wd[s][:n, n:] == 0).all()                                    # columns >= n of the training rows
    assert (Wd[s][n:, n:][off_diag] == 0).all() and (Wd[s][n:, :n] == 0).all()   # padding rows: the identity only
  del Wd, W_h

  # K_* digits: range, padding, and their values
  Ki8_h = Ki8.cpu().numpy()
  Kd = IX.unpack_planes(Ki8_h, nd)
  for s in range(nd):
    lo, hi = (-128, 127) if (radix256 and s > 0) else (-64, 64)
    assert int(Kd[s].min()) >= lo and int(Kd[s].max()) <= hi, (s, Kd[s].min(), Kd[s].max())
    assert (Kd[s][M_CAND:] == 0).all() and (Kd[s][:, n:] == 0).all()
  if not fused:
    Ks = _copy(D, post, 'Ks', (chunk, npad), torch.float64).cpu().numpy()[:m_rows]
    _check_digits_rowwise(Ki8_h, Ks * (1.0 / colscale), radix256)
  else:
    # the digits round v 2^-F to 2^-39 (radix 256) or 2^-42 (radix 128); v itself differs from the reference-order
    # kernel value by tens of ulp: the squared distance |x|^2 + |y|^2 - 2 x.y is rounded in another order (measured:
    # about 17 ulp of |K| for kstar_seg at N = 5000), hence 2^-45 |K|, at most 1/64 of the digits' 2^-40 colscale
    Kref = D.device.kernel_matrix(kern, Cand, X)
    recon = IX.reconstruct([a[:M_CAND, :n] for a in Kd], radix256) * colscale
    tol = 2.0 ** (-40 if radix256 else -43) * colscale + 2.0 ** -45 * np.abs(Kref)
    assert (np.abs(recon - Kref) <= tol).all(), np.max(np.abs(recon - Kref) / tol)
    # the exact check: the fp64-row twin of the producer (kstar_seg<ROWS64>, or kstar_fast's fp64 rows) forms the same
    # values, so the planes are exactly its digits -- in kstar_fast's own radix-128 expansion for that scheme -- and
    # kstar_seg's mu is the twin's, bit for bit
    post.set_option('score_impl', 0)
    if producer != 'kstar_seg':
      post.set_option('kstar_rows64', 0)
    mu_twin, _ = post.eval(Cand, mean_const=1.0)
    assert post.query('last_used_i8') == 0.0
    Ks = _copy(D, post, 'Ks', (chunk, npad), torch.float64).cpu().numpy()[:m_rows]
    want = IX.digits_radix256(Ks * (1.0 / colscale)) if radix256 else IX.digits_radix128_split(Ks * (1.0 / colscale))
    for s in range(nd):
      bad = np.argwhere(Kd[s] != want[s])
      assert len(bad) == 0, ('digit', s, 'differs from the twin in', len(bad), 'entries; first', tuple(bad[0]))
    if producer == 'kstar_seg':
      assert _bits_equal(mu_i8, mu_twin)
  del Kd

  # D: the production `partial`, from the copied planes, row scales and column scale
  ref = _partial_dev(D, _unpack_dev(D, Wi8, nd), _unpack_dev(D, Ki8, nd), rowscale, colscale, radix256)
  bad = np.argwhere(partial.view(np.int64) != ref.view(np.int64))
  assert len(bad) == 0, ('partial differs in', len(bad), 'entries; first', tuple(bad[0]),
                         partial[tuple(bad[0])], ref[tuple(bad[0])])
