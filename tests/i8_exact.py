"""
Exact restatement of the int8 scoring path (dragonfly_b200/csrc/gemm_i8.cuh and its digit producers in kernels.cu),
shared by the CPU tests (test_host_logic.py) and the GPU tests (test_gpu_i8_exact.py).

Everything the kernel does before its epilogue is integer arithmetic, and its epilogue is a fixed sequence of fp64
operations, so `partial` is a deterministic function of the digit planes, the row scales and the column scale.  This
module computes that function:
  * digit expansions of both schemes (radix 256: digits_radix256; radix 128: the loop of slice_i8_kernel, and the
    split form kstar_fast_kernel writes, which expands the same integer);
  * the pair-interleaved plane layout the producers write and the kernel reads (kb = 32);
  * the group sums G_d = sum_{s+t=d} A_s B_t^T with the triangular skip of W: every product and every partial sum
    is an integer below 15 K 2^14 < 2^53, so any fp64 GEMM (numpy's, or torch's on the device) is exact;
  * the epilogue, operation by operation in the kernel's order, with its one contracted multiply-add emulated exactly.
"""
from fractions import Fraction

import numpy as np

TILE = 128            # rows of W per row block (I8_BM)
KB = 32               # k-values per interleave block of the digit planes
N_PLANES = 3


def tile_n(radix256):
  """ Candidates per tile of the contraction (i8_tile_n in gemm_tma.h). """
  return 64 if radix256 else 32


def n_digits(radix256):
  return 5 if radix256 else 6


def digit_weights(radix256):
  """ Weight of digit s (0-based): radix 256 2^-(8 s + 7), radix 128 2^-(7 s + 7). """
  return [2.0 ** -(8 * s + 7) if radix256 else 2.0 ** -(7 * s + 7) for s in range(n_digits(radix256))]


def groups(radix256):
  """ Kept digit groups d = s + t (1-based digits) and their weights, largest group first. """
  if radix256:
    return [(d, 2.0 ** -(8 * d - 2)) for d in range(6, 1, -1)]      # the 15 products with s + t <= 6
  return [(d, 2.0 ** -(7 * d)) for d in range(7, 1, -1)]            # all 21 products


# ---- digit expansions ------------------------------------------------------------------------------------------------
def digits_radix256(x):
  """ NumPy restatement of digits_radix256 (kernels.cu): five signed digits of |x| <= 1/2,
      x ~ a0 2^-7 + a1 2^-15 + a2 2^-23 + a3 2^-31 + a4 2^-39. """
  x = np.asarray(x, dtype=np.float64)
  hi = np.rint(x * 2.0 ** 15)                      # round-half-even, like the magic-number trick
  rem = x * 2.0 ** 15 - hi                         # exact
  lo = np.rint(rem * 2.0 ** 24).astype(np.int64)
  hi = hi.astype(np.int64)
  s8 = lambda v: ((v + 128) % 256) - 128           # sign-extended low byte
  a4 = s8(lo); r = (lo - a4) >> 8
  a3 = s8(r); r = (r - a3) >> 8
  a2 = s8(r); hi = hi + ((r - a2) >> 8)
  a1 = s8(hi); a0 = (hi - a1) >> 8
  return [a0, a1, a2, a3, a4]


def digits_radix128(x):
  """ NumPy restatement of the radix-128 loop of slice_i8_kernel (kernels.cu): six signed digits of |x| < 1/2,
      y = 128 x, a = rint(y), x <- y - a (all exact in fp64); x ~ sum_s a_s 2^-7(s+1). """
  x = np.array(x, dtype=np.float64)
  out = []
  for _ in range(6):
    y = x * 128.0
    a = np.rint(y)
    x = y - a
    out.append(a.astype(np.int64))
  return out


def digits_radix128_split(x):
  """ NumPy restatement of the radix-128 digits of kstar_fast_kernel<..., I8OUT> (kernels.cu): hi = rint(x 2^21) and
      lo = rint((x 2^21 - hi) 2^21), each 21-bit half split into three digits by a1 = (w + 8192) >> 14,
      a2 = (r1 + 64) >> 7, a3 = r1 - 128 a2.  The same integer rint(x 2^42) as digits_radix128, but where a half's
      low bits sit exactly half-way its digits are rounded up, not to the nearest of the remainder: a different,
      equally valid expansion (digits in [-64, 64]). """
  x = np.asarray(x, dtype=np.float64)
  hi = np.rint(x * 2.0 ** 21)
  lo = np.rint((x * 2.0 ** 21 - hi) * 2.0 ** 21).astype(np.int64)
  out = []
  for w in (hi.astype(np.int64), lo):
    a1 = (w + 8192) >> 14
    r1 = w - (a1 << 14)
    a2 = (r1 + 64) >> 7
    out += [a1, a2, r1 - (a2 << 7)]
  return out


def digits(x, radix256):
  return digits_radix256(x) if radix256 else digits_radix128(x)


def reconstruct(dg, radix256):
  """ sum_s a_s w_s in fp64 (exact for the digits of an fp64 value: at most 46 significant bits). """
  out = np.zeros(np.shape(dg[0]), dtype=np.float64)
  for a, w in zip(dg, digit_weights(radix256)):
    out += np.asarray(a, dtype=np.float64) * w
  return out


# ---- pair-interleaved planes -----------------------------------------------------------------------------------------
def pack_planes(dg):
  """ Digits (list of rows x cols integer arrays) -> int8 planes (3, rows, 2 cols).  The byte of (digit s, 0-based;
      row r; column k) sits at (s // 2) plane_bytes + r 2 cols + (k // 32) 64 + (s % 2) 32 + k % 32. """
  rows, cols = np.shape(dg[0])
  assert cols % KB == 0 and len(dg) <= 2 * N_PLANES
  planes = np.zeros((N_PLANES, rows, 2 * cols), dtype=np.int8)
  for s, a in enumerate(dg):
    planes[s // 2].reshape(rows, cols // KB, 2, KB)[:, :, s % 2, :] = np.asarray(a).reshape(rows, cols // KB, KB)
  return planes


def unpack_planes(planes, n):
  """ Inverse of pack_planes: the first n digits (5 for radix 256, whose sixth slot no kernel reads). """
  planes = np.asarray(planes)
  _, rows, cols2 = planes.shape
  cols = cols2 // 2
  return [planes[s // 2].reshape(rows, cols // KB, 2, KB)[:, :, s % 2, :].reshape(rows, cols).astype(np.int64)
          for s in range(n)]


def triangular_keep(rows, K):
  """ keep[r, k]: row block r // 128 contracts only k < min(K, 128 (r // 128 + 1)) (W is lower triangular). """
  limit = np.minimum(K, (np.arange(rows) // TILE + 1) * TILE)
  return np.arange(K)[None, :] < limit[:, None]


# ---- group sums ------------------------------------------------------------------------------------------------------
def group_sums(A, Bd, radix256, matmul=None):
  """ G_d = sum_{s+t=d} A_s B_t^T for the kept groups, as fp64 arrays of exact integers.  A: the W digits, already
      masked with triangular_keep; Bd: the K_* digits.  matmul(a, b) = a b^T in fp64 (numpy by default; the GPU
      tests pass a torch one and their digit arrays as device tensors). """
  if matmul is None:
    matmul = lambda a, b: np.asarray(a, dtype=np.float64) @ np.asarray(b, dtype=np.float64).T
  nd = n_digits(radix256)
  G = {}
  for d, _ in groups(radix256):
    acc = None
    for s in range(1, nd + 1):
      t = d - s
      if 1 <= t <= nd:
        p = matmul(A[s - 1], Bd[t - 1])
        acc = p if acc is None else acc + p
    G[d] = acc
  return G


# ---- fp64 epilogue -----------------------------------------------------------------------------------------------------
def fma_fraction(a, b, c):
  """ Correctly rounded a b + c of three floats (CPython rounds int / int correctly). """
  return float(Fraction(a) * Fraction(b) + Fraction(c))


def _two_sum(a, b):
  s = a + b
  bb = s - a
  return s, (a - (s - bb)) + (b - bb)


def _split(a):
  c = 134217729.0 * a                              # 2^27 + 1
  hi = c - (c - a)
  return hi, a - hi


def _two_prod(a, b):
  p = a * b
  ah, al = _split(a)
  bh, bl = _split(b)
  return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _round_to_odd_sum(a, b):
  """ a + b rounded to odd: of the two floats around an inexact sum, the one with an odd last significand bit. """
  u, e = _two_sum(a, b)
  odd = (u.view(np.int64) & 1) == 1
  toward = np.nextafter(u, np.where(e > 0, np.inf, -np.inf))
  return np.where((e == 0) | odd, u, toward)


def fma_vec(a, b, c):
  """ Vectorised correctly rounded a b + c (Boldo & Melquiond, "Emulation of FMA and correctly rounded sums: proved
      algorithms using rounding to odd", IEEE TC 2008): (uh, ul) = a b exactly, (th, tl) = c + uh exactly,
      result = RN(th + RO(tl + ul)).  The exact product needs no underflow in its low part: entries with a tiny
      non-zero product, or huge operands, go through Fraction instead. """
  a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
  with np.errstate(over='ignore', invalid='ignore'):
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    out = th + _round_to_odd_sum(tl, ul)
  prod = np.abs(a) * np.abs(b)
  slow = ((prod < 2.0 ** -900) & (a != 0) & (b != 0)) | (np.abs(a) > 2.0 ** 500) | (np.abs(b) > 2.0 ** 500) | \
         (np.abs(c) > 2.0 ** 1000) | ~np.isfinite(a) | ~np.isfinite(b) | ~np.isfinite(c)
  if slow.any():
    out = np.array(out)
    for i in zip(*np.nonzero(slow)):
      out[i] = fma_fraction(float(a[i]), float(b[i]), float(c[i])) if np.isfinite([a[i], b[i], c[i]]).all() \
          else a[i] * b[i] + c[i]
  return out


def epilogue(G, rowscale, colscale, radix256):
  """ score_i8_kernel's epilogue in its order of operations, per row block and column:
        v = G_last w_last;  v = fma(G_d, w_d, v) from the smallest weight up (every G w is exact: plain adds);
        v *= rowscale[r] colscale;
        per warp w (tile rows 16 w .. 16 w + 15) and row group g: x_g = fma(v(r1), v(r1), v(r0)^2), r0 = 16 w + g,
        r1 = r0 + 8 (the compiler contracts `cs += v * v` into a DFMA);
        butterfly over the row groups: ((x0 + x1) + (x2 + x3)) + ((x4 + x5) + (x6 + x7));
        t = y_0, t += y_w for w = 1 .. 7.
      G: {d: rows x cols fp64 arrays} (rows = n_rb 128); returns partial (n_rb, cols). """
  gs = groups(radix256)
  v = None
  for d, w in gs:
    t = np.asarray(G[d], dtype=np.float64) * w
    v = t if v is None else t + v
  rows, cols = v.shape
  rs = np.asarray(rowscale, dtype=np.float64) * float(colscale)
  v = v * rs[:, None]
  n_rb = rows // TILE
  v = v.reshape(n_rb, 8, 2, 8, cols)                 # (row block, warp, half, row group, column)
  x = fma_vec(v[:, :, 1], v[:, :, 1], v[:, :, 0] * v[:, :, 0])    # (n_rb, 8 warps, 8 groups, cols)
  y = ((x[:, :, 0] + x[:, :, 1]) + (x[:, :, 2] + x[:, :, 3])) + ((x[:, :, 4] + x[:, :, 5]) + (x[:, :, 6] + x[:, :, 7]))
  t = y[:, 0]
  for w in range(1, 8):
    t = t + y[:, w]
  return t


def row_scales(W):
  """ row_exponent_kernel: rowscale_i = 2^(e_i + 1) with max_k |W_ik| = f 2^e_i, f in [1/2, 1) (2 for a zero row). """
  mx = np.abs(np.asarray(W, dtype=np.float64)).max(axis=1)
  e = np.where(mx > 0, np.frexp(mx)[1], 0)
  return np.ldexp(1.0, e + 1)


def col_scale(kss):
  """ i8_colscale (api.cu): 2^(e + 1) for kss (1 + 1e-9) = f 2^e. """
  return float(np.ldexp(1.0, np.frexp(kss * (1.0 + 1e-9))[1] + 1))


def partial_reference(A, Bd, rowscale, colscale, radix256, matmul=None):
  """ The kernel's `partial` from the digit arrays: A = W digits (rows a multiple of 128, K columns), Bd = K_* digits
      (candidates x K).  Masks A with the triangular skip first. """
  rows, K = np.shape(A[0])
  if matmul is None:
    keep = triangular_keep(rows, K)
    Am = [np.where(keep, a, 0) for a in A]
  else:
    Am = A                                          # the caller masks device tensors itself
  G = group_sums(Am, Bd, radix256, matmul)
  G = {d: (g.cpu().numpy() if hasattr(g, 'cpu') else np.asarray(g)) for d, g in G.items()}
  return epilogue(G, rowscale, colscale, radix256)
