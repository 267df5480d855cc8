"""
NumPy restatement of the seed selection of dfb_score_argmax's bound pass (kernels.cu: seed_key, seed_hist_kernel,
seed_threshold_kernel, seed_flag_kernel, seed_pick_kernel).  Shared by test_prune_seed_host.py (CPU) and
test_gpu_prune_seed.py (device).

The bounds ub of one screen launch are ordered by an order-preserving 64-bit key (NaN above everything).  tau is the
largest 32-bit key prefix with at least K rows at or above it (0 when there are fewer than K rows).  The seeds are
every row whose prefix exceeds tau (fewer than K of them) and then the rows at tau in row order while there are fewer
than 2K seeds in all.
"""
import numpy as np

TOP = np.uint64(1) << np.uint64(63)


def seed_keys(ub):
  ub = np.ascontiguousarray(ub, dtype=np.float64)
  b = ub.view(np.uint64)
  k = np.where(b & TOP, ~b, b | TOP)
  k[np.isnan(ub)] = np.uint64(0xffffffffffffffff)
  return k


def threshold(prefix, K):
  """ tau from the sorted prefixes: the K-th largest, or 0 with fewer than K rows. """
  if len(prefix) < K:
    return np.uint64(0)
  return np.sort(prefix)[len(prefix) - K]


def threshold_two_level(prefix, K):
  """ tau as the device finds it: two 2^16-bin histograms, each scanned from the top. """
  def level(bins, need):
    hist = np.bincount(bins.astype(np.int64), minlength=1 << 16)
    above = np.concatenate([np.cumsum(hist[::-1])[::-1][1:], [0]])   # rows in higher bins
    ok = np.flatnonzero(above + hist >= need)
    b = int(ok.max()) if len(ok) else 0
    return b, int(above[b])
  hi = prefix >> np.uint64(16)
  b0, above0 = level(hi, K)
  lo = (prefix[hi == np.uint64(b0)] & np.uint64(0xffff))
  b1, above1 = level(lo, K - above0)
  return np.uint64((b0 << 16) | b1), above0 + above1


def select_seeds(ub, K):
  """ The seeds' rows, ascending. """
  p = seed_keys(ub) >> np.uint64(32)
  tau = threshold(p, K)
  gt = p > tau
  eq = np.flatnonzero(p == tau)
  sel = gt.copy()
  sel[eq[:max(0, 2 * K - int(gt.sum()))]] = True
  return np.flatnonzero(sel)
