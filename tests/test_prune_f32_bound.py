"""
The certified single-precision upper bound of mu behind the bound pass of dfb_score_argmax (kernels.cu:
prune_bound_kernel; derivation in prune_bound_ref.py), on the CPU.

An emulation of the kernel's fp32 operation sequence, with every ex2 / rsqrt result moved adversarially by the size of
the PTX ISA's stated maximum error in either direction, must give mu_bar = mu32 + E >= mu_exact + mu_bound -- the
largest fp64 mu any K_* producer may return (kstar_ref.py) -- for SE and Matern 1/2, 3/2, 5/2 at d = 1..8: coincident
and near-coincident points, far points where k underflows in fp32, bandwidths 0.02..5, large |alpha| with
cancellation, and coordinates up to the point where the bound refuses (mu_bar = +inf).  The largest |mu32 - mu_exact|
/ E is reported; it stays below 1, and above a floor that keeps E from being absurdly loose.
"""
import numpy as np
import pytest

import kstar_ref as R
import prune_bound_ref as PB

LD = np.longdouble
CASES = [(kname, d) for kname in R.KINDS for d in range(1, 9)]
RATIO_FLOOR = 1e-2


def _inputs(rs, d, layout):
  """ (bw, X, C, alpha) of one layout. """
  n, m = 120, 160
  if layout == 'unit':
    bw = 0.02 + 4.98 * rs.random_sample(d) ** 3                     # bandwidths 0.02 .. 5
    X = rs.random_sample((n, d))
    C = rs.random_sample((m, d))
  elif layout == 'offset':                                           # far from the origin: large uncentred norms
    bw = np.full(d, 0.5)
    X = 2000.0 + rs.random_sample((n, d))
    C = 2000.0 + rs.random_sample((m, d))
  else:                                                              # candidates 10^5 away: the bound refuses
    bw = np.full(d, 0.5)
    X = rs.random_sample((n, d))
    C = 5e4 + rs.random_sample((m, d))
  C[:20] = X[:20]                                                    # on training points
  C[20:40] = X[20:40] * (1.0 + 1e-9 * rs.standard_normal((20, d)))   # next to them
  C[40:60] = X[40:60] + 30.0 * bw                                    # far: k underflows in fp32
  alpha = rs.standard_normal(n) * 10.0 ** rs.uniform(0, 5, n)       # large, mixed signs: cancellation
  return bw, X, C, alpha


def _check(kname, d, layout, seed):
  kind, p = R.KINDS[kname]
  rs = np.random.RandomState(seed)
  bw, X, C, alpha = _inputs(rs, d, layout)
  scale, mean = 1.7, -0.4
  K = R.kernel_exact(kind, p, scale, bw, C, X)
  mu_exact = (K @ alpha.astype(LD)).astype(np.float64) + mean
  mb = R.mu_bound(alpha, K.astype(np.float64), R.kstar_bound(kind, p, scale, bw, C, X), mean)
  worst = 0.0
  for de in (-PB.DOC_APPROX, PB.DOC_APPROX):
    for dr in (-PB.DOC_APPROX, PB.DOC_APPROX):
      mu32, E = PB.emulate(kind, p, scale, bw, C, X, alpha, mean, de, dr)
      fin = np.isfinite(E)
      assert (mu32 + E >= mu_exact + mb).all(), np.flatnonzero(mu32 + E < mu_exact + mb)[:5]
      if fin.any():
        worst = max(worst, float(np.max(np.abs(mu32 - mu_exact)[fin] / E[fin])))
  return worst, fin


@pytest.mark.parametrize('kname,d', CASES)
def test_bound_holds_and_is_not_loose(kname, d):
  worst, fin = _check(kname, d, 'unit', 100 + d)
  print('%s d=%d: max |mu32 - mu_exact| / E = %.3e' % (kname, d, worst))
  assert fin.all()
  assert RATIO_FLOOR <= worst <= 1.0


@pytest.mark.parametrize('kname', list(R.KINDS))
def test_large_coordinates(kname):
  """ Coordinates ~4000 after scaling (the centring keeps X + R small, the fp64 producers' term grows with |x~|^2);
      candidates 10^5 away from the training box: the bound refuses (mu_bar = +inf) and the screen keeps them. """
  worst, fin = _check(kname, 6, 'offset', 7)
  assert fin.all() and worst <= 1.0
  _, fin = _check(kname, 6, 'refuse', 8)
  assert not fin[60:].any()                                         # rows 0..59 sit next to the data
