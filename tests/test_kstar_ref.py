"""
The extended-precision kernel reference and the forward-error bound of tests/kstar_ref.py, checked on the CPU against
the fp64 oracle (oracle/gp_oracle.py OSEKernel, OMaternKernel): a bound that the oracle itself breaks is wrong, and a
bound that no fp64 evaluation comes near is too loose to catch anything.
"""
import numpy as np
import pytest

import kstar_ref as R
from oracle import gp_oracle as O

BANDWIDTHS = (0.02, 0.1, 0.5, 1.0, 5.0)
RATIO_FLOOR = 1e-3
_ratios = {}


def _points(d, seed):
  """ 40 training points in [0, 1]^d; candidates: 40 random points, 8 copies of training points and training
      points moved by 1e-9 .. 1e-3 along a random direction (8 each). """
  rs = np.random.RandomState(seed)
  X = rs.random_sample((40, d))
  cand = [rs.random_sample((40, d)), X[:8].copy()]
  for eps in (1e-9, 1e-7, 1e-5, 1e-3):
    v = rs.standard_normal((8, d))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    cand.append(X[8:16] + eps * v)
  return np.vstack(cand), X


def _oracle(kind, p, d, scale, bw):
  if kind == 'se':
    return O.OSEKernel(d, scale, list(bw))
  return O.OMaternKernel(d, p + 0.5, scale, list(bw))


@pytest.mark.parametrize('kname', list(R.KINDS))
@pytest.mark.parametrize('d', list(range(1, 18)))
def test_oracle_kernel_values_lie_within_the_bound(kname, d):
  kind, p = R.KINDS[kname]
  Xc, X = _points(d, 100 * d + p + (kind == 'se'))
  worst = 0.0
  for i, bw0 in enumerate(BANDWIDTHS):
    rs = np.random.RandomState(i)
    bw = bw0 * (1.0 + 0.25 * rs.random_sample(d))       # per-dimension bandwidths around bw0
    scale = 0.7 + i
    K_o = _oracle(kind, p, d, scale, bw)(Xc, X)
    K_x = R.kernel_exact(kind, p, scale, bw, Xc, X)
    B = R.kstar_bound(kind, p, scale, bw, Xc, X)
    err = np.abs(K_o.astype(np.longdouble) - K_x).astype(np.float64)
    assert (err <= B).all(), (bw0, np.max(err / B), np.unravel_index(np.argmax(err / B), err.shape))
    # and it is a statement about fp64 rounding, not about K: Matern-1/2 turns the residue of D^2 ~ u |x / bw|^2 at
    # coincident points into sqrt(u) |x / bw| of K, the smooth kernels keep it at O(u |x / bw|^2) (|x / bw|^2 reaches
    # 17 / 0.02^2 here)
    assert (B <= (1e-3 if kname == 'matern12' else 1e-8) * scale).all()
    worst = max(worst, float(np.max(err / B)))
  _ratios[(kname, d)] = worst


def test_the_bound_is_not_vacuous():
  """ Across all cases of the test above, the largest observed error reaches at least RATIO_FLOOR of its bound
      (measured: 0.3 to 0.5, Matern-1/2 at coincident points). """
  if len(_ratios) < 4 * 17:
    for kname in R.KINDS:
      for d in range(1, 18):
        if (kname, d) not in _ratios:
          test_oracle_kernel_values_lie_within_the_bound(kname, d)
  worst = max(_ratios.values())
  print('largest |K_oracle - K_exact| / bound: %.3g' % worst)
  for kname in R.KINDS:
    print('  %s: %.3g' % (kname, max(v for (k, _), v in _ratios.items() if k == kname)))
  assert worst >= RATIO_FLOOR, worst
  assert worst <= 1.0


def test_mu_bound_covers_the_sum():
  rs = np.random.RandomState(5)
  Xc, X = _points(6, 7)
  bw = np.full(6, 0.3)
  K_x = R.kernel_exact('matern', 2, 1.3, bw, Xc, X)
  B = R.kstar_bound('matern', 2, 1.3, bw, Xc, X)
  K_hat = K_x.astype(np.float64)
  alpha = rs.standard_normal(X.shape[0]) * 1e3
  mu_exact = (K_x * alpha.astype(np.longdouble)).sum(axis=1)
  mu_hat = K_hat @ alpha
  mb = R.mu_bound(alpha, K_hat, B)
  assert (np.abs(mu_hat.astype(np.longdouble) - mu_exact).astype(np.float64) <= mb).all()
  assert (mb <= 1e-9 * np.abs(alpha).sum()).all()
