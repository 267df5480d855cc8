"""
The two facts the bound pass of dfb_score_argmax (api.cu: bound_pass_applies, run_bound_pass) rests on, on the CPU.

Variance floor: for K = k(X, X) of a stationary kernel, s > 0 the diagonal added to it and any x*,
    sigma^2(x*) = k** - k^T (K + s I)^-1 k >= k** s / (tr K + s),
so that no candidate the screen drops can have a negative fp64 variance (a NaN score, np.argmax's winner) while the
floor exceeds the int8 error bound.  Checked with Cholesky solves on random SE / Matern kernels, N up to 2000, s from
1e-8 to 1e-1 of k**, uniform and clustered X (the floor is attained when every point coincides).

Monotonicity: EI, UCB with beta >= 0 and PI below the incumbent are non-decreasing in sigma -- a NumPy restatement of
the device formulas (kernels.cu: acq_score; scipy's ndtr is the reference's norm.cdf) on a dense grid -- up to
rounding far below the screen's pad of 1e-9 of the score scale.  PI above the incumbent falls with sigma, which is why
the screen keeps those candidates.
"""
import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve
from scipy.special import ndtr

EPS = np.finfo(np.float64).eps


def _kernel(kind, X1, X2, bw, scale):
  d2 = (((X1[:, None, :] - X2[None, :, :]) / bw) ** 2).sum(axis=2)
  if kind == 'se':
    return scale * np.exp(-0.5 * d2)
  r = np.sqrt(d2)
  if kind == 'matern12':
    return scale * np.exp(-r)
  if kind == 'matern32':
    return scale * (1.0 + np.sqrt(3.0) * r) * np.exp(-np.sqrt(3.0) * r)
  return scale * (1.0 + np.sqrt(5.0) * r + 5.0 / 3.0 * d2) * np.exp(-np.sqrt(5.0) * r)


def _variance(K, kstar, kss, s):
  cf = cho_factor(K + s * np.eye(len(K)), lower=True)
  v = cho_solve(cf, kstar.T)
  return kss - np.einsum('ij,ji->i', kstar, v)


CASES = [(kind, n, s, layout) for kind in ('se', 'matern12', 'matern32', 'matern52')
         for n, s, layout in ((200, 1e-1, 'uniform'), (500, 1e-4, 'uniform'), (2000, 1e-8, 'uniform'),
                              (2000, 1e-2, 'uniform'), (300, 1e-6, 'clustered'), (1000, 1e-3, 'clustered'))]


@pytest.mark.parametrize('kind,n,s_rel,layout', CASES)
def test_variance_floor(kind, n, s_rel, layout):
  rs = np.random.RandomState(n + int(-np.log10(s_rel)) + len(kind))
  d = 4
  scale = 0.7
  bw = 0.2 + 0.5 * rs.random_sample(d)
  if layout == 'uniform':
    X = rs.random_sample((n, d))
    C = np.vstack([rs.random_sample((300, d)), X[:100], X[:50] + 1e-6 * rs.standard_normal((50, d))])
  else:          # a few tight clusters: K is close to rank 3, lambda_max close to tr K / 3
    centres = rs.random_sample((3, d))
    X = centres[rs.randint(0, 3, n)] + 1e-4 * rs.standard_normal((n, d))
    C = np.vstack([centres, X[:100], rs.random_sample((100, d))])
  s = s_rel * scale
  K = _kernel(kind, X, X, bw, scale)
  var = _variance(K, _kernel(kind, C, X, bw, scale), scale, s)
  floor = scale * s / (np.trace(K) + s)
  # the Cholesky solve itself is accurate to about n eps k** on sigma^2
  tol = 4.0 * n * EPS * scale
  assert (var >= floor - tol).all(), (float(np.min(var / floor)), float(floor))


def test_variance_floor_is_attained_by_coincident_points():
  """ Every training point at x*: K = k** 1 1^T, lambda_max = tr K, and sigma^2 equals the floor. """
  n, kss, s = 64, 1.3, 1e-3
  K = np.full((n, n), kss)
  var = _variance(K, np.full((1, n), kss), kss, s)[0]
  floor = kss * s / (n * kss + s)
  assert abs(var - floor) <= 1e-9 * floor + 8 * n * EPS * kss


# ---- monotonicity in sigma -------------------------------------------------------------------------------------------
def _ei(mu, sd, best):                    # sigma * (z Phi(z) + phi(z)), z = (mu - best) / sigma
  z = (mu - best) / sd
  return sd * (z * ndtr(z) + np.exp(z * z * -0.5) / 2.50662827463100050242)


def _pi(mu, sd, best):
  return ndtr((mu - best) / sd)


def _ucb(mu, sd, beta):
  return mu + beta * sd


SIGMA = np.geomspace(1e-6, 1e3, 20001)
GAPS = np.concatenate([-np.geomspace(1e3, 1e-8, 60), [0.0], np.geomspace(1e-8, 1e3, 60)])     # mu - best


def _max_drop(scores):
  """ Largest decrease along sigma (axis 1), relative to the score scale of the row. """
  drop = -np.diff(scores, axis=1)
  scale = np.maximum(np.abs(scores).max(axis=1, keepdims=True), 1e-300)
  return float((drop / scale).max())


def test_ei_is_non_decreasing_in_sigma():
  scores = _ei(GAPS[:, None], SIGMA[None, :], 0.0)
  assert _max_drop(scores) <= 1e-12


@pytest.mark.parametrize('beta', [0.0, 0.5, 3.0, 50.0])
def test_ucb_is_non_decreasing_in_sigma(beta):
  mu = np.linspace(-5.0, 5.0, 41)
  scores = _ucb(mu[:, None], SIGMA[None, :], beta)
  assert (np.diff(scores, axis=1) >= 0.0).all()


def test_pi_below_the_incumbent_is_non_decreasing_in_sigma():
  gaps = GAPS[GAPS < 0.0]
  scores = _pi(gaps[:, None], SIGMA[None, :], 0.0)
  assert _max_drop(scores) <= 1e-12


def test_pi_above_the_incumbent_falls_with_sigma():
  """ The case the screen must not bound (it keeps every candidate with mu >= the incumbent). """
  gaps = GAPS[GAPS > 0.0]
  scores = _pi(gaps[:, None], SIGMA[None, :], 0.0)
  assert (np.diff(scores, axis=1) <= 1e-15).all()
  assert (scores[:, 0] > scores[:, -1]).all()
