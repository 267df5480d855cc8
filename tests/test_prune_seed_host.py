"""
The seed selection of the bound pass restated in NumPy (prune_seed_ref.py), on the CPU: the key orders doubles as
they compare with NaN above everything, the device's two-level histogram finds the same threshold as a sort, and the
seeds are the rows above the threshold plus the ties at it in row order, K to 2K rows -- in the cases
test_gpu_prune_seed.py sends through the device.
"""
import numpy as np
import pytest

import prune_seed_ref as S


def _brute(ub, K):
  """ By definition: sort by key, descending, ties in row order; the K-th key's 32-bit prefix is tau. """
  p = S.seed_keys(ub) >> np.uint64(32)
  m = len(ub)
  if m < K:
    return np.arange(m)
  order = sorted(range(m), key=lambda i: (-int(p[i]), i))
  tau = p[order[K - 1]]
  above = [i for i in range(m) if p[i] > tau]
  ties = [i for i in range(m) if p[i] == tau][:2 * K - len(above)]
  return np.array(sorted(above + ties), dtype=np.int64)


def test_key_orders_like_the_doubles():
  rs = np.random.RandomState(3)
  v = np.concatenate([rs.standard_normal(500) * 10.0 ** rs.randint(-300, 300, 500),
                      [0.0, np.inf, -np.inf, 5e-324, -5e-324, np.finfo(np.float64).max]])
  k = S.seed_keys(v)
  order_v = np.argsort(v, kind='stable')
  assert (np.diff(k[order_v].astype(object)) >= 0).all()
  strict = np.diff(v[order_v]) > 0
  assert (k[order_v][1:][strict] > k[order_v][:-1][strict]).all()
  nan = np.array([np.nan, -np.nan, np.frombuffer(np.uint64(0x7ff0000000000001).tobytes(), np.float64)[0]])
  assert (S.seed_keys(nan) == np.uint64(0xffffffffffffffff)).all()
  assert (S.seed_keys(nan).min() > k.max())
  assert S.seed_keys(np.array([-0.0]))[0] + np.uint64(1) == S.seed_keys(np.array([0.0]))[0]


def _cases():
  rs = np.random.RandomState(7)
  c = {}
  c['random'] = (rs.standard_normal(20000), 256)
  c['negative_ucb'] = (-100.0 - rs.random_sample(20000), 128)
  u = rs.random_sample(5000)
  u[rs.randint(0, 5000, 300)] = 0.9999                       # many exact ties, straddling the threshold at K = 128
  c['ties_at_tau'] = (u, 128)
  u = rs.random_sample(5000); u[[17, 4000]] = np.nan; u[[5, 900, 901]] = np.inf
  c['nan_and_inf'] = (u, 64)
  c['all_equal'] = (np.full(7000, 1.25), 512)
  c['fewer_than_k'] = (rs.random_sample(300), 512)
  c['exactly_k'] = (rs.random_sample(512), 512)
  c['k_one'] = (rs.random_sample(1000), 1)
  u = rs.random_sample(3000); u[:] = np.round(u * 8) / 8        # a few values, prefix ties everywhere
  c['few_values'] = (u, 100)
  return c


@pytest.mark.parametrize('name', sorted(_cases()))
def test_selection_matches_the_definition(name):
  ub, K = _cases()[name]
  got = S.select_seeds(ub, K)
  assert (got == _brute(ub, K)).all()
  m = len(ub)
  assert min(K, m) <= len(got) <= 2 * K
  p = S.seed_keys(ub) >> np.uint64(32)
  tau, above = S.threshold_two_level(p, K)
  assert tau == S.threshold(p, K)
  assert above == int((p > tau).sum()) and above < K


def test_special_cases():
  cases = _cases()
  ub, K = cases['all_equal']
  assert (S.select_seeds(ub, K) == np.arange(2 * K)).all()          # the first 2K rows
  ub, K = cases['fewer_than_k']
  assert (S.select_seeds(ub, K) == np.arange(len(ub))).all()
  ub, K = cases['nan_and_inf']
  got = set(S.select_seeds(ub, K).tolist())
  assert {17, 4000, 5, 900, 901} <= got
  ub, K = cases['ties_at_tau']
  got = S.select_seeds(ub, K)
  ties = np.flatnonzero(ub == 0.9999)
  assert len(got) == 2 * K and (got[np.isin(got, ties)] == ties[:len(got) - int((ub > 0.9999).sum())]).all()
