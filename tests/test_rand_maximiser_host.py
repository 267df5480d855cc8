"""
The `rand` acquisition maximiser on the host (no GPU): `asy_ucb` and `asy_ts` through a fake GP whose fused session
scores candidate slabs with NumPy.  Every candidate source -- Euclidean host (streamed MT19937) and device rows,
Cartesian-product host draws and device rows -- must return np.argmax's point over the concatenated scores (ties and
NaN included), leave the global MT19937 stream where the reference leaves it, make the same sequence of scoring calls
(rows, row offset, seed, normals), and drain the stream when a slab's scoring raises.
"""
from argparse import Namespace

import numpy as np
import pytest
import torch

from dragonfly_b200 import cartesian_product_gp as cp
from dragonfly_b200 import dist as dfb_dist
from dragonfly_b200 import domains
from dragonfly_b200 import gpb_acquisitions as A
from dragonfly_b200 import kernel as K

M = 300
CHUNK = 16
SLAB = 64                # STREAM_SLAB_ROWS here: host slabs of 64 rows, device slabs of 128


def _unit(seed, rows, cols):
  """ Deterministic stand-in for the device's counter-based uniforms of (seed, row, column). """
  r = np.asarray(rows, dtype=np.float64).reshape(-1, 1)
  c = np.arange(cols, dtype=np.float64).reshape(1, -1)
  return np.mod((seed % 9973) * 0.6180339887 + r * 0.7548776662 + c * 0.5698402910 + r * r * 1e-4, 1.0)


class _FakePost(object):

  def fill_candidates(self, seed, row0, m, bounds, out=None):
    b = np.asarray(bounds, dtype=np.float64)
    vals = torch.from_numpy(b[:, 0] + _unit(seed, np.arange(row0, row0 + m), len(b)) * (b[:, 1] - b[:, 0]))
    if out is None:
      return vals
    out.copy_(vals)
    return out

  def fill_mixed_candidates(self, seed, row0, m, kinds, bounds, n_levels, out=None):
    from dragonfly_b200 import _lib
    b = np.asarray(bounds, dtype=np.float64).reshape(-1, 2)
    u = _unit(seed, np.arange(row0, row0 + m), len(kinds))
    vals = b[:, 0] + u * (b[:, 1] - b[:, 0])
    for c, kind in enumerate(kinds):
      if kind == _lib.DFB_CAND_INTEGER:
        vals[:, c] = np.trunc(vals[:, c])
      elif kind == _lib.DFB_CAND_CATEGORICAL:
        vals[:, c] = np.minimum(np.floor(u[:, c] * n_levels[c]), n_levels[c] - 1)
    vals = torch.from_numpy(vals)
    if out is None:
      return vals
    out.copy_(vals)
    return out


def _scores(X, nan):
  """ Coarse scores (many ties); with nan, NaN on a band of the first column. """
  X = np.asarray(X, dtype=np.float64)
  vals = np.floor(4.0 * (np.sin(3.0 * X[:, 0]) + 0.5 * X[:, 1])) / 4.0
  if nan:
    vals[(X[:, 0] > 0.55) & (X[:, 0] < 0.6)] = np.nan
  return vals


def _ts_normals(seed, rows):
  return np.sin(1.7 * (seed % 997) + 1.3 * np.asarray(rows, dtype=np.float64))


def _host(pts):
  return pts.numpy() if isinstance(pts, torch.Tensor) else np.asarray(pts)


class _FakeSession(object):

  def __init__(self, trace, nan, fail_at):
    self.trace, self.nan, self.fail_at, self.post = trace, nan, fail_at, _FakePost()

  def slab_rows(self, target):
    return max(1, int(target) // CHUNK) * CHUNK

  def _check(self):
    if len(self.trace) == self.fail_at:
      raise RuntimeError('scoring failed')

  def score(self, pts, want_scores=False):
    X = _host(pts)
    self.trace.append(('score', len(X)))
    self._check()
    vals = _scores(X, self.nan)
    i = int(np.argmax(vals))
    return vals[i], i, None

  def score_ts(self, pts, z=None, seed=0, row0=0, want_scores=False):
    X = _host(pts)
    self.trace.append(('ts', len(X), int(row0), int(seed), None if z is None else (len(z), float(z[0]))))
    self._check()
    if z is None:
      z = _ts_normals(seed, np.arange(row0, row0 + len(X)))
    vals = _scores(X, self.nan) + np.asarray(z)
    i = int(np.argmax(vals))
    return vals[i], i, None, 0


class _FakeGP(object):
  ucb_dim = 2.0

  def __init__(self, kernel, nan=False, fail_at=-1):
    self.kernel, self.trace, self.nan, self.fail_at = kernel, [], nan, fail_at

  def _fused_session(self, acq, halluc=None, **kwargs):
    from contextlib import contextmanager

    @contextmanager
    def session():
      yield _FakeSession(self.trace, self.nan, self.fail_at)
    return session()


EUC_BOUNDS = [[0.0, 1.0], [-1.0, 2.0]]


def _euc():
  return domains.EuclideanDomain(EUC_BOUNDS), K.SEKernel(2, 1.0, [1.0, 1.0])


def _cp():
  dom = domains.CartesianProductDomain([
      domains.EuclideanDomain([[0.0, 1.0], [-1.0, 2.0]]), domains.IntegralDomain([[0, 6]]),
      domains.ProdDiscreteDomain([['a', 'b', 'c'], ['x', 'y']]), domains.ProdDiscreteNumericDomain([[1, 2, 4]])])
  kern = cp.CartesianProductKernel(1.0, [K.SEKernel(2, 1.0, [1.0, 1.0]), K.SEKernel(1, 1.0, [1.0]),
                                         K.HammingKernel(2), K.SEKernel(1, 1.0, [1.0])])
  return dom, kern


def _anc(dom, mode):
  return Namespace(domain=dom, max_evals=M, acq_opt_method='rand', t=7, handle_parallel='halluc',
                   eval_points_in_progress=[], is_mf=False, candidate_rng=mode)


def _enc(pt):
  if isinstance(pt, list):
    return [np.asarray(p).tolist() for p in pt]
  return np.asarray(pt).tolist()


def _device_seed():
  return (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))


def _expected(case, mode, nan):
  """ (point, RNG state after the call) of one np.argmax over every candidate, replayed from seed 0. """
  np.random.seed(0)
  if case == 'euc':
    if mode == 'numpy':
      rows = A.draw_candidates(EUC_BOUNDS, M)
    else:
      rows = _FakePost().fill_candidates(_device_seed(), 0, M, EUC_BOUNDS).numpy()
    return _enc(rows[int(np.argmax(_scores(rows, nan)))]), np.random.get_state()
  dom, kern = _cp()
  parts = A._cp_parts(dom, kern)
  if mode == 'numpy':
    rows, draws = A.draw_cp_candidates(parts, M)
    z = np.random.normal(size=M) if case == 'cp_ts' else 0.0
    i = int(np.argmax(_scores(rows, nan) + z))
    return _enc(A.point_from_draws(parts, draws, i)), np.random.get_state()
  seed = _device_seed()
  kinds, bounds, n_levels, luts = A._cp_device_layout(parts)
  raw = _FakePost().fill_mixed_candidates(seed, 0, M, kinds, bounds, n_levels).numpy()
  rows = raw.copy()
  for c, lut in enumerate(luts):
    if lut is not None:
      rows[:, c] = lut[raw[:, c].astype(int)]
  z = _ts_normals(seed, np.arange(M)) if case == 'cp_ts' else 0.0
  i = int(np.argmax(_scores(rows, nan) + z))
  return _enc(A._cp_point_from_device_row(parts, raw[i])), np.random.get_state()


def _run(case, mode, nan=False, fail_at=-1):
  dom, kern = _euc() if case == 'euc' else _cp()
  gp = _FakeGP(kern, nan, fail_at)
  np.random.seed(0)
  fn = A.asy_ts if case == 'cp_ts' else A.asy_ucb
  try:
    pt = fn(gp, _anc(dom, mode))
  except RuntimeError:
    pt = None
  return pt, np.random.get_state(), gp.trace


def _same_state(a, b):
  return a[0] == b[0] and (a[1] == b[1]).all() and tuple(a[2:]) == tuple(b[2:])


# The scoring calls each case makes: ('score', rows) for the acquisition, ('ts', rows, row0, seed, (len(z), z[0]) or
# None) for Thompson sampling.
SEED0 = 450225092572785199
TRACES = {
  ('euc', 'numpy'): [('score', 32), ('score', 64), ('score', 64), ('score', 64), ('score', 64), ('score', 12)],
  ('euc', 'device'): [('score', 128), ('score', 128), ('score', 44)],
  ('cp_ucb', 'numpy'): [('score', 64), ('score', 64), ('score', 64), ('score', 64), ('score', 44)],
  ('cp_ucb', 'device'): [('score', 128), ('score', 128), ('score', 44)],
  ('cp_ts', 'numpy'): [('ts', 64, 0, 0, (64, -0.324062081632058)), ('ts', 64, 0, 0, (64, 0.1948961564830784)),
                       ('ts', 64, 0, 0, (64, -0.05245121777786827)), ('ts', 64, 0, 0, (64, 1.8873187763318435)),
                       ('ts', 44, 0, 0, (44, 0.6729189302793982))],
  ('cp_ts', 'device'): [('ts', 128, 0, SEED0, None), ('ts', 128, 128, SEED0, None), ('ts', 44, 256, SEED0, None)],
}
CASES = sorted(TRACES)


@pytest.fixture(autouse=True)
def _small_slabs(monkeypatch):
  monkeypatch.setattr(A, 'STREAM_SLAB_ROWS', SLAB)
  monkeypatch.setattr(A, '_shard_info', lambda: (0, 1, None))


@pytest.mark.parametrize('nan', [False, True])
@pytest.mark.parametrize('case,mode', CASES)
def test_point_rng_and_trace(case, mode, nan):
  pt, state, trace = _run(case, mode, nan)
  want_pt, want_state = _expected(case, mode, nan)
  assert _enc(pt) == want_pt
  assert _same_state(state, want_state)
  assert trace == TRACES[(case, mode)]


def test_cases_have_ties_and_nan():
  np.random.seed(0)
  vals = _scores(A.draw_candidates(EUC_BOUNDS, M), False)
  assert (vals == vals.max()).sum() > 1
  np.random.seed(0)
  vals = _scores(A.draw_candidates(EUC_BOUNDS, M), True)
  assert np.isnan(vals).sum() > 1


@pytest.mark.parametrize('case,mode', CASES)
def test_a_failing_slab_still_consumes_the_whole_draw(case, mode):
  pt, state, trace = _run(case, mode, fail_at=2)
  _, want_state = _expected(case, mode, False)
  assert pt is None and len(trace) == 2
  assert _same_state(state, want_state)


def _two_rank_run(monkeypatch, mode, rank, joined):
  """ One rank of a two-rank run: the collectives record this rank's winner and answer with `joined` (or echo). """
  sent = []

  def argmax(score, index, device=None):
    sent.append((score, index, None))
    return joined[:2] if joined else (score, index)

  def argmax_point(score, index, point, dim, device=None):
    sent.append((score, index, None if point is None else np.array(point)))
    return joined if joined else (score, index, point)
  monkeypatch.setattr(A, '_shard_info', lambda: (rank, 2, None))
  monkeypatch.setattr(dfb_dist, 'all_reduce_argmax', argmax)
  monkeypatch.setattr(dfb_dist, 'all_reduce_argmax_point', argmax_point)
  pt, state, trace = _run('euc', mode, nan=False)
  return pt, state, trace, sent[0]


@pytest.mark.parametrize('mode', ['numpy', 'device'])
def test_two_ranks(monkeypatch, mode):
  local = [_two_rank_run(monkeypatch, mode, r, None)[3] for r in range(2)]
  assert local[0][1] < M // 2 <= local[1][1]
  s, i = dfb_dist.reduce_pairs([l[0] for l in local], [l[1] for l in local])
  joined = (s, i, [l[2] for l in local if l[1] == i][0])
  want_pt, want_state = _expected('euc', mode, False)
  traces = []
  for r in range(2):
    pt, state, trace, _ = _two_rank_run(monkeypatch, mode, r, joined)
    assert _enc(pt) == want_pt
    assert _same_state(state, want_state)
    traces.append(trace)
  want = {'numpy': [[('score', 32), ('score', 64), ('score', 54)], [('score', 10), ('score', 64), ('score', 64),
                                                                       ('score', 12)]],
          'device': [[('score', 128), ('score', 22)], [('score', 128), ('score', 22)]]}[mode]
  assert traces == want


def test_scorer_only_maximiser_checks_the_candidate_rng():
  anc = Namespace(domain=domains.EuclideanDomain(EUC_BOUNDS), max_evals=10, candidate_rng='philox')
  scorer = lambda pts: (0.0, 0, None)
  with pytest.raises(ValueError):
    A._fused_maximise(scorer, anc)
  anc.candidate_rng = 'device'
  with pytest.raises(NotImplementedError):
    A._fused_maximise(scorer, anc)
