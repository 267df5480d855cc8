"""
Host logic of the joint Thompson draw (gp_core.GP._draw_samples_on, gp_core.joint_draw_on_device,
gpb_acquisitions._ts_cols) with a NumPy stand-in for DevicePosterior: which form a draw takes for a given M, the
global RNG, one factorisation per call, stable_cholesky's jitter ladder, and the oracle's joint draw against the
reference's golden (tests/golden/ts_joint.npz).  No GPU.
"""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import gp_oracle as O
from dragonfly_b200 import gp_core, gpb_acquisitions


class StandInPost(object):
  """ What _draw_samples_on needs of DevicePosterior.  ts_draws records (m, S, jitter) and returns zeros + mu, or
      -- with fail_below -- info = 1 while jitter < fail_below. """
  TS_BLOCK = 4096
  TS_JOINT_MAX = 16384

  def __init__(self, max_diag=2.0, fail_below=None):
    self.calls = []
    self.max_diag, self.fail_below = max_diag, fail_below

  def ts_draws(self, Xc, Ut, mean_const=0.0, jitter=0.0):
    m, S = len(Xc), Ut.shape[0]
    assert Ut.shape == (S, m)
    self.calls.append((m, S, jitter))
    if self.fail_below is not None and not jitter >= self.fail_below:
      return 1, None, self.max_diag
    return 0, torch.from_numpy(np.full((S, m), float(mean_const)) + 0.0 * Ut), self.max_diag


class StandInGP(object):
  """ The two GP helpers _draw_samples_on calls. """
  def _test_matrix(self, X):
    return X

  def _mean_const_for(self, X):
    return 0.5


def draw(post, S, M):
  X = np.zeros((M, 2))
  return gp_core.GP._draw_samples_on(StandInGP(), post, S, X)


@pytest.mark.parametrize('M,joint', [(4096, False), (4097, True), (16384, True), (16385, False)])
def test_path_is_chosen_by_m(M, joint):
  post = StandInPost()
  out = draw(post, 3, M)
  assert out.shape == (3, M) and (out == 0.5).all()
  ms = [c[0] for c in post.calls]
  if joint:
    assert ms == [M]
  else:
    assert max(ms) <= 4096 and sum(ms) == M


@pytest.mark.parametrize('M', [4096, 6000, 16385])
def test_global_rng_advances_as_one_normal_matrix(M):
  np.random.seed(8)
  draw(StandInPost(), 5, M)
  after = np.random.random(4)
  np.random.seed(8)
  np.random.normal(size=(M, 5))
  assert (np.random.random(4) == after).all()


def test_joint_draw_passes_the_normals_transposed():
  seen = []

  class Recording(StandInPost):
    def ts_draws(self, Xc, Ut, mean_const=0.0, jitter=0.0):
      seen.append(np.array(Ut))
      return StandInPost.ts_draws(self, Xc, Ut, mean_const, jitter)
  np.random.seed(4)
  draw(Recording(), 7, 5000)
  np.random.seed(4)
  U = np.random.normal(size=(5000, 7))
  assert len(seen) == 1 and (seen[0] == U.T).all()


def test_many_draws_factorise_once():
  post = StandInPost()
  draw(post, 300, 5000)
  assert post.calls == [(5000, 300, 0.0)]
  post = StandInPost()
  draw(post, 300, 4000)                     # the block form: passes of <= 256 draws
  assert [c[1] for c in post.calls] == [256, 44]


def test_jitter_ladder_powers():
  max_diag = 3.0
  post = StandInPost(max_diag=max_diag, fail_below=(10 ** -7) * max_diag * (1 - 1e-12))
  smp, power = gp_core.joint_draw_on_device(post, np.zeros((5000, 2)), np.zeros((2, 5000)), 0.0)
  assert power == -7 and smp.shape == (2, 5000)
  assert [c[2] for c in post.calls] == [0.0] + [(10 ** p) * max_diag for p in range(-11, -6)]


def test_jitter_ladder_gives_up_at_power_five():
  max_diag = 3.0
  post = StandInPost(max_diag=max_diag, fail_below=np.inf)
  with pytest.raises(ValueError):
    gp_core.joint_draw_on_device(post, np.zeros((5000, 2)), np.zeros((1, 5000)), 0.0)
  assert [c[2] for c in post.calls] == [0.0] + [(10 ** p) * max_diag for p in range(-11, 5)]


def test_ranks_do_not_split_a_joint_draw(monkeypatch):
  monkeypatch.setattr(gpb_acquisitions, '_shard_info', lambda: (1, 2, None))

  class G(object):
    _post = StandInPost()
  assert gpb_acquisitions._ts_cols(G(), 4096) is not None        # one block: sharded as before
  assert gpb_acquisitions._ts_cols(G(), 4097) is None
  assert gpb_acquisitions._ts_cols(G(), 16384) is None
  cols = gpb_acquisitions._ts_cols(G(), 16385)       # above the cap: rank 1's whole blocks
  assert cols is not None and cols[0] % 4096 == 0 and cols[0] > 0 and cols[1] == 16385


def _golden_gp(g):
  kern = O.OMaternKernel(6, 2.5, float(g['scale1']), g['bws1'])
  return O.OGP(g['X'], g['Y1'], kern, lambda x: np.array([float(g['mean1'])] * len(x)), float(g['noise1']))


def test_oracle_joint_draw_reproduces_the_golden():
  g = load_golden('ts_joint')
  gp = _golden_gp(g)
  mu, covar = gp.eval(g['C'], 'covar')
  assert np.abs(mu - g['mu']).max() <= 1e-10
  assert np.abs(np.diag(covar) - g['covar_diag']).max() <= 1e-10
  idx = g['covar_idx']
  assert np.abs(covar[idx[:, 0], idx[:, 1]] - g['covar_vals']).max() <= 1e-10
  samples = O.draw_gaussian_samples_with_normals(mu, covar, g['U'])
  assert np.abs(samples - g['samples']).max() <= 1e-7
  assert (samples.argmax(axis=1) == g['samples'].argmax(axis=1)).all()
