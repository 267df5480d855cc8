"""
The posterior build's diagonal-block Cholesky (kernels.cu: chol_diag_kernel, one column block at a time) against the
elimination of the batched LML builds (chol_diag_block) on the device (-m gpu), through dfb_debug_chol_diag: for every input the
two must leave the same bits in the block (L, d_j on the diagonal, zeros above) and in L^-1, and report the same info.

Inputs, all seeded: kernel matrices (SE, Matern 1/2, 3/2, 5/2) with noise from 1 down to 1e-10 of the scale; random
SPD blocks; identity-padded last blocks (n mod 128 = 1, 8 -- the last block of N = 5000 --, 37, 127); Schur
complements A22 - L21 L21^T of kernel matrices, the blocks a blocked factorisation meets part-way; a non-positive
pivot at j in {0, 1, 31, 32, 33, 63, 64, 95, 96, 127}; NaN entries; -0.0 entries; an infinite pivot and an L^-1 that
overflows (rows with non-finite values); symmetric indefinite blocks.  On failure neither elimination may write
anything: the block stays the input's copy and L^-1 the NaN sentinel the outputs are filled with.
"""
from argparse import Namespace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NB = 128
BAD_PIVOTS = [0, 1, 31, 32, 33, 63, 64, 95, 96, 127]


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import device, _lib
  _lib.load()
  return Namespace(torch=torch, post=device.DevicePosterior(64))


def _bits(G, t):
  return t.contiguous().view(G.torch.int64).cpu().numpy()


def _run(G, A):
  """ Both eliminations on the host block A (128 x 128, or a device view); returns (info, blk, dinv) of each. """
  blk = A if isinstance(A, G.torch.Tensor) else G.torch.from_numpy(np.ascontiguousarray(A)).cuda()
  return [G.post.debug_chol_diag(which, blk) for which in (0, 1)], blk


def _check_same(G, A, expect_info=None):
  (r0, r1), blk = _run(G, A)
  info0, b0, d0 = r0
  info1, b1, d1 = r1
  assert info1 == info0, (info0, info1)
  if expect_info is not None:
    assert info0 == expect_info, (info0, expect_info)
  bits_b0, bits_b1, bits_d0, bits_d1 = _bits(G, b0), _bits(G, b1), _bits(G, d0), _bits(G, d1)
  nb, nd = int((bits_b0 != bits_b1).sum()), int((bits_d0 != bits_d1).sum())
  assert nb == 0 and nd == 0, 'info %d: %d block and %d L^-1 elements differ' % (info0, nb, nd)
  if info0 != 0:
    sentinel = G.torch.full((1,), float('nan'), dtype=G.torch.float64).view(G.torch.int64).item()
    assert (bits_b1 == _bits(G, blk)).all(), 'a failed elimination wrote to the block'
    assert (bits_d1 == sentinel).all(), 'a failed elimination wrote to L^-1'
  return info0, b1.cpu().numpy(), d1.cpu().numpy()


def _kernel_matrix(rng, kind, n, d=6, scale=2.0):
  X = rng.uniform(0.0, 1.0, size=(n, d))
  bw = rng.uniform(0.2, 0.8, size=d)
  Z = X / bw
  D2 = np.maximum(((Z[:, None, :] - Z[None, :, :]) ** 2).sum(-1), 0.0)
  r = np.sqrt(D2)
  if kind == 'se':
    K = np.exp(-0.5 * D2)
  elif kind == 'm12':
    K = np.exp(-r)
  elif kind == 'm32':
    K = (1 + np.sqrt(3) * r) * np.exp(-np.sqrt(3) * r)
  else:
    K = (1 + np.sqrt(5) * r + 5.0 / 3.0 * D2) * np.exp(-np.sqrt(5) * r)
  return scale * K


def _spd(rng, n=NB):
  M = rng.standard_normal((n, n))
  return M @ M.T / n + 0.1 * np.eye(n)


KINDS = ['se', 'm12', 'm32', 'm52']
NOISES = [1.0, 1e-2, 1e-4, 1e-6, 1e-8, 1e-10]


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('noise', NOISES)
def test_kernel_blocks(G, kind, noise):
  rng = np.random.default_rng(100 * KINDS.index(kind) + NOISES.index(noise))
  A = _kernel_matrix(rng, kind, NB)
  A[np.diag_indices(NB)] += noise * 2.0
  info, L, Dinv = _check_same(G, A)
  if noise >= 1e-4:
    assert info == 0
    Lf = np.tril(L, -1) + np.diag(np.diag(L))
    assert np.abs(Lf @ Lf.T - A).max() <= 1e-12 * np.abs(A).max()
    assert np.abs(Dinv @ Lf - np.eye(NB)).max() <= 1e-8


@pytest.mark.parametrize('seed', range(6))
def test_random_spd(G, seed):
  rng = np.random.default_rng(1000 + seed)
  A = _spd(rng)
  if seed % 2:
    A = A * 10.0 ** rng.uniform(-200, 200)        # scales outside the pivot sequence's fast range
  assert _check_same(G, A)[0] == 0


@pytest.mark.parametrize('rem', [1, 8, 37, 127])
def test_identity_padding(G, rem):
  rng = np.random.default_rng(rem)
  A = np.eye(NB)
  K = _kernel_matrix(rng, 'm52', rem)
  K[np.diag_indices(rem)] += 1e-6
  A[:rem, :rem] = K
  assert _check_same(G, A)[0] == 0


@pytest.mark.parametrize('kind,k', [('m52', 1), ('se', 2), ('m32', 3), ('m12', 1)])
def test_schur_complement(G, kind, k):
  """ The trailing block a factorisation meets after k block steps (formed on the host: both eliminations take it). """
  rng = np.random.default_rng(7 * k + len(kind))
  n = (k + 1) * NB
  A = _kernel_matrix(rng, kind, n)
  A[np.diag_indices(n)] += 1e-6 * 2.0
  L11 = np.linalg.cholesky(A[:k * NB, :k * NB])
  L21 = np.linalg.solve(L11, A[:k * NB, k * NB:]).T
  S = A[k * NB:, k * NB:] - L21 @ L21.T
  _check_same(G, S)


def test_leading_dimension(G):
  """ The block as a view into a wider matrix (ld = 384). """
  rng = np.random.default_rng(5)
  A = _kernel_matrix(rng, 'm52', 3 * NB)
  A[np.diag_indices(3 * NB)] += 1e-4
  At = G.torch.from_numpy(A).cuda()
  assert _check_same(G, At[NB:2 * NB, NB:2 * NB])[0] == 0


@pytest.mark.parametrize('j', BAD_PIVOTS)
def test_non_positive_pivot(G, j):
  rng = np.random.default_rng(j)
  L = np.tril(rng.standard_normal((NB, NB)) / np.sqrt(NB), -1) + np.diag(rng.uniform(1.0, 2.0, NB))
  D = np.ones(NB)
  D[j] = -1.0
  A = (L * D) @ L.T
  _check_same(G, A, expect_info=j + 1)
  A[j, j] = 0.0                                      # an exactly zero first pivot (j = 0), else a cancelled one
  _check_same(G, A)


@pytest.mark.parametrize('where', ['diag0', 'diag64', 'lower', 'upper_only', 'last'])
def test_nan_entries(G, where):
  rng = np.random.default_rng(11)
  A = _spd(rng)
  if where == 'diag0':
    A[0, 0] = np.nan
  elif where == 'diag64':
    A[64, 64] = np.nan
  elif where == 'lower':
    A[90, 40] = np.nan
  elif where == 'upper_only':
    A[40, 90] = np.nan                               # above the diagonal: never read
  else:
    A[127, 126] = np.nan
  info, _, _ = _check_same(G, A)
  assert (info == 0) == (where == 'upper_only')


@pytest.mark.parametrize('case', ['diagonal', 'banded', 'kernel'])
def test_negative_zero_entries(G, case):
  rng = np.random.default_rng(13)
  if case == 'diagonal':
    A = np.diag(rng.uniform(0.5, 2.0, NB))
    A[A == 0.0] = -0.0
  elif case == 'banded':
    A = np.diag(rng.uniform(2.0, 3.0, NB))
    off = rng.uniform(-0.5, 0.5, NB - 1)
    A[np.arange(1, NB), np.arange(NB - 1)] = off
    A[np.arange(NB - 1), np.arange(1, NB)] = off
    A[A == 0.0] = -0.0
  else:
    A = _kernel_matrix(rng, 'm12', NB)
    A[np.diag_indices(NB)] += 1e-3
    A[rng.random((NB, NB)) < 0.2] = -0.0
    iu = np.triu_indices(NB, 1)
    A[iu] = A.T[iu]                                  # symmetric, keeping the -0.0 of the lower triangle
    A[np.diag_indices(NB)] = np.abs(A).sum(1) + 1.0  # diagonally dominant
  assert _check_same(G, A)[0] == 0


def test_infinite_pivot(G):
  A = _spd(np.random.default_rng(17))
  A[50, 50] = np.inf                                 # passes the pivot test: d = inf, 1 / d = 0
  _check_same(G, A)


def test_overflowing_inverse(G):
  """ A = L L^T for the bidiagonal L = (2^-20 on the diagonal, 1 below it), exact in floating point: every pivot is
  2^-40, and L^-1 = (-1)^(i-j) 2^(20 (i-j+1)) overflows 52 rows below the diagonal, so rows end with non-finite
  values. """
  d = 2.0 ** -20
  A = np.diag(np.full(NB, 1.0 + d * d))
  A[0, 0] = d * d
  A[np.arange(1, NB), np.arange(NB - 1)] = d
  A[np.arange(NB - 1), np.arange(1, NB)] = d
  info, _, Dinv = _check_same(G, A)
  assert info == 0 and not np.isfinite(Dinv).all()


@pytest.mark.parametrize('seed', range(4))
def test_symmetric_indefinite(G, seed):
  rng = np.random.default_rng(31 + seed)
  M = rng.standard_normal((NB, NB))
  A = M + M.T + (NB / 4.0) * np.eye(NB)
  _check_same(G, A)
