"""
The posterior build's error bounds (tests/build_ref.py) on the CPU, against the NumPy emulation of the blocked
algorithm: they hold with margin over random, clustered and ill-conditioned matrices at the tile edges, and each of the
defects a broken schedule or kernel would produce violates one of them by a wide factor.
"""
import numpy as np
import pytest

import build_ref as BR

SIZES = [1, 127, 128, 129, 300]
MARGIN = 0.5          # a bound that holds must hold with at least this much to spare
WIDE = 1e3            # a defect must exceed its bound by at least this factor


def test_long_double_is_extended():
  assert np.finfo(np.longdouble).nmant >= 63


def se_matrix(X, bw):
  d2 = (((X[:, None, :] - X[None, :, :]) / bw) ** 2).sum(-1)
  return np.exp(-0.5 * d2)


def make_case(kind, n, seed=0):
  """ (A, y, npad): an SE kernel matrix + noise on the diagonal, identity on the padding. """
  rs = np.random.RandomState(1000 * n + seed)
  if kind == 'random':
    X, noise = rs.random_sample((n, 3)), 1e-2
  elif kind == 'well':                         # well-conditioned: stays positive definite under every defect
    X, noise = rs.random_sample((n, 3)), 0.5
  elif kind == 'clustered':                    # a few tight clusters: many nearly equal rows
    X = rs.random_sample((4, 3))[rs.randint(0, 4, n)] + 1e-3 * rs.standard_normal((n, 3))
    noise = 1e-6
  else:                                        # ill-conditioned: clustered points and noise 1e-10 of the scale
    X = rs.random_sample((3, 3))[rs.randint(0, 3, n)] + 1e-4 * rs.standard_normal((n, 3))
    noise = 1e-10
  K = 1.7 * se_matrix(X, 0.05 if kind == 'well' else 0.4)
  npad = -(-n // BR.T) * BR.T
  y = BR.pad_vector(rs.standard_normal(n), npad)
  return BR.pad_matrix(K, noise, npad), y, npad, noise


def run(A, y, n, **kw):
  L, W, v, alpha = BR.emulate(A, y, **kw)
  lml_full, lml_v = BR.emulate_lml(L, v, y, alpha, n)
  return L, W, v, alpha, lml_full, lml_v


@pytest.mark.parametrize('kind', ['random', 'clustered', 'ill'])
@pytest.mark.parametrize('n', SIZES)
def test_bounds_hold_on_the_emulation(kind, n):
  A, y, npad, _ = make_case(kind, n)
  L, W, v, alpha, lml_full, lml_v = run(A, y, n)
  r = BR.check_build(A, y, L, W, v, alpha=alpha, lml=lml_full, lml_quad='alpha', n=n)
  r['lml_v'] = BR.check_build(A, y, L, W, v, lml=lml_v, lml_quad='v', n=n)['lml']
  assert max(r.values()) <= MARGIN, r


@pytest.mark.parametrize('n', [129, 300])
def test_diagonal_tiles_of_W_are_the_explicit_inverses(n):
  """ The X tile (J, J) is an exact identity until step J, so the panel leaves D_J^T there bit for bit. """
  A, y, npad, _ = make_case('random', n)
  L, W, _, _ = BR.emulate(A, y)
  from scipy.linalg import solve_triangular
  for J in range(npad // BR.T):
    s = BR.blk(J)
    # the emulation computed D_J from the diagonal tile of the trailing matrix; recompute it from L's tile
    D = np.tril(solve_triangular(L[s, s], np.eye(BR.T), lower=True))
    assert np.array_equal(W[s, s], D)


def test_padding_row_is_exact_on_the_emulation():
  A, y, npad, _ = make_case('random', 300)
  L, W, v, alpha = BR.emulate(A, y)
  assert (L[300:, :300] == 0).all() and (np.diag(L)[300:] == 1).all()
  assert (W[300:, :300] == 0).all() and (np.diag(W)[300:] == 1).all()
  assert (v[300:] == 0).all() and (alpha[300:] == 0).all()


def defect_ratio(defect):
  n = 300
  A, y, npad, noise = make_case('well', n)
  if defect in ('drop_slab', 'tile_twice', 'stale_D'):
    L, W, v, alpha = BR.emulate(A, y, defect=defect, at=1)
  elif defect == 'noise_twice':
    A2 = A.copy()
    A2[157, 157] += noise
    L, W, v, alpha = BR.emulate(A2, y)
  else:                                        # 'W_padding_row': one entry of a padding row of W (left of its tile)
    L, W, v, alpha = BR.emulate(A, y)
    W = W.copy()
    W[npad - 1, 5] = 2.0 ** -40
  r = BR.check_build(A, y, L, W, v, alpha=alpha, n=n)
  return r


@pytest.mark.parametrize('defect,which', [('drop_slab', 'L'), ('tile_twice', 'L'), ('stale_D', 'D'),
                                          ('noise_twice', 'L'), ('W_padding_row', 'W')])
def test_each_defect_violates_a_bound_widely(defect, which):
  r = defect_ratio(defect)
  print('%s: residual / bound = %s' % (defect, {k: '%.3g' % x for k, x in r.items()}))
  assert r[which] >= WIDE, ('%s: residual / bound of %s is only %.3g' % (defect, which, r[which]), r)
