"""
The joint Thompson draw over 4096 < M <= 16384 candidates (-m gpu): dfb_ts_draws / dfb_eval_covar on the joint
workspace (the covariance in row slabs, the factor-only mode of the blocked factorisation, the L U product in passes
of 256 draws) against the 4096-candidate block path bit for bit, against fp64 backward-error bounds, and against the
UNMODIFIED reference (tests/golden/ts_joint.npz, M = 6000).
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest

import build_ref as BR
import contract_ref as CR
from conftest import load_golden

pytestmark = pytest.mark.gpu

T = 128
SAMPLE_TOL = 2e-6           # |device - reference| of a posterior draw (the block path's tolerance)
VAR_TOL = 1e-8


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, gp_core, device, _lib, domains, mf_gp
  from dragonfly_b200 import gpb_acquisitions as acq
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  from oracle import gp_oracle as O
  _lib.load()
  return Namespace(torch=torch, kernel=kernel, gp_core=gp_core, device=device, lib=_lib, domains=domains,
                   mf_gp=mf_gp, acq=acq, moo=moo, O=O)


def _copy(B, post, name, count):
  t = B.torch.empty((count,), dtype=B.torch.float64, device=post.device)
  B.lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), C.c_void_p(t.data_ptr()), t.numel() * 8), 'dfb_debug_copy')
  return t.cpu().numpy()


def bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def assert_same(a, b, what):
  a, b = np.asarray(a), np.asarray(b)
  assert a.shape == b.shape, (what, a.shape, b.shape)
  bad = np.argwhere(bits(a) != bits(b))
  assert len(bad) == 0, (what, 'differs in', len(bad), 'entries; first', tuple(bad[0]))


def joint_cov(B, post, m):
  """ The joint buffer js_Cov as its q x q matrix (q = m rounded up to 128). """
  mj = -(-post._js_m // T) * T
  q = -(-m // T) * T
  return _copy(B, post, 'js_Cov', mj * mj)[:q * q].reshape(q, q)


def block_cov(B, post, m):
  q = -(-m // T) * T
  mb = -(-post._ts_mb // T) * T
  return _copy(B, post, 'ts_Cov', mb * mb)[:q * q].reshape(q, q)


def block_T(B, post, m):
  q = -(-m // T) * T
  mb = -(-post._ts_mb // T) * T
  return _copy(B, post, 'ts_T', (2 * mb + T) * mb)[:(2 * q + T) * q].reshape(2 * q + T, q)


def with_chunk(B, chunk, make):
  """ make() with new posteriors at scoring chunk `chunk` (0: the library default). """
  B.gp_core.DEFAULT_CHUNK[0] = chunk
  try:
    return make()
  finally:
    B.gp_core.DEFAULT_CHUNK[0] = 0


def matern_gp(B, n, seed=3, d=6, chunk=0):
  rs = np.random.RandomState(seed)
  X = rs.random_sample((n, d))
  Y = np.sin(3 * X).sum(axis=1)
  gp = with_chunk(B, chunk, lambda: B.gp_core.GP(X, Y, B.kernel.MaternKernel(d, 2.5, 1.3, [0.4] * d),
                                                 B.gp_core.ConstantMean(0.1), 1e-3 * 1.3))
  return gp, rs


def slabs(post, M):
  """ Row slabs the joint covariance is formed in (one scoring chunk each). """
  return -(-(-(-M // T) * T) // int(post.query('chunk')))


def factor_rows_ratio(L, A, rows):
  """ tests/build_ref.py's diagonal-tile / panel bound (items 1-2) on the given rows of the factor-only mode's L
      against A = Sigma + jI with identity padding, residual in long double (contract_ref.factor_check on a row
      subset: the whole matrix is out of reach of a long-double product at these sizes). """
  q = L.shape[0]
  bound = BR.tall_bound(L[rows], A[rows], L, CR._FactorBlocks(L), row_block=rows // T)
  res = BR.factor_residual(L, A, rows)
  return BR._ratio(res, bound, np.arange(q)[None, :] <= rows[:, None])


def padded_input(sig, M, jitter):
  """ Sigma + jitter I (lower triangle mirrored) with identity padding: what the factorisation starts from. """
  q = sig.shape[0]
  A = np.tril(sig) + np.tril(sig, -1).T
  A[M:, :] = 0.0
  A[:, M:] = 0.0
  idx = np.arange(M)
  A[idx, idx] = A[idx, idx] + np.float64(jitter)
  A[np.arange(M, q), np.arange(M, q)] = 1.0
  return A


# ---- 1. the leading block, bit for bit --------------------------------------------------------------------------------
@pytest.mark.parametrize('M,n', [(9000, 1100), (16384, 1100), (9000, 5000), (16384, 5000)])
def test_leading_block_is_the_block_path(B, M, n):
  """ At N = 5000 the scoring chunk is 6528 rows, so the covariance is formed in 2 (M = 9000) or 3 (M = 16384) slabs. """
  gp, rs = matern_gp(B, n)
  post = gp._post
  print('slabs M=%d n=%d: %d' % (M, n, slabs(post, M)))
  Xc = rs.random_sample((M, 6))
  S = 6
  Ut = rs.standard_normal((S, M))
  mu_j, cov_j = post.eval_covar(Xc[:M], mean_const=0.1)
  assert cov_j.shape == (M, M)
  sig_j = joint_cov(B, post, M)
  mu_b, cov_b = post.eval_covar(Xc[:4096], mean_const=0.1)
  sig_b = block_cov(B, post, 4096)
  assert_same(sig_j[:4096, :4096], sig_b, 'Sigma leading block')
  assert_same(cov_j[:4096, :4096], cov_b, 'eval_covar leading block')
  assert_same(mu_j[:4096], mu_b, 'mu leading block')
  del cov_j
  info, smp_j, _ = post.ts_draws(Xc, Ut, mean_const=0.1)
  assert info == 0
  L_j = joint_cov(B, post, M)
  info, smp_b, _ = post.ts_draws(Xc[:4096], np.ascontiguousarray(Ut[:, :4096]), mean_const=0.1)
  assert info == 0
  L_b = np.tril(block_T(B, post, 4096)[:4096])
  assert_same(np.tril(L_j[:4096, :4096]), L_b, 'L leading block')
  assert_same(smp_j.cpu().numpy()[:, :4096], smp_b.cpu().numpy(), 'samples leading block')
  assert np.isfinite(smp_j.cpu().numpy()).all()


# ---- 2. covariance bound ------------------------------------------------------------------------------------------------
def _tile_rows(M, tiles):
  return np.concatenate([np.arange(t * T, min(M, (t + 1) * T)) for t in tiles])


@pytest.mark.parametrize('M,n,chunk', [(4097, 300, 0), (6000, 1000, 0), (16384, 700, 0), (4097, 300, 1024),
                                       (6000, 1000, 1024), (16384, 700, 1024)])
def test_covariance_tiles_meet_the_bound(B, M, n, chunk):
  """ Whole tiles spread over the joint covariance (off-diagonal tiles included; with chunk = 1024 they sit in
      different row slabs, among them both sides of slab boundaries) equal the block covariance of the same candidates
      bit for bit, and that meets contract_ref's covariance bound.  n is not a multiple of 128. """
  gp, rs = matern_gp(B, n, seed=5, chunk=chunk)
  post = gp._post
  Xc = rs.random_sample((M, 6))
  post.eval_covar(Xc)
  sig = joint_cov(B, post, M)
  nt = -(-M // T)
  tiles = sorted(set([0, 1, 7, 8, nt // 2 - 1, nt // 2, nt - 2, nt - 1]))   # 8 tiles: within a 1024-row block
  rows = _tile_rows(M, tiles)
  _, cov_s = post.eval_covar(Xc[rows])
  assert_same(sig[np.ix_(rows, rows)], cov_s, 'joint tiles vs block covariance of the same candidates')
  npad = int(post.query('npad')); chunk = int(post.query('chunk'))
  Ks = _copy(B, post, 'Ks', chunk * npad).reshape(chunk, npad)[:len(rows)]
  W = _copy(B, post, 'W', npad * npad).reshape(npad, npad)
  r = CR.covariance_check(cov_s, Ks, W, ('matern', 2, 1.3, np.array([0.4] * 6), Xc[rows]))
  print('RATIO covariance M=%d n=%d chunk=%d slabs=%d %.3g' % (M, n, chunk, slabs(post, M), r))
  assert r <= 1.0


def test_every_lower_tile_is_the_block_covariance(B):
  """ M = 16384 at N = 5000 (three row slabs of 6528): every lower tile of the joint covariance, and mu, equal the
      block covariance of the same candidates bit for bit -- the tiles are taken 16 x 16 groups at a time, two groups
      (4096 candidates) per block call.  Together with the bound on blocks (C3 and the test above) every tile meets
      the covariance bound. """
  gp, rs = matern_gp(B, 5000, seed=6)
  post = gp._post
  M, G = 16384, 16
  Xc = rs.random_sample((M, 6))
  mu_j, _ = post.eval_covar(Xc)
  assert slabs(post, M) == 3
  sig = joint_cov(B, post, M)
  groups = [np.arange(g * G * T, (g + 1) * G * T) for g in range(M // (G * T))]
  for a in range(len(groups)):
    for b in range(a + 1):
      rows = np.concatenate((groups[b], groups[a])) if a != b else groups[a]
      mu_b, cov_b = post.eval_covar(Xc[rows])
      assert_same(sig[np.ix_(rows, rows)][np.tril_indices(len(rows))], cov_b[np.tril_indices(len(rows))],
                  'lower tiles of groups (%d, %d)' % (a, b))
      assert_same(mu_j[rows], mu_b, 'mu of groups (%d, %d)' % (a, b))


def test_covariance_on_a_hallucinated_posterior(B):
  """ 50 evaluations in progress on N = 600 exceed the padded size (640), so a fresh (N + q)-point posterior is built,
      with its own joint workspace: its tiles equal its block covariance of the same candidates bit for bit, meet the
      covariance bound, and GP.eval_with_hallucinated_observations returns that covariance. """
  gp, rs = matern_gp(B, 600, seed=8)
  M = 5000
  Xc = rs.random_sample((M, 6))
  H = list(rs.random_sample((50, 6)))
  mu_e, cov_e = gp.eval_with_hallucinated_observations(Xc, H, 'covar')
  with gp._hallucinated(H) as post:
    assert post is not gp._post and post.n == 650
    mu, cov = post.eval_covar(Xc, mean_const=0.1)
    assert_same(cov, cov_e, 'eval_with_hallucinated_observations vs the augmented posterior')
    sig = joint_cov(B, post, M)
    nt = -(-M // T)
    rows = _tile_rows(M, [0, 5, nt // 2, nt - 1])
    _, cov_s = post.eval_covar(Xc[rows])
    assert_same(sig[np.ix_(rows, rows)], cov_s, 'augmented joint tiles vs block covariance')
    npad = int(post.query('npad')); chunk = int(post.query('chunk'))
    Ks = _copy(B, post, 'Ks', chunk * npad).reshape(chunk, npad)[:len(rows)]
    W = _copy(B, post, 'W', npad * npad).reshape(npad, npad)
  r = CR.covariance_check(cov_s, Ks, W, ('matern', 2, 1.3, np.array([0.4] * 6), Xc[rows]))
  print('RATIO covariance hallucinated %.3g' % r)
  assert r <= 1.0


# ---- 3. factor residual -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,chunk', [(4097, 0), (6000, 1024)])
def test_factor_meets_the_build_bound(B, M, chunk):
  """ The factor-only mode against build_ref's diagonal-tile / panel bound, on the rows of the last row block (beyond
      the leading 4096, where the leading-block test does not reach) and of the first. """
  gp, rs = matern_gp(B, 700, seed=10, chunk=chunk)
  post = gp._post
  Xc = rs.random_sample((M, 6))
  post.eval_covar(Xc)
  sig = joint_cov(B, post, M)
  j = 1e-9 * float(np.diag(sig)[:M].max())
  info, _, _ = post.ts_draws(Xc, rs.standard_normal((1, M)), mean_const=0.1, jitter=j)
  assert info == 0
  L = np.tril(joint_cov(B, post, M))
  q = L.shape[0]
  rows = np.r_[0:T, q - T:q]
  r = factor_rows_ratio(L, padded_input(sig, M, j), rows)
  print('RATIO factor (build bound) M=%d chunk=%d %.3g' % (M, chunk, r))
  assert r <= 1.0


@pytest.mark.parametrize('M', [6000, 16384])
def test_factor_backward_error(B, M):
  """ The factor-only mode's L against Sigma + jI: |fl(L L^T) - A| <= 4 q u |L| |L|^T + 2 u |A| elementwise (q = the
      padded order; the Cholesky backward error, the panel's multiply by inv(L_kk) at a jitter of 1e-6 of the
      largest variance, and the fp64 evaluation of L L^T on the device). """
  t = B.torch
  gp, rs = matern_gp(B, 900, seed=9)
  post = gp._post
  Xc = rs.random_sample((M, 6))
  post.eval_covar(Xc)
  A = t.from_numpy(joint_cov(B, post, M)).cuda()
  j = 1e-6 * float(A.diagonal().max())
  A = t.tril(A) + t.tril(A, -1).T
  A.diagonal().add_(j)
  q = A.shape[0]
  A[M:, :] = 0; A[:, M:] = 0
  A.diagonal()[M:] = 1.0
  info, _, _ = post.ts_draws(Xc, rs.standard_normal((1, M)), jitter=j)
  assert info == 0
  L = t.tril(t.from_numpy(joint_cov(B, post, M)).cuda())
  u = 2.0 ** -53
  res = (L @ L.T - A).abs()
  bound = 4 * q * u * (L.abs() @ L.abs().T) + 2 * u * A.abs() + 1e-300
  ratio = float((res / bound).max())
  print('RATIO factor M=%d %.3g' % (M, ratio))
  assert ratio <= 1.0


# ---- 4. against the reference ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module', params=[0, 1024], ids=['chunk_default', 'chunk_1024'])
def golden_gps(B, request):
  """ The golden's GPs at the default scoring chunk (one slab) and at a chunk of 1024 rows (six slabs). """
  g = load_golden('ts_joint')

  def make():
    gp1 = B.gp_core.GP(g['X'], g['Y1'], B.kernel.MaternKernel(6, 2.5, float(g['scale1']), list(g['bws1'])),
                       B.gp_core.ConstantMean(float(g['mean1'])), float(g['noise1']))
    gp2 = B.gp_core.GP(g['X'], g['Y2'], B.kernel.SEKernel(6, float(g['scale2']), list(g['bws2'])),
                       B.gp_core.ConstantMean(float(g['mean2'])), float(g['noise2']))
    return gp1, gp2
  gp1, gp2 = with_chunk(B, request.param, make)
  if request.param:
    assert slabs(gp1._post, len(g['C'])) == 6
  return g, gp1, gp2


def test_samples_and_covariance_match_the_reference(B, golden_gps):
  g, gp1, _ = golden_gps
  np.random.seed(11)
  S = gp1.draw_samples(4, g['C'])
  assert np.abs(S - g['samples']).max() <= SAMPLE_TOL
  assert (S.argmax(axis=1) == g['samples'].argmax(axis=1)).all()
  mu, cov = gp1.eval(g['C'], 'covar')
  idx = g['covar_idx']
  assert np.abs(np.diag(cov) - g['covar_diag']).max() <= VAR_TOL
  assert np.abs(cov[idx[:, 0], idx[:, 1]] - g['covar_vals']).max() <= VAR_TOL
  assert np.abs(mu - g['mu']).max() <= 1e-10


def test_recommendations_match_the_reference(B, golden_gps):
  g, gp1, gp2 = golden_gps
  dom = B.domains.EuclideanDomain([[0, 1]] * 6)
  anc = Namespace(max_evals=6000, t=len(g['X']), domain=dom, acq_opt_method='rand', handle_parallel='halluc',
                  eval_points_in_progress=[], is_mf=False, obj_weights=g['weights'], reference_point=list(g['refs']),
                  curr_max_val=float(g['Y1'].max()), mf_strategy=None)
  np.random.seed(int(g['asy_ts_seed']))
  pt = B.acq.asy.ts(gp1, anc)
  assert (np.asarray(pt) == g['asy_ts_point']).all()
  np.random.seed(int(g['lin_ts_seed']))
  pt = B.moo.asy.lin_ts([gp1, gp2], anc)
  assert (np.asarray(pt) == g['lin_ts_point']).all()


# ---- 5. jitter ----------------------------------------------------------------------------------------------------------
def test_jitter_ladder_matches_the_oracle(B):
  gp, rs = matern_gp(B, 400, seed=12)
  Xc = rs.random_sample((4500, 6))
  Xc[4000:4050] = Xc[10]                          # 50 copies of one candidate: the covariance is singular
  Ut = rs.standard_normal((2, 4500))
  _, power = B.gp_core.joint_draw_on_device(gp._post, Xc, Ut, 0.1)
  ogp = B.O.OGP(gp.X, gp.Y, B.O.OMaternKernel(6, 2.5, 1.3, [0.4] * 6), lambda x: np.array([0.1] * len(x)), 1e-3 * 1.3)
  _, cov = ogp.eval(Xc, 'covar')
  _, power_o = B.O.stable_cholesky(cov)
  print('jitter power device %s oracle %s' % (power, power_o))
  assert power_o is not None and power == power_o


# ---- 6. above the cap ----------------------------------------------------------------------------------------------------
def test_above_the_cap_stays_in_blocks(B):
  gp, rs = matern_gp(B, 500, seed=14)
  Xc = rs.random_sample((16385, 6))
  np.random.seed(21)
  S = gp.draw_samples(2, Xc)
  np.random.seed(21)
  U = np.random.normal(size=(16385, 2))
  for lo, hi in [(0, 4096), (12288, 16384), (16384, 16385)]:
    info, smp, _ = gp._post.ts_draws(Xc[lo:hi], np.ascontiguousarray(U[lo:hi].T), mean_const=gp._mean_const)
    assert info == 0
    assert_same(S[:, lo:hi], smp.cpu().numpy(), 'block [%d, %d)' % (lo, hi))


# ---- 7. MF and ExpDecay ----------------------------------------------------------------------------------------------------
def test_mf_posterior_joint_draw(B):
  """ An MF [z || x] posterior: the joint draw over 7000 candidates, whose leading block is the block draw. """
  rs = np.random.RandomState(17)
  n = 300
  Z, X = rs.random_sample((n, 1)), rs.random_sample((n, 4))
  Y = np.sin(3 * X).sum(axis=1) * (1 - 0.2 * Z[:, 0])
  kF = B.kernel.SEKernel(1, 1.0, [0.7]); kD = B.kernel.MaternKernel(4, 2.5, 1.0, [0.4] * 4)
  mfgp = B.mf_gp.EuclideanMFGP(list(Z), list(X), list(Y), None, 1.1, kF, kD, B.gp_core.ConstantMean(0.2), 1e-3)
  ZX = mfgp.get_ZX_matrix(list(rs.random_sample((7000, 1))), list(rs.random_sample((7000, 4))))
  np.random.seed(31)
  S = mfgp.draw_samples(3, ZX)
  np.random.seed(31)
  U = np.random.normal(size=(7000, 3))
  Xm = np.asarray(mfgp._test_matrix(ZX))
  info, smp, _ = mfgp._post.ts_draws(Xm[:4096], np.ascontiguousarray(U[:4096].T), mean_const=0.2)
  assert info == 0
  assert S.shape == (3, 7000) and np.isfinite(S).all()
  assert_same(S[:, :4096], smp.cpu().numpy(), 'MF leading block')


def test_expdecay_kernel_joint_draw(B):
  """ A non-stationary (ExpDecay) kernel over 6000 candidates: joint covariance tiles equal the block covariance of
      the same candidates bit for bit; the kernel is smooth enough that the covariance needs stable_cholesky's
      ladder, and the draw is mu + L U with the factor the device left. """
  rs = np.random.RandomState(19)
  n = 250
  X = rs.random_sample((n, 2))
  Y = np.cos(2 * X).sum(axis=1)
  gp = B.gp_core.GP(X, Y, B.kernel.ExpDecayKernel(2, 1.0, 0.1, [1.0, 2.0]), B.gp_core.ConstantMean(0.0), 1e-3)
  post = gp._post
  M = 6000
  Xc = rs.random_sample((M, 2))
  mu, _ = post.eval_covar(Xc)
  sig = joint_cov(B, post, M)
  rows = _tile_rows(M, [0, 20, 46])
  _, cov_s = post.eval_covar(Xc[rows])
  assert_same(sig[np.ix_(rows, rows)], cov_s, 'ExpDecay joint tiles vs block covariance')
  Ut = rs.standard_normal((2, M))
  smp, power = B.gp_core.joint_draw_on_device(post, Xc, Ut, 0.0)
  print('ExpDecay jitter power', power)
  Lq = np.tril(joint_cov(B, post, M))
  L = Lq[:M, :M]
  ref = mu[None, :] + Ut @ L.T
  assert smp.shape == (2, M) and np.isfinite(smp).all()
  assert np.abs(smp - ref).max() <= 1e-11 * (1 + np.abs(L).sum(axis=1).max())
  # the factor itself, at the jitter the ladder reached (its scale is max diag Sigma, as on the device)
  j = 0.0 if power is None else (10 ** power) * float(np.diag(sig)[:M].max())
  q = Lq.shape[0]
  r = factor_rows_ratio(Lq, padded_input(sig, M, j), np.r_[0:T, q - T:q])
  print('RATIO ExpDecay factor (build bound) %.3g' % r)
  assert r <= 1.0
