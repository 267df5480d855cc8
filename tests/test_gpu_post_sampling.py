"""
dfb_lml_batch and the device post_sampling fit (-m gpu): the batch kernel against the NumPy oracle's LML and bit for
bit against dfb_build_posterior(DFB_BUILD_LML_ONLY); its independence of batch size and position; non-positive-definite
items; hp_grid.lml_batch_for_hyperparams on both sides of LML_BATCH_MAX_N; and post_sampling.post_sample_hps on the
device against the reference's own fits (golden post_sampling.npz).
"""
import numpy as np
import pytest

from conftest import load_golden
import post_sampling_ref as R

pytestmark = pytest.mark.gpu

NS = [1, 2, 63, 127, 128, 129, 255, 256, 257, 511, 512]


@pytest.fixture(scope='module')
def mods():
  import torch
  assert torch.cuda.is_available()
  from dragonfly_b200 import hp_grid, device, kernel, _lib
  from dragonfly_b200.gp_core import stable_cholesky_on_device
  return hp_grid, device, kernel, _lib, stable_cholesky_on_device


def _kernels(K, d, rs):
  """ SE, Matern 1/2, 3/2, 5/2 on d coordinates and the MF product (fidelity SE on coordinate 0, domain Matern). """
  def bws(k):
    return list(0.2 + rs.random_sample(k))
  out = [K.SEKernel(d, 0.5 + rs.random_sample(), bws(d))]
  out += [K.MaternKernel(d, nu, 0.5 + rs.random_sample(), bws(d)) for nu in (0.5, 1.5, 2.5)]
  if d >= 2:
    out.append(K.CoordinateProductKernel(d, 0.5 + rs.random_sample(),
                                         [K.SEKernel(1, 1.0, bws(1)), K.MaternKernel(d - 1, 2.5, 1.0, bws(d - 1))],
                                         [[0], list(range(1, d))]))
  return out


def _data(n, d, seed):
  rs = np.random.RandomState(seed)
  X = rs.random_sample((n, d))
  return X, np.sin(3 * X[:, 0]) + X.sum(1) + 0.1 * rs.randn(n), rs


def _items(K, d, rs, B):
  kerns = _kernels(K, d, rs)
  kern = [kerns[i % len(kerns)] for i in range(B)]
  return kern, list(1e-3 + 0.05 * rs.random_sample(B)), list(rs.randn(B))


def _build_lml(post, desc_of, X, Y, kern, noise, mean, _lib):
  post.set_train(X, Y - mean)
  post.set_kernel(desc_of(kern))
  return post.build(noise, 0.0, _lib.DFB_BUILD_LML_ONLY)


@pytest.mark.parametrize('n', NS)
def test_lml_batch_against_oracle_and_build_posterior(mods, n):
  hp_grid, device, K, _lib, _ = mods
  d = 3
  X, Y, rs = _data(n, d, n)
  desc_of = lambda k: K.build_descriptor(k, train_dim=d, cand_dim=d)
  kern, noise, mean = _items(K, d, rs, 7)
  post = device.DevicePosterior(n)
  post.set_train(X, Y)
  lmls, infos = post.lml_batch([desc_of(k) for k in kern], noise, mean)
  assert (infos == 0).all()
  single = device.DevicePosterior(n)
  for i in range(len(kern)):
    ref = R.O.OGP(X, Y, R.oracle_kernel(kern[i]), lambda x, c=mean[i]: np.array([c] * len(x)), noise[i])
    np.testing.assert_allclose(lmls[i], ref.compute_log_marginal_likelihood(), rtol=1e-10, atol=0)
    info, lml = _build_lml(single, desc_of, X, Y, kern[i], noise[i], mean[i], _lib)
    assert info == 0 and lmls[i] == lml          # the same arithmetic as the LML-only build: bit for bit


@pytest.mark.parametrize('B', [1, 64, 300])
def test_lml_batch_sizes_and_positions(mods, B):
  hp_grid, device, K, _lib, _ = mods
  d, n = 4, 257
  X, Y, rs = _data(n, d, B)
  desc_of = lambda k: K.build_descriptor(k, train_dim=d, cand_dim=d)
  kern, noise, mean = _items(K, d, rs, B)
  descs = [desc_of(k) for k in kern]
  post = device.DevicePosterior(n, chunk=2048 if B == 300 else 0)   # 300 items exceed a 2048-row chunk buffer
  post.set_train(X, Y)
  lmls, infos = post.lml_batch(descs, noise, mean)
  assert (infos == 0).all()
  single = device.DevicePosterior(n)
  for i in sorted(set([0, B - 1, B // 2, min(5, B - 1)])):
    ref = R.O.OGP(X, Y, R.oracle_kernel(kern[i]), lambda x, c=mean[i]: np.array([c] * len(x)), noise[i])
    np.testing.assert_allclose(lmls[i], ref.compute_log_marginal_likelihood(), rtol=1e-10, atol=0)
    assert lmls[i] == _build_lml(single, desc_of, X, Y, kern[i], noise[i], mean[i], _lib)[1]
  # an item's value does not depend on its position or on the rest of the batch
  post.set_train(X, Y)
  alone, _ = post.lml_batch(descs[-1:], noise[-1:], mean[-1:])
  assert alone[0] == lmls[-1]
  rev, _ = post.lml_batch(descs[::-1][:7], noise[::-1][:7], mean[::-1][:7])
  np.testing.assert_array_equal(rev, lmls[::-1][:7])


def test_not_positive_definite_items(mods):
  hp_grid, device, K, _lib, stable_cholesky_on_device = mods
  d, n = 2, 150
  rs = np.random.RandomState(7)
  base = rs.random_sample((60, d))
  X = base[rs.randint(0, 60, n)]                 # duplicated rows: K is singular without noise
  Y = X.sum(1) + 0.1 * rs.randn(n)
  layout = hp_grid.EuclideanHPLayout(d, 'se', mean_func_type='tune', noise_var_type='value', noise_var_value=0.0)
  hps = np.array([[rs.randn(), np.log(1 + rs.random_sample()), np.log(0.5 + rs.random_sample()),
                   np.log(0.5 + rs.random_sample())] for _ in range(6)])
  descs, means = [], []
  for hp in hps:
    mean_const, _, kern = layout.unpack(hp, Y)
    descs.append(K.build_descriptor(kern, train_dim=d, cand_dim=d))
    means.append(mean_const)
  post = device.DevicePosterior(n)
  post.set_train(X, Y)
  _, infos = post.lml_batch(descs, [0.0] * 6, means)
  assert (infos != 0).any()
  single = device.DevicePosterior(n)
  for i in range(6):
    single.set_train(X, Y - means[i])
    single.set_kernel(descs[i])
    assert infos[i] == single.build(0.0, 0.0, _lib.DFB_BUILD_LML_ONLY)[0]
  vals, _ = hp_grid.lml_batch_for_hyperparams(X, Y, hps, layout)
  for i in range(6):
    single.set_train(X, Y - means[i])
    single.set_kernel(descs[i])
    want, _ = stable_cholesky_on_device(single, 0.0, flags=_lib.DFB_BUILD_LML_ONLY)
    assert vals[i] == want


def test_above_the_cap_the_wrapper_is_lml_for_hyperparams(mods):
  hp_grid, _, _, _, _ = mods
  n, d = hp_grid.LML_BATCH_MAX_N + 88, 3
  X, Y, rs = _data(n, d, 11)
  layout = hp_grid.EuclideanHPLayout(d, 'matern', nu=-1.0, mean_func_type='tune', noise_var_type='tune')
  bounds, _ = layout.bounds(X, Y, tune_nu=True)
  hps = bounds[:, 0] + (bounds[:, 1] - bounds[:, 0]) * rs.random_sample((9, len(bounds)))
  nus = [0.5, 1.5, 2.5] * 3
  a, _ = hp_grid.lml_batch_for_hyperparams(X, Y, hps, layout, nus=nus)
  b, _ = hp_grid.lml_for_hyperparams(X, Y, hps, layout, nus=nus)
  np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize('tag', R.CONFIGS)
def test_device_sampler_reproduces_the_reference(mods, tag):
  from dragonfly_b200 import post_sampling
  from dragonfly_b200.gp_core import GP, ConstantMean
  g = load_golden('post_sampling')
  X, Y, layout, bounds, dscr_vals, kw = R.config(g, tag)

  def build(cts, dscr):
    mean_const, noise_var, kern = layout.unpack(cts, Y, dscr[0] if len(dscr) else None)
    return GP(list(X), list(Y), kern, ConstantMean(mean_const), noise_var)
  stats = post_sampling.PostSamplingStats()
  np.random.seed(int(g[tag + '_seed']))
  res = post_sampling.post_sample_hps(X, Y, layout, bounds, dscr_vals, build_gp=build, stats=stats, **kw)
  fingerprint = np.array([np.random.random() for _ in range(4)])
  np.testing.assert_array_equal(fingerprint, g[tag + '_fingerprint'])
  assert res[0] == str(g[tag + '_kind'])
  cts, dscr = res[2] if res[0] == 'post_fitted_gp' else res[1:3]
  np.testing.assert_array_equal(cts, g[tag + '_cts'])
  np.testing.assert_array_equal(dscr, g[tag + '_dscr'])
  assert stats.consumed == len(g[tag + '_trace_lml'])
  if res[0] == 'post_fitted_gp':
    np.testing.assert_allclose(res[1].compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-10)
