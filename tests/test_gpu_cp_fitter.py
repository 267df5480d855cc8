"""
dfb_lml_batch_mixed and the device fits of Cartesian-product GPs (-m gpu): the batch kernel with HAMMING factors bit for
bit against dfb_build_posterior(DFB_BUILD_LML_ONLY) and against the NumPy oracle, its independence of batch size and
position, non-positive-definite items, hp_grid.lml_batch_for_hyperparams on both sides of LML_BATCH_MAX_N, and
hp_grid.fit_gp / post_sampling.post_sample_hps on the device against the reference's CPGPFitter (golden cp_fitter.npz).
"""
import numpy as np
import pytest

from conftest import load_golden
import cp_fitter_ref as R

pytestmark = pytest.mark.gpu

NS = [1, 127, 128, 129, 255, 256, 384, 511, 512]


@pytest.fixture(scope='module')
def mods():
  import torch
  assert torch.cuda.is_available()
  from dragonfly_b200 import hp_grid, device, kernel, cartesian_product_gp, _lib
  from dragonfly_b200.gp_core import stable_cholesky_on_device
  return hp_grid, device, kernel, cartesian_product_gp, _lib, stable_cholesky_on_device


HAMMING_DIMS = (1, 2, 3, 9)
D = 2 + 1 + sum(HAMMING_DIMS)           # [e0, e1 | i | codes of the four Hamming parts]


def _data(n, seed):
  """ rows [e0, e1, i, categorical codes ...]: 2-4 levels per categorical coordinate """
  rs = np.random.RandomState(seed)
  E = rs.random_sample((n, 2))
  I = rs.randint(0, 6, size=(n, 1)).astype(np.float64)
  C = np.concatenate([rs.randint(0, 2 + q % 3, size=(n, 1)) for q in range(sum(HAMMING_DIMS))], axis=1)
  X = np.ascontiguousarray(np.concatenate((E, I, C.astype(np.float64)), axis=1))
  Y = np.sin(3 * E[:, 0]) + 0.2 * I[:, 0] + 0.3 * (C[:, 0] == 1) - 0.2 * C[:, 5] + 0.05 * rs.randn(n)
  return X, Y, rs


def _weights(k, rs):
  w = 0.1 + rs.random_sample(k)
  return list(w / w.sum())


def _kernels(K, CP, rs):
  """ CP kernels over [Euclidean(2) | Integral(1) | Hamming parts ...] with different Hamming dims, plus Euclidean-only
      coordinate products on the same rows (no HAMMING factor). """
  out = []
  for ham in ((1,), (2,), (3,), (9,), (1, 2, 3, 9)):
    kids = [K.SEKernel(2, 1.0, list(0.3 + rs.random_sample(2))), K.MaternKernel(1, 2.5, 1.0, [1.0 + rs.random_sample()])]
    coords = [[0, 1], [2]]
    off = 3
    for h in HAMMING_DIMS:
      if h in ham:
        kids.append(K.HammingKernel(_weights(h, rs)))
        coords.append(list(range(off, off + h)))
      off += h
    out.append(K.CoordinateProductKernel(D, 0.5 + rs.random_sample(), kids, coords))
  out.append(K.CoordinateProductKernel(D, 0.7, [K.MaternKernel(2, 1.5, 1.0, [0.4, 0.6]),
                                                K.SEKernel(1, 1.0, [2.0])], [[0, 1], [2]]))
  return out


def _oracle(kern):
  from oracle import gp_oracle as O
  import hamming_ref as H
  kids = []
  for k in kern.kernel_list:
    hp = k.hyperparams
    if 'dim_weights' in hp:
      kids.append(H.OHammingKernel(hp['dim_weights']))
    elif 'nu' in hp:
      kids.append(O.OMaternKernel(k.dim, hp['nu'], hp['scale'], hp['dim_bandwidths']))
    else:
      kids.append(O.OSEKernel(k.dim, hp['scale'], hp['dim_bandwidths']))
  return O.OCoordinateProductKernel(D, kern.hyperparams['scale'], kids, kern.coordinate_list)


def _single(post, K, X, Y, kern, noise, mean, _lib):
  post.set_train(X, Y - mean)
  post.set_kernel(K.build_descriptor(kern, train_dim=D, cand_dim=D))
  return post.build(noise, 0.0, _lib.DFB_BUILD_LML_ONLY)


@pytest.mark.parametrize('n', NS)
def test_lml_batch_mixed_bit_for_bit_and_against_oracle(mods, n):
  hp_grid, device, K, CP, _lib, _ = mods
  from oracle import gp_oracle as O
  X, Y, rs = _data(n, n)
  kern = _kernels(K, CP, rs)
  noise = list(1e-3 + 0.05 * rs.random_sample(len(kern)))
  mean = list(0.3 * rs.randn(len(kern)))
  post = device.DevicePosterior(n)
  post.set_train(X, Y)
  lmls, infos = post.lml_batch([K.build_descriptor(k, train_dim=D, cand_dim=D) for k in kern], noise, mean, mixed=True)
  assert (infos == 0).all()
  single = device.DevicePosterior(n)
  for i, k in enumerate(kern):
    info, lml = _single(single, K, X, Y, k, noise[i], mean[i], _lib)
    assert info == 0 and lmls[i] == lml                       # the LML-only build's arithmetic: bit for bit
    ref = O.OGP(X, Y, _oracle(k), lambda x, c=mean[i]: np.array([c] * len(x)), noise[i])
    np.testing.assert_allclose(lmls[i], ref.compute_log_marginal_likelihood(), rtol=1e-10, atol=0)


@pytest.mark.parametrize('B', [1, 7, 300])
def test_lml_batch_mixed_sizes_and_positions(mods, B):
  hp_grid, device, K, CP, _lib, _ = mods
  n = 200
  X, Y, rs = _data(n, 5)
  kinds = _kernels(K, CP, rs)
  kern = [kinds[(3 * i + 1) % len(kinds)] for i in range(B)]
  noise = [0.01 + 0.001 * (i % 5) for i in range(B)]
  mean = [0.1 * (i % 3) for i in range(B)]
  post = device.DevicePosterior(n)
  post.set_train(X, Y)
  descs = [K.build_descriptor(k, train_dim=D, cand_dim=D) for k in kern]
  lmls, infos = post.lml_batch(descs, noise, mean, mixed=True)
  assert (infos == 0).all()
  for i in sorted(set([0, B - 1, B // 2])):                    # alone, and in reverse order
    one, _ = post.lml_batch([descs[i]], [noise[i]], [mean[i]], mixed=True)
    assert one[0] == lmls[i]
  rev, _ = post.lml_batch(descs[::-1], noise[::-1], mean[::-1], mixed=True)
  np.testing.assert_array_equal(rev[::-1], lmls)


def test_non_pd_item_and_its_rebuild(mods):
  hp_grid, device, K, CP, _lib, stable = mods
  # one Hamming part of 3 levels on 40 points and no noise: K has rank 3
  lay = hp_grid.CartesianProductHPLayout([('prod_discrete', 1, 'hamming'), ('euclidean', 1, 'se')],
                                         mean_func_type='const', noise_var_type='value', noise_var_value=0.0)
  rs = np.random.RandomState(2)
  pts = [[[['a', 'b', 'c'][i % 3]], np.array([0.5])] for i in range(40)]
  Y = rs.randn(40)
  X = lay.encode(pts)
  hps = np.array([[0.0, 0.0], [0.5, -1.0]])
  _, _, kern = lay.unpack(hps[0], Y)
  post = device.DevicePosterior(40)
  post.set_train(X, Y)
  lmls, infos = post.lml_batch([K.build_descriptor(kern, train_dim=2, cand_dim=2)], [0.0], [0.0], mixed=True)
  info_single, _ = _single_flat(post, K, X, Y, kern, _lib)
  assert infos[0] > 0 and np.isnan(lmls[0]) and infos[0] == info_single
  vals, _ = hp_grid.lml_batch_for_hyperparams(X, Y, hps, lay)
  ref, _ = hp_grid.lml_for_hyperparams(X, Y, hps, lay, lanes=1)
  assert np.isfinite(vals).all()
  np.testing.assert_array_equal(vals, ref)                      # the jitter ladder of stable_cholesky_on_device


def _single_flat(post, K, X, Y, kern, _lib):
  post.set_train(X, Y)
  post.set_kernel(K.build_descriptor(kern, train_dim=X.shape[1], cand_dim=X.shape[1]))
  return post.build(0.0, 0.0, _lib.DFB_BUILD_LML_ONLY)


def test_lane_path_above_the_batch_cap(mods):
  hp_grid, device, K, CP, _lib, _ = mods
  g = load_golden('cp_fitter')
  lay = R.layout('M')
  rs = np.random.RandomState(4)
  base = R.points(g, 'M')
  pts = [base[i % len(base)] for i in range(600)]
  pts = [[p[0] + 0.01 * rs.randn(2), p[1], p[2], p[3]] for p in pts]
  Y = np.array([np.sin(3 * p[0][0]) + 0.1 * p[1][0] for p in pts]) + 0.05 * rs.randn(600)
  X = lay.encode(pts)
  b = lay.bounds(pts, Y)[0]
  hps = b[:, 0] + rs.random_sample((6, len(b))) * (b[:, 1] - b[:, 0])
  assert len(X) > hp_grid.LML_BATCH_MAX_N
  vals, _ = hp_grid.lml_batch_for_hyperparams(X, Y, hps, lay)
  for h, v in zip(hps, vals):
    np.testing.assert_allclose(v, R.oracle_lml(X, Y, lay, h, ()), rtol=1e-10, atol=0)


@pytest.mark.parametrize('method', R.ML_METHODS)
@pytest.mark.parametrize('tag', R.CONFIGS)
def test_device_ml_fits_match_the_reference(mods, tag, method):
  hp_grid = mods[0]
  g = load_golden('cp_fitter')
  key = '%s_%s_' % (tag, method)
  lay = R.layout(tag)
  np.random.seed(int(g[key + 'seed']))
  res = hp_grid.fit_gp(R.points(g, tag), g[tag + '_Y'], lay, g[tag + '_bounds'], R.dscr_vals(g, tag), method=method,
                       max_evals=int(g[key + 'max_evals']))
  fingerprint = np.array([np.random.random() for _ in range(4)])
  assert res[0] == str(g[key + 'kind'])
  if res[0] == 'fitted_gp':
    _, gp, (cts, dscr) = res
    np.testing.assert_array_equal(cts, g[key + 'cts'])
    np.testing.assert_array_equal(np.array(dscr, dtype=np.float64), g[key + 'dscr'])
    np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[key + 'lml']), rtol=1e-10, atol=0)
  else:
    _, cts, dscr, _, probs = res
    np.testing.assert_array_equal(cts, g[key + 'cts'])
    np.testing.assert_allclose(probs, g[key + 'probs'], rtol=1e-10, atol=1e-300)
  np.testing.assert_array_equal(fingerprint, g[key + 'fingerprint'])


def test_device_post_sampling_matches_the_reference(mods):
  from dragonfly_b200 import post_sampling
  g = load_golden('cp_fitter')
  lay = R.layout('M')
  trace = []
  np.random.seed(int(g['PM_seed']))
  res = post_sampling.post_sample_hps(R.points(g, 'M'), g['PM_Y'], lay, g['PM_bounds'], R.dscr_vals(g, 'PM'),
                                      num_samples=int(g['PM_num_samples']), offset=int(g['PM_offset']),
                                      burn=int(g['PM_burn']), build_gp=lambda c, d: None, trace=trace)
  fingerprint = np.array([np.random.random() for _ in range(4)])
  assert res[0] == str(g['PM_kind'])
  np.testing.assert_array_equal(res[1], g['PM_cts'])
  np.testing.assert_array_equal(fingerprint, g['PM_fingerprint'])
  np.testing.assert_array_equal(np.array([h for h, _ in trace]), g['PM_trace_cts'])
  np.testing.assert_allclose([v for _, v in trace], g['PM_trace_lml'], rtol=1e-10, atol=0)
