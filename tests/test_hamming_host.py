"""
Categorical parts on the host (no GPU): the category encoding of HammingKernel, its lowering to the HAMMING factor of
the descriptor (include/dfb200.h), the parity-mode draw of Cartesian-product candidates against the reference's
sample_from_cp_domain (golden hamming.npz, 3), and the Hamming oracle (tests/hamming_ref.py) against the reference's
Gram blocks and CPGP (goldens 1-2).
"""
import json

import numpy as np
import pytest

from conftest import load_golden
from oracle import gp_oracle as O
import hamming_ref as R

from dragonfly_b200 import _lib, domains
from dragonfly_b200 import kernel as K
from dragonfly_b200 import cartesian_product_gp as cp
from dragonfly_b200 import gpb_acquisitions as acq


# ---- encoding ---------------------------------------------------------------------------------------------------
def test_codes_follow_python_equality():
  t = K.CategoryCodes()
  assert [t.encode(v) for v in ['a', 'b', 'a', np.str_('b'), 1, 1.0, True, np.int64(1), '1', 2]] == \
         [0, 1, 0, 1, 2, 2, 2, 2, 3, 4]
  assert t.encode('a') == 0                                 # the table only grows


def test_nan_and_unhashable_categories_are_refused():
  t = K.CategoryCodes()
  for bad in (float('nan'), np.float64('nan'), np.nan):
    with pytest.raises(ValueError):
      t.encode(bad)
  with pytest.raises(ValueError):
    t.encode(['a'])
  assert t.codes == {}


def test_drawn_value_is_encoded_after_numpy_promotion():
  """ np.array([1, 'x'])[k] is np.str_('1'), not 1: the drawn value is what gets a code """
  kern = K.HammingKernel([1.0])
  dom = domains.CartesianProductDomain([domains.ProdDiscreteDomain([[1, 'x']])])
  wrapper = cp.CartesianProductKernel(1.0, [kern])
  parts = acq._cp_parts(dom, wrapper)
  np.random.seed(3)
  rows, draws = acq.draw_cp_candidates(parts, 40)
  pts = [acq.point_from_draws(parts, draws, i) for i in range(40)]
  assert {type(p[0][0]) for p in pts} == {np.str_}
  assert set(kern.category_codes.codes) == {'1', 'x'}
  assert 1 not in kern.category_codes.codes
  one = kern.category_codes.encode('1')
  assert all((r[0] == one) == (p[0][0] == '1') for r, p in zip(rows, pts))


def test_flatten_parts_codes_categorical_parts_and_keeps_euclidean_rows():
  kern = cp.CartesianProductKernel(1.0, [K.SEKernel(2, 1.0, [1.0, 1.0]), K.HammingKernel(2)])
  X = [[np.array([0.5, 0.25]), ['u', 7]], [np.array([1.0, 2.0]), ['v', 7]], [np.array([0.0, 0.0]), ['u', 'w']]]
  M = cp.flatten_parts(X, kern)
  # one table per Hamming factor, shared by its coordinates: u -> 0, 7 -> 1, v -> 2, w -> 3
  np.testing.assert_array_equal(M, [[0.5, 0.25, 0, 1], [1.0, 2.0, 2, 1], [0.0, 0.0, 0, 3]])
  assert cp.flatten_parts(X[1:2], kern)[0, 2] == 2          # one table for every call
  Xe = [[np.array([0.5, 0.25]), [3.0]], [np.array([1.0, 2.0]), [4.0]]]
  np.testing.assert_array_equal(cp.flatten_parts(Xe), [[0.5, 0.25, 3.0], [1.0, 2.0, 4.0]])


# ---- descriptor -------------------------------------------------------------------------------------------------
def test_hamming_kernel_weights():
  np.testing.assert_array_equal(K.HammingKernel(4).hyperparams['dim_weights'], np.ones(4) / 4.0)
  assert K.HammingKernel([0.1, 0.2, 0.7]).dim == 3


def test_descriptor_lowering():
  kern = R.make_kernel(K, cp, 1.3)
  d = K.build_descriptor(kern, train_dim=7, cand_dim=7)
  assert (d.n_terms, d.n_factors, d.n_slots) == (1, 4, 7)
  kinds = [d.factors[f].kind for f in range(4)]
  assert kinds == [_lib.DFB_BASE_SE, _lib.DFB_BASE_MATERN, _lib.DFB_BASE_HAMMING, _lib.DFB_BASE_MATERN]
  h = d.factors[2]
  assert (h.p, h.n_dims, h.slot_off, h.scale) == (0, 3, 3, 1.0)
  assert [d.slot_bandwidth[s] for s in range(3, 6)] == [0.5, 0.2, 0.3]
  assert [d.slot_train_coord[s] for s in range(3, 6)] == [3, 4, 5]
  assert K.is_stationary(d)
  # kss = ((scale k_0) k_1) k_2 ... with k(x, x) of each factor: SE scale, Matern scale * norm, Hamming sum(w)
  assert d.term_pre_scale[0] == 1.3
  assert d.kss == ((((1.3 * d.factors[0].scale) * K._base_at_zero(_f(d, 1))) * ((0.5 + 0.2) + 0.3)) *
                   K._base_at_zero(_f(d, 3)))


def _f(d, i):
  fd = d.factors[i]
  f = K._Factor()
  f.kind, f.p, f.scale, f.coeffs, f.gamma_ratio = fd.kind, fd.p, fd.scale, list(fd.coeffs), fd.gamma_ratio
  return f


def test_hamming_kss_uses_numpy_pairwise_order():
  w = np.array([0.1, 0.2, 0.3, 0.05, 0.15, 0.12, 0.08, 0.33, 0.17])
  d = K.build_descriptor(K.HammingKernel(w))
  assert d.kss == float(np.add.reduce(w))
  r = [w[q] for q in range(8)]
  r[0] += w[8] * 0                                          # 9 terms: eight accumulators, then the tail
  pair = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
  assert d.kss == pair + w[8]


def test_weights_that_check_desc_refuses():
  """ check_desc (api.cu): HAMMING weights finite and >= 0; the host passes them through unchanged """
  d = K.build_descriptor(K.HammingKernel([0.5, 0.0]))
  assert [d.slot_bandwidth[s] for s in range(2)] == [0.5, 0.0]
  for bad in ([0.5, -0.1], [np.inf, 0.1], [np.nan, 0.1]):
    d = K.build_descriptor(K.HammingKernel(bad))
    w = [d.slot_bandwidth[s] for s in range(2)]
    assert not all(np.isfinite(v) and v >= 0 for v in w)


def test_hamming_is_not_an_esp_child():
  with pytest.raises(NotImplementedError):
    K.build_descriptor(K.ESPKernel(1.0, 1, [K.HammingKernel(1)]))


# ---- parity-mode draw (golden 3) --------------------------------------------------------------------------------
def test_parity_draw_matches_sample_from_cp_domain():
  g = load_golden('hamming')
  levels, numeric_levels, scale, _, _ = R.golden_problem(g)
  dom = R.make_domain(domains, levels, numeric_levels)
  kern = R.make_kernel(K, cp, scale)
  parts = acq._cp_parts(dom, kern)
  np.random.seed(21)
  rows, draws = acq.draw_cp_candidates(parts, 50)
  st = np.random.get_state()
  np.testing.assert_array_equal(st[1], g['S_state'])
  assert st[2] == int(g['S_pos'])
  want = json.loads(str(g['S']))
  got = [R.jencode(acq.point_from_draws(parts, draws, i)) for i in range(50)]
  assert got == want
  # the candidate rows are the points' columns, categories coded by the Hamming factor's table
  codes = kern.kernel_list[2].category_codes
  for i in (0, 17, 49):
    pt = acq.point_from_draws(parts, draws, i)
    np.testing.assert_array_equal(rows[i], list(pt[0]) + [float(pt[1][0])] + [codes.encode(v) for v in pt[2]] +
                                  [float(pt[3][0])])


def test_reference_domain_objects_by_duck_typing():
  """ a domain object with the reference's attribute names works (here: a stand-in with get_type / bounds) """
  class Dom(object):
    def __init__(self, t, **kw):
      self.t = t
      self.__dict__.update(kw)
    def get_type(self):
      return self.t
    def get_dim(self):
      return len(getattr(self, 'bounds', getattr(self, 'list_of_list_of_items', [])))
  dom = Dom('cartesian_product', list_of_domains=[Dom('euclidean', bounds=np.array([[0, 1]])),
                                                  Dom('prod_discrete', list_of_list_of_items=[['a', 'b']])])
  parts = acq._cp_parts(dom, cp.CartesianProductKernel(1.0, [K.SEKernel(1, 1.0, [1.0]), K.HammingKernel(1)]))
  assert [p.type for p in parts] == ['euclidean', 'prod_discrete']


def test_refusals():
  kern = cp.CartesianProductKernel(1.0, [K.SEKernel(1, 1.0, [1.0])])
  class Constrained(domains.CartesianProductDomain):
    def has_constraints(self):
      return True
  with pytest.raises(NotImplementedError):
    acq._cp_parts(Constrained([domains.EuclideanDomain([[0, 1]])]), kern)
  with pytest.raises(NotImplementedError):    # a prod_discrete part under SE
    acq._cp_parts(domains.CartesianProductDomain([domains.ProdDiscreteDomain([['a', 'b']])]), kern)


# ---- the oracle against the reference (goldens 1-2) ------------------------------------------------------------
def test_oracle_hamming_blocks_bit_for_bit():
  g = load_golden('hamming')
  for ci, m in enumerate(json.loads(str(g['hk_meta']))):
    codes = {}
    enc = lambda X: np.array([[codes.setdefault(R.jvalue(v), len(codes)) for v in r] for r in X], dtype=np.float64)
    X1, X2 = enc(m['X1']), enc(m['X2'])
    k = R.OHammingKernel(m['dim'] if m['weights'] is None else m['weights'])
    np.testing.assert_array_equal(k(X1, X2), g['hk%d_K' % ci])
    np.testing.assert_array_equal(k(X1, X1), g['hk%d_Kss' % ci])


def test_oracle_cpgp_against_the_reference():
  g = load_golden('hamming')
  _, _, scale, noise_var, mean_const = R.golden_problem(g)
  codes = {}
  X = R.encode_points(R.golden_points(g, 'X'), codes)
  C = R.encode_points(R.golden_points(g, 'C'), codes)
  H = R.encode_points(R.golden_points(g, 'H'), codes)
  gp = O.OGP(X, g['Y'], R.oracle_kernel(scale), lambda x: np.array([mean_const] * len(x)), noise_var)
  np.testing.assert_allclose(gp.K_trtr_wo_noise[:16], g['K'], rtol=0, atol=1e-13)
  np.testing.assert_allclose(gp.L[:16], g['L'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(gp.alpha, g['alpha'], rtol=1e-9, atol=1e-9)
  assert abs(gp.compute_log_marginal_likelihood() - float(g['lml'])) <= 1e-9 * abs(float(g['lml']))
  mu, sd = gp.eval(C, 'std')
  assert np.max(np.abs(mu - g['mu'])) <= 1e-10
  assert np.max(np.abs(sd ** 2 - g['sd'] ** 2)) <= 1e-8
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:100], H, 'std')
  assert np.max(np.abs(mu_h - g['mu_h'])) <= 1e-10
  assert np.max(np.abs(sd_h ** 2 - g['sd_h'] ** 2)) <= 1e-8
