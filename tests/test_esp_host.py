"""
ESP kernel on the host side (no GPU): the descriptor's ESP form (dfb_kernel_desc.esp_order, include/dfb200.h), its
validation, the kernel classes, and the forward-error bound of tests/esp_ref.py against the NumPy restatement of the
reference's recurrence.
"""
import math

import numpy as np
import pytest

from dragonfly_b200 import kernel as K, _lib, mf_gp
import esp_ref as E


def test_classes_mirror_the_reference():
  k = K.ESPKernelSE(3, 1.7, 2, [0.3, 0.4, 0.5])
  assert k.dim == 3 and k.hyperparams == {'scale': 1.7, 'order': 2} and k.is_guaranteed_psd()
  assert [c.hyperparams['dim_bandwidths'].tolist() for c in k.kernel_list] == [[0.3], [0.4], [0.5]]
  assert all(c.hyperparams['scale'] == 1.0 and c.dim == 1 for c in k.kernel_list)
  m = K.ESPKernelMatern(2, [0.5, 2.5], 1.0, 2, [0.3, 0.4])
  assert [c.hyperparams['nu'] for c in m.kernel_list] == [0.5, 2.5]
  for order in (0, 4):
    with pytest.raises(ValueError):
      K.ESPKernelSE(3, 1.0, order, [0.3, 0.4, 0.5])
  g = mf_gp.EuclideanGP._get_kernel_from_type('esp', dict(dim=2, scale=1.1, order=1, dim_bandwidths=[0.2, 0.3]))
  assert type(g).__name__ == 'ESPKernelSE' and g.hyperparams['order'] == 1


@pytest.mark.parametrize('kind', ['se', 'matern'])
def test_descriptor_fields(kind):
  bws = [0.3, 0.4, 0.5, 0.6]
  nus = [0.5, 1.5, 2.5, 1.5]
  k = K.ESPKernelSE(4, 1.7, 3, bws) if kind == 'se' else K.ESPKernelMatern(4, nus, 1.7, 3, bws)
  d = K.build_descriptor(k)
  assert (d.n_terms, d.n_factors, d.n_slots, d.esp_order) == (4, 4, 4, 3)
  assert d.post_scale == 1.7
  for t in range(4):
    assert d.term_first_factor[t] == t and d.term_pre_scale[t] == 1.0
    f = d.factors[t]
    assert (f.n_dims, f.slot_off) == (1, t)
    assert d.slot_train_coord[t] == t and d.slot_cand_coord[t] == t and d.slot_bandwidth[t] == bws[t]
    assert f.kind == (_lib.DFB_BASE_SE if kind == 'se' else _lib.DFB_BASE_MATERN)
    if kind == 'matern':
      assert f.p == int(nus[t])
  assert d.term_first_factor[4] == 4
  # every child is 1 at distance 0 (scale 1, Matern normalised), so k(x, x) = scale * C(4, 3)
  assert d.kss == pytest.approx(1.7 * math.comb(4, 3), rel=1e-15)
  # plain kernels keep esp_order = 0
  assert K.build_descriptor(K.SEKernel(2, 1.0, [0.3, 0.4])).esp_order == 0


def test_duck_typing_by_class_name():
  class ESPKernel(object):                   # a stand-in for the reference's own class
    def __init__(self):
      self.dim = 2
      self.kernel_list = [K.SEKernel(1, 1.0, [0.3]), K.MaternKernel(1, 1.5, 1.0, [0.4])]
      self.hyperparams = {'scale': 2.0, 'order': 2}

  d = K.build_descriptor(ESPKernel())
  assert (d.n_terms, d.esp_order, d.post_scale) == (2, 2, 2.0)
  assert d.factors[1].kind == _lib.DFB_BASE_MATERN


def test_nested_esp_is_refused():
  esp = K.ESPKernelSE(2, 1.0, 1, [0.3, 0.4])
  with pytest.raises(NotImplementedError):
    K.build_descriptor(K.AdditiveKernel(1.0, [esp, K.SEKernel(1, 1.0, [0.2])], [[0, 1], [2]]))
  with pytest.raises(NotImplementedError):
    K.build_descriptor(K.CoordinateProductKernel(3, 1.0, [K.SEKernel(1, 1.0, [0.2]), esp], [[0], [1, 2]]))
  with pytest.raises(NotImplementedError):       # children must be 1-D
    K.build_descriptor(K.ESPKernel(1.0, 1, [K.SEKernel(2, 1.0, [0.3, 0.4])]))


def test_descriptor_validation():
  base = lambda: K.build_descriptor(K.ESPKernelSE(3, 1.0, 2, [0.3, 0.4, 0.5]))
  K.check_esp_descriptor(base())
  for mutate in (lambda d: setattr(d, 'esp_order', 4),           # order > n_terms
                 lambda d: setattr(d, 'esp_order', -1),
                 lambda d: d.term_pre_scale.__setitem__(1, 2.0),   # pre_scale != 1
                 lambda d: setattr(d.factors[2], 'n_dims', 2)):    # a 2-slot factor
    d = base()
    mutate(d)
    with pytest.raises(ValueError):
      K.check_esp_descriptor(d)
  # a term of two factors
  d = K.build_descriptor(K.CoordinateProductKernel(2, 1.0, [K.SEKernel(1, 1.0, [0.2]), K.SEKernel(1, 1.0, [0.3])],
                                                   [[0], [1]]))
  d.esp_order = 1
  with pytest.raises(ValueError):
    K.check_esp_descriptor(d)


def test_host_recurrence_matches_the_oracle():
  rs = np.random.RandomState(0)
  v = [rs.random_sample((5, 7)) for _ in range(6)]
  for order in range(1, 7):
    assert np.array_equal(K.esp_combine(v, order), E.esp_in_reference_order(v, order))


G_NUS = (0.5, 1.5, 2.5)


def _golden_cases(g):
  for key in g.files:
    if key.startswith('K_'):
      _, kind, d, r = key.split('_')
      yield kind, int(d), int(r), key


def test_oracle_against_the_reference_kernel_blocks():
  """ The NumPy restatement against K blocks recorded from the unmodified reference (golden esp.npz): SE and Matern
      with per-dimension nu, d = 1, 2, 4, 8 at every order and d = 20. """
  from conftest import load_golden
  g = load_golden('esp')
  worst = 0.0
  for kind, d, r, key in _golden_cases(g):
    X1, X2 = g['X1_%d_%d' % (d, r)], g['X2_%d_%d' % (d, r)]
    bws = list(0.3 + 0.5 * np.random.RandomState(100 + d).random_sample(d)) if d < 20 else [2.0] * d
    nus = [G_NUS[t % 3] for t in range(d)] if kind == 'matern' else None
    ours = E.oracle_kernel(kind, 1.3, r, bws, nus)(X1, X2)
    b = E.esp_bound(kind, 1.3, r, bws, X1, X2, nus)
    assert np.all(np.abs(ours - g[key]) <= 2 * b), key
    worst = max(worst, float(np.max(np.abs(ours - g[key]) / b)))
  print('oracle vs reference K blocks: max |dK| / bound = %.3g' % worst)


def test_oracle_gp_against_the_reference_gp():
  from conftest import load_golden
  from oracle import gp_oracle as O
  g = load_golden('esp')
  d, r = int(g['gp_d']), int(g['gp_order'])
  ok = E.oracle_kernel('matern', float(g['gp_scale']), r, list(g['gp_bws']), [G_NUS[t % 3] for t in range(d)])
  mc = float(g['gp_mean'])
  ogp = O.OGP(g['gp_X'], g['gp_Y'], ok, lambda x: np.array([mc] * len(x)), float(g['gp_noise']))
  np.testing.assert_allclose(ogp.L[:16], g['L_rows'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(ogp.alpha, g['alpha'], rtol=1e-9, atol=1e-9)
  np.testing.assert_allclose(ogp.compute_log_marginal_likelihood(), float(g['lml']), rtol=1e-11)
  mu, var = O.eval_std_diag(ogp, g['gp_C'])
  np.testing.assert_allclose(mu, g['mu'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(var, g['sd'] ** 2, rtol=0, atol=1e-8)
  mu_h, var_h = O.eval_std_diag(ogp, g['gp_C'][:200], g['Xh'])
  np.testing.assert_allclose(mu_h, g['mu_h'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(var_h, g['sd_h'] ** 2, rtol=0, atol=1e-8)
  S = ogp.draw_samples_with_normals(g['gp_C'][:64], g['ts_U'])
  np.testing.assert_allclose(S, g['ts_samples'], rtol=0, atol=1e-9)


FITTER_CASES = [(kind, method) for kind in ('se', 'matern') for method in ('rand', 'rand_exp_sampling', 'pdoo')]


def _dscr_vals(g, tag):
  return [list(g[tag + '_dscr_vals_%d' % i]) for i in range(int(g[tag + '_n_dscr']))]


@pytest.mark.parametrize('kind,method', FITTER_CASES)
def test_fit_gp_selects_what_the_reference_esp_fitter_selects(kind, method, monkeypatch):
  """ hp_grid.fit_gp with an ESP layout, LMLs from the oracle: the same candidates, the same selected hps and the same
      probabilities as the reference's EuclideanGPFitter with kernel_type 'esp' (golden fitter_esp.npz). """
  from conftest import load_golden
  from oracle import gp_oracle as O
  from dragonfly_b200 import hp_grid
  g = load_golden('fitter_esp')
  tag = '%s_%s' % (kind, method)
  X, Y = g['X'], g['Y']
  layout = hp_grid.EuclideanHPLayout(3, 'esp', esp_kernel_type=kind, mean_func_type=str(g['mean_func_type']),
                                     noise_var_type=str(g['noise_var_type']))
  b, dv = layout.bounds(X, Y)
  assert (b == g[tag + '_bounds']).all() and dv == _dscr_vals(g, tag)

  def oracle_of(kern):
    nus = [c.hyperparams['nu'] for c in kern.kernel_list] if kind == 'matern' else None
    bws = [float(c.hyperparams['dim_bandwidths'][0]) for c in kern.kernel_list]
    return E.oracle_kernel(kind, kern.hyperparams['scale'], kern.hyperparams['order'], bws, nus)
  calls = []

  def oracle_lmls(X_, Y_, hps, layout_, nus=None, post=None, device=None, lanes=None, groupings=None):
    calls.append(len(hps))
    out = []
    for i, hp in enumerate(hps):
      m, nv, k = layout_.unpack(hp, Y_, None if nus is None else nus[i])
      out.append(O.OGP(X_, Y_, oracle_of(k), lambda x, c=m: np.array([c] * len(x)), nv).compute_log_marginal_likelihood())
    return np.array(out), post
  monkeypatch.setattr(hp_grid, 'lml_for_hyperparams', oracle_lmls)

  def oracle_gp(Xl, Yl, kern, mean, noise):
    return O.OGP(np.array(Xl), np.array(Yl), oracle_of(kern), mean, noise)
  np.random.seed(5)
  res = hp_grid.fit_gp(X, Y, layout, g[tag + '_bounds'], _dscr_vals(g, tag), method=method,
                       max_evals=int(g[tag + '_max_evals']), gp_factory=oracle_gp)
  if method == 'rand_exp_sampling':
    _, cts, dscr, other, probs = res
    assert (cts == g[tag + '_cts']).all() and (np.array(dscr) == g[tag + '_dscr']).all()
    np.testing.assert_allclose(probs, g[tag + '_probs'], rtol=1e-9, atol=1e-15)
    assert calls == [len(cts)]
  else:
    _, gp, (cts, dscr) = res
    assert (np.array(cts) == g[tag + '_cts']).all() and (np.array(dscr) == g[tag + '_dscr']).all()
    np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-11)
    mu, sd = gp.eval(g[tag + '_C'], 'std')
    np.testing.assert_allclose(mu, g[tag + '_mu'], atol=1e-10)
    np.testing.assert_allclose(sd, g[tag + '_sd'], atol=1e-9)


def test_layout_from_an_esp_fitter():
  from argparse import Namespace
  from dragonfly_b200 import hp_grid
  opt = Namespace(mean_func_type='median', noise_var_type='tune', kernel_type='esp', esp_kernel_type='matern',
                  esp_order=-1, esp_matern_nu=-1.0, use_additive_gp=False)
  lay = hp_grid.layout_from_fitter(Namespace(options=opt, dim=4, kernel_type='esp'))
  assert (lay.kernel_type, lay.esp_kernel_type, lay.esp_order) == ('esp', 'matern', -1)
  m, nv, k = lay.unpack(np.zeros(6), np.arange(5.0), (1.5, 3))
  assert type(k).__name__ == 'ESPKernelMatern' and k.hyperparams['order'] == 3
  assert [c.hyperparams['nu'] for c in k.kernel_list] == [1.5] * 4
  opt.use_additive_gp = True                     # ESP with use_additive_gp falls through to the reference
  assert hp_grid.layout_from_fitter(Namespace(options=opt, dim=4, kernel_type='esp')) is None


CASES = [('se', d, r, bw) for d in (1, 2, 4, 8) for r in range(1, d + 1) for bw in (0.05, 0.4)] + \
        [('matern', d, r, 0.3) for d in (2, 4, 8) for r in range(1, d + 1)] + \
        [('se', 12, 12, 2.0), ('se', 20, 1, 0.5), ('se', 20, 3, 0.5), ('se', 20, 10, 2.0), ('se', 20, 20, 2.0)]


def test_oracle_within_the_forward_error_bound():
  """ The reference-order recurrence (the oracle, fp64) against the extended-precision value: the measured ratio
      |K^ - K| / bound stays below 1 for every case. """
  worst = 0.0
  for kind, d, r, bw in CASES:
    rs = np.random.RandomState(d * 100 + r)
    X, Y = rs.random_sample((60, d)), rs.random_sample((50, d))
    bws = list(bw * (1.0 + 0.5 * rs.random_sample(d)))
    nus = [(0.5, 1.5, 2.5)[t % 3] for t in range(d)] if kind == 'matern' else None
    ok = E.oracle_kernel(kind, 1.3, r, bws, nus)
    Kh = ok(X, Y)
    ex = E.esp_exact(kind, 1.3, r, bws, X, Y, nus)
    b = E.esp_bound(kind, 1.3, r, bws, X, Y, nus)
    ratio = float(np.max(np.abs(Kh.astype(E.LD) - ex) / b))
    worst = max(worst, ratio)
    assert ratio < 1.0, (kind, d, r, bw, ratio)
  print('ESP recurrence: max |K^ - K| / bound = %.3g over %d cases' % (worst, len(CASES)))
