"""
CPU tests of Cartesian-product (CP) GP fitting (no GPU): hp_grid.CartesianProductHPLayout against the reference's
CPGPFitter (golden cp_fitter.npz) -- bounds, discrete values, param_order, the kernels it unpacks -- and hp_grid.fit_gp /
post_sampling.post_sample_hps with the NumPy oracle's LMLs in place of the device's: the same selections, probabilities,
samples, LML calls and global RNG state as the reference.  Also the routing of fit_gp_on_fitter for CP fitters.
"""
import json
from argparse import Namespace

import numpy as np
import pytest

from dragonfly_b200 import hp_grid, post_sampling, domains
import cp_fitter_ref as R


@pytest.mark.parametrize('tag', R.CONFIGS)
def test_layout_bounds_and_param_order(golden, tag):
  g = golden('cp_fitter')
  lay = R.layout(tag)
  cts, dscr, order = lay.bounds_and_order(R.points(g, tag), g[tag + '_Y'])
  np.testing.assert_array_equal(cts, g[tag + '_bounds'])
  assert dscr == R.dscr_vals(g, tag)
  assert order == json.loads(str(g[tag + '_param_order']))
  assert lay.num_hps() == len(cts) and lay.num_dscr() == len(dscr)
  np.testing.assert_array_equal(lay.bounds(R.points(g, tag), g[tag + '_Y'])[0], cts)


@pytest.mark.parametrize('tag', R.CONFIGS)
def test_unpacked_kernels_against_the_reference(golden, tag):
  g = golden('cp_fitter')
  lay = R.layout(tag)
  X = lay.encode(R.points(g, tag))
  Y = g[tag + '_Y']
  for k, (cts, dscr) in enumerate(zip(g[tag + '_fixed_cts'], g[tag + '_fixed_dscr'])):
    mean_const, noise_var, kern = lay.unpack(cts, Y, tuple(dscr))
    for child, table in zip(kern.kernel_list, lay.codes):
      if table is not None:
        assert child.category_codes is table          # one encoding for the rows and every kernel
    K = R.oracle_kernel(kern)(X[:16], X)
    np.testing.assert_allclose(K, g[tag + '_fixed_K'][k], rtol=0, atol=1e-13)
    np.testing.assert_allclose(R.oracle_lml(X, Y, lay, cts, dscr), g[tag + '_fixed_lml'][k], rtol=1e-10, atol=0)


def _oracle_fit(g, tag, method, monkeypatch):
  lay = R.layout(tag)
  pts, Y = R.points(g, tag), g[tag + '_Y']
  X = lay.encode(pts)
  calls = []

  def batch(X_, Y_, hps, layout, nus=None, post=None, device=None):
    assert layout is lay and np.array_equal(X_, X)
    vals = np.array([R.oracle_lml(X, Y, lay, h, () if nus is None else nus[i]) for i, h in enumerate(hps)])
    calls.extend(vals)
    return vals, None
  monkeypatch.setattr(hp_grid, 'lml_batch_for_hyperparams', batch)
  np.random.seed(int(g['%s_%s_seed' % (tag, method)]))
  res = hp_grid.fit_gp(pts, Y, lay, g[tag + '_bounds'], R.dscr_vals(g, tag), method=method,
                       max_evals=int(g['%s_%s_max_evals' % (tag, method)]), build_gp=lambda c, d, grp: (c, d))
  fingerprint = np.array([np.random.random() for _ in range(4)])
  return res, fingerprint, calls


@pytest.mark.parametrize('method', R.ML_METHODS)
@pytest.mark.parametrize('tag', R.CONFIGS)
def test_ml_fits_reproduce_the_reference(golden, tag, method, monkeypatch):
  g = golden('cp_fitter')
  key = '%s_%s_' % (tag, method)
  res, fingerprint, calls = _oracle_fit(g, tag, method, monkeypatch)
  assert res[0] == str(g[key + 'kind'])
  if method in ('rand', 'rand_exp_sampling'):
    np.testing.assert_allclose(calls, g[key + 'calls'], rtol=1e-10, atol=0)
  else:
    # PDOO evaluates each point once (its cache); the reference calls the objective again for a revisited cell
    calls = np.array(calls)
    for v in g[key + 'calls']:
      assert np.min(np.abs(calls - v)) <= 1e-10 * abs(v)
  if res[0] == 'fitted_gp':
    cts, dscr = res[2]
    np.testing.assert_array_equal(cts, g[key + 'cts'])
    np.testing.assert_array_equal(np.array(dscr, dtype=np.float64), g[key + 'dscr'])
  else:
    _, cts, dscr, other, probs = res
    np.testing.assert_array_equal(cts, g[key + 'cts'])
    np.testing.assert_array_equal(np.array(dscr, dtype=np.float64).reshape(g[key + 'dscr'].shape), g[key + 'dscr'])
    np.testing.assert_allclose(probs, g[key + 'probs'], rtol=1e-10, atol=1e-300)
  np.testing.assert_array_equal(fingerprint, g[key + 'fingerprint'])


@pytest.mark.parametrize('depth', [1, 8])
def test_post_sampling_reproduces_the_reference(golden, depth):
  g = golden('cp_fitter')
  lay = R.layout('M')
  pts, Y = R.points(g, 'M'), g['PM_Y']
  X = lay.encode(pts)
  trace = []
  np.random.seed(int(g['PM_seed']))
  res = post_sampling.post_sample_hps(pts, Y, lay, g['PM_bounds'], R.dscr_vals(g, 'PM'),
                                      num_samples=int(g['PM_num_samples']), offset=int(g['PM_offset']),
                                      burn=int(g['PM_burn']), build_gp=lambda c, d: (c, d),
                                      lml_batch=R.oracle_lml_batch(X, Y, lay), depth=depth, trace=trace)
  fingerprint = np.array([np.random.random() for _ in range(4)])
  assert res[0] == str(g['PM_kind'])
  np.testing.assert_array_equal(res[1], g['PM_cts'])
  np.testing.assert_array_equal(fingerprint, g['PM_fingerprint'])
  assert len(trace) == len(g['PM_trace_lml'])
  np.testing.assert_array_equal(np.array([h for h, _ in trace]), g['PM_trace_cts'])
  np.testing.assert_allclose([v for _, v in trace], g['PM_trace_lml'], rtol=1e-10, atol=0)


def test_layout_refuses_what_the_reference_cannot_build():
  ok = [('euclidean', 2, 'matern'), ('prod_discrete', 2, 'hamming')]
  hp_grid.CartesianProductHPLayout(ok)
  for bad in ([('euclidean', 2, 'matern', 'default', True)],         # use_same_bandwidth: AttributeError there
              [('euclidean', 2, 'matern', -1)],                      # integer nu < 0: a discrete hp never set up
              [('euclidean', 2, 'poly')], [('euclidean', 2, 'esp')], [('integral', 1, 'expdecay')],
              [('prod_discrete', 2, 'se')], [('neural_network', 1, 'otmann')], [('discrete_euclidean', 2, 'matern')]):
    with pytest.raises(NotImplementedError):
      hp_grid.CartesianProductHPLayout(ok + bad)


def test_encode_shares_one_table_per_hamming_part():
  lay = hp_grid.CartesianProductHPLayout([('prod_discrete', 2, 'hamming'), ('euclidean', 1, 'se'),
                                          ('prod_discrete', 1, 'hamming')])
  rows = lay.encode([[['a', 1], np.array([0.5]), ['a']], [[1, 'a'], np.array([0.25]), [True]]])
  # Python equality: 1 == True, so the third part codes both values alike; the first part's table is its own
  np.testing.assert_array_equal(rows, [[0, 1, 0.5, 0], [1, 0, 0.25, 1]])
  _, _, kern = lay.unpack([0.0, 0.0, 0.3, 0.1], np.zeros(2))
  assert kern.kernel_list[0].category_codes is lay.codes[0] and kern.kernel_list[2].category_codes is lay.codes[2]
  np.testing.assert_array_equal(kern.kernel_list[0].hyperparams['dim_weights'], [0.3, 0.7])


# ---- routing (fit_gp_on_fitter) ------------------------------------------------------------------------------------
def _cp_fitter(crit='ml', method='rand', ordering=None, **opt_kw):
  opt = dict(mean_func_type='tune', noise_var_type='tune', hp_tune_criterion=crit, post_hp_tune_method='slice',
             post_hp_tune_offset=25, post_hp_tune_burn=-1, dom_euc_kernel_type='default', dom_int_kernel_type='default',
             dom_disc_kernel_type='default', dom_disc_num_kernel_type='default', dom_euc_matern_nu='default',
             dom_int_matern_nu='default', dom_disc_num_matern_nu='default', dom_euc_use_same_bandwidth=False,
             dom_int_use_same_bandwidth=False, dom_disc_num_use_same_bandwidth=False,
             dom_disc_hamming_use_same_weight=False, dom_euc_use_additive_gp=False, dom_int_use_additive_gp=False)
  opt.update(opt_kw)
  dom = domains.CartesianProductDomain([domains.EuclideanDomain([[0, 1], [0, 1]]), domains.IntegralDomain([[0, 4]]),
                                        domains.ProdDiscreteDomain([['a', 'b'], ['c', 'd', 'e']])])
  X = [[np.array([0.1 * i, 0.2]), [i % 5], [['a', 'b'][i % 2], ['c', 'd', 'e'][i % 3]]] for i in range(8)]
  return Namespace(options=Namespace(**opt), domain=dom, domain_kernel_ordering=ordering or [''] * 3,
                   domain_lists_of_dists=[None] * 3, X=X, Y=list(np.arange(8.0)), ml_hp_tune_opt_method=method,
                   hp_tune_max_evals=50, cts_hp_bounds=np.zeros((7, 2)), dscr_hp_vals=[],
                   build_gp=lambda c, d, other_gp_params=None: ('built', c, d))


def _route(fitter, monkeypatch, crit):
  seen = []
  monkeypatch.setattr(hp_grid, 'fit_gp', lambda *a, **k: seen.append(('ml', a, k)) or 'device')
  monkeypatch.setattr(post_sampling, 'post_sample_hps', lambda *a, **k: seen.append(('post', a, k)) or 'device')
  out = hp_grid.fit_gp_on_fitter(fitter, lambda f, n, c: seen.append(('reference', n, c)) or 'reference', 1, crit)
  return out, seen


@pytest.mark.parametrize('crit', ['ml', 'post_sampling'])
def test_cp_fitter_goes_to_the_device(monkeypatch, crit):
  out, seen = _route(_cp_fitter(crit), monkeypatch, crit)
  assert out == 'device'
  _, args, kw = seen[0]
  lay = args[2]
  assert isinstance(lay, hp_grid.CartesianProductHPLayout)
  assert [(p.dom_type, p.dim, p.kernel_type) for p in lay.parts] == \
      [('euclidean', 2, 'matern'), ('integral', 1, 'matern'), ('prod_discrete', 2, 'hamming')]
  assert args[0] is not None and len(args[0]) == 8            # list-of-parts points: the layout encodes them
  if crit == 'ml':
    assert kw['build_gp']([1.0], [], None) == ('built', [1.0], [])
  # a kernel ordering entry overrides the options; tuned nus on the ml path
  out, seen = _route(_cp_fitter(crit, ordering=['se', '', 'hamming'], dom_int_matern_nu=-1.0), monkeypatch, crit)
  lay = seen[0][1][2] if seen[0][0] != 'reference' else None
  if crit == 'ml':
    assert out == 'device' and lay.parts[0].kernel_type == 'se' and lay.num_dscr() == 1
  else:
    assert out == 'reference'                                  # the reference's sampler mis-indexes tuned nus here


@pytest.mark.parametrize('what', ['same_bandwidth', 'integer_nu', 'poly', 'additive', 'cpmf', 'dists', 'nuts',
                                  'mean_func'])
def test_out_of_scope_cp_fitters_go_to_the_reference(monkeypatch, what):
  crit = 'post_sampling' if what == 'nuts' else 'ml'
  kw = dict(same_bandwidth=dict(dom_euc_use_same_bandwidth=True), integer_nu=dict(dom_int_matern_nu=-1),
            poly=dict(dom_euc_kernel_type='poly'), additive=dict(dom_euc_use_additive_gp=True),
            nuts=dict(post_hp_tune_method='nuts'), mean_func=dict(mean_func=lambda x: x)).get(what, {})
  fitter = _cp_fitter(crit, **kw)
  if what == 'cpmf':
    fitter.fidel_space = fitter.domain
  if what == 'dists':
    fitter.domain_lists_of_dists = [None, None, [np.zeros((8, 8))]]
  out, seen = _route(fitter, monkeypatch, crit)
  assert out == 'reference' and seen == [('reference', 1, crit)]
