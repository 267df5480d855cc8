"""
CPU tests of dragonfly_b200.post_sampling (no GPU): the speculative slice / Metropolis sampler driven by the NumPy
oracle's LML against the reference's own post_sampling fits (golden post_sampling.npz) -- the call trace, the samples
and the global RNG state after the fit -- and the routing of fit_gp_on_fitter for 'post_sampling'.
"""
from argparse import Namespace

import numpy as np
import pytest

from dragonfly_b200 import hp_grid, post_sampling
import post_sampling_ref as R


def _fit(g, tag, depth, seed_offset=0):
  X, Y, layout, bounds, dscr_vals, kw = R.config(g, tag)
  stats, trace = post_sampling.PostSamplingStats(), []
  np.random.seed(int(g[tag + '_seed']) + seed_offset)
  res = post_sampling.post_sample_hps(X, Y, layout, bounds, dscr_vals, build_gp=lambda c, d: (c, d),
                                      lml_batch=R.oracle_lml_batch(X, Y, layout), depth=depth, stats=stats,
                                      trace=trace, **kw)
  fingerprint = np.array([np.random.random() for _ in range(4)])
  return res, fingerprint, stats, trace


def _check_result(g, tag, res, fingerprint):
  assert res[0] == str(g[tag + '_kind'])
  if res[0] == 'post_fitted_gp':
    cts, dscr = res[2]
    assert res[1][0] is cts[0] or np.array_equal(res[1][0], cts[0])
  else:
    _, cts, dscr, other = res
    assert other == [None] * len(cts)
  np.testing.assert_array_equal(cts, g[tag + '_cts'])
  np.testing.assert_array_equal(dscr, g[tag + '_dscr'])
  np.testing.assert_array_equal(fingerprint, g[tag + '_fingerprint'])


def _check_trace(g, tag, trace):
  n_cts = len(g[tag + '_bounds'])
  assert len(trace) == len(g[tag + '_trace_lml'])
  hps = np.array([h for h, _ in trace])
  np.testing.assert_array_equal(hps[:, :n_cts], g[tag + '_trace_cts'])
  np.testing.assert_array_equal(hps[:, n_cts:], g[tag + '_trace_dscr'])
  np.testing.assert_allclose([v for _, v in trace], g[tag + '_trace_lml'], rtol=1e-10, atol=0)


@pytest.mark.parametrize('tag', R.CONFIGS)
def test_depth_one_reproduces_the_reference(golden, tag):
  g = golden('post_sampling')
  res, fingerprint, stats, trace = _fit(g, tag, 1)
  _check_result(g, tag, res, fingerprint)
  _check_trace(g, tag, trace)
  assert stats.consumed == len(trace)
  if tag == 'A':
    assert int(g['A_metropolis_out_of_range']) > 0          # a proposal outside the category ids: prior -inf


@pytest.mark.parametrize('depth', [2, 8, 32])
@pytest.mark.parametrize('tag', R.CONFIGS)
def test_speculation_changes_no_sample(golden, tag, depth):
  g = golden('post_sampling')
  res, fingerprint, stats, trace = _fit(g, tag, depth)
  _check_result(g, tag, res, fingerprint)
  _check_trace(g, tag, trace)
  assert stats.evaluated >= len(set(tuple(h.tolist()) for h, _ in trace))
  if depth == 32:
    # no chain runs 32 points deep here: two batches per slice sample (stepping out, shrinkage), plus at most one per
    # chain for its starting point or its Metropolis categories
    n_hps = len(g[tag + '_bounds']) + len(g[tag + '_dscr_vals'])
    assert stats.round_trips <= 2 * R.num_slice_samples(g, tag) + n_hps


def test_speculation_saves_round_trips(golden):
  g = golden('post_sampling')
  _, _, one, _ = _fit(g, 'B', 1)
  _, _, eight, _ = _fit(g, 'B', 8)
  assert one.consumed == eight.consumed
  assert eight.round_trips < one.round_trips
  assert eight.round_trips <= 2 * R.num_slice_samples(g, 'B') + 5


def test_default_burn_in_is_not_clipped(golden):
  g = golden('post_sampling')
  X, Y, layout, bounds, dscr_vals, kw = R.config(g, 'B')
  assert kw['burn'] == -1
  stats = post_sampling.PostSamplingStats()
  calls = []

  def counting(cts_rows, dscr_rows):
    calls.append(len(cts_rows))
    return R.oracle_lml_batch(X, Y, layout)(cts_rows, dscr_rows)
  np.random.seed(int(g['B_seed']))
  post_sampling.post_sample_hps(X, Y, layout, bounds, dscr_vals, build_gp=lambda c, d: None, lml_batch=counting,
                                depth=1, stats=stats, **kw)
  # 5 hps: int(sqrt(5) * 100) = 223 burn-in samples per hp (the reference's np.clip to [100, 2000] is discarded)
  assert R.num_slice_samples(g, 'B') == 5 * (223 + 1)
  assert stats.consumed == len(g['B_trace_lml'])


# ---- routing (fit_gp_on_fitter) ------------------------------------------------------------------------------------
def _fitter(crit='post_sampling', method='slice', **opt_kw):
  opt = dict(mean_func_type='tune', noise_var_type='tune', kernel_type='matern', matern_nu=-1.0,
             hp_tune_criterion=crit, post_hp_tune_method=method, post_hp_tune_offset=25, post_hp_tune_burn=-1)
  opt.update(opt_kw)
  rs = np.random.RandomState(0)
  X = rs.random_sample((12, 3))
  return Namespace(options=Namespace(**opt), dim=3, X=list(X), Y=list(X.sum(1)),
                   cts_hp_bounds=np.array([[-1, 1], [-5, -1], [-2, 2], [-3, 1], [-3, 1], [-3, 1]]),
                   dscr_hp_vals=[[0.5, 1.5, 2.5]])


def _route(fitter, monkeypatch):
  seen = []
  monkeypatch.setattr(post_sampling, 'post_sample_hps', lambda *a, **k: seen.append(('device', a, k)) or 'device')
  out = hp_grid.fit_gp_on_fitter(fitter, lambda f, n, c: seen.append(('reference', n, c)) or 'reference', 4,
                                 'post_sampling')
  return out, seen


def test_slice_on_a_covered_layout_goes_to_the_device_sampler(monkeypatch):
  out, seen = _route(_fitter(), monkeypatch)
  assert out == 'device'
  _, args, kw = seen[0]
  assert isinstance(args[2], hp_grid.EuclideanHPLayout) and kw['num_samples'] == 4
  assert kw['offset'] == 25 and kw['burn'] == -1
  out, _ = _route(_fitter(kernel_type='se'), monkeypatch)
  assert out == 'device'
  mf = Namespace(options=Namespace(mean_func_type='tune', noise_var_type='tune', fidel_kernel_type='se',
                                   domain_kernel_type='matern', fidel_matern_nu=2.5, domain_matern_nu=-1.0,
                                   domain_use_additive_gp=False, hp_tune_criterion='post_sampling',
                                   post_hp_tune_method='slice', post_hp_tune_offset=3, post_hp_tune_burn=10),
                 fidel_dim=1, domain_dim=2, ZZ=[[0.1], [0.9]], XX=[[0.2, 0.3], [0.4, 0.5]], YY=[1.0, 2.0],
                 cts_hp_bounds=np.zeros((6, 2)), dscr_hp_vals=[[0.5, 1.5, 2.5]])
  out, seen = _route(mf, monkeypatch)
  assert out == 'device'
  np.testing.assert_array_equal(seen[0][1][0], [[0.1, 0.2, 0.3], [0.9, 0.4, 0.5]])


@pytest.mark.parametrize('what', ['nuts', 'additive', 'esp', 'expdecay', 'cpgp'])
def test_everything_else_goes_to_the_reference(monkeypatch, what):
  if what == 'nuts':
    fitter = _fitter(method='nuts')
  elif what == 'additive':
    fitter = _fitter(use_additive_gp=True)
  elif what == 'esp':
    fitter = _fitter(kernel_type='esp', esp_kernel_type='se', esp_order=-1)
  elif what == 'expdecay':
    fitter = Namespace(options=Namespace(mean_func_type='tune', noise_var_type='tune', fidel_kernel_type='expdecay',
                                         domain_kernel_type='se', domain_use_additive_gp=False,
                                         hp_tune_criterion='post_sampling', post_hp_tune_method='slice'),
                       fidel_dim=1, domain_dim=2)
  else:
    fitter = Namespace(options=Namespace(hp_tune_criterion='post_sampling', post_hp_tune_method='slice',
                                         mean_func_type='tune', noise_var_type='tune'))
  out, seen = _route(fitter, monkeypatch)
  assert out == 'reference' and seen == [('reference', 4, 'post_sampling')]
