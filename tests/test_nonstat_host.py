"""
Poly and ExpDecay kernels on the host side (no GPU): the kernel classes, their descriptor form (factor kinds POLY and
EXPDECAY, kss = NaN, include/dfb200.h), the refusals, the NumPy restatement (tests/nonstat_ref.py) against fixtures
recorded from the unmodified reference (golden nonstat.npz, fitter_expdecay.npz) and the multi-fidelity fitter's
hyper-parameter layout with an ExpDecay fidelity kernel.
"""
import math
from argparse import Namespace

import numpy as np
import pytest

from conftest import load_golden
from dragonfly_b200 import kernel as K, _lib, mf_gp, hp_grid
from oracle import gp_oracle as O
import nonstat_ref as R


def test_classes_mirror_the_reference():
  p = K.PolyKernel(3, 2, 1.5, [0.5, 1.0, 2.0])
  assert p.dim == 3 and set(p.hyperparams) == {'order', 'scale', 'dim_scalings'} and p.is_guaranteed_psd()
  assert p.hyperparams['dim_scalings'].tolist() == [0.5, 1.0, 2.0]
  assert K.PolyKernel(2, 1, 1.0, 0.7).hyperparams['dim_scalings'].tolist() == [0.7, 0.7]
  with pytest.raises(ValueError):
    K.PolyKernel(3, 2, 1.5, [0.5, 1.0])
  e = K.ExpDecayKernel(2, 1.1, 0.3, 1.5)              # a scalar power is broadcast to every dimension
  assert e.hyperparams == {'scale': 1.1, 'offset': 0.3, 'powers': [1.5, 1.5]} and e.is_guaranteed_psd()
  g = mf_gp.EuclideanGP._get_kernel_from_type('poly', dict(dim=2, order=3, scale=0.9, dim_scalings=[0.2, 0.3]))
  assert type(g).__name__ == 'PolyKernel' and g.hyperparams['order'] == 3


def test_descriptor_fields():
  d = K.build_descriptor(K.PolyKernel(3, 5, 1.5, [0.5, 1.0, 2.0]))
  f = d.factors[0]
  assert (d.n_terms, d.n_factors, d.n_slots, d.esp_order) == (1, 1, 3, 0)
  assert (f.kind, f.p, f.n_dims, f.slot_off, f.scale) == (_lib.DFB_BASE_POLY, 5, 3, 0, 1.5)
  assert list(d.slot_bandwidth)[:3] == [0.5, 1.0, 2.0] and math.isnan(d.kss)
  d = K.build_descriptor(K.ExpDecayKernel(2, 1.1, 0.3, [1.0, 2.0]))
  f = d.factors[0]
  assert (f.kind, f.p, f.n_dims, f.scale, f.s2) == (_lib.DFB_BASE_EXPDECAY, 0, 2, 1.1, 0.3)
  assert list(d.slot_bandwidth)[:2] == [1.0, 2.0] and math.isnan(d.kss)
  # the MF product ((scale k_F) k_D): one term, the ExpDecay value (offset included) as one factor
  mf = K.CoordinateProductKernel(4, 2.5, [K.ExpDecayKernel(1, 1.0, 0.05, [1.7]), K.MaternKernel(3, 2.5, 1.0, [0.4] * 3)],
                                 [[0], [1, 2, 3]])
  d = K.build_descriptor(mf)
  assert (d.n_terms, d.n_factors, d.post_scale, d.term_pre_scale[0]) == (1, 2, 1.0, 2.5)
  assert [d.factors[i].kind for i in range(2)] == [_lib.DFB_BASE_EXPDECAY, _lib.DFB_BASE_MATERN]
  assert list(d.slot_train_coord)[:4] == [0, 1, 2, 3] and math.isnan(d.kss)


def test_kss_is_nan_exactly_when_a_factor_is_non_stationary():
  se = lambda: K.SEKernel(2, 1.3, [0.4, 0.5])
  stationary = [se(), K.MaternKernel(2, 1.5, 0.7, [0.3, 0.4]),
                K.AdditiveKernel(1.0, [se(), K.SEKernel(1, 1.0, [0.2])], [[0, 1], [2]]),
                K.CoordinateProductKernel(3, 2.0, [se(), K.SEKernel(1, 1.0, [0.2])], [[0, 1], [2]]),
                K.ESPKernelSE(3, 1.0, 2, [0.3, 0.4, 0.5])]
  non_stationary = [K.PolyKernel(2, 1, 1.0, [1.0, 1.0]), K.ExpDecayKernel(2, 1.0, 0.1, 1.0),
                    K.AdditiveKernel(1.0, [se(), K.PolyKernel(1, 2, 1.0, [0.5])], [[0, 1], [2]]),
                    K.CoordinateProductKernel(3, 2.0, [K.ExpDecayKernel(1, 1.0, 0.1, 2.0), se()], [[0], [1, 2]])]
  for k in stationary:
    d = K.build_descriptor(k)
    assert K.is_stationary(d) and np.isfinite(d.kss) and d.kss > 0, k
  for k in non_stationary:
    d = K.build_descriptor(k)
    assert not K.is_stationary(d) and math.isnan(d.kss), k


def test_duck_typing_by_class_name():
  class PolyKernel(object):                  # stand-ins for the reference's own classes
    def __init__(self):
      self.dim = 2
      self.hyperparams = {'order': 2, 'scale': 0.5, 'dim_scalings': np.array([1.5, 0.5])}

  class ExpDecayKernel(object):
    def __init__(self):
      self.dim = 1
      self.hyperparams = {'scale': 1.0, 'offset': 0.2, 'powers': [2.0]}

  d = K.build_descriptor(PolyKernel())
  assert (d.factors[0].kind, d.factors[0].p, d.factors[0].scale) == (_lib.DFB_BASE_POLY, 2, 0.5)
  d = K.build_descriptor(ExpDecayKernel())
  assert (d.factors[0].kind, d.factors[0].s2, d.slot_bandwidth[0]) == (_lib.DFB_BASE_EXPDECAY, 0.2, 2.0)


def test_refusals():
  for order in (1.5, 2.0000001, -1):
    with pytest.raises(NotImplementedError):
      K.build_descriptor(K.PolyKernel(2, order, 1.0, [1.0, 1.0]))
  K.build_descriptor(K.PolyKernel(2, 2.0, 1.0, [1.0, 1.0]))          # an integral float order is an integer order
  for child in (K.PolyKernel(1, 2, 1.0, [1.0]), K.ExpDecayKernel(1, 1.0, 0.1, 1.0)):
    with pytest.raises(NotImplementedError):
      K.build_descriptor(K.ESPKernel(1.0, 1, [K.SEKernel(1, 1.0, [0.3]), child]))
  with pytest.raises(NotImplementedError):
    hp_grid.EuclideanMFHPLayout(1, 3, 'poly', 'se')
  with pytest.raises(NotImplementedError):
    hp_grid.EuclideanMFHPLayout(1, 3, 'se', 'expdecay')


def _mf_fitter(fidel, domain):
  opt = Namespace(mean_func_type='tune', noise_var_type='tune', fidel_kernel_type=fidel, domain_kernel_type=domain,
                  fidel_matern_nu=2.5, domain_matern_nu=2.5, domain_use_additive_gp=False)
  return Namespace(options=opt, fidel_dim=1, domain_dim=3)


def test_layout_from_an_mf_fitter():
  lay = hp_grid.layout_from_fitter(_mf_fitter('expdecay', 'matern'))
  assert type(lay) is hp_grid.EuclideanMFExpDecayHPLayout
  assert (lay.fidel_kernel_type, lay.domain_kernel_type, lay.num_hps()) == ('expdecay', 'matern', 8)
  assert type(hp_grid.layout_from_fitter(_mf_fitter('se', 'matern'))) is hp_grid.EuclideanMFHPLayout
  # the reference's fitter raises for a Poly fidelity or domain kernel: those stay with the reference
  assert hp_grid.layout_from_fitter(_mf_fitter('poly', 'se')) is None
  assert hp_grid.layout_from_fitter(_mf_fitter('expdecay', 'poly')) is None
  assert hp_grid.layout_from_fitter(_mf_fitter('se', 'poly')) is None


def test_oracle_against_the_reference_kernel_blocks():
  g = load_golden('nonstat')
  for d in (1, 2, 4, 8):
    for order in (1, 2, 3, 5):
      ours = R.OPolyKernel(d, order, 0.8, g['poly_scal_%d' % d])(g['poly_X1_%d_%d' % (d, order)],
                                                                  g['poly_X2_%d_%d' % (d, order)])
      np.testing.assert_allclose(ours, g['poly_K_%d_%d' % (d, order)], rtol=1e-14, atol=0)
  for i in range(4):
    d, scale, offset = g['ed_meta_%d' % i]
    pw = g['ed_powers_%d' % i]
    powers = list(pw) if pw.ndim else float(pw)           # case 3: one scalar power for every dimension
    ours = R.OExpDecayKernel(int(d), scale, offset, powers)(g['ed_X1_%d' % i], g['ed_X2_%d' % i])
    assert np.array_equal(ours, g['ed_K_%d' % i]), i
  cp = O.OCoordinateProductKernel(4, 1.4, [R.OExpDecayKernel(1, 1.0, 0.15, [2.0]),
                                           O.OMaternKernel(3, 2.5, 1.0, [0.5, 0.7, 0.9])], [[0], [1, 2, 3]])
  np.testing.assert_allclose(cp(g['cp_X1'], g['cp_X2']), g['cp_K'], rtol=1e-15, atol=0)


def mf_oracle_gp(g):
  kern = O.OCoordinateProductKernel(5, float(g['mf_scale']), [R.OExpDecayKernel(1, 1.0, float(g['mf_offset']),
                                                                                g['mf_powers']),
                                                              O.OMaternKernel(4, 2.5, 1.0, g['mf_bws'])],
                                    [[0], [1, 2, 3, 4]])
  mc = float(g['mf_mean'])
  return O.OGP(np.concatenate((g['mf_Z'], g['mf_Xd']), axis=1), g['mf_Y'], kern, lambda x: np.array([mc] * len(x)),
               float(g['mf_noise']))


def test_oracle_gps_against_the_reference_gps():
  g = load_golden('nonstat')
  ogp = mf_oracle_gp(g)
  np.testing.assert_allclose(ogp.L[:16], g['mf_L_rows'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(ogp.alpha, g['mf_alpha'], rtol=1e-9, atol=1e-9)
  np.testing.assert_allclose(ogp.compute_log_marginal_likelihood(), float(g['mf_lml']), rtol=1e-11)
  for fz in (0.2, 0.6, 1.0):
    tag = ('%g' % fz).replace('.', 'p')
    mu, var = O.eval_std_diag(ogp, O.mf_zx(np.array([fz]), g['mf_Cx']))
    np.testing.assert_allclose(mu, g['mf_mu_' + tag], rtol=0, atol=1e-10)
    np.testing.assert_allclose(var, g['mf_sd_' + tag] ** 2, rtol=0, atol=1e-8)
  mc = float(g['poly_gp_mean'])
  pgp = O.OGP(g['poly_gp_X'], g['poly_gp_Y'], R.OPolyKernel(4, 2, float(g['poly_gp_scale']), g['poly_gp_scal']),
              lambda x: np.array([mc] * len(x)), float(g['poly_gp_noise']))
  np.testing.assert_allclose(pgp.L[:16], g['poly_gp_L_rows'], rtol=0, atol=1e-12)
  np.testing.assert_allclose(pgp.compute_log_marginal_likelihood(), float(g['poly_gp_lml']), rtol=1e-11)
  mu, var = O.eval_std_diag(pgp, g['poly_gp_C'])
  np.testing.assert_allclose(mu, g['poly_gp_mu'], rtol=0, atol=1e-10)
  np.testing.assert_allclose(var, g['poly_gp_sd'] ** 2, rtol=0, atol=1e-8)


def oracle_of_mf(kern):
  """ The oracle twin of the MF layout's CoordinateProductKernel([ExpDecayKernel, SE / Matern kernel]). """
  kf, kd = kern.kernel_list
  hp = kf.hyperparams
  of = R.OExpDecayKernel(kf.dim, hp['scale'], hp['offset'], hp['powers'])
  bws = np.asarray(kd.hyperparams['dim_bandwidths'], dtype=np.float64)
  od = O.OSEKernel(kd.dim, kd.hyperparams['scale'], bws) if type(kd).__name__ == 'SEKernel' else \
      O.OMaternKernel(kd.dim, kd.hyperparams['nu'], kd.hyperparams['scale'], bws)
  return O.OCoordinateProductKernel(kern.dim, kern.hyperparams['scale'], [of, od], kern.coordinate_list)


def test_mf_layout_unpacks_the_reference_fitters_kernel():
  """ [mean] [log noise] log scale, log offset, log power, log domain bandwidths -> the kernel the reference's
      EuclideanMFGPFitter builds: its LML and eval (golden fitter_expdecay.npz, method 'rand'). """
  g = load_golden('fitter_expdecay')
  X, Y = np.concatenate((g['Z'], g['X']), axis=1), g['Y']
  for dom in ('se', 'matern'):
    tag = dom + '_rand'
    lay = hp_grid.EuclideanMFExpDecayHPLayout(1, 3, dom, domain_nu=float(g[tag + '_domain_matern_nu']),
                                              mean_func_type=str(g['mean_func_type']),
                                              noise_var_type=str(g['noise_var_type']))
    cts = g[tag + '_cts']
    assert lay.num_hps() == len(cts) == len(g[tag + '_bounds'])
    mc, nv, kern = lay.unpack(cts, Y)
    kf = kern.kernel_list[0]
    assert type(kf).__name__ == 'ExpDecayKernel' and kf.hyperparams['scale'] == 1.0
    assert kf.hyperparams['offset'] == np.exp(cts[3]) and list(kf.hyperparams['powers']) == [np.exp(cts[4])]
    assert (mc, nv, kern.hyperparams['scale']) == (cts[0], np.exp(cts[1]), np.exp(cts[2]))
    ogp = O.OGP(X, Y, oracle_of_mf(kern), lambda x, c=mc: np.array([c] * len(x)), nv)
    np.testing.assert_allclose(ogp.compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-11)
    mu, var = O.eval_std_diag(ogp, np.concatenate((g[tag + '_Cz'], g[tag + '_Cx']), axis=1))
    np.testing.assert_allclose(mu, g[tag + '_mu'], rtol=0, atol=1e-10)
    np.testing.assert_allclose(var, g[tag + '_sd'] ** 2, rtol=0, atol=1e-8)


@pytest.mark.parametrize('dom,method', [(d, m) for d in ('se', 'matern') for m in ('rand', 'rand_exp_sampling')])
def test_fit_gp_selects_what_the_reference_mf_fitter_selects(dom, method, monkeypatch):
  """ hp_grid.fit_gp with the MF layout, LMLs from the oracle: the same candidates, hps and probabilities as the
      reference's EuclideanMFGPFitter with fidel_kernel_type 'expdecay'. """
  g = load_golden('fitter_expdecay')
  tag = '%s_%s' % (dom, method)
  X, Y = np.concatenate((g['Z'], g['X']), axis=1), g['Y']
  lay = hp_grid.EuclideanMFExpDecayHPLayout(1, 3, dom, domain_nu=float(g[tag + '_domain_matern_nu']),
                                            mean_func_type=str(g['mean_func_type']),
                                            noise_var_type=str(g['noise_var_type']))

  def oracle_lmls(X_, Y_, hps, layout_, nus=None, post=None, device=None, lanes=None, groupings=None):
    out = []
    for hp in hps:
      m, nv, k = layout_.unpack(hp, Y_)
      out.append(O.OGP(X_, Y_, oracle_of_mf(k), lambda x, c=m: np.array([c] * len(x)), nv)
                 .compute_log_marginal_likelihood())
    return np.array(out), post
  monkeypatch.setattr(hp_grid, 'lml_for_hyperparams', oracle_lmls)

  def oracle_gp(Xl, Yl, kern, mean, noise):
    return O.OGP(np.array(Xl), np.array(Yl), oracle_of_mf(kern), mean, noise)
  np.random.seed(5)
  res = hp_grid.fit_gp(X, Y, lay, g[tag + '_bounds'], [], method=method, max_evals=int(g[tag + '_max_evals']),
                       gp_factory=oracle_gp)
  if method == 'rand_exp_sampling':
    _, cts, _, _, probs = res
    assert (cts == g[tag + '_cts']).all()
    np.testing.assert_allclose(probs, g[tag + '_probs'], rtol=1e-9, atol=1e-15)
  else:
    _, gp, (cts, _) = res
    assert (np.array(cts) == g[tag + '_cts']).all()
    np.testing.assert_allclose(gp.compute_log_marginal_likelihood(), float(g[tag + '_lml']), rtol=1e-11)


def test_expdecay_mf_layout():
  """ EuclideanMFExpDecayHPLayout: [mean]? [log noise]? log scale, log offset, log power x fidel_dim, log domain
      bandwidths (euclidean_gp.py:521-541, 871-877); the fidelity kernel has scale 1 and no bandwidths, so
      fidel_use_same_bandwidth plays no part.  EuclideanMFHPLayout itself keeps SE / Matern fidelity kernels only. """
  ed = hp_grid.EuclideanMFExpDecayHPLayout(2, 2, 'se', domain_use_same_bandwidth=False, mean_func_type='median',
                                           noise_var_type='value', noise_var_value=0.07)
  assert isinstance(ed, hp_grid.EuclideanMFHPLayout) and ed.fidel_kernel_type == 'expdecay'
  m, nv, kern = ed.unpack([np.log(2.0), np.log(0.05), np.log(1.5), np.log(3.0), np.log(0.1), np.log(0.9)],
                          np.array([1.0, 5.0, 2.0]))
  assert (m, nv, ed.num_hps(), ed.tuned_nus()) == (2.0, 0.07, 6, [False, False])
  kF, kD = kern.kernel_list
  assert type(kF).__name__ == 'ExpDecayKernel' and kF.hyperparams['scale'] == 1.0
  np.testing.assert_allclose([kF.hyperparams['offset']] + list(kF.hyperparams['powers']), [0.05, 1.5, 3.0])
  np.testing.assert_allclose(kD.hyperparams['dim_bandwidths'], [0.1, 0.9])
  assert kern.coordinate_list == [[0, 1], [2, 3]] and abs(kern.hyperparams['scale'] - 2.0) < 1e-15
  tuned = hp_grid.EuclideanMFExpDecayHPLayout(1, 3, 'matern', domain_nu=-1.0, mean_func_type='tune',
                                              noise_var_type='tune')
  assert tuned.num_hps() == 8 and tuned.tuned_nus() == [False, True]
  _, _, kern = tuned.unpack(np.zeros(8), np.arange(5.0), nu=1.5)
  assert kern.kernel_list[1].hyperparams['nu'] == 1.5
  for dom in ('poly', 'expdecay'):
    with pytest.raises(NotImplementedError):
      hp_grid.EuclideanMFExpDecayHPLayout(1, 2, dom)
  for fidel, dom in (('poly', 'se'), ('se', 'poly'), ('expdecay', 'se'), ('se', 'expdecay')):
    with pytest.raises(NotImplementedError):
      hp_grid.EuclideanMFHPLayout(1, 2, fidel, dom)
