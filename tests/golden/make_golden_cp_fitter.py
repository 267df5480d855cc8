"""
Generates tests/golden/cp_fitter.npz: the UNMODIFIED reference's CPGPFitter (cartesian_product_gp.py:325-391) on two
Cartesian-product domains, under a seeded global RNG.  Run from the repository root with the reference source tree in
$DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore \
        tests/golden/make_golden_cp_fitter.py

Configurations:
  M  the mixed domain of tests/golden/hamming.npz: Euclidean(2) x Integral(1) x ProdDiscrete(3 dims, 2-5 levels) x
     ProdDiscreteNumeric(1), default options (Matern 5/2 numeric parts, three Hamming weights), tuned mean and noise;
  T  Euclidean(2) x ProdDiscrete(2 dims) x Integral(1) with both Matern nus tuned (dom_euc_matern_nu =
     dom_int_matern_nu = -1.0): two discrete hps and one linear Hamming weight.
Per configuration: the points (JSON, hamming_ref.jpoint), Y, cts_hp_bounds, dscr_hp_vals and param_order; the first 16
rows of K and the LML of fitter.build_gp at three fixed hp vectors; seeded fits with ml_hp_tune_opt rand,
rand_exp_sampling, pdoo and direct (PDOO where the Fortran DIRECT is not built) -- the selected hps (or the samples and
their probabilities), the LML of every _tuning_objective call and four np.random.random() draws after the fit (RNG
fingerprint) -- and, for M, a post_sampling / slice fit recorded by make_golden_post_sampling.run (T has discrete hps,
which the reference's sampler mis-indexes on CP fitters: see main).  Every seed is the first whose
smallest relative margin (the gap between the two largest distinct LMLs of an ml fit, every acceptance comparison of
the sampler) exceeds 1e-7, far above the ~1e-14 rounding of the reference's eigen-projection (project_first).
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import dragonfly  # noqa: E402
from dragonfly.gp.cartesian_product_gp import CPGPFitter, cartesian_product_gp_args  # noqa: E402
from dragonfly.exd.domains import (EuclideanDomain, IntegralDomain, ProdDiscreteDomain,  # noqa: E402
                                   ProdDiscreteNumericDomain, CartesianProductDomain)
from dragonfly.exd.cp_domain_utils import sample_from_cp_domain  # noqa: E402
from dragonfly.utils.option_handler import load_options  # noqa: E402
import make_golden_post_sampling as P  # noqa: E402
from make_golden_hamming import jpoint  # noqa: E402

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

MIN_MARGIN = 1e-7
ML_METHODS = ('rand', 'rand_exp_sampling', 'pdoo', 'direct')
ML_EVALS = 40


def domain_m():
  return CartesianProductDomain([EuclideanDomain([[0, 1], [-1, 2]]), IntegralDomain([[0, 6]]),
                                 ProdDiscreteDomain([['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']]),
                                 ProdDiscreteNumericDomain([[0.5, 1.0, 2.0, 4.0]])])


def objective_m(pt):
  e, i, c, n = pt
  return (np.sin(3 * e[0]) + 0.3 * e[1] - 0.1 * (i[0] - 3) ** 2 + (0.4 if c[0] == 'b' else 0.0) +
          (0.3 if c[2] in ('q', 's') else -0.1) + 0.2 * np.log(n[0]))


def domain_t():
  return CartesianProductDomain([EuclideanDomain([[0, 1], [0, 1]]), ProdDiscreteDomain([['u', 'v', 'w'], [0, 1]]),
                                 IntegralDomain([[-3, 3]])])


def objective_t(pt):
  e, c, i = pt
  return np.cos(4 * e[0]) * e[1] + (0.5 if c[0] == 'v' else 0.0) - 0.3 * c[1] + 0.05 * i[0] ** 2


CONFIGS = {
    'M': (domain_m, objective_m, 30, {}),
    'T': (domain_t, objective_t, 25, dict(dom_euc_matern_nu=-1.0, dom_int_matern_nu=-1.0)),
}


def data(tag):
  make_dom, obj, n, _ = CONFIGS[tag]
  rs_state = np.random.get_state()
  np.random.seed({'M': 5, 'T': 6}[tag])
  X = sample_from_cp_domain(make_dom(), n)
  Y = np.array([obj(x) for x in X]) + 0.05 * np.random.standard_normal(n)
  np.random.set_state(rs_state)
  return X, Y


def make_fitter(tag, X, Y, **opt_kw):
  make_dom, _, _, dom_opts = CONFIGS[tag]
  opt = load_options(cartesian_product_gp_args)
  opt.mean_func_type = 'tune'
  opt.noise_var_type = 'tune'
  for k, v in list(dom_opts.items()) + list(opt_kw.items()):
    setattr(opt, k, v)
  dom = make_dom()
  return CPGPFitter(list(X), list(Y), dom, domain_kernel_ordering=[''] * dom.num_domains, options=opt)


def fixed_hps(fitter):
  """ three hp vectors: the bounds' midpoint with the first discrete values, two uniform draws with the last / middle """
  b = np.array(fitter.cts_hp_bounds)
  rs = np.random.RandomState(17)
  cts = [0.5 * (b[:, 0] + b[:, 1])] + [b[:, 0] + rs.random_sample(len(b)) * (b[:, 1] - b[:, 0]) for _ in range(2)]
  dv = fitter.dscr_hp_vals
  dscr = [[v[0] for v in dv], [v[-1] for v in dv], [v[len(v) // 2] for v in dv]]
  return cts, dscr


def ml_fit(tag, method, X, Y, out):
  for seed in range(1, 50):
    fitter = make_fitter(tag, X, Y, hp_tune_criterion='ml', ml_hp_tune_opt=method, hp_tune_max_evals=ML_EVALS)
    calls = []
    orig = fitter._tuning_objective

    def logged(cts, dscr, *a, **k):
      v = orig(cts, dscr, *a, **k)
      calls.append(float(v))
      return v
    fitter._tuning_objective = logged
    np.random.seed(seed)
    res = fitter.fit_gp()
    fingerprint = np.array([np.random.random() for _ in range(4)])
    vals = np.unique(np.array(calls))[::-1]
    margin = float((vals[0] - vals[1]) / abs(vals[0]))
    key = '%s_%s_' % (tag, method)
    print(tag, method, 'seed', seed, 'calls', len(calls), 'margin %.2e' % margin)
    if margin <= MIN_MARGIN:
      continue
    out[key + 'seed'] = seed
    out[key + 'method_resolved'] = fitter.ml_hp_tune_opt_method
    out[key + 'max_evals'] = fitter.hp_tune_max_evals
    out[key + 'calls'] = np.array(calls)
    out[key + 'fingerprint'] = fingerprint
    out[key + 'margin'] = margin
    out[key + 'kind'] = res[0]
    if res[0] == 'fitted_gp':
      _, gp, (cts, dscr) = res
      out[key + 'cts'] = np.array(cts, dtype=np.float64)
      out[key + 'dscr'] = np.array(dscr, dtype=np.float64)
      out[key + 'lml'] = gp.compute_log_marginal_likelihood()
    else:
      _, cts, dscr, _, probs = res
      out[key + 'cts'] = np.array(cts, dtype=np.float64)
      out[key + 'dscr'] = np.array(dscr, dtype=np.float64).reshape(len(cts), len(fitter.dscr_hp_vals))
      out[key + 'probs'] = np.array(probs)
    return
  raise RuntimeError('no seed with a margin above %g for %s %s' % (MIN_MARGIN, tag, method))


def main():
  P.REC.install()
  out = {}
  for tag in CONFIGS:
    X, Y = data(tag)
    fitter = make_fitter(tag, X, Y)
    out[tag + '_points'] = np.array(json.dumps([jpoint(x) for x in X]))
    out[tag + '_Y'] = Y
    out[tag + '_bounds'] = np.array(fitter.cts_hp_bounds)
    out[tag + '_dscr_vals'] = np.array(fitter.dscr_hp_vals, dtype=np.float64).reshape(len(fitter.dscr_hp_vals), 3)
    out[tag + '_param_order'] = np.array(json.dumps(fitter.param_order))
    cts, dscr = fixed_hps(fitter)
    out[tag + '_fixed_cts'] = np.array(cts)
    out[tag + '_fixed_dscr'] = np.array(dscr, dtype=np.float64).reshape(3, len(fitter.dscr_hp_vals))
    Ks, lmls = [], []
    for c, d in zip(cts, dscr):
      gp = fitter.build_gp(list(c), list(d))
      Ks.append(np.array(gp.K_trtr_wo_noise[:16]))
      lmls.append(gp.compute_log_marginal_likelihood())
    out[tag + '_fixed_K'] = np.array(Ks)
    out[tag + '_fixed_lml'] = np.array(lmls)
    for method in ML_METHODS:
      ml_fit(tag, method, X, Y, out)
    if fitter.dscr_hp_vals:
      # the sampler takes hp i as discrete when param_order[i] says so (gp_core.py:689-697), but CPGPFitter lists a
      # part's nu before its bandwidths: the vector and param_order disagree and the fit fails or mixes them up
      continue

    def post_fitter(tag=tag, X=X, Y=Y):
      f = make_fitter(tag, X, Y, hp_tune_criterion='post_sampling', post_hp_tune_method='slice',
                      post_hp_tune_offset=2, post_hp_tune_burn=8)
      return f, np.array(json.dumps([jpoint(x) for x in X])), Y, None
    P.run('P' + tag, post_fitter, 3, out, range(1, 50))
  np.savez_compressed(os.path.join(HERE, 'cp_fitter.npz'), **out)
  print(sorted(out))


if __name__ == '__main__':
  main()
