"""
Generates tests/golden/fitter.npz: the UNMODIFIED reference's EuclideanGPFitter.fit_gp (gp_core.py:783-821,
euclidean_gp.py:153-345) with hp_tune_criterion='ml' and the three continuous-hp optimisers that the device path
batches ('rand', 'rand_exp_sampling', 'pdoo'), under a seeded global RNG.  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_fitter.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402
from dragonfly.gp.euclidean_gp import EuclideanGPFitter, euclidean_gp_args  # noqa
from dragonfly.utils.option_handler import load_options  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])


def main():
  rs = np.random.RandomState(0)
  X = rs.random_sample((60, 3)); Y = np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2]
  out = dict(X=X, Y=Y)
  for method, evals in [('rand', 40), ('rand_exp_sampling', 40), ('pdoo', 60)]:
    options = load_options(euclidean_gp_args)
    options.kernel_type = 'matern'; options.matern_nu = -1.0
    options.hp_tune_criterion = 'ml'; options.ml_hp_tune_opt = method; options.hp_tune_max_evals = evals
    np.random.seed(5)
    fitter = EuclideanGPFitter(list(X), list(Y), options)
    res = fitter.fit_gp()
    out[method + '_bounds'] = np.array(fitter.cts_hp_bounds)
    out[method + '_dscr_vals'] = np.array(fitter.dscr_hp_vals)
    out[method + '_max_evals'] = fitter.hp_tune_max_evals
    out['mean_func_type'] = options.mean_func_type; out['noise_var_type'] = options.noise_var_type
    if res[0] == 'fitted_gp':
      _, gp, (cts, dscr) = res
      out[method + '_cts'] = np.array(cts); out[method + '_dscr'] = np.array(dscr)
      out[method + '_lml'] = gp.compute_log_marginal_likelihood()
      C = rs.random_sample((50, 3))
      mu, sd = gp.eval(C, 'std')
      out[method + '_C'] = C; out[method + '_mu'] = mu; out[method + '_sd'] = sd
      print(method, cts, dscr, out[method + '_lml'])
    else:
      _, cts, dscr, other, probs = res
      out[method + '_cts'] = np.array(cts); out[method + '_dscr'] = np.array(dscr); out[method + '_probs'] = probs
      print(method, np.array(cts).shape, np.array(dscr).shape, probs.max(), other[:2])
  np.savez_compressed(os.path.join(HERE, 'fitter.npz'), **out)


if __name__ == '__main__':
  main()
