"""
Generates tests/golden/fitter_esp.npz: the UNMODIFIED reference's EuclideanGPFitter.fit_gp (gp_core.py:783-821,
euclidean_gp.py:205-345) with kernel_type='esp', hp_tune_criterion='ml', both child kinds (esp_kernel_type 'se' with the
order tuned, 'matern' with nu and order tuned) and the three continuous-hp optimisers the device path batches ('rand',
'rand_exp_sampling', 'pdoo'), under a seeded global RNG.  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_fitter_esp.py
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
  rs = np.random.RandomState(1)
  X = rs.random_sample((50, 3)); Y = np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2]
  out = dict(X=X, Y=Y)
  for kind in ('se', 'matern'):
    for method, evals in [('rand', 30), ('rand_exp_sampling', 40), ('pdoo', 40)]:
      tag = '%s_%s' % (kind, method)
      options = load_options(euclidean_gp_args)
      options.kernel_type = 'esp'; options.esp_kernel_type = kind
      options.hp_tune_criterion = 'ml'; options.ml_hp_tune_opt = method; options.hp_tune_max_evals = evals
      np.random.seed(5)
      fitter = EuclideanGPFitter(list(X), list(Y), options)
      res = fitter.fit_gp()
      out[tag + '_bounds'] = np.array(fitter.cts_hp_bounds)
      out[tag + '_n_dscr'] = len(fitter.dscr_hp_vals)
      for i, vals in enumerate(fitter.dscr_hp_vals):
        out[tag + '_dscr_vals_%d' % i] = np.array(vals)
      out[tag + '_max_evals'] = fitter.hp_tune_max_evals
      out['mean_func_type'] = options.mean_func_type; out['noise_var_type'] = options.noise_var_type
      if res[0] == 'fitted_gp':
        _, gp, (cts, dscr) = res
        out[tag + '_cts'] = np.array(cts); out[tag + '_dscr'] = np.array(dscr)
        out[tag + '_lml'] = gp.compute_log_marginal_likelihood()
        C = rs.random_sample((40, 3))
        mu, sd = gp.eval(C, 'std')
        out[tag + '_C'] = C; out[tag + '_mu'] = mu; out[tag + '_sd'] = sd
        print(tag, cts, dscr, out[tag + '_lml'])
      else:
        _, cts, dscr, other, probs = res
        out[tag + '_cts'] = np.array(cts); out[tag + '_dscr'] = np.array(dscr); out[tag + '_probs'] = probs
        print(tag, np.array(cts).shape, np.array(dscr).shape, probs.max())
  np.savez_compressed(os.path.join(HERE, 'fitter_esp.npz'), **out)


if __name__ == '__main__':
  main()
