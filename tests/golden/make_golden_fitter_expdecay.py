"""
Generates tests/golden/fitter_expdecay.npz: the UNMODIFIED reference's EuclideanMFGPFitter.fit_gp (gp_core.py:783-821,
euclidean_gp.py:418-716) with fidel_kernel_type='expdecay', domain_kernel_type 'se' and 'matern', hp_tune_criterion='ml'
and the continuous-hp optimisers 'rand' and 'rand_exp_sampling', under np.random.seed(5).  Run with the reference source
tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_fitter_expdecay.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402
from dragonfly.gp.euclidean_gp import EuclideanMFGPFitter, euclidean_mf_gp_args  # noqa
from dragonfly.utils.option_handler import load_options  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])


def main():
  rs = np.random.RandomState(1)
  Z = rs.random_sample((60, 1)); X = rs.random_sample((60, 3))
  Y = (np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2]) * (0.5 + 0.5 * Z[:, 0])
  out = dict(Z=Z, X=X, Y=Y)
  for dom in ('se', 'matern'):
    for method, evals in [('rand', 30), ('rand_exp_sampling', 40)]:
      tag = '%s_%s' % (dom, method)
      options = load_options(euclidean_mf_gp_args)
      options.fidel_kernel_type = 'expdecay'; options.domain_kernel_type = dom
      options.hp_tune_criterion = 'ml'; options.ml_hp_tune_opt = method; options.hp_tune_max_evals = evals
      np.random.seed(5)
      fitter = EuclideanMFGPFitter(list(Z), list(X), list(Y), options)
      res = fitter.fit_gp()
      out[tag + '_bounds'] = np.array(fitter.cts_hp_bounds)
      out[tag + '_n_dscr'] = len(fitter.dscr_hp_vals)
      for i, vals in enumerate(fitter.dscr_hp_vals):
        out[tag + '_dscr_vals_%d' % i] = np.array(vals)
      out[tag + '_max_evals'] = fitter.hp_tune_max_evals
      out['mean_func_type'] = options.mean_func_type; out['noise_var_type'] = options.noise_var_type
      out[tag + '_domain_matern_nu'] = options.domain_matern_nu
      if res[0] == 'fitted_gp':
        _, gp, (cts, dscr) = res
        out[tag + '_cts'] = np.array(cts); out[tag + '_dscr'] = np.array(dscr)
        out[tag + '_lml'] = gp.compute_log_marginal_likelihood()
        Cz, Cx = rs.random_sample((40, 1)), rs.random_sample((40, 3))
        mu, sd = gp.eval_at_fidel(list(Cz), list(Cx), uncert_form='std')
        out[tag + '_Cz'] = Cz; out[tag + '_Cx'] = Cx; out[tag + '_mu'] = mu; out[tag + '_sd'] = sd
        print(tag, len(cts), cts, dscr, out[tag + '_lml'])
      else:
        _, cts, dscr, other, probs = res
        out[tag + '_cts'] = np.array(cts); out[tag + '_dscr'] = np.array(dscr); out[tag + '_probs'] = probs
        print(tag, np.array(cts).shape, np.array(dscr).shape, probs.max())
  np.savez_compressed(os.path.join(HERE, 'fitter_expdecay.npz'), **out)


if __name__ == '__main__':
  main()
