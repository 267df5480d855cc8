"""
Generates tests/golden/fitter_add.npz: the UNMODIFIED reference's EuclideanGPFitter.fit_gp with use_additive_gp
(euclidean_gp.py:312-323, 718-776) for ml_hp_tune_opt 'rand' and 'rand_exp_sampling', seeded.  Authoring container:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_fitter_add.py
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
  d = 5
  X = rs.random_sample((40, d)); Y = np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2] - (X[:, 3] - 0.5) ** 2 + 0.3 * X[:, 4]
  out = dict(X=X, Y=Y)
  for method, evals in [('rand', 20), ('rand_exp_sampling', 25)]:
    options = load_options(euclidean_gp_args)
    options.kernel_type = 'matern'; options.matern_nu = -1.0
    options.use_additive_gp = True; options.add_max_group_size = 3; options.num_groups_per_group_size = 2
    options.hp_tune_criterion = 'ml'; options.ml_hp_tune_opt = method; options.hp_tune_max_evals = evals
    np.random.seed(7)
    fitter = EuclideanGPFitter(list(X), list(Y), options)
    res = fitter.fit_gp()
    out[method + '_bounds'] = np.array(fitter.cts_hp_bounds)
    out[method + '_dscr_vals_nu'] = np.array(fitter.dscr_hp_vals[0])
    out[method + '_dscr_vals_grp'] = np.array(fitter.dscr_hp_vals[1])
    out[method + '_max_evals'] = fitter.hp_tune_max_evals
    out['mean_func_type'] = options.mean_func_type; out['noise_var_type'] = options.noise_var_type
    if res[0] == 'fitted_gp':
      _, gp, (cts, dscr) = res
      out[method + '_cts'] = np.array(cts); out[method + '_dscr'] = np.array(dscr)
      out[method + '_lml'] = gp.compute_log_marginal_likelihood()
      out[method + '_groupings'] = np.array([g + [-1] * (3 - len(g)) for g in gp.kernel.groupings])
      C = rs.random_sample((30, d))
      mu, sd = gp.eval(C, 'std')
      out[method + '_C'] = C; out[method + '_mu'] = mu; out[method + '_sd'] = sd
      print(method, cts, dscr, gp.kernel.groupings, out[method + '_lml'])
    else:
      _, cts, dscr, other, probs = res
      out[method + '_cts'] = np.array(cts); out[method + '_dscr'] = np.array(dscr); out[method + '_probs'] = probs
      out[method + '_groupings'] = np.array([[g + [-1] * (3 - len(g)) for g in o.add_gp_groupings] +
                                             [[-1] * 3] * (5 - len(o.add_gp_groupings)) for o in other])
      print(method, np.array(cts).shape, np.array(dscr)[:3].tolist(), probs.max(), other[0].add_gp_groupings)
  np.savez_compressed(os.path.join(HERE, 'fitter_add.npz'), **out)


if __name__ == '__main__':
  main()
