"""
Golden vectors for the `ga` acquisition maximiser on a mixed Cartesian-product domain, from the UNMODIFIED reference.
The domain has bench_mixed's shape ([Euclidean(2), Integral(1), ProdDiscrete(3 dims, 3/2/5 levels),
ProdDiscreteNumeric(1)], SE x Matern x Hamming x Matern), with string categories only: the reference asserts that every
point it evaluates is a member of the domain, and a category that NumPy promotes ([1, 'x'] draws '1') is not.
  seeded asy_ucb / asy_ei / asy_pi / asy_ttei with acq_opt_method 'ga', budgets 300 to 1000, with 0 and 2 evaluations in
  progress; one syn_ei batch of two; one asy_ei with 'ga-pdoo'; one multi-objective mo_lin_asy_ucb with 'ga'.
For every GA call: the query log (every point in evaluation order, with its value), read from the history that
cp_ga_optimiser_from_proc_args returns, and the smallest selection margin -- the distance of each uniform that
sample_according_to_exp_probs consumes from a boundary of its CDF.  Per run: the returned point and the MT19937 state
afterwards.  Seeds are kept only when every margin is at least 1e-9, so that the 1e-10 / 1e-8 device contract on mu /
sigma^2 cannot move a parent selection.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF:tests/golden python tests/golden/make_golden_cp_ga.py
"""
import json
import os
from argparse import Namespace

import numpy as np
import dragonfly
from dragonfly.gp.cartesian_product_gp import CPGP
from dragonfly.exd.domains import (EuclideanDomain, IntegralDomain, ProdDiscreteDomain, ProdDiscreteNumericDomain,
                                   CartesianProductDomain)
from dragonfly.exd.cp_domain_utils import sample_from_cp_domain
from dragonfly.opt import cp_ga_optimiser, ga_optimiser
from dragonfly.opt import gpb_acquisitions as ref_acq
from dragonfly.opt import multiobjective_gpb_acquisitions as ref_moo

from make_golden_hamming import jpoint, make_kernel, SCALE, NOISE_VAR, NUMERIC_LEVELS
from make_golden_moo_cp import make_kernel2, SCALE2, NOISE_VAR2, WEIGHTS, REFS

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

LEVELS = [['a', 'b', 'c'], ['w', 'x'], ['p', 'q', 'r', 's', 't']]
N_TRAIN = 60
MIN_MARGIN = 1e-9
_CALLS, _MARGINS = [], []
_original_ga = cp_ga_optimiser.cp_ga_optimiser_from_proc_args
_original_sample = ga_optimiser.sample_according_to_exp_probs


def _recording_ga(*args, **kwargs):
  max_val, max_pt, history = _original_ga(*args, **kwargs)
  _CALLS.append(dict(points=[jpoint(x) for x in history.query_points],
                     vals=[float(np.asarray(v).ravel()[0]) for v in history.query_vals]))
  return max_val, max_pt, history


def _recording_sample(fitness_vals, num_samples, replace=False, scaling_param=None, scaling_const=None,
                      sample_uniformly_if_fail=False):
  vals = np.array(fitness_vals, dtype=np.float64).ravel()
  p = np.exp((vals - vals.mean()) / (scaling_const * (vals.std() + 0.0001)))
  p = p / p.sum()
  if not np.isfinite(p.sum()):
    p = np.ones((len(vals),)) / float(len(vals))
  state = np.random.get_state()
  u = np.random.random_sample(num_samples)
  np.random.set_state(state)
  cdf = p.cumsum()
  cdf /= cdf[-1]
  _MARGINS.append(float(np.abs(u[:, None] - cdf[None, :]).min()))
  return _original_sample(fitness_vals, num_samples, replace, scaling_param, scaling_const, sample_uniformly_if_fail)


cp_ga_optimiser.cp_ga_optimiser_from_proc_args = _recording_ga
ga_optimiser.sample_according_to_exp_probs = _recording_sample


def make_domain():
  return CartesianProductDomain([EuclideanDomain([[0, 1], [-1, 2]]), IntegralDomain([[0, 6]]),
                                 ProdDiscreteDomain(LEVELS), ProdDiscreteNumericDomain(NUMERIC_LEVELS)])


def objective(pt):
  e, i, c, n = pt
  return (np.sin(3 * e[0]) + 0.3 * e[1] - 0.1 * (i[0] - 3) ** 2 + (0.4 if c[0] == 'b' else 0.0) +
          (0.3 if c[2] in ('q', 's') else -0.1) + (0.2 if c[1] == 'x' else 0.0) + 0.2 * np.log(n[0]))


def objective2(pt):
  e, i, c, n = pt
  return (np.cos(2 * e[1]) - 0.5 * (e[0] - 0.3) ** 2 + 0.05 * i[0] + (0.3 if c[1] == 'x' else -0.2) +
          (0.2 if c[0] in ('a', 'c') else 0.0) - 0.1 * n[0])


CASES = [('ucb', 'ga', 300, 0), ('ucb', 'ga', 1000, 2), ('ei', 'ga', 500, 0), ('ei', 'ga', 700, 2),
         ('pi', 'ga', 400, 0), ('pi', 'ga', 600, 2), ('ttei', 'ga', 800, 0), ('ttei', 'ga', 500, 2),
         ('syn_ei', 'ga', 300, 0), ('ei', 'ga-pdoo', 300, 0), ('mo_lin_ucb', 'ga', 400, 0)]


def main():
  dom = make_domain()
  np.random.seed(11)
  X = sample_from_cp_domain(dom, N_TRAIN)
  H = sample_from_cp_domain(dom, 2)
  Y = np.array([objective(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  Y2 = np.array([objective2(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  mean_const, mean_const2 = float(np.median(Y)), float(np.median(Y2))
  gp = CPGP(X, list(Y), make_kernel(), lambda x: np.array([mean_const] * len(x)), NOISE_VAR)
  gp2 = CPGP(X, list(Y2), make_kernel2(), lambda x: np.array([mean_const2] * len(x)), NOISE_VAR2)
  curr_max = float(np.max(Y))
  out = dict(X=np.array(json.dumps([jpoint(x) for x in X])), H=np.array(json.dumps([jpoint(x) for x in H])), Y=Y, Y2=Y2,
             meta=np.array([SCALE, NOISE_VAR, mean_const]), meta2=np.array([SCALE2, NOISE_VAR2, mean_const2]),
             levels=np.array(json.dumps(LEVELS)), numeric_levels=np.array(json.dumps(NUMERIC_LEVELS)),
             weights=np.array(WEIGHTS), refs=np.array(REFS), t=np.array(len(X)), curr_max=np.array(curr_max),
             beta=np.array(ref_acq._get_ucb_beta_th(ref_acq._get_gp_ucb_dim(gp), len(X))),
             mo_beta=np.array(ref_moo._get_ucb_beta_th(dom.dim, len(X))))

  def anc(method, max_evals, halluc):
    return Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=len(X), handle_parallel='halluc',
                     eval_points_in_progress=H[:halluc], is_mf=False, curr_max_val=curr_max, obj_weights=WEIGHTS,
                     reference_point=REFS)

  def call(name, method, max_evals, halluc):
    if name == 'syn_ei':
      return ref_acq.syn.ei(2, gp, anc(method, max_evals, halluc))
    if name == 'mo_lin_ucb':
      return ref_moo.asy.lin_ucb([gp, gp2], anc(method, max_evals, halluc))
    return getattr(ref_acq.asy, name)(gp, anc(method, max_evals, halluc))

  runs = []
  for k, (name, method, max_evals, halluc) in enumerate(CASES):
    seed = 900 + 10 * k
    while True:
      del _CALLS[:], _MARGINS[:]
      np.random.seed(seed)
      pt = call(name, method, max_evals, halluc)
      if min(_MARGINS) >= MIN_MARGIN:
        break
      seed += 1
    st = np.random.get_state()
    pts = pt if name == 'syn_ei' else [pt]
    runs.append(dict(name=name, method=method, max_evals=max_evals, halluc=halluc, seed=seed,
                     points=[jpoint(p) for p in pts], calls=[len(c['vals']) for c in _CALLS], margin=min(_MARGINS)))
    out['run%d_log' % k] = np.array(json.dumps([c['points'] for c in _CALLS]))
    out['run%d_vals' % k] = np.concatenate([c['vals'] for c in _CALLS])
    out['run%d_state' % k] = np.asarray(st[1])
    out['run%d_pos' % k] = np.array(st[2])
    out['run%d_has_gauss' % k] = np.array(st[3])
    out['run%d_cached_gauss' % k] = np.array(st[4])
  out['runs'] = np.array(json.dumps(runs))
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cp_ga.npz'), **out)
  print(json.dumps([{k: v for k, v in r.items() if k != 'points'} for r in runs]))


if __name__ == '__main__':
  main()
