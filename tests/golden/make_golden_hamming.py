"""
Golden vectors for categorical and mixed Cartesian-product domains, from the UNMODIFIED reference:
  1. dragonfly.gp.kernel.HammingKernel Gram blocks (pairwise_hamming_kernel, general_utils.py:113-146): string, int and
     mixed-type categories, uniform and non-uniform weights, dims 1, 3 and 9;
  2. a dragonfly.gp.cartesian_product_gp.CPGP on [Euclidean(2), Integral(1), ProdDiscrete(3 dims, 2-5 levels),
     ProdDiscreteNumeric(1)] with SE / Matern / Hamming / Matern factors (default handle_non_psd_kernels): K rows, the
     first rows of L, alpha, the LML, eval mean / std and the hallucinated eval;
  3. sample_from_cp_domain on that domain for a fixed seed, and the MT19937 state after it;
  4. seeded asy_ucb / asy_ei / asy_pi / asy_ttei with acq_opt_method='rand' on that domain (with and without
     hallucinations), and the MT19937 state after each.
Categories and points are stored as JSON strings (values and NumPy type names), never pickled.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python tests/golden/make_golden_hamming.py
"""
import json
import os
from argparse import Namespace

import numpy as np
import dragonfly
from dragonfly.gp.kernel import SEKernel, MaternKernel, HammingKernel, CartesianProductKernel
from dragonfly.gp.cartesian_product_gp import CPGP
from dragonfly.exd.domains import (EuclideanDomain, IntegralDomain, ProdDiscreteDomain, ProdDiscreteNumericDomain,
                                   CartesianProductDomain)
from dragonfly.exd.cp_domain_utils import sample_from_cp_domain
from dragonfly.opt import gpb_acquisitions as ref_acq

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

LEVELS = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']]
NUMERIC_LEVELS = [[0.5, 1.0, 2.0, 4.0]]
SCALE, NOISE_VAR = 1.3, 0.02


def jval(v):
  """ one category / coordinate value -> [JSON value, NumPy / Python type name] """
  if isinstance(v, np.generic):
    return [v.item(), type(v).__name__]
  return [v, type(v).__name__]


def jpoint(pt):
  """ a list-of-parts point -> per part [[value, type name], ...]; an ndarray part carries its dtype's name """
  return [[[x, part.dtype.name] for x in part.tolist()] if isinstance(part, np.ndarray) else [jval(v) for v in part]
          for part in pt]


def make_domain():
  return CartesianProductDomain([EuclideanDomain([[0, 1], [-1, 2]]), IntegralDomain([[0, 6]]),
                                 ProdDiscreteDomain(LEVELS), ProdDiscreteNumericDomain(NUMERIC_LEVELS)])


def make_kernel():
  return CartesianProductKernel(SCALE, [SEKernel(2, 1.0, [0.4, 0.9]), MaternKernel(1, 2.5, 1.0, [2.5]),
                                        HammingKernel([0.5, 0.2, 0.3]), MaternKernel(1, 1.5, 1.0, [1.2])])


def objective(pt):
  e, i, c, n = pt
  return (np.sin(3 * e[0]) + 0.3 * e[1] - 0.1 * (i[0] - 3) ** 2 + (0.4 if c[0] == 'b' else 0.0) +
          (0.3 if c[2] in ('q', 's') else -0.1) + 0.2 * np.log(n[0]))


def hamming_blocks(out):
  rs = np.random.RandomState(11)
  cases = [
      (['u', 'v', 'w'], 1, None),
      ([0, 1, 2, 3], 3, [0.2, 0.5, 0.3]),
      ([1, 'a', 2.5, 'b', True], 9, [0.05, 0.1, 0.15, 0.2, 0.05, 0.1, 0.15, 0.1, 0.1]),
      (['s', 't'], 3, 3),
  ]
  meta = []
  for ci, (vals, dim, wts) in enumerate(cases):
    n1, n2 = 37, 23
    X1 = [[vals[k] for k in rs.randint(0, len(vals), size=dim)] for _ in range(n1)]
    X2 = [[vals[k] for k in rs.randint(0, len(vals), size=dim)] for _ in range(n2)]
    kern = HammingKernel(dim if wts is None else wts)
    out['hk%d_K' % ci] = kern(X1, X2)
    out['hk%d_Kss' % ci] = kern(X1, X1)
    meta.append(dict(X1=[[jval(v) for v in r] for r in X1], X2=[[jval(v) for v in r] for r in X2],
                     weights=None if wts is None else wts, dim=dim))
  out['hk_meta'] = np.array(json.dumps(meta))


def main():
  out = {}
  hamming_blocks(out)
  dom = make_domain()
  np.random.seed(7)
  X = sample_from_cp_domain(dom, 160)
  C = sample_from_cp_domain(dom, 300)
  H = sample_from_cp_domain(dom, 3)
  Y = np.array([objective(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  mean_const = float(np.median(Y))
  gp = CPGP(X, list(Y), make_kernel(), lambda x: np.array([mean_const] * len(x)), NOISE_VAR)
  mu, sd = gp.eval(C, 'std')
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:100], H, 'std')
  out.update(X=np.array(json.dumps([jpoint(x) for x in X])), C=np.array(json.dumps([jpoint(x) for x in C])),
             H=np.array(json.dumps([jpoint(x) for x in H])), Y=Y, meta=np.array([SCALE, NOISE_VAR, mean_const]),
             K=gp.K_trtr_wo_noise[:16], L=gp.L[:16], alpha=gp.alpha, lml=np.array(gp.compute_log_marginal_likelihood()),
             mu=mu, sd=sd, mu_h=mu_h, sd_h=sd_h, levels=np.array(json.dumps(LEVELS)),
             numeric_levels=np.array(json.dumps(NUMERIC_LEVELS)))
  # 3. the sampler
  np.random.seed(21)
  S = sample_from_cp_domain(dom, 50)
  st = np.random.get_state()
  out.update(S=np.array(json.dumps([jpoint(x) for x in S])), S_state=np.asarray(st[1]), S_pos=np.array(st[2]))
  # 4. the acquisitions
  runs = []
  for k, (name, halluc) in enumerate([('ucb', 0), ('ei', 0), ('pi', 0), ('ttei', 0), ('ucb', 2), ('ei', 2),
                                      ('ttei', 2)]):
    np.random.seed(100 + k)
    anc = Namespace(domain=dom, max_evals=2000, acq_opt_method='rand', t=len(X), curr_max_val=float(np.max(Y)),
                    handle_parallel='halluc', eval_points_in_progress=H[:halluc], is_mf=False)
    pt = getattr(ref_acq.asy, name)(gp, anc)
    st = np.random.get_state()
    runs.append(dict(name=name, halluc=halluc, seed=100 + k, point=jpoint(pt)))
    out['acq%d_state' % k] = np.asarray(st[1])
    out['acq%d_pos' % k] = np.array(st[2])
  out['acq_runs'] = np.array(json.dumps(runs))
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'hamming.npz'), **out)
  print({k: np.shape(v) for k, v in out.items()})
  print(runs)


if __name__ == '__main__':
  main()
