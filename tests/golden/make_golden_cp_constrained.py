"""
Golden vectors of the constrained draw on a mixed Cartesian-product domain, from the UNMODIFIED reference loaded through
load_config: a float of dim 2, a scalar float, an int, a discrete string and a discrete numeric variable, with
constraints modelled on the reference's examples (a norm, a builtin sum, np.sqrt, string equality, int arithmetic, a
discrete-numeric value) and one callable (constraint_fns.z_or_n).  Recorded: the domain's orderings, and for seeded
calls of sample_from_cp_domain and of the `rand` maximiser's draw (exd_utils._rand_maximise_vectorised_objective_in_cp_
domain with a zero objective) the kept count, the points and the MT19937 state after the call -- including calls whose
kept count exceeds M (a maximiser draw of more than one sample_from_cp_domain call) and one that needs several rounds.
Then the GA's constrained initial pool (get_cp_domain_initial_qinfos with latin_hc), and seeded acquisitions on a CPGP
fitted to constrained points: asy EI / UCB / PI / TTEI and TS with 'rand', TS with 'ga', a hallucinated syn_ucb batch,
EI with the default 'ga', and the multi-objective lin_ucb / tch_ts -- each with its point and the MT19937 state after
it.  Seeds of the 'rand' cases are kept only when the winning gap of every scored draw is at least 1e-6.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF:tests/golden python tests/golden/make_golden_cp_constrained.py
"""
import json
import os

from argparse import Namespace

import numpy as np
import dragonfly
from dragonfly.exd.cp_domain_utils import load_config, sample_from_cp_domain
from dragonfly.exd import exd_utils
from dragonfly.exd.exd_utils import get_cp_domain_initial_qinfos
from dragonfly.gp.kernel import SEKernel, MaternKernel, HammingKernel
from dragonfly.gp.cartesian_product_gp import CPGP, CartesianProductKernel
from dragonfly.opt import gpb_acquisitions as ref_acq
from dragonfly.opt import multiobjective_gpb_acquisitions as ref_moo

from constraint_fns import z_or_n

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

VARS = [{'name': 'x', 'type': 'float', 'min': 0, 'max': 1, 'dim': 2},
        {'name': 'z', 'type': 'float', 'min': -1, 'max': 2},
        {'name': 'n', 'type': 'int', 'min': 0, 'max': 6},
        {'name': 'c', 'type': 'discrete', 'items': ['a', 'b', 'c']},
        {'name': 'w', 'type': 'discrete_numeric', 'items': [0.5, 1.0, 2.0, 4.0]}]
CONSTRAINTS = ['np.linalg.norm(x[0:2]) + z <= 1.5',
               "c != 'b' or n > 2",
               'sum(x) + np.sqrt(abs(z)) * w <= 3.5',
               'n * 2 - 3 <= 7 or x[0] < 0.5',
               z_or_n]


def config(constraints):
  return load_config({'domain': [dict(v) for v in VARS],
                      'domain_constraints': [{'constraint': c} for c in constraints]})


def jval(v):
  if isinstance(v, np.ndarray):
    return [jval(e) for e in v]
  if isinstance(v, (list, tuple)):
    return [jval(e) for e in v]
  if isinstance(v, (np.integer, int)) and not isinstance(v, bool):
    return int(v)
  if isinstance(v, (np.floating, float)):
    return float(v)
  return str(v)


MIN_GAP = 1e-6
SCALE, NOISE_VAR = 1.2, 0.02
_RECORD = []
_original = exd_utils._rand_maximise_vectorised_objective_in_cp_domain


def _recording(obj, domain, max_evals, return_history=False):
  max_val, max_pt, history = _original(obj, domain, max_evals, return_history=True)
  vals = np.array([float(np.asarray(v).ravel()[0]) for v in history.query_vals])
  idx = int(np.argmax(vals))
  _RECORD.append(float(vals[idx] - np.delete(vals, idx).max()) if len(vals) > 1 else np.inf)
  if return_history:
    return max_val, max_pt, history
  return max_val, max_pt


def make_kernel():
  return CartesianProductKernel(SCALE, [SEKernel(3, 1.0, [0.4, 0.9, 1.1]), MaternKernel(1, 2.5, 1.0, [2.5]),
                                        HammingKernel([1.0]), MaternKernel(1, 1.5, 1.0, [1.2])])


def objective(pt, k=0):
  e, i, c, w = pt
  if k == 0:
    return np.sin(3 * e[0]) + 0.3 * e[1] - 0.2 * e[2] - 0.05 * (i[0] - 3) ** 2 + (0.4 if c[0] == 'b' else 0.0) + \
        0.1 * np.log(w[0])
  return np.cos(2 * e[1]) - 0.5 * (e[0] - 0.3) ** 2 + 0.05 * i[0] + (0.3 if c[0] == 'c' else -0.1) - 0.1 * w[0]


def acquisitions(dom, out):
  """ the GA pool and the seeded acquisitions on the constrained domain """
  np.random.seed(31)
  pool = [q.point for q in get_cp_domain_initial_qinfos(dom, 17)]
  st = np.random.get_state()
  out['pool'] = np.array(json.dumps([jval(p) for p in pool]))
  out['pool_state'], out['pool_pos'] = np.asarray(st[1]), np.array(st[2])
  np.random.seed(32)
  X = sample_from_cp_domain(dom, 60)
  H = sample_from_cp_domain(dom, 2)
  Y = np.array([objective(x) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  Y2 = np.array([objective(x, 1) for x in X]) + 0.05 * np.random.standard_normal(len(X))
  mc, mc2 = float(np.median(Y)), float(np.median(Y2))
  gp = CPGP(X, list(Y), make_kernel(), lambda x: np.array([mc] * len(x)), NOISE_VAR)
  gp2 = CPGP(X, list(Y2), make_kernel(), lambda x: np.array([mc2] * len(x)), NOISE_VAR)
  out['X'] = np.array(json.dumps([jval(x) for x in X]))
  out['H'] = np.array(json.dumps([jval(x) for x in H]))
  out['Y'], out['Y2'], out['meta'] = Y, Y2, np.array([SCALE, NOISE_VAR, mc, mc2])

  def anc(method, max_evals, halluc):
    return Namespace(domain=dom, max_evals=max_evals, acq_opt_method=method, t=len(X), curr_max_val=float(np.max(Y)),
                     handle_parallel='halluc', eval_points_in_progress=H[:halluc], is_mf=False,
                     obj_weights=[0.6, 0.4], reference_point=[float(np.min(Y)), float(np.min(Y2))])
  cases = [('ei', 'rand', 300, 0), ('ucb', 'rand', 300, 0), ('pi', 'rand', 300, 0), ('ttei', 'rand', 300, 0),
           ('ts', 'rand', 200, 0), ('ts', 'ga', 60, 0), ('syn_ucb', 'rand', 150, 0), ('ei', 'ga', 40, 0),
           ('ucb', 'rand', 300, 2), ('lin_ucb', 'rand', 200, 0), ('tch_ts', 'rand', 200, 0)]
  runs = []
  exd_utils._rand_maximise_vectorised_objective_in_cp_domain = _recording
  try:
    for k, (name, method, max_evals, halluc) in enumerate(cases):
      seed = 700 + 10 * k
      while True:
        del _RECORD[:]
        np.random.seed(seed)
        if name == 'syn_ucb':
          pts = ref_acq.syn.ucb(3, gp, anc(method, max_evals, halluc))
        elif name in ('lin_ucb', 'tch_ts'):
          pts = [getattr(ref_moo.asy, name)([gp, gp2], anc(method, max_evals, halluc))]
        else:
          pts = [getattr(ref_acq.asy, name)(gp, anc(method, max_evals, halluc))]
        if not _RECORD or min(_RECORD) >= MIN_GAP:
          break
        seed += 1
      st = np.random.get_state()
      runs.append(dict(name=name, method=method, max_evals=max_evals, halluc=halluc, seed=seed,
                       points=[jval(p) for p in pts]))
      out['acq%d_state' % k], out['acq%d_pos' % k] = np.asarray(st[1]), np.array(st[2])
      out['acq%d_gauss' % k] = np.array([st[3], st[4]])
  finally:
    exd_utils._rand_maximise_vectorised_objective_in_cp_domain = _original
  out['acq_runs'] = np.array(json.dumps(runs))
  return runs


def main():
  dom = config(CONSTRAINTS).domain
  o = dom.domain_info.config_orderings
  out = dict(orderings=np.array(json.dumps(dict(raw_name_ordering=o.raw_name_ordering, index_ordering=o.index_ordering,
                                                dim_ordering=o.dim_ordering))),
             types=np.array(json.dumps([d.get_type() for d in dom.list_of_domains])))
  runs = []
  # (kind, constraints, M, seed): 'sample' = one sample_from_cp_domain call, 'rand' = the maximiser's draw
  cases = [('sample', 'all', 50, 11), ('sample', 'all', 1, 12), ('rand', 'all', 200, 13),
           ('rand', 'tight', 40, 14), ('sample', 'tight', 40, 15)]
  tight = CONSTRAINTS + ['z <= -0.8']
  for k, (kind, which, M, seed) in enumerate(cases):
    d = dom if which == 'all' else config(tight).domain
    np.random.seed(seed)
    if kind == 'sample':
      pts = sample_from_cp_domain(d, M, verbose_constraint_satisfaction=False)
    else:
      _, _, hist = exd_utils._rand_maximise_vectorised_objective_in_cp_domain(lambda x: 0.0, d, M, return_history=True)
      pts = hist.query_points
    st = np.random.get_state()
    runs.append(dict(kind=kind, which=which, M=M, seed=seed, count=len(pts), points=[jval(p) for p in pts]))
    out['state%d' % k] = np.asarray(st[1])
    out['pos%d' % k] = np.array(st[2])
    out['gauss%d' % k] = np.array([st[3], st[4]])
  out['runs'] = np.array(json.dumps(runs))
  acq_runs = acquisitions(dom, out)
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cp_constrained.npz'), **out)
  print(json.dumps([{k: v for k, v in r.items() if k != 'points'} for r in runs + acq_runs]))


if __name__ == '__main__':
  main()
