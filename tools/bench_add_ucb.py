"""
Add-UCB with the sequential maximisers: one asy.add_ucb call on the c3_additive40_add_ucb workload (40 dimensions,
7 groups) at N = 2000 and 5000, with the bandit's default budgets at t = N (gp_bandit.py:726-738: 'direct'
clip(25 sqrt(1000), 1000, 3e4) = 1000 evaluations, 'pdoo' clip(50 sqrt(1000), 2000, 6e4) = 2000; the 'direct' call runs
PDOO, as the reference does without its Fortran DIRECT).  Three arms, alternated, median of --steps after --warmup:
  grouped    the library path: all groups' PDOO searches in lock-step, each round one dfb_score_groups call
  per_group  the same lock-step search, each group's points of a round scored through that group's own fused session
             (dfb_set_test_kernel + dfb_eval): one device call per group and round
  host       the same search scored by the NumPy oracle, one point per call as the reference does, on --host-budget
             evaluations per group, extrapolated per evaluation
Per arm: wall time per call, device calls, and the bytes of W = L^-1 the contractions read (lower triangle, computed from
the shapes: every 8-row launch of the row-streaming contraction streams it once).  Prints one JSON line with the card's
name and power limit read in the same run.

  python tools/bench_add_ucb.py [--steps 3] [--warmup 1] [--host-budget 140]
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_mixed import _card  # noqa: E402

BUDGETS = {'direct': 1000, 'pdoo': 2000}


def _w_bytes(n, rows_per_call):
  """ Bytes of W's lower triangle the row-streaming contraction reads for calls of the given row counts. """
  tri = 8.0 * n * (n + 1) / 2
  return sum(((r + 7) // 8) * tri for r in rows_per_call)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--warmup', type=int, default=1)
  ap.add_argument('--sizes', type=str, default='2000,5000')
  ap.add_argument('--host-budget', type=int, default=140)
  args = ap.parse_args()
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('bench_add_ucb needs a GPU')
  from dragonfly_b200 import synth_data, kernel, gp_core, doo, domains
  from dragonfly_b200 import gpb_acquisitions as A
  from oracle import gp_oracle as O
  sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
  import bench
  card, power = _card()
  out = {'tool': 'bench_add_ucb', 'card': card, 'power_limit': power, 'steps': args.steps, 'results': []}
  for n in [int(s) for s in args.sizes.split(',')]:
    w = synth_data.make_workload('c3_additive40_add_ucb', n_train=n, n_cand=16)
    spec = w['kernel']
    sub = [kernel.MaternKernel(k['dim'], k['nu'], k['scale'], k['dim_bandwidths']) for k in spec['kernels']]
    add = kernel.AdditiveKernel(spec['scale'], sub, spec['groupings'])
    gp = gp_core.GP(w['X'], w['Y'], add, gp_core.ConstantMean(w['mean_const']), w['noise_var'])
    groups = spec['groupings']
    descs = [gp._group_test_descriptor(add, sub[j], groups[j], w['dim']) for j in range(len(groups))]
    post = gp._device_posterior()
    ogp = O.OGP(w['X'], w['Y'], bench.oracle_kernel(O, spec), lambda x: np.array([w['mean_const']] * len(x)),
                w['noise_var'])
    okern = bench.oracle_kernel(O, spec)
    dom = domains.EuclideanDomain([[0, 1]] * w['dim'])
    for method, budget in BUDGETS.items():
      anc = Namespace(curr_acq='add_ucb', max_evals=budget, t=n, domain=dom, acq_opt_method=method,
                      domain_bounds=np.array(dom.bounds), handle_parallel='halluc', eval_points_in_progress=[],
                      is_mf=False, curr_max_val=0.0)
      betas = [A._get_add_ucb_beta_th(len(g), n) for g in groups]
      rows = {'grouped': [], 'per_group': []}
      real = post.score_groups

      def grouped():
        def counted(*a):
          rows['grouped'].append(len(a[2]))
          return real(*a)
        post.score_groups = counted
        try:
          return A.asy.add_ucb(gp, anc)
        finally:
          del post.score_groups

      def per_group():
        def score(requests):
          vals = []
          for j, X in requests:
            with gp._fused_session(None, [], test_desc=descs[j], mean_const=0.0) as sess:
              mu, sd = sess.post.eval(X, 0.0)
            rows['per_group'].append(len(X))
            vals.append(mu + betas[j] * sd)
          return vals
        found = doo.pdoo_maximise_lockstep(score, [np.asarray(anc.domain_bounds)[g] for g in groups],
                                           budget // len(groups))
        ret = np.zeros(w['dim'])
        for (_, p), g in zip(found, groups):
          ret[g] = p
        return ret
      arms = {'grouped': grouped, 'per_group': per_group}
      times = {k: [] for k in arms}
      pts = {}
      for it in range(args.warmup + args.steps):
        for name, fn in arms.items():
          rows[name].clear()
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          pts[name] = fn()
          torch.cuda.synchronize()
          if it >= args.warmup:
            times[name].append(time.perf_counter() - t0)
      assert (pts['grouped'] == pts['per_group']).all(), 'the grouped and per-group arms disagree'
      # host: the oracle, one point per call, on a smaller budget per group; extrapolated per evaluation
      hb = min(args.host_budget, budget // len(groups))
      t0 = time.perf_counter()
      n_host = 0
      for j, g in enumerate(groups):
        def one(x, j=j):
          return float(O.add_ucb_group_scores(ogp, okern, j, np.asarray(x).reshape(1, -1), n)[0][0])
        doo.pdoo_maximise(one, np.asarray(anc.domain_bounds)[g], hb, vectorised=False)
        n_host += len(doo.pdoo_maximise.last_search.query_vals)
      host_per_eval = (time.perf_counter() - t0) / max(n_host, 1)
      n_evals = sum(len(s.query_vals) for s in doo.pdoo_maximise_lockstep.last_searches)
      res = {'n': n, 'method': method, 'budget': budget, 'evaluations': n_evals,
             'rounds': doo.pdoo_maximise_lockstep.last_rounds,
             'host_s_per_call_extrapolated': host_per_eval * n_evals}
      for name in arms:
        res[name] = {'s_per_call': float(np.median(times[name])), 'device_calls': len(rows[name]),
                     'w_gb_read': _w_bytes(n, rows[name]) / 1e9}
      out['results'].append(res)
      print(json.dumps(res), flush=True)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
