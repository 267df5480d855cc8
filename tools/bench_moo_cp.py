"""
The multi-objective acquisitions on a mixed Cartesian-product domain: the domain and first CPGP of tools/bench_mixed.py
([Euclidean(2), Integral(1), ProdDiscrete(3 dims, 2-5 levels), ProdDiscreteNumeric(1)] under SE x Matern x Hamming x
Matern, N = 2000) plus a second objective under the kernel of tests/golden/moo_cp.npz's second CPGP.  One asy.lin_ts and
one asy.tch_ucb call at 1.2 x 10^5 candidates (the reference's cap of 3 x 10^4 for a CP domain, times 4 for Thompson
sampling) and at 10^6, in both candidate modes, arms alternated:
  parity  candidate_rng 'numpy': the reference's candidates (and, for TS, np.random.normal(size=(M, 2))) on the host,
          scored in device slabs: one dfb_eval per objective, then dfb_moo_score_argmax(_ts)
  device  candidate_rng 'device': rows from dfb_fill_mixed_candidates, TS normals made in the scoring kernel
and host arms that score the reference's way -- one oracle call per point and objective (exd_utils.py:247-274): a 1 x 1
draw for TS, an eval for UCB -- on a few hundred points, reported as rates.  Prints one JSON line with the median wall
time per call and candidates/s of each arm, the card's name and its power limit read in the same run.

  python tools/bench_moo_cp.py [--steps 3] [--warmup 1] [--host-m 300]
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_mixed import _card  # noqa: E402

ACQS = ('lin_ts', 'tch_ucb')
SIZES = (120000, 1000000)
WEIGHTS, REFS = [0.6, 0.4], [0.1, -1.0]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=3)
  ap.add_argument('--warmup', type=int, default=1)
  ap.add_argument('--n', type=int, default=2000)
  ap.add_argument('--host-m', type=int, default=300)
  args = ap.parse_args()
  import torch
  from dragonfly_b200 import kernel, cartesian_product_gp as cp, gpb_acquisitions as acq, domains, _lib
  from dragonfly_b200 import multiobjective_gpb_acquisitions as moo
  from oracle import gp_oracle as O
  import hamming_ref as R
  import moo_cp_ref as T
  _lib.load()
  levels, numeric_levels = [['a', 'b', 'c'], [1, 'x'], ['p', 'q', 'r', 's', 't']], [[0.5, 1.0, 2.0, 4.0]]
  dom = R.make_domain(domains, levels, numeric_levels)
  kerns = [R.make_kernel(kernel, cp, 1.3), T.make_kernel2(kernel, cp, 0.7)]
  parts = acq._cp_parts(dom, kerns[0])
  np.random.seed(0)
  Xr, draws = acq.draw_cp_candidates(parts, args.n)
  X = [acq.point_from_draws(parts, draws, i) for i in range(args.n)]
  Ys = [np.sin(3 * Xr[:, 0]) + 0.3 * Xr[:, 1] - 0.1 * (Xr[:, 2] - 3) ** 2 + 0.4 * (Xr[:, 3] == 1) +
        0.2 * np.log(Xr[:, 6]) + 0.05 * np.random.standard_normal(args.n),
        np.cos(2 * Xr[:, 1]) - 0.5 * (Xr[:, 0] - 0.3) ** 2 + 0.05 * Xr[:, 2] - 0.1 * Xr[:, 6] +
        0.05 * np.random.standard_normal(args.n)]
  mcs = [float(np.median(Y)) for Y in Ys]
  noise = [0.02, 0.01]
  gps = [cp.CPGP(X, list(Y), kern, (lambda c: (lambda x: np.array([c] * len(x))))(mc), nv)
         for Y, kern, mc, nv in zip(Ys, kerns, mcs, noise)]
  arms = [(name, M, mode) for name in ACQS for M in SIZES for mode in ('numpy', 'device')]
  times = dict((arm, []) for arm in arms)
  for step in range(args.warmup + args.steps):
    for name in ACQS:
      for M in SIZES:
        for mode in (('numpy', 'device') if step % 2 == 0 else ('device', 'numpy')):     # alternate the arms
          anc = Namespace(domain=dom, max_evals=M, acq_opt_method='rand', t=args.n, handle_parallel='halluc',
                          eval_points_in_progress=[], is_mf=False, candidate_rng=mode, obj_weights=WEIGHTS,
                          reference_point=REFS)
          np.random.seed(step)
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          getattr(moo.asy, name)(gps, anc)
          t1 = time.perf_counter()
          if step >= args.warmup:
            times[(name, M, mode)].append(t1 - t0)
  result = {}
  for (name, M, mode), ts in times.items():
    s = float(np.median(ts))
    result['%s_%s_%d' % (name, 'parity' if mode == 'numpy' else 'device', M)] = dict(s_per_call=round(s, 4),
                                                                                    cand_per_s=round(M / s, 1))
  # host arms: the reference's one-point calls per objective -- draw_samples(1, [x]) (a 1 x 1 covariance, its Cholesky
  # factor, one normal) for TS, eval([x], 'std') for UCB
  codes = {}
  okerns = [R.oracle_kernel(1.3), T.oracle_kernel2(0.7)]
  ogps = [O.OGP(R.encode_points(X, codes), Y, okern, (lambda c: (lambda x: np.array([c] * len(x))))(mc), nv)
          for Y, okern, mc, nv in zip(Ys, okerns, mcs, noise)]
  beta = O.moo_ucb_beta_th(dom.dim, args.n)
  np.random.seed(1)
  _, hdraws = acq.draw_cp_candidates(parts, args.host_m)
  pts = [acq.point_from_draws(parts, hdraws, i) for i in range(args.host_m)]
  for name in ACQS:
    t0 = time.perf_counter()
    vals = []
    for p in pts:
      row = R.encode_points([p], codes)
      if name == 'lin_ts':
        s = 0.0
        for ogp, w in zip(ogps, WEIGHTS):
          mu, cov = ogp.eval(row, 'covar')
          L, _ = O.stable_cholesky(cov)
          s += (L.dot(np.random.normal(size=(1, 1))).T + mu).ravel() * w
      else:
        mus, sds = zip(*[ogp.eval(row, 'std') for ogp in ogps])
        s = T.scalarise(name, mus, sds, WEIGHTS, REFS, beta)
      vals.append(float(np.asarray(s).ravel()[0]))
    int(np.argmax(vals))
    s = time.perf_counter() - t0
    result['%s_host_one_point_%d' % (name, args.host_m)] = dict(s_per_call=round(s, 4),
                                                                 cand_per_s=round(args.host_m / s, 1))
  name, plimit = _card()
  print(json.dumps(dict(bench='moo_cp', n=args.n, steps=args.steps, card=name, power_limit=plimit, arms=result)))


if __name__ == '__main__':
  main()
