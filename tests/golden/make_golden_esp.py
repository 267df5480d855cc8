"""
Generates tests/golden/esp.npz: the UNMODIFIED reference's ESP kernels (dragonfly/gp/kernel.py:671-744, ESPKernelSE and
ESPKernelMatern with per-dimension nu) and a GP built on one.  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_esp.py

Records
  K blocks (30 x 20) of ESPKernelSE and of ESPKernelMatern (nu cycling 0.5, 1.5, 2.5 over the dimensions) at
    d in {1, 2, 4, 8} and every order, and at d = 20, orders 1, 2, 3, 10, 20;
  a GP (d = 4, order 2, N = 240): the first rows of L, alpha, the LML, eval mu / sd, a hallucinated eval, the points
    asy_ei / asy_ucb return under a seeded global RNG (random_maximise over 1500 uniform candidates);
  draw_samples at 64 points with the normals it drew (recovered from the same seed).
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402  (the reference; needs the shim + $DRAGONFLY_REF on PYTHONPATH)
from dragonfly.gp.kernel import ESPKernelSE, ESPKernelMatern  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__

NUS = (0.5, 1.5, 2.5)


def nus_of(d):
  return [NUS[t % 3] for t in range(d)]


def bws_of(d):
  return list(0.3 + 0.5 * np.random.RandomState(100 + d).random_sample(d)) if d < 20 else [2.0] * d


def main():
  out = {}
  cases = [(d, r) for d in (1, 2, 4, 8) for r in range(1, d + 1)] + [(20, r) for r in (1, 2, 3, 10, 20)]
  for d, r in cases:
    rs = np.random.RandomState(d * 31 + r)
    X1, X2 = rs.random_sample((30, d)), rs.random_sample((20, d))
    bws = bws_of(d)
    out['K_se_%d_%d' % (d, r)] = ESPKernelSE(d, 1.3, r, np.array(bws))(X1, X2)
    out['K_matern_%d_%d' % (d, r)] = ESPKernelMatern(d, nus_of(d), 1.3, r, np.array(bws))(X1, X2)
    out['X1_%d_%d' % (d, r)], out['X2_%d_%d' % (d, r)] = X1, X2
  # a GP on an ESP-Matern kernel
  d, r = 4, 2
  rs = np.random.RandomState(5)
  X = rs.random_sample((240, d))
  Y = np.sin(3 * X[:, 0]) + X[:, 1] * X[:, 2] - (X[:, 3] - 0.4) ** 2 + 0.05 * rs.standard_normal(240)
  C = rs.random_sample((400, d))
  bws, scale, noise, mc = [0.4, 0.5, 0.6, 0.7], 0.8, 0.01, float(np.median(Y))
  kern = ESPKernelMatern(d, nus_of(d), scale, r, np.array(bws))
  gp = GP(list(X), list(Y), kern, lambda x: np.array([mc] * len(x)), noise)
  mu, sd = gp.eval(C, 'std')
  Xh = rs.random_sample((3, d))
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:200], list(Xh), 'std')
  t, curr_best = 240, float(np.max(Y))
  pts = {}
  for name in ('ei', 'ucb'):
    dom = EuclideanDomain([[0, 1]] * d)
    anc = Namespace(curr_acq=name, max_evals=1500, t=t, domain=dom, curr_max_val=curr_best,
                    eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                    is_mf=False, domain_bounds=np.array(dom.bounds))
    np.random.seed(7)
    pts['pt_' + name] = getattr(ref_acq.asy, name)(gp, anc)
  S, Cts = 6, C[:64]
  np.random.seed(2)
  samples = gp.draw_samples(S, Cts)
  np.random.seed(2)
  U = np.random.normal(size=(len(Cts), S))
  out.update(gp_X=X, gp_Y=Y, gp_C=C, gp_bws=np.array(bws), gp_scale=scale, gp_noise=noise, gp_mean=mc, gp_d=d,
             gp_order=r, L_rows=gp.L[:16], alpha=gp.alpha, lml=gp.compute_log_marginal_likelihood(), mu=mu, sd=sd,
             Xh=Xh, mu_h=mu_h, sd_h=sd_h, t=t, curr_best=curr_best, ts_U=U, ts_samples=samples, **pts)
  path = os.path.join(HERE, 'esp.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in out.items()})
  print('wrote %s (%.1f KB)' % (path, os.path.getsize(path) / 1024.0))


if __name__ == '__main__':
  main()
