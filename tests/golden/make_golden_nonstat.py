"""
Generates tests/golden/nonstat.npz: the UNMODIFIED reference's non-stationary kernels PolyKernel and ExpDecayKernel
(dragonfly/gp/kernel.py:331-433) and GPs built on them.  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore tests/golden/make_golden_nonstat.py

Records
  K blocks (30 x 20) of PolyKernel at orders 1, 2, 3, 5 and d = 1, 2, 4, 8 with unequal dim_scalings;
  K blocks of ExpDecayKernel at dims 1, 2, 3 (powers with 1 and 2 among them, a scalar power, non-zero offsets);
  a CartesianProductKernel([ExpDecayKernel, MaternKernel]) block on points given as per-part lists;
  an EuclideanMFGP with ExpDecay (fidelity, dz = 1) x Matern-2.5 (domain, dx = 4), N = 300: the first rows of L, alpha,
    the LML, K's diagonal, eval_at_fidel mu / sd at fidelities 0.2, 0.6 and 1, a hallucinated eval, asy.ucb / asy.ei on
    the fidel_to_opt slice under a seeded RNG, a BOCA fidelity and point (tests/golden/fake_mf_caller.py), and
    draw_mf_samples with the normals it drew;
  a GP on PolyKernel (order 2, d = 4, noise 0.01), N = 150: L rows, alpha, LML, eval mu / sd and an asy.ei point.
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
sys.path.insert(0, HERE)

import dragonfly  # noqa: E402  (the reference; needs the shim + $DRAGONFLY_REF on PYTHONPATH)
from dragonfly.gp.kernel import PolyKernel, ExpDecayKernel, MaternKernel, CartesianProductKernel  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.gp.euclidean_gp import EuclideanMFGP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa
from fake_mf_caller import FakeMFCaller  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__

EXPDECAY_CASES = [(1, [1.0], 1.3, 0.2), (2, [2.0, 1.0], 0.7, 0.05), (3, [1.0, 2.0, 0.7], 1.1, 0.3), (2, 1.5, 0.9, 0.1)]


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def anc(acq, max_evals, t, d, curr_max, **kw):
  dom = EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq=acq, max_evals=max_evals, t=t, domain=dom, curr_max_val=curr_max,
                   eval_points_in_progress=[], acq_opt_method='rand', handle_parallel='halluc', mf_strategy=None,
                   is_mf=False, domain_bounds=np.array(dom.bounds), **kw)


def kernel_blocks(out):
  for d in (1, 2, 4, 8):
    scal = list(0.4 + 0.9 * np.random.RandomState(200 + d).random_sample(d))
    for order in (1, 2, 3, 5):
      rs = np.random.RandomState(10 * d + order)
      X1, X2 = rs.random_sample((30, d)) * 2 - 0.5, rs.random_sample((20, d)) * 2 - 0.5
      out['poly_K_%d_%d' % (d, order)] = PolyKernel(d, order, 0.8, np.array(scal))(X1, X2)
      out['poly_X1_%d_%d' % (d, order)], out['poly_X2_%d_%d' % (d, order)] = X1, X2
    out['poly_scal_%d' % d] = np.array(scal)
  for i, (d, powers, scale, offset) in enumerate(EXPDECAY_CASES):
    rs = np.random.RandomState(50 + i)
    X1, X2 = rs.random_sample((30, d)), rs.random_sample((20, d))
    out['ed_K_%d' % i] = ExpDecayKernel(d, scale, offset, powers)(X1, X2)
    out['ed_X1_%d' % i], out['ed_X2_%d' % i] = X1, X2
    out['ed_powers_%d' % i], out['ed_meta_%d' % i] = np.asarray(powers), np.array([d, scale, offset])
  # Cartesian product: part 0 a 1-D ExpDecay, part 1 a 3-D Matern-2.5
  rs = np.random.RandomState(70)
  pts = lambda k: [[rs.random_sample(1), rs.random_sample(3)] for _ in range(k)]
  P1, P2 = pts(30), pts(20)
  kern = CartesianProductKernel(1.4, [ExpDecayKernel(1, 1.0, 0.15, [2.0]), MaternKernel(3, 2.5, 1.0, [0.5, 0.7, 0.9])])
  out['cp_K'] = kern(P1, P2)
  flat = lambda P: np.array([np.concatenate(p) for p in P])
  out['cp_X1'], out['cp_X2'] = flat(P1), flat(P2)


def mf_gp(out):
  rs = np.random.RandomState(0)
  n, dz, dx = 300, 1, 4
  Z = rs.random_sample((n, dz)); Xd = rs.random_sample((n, dx))
  Y = (np.sin(3 * Xd[:, 0]) + Xd[:, 1] * Xd[:, 2] - (Xd[:, 3] - 0.4) ** 2) * (0.6 + 0.4 * Z[:, 0]) + \
      0.02 * rs.standard_normal(n)
  powers, offset = [1.7], 0.05
  kF = ExpDecayKernel(dz, 1.0, offset, powers); kD = MaternKernel(dx, 2.5, 1.0, [0.4, 0.5, 0.6, 0.7])
  scale = float(Y.var()); noise = 0.01 * float(Y.var()); m0 = float(np.median(Y))
  mfgp = EuclideanMFGP(list(Z), list(Xd), list(Y), None, scale, kF, kD, const_mean(m0), noise)
  Cx = np.random.RandomState(1).random_sample((500, dx))
  evals = {}
  for fz in (0.2, 0.6, 1.0):
    tag = ('%g' % fz).replace('.', 'p')
    mu, sd = mfgp.eval_at_fidel([np.array([fz])] * len(Cx), list(Cx), uncert_form='std')
    evals['mf_mu_' + tag], evals['mf_sd_' + tag] = mu, sd
  Zh, Xh = rs.random_sample((3, dz)), rs.random_sample((3, dx))
  mu_h, sd_h = mfgp.eval_at_fidel_with_hallucinated_observations(
      [np.array([1.0])] * 200, list(Cx[:200]), list(Zh), list(Xh), uncert_form='std')
  f2o = np.array([1.0])
  pts = {}
  for name in ('ucb', 'ei'):
    np.random.seed(7)
    f2o_gp = ref_acq._get_fidel_to_opt_gp(mfgp, f2o)
    pts['mf_pt_' + name] = getattr(ref_acq.asy, name)(f2o_gp, anc(name, 1500, n, dx, float(Y.max())))
  caller = FakeMFCaller([1.0])
  for coeff in (1e-4, 0.5):
    tag = str(coeff).replace('.', 'p').replace('-', 'm')
    np.random.seed(8)
    a = anc('ucb', 600, n, dx, float(Y.max()), boca_thresh_coeff=coeff, y_range=float(Y.max() - Y.min()),
            boca_max_low_fidel_cost_ratio=0.9)
    a.is_mf = True
    a.eval_fidel_points_in_progress = []
    fid, pt = ref_acq.boca(ref_acq.asy.ucb, mfgp, a, caller)
    pts['mf_boca_fidel_' + tag] = np.asarray(fid, dtype=np.float64)
    pts['mf_boca_point_' + tag] = pt
  S, Zs, Xs = 6, rs.random_sample((48, dz)), rs.random_sample((48, dx))
  np.random.seed(2)
  samples = mfgp.draw_mf_samples(S, list(Zs), list(Xs))
  np.random.seed(2)
  U = np.random.normal(size=(len(Xs), S))
  out.update(mf_Z=Z, mf_Xd=Xd, mf_Y=Y, mf_powers=np.array(powers), mf_offset=offset, mf_bws=np.array([0.4, 0.5, 0.6, 0.7]),
             mf_scale=scale, mf_noise=noise, mf_mean=m0, mf_Cx=Cx, mf_L_rows=mfgp.L[:16], mf_alpha=mfgp.alpha,
             mf_lml=mfgp.compute_log_marginal_likelihood(), mf_Kdiag=np.diag(mfgp.K_trtr_wo_noise), mf_Zh=Zh, mf_Xh=Xh,
             mf_mu_h=mu_h, mf_sd_h=sd_h, mf_t=n, mf_Zs=Zs, mf_Xs=Xs, mf_ts_U=U, mf_ts_samples=samples, **evals, **pts)


def poly_gp(out):
  rs = np.random.RandomState(4)
  n, d = 150, 4
  X = rs.random_sample((n, d))
  Y = X[:, 0] * X[:, 1] - 0.5 * X[:, 2] ** 2 + 0.3 * X[:, 3] + 0.05 * rs.standard_normal(n)
  scal, scale, noise, m0 = [0.9, 1.2, 0.7, 1.1], 0.6, 0.01, float(np.median(Y))
  gp = GP(list(X), list(Y), PolyKernel(d, 2, scale, np.array(scal)), const_mean(m0), noise)
  C = rs.random_sample((400, d))
  mu, sd = gp.eval(C, 'std')
  np.random.seed(11)
  pt = ref_acq.asy.ei(gp, anc('ei', 1500, n, d, float(Y.max())))
  out.update(poly_gp_X=X, poly_gp_Y=Y, poly_gp_scal=np.array(scal), poly_gp_scale=scale, poly_gp_noise=noise,
             poly_gp_mean=m0, poly_gp_C=C, poly_gp_L_rows=gp.L[:16], poly_gp_alpha=gp.alpha,
             poly_gp_lml=gp.compute_log_marginal_likelihood(), poly_gp_mu=mu, poly_gp_sd=sd, poly_gp_pt_ei=pt,
             poly_gp_t=n)


def main():
  out = {}
  kernel_blocks(out)
  mf_gp(out)
  poly_gp(out)
  path = os.path.join(HERE, 'nonstat.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in out.items()})
  print('wrote %s (%.1f KB)' % (path, os.path.getsize(path) / 1024.0))


if __name__ == '__main__':
  main()
