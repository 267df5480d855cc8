"""
Generates tests/golden/*.npz by running the UNMODIFIED reference (dragonfly-opt 0.1.7 under
$DRAGONFLY_REF) on small seeded inputs.  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF \
        python -W ignore tests/golden/make_golden.py

The tests read only the committed fixtures.  Each fixture holds
the inputs (X, Y, candidates, hyper-parameters, normal draws) and the reference's outputs, so both
the NumPy oracle (tests/test_oracle_golden.py) and the CUDA path (tests/test_gpu_parity.py) are
checked against the reference itself.
"""
import os
import sys
from argparse import Namespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402  (the reference; needs the shim + $DRAGONFLY_REF on PYTHONPATH)
from dragonfly.gp.kernel import SEKernel, MaternKernel, AdditiveKernel, CoordinateProductKernel  # noqa
from dragonfly.gp.gp_core import GP  # noqa
from dragonfly.gp.euclidean_gp import EuclideanMFGP  # noqa
from dragonfly.opt import gpb_acquisitions as ref_acq  # noqa
from dragonfly.exd.domains import EuclideanDomain  # noqa
from dragonfly.utils import general_utils as ref_gu  # noqa

from dragonfly_b200 import synth_data  # noqa

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF']), dragonfly.__file__


def const_mean(c):
  return lambda x: np.array([c] * len(x))


def anc(acq, max_evals, t, d, curr_max, in_progress=(), **kw):
  dom = EuclideanDomain([[0, 1]] * d)
  return Namespace(curr_acq=acq, max_evals=max_evals, t=t, domain=dom, curr_max_val=curr_max,
                   eval_points_in_progress=list(in_progress), acq_opt_method='rand',
                   handle_parallel='halluc', mf_strategy=None, is_mf=False,
                   domain_bounds=np.array(dom.bounds), **kw)


def save(name, **arrs):
  path = os.path.join(HERE, name + '.npz')
  np.savez_compressed(path, **{k: np.asarray(v) for k, v in arrs.items()})
  print('wrote %s (%.1f KB)' % (path, os.path.getsize(path) / 1024.0))


def known_answers():
  """ The reference's own known-answer vectors: unittest_general_utils.py:26-35,
      unittest_kernel.py:37-54,82-124 -- evaluated by the reference code. """
  X1 = np.array([[1, 2, 3], [1, 2, 4], [2, 3, 4.5]])
  X2 = np.array([[1, 2, 4], [1, 2, 5], [2, 3, 5]])
  d2 = ref_gu.dist_squared(X1, X2)
  assert (d2 == np.array([[1, 4, 6], [0, 1, 3], [2.25, 2.25, 0.25]])).all()
  data_1 = np.array([[1, 2], [3, 4.5]])
  data_2 = np.array([[1, 2], [3, 4]])
  bws = [0.1, 1]
  se = SEKernel(2, 2, bws)
  out = dict(ds_X1=X1, ds_X2=X2, ds_true=d2, data_1=data_1, data_2=data_2, bws=bws,
             se_scale=2.0, se_11=se(data_1), se_22=se(data_2), se_12=se(data_1, data_2),
             matern_scale=2.1)
  for nu in [0.5, 1.5, 2.5]:
    mk = MaternKernel(2, nu, 2.1, bws)
    tag = str(nu).replace('.', 'p')
    out['matern_%s_11' % tag] = mk(data_1)
    out['matern_%s_22' % tag] = mk(data_2)
    out['matern_%s_12' % tag] = mk(data_1, data_2)
    out['matern_%s_norm_constant' % tag] = mk.norm_constant
  save('known_answers', **out)


def case_c1_se():
  """ C1 scale: Branin 2-D, SE, N=50, every acquisition + the end-to-end asy_* calls. """
  w = synth_data.make_workload('c1_branin_se_ei', n_cand=2000)
  X, Y, C = w['X'], w['Y'], w['candidates']
  k = w['kernel']
  kern = SEKernel(2, k['scale'], k['dim_bandwidths'])
  gp = GP(X, Y, kern, const_mean(w['mean_const']), w['noise_var'])
  mu, sd = gp.eval(C, 'std')
  mu_none, _ = gp.eval(C, 'none')
  t = 50
  beta = ref_acq._get_ucb_beta_th(2, t)
  curr_best = float(Y.max())
  z = (mu - curr_best) / sd
  ei = sd * ref_acq._expected_improvement_for_norm_diff(z)
  pi = ref_acq.normal_distro.cdf(z)
  ucb = mu + beta * sd
  ref_idx = int(ei.argmax())
  comb = np.sqrt(sd[ref_idx] ** 2 + sd ** 2)
  ttei = comb * ref_acq._expected_improvement_for_norm_diff((mu - mu[ref_idx]) / comb)
  # end-to-end through maximise_acquisition / random_maximise with the global NumPy RNG
  e2e = {}
  for acq_name in ['ei', 'ucb', 'pi']:
    np.random.seed(7)
    pt = getattr(ref_acq.asy, acq_name)(gp, anc(acq_name, 1500, t, 2, curr_best))
    np.random.seed(7)
    U = np.random.random((1500, 2))
    e2e['e2e_%s_point' % acq_name] = pt
    e2e['e2e_U'] = U
  # hallucinated observations (q = 3 pending points)
  Xh = np.random.RandomState(3).random_sample((3, 2))
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:800], list(Xh), 'std')
  np.random.seed(7)
  pt_h = ref_acq.asy.ucb(gp, anc('ucb', 1000, t, 2, curr_best, in_progress=list(Xh)))
  save('c1_se', X=X, Y=Y, C=C, scale=k['scale'], bws=k['dim_bandwidths'], mean_const=w['mean_const'],
       noise_var=w['noise_var'], K=gp.K_trtr_wo_noise, L=gp.L, alpha=gp.alpha,
       lml=gp.compute_log_marginal_likelihood(), mu=mu, sd=sd, mu_none=mu_none, t=t, beta=beta,
       curr_best=curr_best, ei=ei, pi=pi, ucb=ucb, ttei=ttei, ttei_ref_idx=ref_idx,
       argmax_ei=int(ei.argmax()), argmax_pi=int(pi.argmax()), argmax_ucb=int(ucb.argmax()),
       argmax_ttei=int(ttei.argmax()), Xh=Xh, mu_h=mu_h, sd_h=sd_h, e2e_h_point=pt_h, **e2e)


def case_matern():
  """ Hartmann-6, Matern nu in {0.5, 1.5, 2.5}, N=300. """
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=300, n_cand=1500)
  X, Y, C = w['X'], w['Y'], w['candidates']
  k = w['kernel']
  out = dict(X=X, Y=Y, C=C, scale=k['scale'], bws=k['dim_bandwidths'], mean_const=w['mean_const'],
             noise_var=w['noise_var'], t=300)
  for nu in [0.5, 1.5, 2.5]:
    tag = str(nu).replace('.', 'p')
    kern = MaternKernel(6, nu, k['scale'], k['dim_bandwidths'])
    gp = GP(X, Y, kern, const_mean(w['mean_const']), w['noise_var'])
    mu, sd = gp.eval(C, 'std')
    beta = ref_acq._get_ucb_beta_th(6, 300)
    ucb = mu + beta * sd
    z = (mu - Y.max()) / sd
    ei = sd * ref_acq._expected_improvement_for_norm_diff(z)
    out.update({'alpha_' + tag: gp.alpha, 'Ldiag_' + tag: np.diag(gp.L), 'Lsub_' + tag: gp.L[::7, ::5],
                'Ksub_' + tag: gp.K_trtr_wo_noise[::7, ::5],
                'lml_' + tag: gp.compute_log_marginal_likelihood(), 'mu_' + tag: mu, 'sd_' + tag: sd,
                'ucb_' + tag: ucb, 'ei_' + tag: ei, 'argmax_ucb_' + tag: int(ucb.argmax()),
                'argmax_ei_' + tag: int(ei.argmax()), 'Kstar_sub_' + tag: kern(C[:64], X)})
  out['beta'] = ref_acq._get_ucb_beta_th(6, 300)
  out['curr_best'] = float(Y.max())
  save('matern_h6', **out)


def case_additive():
  """ Additive GP + Add-UCB (gpb_acquisitions.py:139-189), d=10 in groups of 4/4/2. """
  rs = np.random.RandomState(0)
  n, d = 200, 10
  X = rs.random_sample((n, d))
  Y = synth_data.tiled(synth_data.park1, 4, X)
  groups = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
  sub = [MaternKernel(4, 2.5, 1.0, [0.5] * 4), SEKernel(4, 1.0, [0.4, 0.5, 0.6, 0.7]),
         MaternKernel(2, 1.5, 1.0, [0.3, 0.45])]
  scale = float(Y.var()) / 3.0
  kern = AdditiveKernel(scale, sub, groups)
  noise = 0.01 * float(Y.var())
  m0 = float(np.median(Y))
  gp = GP(X, Y, kern, const_mean(m0), noise)
  C = np.random.RandomState(1).random_sample((900, d))
  mu, sd = gp.eval(C, 'std')
  t = n
  out = dict(X=X, Y=Y, C=C, scale=scale, noise_var=noise, mean_const=m0, t=t, alpha=gp.alpha,
             Ldiag=np.diag(gp.L), lml=gp.compute_log_marginal_likelihood(), mu=mu, sd=sd,
             Ksub=gp.K_trtr_wo_noise[::5, ::3])
  # per-group scores on supplied sub-domain candidates: replicate _add_ucb_acq_j exactly
  Xtr = np.array(gp.X)
  for j, (grp, kj) in enumerate(zip(groups, sub)):
    Cj = np.random.RandomState(10 + j).random_sample((300, len(grp)))
    beta_j = ref_acq._get_add_ucb_beta_th(len(grp), t)
    K_tetr_j = scale * kj(Cj, Xtr[:, grp])
    mu_j = K_tetr_j.dot(gp.alpha) + 0
    V_j = ref_gu.solve_lower_triangular(gp.L, K_tetr_j.T)
    cov_j = scale * kj(Cj, Cj) - V_j.T.dot(V_j)
    sd_j = np.sqrt(np.diag(cov_j))
    out['Cj_%d' % j] = Cj
    out['mu_j_%d' % j] = mu_j
    out['sd_j_%d' % j] = sd_j
    out['score_j_%d' % j] = mu_j + beta_j * sd_j
    out['argmax_j_%d' % j] = int((mu_j + beta_j * sd_j).argmax())
  # end-to-end asy_add_ucb with the global RNG: 3 groups x (900 // 3) candidates
  np.random.seed(11)
  pt = ref_acq.asy.add_ucb(gp, anc('add_ucb', 900, t, d, float(Y.max())))
  np.random.seed(11)
  Us = [np.random.random((300, len(g))) for g in groups]
  out['e2e_point'] = pt
  for j, U in enumerate(Us):
    out['e2e_U_%d' % j] = U
  save('additive', **out)


def case_mf():
  """ Multi-fidelity product kernel (euclidean_gp.py:347-403) + the fidel_to_opt slice used by
      BOCA step 1 (gpb_acquisitions.py:314-332). """
  rs = np.random.RandomState(0)
  n, dz, dx = 150, 1, 4
  Z = rs.random_sample((n, dz)); Xd = rs.random_sample((n, dx))
  Y = synth_data.park1(Xd) * (0.7 + 0.3 * Z[:, 0])
  kF = SEKernel(dz, 1.0, [0.7]); kD = MaternKernel(dx, 2.5, 1.0, [0.4] * dx)
  scale = float(Y.var()); noise = 0.01 * float(Y.var()); m0 = float(np.median(Y))
  mfgp = EuclideanMFGP(list(Z), list(Xd), list(Y), None, scale, kF, kD, const_mean(m0), noise)
  Cx = np.random.RandomState(1).random_sample((700, dx))
  Cz = np.random.RandomState(2).random_sample((700, dz))
  mu, sd = mfgp.eval_at_fidel(list(Cz), list(Cx), uncert_form='std')
  f2o = np.array([1.0])
  boca_gp = ref_acq._get_fidel_to_opt_gp(mfgp, f2o)
  mu_f, sd_f = boca_gp.eval(Cx, uncert_form='std')
  beta = ref_acq._get_ucb_beta_th(dx, n)
  ucb_f = mu_f + beta * sd_f
  save('mf', Z=Z, Xd=Xd, Y=Y, scale=scale, noise_var=noise, mean_const=m0, Cx=Cx, Cz=Cz,
       alpha=mfgp.alpha, Ldiag=np.diag(mfgp.L), lml=mfgp.compute_log_marginal_likelihood(),
       mu=mu, sd=sd, f2o=f2o, mu_f=mu_f, sd_f=sd_f, beta=beta, ucb_f=ucb_f,
       argmax_ucb_f=int(ucb_f.argmax()), t=n)


def case_ts():
  """ Thompson sampling: draw_samples with the normal matrix recovered from the seed
      (gp_core.py:250-254, general_utils.py:224-232). """
  w = synth_data.make_workload('c5_park1_20_ts', n_train=120, n_cand=256)
  X, Y, C = w['X'], w['Y'], w['candidates']
  k = w['kernel']
  kern = MaternKernel(20, 2.5, k['scale'], k['dim_bandwidths'])
  gp = GP(X, Y, kern, const_mean(w['mean_const']), w['noise_var'])
  S = 8
  np.random.seed(2)
  samples = gp.draw_samples(S, C)
  np.random.seed(2)
  U = np.random.normal(size=(len(C), S))
  mu, covar = gp.eval(C, 'covar')
  save('ts', X=X, Y=Y, C=C, scale=k['scale'], bws=k['dim_bandwidths'], mean_const=w['mean_const'],
       noise_var=w['noise_var'], U=U, samples=samples, mu=mu, covar_diag=np.diag(covar),
       argmax=samples.argmax(axis=1))


def case_jitter():
  """ stable_cholesky's jitter ladder (general_utils.py:183-203): duplicated training points and
      zero noise make K singular; the reference adds 10^p max(diag K). """
  rs = np.random.RandomState(5)
  X = rs.random_sample((40, 3))
  X = np.concatenate((X, X[:10]), axis=0)
  Y = np.sin(X.sum(axis=1))
  kern = SEKernel(3, 1.3, [0.9, 1.1, 1.0])
  gp = GP(X, Y, kern, const_mean(0.0), 0.0)
  K = gp.K_trtr_wo_noise
  # which power succeeded?
  power = None
  for p in range(-11, 5):
    try:
      Lp = np.linalg.cholesky(K + (10 ** p) * np.diag(K).max() * np.eye(len(K)))
      if np.allclose(Lp, gp.L, rtol=0, atol=0):
        power = p
        break
    except np.linalg.LinAlgError:
      continue
  C = rs.random_sample((100, 3))
  mu, sd = gp.eval(C, 'std')
  save('jitter', X=X, Y=Y, scale=1.3, bws=[0.9, 1.1, 1.0], L=gp.L, alpha=gp.alpha,
       power=-999 if power is None else power, C=C, mu=mu, sd=sd)


def case_lml_grid():
  """ The hyper-parameter 'grid' objective (gp_core.py:551-563): LML of the GP built from each
      hp vector [log noise, log scale, log bw x d], Matern-2.5. """
  w = synth_data.make_workload('c2_hartmann6_matern_ucb', n_train=200, n_cand=10)
  X, Y = w['X'], w['Y']
  rs = np.random.RandomState(9)
  H, d = 12, 6
  hps = np.concatenate((np.log(Y.var()) + rs.uniform(-6, -2, (H, 1)),
                        np.log(Y.var()) + rs.uniform(-1, 1, (H, 1)),
                        rs.uniform(np.log(0.1), np.log(2.0), (H, d))), axis=1)
  lmls = []
  m0 = float(np.median(Y))
  for hp in hps:
    kern = MaternKernel(d, 2.5, np.exp(hp[1]), np.exp(hp[2:]))
    gp = GP(X, Y, kern, const_mean(m0), np.exp(hp[0]))
    lmls.append(gp.compute_log_marginal_likelihood())
  save('lml_grid', X=X, Y=Y, hps=hps, lmls=np.array(lmls), mean_const=m0)


def case_extra():
  """ TTEI / synchronous batches / covariance / Thompson e2e / BOCA -- the remaining operator-table
      entries, end to end through the reference with the global RNG seeded. """
  from fake_mf_caller import FakeMFCaller
  w = synth_data.make_workload('c1_branin_se_ei', n_cand=2000)
  X, Y, C = w['X'], w['Y'], w['candidates']
  k = w['kernel']
  kern = SEKernel(2, k['scale'], k['dim_bandwidths'])
  gp = GP(X, Y, kern, const_mean(w['mean_const']), w['noise_var'])
  out = dict(X=X, Y=Y, C=C, scale=k['scale'], bws=k['dim_bandwidths'], mean_const=w['mean_const'],
             noise_var=w['noise_var'], t=50, curr_best=float(Y.max()))
  # TTEI: one seed per branch of the coin flip (gpb_acquisitions.py:284)
  seeds = {}
  for seed in range(40):
    np.random.seed(seed)
    branch = 'ei' if np.random.random() < 0.5 else 'tt'
    if branch not in seeds:
      seeds[branch] = seed
    if len(seeds) == 2:
      break
  for branch, seed in seeds.items():
    np.random.seed(seed)
    out['ttei_%s_seed' % branch] = seed
    out['ttei_%s_point' % branch] = ref_acq.asy.ttei(gp, anc('ttei', 1200, 50, 2, float(Y.max())))
  # synchronous batches: worker k sees the previous picks as hallucinations
  for name in ['ucb', 'ei']:
    np.random.seed(21)
    pts = getattr(ref_acq.syn, name)(3, gp, anc(name, 800, 50, 2, float(Y.max())))
    out['syn_%s_points' % name] = np.array(pts)
  # full covariance on 96 candidates
  mu, covar = gp.eval(C[:96], 'covar')
  out['covar_mu'] = mu
  out['covar'] = covar
  # Thompson sampling end to end (single joint draw over all candidates)
  np.random.seed(4)
  out['ts_point'] = ref_acq.asy.ts(gp, anc('ts', 700, 50, 2, float(Y.max())))
  np.random.seed(4)
  out['ts_point_halluc'] = ref_acq.asy.ts(gp, anc('ts', 500, 50, 2, float(Y.max()),
                                                in_progress=list(C[:2])))
  save('extra_c1', **out)

  # BOCA on the MF GP of case_mf
  rs = np.random.RandomState(0)
  n, dz, dx = 150, 1, 4
  Z = rs.random_sample((n, dz)); Xd = rs.random_sample((n, dx))
  Ymf = synth_data.park1(Xd) * (0.7 + 0.3 * Z[:, 0])
  kF = SEKernel(dz, 1.0, [0.7]); kD = MaternKernel(dx, 2.5, 1.0, [0.4] * dx)
  scale = float(Ymf.var()); noise = 0.01 * float(Ymf.var()); m0 = float(np.median(Ymf))
  mfgp = EuclideanMFGP(list(Z), list(Xd), list(Ymf), None, scale, kF, kD, const_mean(m0), noise)
  caller = FakeMFCaller([1.0])
  res = {}
  for coeff in [1e-4, 0.5]:
    np.random.seed(8)
    a = anc('ucb', 600, n, dx, float(Ymf.max()), boca_thresh_coeff=coeff,
            y_range=float(Ymf.max() - Ymf.min()), boca_max_low_fidel_cost_ratio=0.9)
    a.is_mf = True
    a.eval_fidel_points_in_progress = []
    fid, pt = ref_acq.boca(ref_acq.asy.ucb, mfgp, a, caller)
    tag = str(coeff).replace('.', 'p').replace('-', 'm')
    res['boca_fidel_%s' % tag] = np.asarray(fid, dtype=np.float64)
    res['boca_point_%s' % tag] = pt
  # additive domain kernel: add_ucb_for_boca
  groups = [[0, 1], [2, 3]]
  kDa = AdditiveKernel(1.0, [MaternKernel(2, 2.5, 1.0, [0.4, 0.5]), SEKernel(2, 1.0, [0.3, 0.6])], groups)
  mfgp_a = EuclideanMFGP(list(Z), list(Xd), list(Ymf), None, scale / 2, kF, kDa, const_mean(m0), noise)
  np.random.seed(9)
  a = anc('add_ucb', 600, n, dx, float(Ymf.max()), boca_thresh_coeff=1e-4,
          y_range=float(Ymf.max() - Ymf.min()), boca_max_low_fidel_cost_ratio=0.9)
  a.is_mf = True
  a.eval_fidel_points_in_progress = []
  fid, pt = ref_acq.boca(None, mfgp_a, a, caller)
  res['boca_add_fidel'] = np.asarray(fid, dtype=np.float64)
  res['boca_add_point'] = pt
  res['alpha_add'] = mfgp_a.alpha
  save('extra_mf', Z=Z, Xd=Xd, Y=Ymf, scale=scale, noise_var=noise, mean_const=m0, **res)


if __name__ == '__main__':
  if len(sys.argv) > 1 and sys.argv[1] == 'extra':
    case_extra()
    sys.exit(0)
  known_answers()
  case_c1_se()
  case_matern()
  case_additive()
  case_mf()
  case_ts()
  case_jitter()
  case_lml_grid()
  case_extra()
