"""
Drop-in for dragonfly.opt.multiobjective_gpb_acquisitions (multiobjective_gpb_acquisitions.py:19-125):
the linear / Tchebychev scalarisations of several GPs' UCBs or Thompson draws over one set of random
candidates (SURVEY.md 8f rank 3).  Pure re-use of the hot path: every GP scores the SAME
device-resident candidate matrix with dfb_eval (mu, sd in fp64) or a joint posterior draw, and one
launch of dfb_moo_score_argmax scalarises the objectives in the reference's operation order and
takes random_maximise's arg-max (oper_utils.py:70-80).  Same names, arguments and anc_data fields
(obj_weights, reference_point) as the reference; `asy`, `syn`, `seq` tables at the bottom.

On Cartesian-product domains (CPMultiObjectiveGPBandit, multiobjective_gp_bandit.py:638-757) the reference's `rand`
maximiser calls the acquisition one point at a time (exd_utils.py:247-274): every objective's UCB, or its own 1 x 1
posterior draw, per candidate.  _mo_cp scores every candidate in device slabs: one dfb_eval per objective, then one
dfb_moo_score_argmax (UCB) or dfb_moo_score_argmax_ts (TS, the marginal draws fused into the scalarisation).
"""
from argparse import Namespace
from contextlib import ExitStack

import numpy as np

from . import _lib
from .gpb_acquisitions import (draw_candidates, _check_rand_euclidean, _halluc_points,
                               _delegate_to_reference_maximiser, _sharded_argmax, _draw_one_sample,
                               _ts_cols, _shard_info, _ts_anc_data, _is_cp_domain, _cp_parts, _cp_device_layout,
                               _cp_candidate_source, _cp_other_maximiser, _encode_levels, _slab_argmax, _candidate_rng,
                               _check_nonpos)


def _get_ucb_beta_th(dim, time_step):
  """ :73-75 (0.2, not the single-objective 0.5) """
  return np.sqrt(0.2 * dim * np.log(2 * dim * time_step + 1))


def _device_candidates(gps, rand_pts):
  import torch
  post = gps[0]._post
  return torch.from_numpy(np.ascontiguousarray(rand_pts)).to(post.device), post


def _mo_ucb(kind, gps, anc_data):
  beta_th = _get_ucb_beta_th(anc_data.domain.dim, anc_data.t)
  weights = list(anc_data.obj_weights)
  refs = list(anc_data.reference_point) if kind == _lib.DFB_MOO_TCH_UCB else None
  if _is_cp_domain(anc_data):
    if anc_data.acq_opt_method in ['rand']:
      return _mo_cp(kind, gps, anc_data, weights, refs, beta_th)
    return _cp_other_maximiser(lambda pts: _mo_cp_ucb_scores(kind, gps, pts, weights, refs, beta_th), anc_data)
  if not _check_rand_euclidean(anc_data):
    def acquisition(x):
      return _mo_ucb_scores(kind, gps, np.asarray(x, dtype=np.float64), weights, refs, beta_th)
    return _delegate_to_reference_maximiser(acquisition, anc_data)
  rand_pts = draw_candidates(anc_data.domain.bounds, anc_data.max_evals)

  def scorer(lo, hi):
    """ This rank's rows (all of them in a single process): one upload, one dfb_eval per objective. """
    Xd, post = _device_candidates(gps, rand_pts[lo:hi])
    mus, sds = [], []
    for gp in gps:
      mu, sd = gp.eval(Xd, uncert_form='std')     # CUDA tensors
      mus.append(mu); sds.append(sd)
    return post.moo_score_argmax(kind, mus, sds, weights, refs, beta_th)

  return rand_pts[_sharded_argmax(scorer, len(rand_pts))]


def _mo_ucb_scores(kind, gps, X, weights, refs, beta_th):
  """ The scalarised UCB of every row of X (host ndarray in, host ndarray out). """
  Xd, post = _device_candidates(gps, X)
  mus, sds = zip(*[gp.eval(Xd, uncert_form='std') for gp in gps])
  _, _, sc = post.moo_score_argmax(kind, list(mus), list(sds), weights, refs, beta_th, want_scores=True)
  return sc.cpu().numpy()


def _mo_cp_ucb_scores(kind, gps, pts, weights, refs, beta_th):
  """ The scalarised UCB of a list of list-of-parts points (host ndarray out): each objective evaluates the points in
      its own category coding. """
  mus, sds = zip(*[gp.eval(pts, uncert_form='std') for gp in gps])
  _, _, sc = gps[0]._post.moo_score_argmax(kind, list(mus), list(sds), weights, refs, beta_th, want_scores=True)
  return sc.cpu().numpy()


def mo_lin_asy_ucb(gps, anc_data):
  """ :79-91 -- sum_k w_k mu_k + beta_th sqrt(sum_k w_k^2 sigma_k^2) """
  return _mo_ucb(_lib.DFB_MOO_LIN_UCB, gps, anc_data)


def mo_tch_asy_ucb(gps, anc_data):
  """ :94-107 -- min_k (mu_k + beta_th sqrt(sigma_k) - ref_k) / w_k  (the reference names the std
      `sigma2` and takes its square root; reproduced as written) """
  return _mo_ucb(_lib.DFB_MOO_TCH_UCB, gps, anc_data)


def _mo_ts(kind, gps, anc_data):
  anc_data = _ts_anc_data(anc_data)              # :23-26 -- always the random maximiser, 4x the evaluations
  if _is_cp_domain(anc_data):
    return _mo_cp(kind, gps, anc_data, list(anc_data.obj_weights),
                  list(anc_data.reference_point) if kind == _lib.DFB_MOO_TCH_VAL else None)
  halluc = _halluc_points(anc_data)
  rand_pts = draw_candidates(anc_data.domain.bounds, anc_data.max_evals)
  # one joint draw per objective, in order (global RNG); under torch.distributed each rank computes only
  # its blocks of candidates (the same blocks for every objective)
  samples = [_draw_one_sample(gp, rand_pts, halluc) for gp in gps]
  refs = list(anc_data.reference_point) if kind == _lib.DFB_MOO_TCH_VAL else None
  cols = _ts_cols(gps[0], len(rand_pts))
  lo, hi = (0, len(rand_pts)) if cols is None else cols
  if hi > lo:
    best, idx, _ = gps[0]._post.moo_score_argmax(kind, [v[lo:hi] for v in samples], None,
                                                 list(anc_data.obj_weights), refs)
    idx += lo
  else:
    best, idx = 0.0, -1
  if cols is not None:
    from . import dist as dfb_dist
    _, idx = dfb_dist.all_reduce_argmax(best, idx, device=_shard_info()[2])
  return rand_pts[idx]


def _mo_cp(kind, gps, anc_data, weights, refs, beta_th=0.0):
  """ The `rand` maximiser of the multi-objective acquisitions on a CP domain (anc_data of TS already forced to 'rand'):
      the reference's candidates (candidate_rng 'numpy') or the device's (candidate_rng 'device'), the arg-max in
      np.argmax order.  Each slab is uploaded once, as level indices; every objective's rows use its own Hamming codes
      (one matrix for all when their tables agree) for its dfb_eval.
        UCB kinds  dfb_moo_score_argmax of (mu_k, sd_k), from the GPs themselves (:79-107 call gp.eval).
        VAL kinds  Thompson sampling: candidate i's value of objective k is its own 1 x 1 draw fl(fl(sd_ik z_ik) + mu_ik)
                   (gp_core.py:250-261), with the normals the reference's one-point calls consume -- candidate-major,
                   objective-minor, which np.random.normal(size=(M, K)) after the candidates reproduces, the legacy
                   generator's cached Gaussian included -- or the device's normals of the seed.  Evaluations in progress
                   give each objective the variance of its GP augmented with them and the GP's own mean.  A variance
                   that is not > 0 raises ValueError, as the reference's stable_cholesky does. """
  if not 1 <= len(gps) <= _lib.DFB_MOO_MAX_OBJ:
    raise NotImplementedError('%d objectives: the device scalarises 1 to %d.' % (len(gps), _lib.DFB_MOO_MAX_OBJ))
  if getattr(anc_data, 'is_mf', False) or any(hasattr(gp, 'fidel_space_kernel') or hasattr(gp, 'mfgp') for gp in gps):
    raise NotImplementedError('Multi-objective acquisitions with multi-fidelity GPs are outside the GPU hot-path scope.')
  parts = [_cp_parts(anc_data.domain, gp.kernel) for gp in gps]
  if _shard_info()[1] > 1:
    raise NotImplementedError('Cartesian-product candidate draws are not sharded across ranks.')
  import torch
  ts = kind in (_lib.DFB_MOO_LIN_VAL, _lib.DFB_MOO_TCH_VAL)
  mode = _candidate_rng(anc_data)
  M, K = int(anc_data.max_evals), len(gps)
  luts = [_cp_device_layout(p)[3] for p in parts]
  same = lambda a, b: (a is None) == (b is None) and (a is None or np.array_equal(a, b))
  shared = all(all(map(same, lk, luts[0])) for lk in luts[1:])
  halluc = _halluc_points(anc_data) if ts else []
  with ExitStack() as stack:
    sessions = [stack.enter_context(gp._fused_session(None, halluc)) for gp in gps]
    posts = [sess.post for sess in sessions]
    source, seed = _cp_candidate_source(posts[0], sessions[0].slab_rows, parts[0], M, mode, levels=True,
                                        domain=anc_data.domain)
    z = np.random.normal(size=(source.hi, K)) if ts and mode == 'numpy' else None
    nonpos = 0

    def score(pts, r0):
      nonlocal nonpos
      X = torch.as_tensor(pts, dtype=torch.float64).to(posts[0].device)
      Xs = [_encode_levels(X, luts[0])] * K if shared else [_encode_levels(X.clone(), lk) for lk in luts]
      mus, sds = zip(*[gp._eval_on(post, Xk, True) for gp, post, Xk in zip(gps, posts, Xs)])
      if not ts:
        return posts[0].moo_score_argmax(kind, list(mus), list(sds), weights, refs, beta_th)
      res = posts[0].moo_score_argmax_ts(kind, list(mus), list(sds), weights, refs, seed=seed or 0, row0=r0,
                                         z=None if z is None else z[r0:r0 + len(pts)])
      nonpos += int(res[3])
      return res
    best = _slab_argmax(source, score)
  _check_nonpos(nonpos)
  return source.point(*best)


def mo_lin_asy_ts(gps, anc_data):
  """ :19-41 """
  return _mo_ts(_lib.DFB_MOO_LIN_VAL, gps, anc_data)


def mo_tch_asy_ts(gps, anc_data):
  """ :44-68 """
  return _mo_ts(_lib.DFB_MOO_TCH_VAL, gps, anc_data)


asy = Namespace(lin_ts=mo_lin_asy_ts, tch_ts=mo_tch_asy_ts, lin_ucb=mo_lin_asy_ucb, tch_ucb=mo_tch_asy_ucb)
syn = Namespace()      # the reference has none either (:118-120)
seq = Namespace(lin_ts=mo_lin_asy_ts, tch_ts=mo_tch_asy_ts, lin_ucb=mo_lin_asy_ucb, tch_ucb=mo_tch_asy_ucb)
