"""
Drop-in for dragonfly.opt.multiobjective_gpb_acquisitions (multiobjective_gpb_acquisitions.py:19-125):
the linear / Tchebychev scalarisations of several GPs' UCBs or Thompson draws over one set of random
candidates (SURVEY.md 8f rank 3).  Pure re-use of the hot path: every GP scores the SAME
device-resident candidate matrix with dfb_eval (mu, sd in fp64) or a joint posterior draw, and one
launch of dfb_moo_score_argmax scalarises the objectives in the reference's operation order and
takes random_maximise's arg-max (oper_utils.py:70-80).  Same names, arguments and anc_data fields
(obj_weights, reference_point) as the reference; `asy`, `syn`, `seq` tables at the bottom.
"""
from argparse import Namespace

import numpy as np

from . import _lib
from .gpb_acquisitions import (draw_candidates, _check_rand_euclidean, _halluc_points,
                               _delegate_to_reference_maximiser, _sharded_argmax, _draw_one_sample,
                               _ts_cols, _shard_info, _ts_anc_data)


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


def mo_lin_asy_ucb(gps, anc_data):
  """ :79-91 -- sum_k w_k mu_k + beta_th sqrt(sum_k w_k^2 sigma_k^2) """
  return _mo_ucb(_lib.DFB_MOO_LIN_UCB, gps, anc_data)


def mo_tch_asy_ucb(gps, anc_data):
  """ :94-107 -- min_k (mu_k + beta_th sqrt(sigma_k) - ref_k) / w_k  (the reference names the std
      `sigma2` and takes its square root; reproduced as written) """
  return _mo_ucb(_lib.DFB_MOO_TCH_UCB, gps, anc_data)


def _mo_ts(kind, gps, anc_data):
  anc_data = _ts_anc_data(anc_data)              # :23-26 -- always the random maximiser, 4x the evaluations
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


def mo_lin_asy_ts(gps, anc_data):
  """ :19-41 """
  return _mo_ts(_lib.DFB_MOO_LIN_VAL, gps, anc_data)


def mo_tch_asy_ts(gps, anc_data):
  """ :44-68 """
  return _mo_ts(_lib.DFB_MOO_TCH_VAL, gps, anc_data)


asy = Namespace(lin_ts=mo_lin_asy_ts, tch_ts=mo_tch_asy_ts, lin_ucb=mo_lin_asy_ucb, tch_ucb=mo_tch_asy_ucb)
syn = Namespace()      # the reference has none either (:118-120)
seq = Namespace(lin_ts=mo_lin_asy_ts, tch_ts=mo_tch_asy_ts, lin_ucb=mo_lin_asy_ucb, tch_ucb=mo_tch_asy_ucb)
