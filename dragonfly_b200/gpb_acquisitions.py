"""
Drop-in for the acquisition operator table of dragonfly/opt/gpb_acquisitions.py (:443-471): the
`asy` / `syn` / `seq` Namespaces of fn(gp, anc_data) -> point, with the same anc_data fields
(gp_bandit.py:462-484), the same use of NumPy's global RNG for candidates and coin flips, and the
same return values -- but the objective evaluation AND the arg-max of `random_maximise`
(oper_utils.py:59-80) run as one fused device call (dfb_score_argmax) instead of
gp.eval(.., 'std') + scipy.stats + np.argmax on M x N / M x M host temporaries.

Scope: acq_opt_method == 'rand' on Euclidean domains, which is the vectorised branch of
maximise_acquisition (gpb_acquisitions.py:29-31).  The sequential one-point maximisers
(DIRECT / PDOO, :32-37) are host tree searches outside the hot path; when a Dragonfly install is
importable they are delegated to its own maximise_with_method with the device-backed gp.eval as
the objective, otherwise they raise.
"""
from argparse import Namespace
from contextlib import contextmanager
from copy import copy

import numpy as np

from .device import make_acq_desc
from .kernel import build_descriptor
from .domains import EuclideanDomain


# ---------------------------------------------------------------------------------------------
# Candidate generation: random_sample (oper_utils.py:59-67) + map_to_bounds (general_utils.py:25-27)
# ---------------------------------------------------------------------------------------------
def map_to_bounds(pts, bounds):
  bounds = np.asarray(bounds, dtype=np.float64)
  return pts * (bounds[:, 1] - bounds[:, 0]) + bounds[:, 0]


def draw_candidates(bounds, max_evals):
  """ rand_pts = map_to_bounds(np.random.random((int(max_evals), dim)), bounds) -- consumes the
      global MT19937 stream exactly like the reference, so seeded runs pick identical candidates. """
  dim = len(bounds)
  return map_to_bounds(np.random.random((int(max_evals), dim)), bounds)


def _check_rand_euclidean(anc_data):
  if anc_data.domain.get_type() != 'euclidean':
    raise NotImplementedError('Only Euclidean domains are on the GPU hot path.')
  return anc_data.acq_opt_method in ['rand']


# Multi-GPU (SURVEY.md 8e): when torch.distributed is initialised with more than one rank, every rank runs
# the same acquisition call in lock-step -- same seed, hence the same candidate matrix -- scores only its
# contiguous shard of the rows on its own GPU and joins with ONE 16-byte all-gather (dist.all_reduce_argmax).
# The recommendation is identical on every rank and to the single-process result, for any world size.
SHARD_ACROSS_RANKS = True


def _shard_info():
  """ (rank, world, device for the collective's 16-byte buffers) -- (0, 1, None) when not distributed. """
  if not SHARD_ACROSS_RANKS:
    return 0, 1, None
  import torch
  import torch.distributed as tdist
  if not (tdist.is_available() and tdist.is_initialized()) or tdist.get_world_size() < 2:
    return 0, 1, None
  dev = torch.device('cuda', torch.cuda.current_device()) if tdist.get_backend() == 'nccl' else None
  return tdist.get_rank(), tdist.get_world_size(), dev


def _sharded_argmax(scorer, n_rows, align=1):
  """ scorer(lo, hi) -> (best_score, best_index_within_the_slice) over global rows [lo, hi); returns the
      global arg-max index (np.argmax order).  `align` keeps shard boundaries on multiples of a block size. """
  rank, world, dev = _shard_info()
  if world == 1:
    return int(scorer(0, n_rows)[1])
  from . import dist as dfb_dist
  n_units = (n_rows + align - 1) // align
  u_lo, u_hi = dfb_dist.shard_bounds(n_units, rank, world)
  lo, hi = min(u_lo * align, n_rows), min(u_hi * align, n_rows)
  if hi > lo:
    best, idx = scorer(lo, hi)[:2]
    best, idx = float(best), int(idx) + lo
  else:
    best, idx = 0.0, -1
  _, gidx = dfb_dist.all_reduce_argmax(best, idx, device=dev)
  return int(gidx)


# Candidate source of the `rand` maximiser.
#   'numpy'  (default, parity mode): np.random.random((max_evals, d)) from the GLOBAL MT19937 stream, exactly the
#            rows the reference draws (oper_utils.py:59-67) -- every rank consumes the whole stream, in slabs, on a
#            producer thread that overlaps with the device scoring of the previous slab; a rank uploads and keeps only
#            the rows of its own shard.
#   'device' (throughput mode): a counter-based Philox4x32-10 stream keyed by (seed, GLOBAL row index, coordinate)
#            generated on the GPU (dfb_fill_candidates): no host RNG, no host->device copy, nothing proportional to
#            max_evals on the host, and a rank generates its own shard only; the seed is two draws from the global
#            NumPy stream, so seeded runs are reproducible and every rank agrees.  Different candidates than the
#            reference's, same distribution.  Select per call with anc_data.candidate_rng or module-wide here.
CANDIDATE_RNG = 'numpy'
STREAM_SLAB_ROWS = 1 << 18


_PINNED_SLABS = {}


def _pinned_slab_buffers(rows, dim, count=4):
  """ `count` page-locked (rows, dim) staging arrays (NumPy views of pinned torch tensors), cached: the slabs of the
      streamed draw are mapped to bounds straight into them, so the device call's host->device copies are real DMA
      instead of the driver's pageable staging.  None without CUDA (the CPU tests). """
  try:
    import torch
    if not torch.cuda.is_available():
      return None
  except Exception:  # pylint: disable=broad-except
    return None
  key = (int(rows), int(dim))
  if key not in _PINNED_SLABS:
    if len(_PINNED_SLABS) > 8:
      _PINNED_SLABS.clear()
    bufs = [torch.empty((key[0], key[1]), dtype=torch.float64, pin_memory=True) for _ in range(count)]
    _PINNED_SLABS[key] = (bufs, [b.numpy() for b in bufs])
  return _PINNED_SLABS[key][1]


def _slab_schedule(max_evals, slab, unit):
  """ Row ranges of the streamed draw: short slabs first -- 2 scoring chunks, then x4 per slab -- so that the device starts
      after ~0.5 ms of drawing and never waits for the producer (MT19937 draws a 6-column row in ~36 ns, the device scores
      one in ~160 ns at N = 5000: a slab four times the previous one is drawn while the previous one is scored), then
      full slabs. """
  starts, r0 = [], 0
  rows = 2 * unit
  while unit > 0 and rows < slab and r0 + rows < max_evals:
    starts.append((r0, rows)); r0 += rows
    rows *= 4
  while r0 < max_evals:
    rows = min(slab, max_evals - r0)
    starts.append((r0, rows)); r0 += rows
  return starts


def _maximise_streamed(score, bounds, max_evals, slab, unit=0):
  """ random_maximise (oper_utils.py:70-80) with the candidate draw pipelined against the scoring.
      score(pts) -> (best_score, best_index_within_pts, ...).  np.random.random((M, d)) and consecutive
      np.random.random((m_k, d)) slabs consume the MT19937 stream identically (row-major fill), so the candidates
      -- and the state the global RNG is left in -- are the reference's.  `unit` = rows of one scoring chunk. """
  import queue
  import threading
  from . import dist as dfb_dist
  M, dim = int(max_evals), len(bounds)
  rank, world, dev = _shard_info()
  lo_r, hi_r = dfb_dist.shard_bounds(M, rank, world) if world > 1 else (0, M)
  starts = _slab_schedule(M, slab, unit) if M > 0 else []
  q = queue.Queue(maxsize=2)
  bnds = np.asarray(bounds, dtype=np.float64)
  width, low = bnds[:, 1] - bnds[:, 0], bnds[:, 0]
  # staging buffers sized by the largest slab actually scheduled (never by the nominal slab size), and only while they
  # stay modest: 4 x 256 MB at most
  rows_max = max([r for _, r in starts] or [0])
  pinned = _pinned_slab_buffers(rows_max, dim) if (len(starts) > 1 and rows_max * dim * 8 <= (256 << 20)) else None

  def _producer():
    try:
      for k, (r0, rows) in enumerate(starts):
        raw = np.random.random((rows, dim))
        if not min(hi_r, r0 + rows) > max(lo_r, r0):
          q.put((r0, None))                            # another rank's rows: drawn (the stream must advance), not mapped
          continue
        if pinned is not None:
          pts = pinned[k % len(pinned)][:rows]
          np.multiply(raw, width, out=pts)             # map_to_bounds: pts * (hi - lo) + lo, written in place
          np.add(pts, low, out=pts)
        else:
          pts = raw * width + low
        q.put((r0, pts))
    except BaseException as exc:  # pylint: disable=broad-except
      q.put(exc)

  if len(starts) > 1:
    th = threading.Thread(target=_producer, daemon=True)
    th.start()
  else:
    th = None
    _producer()
  best_s, best_i, best_pt, err = 0.0, -1, None, None
  for _ in starts:
    item = q.get()
    if isinstance(item, BaseException):
      err = item
      break
    if err is not None:
      continue            # keep draining: the global RNG must end where the reference leaves it
    r0, pts = item
    if pts is None:
      continue
    a, b = max(lo_r, r0), min(hi_r, r0 + len(pts))
    if b <= a:
      continue
    try:
      res = score(pts[a - r0:b - r0])
    except BaseException as exc:  # pylint: disable=broad-except
      err = exc
      continue
    s, gi = float(res[0]), a + int(res[1])
    if dfb_dist.better(s, gi, best_s, best_i):
      best_s, best_i, best_pt = s, gi, np.array(pts[gi - r0], dtype=np.float64)
  if th is not None:
    th.join()
  if err is not None:
    raise err
  if world > 1:
    best_s, best_i, best_pt = dfb_dist.all_reduce_argmax_point(best_s, best_i, best_pt, dim, device=dev)
  return best_pt


def _maximise_device_candidates(session, bounds, max_evals):
  """ Throughput mode of the `rand` maximiser: candidates generated on the device by global row index. """
  from . import dist as dfb_dist
  M = int(max_evals)
  seed = (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))
  rank, world, dev = _shard_info()
  lo_r, hi_r = dfb_dist.shard_bounds(M, rank, world) if world > 1 else (0, M)
  slab = session.slab_rows(2 * STREAM_SLAB_ROWS)
  best_s, best_i, buf = 0.0, -1, None
  for r0 in range(lo_r, hi_r, slab):
    m = min(slab, hi_r - r0)
    if buf is None:
      buf = session.post.fill_candidates(seed, r0, m, bounds)
      pts = buf
    else:
      pts = session.post.fill_candidates(seed, r0, m, bounds, out=buf[:m])
    res = session.score(pts)
    s, gi = float(res[0]), r0 + int(res[1])
    if dfb_dist.better(s, gi, best_s, best_i):
      best_s, best_i = s, gi
  if world > 1:
    best_s, best_i = dfb_dist.all_reduce_argmax(best_s, best_i, device=dev)
  return session.post.fill_candidates(seed, int(best_i), 1, bounds).cpu().numpy()[0]


def _fused_maximise(scorer, anc_data, bounds=None, session=None):
  """ maximise_acquisition (:23-40) for the `rand` method: candidates scored slab by slab through fused device
      calls (per rank), the arg-max point returned.  `session` (a context-manager factory, GP._fused_session) binds
      hallucinations / test kernel once for all slabs; a plain `scorer(pts)` callable works too. """
  bounds = anc_data.domain.bounds if bounds is None else bounds
  mode = getattr(anc_data, 'candidate_rng', None) or CANDIDATE_RNG
  if session is None:
    if mode == 'device':
      raise NotImplementedError('device candidate generation needs a GP session')
    return _maximise_streamed(scorer, bounds, anc_data.max_evals, STREAM_SLAB_ROWS)
  with session() as sess:
    if mode == 'device':
      return _maximise_device_candidates(sess, bounds, anc_data.max_evals)
    if mode != 'numpy':
      raise ValueError("candidate_rng should be 'numpy' or 'device'.")
    return _maximise_streamed(sess.score, bounds, anc_data.max_evals, sess.slab_rows(STREAM_SLAB_ROWS),
                              unit=sess.slab_rows(1))


def _reference_fortran_direct_available():
  """ True when a Dragonfly install with its Fortran DIRECT extension is importable: only then does the
      reference's 'direct' differ from PDOO (oper_utils.py:23-31, 121-137). """
  try:
    from dragonfly.utils import oper_utils as ref_oper  # pylint: disable=import-error
  except Exception:  # pylint: disable=broad-except
    return False
  return getattr(ref_oper, 'direct_ft_wrap', None) is not None


def _delegate_to_reference_maximiser(acq_fn, anc_data, deterministic=True):
  """ The non-vectorised maximisers of maximise_acquisition (:29-37).  `acq_fn` takes a (k, d) array.
      'pdoo' -- and 'direct' wherever the reference itself would fall back to PDOO because its Fortran DIRECT is
      not built (oper_utils.py:121-137) -- run the batched PDOO of dragonfly_b200/doo.py: the same search as
      dragonfly/utils/doo.py with the two children of every split scored in one device call.  Fortran DIRECT
      itself stays the reference's (a sequential host code driving the device-backed objective point by point). """
  method = str(anc_data.acq_opt_method).lower()
  if method.startswith('pdoo') or (method.startswith('direct') and not _reference_fortran_direct_available()):
    from .doo import pdoo_maximise
    if deterministic:
      _, opt_pt, _ = pdoo_maximise(lambda X: acq_fn(np.asarray(X, dtype=np.float64)), anc_data.domain.bounds,
                                   anc_data.max_evals)
    else:       # a random objective (asy_rand): one call per evaluation, like the reference, nothing cached
      _, opt_pt, _ = pdoo_maximise(lambda x: acq_fn(np.asarray(x, dtype=np.float64).reshape((1, -1))),
                                   anc_data.domain.bounds, anc_data.max_evals, vectorised=False, deterministic=False)
    return opt_pt
  try:
    from dragonfly.exd.exd_utils import maximise_with_method  # pylint: disable=import-error
  except ImportError:
    raise NotImplementedError(
        "acq_opt_method '%s' is a sequential host maximiser outside the GPU hot path; 'rand', 'pdoo' and "
        "'direct' (as PDOO) are served without a Dragonfly install." % (anc_data.acq_opt_method))
  acquisition = lambda x: acq_fn(np.asarray(x).reshape((1, -1)))
  _, opt_pt = maximise_with_method(anc_data.acq_opt_method, acquisition, anc_data.domain,
                                   anc_data.max_evals)
  return opt_pt


# ---------------------------------------------------------------------------------------------
# Parallel strategy: hallucinated observations (:43-64)
# ---------------------------------------------------------------------------------------------
def _halluc_points(anc_data):
  if anc_data.handle_parallel == 'halluc' and len(anc_data.eval_points_in_progress) > 0:
    if getattr(anc_data, 'is_mf', False):
      return list(anc_data.eval_fidel_points_in_progress)
    return list(anc_data.eval_points_in_progress)
  return []


def _posterior_for(gp, anc_data):
  """ The device posterior the acquisition scores against: the GP's own, or the one augmented with
      the evaluations in progress (variance only; means from the un-augmented GP). """
  halluc = _halluc_points(anc_data)
  if len(halluc) == 0:
    return gp._device_posterior()
  return gp._device_posterior(halluc)


def _get_gp_eval_for_parallel_strategy(gp, anc_data, uncert_form='std'):
  """ :43-64 -- host-callable eval closure (used by TTEI's reference point and the delegated
      sequential maximisers). """
  halluc = _halluc_points(anc_data)
  if len(halluc) > 0:
    return lambda x: gp.eval_with_hallucinated_observations(x, halluc, uncert_form=uncert_form)
  return lambda x: gp.eval(x, uncert_form=uncert_form)


def _get_syn_recommendations_from_asy(asy_acq, num_workers, list_of_gps, anc_datas):
  """ Transcribed from the reference's :90-115 (host glue, kept as is) -- worker k sees the previous k-1 picks as
      hallucinations. """
  def _next(objs):
    ret = objs.pop(0)
    return ret, objs + [ret]
  if not hasattr(list_of_gps, '__iter__'):
    list_of_gps = [list_of_gps] * num_workers
  if not hasattr(anc_datas, '__iter__'):
    anc_datas = [anc_datas] * num_workers
  list_of_gps = [copy(gp) for gp in list_of_gps]
  anc_datas = [copy(ad) for ad in anc_datas]
  next_gp, list_of_gps = _next(list_of_gps)
  next_anc_data, anc_datas = _next(anc_datas)
  recommendations = [asy_acq(next_gp, next_anc_data)]
  for _ in range(1, num_workers):
    next_gp, list_of_gps = _next(list_of_gps)
    next_anc_data, anc_datas = _next(anc_datas)
    next_anc_data.eval_points_in_progress = recommendations
    recommendations.append(asy_acq(next_gp, next_anc_data))
  return recommendations


# ---------------------------------------------------------------------------------------------
# UCB (:202-227)
# ---------------------------------------------------------------------------------------------
def _get_gp_ucb_dim(gp):
  """ transcribed from the reference's :202-209 """
  if hasattr(gp, 'ucb_dim') and gp.ucb_dim is not None:
    return gp.ucb_dim
  elif hasattr(gp.kernel, 'dim'):
    return gp.kernel.dim
  return 3.0


def _get_ucb_beta_th(dim, time_step):
  """ transcribed from the reference's :211-213 """
  return np.sqrt(0.5 * dim * np.log(2 * dim * time_step + 1))


def asy_ucb(gp, anc_data):
  beta_th = _get_ucb_beta_th(_get_gp_ucb_dim(gp), anc_data.t)
  if _check_rand_euclidean(anc_data):
    acq = make_acq_desc('ucb', beta=beta_th)
    return _fused_maximise(None, anc_data, session=lambda: gp._fused_session(acq, _halluc_points(anc_data)))
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _ucb_acq(x):
    mu, sigma = gp_eval(x)
    return mu + beta_th * sigma
  return _delegate_to_reference_maximiser(_ucb_acq, anc_data)


def syn_ucb(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_ucb, num_workers, list_of_gps, anc_datas)


# ---------------------------------------------------------------------------------------------
# PI (:230-243), EI (:246-265), TTEI (:268-298)
# ---------------------------------------------------------------------------------------------
def asy_pi(gp, anc_data):
  curr_best = anc_data.curr_max_val
  if _check_rand_euclidean(anc_data):
    acq = make_acq_desc('pi', best=curr_best)
    return _fused_maximise(None, anc_data, session=lambda: gp._fused_session(acq, _halluc_points(anc_data)))
  from scipy.stats import norm as normal_distro
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _pi_acq(x):
    mu, sigma = gp_eval(x)
    return normal_distro.cdf((mu - curr_best) / sigma)
  return _delegate_to_reference_maximiser(_pi_acq, anc_data)


def syn_pi(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_pi, num_workers, list_of_gps, anc_datas)


def asy_ei(gp, anc_data):
  curr_best = anc_data.curr_max_val
  if _check_rand_euclidean(anc_data):
    acq = make_acq_desc('ei', best=curr_best)
    return _fused_maximise(None, anc_data, session=lambda: gp._fused_session(acq, _halluc_points(anc_data)))
  from scipy.stats import norm as normal_distro
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _ei_acq(x):
    mu, sigma = gp_eval(x)
    z = (mu - curr_best) / sigma
    return sigma * (z * normal_distro.cdf(z) + normal_distro.pdf(z))
  return _delegate_to_reference_maximiser(_ei_acq, anc_data)


def syn_ei(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_ei, num_workers, list_of_gps, anc_datas)


def _ttei(gp, anc_data, ref_point):
  """ :269-280 -- expected improvement over the reference arm. """
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  ref_mean, ref_std = gp_eval([ref_point])
  ref_mean = float(ref_mean[0])
  ref_std = float(ref_std[0])
  if _check_rand_euclidean(anc_data):
    acq = make_acq_desc('ttei', ref_mean=ref_mean, ref_std=ref_std)
    return _fused_maximise(None, anc_data, session=lambda: gp._fused_session(acq, _halluc_points(anc_data)))
  from scipy.stats import norm as normal_distro
  def _tt_ei_acq(x):
    mu, sigma = gp_eval(x)
    comb_std = np.sqrt(ref_std ** 2 + sigma ** 2)
    z = (mu - ref_mean) / comb_std
    return comb_std * (z * normal_distro.cdf(z) + normal_distro.pdf(z))
  return _delegate_to_reference_maximiser(_tt_ei_acq, anc_data)


def asy_ttei(gp, anc_data):
  """ :282-294 -- coin flip between the EI point and the best challenger of the EI point. """
  if np.random.random() < 0.5:
    return asy_ei(gp, anc_data)
  max_acq_opt_evals = anc_data.max_evals
  anc_data = copy(anc_data)
  anc_data.max_evals = max_acq_opt_evals // 2
  ei_argmax = asy_ei(gp, anc_data)
  return _ttei(gp, anc_data, ei_argmax)


def syn_ttei(num_workers, list_of_gps, anc_data):
  return _get_syn_recommendations_from_asy(asy_ttei, num_workers, list_of_gps, anc_data)


# ---------------------------------------------------------------------------------------------
# Add-UCB (:134-199)
# ---------------------------------------------------------------------------------------------
def _get_add_ucb_beta_th(dim, time_step):
  return np.sqrt(0.2 * dim * np.log(2 * dim * time_step + 1))


def _add_ucb(gp, add_kernel, mean_funcs, anc_data):
  """ :139-189.  Per group j the candidates live in the d_j-dimensional sub-box; K_*j =
      scale * k_j(X*_j, X[:, g_j]) is scored against the FULL additive GP's L and alpha. """
  if mean_funcs is not None:
    raise NotImplementedError('Add-UCB with per-group mean functions is not used by GPBandit '
                              '(asy_add_ucb passes None).')
  if not _check_rand_euclidean(anc_data):
    raise NotImplementedError("Add-UCB on device needs acq_opt_method == 'rand'.")
  kernel_list = add_kernel.kernel_list
  groupings = add_kernel.groupings
  total_max_evals = anc_data.max_evals
  domain_bounds = np.asarray(anc_data.domain_bounds)
  num_groups = len(kernel_list)
  group_points = []
  num_coordinates = 0
  anc_data.max_evals = total_max_evals // num_groups
  train_dim = gp._train_matrix().shape[1]
  for group_j, kernel_j in zip(groupings, kernel_list):
    betath_j = _get_add_ucb_beta_th(len(group_j), anc_data.t)
    desc_j = gp._group_test_descriptor(add_kernel, kernel_j, group_j, train_dim)
    acq = make_acq_desc('ucb', beta=betath_j)
    anc_data_j = copy(anc_data)
    anc_data_j.domain = EuclideanDomain(domain_bounds[group_j])
    point_j = _fused_maximise(None, anc_data_j, session=lambda _d=desc_j, _a=acq: gp._fused_session(
        _a, [], test_desc=_d, mean_const=0.0))
    group_points.append(point_j)
    num_coordinates += len(point_j)
  anc_data.max_evals = total_max_evals
  ret = np.zeros((num_coordinates,))
  for point_j, group_j in zip(group_points, groupings):
    ret[group_j] = point_j
  return ret


def asy_add_ucb(gp, anc_data):
  return _add_ucb(gp, gp.kernel, None, anc_data)


def syn_add_ucb(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_add_ucb, num_workers, list_of_gps, anc_datas)


# ---------------------------------------------------------------------------------------------
# Thompson sampling (:118-131)
# ---------------------------------------------------------------------------------------------
def asy_ts(gp, anc_data):
  """ :119-127 -- always the random maximiser with 4x the evaluations; the objective is one joint
      posterior draw over all candidates (gp.draw_samples(1, x)). """
  anc_data = copy(anc_data)
  if anc_data.acq_opt_method != 'rand':
    anc_data.acq_opt_method = 'rand'
    anc_data.max_evals = 4 * anc_data.max_evals
  halluc = _halluc_points(anc_data)
  rand_pts = draw_candidates(anc_data.domain.bounds, anc_data.max_evals)
  sample = _draw_one_sample(gp, rand_pts, halluc)
  return rand_pts[_argmax_of_sharded_sample(sample)]


def _ts_block(gp):
  post = getattr(gp, '_post', None) or getattr(getattr(gp, 'mfgp', None), '_post', None)
  return int(getattr(post, 'TS_BLOCK', 4096))


def _ts_cols(gp, n_rows):
  """ This rank's share [lo, hi) of the candidate rows, in whole TS blocks; None when not distributed. """
  rank, world, _ = _shard_info()
  if world == 1:
    return None
  from . import dist as dfb_dist
  blk = _ts_block(gp)
  b_lo, b_hi = dfb_dist.shard_bounds((n_rows + blk - 1) // blk, rank, world)
  return (min(b_lo * blk, n_rows), min(b_hi * blk, n_rows))


def _draw_one_sample(gp, rand_pts, halluc):
  """ One joint posterior draw over the candidates (gp_core.py:250-261).  Under torch.distributed each rank
      computes only its share of the independent 4096-candidate blocks (DESIGN.md 7) -- the normals are still
      drawn for ALL candidates so that every rank consumes the global RNG like the single-process run -- and
      the entries of the other ranks' blocks are -inf. """
  cols = _ts_cols(gp, len(rand_pts))
  kw = {} if cols is None else {'cols': cols}
  if len(halluc) > 0:
    return gp.draw_samples_with_hallucinated_observations(1, rand_pts, halluc, **kw).ravel()
  return gp.draw_samples(1, rand_pts, **kw).ravel()


def _argmax_of_sharded_sample(sample):
  """ np.argmax of a sample vector whose foreign-shard entries are -inf, joined across ranks. """
  rank, world, dev = _shard_info()
  idx = int(sample.argmax())
  if world == 1:
    return idx
  from . import dist as dfb_dist
  own = np.isfinite(sample) | np.isnan(sample) | (sample == np.inf)
  if not own.any():
    best, idx = 0.0, -1
  else:
    best = float(sample[idx])
  _, gidx = dfb_dist.all_reduce_argmax(best, idx, device=dev)
  return int(gidx)


def syn_ts(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_ts, num_workers, list_of_gps, anc_datas)


# ---------------------------------------------------------------------------------------------
# Random (:300-311)
# ---------------------------------------------------------------------------------------------
def asy_rand(_, anc_data):
  """ :301-307 -- the objective is np.random.random((1,)) whatever its argument.  With the `rand` maximiser the
      vectorised objective returns ONE uniform for the whole candidate matrix, so the arg-max is candidate 0;
      the sequential maximisers call it point by point (one uniform per evaluation), so they run as in the
      reference and consume the global RNG like it. """
  if not _check_rand_euclidean(anc_data):
    return _delegate_to_reference_maximiser(lambda x: np.random.random((1,)), anc_data, deterministic=False)
  rand_pts = draw_candidates(anc_data.domain.bounds, anc_data.max_evals)
  np.random.random((1,))
  return rand_pts[0]


def syn_rand(num_workers, list_of_gps, anc_data):
  return _get_syn_recommendations_from_asy(asy_rand, num_workers, list_of_gps, anc_data)


# ---------------------------------------------------------------------------------------------
# Multi-fidelity: the fidel_to_opt slice used by BOCA step 1 (:314-332)
# ---------------------------------------------------------------------------------------------
class _FidelToOptGP(object):
  """ Every candidate row gets the same fidelity prefix z = fidel_to_opt before it reaches the
      MF-GP (mfgp.eval_at_fidel([fidel_to_opt] * len(x), x)). """

  def __init__(self, mfgp, fidel_to_opt):
    self.mfgp = mfgp
    self.fidel_to_opt = np.asarray(fidel_to_opt, dtype=np.float64).reshape(-1)
    self.kernel = mfgp.get_domain_kernel()

  def _zx(self, x):
    x = np.asarray(x, dtype=np.float64)
    if x.ndim == 1:
      x = x.reshape(1, -1)
    return self.mfgp.get_ZX_matrix(np.repeat(self.fidel_to_opt.reshape(1, -1), len(x), axis=0), x)

  def eval(self, x, *args, **kwargs):
    return self.mfgp.eval(self._zx(x), *args, **kwargs)

  def eval_with_hallucinated_observations(self, x, halluc_fidel_pts, *args, **kwargs):
    return self.mfgp.eval_with_hallucinated_observations(self._zx(x), halluc_fidel_pts, *args,
                                                         **kwargs)

  def draw_samples(self, n, x, *args, **kwargs):
    return self.mfgp.draw_samples(n, self._zx(x), *args, **kwargs)

  def draw_samples_with_hallucinated_observations(self, n, x, halluc_fidel_pts, *args, **kwargs):
    return self.mfgp.draw_samples_with_hallucinated_observations(n, self._zx(x), halluc_fidel_pts,
                                                                 *args, **kwargs)

  def _zx_any(self, x):
    """ _zx for host rows or a CUDA tensor of rows (device-generated candidates). """
    try:
      import torch
    except ImportError:
      torch = None
    if torch is not None and isinstance(x, torch.Tensor):
      z = torch.as_tensor(self.fidel_to_opt, dtype=x.dtype, device=x.device).reshape(1, -1).expand(len(x), -1)
      ordering = np.argsort(list(self.mfgp.fidel_coords) + list(self.mfgp.domain_coords))
      return torch.cat((z, x), dim=1)[:, torch.as_tensor(ordering, device=x.device)].contiguous()
    return self._zx(x)

  def _fused_score(self, acq, pts, halluc, **kwargs):
    return self.mfgp._fused_score(acq, self._zx(pts), halluc, **kwargs)

  @contextmanager
  def _fused_session(self, acq, halluc=None, **kwargs):
    with self.mfgp._fused_session(acq, halluc, **kwargs) as sess:
      yield _PrefixedSession(sess, self._zx_any)


class _PrefixedSession(object):
  """ A GP._fused_session whose candidate rows get the fidel_to_opt prefix before they are scored. """

  def __init__(self, sess, prefix):
    self.sess, self.prefix, self.post = sess, prefix, sess.post

  def score(self, pts, want_scores=False):
    return self.sess.score(self.prefix(pts), want_scores=want_scores)

  def slab_rows(self, target):
    return self.sess.slab_rows(target)


def _get_fidel_to_opt_gp(mfgp, fidel_to_opt):
  return _FidelToOptGP(mfgp, fidel_to_opt)


def _add_ucb_for_boca(mfgp, fidel_to_opt, mean_funcs, anc_data):
  """ :334-388 -- Add-UCB on the z = fidel_to_opt slice of an MF-GP whose domain kernel is additive:
      K_*j = scale * k_F(Z_train, z) o k_j(X*_j, X[:, g_j]),  K**_j = scale * k_F(z, z) * k_j(X*_j, X*_j),
      scored against the MF-GP's full L and alpha. """
  if mean_funcs is not None:
    raise NotImplementedError('per-group mean functions are not used by GPBandit.')
  if not _check_rand_euclidean(anc_data):
    raise NotImplementedError("Add-UCB on device needs acq_opt_method == 'rand'.")
  from .kernel import CoordinateProductKernel
  domain_kernel_list = mfgp.domain_kernel.kernel_list
  groupings = mfgp.domain_kernel.groupings
  total_max_evals = anc_data.max_evals
  kern_scale = mfgp.kernel.hyperparams['scale']
  domain_bounds = np.asarray(anc_data.domain_bounds)
  num_groups = len(domain_kernel_list)
  f2o = np.asarray(fidel_to_opt, dtype=np.float64).reshape(-1)
  dz = len(f2o)
  train_dim = mfgp._train_matrix().shape[1]
  group_points = []
  num_coordinates = 0
  anc_data.max_evals = total_max_evals // num_groups
  for group_j, kernel_j in zip(groupings, domain_kernel_list):
    d_j = len(group_j)
    betath_j = _get_add_ucb_beta_th(d_j, anc_data.t)
    prod_j = CoordinateProductKernel(dz + d_j, kern_scale, [mfgp.fidel_kernel, kernel_j],
                                     [list(range(dz)), list(range(dz, dz + d_j))])
    train_coords = [mfgp.fidel_coords[i] for i in range(dz)] + \
                   [mfgp.domain_coords[int(g)] for g in group_j]
    desc_j = build_descriptor(prod_j, train_dim=train_dim, cand_dim=dz + d_j,
                              train_coords=train_coords, cand_coords=list(range(dz + d_j)))
    acq = make_acq_desc('ucb', beta=betath_j)
    anc_data_j = copy(anc_data)
    anc_data_j.domain = EuclideanDomain(domain_bounds[group_j])
    def scorer(pts, _d=desc_j, _a=acq):
      zx = np.concatenate((np.repeat(f2o.reshape(1, -1), len(pts), axis=0), pts), axis=1)
      return mfgp._fused_score(_a, zx, [], test_desc=_d, mean_const=0.0)
    point_j = _fused_maximise(scorer, anc_data_j)
    group_points.append(point_j)
    num_coordinates += len(point_j)
  anc_data.max_evals = total_max_evals
  ret = np.zeros((num_coordinates,))
  for point_j, group_j in zip(group_points, groupings):
    ret[group_j] = point_j
  return ret


def asy_add_ucb_for_boca(mfgp, fidel_to_opt, anc_data):
  return _add_ucb_for_boca(mfgp, fidel_to_opt, None, anc_data)


def boca(select_pt_func, mfgp, anc_data, func_caller):
  """ :399-439 -- BOCA: (1) pick x with an ordinary acquisition on the fidel_to_opt slice (the
      batched device path), (2) evaluate sigma at the candidate fidelities of that single x and
      threshold against cost ratio x information gap (tiny; host logic kept as in the reference). """
  if anc_data.curr_acq == 'add_ucb':
    next_eval_point = asy_add_ucb_for_boca(mfgp, func_caller.fidel_to_opt, anc_data)
  else:
    fidel_to_opt_gp = _get_fidel_to_opt_gp(mfgp, func_caller.fidel_to_opt)
    next_eval_point = select_pt_func(fidel_to_opt_gp, anc_data)
  candidate_fidels, cost_ratios = func_caller.get_candidate_fidels_and_cost_ratios(
      next_eval_point, filter_by_cost=True)
  num_candidates = len(candidate_fidels)
  cost_ratios = np.array(cost_ratios)
  sqrt_cost_ratios = np.sqrt(cost_ratios)
  information_gaps = np.array(func_caller.get_information_gap(candidate_fidels))
  _, cand_fidel_stds = mfgp.eval_at_fidel(candidate_fidels, [next_eval_point] * num_candidates,
                                          uncert_form='std')
  cand_fidel_stds = cand_fidel_stds / np.sqrt(mfgp.kernel.hyperparams['scale'])
  std_thresholds = anc_data.boca_thresh_coeff * anc_data.y_range * sqrt_cost_ratios * \
                   information_gaps
  qualifying_idxs = np.where(cand_fidel_stds > std_thresholds)[0]
  if len(qualifying_idxs) == 0:
    next_eval_fidel = func_caller.fidel_to_opt
  else:
    qualifying_fidels = [candidate_fidels[idx] for idx in qualifying_idxs]
    qualifying_sqrt_cost_ratios = sqrt_cost_ratios[qualifying_idxs]
    qualifying_cost_ratios = cost_ratios[qualifying_idxs]
    next_eval_fidel_idx = qualifying_sqrt_cost_ratios.argmin()
    if qualifying_cost_ratios[next_eval_fidel_idx] > anc_data.boca_max_low_fidel_cost_ratio:
      next_eval_fidel = func_caller.fidel_to_opt
    else:
      next_eval_fidel = qualifying_fidels[next_eval_fidel_idx]
  return next_eval_fidel, next_eval_point


# The operator tables looked up by name at gp_bandit.py:490,510,651,681 ---------------------------
syn = Namespace(ucb=syn_ucb, add_ucb=syn_add_ucb, ei=syn_ei, pi=syn_pi, ttei=syn_ttei, ts=syn_ts,
                rand=syn_rand)
asy = Namespace(ucb=asy_ucb, add_ucb=asy_add_ucb, ei=asy_ei, pi=asy_pi, ttei=asy_ttei, ts=asy_ts,
                rand=asy_rand)
seq = Namespace(ucb=asy_ucb, add_ucb=asy_add_ucb, ei=asy_ei, pi=asy_pi, ttei=asy_ttei, ts=asy_ts,
                rand=asy_rand)
