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


def _is_cp_domain(anc_data):
  return anc_data.domain.get_type() == 'cartesian_product'


# ---------------------------------------------------------------------------------------------
# Cartesian-product domains (maximise_acquisition's CP branch, :35-37; exd_utils.py:219-289)
# ---------------------------------------------------------------------------------------------
_CP_NUMERIC = ('euclidean', 'integral')
_CP_DISCRETE = ('prod_discrete', 'prod_discrete_numeric')


class _CPPart(object):
  """ One part of a CP domain as candidate columns: its type, column count, bounds (numeric parts), the lists of levels
      (discrete parts) and, for a part under a Hamming factor, that factor's CategoryCodes table. """
  __slots__ = ('type', 'dim', 'bounds', 'levels', 'codes')


def _cp_parts(domain, kernel=None):
  """ The parts of a CP domain in domain order; raises for what the device does not serve (constraints it cannot read,
      NN and discrete-Euclidean parts, nested CP domains).  kernel None: the parts without Hamming tables (and without checking
      the GP's kernel against the domain). """
  from .kernel import category_codes, _kind_of
  from .constraints import readable
  if _has_constraints(domain) and not readable(domain):
    raise NotImplementedError('A constrained Cartesian-product domain needs its constraint list, raw name ordering, '
                              'get_raw_point and constraints_are_satisfied to be served on the GPU.')
  kernel_list = getattr(kernel, 'kernel_list', None) if kernel is not None else [None] * len(domain.list_of_domains)
  if kernel_list is None or len(kernel_list) != len(domain.list_of_domains):
    raise NotImplementedError('A Cartesian-product domain needs a CPGP whose kernel has one factor per part.')
  parts = []
  for dom, kern in zip(domain.list_of_domains, kernel_list):
    p = _CPPart()
    p.type = dom.get_type()
    p.bounds, p.levels, p.codes = None, None, None
    if p.type in _CP_NUMERIC:
      p.bounds = np.asarray(dom.bounds)
      p.dim = len(p.bounds)
    elif p.type in _CP_DISCRETE:
      p.levels = [list(loi) for loi in dom.list_of_list_of_items]
      p.dim = len(p.levels)
      if kern is None:
        pass
      elif _kind_of(kern) == 'HammingKernel':
        p.codes = category_codes(kern)
      elif p.type != 'prod_discrete_numeric':
        raise NotImplementedError('A prod_discrete part needs a HammingKernel factor.')
    else:
      raise NotImplementedError("Domain parts of type '%s' are outside the GPU hot-path scope." % (p.type))
    parts.append(p)
  return parts


def _has_constraints(domain):
  has_constraints = getattr(domain, 'has_constraints', None)
  return has_constraints is not None and bool(has_constraints())


def _level_columns(p, level_values):
  """ The candidate column values of one discrete coordinate's levels: Hamming codes, or the numeric values. """
  if p.codes is not None:
    return np.array([p.codes.encode(v) for v in level_values], dtype=np.float64)
  return np.asarray(level_values, dtype=np.float64)


def draw_cp_candidates(parts, max_evals):
  """ sample_from_cp_domain_without_constraints (cp_domain_utils.py:448-489) for M = max_evals points, part by part in
      domain order, consuming the global MT19937 stream exactly as the reference does:
        euclidean  map_to_bounds(np.random.random((M, d_j)), bounds)                    oper_utils.py:318-326
        integral   the same, then .astype(int)                                           oper_utils.py:337-340
        discrete   one np.random.choice(levels_q) per point and coordinate, point-major  oper_utils.py:342-360
      The last is drawn as ONE np.random.randint(0, n_q) over the (M, d_j) grid of level counts: the legacy generator
      draws a broadcast randint element by element in C order with the same bounded-integer routine as choice's scalar
      randint(0, n_q) (n_q = 1 draws nothing in both), so the stream advances identically.  The drawn value is
      np.array(levels_q)[idx] -- NumPy's promotion applies ([1, 'a'] draws '1') -- and that value is what gets encoded.
      Returns (rows, draws): the (M, sum d_j) float64 candidate matrix and per part what point_from_draws needs. """
  M = int(max_evals)
  cols, draws = [], []
  for p in parts:
    if p.type in _CP_NUMERIC:
      vals = map_to_bounds(np.random.random((M, p.dim)), p.bounds)
      if p.type == 'integral':
        vals = vals.astype(int)
      cols.append(np.asarray(vals, dtype=np.float64))
      draws.append(vals)
    else:
      n_levels = np.array([len(loi) for loi in p.levels], dtype=np.int64)
      idx = np.random.randint(0, np.broadcast_to(n_levels, (M, p.dim))) if M > 0 else np.zeros((0, p.dim), np.int64)
      c = np.empty((M, p.dim), dtype=np.float64)
      for q in range(p.dim):
        arr = np.array(p.levels[q])
        c[:, q] = _level_columns(p, [arr[k] for k in range(len(arr))])[idx[:, q]]
      cols.append(c)
      draws.append(idx)
  rows = np.ascontiguousarray(np.concatenate(cols, axis=1)) if cols else np.zeros((M, 0))
  return rows, draws


def point_from_draws(parts, draws, i):
  """ Point i of draw_cp_candidates in the reference's list-of-parts form: ndarray rows for Euclidean parts, int arrays
      for integral parts, lists of NumPy scalars (np.array(levels_q)[idx]) for discrete parts. """
  pt = []
  for p, d in zip(parts, draws):
    if p.type in _CP_NUMERIC:
      pt.append(d[i])
    else:
      pt.append([np.array(p.levels[q])[int(d[i, q])] for q in range(p.dim)])
  return pt


def _cp_device_layout(parts):
  """ Column kinds, bounds and level counts of dfb_fill_mixed_candidates for the parts, plus per discrete part the
      level -> column value tables (the device draws level indices). """
  from . import _lib
  kinds, bounds, n_levels, luts = [], [], [], []
  for p in parts:
    for q in range(p.dim):
      if p.type in _CP_NUMERIC:
        kinds.append(_lib.DFB_CAND_REAL if p.type == 'euclidean' else _lib.DFB_CAND_INTEGER)
        bounds.append([float(p.bounds[q][0]), float(p.bounds[q][1])])
        n_levels.append(0)
        luts.append(None)
      else:
        arr = np.array(p.levels[q])
        kinds.append(_lib.DFB_CAND_CATEGORICAL)
        bounds.append([0.0, 0.0])
        n_levels.append(len(arr))
        luts.append(_level_columns(p, [arr[k] for k in range(len(arr))]))
  return kinds, bounds, n_levels, luts


def _cp_device_rows(post, seed, r0, m, layout, out=None):
  """ Rows r0 .. r0+m-1 of the device-generated CP candidates, category columns mapped from level index to their column
      value (a Hamming code or the level's number) on the device. """
  kinds, bounds, n_levels, luts = layout
  return _encode_levels(post.fill_mixed_candidates(seed, r0, m, kinds, bounds, n_levels, out=out), luts)


def _encode_levels(pts, luts):
  """ Maps, in place, the category columns of a tensor of CP candidate rows from level index to column value: column c
      through luts[c] (_cp_device_layout), unless that is None or the identity. """
  import torch
  for c, lut in enumerate(luts):
    if lut is not None and not np.array_equal(lut, np.arange(len(lut), dtype=np.float64)):
      lut_d = torch.as_tensor(lut, device=pts.device)
      pts[:, c] = lut_d[pts[:, c].long()]
  return pts


def _cp_point_from_device_row(parts, row):
  """ The list-of-parts point of one row of dfb_fill_mixed_candidates (categorical columns as level indices). """
  pt, c = [], 0
  for p in parts:
    vals = row[c:c + p.dim]
    if p.type == 'euclidean':
      pt.append(np.array(vals, dtype=np.float64))
    elif p.type == 'integral':
      pt.append(np.array(vals).astype(int))
    else:
      pt.append([np.array(p.levels[q])[int(vals[q])] for q in range(p.dim)])
    c += p.dim
  return pt


def _cp_candidate_source(post, slab_rows, parts, M, mode, levels=False, domain=None):
  """ The M candidates of the `rand` maximiser on a CP domain as an _IndexedRows, and the seed of the device's candidates
      (None in 'numpy' mode).  'numpy' draws the reference's points (draw_cp_candidates) in host slabs of
      slab_rows(STREAM_SLAB_ROWS) rows; 'device' generates them with dfb_fill_mixed_candidates on `post`, keyed by (seed,
      global row, column), in slabs of slab_rows(2 STREAM_SLAB_ROWS).  levels: category columns hold level indices
      instead of the parts' column values (_encode_levels maps them).  A constrained domain's candidates are the rows
      its constraints keep (_constrained_source); their number, source.hi, may then differ from M. """
  if domain is not None and _has_constraints(domain):
    return _constrained_source(post, slab_rows, parts, M, mode, levels, domain)
  if mode == 'device':
    seed = _device_seed()
    kinds, bounds, n_levels, luts = _cp_device_layout(parts)
    layout = (kinds, bounds, n_levels, [None] * len(luts) if levels else luts)
    return _IndexedRows(
        slab_rows(2 * STREAM_SLAB_ROWS), 0, M, lambda r0, m, out: _cp_device_rows(post, seed, r0, m, layout, out),
        lambda i: _cp_point_from_device_row(
            parts, post.fill_mixed_candidates(seed, i, 1, kinds, bounds, n_levels).cpu().numpy()[0])), seed
  rows, draws = draw_cp_candidates(parts, M)
  if levels:
    rows = _level_rows(draws)
  return _IndexedRows(slab_rows(STREAM_SLAB_ROWS), 0, M, lambda r0, m, out: rows[r0:r0 + m],
                      lambda i: point_from_draws(parts, draws, i)), None


def _level_rows(draws):
  return np.ascontiguousarray(np.concatenate([np.asarray(d, dtype=np.float64) for d in draws], axis=1))


# ---------------------------------------------------------------------------------------------
# Constrained CP domains: the reference's constrained draw (cp_domain_utils.py:401-444) filtered on the device by the
# compiled constraints (constraints.py), undecided and residue rows settled on the host by the domain's own evaluator
# ---------------------------------------------------------------------------------------------
MAX_CONSTRAINED_TRIES = 10


def constrained_rand_draw(parts, M, keep_round):
  """ The candidates of _rand_maximise_vectorised_objective_in_cp_domain (exd_utils.py:247-274) on a constrained domain:
      calls of sample_from_cp_domain(domain, M) (cp_domain_utils.py:401-444) until M points are kept, or some are and
      five calls are spent -- so more than M may be kept.  A call draws at most 10 rounds, max(10, 2M) rows first and 2M
      after (draw_cp_candidates, the reference's MT19937 consumption), keeps each round's accepted rows in order and
      stops, truncated to M, once M are kept.  keep_round(rows, draws, need) -> (chunk, k) keeps the first k <= need
      accepted rows of a round.  Where the reference would draw forever because nothing is ever accepted, this warns
      as it does at the 10th empty call and raises ValueError.  Returns (chunks, number kept). """
  from warnings import warn
  chunks, total, tries = [], 0, 0
  while not (total >= M or (total > 0 and tries >= 5)):
    got = constrained_sample(parts, M, keep_round, chunks)
    total += got
    tries += 1
    if total == 0 and tries % MAX_CONSTRAINED_TRIES == 0:
      warn(('Sampling from domain failed despite %d attempts -- will continue trying but consider reparametrising '
            'your domain if this problem persists.') % (tries))
      raise ValueError('No point of the constrained domain was accepted in %d calls of %d draws.' % (tries, 20 * M))
  return chunks, total


def constrained_sample(parts, M, keep_round, chunks):
  """ One sample_from_cp_domain(domain, M) call of constrained_rand_draw: appends its kept chunks, returns their count. """
  got, n_draw = 0, max(10, 2 * M)
  for _ in range(10):
    rows, draws = draw_cp_candidates(parts, n_draw)
    chunk, k = keep_round(rows, draws, M - got)
    if k > 0:
      chunks.append(chunk)
    got += k
    if got >= M:
      break
    n_draw = 2 * M
  return got


def _constrained_source(post, slab_rows, parts, M, mode, levels, domain):
  """ _cp_candidate_source on a constrained domain.  'numpy': constrained_rand_draw, each round uploaded once, given a
      status per row by dfb_constraint_status, its undecided (and, with residue constraints, accepted) rows settled on
      the host through point_from_draws, and compacted on the device (dfb_compact_rows).  'device': the first M accepted
      rows of the device's candidate stream in row order, scanned block by block until M are found or the rows the
      reference's five calls could draw at most are spent; ValueError when none is accepted. """
  import torch
  from .constraints import compile_filter
  filt = compile_filter(domain, parts, levels=levels)
  prog = filt.desc()
  dev = post.device

  def status_of(rows_dev, point_of, need):
    """ The rows' statuses, the host's share settled in row order up to the first `need` accepted rows. """
    status, counts = post.constraint_status(prog, rows_dev)
    if counts[2] > 0 or (filt.residue and counts[1] > 0):
      status.copy_(torch.from_numpy(filt.settle(status.cpu().numpy(), point_of, need)))
    return status

  if mode == 'device':
    seed = _device_seed()
    kinds, bounds, n_levels, luts = _cp_device_layout(parts)
    block = slab_rows(2 * STREAM_SLAB_ROWS)
    cap = 5 * (max(10, 2 * M) + 9 * 2 * M)
    kept = torch.empty((M, len(kinds)), dtype=torch.float64, device=dev)
    kept_idx = torch.empty((M,), dtype=torch.int64, device=dev)
    got, r0, lv, coded = 0, 0, None, None
    while got < M and r0 < cap:
      m = min(block, cap - r0)
      lv = post.fill_mixed_candidates(seed, r0, m, kinds, bounds, n_levels, out=None if lv is None else lv[:m])
      rows = lv if levels else _encode_levels(torch.clone(lv) if coded is None else coded[:m].copy_(lv), luts)
      coded = None if levels else rows
      host_rows = {}

      def point_of(i, lv=lv):
        if not host_rows:              # the level rows the host may need, copied once per block
          st = status_now[0]
          idx = filt.host_rows(st)
          host_rows['idx'] = idx
          host_rows['rows'] = lv[torch.from_numpy(idx).to(dev)].cpu().numpy()
        k = int(np.searchsorted(host_rows['idx'], i))
        return _cp_point_from_device_row(parts, host_rows['rows'][k])
      status_now = [None]
      status, counts = post.constraint_status(prog, rows)
      if counts[2] > 0 or (filt.residue and counts[1] > 0):
        status_now[0] = status.cpu().numpy()
        status.copy_(torch.from_numpy(filt.settle(status_now[0], point_of, M - got)))
      rows_k, idx_k = post.compact_rows(rows, status, idx_base=r0)
      take = min(int(rows_k.shape[0]), M - got)
      kept[got:got + take] = rows_k[:take]
      kept_idx[got:got + take] = idx_k[:take]
      got += take
      r0 += m
    if got == 0:
      raise ValueError('No point of the constrained domain was accepted in %d device draws.' % (r0))
    return _IndexedRows(block, 0, got, lambda a, m, out: kept[a:a + m], lambda i: _cp_point_from_device_row(
        parts, post.fill_mixed_candidates(seed, int(kept_idx[i]), 1, kinds, bounds, n_levels).cpu().numpy()[0])), seed

  def keep_round(rows, draws, need):
    X = _level_rows(draws) if levels else rows
    rows_dev = torch.from_numpy(np.ascontiguousarray(X)).to(dev)
    status = status_of(rows_dev, lambda i: point_from_draws(parts, draws, i), need)
    rows_k, idx_k = post.compact_rows(rows_dev, status)
    k = min(int(rows_k.shape[0]), need)
    sel = idx_k[:k].cpu().numpy()
    return (rows_k[:k].clone(), [d[sel] for d in draws]), k

  chunks, total = constrained_rand_draw(parts, M, keep_round)
  kept = torch.cat([c[0] for c in chunks]) if len(chunks) > 1 else chunks[0][0]
  draws = [np.concatenate([c[1][j] for c in chunks]) for j in range(len(parts))]
  return _IndexedRows(slab_rows(STREAM_SLAB_ROWS), 0, total, lambda a, m, out: kept[a:a + m],
                      lambda i: point_from_draws(parts, draws, i)), None


def _cp_fused_maximise(gp, anc_data, acq):
  """ maximise_acquisition on a CP domain with acq_opt_method 'rand' (_rand_maximise_vectorised_objective_in_cp_domain,
      exd_utils.py:247-274): the reference scores its sampled points one gp.eval at a time; here every candidate is
      scored in fused device slabs and the arg-max follows np.argmax over the per-point values (first index on ties).
      candidate_rng 'numpy' draws the reference's points (draw_cp_candidates), 'device' draws them with
      dfb_fill_mixed_candidates keyed by (seed, global row, column).  acq None scores Thompson sampling's marginal draws
      instead (_cp_ts): with the normals drawn right after the reference's points, or the device's normals of the seed. """
  parts = _cp_parts(anc_data.domain, gp.kernel)
  if _shard_info()[1] > 1:
    raise NotImplementedError('Cartesian-product candidate draws are not sharded across ranks.')
  mode = _candidate_rng(anc_data)
  M = int(anc_data.max_evals)
  with gp._fused_session(acq, _halluc_points(anc_data)) as sess:
    source, seed = _cp_candidate_source(sess.post, sess.slab_rows, parts, M, mode, domain=anc_data.domain)
    if acq is not None:
      return source.point(*_slab_argmax(source, lambda pts, r0: sess.score(pts)))
    z = np.random.normal(size=source.hi) if mode == 'numpy' else None
    nonpos = 0

    def score_ts(pts, r0):
      nonlocal nonpos
      res = sess.score_ts(pts, seed=seed, row0=r0) if z is None else sess.score_ts(pts, z=z[r0:r0 + len(pts)])
      nonpos += int(res[3])
      return res
    best = _slab_argmax(source, score_ts)
    _check_nonpos(nonpos)
    return source.point(*best)


def _check_nonpos(nonpos):
  """ The reference's stable_cholesky raises for a 1 x 1 covariance that is not > 0 (general_utils.py:183-203). """
  if nonpos > 0:
    raise ValueError('Could not compute Cholesky decomposition despite adding jitter to the diagonal: the posterior '
                     'variance of %d candidate(s) is not positive. This is likely because the M is not positive '
                     'semi-definite or has infinities/nans.' % (nonpos))


def _cp_other_maximiser(acq_fn, anc_data, gp=None, acq=None):
  """ The non-'rand' maximisers on a CP domain.  'direct' / 'pdoo' on a domain of Euclidean parts only: PDOO over the
      flattened bounds, the point regrouped into parts (maximise_with_method_on_product_euclidean_spaces,
      exd_utils.py:219-244).  'ga' and 'ga-<method>' run the reference's GA restated in ga.py, each batch it allows
      scored in one call: with the device descriptor acq in one fused session on gp (evaluations in progress appended
      once), else with acq_fn.  acq_fn takes a list of list-of-parts points. """
  method = str(anc_data.acq_opt_method).lower()
  if method.startswith(('direct', 'pdoo')):
    doms = anc_data.domain.list_of_domains
    if any(d.get_type() != 'euclidean' for d in doms):
      raise NotImplementedError("'%s' on a Cartesian-product domain needs Euclidean parts only; use 'rand'." % (method))
    dims = [int(d.get_dim()) for d in doms]
    starts = np.concatenate(([0], np.cumsum(dims))).astype(int)
    regroup = lambda x: [np.asarray(x)[starts[j]:starts[j + 1]] for j in range(len(dims))]
    flat = copy(anc_data)
    flat.domain = EuclideanDomain(np.concatenate([np.asarray(d.bounds, dtype=np.float64) for d in doms]))
    flat_fn = lambda X: acq_fn([regroup(x) for x in np.asarray(X, dtype=np.float64)])
    return regroup(_delegate_to_reference_maximiser(flat_fn, flat))
  if method.startswith('ga'):
    from . import ga
    parts = _cp_parts(anc_data.domain, None if gp is None else gp.kernel)
    constrained = anc_data.domain if _has_constraints(anc_data.domain) else None
    cons_kw = {} if constrained is None else {'domain': constrained}
    if _shard_info()[1] > 1:
      raise NotImplementedError('The GA maximiser of Cartesian-product domains is not sharded across ranks.')
    if gp is None or acq is None:
      return ga.maximise(acq_fn, parts, method, anc_data.max_evals, **cons_kw)
    if constrained is not None and _candidate_rng(anc_data) == 'device':
      raise NotImplementedError("The device GA (candidate_rng='device') does not serve constrained Cartesian-product "
                                "domains; use candidate_rng='numpy' or acq_opt_method 'rand'.")
    seed = _device_seed() if _candidate_rng(anc_data) == 'device' else None
    with gp._fused_session(acq, _halluc_points(anc_data)) as sess:
      search = None if seed is None else (lambda: ga.device_search(sess, parts, anc_data.max_evals, seed))
      return ga.maximise(lambda pts: sess.score(pts, want_scores=True)[2], parts, method, anc_data.max_evals,
                         search=search, **cons_kw)
  raise NotImplementedError("acq_opt_method '%s' is not served on Cartesian-product domains; use 'rand'."
                            % (anc_data.acq_opt_method))


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


def _candidate_rng(anc_data):
  """ The candidate source of one `rand` maximisation: anc_data.candidate_rng, else CANDIDATE_RNG. """
  mode = getattr(anc_data, 'candidate_rng', None) or CANDIDATE_RNG
  if mode not in ('numpy', 'device'):
    raise ValueError("candidate_rng should be 'numpy' or 'device'.")
  return mode


def _device_seed():
  """ The seed of the device's candidates (and normals): two draws from the global NumPy stream. """
  return (int(np.random.randint(0, 2 ** 31 - 1)) << 31) | int(np.random.randint(0, 2 ** 31 - 1))


def _slab_argmax(source, score):
  """ random_maximise's arg-max (oper_utils.py:70-80) over a candidate source: score(pts, r0) -> (best_score,
      best_index_within_pts, ...) for every slab of this rank's rows, folded in np.argmax order (first index on ties,
      NaN counts as the maximum) and joined across the ranks the source is sharded over.  Returns (global index, row):
      the row is a copy of the winning host row when the source has row_dim set (slab buffers are reused; the row
      rides along the 16-byte join), else None and source.point regenerates it from the index.  When a score call
      raises, the source is closed -- the streamed draw still consumes the whole stream -- before the error propagates. """
  from . import dist as dfb_dist
  best_s, best_i, best_row = 0.0, -1, None
  slabs = source.slabs()
  try:
    for r0, pts in slabs:
      res = score(pts, r0)
      s, gi = float(res[0]), r0 + int(res[1])
      if dfb_dist.better(s, gi, best_s, best_i):
        best_s, best_i = s, gi
        if source.row_dim is not None:
          best_row = np.array(pts[gi - r0], dtype=np.float64)
  finally:
    slabs.close()
  _, world, dev = source.shard
  if world > 1 and source.row_dim is not None:
    best_s, best_i, best_row = dfb_dist.all_reduce_argmax_point(best_s, best_i, best_row, source.row_dim, device=dev)
  elif world > 1:
    best_s, best_i = dfb_dist.all_reduce_argmax(best_s, best_i, device=dev)
  return best_i, best_row


class _StreamedRows(object):
  """ Candidate source 'numpy' on a Euclidean domain, drawn slab by slab on a producer thread: np.random.random((M, d))
      and consecutive np.random.random((m_k, d)) slabs consume the MT19937 stream identically (row-major fill), so the
      candidates -- and the state the global RNG is left in -- are the reference's.  `unit` = rows of one scoring chunk. """

  def __init__(self, bounds, max_evals, slab, unit=0):
    self.bounds = np.asarray(bounds, dtype=np.float64)
    self.M, self.row_dim = int(max_evals), len(self.bounds)
    self.slab, self.unit = slab, unit
    self.shard = _shard_info()

  def slabs(self):
    import queue
    import threading
    from . import dist as dfb_dist
    M, dim = self.M, self.row_dim
    rank, world, _ = self.shard
    lo_r, hi_r = dfb_dist.shard_bounds(M, rank, world) if world > 1 else (0, M)
    starts = _slab_schedule(M, self.slab, self.unit) if M > 0 else []
    q = queue.Queue(maxsize=2)
    width, low = self.bounds[:, 1] - self.bounds[:, 0], self.bounds[:, 0]
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
    pending = len(starts)
    try:
      while pending:
        item = q.get()
        pending -= 1
        if isinstance(item, BaseException):
          pending = 0
          raise item
        r0, pts = item
        if pts is None:
          continue
        a, b = max(lo_r, r0), min(hi_r, r0 + len(pts))
        if b > a:
          yield a, pts[a - r0:b - r0]
    finally:
      while pending:        # closed early: keep draining, the global RNG must end where the reference leaves it
        pending -= 1
        if isinstance(q.get(), BaseException):
          break
      if th is not None:
        th.join()

  def point(self, i, row):
    return row


class _IndexedRows(object):
  """ Candidates addressed by global row index: rows lo .. hi-1 in slabs, fill(r0, m, out) returning rows r0 .. r0+m-1
      (device sources write them into out, the previous slab's buffer, when it is not None), point_of(i) the point of
      row i. """
  row_dim = None

  def __init__(self, slab, lo, hi, fill, point_of, shard=(0, 1, None)):
    self.slab, self.lo, self.hi, self.fill, self.point_of, self.shard = slab, lo, hi, fill, point_of, shard

  def slabs(self):
    buf = None
    for r0 in range(self.lo, self.hi, self.slab):
      m = min(self.slab, self.hi - r0)
      buf = self.fill(r0, m, None if buf is None else buf[:m])
      yield r0, buf

  def point(self, i, row):
    return self.point_of(int(i))


def _maximise_streamed(score, bounds, max_evals, slab, unit=0):
  """ random_maximise (oper_utils.py:70-80) over the streamed host draw (_StreamedRows): score(pts) -> (best_score,
      best_index_within_pts, ...) per slab; returns the arg-max point. """
  source = _StreamedRows(bounds, max_evals, slab, unit)
  return source.point(*_slab_argmax(source, lambda pts, r0: score(pts)))


def _fused_maximise(scorer, anc_data, session=None):
  """ maximise_acquisition (:23-40) for the `rand` method on a Euclidean domain: candidates scored slab by slab
      through fused device calls (per rank), the arg-max point returned.  `session` (a context-manager factory,
      GP._fused_session) binds hallucinations / test kernel once for all slabs; a plain `scorer(pts)` callable works
      too, on host candidates. """
  from . import dist as dfb_dist
  bounds, M = anc_data.domain.bounds, int(anc_data.max_evals)
  mode = _candidate_rng(anc_data)
  if session is None:
    if mode == 'device':
      raise NotImplementedError('device candidate generation needs a GP session')
    return _maximise_streamed(scorer, bounds, M, STREAM_SLAB_ROWS)
  with session() as sess:
    if mode == 'numpy':
      return _maximise_streamed(sess.score, bounds, M, sess.slab_rows(STREAM_SLAB_ROWS), unit=sess.slab_rows(1))
    seed = _device_seed()
    shard = _shard_info()
    lo, hi = dfb_dist.shard_bounds(M, shard[0], shard[1]) if shard[1] > 1 else (0, M)
    fill = lambda r0, m, out: sess.post.fill_candidates(seed, r0, m, bounds, out=out)
    source = _IndexedRows(sess.slab_rows(2 * STREAM_SLAB_ROWS), lo, hi, fill,
                          lambda i: fill(i, 1, None).cpu().numpy()[0], shard)
    return source.point(*_slab_argmax(source, lambda pts, r0: sess.score(pts)))


def _reference_fortran_direct_available():
  """ True when a Dragonfly install with its Fortran DIRECT extension is importable: only then does the
      reference's 'direct' differ from PDOO (oper_utils.py:23-31, 121-137). """
  try:
    from dragonfly.utils import oper_utils as ref_oper  # pylint: disable=import-error
  except Exception:  # pylint: disable=broad-except
    return False
  return getattr(ref_oper, 'direct_ft_wrap', None) is not None


def _uses_device_pdoo(anc_data):
  """ True when maximise_acquisition ends in PDOO: 'pdoo', or 'direct' without the reference's Fortran DIRECT
      (oper_utils.py:121-137). """
  method = str(anc_data.acq_opt_method).lower()
  return method.startswith('pdoo') or (method.startswith('direct') and not _reference_fortran_direct_available())


def _delegate_to_reference_maximiser(acq_fn, anc_data, deterministic=True):
  """ The non-vectorised maximisers of maximise_acquisition (:29-37).  `acq_fn` takes a (k, d) array.
      'pdoo' -- and 'direct' wherever the reference itself would fall back to PDOO because its Fortran DIRECT is
      not built (oper_utils.py:121-137) -- run the batched PDOO of dragonfly_b200/doo.py: the same search as
      dragonfly/utils/doo.py with the two children of every split scored in one device call.  Fortran DIRECT
      itself stays the reference's (a sequential host code driving the device-backed objective point by point). """
  if _uses_device_pdoo(anc_data):
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
  elif hasattr(gp.kernel, 'dim') and type(gp.kernel).__name__ != 'CartesianProductKernel':
    # the reference's CartesianProductKernel has no `dim` (kernel.py:504-518); ours carries one for the descriptor
    return gp.kernel.dim
  return 3.0


def _maximise_acq(gp, anc_data, acq, acq_fn):
  """ maximise_acquisition (:23-40) of the acquisitions below: the fused 'rand' maximiser (device descriptor acq) on
      Cartesian-product and Euclidean domains, else the other maximisers with the host objective acq_fn (on a CP
      domain it takes a list of list-of-parts points). """
  if _is_cp_domain(anc_data):
    if anc_data.acq_opt_method in ['rand']:
      return _cp_fused_maximise(gp, anc_data, acq)
    return _cp_other_maximiser(acq_fn, anc_data, gp, acq)
  if _check_rand_euclidean(anc_data):
    return _fused_maximise(None, anc_data, session=lambda: gp._fused_session(acq, _halluc_points(anc_data)))
  return _delegate_to_reference_maximiser(acq_fn, anc_data)


def _get_ucb_beta_th(dim, time_step):
  """ transcribed from the reference's :211-213 """
  return np.sqrt(0.5 * dim * np.log(2 * dim * time_step + 1))


def asy_ucb(gp, anc_data):
  beta_th = _get_ucb_beta_th(_get_gp_ucb_dim(gp), anc_data.t)
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _ucb_acq(x):
    mu, sigma = gp_eval(x)
    return mu + beta_th * sigma
  return _maximise_acq(gp, anc_data, make_acq_desc('ucb', beta=beta_th), _ucb_acq)


def syn_ucb(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_ucb, num_workers, list_of_gps, anc_datas)


# ---------------------------------------------------------------------------------------------
# PI (:230-243), EI (:246-265), TTEI (:268-298)
# ---------------------------------------------------------------------------------------------
def asy_pi(gp, anc_data):
  curr_best = anc_data.curr_max_val
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _pi_acq(x):
    from scipy.stats import norm as normal_distro
    mu, sigma = gp_eval(x)
    return normal_distro.cdf((mu - curr_best) / sigma)
  return _maximise_acq(gp, anc_data, make_acq_desc('pi', best=curr_best), _pi_acq)


def syn_pi(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_pi, num_workers, list_of_gps, anc_datas)


def asy_ei(gp, anc_data):
  curr_best = anc_data.curr_max_val
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  def _ei_acq(x):
    from scipy.stats import norm as normal_distro
    mu, sigma = gp_eval(x)
    z = (mu - curr_best) / sigma
    return sigma * (z * normal_distro.cdf(z) + normal_distro.pdf(z))
  return _maximise_acq(gp, anc_data, make_acq_desc('ei', best=curr_best), _ei_acq)


def syn_ei(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_ei, num_workers, list_of_gps, anc_datas)


def _ttei(gp, anc_data, ref_point):
  """ :269-280 -- expected improvement over the reference arm. """
  gp_eval = _get_gp_eval_for_parallel_strategy(gp, anc_data, 'std')
  ref_mean, ref_std = gp_eval([ref_point])
  ref_mean = float(ref_mean[0])
  ref_std = float(ref_std[0])
  def _tt_ei_acq(x):
    from scipy.stats import norm as normal_distro
    mu, sigma = gp_eval(x)
    comb_std = np.sqrt(ref_std ** 2 + sigma ** 2)
    z = (mu - ref_mean) / comb_std
    return comb_std * (z * normal_distro.cdf(z) + normal_distro.pdf(z))
  return _maximise_acq(gp, anc_data, make_acq_desc('ttei', ref_mean=ref_mean, ref_std=ref_std), _tt_ei_acq)


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


def _add_ucb_groups(anc_data, groupings, maximise_group, score_groups):
  """ The group loop of Add-UCB (:139-189, :334-388): group j's UCB, with the beta of its d_j coordinates, is maximised
      over the d_j-dimensional sub-box with max_evals // (number of groups) evaluations, and the group points are put back
      into one point.  'rand': maximise_group(j, acq_desc, anc_data_j) -> point_j, group by group.  PDOO: one search per
      group, all driven in lock-step so that each round's points of every group are scored in one
      score_groups([(j, X_j), ...], betas) -> [values_j, ...] call.  Other methods (Fortran DIRECT): the reference's
      maximiser per group on the one-point objective score_groups([(j, x)], betas). """
  rand = _check_rand_euclidean(anc_data)
  domain_bounds = np.asarray(anc_data.domain_bounds)
  betas = [_get_add_ucb_beta_th(len(group_j), anc_data.t) for group_j in groupings]
  anc_datas = []
  for group_j in groupings:
    anc_data_j = copy(anc_data)
    anc_data_j.max_evals = anc_data.max_evals // len(groupings)
    anc_data_j.domain = EuclideanDomain(domain_bounds[group_j])
    anc_datas.append(anc_data_j)
  if rand:
    group_points = [maximise_group(j, make_acq_desc('ucb', beta=betas[j]), anc_data_j)
                    for j, anc_data_j in enumerate(anc_datas)]
  elif _uses_device_pdoo(anc_data):
    from .doo import pdoo_maximise_lockstep
    found = pdoo_maximise_lockstep(lambda requests: score_groups(requests, betas),
                                   [domain_bounds[group_j] for group_j in groupings], anc_datas[0].max_evals)
    group_points = [pt for _, pt in found]
  else:
    group_points = [_delegate_to_reference_maximiser(
        lambda X, j=j: score_groups([(j, np.asarray(X, dtype=np.float64))], betas)[0], anc_data_j)
                    for j, anc_data_j in enumerate(anc_datas)]
  ret = np.zeros((sum(len(point_j) for point_j in group_points),))
  for point_j, group_j in zip(group_points, groupings):
    ret[group_j] = point_j
  return ret


def _group_calls(descs, groups):
  """ The groups of one round split into dfb_score_groups calls, in order: each call holds at most DFB_MAX_GROUPS
      groups whose descriptors together use at most DFB_MAX_SLOTS slots and DFB_MAX_FACTORS factors. """
  from . import _lib
  calls, cur, slots, factors = [], [], 0, 0
  for j in groups:
    s, f = int(descs[j].n_slots), int(descs[j].n_factors)
    if cur and (len(cur) == _lib.DFB_MAX_GROUPS or slots + s > _lib.DFB_MAX_SLOTS or
                factors + f > _lib.DFB_MAX_FACTORS):
      calls.append(cur)
      cur, slots, factors = [], 0, 0
    cur.append(j)
    slots, factors = slots + s, factors + f
  if cur:
    calls.append(cur)
  return calls


def _group_scorer(post, descs, prefix=None):
  """ score_groups of _add_ucb_groups on a device posterior: the rows of all requests -- each group's points, after
      `prefix` (a fixed leading block of coordinates) when given -- in dfb_score_groups calls that pass only the groups
      of the round (one call unless they exceed the entry's limits on groups, slots and factors, _group_calls). """
  def score_one_call(requests, betas):
    rows = [np.asarray(X, dtype=np.float64).reshape(len(X), -1) for _, X in requests]
    if prefix is not None:
      rows = [np.concatenate((np.repeat(prefix.reshape(1, -1), len(R), axis=0), R), axis=1) for R in rows]
    present = list(dict.fromkeys(j for j, _ in requests))
    local = {j: k for k, j in enumerate(present)}
    X = np.zeros((sum(len(R) for R in rows), max(R.shape[1] for R in rows)))
    groups = np.empty((len(X),), dtype=np.int32)
    r0, bounds = 0, []
    for (j, _), R in zip(requests, rows):
      X[r0:r0 + len(R), :R.shape[1]] = R
      groups[r0:r0 + len(R)] = local[j]
      bounds.append((r0, r0 + len(R)))
      r0 += len(R)
    scores = post.score_groups([descs[j] for j in present], [betas[j] for j in present], X, groups)
    return [scores[a:b] for a, b in bounds]

  def score_groups(requests, betas):
    out = {}
    for call in _group_calls(descs, list(dict.fromkeys(j for j, _ in requests))):
      members = set(call)
      part = [(k, r) for k, r in enumerate(requests) if r[0] in members]
      for (k, _), vals in zip(part, score_one_call([r for _, r in part], betas)):
        out[k] = vals
    return [out[k] for k in range(len(requests))]
  return score_groups


def _add_ucb(gp, add_kernel, mean_funcs, anc_data):
  """ :139-189.  Per group j the candidates live in the d_j-dimensional sub-box; K_*j =
      scale * k_j(X*_j, X[:, g_j]) is scored against the FULL additive GP's L and alpha. """
  if mean_funcs is not None:
    raise NotImplementedError('Add-UCB with per-group mean functions is not used by GPBandit '
                              '(asy_add_ucb passes None).')
  groupings = add_kernel.groupings
  train_dim = gp._train_matrix().shape[1]
  descs = [gp._group_test_descriptor(add_kernel, add_kernel.kernel_list[j], groupings[j], train_dim)
           for j in range(len(groupings))]

  def maximise_group(j, acq, anc_data_j):
    return _fused_maximise(None, anc_data_j, session=lambda: gp._fused_session(acq, [], test_desc=descs[j],
                                                                               mean_const=0.0))

  return _add_ucb_groups(anc_data, groupings, maximise_group, _group_scorer(gp._device_posterior(), descs))


def asy_add_ucb(gp, anc_data):
  return _add_ucb(gp, gp.kernel, None, anc_data)


def syn_add_ucb(num_workers, list_of_gps, anc_datas):
  return _get_syn_recommendations_from_asy(asy_add_ucb, num_workers, list_of_gps, anc_datas)


# ---------------------------------------------------------------------------------------------
# Thompson sampling (:118-131)
# ---------------------------------------------------------------------------------------------
def _ts_anc_data(anc_data):
  """ :119-124 -- a copy of anc_data for Thompson sampling, which always runs the random maximiser: with 4x the
      evaluations when another maximiser was asked for. """
  anc_data = copy(anc_data)
  if anc_data.acq_opt_method != 'rand':
    anc_data.acq_opt_method = 'rand'
    anc_data.max_evals = 4 * anc_data.max_evals
  return anc_data


def asy_ts(gp, anc_data):
  """ :119-127 -- always the random maximiser with 4x the evaluations; the objective is one joint
      posterior draw over all candidates (gp.draw_samples(1, x)). """
  anc_data = _ts_anc_data(anc_data)
  if _is_cp_domain(anc_data):
    return _cp_ts(gp, anc_data)
  halluc = _halluc_points(anc_data)
  rand_pts = draw_candidates(anc_data.domain.bounds, anc_data.max_evals)
  sample = _draw_one_sample(gp, rand_pts, halluc)
  return rand_pts[_argmax_of_sharded_sample(sample)]


def _cp_ts(gp, anc_data):
  """ asy_ts on a CP domain (anc_data already forced to 'rand').  The reference's vectorised objective is called one
      point at a time there (exd_utils.py:247-274), so each candidate gets its own 1 x 1 draw: sqrt(sigma^2) z + mu with
      one np.random.normal(size=(1, 1)) per candidate, in candidate order (gp_core.py:250-261, general_utils.py:224-232).
      Legacy NumPy draws normals in pairs and caches the second, so np.random.normal(size=M) after the candidates gives
      the same M normals and leaves the stream where the M one-normal calls leave it.  Every candidate is scored in
      fused device slabs (dfb_score_argmax_ts) and the arg-max follows np.argmax.  candidate_rng 'device' generates the
      rows (dfb_fill_mixed_candidates) and the normals (in the scoring kernel) from one seed.  A candidate whose variance
      is not > 0 raises ValueError, as the reference's stable_cholesky does. """
  if getattr(anc_data, 'is_mf', False) or hasattr(gp, 'fidel_space_kernel') or hasattr(gp, 'mfgp'):
    raise NotImplementedError('Thompson sampling with a multi-fidelity GP on a Cartesian-product domain is outside the '
                              'GPU hot-path scope.')
  return _cp_fused_maximise(gp, anc_data, None)


def _ts_limits(gp):
  """ (TS_BLOCK, TS_JOINT_MAX) of the GP's device posterior. """
  post = getattr(gp, '_post', None) or getattr(getattr(gp, 'mfgp', None), '_post', None)
  return int(getattr(post, 'TS_BLOCK', 4096)), int(getattr(post, 'TS_JOINT_MAX', 16384))


def _ts_cols(gp, n_rows):
  """ This rank's share [lo, hi) of the candidate rows, in whole TS blocks; None when not distributed, and when
      the candidates take one joint draw (TS_BLOCK < n_rows <= TS_JOINT_MAX): every rank then computes the whole
      draw. """
  rank, world, _ = _shard_info()
  if world == 1:
    return None
  blk, joint_max = _ts_limits(gp)
  if blk < n_rows <= joint_max:
    return None
  from . import dist as dfb_dist
  b_lo, b_hi = dfb_dist.shard_bounds((n_rows + blk - 1) // blk, rank, world)
  return (min(b_lo * blk, n_rows), min(b_hi * blk, n_rows))


def _draw_one_sample(gp, rand_pts, halluc):
  """ One joint posterior draw over the candidates (gp_core.py:250-261).  Up to TS_JOINT_MAX candidates every rank
      computes the whole joint draw.  Above it, under torch.distributed, each rank computes only its share of the
      independent 4096-candidate blocks (DESIGN.md 7) -- the normals are still drawn for ALL candidates so that every
      rank consumes the global RNG like the single-process run -- and the entries of the other ranks' blocks are
      -inf. """
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
  from .kernel import CoordinateProductKernel
  groupings = mfgp.domain_kernel.groupings
  kern_scale = mfgp.kernel.hyperparams['scale']
  f2o = np.asarray(fidel_to_opt, dtype=np.float64).reshape(-1)
  dz = len(f2o)
  train_dim = mfgp._train_matrix().shape[1]
  descs = []
  for j, group_j in enumerate(groupings):
    d_j = len(group_j)
    prod_j = CoordinateProductKernel(dz + d_j, kern_scale, [mfgp.fidel_kernel, mfgp.domain_kernel.kernel_list[j]],
                                     [list(range(dz)), list(range(dz, dz + d_j))])
    train_coords = [mfgp.fidel_coords[i] for i in range(dz)] + \
                   [mfgp.domain_coords[int(g)] for g in group_j]
    descs.append(build_descriptor(prod_j, train_dim=train_dim, cand_dim=dz + d_j,
                                  train_coords=train_coords, cand_coords=list(range(dz + d_j))))

  def maximise_group(j, acq, anc_data_j):
    def scorer(pts):
      zx = np.concatenate((np.repeat(f2o.reshape(1, -1), len(pts), axis=0), pts), axis=1)
      return mfgp._fused_score(acq, zx, [], test_desc=descs[j], mean_const=0.0)
    return _fused_maximise(scorer, anc_data_j)

  return _add_ucb_groups(anc_data, groupings, maximise_group,
                         _group_scorer(mfgp._device_posterior(), descs, prefix=f2o))


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
