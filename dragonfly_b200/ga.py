"""
The `ga` acquisition maximiser of Cartesian-product domains (maximise_with_method_on_cp_domain, exd_utils.py:290-337),
restated without the experiment-design machinery the reference runs it through (CPGAOptimiser in a BlackboxOptimiser
with a one-worker SyntheticWorkerManager, cp_ga_optimiser.py, ga_optimiser.py, exd_core.py).

The search queries the same points in the same order and consumes the global MT19937 stream exactly as the reference
does, so seeded runs return the reference's point.  What changes is how the points are scored: the reference evaluates
one point per step, one device round trip each; here the initial pool is scored as one batch and every epoch's mutations
(five, the reference's num_mutations_per_epoch) as one batch.  That is exact because an epoch's mutations are all drawn
before the first of them is evaluated and nothing the search reads changes until they have been.

  initial pool  init_capital = clip(5 dim, max(5, 0.025 B), max(5, 0.075 B)) (exd_core.py:304-307) with capital_type
                'return_value': points are dispatched until the capital spent (one per evaluation) reaches it, i.e.
                ceil(init_capital) of them, drawn int(init_capital) at a time by get_cp_domain_initial_qinfos with
                latin_hc for Euclidean and integral parts (oper_utils.py:286-340).  The loop takes one point more
                from the pool than it dispatches, so a second pool is drawn whenever the first runs out: its first
                point is evaluated when init_capital is fractional, none of it when it is whole.
  epochs        GAOptimiser.generate_new_eval_points (ga_optimiser.py:70-132): parents by
                sample_according_to_exp_probs over every value so far (scaling_const 2, uniform when the probabilities
                are not finite, general_utils.py:366-385), each parent mutated part by part with the default operators
                (cp_ga_optimiser.py:27-121), the mutations shuffled and filtered by domain membership, retried with
                int(1.2 k + 1) mutations when none survive, ValueError after 51 tries.
  budget        the main loop runs while the capital spent is below B; it ends after ceil(B) + 1 evaluations in all
                (at least the pool); mutations left over when it ends are never evaluated.
  result        the first point with the largest value (BlackboxOptimiser keeps the best with a strict >).
Every evaluated point is asserted to be a member of the domain (experiment_caller.py:148), as in the reference.
"""
from argparse import Namespace
from copy import copy
from numbers import Number

import numpy as np

NUM_MUTATIONS_PER_EPOCH = 5
SCALING_CONST = 2.0
MAX_TRIES = 51


# ---------------------------------------------------------------------------------------------
# The initial pool: get_cp_domain_initial_qinfos with latin_hc (exd_utils.py:129-148, oper_utils.py:286-340)
# ---------------------------------------------------------------------------------------------
def latin_hc_indices(dim, num_samples):
  """ oper_utils.py:286-296: one np.random.randint(num_samples - i, size=dim) per row, each column a shrinking list. """
  index_set = [list(range(num_samples)) for _ in range(dim)]
  lhs_indices = []
  for i in range(num_samples):
    curr_idx_idx = np.random.randint(num_samples - i, size=dim)
    lhs_indices.append([index_set[j].pop(int(curr_idx_idx[j])) for j in range(dim)])
  return lhs_indices


def latin_hc_sampling(dim, num_samples):
  """ oper_utils.py:298-316: Latin hyper-cube sampling in the unit cube. """
  if num_samples == 0:
    return np.zeros((0, dim))
  elif num_samples == 1:
    return 0.5 * np.ones((1, dim))
  lower = np.linspace(0, 1, num_samples + 1)[:num_samples]
  width = lower[1] - lower[0]
  idx = np.array(latin_hc_indices(dim, num_samples), dtype=np.int64).reshape(num_samples, dim)
  return lower[idx] + width * np.random.random((num_samples, dim))


def draw_cp_initial_pool(parts, num_samples):
  """ sample_from_cp_domain_without_constraints (cp_domain_utils.py:448-489) with latin_hc for Euclidean and integral
      parts and one np.random.choice per point and coordinate for discrete parts (drawn as draw_cp_candidates does):
      the list of num_samples list-of-parts points, consuming the global MT19937 stream as the reference does. """
  from .gpb_acquisitions import map_to_bounds
  n = int(num_samples)
  cols = []
  for p in parts:
    if p.type in ('euclidean', 'integral'):
      vals = map_to_bounds(latin_hc_sampling(p.dim, n), p.bounds)
      cols.append([v.astype(int) for v in vals] if p.type == 'integral' else list(vals))
    else:
      n_levels = np.array([len(loi) for loi in p.levels], dtype=np.int64)
      idx = np.random.randint(0, np.broadcast_to(n_levels, (n, p.dim))) if n > 0 else np.zeros((0, p.dim), np.int64)
      arrs = [np.array(loi) for loi in p.levels]
      cols.append([[arrs[q][int(idx[i, q])] for q in range(p.dim)] for i in range(n)])
  return [[c[i] for c in cols] for i in range(n)]


def draw_constrained_pool(parts, domain, num_samples):
  """ get_cp_domain_initial_qinfos on a constrained domain (exd_utils.py:129-148): sample_from_cp_domain
      (cp_domain_utils.py:401-444) with latin_hc, i.e. at most 10 rounds of draw_cp_initial_pool -- max(10, 2n) points,
      then 2n -- each filtered by the domain's own constraints_are_satisfied, truncated to n once n are kept.  Fewer
      than n come back when ten rounds do not find them, as in the reference. """
  n = int(num_samples)
  ret, n_draw = [], max(10, 2 * n)
  for _ in range(10):
    ret.extend(pt for pt in draw_cp_initial_pool(parts, n_draw) if domain.constraints_are_satisfied(pt))
    if len(ret) >= n:
      return ret[:n]
    n_draw = 2 * n
  return ret


# ---------------------------------------------------------------------------------------------
# Domain membership (domains.py:90-131, 271-318, 418-428) and the mutation operators (cp_ga_optimiser.py:27-121)
# ---------------------------------------------------------------------------------------------
def _within_bounds(bounds, x):
  bounds = np.asarray(bounds)
  x = np.asarray(x)
  return bool(np.all(x >= bounds[:, 0]) and np.all(x <= bounds[:, 1]))


def _part_is_member(p, x):
  if p.type == 'euclidean':
    return _within_bounds(p.bounds, x)
  if p.type == 'integral':
    return all(isinstance(v, (int, np.int64)) for v in x) and _within_bounds(p.bounds, x)
  if not hasattr(x, '__iter__') or len(x) != p.dim:
    return False
  if p.type == 'prod_discrete':
    return all(v in loi for v, loi in zip(x, p.levels))
  return all(isinstance(v, Number) and any(abs(v - e) < 1e-8 for e in loi) for v, loi in zip(x, p.levels))


def is_a_member(parts, pt, domain=None):
  """ CartesianProductDomain.is_a_member (domains.py:418-428): every part's membership, then, for a constrained domain,
      the domain's own constraints_are_satisfied. """
  if not (hasattr(pt, '__iter__') and len(pt) == len(parts) and all(_part_is_member(p, x) for p, x in zip(parts, pt))):
    return False
  return domain is None or bool(domain.constraints_are_satisfied(pt))


def _gauss_perturbation(x, bounds):
  bounds = np.asarray(bounds)
  sigmas = [(b[1] - b[0]) / 10 for b in bounds]
  return np.clip(np.array(x) + np.random.normal(scale=sigmas), bounds[:, 0], bounds[:, 1])


def mutate_part(p, x):
  """ The default mutation operator of one part (get_default_mutation_op, cp_ga_optimiser.py:124-145). """
  if p.type == 'euclidean':
    return _gauss_perturbation(x, p.bounds)
  if p.type == 'integral':
    return _gauss_perturbation(x, p.bounds).round().astype(int)
  if p.type == 'prod_discrete':                       # prod_discrete_random_mutation
    ret = [copy(v) for v in x]
    change_idx = np.random.choice(len(x))
    change_list = copy(p.levels[change_idx])
    change_list.remove(x[change_idx])                 # ValueError for a value NumPy promoted ([1, 'a'] draws '1')
    ret[change_idx] = np.random.choice(change_list)   # ValueError for a coordinate with one level
    return ret
  ret = []                                            # prod_discrete_numeric_exp_mutation, uniform_prob 0.2
  for idx, loi in enumerate(p.levels):
    probs = np.exp(-np.abs(loi - x[idx]))
    probs = probs / probs.sum()
    ret.append(np.random.choice(loi, p=0.8 * probs + 0.2 * np.ones((len(probs),)) / float(len(probs))))
  return ret


def sample_parents(vals, num):
  """ sample_according_to_exp_probs(vals, num, replace=True, scaling_const=2, sample_uniformly_if_fail=True)
      (general_utils.py:366-385). """
  vals = np.asarray(vals, dtype=np.float64)
  probs = np.exp((vals - vals.mean()) / (SCALING_CONST * (vals.std() + 0.0001)))
  probs = probs / probs.sum()
  if not np.isfinite(probs.sum()):
    probs = np.ones((len(vals),)) / float(len(vals))
  return np.random.choice(len(vals), num, p=probs, replace=True)


def mutation_epoch(parts, points, vals, domain=None):
  """ GAOptimiser.generate_new_eval_points with CPGAOptimiser._mutation_op (ga_optimiser.py:97-132,
      cp_ga_optimiser.py:159-183): the new points to evaluate, in order.  domain: a constrained domain whose constraints
      filter the mutations too. """
  num_tries, k = 0, NUM_MUTATIONS_PER_EPOCH
  while True:
    num_tries += 1
    counts = np.bincount(sample_parents(vals, k), minlength=len(points))
    ret = []
    for idx in np.flatnonzero(counts):
      for _ in range(int(counts[idx])):
        ret.append([mutate_part(p, x) for p, x in zip(parts, points[idx])])
    np.random.shuffle(ret)
    members = [pt for pt in ret if (is_a_member(parts, pt) if domain is None else is_a_member(parts, pt, domain))]
    if members:
      return members
    if num_tries >= MAX_TRIES:
      raise ValueError(('Could not generate any points in domain from given mutation operator despite %d tries with '
                        'up to %d candidates. Quitting now.') % (num_tries, k))
    k = int(k * 1.2 + 1)


# ---------------------------------------------------------------------------------------------
# The search
# ---------------------------------------------------------------------------------------------
def init_capital(dim, max_evals):
  """ exd_core.py:304-307 """
  return np.clip(5 * dim, max(5.0, 0.025 * max_evals), max(5.0, 0.075 * max_evals))


def ga_budget(parts, max_evals):
  """ (init_capital, points in the initial pool, evaluations in all) of a search with budget max_evals. """
  cap = init_capital(sum(p.dim for p in parts), float(max_evals))
  n_pool = int(np.ceil(cap))
  return cap, n_pool, max(n_pool, int(np.ceil(float(max_evals))) + 1)


def ga_maximise(score, parts, max_evals, log=None, domain=None):
  """ The reference's CP GA with score(list of points) -> their values (one call per batch).  Returns (max_val,
      max_pt); log, when a list, receives (points, values) of every scored batch in order.  domain: a constrained
      domain -- the initial pool is its constrained draw and its constraints filter the mutations. """
  cap, n_pool, n_total = ga_budget(parts, max_evals)
  pool = []
  while len(pool) <= n_pool:           # the loop pops one point more than it dispatches, then sees the capital spent
    pool.extend(draw_cp_initial_pool(parts, int(cap)) if domain is None else
                draw_constrained_pool(parts, domain, int(cap)))
  pool = pool[:n_pool]
  points, vals = [], np.zeros((0,))

  def evaluate(batch):
    nonlocal vals
    for pt in batch:
      assert is_a_member(parts, pt) if domain is None else is_a_member(parts, pt, domain)
    v = np.asarray(score(batch), dtype=np.float64).reshape(-1)
    if log is not None:
      log.append((batch, v))
    points.extend(batch)
    vals = np.concatenate((vals, v))

  evaluate(pool)
  while len(points) < n_total:
    evaluate(mutation_epoch(parts, points, vals, domain)[:n_total - len(points)])
  ok = np.flatnonzero(vals == np.nanmax(vals)) if not np.all(np.isnan(vals)) else []
  if len(ok) == 0:
    return -np.inf, None
  return vals[ok[0]], points[ok[0]]


def ga_follow_up(score, parts, ga_val, ga_pt, method, max_evals):
  """ The `ga-<method>` follow-up (exd_utils.py:292-330): `method` over the Euclidean parts with the other parts fixed
      at the GA's point, kept when its value is larger.  'pdoo', and 'direct' without the reference's Fortran DIRECT,
      run the batched PDOO of doo.py; any other method (Fortran DIRECT, 'rand', ...) is the reference's own
      maximise_with_method_on_product_euclidean_spaces from a Dragonfly install, scoring one point per call. """
  from .doo import pdoo_maximise
  from .gpb_acquisitions import _reference_fortran_direct_available
  euc = [j for j, p in enumerate(parts) if p.type == 'euclidean']
  dims = [parts[j].dim for j in euc]
  starts = np.concatenate(([0], np.cumsum(dims))).astype(int)

  def swap(x):
    pt = list(ga_pt)
    for k, j in enumerate(euc):
      pt[j] = np.asarray(x)[starts[k]:starts[k + 1]]
    return pt
  if method == 'pdoo' or (method == 'direct' and not _reference_fortran_direct_available()):
    bounds = np.concatenate([np.asarray(parts[j].bounds, dtype=np.float64) for j in euc])
    euc_val, euc_pt, _ = pdoo_maximise(lambda X: score([swap(x) for x in np.asarray(X, dtype=np.float64)]), bounds,
                                       max_evals)
    euc_pt = swap(euc_pt)
  else:
    try:
      from dragonfly.exd.exd_utils import maximise_with_method_on_product_euclidean_spaces  # pylint: disable=import-error
    except ImportError:
      raise NotImplementedError("'ga-%s' on a Cartesian-product domain needs a Dragonfly install; 'ga-pdoo' runs "
                                "without one." % (method))
    doms = [Namespace(dim=parts[j].dim, bounds=parts[j].bounds) for j in euc]
    euc_val, euc_parts = maximise_with_method_on_product_euclidean_spaces(
        method, lambda xs: score([swap(np.concatenate([np.asarray(x, dtype=np.float64) for x in xs]))]), doms,
        max_evals)
    euc_pt = swap(np.concatenate([np.asarray(x, dtype=np.float64) for x in euc_parts]))
  if euc_val > ga_val:
    return euc_val, euc_pt
  return ga_val, ga_pt


def maximise(score, parts, method, max_evals, log=None, search=None, domain=None):
  """ maximise_with_method_on_cp_domain for method 'ga' or 'ga-<method>': returns the point.  log, domain: see
      ga_maximise.  search() -> (max_val, max_pt) replaces the parity GA (the device GA of device_search).  The
      follow-up over the Euclidean parts ignores the constraints, as the reference's does. """
  names = str(method).lower().split('-')
  if search is not None:
    val, pt = search()
  else:
    val, pt = ga_maximise(score, parts, max_evals, log) if domain is None else \
        ga_maximise(score, parts, max_evals, log, domain=domain)
  if len(names) == 2 and any(p.type == 'euclidean' for p in parts):
    val, pt = ga_follow_up(score, parts, val, pt, names[1], max_evals)
  return pt


# ---------------------------------------------------------------------------------------------
# Device mode (candidate_rng 'device'): the same search on the GPU, driven by Philox (dfb_ga_maximise)
# ---------------------------------------------------------------------------------------------
_PART_KINDS = {'euclidean': 0, 'integral': 1, 'prod_discrete': 2, 'prod_discrete_numeric': 3}   # DFB_GA_PART_*


def device_desc(parts):
  """ The dfb_ga_desc of the parts: the columns of dfb_fill_mixed_candidates, per categorical column its level ->
      column value table (and for prod_discrete_numeric parts the levels' numbers), the parts' column ranges. """
  from . import _lib
  from .gpb_acquisitions import _cp_device_layout
  kinds, bounds, n_levels, luts = _cp_device_layout(parts)
  if len(kinds) > _lib.DFB_GA_MAX_COLS or len(parts) > _lib.DFB_GA_MAX_PARTS:
    raise NotImplementedError('The device GA serves up to %d columns in %d parts.' % (_lib.DFB_GA_MAX_COLS,
                                                                                     _lib.DFB_GA_MAX_PARTS))
  g = _lib.GaDesc()
  g.d, g.n_parts = len(kinds), len(parts)
  lut, c = [], 0
  for j, p in enumerate(parts):
    g.part_kind[j], g.part_c0[j], g.part_c1[j] = _PART_KINDS[p.type], c, c + p.dim
    for q in range(p.dim):
      col = c + q
      g.kind[col] = kinds[col]
      g.lo[col], g.hi[col] = bounds[col]
      if luts[col] is None:
        continue
      if p.type == 'prod_discrete' and n_levels[col] < 2:
        raise ValueError("a cannot be empty unless no samples are taken: coordinate %d of a prod_discrete part has one "
                         "level, so no other level can be chosen." % (q))
      g.n_levels[col], g.lut_off[col] = n_levels[col], len(lut)
      lut.extend(float(v) for v in luts[col])
      if p.type == 'prod_discrete_numeric':
        g.val_off[col] = len(lut)
        lut.extend(float(v) for v in p.levels[q])
    c += p.dim
  if len(lut) > _lib.DFB_GA_MAX_LUT:
    raise NotImplementedError('The device GA holds up to %d category values.' % (_lib.DFB_GA_MAX_LUT))
  for k, v in enumerate(lut):
    g.lut[k] = v
  return g


def device_search(sess, parts, max_evals, seed):
  """ dfb_ga_maximise on the session's posterior and acquisition: returns (max_val, max_pt). """
  from .gpb_acquisitions import _cp_point_from_device_row
  _, n_pool, n_total = ga_budget(parts, max_evals)
  mean_const = sess._slab(sess.gp.X[:1])[1]
  val, idx, row, _, _ = sess.post.ga_maximise(sess.acq, mean_const, device_desc(parts), seed, n_pool, n_total)
  if idx < 0:
    return -np.inf, None
  return val, _cp_point_from_device_row(parts, row)
