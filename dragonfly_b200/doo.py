"""
Parallel deterministic optimistic optimisation (PDOO) of an acquisition, with the children of every split scored
in ONE batched call -- SURVEY.md 8f rank 4.

What it replaces: dragonfly/utils/doo.py (OptTree.run_PDOO / run_DOO / split_children / querie, pdoo_wrap) as
driven by pdoo_maximise (dragonfly/utils/oper_utils.py:257-271: K = 2, tol = 1e-3, nu_max = 1, C_init = 0.8,
rho_max = 0.9, POO_mult = 0.5) -- the maximiser the reference ends up in for acq_opt_method 'pdoo', and for the
default 'direct' whenever its Fortran DIRECT extension is not built (oper_utils.py:121-137).  The reference
evaluates the acquisition one point per Python call (gpb_acquisitions.py:33-37, doo.py:117-125); here the K
children of the splits of ALL N passes of a round go to the device together (a speculative lock-step prefetch,
see PDOOSearch; GP.eval's row-streaming path serves up to 32 points), which is the only change: the search itself -- cell geometry, optimistic bounds, fidelity bookkeeping, evaluation cache,
priority order, budget accounting, the final selection -- is restated so that, for the same objective values, it
visits the same cells in the same order and returns the same point (tests/test_host_logic.py pins it on the
reference's own runs, tests/golden/pdoo.npz).

The objective here never depends on the "fidelity" z (cost 1 per evaluation), but z still decides when a cached
cell is re-evaluated (|z_old - z| > tol) and enters the bounds, so it is carried exactly as in the reference.
"""
import heapq

import numpy as np


class _Leaf(object):
  """ A cell with its value and optimistic bound; ordered for heapq so that the LARGEST bound pops first and
      equal bounds compare equal (doo.py:84-91). """
  __slots__ = ('cell', 'value', 'fidelity', 'bound', 'height', 'split_dim')

  def __init__(self, cell, value, fidelity, bound, height, split_dim):
    self.cell, self.value, self.fidelity = cell, value, fidelity
    self.bound, self.height, self.split_dim = bound, height, split_dim

  def __lt__(self, other):
    return other.bound < self.bound

  def __eq__(self, other):
    return other.bound == self.bound


class _PassState(object):
  """ What a DOO pass reads and writes besides its own heap: the evaluation cache, the smoothness constant C and whether
      evaluations are recorded.  The exact run shares one state over all passes (as the reference's OptTree does); the
      speculative prefetch gives every pass a private one. """

  def __init__(self, C, record):
    self.cache, self.C, self.record = {}, C, record


class PDOOSearch(object):
  """ One PDOO run over the unit cube; `batch_obj(P)` maps an (k, d) array of NORMALISED points to k values.

      Batching (SURVEY 8f rank 4).  The search is written as generators that YIELD the cells whose objective value they
      need and receive the values back, so the same code runs in two ways:
        * exact run: the N DOO passes one after the other on a shared cache, as the reference does;
        * speculative prefetch (first): the N passes advance in LOCK-STEP, each on a private cache, and the children of
          the splits of ALL passes of a round go to the device in one call (N x K points instead of K).  It only fills a
          value table keyed by cell -- the objective is a deterministic function of the cell midpoint -- from which the
          exact run is then served; what the prefetch did not foresee (the shared cache changes a pass's budget slightly)
          is evaluated on demand.  The search therefore visits exactly the cells of the one-point-per-call reference, in
          the same order, with ~N times fewer device calls. """

  PREFETCH_GROUP = 32          # points per device call of the prefetch (dfb_eval's row-streaming path serves <= 32)

  def __init__(self, batch_obj, dim, total_budget, nu_max=1.0, rho_max=0.9, K=2, C_init=0.8, tol=1e-3, prefetch=True,
               deterministic=True):
    self.batch_obj, self.dim = batch_obj, dim
    self.deterministic = deterministic      # False (e.g. asy_rand's random objective): every evaluation is a fresh call
    prefetch = prefetch and deterministic
    self.total_budget, self.nu_max, self.rho_max, self.K = total_budget, nu_max, rho_max, K
    self.tol, self.prefetch = tol, prefetch
    self.state = _PassState(C_init, True)
    self.values = {}                 # cell -> objective value at its midpoint (filled by both phases)
    self.query_pts, self.query_vals = [], []
    self.num_device_calls = 0
    self.num_prefetched = 0

  @property
  def C(self):
    return self.state.C

  @property
  def cache(self):
    return self.state.cache

  # -- objective values of a group of cells: value table first, the rest in batched calls ---------------------------------
  def _fetch(self, cells, group=None):
    """ The values of `cells`: yields the cells missing from the value table, `group` at a time (all at once when None),
        receives their values and files them.  A non-deterministic objective gets every cell, every time. """
    if not self.deterministic:
      got = yield list(cells)
      self.num_device_calls += 1
      return [float(v) for v in np.asarray(got, dtype=np.float64).reshape(-1)]
    miss = [c for c in dict.fromkeys(cells) if c not in self.values]
    step = len(miss) if not group else group
    for s0 in range(0, len(miss), max(step, 1)):
      part = miss[s0:s0 + step]
      got = np.asarray((yield part), dtype=np.float64).reshape(-1)
      self.num_device_calls += 1
      for c, v in zip(part, got):
        self.values[c] = float(v)
    return [self.values[c] for c in cells]

  def _score(self, cells):
    """ batch_obj at the midpoints of the cells. """
    return self.batch_obj(np.array([[(lo + hi) / 2.0 for (lo, hi) in c] for c in cells]))

  def _eval_cells(self, cells, group=None):
    return self._drive(self._fetch(cells, group), self._score)

  @staticmethod
  def _drive(gen, evaluate):
    """ Runs a generator to completion, answering every yielded list of cells with evaluate(cells). """
    try:
      need = next(gen)
      while True:
        need = gen.send(evaluate(need))
    except StopIteration as stop:
      return stop.value

  # -- evaluation of a group of cells (one split's children, or the root) ---------------------------------------
  def _fidelity(self, diam, C):
    return min(max(1 - diam / C, self.tol), 1.0)

  def _score_cells(self, st, cells, height, rho, nu, split_dim):
    """ doo.py:127-158 for each cell IN ORDER, with the needed objective values requested in one go.
        Which cells need a value does not depend on the values themselves unless C doubles mid-group (it cannot
        for an objective that ignores z: a re-evaluation returns the cached value); that case asks again, cell by
        cell, to stay exact. """
    diam = nu * (rho ** height)
    C_before = st.C
    z = self._fidelity(diam, st.C)
    need = [c for c in cells if not (c in st.cache and abs(st.cache[c].fidelity - z) <= self.tol)]
    values = {}
    if need:
      got = yield need
      values = dict(zip(need, [float(v) for v in got]))
    leaves, cost = [], 0
    for c in cells:
      if st.C != C_before:           # C doubled inside this group: the remaining cells see a new z
        z = self._fidelity(diam, st.C)
        if c not in values and not (c in st.cache and abs(st.cache[c].fidelity - z) <= self.tol):
          got = yield [c]
          values[c] = float(got[0])
      if c in st.cache:
        known = st.cache[c]
        if abs(known.fidelity - z) <= self.tol:
          value, spent = known.value, 0
        else:
          value = self._record(st, c, values[c])
          if abs(value - known.value) > st.C * abs(known.fidelity - z):
            st.C = 2.0 * st.C
          known.value, known.fidelity = value, z
          spent = 1.0
      else:
        value = self._record(st, c, values[c])
        st.cache[c] = _Leaf(c, value, z, diam + st.C * (1.0 - z) + value, height, split_dim)
        spent = 1.0
      leaves.append(_Leaf(c, value, z, diam + st.C * (1.0 - z) + value, height, split_dim))
      cost += spent
    return leaves, cost

  def _record(self, st, cell, value):
    if st.record and len(self.query_vals) <= self.total_budget:
      self.query_pts.append(np.array([(lo + hi) / 2.0 for (lo, hi) in cell]))
      self.query_vals.append(value)
    return value

  # -- one DOO pass (doo.py:188-230) -----------------------------------------------------------------------------------
  def _split(self, st, leaf, rho, nu):
    spans = [abs(hi - lo) for (lo, hi) in leaf.cell]
    d = int(np.argmax(spans))
    if d == leaf.split_dim:
      d = (leaf.split_dim - 1) % len(leaf.cell)
    edges = np.linspace(leaf.cell[d][0], leaf.cell[d][1], self.K + 1)
    kids = [tuple((edges[i], edges[i + 1]) if j == d else side for j, side in enumerate(leaf.cell))
            for i in range(self.K)]
    return (yield from self._score_cells(st, kids, leaf.height + 1, rho, nu, d))

  def _doo_pass(self, st, budget, nu, rho):
    root = tuple((0, 1) for _ in range(self.dim))
    leaves, cost = yield from self._score_cells(st, [root], 0, rho, nu, 0)
    heap = []
    heapq.heappush(heap, leaves[0])
    seen = {}
    while cost <= budget:
      top = heapq.heappop(heap)
      seen[top.cell] = (top.value, top.fidelity, top.height)
      kids, spent = yield from self._split(st, top, rho, nu)
      if top.cell == kids[0].cell:
        break
      cost = cost + spent
      for kid in kids:
        heapq.heappush(heap, kid)
    while heap:
      leaf = heapq.heappop(heap)
      seen[leaf.cell] = (leaf.value, leaf.fidelity, leaf.height)
    best, pick = float('-inf'), None
    for cell, (value, fidelity, height) in seen.items():
      if value - st.C * (1.0 - fidelity) > best:
        best = value - st.C * (1.0 - fidelity)
        pick = (value, fidelity, np.array([(lo + hi) / 2 for (lo, hi) in cell]), height)
    return pick[0], pick[1], pick[2], cost, pick[3]

  # -- speculative lock-step prefetch of all passes ------------------------------------------------------------------
  def _prefetch_all(self, budget, rhos):
    gens = [self._doo_pass(_PassState(self.state.C, False), budget, self.nu_max, rho) for rho in rhos]
    wants = {}
    for i, gen in enumerate(gens):
      try:
        wants[i] = next(gen)
      except StopIteration:
        pass
    while wants:
      cells = [c for i in sorted(wants) for c in wants[i]]
      before = len(self.values)
      yield from self._fetch(cells, group=self.PREFETCH_GROUP)
      self.num_prefetched += len(self.values) - before
      nxt = {}
      for i in sorted(wants):
        try:
          nxt[i] = gens[i].send([self.values[c] for c in wants[i]])
        except StopIteration:
          pass
      wants = nxt

  def _exact_pass(self, budget, rho):
    """ One DOO pass on the shared state, its requests answered from the value table (misses fetched on demand). """
    gen = self._doo_pass(self.state, budget, self.nu_max, rho)
    try:
      need = next(gen)
      while True:
        need = gen.send((yield from self._fetch(need)))
    except StopIteration as stop:
      return stop.value

  # -- the sweep over rho (doo.py:232-251) ------------------------------------------------------------------------------
  def steps(self, mult=0.5):
    """ The whole search as a generator: yields lists of cells whose objective values it needs (never more than
        PREFETCH_GROUP in the prefetch), receives their values, and returns (passes, index of the chosen pass). """
    Dm = int(np.log(self.K) / np.log(1 / self.rho_max))
    n = self.total_budget / 1.0
    N = int(mult * Dm * np.log(n / np.log(n)))
    budget = self.total_budget / float(N)
    rhos = [(self.rho_max) ** (float(N) / (N - i)) for i in range(N)]
    if self.prefetch and N > 1:
      yield from self._prefetch_all(budget, rhos)
    passes = []
    for rho in rhos:
      passes.append((yield from self._exact_pass(budget, rho)))
    adjusted = [p[0] - self.state.C * (1 - p[1]) for p in passes]
    return passes, int(np.argmax(adjusted))

  def run(self, mult=0.5):
    return self._drive(self.steps(mult), self._score)


def run_lockstep(searches, score, mult=0.5):
  """ Runs several searches together: every round, the cells that all unfinished searches request go to ONE call
      score([(i, cells_i), ...]) -> [values_i, ...] (i = the search's index, in increasing order).  Each search sees only
      its own values, so it visits the cells it visits when run alone, in the same order, and returns the same result.
      Returns ([search.run()'s result per search], the number of rounds). """
  gens = [s.steps(mult) for s in searches]
  results, wants = [None] * len(gens), {}
  for i, gen in enumerate(gens):
    try:
      wants[i] = next(gen)
    except StopIteration as stop:
      results[i] = stop.value
  rounds = 0
  while wants:
    order = sorted(wants)
    got = score([(i, wants[i]) for i in order])
    rounds += 1
    nxt = {}
    for i, vals in zip(order, got):
      try:
        nxt[i] = gens[i].send(vals)
      except StopIteration as stop:
        results[i] = stop.value
    wants = nxt
  return results, rounds


def pdoo_maximise(obj, bounds, max_evals, vectorised=True, deterministic=True):
  """ oper_utils.py:257-271 + doo.py:253-260: returns (max_val, max_pt, None).  `obj` takes an (k, d) array of
      points in the ORIGINAL coordinates and returns k values when `vectorised` (the acquisition closures of
      gpb_acquisitions do); otherwise it is called one point at a time like the reference does. """
  bounds = np.array(bounds)
  lo, width = bounds[:, 0], bounds[:, 1] - bounds[:, 0]

  def batch_obj(P):
    X = P * width + lo                                         # map_to_bounds (general_utils.py:25-27)
    if vectorised:
      return obj(X)
    return np.array([float(obj(x)) for x in X])
  search = PDOOSearch(batch_obj, len(bounds), float(max_evals), nu_max=1.0, rho_max=0.9, K=2, C_init=0.8,
                      tol=1e-3, deterministic=deterministic)
  passes, index = search.run(0.5)
  max_pt = passes[index][2] * width + lo
  pdoo_maximise.last_search = search            # diagnostics: query sequence, number of batched calls
  return passes[index][0], max_pt, None


pdoo_maximise.last_search = None


def pdoo_maximise_lockstep(score, list_of_bounds, max_evals):
  """ pdoo_maximise over each of several boxes with the same budget, the searches run in lock-step (run_lockstep):
      score([(i, X_i), ...]) -> [values_i, ...] gets, per round, the points X_i in box i's ORIGINAL coordinates that
      search i needs.  Returns [(max_val, max_pt) per box]; pdoo_maximise_lockstep.last_searches and .last_rounds keep the
      searches (query sequences) and the number of score calls. """
  boxes = [np.array(b, dtype=np.float64) for b in list_of_bounds]
  searches = [PDOOSearch(None, len(b), float(max_evals), nu_max=1.0, rho_max=0.9, K=2, C_init=0.8, tol=1e-3)
              for b in boxes]

  def score_cells(requests):
    pts = [(i, np.array([[(lo + hi) / 2.0 for (lo, hi) in c] for c in cells]) * (boxes[i][:, 1] - boxes[i][:, 0])
            + boxes[i][:, 0]) for i, cells in requests]
    return score(pts)
  results, rounds = run_lockstep(searches, score_cells, 0.5)
  pdoo_maximise_lockstep.last_searches, pdoo_maximise_lockstep.last_rounds = searches, rounds
  out = []
  for b, (passes, index) in zip(boxes, results):
    out.append((passes[index][0], passes[index][2] * (b[:, 1] - b[:, 0]) + b[:, 0]))
  return out


pdoo_maximise_lockstep.last_searches, pdoo_maximise_lockstep.last_rounds = None, 0
