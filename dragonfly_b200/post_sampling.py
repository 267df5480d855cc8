"""
GPFitter.fit_gp for hp_tune_criterion 'post_sampling' with post_hp_tune_method 'slice' (gp_core.py:592-726, 811-821):
every continuous hyper-parameter in turn through a fresh slice sampler (sampling/slice.py:37-108), every discrete one
(the Matern nu) through a Metropolis chain over its category ids (sampling/metropolis.py:122-164), the log-probability
of a vector being the sum of its uniform / categorical priors plus the GP's log marginal likelihood.

The sample sequence and the global NumPy RNG consumption are the reference's; what changes is how the LMLs are
obtained.  The reference evaluates them one at a time, each a fresh GP build.  Here they come in batches
(`lml_batch`, by default hp_grid.lml_batch_for_hyperparams: one dfb_lml_batch launch), by speculation:
  stepping out    the points of both chains ql - k w, qr + k w (k < depth, formed by repeated subtraction / addition
                  as the reference forms them) are evaluated at once; out-of-bound points cost nothing (prior -inf);
                  the prefix the reference would have evaluated is consumed, a chain that runs past `depth` asks for
                  another batch;
  shrinkage       `depth` uniforms are drawn ahead, the proposals the reference would make if each were rejected are
                  evaluated at once (a rejection moves the interval by a rule that needs no LML), the first accepted
                  one is taken and the RNG is rewound to consume exactly the uniforms the reference consumes;
  Metropolis      all categories of the discrete hp are evaluated on the first miss of a chain (the other hps do not
                  move during it);
  cache           logp at the start of each slice sample is the value of the point accepted last: LMLs are cached on
                  the exact hp vector (the device values are deterministic).
Without ever-rejected speculation an LML is evaluated once, so the consumed sequence -- and every acceptance decision
-- is the reference's; a slice sample costs two round trips when neither chain exceeds `depth`.
"""
import numpy as np

from .hp_grid import lml_batch_for_hyperparams, LML_BATCH_MAX_N

# Speculation depth where one batch is one dfb_lml_batch launch (N <= LML_BATCH_MAX_N).  Above the cap every LML is a
# build of its own, so speculation only adds builds: depth 1 there (DESIGN.md 10: 37.7 s against 96.6 s per fit at
# N = 1000).
DEFAULT_DEPTH = 8


class PostSamplingStats(object):
  """ Counters of one fit: LMLs the reference would compute (`consumed`, the calls of _tuning_objective_post_sampling),
      LMLs evaluated (consumed once each, plus the speculative ones never consumed), and batches (`round_trips`). """

  def __init__(self):
    self.consumed = 0
    self.evaluated = 0
    self.round_trips = 0


def device_lml_batch(X, Y, layout, device=None, batch_fn=lml_batch_for_hyperparams):
  """ The sampler's default LML source: batch_fn (lml_batch_for_hyperparams or lml_for_hyperparams) on one posterior
      that is kept across calls, each item with what the layout takes for its discrete hps (HPLayout.dscr_arg). """
  state = {'post': None}

  def lml_batch(cts_rows, dscr_rows):
    nus = [layout.dscr_arg(d) for d in dscr_rows]
    if all(nu is None for nu in nus):
      nus = None
    vals, state['post'] = batch_fn(X, Y, np.array(cts_rows), layout, nus=nus, post=state['post'], device=device)
    return vals
  return lml_batch


def _tune_params(scale, acc_rate):
  """ metropolis.py:243-279 """
  if acc_rate < 0.001:
    scale *= 0.1
  elif acc_rate < 0.05:
    scale *= 0.5
  elif acc_rate < 0.2:
    scale *= 0.9
  elif acc_rate > 0.95:
    scale *= 10.0
  elif acc_rate > 0.75:
    scale *= 2.0
  elif acc_rate > 0.5:
    scale *= 1.1
  return scale


class _Sampler(object):
  """ The state of _sample_cts_dscr_hps_for_post_sampling: the hp vector, the priors and the LML cache. """

  def __init__(self, cts_hp_bounds, dscr_hp_vals, lml_batch, depth, stats, trace):
    self.lower = [float(b[0]) for b in cts_hp_bounds]              # ContinuousUniform(bounds[0], bounds[-1])
    self.upper = [float(b[-1]) for b in cts_hp_bounds]
    self.cats = [list(v) for v in dscr_hp_vals]                    # Categorical(vals, uniform p)
    self.probs = [np.repeat(1.0 / len(v), len(v)) for v in dscr_hp_vals]
    self.n_cts = len(self.lower)
    self.num_hps = self.n_cts + len(self.cats)
    self.lml_batch, self.depth, self.stats, self.trace = lml_batch, max(1, int(depth)), stats, trace
    self.cache = {}
    self.hps = np.ones((self.num_hps,))

  # ---- priors (gp_core.py:611-618) -----------------------------------------------------------------------------------
  def _cat_id(self, k, category):
    """ Categorical.get_id (distributions/discrete.py:152-156) """
    if category is None or np.isnan(category):
      return -1
    return self.cats[k].index(category)

  def prior(self, h):
    lp = 0
    for i in range(self.n_cts):
      x = h[i]
      lp += -np.inf if (x < self.lower[i] or x > self.upper[i]) else -np.log(self.upper[i] - self.lower[i])
    for k in range(len(self.cats)):
      value = self._cat_id(k, h[self.n_cts + k])
      lp += -np.inf if (value < 0 or value >= len(self.cats[k])) else np.log(self.probs[k][value])
    return lp

  # ---- LMLs ------------------------------------------------------------------------------------------------------------
  def with_hp(self, i, x):
    h = self.hps.copy()
    h[i] = x
    return h

  def prefetch(self, vectors):
    """ One batch for every vector whose prior is finite and whose LML is not cached yet. """
    todo, keys = [], set()
    for h in vectors:
      key = tuple(h.tolist())
      if key in self.cache or key in keys or not np.isfinite(self.prior(h)):
        continue
      keys.add(key)
      todo.append(h)
    if not todo:
      return
    vals = self.lml_batch([h[:self.n_cts] for h in todo], [h[self.n_cts:] for h in todo])
    self.stats.round_trips += 1
    self.stats.evaluated += len(todo)
    for h, v in zip(todo, vals):
      self.cache[tuple(h.tolist())] = float(v)

  def logp(self, h):
    """ _logp (gp_core.py:596-622) of the vector h: the priors in index order, then the LML. """
    lp = self.prior(h)
    if not np.isfinite(lp):
      return lp
    key = tuple(h.tolist())
    if key not in self.cache:
      self.prefetch([h])
    val = self.cache[key]
    self.stats.consumed += 1
    if self.trace is not None:
      self.trace.append((h.copy(), val))
    lp += val
    return lp

  # ---- continuous: Slice._sample (slice.py:37-87) for one coordinate ---------------------------------------------
  def slice_sample(self, i, q0, w, n_tunes):
    q = q0
    y = self.logp(self.with_hp(i, q)) - np.random.standard_exponential()
    ql = q - np.random.uniform(0, w)
    qr = q + w
    left, right = [ql], [qr]
    k_left = k_right = 0
    lefts_done = rights_done = False
    while True:
      # extend both chains to `depth` points past what is consumed, stopping at the first out-of-bound point
      for pts, sign in ((left, -1.0), (right, 1.0)):
        while len(pts) < (k_left if sign < 0 else k_right) + self.depth and self.lower[i] <= pts[-1] <= self.upper[i]:
          pts.append(pts[-1] - w if sign < 0 else pts[-1] + w)
      lo_need = [] if lefts_done else left[k_left:k_left + self.depth]
      hi_need = [] if rights_done else right[k_right:k_right + self.depth]
      self.prefetch([self.with_hp(i, x) for x in lo_need + hi_need])
      while not lefts_done and k_left < len(left) and self._cached_or_out(i, left[k_left]):
        if y < self.logp(self.with_hp(i, left[k_left])):
          k_left += 1
        else:
          lefts_done = True
      if not lefts_done:
        continue
      while not rights_done and k_right < len(right) and self._cached_or_out(i, right[k_right]):
        if y < self.logp(self.with_hp(i, right[k_right])):
          k_right += 1
        else:
          rights_done = True
      if rights_done:
        break
    ql, qr = left[k_left], right[k_right]
    # shrinkage: the proposals of `depth` uniforms drawn ahead, as if each were rejected
    while True:
      state = np.random.get_state()
      us = [np.random.rand() for _ in range(self.depth)]
      props, bounds = [], []
      l, r = ql, qr
      for u in us:
        p = (r - l) * u + l
        props.append(p)
        bounds.append((l, r))
        if p > q0:
          r = p
        elif p < q0:
          l = p
      self.prefetch([self.with_hp(i, p) for p in props])
      accepted = None
      for k, p in enumerate(props):
        if not self.logp(self.with_hp(i, p)) < y:
          accepted = k
          break
      if accepted is None:
        ql, qr = l, r
        continue
      np.random.set_state(state)
      for _ in range(accepted + 1):
        np.random.rand()
      q = props[accepted]
      ql, qr = bounds[accepted]
      break
    w = w * (n_tunes / (n_tunes + 1)) + (qr - ql) / (n_tunes + 1)
    return q, w

  def _cached_or_out(self, i, x):
    h = self.with_hp(i, x)
    return tuple(h.tolist()) in self.cache or not np.isfinite(self.prior(h))

  def slice_chain(self, i, init, num_samples, burn):
    """ Slice(model).sample(init, num_samples, burn) (slice.py:89-108) with w = 1 and tuning on. """
    w, n_tunes = 1., 0.
    q0 = float(init)
    for _ in range(burn):
      q0, w = self.slice_sample(i, q0, w, n_tunes)
      n_tunes += 1
    samples = np.zeros(num_samples)
    for s in range(num_samples):
      q0, w = self.slice_sample(i, q0, w, n_tunes)
      n_tunes += 1
      samples[s] = q0
    return samples

  # ---- discrete: Metropolis(model, True).sample over category ids (metropolis.py:97-164) ----------------------------
  def category_vector(self, i, cat_id):
    """ hps with entry i set from a category id the way _logp does it: get_category, None (NaN) outside the ids. """
    k = i - self.n_cts
    val = self.cats[k][int(cat_id)] if 0 <= cat_id < len(self.cats[k]) else None
    return self.with_hp(i, np.nan if val is None else val)

  def metropolis_chain(self, i, init_id, num_samples):
    scaling = np.atleast_1d(1.).astype('d')
    steps_until_tune, accepted_count = 100, 0
    q0 = np.array([init_id])
    samples = np.zeros([num_samples, 1])
    self.prefetch([self.category_vector(i, c) for c in [int(init_id)] + list(range(len(self.cats[i - self.n_cts])))])
    for s in range(num_samples):
      if not steps_until_tune:
        scaling = _tune_params(scaling, accepted_count / float(100))
        steps_until_tune = 100
        accepted_count = 0
      delta = np.random.normal(scale=np.ones(1)) * scaling
      delta = np.round(delta, 0).astype('int64')
      q0 = q0.astype('int64')
      q = (q0 + delta).astype('int64')
      val = self.logp(self.category_vector(i, q.item())) - self.logp(self.category_vector(i, q0.item()))
      mr = min(1, np.exp(val))
      if np.isfinite(mr) and np.random.uniform() < mr:
        q_new, acc = q, True
      else:
        q_new, acc = q0, False
      accepted_count += acc
      steps_until_tune -= 1
      samples[s] = q_new
      q0 = samples[s]
    return samples[:, 0]


def post_sample_hps(X, Y, layout, cts_hp_bounds, dscr_hp_vals=(), num_samples=1, offset=25, burn=-1, build_gp=None,
                    lml_batch=None, depth=None, device=None, stats=None, trace=None):
  """ GPFitter.fit_gp(num_samples, 'post_sampling') with the slice sampler (gp_core.py:592-726, 811-821) on any
      hp_grid.HPLayout.  `cts_hp_bounds` / `dscr_hp_vals` are the fitter's; `offset` and `burn`
      its post_hp_tune_offset / post_hp_tune_burn (-1: int(sqrt(num_hps) * 100), unclipped as in the reference).
      `build_gp(cts, dscr)` builds the returned GP when num_samples == 1.  `lml_batch(cts_rows, dscr_rows)` returns the
      LMLs of a batch (default: device_lml_batch); `depth` bounds the speculation (default: DEFAULT_DEPTH up to
      LML_BATCH_MAX_N training points, 1 above).  `stats` (PostSamplingStats) and
      `trace` (a list: (hp vector, LML) per consumed LML, in the reference's order) are filled when given.  Returns
      ('post_fitted_gp', gp, (cts, dscr)) or ('post_sample_hps_with_probs', cts, dscr, [None] * num_samples).
      X holds the points the layout's rows() takes: with a CartesianProductHPLayout CPGPFitter's list-of-parts points
      (encoded here), and there may then be a discrete hp per tuned Matern part: each has its own Metropolis chain, and
      every LML item gets the whole tuple. """
  X = layout.rows(X)
  Y = np.asarray(Y, dtype=np.float64)
  dscr_hp_vals = [list(v) for v in dscr_hp_vals]
  if layout.max_dscr_hps is not None and len(dscr_hp_vals) > layout.max_dscr_hps:
    raise NotImplementedError('More discrete hyper-parameters than the layout takes on the device path.')
  if lml_batch is None:
    lml_batch = device_lml_batch(X, Y, layout, device=device)
  if depth is None:
    depth = DEFAULT_DEPTH if len(X) <= LML_BATCH_MAX_N else 1
  stats = PostSamplingStats() if stats is None else stats
  S = _Sampler(cts_hp_bounds, dscr_hp_vals, lml_batch, depth, stats, trace)
  n_cts, num_hps = S.n_cts, S.num_hps
  best_cts_hps = np.zeros([num_samples, n_cts])
  best_dscr_hps = np.zeros([num_samples, len(dscr_hp_vals)])
  total_samples = (num_samples - 1) * offset + 1
  cts_hps = np.zeros([total_samples, n_cts])
  dscr_hps = np.zeros([total_samples, len(dscr_hp_vals)])
  if burn == -1:
    burn = int(np.sqrt(num_hps) * 100)
  for i in range(n_cts):
    S.hps[i] = (S.lower[i] + S.upper[i]) / 2                      # ContinuousUniform.get_mean
  for i in range(n_cts, num_hps):
    k = i - n_cts
    draw = np.random.multinomial(1, S.probs[k], 1)                 # Categorical.draw_samples('random', 1)
    S.hps[i] = S.cats[k][int(np.argmax(draw, len(draw.shape) - 1)[0])]
  order = list(range(num_hps))
  np.random.shuffle(order)
  for i in order:
    if i < n_cts:
      cts_hps[:, i] = S.slice_chain(i, S.hps[i], total_samples, burn)
      S.hps[i] = cts_hps[0, i]
    else:
      k = i - n_cts
      ids = S.metropolis_chain(i, S._cat_id(k, S.hps[i]), total_samples)
      for j, val in enumerate(ids):
        dscr_hps[j, k] = S.cats[k][int(val)] if 0 <= int(val) < len(S.cats[k]) else np.nan
      S.hps[i] = dscr_hps[0, k]
  for i in range(num_samples):
    best_cts_hps[i, :] = cts_hps[i * offset, :]
    best_dscr_hps[i, :] = dscr_hps[i * offset, :]
  if num_samples == 1:
    return 'post_fitted_gp', build_gp(best_cts_hps[0], best_dscr_hps[0]), (best_cts_hps, best_dscr_hps)
  return 'post_sample_hps_with_probs', best_cts_hps, best_dscr_hps, [None] * num_samples
