"""
Generates tests/golden/post_sampling.npz: the UNMODIFIED reference's GPFitter.fit_gp(num_samples, 'post_sampling') with
the slice sampler (gp_core.py:592-726, 811-821) under a seeded global RNG, with every _tuning_objective_post_sampling
call logged (hp vector, discrete values, LML).  Run with the reference source tree in $DRAGONFLY_REF:

    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python -W ignore \
        tests/golden/make_golden_post_sampling.py

Configurations: A EuclideanGPFitter, Matern with tuned nu (Metropolis over its ids), tuned mean and noise, N = 40,
d = 3, 4 samples, offset 3, burn 20; B SE, 1 sample, the default (unclipped) burn-in; C EuclideanMFGPFitter (fidelity
dimension 1, domain dimension 2), 3 samples, burn 10.  Per configuration: inputs and options, the returned cts / dscr,
the call trace, four np.random.random() draws after the fit (RNG fingerprint) and the smallest relative margin of any
acceptance comparison -- the seed is the first one whose margin exceeds 1e-7, so that LMLs that differ from these in
the 10th digit take every decision the same way.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

import dragonfly  # noqa: E402
from dragonfly.gp.euclidean_gp import EuclideanGPFitter, EuclideanMFGPFitter, euclidean_gp_args, \
    euclidean_mf_gp_args  # noqa: E402
from dragonfly.distributions.model import Model  # noqa: E402
from dragonfly.sampling.slice import Slice  # noqa: E402
from dragonfly.sampling.metropolis import Metropolis  # noqa: E402
from dragonfly.utils.option_handler import load_options  # noqa: E402

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])

MIN_MARGIN = 1e-7


class Recorder(object):
  """ Wraps (does not restate) Model.logp, np.random.standard_exponential / uniform, Slice._sample and
      Metropolis._sample to collect the operands of every acceptance comparison. """

  def __init__(self):
    self.events, self.margins, self.out_of_range = None, [], 0

  def install(self):
    rec = self
    orig_logp, orig_exp, orig_unif = Model.logp, np.random.standard_exponential, np.random.uniform
    orig_slice, orig_metro = Slice._sample, Metropolis._sample

    def logp(self, x):
      v = orig_logp(self, x)
      if rec.events is not None:
        rec.events.append(('lp', float(v)))
      return v

    def sexp(*a, **k):
      v = orig_exp(*a, **k)
      if rec.events is not None:
        rec.events.append(('exp', float(v)))
      return v

    def unif(*a, **k):
      v = orig_unif(*a, **k)
      if rec.events is not None and not a and not k:
        rec.events.append(('u', float(v)))
      return v

    def slice_sample(self, q0):
      rec.events = []
      q = orig_slice(self, q0)
      ev, rec.events = rec.events, None
      assert ev[0][0] == 'lp' and ev[1][0] == 'exp'
      y = ev[0][1] - ev[1][1]
      for kind, v in ev[2:]:
        if kind == 'lp' and np.isfinite(v):
          rec.margins.append(abs(y - v) / max(abs(v), 1e-300))
      return q

    def metro_sample(self, q0):
      rec.events = []
      q = orig_metro(self, q0)
      ev, rec.events = rec.events, None
      lp_q, lp_q0 = ev[0][1], ev[1][1]
      if not np.isfinite(lp_q):
        rec.out_of_range += 1
      if len(ev) > 2:
        mr = min(1, np.exp(lp_q - lp_q0))
        if 0 < mr < 1:
          rec.margins.append(abs(ev[2][1] - mr) / mr)
      return q

    Model.logp, np.random.standard_exponential, np.random.uniform = logp, sexp, unif
    Slice._sample, Metropolis._sample = slice_sample, metro_sample


REC = Recorder()


def run(tag, make_fitter, num_samples, out, seeds):
  for seed in seeds:
    fitter, X, Y, Z = make_fitter()
    trace = []
    orig = fitter._tuning_objective_post_sampling

    def logged(cts, dscr, *a, **k):
      v = orig(cts, dscr, *a, **k)
      trace.append((np.array(cts, dtype=np.float64).copy(), np.array(dscr, dtype=np.float64).copy(), float(v)))
      return v
    fitter._tuning_objective_post_sampling = logged
    REC.margins, REC.out_of_range = [], 0
    np.random.seed(seed)
    res = fitter.fit_gp(num_samples, 'post_sampling')
    fingerprint = np.array([np.random.random() for _ in range(4)])
    margin = min(REC.margins)
    print(tag, 'seed', seed, 'calls', len(trace), 'margin %.2e' % margin, 'metropolis out of range', REC.out_of_range)
    if margin <= MIN_MARGIN:
      continue
    opt = fitter.options
    out[tag + '_seed'] = seed
    out[tag + '_X'] = X; out[tag + '_Y'] = Y
    if Z is not None:
      out[tag + '_Z'] = Z
    out[tag + '_bounds'] = np.array(fitter.cts_hp_bounds)
    out[tag + '_dscr_vals'] = np.array(fitter.dscr_hp_vals, dtype=np.float64).reshape(len(fitter.dscr_hp_vals), 3)
    out[tag + '_num_samples'] = num_samples
    out[tag + '_offset'] = opt.post_hp_tune_offset; out[tag + '_burn'] = opt.post_hp_tune_burn
    out[tag + '_mean_func_type'] = opt.mean_func_type; out[tag + '_noise_var_type'] = opt.noise_var_type
    out[tag + '_trace_cts'] = np.array([t[0] for t in trace])
    out[tag + '_trace_dscr'] = np.array([t[1] for t in trace]).reshape(len(trace), len(fitter.dscr_hp_vals))
    out[tag + '_trace_lml'] = np.array([t[2] for t in trace])
    out[tag + '_fingerprint'] = fingerprint
    out[tag + '_margin'] = margin
    out[tag + '_metropolis_out_of_range'] = REC.out_of_range
    if res[0] == 'post_fitted_gp':
      _, gp, (cts, dscr) = res
      out[tag + '_lml'] = gp.compute_log_marginal_likelihood()
    else:
      _, cts, dscr, _ = res
    out[tag + '_kind'] = res[0]
    out[tag + '_cts'] = np.array(cts); out[tag + '_dscr'] = np.array(dscr)
    return
  raise RuntimeError('no seed with a margin above %g for %s' % (MIN_MARGIN, tag))


def main():
  REC.install()
  rs = np.random.RandomState(3)
  out = {}

  def fitter_a():
    X = rs.random_sample((40, 3)); Y = np.sin(4 * X[:, 0]) + X[:, 1] * X[:, 2] + 0.05 * rs.randn(40)
    opt = load_options(euclidean_gp_args)
    opt.kernel_type = 'matern'; opt.matern_nu = -1.0; opt.mean_func_type = 'tune'; opt.noise_var_type = 'tune'
    opt.hp_tune_criterion = 'post_sampling'; opt.post_hp_tune_method = 'slice'
    opt.post_hp_tune_offset = 3; opt.post_hp_tune_burn = 20
    return EuclideanGPFitter(list(X), list(Y), opt), X, Y, None
  run('A', fitter_a, 4, out, range(1, 50))

  def fitter_b():
    X = rs.random_sample((30, 2)); Y = np.cos(3 * X[:, 0]) - X[:, 1] ** 2 + 0.05 * rs.randn(30)
    opt = load_options(euclidean_gp_args)
    opt.kernel_type = 'se'; opt.mean_func_type = 'tune'; opt.noise_var_type = 'tune'
    opt.hp_tune_criterion = 'post_sampling'; opt.post_hp_tune_method = 'slice'; opt.post_hp_tune_burn = -1
    return EuclideanGPFitter(list(X), list(Y), opt), X, Y, None
  run('B', fitter_b, 1, out, range(1, 50))

  def fitter_c():
    Z = rs.random_sample((36, 1)); X = rs.random_sample((36, 2))
    Y = np.sin(3 * X[:, 0]) + X[:, 1] - 0.3 * (1 - Z[:, 0]) + 0.05 * rs.randn(36)
    opt = load_options(euclidean_mf_gp_args)
    opt.fidel_kernel_type = 'se'; opt.domain_kernel_type = 'matern'; opt.domain_matern_nu = 2.5
    opt.mean_func_type = 'tune'; opt.noise_var_type = 'tune'
    opt.hp_tune_criterion = 'post_sampling'; opt.post_hp_tune_method = 'slice'
    opt.post_hp_tune_offset = 3; opt.post_hp_tune_burn = 10
    return EuclideanMFGPFitter(list(Z), list(X), list(Y), opt), X, Y, Z
  run('C', fitter_c, 3, out, range(1, 50))
  assert out['A_metropolis_out_of_range'] > 0, 'golden A never proposes a category id outside the range'
  np.savez_compressed(os.path.join(HERE, 'post_sampling.npz'), **out)


if __name__ == '__main__':
  main()
