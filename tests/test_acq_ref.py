"""
The reference of the acquisition epilogue (tests/acq_ref.py) on its own, without a GPU:
  * its forward-error bounds hold for the device's operation sequence with erf, erfc and exp pushed adversarially by
    their documented maximum ulp errors, against mpmath, on a dense z grid over [-40, 40] with z = +-1 and its
    neighbours (the erf / erfc branch), the points where phi and erfc underflow, and sd down to subnormal;
  * the bounds are not vacuous: for |z| <= 5 each is at most a small stated multiple of u times the term magnitudes;
  * SciPy's norm.cdf / norm.pdf in the reference's formulas meet the cephes-side bound;
  * the int8 pass's allowance E (i8_score_err) bounds |S(sd64) - S(sd8)| for every sd64 the sigma^2 error model allows,
    for every kind, over sd8 and b2 across decades (so do the constants 0.4 >= sup phi and 0.25 >= sup |z phi|);
  * the bound pass's ub (acq at mu_bar >= mu and sqrt(k**) >= sd) plus the shortlist's pad is at least the fp64 score
    for EI, UCB with beta >= 0 and PI below the incumbent, on the device sequence under the same adversarial pushes;
  * the self-check's rule does not count rounding noise as a violation of the error model.
"""
import mpmath as mp
import numpy as np
import pytest
from scipy import special, stats

import acq_ref as R
from test_kstar_prune_bound import GAPS, SIGMA          # the sigma monotonicity grids of the bound pass

U = R.U
K = R.ULP_CUDA


def _pushes():
  """ erf, erfc, exp each moved by its whole documented error: all up, all down, and the two mixed patterns that push
  Phi and phi (hence z Phi and phi) apart. """
  for s in ((1, 1, 1), (-1, -1, -1), (1, -1, 1), (-1, 1, -1)):
    yield R.pushed_fns(s[0] * K['erf'], s[1] * K['erfc'], s[2] * K['exp'])


def _z_grid():
  pos = np.geomspace(1e-12, 40.0, 700)
  z = np.concatenate([-pos[::-1], [0.0, -0.0], pos, np.linspace(-6.0, 6.0, 241)])
  edges = []
  for c in (1.0, -1.0,                                     # |x| = 1/sqrt 2: the erf / erfc branch
            37.5, -37.5, 38.4674, -38.4674, 38.5, -38.5,   # erfc(|x|) subnormal, then 0; phi's exp underflows
            26.5 * np.sqrt(2.0), -26.5 * np.sqrt(2.0)):
    edges += [c, np.nextafter(c, np.inf), np.nextafter(c, -np.inf)]
  # the doubles just around the branch point itself, x = z / sqrt 2 straddling fl(1/sqrt 2)
  zb = R.SQRT1_2 / R.SQRT1_2
  for k in range(-4, 5):
    edges.append(zb + k * np.spacing(1.0))
  return np.unique(np.concatenate([z, edges]))


Z = _z_grid()
SD = [1.0, 3.7e-3, 2.5e5, 1e-300, 5e-320]                  # the last two: subnormal-range scores and quotients


def _check_within(kind, mean, sd, **kw):
  """ Every finite device-sequence score under every push lies within the bound of the exact value. """
  bnd = R.bound(kind, mean, sd, **kw)
  worst = 0.0
  for fns in _pushes():
    s = R.acq(kind, mean, sd, fns=fns, **kw)
    fin = np.isfinite(s) & np.isfinite(bnd)
    assert (np.isfinite(s) == np.isfinite(R.acq(kind, mean, sd, **kw))).all()
    err = R.errors(kind, np.where(fin, s, np.nan), mean, sd, **kw)
    ok = ~fin | (err <= bnd)
    assert ok.all(), (kind, np.asarray(mean)[~ok][:5], np.asarray(sd)[~ok][:5] if np.ndim(sd) else sd,
                      err[~ok][:5], bnd[~ok][:5])
    worst = max(worst, float(np.nanmax(np.where(fin, err / bnd, np.nan))))
  return worst


@pytest.mark.parametrize('sd', SD)
@pytest.mark.parametrize('kind', [R.EI, R.PI])
def test_device_sequence_within_the_bound(kind, sd):
  mean = Z * sd                     # z = fl(fl(mean - 0) / sd): the grid's z up to the rounding of the product
  _check_within(kind, mean, sd, best=0.0)


@pytest.mark.parametrize('ref_std', ['zero', 'tiny', 'comparable', 'large'])
@pytest.mark.parametrize('sd', [1.0, 2.5e5, 1e-300])
def test_ttei_within_the_bound(sd, ref_std):
  rs = {'zero': 0.0, 'tiny': 1e-12 * sd, 'comparable': 0.7 * sd, 'large': 1e3 * sd}[ref_std]
  comb = np.sqrt(rs * rs + sd * sd)
  _check_within(R.TTEI, 1.5 + Z[::3] * comb, sd, ref_mean=1.5, ref_std=rs)


def test_ucb_and_ts_within_the_bound():
  rs = np.random.RandomState(0)
  mean = np.concatenate([rs.standard_normal(300) * 10.0 ** rs.randint(-300, 300, 300), [0.0, -0.0, 1e9, -1e15]])
  sd = np.abs(rs.standard_normal(mean.size)) * 10.0 ** rs.randint(-300, 300, mean.size)
  for beta in (0.0, 2.5, -3.0, 1e-3):
    s = R.acq(R.UCB, mean, sd, beta=beta)
    err = R.errors(R.UCB, s, mean, sd, beta=beta)
    assert (err <= R.bound(R.UCB, mean, sd, beta=beta)).all()
  z = rs.standard_normal(mean.size) * 3.0
  s = R.acq(R.TS, mean, sd, z=z)
  assert (R.errors(R.TS, s, mean, sd, z=z) <= R.bound(R.TS, mean, sd, z=z)).all()


def test_sigma_restatement_on_edges():
  """ sigma(): sequential sum of the partial rows, sqrt(kss - vn) without a clamp: NaN, -0.0, 0 and subnormal. """
  kss = np.array([1.0, 1.0, 1.0, 1e-310, 0.0, -0.0])
  partial = np.array([[0.5, 0.75, 1.0, 0.0, 0.0, 0.0], [0.5, 0.5, 0.0, 0.0, 0.0, 0.0]])
  sd = R.sigma(partial, kss)
  assert sd[0] == 0.0 and np.isnan(sd[1]) and sd[2] == 0.0 and 0.0 < sd[3] < 1e-150
  assert sd[4] == 0.0 and np.signbit(sd[5]) and sd[5] == 0.0


# ---- the bounds are not vacuous -------------------------------------------------------------------------------------
# For |z| <= 5 each bound is at most C u times the term magnitudes (acq_ref.magnitude).  C follows from the parameters:
# erfc's 5 ulps and the branch's 0.5 halve to ~2.5 u of Phi, exp's 1 ulp and the divisions add ~3 u of phi, and z's own
# rounding enters through Phi and |z| phi: a few tens of u.
NOT_VACUOUS = {R.EI: 48.0, R.PI: 48.0, R.TTEI: 64.0, R.UCB: 2.0, R.TS: 2.0}


@pytest.mark.parametrize('kind', [R.EI, R.PI, R.TTEI, R.UCB, R.TS])
def test_bounds_are_not_vacuous(kind):
  z = np.linspace(-5.0, 5.0, 2001)
  for sd in (1.0, 3.7e-3, 2.5e5):
    kw = {'ref_mean': 0.0, 'ref_std': 0.3 * sd} if kind == R.TTEI else {'beta': 2.0, 'z': z} if kind in (R.UCB, R.TS) \
        else {'best': 0.0}
    mean = z * sd
    ratio = R.bound(kind, mean, sd, **kw) / (U * R.magnitude(kind, mean, sd, **kw))
    ratio = ratio[np.abs(mean) > 1e-280]
    assert np.nanmax(ratio) <= NOT_VACUOUS[kind], (kind, sd, float(np.nanmax(ratio)))


# ---- SciPy (cephes ndtr, NumPy exp) meets the reference-side bound -------------------------------------------------
def _scipy(kind, mean, sd, best=0.0, ref_mean=0.0, ref_std=0.0):
  """ gpb_acquisitions.py's formulas on scipy.stats.norm, as the reference evaluates them. """
  with np.errstate(all='ignore'):
    if kind == R.PI:
      return stats.norm.cdf((mean - best) / sd)
    if kind == R.EI:
      z = (mean - best) / sd
      return sd * (z * stats.norm.cdf(z) + stats.norm.pdf(z))
    comb = np.sqrt(ref_std ** 2 + sd ** 2)
    z = (mean - ref_mean) / comb
    return comb * (z * stats.norm.cdf(z) + stats.norm.pdf(z))


@pytest.mark.parametrize('kind', [R.EI, R.PI, R.TTEI])
def test_scipy_meets_the_cephes_bound(kind):
  kw = {'ref_mean': 0.0, 'ref_std': 0.5} if kind == R.TTEI else {'best': 0.0}
  for sd in (1.0, 3.7e-3, 1e-300):
    mean = Z * sd
    s = _scipy(kind, mean, sd, **kw)
    bnd = R.bound(kind, mean, sd, ulp=R.ULP_CEPHES, **kw)
    fin = np.isfinite(s) & np.isfinite(bnd)
    err = R.errors(kind, np.where(fin, s, np.nan), mean, sd, **kw)
    ok = ~fin | (err <= bnd)
    assert ok.all(), (kind, sd, mean[~ok][:5], err[~ok][:5], bnd[~ok][:5])


def test_cephes_ulp_parameters_cover_scipy():
  """ The measured parameters of ULP_CEPHES: scipy's erf, erfc and NumPy's exp within them against mpmath. """
  c = R.ULP_CEPHES
  for x in np.concatenate([np.linspace(R.SQRT1_2, c['erfc_zero'], 1500), [1.0, 2.0, 26.0]]):
    ex = mp.erfc(mp.mpf(float(x)))
    err = float(abs(mp.mpf(float(special.erfc(x))) - ex))
    assert err <= (c['erfc'] + c['erfc_x2'] * x * x) * np.spacing(float(ex)), x
  for x in np.linspace(np.nextafter(c['erfc_zero'], np.inf), 27.3, 50):
    assert special.erfc(x) == 0.0 and mp.erfc(mp.mpf(float(x))) > 0            # the flush the bound allows for
  for x in np.linspace(-R.SQRT1_2, R.SQRT1_2, 501):
    ex = mp.erf(mp.mpf(float(x)))
    assert float(abs(mp.mpf(float(special.erf(x))) - ex)) <= c['erf'] * np.spacing(abs(float(ex))), x
  for w in np.linspace(-745.0, 0.0, 1501):
    ex = mp.exp(mp.mpf(float(w)))
    assert float(abs(mp.mpf(float(np.exp(w))) - ex)) <= c['exp'] * np.spacing(float(ex)), w


# ---- the allowance E of the int8 pass -------------------------------------------------------------------------------
def test_the_constants_behind_the_allowance():
  """ sup phi = phi(0) = 1/sqrt(2 pi) < 0.4; sup |z phi(z)| = phi(1) (d/dz z phi = (1 - z^2) phi) < 0.25. """
  assert 1 / mp.sqrt(2 * mp.pi) < mp.mpf('0.4')
  assert mp.npdf(1) < mp.mpf('0.25')
  zs = [mp.mpf(k) / 1000 for k in range(0, 6001)]
  assert max(z * mp.npdf(z) for z in zs) == mp.npdf(1)
  assert R.SENS[R.EI] >= 1 / mp.sqrt(2 * mp.pi) and R.SENS[R.TTEI] >= 1 / mp.sqrt(2 * mp.pi)
  assert R.SENS[R.PI] >= mp.npdf(1)


B2 = [1e-18, 1e-15, 1e-12, 1e-9, 5e-9]
ZS = [-5.0, -1.0, -0.3, 0.0, 0.3, 1.0, 5.0]


def _sd8s(b2):
  r = np.sqrt(b2)
  return [r * (1 + 2.0 ** -20), r * 1.5, r * 10.0] + [s for s in (1e-6, 1e-3, 1.0, 1e3) if s > 10.0 * r]


def _certify(kind, sd8, b2, sens, **kw):
  e = float(R.score_err(kind, sd8, b2, sens))
  assert e >= 0.0
  sup = R.allowance_sup(kind, sd8, b2, **kw)
  assert sup <= mp.mpf(e), (kind, sd8, b2, kw, float(sup), e)
  return float(sup / e) if e > 0 else 0.0


@pytest.mark.parametrize('kind', [R.UCB, R.EI, R.PI])
def test_allowance_is_certified(kind):
  worst = 0.0
  for b2 in B2:
    for sd8 in _sd8s(b2):
      if kind == R.UCB:
        for beta in (0.0, 0.5, 3.0, -2.0, 50.0):
          worst = max(worst, _certify(kind, sd8, b2, R.sens_of(kind, beta), mean=1.0, beta=beta))
      else:
        for z in ZS:
          worst = max(worst, _certify(kind, sd8, b2, R.sens_of(kind), mean=z * sd8, best=0.0))
  assert worst <= 1.0


@pytest.mark.parametrize('ref_std', ['zero', 'tiny', 'comparable', 'large'])
def test_allowance_is_certified_for_ttei(ref_std):
  for b2 in B2:
    for sd8 in _sd8s(b2):
      rs = {'zero': 0.0, 'tiny': 1e-12 * sd8, 'comparable': sd8, 'large': 1e3 * sd8}[ref_std]
      comb = np.sqrt(rs * rs + sd8 * sd8)
      for z in ZS:
        _certify(R.TTEI, sd8, b2, R.sens_of(R.TTEI), mean=z * comb, ref_mean=0.0, ref_std=rs)


def test_allowance_is_certified_for_ts():
  for b2 in B2:
    for sd8 in _sd8s(b2):
      for z in (-9.0, -8.6, -3.0, -0.1, 0.0, 0.7, 4.0, 9.0):
        _certify(R.TS, sd8, b2, abs(z), mean=2.0, z=z)


def test_allowance_edges():
  """ i8_score_err: -1 at sd <= sqrt(b2) and for NaN sd; PI capped at 1, and 1 when sd - b2 / sd <= 0. """
  b2 = 1e-12
  e = R.score_err(R.EI, np.array([1e-6, np.nextafter(1e-6, 1), 0.0, -0.0, np.nan, np.inf]), b2, 0.4)
  assert (e[[0, 2, 3, 4]] == -1.0).all() and e[1] > 0.0 and e[5] == 0.0
  p = R.score_err(R.PI, np.array([np.nextafter(1e-6, 1), 1.0000001e-6, 1e-3]), b2, 0.25)
  assert p[0] == 1.0 and 0.0 < p[2] < 1.0


# ---- the bound pass: ub + pad >= score on the device sequence -------------------------------------------------------
def _pad(kind, sk, beta=0.0, mean_const=0.0, best=0.0):
  """ api.cu: score_argmax_impl's pad = 1e-9 scale. """
  if kind == R.UCB:
    scale = (1.0 + abs(beta)) * sk + abs(mean_const)
  elif kind == R.PI:
    scale = 1.0
  else:
    scale = sk + abs(mean_const) + abs(best)
  return 1e-9 * scale


def _push(sign):
  return R.beyond_fns(sign)


@pytest.mark.parametrize('kind', [R.EI, R.PI, R.UCB])
def test_bound_pass_ub_covers_the_score_under_pushed_functions(kind):
  """ ub = acq(mu_bar, sqrt(k**)) evaluated with erf / erfc / exp pushed down, the score at (mu, sd) with them pushed
  up (beyond the device's documented errors, acq_ref.beyond_fns): ub + pad >= score wherever the bound pass applies
  (EI, UCB with beta >= 0, PI with mu_bar below the incumbent), with pad = 1e-9 scale as api.cu forms it. """
  gaps = GAPS[GAPS < 0.0] if kind == R.PI else GAPS
  for shift in (0, 1, 300):
    sd = SIGMA[:SIGMA.size - shift]
    sk = SIGMA[shift:]                                      # sqrt(k**) >= sd
    for mean_const in (0.0, 1e6):
      for bump in (0.0, 1e-12, 1e-6):
        mu = mean_const + gaps[:, None]
        mub = mu + bump * np.abs(mu) if bump else mu       # mu_bar >= mu
        if kind == R.UCB:
          for beta in (0.0, 0.5, 3.0, 50.0):
            ub = R.acq(kind, mub, sk[None, :], beta=beta)
            s = R.acq(kind, mu, sd[None, :], beta=beta)
            assert (ub + _pad(kind, sk, beta, mean_const)[None, :] >= s).all()
        else:
          # the incumbent at the mean function, or (EI) a mean function far above it
          for best in ((mean_const,) if kind == R.PI or mean_const == 0.0 else (mean_const, 0.0)):
            ub = R.acq(kind, mub, sk[None, :], best=best, fns=_push(-1))
            s = R.acq(kind, mu, sd[None, :], best=best, fns=_push(1))
            pad = np.array([_pad(kind, v, mean_const=mean_const, best=best) for v in sk]) if kind != R.PI else 1e-9
            ok = ub + pad >= s
            # stated for posterior means within 1e6 sqrt(k**) of the mean function: beyond, one ulp of an EI score
            # ~ mu - best may outgrow the pad and the rounding of z and sd z leave ub an ulp below the score
            far = np.abs(mu - mean_const) > 1e6 * sk[None, :]
            assert (ok | far).all(), (kind, shift, mean_const, best, bump, float((s - ub)[~ok & ~far].max()))


# ---- the self-check's rule ------------------------------------------------------------------------------------------
def _model_pairs(rs, n, b2):
  """ (sd8, sd64) with sd8 > sqrt(b2) and |sd64^2 - sd8^2| <= b2: the sigma^2 error model holds. """
  sd8 = np.sqrt(b2) * 10.0 ** rs.uniform(0.001, 4.0, n)
  t = rs.uniform(-1.0, 1.0, n)
  sd64 = np.sqrt(np.maximum(sd8 * sd8 + t * b2 * (1 - 1e-9), 0.0))
  return sd8, sd64


@pytest.mark.parametrize('kind', [R.UCB, R.TS])
def test_selfcheck_does_not_count_rounding_noise(kind):
  """ With a large mean offset one ulp of the score exceeds E: the rule without the slack would void the int8 pass on
  rounding alone, the rule with it counts nothing while the sigma^2 model holds. """
  rs = np.random.RandomState(5)
  bare = 0
  for b2 in (1e-12, 3e-9):
    sd8, sd64 = _model_pairs(rs, 4000, b2)
    for mean in (0.0, 1.0, -37.0, 1e6, 1e9, -3e12, 1e15):
      if kind == R.UCB:
        beta = 3.0
        s8, s64 = R.acq(R.UCB, mean, sd8, beta=beta), R.acq(R.UCB, mean, sd64, beta=beta)
        e = R.score_err(R.UCB, sd8, b2, abs(beta))
      else:
        z = rs.standard_normal(sd8.size) * 3.0
        s8, s64 = R.acq(R.TS, mean, sd8, z=z), R.acq(R.TS, mean, sd64, z=z)
        e = R.score_err(R.TS, sd8, b2, np.abs(z))
      assert R.selfcheck(s8, e, s64) == 0, (b2, mean)
      bare += int((np.abs(s8 - s64) > e).sum())
  assert bare > 0              # the case the slack is for does occur


def test_selfcheck_rule_counts_model_violations():
  b2, beta = 1e-10, 2.0
  sd8 = np.array([1e-3, 1e-2, 1.0])
  sd64 = np.sqrt(sd8 * sd8 + 4.0 * b2)                      # the model fails by a factor 4
  s8, s64 = R.acq(R.UCB, 0.5, sd8, beta=beta), R.acq(R.UCB, 0.5, sd64, beta=beta)
  e = R.score_err(R.UCB, sd8, b2, beta)
  assert R.selfcheck(s8, e, s64) == 3
  assert R.selfcheck(s8, np.full(3, -1.0), s64) == 0        # E < 0: not checked
  assert R.selfcheck(s8, e, np.array([np.nan, s64[1], s64[2]])) == 3


# ---- np.argmax order and the shortlist rule ------------------------------------------------------------------------
def test_argmax_order():
  assert R.argmax([1.0, 3.0, 3.0, 2.0]) == 1
  assert R.argmax([1.0, np.nan, 3.0, np.nan]) == 1
  assert R.argmax([-np.inf, -np.inf]) == 0
  assert R.argmax([np.nan, np.inf]) == 0 and R.argmax([0.0, np.inf, np.nan]) == 2
  assert R.argmax([-0.0, 0.0]) == 0


def test_keep_rule():
  s = np.array([1.0, 0.5, np.nan, 0.2, 0.9])
  e = np.array([0.0, 0.5, 0.1, -1.0, 0.05])
  k = R.keep(s, e, 1.0, 0.05)
  assert k.tolist() == [True, True, True, True, True]
  k = R.keep(s, e, 1.0, 0.0)
  assert k.tolist() == [True, True, True, True, False]      # 0.5 + 0.5 == 1.0 - 0: kept at equality
