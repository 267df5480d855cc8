"""
The acquisition epilogue on the device (-m gpu) against the extended-precision reference of tests/acq_ref.py:
  A1  UCB, EI, PI, TTEI and TS from the real acq_kernel (dfb_debug_acq) on synthetic (mu, partials, k**) over z in
      [-40, 40], z = +-1 +- 1 ulp, sigma^2 = 0, -0.0, negative and subnormal, mu - best = +-0, infinite mu, best and
      beta, TTEI with ref_std = 0 and sigma = 0: every finite score within the device bound of the mpmath value, the NaN,
      infinity, zero and subnormal positions those of the NumPy restatement, UCB, TS and sigma bit for bit;
  A2  the same bound on a real posterior (Matern-5/2, N = 1100): scores of dfb_score_argmax against dfb_eval's mu, sd;
  A3  the arg-max across block and chunk edges equals np.argmax of the returned scores (NaN first, lowest index);
  A4  the shortlist equals the keep rule applied to the device's own scores and allowances;
  A5  the allowance E on the device -- with the sensitivity dfb_score_argmax uses -- bounds the extended-precision
      supremum and its constants are at least sup phi and sup |z phi|, the self-check counts what its rule says,
      and the int8 path with a large mean offset reports no self-check violation;
  A6  the bound pass's ub + pad is at least the fp64 score of the same row, at kernel scales 1e-2 .. 1e4;
  A7  the golden arg-max assertions of test_gpu_parity.py (c1 UCB, EI, PI, TTEI; matern_h6 UCB, EI) and the headline
      EI / UCB of test_gpu_baseline_sizes.py have a top-two margin above 1e12 times the combined device + cephes error
      of the epilogue.
"""
from argparse import Namespace

import numpy as np
import pytest

import acq_ref as R

pytestmark = pytest.mark.gpu

CHUNK = 1024


@pytest.fixture(scope='module')
def G():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import device, kernel, synth_data, _lib
  _lib.load()
  return Namespace(torch=torch, device=device, kernel=kernel, synth=synth_data, lib=_lib,
                   post=device.DevicePosterior(64, chunk=CHUNK))


def _cuda(G, a):
  return G.torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _np(t):
  return t.cpu().numpy()


def _bits(a):
  return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _desc(G, kind, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0):
  a = G.lib.AcqDesc()
  a.kind, a.beta, a.best, a.ref_mean, a.ref_std = kind, float(beta), float(best), float(ref_mean), float(ref_std)
  return a


def _run(G, kind, mean, partial, kss, z=None, **kw):
  par = {k: kw.pop(k) for k in ('beta', 'best', 'ref_mean', 'ref_std') if k in kw}
  return G.post.debug_acq(_desc(G, kind, **par), _cuda(G, mean), _cuda(G, partial) if partial is not None else None,
                          _cuda(G, kss), z=_cuda(G, z) if z is not None else None, **kw)


def _classes(s):
  s = np.asarray(s)
  with np.errstate(all='ignore'):
    return np.stack([np.isnan(s), np.isposinf(s), np.isneginf(s), s == 0, np.signbit(s),
                     np.isfinite(s) & (np.abs(s) < 2.2250738585072014e-308) & (s != 0)])


# ---- A1: synthetic inputs -------------------------------------------------------------------------------------------
def _synthetic(rs):
  """ (mean, partial (2 x m), kss, best): the z grid at several sd, plus the sigma^2 and mu - best edges. """
  pos = np.geomspace(1e-9, 40.0, 160)
  z = np.concatenate([-pos[::-1], [0.0, -0.0], pos, [1.0, -1.0, np.nextafter(1.0, 2), np.nextafter(1.0, 0),
                                                       np.nextafter(-1.0, -2), np.nextafter(-1.0, 0)]])
  rows = []
  for sd_t in (1.0, 3.7e-3, 2.5e5, 1e-160):
    vn = rs.uniform(0.0, 1.0, (2, z.size)) * sd_t * sd_t
    kss = sd_t * sd_t + vn[0] + vn[1]
    rows.append((z, vn, kss))
  best = 0.75
  zz = np.concatenate([r[0] for r in rows])
  part = np.concatenate([r[1] for r in rows], axis=1)
  kss = np.concatenate([r[2] for r in rows])
  sd = R.sigma(part, kss)
  mean = best + zz * sd
  # edges: sigma^2 = 0, -0.0, negative, subnormal; mu - best = +-0 (at sigma > 0 and at sigma = 0); a NaN mu
  e_kss = np.array([0.5, -0.0, 0.25, 1e-310, 1e-318, 1.0, 1.0, 0.5, 0.5, 1.0])
  e_part = np.array([[0.25, 0.0, 0.5, 0.0, 0.0, 0.0, 0.0, 0.25, 0.25, 0.0],
                     [0.25, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.25, 0.25, 0.0]])
  e_mean = np.array([best + 1.0, best, best - 2.0, best + 1e-160, best, best, best, best, best - 1.0, np.nan])
  return (np.concatenate([mean, e_mean]), np.concatenate([part, e_part], axis=1), np.concatenate([kss, e_kss]), best)


def _check_scores(kind, s_dev, mean, sd, **kw):
  s_ref = R.acq(kind, mean, sd, **kw)
  np.testing.assert_array_equal(_classes(s_dev), _classes(s_ref))
  if kind in (R.UCB, R.TS):
    assert (_bits(s_dev) == _bits(s_ref)).all()
  pos = (np.sqrt(kw.get('ref_std', 0.0) ** 2 + sd * sd) > 0) if kind == R.TTEI else (sd > 0)
  fin = np.isfinite(s_dev) & pos
  bnd = R.bound(kind, mean, sd, **kw)
  err = R.errors(kind, np.where(fin, s_dev, np.nan), mean, np.where(fin, sd, 1.0), **kw)
  ok = ~fin | (err <= bnd)
  assert ok.all(), (kind, mean[~ok][:4], sd[~ok][:4], err[~ok][:4], bnd[~ok][:4])
  return float(np.nanmax(np.where(fin, err / bnd, np.nan)))


@pytest.mark.parametrize('name', ['ucb', 'ei', 'pi', 'ttei', 'ts'])
def test_a1_synthetic_scores(G, name):
  kind = R.KINDS[name]
  rs = np.random.RandomState(11)
  mean, part, kss, best = _synthetic(rs)
  sd_ref = R.sigma(part, kss)
  variants = {'ucb': [dict(beta=2.5), dict(beta=0.0), dict(beta=-1.5)],
              'ei': [dict(best=best)], 'pi': [dict(best=best)],
              'ttei': [dict(ref_mean=best, ref_std=0.0), dict(ref_mean=best, ref_std=0.3),
                       dict(ref_mean=best, ref_std=1e-170)],
              'ts': [dict(z=rs.standard_normal(mean.size) * 3.0)]}[name]
  worst = 0.0
  for kw in variants:
    out = _run(G, kind, mean, part, kss, **kw)
    sd = _np(out.sd)
    assert (_bits(sd) == _bits(sd_ref)).all()
    s = _np(out.scores)
    worst = max(worst, _check_scores(kind, s, mean, sd, **kw))
    assert out.index == R.argmax(s) and (_bits(out.score) == _bits(s[out.index]))
  print('A1 %s: largest |error| / bound = %.3f' % (name, worst))


def test_a1_ei_bit_for_bit_where_the_functions_are_exact(G):
  """ z >= 40: erfc(z / sqrt 2) < 2^-1074 / 2 and exp(-z^2 / 2) underflows, so Phi = 1 and phi ~ 0 are exact after
  rounding whatever the functions' few ulps, and EI = fl(sd fl((mean - best) / sd)), TTEI = fl(comb fl(d / comb)):
  the score pins the rounding of z itself. """
  rs = np.random.RandomState(13)
  m = 4000
  sd = 10.0 ** rs.uniform(-6.0, 3.0, m)
  z = 10.0 ** rs.uniform(np.log10(40.0), 8.0, m)
  best = rs.uniform(-5.0, 5.0, m)
  mean = best + z * sd
  kss = sd * sd
  sd_dev = R.sigma(np.zeros((0, m)), kss)
  for kind in (R.EI, R.TTEI):
    for b in (0.25, -3.0):
      kw = dict(best=b) if kind == R.EI else dict(ref_mean=b, ref_std=0.3 * b * b)
      mb = mean - best + b
      out = _run(G, kind, mb, None, kss, **kw)
      s = _np(out.scores)
      with np.errstate(all='ignore'):
        comb = np.sqrt(kw.get('ref_std', 0.0) ** 2 + sd_dev * sd_dev) if kind == R.TTEI else sd_dev
        zc = (mb - b) / comb
      sel = zc >= 40.0
      assert sel.sum() > m // 2
      want = comb * zc
      assert (_bits(s[sel]) == _bits(want[sel])).all(), (kind, int((_bits(s[sel]) != _bits(want[sel])).sum()))


def test_a1_ts_generated_normals(G):
  rs = np.random.RandomState(12)
  mean, part, kss, _ = _synthetic(rs)
  out = _run(G, R.TS, mean, part, kss, seed=77)
  z = _np(G.post.fill_rng(77, 0, 1, mean.size)[0])
  s = _np(out.scores)
  assert (_bits(s) == _bits(R.acq(R.TS, mean, _np(out.sd), z=z))).all()


@pytest.mark.parametrize('case', ['mean_inf', 'best_inf', 'beta_inf'])
def test_a1_infinite_inputs(G, case):
  m = 6
  kss = np.array([1.0, 1.0, 0.0, 4.0, 1.0, 1.0])
  mean = np.array([np.inf, -np.inf, 1.0, 0.0, np.inf, 2.0]) if case == 'mean_inf' else np.linspace(-1, 1, m)
  best = np.inf if case == 'best_inf' else (-np.inf if case == 'mean_inf' else 0.0)
  beta = np.inf if case == 'beta_inf' else 1.0
  sd = R.sigma(np.zeros((0, m)), kss)
  for kind, kw in ((R.UCB, dict(beta=beta)), (R.EI, dict(best=best)), (R.PI, dict(best=best)),
                   (R.TTEI, dict(ref_mean=best, ref_std=0.0))):
    out = _run(G, kind, mean, None, kss, **kw)
    s = _np(out.scores)
    np.testing.assert_array_equal(_classes(s), _classes(R.acq(kind, mean, sd, **kw)))
    assert out.index == R.argmax(s)


# ---- A2: a real posterior -------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def real(G):
  rs = np.random.RandomState(21)
  X = rs.random_sample((1100, 6))
  Y = G.synth.hartmann6(X)
  Y = Y - float(np.median(Y))
  kern = G.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)
  C = rs.random_sample((3000, 6))
  posts = {}
  for impl in (0, 2):
    p = G.device.DevicePosterior(1108, chunk=CHUNK)
    p.set_option('score_impl', impl)
    p.set_kernel(G.kernel.build_descriptor(kern))
    p.set_train(X, Y)
    assert p.build(0.01 * float(Y.var()))[0] == 0
    posts[impl] = p
  return Namespace(X=X, Y=Y, C=C, posts=posts, kern=kern)


@pytest.mark.parametrize('impl', [0, 2])
@pytest.mark.parametrize('name', ['ucb', 'ei', 'pi', 'ttei'])
def test_a2_real_posterior_scores_within_the_bound(G, real, impl, name):
  post = real.posts[impl]
  mu, sd = post.eval(real.C)
  best = float(real.Y.max())
  kw = {'ucb': dict(beta=2.2), 'ei': dict(best=best), 'pi': dict(best=best),
        'ttei': dict(ref_mean=float(mu[7]), ref_std=float(sd[7]))}[name]
  kind = R.KINDS[name]
  bs, bi, s = post.score_argmax(_desc(G, kind, **kw), real.C, want_scores=True)
  assert post.query('last_used_i8') == 0.0
  ratio = _check_scores(kind, s, mu, sd, **kw)
  assert bi == R.argmax(s) and _bits(bs) == _bits(s[bi])
  print('A2 %s impl %d: largest |error| / bound = %.3f' % (name, impl, ratio))


# ---- A3: the arg-max across edges -----------------------------------------------------------------------------------
def _argmax_case(G, scores):
  """ UCB with beta = 0 and sd = 1: the score is mu itself (mu + 0, so -0.0 reads as +0.0). """
  m = scores.size
  out = _run(G, R.UCB, scores, None, np.ones(m), beta=0.0)
  s = _np(out.scores)
  want = R.argmax(s)
  assert out.index == want, (m, out.index, want)
  assert _bits(out.score) == _bits(s[want])


@pytest.mark.parametrize('m', [1, 255, 256, 257, CHUNK - 1, CHUNK + 1, 3 * CHUNK + 17])
def test_a3_argmax_edges(G, m):
  rs = np.random.RandomState(m)
  base = rs.uniform(-1.0, 0.0, m)
  _argmax_case(G, base)
  for i, j in ((255, 256), (CHUNK - 1, CHUNK), (m - 2, m - 1), (0, m - 1)):     # exact ties across block / chunk edges
    if 0 <= i < j < m:
      s = base.copy()
      s[i] = s[j] = 5.0
      _argmax_case(G, s)
      s[j] = np.nextafter(5.0, 6.0)
      _argmax_case(G, s)
  s = base.copy()
  s[m - 1] = np.nan                                           # NaN in the last (partial) block
  _argmax_case(G, s)
  if m > 3:
    s[m // 2] = np.nan
    _argmax_case(G, s)
  _argmax_case(G, np.full(m, -np.inf))
  s = np.full(m, np.nan)
  s[m // 2] = np.inf                                          # one +inf among NaNs: the first NaN wins
  _argmax_case(G, s)
  s = np.full(m, -np.inf)
  s[m - 1] = np.inf
  _argmax_case(G, s)


# ---- A4: the shortlist ----------------------------------------------------------------------------------------------
def _shortlist(G, out, m):
  n = min(out.count, 4096)
  idx = _np(G.post.debug_buffer('list_idx', G.torch.int64, 4096))[:n]
  s8 = _np(G.post.debug_buffer('list_s8', G.torch.float64, 4096))[:n]
  err = _np(G.post.debug_buffer('list_err', G.torch.float64, 4096))[:n]
  return idx, s8, err


def _check_shortlist(G, kind, mean, kss, b2, sens, pad, init, z=None, **kw):
  m = mean.size
  out = _run(G, kind, mean, None, kss, z=z, b2=b2, sens=sens, pad=pad, best_lb=init, **kw)
  s, sd = _np(out.scores), _np(out.sd)
  e = R.score_err(kind, sd, b2, np.abs(z) if kind == R.TS else sens)
  lbs = R.running_best_lb(s, e, CHUNK, init)
  assert _bits(out.best_lb) == _bits(lbs[-1])
  want = R.shortlist(s, e, CHUNK, pad, init)
  assert out.count == want.size
  idx, s8, err = _shortlist(G, out, m)
  order = np.argsort(idx)
  assert (idx[order] == np.sort(want)).all()
  assert (_bits(s8[order]) == _bits(s[idx[order]])).all()
  assert (_bits(err[order]) == _bits(np.where(np.isnan(s[idx[order]]), -1.0, e[idx[order]]))).all()
  return out, s, e


def test_a4_shortlist_edges(G):
  m = 2 * CHUNK + 300
  rs = np.random.RandomState(41)
  b2, beta, pad = 2.0 ** -20, 1.0, 2.0 ** -10
  mean = rs.uniform(-3.0, -0.5, m)
  kss = np.ones(m)
  init = 1.0                                   # above every lower bound: the keep threshold is init - pad throughout
  E = beta * b2                                # sd = 1, s = mean + 1
  mean[[5, CHUNK + 3, m - 1]] = (init - pad - E) - 1.0                      # s + E == best_lb - pad exactly: kept
  mean[[6, CHUNK + 4]] = np.nextafter(init - pad - E, -1) - 1.0            # just below: dropped
  mean[[7, 2 * CHUNK + 1]] = np.nan                         # NaN score, finite sigma
  kss[[8, CHUNK + 9]] = b2                                  # sd = sqrt(b2): E = -1, always kept
  kss[10] = b2 * 0.25
  out, s, e = _check_shortlist(G, R.UCB, mean, kss, b2, beta, pad, init, beta=beta)
  assert s[5] + e[5] == init - pad and s[6] + e[6] < init - pad and out.best_lb == init
  for kind, kw, sens in ((R.EI, dict(best=0.3), 0.4), (R.PI, dict(best=0.3), 0.25),
                         (R.TTEI, dict(ref_mean=0.3, ref_std=0.2), 0.4)):
    _check_shortlist(G, kind, rs.uniform(-1.0, 1.0, m), rs.uniform(1e-6, 2.0, m), 1e-9, sens, 1e-3, -np.inf, **kw)
  z = rs.standard_normal(m) * 3.0
  _check_shortlist(G, R.TS, rs.uniform(-1.0, 1.0, m), rs.uniform(1e-6, 2.0, m), 1e-9, 0.0, 1e-3, -np.inf, z=z)


def test_a4_shortlist_overflow(G):
  m = CHUNK
  mean = np.zeros(m)                           # every candidate within reach, fewer than the cap of 4096
  out = _run(G, R.UCB, mean, None, np.ones(m), beta=1.0, b2=1e-9, sens=1.0, pad=1.0)
  assert out.count == m
  big = 4096 + 3 * CHUNK + 5                   # several chunks of ties: the list overflows, the count says so
  out = _run(G, R.UCB, np.zeros(big), None, np.ones(big), beta=1.0, b2=1e-9, sens=1.0, pad=1.0)
  assert out.count > 4096


# ---- A5: the allowance and the self-check on the device -------------------------------------------------------------
@pytest.mark.parametrize('name', ['ucb', 'ei', 'pi', 'ttei', 'ts'])
def test_a5_allowance_covers_the_supremum(G, name):
  kind = R.KINDS[name]
  worst = 0.0
  for b2 in (1e-18, 1e-12, 5e-9):
    r = np.sqrt(b2)
    sd8 = np.array([r * (1 + 2.0 ** -20), r * 1.5, r * 10.0, 1e-3, 1.0, 1e3])
    sd8 = sd8[sd8 > r]
    zs = np.array([-5.0, -1.0, 0.0, 1.0, 5.0])
    sdv, zv = np.repeat(sd8, zs.size), np.tile(zs, sd8.size)
    kw = {'ucb': dict(beta=3.0), 'ei': dict(best=0.0), 'pi': dict(best=0.0),
          'ttei': dict(ref_mean=0.0, ref_std=0.5), 'ts': dict(z=zv * 1.7)}[name]
    comb = np.sqrt(0.25 + sdv * sdv) if kind == R.TTEI else sdv
    mean = zv * comb
    out = _run(G, kind, mean, None, sdv * sdv, b2=b2, pad=np.inf, **kw)      # sens: what dfb_score_argmax uses
    sd_dev = _np(out.sd)
    idx, s8, err = _shortlist(G, out, mean.size)
    assert out.count == mean.size
    e = np.empty(mean.size)
    e[idx] = err
    sens = np.abs(kw['z']) if kind == R.TS else R.sens_of(kind, kw.get('beta', 0.0))
    assert (_bits(e) == _bits(R.score_err(kind, sd_dev, b2, sens))).all()
    _check_sensitivity(kind, sd_dev, b2, e, kw)
    for i in range(mean.size):
      if e[i] < 0:
        assert not sd_dev[i] > r
        continue
      kwi = dict(kw)
      if kind == R.TS:
        kwi['z'] = float(kw['z'][i])
      sup = R.allowance_sup(kind, sd_dev[i], b2, mean=mean[i], **kwi)
      assert sup <= R.mp.mpf(float(e[i])), (name, b2, sd_dev[i], mean[i], float(sup), e[i])
      worst = max(worst, float(sup / R.mp.mpf(float(e[i]))) if e[i] > 0 else 0.0)
  print('A5 %s: largest sup / E = %.4f' % (name, worst))


def _check_sensitivity(kind, sd, b2, e, kw):
  """ The constant behind the device's allowance, recovered from E itself, is at least the supremum it stands for:
  sup phi = phi(0) (EI, TTEI), sup |z phi(z)| = phi(1) (PI), |beta| (UCB), |z_i| (TS). """
  ok = e > 0
  with np.errstate(all='ignore'):
    q = b2 / sd                                                # fl(b2 / sd), as i8_score_err forms it
    if kind == R.PI:
      ok &= e < 1.0
      c = e * (sd - q) / q
      need = float(R.mp.npdf(1))
    elif kind in (R.EI, R.TTEI):
      c, need = e / q, float(R.mp.npdf(0))
    elif kind == R.UCB:
      c, need = e / q, abs(kw['beta'])
    else:
      c, need = e / q, np.abs(kw['z'])
  need = np.broadcast_to(need, e.shape)
  assert (c[ok] * (1 + 1e-12) >= need[ok]).all(), (kind, float(np.min(c[ok] / need[ok])))


def test_a5_selfcheck_counts_its_rule(G):
  rs = np.random.RandomState(51)
  n = 3000
  b2 = 3e-9
  sd8 = np.sqrt(b2) * 10.0 ** rs.uniform(0.01, 3.0, n)
  t = rs.uniform(-1.0, 1.0, n)
  viol = rs.random_sample(n) < 0.1
  sd64 = np.sqrt(sd8 * sd8 + t * b2 * np.where(viol, 8.0, 0.999))     # 10 % break the sigma^2 model
  mean = np.where(rs.random_sample(n) < 0.5, 0.3, 1e12)                # half with a large mean offset
  s8, s64 = R.acq(R.UCB, mean, sd8, beta=3.0), R.acq(R.UCB, mean, sd64, beta=3.0)
  e = R.score_err(R.UCB, sd8, b2, 3.0)
  e[::97] = -1.0
  s64[::89] = np.nan
  count, ratio = G.post.debug_selfcheck(_cuda(G, s8), _cuda(G, e), _cuda(G, s64))
  assert count == R.selfcheck(s8, e, s64), (count, R.selfcheck(s8, e, s64))
  assert count > 0


@pytest.mark.parametrize('mean_const', [0.0, 1e6, 1e9, -1e12])
def test_a5_int8_path_with_a_large_mean_offset(G, mean_const):
  """ score_impl = 1 with small k** (the guard admits it) and a large mean offset: the self-check must not void the
  int8 pass on rounding alone, and the arg-max is the fp64 one. """
  rs = np.random.RandomState(52)
  X = rs.random_sample((1100, 6))
  Y = G.synth.hartmann6(X) * 1e-2
  Y = Y - float(np.median(Y))
  kern = G.kernel.MaternKernel(6, 2.5, float(Y.var()), 0.3)
  C = rs.random_sample((4000, 6))
  res = {}
  for impl in (1, 0):
    p = G.device.DevicePosterior(1108, chunk=CHUNK)
    p.set_option('score_impl', impl)
    p.set_kernel(G.kernel.build_descriptor(kern))
    p.set_train(X, Y)
    assert p.build(0.01 * float(Y.var()))[0] == 0
    for name in ('ucb', 'ei'):
      acq = _desc(G, R.KINDS[name], beta=3.0, best=mean_const + float(Y.max()))
      bs, bi, _ = p.score_argmax(acq, C, mean_const=mean_const)
      res[(impl, name)] = (bs, bi)
      if impl == 1:
        v = p.query('last_selfcheck_violations')
        print('A5 mean_const %g %s: used_i8 %d shortlist %d violations %d ratio %.3g b2 %.3g' % (
            mean_const, name, p.query('last_used_i8'), p.query('last_shortlist'), v,
            p.query('last_selfcheck_ratio'), p.query('i8_sigma2_bound')))
        assert p.query('last_used_i8') == 1.0
        assert v == 0.0
  for name in ('ucb', 'ei'):
    assert res[(1, name)][1] == res[(0, name)][1] and _bits(res[(1, name)][0]) == _bits(res[(0, name)][0])


# ---- A6: the bound pass's ub ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('scale', [1e-2, 1.0, 1e2, 1e4])
@pytest.mark.parametrize('mean_const', [0.0, 1e3, 1e6])
def test_a6_bound_pass_ub_covers_the_score(G, scale, mean_const):
  rs = np.random.RandomState(61)
  X = rs.random_sample((1100, 6))
  Y = G.synth.hartmann6(X)
  Y = (Y - float(np.median(Y))) * np.sqrt(scale / float(Y.var()))
  kern = G.kernel.MaternKernel(6, 2.5, scale, 0.3)
  noise = 0.01 * scale
  C = G.torch.from_numpy(rs.random_sample((3 * CHUNK, 6))).cuda()
  pr = G.device.DevicePosterior(1108, chunk=CHUNK)
  pr.set_option('score_impl', 2)
  if scale > 1.0:
    pr.set_option('i8_unguarded', 1)           # the int8 guard (b2 <= 5e-9 absolute) would keep the bound pass off
  pr.set_kernel(G.kernel.build_descriptor(kern))
  pr.set_train(X, Y)
  assert pr.build(noise)[0] == 0
  ex = G.device.DevicePosterior(1108, chunk=CHUNK)
  ex.set_option('score_impl', 0)
  ex.set_kernel(G.kernel.build_descriptor(kern))
  ex.set_train(X, Y)
  assert ex.build(noise)[0] == 0
  sk = np.sqrt(scale)
  ran = 0
  for name in ('ei', 'pi', 'ucb'):
    best = mean_const + float(Y.max())
    acq = _desc(G, R.KINDS[name], beta=2.0, best=best)
    bs, bi, _ = pr.score_argmax(acq, C, mean_const=mean_const)
    if pr.query('last_seed_rows') == 0:
      continue                                 # the int8 guard or the variance floor keeps the bound pass off
    ran += 1
    ub = _np(pr.debug_buffer('prune_ub', G.torch.float64, int(pr.query('keep_cap'))))[:C.shape[0]]
    _, bi0, s = ex.score_argmax(acq, C, mean_const=mean_const, want_scores=True)
    s = _np(s)
    assert bi == bi0
    scl = {'ucb': 3.0 * sk + abs(mean_const), 'pi': 1.0, 'ei': sk + abs(mean_const) + abs(best)}[name]
    pad = 1e-9 * scl
    gap = (ub + pad) - s
    assert (gap >= 0).all(), (name, scale, mean_const, float(gap.min()))
    tight = np.min(np.where(np.isfinite(ub), gap / pad, np.inf))
    print('A6 scale %g mean_const %g %s: min (ub + pad - score) / pad = %.6g' % (scale, mean_const, name, tight))
  assert ran == 3


# ---- A7: the margin of the golden arg-max assertions ----------------------------------------------------------------
MARGIN = 1e12          # the smallest top-two gap of these cases, in units of the combined error bound, is 1.4e12


def _margin(kind, scores, mean, sd, **kw):
  """ top-two gap of the reference's scores and the combined device + cephes bound at those two candidates. """
  i1 = R.argmax(scores)
  rest = np.where(np.arange(scores.size) == i1, -np.inf, scores)
  i2 = R.argmax(rest)
  idx = np.array([i1, i2])
  b = (R.bound(kind, mean[idx], sd[idx], **kw) + R.bound(kind, mean[idx], sd[idx], ulp=R.ULP_CEPHES, **kw)).sum()
  return float(scores[i1] - scores[i2]), float(b)


def _golden_cases():
  from conftest import load_golden
  g = load_golden('c1_se')
  ri = int(g['ttei_ref_idx'])
  yield 'c1_ucb', R.UCB, g['ucb'], g['mu'], g['sd'], dict(beta=float(g['beta']))
  yield 'c1_ei', R.EI, g['ei'], g['mu'], g['sd'], dict(best=float(g['curr_best']))
  yield 'c1_pi', R.PI, g['pi'], g['mu'], g['sd'], dict(best=float(g['curr_best']))
  yield 'c1_ttei', R.TTEI, g['ttei'], g['mu'], g['sd'], dict(ref_mean=float(g['mu'][ri]), ref_std=float(g['sd'][ri]))
  h = load_golden('matern_h6')
  for tag in ('0p5', '1p5', '2p5'):
    yield 'h6_ucb_' + tag, R.UCB, h['ucb_' + tag], h['mu_' + tag], h['sd_' + tag], dict(beta=float(h['beta']))
    yield 'h6_ei_' + tag, R.EI, h['ei_' + tag], h['mu_' + tag], h['sd_' + tag], dict(best=float(h['curr_best']))


def test_a7_golden_argmax_margins():
  for name, kind, scores, mean, sd, kw in _golden_cases():
    gap, b = _margin(kind, np.asarray(scores), np.asarray(mean), np.asarray(sd), **kw)
    print('A7 %s: top-two gap %.3e, epilogue error bound %.3e (%.1e x)' % (name, gap, b, gap / b))
    assert gap > MARGIN * b, name


def test_a7_baseline_size_margins():
  """ The headline workload of test_gpu_baseline_sizes.py (N = 5000, 2560 candidates) on the oracle's mu and sigma. """
  from dragonfly_b200 import synth_data
  from oracle import gp_oracle as O
  w = synth_data.make_workload('headline_hartmann6_matern_ei', n_cand=2560)
  k = w['kernel']
  ogp = O.OGP(w['X'], w['Y'], O.OMaternKernel(6, 2.5, k['scale'], k['dim_bandwidths']),
              lambda x: np.array([w['mean_const']] * len(x)), w['noise_var'])
  mu, var = O.eval_std_diag(ogp, w['candidates'])
  sd = np.sqrt(var)
  best = float(w['Y'].max())
  beta = O.ucb_beta_th(6, 5000)
  for name, kind, scores, kw in (('ei', R.EI, O.acq_ei(mu, sd, best), dict(best=best)),
                                 ('ucb', R.UCB, O.acq_ucb(mu, sd, beta), dict(beta=beta))):
    gap, b = _margin(kind, np.asarray(scores), mu, sd, **kw)
    print('A7 headline %s: top-two gap %.3e, epilogue error bound %.3e (%.1e x)' % (name, gap, b, gap / b))
    assert gap > MARGIN * b, name
