"""
The single-precision screen of dfb_score_argmax's bound pass (kernels.cu: prune_bound_kernel) on the device (-m gpu).

mu_bar, read through dfb_mu_upper_bound, must be at least the fp64 mu of every K_* producer -- mean-only dfb_eval
(SEG_MU), the fp64 rows of score_impl = 0 (SEG_ROWS64) and the round-1 kernels of kstar_seg = 0 (FAST_ROWS) -- for
every (kind, d <= 8), on training points, far away, under hallucinated points and at the headline; it is
deterministic and the same for every candidate memory space.  The approximate ex2 / rsqrt instructions it uses must
stay within the error the bound assumes (tests/prune_bound_ref.py: EPS_APPROX), checked once over every float input
in the range the kernel gives them.  At the headline the screen keeps at most 1 % more candidates than an exact-mu
screen against the seed chunk's fp64 maximum would, and the arg-max stays bit-identical with and without the screen
under the digit and K_* options the screen now serves.
"""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest
from scipy.special import ndtr

import kstar_ref as R
import prune_bound_ref as PB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def B():
  import torch
  assert torch.cuda.is_available(), 'these tests need a CUDA device'
  from dragonfly_b200 import kernel, device, synth_data, _lib
  _lib.load()
  return Namespace(torch=torch, kernel=kernel, device=device, synth=synth_data, lib=_lib)


def _post(B, X, Y, kern, noise, chunk=0, **opts):
  post = B.device.DevicePosterior(len(X) + 8, chunk=chunk)
  for k, v in opts.items():
    post.set_option(k, v)
  post.set_kernel(B.kernel.build_descriptor(kern))
  post.set_train(X, Y)
  assert post.build(noise)[0] == 0
  return post


def mu_upper_bound(B, post, Xc, mean_const=0.0, space='device'):
  """ dfb_mu_upper_bound for a host array; space 'device', 'pinned' or 'pageable'. """
  torch = B.torch
  Xh = np.ascontiguousarray(np.asarray(Xc, dtype=np.float64))
  m, dc = Xh.shape
  if space == 'device':
    Xd = torch.from_numpy(Xh).cuda()
    out = torch.empty((m,), dtype=torch.float64, device='cuda')
    B.lib.check(post.lib.dfb_mu_upper_bound(post.h, C.c_void_p(Xd.data_ptr()), m, dc, B.lib.DFB_DEVICE,
                                            float(mean_const), C.c_void_p(out.data_ptr())), 'dfb_mu_upper_bound')
    return out.cpu().numpy()
  if space == 'pinned':
    t = torch.empty((m, dc), dtype=torch.float64, pin_memory=True)
    t.numpy()[:] = Xh
    Xh = t.numpy()
  out = np.empty((m,), dtype=np.float64)
  B.lib.check(post.lib.dfb_mu_upper_bound(post.h, Xh.ctypes.data_as(C.c_void_p), m, dc, B.lib.DFB_HOST,
                                          float(mean_const), out.ctypes.data_as(C.c_void_p)), 'dfb_mu_upper_bound')
  return out


def test_approx_instructions_within_the_assumed_error(B):
  post = B.device.DevicePosterior(64)
  for which, name in ((0, 'ex2.approx.ftz.f32 on [-126, 0]'), (1, 'rsqrt.approx.ftz.f32 on [2^-120, 2^126)')):
    err = C.c_double(0.0)
    B.lib.check(post.lib.dfb_debug_approx_error(post.h, which, C.byref(err)), 'dfb_debug_approx_error')
    print('%s: max relative error %.3e = 2^%.2f (assumed 2^%.0f)' % (name, err.value, np.log2(err.value),
                                                                     np.log2(PB.EPS_APPROX)))
    assert 0.0 < err.value <= PB.EPS_APPROX


def _all_fp64_mus(B, post, C_, mean_const):
  """ mu of mean-only dfb_eval, of the fp64-row producer and of the round-1 kernels. """
  mus = [post.eval(C_, mean_const=mean_const, want_std=False)[0]]
  post.set_option('score_impl', 0)
  mus.append(post.eval(C_, mean_const=mean_const)[0])
  post.set_option('kstar_seg', 0)
  mus.append(post.eval(C_, mean_const=mean_const)[0])
  mus.append(post.eval(C_, mean_const=mean_const, want_std=False)[0])
  post.set_option('kstar_seg', 1)
  post.set_option('score_impl', 2)
  return mus


@pytest.mark.parametrize('d', list(range(1, 9)))
@pytest.mark.parametrize('kname', list(R.KINDS))
def test_bound_holds_for_every_producer(B, kname, d):
  kind, p = R.KINDS[kname]
  rs = np.random.RandomState(70 + d)
  X = rs.random_sample((400, d)); Y = np.sin(3.0 * X).sum(axis=1); Y -= Y.mean()
  bw = list(0.05 + 0.6 * rs.random_sample(d))
  kern = B.kernel.SEKernel(d, 1.3, bw) if kind == 'se' else B.kernel.MaternKernel(d, p + 0.5, 1.3, bw)
  post = _post(B, X, Y, kern, 1e-4)
  C_ = rs.random_sample((3000, d))
  C_[:60] = X[:60]                                                       # on training points
  C_[60:120] = X[60:120] + 1e-7 * rs.standard_normal((60, d))           # next to them
  C_[120:200] = 5.0 + 20.0 * rs.random_sample((80, d))                   # far: k underflows in fp32
  C_[200, 0] = np.nan
  mub = mu_upper_bound(B, post, C_, mean_const=0.3)
  assert np.isnan(mub[200]) and not np.isnan(np.delete(mub, 200)).any()
  for mu in _all_fp64_mus(B, post, C_, 0.3):
    ok = np.delete(mub >= mu, 200)
    assert ok.all(), (np.flatnonzero(~ok)[:5], float(np.max(np.delete(mu - mub, 200))))
  slack = np.delete(mub - _all_fp64_mus(B, post, C_, 0.3)[0], 200)
  print('%s d=%d: mu_bar - mu median %.2e, max %.2e' % (kname, d, np.median(slack), slack.max()))


def test_bound_holds_under_hallucinated_points(B):
  rs = np.random.RandomState(5)
  X = rs.random_sample((600, 6)); Y = np.cos(2.0 * X).sum(axis=1); Y -= Y.mean()
  post = _post(B, X, Y, B.kernel.MaternKernel(6, 2.5, 0.8, 0.3), 1e-3)
  _, alpha, _ = post.get_state(want_alpha=True)
  Xh = rs.random_sample((5, 6))
  assert post.extend(Xh, np.zeros(5), save=True)[0] == 0
  post.set_alpha(alpha)                     # alpha = 0 on the hallucinated points
  try:
    C_ = np.vstack([rs.random_sample((2000, 6)), Xh])
    mub = mu_upper_bound(B, post, C_)
    for mu in _all_fp64_mus(B, post, C_, 0.0):
      assert (mub >= mu).all()
  finally:
    post.restore(600)


# ---- the headline ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def headline(B):
  w = B.synth.make_workload('headline_hartmann6_matern_ei', n_cand=16)
  k = w['kernel']
  kern = B.kernel.MaternKernel(6, 2.5, k['scale'], k['dim_bandwidths'])
  Yc = w['Y'] - w['mean_const']
  post = _post(B, w['X'], Yc, kern, w['noise_var'])
  host = np.random.RandomState(1000).random_sample((1000000, 6))           # bench.py's rank-0 candidates
  return Namespace(w=w, k=k, kern=kern, Yc=Yc, post=post, host=host)


def test_headline_bound_deterministic_and_space_independent(B, headline):
  post, w = headline.post, headline.w
  mub = mu_upper_bound(B, post, headline.host, w['mean_const'])
  mu = post.eval(B.torch.from_numpy(headline.host).cuda(), mean_const=w['mean_const'], want_std=False)[0].cpu().numpy()
  assert (mub >= mu).all()
  print('headline: mu_bar - mu median %.2e, max %.2e' % (np.median(mub - mu), (mub - mu).max()))
  again = mu_upper_bound(B, post, headline.host, w['mean_const'])
  assert (again.view(np.int64) == mub.view(np.int64)).all()
  sub = headline.host[:200000]
  for space in ('pinned', 'pageable'):
    other = mu_upper_bound(B, post, sub, w['mean_const'], space=space)
    assert (other.view(np.int64) == mub[:200000].view(np.int64)).all(), space


def _ei(mu, sd, best):
  z = (mu - best) / sd
  return sd * (z * ndtr(z) + np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi))


def test_headline_survivors_close_to_an_exact_screen(B, headline):
  post, w = headline.post, headline.w
  chunk = int(post.query('chunk'))
  Cd = B.torch.from_numpy(headline.host).cuda()
  acq = B.device.make_acq_desc('ei', best=float(w['Y'].max()))
  post.score_argmax(acq, Cd, mean_const=w['mean_const'])
  surv = post.query('last_survivors')
  seed_best = post.score_argmax(acq, Cd[:chunk], mean_const=w['mean_const'])[0]
  mu = post.eval(Cd[chunk:], mean_const=w['mean_const'], want_std=False)[0].cpu().numpy()
  kss = float(B.kernel.build_descriptor(headline.kern).kss)
  ub = _ei(mu, np.sqrt(kss), float(w['Y'].max()))
  count = int((ub >= seed_best).sum())
  print('headline EI: survivors %d, exact-mu screen against the seed maximum %d' % (surv, count))
  assert surv <= 1.01 * count


@pytest.mark.parametrize('opts', [{}, {'i8_radix': 0}, {'kstar_seg': 0}])
def test_headline_argmax_bit_identical(B, headline, opts):
  w = headline.w
  Cd = B.torch.from_numpy(headline.host).cuda()
  acq = B.device.make_acq_desc('ei', best=float(w['Y'].max()))
  res = []
  for extra in ({'prune': 1}, {'prune': 0}, {'score_impl': 0}):
    p = _post(B, w['X'], headline.Yc, headline.kern, w['noise_var'], **dict(opts, **extra))
    s, i, _ = p.score_argmax(acq, Cd, mean_const=w['mean_const'])
    if extra.get('prune') == 1:
      assert p.query('last_used_i8') == 1.0 and p.query('last_pruned_candidates') > 0
    res.append((np.float64(s).view(np.int64), i))
    del p
  assert res[0] == res[1] == res[2], res
