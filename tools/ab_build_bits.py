"""Bit-for-bit A/B of the posterior build between two libraries (DFB200_LIB), each run in its own process.

Compares the tall factorisation matrix T (dfb_debug_copy "T": L, L^-T and (L^-1 y)^T), W = L^-1, alpha, the LML and
`info` for full, NO_ALPHA and LML-only builds at N = 1, 127, 128, 129, 300, 1100 and 5000 with the look-ahead
schedule on and off; a build with jitter; a build that is not positive definite; an extend + restore; one Thompson
block (dfb_eval_covar and dfb_ts_draws).  Buffers are compared by SHA-256 of their bytes, scalars by their bit pattern.

Usage: python tools/ab_build_bits.py OLD.so NEW.so      (exit status 1 on any difference)"""
import hashlib
import json
import os
import struct
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = (1, 127, 128, 129, 300, 1100, 5000)


def digest(t):
  return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


def bits(x):
  return None if x is None else struct.pack('<d', float(x)).hex()


def run_child():
  sys.path.insert(0, ROOT)
  import numpy as np
  import torch
  from dragonfly_b200 import synth_data, kernel, device, _lib
  spec = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=5000, n_cand=16)
  ks = spec['kernel']
  desc = kernel.build_descriptor(kernel.MaternKernel(6, 2.5, ks['scale'], ks['dim_bandwidths']))
  noise = spec['noise_var']
  out = {}

  def buffers(post, key, info, lml):
    npad = (post.n + 127) // 128 * 128
    rec = {'info': int(info), 'lml': bits(lml)}
    for name, count in (('T', (2 * npad + 128) * npad), ('W', npad * npad), ('alpha', npad)):
      buf = torch.empty(count, dtype=torch.float64, device='cuda')
      _lib.check(post.lib.dfb_debug_copy(post.h, name.encode(), buf.data_ptr(), 8 * count), 'dfb_debug_copy')
      rec[name] = digest(buf)
    out[key] = rec

  flag_sets = (('full', _lib.DFB_BUILD_FULL), ('no_alpha', _lib.DFB_BUILD_NO_ALPHA),
               ('lml_only', _lib.DFB_BUILD_LML_ONLY))
  for n in SIZES:
    w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=n, n_cand=16)
    yc = w['Y'] - w['mean_const']
    for la in (0, 1):
      post = device.DevicePosterior(n)
      post.set_option('lookahead', la)
      post.set_kernel(desc)
      post.set_train(w['X'], yc)
      for name, flags in flag_sets:
        info, lml = post.build(noise, 0.0, flags)
        buffers(post, 'N%d_la%d_%s' % (n, la, name), info, lml)
      if n == 1100:
        info, lml = post.build(noise, 1e-6 * ks['scale'], _lib.DFB_BUILD_FULL)
        buffers(post, 'N%d_la%d_jitter' % (n, la), info, lml)
        info, lml = post.build(-2.0 * ks['scale'], 0.0, _lib.DFB_BUILD_FULL)
        buffers(post, 'N%d_la%d_not_pd' % (n, la), info, lml)
      del post
  # extend + restore: N = 1100 -> 1120 inside the same padded size
  w = synth_data.make_workload('headline_hartmann6_matern_ei', n_train=1120, n_cand=16)
  yc = w['Y'] - w['mean_const']
  post = device.DevicePosterior(1120)
  post.set_kernel(desc)
  post.set_train(w['X'][:1100], yc[:1100])
  post.build(noise, 0.0, _lib.DFB_BUILD_FULL)
  info, lml = post.extend(w['X'][1100:], yc[1100:], save=True)
  buffers(post, 'extend', info, lml)
  post.restore(1100)
  buffers(post, 'restore', 0, None)
  # one Thompson block: its covariance and its draws (the draws factorise the block's covariance)
  rc = np.random.RandomState(7)
  Xc = rc.random_sample((700, 6))
  mu, cov = post.eval_covar(Xc, 0.0)
  Ut = rc.standard_normal((4, 700))
  info, samples, mx = post.ts_draws(Xc, Ut, 0.0, 0.0)
  out['ts'] = {'mu': hashlib.sha256(mu.tobytes()).hexdigest(), 'cov': hashlib.sha256(cov.tobytes()).hexdigest(),
               'info': int(info), 'samples': digest(samples), 'max_diag': bits(mx)}
  return out


def main():
  if len(sys.argv) == 2 and sys.argv[1] == '--child':
    print(json.dumps(run_child()), flush=True)
    return 0
  libs = sys.argv[1:3]
  res = []
  for lib in libs:
    env = dict(os.environ, DFB200_LIB=os.path.abspath(lib))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), '--child'], env=env, capture_output=True,
                       text=True, check=True)
    res.append(json.loads(r.stdout.strip().splitlines()[-1]))
  a, b = res
  bad = [k for k in a if a[k] != b.get(k)] + [k for k in b if k not in a]
  for k in a:
    print('%-24s %s  info %s' % (k, 'equal' if a[k] == b.get(k) else 'DIFFERENT', a[k].get('info')))
  print('%d comparisons, %d different' % (len(a), len(bad)))
  return 1 if bad else 0


if __name__ == '__main__':
  sys.exit(main())
