"""
Golden vectors for the log-marginal-likelihood gradients (SURVEY 8f rank 2):
GP.compute_grad_log_marginal_likelihood (gp_core.py:229-240) with Kernel.gradient (kernel.py:202-217, 301-322) of
the UNMODIFIED reference.  The reference indexes hyperparams['dim_bandwidths'][0, j]; that is defined only when the
bandwidths were handed over as a (d, 1) column, which is how the kernels are built here.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python tests/golden/make_golden_grad.py
"""
import os
import numpy as np
import dragonfly
from dragonfly.gp.kernel import SEKernel, MaternKernel
from dragonfly.gp.gp_core import GP

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])


def main():
  out = {}
  rs = np.random.RandomState(7)
  cases = [('se3', 300, 3, 'se', None), ('m25_6', 400, 6, 'matern', 2.5), ('m15_2', 200, 2, 'matern', 1.5),
           ('m05_4', 250, 4, 'matern', 0.5)]
  for name, n, d, kind, nu in cases:
    X = rs.random_sample((n, d))
    Y = np.sin(3 * X.sum(axis=1)) + 0.1 * rs.standard_normal(n)
    bw = 0.2 + 0.6 * rs.random_sample(d)
    scale = 1.7
    noise_var = 0.05
    mean_const = float(np.median(Y))
    col = bw.reshape(d, 1)
    kern = SEKernel(d, scale, col) if kind == 'se' else MaternKernel(d, nu, scale, col)
    gp = GP(list(X), list(Y), kern, lambda x, m=mean_const: np.array([m] * len(x)), noise_var)
    params = [('scale', ()), ('noise_var', ()), ('noise_mean', ()), ('same_dim_bandwidths', ())]
    params += [('dim_bandwidths', (j,)) for j in range(d)]
    grads = np.array([gp.compute_grad_log_marginal_likelihood(p, *a) for p, a in params])
    out[name + '_X'] = X; out[name + '_Y'] = Y; out[name + '_bw'] = bw
    out[name + '_meta'] = np.array([scale, noise_var, mean_const, -1.0 if nu is None else nu])
    out[name + '_grads'] = grads
    out[name + '_lml'] = np.array(gp.compute_log_marginal_likelihood())
    # kernel-gradient sub-blocks (rows 0..7) for the oracle's own pinning
    out[name + '_G_same'] = kern.gradient('same_dim_bandwidths', X[:8], X)
    out[name + '_G_dim1'] = kern.gradient('dim_bandwidths', list(X), list(X), 1)[:8]
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'grad.npz'), **out)
  print({k: v.shape for k, v in out.items()})


if __name__ == '__main__':
  main()
