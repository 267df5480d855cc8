"""
Golden vectors for the Cartesian-product GP over Euclidean-type domains: the UNMODIFIED reference's
dragonfly.gp.cartesian_product_gp.CPGP with dragonfly.gp.kernel.CartesianProductKernel (kernel.py:504-538) at its
default handle_non_psd_kernels='project_first'.

Run from the repository root with the reference source tree in $DRAGONFLY_REF:
  PYTHONPATH=oracle/ref_shim:$DRAGONFLY_REF python tests/golden/make_golden_cpgp.py
"""
import os
import numpy as np
import dragonfly
from dragonfly.gp.kernel import SEKernel, MaternKernel, CartesianProductKernel
from dragonfly.gp.cartesian_product_gp import CPGP

assert dragonfly.__file__.startswith(os.environ['DRAGONFLY_REF'])


def main():
  rs = np.random.RandomState(3)
  n, m = 240, 500
  def pts(k):
    return [[rs.random_sample(2), rs.random_sample(3), rs.random_sample(1)] for _ in range(k)]
  X, C = pts(n), pts(m)
  flat = lambda P: np.array([np.concatenate(p) for p in P])
  Xf = flat(X)
  Y = np.sin(3 * Xf[:, 0]) + Xf[:, 2] * Xf[:, 3] - (Xf[:, 5] - 0.3) ** 2 + 0.05 * rs.standard_normal(n)
  scale, noise_var, mean_const = 1.3, 0.02, float(np.median(Y))
  kern = CartesianProductKernel(scale, [SEKernel(2, 1.0, [0.4, 0.6]), MaternKernel(3, 2.5, 1.0, [0.5, 0.7, 0.9]),
                                        MaternKernel(1, 1.5, 1.0, [0.3])])
  gp = CPGP(X, list(Y), kern, lambda x: np.array([mean_const] * len(x)), noise_var)
  mu, sd = gp.eval(C, 'std')
  halluc = pts(3)
  mu_h, sd_h = gp.eval_with_hallucinated_observations(C[:100], halluc, 'std')
  out = dict(X=Xf, Y=Y, C=flat(C), H=flat(halluc), meta=np.array([scale, noise_var, mean_const]), K=gp.K_trtr_wo_noise[:16],
             mu=mu, sd=sd, mu_h=mu_h, sd_h=sd_h, lml=np.array(gp.compute_log_marginal_likelihood()), alpha=gp.alpha)
  np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cpgp.npz'), **out)
  print({k: np.shape(v) for k, v in out.items()})


if __name__ == '__main__':
  main()
