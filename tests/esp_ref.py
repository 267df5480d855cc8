"""
NumPy restatement of the reference's ESP kernel (dragonfly/gp/kernel.py:671-744, ESPKernel._child_evaluate) in its
operation order, an extended-precision value of the same kernel, and a per-entry forward-error bound that every fp64
evaluation of the reference's recurrence meets.  Shared by the CPU tests (test_esp_host.py) and the GPU tests
(test_gpu_esp.py).

esp_bound, the derivation.  v_t >= 0 are the exact child values (1-D SE / Matern of scale 1), v^_t the computed ones,
|v^_t - v_t| <= B_t with B_t = tests/kstar_ref.kstar_bound of the 1-D child.  r = order, d = number of children, u = 2^-53.

 1. Child errors.  e_r is multilinear with non-negative coefficients, so for |v^ - v| <= B (v >= 0)
        |e_r(v^) - e_r(v)| <= e_r(v + B) - e_r(v).
 2. Power sums.  p^_i = fl(sum_t fl(v^_t^i)) with v^_t^i from one product (i = 2) or pow (within 2 ulp); the d-term sum of
    non-negative numbers adds gamma_d.  So p^_i = p_i (1 + theta_i), |theta_i| <= gamma_{d+3}, p_i = sum_t v^_t^i.
 3. Newton-Girard.  Let E_0 = 1, E_m = (sum_{i<=m} E_{m-i} P_i) / m with P_i = sum_t w_t^i, w = v + B (every sign
    positive, every quantity at its largest): by induction |e_m(v^)| <= E_m.  With delta_m = |e^_m - e_m(v^)|, the
    m products and m - 1 additions of step m round with gamma_{m+1} relative to sum_i |e^_{m-i}| p^_i, the inputs carry
    delta_{m-i} p^_i + |e_{m-i}| |p^_i - p_i|, and the division rounds once:
        delta_m <= phi_m E_m,  phi_m = phi_{m-1} + (d + m + 5) u + O(u^2),
    so phi_r = (r (d + 6) + r (r + 1) / 2) u, with 1 % added for the O(u^2) terms (r, d <= 48).
 4. K = scale e_r: one more rounding, u |K|.
 Altogether |K^ - K| <= |scale| ((e_r(w) - e_r(v)) + phi_r E_r) + u |scale| E_r + 1e-290 |scale|.
The bound is relative to E_r, the all-positive recurrence, which is what the cancellation of Newton-Girard at high
order loses against: at d = 20, r = 20, E_r / e_r is ~1e5.
"""
import numpy as np

from oracle import gp_oracle as O
import kstar_ref as KR

U = 2.0 ** -53
LD = np.longdouble


def _power(v, i):
  """ v^i the way NumPy's `array ** i` forms it: a copy for 1, a square for 2, pow otherwise. """
  if i == 1:
    return v
  return v * v if i == 2 else np.power(v, float(i))


def esp_in_reference_order(child_vals, r):
  """ e_r of the child matrices, every operation in the reference's order (kernel.py:710-726): the power sums run over
      the children in order from a zero matrix, then step m of Newton-Girard adds the signed terms e_{m-i} p_i for
      i = 1..m to a zero matrix and divides by m. """
  zero = np.zeros_like(child_vals[0])
  psum = {i: zero for i in range(1, r + 1)}
  for i in psum:
    for v in child_vals:
      psum[i] = psum[i] + _power(v, i)
  e = {0: np.ones_like(zero)}
  for m in range(1, r + 1):
    acc = zero
    for i in range(1, m + 1):
      acc = acc + (e[m - i] if i % 2 else -e[m - i]) * psum[i]
    e[m] = acc / m
  return e[r]


class OESPKernel(O.OKernel):
  """ scale * e_order of the 1-D children k_t(X1[:, t], X2[:, t]) (kernel.py:671-744). """

  def __init__(self, scale, order, kernel_list):
    self.dim = len(kernel_list)
    self.kernel_list = kernel_list
    self.hyperparams = {'scale': scale, 'order': order}

  def _evaluate(self, X1, X2):
    kids = [k(X1[:, [t]], X2[:, [t]]) for t, k in enumerate(self.kernel_list)]
    return self.hyperparams['scale'] * esp_in_reference_order(kids, self.hyperparams['order'])


def oracle_kernel(kind, scale, order, bws, nus=None):
  """ OESPKernel with 1-D OSEKernel / OMaternKernel children of scale 1 (ESPKernelSE / ESPKernelMatern). """
  if kind == 'se':
    kids = [O.OSEKernel(1, 1.0, [b]) for b in bws]
  else:
    kids = [O.OMaternKernel(1, nu, 1.0, [b]) for nu, b in zip(nus, bws)]
  return OESPKernel(scale, order, kids)


def _children(kind, bws, nus, Xc, X, exact):
  out = []
  for t, b in enumerate(bws):
    ck, p = ('se', 0) if kind == 'se' else ('matern', int(nus[t]))
    f = KR.kernel_exact if exact else KR.kstar_bound
    out.append(np.asarray(f(ck, p, 1.0, [b], Xc[:, t:t + 1], X[:, t:t + 1]), dtype=LD))
  return out


def _esp_dp(vals, order):
  """ e_order by the product recurrence e_k <- e_k + v e_{k-1} (no cancellation), in longdouble. """
  e = [np.ones(vals[0].shape, dtype=LD)] + [np.zeros(vals[0].shape, dtype=LD) for _ in range(order)]
  for v in vals:
    for k in range(order, 0, -1):
      e[k] = e[k] + v * e[k - 1]
  return e[order]


def esp_exact(kind, scale, order, bws, Xc, X, nus=None):
  """ scale * e_order of the longdouble child values, (m, n) longdouble. """
  return LD(scale) * _esp_dp(_children(kind, bws, nus, Xc, X, True), order)


def esp_bound(kind, scale, order, bws, Xc, X, nus=None):
  """ Per-entry bound on |K^ - K| (module docstring), (m, n) float64. """
  v = _children(kind, bws, nus, Xc, X, True)
  B = _children(kind, bws, nus, Xc, X, False)
  w = [a + b for a, b in zip(v, B)]
  d, r = len(bws), int(order)
  P = [None] + [sum(x ** i for x in w) for i in range(1, r + 1)]
  E = [np.ones(v[0].shape, dtype=LD)] + [None] * r
  for m in range(1, r + 1):
    E[m] = sum(E[m - i] * P[i] for i in range(1, m + 1)) / LD(m)
  phi = LD((r * (d + 6) + r * (r + 1) / 2) * U * 1.01)
  s = abs(LD(scale))
  b = s * ((_esp_dp(w, r) - _esp_dp(v, r)) + phi * E[r]) + LD(U) * s * E[r] + LD(1e-290) * s
  return b.astype(np.float64)
