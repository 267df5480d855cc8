"""
The callable constraint of the constrained Cartesian-product fixture (make_golden_cp_constrained.py): it receives the
raw point [x, z, n, c, w] and is imported by the generator and by the tests alike.
"""


def z_or_n(x):
  return bool(x[1] >= 0.0 or x[2] % 2 == 0)
