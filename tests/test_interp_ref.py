"""
The extended-precision reference and the forward-error bound of tests/interp_ref.py, checked on the CPU against the
fp64 NumPy oracles of the same kernel objects (oracle/gp_oracle.py, tests/nonstat_ref.py, tests/hamming_ref.py): a
bound that an oracle breaks is wrong, one that no fp64 evaluation comes near is too loose to catch anything, and one
that a defect of the interpreter's kind does not break by 10x catches nothing.  Also NumPy's summation order, which
the device's numpy_add_reduce restates, bit for bit.
"""
import numpy as np
import pytest

import interp_ref as IR
import kstar_ref as KR
from dragonfly_b200 import kernel as K
from dragonfly_b200.cartesian_product_gp import CartesianProductKernel

RATIO_FLOOR = 1e-3
DEFECT_FACTOR = 10.0
CASES = IR.catalogue(K, CartesianProductKernel, small=True)
_ratios = {}


def _err(vals, exact):
  return np.abs(np.asarray(vals, dtype=np.float64).astype(np.longdouble) - exact).astype(np.float64)


@pytest.mark.parametrize('case', CASES, ids=[c.name for c in CASES])
def test_oracle_values_lie_within_the_bound(case):
  K_o = IR.oracle_of(case.kern)(case.Xc, case.X)
  K_x, B = IR.evaluate(case.kern, case.Xc, case.X)
  err = _err(K_o, K_x)
  assert (err <= B).all(), (float(np.max(err / B)), np.unravel_index(np.argmax(err / B), err.shape))
  # the diagonal form: k(x, x) of the candidates
  d_o = np.diag(IR.oracle_of(case.kern)(case.Xc, case.Xc))
  d_x, d_B = IR.evaluate(case.kern, case.Xc, case.Xc, diag=True)
  d_err = _err(d_o, d_x)
  assert (d_err <= d_B).all(), float(np.max(d_err / d_B))
  worst = max(float(np.max(err / B)), float(np.max(d_err / d_B)))
  _ratios[case.construct] = max(_ratios.get(case.construct, 0.0), worst)


def test_the_bound_is_not_vacuous():
  """ Per construct, the largest observed |oracle - exact| / bound over the catalogue reaches RATIO_FLOOR. """
  for case in CASES:
    if case.construct not in _ratios:
      test_oracle_values_lie_within_the_bound(case)
  for construct in sorted(_ratios):
    print('largest |K_oracle - K_exact| / bound, %-10s %.3g' % (construct, _ratios[construct]))
  for construct, worst in _ratios.items():
    assert RATIO_FLOOR <= worst <= 1.0, (construct, worst)


def test_the_diagonal_form_is_the_diagonal():
  case = [c for c in CASES if c.name == 'prod-over-additive'][0]
  K_x, B = IR.evaluate(case.kern, case.Xc, case.Xc)
  d_x, d_B = IR.evaluate(case.kern, case.Xc, case.Xc, diag=True)
  assert np.array_equal(np.diag(K_x), d_x) and np.array_equal(np.diag(B), d_B)


@pytest.mark.parametrize('d', list(range(1, 18)))
def test_matern72_oracle_values_lie_within_the_kstar_bound(d):
  """ kstar_ref's bound with the Matern-7/2 constant (pow in the polynomial) against the NumPy oracle, coincident and
      nearly coincident pairs included, at bandwidths 0.02 .. 5 """
  from oracle import gp_oracle as O
  X, Xc = _pts(d, seed=50 + d)
  worst = 0.0
  for i, bw0 in enumerate((0.02, 0.1, 0.5, 1.0, 5.0)):
    bw = bw0 * (1.0 + 0.25 * np.random.RandomState(i).random_sample(d))
    K_o = O.OMaternKernel(d, 3.5, 0.7 + i, list(bw))(Xc, X)
    K_x = KR.kernel_exact('matern', 3, 0.7 + i, bw, Xc, X)
    B = KR.kstar_bound('matern', 3, 0.7 + i, bw, Xc, X)
    err = _err(K_o, K_x)
    assert (err <= B).all(), (bw0, float(np.max(err / B)))
    assert (B <= 1e-8 * (0.7 + i)).all()
    worst = max(worst, float(np.max(err / B)))
  assert worst >= RATIO_FLOOR, worst          # not vacuous


# ---- injected defects ---------------------------------------------------------------------------------------------------
def _pts(D, n=40, m=48, seed=3, lo=0.0, hi=1.0):
  return IR.points(np.random.RandomState(seed), D, n, m, lo, hi)


def _breaks(kern, Xc, X, defective, cols1=None, cols2=None):
  K_x, B = IR.evaluate(kern, Xc, X, cols1=cols1, cols2=cols2)
  ratio = float(np.max(_err(defective, K_x) / B))
  assert ratio >= DEFECT_FACTOR, ratio
  return ratio


def _se_d2_dropping_tail(A, B, drop):
  """ dist_squared's (|y|^2 + |x|^2) - 2 x.y with term `drop` of the candidates' squared norm left out """
  sq1 = (A ** 2)
  sq1[:, drop] = 0.0
  return np.clip((B ** 2).sum(axis=1)[None, :] + sq1.sum(axis=1)[:, None] - 2 * A.dot(B.T), 0.0, np.inf)


@pytest.mark.parametrize('kname', ['se', 'matern12', 'matern72'])
def test_defect_last_slot_of_a_factor_dropped(kname):
  kind, p = KR.INTERP_KINDS[kname]
  bw = [0.4, 0.5, 0.6, 0.7, 0.8]
  make = lambda d: K.SEKernel(d, 1.3, bw[:d]) if kind == 'se' else K.MaternKernel(d, p + 0.5, 1.3, bw[:d])
  X, Xc = _pts(5)
  _breaks(make(5), Xc, X, IR.oracle_of(make(4))(Xc[:, :4], X[:, :4]))


def test_defect_factor_reads_the_previous_factors_slots():
  kern = K.CoordinateProductKernel(4, 0.9, [K.SEKernel(2, 1.0, [0.4, 0.5]), K.MaternKernel(2, 2.5, 1.0, [0.6, 0.7])],
                                   [[0, 1], [2, 3]])
  X, Xc = _pts(4)
  bad = IR.oracle_of(K.CoordinateProductKernel(4, 0.9, kern.kernel_list, [[0, 1], [0, 1]]))(Xc, X)
  _breaks(kern, Xc, X, bad)


def _additive():
  return K.AdditiveKernel(0.35, [K.SEKernel(2, 1.0, [0.4, 0.5]), K.MaternKernel(1, 1.5, 0.7, [0.6]),
                                 K.MaternKernel(1, 0.5, 0.2, [0.9])], [[0, 1], [2], [3]])


def test_defect_term_dropped():
  kern = _additive()
  X, Xc = _pts(4)
  bad = IR.oracle_of(K.AdditiveKernel(0.35, kern.kernel_list[:2], kern.groupings[:2]))(Xc, X)
  _breaks(kern, Xc, X, bad)


def test_defect_pre_scale_twice_and_post_scale_missing():
  X, Xc = _pts(4)
  prod = K.CoordinateProductKernel(4, 0.7, [K.SEKernel(2, 1.0, [0.4, 0.5]), K.MaternKernel(2, 2.5, 1.0, [0.6, 0.7])],
                                   [[0, 1], [2, 3]])
  _breaks(prod, Xc, X, 0.7 * IR.oracle_of(prod)(Xc, X))
  add = _additive()
  _breaks(add, Xc, X, IR.oracle_of(add)(Xc, X) / 0.35)


def _expdecay_values(scale, offset, powers, Xc, X, where):
  """ ExpDecay with its offset added before the product chain, or omitted """
  ret = (scale + offset if where == 'before' else scale) * np.ones((Xc.shape[0], X.shape[0]))
  for i in range(len(powers)):
    ret *= 1 / (1 + np.add.outer(Xc[:, i], X[:, i])) ** powers[i]
  return ret


@pytest.mark.parametrize('where', ['before', 'omitted'])
def test_defect_expdecay_offset(where):
  kern = K.CoordinateProductKernel(3, 1.3, [K.ExpDecayKernel(2, 0.8, 0.1, [1.0, 2.0]), K.MaternKernel(1, 1.5, 1.0, [0.5])],
                                   [[0, 1], [2]])
  X, Xc = _pts(3)
  bad = 1.3 * _expdecay_values(0.8, 0.1, [1.0, 2.0], Xc, X, where) * IR.oracle_of(kern.kernel_list[1])(Xc[:, 2:], X[:, 2:])
  _breaks(kern, Xc, X, bad)


@pytest.mark.parametrize('order', [1, 2, 3, 7])
def test_defect_poly_without_its_plus_one(order):
  w = np.array([0.5, 0.7, 0.3, 0.6])
  kern = K.PolyKernel(4, order, 0.8, list(w))
  X, Xc = _pts(4, lo=-1.5, hi=1.5)
  _breaks(kern, Xc, X, 0.8 * ((Xc * w).dot((X * w).T)) ** order)


@pytest.mark.parametrize('order', [1, 2, 3, 7])
def test_defect_poly_scaling_divided(order):
  w = np.array([0.5, 0.7, 0.3, 0.6])
  kern = K.PolyKernel(4, order, 0.8, list(w))
  X, Xc = _pts(4, lo=-1.5, hi=1.5)
  _breaks(kern, Xc, X, 0.8 * ((Xc / w).dot((X / w).T) + 1) ** order)


@pytest.mark.parametrize('kname', ['se', 'poly', 'expdecay'])
def test_defect_coordinate_maps_swapped_on_a_test_kernel(kname):
  """ An Add-UCB group kernel: candidate columns 0 .. 2 against training columns g; the defect reads the candidates'
      columns g and the training points' 0 .. 2. """
  g = [5, 1, 3]
  kern = {'se': K.SEKernel(3, 1.1, [0.4, 0.5, 0.6]), 'poly': K.PolyKernel(3, 2, 0.9, [0.5, 0.7, 0.3]),
          'expdecay': K.ExpDecayKernel(3, 1.0, 0.2, [1.0, 0.5, 2.0])}[kname]
  X, Xc = _pts(6)
  bad = IR.oracle_of(kern)(Xc[:, g], X[:, :3])
  _breaks(kern, Xc, X, bad, cols1=[0, 1, 2], cols2=g)


@pytest.mark.parametrize('kname', ['se', 'matern52'])
def test_defect_pairwise_tail_term_of_the_norm_dropped(kname):
  """ d = 17: eight accumulators over 16 terms and a one-term tail; the tail's term left out of |x|^2 """
  d = 17
  bw = np.full(d, 1.2)
  kern = K.SEKernel(d, 1.0, list(bw)) if kname == 'se' else K.MaternKernel(d, 2.5, 1.0, list(bw))
  X, Xc = _pts(d)
  d2 = _se_d2_dropping_tail(Xc / bw, X / bw, d - 1)
  bad = np.exp(-d2 / 2) if kname == 'se' else IR.oracle_of(kern).norm_constant * IR.oracle_of(kern)._unnormalised(
      np.sqrt(d2))
  _breaks(kern, Xc, X, bad)


# ---- NumPy's summation order --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('d', list(range(1, 10)) + [15, 16, 17, 24, 31, 64, 128])
def test_numpy_add_reduce_restatement_is_numpys_sum(d):
  """ kernels.cu numpy_add_reduce, restated on the host, gives NumPy's (np.equal(a, b) * w).sum(axis=1) bit for bit;
      the weights spread over 2^-20 .. 2^20, so that another association order changes the result. """
  rs = np.random.RandomState(d)
  w = 2.0 ** rs.uniform(-20, 20, size=d)
  A = rs.randint(0, 2, size=(200, d)).astype(np.float64)
  B = rs.randint(0, 2, size=(200, d)).astype(np.float64)
  eq = np.equal(A, B)
  want = (eq * w).sum(axis=1)
  got = np.array([IR.numpy_add_reduce(row) for row in eq * w])
  assert np.array_equal(want.view(np.int64), got.view(np.int64))
  want1 = np.add.reduce(w)
  assert IR.numpy_add_reduce(w) == want1
  if d >= 16:
    # the order matters at these weights: a plain left-to-right sum differs somewhere
    seq = np.array([sum(float(x) for x in row) for row in eq * w])
    assert not np.array_equal(seq, want)
