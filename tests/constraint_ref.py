"""
NumPy oracle of dfb_constraint_status: the compiled constraint program of dragonfly_b200/constraints.py interpreted over
many rows at once, every value and radius formed with the device's operations in the device's order (IEEE round to
nearest, no contraction).  exp and log are NumPy's here and CUDA's there; everything else agrees bit for bit.
"""
import numpy as np

from dragonfly_b200.constraints import OP, REJECT, ACCEPT, UNDECIDED

EPS2, EF2, EF4, EF8 = 2.0 ** -52, 2.0 ** -43, 2.0 ** -42, 2.0 ** -41
INFL, TINY, TINYF, ILIM = 1.0 + 2.0 ** -48, 2.0 ** -1070, 2.0 ** -1000, 2.0 ** 53
MAX = np.finfo(np.float64).max


def infl(x):
  return x * INFL + TINY


def fin(x):
  return np.abs(x) <= MAX


def known(r):
  return r <= MAX


def _compare(op, a, ra, b, rb):
  exact = (ra == 0) & (rb == 0)
  t = {OP['lt']: a < b, OP['le']: a <= b, OP['gt']: a > b, OP['ge']: a >= b, OP['eq']: a == b, OP['ne']: a != b}[op]
  d = (a - b) if op in (OP['gt'], OP['ge']) else (b - a)
  s = infl((ra + rb) + EPS2 * np.abs(d))
  if op == OP['eq']:
    ap = np.where(np.abs(d) > s, 0.0, 2.0)
  elif op == OP['ne']:
    ap = np.where(np.abs(d) > s, 1.0, 2.0)
  else:
    ap = np.where(d > s, 1.0, np.where(d < -s, 0.0, 2.0))
  bad = ~(fin(a) & fin(b) & known(ra) & known(rb))
  return np.where(exact, t.astype(np.float64), np.where(bad, 2.0, ap))


def _sqrt_radius(a, ra, c):
  e = ra / c
  ap = infl(e + EPS2 * (c + e))
  return np.where(ra == 0, 0.0, np.where(fin(a) & known(ra) & (a > ra), ap, np.inf))


def status(f, rows):
  """ The status byte of every row of rows (m x n_cols float64) under ConstraintFilter f. """
  rows = np.asarray(rows, dtype=np.float64)
  m = len(rows)
  st = np.full(m, ACCEPT, dtype=np.uint8)
  V, R = [], []
  with np.errstate(all='ignore'):
    for op, arg, arg2, val in zip(f.op, f.arg, f.arg2, f.val):
      op, arg, arg2 = int(op), int(arg), int(arg2)
      if op in (OP['col'], OP['const'], OP['lookup']):
        if op == OP['const']:
          V.append(np.full(m, val)); R.append(np.zeros(m))
        elif op == OP['col']:
          V.append(rows[:, arg].copy()); R.append(np.zeros(m))
        else:
          key = rows[:, arg]
          c, r = np.full(m, 2.0), np.full(m, np.inf)
          for j in reversed(range(arg2, arg2 + int(val))):     # the first equal key wins
            hit = key == f.tab_key[j]
            c, r = np.where(hit, f.tab_val[j], c), np.where(hit, 0.0, r)
          V.append(c); R.append(r)
      elif OP['add'] <= op <= OP['div']:
        b, rb, a, ra = V.pop(), R.pop(), V.pop(), R.pop()
        c = {OP['add']: a + b, OP['sub']: a - b, OP['mul']: a * b, OP['div']: a / b}[op]
        if op in (OP['add'], OP['sub']):
          ap = infl((ra + rb) + EPS2 * np.abs(c))
        else:
          lin = np.abs(a) * rb + np.abs(b) * ra
          if op == OP['mul']:
            e = lin + ra * rb
          else:
            e = np.where(np.abs(b) > rb, lin / (np.abs(b) * (np.abs(b) - rb)), np.inf)
          ap = infl(e + EPS2 * (np.abs(c) + e))
        bad = ~(fin(a) & fin(b) & fin(c) & known(ra) & known(rb))
        r = np.where((ra == 0) & (rb == 0), 0.0, np.where(bad, np.inf, ap))
        if arg == 1:
          r = np.where(np.abs(c) < ILIM, r, np.inf)
        V.append(c); R.append(r)
      elif op == OP['neg']:
        V[-1] = -V[-1]
      elif op == OP['abs']:
        V[-1] = np.abs(V[-1])
      elif op == OP['sqrt']:
        a, ra = V.pop(), R.pop()
        c = np.sqrt(a)
        V.append(c); R.append(_sqrt_radius(a, ra, c))
      elif op == OP['exp']:
        a, ra = V.pop(), R.pop()
        c = np.exp(a)
        ok = fin(a) & (ra <= 1.0) & fin(c)
        V.append(c); R.append(np.where(ok, infl(c * (2.5 * ra + EF8) + TINYF), np.inf))
      elif op == OP['log']:
        a, ra = V.pop(), R.pop()
        c = np.log(a)
        e = ra / (a - ra)
        ok = fin(a) & known(ra) & (a > ra)
        V.append(c); R.append(np.where(ok, infl((1.25 * e + EF4 * (np.abs(c) + e)) + TINYF), np.inf))
      elif op == OP['pow']:
        a, ra = V.pop(), R.pop()
        if arg == 0:
          c, r = np.ones(m), np.zeros(m)
        elif arg == 1:
          c, r = a, ra
        else:
          c = a
          for _ in range(1, arg):
            c = c * a
          if arg2 == 1:
            r = np.where((ra == 0) & (np.abs(c) < ILIM), 0.0, np.inf)
          else:
            mm = np.abs(a) + ra
            pm = mm
            for _ in range(2, arg):
              pm = pm * mm
            e = (float(arg) * pm) * ra
            rel = float(arg) * EPS2 + EF2
            ap = infl((1.25 * e + (np.abs(c) + e) * rel) + TINYF)
            r = np.where(fin(a) & fin(c) & known(ra), ap, np.inf)
        V.append(c); R.append(r)
      elif op in (OP['min'], OP['max']):
        b, rb, a, ra = V.pop(), R.pop(), V.pop(), R.pop()
        c = np.where(b < a, b, a) if op == OP['min'] else np.where(b > a, b, a)
        bad = ~(fin(a) & fin(b) & known(ra) & known(rb))
        V.append(c); R.append(np.where((ra == 0) & (rb == 0), 0.0, np.where(bad, np.inf, np.maximum(ra, rb))))
      elif op in (OP['npsum'], OP['norm']):
        xs, rs_in = V[-arg:], R[-arg:]
        del V[-arg:], R[-arg:]
        s = xs[0] if op == OP['npsum'] else xs[0] * xs[0]
        Rs, A, ok = rs_in[0], np.abs(xs[0]), fin(xs[0])
        for y, ry in zip(xs[1:], rs_in[1:]):
          s = s + (y if op == OP['npsum'] else y * y)
          Rs = Rs + ry
          A = A + np.abs(y)
          ok = ok & fin(y)
        if op == OP['npsum']:
          ap = infl(Rs + (float(arg) * EPS2) * (A + Rs))
          r = np.where(ok & fin(A) & known(Rs), ap, np.inf)
          if arg <= 2:
            r = np.where(Rs == 0, 0.0, r)
          c = s
        else:
          rsq = infl((float(arg) * EPS2) * s + TINYF)
          c = np.sqrt(s)
          r = _sqrt_radius(s, rsq, c)
          zero = A == 0
          c = np.where(zero, 0.0, c)
          r = np.where(zero, 0.0, r)
          bad = ~(ok & (Rs == 0) & fin(s))
          c = np.where(bad, s, c)
          r = np.where(bad, np.inf, r)
        V.append(c); R.append(r)
      elif OP['lt'] <= op <= OP['ne']:
        b, rb, a, ra = V.pop(), R.pop(), V.pop(), R.pop()
        V.append(_compare(op, a, ra, b, rb)); R.append(np.zeros(m))
      elif op in (OP['and'], OP['or']):
        b, a = V.pop(), V.pop()
        del R[-2:]
        if op == OP['and']:
          c = np.where((a == 0) | (b == 0), 0.0, np.where((a == 1) & (b == 1), 1.0, 2.0))
        else:
          c = np.where((a == 1) | (b == 1), 1.0, np.where((a == 0) & (b == 0), 0.0, 2.0))
        V.append(c); R.append(np.zeros(m))
      elif op == OP['not']:
        V[-1] = np.where(V[-1] == 2, 2.0, 1.0 - V[-1])
      else:                                                   # accept
        b = V.pop(); R.pop()
        st = np.where(st == REJECT, REJECT, np.where(b == 0, REJECT, np.where(b == 2, UNDECIDED, st))).astype(np.uint8)
  assert not V
  return st
