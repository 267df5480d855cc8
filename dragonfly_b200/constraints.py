"""
Domain constraints of a Cartesian-product domain compiled to a certified device filter.

The reference checks every drawn point with domain.constraints_are_satisfied (domains.py:350-460): the point is
reordered into its raw form (get_raw_point), every string constraint is eval'd with the raw variables bound, every
callable is called on the raw point, and the point is kept iff all of them return True.  Here the string constraints
are parsed (Python `ast`, nothing is eval'd per point) into a small stack program that the device runs over candidate
rows (dfb_constraint_status); whatever the compiler does not take stays on the host as the *residue*.

Certified evaluation.  Every value the program computes carries a radius that bounds the distance between the device's
value and the one NumPy computes for the same raw point.  Operations the device repeats exactly -- IEEE + - * / and sqrt
in the reference's order, integer arithmetic below 2^53, table lookups -- keep radius 0; exp, log, np.sum over three
or more terms, np.linalg.norm and powers x**k (k >= 2) get a forward-error bound that covers both implementations; an
interval that touches a function's domain boundary (sqrt, log, a divisor) is unknown.  A comparison is decided when its
margin exceeds the radii, and constraints combine in three-valued logic.  A row's status is REJECT, ACCEPT or UNDECIDED;
UNDECIDED rows, and ACCEPT rows when residue constraints exist, are settled on the host by the domain's own evaluator,
so the kept set is exactly the reference's.  One divergence: a residue constraint is not called on a row that a
compiled constraint rejects, so a residue callable that would raise there does not.

What compiles: raw variable names, constants, constant integer indexing and constant slices of vector variables, unary
-, + - * /, ** by a constant integer 0..8, abs / np.abs, np.sqrt, np.exp, np.log, builtin sum (left to right from 0),
np.sum, np.linalg.norm of a vector (2-norm), min / max of scalars, chained comparisons of numbers, and / or / not of
booleans.  A sub-expression that depends on one single-coordinate discrete variable only (c != 'b', c in ['a', 'b'], a
discrete-numeric value) is tabulated over that variable's levels by Python's own evaluation and looked up on the device
by the column value the rows hold.  Everything else -- other calls or attributes, names outside the raw ordering,
vector-valued results, and / or over non-booleans, callables and .py constraints -- is residue.
"""
import ast

import numpy as np

# opcodes of dfb_cons_prog (include/dfb200.h)
OPS = ['col', 'const', 'lookup', 'add', 'sub', 'mul', 'div', 'neg', 'abs', 'sqrt', 'exp', 'log', 'pow', 'min', 'max',
       'npsum', 'norm', 'lt', 'le', 'gt', 'ge', 'eq', 'ne', 'and', 'or', 'not', 'accept']
OP = {name: k for k, name in enumerate(OPS)}
MAX_OPS, MAX_STACK, MAX_TAB, MAX_VEC = 128, 16, 64, 16
REJECT, ACCEPT, UNDECIDED = 0, 1, 2
INT_LIMIT = float(2 ** 53)

# names bound as locals inside the reference's evaluate_strings_with_given_variables: a raw variable of one of these
# names does not evaluate to its value there, so constraints naming them stay on the host
_EVALUATOR_LOCALS = {'strs_to_execute', 'variable_dict', 'got_list_of_constraints', 'key', 'value', 'ret', 'elem',
                     'curr_result'}
_PURE_BUILTINS = {'abs', 'min', 'max', 'sum', 'len', 'float', 'int', 'str', 'bool', 'round'}
_PURE_NP = {'abs', 'absolute', 'sqrt', 'exp', 'log', 'sum', 'linalg.norm', 'pi', 'e', 'inf', 'nan'}
_NP_UNARY = {'abs': 'abs', 'absolute': 'abs', 'sqrt': 'sqrt', 'exp': 'exp', 'log': 'log'}


class _Residue(Exception):
  pass


class _Var(object):
  """ A raw variable: its candidate columns (a scalar has one and vector False) and the kind of its part. """
  __slots__ = ('cols', 'vector', 'kind')

  def __init__(self, cols, vector, kind):
    self.cols, self.vector, self.kind = cols, vector, kind


def column_map(domain, parts):
  """ name -> _Var, read by passing a probe point through the domain's own get_raw_point: the probe holds each
      coordinate's candidate-column index (numeric parts as float arrays, discrete parts as lists), and get_raw_point
      only slices and reorders, so each raw variable comes back as the column(s) it occupies. """
  probe, kinds, c0 = [], [], 0
  for p in parts:
    if p.type in ('euclidean', 'integral'):
      probe.append(np.arange(c0, c0 + p.dim, dtype=np.float64))
    else:
      probe.append(list(range(c0, c0 + p.dim)))
    kinds += [p.type] * p.dim
    c0 += p.dim
  out = {}
  for name, v in zip(domain.raw_name_ordering, domain.get_raw_point(probe)):
    if isinstance(v, (np.ndarray, list)):
      cols = [int(c) for c in v]
      out[name] = _Var(cols, True, kinds[cols[0]] if cols else None)
    else:
      out[name] = _Var([int(v)], False, kinds[int(v)])
  return out


def _scalar_kind(v):
  """ 'bool' / 'int' / 'float' of a value the device can hold exactly with NumPy's semantics, else None. """
  if isinstance(v, (bool, np.bool_)):
    return 'bool'
  if isinstance(v, (int, np.int64)) and abs(int(v)) < 2 ** 53:
    return 'int'
  if type(v) in (float, np.float64):
    return 'float'
  return None


class _Compiler(object):

  def __init__(self, cmap, parts, globs, levels):
    self.cmap, self.globs, self.levels = cmap, globs, levels
    self.tab_key, self.tab_val = [], []
    self.col_levels = {}
    c0 = 0
    for p in parts:
      for q in range(p.dim):
        if p.levels is not None:
          from .gpb_acquisitions import _level_columns
          arr = np.array(p.levels[q])
          vals = [arr[k] for k in range(len(arr))]
          keys = np.arange(len(vals), dtype=np.float64) if levels else _level_columns(p, vals)
          self.col_levels[c0 + q] = (vals, keys)
      c0 += p.dim

  # -- helpers ---------------------------------------------------------------------------------------------------
  def _names(self, node):
    return {n.id for n in ast.walk(node) if isinstance(n, ast.Name)}

  def _pure(self, node):
    """ True when every call and attribute of the sub-expression is a pure function or constant of Python or NumPy, so
        that evaluating it once per level (or once in all) is evaluating it per point. """
    for n in ast.walk(node):
      if isinstance(n, ast.Call):
        f = n.func
        if isinstance(f, ast.Name):
          if f.id not in _PURE_BUILTINS or f.id in self.cmap or f.id in self.globs:
            return False
        elif self._np_func(f) not in _PURE_NP:
          return False
      elif isinstance(n, ast.Attribute) and self._np_func(n) not in _PURE_NP and not (
          isinstance(n.value, ast.Name) and n.value.id == 'np' and n.attr == 'linalg'):
        return False
    return True

  def _raw_deps(self, node):
    return {n for n in self._names(node) if n in self.cmap}

  def _eval(self, node, bindings):
    code = compile(ast.Expression(body=node), '<constraint>', 'eval')
    return eval(code, self.globs, dict(bindings))  # pylint: disable=eval-used

  def _tabulate(self, node):
    """ A sub-expression of constants or of one single-coordinate discrete variable, evaluated by Python: a constant or
        a lookup table keyed by the column values of the variable's levels.  None when it does not reduce to a bool or
        number (the parent may). """
    names = self._names(node)
    if names & _EVALUATOR_LOCALS or not self._pure(node):
      return None
    deps = self._raw_deps(node)
    if not deps:
      try:
        v = self._eval(node, {})
      except Exception:  # pylint: disable=broad-except
        return None
      k = _scalar_kind(v)
      return None if k is None else (k, [('const', 0, 0, float(v))])
    if len(deps) != 1:
      return None
    var = self.cmap[next(iter(deps))]
    if var.vector or var.cols[0] not in self.col_levels:
      return None
    vals, keys = self.col_levels[var.cols[0]]
    if len(set(keys.tolist())) != len(keys):
      return None
    try:
      outs = [self._eval(node, {next(iter(deps)): v}) for v in vals]
    except Exception:  # pylint: disable=broad-except
      return None
    kinds = {_scalar_kind(v) for v in outs}
    if None in kinds or ('bool' in kinds and len(kinds) > 1):
      return None
    kind = 'bool' if kinds == {'bool'} else ('int' if kinds == {'int'} else 'float')
    off = len(self.tab_key)
    self.tab_key += [float(k) for k in keys]
    self.tab_val += [float(v) for v in outs]
    if len(self.tab_key) > MAX_TAB:
      raise _Residue('lookup tables too large')
    return kind, [('lookup', var.cols[0], off, float(len(keys)))]

  def _scalar(self, node):
    kind, code = self.node(node)
    if kind not in ('int', 'float'):
      raise _Residue('not a number')
    return kind, code

  def _vector(self, node):
    """ (element kind, columns) of a vector variable or a constant slice of one. """
    if isinstance(node, ast.Name) and node.id in self.cmap and self.cmap[node.id].vector:
      var = self.cmap[node.id]
    elif isinstance(node, ast.Subscript) and isinstance(node.slice, ast.Slice):
      kind, cols = self._vector(node.value)
      sl = slice(*[None if e is None else self._const_int(e) for e in (node.slice.lower, node.slice.upper,
                                                                       node.slice.step)])
      return kind, cols[sl]
    else:
      raise _Residue('not a vector')
    if var.kind not in ('euclidean', 'integral'):
      raise _Residue('vector of a discrete variable')
    return ('float' if var.kind == 'euclidean' else 'int'), list(var.cols)

  def _const_int(self, node):
    v = self._tabulate(node)
    if v is None or v[0] != 'int':
      raise _Residue('index is not a constant integer')
    return int(v[1][0][3])

  # -- nodes -----------------------------------------------------------------------------------------------------
  def node(self, node):
    tab = self._tabulate(node)
    if tab is not None:
      return tab
    if isinstance(node, ast.Name):
      var = self.cmap.get(node.id)
      if var is None or node.id in _EVALUATOR_LOCALS or var.vector or var.kind not in ('euclidean', 'integral'):
        raise _Residue('name %s' % node.id)
      return ('float' if var.kind == 'euclidean' else 'int'), [('col', var.cols[0], 0, 0.0)]
    if isinstance(node, ast.Subscript):
      if isinstance(node.slice, ast.Slice):
        raise _Residue('vector value')
      kind, cols = self._vector(node.value)
      k = self._const_int(node.slice)
      if not -len(cols) <= k < len(cols):
        raise _Residue('index out of range')
      return kind, [('col', cols[k], 0, 0.0)]
    if isinstance(node, ast.UnaryOp):
      if isinstance(node.op, ast.Not):
        kind, code = self.node(node.operand)
        if kind != 'bool':
          raise _Residue('not of a non-bool')
        return 'bool', code + [('not', 0, 0, 0.0)]
      kind, code = self._scalar(node.operand)
      if isinstance(node.op, ast.UAdd):
        return kind, code
      if isinstance(node.op, ast.USub):
        return kind, code + [('neg', 0, 0, 0.0)]
      raise _Residue('unary operator')
    if isinstance(node, ast.BinOp):
      if isinstance(node.op, ast.Pow):
        kind, code = self._scalar(node.left)
        k = self._const_int(node.right)
        if not 0 <= k <= 8:
          raise _Residue('exponent')
        return kind, code + [('pow', k, int(kind == 'int'), 0.0)]
      ops = {ast.Add: 'add', ast.Sub: 'sub', ast.Mult: 'mul', ast.Div: 'div'}
      if type(node.op) not in ops:
        raise _Residue('binary operator')
      lk, lc = self._scalar(node.left)
      rk, rc = self._scalar(node.right)
      op = ops[type(node.op)]
      kind = 'int' if (lk == rk == 'int' and op != 'div') else 'float'
      return kind, lc + rc + [(op, int(kind == 'int'), 0, 0.0)]
    if isinstance(node, ast.BoolOp):
      op = 'and' if isinstance(node.op, ast.And) else 'or'
      code = []
      for j, v in enumerate(node.values):
        kind, c = self.node(v)
        if kind != 'bool':
          raise _Residue('and / or of a non-bool')
        code += c + ([(op, 0, 0, 0.0)] if j > 0 else [])
      return 'bool', code
    if isinstance(node, ast.Compare):
      ops = {ast.Lt: 'lt', ast.LtE: 'le', ast.Gt: 'gt', ast.GtE: 'ge', ast.Eq: 'eq', ast.NotEq: 'ne'}
      code, left = [], node.left
      for j, (cop, right) in enumerate(zip(node.ops, node.comparators)):
        if type(cop) not in ops:
          raise _Residue('comparison')
        code += self._scalar(left)[1] + self._scalar(right)[1] + [(ops[type(cop)], 0, 0, 0.0)]
        if j > 0:
          code.append(('and', 0, 0, 0.0))
        left = right
      return 'bool', code
    if isinstance(node, ast.Call):
      return self._call(node)
    raise _Residue(type(node).__name__)

  def _np_func(self, func):
    """ 'abs' / 'sqrt' / ... / 'sum' / 'norm' for np.<f> and np.linalg.norm, when np is NumPy in the evaluator. """
    if self.globs.get('np') is not np or 'np' in self.cmap:
      return None
    if isinstance(func, ast.Attribute) and isinstance(func.value, ast.Name) and func.value.id == 'np':
      return func.attr
    if (isinstance(func, ast.Attribute) and func.attr == 'norm' and isinstance(func.value, ast.Attribute) and
        func.value.attr == 'linalg' and isinstance(func.value.value, ast.Name) and func.value.value.id == 'np'):
      return 'linalg.norm'
    return None

  def _call(self, node):
    if node.keywords:
      raise _Residue('keyword arguments')
    builtin = node.func.id if (isinstance(node.func, ast.Name) and node.func.id not in self.cmap and
                               node.func.id not in self.globs) else None
    npf = self._np_func(node.func)
    args = node.args
    if (builtin == 'abs' or npf in _NP_UNARY) and len(args) == 1:
      kind, code = self._scalar(args[0])
      op = 'abs' if builtin == 'abs' else _NP_UNARY[npf]
      return (kind if op == 'abs' else 'float'), code + [(op, 0, 0, 0.0)]
    if builtin == 'sum' and len(args) == 1:
      kind, cols = self._vector(args[0])
      code = [('const', 0, 0, 0.0)]
      for c in cols:
        code += [('col', c, 0, 0.0), ('add', int(kind == 'int'), 0, 0.0)]
      return kind, code
    if npf in ('sum', 'linalg.norm') and len(args) == 1:
      kind, cols = self._vector(args[0])
      if not 1 <= len(cols) <= MAX_VEC:
        raise _Residue('vector length')
      code = [('col', c, 0, 0.0) for c in cols]
      if npf == 'sum' and kind == 'int':                  # integer sums are exact in any order
        return 'int', code + [('add', 1, 0, 0.0)] * (len(cols) - 1)
      if npf == 'linalg.norm' and kind == 'int':          # x.dot(x) in int64, then sqrt
        code = []
        for j, c in enumerate(cols):
          code += [('col', c, 0, 0.0), ('col', c, 0, 0.0), ('mul', 1, 0, 0.0)] + ([('add', 1, 0, 0.0)] if j else [])
        return 'float', code + [('sqrt', 0, 0, 0.0)]
      return 'float', code + [('npsum' if npf == 'sum' else 'norm', len(cols), 0, 0.0)]
    if builtin in ('min', 'max') and len(args) >= 1:
      if len(args) == 1:
        kind, cols = self._vector(args[0])
        items = [(kind, [('col', c, 0, 0.0)]) for c in cols]
      else:
        items = [self._scalar(a) for a in args]
      if not items:
        raise _Residue('empty min / max')
      code = list(items[0][1])
      for _, c in items[1:]:
        code += c + [(builtin, 0, 0, 0.0)]
      kinds = {k for k, _ in items}
      return ('int' if kinds == {'int'} else 'float'), code
    raise _Residue('call')


def _stack_depth(code):
  depth, peak = 0, 0
  pops = {'col': -1, 'const': -1, 'lookup': -1, 'neg': 0, 'abs': 0, 'sqrt': 0, 'exp': 0, 'log': 0, 'pow': 0,
          'not': 0, 'accept': 1}
  for op, arg, _, _ in code:
    if op in ('npsum', 'norm'):
      depth -= arg - 1
    else:
      depth -= pops.get(op, 1)
    peak = max(peak, depth)
  return peak


class ConstraintFilter(object):
  """ A domain's constraints split into the device program (ops, arg, arg2, val and the lookup tables) and the host
      residue.  n_compiled: constraints in the program; residue: indices of the constraints left on the host. """

  def __init__(self, domain, code, tab_key, tab_val, n_compiled, residue, n_cols):
    self.domain, self.code, self.n_compiled, self.residue, self.n_cols = domain, code, n_compiled, residue, n_cols
    self.op = np.array([OP[c[0]] for c in code], dtype=np.int32)
    self.arg = np.array([c[1] for c in code], dtype=np.int32)
    self.arg2 = np.array([c[2] for c in code], dtype=np.int32)
    self.val = np.array([c[3] for c in code], dtype=np.float64)
    self.tab_key = np.array(tab_key, dtype=np.float64)
    self.tab_val = np.array(tab_val, dtype=np.float64)

  def desc(self):
    """ The dfb_cons_prog descriptor of the program. """
    from . import _lib
    d = _lib.ConsProg()
    d.n_ops, d.n_tab, d.n_cols = len(self.op), len(self.tab_key), self.n_cols
    d.op[:len(self.op)] = self.op.tolist()
    d.arg[:len(self.op)] = self.arg.tolist()
    d.arg2[:len(self.op)] = self.arg2.tolist()
    d.val[:len(self.op)] = self.val.tolist()
    d.tab_key[:len(self.tab_key)] = self.tab_key.tolist()
    d.tab_val[:len(self.tab_key)] = self.tab_val.tolist()
    return d

  def host_rows(self, status):
    """ Indices of the rows whose status the host must settle with the domain's own evaluator. """
    status = np.asarray(status)
    if self.residue:
      return np.flatnonzero(status != REJECT)
    return np.flatnonzero(status == UNDECIDED)

  def settle(self, status, point_of, need=None):
    """ status with the rows of host_rows decided by domain.constraints_are_satisfied(point_of(i)), in row order.  need:
        only the first `need` accepted rows matter -- the host stops once they are known and rejects the host rows after
        them, so at most need accepted rows (plus the rejected ones before them) are evaluated. """
    status = np.array(status, dtype=np.uint8)
    host = self.host_rows(status)
    fixed = (status == ACCEPT)
    fixed[host] = False
    before = np.concatenate(([0], np.cumsum(fixed)))       # fixed ACCEPT rows before row i
    got = 0
    for k, i in enumerate(host):
      if need is not None and before[i] + got >= need:
        status[host[k:]] = REJECT
        break
      ok = self.domain.constraints_are_satisfied(point_of(int(i)))
      status[i] = ACCEPT if ok else REJECT
      got += int(bool(ok))
    return status


def readable(domain):
  """ True when the constraints of a constrained domain can be read: the list, the raw orderings and the evaluator. """
  return all(getattr(domain, a, None) is not None for a in ('domain_constraints', 'raw_name_ordering', 'get_raw_point',
                                                              'constraints_are_satisfied'))


def compile_filter(domain, parts, levels=False):
  """ The ConstraintFilter of a constrained domain whose candidate columns are laid out by `parts` (gpb_acquisitions
      ._cp_parts).  levels: the rows hold level indices in discrete columns instead of their column values. """
  cmap = column_map(domain, parts)
  evaluator = getattr(domain, 'str_constraint_evaluator', None)
  globs = getattr(evaluator, '__globals__', None) or {'np': np}
  comp = _Compiler(cmap, parts, globs, levels)
  code, residue, n_compiled = [], [], 0
  for idx, c in enumerate(domain.domain_constraints):
    con = c['constraint']
    if not isinstance(con, str) or con.endswith('.py'):
      residue.append(idx)
      continue
    n_key = len(comp.tab_key)
    try:
      kind, cc = comp.node(ast.parse(con.strip(), mode='eval').body)
      if kind != 'bool':
        raise _Residue('not a bool')
      cc = cc + [('accept', 0, 0, 0.0)]
      if len(code) + len(cc) > MAX_OPS or _stack_depth(cc) > MAX_STACK:
        raise _Residue('program too large')
    except (_Residue, SyntaxError, RecursionError):
      del comp.tab_key[n_key:], comp.tab_val[n_key:]
      residue.append(idx)
      continue
    code += cc
    n_compiled += 1
  return ConstraintFilter(domain, code, comp.tab_key, comp.tab_val, n_compiled, residue,
                          sum(p.dim for p in parts))
