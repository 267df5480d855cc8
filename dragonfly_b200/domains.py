"""
Minimal mirrors of the domains on the hot path (dragonfly/exd/domains.py): EuclideanDomain (:71-115), and the parts of
a Cartesian-product domain the device serves -- IntegralDomain (:109-146), ProdDiscreteDomain (:254-295),
ProdDiscreteNumericDomain (:298-331) and CartesianProductDomain (:334-480).  anc_data.domain only needs get_type(),
get_dim(), .bounds / .list_of_list_of_items / .list_of_domains and has_constraints(); the reference's own domain
objects provide the same and work as well.  A CartesianProductDomain may carry the reference's domain constraints
(domains.py:350-460) with the orderings of the config it came from (cp_domain_utils.py:169-294).
"""
import numpy as np


class EuclideanDomain(object):
  """ Domain for Euclidean spaces: bounds is a (dim, 2) array of [lower, upper]. """

  def __init__(self, bounds):
    self.bounds = np.array(bounds, dtype=np.float64)
    self.diameter = np.linalg.norm(self.bounds[:, 1] - self.bounds[:, 0])
    self.dim = len(bounds)

  def get_type(self):
    return 'euclidean'

  def get_dim(self):
    return self.dim

  def is_a_member(self, point):
    point = np.asarray(point)
    return bool(len(point) == self.dim and np.all(point >= self.bounds[:, 0])
                and np.all(point <= self.bounds[:, 1]))

  def __str__(self):
    return 'Euclidean: %s' % (self.bounds.tolist())


class IntegralDomain(object):
  """ Vectors of integers in [lower, upper] per coordinate; bounds is a (dim, 2) integer array. """

  def __init__(self, bounds):
    self.bounds = np.array(bounds, dtype=np.int64)
    self.diameter = np.linalg.norm(self.bounds[:, 1] - self.bounds[:, 0])
    self.dim = len(bounds)

  def get_type(self):
    return 'integral'

  def get_dim(self):
    return self.dim

  def __str__(self):
    return 'Integral: %s' % (self.bounds.tolist())


class ProdDiscreteDomain(object):
  """ A product of finite sets of categories: list_of_list_of_items[q] lists the values of coordinate q. """

  def __init__(self, list_of_list_of_items):
    self.list_of_list_of_items = list_of_list_of_items
    self.dim = len(list_of_list_of_items)
    self.size = np.prod([len(loi) for loi in list_of_list_of_items])

  def get_type(self):
    return 'prod_discrete'

  def get_dim(self):
    return self.dim

  def __str__(self):
    return 'ProdDiscrete: %s' % (self.list_of_list_of_items)


class ProdDiscreteNumericDomain(ProdDiscreteDomain):
  """ A product of finite sets of numbers. """

  def __init__(self, list_of_list_of_items):
    if not all(all(isinstance(v, (int, float, np.integer, np.floating)) for v in loi)
               for loi in list_of_list_of_items):
      raise ValueError('list_of_list_of_items must of a list where each element is a list of numeric objects.')
    super(ProdDiscreteNumericDomain, self).__init__(list_of_list_of_items)

  def get_type(self):
    return 'prod_discrete_numeric'


def evaluate_strings_with_given_variables(strs_to_execute, variable_dict=None):
  """ general_utils.py:236-258: each string eval'd with the variables bound and this module's globals (np, ...). """
  return [eval(elem, globals(), dict(variable_dict or {})) for elem in strs_to_execute]  # pylint: disable=eval-used


def _flatten(L):
  """ general_utils.flatten_list_of_objects_and_iterables (:311-321). """
  ret = []
  for elem in L:
    if hasattr(elem, '__iter__') and not isinstance(elem, str):
      ret.extend(elem)
    else:
      ret.append(elem)
  return ret


def _unpack_vectorised_domain(x, dim_ordering):
  """ cp_domain_utils.py:306-318 """
  ret, counter = [None] * len(dim_ordering), 0
  for idx, num_dims in enumerate(dim_ordering):
    if num_dims == '':
      ret[idx] = x[counter]
      counter += 1
    else:
      ret[idx] = x[counter:counter + num_dims]
      counter += num_dims
  assert counter == len(x)
  return ret


class CartesianProductDomain(object):
  """ The Cartesian product of list_of_domains; a point is a list whose j-th element lies in list_of_domains[j].
      domain_constraints (optional): the reference's list of {'name', 'constraint'} dicts, a constraint being a Python
      expression string over the raw variable names or a callable of the raw point; it needs the config's orderings
      (raw_name_ordering, index_ordering, dim_ordering) to form raw points.  Without it has_constraints() is False. """

  def __init__(self, list_of_domains, domain_constraints=None, raw_name_ordering=None, index_ordering=None,
               dim_ordering=None):
    self.list_of_domains = list_of_domains
    self.num_domains = len(list_of_domains)
    self.dim = sum([dom.get_dim() for dom in self.list_of_domains])
    self._has_constraints = domain_constraints is not None
    if raw_name_ordering is not None:
      self.raw_name_ordering = list(raw_name_ordering)
      self.index_ordering, self.dim_ordering = index_ordering, dim_ordering
    if self._has_constraints:
      if raw_name_ordering is None:
        raise ValueError('A constrained domain needs the orderings of its raw variables.')
      self.str_constraint_evaluator = evaluate_strings_with_given_variables
      self.domain_constraints = list(domain_constraints)
      self.num_domain_constraints = len(self.domain_constraints)
      cons = [c['constraint'] for c in self.domain_constraints]
      if any(isinstance(c, str) and c.endswith('.py') for c in cons):
        raise ValueError('Constraints can be specified in a python file only when using a configuration file.')
      self.eval_as_str_idxs = [k for k, c in enumerate(cons) if isinstance(c, str)]
      self.eval_as_pyfunc_idxs = [k for k, c in enumerate(cons) if hasattr(c, '__call__')]
      self.str_constraints = [cons[k] for k in self.eval_as_str_idxs]
      self.pyfunc_constraints = [cons[k] for k in self.eval_as_pyfunc_idxs]

  def get_type(self):
    return 'cartesian_product'

  def get_dim(self):
    return self.dim

  def has_constraints(self):
    return self._has_constraints

  def get_raw_point(self, proc_x):
    """ get_raw_point_from_processed_point (cp_domain_utils.py:342-361) for a Cartesian-product domain. """
    repacked_x = []
    for idx, raw_dim in enumerate(self.dim_ordering):
      if isinstance(raw_dim, list):
        repacked_x.append(_unpack_vectorised_domain(proc_x[idx], raw_dim))
      elif raw_dim == '':
        repacked_x.append(proc_x[idx])
      else:
        repacked_x.append([proc_x[idx]])
    repacked_x = _flatten(repacked_x)
    ordering = _flatten(self.index_ordering)
    ret = [None] * len(ordering)
    for orig_idx, ordered_idx in enumerate(ordering):
      ret[ordered_idx] = repacked_x[orig_idx]
    return ret

  def constraints_are_satisfied(self, point):
    """ domains.py:427-440: every constraint evaluated on the raw point; each must return a bool. """
    if not self._has_constraints:
      return True
    raw_point = self.get_raw_point(point)
    names = dict(zip(self.raw_name_ordering, raw_point))
    ret_all = [None] * self.num_domain_constraints
    for k, v in zip(self.eval_as_str_idxs, self.str_constraint_evaluator(self.str_constraints, names)):
      ret_all[k] = v
    for k, fn in zip(self.eval_as_pyfunc_idxs, self.pyfunc_constraints):
      ret_all[k] = fn(raw_point)
    for idx, elem in enumerate(ret_all):
      if not isinstance(elem, (bool, np.bool_)):
        raise ValueError('Constraint %d:%s returned %s. It should return type bool.' % (
            idx, self.domain_constraints[idx].get('name'), str(elem)))
    return all(ret_all)

  def __str__(self):
    return 'CartProd(N=%d,d=%d)::[%s]' % (self.num_domains, self.dim,
                                          ', '.join([str(d) for d in self.list_of_domains]))
