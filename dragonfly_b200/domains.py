"""
Minimal mirrors of the domains on the hot path (dragonfly/exd/domains.py): EuclideanDomain (:71-115), and the parts of
a Cartesian-product domain the device serves -- IntegralDomain (:109-146), ProdDiscreteDomain (:254-295),
ProdDiscreteNumericDomain (:298-331) and CartesianProductDomain (:334-480).  anc_data.domain only needs get_type(),
get_dim(), .bounds / .list_of_list_of_items / .list_of_domains and has_constraints(); the reference's own domain
objects provide the same and work as well.
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


class CartesianProductDomain(object):
  """ The Cartesian product of list_of_domains; a point is a list whose j-th element lies in list_of_domains[j].
      Constraints are not mirrored: has_constraints() is False. """

  def __init__(self, list_of_domains):
    self.list_of_domains = list_of_domains
    self.num_domains = len(list_of_domains)
    self.dim = sum([dom.get_dim() for dom in self.list_of_domains])

  def get_type(self):
    return 'cartesian_product'

  def get_dim(self):
    return self.dim

  def has_constraints(self):
    return False

  def __str__(self):
    return 'CartProd(N=%d,d=%d)::[%s]' % (self.num_domains, self.dim,
                                          ', '.join([str(d) for d in self.list_of_domains]))
