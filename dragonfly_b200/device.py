"""
Device-side objects behind the Python host: a `DevicePosterior` wraps one libdfb200 handle plus the
torch-owned workspace it computes in.  PyTorch appears here only as the allocator of device buffers
and the owner of CUDA streams; every numeric result comes from libdfb200's CUDA kernels.
"""
import ctypes as C
import weakref

import numpy as np
import torch

from . import _lib
from .kernel import build_descriptor


def _require_cuda(device=None):
  if not torch.cuda.is_available():
    raise RuntimeError('dragonfly_b200 needs a CUDA device (H100, sm_90a); none is visible and '
                       'there is no CPU fallback.')
  if device is None:
    device = torch.cuda.current_device()
  return torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)


def _dev_f64(arr, device):
  """ Host array-like or torch tensor -> contiguous fp64 CUDA tensor on `device`. """
  if isinstance(arr, torch.Tensor):
    return arr.to(device=device, dtype=torch.float64).contiguous()
  return torch.from_numpy(np.ascontiguousarray(np.asarray(arr, dtype=np.float64))).to(device)


# Options applied to every new DevicePosterior (name -> int), e.g. {'score_impl': 0} to force the fp64
# DMMA contraction everywhere.  See dfb_set_option in include/dfb200.h.
DEFAULT_OPTIONS = {}

# A BO loop builds a fresh GP (hence a fresh handle) every iteration; the ~1.3 GB workspace of an N = 5000
# posterior is recycled through this small per-(device, size) pool rather than through cudaMalloc /
# cudaFree, whose cost (tens of ms, variable) would otherwise sit inside every build_posterior.
_WORKSPACE_POOL = {}
_WORKSPACE_POOL_DEPTH = 2


def _take_workspace(key, dev):
  free = _WORKSPACE_POOL.get(key)
  if free:
    return free.pop()
  return torch.empty(key[1] + 256, dtype=torch.uint8, device=dev)


def _give_workspace(key, ws):
  if ws is None:
    return
  free = _WORKSPACE_POOL.setdefault(key, [])
  if len(free) < _WORKSPACE_POOL_DEPTH:
    free.append(ws)


def release_workspaces():
  """ Drops the pooled workspaces (returns the memory to torch's allocator). """
  _WORKSPACE_POOL.clear()


class DevicePosterior(object):
  """ One handle + workspace.  Immutable once built (GP objects replace, never mutate, it), so
      shallow / deep copies of a GP may share it (gpb_acquisitions.py:104, unittest_mf_gp.py:109). """

  def __init__(self, n_max, device=None, chunk=0):
    self.lib = _lib.load()
    self.device = _require_cuda(device)
    self.n_max = int(n_max)
    hp = C.c_void_p()
    _lib.check(self.lib.dfb_create(C.byref(hp), self.device.index), 'dfb_create')
    self.h = hp
    nbytes = self.lib.dfb_workspace_bytes(self.n_max, 0, int(chunk))
    self._pool_key = (self.device.index, int(nbytes))
    self.workspace = _take_workspace(self._pool_key, self.device)
    ptr = (self.workspace.data_ptr() + 255) // 256 * 256
    with torch.cuda.device(self.device):
      stream = torch.cuda.current_stream(self.device).cuda_stream
      _lib.check(self.lib.dfb_set_stream(self.h, C.c_void_p(stream)), 'dfb_set_stream')
      _lib.check(self.lib.dfb_set_workspace(self.h, C.c_void_p(ptr), C.c_size_t(nbytes), self.n_max,
                                            int(chunk)), 'dfb_set_workspace')
    self.n = 0
    self.dim = 0
    self.lml = None
    self._owners = weakref.WeakSet()      # GP objects using this posterior (gp_core.GP._post_is_shared)
    # joint-posterior blocks (covariance / Thompson draws) must fit the handle's scoring chunk
    self.TS_BLOCK = min(DevicePosterior.TS_BLOCK, int(self.query('chunk')))
    for _name, _value in DEFAULT_OPTIONS.items():
      self.set_option(_name, _value)
    self._keep = []      # tensors that must outlive asynchronous use

  def __del__(self):
    try:
      if getattr(self, 'h', None) is not None and self.h.value:
        torch.cuda.synchronize(self.device)
        self.lib.dfb_destroy(self.h)
        self.h = None
        _give_workspace(self._pool_key, self.workspace)
        self.workspace = None
    except Exception:  # pylint: disable=broad-except
      pass

  def bind_current_stream(self):
    """ Issue this handle's work on the calling thread's current torch stream from now on. """
    stream = torch.cuda.current_stream(self.device).cuda_stream
    _lib.check(self.lib.dfb_set_stream(self.h, C.c_void_p(stream)), 'dfb_set_stream')

  # -- model ------------------------------------------------------------------------------------
  def set_kernel(self, desc):
    _lib.check(self.lib.dfb_set_kernel(self.h, C.byref(desc)), 'dfb_set_kernel')

  def set_test_kernel(self, desc):
    if desc is None:
      _lib.check(self.lib.dfb_set_test_kernel(self.h, None), 'dfb_set_test_kernel')
    else:
      _lib.check(self.lib.dfb_set_test_kernel(self.h, C.byref(desc)), 'dfb_set_test_kernel')

  def set_train(self, X, y_centred):
    Xd = _dev_f64(X, self.device)
    yd = _dev_f64(y_centred, self.device)
    self.n, self.dim = int(Xd.shape[0]), int(Xd.shape[1])
    _lib.check(self.lib.dfb_set_train(self.h, C.c_void_p(Xd.data_ptr()), self.n, self.dim,
                                      C.c_void_p(yd.data_ptr())), 'dfb_set_train')
    torch.cuda.synchronize(self.device)

  def build(self, noise_var, jitter=0.0, flags=_lib.DFB_BUILD_FULL):
    """ Returns (info, lml): info > 0 means 'not positive definite' (np.linalg.LinAlgError). """
    lml = C.c_double(0.0)
    info = _lib.check(self.lib.dfb_build_posterior(self.h, float(noise_var), float(jitter), int(flags),
                                                   C.byref(lml)), 'dfb_build_posterior')
    self.lml = lml.value if info == 0 else None
    return info, self.lml

  def lml_batch(self, descs, noise_vars, mean_consts, mixed=False):
    """ dfb_lml_batch on the training set of set_train (pass the raw Y, mean 0): one LML-only build per item, all in one
        launch.  Returns (lmls, infos); an item with info > 0 is not positive definite and its lml is NaN.  mixed: call
        dfb_lml_batch_mixed, which also evaluates HAMMING factors (Cartesian-product kernels with categorical parts). """
    B = len(descs)
    arr = (_lib.KernelDesc * B)(*descs)
    noise = np.ascontiguousarray(noise_vars, dtype=np.float64)
    mean = np.ascontiguousarray(mean_consts, dtype=np.float64)
    assert len(noise) == B and len(mean) == B
    lmls = np.empty(B)
    infos = np.empty(B, dtype=np.int32)
    name = 'dfb_lml_batch_mixed' if mixed else 'dfb_lml_batch'
    _lib.check(getattr(self.lib, name)(self.h, arr, noise.ctypes.data_as(C.POINTER(C.c_double)),
                                       mean.ctypes.data_as(C.POINTER(C.c_double)), B,
                                       lmls.ctypes.data_as(C.POINTER(C.c_double)),
                                       infos.ctypes.data_as(C.POINTER(C.c_int32))), name)
    return lmls, infos

  def capacity(self):
    """ Training points this posterior can hold without a rebuild: its padded size (a multiple of 128). """
    return (self.n + 127) // 128 * 128

  def extend(self, X_new, y_centred_new, flags=_lib.DFB_BUILD_FULL, save=False):
    """ dfb_extend_posterior: appends training points to the built posterior in O(N^2) work.
        Returns (info, lml); info > 0 = the extended matrix is not positive definite (with save=True
        the un-extended posterior is back in place, otherwise it must be rebuilt). """
    Xd = _dev_f64(X_new, self.device)
    yd = _dev_f64(y_centred_new, self.device)
    q = int(Xd.shape[0])
    assert int(Xd.shape[1]) == self.dim and int(yd.shape[0]) == q
    lml = C.c_double(0.0)
    info = _lib.check(self.lib.dfb_extend_posterior(
        self.h, C.c_void_p(Xd.data_ptr()), q, C.c_void_p(yd.data_ptr()),
        int(flags) | (_lib.DFB_EXTEND_SAVE if save else 0), C.byref(lml)), 'dfb_extend_posterior')
    if info == 0:
      self.n += q
      self.lml = lml.value
    return info, (lml.value if info == 0 else None)

  def restore(self, n_before):
    """ dfb_restore_posterior: undoes an extend(..., save=True) bit for bit. """
    _lib.check(self.lib.dfb_restore_posterior(self.h), 'dfb_restore_posterior')
    self.n = int(n_before)

  def lml_gradients(self, dim):
    """ dfb_lml_gradients: [scale, noise_var / noise_var, noise_mean, same_dim_bandwidths, dim_bandwidths[0..d)]. """
    out = (C.c_double * (4 + int(dim)))()
    st = self.lib.dfb_lml_gradients(self.h, out, 4 + int(dim))
    if st == -3:
      raise NotImplementedError(_lib.last_error())
    _lib.check(st, 'dfb_lml_gradients')
    return np.array(out[:], dtype=np.float64)

  def max_diag(self):
    out = C.c_double(0.0)
    _lib.check(self.lib.dfb_get_max_diag(self.h, C.byref(out)), 'dfb_get_max_diag')
    return out.value

  def get_state(self, want_L=False, want_alpha=False, want_K=False):
    L = torch.empty((self.n, self.n), dtype=torch.float64, device=self.device) if want_L else None
    a = torch.empty((self.n,), dtype=torch.float64, device=self.device) if want_alpha else None
    K = torch.empty((self.n, self.n), dtype=torch.float64, device=self.device) if want_K else None
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(self.lib.dfb_get_state(self.h, ptr(L), ptr(a), ptr(K)), 'dfb_get_state')
    return L, a, K

  def set_alpha(self, alpha):
    ad = _dev_f64(alpha, self.device)
    _lib.check(self.lib.dfb_set_alpha(self.h, C.c_void_p(ad.data_ptr()), int(ad.shape[0])),
               'dfb_set_alpha')
    torch.cuda.synchronize(self.device)

  # -- prediction ---------------------------------------------------------------------------------
  def _operands(self, Xc, z=None):
    """ Candidate rows Xc (and normals z) as the scoring calls take them: (X, z, DFB_HOST or DFB_DEVICE, ptr, vec).
        A host Xc stays on the host (the C call copies it) with host outputs, a CUDA tensor stays on the device with
        CUDA outputs.  A C-contiguous float64 host array is used as is, not copied: page-locked slabs must stay
        page-locked to take the double-buffered copies.  ptr(a) is the C pointer of X, z or an output (NULL for None);
        vec() allocates one output vector of len(X) in the same memory space. """
    if isinstance(Xc, torch.Tensor):
      X = _dev_f64(Xc, self.device)
      z = None if z is None else _dev_f64(z, self.device).reshape(-1)
      vec = lambda: torch.empty((int(X.shape[0]),), dtype=torch.float64, device=self.device)
      return X, z, _lib.DFB_DEVICE, lambda a: None if a is None else C.c_void_p(a.data_ptr()), vec
    X = np.ascontiguousarray(np.asarray(Xc, dtype=np.float64))
    z = None if z is None else np.ascontiguousarray(np.asarray(z, dtype=np.float64).reshape(-1))
    vec = lambda: np.empty((X.shape[0],), dtype=np.float64)
    return X, z, _lib.DFB_HOST, lambda a: None if a is None else a.ctypes.data_as(C.c_void_p), vec

  def eval(self, Xc, mean_const=0.0, want_std=True):
    """ Xc: host ndarray (results are host ndarrays, copies inside the C call) or CUDA tensor
        (results are CUDA tensors).  Returns (mu, sd or None). """
    X, _, space, ptr, vec = self._operands(Xc)
    mu, sd = vec(), (vec() if want_std else None)
    _lib.check(self.lib.dfb_eval(self.h, ptr(X), int(X.shape[0]), int(X.shape[1]), space, float(mean_const), ptr(mu),
                                 ptr(sd)), 'dfb_eval')
    return mu, sd

  def score_argmax(self, acq_desc, Xc, mean_const=0.0, want_scores=False):
    """ Fused scoring + arg-max.  Returns (best_score, best_index, scores or None). """
    bs, bi = C.c_double(0.0), C.c_int64(-1)
    X, _, space, ptr, vec = self._operands(Xc)
    sc = vec() if want_scores else None
    _lib.check(self.lib.dfb_score_argmax(self.h, C.byref(acq_desc), ptr(X), int(X.shape[0]), int(X.shape[1]), space,
                                         float(mean_const), ptr(sc), C.byref(bs), C.byref(bi)), 'dfb_score_argmax')
    return bs.value, bi.value, sc

  def score_argmax_ts(self, Xc, mean_const=0.0, z=None, seed=0, row0=0, want_scores=False):
    """ dfb_score_argmax_ts: one marginal posterior draw per candidate, mu_i + sqrt(sigma^2_i) z_i, and its arg-max.
        z: the m normals, kept in the memory space of Xc (host ndarray for a host Xc, CUDA tensor for a CUDA one), or None
        for the device's counter-based normals of (seed, row0 + row).  Returns (best_score, best_index, scores or None,
        the number of candidates whose variance is not > 0). """
    bs, bi, nonpos = C.c_double(0.0), C.c_int64(-1), C.c_int64(0)
    X, z, space, ptr, vec = self._operands(Xc, z)
    assert z is None or int(z.shape[0]) == int(X.shape[0])
    sc = vec() if want_scores else None
    _lib.check(self.lib.dfb_score_argmax_ts(
        self.h, ptr(X), int(X.shape[0]), int(X.shape[1]), space, float(mean_const), ptr(z),
        C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(row0), ptr(sc), C.byref(bs), C.byref(bi), C.byref(nonpos)),
        'dfb_score_argmax_ts')
    return bs.value, bi.value, sc, nonpos.value

  def score_groups(self, descs, betas, X, groups):
    """ dfb_score_groups: Add-UCB's per-group objective of every row, mu + beta_g sd under row r's group descriptor
        descs[groups[r]] (mean 0).  X: host (m, ldx) rows, group g's coordinates in its first descs[g].cand_dim
        columns.  Returns the m scores (host ndarray). """
    G = len(descs)
    arr = (_lib.KernelDesc * G)(*descs)
    b = np.ascontiguousarray(betas, dtype=np.float64)
    X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
    g = np.ascontiguousarray(groups, dtype=np.int32)
    assert len(b) == G and X.ndim == 2 and len(g) == len(X)
    out = np.empty((len(X),), dtype=np.float64)
    _lib.check(self.lib.dfb_score_groups(self.h, arr, b.ctypes.data_as(C.POINTER(C.c_double)), G,
                                         X.ctypes.data_as(C.c_void_p), int(X.shape[0]), int(X.shape[1]),
                                         g.ctypes.data_as(C.POINTER(C.c_int32)),
                                         out.ctypes.data_as(C.c_void_p)), 'dfb_score_groups')
    return out

  # -- joint posterior over one block, or over all candidates: covariance and Thompson draws ---------
  TS_BLOCK = 4096
  # Above TS_BLOCK and up to TS_JOINT_MAX candidates, the covariance and the draws are formed over all candidates at
  # once in a joint workspace (about 8 Mpad^2 + 8 Mpad npad bytes: 2.9 GB at M = 16384, N = 5000), allocated on the
  # first such call and grown when a larger M comes.  The form depends on M alone; a joint call that cannot get its
  # workspace raises.
  TS_JOINT_MAX = 16384

  def _ensure_workspace_for(self, m):
    if m <= self.TS_BLOCK:
      self._ensure_ts_workspace(m)
    elif m <= self.TS_JOINT_MAX:
      self._ensure_joint_workspace(m)
    else:
      raise ValueError('%d candidates: the joint posterior takes at most %d (TS_JOINT_MAX).' % (m, self.TS_JOINT_MAX))

  def _ensure_joint_workspace(self, m):
    if getattr(self, '_js_m', 0) >= m:
      return
    mj = min(self.TS_JOINT_MAX, (int(m) + 1023) // 1024 * 1024)
    # Give the old workspace back before taking a larger one.  The handle still points into it until
    # dfb_set_joint_workspace succeeds, so no capacity is recorded meanwhile: if the allocation below raises, the next
    # joint call allocates again instead of writing into memory the caching allocator may have handed on.
    self._js_m = 0
    self._js_workspace = None
    nbytes = self.lib.dfb_joint_workspace_bytes(self.n_max, mj)
    self._js_workspace = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
    ptr = (self._js_workspace.data_ptr() + 255) // 256 * 256
    _lib.check(self.lib.dfb_set_joint_workspace(self.h, C.c_void_p(ptr), C.c_size_t(nbytes), mj),
               'dfb_set_joint_workspace')
    self._js_m = mj

  def _ensure_ts_workspace(self, m):
    mb = getattr(self, '_ts_mb', 0)
    if mb >= m:
      return
    mb = max(int(m), 512)
    nbytes = self.lib.dfb_ts_workspace_bytes(self.n_max, mb)
    self._ts_workspace = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=self.device)
    ptr = (self._ts_workspace.data_ptr() + 255) // 256 * 256
    _lib.check(self.lib.dfb_set_ts_workspace(self.h, C.c_void_p(ptr), C.c_size_t(nbytes), mb),
               'dfb_set_ts_workspace')
    self._ts_mb = mb

  def eval_covar(self, Xc, mean_const=0.0):
    """ (mu, covar) of GP.eval(X, 'covar') for up to TS_JOINT_MAX candidates (one block up to TS_BLOCK);
        host ndarray in -> host ndarrays out. """
    Xd = _dev_f64(Xc, self.device)
    m, dc = int(Xd.shape[0]), int(Xd.shape[1])
    self._ensure_workspace_for(m)
    mu = torch.empty((m,), dtype=torch.float64, device=self.device)
    cov = torch.empty((m, m), dtype=torch.float64, device=self.device)
    _lib.check(self.lib.dfb_eval_covar(self.h, C.c_void_p(Xd.data_ptr()), m, dc, float(mean_const),
                                       C.c_void_p(mu.data_ptr()), C.c_void_p(cov.data_ptr())),
               'dfb_eval_covar')
    if isinstance(Xc, torch.Tensor):
      return mu, cov
    return mu.cpu().numpy(), cov.cpu().numpy()

  def ts_draws(self, Xc, Ut, mean_const=0.0, jitter=0.0):
    """ One attempt of draw_gaussian_samples on a block (m <= TS_BLOCK, S <= 256), or jointly over all
        m <= TS_JOINT_MAX candidates (any S, one factorisation): returns (info, samples (S, m), max_diag). """
    Xd = _dev_f64(Xc, self.device)
    Ud = _dev_f64(Ut, self.device)
    m, dc = int(Xd.shape[0]), int(Xd.shape[1])
    S = int(Ud.shape[0])
    assert int(Ud.shape[1]) == m
    self._ensure_workspace_for(m)
    out = torch.empty((S, m), dtype=torch.float64, device=self.device)
    mx = C.c_double(0.0)
    info = _lib.check(self.lib.dfb_ts_draws(self.h, C.c_void_p(Xd.data_ptr()), m, dc, float(mean_const),
                                            C.c_void_p(Ud.data_ptr()), S, float(jitter),
                                            C.c_void_p(out.data_ptr()), None, C.byref(mx)),
                      'dfb_ts_draws')
    return info, out, mx.value

  def moo_score_argmax(self, kind, a_list, b_list, weights, refs=None, beta=0.0, want_scores=False):
    """ dfb_moo_score_argmax: scalarise n_obj objectives' device vectors and take the arg-max.
        a_list / b_list: CUDA fp64 tensors (mu_k or sampled values; sd_k or None).
        Returns (best_score, best_index, scores tensor or None). """
    d, m, a_ptrs, b_ptrs, keep = self._moo_operands(kind, a_list, b_list, weights, refs, beta)
    sc = torch.empty((m,), dtype=torch.float64, device=self.device) if want_scores else None
    bs, bi = C.c_double(0.0), C.c_int64(-1)
    _lib.check(self.lib.dfb_moo_score_argmax(
        self.h, C.byref(d), a_ptrs, b_ptrs, m, C.c_void_p(sc.data_ptr()) if want_scores else None,
        C.byref(bs), C.byref(bi)), 'dfb_moo_score_argmax')
    del keep                      # the call has synchronised: the vectors may go
    return bs.value, bi.value, sc

  def moo_score_argmax_ts(self, kind, mu_list, sd_list, weights, refs=None, z=None, seed=0, row0=0, want_scores=False):
    """ dfb_moo_score_argmax_ts: one marginal posterior draw per candidate and objective, fl(fl(sd_k z_k) + mu_k),
        scalarised by kind (DFB_MOO_LIN_VAL / DFB_MOO_TCH_VAL), and its arg-max.  mu_list / sd_list: the objectives'
        dfb_eval vectors (CUDA fp64 tensors); z: the (m, n_obj) normals (host or device), or None for the device's
        counter-based normals of (seed, row0 + row, objective).  Returns (best_score, best_index, scores tensor or None,
        the number of candidates with a variance that is not > 0). """
    d, m, mu_ptrs, sd_ptrs, keep = self._moo_operands(kind, mu_list, sd_list, weights, refs, 0.0)
    zd = None if z is None else _dev_f64(z, self.device)
    assert zd is None or tuple(zd.shape) == (m, len(mu_list))
    sc = torch.empty((m,), dtype=torch.float64, device=self.device) if want_scores else None
    bs, bi, nonpos = C.c_double(0.0), C.c_int64(-1), C.c_int64(0)
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    _lib.check(self.lib.dfb_moo_score_argmax_ts(
        self.h, C.byref(d), mu_ptrs, sd_ptrs, m, ptr(zd), C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(row0),
        ptr(sc), C.byref(bs), C.byref(bi), C.byref(nonpos)), 'dfb_moo_score_argmax_ts')
    del keep
    return bs.value, bi.value, sc, nonpos.value

  def _moo_operands(self, kind, a_list, b_list, weights, refs, beta):
    """ The dfb_moo_desc of n_obj = len(a_list) objectives and the C arrays of their device vectors: (desc, m, a pointers,
        b pointers or None, the device tensors the pointers point into). """
    K = len(a_list)
    d = _lib.MooDesc()
    d.kind, d.n_obj, d.beta = int(kind), K, float(beta)
    for k in range(K):
      d.weight[k] = float(weights[k])
      d.ref[k] = float(refs[k]) if refs is not None else 0.0
    a_t = [_dev_f64(a, self.device) for a in a_list]
    b_t = [_dev_f64(b, self.device) for b in b_list] if b_list is not None else None
    m = int(a_t[0].shape[0])
    assert all(int(t.shape[0]) == m for t in a_t) and (b_t is None or all(int(t.shape[0]) == m for t in b_t))
    PtrArr = C.c_void_p * K
    a_ptrs = PtrArr(*[t.data_ptr() for t in a_t])
    b_ptrs = PtrArr(*[t.data_ptr() for t in b_t]) if b_t is not None else None
    return d, m, a_ptrs, b_ptrs, (a_t, b_t)

  def fill_rng(self, seed, col0, S, m, what=_lib.DFB_RNG_NORMAL, out=None):
    """ dfb_fill_rng: the S x m matrix of counter-based normals / uniforms for global columns col0 .. col0+m-1. """
    if out is None:
      out = torch.empty((int(S), int(m)), dtype=torch.float64, device=self.device)
    _lib.check(self.lib.dfb_fill_rng(self.h, C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(col0), int(S), int(m),
                                     int(what), C.c_void_p(out.data_ptr())), 'dfb_fill_rng')
    return out

  def fill_candidates(self, seed, row0, m, bounds, out=None):
    """ dfb_fill_candidates: rows row0 .. row0+m-1 of the device-generated candidate matrix (m x d CUDA tensor);
        bounds: (d, 2) array-like of [lo, hi]. """
    b = np.ascontiguousarray(np.asarray(bounds, dtype=np.float64))
    d = int(b.shape[0])
    lo = np.ascontiguousarray(b[:, 0]); hi = np.ascontiguousarray(b[:, 1])
    if out is None:
      out = torch.empty((int(m), d), dtype=torch.float64, device=self.device)
    _lib.check(self.lib.dfb_fill_candidates(self.h, C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(row0), int(m), d,
                                            lo.ctypes.data_as(C.POINTER(C.c_double)),
                                            hi.ctypes.data_as(C.POINTER(C.c_double)),
                                            C.c_void_p(out.data_ptr())), 'dfb_fill_candidates')
    return out

  def fill_mixed_candidates(self, seed, row0, m, kinds, bounds, n_levels, out=None):
    """ dfb_fill_mixed_candidates: rows row0 .. row0+m-1 of the device-generated candidate matrix of a Cartesian-product
        domain; kinds: per column DFB_CAND_*; bounds: (d, 2) [lo, hi] (read for real / integer columns); n_levels: per
        column number of categories (read for categorical columns). """
    k = np.ascontiguousarray(np.asarray(kinds, dtype=np.int32))
    b = np.ascontiguousarray(np.asarray(bounds, dtype=np.float64)).reshape(-1, 2)
    lv = np.ascontiguousarray(np.asarray(n_levels, dtype=np.int64))
    d = int(k.shape[0])
    lo = np.ascontiguousarray(b[:, 0]); hi = np.ascontiguousarray(b[:, 1])
    if out is None:
      out = torch.empty((int(m), d), dtype=torch.float64, device=self.device)
    _lib.check(self.lib.dfb_fill_mixed_candidates(
        self.h, C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(row0), int(m), d,
        k.ctypes.data_as(C.POINTER(C.c_int32)), lo.ctypes.data_as(C.POINTER(C.c_double)),
        hi.ctypes.data_as(C.POINTER(C.c_double)), lv.ctypes.data_as(C.POINTER(C.c_int64)),
        C.c_void_p(out.data_ptr())), 'dfb_fill_mixed_candidates')
    return out

  def ga_maximise(self, acq_desc, mean_const, ga_desc, seed, n_init, n_total):
    """ dfb_ga_maximise: the whole GA search on the device.  Returns (best value, best index, best level row, the
        n_total x d level rows, the n_total values), the last two CUDA tensors. """
    d = int(ga_desc.d)
    rows = torch.empty((int(n_total), d), dtype=torch.float64, device=self.device)
    vals = torch.empty((int(n_total),), dtype=torch.float64, device=self.device)
    coded = torch.empty((max(int(n_init), 5), d), dtype=torch.float64, device=self.device)
    bv, bi, row = C.c_double(0.0), C.c_int64(-1), (C.c_double * d)()
    _lib.check(self.lib.dfb_ga_maximise(
        self.h, C.byref(acq_desc), float(mean_const), C.byref(ga_desc), C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF),
        int(n_init), int(n_total), C.c_void_p(rows.data_ptr()), C.c_void_p(vals.data_ptr()),
        C.c_void_p(coded.data_ptr()), C.byref(bv), C.byref(bi), row), 'dfb_ga_maximise')
    return bv.value, bi.value, np.array(row[:], dtype=np.float64), rows, vals

  def ts_argmax(self, samples, idx_base, best, index, reset):
    """ dfb_ts_argmax: fold one block of draws (S x m CUDA tensor) into the running per-draw arg-max. """
    S, m = int(samples.shape[0]), int(samples.shape[1])
    _lib.check(self.lib.dfb_ts_argmax(self.h, C.c_void_p(samples.data_ptr()), int(samples.stride(0)), S, m,
                                      int(idx_base), 1 if reset else 0, C.c_void_p(best.data_ptr()),
                                      C.c_void_p(index.data_ptr())), 'dfb_ts_argmax')

  def launch_count(self):
    return int(self.lib.dfb_launch_count(self.h))

  def set_option(self, name, value):
    _lib.check(self.lib.dfb_set_option(self.h, name.encode('utf-8'), int(value)), 'dfb_set_option')

  def query(self, name):
    out = C.c_double(0.0)
    _lib.check(self.lib.dfb_query(self.h, name.encode('utf-8'), C.byref(out)), 'dfb_query')
    return out.value

  def profile_enable(self, on=True):
    _lib.check(self.lib.dfb_profile_enable(self.h, 1 if on else 0), 'dfb_profile_enable')

  def profile_read(self, cls):
    """ (milliseconds, launches, work units) accumulated for a kernel class; resets it. """
    ms, n, u = C.c_double(0.0), C.c_int64(0), C.c_double(0.0)
    _lib.check(self.lib.dfb_profile_read(self.h, int(cls), C.byref(ms), C.byref(n), C.byref(u)),
               'dfb_profile_read')
    return ms.value, n.value, u.value


def measure_peak(what, device=None):
  """ dfb_measure_peak: 'i8' -> int8 wgmma issue rate (int8 TOP/s), 'f64' -> DMMA issue rate (TFLOP/s). """
  dev = _require_cuda(device)
  out = C.c_double(0.0)
  code = {'i8': _lib.DFB_PEAK_I8, 'f64': _lib.DFB_PEAK_DMMA_F64}[what]
  _lib.check(_lib.load().dfb_measure_peak(dev.index, code, C.byref(out)), 'dfb_measure_peak')
  return out.value


_KM_CACHE = {}


def kernel_matrix(kern, X1, X2, device=None):
  """ Kernel.__call__(X1, X2) on the GPU (dfb_kernel_matrix).  Returns a host ndarray (n1, n2). """
  dev = _require_cuda(device)
  X1d = _dev_f64(np.asarray(X1, dtype=np.float64), dev)
  X2d = _dev_f64(np.asarray(X2, dtype=np.float64), dev)
  n1, d1 = int(X1d.shape[0]), int(X1d.shape[1])
  n2, d2 = int(X2d.shape[0]), int(X2d.shape[1])
  key = (dev.index,)
  post = _KM_CACHE.get(key)
  if post is None or post.n_max < n2:
    post = DevicePosterior(max(n2, 1024), device=dev, chunk=128)
    _KM_CACHE[key] = post
  desc = build_descriptor(kern, train_dim=d1, cand_dim=d1)
  K = torch.empty((n1, n2), dtype=torch.float64, device=dev)
  _lib.check(post.lib.dfb_kernel_matrix(post.h, C.byref(desc), C.c_void_p(X1d.data_ptr()), n1, d1,
                                        C.c_void_p(X2d.data_ptr()), n2, d2,
                                        C.c_void_p(K.data_ptr())), 'dfb_kernel_matrix')
  return K.cpu().numpy()


def make_acq_desc(kind, beta=0.0, best=0.0, ref_mean=0.0, ref_std=0.0):
  a = _lib.AcqDesc()
  a.kind = {'mean': _lib.DFB_ACQ_MEAN, 'ucb': _lib.DFB_ACQ_UCB, 'ei': _lib.DFB_ACQ_EI,
            'pi': _lib.DFB_ACQ_PI, 'ttei': _lib.DFB_ACQ_TTEI}[kind]
  a.beta, a.best, a.ref_mean, a.ref_std = float(beta), float(best), float(ref_mean), float(ref_std)
  return a
