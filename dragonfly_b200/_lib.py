"""
ctypes binding of libdfb200.so (include/dfb200.h) -- the only way the Python host reaches the GPU.

There is deliberately NO fallback: if the shared library is missing, or no H100 (sm_90) device is
visible when a handle is created, this module raises.  PyTorch is used only to own device buffers
(workspace, candidate matrices) and to expose the current CUDA stream.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('DFB200_LIB') or os.path.join(_HERE, 'libdfb200.so')      # DFB200_LIB: A/B builds (tools/)

DFB_MAX_FACTORS = 48
DFB_MAX_TERMS = 48
DFB_MAX_SLOTS = 128
DFB_MAX_MATERN_P = 3
DFB_BASE_SE, DFB_BASE_MATERN, DFB_BASE_POLY, DFB_BASE_EXPDECAY, DFB_BASE_HAMMING = 0, 1, 2, 3, 4
DFB_CAND_REAL, DFB_CAND_INTEGER, DFB_CAND_CATEGORICAL = 0, 1, 2
DFB_DEVICE, DFB_HOST = 0, 1
DFB_ACQ_MEAN, DFB_ACQ_UCB, DFB_ACQ_EI, DFB_ACQ_PI, DFB_ACQ_TTEI, DFB_ACQ_TS_MARGINAL = 0, 1, 2, 3, 4, 5
DFB_BUILD_FULL, DFB_BUILD_LML_ONLY, DFB_BUILD_NO_ALPHA = 0, 1, 2
DFB_EXTEND_SAVE = 16
DFB_MOO_MAX_OBJ = 8
DFB_MAX_GROUPS = 48
DFB_RNG_NORMAL, DFB_RNG_UNIFORM = 0, 1
DFB_PEAK_I8, DFB_PEAK_DMMA_F64 = 0, 1
DFB_MOO_LIN_UCB, DFB_MOO_TCH_UCB, DFB_MOO_LIN_VAL, DFB_MOO_TCH_VAL = 0, 1, 2, 3


class FactorDesc(C.Structure):
  _fields_ = [('kind', C.c_int32), ('p', C.c_int32), ('n_dims', C.c_int32), ('slot_off', C.c_int32),
              ('scale', C.c_double), ('s8', C.c_double), ('s2', C.c_double),
              ('gamma_ratio', C.c_double), ('coeffs', C.c_double * (DFB_MAX_MATERN_P + 1))]


class KernelDesc(C.Structure):
  _fields_ = [('n_terms', C.c_int32), ('n_factors', C.c_int32), ('n_slots', C.c_int32),
              ('train_dim', C.c_int32), ('cand_dim', C.c_int32), ('esp_order', C.c_int32),
              ('post_scale', C.c_double), ('kss', C.c_double),
              ('term_first_factor', C.c_int32 * (DFB_MAX_TERMS + 1)),
              ('term_pre_scale', C.c_double * DFB_MAX_TERMS),
              ('factors', FactorDesc * DFB_MAX_FACTORS),
              ('slot_train_coord', C.c_int32 * DFB_MAX_SLOTS),
              ('slot_cand_coord', C.c_int32 * DFB_MAX_SLOTS),
              ('slot_bandwidth', C.c_double * DFB_MAX_SLOTS)]


class AcqDesc(C.Structure):
  _fields_ = [('kind', C.c_int32), ('reserved', C.c_int32), ('beta', C.c_double),
              ('best', C.c_double), ('ref_mean', C.c_double), ('ref_std', C.c_double)]


class MooDesc(C.Structure):
  _fields_ = [('kind', C.c_int32), ('n_obj', C.c_int32), ('beta', C.c_double),
              ('weight', C.c_double * DFB_MOO_MAX_OBJ), ('ref', C.c_double * DFB_MOO_MAX_OBJ)]


# name -> (restype, argtypes); kept in one table so tests can check it against include/dfb200.h
_P = C.c_void_p
_D = C.c_double
_I32 = C.c_int32
_I64 = C.c_int64
DFB_GA_MAX_COLS, DFB_GA_MAX_PARTS, DFB_GA_MAX_LUT = 32, 16, 256
DFB_GA_PART_REAL, DFB_GA_PART_INTEGER, DFB_GA_PART_CATEGORICAL, DFB_GA_PART_NUMERIC = 0, 1, 2, 3


class GaDesc(C.Structure):
  _fields_ = [('d', C.c_int32), ('n_parts', C.c_int32), ('kind', C.c_int32 * DFB_GA_MAX_COLS),
              ('n_levels', C.c_int32 * DFB_GA_MAX_COLS), ('lut_off', C.c_int32 * DFB_GA_MAX_COLS),
              ('val_off', C.c_int32 * DFB_GA_MAX_COLS), ('part_kind', C.c_int32 * DFB_GA_MAX_PARTS),
              ('part_c0', C.c_int32 * DFB_GA_MAX_PARTS), ('part_c1', C.c_int32 * DFB_GA_MAX_PARTS),
              ('lo', C.c_double * DFB_GA_MAX_COLS), ('hi', C.c_double * DFB_GA_MAX_COLS),
              ('lut', C.c_double * DFB_GA_MAX_LUT)]


DFB_CONS_MAX_OPS, DFB_CONS_MAX_STACK, DFB_CONS_MAX_TAB, DFB_CONS_MAX_VEC = 128, 16, 64, 16
DFB_CONS_REJECT, DFB_CONS_ACCEPT, DFB_CONS_UNDECIDED = 0, 1, 2


class ConsProg(C.Structure):
  _fields_ = [('n_ops', C.c_int32), ('n_tab', C.c_int32), ('n_cols', C.c_int32), ('reserved', C.c_int32),
              ('op', C.c_int32 * DFB_CONS_MAX_OPS), ('arg', C.c_int32 * DFB_CONS_MAX_OPS),
              ('arg2', C.c_int32 * DFB_CONS_MAX_OPS), ('val', C.c_double * DFB_CONS_MAX_OPS),
              ('tab_key', C.c_double * DFB_CONS_MAX_TAB), ('tab_val', C.c_double * DFB_CONS_MAX_TAB)]


PROTOTYPES = {
  'dfb_version': (C.c_int, []),
  'dfb_last_error': (C.c_char_p, []),
  'dfb_create': (C.c_int, [C.POINTER(_P), C.c_int]),
  'dfb_destroy': (None, [_P]),
  'dfb_set_stream': (C.c_int, [_P, _P]),
  'dfb_workspace_bytes': (C.c_size_t, [_I64, _I32, _I64]),
  'dfb_set_workspace': (C.c_int, [_P, _P, C.c_size_t, _I64, _I64]),
  'dfb_set_kernel': (C.c_int, [_P, C.POINTER(KernelDesc)]),
  'dfb_set_test_kernel': (C.c_int, [_P, C.POINTER(KernelDesc)]),
  'dfb_set_train': (C.c_int, [_P, _P, _I64, _I32, _P]),
  'dfb_build_posterior': (C.c_int, [_P, _D, _D, _I32, C.POINTER(_D)]),
  'dfb_lml_batch': (C.c_int, [_P, C.POINTER(KernelDesc), C.POINTER(_D), C.POINTER(_D), _I32, C.POINTER(_D),
                             C.POINTER(_I32)]),
  'dfb_lml_batch_mixed': (C.c_int, [_P, C.POINTER(KernelDesc), C.POINTER(_D), C.POINTER(_D), _I32, C.POINTER(_D),
                                   C.POINTER(_I32)]),
  'dfb_extend_posterior': (C.c_int, [_P, _P, _I64, _P, _I32, C.POINTER(_D)]),
  'dfb_restore_posterior': (C.c_int, [_P]),
  'dfb_get_max_diag': (C.c_int, [_P, C.POINTER(_D)]),
  'dfb_lml_gradients': (C.c_int, [_P, C.POINTER(_D), _I32]),
  'dfb_get_state': (C.c_int, [_P, _P, _P, _P]),
  'dfb_set_alpha': (C.c_int, [_P, _P, _I64]),
  'dfb_eval': (C.c_int, [_P, _P, _I64, _I32, _I32, _D, _P, _P]),
  'dfb_mu_upper_bound': (C.c_int, [_P, _P, _I64, _I32, _I32, _D, _P]),
  'dfb_eval_covar': (C.c_int, [_P, _P, _I64, _I32, _D, _P, _P]),
  'dfb_score_argmax': (C.c_int, [_P, C.POINTER(AcqDesc), _P, _I64, _I32, _I32, _D, _P,
                                 C.POINTER(_D), C.POINTER(_I64)]),
  'dfb_score_groups': (C.c_int, [_P, C.POINTER(KernelDesc), C.POINTER(_D), _I32, _P, _I64, _I32, C.POINTER(_I32),
                                 _P]),
  'dfb_score_argmax_ts': (C.c_int, [_P, _P, _I64, _I32, _I32, _D, _P, C.c_uint64, _I64, _P, C.POINTER(_D),
                                    C.POINTER(_I64), C.POINTER(_I64)]),
  'dfb_moo_score_argmax': (C.c_int, [_P, C.POINTER(MooDesc), C.POINTER(_P), C.POINTER(_P), _I64, _P,
                                     C.POINTER(_D), C.POINTER(_I64)]),
  'dfb_moo_score_argmax_ts': (C.c_int, [_P, C.POINTER(MooDesc), C.POINTER(_P), C.POINTER(_P), _I64, _P, C.c_uint64,
                                        _I64, _P, C.POINTER(_D), C.POINTER(_I64), C.POINTER(_I64)]),
  'dfb_ga_maximise': (C.c_int, [_P, C.POINTER(AcqDesc), _D, C.POINTER(GaDesc), C.c_uint64, _I64, _I64, _P, _P, _P,
                                C.POINTER(_D), C.POINTER(_I64), C.POINTER(_D)]),
  'dfb_kernel_matrix': (C.c_int, [_P, C.POINTER(KernelDesc), _P, _I64, _I32, _P, _I64, _I32, _P]),
  'dfb_ts_workspace_bytes': (C.c_size_t, [_I64, _I64]),
  'dfb_set_ts_workspace': (C.c_int, [_P, _P, C.c_size_t, _I64]),
  'dfb_joint_workspace_bytes': (C.c_size_t, [_I64, _I64]),
  'dfb_set_joint_workspace': (C.c_int, [_P, _P, C.c_size_t, _I64]),
  'dfb_ts_draws': (C.c_int, [_P, _P, _I64, _I32, _D, _P, _I32, _D, _P, _P, C.POINTER(_D)]),
  'dfb_fill_rng': (C.c_int, [_P, C.c_uint64, _I64, _I32, _I64, _I32, _P]),
  'dfb_ts_argmax': (C.c_int, [_P, _P, _I64, _I32, _I64, _I64, _I32, _P, _P]),
  'dfb_fill_candidates': (C.c_int, [_P, C.c_uint64, _I64, _I64, _I32, C.POINTER(_D), C.POINTER(_D), _P]),
  'dfb_fill_mixed_candidates': (C.c_int, [_P, C.c_uint64, _I64, _I64, _I32, C.POINTER(_I32), C.POINTER(_D),
                                          C.POINTER(_D), C.POINTER(_I64), _P]),
  'dfb_constraint_status': (C.c_int, [_P, C.POINTER(ConsProg), _P, _I64, _I64, _P, C.POINTER(_I64)]),
  'dfb_compact_rows': (C.c_int, [_P, _P, _I64, _I32, _I64, _P, _I32, _I64, _P, _P, C.POINTER(_I64)]),
  'dfb_measure_peak': (C.c_int, [C.c_int, C.c_int, C.POINTER(_D)]),
  'dfb_launch_count': (_I64, [_P]),
  'dfb_debug_score_i8': (C.c_int, [_P, _I32, _P, _P, _I32, _I32, _P, _D, _P, _P, _I64]),
  'dfb_debug_copy': (C.c_int, [_P, C.c_char_p, _P, _I64]),
  'dfb_debug_approx_error': (C.c_int, [_P, _I32, C.POINTER(_D)]),
  'dfb_debug_chol_diag': (C.c_int, [_P, _I32, _P, _I64, _P, _P, C.POINTER(_I32)]),
  'dfb_debug_acq': (C.c_int, [_P, C.POINTER(AcqDesc), _P, _P, _I64, _I32, _P, _I64, _P, C.c_uint64, _D, _D, _D, _D,
                              _P, _P, C.POINTER(_D), C.POINTER(_I64), C.POINTER(_D), C.POINTER(_I32)]),
  'dfb_debug_selfcheck': (C.c_int, [_P, _P, _P, _P, _I32, C.POINTER(_I32)]),
  'dfb_set_option': (C.c_int, [_P, C.c_char_p, _I64]),
  'dfb_query': (C.c_int, [_P, C.c_char_p, C.POINTER(_D)]),
  'dfb_profile_enable': (C.c_int, [_P, C.c_int]),
  'dfb_profile_read': (C.c_int, [_P, C.c_int, C.POINTER(_D), C.POINTER(_I64), C.POINTER(_D)]),
}

_lib = None


class DfbError(RuntimeError):
  """ A negative status from libdfb200 (argument or CUDA error). """


def load():
  """ Loads libdfb200.so (once).  Raises ImportError if it has not been built -- no fallback. """
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise ImportError('dragonfly_b200: %s is missing. Build it with `python -c "import '
                      '__graft_entry__ as g; g.build()"` (nvcc, sm_90a). There is no CPU '
                      'fallback.' % (LIB_PATH))
  lib = C.CDLL(LIB_PATH)
  for name, (restype, argtypes) in PROTOTYPES.items():
    fn = getattr(lib, name)     # AttributeError here == header/library mismatch
    fn.restype = restype
    fn.argtypes = argtypes
  _lib = lib
  return lib


def last_error():
  return load().dfb_last_error().decode('utf-8', 'replace')


def check(status, what):
  """ status < 0 -> DfbError; status > 0 is returned to the caller (LAPACK-style info). """
  if status < 0:
    raise DfbError('%s failed (%d): %s' % (what, status, last_error()))
  return status
