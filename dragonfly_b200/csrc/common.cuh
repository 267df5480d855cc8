// Shared declarations for libdfb200.so (sm_90a: H100).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <math.h>
#include "../../include/dfb200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900 || !defined(__CUDA_ARCH_FEAT_SM90_ALL))
#error "libdfb200 is written for sm_90a (H100) only"
#endif

namespace dfb {

constexpr int TILE = 128;            // block size of every blocked algorithm (rows/cols)
constexpr int GEMM_BK = 16;          // k-extent of one pipeline stage (16 doubles = 128 B per row)

void set_error(const char* fmt, ...);

#define DFB_CUDA_OK(expr)                                                               \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      dfb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// k(x, x) is the same for every x -- and the descriptor's kss means something -- unless a factor is POLY or EXPDECAY
// (dfb200.h).  Everything that relies on a constant k(x, x) asks here: the int8 screen, the bound pass, max_diag.
static inline bool kernel_stationary(const dfb_kernel_desc& d) {
  for (int f = 0; f < d.n_factors; f++)
    if (d.factors[f].kind == DFB_BASE_POLY || d.factors[f].kind == DFB_BASE_EXPDECAY) return false;
  return true;
}

// ------------------------------------------------------------------------------------------------
// Device-side view of the posterior state and the workspace carve-up.
// ------------------------------------------------------------------------------------------------
struct ScaledSet {        // scaled training coordinates for one kernel descriptor (SoA, j contiguous)
  double* xs;             // [n_slots][npad]    x~ = x[coord] / bw
  double* nrm;            // [n_factors][npad]  |x~|^2 per factor
};

}  // namespace dfb

namespace dfb {
constexpr int PROF_CLASSES = 14;
constexpr int PROF_RING = 1024;
struct ProfClass {
  cudaEvent_t start[PROF_RING];
  cudaEvent_t stop[PROF_RING];
  double units[PROF_RING];
  int n = 0;
  bool created = false;
  double acc_ms = 0.0, acc_units = 0.0;
  int64_t acc_launches = 0;
};
// TMA maps of one operand of the int8 contraction (make_i8_maps in kernels.cu): its pair-interleaved digit planes and,
// with radix-256 digits, digit 5 alone (the first half of plane 3; the second half is the unused sixth slot)
struct I8Maps {
  CUtensorMap planes, digit5;
};
}  // namespace dfb

// The opaque handle of the C-ABI.
struct dfb_handle {
  bool prof_on = false;
  dfb::ProfClass* prof = nullptr;   // [PROF_CLASSES], allocated on first enable

  int device = 0;
  cudaStream_t stream = 0;
  int64_t launches = 0;

  // workspace
  char* ws = nullptr;
  size_t ws_bytes = 0;
  int64_t n_max = 0, npad_max = 0, chunk = 0;

  // carved pointers (see api.cu: carve())
  double* T = nullptr;        // tall factorisation matrix: (2*npad + TILE) x npad
  double* W = nullptr;        // L^-1, npad x npad, lower triangular, row-major
  double* Dinv = nullptr;     // TILE x TILE inverse of the current diagonal block
  double* X = nullptr;        // n x d training inputs (copy)
  double* yc = nullptr;       // npad centred targets (zero padded)
  double* alpha = nullptr;    // npad (zero padded)
  dfb::ScaledSet tr;          // scaled set for the GP kernel
  dfb::ScaledSet te;          // scaled set for the test kernel (Add-UCB)
  double* Ks = nullptr;       // chunk x npad  K_* rows of the current candidate chunk
  double* partial = nullptr;  // (npad/TILE) x chunk  per-row-block |v|^2 partial sums
  double* mu = nullptr;       // chunk
  double* sd = nullptr;       // chunk
  double* score = nullptr;    // chunk
  double* kssv = nullptr;     // chunk  k(x*, x*) per candidate
  double* stage = nullptr;    // chunk x DFB_MAX_SLOTS host-candidate staging
  double* blk_score = nullptr;  // per-block arg-max scratch
  int64_t* blk_index = nullptr;
  double* best_score = nullptr;  // running best (device)
  int64_t* best_index = nullptr;
  double* red = nullptr;      // small reduction scratch (4 doubles)
  int* info = nullptr;        // factorisation status
  dfb_kernel_desc* d_desc_tr = nullptr;
  dfb_kernel_desc* d_desc_te = nullptr;
  dfb_kernel_desc* d_desc_tmp = nullptr;
  dfb_kernel_desc* d_desc_grp = nullptr;   // DFB_MAX_GROUPS descriptors of dfb_score_groups

  // optional Thompson-sampling workspace (api.cu: carve_ts())
  char* ts_ws = nullptr;
  int64_t ts_mb = 0;          // padded block capacity
  double* ts_Vt = nullptr;    // mbp x npad   (L^-1 K_*^T)^T
  double* ts_cxs = nullptr;   // slots x mbp  scaled candidate coordinates (SoA)
  double* ts_cnrm = nullptr;  // factors x mbp
  double* ts_Cov = nullptr;   // mbp x mbp    posterior covariance
  double* ts_T = nullptr;     // (2 mbp + 128) x mbp factorisation buffer
  double* ts_Ut = nullptr;    // 256 x mbp
  double* ts_Sm = nullptr;    // 256 x mbp
  double* ts_mu = nullptr;    // mbp
  double* ts_red = nullptr;   // 4
  int* ts_info = nullptr;

  // optional joint Thompson-sampling workspace (api.cu: carve_joint()): one covariance over all candidates, factorised
  // in place
  char* js_ws = nullptr;
  int64_t js_mb = 0;          // padded candidate capacity Mpad
  double* js_Vt = nullptr;    // Mpad x npad  (L^-1 K_*^T)^T
  double* js_cxs = nullptr;   // slots x Mpad
  double* js_cnrm = nullptr;  // factors x Mpad
  double* js_Cov = nullptr;   // Mpad x Mpad  posterior covariance, then its Cholesky factor (lower tiles)
  double* js_Ut = nullptr;    // 256 x Mpad
  double* js_Sm = nullptr;    // 256 x Mpad
  double* js_mu = nullptr;    // Mpad
  double* js_red = nullptr;   // 4
  int* js_info = nullptr;

  // TMA path of the scoring contraction (gemm_tma.cuh)
  int gemm_impl = 1;          // 0 = v1 cp.async ring, 1 = v2 TMA + mbarrier ring (default)
  int tma_cb_group = 1 << 20;       // candidate tiles per scheduling group (a sweep found no gain)
  int i8_c2_group = 0;        // int8 kernel: candidate tiles per group of its tile order; 0 = 8 (kernels.cu)
  int last_c2_group = 0;
  int kstar_fast = 1;         // specialised K_* kernel for plain SE / Matern on <= 8 dims
  bool tma_ready = false;
  CUtensorMap tmW;            // W  (npad x npad)
  CUtensorMap tmK;            // Ks (chunk x npad)

  // integer-slice wgmma path (gemm_i8.cuh)
  int score_impl = 2;         // 0 = fp64 DMMA, 1 = int8-slice wgmma everywhere, 2 = auto: int8 pass +
                              // exact fp64 re-score of the shortlist in dfb_score_argmax, fp64 in dfb_eval
  double i8_rowscale_max = 0.0;   // max_i 2^E_i of the current posterior
  int64_t* list_idx = nullptr;    // shortlist (cap entries)
  double* list_X = nullptr;       // cap x DFB_MAX_SLOTS
  int* list_count = nullptr;      // [0] entries wanted (> cap = overflow), [1] self-check violations, [2] max ratio x 1e6
  double* list_s8 = nullptr;      // int8-pass score of each shortlist entry
  double* list_err = nullptr;     // its error allowance E_i (< 0: none -- suspect / NaN)
  double* list_z = nullptr;       // DFB_ACQ_TS_MARGINAL: its normal z_i
  double* ts_z = nullptr;         // DFB_ACQ_TS_MARGINAL: one chunk of normals (host normals staged, or the generated ones)
  int* ts_nonpos = nullptr;       // DFB_ACQ_TS_MARGINAL: candidates of the fp64 pass whose sigma^2 is not > 0
  double* blk_lb = nullptr;       // per-block max of (score - E): certain lower bounds of the fp64 maximum
  double* best_lb = nullptr;      // running maximum of those
  // survivor list of the bound pass of dfb_score_argmax (api.cu)
  int prune = 1;                  // option "prune": 0 = contract every candidate
  int64_t surv_cap = 0;           // 4 chunks
  int64_t* surv_idx = nullptr;    // surv_cap global indices
  double* surv_X = nullptr;       // surv_cap x PRUNE_MAX_DC candidate rows
  int* surv_count = nullptr;      // [0] survivors wanted (> surv_cap = overflow)
  uint32_t* keep_words = nullptr; // keep_cap / 32 ballot words of one screen launch
  int64_t keep_cap = 0;           // rows one screen launch may cover
  int64_t last_survivors = 0, last_pruned = 0;
  int64_t last_selfcheck_violations = 0;
  double last_selfcheck_ratio = 0.0;   // max |s_int8 - s_fp64| / E_i over the last shortlist
  int64_t last_shortlist = 0;     // diagnostics: size of the last shortlist, -1 = overflow -> exact pass
  int last_used_i8 = 0;
  bool i8_ready = false;
  int i8_unguarded = 0;       // diagnostics: use the int8 path even when its a-priori bound exceeds the limit (the error sweep)
  int i8_fuse = 1;            // K_* kernel emits the digit planes itself (no fp64 K_* round trip)
  int kstar_seg = 1;          // second-generation digit kernel (kstar_seg_kernel) where it applies
  int kstar_rows64 = 1;       // ... and its fp64-row form for the materialising K_* build of the fp64 scoring paths
  int8_t* Wi8 = nullptr;      // 3 pair-interleaved planes [npad][2 npad]
  int8_t* Ki8 = nullptr;      // the same for the K_* chunk
  double* cprep = nullptr;    // chunk x 10 scaled candidate rows (cand_prep_kernel)
  double* mu_part = nullptr;  // (npad / 64 + 2) x chunk
  cudaStream_t cp_stream = nullptr;   // H2D copies of page-locked host candidates, one batch ahead (api.cu: CandidateStage)
  cudaEvent_t cp_fork = nullptr, cp_done[2] = {nullptr, nullptr}, cp_free[2] = {nullptr, nullptr};
  double* rowscale = nullptr; // npad  2^E_i
  double* rowinv = nullptr;   // npad  2^-E_i
  dfb::I8Maps tmWi8, tmKi8;
  int i8_radix_opt = -1;      // digit scheme: -1 auto (radix 256 when its bound allows), 0 = 128, 1 = 256
  int i8_radix256 = 0;        // scheme in use for the current posterior (set by prepare_i8)

  // model state
  dfb_kernel_desc desc_tr;
  dfb_kernel_desc desc_te;
  dfb_kernel_desc desc_tmp;
  bool tr_prepped = false, te_prepped = false;
  bool have_kernel = false, have_test_kernel = false, have_train = false, have_post = false;
  bool have_w = false;
  int64_t n = 0, npad = 0;
  int32_t d = 0;
  double noise_plus_jitter = 0.0;
  // look-ahead factorisation (api.cu: factorise_tall): critical path on a high-priority stream, bulk trailing
  // updates on a second one; created on first use, destroyed with the handle
  cudaStream_t fs_hi = nullptr, fs_lo = nullptr;
  cudaEvent_t fe_fork = nullptr, fe_panel = nullptr, fe_rest = nullptr, fe_join_hi = nullptr, fe_join_lo = nullptr;
  int lookahead = 1;          // option "lookahead": 0 = the single-stream schedule
  int small_eval = 1;         // option "small_eval": dfb_eval of <= 16 points streams W's rows (small_sumsq_kernel)
  // dfb_extend_posterior / dfb_restore_posterior
  double* ext_save = nullptr;   // (2*TILE + 1) * npad + TILE doubles
  bool ext_saved = false;
  int64_t ext_saved_n = 0;
  double ext_saved_max_diag = 0.0;
  double max_diag = 0.0;      // max(diag K) + noise_var of the current posterior (dfb_get_max_diag)
  double noise_var = 0.0;     // of the last dfb_build_posterior
};
