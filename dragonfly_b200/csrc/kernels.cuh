// Host-side launchers of the CUDA kernels in kernels.cu (one stream: h->stream).
#pragma once
#include "common.cuh"
#include "gemm.cuh"

namespace dfb {

int launch_prep_scaled(dfb_handle* h, const dfb_kernel_desc* d_desc, int use_train_coords,
                       const double* X, int64_t n, int d, double* xs, double* nrm, int64_t npad);
// ---- K_* stage: kernel rows k(x*, X), mu and k(x*, x*) of a block of candidates ----
// Everything one K_* launch reads and writes.  Which of the fields a producer uses is up to the producer.
struct KstarArgs {
  const dfb_kernel_desc* desc;        // host copy: picks the producer and its template arguments
  const dfb_kernel_desc* d_desc;      // the same descriptor on the device
  int cand_uses_train_coords;         // 1: the candidates are training points (K(X, X) builds)
  const double* xsT; const double* nrmT; int64_t npad_tr;    // scaled training set (launch_prep_scaled)
  const double* alpha;                // NULL: no mu
  const double* Xc; int64_t m; int dc; int64_t m_rows;       // candidates; rows m .. m_rows-1 are written as padding
  int64_t n_valid, n_write;           // training points that count / columns written
  double* Ks; int64_t ldk;            // fp64 rows
  double mean_const; double* mu; double* kss_out;            // mu and k(x*, x*); either may be NULL
  void* planes; int64_t plane_bytes, row_bytes; double inv_colscale;    // int8 digit planes
  const int* abort_count;             // digit and mu-only producers: no-op once *abort_count > SHORTLIST_CAP; may be NULL
  double* cprep; double* mu_part;     // segment-kernel scratch (h->cprep, h->mu_part)
};
enum class KstarWant {
  ROWS,           // fp64 rows (+ mu, k(x*, x*) when asked)
  DIGITS,         // int8 digit planes + mu + k(x*, x*)
  MU,             // mu alone, as ROWS computes it (mean-only dfb_eval)
};
// "plain" of the route table: one term, one SE or Matern (p <= 2) factor on slots 0 .. d-1, d <= 8, no ESP -- the
// kernels specialised on (kind, p, d)
bool kstar_plain(const dfb_kernel_desc& desc);
enum class KstarProducer { SEG_DIGITS, SEG_ROWS64, SEG_MU, FAST_DIGITS, FAST_ROWS, ESP_DIGITS, ESP_ROWS, INTERP_ROWS };
struct KstarRoute {
  KstarProducer producer;
  bool slice_i8;                      // DIGITS served by an fp64 row producer: launch_slice_i8 of a.Ks must follow
};
// The producer of a K_* launch (table in kernels.cu); host logic only
KstarRoute route_kstar(const dfb_handle* h, const KstarArgs& a, KstarWant want);
int launch_kstar(dfb_handle* h, const KstarArgs& a, KstarRoute route);
int launch_init_tall(dfb_handle* h, double* T, int64_t n, int64_t npad, double diag_add,
                     const double* yc, int with_bottom);
int launch_chol_diag(dfb_handle* h, double* T, int64_t ld, int step, double* Dinv, int* info);
int launch_transpose(dfb_handle* h, const double* src, double* dst, int64_t n);
int launch_alpha(dfb_handle* h, const double* Wt, const double* v, double* alpha, int64_t n,
                 int64_t npad);
int launch_lml_reduce(dfb_handle* h, const double* T, const double* yc, const double* alpha,
                      const double* v, int64_t n, int64_t npad, double* out);
int launch_extract_lower(dfb_handle* h, const double* T, int64_t npad, double* L, int64_t n);
int launch_copy_pad(dfb_handle* h, const double* src, int64_t n_src, double* dst, int64_t n_dst);
int launch_copy_rows(dfb_handle* h, const double* src, int64_t ld_src, double* dst, int64_t ld_dst,
                     int64_t rows, int64_t cols);
// Error model of the int8-slice scoring pass handed to the acquisition / shortlist kernels (kernels.cu:
// i8_score_err): |sigma^2_int8 - sigma^2_fp64| <= b2; sens = |beta| (UCB), 0.4 (EI, TTEI), 0.25 (PI).
struct I8ErrModel {
  double b2;       // a-priori bound on |d sigma^2|; 0 = no int8 pass (no lower-bound tracking)
  double sens;
  int kind;        // DFB_ACQ_*
};
constexpr int SHORTLIST_CAP = 4096;
int launch_acq(dfb_handle* h, const dfb_acq_desc& acq, const double* mu, const double* partial,
               int64_t ld_partial, int nrb, const double* kss, int64_t m, int64_t idx_base,
               int want_std, double* sd_out, double* score_out, bool do_argmax,
               const int64_t* idx_map = nullptr, const I8ErrModel* em = nullptr);
int launch_collect_shortlist(dfb_handle* h, const double* score, const double* sd, int64_t mc,
                             int64_t idx_base, const int64_t* idx_map, const I8ErrModel& em, double pad, const double* Xc,
                             int dc);
// bound pass of dfb_score_argmax (plain kernels): keeps the m candidates Xc (device) whose acquisition at
// (mu_bar, sqrt(k**)) reaches *best_lb - pad, mu_bar a certified upper bound of mu, and appends them (x rows, global
// index idx_base + row) to the survivor list in row order; m <= h->keep_cap.  mu_ub non-NULL: writes mu_bar instead
// (no screen).  No-op once *abort_count > SHORTLIST_CAP (abort_count may be NULL).
int launch_prune(dfb_handle* h, const dfb_acq_desc& acq, const dfb_kernel_desc& desc, const dfb_kernel_desc* d_desc,
                 const double* xsT, const double* Xc, int64_t m, int dc, double mean_const, double pad, int64_t idx_base,
                 const int* abort_count, double* mu_ub);
// largest relative error of ex2.approx.ftz.f32 (which = 0) or rsqrt.approx.ftz.f32 (1) over the inputs the bound pass
// gives them, as the bit pattern of a double in *out_bits (device)
int launch_approx_err(dfb_handle* h, int which, unsigned long long* out_bits);
int launch_selfcheck(dfb_handle* h, const double* s64, int count);
int launch_vec_max(dfb_handle* h, const double* v, int64_t n, double* out);
int launch_reset_best(dfb_handle* h);
int launch_fill_rng(dfb_handle* h, uint64_t seed, int64_t col0, int S, int64_t m, int what, double* out);
int launch_fill_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int d, const double* lo,
                           const double* hi, double* out);
int launch_fill_mixed_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int d, const int32_t* kinds,
                                 const double* lo, const double* hi, const int64_t* n_levels, double* out);
int launch_ts_argmax(dfb_handle* h, const double* samples, int64_t ld, int S, int64_t m, int64_t idx_base, int reset,
                     double* best, int64_t* index);
int launch_small_sumsq(dfb_handle* h, const double* W, int64_t ldw, const double* Ks, int64_t ldk, int64_t n_rows,
                       int m, double* part, int64_t ld_part, int* n_warps_out);
int launch_moo(dfb_handle* h, const dfb_moo_desc& d, const double* const* a, const double* const* b, int64_t m,
               double* scores);
int launch_add_row_vector(dfb_handle* h, double* M, int64_t ld, int64_t rows, int64_t cols,
                          const double* v);
int launch_diag_max(dfb_handle* h, const double* M, int64_t ld, int64_t n, double* out);
int launch_fill(dfb_handle* h, double* p, int64_t n, double v);
int launch_set_diag(dfb_handle* h, double* M, int64_t ld, int64_t from, int64_t to, double v, int add);
// LML gradients: reduction of (alpha alpha^T - K^-1) o dK/dparam over lower tiles of row blocks [rb0, rb0 + n_rb)
int launch_lml_grad_tiles(dfb_handle* h, const dfb_kernel_desc* d_desc, const double* xs, const double* nrm, int64_t npad,
                          const double* alpha, const double* Kinv, int64_t ldk, int rb0, int n_rb, int nb, int64_t n,
                          int pstride, double* partial);
int launch_lml_grad_reduce(dfb_handle* h, const double* partial, int64_t n_tiles, int pstride, int n_out,
                           const double* alpha, int64_t n, double* out);

// dfb_lml_batch: B LML-only builds on the handle's training set, one CTA per item (kernels.cu, lml_batch_kernel)
constexpr int LML_BATCH_MAX_NPAD = 4 * TILE;
struct LmlBatchArgs {
  const dfb_kernel_desc* descs; const double* noise; const double* mean;    // B of each (device)
  const double* X; const double* y; int64_t n; int d; int64_t npad;         // training set; y = Y (uncentred), padded
  int ns_max, nf_max;                 // largest n_slots / n_factors in the batch: the staged coordinates per item
  double* scratch; int64_t item_doubles;
  double* red;                        // [B][2]: sum log L_ii, |L^-1 y_c|^2
  int* info;                          // [B]: 0, or 1 + the index of the first non-positive pivot
};
int64_t lml_batch_item_doubles(int64_t npad, int ns, int nf);
// hamming: launch the instantiation that evaluates HAMMING factors (dfb_lml_batch_mixed); without, the Euclidean one
int launch_lml_batch(dfb_handle* h, const LmlBatchArgs& g, int B, bool hamming);

}  // namespace dfb
