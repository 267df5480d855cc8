// C-ABI of libdfb200.so (include/dfb200.h): handle, workspace carve-up and the call sequences.
// No CPU fallback anywhere: every entry point drives CUDA kernels on the handle's stream.
#include <stdarg.h>
#include <new>
#include <stdlib.h>
#include <float.h>
#include <algorithm>
#include <vector>
#include "kernels.cuh"
#include "gemm_tma.h"

namespace dfb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int64_t default_chunk(int64_t npad) {
  int64_t c = ((int64_t)32 << 20) / npad;   // ~256 MB of K_* rows per chunk
  c = c / TILE * TILE;
  if (c < TILE) c = TILE;
  if (c > 65536) c = 65536;
  return c;
}

constexpr int PRUNE_MAX_DC = 8;       // candidate columns the survivor list of the bound pass holds

struct Carver {
  char* base;
  size_t off;
  explicit Carver(char* b) : base(b), off(0) {}
  template <typename T>
  T* take(size_t count) {
    off = (off + 255) / 256 * 256;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

// One definition of the layout, used both to size the workspace and to carve it.
static size_t carve(dfb_handle* h, char* base, int64_t n_max, int64_t chunk) {
  const int64_t npad = round_up(n_max < 1 ? 1 : n_max, TILE);
  if (chunk <= 0) chunk = default_chunk(npad);
  chunk = round_up(chunk, TILE);
  const int64_t nb = npad / TILE;
  Carver c(base);
  double* T = c.take<double>((size_t)(2 * npad + TILE) * npad);
  double* W = c.take<double>((size_t)npad * npad);
  double* Dinv = c.take<double>((size_t)TILE * TILE);
  double* X = c.take<double>((size_t)npad * DFB_MAX_SLOTS);
  double* yc = c.take<double>((size_t)npad);
  double* alpha = c.take<double>((size_t)npad);
  double* tr_xs = c.take<double>((size_t)npad * DFB_MAX_SLOTS);
  double* tr_nrm = c.take<double>((size_t)npad * DFB_MAX_FACTORS);
  double* te_xs = c.take<double>((size_t)npad * DFB_MAX_SLOTS);
  double* te_nrm = c.take<double>((size_t)npad * DFB_MAX_FACTORS);
  double* Ks = c.take<double>((size_t)chunk * npad);
  // three pair-interleaved digit planes (2 bytes per entry each)
  int8_t* Wi8 = c.take<int8_t>((size_t)6 * npad * npad);
  int8_t* Ki8 = c.take<int8_t>((size_t)6 * chunk * npad);
  double* cprep = c.take<double>((size_t)chunk * 10);
  double* mu_part = c.take<double>((size_t)(npad / 64 + 2) * chunk);      // per 64-point block partial sums of mu
  double* rowscale = c.take<double>((size_t)npad);
  double* rowinv = c.take<double>((size_t)npad);
  int64_t* list_idx = c.take<int64_t>((size_t)SHORTLIST_CAP);
  double* list_X = c.take<double>((size_t)SHORTLIST_CAP * DFB_MAX_SLOTS);
  int* list_count = c.take<int>(4);
  double* list_s8 = c.take<double>((size_t)SHORTLIST_CAP);
  double* list_err = c.take<double>((size_t)SHORTLIST_CAP);
  double* blk_lb = c.take<double>((size_t)chunk / 128 + 16);
  double* best_lb = c.take<double>(1);
  double* partial = c.take<double>((size_t)nb * chunk);
  double* mu = c.take<double>((size_t)chunk);
  double* sd = c.take<double>((size_t)chunk);
  double* score = c.take<double>((size_t)chunk);
  double* kssv = c.take<double>((size_t)chunk);
  double* stage = c.take<double>((size_t)chunk * DFB_MAX_SLOTS);
  double* blk_score = c.take<double>((size_t)chunk / 128 + 16);
  int64_t* blk_index = c.take<int64_t>((size_t)chunk / 128 + 16);
  const int64_t surv_cap = 4 * chunk;
  int64_t* surv_idx = c.take<int64_t>((size_t)surv_cap);
  double* surv_X = c.take<double>((size_t)surv_cap * PRUNE_MAX_DC);
  int* surv_count = c.take<int>(4);
  // one screen launch covers a host staging batch (up to chunk x DFB_MAX_SLOTS rows) or ~10^6 device rows
  const int64_t keep_cap = round_up(chunk * DFB_MAX_SLOTS > ((int64_t)1 << 20) ? chunk * DFB_MAX_SLOTS : (int64_t)1 << 20, 32);
  uint32_t* keep_words = c.take<uint32_t>((size_t)keep_cap / 32);
  double* best_score = c.take<double>(1);
  int64_t* best_index = c.take<int64_t>(1);
  double* red = c.take<double>(8);
  int* info = c.take<int>(4);
  dfb_kernel_desc* d0 = c.take<dfb_kernel_desc>(1);
  dfb_kernel_desc* d1 = c.take<dfb_kernel_desc>(1);
  dfb_kernel_desc* d2 = c.take<dfb_kernel_desc>(1);
  dfb_kernel_desc* d_grp = c.take<dfb_kernel_desc>(DFB_MAX_GROUPS);
  // dfb_extend_posterior's snapshot of what it overwrites: the last row block of L, the last block
  // column of L^-T, that block of the y row, alpha
  double* ext_save = c.take<double>((size_t)(2 * TILE + 1) * npad + TILE);
  // dfb_score_argmax_ts: the normals of the shortlist and of one chunk, and the count of non-positive variances
  double* list_z = c.take<double>((size_t)SHORTLIST_CAP);
  double* ts_z = c.take<double>((size_t)chunk);
  int* ts_nonpos = c.take<int>(4);
  if (h != nullptr && base != nullptr) {
    h->ext_save = ext_save;
    h->list_z = list_z; h->ts_z = ts_z; h->ts_nonpos = ts_nonpos;
    h->cprep = cprep; h->mu_part = mu_part;
    h->T = T; h->W = W; h->Dinv = Dinv; h->X = X; h->yc = yc; h->alpha = alpha;
    h->tr.xs = tr_xs; h->tr.nrm = tr_nrm; h->te.xs = te_xs; h->te.nrm = te_nrm;
    h->Ks = Ks; h->Wi8 = Wi8; h->Ki8 = Ki8; h->rowscale = rowscale; h->rowinv = rowinv; h->list_idx = list_idx; h->list_X = list_X; h->list_count = list_count; h->list_s8 = list_s8; h->list_err = list_err; h->blk_lb = blk_lb; h->best_lb = best_lb; h->partial = partial; h->mu = mu; h->sd = sd; h->score = score; h->kssv = kssv; h->stage = stage;
    h->blk_score = blk_score; h->blk_index = blk_index; h->best_score = best_score;
    h->surv_cap = surv_cap; h->surv_idx = surv_idx; h->surv_X = surv_X; h->surv_count = surv_count;
    h->keep_words = keep_words; h->keep_cap = keep_cap;
    h->best_index = best_index; h->red = red; h->info = info;
    h->d_desc_tr = d0; h->d_desc_te = d1; h->d_desc_tmp = d2; h->d_desc_grp = d_grp;
    h->n_max = n_max; h->npad_max = npad; h->chunk = chunk;
  }
  return c.off + 256;
}

static size_t carve_ts(dfb_handle* h, char* base, int64_t n_max, int64_t mb) {
  const int64_t npad = round_up(n_max < 1 ? 1 : n_max, TILE);
  const int64_t mbp = round_up(mb < 1 ? 1 : mb, TILE);
  Carver c(base);
  double* Vt = c.take<double>((size_t)mbp * npad);
  double* cxs = c.take<double>((size_t)mbp * DFB_MAX_SLOTS);
  double* cnrm = c.take<double>((size_t)mbp * DFB_MAX_FACTORS);
  double* Cov = c.take<double>((size_t)mbp * mbp);
  double* T2 = c.take<double>((size_t)(2 * mbp + TILE) * mbp);
  double* Ut = c.take<double>((size_t)256 * mbp);
  double* Sm = c.take<double>((size_t)256 * mbp);
  double* mu = c.take<double>((size_t)mbp);
  double* red = c.take<double>(8);
  int* info = c.take<int>(4);
  if (h != nullptr && base != nullptr) {
    h->ts_Vt = Vt; h->ts_cxs = cxs; h->ts_cnrm = cnrm; h->ts_Cov = Cov; h->ts_T = T2; h->ts_Ut = Ut;
    h->ts_Sm = Sm; h->ts_mu = mu; h->ts_red = red; h->ts_info = info; h->ts_mb = mbp;
  }
  return c.off + 256;
}

// The joint form over up to m candidates: the covariance is factorised in place, so there is one Mpad x Mpad matrix
// and no tall buffer.
static size_t carve_joint(dfb_handle* h, char* base, int64_t n_max, int64_t m) {
  const int64_t npad = round_up(n_max < 1 ? 1 : n_max, TILE);
  const int64_t mp = round_up(m < 1 ? 1 : m, TILE);
  Carver c(base);
  double* Vt = c.take<double>((size_t)mp * npad);
  double* cxs = c.take<double>((size_t)mp * DFB_MAX_SLOTS);
  double* cnrm = c.take<double>((size_t)mp * DFB_MAX_FACTORS);
  double* Cov = c.take<double>((size_t)mp * mp);
  double* Ut = c.take<double>((size_t)256 * mp);
  double* Sm = c.take<double>((size_t)256 * mp);
  double* mu = c.take<double>((size_t)mp);
  double* red = c.take<double>(8);
  int* info = c.take<int>(4);
  if (h != nullptr && base != nullptr) {
    h->js_Vt = Vt; h->js_cxs = cxs; h->js_cnrm = cnrm; h->js_Cov = Cov; h->js_Ut = Ut; h->js_Sm = Sm; h->js_mu = mu;
    h->js_red = red; h->js_info = info; h->js_mb = mp;
  }
  return c.off + 256;
}

static int check_desc(const dfb_kernel_desc* d) {
  if (d == nullptr) { set_error("kernel descriptor is NULL"); return -1; }
  if (d->n_terms < 1 || d->n_terms > DFB_MAX_TERMS || d->n_factors < 1 ||
      d->n_factors > DFB_MAX_FACTORS || d->n_slots < 1 || d->n_slots > DFB_MAX_SLOTS) {
    set_error("kernel descriptor out of range (terms %d, factors %d, slots %d)", d->n_terms,
              d->n_factors, d->n_slots);
    return -1;
  }
  if (d->term_first_factor[0] != 0 || d->term_first_factor[d->n_terms] != d->n_factors) {
    set_error("kernel descriptor: term_first_factor does not cover the factors");
    return -1;
  }
  for (int f = 0; f < d->n_factors; f++) {
    const dfb_factor_desc& fd = d->factors[f];
    if (fd.kind < DFB_BASE_SE || fd.kind > DFB_BASE_HAMMING || fd.n_dims < 1 ||
        fd.slot_off < 0 || fd.slot_off + fd.n_dims > d->n_slots || fd.p < 0 ||
        (fd.kind == DFB_BASE_MATERN && fd.p > DFB_MAX_MATERN_P) ||
        ((fd.kind == DFB_BASE_EXPDECAY || fd.kind == DFB_BASE_HAMMING) && fd.p != 0) ||
        (fd.kind >= DFB_BASE_POLY && !(fd.scale > 0.0 && isfinite(fd.scale))) ||
        (fd.kind == DFB_BASE_EXPDECAY && !isfinite(fd.s2))) {
      set_error("kernel descriptor: bad factor %d", f);
      return -1;
    }
    // slot_bandwidth means a bandwidth, a scaling, a power or a weight depending on the kind (dfb200.h): a slot of a
    // POLY, EXPDECAY or HAMMING factor belongs to that factor alone
    if (fd.kind >= DFB_BASE_POLY) {
      for (int g = 0; g < d->n_factors; g++) {
        const dfb_factor_desc& gd = d->factors[g];
        if (g != f && gd.slot_off < fd.slot_off + fd.n_dims && fd.slot_off < gd.slot_off + gd.n_dims) {
          set_error("kernel descriptor: factor %d shares slots with POLY / EXPDECAY / HAMMING factor %d", g, f);
          return -1;
        }
      }
      for (int q = 0; q < fd.n_dims; q++) {
        const double w = d->slot_bandwidth[fd.slot_off + q];
        if (!isfinite(w) || (fd.kind == DFB_BASE_HAMMING && !(w >= 0.0))) {
          set_error("kernel descriptor: factor %d has a %s %s", f, fd.kind == DFB_BASE_HAMMING ? "negative or non-finite" :
                    "non-finite", fd.kind == DFB_BASE_POLY ? "scaling" : fd.kind == DFB_BASE_HAMMING ? "weight" : "power");
          return -1;
        }
      }
    }
  }
  for (int s = 0; s < d->n_slots; s++) {
    bool bandwidth = true;              // every slot but those of POLY / EXPDECAY factors holds a bandwidth
    for (int f = 0; f < d->n_factors; f++) {
      const dfb_factor_desc& fd = d->factors[f];
      if (fd.kind >= DFB_BASE_POLY && s >= fd.slot_off && s < fd.slot_off + fd.n_dims) bandwidth = false;
    }
    if (d->slot_train_coord[s] < 0 || d->slot_train_coord[s] >= d->train_dim ||
        d->slot_cand_coord[s] < 0 || d->slot_cand_coord[s] >= d->cand_dim ||
        (bandwidth && !(d->slot_bandwidth[s] > 0.0))) {
      set_error("kernel descriptor: bad slot %d", s);
      return -1;
    }
  }
  if (d->esp_order < 0 || d->esp_order > d->n_terms) {
    set_error("kernel descriptor: ESP order %d outside 0 .. n_terms = %d", d->esp_order, d->n_terms);
    return -1;
  }
  if (d->esp_order > 0) {
    for (int t = 0; t < d->n_terms; t++) {
      const int f = d->term_first_factor[t];
      if (d->term_first_factor[t + 1] != f + 1 || d->factors[f].n_dims != 1 || d->term_pre_scale[t] != 1.0) {
        set_error("kernel descriptor: ESP term %d is not one 1-slot factor with pre_scale 1", t);
        return -1;
      }
      if (d->factors[f].kind >= DFB_BASE_POLY) {
        set_error("kernel descriptor: ESP term %d is a POLY / EXPDECAY / HAMMING factor (ESP children are SE or Matern)",
                  t);
        return -1;
      }
    }
  }
  return 0;
}

#define DFB_TRY(expr)        \
  do {                       \
    int _r = (expr);         \
    if (_r != 0) return _r;  \
  } while (0)

static int need(dfb_handle* h, bool ws, bool kern, bool train, bool post, bool w) {
  if (h == nullptr) { set_error("handle is NULL"); return -1; }
  if (ws && h->ws == nullptr) { set_error("no workspace: call dfb_set_workspace first"); return -1; }
  if (kern && !h->have_kernel) { set_error("no kernel: call dfb_set_kernel first"); return -1; }
  if (train && !h->have_train) { set_error("no training data: call dfb_set_train first"); return -1; }
  if (post && !h->have_post) { set_error("no posterior: call dfb_build_posterior first"); return -1; }
  if (w && !h->have_w) { set_error("posterior was built LML-only: W = L^-1 is not available"); return -1; }
  return 0;
}

static int ensure_train_scaled(dfb_handle* h) {
  if (!h->tr_prepped) {
    DFB_TRY(launch_prep_scaled(h, h->d_desc_tr, 1, h->X, h->n, h->d, h->tr.xs, h->tr.nrm, h->npad));
    h->tr_prepped = true;
  }
  return 0;
}

static int ensure_test_scaled(dfb_handle* h) {
  if (h->have_test_kernel && !h->te_prepped) {
    DFB_TRY(launch_prep_scaled(h, h->d_desc_te, 1, h->X, h->n, h->d, h->te.xs, h->te.nrm, h->npad));
    h->te_prepped = true;
  }
  return 0;
}

// The kernel candidates are scored with: the test kernel (Add-UCB) when one is set, else the training kernel.
struct ActiveKernel { const dfb_kernel_desc& desc; const dfb_kernel_desc* d_desc; const ScaledSet& ss; };
static ActiveKernel active_kernel(const dfb_handle* h) {
  if (h->have_test_kernel) return {h->desc_te, h->d_desc_te, h->te};
  return {h->desc_tr, h->d_desc_tr, h->tr};
}

// K(X[row0 : row0 + m_rows], X) of the training kernel into Ks (n_write columns), rows beyond n as padding: the
// posterior build (GP._get_training_kernel_matrix, gp_core.py:149-153), its replay and dfb_get_state.
static int launch_train_kstar(dfb_handle* h, int64_t row0, int64_t m_rows, double* Ks, int64_t ldk, int64_t n_write) {
  KstarArgs ka{};
  ka.desc = &h->desc_tr; ka.d_desc = h->d_desc_tr; ka.cand_uses_train_coords = 1;
  ka.xsT = h->tr.xs; ka.nrmT = h->tr.nrm; ka.npad_tr = h->npad; ka.Xc = h->X + row0 * h->d; ka.m = h->n - row0;
  ka.dc = h->d; ka.m_rows = m_rows; ka.n_valid = h->n; ka.n_write = n_write; ka.Ks = Ks; ka.ldk = ldk;
  return launch_kstar(h, ka, route_kstar(h, ka, KstarWant::ROWS));
}

// ---- optional per-class event timing -------------------------------------------------------------
static int prof_flush(dfb_handle* h, int cls) {
  ProfClass& pc = h->prof[cls];
  if (pc.n == 0) return 0;
  DFB_CUDA_OK(cudaEventSynchronize(pc.stop[pc.n - 1]));
  for (int i = 0; i < pc.n; i++) {
    float ms = 0.f;
    DFB_CUDA_OK(cudaEventElapsedTime(&ms, pc.start[i], pc.stop[i]));
    pc.acc_ms += ms;
    pc.acc_units += pc.units[i];
    pc.acc_launches += 1;
  }
  pc.n = 0;
  return 0;
}
// cls < 0: the interval is not profiled
static int prof_begin(dfb_handle* h, int cls) {
  if (!h->prof_on || cls < 0) return 0;
  ProfClass& pc = h->prof[cls];
  if (!pc.created) {
    for (int i = 0; i < PROF_RING; i++) {
      DFB_CUDA_OK(cudaEventCreate(&pc.start[i]));
      DFB_CUDA_OK(cudaEventCreate(&pc.stop[i]));
    }
    pc.created = true;
  }
  if (pc.n == PROF_RING) DFB_TRY(prof_flush(h, cls));
  DFB_CUDA_OK(cudaEventRecord(pc.start[pc.n], h->stream));
  return 0;
}
static int prof_end(dfb_handle* h, int cls, double units) {
  if (!h->prof_on || cls < 0) return 0;
  ProfClass& pc = h->prof[cls];
  DFB_CUDA_OK(cudaEventRecord(pc.stop[pc.n], h->stream));
  pc.units[pc.n] = units;
  pc.n++;
  return 0;
}

// The blocked right-looking factorisation of the tall matrix [A ; I ; y^T] (factor_tma.cuh):
// top -> L, bottom -> L^-T, y row -> (L^-1 y)^T.
//
// Schedule: chol_diag is a one-CTA, latency-bound kernel run once per step (npad/128 steps), so in the plain
// step-after-step order the other SMs wait for it at every step.  With look-ahead the trailing update of
// step k is split: the column of the NEXT panel (block k+1) is updated first on the critical-path stream, so
// chol_diag(k+1) and the panel solve of step k+1 run while the bulk of update k (column blocks >= k+2) is still
// in flight on a second stream.
//   hi:  chol(k) panel(k) [P_k] wait(R_k-1) next(k)  chol(k+1) panel(k+1) [P_k+1] wait(R_k) next(k+1) ...
//   lo:                   wait(P_k) rest(k) [R_k]                         wait(P_k+1) rest(k+1) [R_k+1]
// next(k) and rest(k-1) both accumulate into column block k+1, hence wait(R_k-1); rest(k) after rest(k-1) by
// stream order.  panel(k) and next(k) take factor_update_kernel's small chain shape, so each spreads over ~4x as many
// SMs as it has 128 x 128 tiles; the bulk launches take its throughput shape.  The arithmetic per element does not
// depend on the shape or the stream: results are bit-identical to the single-stream schedule.
struct StreamSwap {
  dfb_handle* h;
  cudaStream_t user;
  explicit StreamSwap(dfb_handle* hh) : h(hh), user(hh->stream) {}
  ~StreamSwap() { h->stream = user; }
};

static int ensure_factor_streams(dfb_handle* h) {
  if (h->fs_hi != nullptr) return 0;
  int lo = 0, hi = 0;
  DFB_CUDA_OK(cudaDeviceGetStreamPriorityRange(&lo, &hi));      // lo = least, hi = greatest priority
  DFB_CUDA_OK(cudaStreamCreateWithPriority(&h->fs_hi, cudaStreamNonBlocking, hi));
  DFB_CUDA_OK(cudaStreamCreateWithPriority(&h->fs_lo, cudaStreamNonBlocking, lo));
  cudaEvent_t* evs[5] = {&h->fe_fork, &h->fe_panel, &h->fe_rest, &h->fe_join_hi, &h->fe_join_lo};
  for (int i = 0; i < 5; i++) DFB_CUDA_OK(cudaEventCreateWithFlags(evs[i], cudaEventDisableTiming));
  return 0;
}

// One launch of factor_update_kernel inside an interval of profiling class cls (< 0: none).
static int factor_update(dfb_handle* h, const FactorMaps& m, const FactorArgs& g, bool chain, int cls) {
  DFB_TRY(prof_begin(h, cls));
  DFB_TRY(launch_factor_update(h, m, g, chain));
  return prof_end(h, cls, 1.0);
}

// profile: time the stages in the DFB_PROF_BUILD_* classes (the posterior build; not the Thompson blocks).
// top_only: T is the npad x npad square alone, factorised in place (no L^-T rows, no y row; with_bottom is ignored).
// The top's tiles see the same launches and arithmetic in both forms, so its L is bit for bit the tall form's.
static int factorise_tall(dfb_handle* h, double* T, int64_t npad, double* Dinv, int* info,
                          bool with_bottom, bool profile, bool top_only = false) {
  const int nb = (int)(npad / TILE);
  const int c_chol = profile ? DFB_PROF_BUILD_CHOL : -1, c_chain = profile ? DFB_PROF_BUILD_CHAIN : -1;
  const int c_rest = profile ? DFB_PROF_BUILD_REST : -1;
  const bool la = h->lookahead != 0 && nb >= 4;
  FactorMaps maps;
  DFB_TRY(make_factor_maps(&maps, T, top_only ? npad : 2 * npad + TILE, npad, Dinv));
  StreamSwap guard(h);
  if (la) {
    DFB_TRY(ensure_factor_streams(h));
    DFB_CUDA_OK(cudaEventRecord(h->fe_fork, guard.user));
    DFB_CUDA_OK(cudaStreamWaitEvent(h->fs_hi, h->fe_fork, 0));
    DFB_CUDA_OK(cudaStreamWaitEvent(h->fs_lo, h->fe_fork, 0));
  }
  bool rest_pending = false;
  for (int step = 0; step < nb; step++) {
    if (la) h->stream = h->fs_hi;
    DFB_TRY(prof_begin(h, c_chol));
    DFB_TRY(launch_chol_diag(h, T, npad, step, Dinv, info));
    DFB_TRY(prof_end(h, c_chol, 1.0));
    FactorArgs g;
    memset(&g, 0, sizeof(g));
    g.T = T; g.ld = npad; g.step = step; g.nb = nb; g.skip_bottom = with_bottom ? 0 : 1; g.info = info;
    g.top_only = top_only ? 1 : 0;
    g.panel = 1;
    DFB_TRY(factor_update(h, maps, g, true, c_chain));
    if (step + 1 >= nb) continue;
    g.panel = 0;
    if (!la) {
      g.j0 = step + 1; g.j1 = nb;
      DFB_TRY(factor_update(h, maps, g, false, c_rest));
      continue;
    }
    DFB_CUDA_OK(cudaEventRecord(h->fe_panel, h->fs_hi));
    if (rest_pending) DFB_CUDA_OK(cudaStreamWaitEvent(h->fs_hi, h->fe_rest, 0));
    g.j0 = step + 1; g.j1 = step + 2;                 // the next panel's column, on the critical path
    DFB_TRY(factor_update(h, maps, g, true, c_chain));
    if (step + 2 < nb) {
      h->stream = h->fs_lo;
      DFB_CUDA_OK(cudaStreamWaitEvent(h->fs_lo, h->fe_panel, 0));
      g.j0 = step + 2; g.j1 = nb;
      DFB_TRY(factor_update(h, maps, g, false, c_rest));
      DFB_CUDA_OK(cudaEventRecord(h->fe_rest, h->fs_lo));
      rest_pending = true;
    }
  }
  if (la) {
    DFB_CUDA_OK(cudaEventRecord(h->fe_join_hi, h->fs_hi));
    DFB_CUDA_OK(cudaEventRecord(h->fe_join_lo, h->fs_lo));
    DFB_CUDA_OK(cudaStreamWaitEvent(guard.user, h->fe_join_hi, 0));
    DFB_CUDA_OK(cudaStreamWaitEvent(guard.user, h->fe_join_lo, 0));
  }
  return 0;
}

// A-priori bound on the int8-slice path's ABSOLUTE sigma^2 error for the active kernel.
//
// Error model.  One entry of v = L^-1 k_* is a sum over k <= i of digit-truncation and dropped-product terms, each
// bounded by c 2^-q rowscale_i colscale (q = 43 for six radix-128 digits, 40 for five radix-256 digits; the low
// digits of an operand are unrelated to its magnitude, so the terms do not shrink with |W_ik K_k|) and, being
// rounding residues of unrelated numbers, of effectively independent sign: |dv_i| grows like sqrt(n), exactly as
// the rounding error of the fp64 dot product it replaces (whose worst-case bound n eps is never approached either).
// d(sigma^2) = 2 sum_i v_i dv_i has standard deviation <= 2 |v| max_i sd(dv_i) <= 2 sqrt(k(x,x)) max_i sd(dv_i)
// for independent dv_i (|v|^2 <= k(x,x) - sigma^2 <= k(x,x)).  A worst-case (n instead of sqrt(n), aligned signs
// over i) bound would be ~sqrt(n) n / 8 ~ 4 10^4 times larger at N = 5000 and is as unattainable as LAPACK's own.
//
// The constant 8 keeps the bound above every maximum measured over the validation sweep (tools/sweep_i8_bound.py:
// 480 configurations -- N 1024..5000, noise 1e-2..1e-8 of the scale, scale 1e-2..1e4,
// SE / Matern-5/2 / Matern-1/2 / additive / product kernels, both digit schemes, 13056 candidates each, guard off): the
// worst measured / bound ratio is 0.28 (Matern-1/2, N = 1024, radix 256), typically 0.02-0.15; the worst ABSOLUTE error
// among the 185 configurations the guard admits is 1.05e-9 against the 1e-8 contract.  It is NOT a worst-case bound;
// three things keep the arg-max exact in spite of that:
//   (1) the limit below is ABSOLUTE: the int8 pass is used only while the bound is <= 5e-9, half of the
//       north-star's 1e-8 contract on sigma^2, whatever the kernel scale;
//   (2) dfb_score_argmax re-scores in fp64 every candidate whose int8 score, widened by the bound, could reach the
//       fp64 maximum, and returns the fp64 arg-max of those;
//   (3) after that exact pass the int8 and fp64 scores of the shortlist are compared (selfcheck_kernel): a single
//       candidate outside its allowance voids the int8 pass and the whole call is repeated in fp64
//       (query "last_selfcheck_violations" / "last_selfcheck_ratio").
// score_impl = 0 (env DFB200_SCORE=fp64, option "score_impl") switches the int8 path off altogether.
static double i8_colscale(const dfb_kernel_desc& desc) {
  int e = 0;
  frexp(desc.kss * (1.0 + 1e-9), &e);
  return ldexp(1.0, e + 1);
}
static double i8_sigma2_bound(const dfb_handle* h, const dfb_kernel_desc& desc) {
  return 8.0 * h->i8_rowscale_max * sqrt((double)h->n) * i8_colscale(desc) *
         ldexp(1.0, h->i8_radix256 ? -40 : -43) * sqrt(desc.kss);
}
static const double I8_BOUND_LIMIT = 5e-9;     // absolute: half of the 1e-8 sigma^2 contract
// The colscale and the bound rest on one k(x, x) for all candidates: non-stationary kernels are scored in fp64 only.
static bool i8_usable(const dfb_handle* h, const dfb_kernel_desc& desc) {
  if (!h->i8_ready || !kernel_stationary(desc) || !(desc.kss > 0.0)) return false;
  if (h->i8_unguarded) return true;                 // diagnostics only (tools/sweep_i8_bound.py)
  return i8_sigma2_bound(h, desc) <= I8_BOUND_LIMIT;
}

// Digit planes of W = L^-1 for the int8 wgmma path + the tensor maps of both operands.
static int prepare_i8(dfb_handle* h) {
  const int64_t npad = h->npad;
  DFB_TRY(launch_row_exponent(h, h->W, npad, npad, npad, h->rowscale, h->rowinv));
  DFB_TRY(launch_vec_max(h, h->rowscale, h->n, h->red + 4));
  DFB_CUDA_OK(cudaMemcpyAsync(&h->i8_rowscale_max, h->red + 4, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  // Digit scheme: five radix-256 digits (15 products) when the a-priori bound of
  // that coarser expansion passes for the training kernel, else six radix-128 digits (21 products).  The
  // radix-256 groups also need int32 headroom: 5 K 2^14 < 2^31.
  h->i8_radix256 = 0;
  if (h->i8_radix_opt != 0 && npad <= 24576) {
    h->i8_radix256 = 1;
    const dfb_kernel_desc& dtr = h->desc_tr;
    if (h->i8_radix_opt < 0 && dtr.kss > 0.0 && i8_sigma2_bound(h, dtr) > I8_BOUND_LIMIT)
      h->i8_radix256 = 0;
  }
  // pair-interleaved digit planes: 3 planes of rows x (2 * npad) bytes
  DFB_TRY(launch_slice_i8(h, h->W, npad, npad, npad, h->rowinv, 0.0, h->Wi8, 2 * npad * npad, 2 * npad));
  // TMA maps of one K = 32 block per box: one CTA's share of W's 128-row block, one tile of candidates
  DFB_TRY(make_i8_maps(&h->tmWi8, h->Wi8, npad, npad, true, h->i8_radix256 != 0));
  DFB_TRY(make_i8_maps(&h->tmKi8, h->Ki8, npad, h->chunk, false, h->i8_radix256 != 0));
  h->i8_ready = true;
  return 0;
}

// The scoring state of the current posterior, rebuilt on request: with i8 the int8 digit planes of W (when option
// score_impl asks for them), with tma the fp64 TMA maps of W and Ks (when option gemm_impl does).  Both need W = L^-1;
// without it they are only marked not ready.  The TMA maps describe (address, npad) only, so a posterior that changed W
// but not npad keeps them.
static int prepare_scoring(dfb_handle* h, bool i8, bool tma) {
  if (i8) h->i8_ready = false;
  if (tma) h->tma_ready = false;
  if (!h->have_post || !h->have_w) return 0;
  DFB_CUDA_OK(cudaSetDevice(h->device));
  // a non-stationary training kernel never takes the int8 path (i8_usable), so its digit planes are not made
  if (i8 && (h->score_impl == 1 || (h->score_impl == 2 && h->n >= 1024)) && kernel_stationary(h->desc_tr))
    DFB_TRY(prepare_i8(h));
  if (tma && h->gemm_impl == 1) {
    DFB_TRY(make_tensor_map_2d_f64(&h->tmW, h->W, h->npad, h->npad, h->npad));
    DFB_TRY(make_tensor_map_2d_f64(&h->tmK, h->Ks, h->chunk, h->npad, h->npad));
    h->tma_ready = true;
  }
  return 0;
}

// The LML from lml_reduce's sums: quad = |L^-1 y|^2 or y^T alpha, log_det_half = sum log L_ii
static double lml(double quad, double log_det_half, int64_t n) { return -0.5 * quad - log_det_half - 0.5 * (double)n * log(2.0 * M_PI); }

// The tail of a factorisation of [A ; I ; y^T]: W = L^-1 from L^-T (unless LML-only), alpha (DFB_BUILD_FULL), the LML
// sums, then the read-back of the sums and the pivot status.  A non-stationary training kernel reads back 7 sums: red[6]
// is the max(diag K) launch_diag_max left.  end_build (the posterior build) times the tail in
// DFB_PROF_BUILD_TAIL and closes the DFB_PROF_BUILD interval before the read-back.
static int posterior_tail(dfb_handle* h, int32_t flags, bool end_build, double red[7], int* info) {
  const int64_t n = h->n, npad = h->npad;
  const double* Wt = h->T + (size_t)npad * npad;
  const double* v = h->T + (size_t)2 * npad * npad;
  const int c_tail = end_build ? DFB_PROF_BUILD_TAIL : -1;
  DFB_TRY(prof_begin(h, c_tail));
  if (flags != DFB_BUILD_LML_ONLY) DFB_TRY(launch_transpose(h, Wt, h->W, npad));
  if (flags == DFB_BUILD_FULL) DFB_TRY(launch_alpha(h, Wt, v, h->alpha, n, npad));
  DFB_TRY(launch_lml_reduce(h, h->T, h->yc, flags == DFB_BUILD_FULL ? h->alpha : nullptr, v, n, npad, h->red));
  DFB_TRY(prof_end(h, c_tail, 1.0));
  if (end_build) DFB_TRY(prof_end(h, DFB_PROF_BUILD, 1.0));
  const size_t red_bytes = sizeof(double) * (kernel_stationary(h->desc_tr) ? 3 : 7);
  DFB_CUDA_OK(cudaMemcpyAsync(red, h->red, red_bytes, cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(info, h->info, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

// ---- incremental posterior update (SURVEY 8f rank 1) ------------------------------------------------------
// Appending q training points changes only the LAST row block of L (as long as n + q stays inside the same
// padded size): Cholesky row i depends on rows <= i alone.  Rather than re-running the N^3/3 right-looking
// factorisation, the pre-step state of the last block column of the tall matrix [A ; I ; y^T] is rebuilt by
// left-looking products against the finished factor and the last factorisation step is replayed:
//     P    = A[last, :m0] L00^-T = A[last, :m0] W00^T          top, row block nb-1, columns < m0
//     S    = A[last, last] - P P^T                             top, diagonal block
//     Wt_c = -(L00^-T) P^T                                     L^-T rows < m0, last block column
//     y_c  = y[last] - v[:m0] P^T                              y row, last block
// then chol_diag + the panel solve of step nb-1 turn (S, I, Wt_c, y_c) into (L_dd, L_dd^-T, L^-T's last
// block column, v[last]).  Cost 4 N^2 * 128 flops + one 128 x 128 Cholesky instead of 2 N^3 / 3.
static int replay_last_block(dfb_handle* h, int32_t flags, double* lml_out_host) {
  const int64_t n = h->n, npad = h->npad;
  const int nb = (int)(npad / TILE), step = nb - 1;
  const int64_t m0 = (int64_t)step * TILE;
  double* top_row = h->T + m0 * npad;                      // row block nb-1 of the top
  double* mid = h->T + npad * npad;                        // L^-T
  double* yrow = h->T + 2 * npad * npad;                   // y row block (row 0 holds the data)
  h->have_post = h->have_w = false;
  h->tr_prepped = h->te_prepped = false;
  DFB_TRY(ensure_train_scaled(h));
  DFB_CUDA_OK(cudaMemsetAsync(h->info, 0, sizeof(int) * 4, h->stream));
  // A[last, :] = K(X[last], X) + (noise + jitter) I, identity on the padding rows -> Ks scratch (128 x npad)
  DFB_TRY(launch_train_kstar(h, m0, TILE, h->Ks, npad, npad));
  // a non-stationary kernel's max(diag K) can grow with the appended points: the block's diagonal is rebuilt here
  const bool stationary = kernel_stationary(h->desc_tr);
  if (!stationary) DFB_TRY(launch_diag_max(h, h->Ks + m0, npad, n - m0, h->red + 6));
  DFB_TRY(launch_set_diag(h, h->Ks + m0, npad, 0, n - m0, h->noise_plus_jitter, 1));
  DFB_TRY(launch_set_diag(h, h->Ks + m0, npad, n - m0, TILE, 1.0, 0));
  // The four left-looking products have 1 .. nb-1 output tiles with k-depths up to m0 ~ N: each tile's k-range is
  // split over several CTAs (launch_gemm_splitk) so that they fill the GPU; scratch lives in the K_* chunk buffer
  // behind the 128 rows of A.
  const int KS = 8;
  double* scratch = h->Ks + (int64_t)TILE * npad;
  const bool split = step >= 2 && h->chunk >= (int64_t)TILE * (1 + KS);       // KS * 128 x npad doubles of scratch
  GemmArgs g;
  if (step > 0) {
    // P[a][i] = sum_{k <= i} A[a][k] W[i][k]
    memset(&g, 0, sizeof(g));
    g.A = h->Ks; g.lda = npad; g.B = h->W; g.ldb = npad; g.D = top_row; g.ldd = npad; g.alpha = 1.0;
    g.mode = MODE_GENERIC; g.n_rb = 1; g.n_cb = step; g.K = (int)m0; g.tri = 2;
    if (split) DFB_TRY(launch_gemm_splitk(h, g, 4, scratch));
    else DFB_TRY(launch_gemm(h, g, EPI_STORE, step));
    // Wt_c[j][a] = -sum_k Wt[j][k] P[a][k]
    memset(&g, 0, sizeof(g));
    g.A = mid; g.lda = npad; g.B = top_row; g.ldb = npad; g.D = mid + m0; g.ldd = npad; g.alpha = -1.0;
    g.mode = MODE_GENERIC; g.n_rb = step; g.n_cb = 1; g.K = (int)m0;
    if (split) DFB_TRY(launch_gemm_splitk(h, g, 4, scratch));
    else DFB_TRY(launch_gemm(h, g, EPI_STORE, step));
  }
  // S = A[last, last] - P P^T  (K = 0 degenerates to a copy)
  memset(&g, 0, sizeof(g));
  g.A = top_row; g.lda = npad; g.B = top_row; g.ldb = npad; g.C = h->Ks + m0; g.ldc = npad;
  g.D = top_row + m0; g.ldd = npad; g.alpha = -1.0; g.mode = MODE_GENERIC; g.n_rb = 1; g.n_cb = 1; g.K = (int)m0;
  if (split) DFB_TRY(launch_gemm_splitk(h, g, KS, scratch));
  else DFB_TRY(launch_gemm(h, g, EPI_STORE, 1));
  // identity in the diagonal block of L^-T
  DFB_CUDA_OK(cudaMemset2DAsync(mid + m0 * npad + m0, sizeof(double) * npad, 0, sizeof(double) * TILE, TILE, h->stream));
  DFB_TRY(launch_set_diag(h, mid, npad, m0, npad, 1.0, 0));
  // y_c = y[last] - v[:m0] P^T (rows 1..127 of the y block are zero and stay zero)
  DFB_TRY(launch_copy_pad(h, h->yc + m0, n - m0, yrow + m0, TILE));
  memset(&g, 0, sizeof(g));
  g.A = yrow; g.lda = npad; g.B = top_row; g.ldb = npad; g.C = yrow + m0; g.ldc = npad;
  g.D = yrow + m0; g.ldd = npad; g.alpha = -1.0; g.mode = MODE_GENERIC; g.n_rb = 1; g.n_cb = 1; g.K = (int)m0;
  if (split) DFB_TRY(launch_gemm_splitk(h, g, KS, scratch));
  else DFB_TRY(launch_gemm(h, g, EPI_STORE, 1));
  // replay of factorisation step nb-1
  DFB_TRY(launch_chol_diag(h, h->T, npad, step, h->Dinv, h->info));
  FactorMaps maps;
  DFB_TRY(make_factor_maps(&maps, h->T, 2 * npad + TILE, npad, h->Dinv));
  FactorArgs fa;
  memset(&fa, 0, sizeof(fa));
  fa.T = h->T; fa.ld = npad; fa.step = step; fa.nb = nb; fa.panel = 1; fa.info = h->info;
  DFB_TRY(launch_factor_update(h, maps, fa, true));
  double red[7];
  int info = 0;
  DFB_TRY(posterior_tail(h, flags, false, red, &info));
  if (!stationary) h->max_diag = fmax(h->max_diag, red[6] + h->noise_var);
  if (info != 0) {
    set_error("extended matrix is not positive definite: non-positive pivot at index %d", info - 1);
    return info;
  }
  h->have_post = true;
  h->have_w = true;
  DFB_TRY(prepare_scoring(h, true, false));     // npad is unchanged: the fp64 TMA maps stay valid
  if (lml_out_host != nullptr) *lml_out_host = lml((flags == DFB_BUILD_FULL) ? red[1] : red[2], red[0], n);
  return 0;
}

struct ChunkOut {
  double* mu; double* sd; double* score;   // user pointers (space given), may be NULL
};

// Scores m candidates chunk by chunk: K_* rows + mu -> |L^-1 k_*|^2 -> sd / acquisition / arg-max.
struct ChunkMode {
  bool want_std = false, do_argmax = false;
  bool use_i8 = false;                 // int8-slice wgmma contraction instead of fp64 DMMA
  bool collect = false;                // gather the shortlist for the exact re-score
  I8ErrModel em{};                     // int8 error model (collect): bound on |d sigma^2|, score sensitivity
  double pad = 0.0;                    // extra slack of the shortlist test
  const int64_t* idx_map = nullptr;    // global index of each row (re-score passes), NULL = idx_base + row
  int64_t idx_base = 0;                // global index of row 0 when idx_map is NULL
  bool allow_small = false;            // dfb_eval of <= SMALL_EVAL_M points: row-streaming kernel instead of the tile GEMM
  bool keep_scores = false;            // leave the scores of a single-chunk pass in h->score (self-check of the shortlist)
  bool keep_best = false;              // continue the running arg-max and best_lb of an earlier pass instead of resetting them
  // DFB_ACQ_TS_MARGINAL: the pass's m normals in the space of its rows, or NULL for rng_normal(ts_seed, ts_row0 + global
  // index).  The fp64 passes (use_i8 false) count the non-positive variances into h->ts_nonpos.
  const double* ts_z = nullptr;
  uint64_t ts_seed = 0;
  int64_t ts_row0 = 0;
};
constexpr int64_t SMALL_EVAL_M = 32;      // up to four 8-wide passes over W's rows (105 MB each at N = 5000): still ~10x cheaper than one 128-wide tile pass

// Checks the candidates' column count against the active kernel and brings the scaled training sets up to date.
static int prepare_candidates(dfb_handle* h, const ActiveKernel& k, int32_t dc, int32_t space) {
  if (dc != k.desc.cand_dim) { set_error("candidates have %d columns, the kernel descriptor expects %d", dc, k.desc.cand_dim); return -1; }
  if (space == DFB_HOST && dc > DFB_MAX_SLOTS) { set_error("host candidates: dc > %d", DFB_MAX_SLOTS); return -1; }
  DFB_TRY(ensure_train_scaled(h));
  DFB_TRY(ensure_test_scaled(h));
  return 0;
}

// How the rows of the caller's candidate matrix reach the device, step by step.  Steps cover the rows in order and
// never straddle a batch.  Device rows are used in place, as one batch.  Host rows are staged in batches of as many
// whole chunks as h->stage holds (chunk x DFB_MAX_SLOTS doubles), so a 6-column matrix needs one copy per ~21 chunks.
// Page-locked host rows (what the streamed `rand` maximiser hands over) use the buffer as two halves, and the copy of
// batch b+1 runs on h->cp_stream while batch b is scored (cp_done: copy done, cp_free: every step that reads the half
// is done).  Pageable memory keeps the single-buffer copy on the compute stream: its cudaMemcpyAsync would block the
// host on the half's cp_free and stall the launches of the batch in flight.
struct CandidateStage {
  dfb_handle* h = nullptr;
  const double* Xc = nullptr; // the caller's rows
  int64_t m = 0, batch = 0;   // batch: rows per batch
  int32_t dc = 0;
  bool host = false;          // the rows, and so the results, are in host memory
  bool dbuf = false;          // page-locked host rows: two halves, copies one batch ahead on h->cp_stream

  int open(dfb_handle* hh, const double* X, int64_t mm, int32_t d, int32_t space) {
    h = hh; Xc = X; m = batch = mm; dc = d; host = space == DFB_HOST;
    if (!host) return 0;
    const int64_t Mc = h->chunk;
    const int64_t stage_rows = (Mc * DFB_MAX_SLOTS / dc) / Mc * Mc;
    const int64_t half_rows = (stage_rows / Mc / 2) * Mc;
    if (half_rows >= Mc && m > half_rows) {
      cudaPointerAttributes pa;
      if (cudaPointerGetAttributes(&pa, Xc) == cudaSuccess && pa.type == cudaMemoryTypeHost) dbuf = true;
      cudaGetLastError();                                   // an unregistered pointer may leave a sticky-free error behind
    }
    batch = dbuf ? half_rows : stage_rows;
    if (!dbuf) return 0;
    if (h->cp_stream == nullptr) {
      DFB_CUDA_OK(cudaStreamCreateWithFlags(&h->cp_stream, cudaStreamNonBlocking));
      cudaEvent_t* evs[5] = {&h->cp_done[0], &h->cp_free[0], &h->cp_done[1], &h->cp_free[1], &h->cp_fork};
      for (int i = 0; i < 5; i++) DFB_CUDA_OK(cudaEventCreateWithFlags(evs[i], cudaEventDisableTiming));
    }
    DFB_CUDA_OK(cudaEventRecord(h->cp_fork, h->stream));  // the copy stream starts after everything already on the caller's stream
    DFB_CUDA_OK(cudaStreamWaitEvent(h->cp_stream, h->cp_fork, 0));
    return 0;
  }
  // *xc: the device rows of the step that starts at row c0
  int rows(int64_t c0, const double** xc) {
    if (!host) { *xc = Xc + c0 * dc; return 0; }
    const int64_t bi = c0 / batch;
    if (c0 % batch == 0) {                                  // first step of batch bi
      if (bi == 0 || !dbuf) DFB_TRY(copy(bi));
      if (dbuf && (bi + 1) * batch < m) DFB_TRY(copy(bi + 1));
      if (dbuf) DFB_CUDA_OK(cudaStreamWaitEvent(h->stream, h->cp_done[bi & 1], 0));
    }
    *xc = buffer(bi) + (c0 - bi * batch) * dc;
    return 0;
  }
  // Every launch that reads rows c0 .. c0 + mc - 1 is enqueued: after the last step of a batch its half may be refilled.
  int done(int64_t c0, int64_t mc) {
    if (dbuf && (c0 + mc == m || (c0 + mc) % batch == 0))
      DFB_CUDA_OK(cudaEventRecord(h->cp_free[(c0 / batch) & 1], h->stream));
    return 0;
  }
  double* buffer(int64_t bi) const { return h->stage + (dbuf ? (bi & 1) * batch * dc : 0); }
  int copy(int64_t bi) {      // batch bi into its buffer: on the compute stream, or one batch ahead on the copy stream
    const int64_t lo = bi * batch, hi = std::min(m, lo + batch);
    const cudaStream_t s = dbuf ? h->cp_stream : h->stream;
    if (dbuf && bi >= 2) DFB_CUDA_OK(cudaStreamWaitEvent(s, h->cp_free[bi & 1], 0));
    DFB_CUDA_OK(cudaMemcpyAsync(buffer(bi), Xc + lo * dc, sizeof(double) * (hi - lo) * dc, cudaMemcpyHostToDevice, s));
    if (dbuf) DFB_CUDA_OK(cudaEventRecord(h->cp_done[bi & 1], s));
    return 0;
  }
};

// The fp64 tile contraction of the G stage: per 128-row block of W, the partial |L^-1 k_*|^2 of the first m_rows rows
// of h->Ks into h->partial (leading dimension: the chunk).
static int contract_tiles_f64(dfb_handle* h, int64_t m_rows) {
  const int64_t npad = h->npad;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.A = h->W; g.lda = npad; g.B = h->Ks; g.ldb = npad; g.mode = MODE_SCORE;
  g.n_rb = (int)(npad / TILE); g.n_cb = (int)(m_rows / TILE); g.K = (int)npad;
  g.partial = h->partial; g.ld_partial = h->chunk;
  if (h->gemm_impl == 1 && h->tma_ready) {
    ScoreTmaArgs ta;
    ta.n_rb = g.n_rb; ta.n_cb = g.n_cb; ta.K = g.K; ta.partial = g.partial; ta.ld_partial = g.ld_partial;
    ta.cb_group = h->tma_cb_group;
    return launch_score_tma(h, h->tmW, h->tmK, ta);
  }
  return launch_gemm(h, g, EPI_SUMSQ, g.n_rb * g.n_cb);
}

// The row-streaming contraction of dfb_eval applies to m <= SMALL_EVAL_M rows when option small_eval is on and the
// per-warp partials fit h->partial.
static bool small_eval_fits(const dfb_handle* h) {
  return h->small_eval != 0 && (int64_t)((h->n + 7) / 8 * 8) * SMALL_EVAL_M <= (int64_t)(h->npad / TILE) * h->chunk;
}

// Per chunk two stages, back to back on the handle's stream:
//   K: K_* rows / digit planes + mu + k(x*,x*)                                      fp64 pipe
//   G: the contraction |L^-1 k_*|^2 -> sd / acquisition / arg-max / shortlist       tensor pipe (int8) or DMMA
static int run_chunks(dfb_handle* h, const dfb_acq_desc& acq, const double* Xc, int64_t m, int32_t dc,
                      int32_t space, double mean_const, ChunkOut out, const ChunkMode& md) {
  const bool want_std = md.want_std, do_argmax = md.do_argmax;
  const ActiveKernel k = active_kernel(h);
  DFB_TRY(prepare_candidates(h, k, dc, space));
  const int64_t npad = h->npad, Mc = h->chunk;
  const int nb = (int)(npad / TILE);
  if (do_argmax && !md.keep_best) DFB_TRY(launch_reset_best(h));
  const bool i8 = want_std && md.use_i8;
  CandidateStage st;
  DFB_TRY(st.open(h, Xc, m, dc, space));
  const int* abort_count = md.collect ? h->list_count : nullptr;
  const bool small = want_std && md.allow_small && !md.use_i8 && m <= SMALL_EVAL_M && small_eval_fits(h);
  // K_* arguments of every chunk; the candidates, their count and mu are set per chunk
  KstarArgs ka{};
  ka.desc = &k.desc; ka.d_desc = k.d_desc; ka.xsT = k.ss.xs; ka.nrmT = k.ss.nrm; ka.npad_tr = npad; ka.alpha = h->alpha;
  ka.dc = dc; ka.n_valid = h->n; ka.n_write = npad; ka.Ks = h->Ks; ka.ldk = npad; ka.mean_const = mean_const;
  ka.kss_out = want_std ? h->kssv : nullptr; ka.abort_count = abort_count; ka.cprep = h->cprep; ka.mu_part = h->mu_part;
  if (i8) {
    ka.planes = h->Ki8; ka.plane_bytes = 2 * h->chunk * npad; ka.row_bytes = 2 * npad;
    ka.inv_colscale = 1.0 / i8_colscale(k.desc);
  }
  const KstarWant want = !want_std ? KstarWant::MU : i8 ? KstarWant::DIGITS : KstarWant::ROWS;

  for (int64_t c0 = 0; c0 < m; c0 += Mc) {
    const int64_t mc = std::min(m - c0, Mc);
    const int64_t m_rows = round_up(mc, TILE);
    const double* xc_dev;
    DFB_TRY(st.rows(c0, &xc_dev));
    double* mu_dev = (space == DFB_DEVICE && out.mu) ? out.mu + c0 : h->mu;
    double* sd_dev = (space == DFB_DEVICE && out.sd) ? out.sd + c0 : h->sd;
    double* sc_dev = (space == DFB_DEVICE && out.score) ? out.score + c0
                                                         : ((out.score || md.collect || md.keep_scores) ? h->score : nullptr);
    ka.Xc = xc_dev; ka.m = mc; ka.m_rows = m_rows; ka.mu = mu_dev;
    const KstarRoute route = route_kstar(h, ka, want);

    // K stage
    DFB_TRY(prof_begin(h, DFB_PROF_KSTAR));
    DFB_TRY(launch_kstar(h, ka, route));
    if (route.slice_i8)     // K_* = 2^F * digits: |K_*| <= k(x,x) for every supported (stationary, non-negative) kernel
      DFB_TRY(launch_slice_i8(h, h->Ks, npad, m_rows, npad, nullptr, ka.inv_colscale, h->Ki8, ka.plane_bytes,
                              ka.row_bytes));
    DFB_TRY(prof_end(h, DFB_PROF_KSTAR, (double)mc));

    // G stage
    int small_warps = 0;
    if (small) {
      // the padded rows of K_* beyond mc are zero, so an 8-wide pass may run past mc (within the 128-row tile)
      DFB_TRY(prof_begin(h, DFB_PROF_GEMM));
      DFB_TRY(launch_small_sumsq(h, h->W, npad, h->Ks, npad, h->n, (int)mc, h->partial, SMALL_EVAL_M, &small_warps));
      DFB_TRY(prof_end(h, DFB_PROF_GEMM, (double)mc));
    } else if (want_std) {
      DFB_TRY(prof_begin(h, DFB_PROF_GEMM));
      if (md.use_i8) {
        const double colscale = i8_colscale(k.desc);
        DFB_TRY(launch_score_i8_args(h, h->i8_radix256 != 0, h->tmWi8, h->tmKi8, nb,
                                     (int)(m_rows / i8_tile_n(h->i8_radix256)), (int)npad, h->partial, Mc,
                                     h->rowscale, colscale, abort_count));
      } else {
        DFB_TRY(contract_tiles_f64(h, m_rows));
      }
      DFB_TRY(prof_end(h, DFB_PROF_GEMM, (double)mc));
    }
    if (want_std || do_argmax || sc_dev != nullptr) {
      DFB_TRY(prof_begin(h, DFB_PROF_ACQ));
      const int64_t* idx_map = md.idx_map ? md.idx_map + c0 : nullptr;
      const bool ts = acq.kind == DFB_ACQ_TS_MARGINAL;
      TsZ tz;
      memset(&tz, 0, sizeof(tz));
      if (ts) {
        if (md.ts_z != nullptr && st.host) {          // host normals: staged chunk by chunk with their rows
          DFB_CUDA_OK(cudaMemcpyAsync(h->ts_z, md.ts_z + c0, sizeof(double) * mc, cudaMemcpyHostToDevice, h->stream));
          tz.z = h->ts_z;
        } else if (md.ts_z != nullptr) {
          tz.z = md.ts_z + c0;
        }
        tz.seed = md.ts_seed; tz.row0 = md.ts_row0;
        tz.z_out = (tz.z == nullptr && md.collect) ? h->ts_z : nullptr;    // generated normals for the shortlist
        tz.nonpos = md.use_i8 ? nullptr : h->ts_nonpos;
      }
      DFB_TRY(launch_acq(h, acq, mu_dev, h->partial, small ? SMALL_EVAL_M : Mc, small ? small_warps : nb, h->kssv, mc,
                         md.idx_base + c0, want_std ? 1 : 0, want_std ? sd_dev : nullptr, sc_dev, do_argmax, idx_map,
                         md.collect ? &md.em : nullptr, ts ? &tz : nullptr));
      if (md.collect)
        DFB_TRY(launch_collect_shortlist(h, sc_dev, sd_dev, mc, md.idx_base + c0, idx_map, md.em, md.pad, xc_dev, dc,
                                         ts ? (tz.z != nullptr ? tz.z : h->ts_z) : nullptr));
      DFB_TRY(prof_end(h, DFB_PROF_ACQ, (double)mc));
    }
    if (st.host) {
      if (out.mu)
        DFB_CUDA_OK(cudaMemcpyAsync(out.mu + c0, mu_dev, sizeof(double) * mc, cudaMemcpyDeviceToHost, h->stream));
      if (out.sd && want_std)
        DFB_CUDA_OK(cudaMemcpyAsync(out.sd + c0, sd_dev, sizeof(double) * mc, cudaMemcpyDeviceToHost, h->stream));
      if (out.score)
        DFB_CUDA_OK(cudaMemcpyAsync(out.score + c0, sc_dev, sizeof(double) * mc, cudaMemcpyDeviceToHost, h->stream));
    }
    DFB_TRY(st.done(c0, mc));
  }
  return 0;
}

// The bound pass of dfb_score_argmax (see bound_pass_applies): no K_* rows, no contraction, but one screen per step of
// keep_cap device rows or one staging batch of host rows, which appends the candidates whose acquisition bound reaches
// best_lb - pad to the survivor list (global index idx_base + row).  With mu_out it writes mu_bar there instead, a chunk
// per step (dfb_mu_upper_bound).  Void once *abort_count (the seed's shortlist; may be NULL) has overflowed.
static int run_bound_pass(dfb_handle* h, const dfb_acq_desc& acq, const double* Xc, int64_t m, int32_t dc, int32_t space,
                          double mean_const, double pad, int64_t idx_base, const int* abort_count, double* mu_out) {
  const ActiveKernel k = active_kernel(h);
  DFB_TRY(prepare_candidates(h, k, dc, space));
  CandidateStage st;
  DFB_TRY(st.open(h, Xc, m, dc, space));
  const int64_t step = mu_out != nullptr ? h->chunk : std::min(h->keep_cap, st.batch);    // keep_cap >= a host batch
  for (int64_t c0 = 0; c0 < m; c0 += step) {
    const int64_t mc = std::min(m - c0, step);
    const double* xc_dev;
    DFB_TRY(st.rows(c0, &xc_dev));
    double* mu_dev = mu_out == nullptr ? nullptr : space == DFB_DEVICE ? mu_out + c0 : h->mu;
    DFB_TRY(prof_begin(h, DFB_PROF_PRUNE));
    DFB_TRY(launch_prune(h, acq, k.desc, k.d_desc, k.ss.xs, xc_dev, mc, dc, mean_const, pad, idx_base + c0, abort_count,
                         mu_dev));
    DFB_TRY(prof_end(h, DFB_PROF_PRUNE, (double)mc));
    if (st.host && mu_out != nullptr)
      DFB_CUDA_OK(cudaMemcpyAsync(mu_out + c0, mu_dev, sizeof(double) * mc, cudaMemcpyDeviceToHost, h->stream));
    DFB_TRY(st.done(c0, mc));
  }
  return 0;
}

}  // namespace dfb

using namespace dfb;

extern "C" {

int dfb_version(void) { return DFB_VERSION; }

const char* dfb_last_error(void) { return g_err; }

int dfb_create(dfb_handle** out, int device) {
  if (out == nullptr) { set_error("out is NULL"); return -1; }
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    set_error("no CUDA device visible (%s): libdfb200 has no CPU fallback", cudaGetErrorString(e));
    return -2;
  }
  if (device < 0 || device >= count) { set_error("device %d out of range (0..%d)", device, count - 1); return -1; }
  DFB_CUDA_OK(cudaSetDevice(device));
  int cc_major = 0, cc_minor = 0;     // attribute queries: cudaGetDeviceProperties costs milliseconds per call
  DFB_CUDA_OK(cudaDeviceGetAttribute(&cc_major, cudaDevAttrComputeCapabilityMajor, device));
  DFB_CUDA_OK(cudaDeviceGetAttribute(&cc_minor, cudaDevAttrComputeCapabilityMinor, device));
  if (cc_major != 9 || cc_minor != 0) {
    set_error("device %d is sm_%d%d; libdfb200 is built for sm_90a (H100) only", device, cc_major, cc_minor);
    return -2;
  }
  dfb_handle* h = new (std::nothrow) dfb_handle();
  if (h == nullptr) { set_error("out of host memory"); return -2; }
  h->device = device;
  const char* impl = getenv("DFB200_GEMM");       // "v1" = cp.async ring, "tma" = TMA + mbarrier ring
  h->gemm_impl = (impl != nullptr && strcmp(impl, "v1") == 0) ? 0 : 1;   // default: TMA ring
  const char* simpl = getenv("DFB200_SCORE");     // "i8" = int8-slice wgmma contraction
  h->score_impl = 2;                              // auto
  if (simpl != nullptr && strcmp(simpl, "i8") == 0) h->score_impl = 1;
  if (simpl != nullptr && strcmp(simpl, "fp64") == 0) h->score_impl = 0;
  *out = h;
  return 0;
}

void dfb_destroy(dfb_handle* h) {
  if (h == nullptr) return;
  if (h->fs_hi != nullptr) {
    cudaStreamDestroy(h->fs_hi); cudaStreamDestroy(h->fs_lo);
    cudaEventDestroy(h->fe_fork); cudaEventDestroy(h->fe_panel); cudaEventDestroy(h->fe_rest);
    cudaEventDestroy(h->fe_join_hi); cudaEventDestroy(h->fe_join_lo);
  }
  if (h->cp_stream != nullptr) {
    cudaStreamDestroy(h->cp_stream); cudaEventDestroy(h->cp_fork);
    for (int i = 0; i < 2; i++) { cudaEventDestroy(h->cp_done[i]); cudaEventDestroy(h->cp_free[i]); }
  }
  if (h->prof != nullptr) {
    for (int c = 0; c < PROF_CLASSES; c++)
      if (h->prof[c].created)
        for (int i = 0; i < PROF_RING; i++) { cudaEventDestroy(h->prof[c].start[i]); cudaEventDestroy(h->prof[c].stop[i]); }
    delete[] h->prof;
  }
  delete h;
}

int dfb_set_stream(dfb_handle* h, void* cuda_stream) {
  DFB_TRY(need(h, false, false, false, false, false));
  h->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  return 0;
}

size_t dfb_workspace_bytes(int64_t n_max, int32_t n_slots, int64_t chunk) {
  (void)n_slots;
  return carve(nullptr, nullptr, n_max, chunk);
}

int dfb_set_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t n_max, int64_t chunk) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (workspace_dev == nullptr || n_max < 1) { set_error("bad workspace arguments"); return -1; }
  const size_t want = carve(nullptr, nullptr, n_max, chunk);
  if (bytes < want) { set_error("workspace too small: %zu bytes given, %zu needed", bytes, want); return -1; }
  if ((reinterpret_cast<uintptr_t>(workspace_dev) & 255) != 0) { set_error("workspace must be 256-byte aligned"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  h->ws = static_cast<char*>(workspace_dev);
  h->ws_bytes = bytes;
  carve(h, h->ws, n_max, chunk);
  h->have_train = h->have_post = h->have_w = false;
  h->tr_prepped = h->te_prepped = false;
  if (h->have_kernel)
    DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_tr, &h->desc_tr, sizeof(dfb_kernel_desc), cudaMemcpyHostToDevice, h->stream));
  if (h->have_test_kernel)
    DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_te, &h->desc_te, sizeof(dfb_kernel_desc), cudaMemcpyHostToDevice, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dfb_set_kernel(dfb_handle* h, const dfb_kernel_desc* desc) {
  DFB_TRY(need(h, true, false, false, false, false));
  DFB_TRY(check_desc(desc));
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));   // the pageable host copy below must not race
  h->desc_tr = *desc;
  DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_tr, &h->desc_tr, sizeof(dfb_kernel_desc), cudaMemcpyHostToDevice, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  h->have_kernel = true;
  h->tr_prepped = false;
  h->have_post = h->have_w = false;
  return 0;
}

int dfb_set_test_kernel(dfb_handle* h, const dfb_kernel_desc* desc) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (desc == nullptr) { h->have_test_kernel = false; h->te_prepped = false; return 0; }
  DFB_TRY(check_desc(desc));
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  h->desc_te = *desc;
  DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_te, &h->desc_te, sizeof(dfb_kernel_desc), cudaMemcpyHostToDevice, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  h->have_test_kernel = true;
  h->te_prepped = false;
  return 0;
}

int dfb_set_train(dfb_handle* h, const double* X_dev, int64_t n, int32_t d, const double* y_centred_dev) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (n < 1 || n > h->n_max) { set_error("n = %lld outside [1, n_max = %lld]", (long long)n, (long long)h->n_max); return -1; }
  if (d < 1 || d > DFB_MAX_SLOTS) { set_error("d = %d outside [1, %d]", d, DFB_MAX_SLOTS); return -1; }
  if (X_dev == nullptr || y_centred_dev == nullptr) { set_error("X / y pointer is NULL"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  h->n = n; h->d = d; h->npad = round_up(n, TILE);
  DFB_CUDA_OK(cudaMemcpyAsync(h->X, X_dev, sizeof(double) * n * d, cudaMemcpyDeviceToDevice, h->stream));
  DFB_TRY(launch_copy_pad(h, y_centred_dev, n, h->yc, h->npad));
  DFB_TRY(launch_fill(h, h->alpha, h->npad, 0.0));
  h->have_train = true;
  h->tr_prepped = h->te_prepped = false;
  h->have_post = h->have_w = false;
  return 0;
}

int dfb_build_posterior(dfb_handle* h, double noise_var, double jitter, int32_t flags, double* lml_out_host) {
  DFB_TRY(need(h, true, true, true, false, false));
  if (h->desc_tr.train_dim != h->d) { set_error("kernel train_dim %d != data dim %d", h->desc_tr.train_dim, h->d); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  const int64_t n = h->n, npad = h->npad;
  const bool with_bottom = (flags != DFB_BUILD_LML_ONLY);
  h->have_post = h->have_w = false;
  DFB_TRY(prof_begin(h, DFB_PROF_BUILD));
  DFB_CUDA_OK(cudaMemsetAsync(h->info, 0, sizeof(int) * 4, h->stream));
  DFB_CUDA_OK(cudaMemsetAsync(h->T, 0, sizeof(double) * (size_t)(2 * npad + TILE) * npad, h->stream));
  DFB_TRY(prof_begin(h, DFB_PROF_BUILD_KXX));
  DFB_TRY(ensure_train_scaled(h));
  DFB_TRY(launch_train_kstar(h, 0, n, h->T, npad, npad));
  // the jitter ladder's scale max(diag K) + noise: kss for a stationary kernel, else read off the diagonal just built
  const bool stationary = kernel_stationary(h->desc_tr);
  if (!stationary) DFB_TRY(launch_diag_max(h, h->T, npad, n, h->red + 6));
  DFB_TRY(launch_init_tall(h, h->T, n, npad, noise_var + jitter, h->yc, with_bottom ? 1 : 0));
  DFB_TRY(prof_end(h, DFB_PROF_BUILD_KXX, 1.0));
  DFB_TRY(factorise_tall(h, h->T, npad, h->Dinv, h->info, with_bottom, true));
  double red[7];
  int info = 0;
  DFB_TRY(posterior_tail(h, flags, true, red, &info));
  h->max_diag = (stationary ? h->desc_tr.kss : red[6]) + noise_var;
  h->noise_var = noise_var;
  if (info != 0) {
    set_error("matrix is not positive definite: non-positive pivot at index %d", info - 1);
    return info;
  }
  h->noise_plus_jitter = noise_var + jitter;
  h->have_post = true;
  h->have_w = with_bottom;
  DFB_TRY(prof_begin(h, DFB_PROF_BUILD_I8));
  DFB_TRY(prepare_scoring(h, true, true));
  DFB_TRY(prof_end(h, DFB_PROF_BUILD_I8, 1.0));
  if (lml_out_host != nullptr) *lml_out_host = lml((flags == DFB_BUILD_FULL) ? red[1] : red[2], red[0], n);
  return 0;
}

// The body of dfb_lml_batch and dfb_lml_batch_mixed: allow_hamming is the one difference.
static int lml_batch_impl(dfb_handle* h, const dfb_kernel_desc* descs, const double* noise_var,
                          const double* mean_const, int32_t B, double* lml_out, int32_t* info_out, bool allow_hamming) {
  DFB_TRY(need(h, true, false, true, false, false));
  if (B < 0 || (B > 0 && (descs == nullptr || noise_var == nullptr || mean_const == nullptr || lml_out == nullptr ||
                          info_out == nullptr))) {
    set_error("lml_batch: bad arguments");
    return -1;
  }
  if (h->npad > LML_BATCH_MAX_NPAD) {
    set_error("lml_batch: n = %lld above the batch kernel's %d", (long long)h->n, LML_BATCH_MAX_NPAD);
    return -1;
  }
  int ns_max = 1, nf_max = 1;
  bool any_hamming = false;
  for (int b = 0; b < B; b++) {
    DFB_TRY(check_desc(&descs[b]));
    if (descs[b].esp_order != 0) { set_error("lml_batch: item %d is an ESP kernel", b); return -1; }
    for (int f = 0; f < descs[b].n_factors; f++) {
      if (descs[b].factors[f].kind == DFB_BASE_HAMMING) {
        if (!allow_hamming) {
          set_error("lml_batch: item %d has a HAMMING factor (dfb_lml_batch_mixed evaluates them)", b);
          return -1;
        }
        any_hamming = true;
      }
    }
    if (descs[b].train_dim != h->d) {
      set_error("lml_batch: item %d has train_dim %d != data dim %d", b, descs[b].train_dim, h->d);
      return -1;
    }
    ns_max = std::max(ns_max, (int)descs[b].n_slots);
    nf_max = std::max(nf_max, (int)descs[b].n_factors);
  }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  // The K_* chunk buffer is idle outside scoring: it holds the items' parameters, results and factorisation scratch.
  // A batch larger than it holds runs as consecutive launches of what fits.
  const int64_t npad = h->npad;
  const int64_t item = lml_batch_item_doubles(npad, ns_max, nf_max);
  const size_t per_item_bytes = sizeof(dfb_kernel_desc) + 4 * sizeof(double) + sizeof(int) + item * sizeof(double);
  const size_t ks_bytes = (size_t)h->chunk * h->npad_max * sizeof(double);
  const int64_t cap = std::min<int64_t>((int64_t)((ks_bytes - 4096) / per_item_bytes), 65535);
  if (cap < 1) { set_error("lml_batch: workspace too small for one item"); return -1; }
  std::vector<char> up, down;
  for (int b0 = 0; b0 < B; b0 += (int)cap) {
    const int nb_items = (int)std::min<int64_t>(cap, B - b0);
    Carver c(reinterpret_cast<char*>(h->Ks));
    dfb_kernel_desc* d_descs = c.take<dfb_kernel_desc>(nb_items);
    double* d_noise = c.take<double>(nb_items);
    double* d_mean = c.take<double>(nb_items);
    const size_t up_bytes = c.off;
    double* d_red = c.take<double>(2 * (size_t)nb_items);
    const size_t down_off = (reinterpret_cast<char*>(d_red) - reinterpret_cast<char*>(h->Ks));
    int* d_info = c.take<int>(nb_items);
    const size_t down_bytes = c.off - down_off;
    double* scratch = c.take<double>((size_t)item * nb_items);
    up.assign(up_bytes, 0);
    memcpy(up.data() + (reinterpret_cast<char*>(d_descs) - reinterpret_cast<char*>(h->Ks)), descs + b0,
           sizeof(dfb_kernel_desc) * nb_items);
    memcpy(up.data() + (reinterpret_cast<char*>(d_noise) - reinterpret_cast<char*>(h->Ks)), noise_var + b0,
           sizeof(double) * nb_items);
    memcpy(up.data() + (reinterpret_cast<char*>(d_mean) - reinterpret_cast<char*>(h->Ks)), mean_const + b0,
           sizeof(double) * nb_items);
    DFB_CUDA_OK(cudaMemcpyAsync(h->Ks, up.data(), up_bytes, cudaMemcpyHostToDevice, h->stream));
    LmlBatchArgs g;
    g.descs = d_descs; g.noise = d_noise; g.mean = d_mean;
    g.X = h->X; g.y = h->yc; g.n = h->n; g.d = h->d; g.npad = npad;
    g.ns_max = ns_max; g.nf_max = nf_max;
    g.scratch = scratch; g.item_doubles = item;
    g.red = d_red; g.info = d_info;
    DFB_TRY(launch_lml_batch(h, g, nb_items, any_hamming));
    down.resize(down_bytes);
    DFB_CUDA_OK(cudaMemcpyAsync(down.data(), d_red, down_bytes, cudaMemcpyDeviceToHost, h->stream));
    DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
    const double* red = reinterpret_cast<const double*>(down.data());
    const int* info = reinterpret_cast<const int*>(down.data() + (reinterpret_cast<char*>(d_info) -
                                                                   reinterpret_cast<char*>(d_red)));
    for (int b = 0; b < nb_items; b++) {
      info_out[b0 + b] = info[b];
      lml_out[b0 + b] = info[b] != 0 ? NAN : lml(red[2 * b + 1], red[2 * b], h->n);
    }
  }
  return 0;
}

int dfb_lml_batch(dfb_handle* h, const dfb_kernel_desc* descs, const double* noise_var, const double* mean_const,
                  int32_t B, double* lml_out, int32_t* info_out) {
  return lml_batch_impl(h, descs, noise_var, mean_const, B, lml_out, info_out, false);
}

int dfb_lml_batch_mixed(dfb_handle* h, const dfb_kernel_desc* descs, const double* noise_var, const double* mean_const,
                        int32_t B, double* lml_out, int32_t* info_out) {
  return lml_batch_impl(h, descs, noise_var, mean_const, B, lml_out, info_out, true);
}

int dfb_restore_posterior(dfb_handle* h);

int dfb_extend_posterior(dfb_handle* h, const double* X_new_dev, int64_t q, const double* y_centred_new_dev,
                         int32_t flags, double* lml_out_host) {
  DFB_TRY(need(h, true, true, true, true, true));
  const int32_t build_flags = flags & ~DFB_EXTEND_SAVE;
  if (build_flags != DFB_BUILD_FULL && build_flags != DFB_BUILD_NO_ALPHA) { set_error("dfb_extend_posterior: flags must be DFB_BUILD_FULL or DFB_BUILD_NO_ALPHA (| DFB_EXTEND_SAVE)"); return -1; }
  if (q < 1 || X_new_dev == nullptr || y_centred_new_dev == nullptr) { set_error("bad extend arguments (q = %lld)", (long long)q); return -1; }
  if (h->n + q > h->npad) {
    set_error("dfb_extend_posterior: %lld + %lld points do not fit the padded size %lld of this posterior: rebuild",
              (long long)h->n, (long long)q, (long long)h->npad);
    return -1;
  }
  if (h->ext_saved) { set_error("dfb_extend_posterior: a saved extension is active, call dfb_restore_posterior first"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  const int64_t n0 = h->n, npad = h->npad;
  const int64_t m0 = npad - TILE;
  if (flags & DFB_EXTEND_SAVE) {
    double* s = h->ext_save;
    DFB_CUDA_OK(cudaMemcpyAsync(s, h->T + m0 * npad, sizeof(double) * TILE * npad, cudaMemcpyDeviceToDevice, h->stream));
    DFB_CUDA_OK(cudaMemcpy2DAsync(s + TILE * npad, sizeof(double) * TILE, h->T + npad * npad + m0, sizeof(double) * npad,
                                  sizeof(double) * TILE, (size_t)npad, cudaMemcpyDeviceToDevice, h->stream));
    DFB_CUDA_OK(cudaMemcpyAsync(s + 2 * TILE * npad, h->T + 2 * npad * npad + m0, sizeof(double) * TILE,
                                cudaMemcpyDeviceToDevice, h->stream));
    DFB_CUDA_OK(cudaMemcpyAsync(s + 2 * TILE * npad + TILE, h->alpha, sizeof(double) * npad, cudaMemcpyDeviceToDevice, h->stream));
    h->ext_saved_n = n0;
    h->ext_saved_max_diag = h->max_diag;
  }
  DFB_CUDA_OK(cudaMemcpyAsync(h->X + n0 * h->d, X_new_dev, sizeof(double) * q * h->d, cudaMemcpyDeviceToDevice, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(h->yc + n0, y_centred_new_dev, sizeof(double) * q, cudaMemcpyDeviceToDevice, h->stream));
  h->n = n0 + q;
  if (h->n_max < h->n) h->n_max = h->n;
  const int r = replay_last_block(h, build_flags, lml_out_host);
  if (flags & DFB_EXTEND_SAVE) {
    h->ext_saved = true;
    if (r > 0) {                       // not positive definite: put the un-extended posterior back
      char msg[512];
      snprintf(msg, sizeof(msg), "%s", g_err);
      DFB_TRY(dfb_restore_posterior(h));
      set_error("%s", msg);
    }
  }
  return r;
}

int dfb_restore_posterior(dfb_handle* h) {
  DFB_TRY(need(h, true, true, true, false, false));
  if (!h->ext_saved) { set_error("dfb_restore_posterior: nothing saved"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  const int64_t npad = h->npad, m0 = npad - TILE, n0 = h->ext_saved_n;
  const double* s = h->ext_save;
  DFB_CUDA_OK(cudaMemcpyAsync(h->T + m0 * npad, s, sizeof(double) * TILE * npad, cudaMemcpyDeviceToDevice, h->stream));
  DFB_CUDA_OK(cudaMemcpy2DAsync(h->T + npad * npad + m0, sizeof(double) * npad, s + TILE * npad, sizeof(double) * TILE,
                                sizeof(double) * TILE, (size_t)npad, cudaMemcpyDeviceToDevice, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(h->T + 2 * npad * npad + m0, s + 2 * TILE * npad, sizeof(double) * TILE,
                              cudaMemcpyDeviceToDevice, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(h->alpha, s + 2 * TILE * npad + TILE, sizeof(double) * npad, cudaMemcpyDeviceToDevice, h->stream));
  DFB_TRY(launch_fill(h, h->yc + n0, npad - n0, 0.0));           // zero the appended targets
  h->n = n0;
  h->max_diag = h->ext_saved_max_diag;
  h->ext_saved = false;
  h->tr_prepped = h->te_prepped = false;
  DFB_TRY(launch_transpose(h, h->T + npad * npad, h->W, npad));
  h->have_post = h->have_w = true;
  DFB_TRY(prepare_scoring(h, true, false));     // npad is unchanged: the fp64 TMA maps stay valid
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dfb_lml_gradients(dfb_handle* h, double* out_host, int32_t n_out) {
  DFB_TRY(need(h, true, true, true, true, true));
  const dfb_kernel_desc& desc = h->desc_tr;
  if (desc.n_terms != 1 || desc.n_factors != 1 || desc.esp_order != 0 ||
      (desc.factors[0].kind != DFB_BASE_SE && desc.factors[0].kind != DFB_BASE_MATERN)) {
    // the reference's composite, ESP, Poly, ExpDecay and Hamming kernels inherit Kernel._child_gradient, which raises
    // (kernel.py:123-125)
    set_error("LML gradients are defined for plain SE / Matern kernels only (kernel has %d terms, %d factors, "
              "ESP order %d, first factor kind %d)", desc.n_terms, desc.n_factors, desc.esp_order, desc.factors[0].kind);
    return -3;
  }
  const int D = desc.factors[0].n_dims;
  const int P = 4 + D;
  if (out_host == nullptr || n_out < P) { set_error("lml_gradients: out needs 4 + d = %d entries", P); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  const int64_t npad = h->npad;
  const int nb = (int)(npad / TILE);
  const int64_t n_tiles = (int64_t)nb * (nb + 1) / 2;
  if (n_tiles * P > (int64_t)nb * h->chunk || P > h->chunk) {
    set_error("lml_gradients: scoring chunk %lld too small for %lld tile partials", (long long)h->chunk, (long long)n_tiles);
    return -1;
  }
  DFB_TRY(ensure_train_scaled(h));
  // K^-1 = W^T W row-block stripe by stripe into the K_* chunk buffer (chunk rows x npad), each followed by the
  // fused reduction against the kernel derivatives.  L^-T sits in the middle block of the tall matrix.
  const double* Wt = h->T + (size_t)npad * npad;
  const int stripe = (int)((h->chunk / TILE) < nb ? (h->chunk / TILE) : nb);
  for (int rb0 = 0; rb0 < nb; rb0 += stripe) {
    const int R = (nb - rb0 < stripe) ? nb - rb0 : stripe;
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.A = Wt + (int64_t)rb0 * TILE * npad; g.lda = npad; g.B = Wt; g.ldb = npad; g.D = h->Ks; g.ldd = npad;
    g.alpha = 1.0; g.mode = MODE_GENERIC; g.n_rb = R; g.n_cb = nb; g.K = (int)npad; g.tri = 3; g.lower_only = 1;
    g.rb0 = rb0;
    DFB_TRY(launch_gemm(h, g, EPI_STORE, R * nb));
    DFB_TRY(launch_lml_grad_tiles(h, h->d_desc_tr, h->tr.xs, h->tr.nrm, npad, h->alpha, h->Ks, npad, rb0, R, nb, h->n, P,
                                  h->partial));
  }
  DFB_TRY(launch_lml_grad_reduce(h, h->partial, n_tiles, P, P, h->alpha, h->n, h->score));
  DFB_CUDA_OK(cudaMemcpyAsync(out_host, h->score, sizeof(double) * P, cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  // 1/2 tr(.) (gp_core.py:240); slot 1 still lacks the factor noise_var, slot 2 is sum(alpha) as is
  for (int p = 0; p < P; p++) if (p != 2) out_host[p] *= 0.5;
  return 0;
}

int dfb_get_max_diag(dfb_handle* h, double* out_host) {
  DFB_TRY(need(h, true, true, true, false, false));
  if (out_host == nullptr) { set_error("out is NULL"); return -1; }
  *out_host = h->max_diag;
  return 0;
}

int dfb_get_state(dfb_handle* h, double* L_dev, double* alpha_dev, double* K_dev) {
  DFB_TRY(need(h, true, true, true, true, false));
  DFB_CUDA_OK(cudaSetDevice(h->device));
  if (L_dev) DFB_TRY(launch_extract_lower(h, h->T, h->npad, L_dev, h->n));
  if (alpha_dev) DFB_TRY(launch_copy_pad(h, h->alpha, h->n, alpha_dev, h->n));
  if (K_dev) DFB_TRY(launch_train_kstar(h, 0, h->n, K_dev, h->n, h->n));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dfb_set_alpha(dfb_handle* h, const double* alpha_dev, int64_t n) {
  DFB_TRY(need(h, true, true, true, false, false));
  if (alpha_dev == nullptr || n < 0 || n > h->n) { set_error("bad alpha arguments"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_TRY(launch_copy_pad(h, alpha_dev, n, h->alpha, h->npad));
  return 0;
}

int dfb_eval(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space, double mean_const,
             double* mu, double* sd) {
  DFB_TRY(need(h, true, true, true, true, sd != nullptr));
  if (m < 0 || (m > 0 && (Xc == nullptr || mu == nullptr))) { set_error("bad eval arguments"); return -1; }
  if (m == 0) return 0;
  DFB_CUDA_OK(cudaSetDevice(h->device));
  dfb_acq_desc acq;
  memset(&acq, 0, sizeof(acq));
  acq.kind = DFB_ACQ_MEAN;
  ChunkOut out = {mu, sd, nullptr};
  ChunkMode md;
  md.want_std = sd != nullptr;
  md.use_i8 = (sd != nullptr) && (h->score_impl == 1) && i8_usable(h, active_kernel(h).desc);
  md.allow_small = h->small_eval != 0;
  h->last_used_i8 = md.use_i8 ? 1 : 0;
  DFB_TRY(run_chunks(h, acq, Xc, m, dc, space, mean_const, out, md));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

// dfb_score_groups.  The groups' descriptors go to h->d_desc_grp and their scaled training sets side by side into the
// test-kernel set h->te (group g from slot / factor offset sum_{g' < g} n_slots / n_factors), which is re-prepared when
// a test kernel is next used.  Rows are put in group order, staged packed (each group's rows with its own column count),
// and scored SMALL_EVAL_M at a time: per group present in a pass, one K_* launch writes its rows' K_*, mu and k(x*, x*)
// at their place in the pass; one contraction covers the pass; per group, one acquisition launch with its beta.
int dfb_score_groups(dfb_handle* h, const dfb_kernel_desc* descs, const double* betas, int32_t n_groups,
                     const double* X_host, int64_t m, int32_t ldx, const int32_t* group_host, double* scores_host) {
  DFB_TRY(need(h, true, true, true, true, true));
  if (descs == nullptr || betas == nullptr || n_groups < 1 || n_groups > DFB_MAX_GROUPS) {
    set_error("score_groups: n_groups = %d outside [1, %d] or NULL descriptors", n_groups, DFB_MAX_GROUPS);
    return -1;
  }
  if (ldx < 1 || ldx > DFB_MAX_SLOTS) {
    set_error("score_groups: ldx = %d outside [1, %d]", ldx, DFB_MAX_SLOTS);
    return -1;
  }
  if (m < 0 || (m > 0 && (X_host == nullptr || group_host == nullptr || scores_host == nullptr))) {
    set_error("bad score_groups arguments (m = %lld)", (long long)m);
    return -1;
  }
  std::vector<int> slot_off(n_groups + 1, 0), fac_off(n_groups + 1, 0);
  for (int g = 0; g < n_groups; g++) {
    DFB_TRY(check_desc(&descs[g]));
    slot_off[g + 1] = slot_off[g] + descs[g].n_slots;
    fac_off[g + 1] = fac_off[g] + descs[g].n_factors;
  }
  if (slot_off[n_groups] > DFB_MAX_SLOTS || fac_off[n_groups] > DFB_MAX_FACTORS) {
    set_error("score_groups: the groups use %d slots and %d factors (at most %d and %d)", slot_off[n_groups],
              fac_off[n_groups], DFB_MAX_SLOTS, DFB_MAX_FACTORS);
    return -1;
  }
  for (int64_t r = 0; r < m; r++) {
    if (group_host[r] < 0 || group_host[r] >= n_groups) {
      set_error("score_groups: row %lld has group %d", (long long)r, group_host[r]);
      return -1;
    }
    if (descs[group_host[r]].cand_dim > ldx) {
      set_error("score_groups: group %d has %d columns, the rows %d", group_host[r], descs[group_host[r]].cand_dim, ldx);
      return -1;
    }
  }
  if (m == 0) return 0;
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_TRY(ensure_train_scaled(h));
  const int64_t npad = h->npad;
  DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_grp, descs, sizeof(dfb_kernel_desc) * n_groups, cudaMemcpyHostToDevice,
                              h->stream));
  h->te_prepped = false;
  for (int g = 0; g < n_groups; g++)
    DFB_TRY(launch_prep_scaled(h, h->d_desc_grp + g, 1, h->X, h->n, h->d, h->te.xs + slot_off[g] * npad,
                               h->te.nrm + fac_off[g] * npad, npad));

  // rows in group order (stable), packed
  std::vector<int64_t> order(m);
  for (int64_t r = 0; r < m; r++) order[r] = r;
  std::stable_sort(order.begin(), order.end(), [&](int64_t a, int64_t b) { return group_host[a] < group_host[b]; });
  const bool small = small_eval_fits(h);
  // a batch: as many whole passes as the staging buffer (chunk x DFB_MAX_SLOTS) and h->score (chunk) hold
  const int64_t batch = std::min(h->chunk, h->chunk * DFB_MAX_SLOTS / ldx) / SMALL_EVAL_M * SMALL_EVAL_M;
  std::vector<double> packed, sorted_scores(m);
  for (int64_t b0 = 0; b0 < m; b0 += batch) {
    const int64_t bm = std::min(batch, m - b0);
    packed.clear();
    std::vector<int64_t> col0(bm);                        // offset of each row's coordinates in `packed`
    for (int64_t i = 0; i < bm; i++) {
      const int64_t r = order[b0 + i];
      const int dc = descs[group_host[r]].cand_dim;
      col0[i] = (int64_t)packed.size();
      packed.insert(packed.end(), X_host + r * ldx, X_host + r * ldx + dc);
    }
    DFB_CUDA_OK(cudaMemcpyAsync(h->stage, packed.data(), sizeof(double) * packed.size(), cudaMemcpyHostToDevice,
                                h->stream));
    for (int64_t p0 = 0; p0 < bm; p0 += SMALL_EVAL_M) {
      const int64_t pm = std::min<int64_t>(SMALL_EVAL_M, bm - p0);
      // segments [s0, s1) of one group within the pass
      std::vector<int64_t> seg;
      for (int64_t i = 0; i < pm; i++)
        if (i == 0 || group_host[order[b0 + p0 + i]] != group_host[order[b0 + p0 + i - 1]]) seg.push_back(i);
      seg.push_back(pm);
      DFB_TRY(prof_begin(h, DFB_PROF_KSTAR));
      for (size_t s = 0; s + 1 < seg.size(); s++) {
        const int64_t s0 = seg[s], cnt = seg[s + 1] - s0;
        const int g = group_host[order[b0 + p0 + s0]];
        KstarArgs ka{};
        ka.desc = &descs[g]; ka.d_desc = h->d_desc_grp + g;
        ka.xsT = h->te.xs + slot_off[g] * npad; ka.nrmT = h->te.nrm + fac_off[g] * npad; ka.npad_tr = npad;
        ka.alpha = h->alpha; ka.Xc = h->stage + col0[p0 + s0]; ka.m = cnt; ka.dc = descs[g].cand_dim;
        ka.m_rows = (cnt + 1) / 2 * 2;                   // rows past cnt are overwritten by the next group's launch
        ka.n_valid = h->n; ka.n_write = npad; ka.Ks = h->Ks + s0 * npad; ka.ldk = npad; ka.mean_const = 0.0;
        ka.mu = h->mu + s0; ka.kss_out = h->kssv + s0; ka.cprep = h->cprep; ka.mu_part = h->mu_part;
        DFB_TRY(launch_kstar(h, ka, route_kstar(h, ka, KstarWant::ROWS)));
      }
      DFB_TRY(prof_end(h, DFB_PROF_KSTAR, (double)pm));
      DFB_TRY(prof_begin(h, DFB_PROF_GEMM));
      int n_part = (int)(npad / TILE);
      int64_t ld_part = h->chunk;
      if (small) {
        DFB_TRY(launch_small_sumsq(h, h->W, npad, h->Ks, npad, h->n, (int)pm, h->partial, SMALL_EVAL_M, &n_part));
        ld_part = SMALL_EVAL_M;
      } else {
        DFB_TRY(contract_tiles_f64(h, round_up(pm, TILE)));
      }
      DFB_TRY(prof_end(h, DFB_PROF_GEMM, (double)pm));
      DFB_TRY(prof_begin(h, DFB_PROF_ACQ));
      for (size_t s = 0; s + 1 < seg.size(); s++) {
        const int64_t s0 = seg[s], cnt = seg[s + 1] - s0;
        dfb_acq_desc acq;
        memset(&acq, 0, sizeof(acq));
        acq.kind = DFB_ACQ_UCB;
        acq.beta = betas[group_host[order[b0 + p0 + s0]]];
        DFB_TRY(launch_acq(h, acq, h->mu + s0, h->partial + s0, ld_part, n_part, h->kssv + s0, cnt, 0, 1, nullptr,
                           h->score + p0 + s0, false));
      }
      DFB_TRY(prof_end(h, DFB_PROF_ACQ, (double)pm));
    }
    DFB_CUDA_OK(cudaMemcpyAsync(sorted_scores.data() + b0, h->score, sizeof(double) * bm, cudaMemcpyDeviceToHost,
                                h->stream));
    DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  }
  for (int64_t i = 0; i < m; i++) scores_host[order[i]] = sorted_scores[i];
  return 0;
}

int dfb_mu_upper_bound(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space, double mean_const,
                       double* mu_ub_out) {
  DFB_TRY(need(h, true, true, true, true, false));
  if (m < 0 || (m > 0 && (Xc == nullptr || mu_ub_out == nullptr))) { set_error("bad mu_upper_bound arguments"); return -1; }
  if (h->have_test_kernel || !kstar_plain(h->desc_tr)) {
    set_error("dfb_mu_upper_bound: the bound pass serves plain SE / Matern kernels on <= 8 dims without a test kernel");
    return -1;
  }
  if (m == 0) return 0;
  DFB_CUDA_OK(cudaSetDevice(h->device));
  dfb_acq_desc acq;
  memset(&acq, 0, sizeof(acq));
  DFB_TRY(run_bound_pass(h, acq, Xc, m, dc, space, mean_const, 0.0, 0, nullptr, mu_ub_out));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dfb_debug_approx_error(dfb_handle* h, int32_t which, double* out_host) {
  DFB_TRY(need(h, true, false, false, false, false));
  if ((which != 0 && which != 1) || out_host == nullptr) { set_error("bad approx_error arguments"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  unsigned long long* bits = reinterpret_cast<unsigned long long*>(h->red);
  DFB_TRY(launch_approx_err(h, which, bits));
  unsigned long long v = 0;
  DFB_CUDA_OK(cudaMemcpyAsync(&v, bits, sizeof(v), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  memcpy(out_host, &v, sizeof(double));
  return 0;
}

// ---- bound pass of dfb_score_argmax ---------------------------------------------------------------------------------
// Most candidates of a large random batch cannot reach the arg-max, and proving so needs an upper bound of mu alone:
//   (1) ub = acq(mu_bar, sqrt(k**)) >= the fp64 score of the exact pass.  mu_bar (kernels.cu: prune_bound_kernel, in
//       single precision) is at least the fp64 mu of every K_* producer.  EI and UCB with beta >= 0 are
//       non-decreasing in mu and in sigma, PI is non-decreasing in mu and, for mu_bar < the incumbent (z < 0), in
//       sigma; the device's fp64 variance fl(k** - sum of partials) with every partial >= 0 is at most k** in floating
//       point as well.  The ulp-level non-monotonicity of the ndtr / erfc formulas is dwarfed by the shortlist's pad
//       (1e-9 of the score scale).
//   (2) best_lb <= the final fp64 maximum (argmax_merge_kernel: a maximum of certain lower bounds).
// So a candidate with ub < best_lb - pad has an fp64 score below the maximum: every candidate whose fp64 score equals
// the maximum, ties included, survives, the shortlist of the passes that follow contains all of them, and the fp64
// arg-max over it -- index and score -- is the one the full pass returns, bit for bit.
// (3) No dropped candidate can be a NaN winner (a negative fp64 variance gives a NaN score, and np.argmax takes the
//     first NaN): see bound_pass_applies.
// Order: (a) chunk 0 scored as today (collect mode) seeds best, best_lb and the shortlist; (b) the bound pass over
// rows chunk.. (run_bound_pass: one screen + gather per step) fills the survivor list; (c) one read-back of the
// survivor count; (d) the survivors are scored like any
// other chunk (collect mode, indices mapped back), continuing the arg-max of (a); the caller then re-scores the
// shortlist in fp64 and runs the self-check unchanged.  A survivor list that overflows (4 chunks) voids the screen:
// chunks 1.. are then scored as today, still continuing the seed's state.
static bool bound_pass_applies(const dfb_handle* h, const dfb_acq_desc& acq, const dfb_kernel_desc& desc, int64_t m,
                               int32_t dc, double b2) {
  if (!h->prune || h->have_test_kernel || m <= h->chunk || dc > PRUNE_MAX_DC || !kstar_plain(desc)) return false;
  if (!(acq.kind == DFB_ACQ_EI || acq.kind == DFB_ACQ_PI || (acq.kind == DFB_ACQ_UCB && acq.beta >= 0.0))) return false;
  // Variance floor.  K: the noiseless training kernel matrix, s: the diagonal actually added (noise + jitter, for every
  // point, hallucinated ones included), k = K(X, x*).  The joint covariance [[K, k], [k^T, k**]] is PSD, so
  // k^T K^+ k <= k**, and in the eigenbasis of K (c_i = u_i^T k, eigenvalues l_i <= l_max <= tr K = n k(x, x)):
  //   k^T (K + s I)^-1 k = sum_i (c_i^2 / l_i) l_i / (l_i + s) <= k** l_max / (l_max + s)
  //   sigma^2 = k** - k^T (K + s I)^-1 k >= k** s / (l_max + s) >= k** s / (tr K + s).
  // Screening is allowed only when this floor exceeds both the int8 error bound b2 and n eps k** (a worst-case bound
  // on the fp64 contraction's own rounding): then no candidate's fp64 variance is negative.  At the headline
  // (N = 5000) the floor is ~3e-7 against b2 ~ 3e-9.
  const double s = h->noise_plus_jitter, kss = desc.kss;
  const double floor = kss * s / ((double)h->n * kss + s);
  return floor > b2 && floor > (double)h->n * DBL_EPSILON * kss;
}

static int run_chunks_pruned(dfb_handle* h, const dfb_acq_desc& acq, const double* Xc, int64_t m, int32_t dc,
                             int32_t space, double mean_const, const ChunkMode& md) {
  const int64_t Mc = h->chunk;
  const ChunkOut none = {nullptr, nullptr, nullptr};
  const double* rest = Xc + Mc * dc;
  DFB_TRY(run_chunks(h, acq, Xc, Mc, dc, space, mean_const, none, md));                 // (a)
  DFB_CUDA_OK(cudaMemsetAsync(h->surv_count, 0, sizeof(int), h->stream));
  DFB_TRY(run_bound_pass(h, acq, rest, m - Mc, dc, space, mean_const, md.pad, Mc, h->list_count, nullptr));  // (b)
  int surv = 0;
  DFB_CUDA_OK(cudaMemcpyAsync(&surv, h->surv_count, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));                                        // (c)
  h->last_survivors = surv;
  ChunkMode cont = md;
  cont.keep_best = true;
  if (surv > h->surv_cap) {                         // overflow: every candidate of chunks 1.. is contracted
    h->last_pruned = 0;
    cont.idx_base = Mc;
    return run_chunks(h, acq, rest, m - Mc, dc, space, mean_const, none, cont);
  }
  h->last_pruned = m - Mc - surv;
  if (surv == 0) return 0;
  cont.idx_map = h->surv_idx;
  return run_chunks(h, acq, h->surv_X, surv, dc, DFB_DEVICE, mean_const, none, cont);   // (d)
}

// The running arg-max (score, index) of the handle, read back
static int read_best(dfb_handle* h, double* best_score_host, int64_t* best_index_host) {
  double bs = 0.0; int64_t bi = -1;
  DFB_CUDA_OK(cudaMemcpyAsync(&bs, h->best_score, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(&bi, h->best_index, sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  if (best_score_host) *best_score_host = bs;
  if (best_index_host) *best_index_host = bi;
  return 0;
}

// The body of dfb_score_argmax and dfb_score_argmax_ts.  base: the normals of DFB_ACQ_TS_MARGINAL (ChunkMode::ts_*),
// else default.  TS: every fp64 pass starts h->ts_nonpos from 0, so it ends holding the count of the pass that decided.
static int score_argmax_impl(dfb_handle* h, const dfb_acq_desc* acq, const double* Xc, int64_t m, int32_t dc,
                             int32_t space, double mean_const, double* scores, double* best_score_host,
                             int64_t* best_index_host, const ChunkMode& base) {
  const bool want_std = (acq->kind != DFB_ACQ_MEAN);
  const bool ts = acq->kind == DFB_ACQ_TS_MARGINAL;
  ChunkOut out = {nullptr, nullptr, scores};
  const dfb_kernel_desc& desc = active_kernel(h).desc;
  // A caller that asks for the full score vector gets fp64 scores (parity use); the shortlist scheme
  // only guarantees the arg-max, so the int8 pass is reserved for arg-max-only calls unless forced.
  const bool fast = want_std && h->score_impl != 0 && i8_usable(h, desc) &&
                    (scores == nullptr || h->score_impl == 1);
  ChunkMode exact = base;                // the fp64 arg-max
  exact.want_std = want_std; exact.do_argmax = true;
  ChunkMode md = exact;
  md.use_i8 = fast;
  h->last_used_i8 = fast ? 1 : 0;
  h->last_shortlist = 0;
  h->last_selfcheck_violations = 0;
  h->last_selfcheck_ratio = 0.0;
  h->last_survivors = 0;
  h->last_pruned = 0;
  bool need_exact_pass = !fast;
  if (fast) {
    // Pass 1: int8-slice scoring of everything, collecting the shortlist of candidates whose fp64 score could be
    // the maximum under the error model (kernels.cu: i8_score_err / collect_shortlist_kernel).  The pass is void
    // -- and its remaining launches return at once -- as soon as the shortlist overflows (masses of exact ties).
    const double sk = sqrt(desc.kss);
    double scale = sk;                    // natural score scale, for the slack only
    if (acq->kind == DFB_ACQ_UCB) scale = (1.0 + fabs(acq->beta)) * sk + fabs(mean_const);
    else if (acq->kind == DFB_ACQ_PI) scale = 1.0;
    else if (ts) scale = 9.0 * sk + fabs(mean_const);     // UCB's with |z| <= 8 (Box-Muller's on 53-bit uniforms: 8.6)
    md.collect = true;
    md.em.b2 = i8_sigma2_bound(h, desc);
    md.em.kind = acq->kind;
    md.em.sens = (acq->kind == DFB_ACQ_UCB) ? fabs(acq->beta) : (acq->kind == DFB_ACQ_PI ? 0.25 : 0.4);   // TS: |z_i|
    md.pad = 1e-9 * scale;
    DFB_CUDA_OK(cudaMemsetAsync(h->list_count, 0, sizeof(int) * 4, h->stream));
    if (scores == nullptr && bound_pass_applies(h, *acq, desc, m, dc, md.em.b2))
      DFB_TRY(run_chunks_pruned(h, *acq, Xc, m, dc, space, mean_const, md));
    else
      DFB_TRY(run_chunks(h, *acq, Xc, m, dc, space, mean_const, out, md));
    int count = 0;
    DFB_CUDA_OK(cudaMemcpyAsync(&count, h->list_count, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
    if (count > SHORTLIST_CAP || count > h->chunk) {
      h->last_shortlist = -1;          // too many candidates within reach of the maximum: exact pass over everything
      need_exact_pass = true;
    } else {
      // Pass 2: exact fp64 (DMMA) re-score of the shortlist; indices map back to the caller's rows.  Then the
      // self-check: int8 vs fp64 score of every listed candidate against its allowance.
      h->last_shortlist = count;
      ChunkMode ex = exact;
      ex.idx_map = h->list_idx; ex.keep_scores = true;
      if (ts) {
        ex.ts_z = h->list_z;                         // the normals of the first pass
        DFB_CUDA_OK(cudaMemsetAsync(h->ts_nonpos, 0, sizeof(int), h->stream));
      }
      ChunkOut none = {nullptr, nullptr, nullptr};
      DFB_TRY(run_chunks(h, *acq, h->list_X, count, dc, DFB_DEVICE, mean_const, none, ex));
      DFB_TRY(launch_selfcheck(h, h->score, count));
      int chk[2] = {0, 0};
      DFB_CUDA_OK(cudaMemcpyAsync(chk, h->list_count + 1, sizeof(chk), cudaMemcpyDeviceToHost, h->stream));
      DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
      h->last_selfcheck_violations = chk[0];
      h->last_selfcheck_ratio = (double)chk[1] * 1e-6;
      if (chk[0] > 0) need_exact_pass = true;      // the error model failed on a candidate that matters: fp64
    }
  }
  if (need_exact_pass) {
    if (ts) DFB_CUDA_OK(cudaMemsetAsync(h->ts_nonpos, 0, sizeof(int), h->stream));
    DFB_TRY(run_chunks(h, *acq, Xc, m, dc, space, mean_const, out, exact));
  }
  return read_best(h, best_score_host, best_index_host);
}

int dfb_score_argmax(dfb_handle* h, const dfb_acq_desc* acq, const double* Xc, int64_t m, int32_t dc,
                     int32_t space, double mean_const, double* scores, double* best_score_host,
                     int64_t* best_index_host) {
  if (acq == nullptr) { set_error("acq is NULL"); return -1; }
  const bool want_std = (acq->kind != DFB_ACQ_MEAN);
  DFB_TRY(need(h, true, true, true, true, want_std));
  if (m < 1 || Xc == nullptr) { set_error("bad score arguments (m = %lld)", (long long)m); return -1; }
  if (acq->kind < DFB_ACQ_MEAN || acq->kind > DFB_ACQ_TTEI) { set_error("unknown acquisition kind %d", acq->kind); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  return score_argmax_impl(h, acq, Xc, m, dc, space, mean_const, scores, best_score_host, best_index_host, ChunkMode());
}

int dfb_score_argmax_ts(dfb_handle* h, const double* Xc, int64_t m, int32_t dc, int32_t space, double mean_const,
                        const double* z, uint64_t seed, int64_t row0, double* scores, double* best_score_host,
                        int64_t* best_index_host, int64_t* n_nonpos_host) {
  DFB_TRY(need(h, true, true, true, true, true));
  if (m < 1 || Xc == nullptr || row0 < 0 || (space != DFB_HOST && space != DFB_DEVICE)) {
    set_error("bad score_ts arguments (m = %lld, row0 = %lld)", (long long)m, (long long)row0);
    return -1;
  }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  dfb_acq_desc acq;
  memset(&acq, 0, sizeof(acq));
  acq.kind = DFB_ACQ_TS_MARGINAL;
  ChunkMode base;
  base.ts_z = z; base.ts_seed = seed; base.ts_row0 = row0;
  DFB_TRY(score_argmax_impl(h, &acq, Xc, m, dc, space, mean_const, scores, best_score_host, best_index_host, base));
  if (n_nonpos_host != nullptr) {
    int nonpos = 0;
    DFB_CUDA_OK(cudaMemcpyAsync(&nonpos, h->ts_nonpos, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
    *n_nonpos_host = nonpos;
  }
  return 0;
}

int dfb_moo_score_argmax(dfb_handle* h, const dfb_moo_desc* desc, const double* const* a_dev,
                         const double* const* b_dev, int64_t m, double* scores_dev,
                         double* best_score_host, int64_t* best_index_host) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (desc == nullptr || a_dev == nullptr || m < 1) { set_error("bad moo arguments (m = %lld)", (long long)m); return -1; }
  if (desc->kind < DFB_MOO_LIN_UCB || desc->kind > DFB_MOO_TCH_VAL) { set_error("unknown scalarisation kind %d", desc->kind); return -1; }
  if (desc->n_obj < 1 || desc->n_obj > DFB_MOO_MAX_OBJ) { set_error("n_obj = %d outside [1, %d]", desc->n_obj, DFB_MOO_MAX_OBJ); return -1; }
  const bool ucb = desc->kind == DFB_MOO_LIN_UCB || desc->kind == DFB_MOO_TCH_UCB;
  for (int k = 0; k < desc->n_obj; k++)
    if (a_dev[k] == nullptr || (ucb && (b_dev == nullptr || b_dev[k] == nullptr))) { set_error("objective %d: NULL vector", k); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_TRY(launch_reset_best(h));
  DFB_TRY(launch_moo(h, *desc, a_dev, ucb ? b_dev : nullptr, m, scores_dev));
  return read_best(h, best_score_host, best_index_host);
}

int dfb_moo_score_argmax_ts(dfb_handle* h, const dfb_moo_desc* desc, const double* const* mu_dev,
                            const double* const* sd_dev, int64_t m, const double* z_dev, uint64_t seed,
                            int64_t row0, double* scores_dev, double* best_score_host,
                            int64_t* best_index_host, int64_t* n_nonpos_host) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (desc == nullptr || mu_dev == nullptr || sd_dev == nullptr || m < 1 || row0 < 0) {
    set_error("bad moo_ts arguments (m = %lld, row0 = %lld)", (long long)m, (long long)row0);
    return -1;
  }
  if (desc->kind != DFB_MOO_LIN_VAL && desc->kind != DFB_MOO_TCH_VAL) { set_error("scalarisation kind %d is not a VAL kind", desc->kind); return -1; }
  if (desc->n_obj < 1 || desc->n_obj > DFB_MOO_MAX_OBJ) { set_error("n_obj = %d outside [1, %d]", desc->n_obj, DFB_MOO_MAX_OBJ); return -1; }
  for (int k = 0; k < desc->n_obj; k++)
    if (mu_dev[k] == nullptr || sd_dev[k] == nullptr) { set_error("objective %d: NULL vector", k); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_TRY(launch_reset_best(h));
  DFB_CUDA_OK(cudaMemsetAsync(h->ts_nonpos, 0, sizeof(int), h->stream));
  TsZ tz;
  memset(&tz, 0, sizeof(tz));
  tz.z = z_dev; tz.seed = seed; tz.row0 = row0; tz.nonpos = h->ts_nonpos;
  DFB_TRY(launch_moo(h, *desc, mu_dev, sd_dev, m, scores_dev, &tz));
  if (n_nonpos_host != nullptr) {
    int nonpos = 0;
    DFB_CUDA_OK(cudaMemcpyAsync(&nonpos, h->ts_nonpos, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
    *n_nonpos_host = nonpos;
  }
  return read_best(h, best_score_host, best_index_host);
}

int dfb_ga_maximise(dfb_handle* h, const dfb_acq_desc* acq, double mean_const, const dfb_ga_desc* desc, uint64_t seed,
                    int64_t n_init, int64_t n_total, double* rows_dev, double* vals_dev, double* coded_dev,
                    double* best_value_host, int64_t* best_index_host, double* best_row_host) {
  DFB_TRY(need(h, true, true, true, true, true));
  if (acq == nullptr || desc == nullptr || rows_dev == nullptr || vals_dev == nullptr || coded_dev == nullptr) {
    set_error("ga_maximise: NULL argument"); return -1;
  }
  if (acq->kind < DFB_ACQ_UCB || acq->kind > DFB_ACQ_TTEI) { set_error("ga_maximise: acquisition kind %d", acq->kind); return -1; }
  const dfb_ga_desc& g = *desc;
  if (g.d < 1 || g.d > DFB_GA_MAX_COLS || g.n_parts < 1 || g.n_parts > DFB_GA_MAX_PARTS || n_init < 1 ||
      n_total < n_init) {
    set_error("bad ga_maximise arguments (d = %d, parts = %d, n_init = %lld, n_total = %lld)", g.d, g.n_parts,
              (long long)n_init, (long long)n_total);
    return -1;
  }
  int next = 0;
  for (int p = 0; p < g.n_parts; p++) {
    const int c0 = g.part_c0[p], c1 = g.part_c1[p], kind = g.part_kind[p];
    if (c0 != next || c1 <= c0 || c1 > g.d || kind < DFB_GA_PART_REAL || kind > DFB_GA_PART_NUMERIC) {
      set_error("ga_maximise: bad part %d", p); return -1;
    }
    next = c1;
    for (int c = c0; c < c1; c++) {
      const bool cat = kind >= DFB_GA_PART_CATEGORICAL;
      if (g.kind[c] != (cat ? DFB_CAND_CATEGORICAL : (kind == DFB_GA_PART_REAL ? DFB_CAND_REAL : DFB_CAND_INTEGER)) ||
          (!cat && !(g.lo[c] <= g.hi[c])) ||
          (cat && (g.n_levels[c] < (kind == DFB_GA_PART_CATEGORICAL ? 2 : 1) || g.lut_off[c] < 0 ||
                   g.lut_off[c] + g.n_levels[c] > DFB_GA_MAX_LUT)) ||
          (kind == DFB_GA_PART_NUMERIC && (g.val_off[c] < 0 || g.val_off[c] + g.n_levels[c] > DFB_GA_MAX_LUT))) {
        set_error("ga_maximise: bad column %d of part %d", c, p); return -1;
      }
    }
  }
  if (next != g.d) { set_error("ga_maximise: the parts cover %d of %d columns", next, g.d); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  int64_t n_levels[DFB_GA_MAX_COLS];
  for (int c = 0; c < g.d; c++) n_levels[c] = g.kind[c] == DFB_CAND_CATEGORICAL ? g.n_levels[c] : 0;
  ChunkMode md;
  md.want_std = true;
  md.allow_small = h->small_eval != 0;
  // the initial pool
  DFB_TRY(launch_fill_mixed_candidates(h, seed, 0, n_init, g.d, g.kind, g.lo, g.hi, n_levels, rows_dev));
  DFB_TRY(launch_ga_encode(h, g, rows_dev, n_init, coded_dev));
  ChunkOut out = {nullptr, nullptr, vals_dev};
  DFB_TRY(run_chunks(h, *acq, coded_dev, n_init, g.d, DFB_DEVICE, mean_const, out, md));
  // epochs: no launch waits on the host
  for (int64_t r0 = n_init; r0 < n_total; r0 += 5) {
    const int c = (int)std::min<int64_t>(5, n_total - r0);
    DFB_TRY(launch_ga_epoch(h, g, seed, r0, c, rows_dev, vals_dev, coded_dev));
    ChunkOut oe = {nullptr, nullptr, vals_dev + r0};
    DFB_TRY(run_chunks(h, *acq, coded_dev, c, g.d, DFB_DEVICE, mean_const, oe, md));
  }
  DFB_TRY(launch_ga_best(h, g, rows_dev, vals_dev, n_total, coded_dev));
  double res[2 + DFB_GA_MAX_COLS];
  DFB_CUDA_OK(cudaMemcpyAsync(res, coded_dev, sizeof(double) * (2 + g.d), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  if (best_value_host) *best_value_host = res[0];
  if (best_index_host) *best_index_host = (int64_t)res[1];
  if (best_row_host) for (int c = 0; c < g.d; c++) best_row_host[c] = res[2 + c];
  return 0;
}

int dfb_kernel_matrix(dfb_handle* h, const dfb_kernel_desc* desc, const double* X1_dev, int64_t n1,
                      int32_t d1, const double* X2_dev, int64_t n2, int32_t d2, double* K_dev) {
  DFB_TRY(need(h, true, false, false, false, false));
  DFB_TRY(check_desc(desc));
  if (n1 < 1 || n2 < 1 || X1_dev == nullptr || X2_dev == nullptr || K_dev == nullptr) { set_error("bad kernel_matrix arguments"); return -1; }
  if (d1 != d2 || d1 != desc->train_dim) { set_error("kernel_matrix: dims %d, %d vs kernel train_dim %d", d1, d2, desc->train_dim); return -1; }
  const int64_t np2 = round_up(n2, TILE);
  if (np2 > h->npad_max) { set_error("kernel_matrix: n2 = %lld exceeds the workspace (n_max = %lld)", (long long)n2, (long long)h->n_max); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  h->desc_tmp = *desc;
  DFB_CUDA_OK(cudaMemcpyAsync(h->d_desc_tmp, &h->desc_tmp, sizeof(dfb_kernel_desc), cudaMemcpyHostToDevice, h->stream));
  h->te_prepped = false;   // the test-kernel scaled set is used as scratch
  DFB_TRY(launch_prep_scaled(h, h->d_desc_tmp, 1, X2_dev, n2, d2, h->te.xs, h->te.nrm, np2));
  KstarArgs ka{};
  ka.desc = &h->desc_tmp; ka.d_desc = h->d_desc_tmp; ka.cand_uses_train_coords = 1;
  ka.xsT = h->te.xs; ka.nrmT = h->te.nrm; ka.npad_tr = np2; ka.Xc = X1_dev; ka.m = n1; ka.dc = d1; ka.m_rows = n1;
  ka.n_valid = n2; ka.n_write = n2; ka.Ks = K_dev; ka.ldk = n2;
  DFB_TRY(launch_kstar(h, ka, route_kstar(h, ka, KstarWant::ROWS)));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

// The buffers one posterior covariance is formed in: the block workspace's (ts_*, m <= its mb and the chunk) or the
// joint workspace's (js_*, every candidate at once).
struct CovBufs {
  double* Vt; double* cxs; double* cnrm; double* Cov; double* mu;
  bool joint;
};

// Block form when the TS workspace holds the m candidates within one scoring chunk, else the joint form when the joint
// workspace holds them, else an error.  A caller that sets both picks the form by which workspace can hold m.
static int cov_bufs(dfb_handle* h, int64_t m, CovBufs* b) {
  const int64_t mbp = round_up(m, TILE);
  if (m < 1) { set_error("posterior covariance of %lld candidates", (long long)m); return -1; }
  if (h->ts_ws != nullptr && mbp <= h->ts_mb && mbp <= h->chunk) {
    *b = CovBufs{h->ts_Vt, h->ts_cxs, h->ts_cnrm, h->ts_Cov, h->ts_mu, false};
    return 0;
  }
  if (h->js_ws != nullptr && mbp <= h->js_mb) {
    *b = CovBufs{h->js_Vt, h->js_cxs, h->js_cnrm, h->js_Cov, h->js_mu, true};
    return 0;
  }
  if (h->ts_ws == nullptr && h->js_ws == nullptr) {
    set_error("no Thompson-sampling workspace: call dfb_set_ts_workspace or dfb_set_joint_workspace first");
    return -1;
  }
  set_error("%lld candidates exceed the TS workspace (%lld) / chunk (%lld) and the joint workspace (%lld)",
            (long long)m, (long long)h->ts_mb, (long long)h->chunk, (long long)h->js_mb);
  return -1;
}

// mu and the padded posterior covariance (b.Cov, ld = mbp) of m candidates:
// K_* -> V^T = K_* W^T -> Cov = K** - V^T V    (gp_core.py:173-181)
// K_* and K** are formed in row slabs of at most one scoring chunk (the K_* buffer and the candidate staging hold one
// chunk); a block (mbp <= chunk) is one slab.  Every tile of Cov is one DMMA contraction of depth npad over the same
// V^T rows whatever the slab and the grid, so the leading q x q of a joint covariance is bit for bit the covariance of
// its first q candidates.
static int posterior_covariance(dfb_handle* h, const CovBufs& b, const double* Xc_dev, int64_t m, int32_t dc,
                                double mean_const, int64_t* mbp_out, bool lower_only) {
  const ActiveKernel k = active_kernel(h);
  if (dc != k.desc.cand_dim) { set_error("candidates have %d columns, the kernel descriptor expects %d", dc, k.desc.cand_dim); return -1; }
  const int64_t mbp = round_up(m, TILE);
  DFB_TRY(ensure_train_scaled(h));
  DFB_TRY(ensure_test_scaled(h));
  const int64_t npad = h->npad;
  const int nb = (int)(npad / TILE), mbb = (int)(mbp / TILE);
  KstarArgs ka{};
  GemmArgs g;
  for (int64_t r0 = 0; r0 < mbp; r0 += h->chunk) {
    const int64_t rows = std::min(h->chunk, mbp - r0);
    // K_* rows (zero rows beyond m) and mu
    ka = KstarArgs{};
    ka.desc = &k.desc; ka.d_desc = k.d_desc; ka.xsT = k.ss.xs; ka.nrmT = k.ss.nrm; ka.npad_tr = npad; ka.alpha = h->alpha;
    ka.Xc = Xc_dev + r0 * dc; ka.m = std::min(m - r0, rows); ka.dc = dc; ka.m_rows = rows; ka.n_valid = h->n;
    ka.n_write = npad; ka.Ks = h->Ks; ka.ldk = npad;
    ka.mean_const = mean_const; ka.mu = b.mu + r0; ka.cprep = h->cprep; ka.mu_part = h->mu_part;
    DFB_TRY(launch_kstar(h, ka, route_kstar(h, ka, KstarWant::ROWS)));
    // V^T[a][i] = sum_{k <= i} K_*[a][k] W[i][k]
    memset(&g, 0, sizeof(g));
    g.A = h->Ks; g.lda = npad; g.B = h->W; g.ldb = npad; g.D = b.Vt + r0 * npad; g.ldd = npad; g.alpha = 1.0;
    g.mode = MODE_GENERIC; g.n_rb = (int)(rows / TILE); g.n_cb = nb; g.K = (int)npad; g.tri = 2;
    DFB_TRY(launch_gemm(h, g, EPI_STORE, g.n_rb * nb));
  }
  // K** = kernel(X_test, X_test) (gp_core.py:179) with the candidates as both sides
  DFB_TRY(launch_prep_scaled(h, k.d_desc, 0, Xc_dev, m, dc, b.cxs, b.cnrm, mbp));
  for (int64_t r0 = 0; r0 < mbp; r0 += h->chunk) {
    const int64_t rows = std::min(h->chunk, mbp - r0);
    ka.Xc = Xc_dev + r0 * dc; ka.m = std::min(m - r0, rows); ka.m_rows = rows;
    ka.xsT = b.cxs; ka.nrmT = b.cnrm; ka.npad_tr = mbp; ka.alpha = nullptr; ka.n_valid = m; ka.n_write = mbp;
    ka.Ks = b.Cov + r0 * mbp; ka.ldk = mbp; ka.mean_const = 0.0; ka.mu = nullptr;
    DFB_TRY(launch_kstar(h, ka, route_kstar(h, ka, KstarWant::ROWS)));
  }
  // Cov = K** - V^T V
  memset(&g, 0, sizeof(g));
  g.A = b.Vt; g.lda = npad; g.B = b.Vt; g.ldb = npad; g.C = b.Cov; g.ldc = mbp;
  g.D = b.Cov; g.ldd = mbp; g.alpha = -1.0; g.mode = MODE_GENERIC; g.n_rb = mbb; g.n_cb = mbb;
  g.K = (int)npad;
  g.lower_only = lower_only ? 1 : 0;     // the factorisation that follows reads the lower triangle only
  DFB_TRY(launch_gemm(h, g, EPI_STORE, mbb * mbb));
  *mbp_out = mbp;
  return 0;
}

size_t dfb_ts_workspace_bytes(int64_t n_max, int64_t mb) { return carve_ts(nullptr, nullptr, n_max, mb); }

int dfb_set_ts_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t mb) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (workspace_dev == nullptr || mb < 1) { set_error("bad TS workspace arguments"); return -1; }
  const size_t want = carve_ts(nullptr, nullptr, h->n_max, mb);
  if (bytes < want) { set_error("TS workspace too small: %zu bytes given, %zu needed", bytes, want); return -1; }
  if ((reinterpret_cast<uintptr_t>(workspace_dev) & 255) != 0) { set_error("TS workspace must be 256-byte aligned"); return -1; }
  h->ts_ws = static_cast<char*>(workspace_dev);
  carve_ts(h, h->ts_ws, h->n_max, mb);
  return 0;
}

size_t dfb_joint_workspace_bytes(int64_t n_max, int64_t m) { return carve_joint(nullptr, nullptr, n_max, m); }

int dfb_set_joint_workspace(dfb_handle* h, void* workspace_dev, size_t bytes, int64_t m) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (workspace_dev == nullptr || m < 1) { set_error("bad joint workspace arguments"); return -1; }
  const size_t want = carve_joint(nullptr, nullptr, h->n_max, m);
  if (bytes < want) { set_error("joint workspace too small: %zu bytes given, %zu needed", bytes, want); return -1; }
  if ((reinterpret_cast<uintptr_t>(workspace_dev) & 255) != 0) { set_error("joint workspace must be 256-byte aligned"); return -1; }
  h->js_ws = static_cast<char*>(workspace_dev);
  carve_joint(h, h->js_ws, h->n_max, m);
  return 0;
}

int dfb_eval_covar(dfb_handle* h, const double* Xc_dev, int64_t m, int32_t dc, double mean_const,
                   double* mu_dev, double* covar_dev) {
  DFB_TRY(need(h, true, true, true, true, true));
  if (Xc_dev == nullptr || mu_dev == nullptr || covar_dev == nullptr) { set_error("bad eval_covar arguments"); return -1; }
  CovBufs b;
  DFB_TRY(cov_bufs(h, m, &b));
  DFB_CUDA_OK(cudaSetDevice(h->device));
  int64_t mbp = 0;
  DFB_TRY(posterior_covariance(h, b, Xc_dev, m, dc, mean_const, &mbp, false));
  DFB_TRY(launch_copy_pad(h, b.mu, m, mu_dev, m));
  DFB_TRY(launch_copy_rows(h, b.Cov, mbp, covar_dev, m, m, m));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

// The joint draw: Cov + jitter I (identity padding) factorised in place by the factor-only mode, then samples^T = L U
// in passes of <= 256 draws over the one factor.
static int joint_draws(dfb_handle* h, const CovBufs& b, const double* Xc_dev, int64_t m, int32_t dc, double mean_const,
                       const double* Ut_dev, int32_t S, double jitter, double* samples_dev, int64_t* mbp_out) {
  int64_t mbp = 0;
  DFB_TRY(prof_begin(h, DFB_PROF_TS_COV));
  DFB_TRY(posterior_covariance(h, b, Xc_dev, m, dc, mean_const, &mbp, true));
  DFB_TRY(prof_end(h, DFB_PROF_TS_COV, 1.0));
  DFB_TRY(launch_diag_max(h, b.Cov, mbp, m, h->js_red));
  DFB_CUDA_OK(cudaMemsetAsync(h->js_info, 0, sizeof(int) * 4, h->stream));
  DFB_TRY(launch_set_diag(h, b.Cov, mbp, 0, m, jitter, 1));
  DFB_TRY(launch_set_diag(h, b.Cov, mbp, m, mbp, 1.0, 0));
  DFB_TRY(prof_begin(h, DFB_PROF_TS_FACTOR));
  DFB_TRY(factorise_tall(h, b.Cov, mbp, h->Dinv, h->js_info, false, false, true));
  DFB_TRY(prof_end(h, DFB_PROF_TS_FACTOR, 1.0));
  DFB_TRY(prof_begin(h, DFB_PROF_TS_PRODUCT));
  for (int32_t s0 = 0; s0 < S; s0 += 256) {
    const int32_t s = std::min(256, S - s0);
    const int64_t Sp = round_up(s, TILE);
    DFB_CUDA_OK(cudaMemsetAsync(h->js_Ut, 0, sizeof(double) * (size_t)Sp * mbp, h->stream));
    DFB_TRY(launch_copy_rows(h, Ut_dev + (int64_t)s0 * m, m, h->js_Ut, mbp, s, m));
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.A = h->js_Ut; g.lda = mbp; g.B = b.Cov; g.ldb = mbp; g.D = h->js_Sm; g.ldd = mbp; g.alpha = 1.0;
    g.mode = MODE_GENERIC; g.n_rb = (int)(Sp / TILE); g.n_cb = (int)(mbp / TILE); g.K = (int)mbp; g.tri = 2;
    g.info = h->js_info;
    DFB_TRY(launch_gemm(h, g, EPI_STORE, g.n_rb * g.n_cb));
    DFB_TRY(launch_add_row_vector(h, h->js_Sm, mbp, s, m, b.mu));
    DFB_TRY(launch_copy_rows(h, h->js_Sm, mbp, samples_dev + (int64_t)s0 * m, m, s, m));
  }
  DFB_TRY(prof_end(h, DFB_PROF_TS_PRODUCT, 1.0));
  *mbp_out = mbp;
  return 0;
}

int dfb_ts_draws(dfb_handle* h, const double* Xc_dev, int64_t m, int32_t dc, double mean_const,
                 const double* Ut_dev, int32_t S, double jitter, double* samples_dev, double* mu_dev,
                 double* max_diag_host) {
  DFB_TRY(need(h, true, true, true, true, true));
  if (Xc_dev == nullptr || Ut_dev == nullptr || samples_dev == nullptr || S < 1) { set_error("bad ts_draws arguments"); return -1; }
  CovBufs b;
  DFB_TRY(cov_bufs(h, m, &b));
  if (!b.joint && S > 256) { set_error("bad ts_draws arguments (a block takes 1 <= S <= 256)"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  int64_t mbp = 0;
  const double* red = h->ts_red;
  const int* dinfo = h->ts_info;
  if (b.joint) {
    DFB_TRY(joint_draws(h, b, Xc_dev, m, dc, mean_const, Ut_dev, S, jitter, samples_dev, &mbp));
    red = h->js_red; dinfo = h->js_info;
  } else {
    DFB_TRY(posterior_covariance(h, b, Xc_dev, m, dc, mean_const, &mbp, true));
    DFB_TRY(launch_diag_max(h, h->ts_Cov, mbp, m, h->ts_red));
    // stable_cholesky(K) (general_utils.py:224-229): factorise Cov + jitter I (identity padding)
    DFB_CUDA_OK(cudaMemsetAsync(h->ts_info, 0, sizeof(int) * 4, h->stream));
    DFB_CUDA_OK(cudaMemsetAsync(h->ts_T, 0, sizeof(double) * (size_t)(2 * mbp + TILE) * mbp, h->stream));
    DFB_TRY(launch_copy_rows(h, h->ts_Cov, mbp, h->ts_T, mbp, mbp, mbp));
    DFB_TRY(launch_set_diag(h, h->ts_T, mbp, 0, m, jitter, 1));
    DFB_TRY(launch_set_diag(h, h->ts_T, mbp, m, mbp, 1.0, 0));
    DFB_TRY(factorise_tall(h, h->ts_T, mbp, h->Dinv, h->ts_info, false, false));
    // samples^T = L_post U: samples[s][a] = sum_{b <= a} U^T[s][b] L[a][b]
    const int64_t Sp = round_up(S, TILE);
    DFB_CUDA_OK(cudaMemsetAsync(h->ts_Ut, 0, sizeof(double) * (size_t)Sp * mbp, h->stream));
    DFB_TRY(launch_copy_rows(h, Ut_dev, m, h->ts_Ut, mbp, S, m));
    GemmArgs g;
    memset(&g, 0, sizeof(g));
    g.A = h->ts_Ut; g.lda = mbp; g.B = h->ts_T; g.ldb = mbp; g.D = h->ts_Sm; g.ldd = mbp; g.alpha = 1.0;
    g.mode = MODE_GENERIC; g.n_rb = (int)(Sp / TILE); g.n_cb = (int)(mbp / TILE); g.K = (int)mbp; g.tri = 2;
    g.info = h->ts_info;
    DFB_TRY(launch_gemm(h, g, EPI_STORE, g.n_rb * g.n_cb));
    DFB_TRY(launch_add_row_vector(h, h->ts_Sm, mbp, S, m, h->ts_mu));
    DFB_TRY(launch_copy_rows(h, h->ts_Sm, mbp, samples_dev, m, S, m));
  }
  if (mu_dev != nullptr) DFB_TRY(launch_copy_pad(h, b.mu, m, mu_dev, m));
  double mx = 0.0;
  int info = 0;
  DFB_CUDA_OK(cudaMemcpyAsync(&mx, red, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaMemcpyAsync(&info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  if (max_diag_host != nullptr) *max_diag_host = mx;
  if (info != 0) { set_error("posterior covariance is not positive definite at jitter %g (pivot %d)", jitter, info - 1); return info; }
  return 0;
}

int dfb_fill_rng(dfb_handle* h, uint64_t seed, int64_t col0, int32_t S, int64_t m, int32_t what, double* out_dev) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (out_dev == nullptr || S < 1 || m < 1 || col0 < 0 || (what != DFB_RNG_NORMAL && what != DFB_RNG_UNIFORM)) { set_error("bad fill_rng arguments"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  return launch_fill_rng(h, seed, col0, S, m, what, out_dev);
}

int dfb_fill_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int32_t d, const double* lo_host,
                        const double* hi_host, double* out_dev) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (out_dev == nullptr || lo_host == nullptr || hi_host == nullptr || m < 1 || row0 < 0 || d < 1 || d > DFB_MAX_SLOTS) {
    set_error("bad fill_candidates arguments (m = %lld, d = %d)", (long long)m, d);
    return -1;
  }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  return launch_fill_candidates(h, seed, row0, m, d, lo_host, hi_host, out_dev);
}

int dfb_fill_mixed_candidates(dfb_handle* h, uint64_t seed, int64_t row0, int64_t m, int32_t d, const int32_t* kinds_host,
                              const double* lo_host, const double* hi_host, const int64_t* n_levels_host, double* out_dev) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (out_dev == nullptr || kinds_host == nullptr || lo_host == nullptr || hi_host == nullptr || m < 1 || row0 < 0 ||
      d < 1 || d > DFB_MAX_SLOTS) {
    set_error("bad fill_mixed_candidates arguments (m = %lld, d = %d)", (long long)m, d);
    return -1;
  }
  for (int s = 0; s < d; s++) {
    const int k = kinds_host[s];
    if (k < DFB_CAND_REAL || k > DFB_CAND_CATEGORICAL ||
        (k == DFB_CAND_CATEGORICAL && (n_levels_host == nullptr || n_levels_host[s] < 1 ||
                                       n_levels_host[s] > ((int64_t)1 << 52)))) {
      set_error("fill_mixed_candidates: bad column %d (kind %d)", s, k);
      return -1;
    }
  }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  return launch_fill_mixed_candidates(h, seed, row0, m, d, kinds_host, lo_host, hi_host, n_levels_host, out_dev);
}

int dfb_ts_argmax(dfb_handle* h, const double* samples_dev, int64_t ld, int32_t S, int64_t m, int64_t idx_base,
                  int32_t reset, double* best_dev, int64_t* index_dev) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (samples_dev == nullptr || best_dev == nullptr || index_dev == nullptr || S < 1 || m < 1 || ld < m) { set_error("bad ts_argmax arguments"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  return launch_ts_argmax(h, samples_dev, ld, S, m, idx_base, reset, best_dev, index_dev);
}

int64_t dfb_launch_count(dfb_handle* h) { return h ? h->launches : 0; }

// The production int8 contraction on caller-owned digit planes (tests/test_gpu_i8_exact.py): A = n_rb * 128 rows of
// W digits, B = n_cb tiles of K_* digits, K = n_rb * 128, both in the pair-interleaved three-plane layout of
// gemm_i8.cuh.  Tensor maps and launch as in prepare_i8 / run_chunks; the handle's digit scheme and buffers are untouched.
int dfb_debug_score_i8(dfb_handle* h, int32_t radix256, const void* a_planes_dev, const void* b_planes_dev, int32_t n_rb,
                       int32_t n_cb, const double* rowscale_dev, double colscale, const int32_t* abort_count_dev,
                       double* partial_dev, int64_t ld_partial) {
  DFB_TRY(need(h, false, false, false, false, false));
  const int bn = i8_tile_n(radix256 != 0);
  if (a_planes_dev == nullptr || b_planes_dev == nullptr || rowscale_dev == nullptr || partial_dev == nullptr ||
      n_rb < 1 || n_cb < 1 || ld_partial < (int64_t)n_cb * bn) {
    set_error("bad debug_score_i8 arguments (n_rb %d, n_cb %d, ld_partial %lld)", n_rb, n_cb, (long long)ld_partial);
    return -1;
  }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  const int64_t K = (int64_t)n_rb * TILE, a_rows = K, b_rows = (int64_t)n_cb * bn;
  I8Maps tmA, tmB;
  DFB_TRY(make_i8_maps(&tmA, a_planes_dev, K, a_rows, true, radix256 != 0));
  DFB_TRY(make_i8_maps(&tmB, b_planes_dev, K, b_rows, false, radix256 != 0));
  const int keep_group = h->last_c2_group;
  DFB_TRY(launch_score_i8_args(h, radix256 != 0, tmA, tmB, n_rb, n_cb, (int)K, partial_dev, ld_partial, rowscale_dev,
                               colscale, abort_count_dev));
  h->last_c2_group = keep_group;
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

// Device-to-device copy of one internal buffer of the current state (tests/test_gpu_i8_exact.py); sizes follow from
// the queries "npad" and "chunk".
int dfb_debug_copy(dfb_handle* h, const char* name, void* dst_dev, int64_t bytes) {
  DFB_TRY(need(h, true, false, false, false, false));
  if (name == nullptr || dst_dev == nullptr) { set_error("bad debug_copy arguments"); return -1; }
  const int64_t npad = h->npad, chunk = h->chunk;
  const void* src = nullptr;
  int64_t size = 0;
  if (strcmp(name, "W") == 0) { src = h->W; size = (int64_t)sizeof(double) * npad * npad; }
  else if (strcmp(name, "T") == 0) { src = h->T; size = (int64_t)sizeof(double) * (2 * npad + TILE) * npad; }
  else if (strcmp(name, "alpha") == 0) { src = h->alpha; size = (int64_t)sizeof(double) * npad; }
  else if (strcmp(name, "Wi8") == 0) { src = h->Wi8; size = 3 * 2 * npad * npad; }
  else if (strcmp(name, "rowscale") == 0) { src = h->rowscale; size = (int64_t)sizeof(double) * npad; }
  else if (strcmp(name, "Ki8") == 0) { src = h->Ki8; size = 3 * 2 * chunk * npad; }
  else if (strcmp(name, "Ks") == 0) { src = h->Ks; size = (int64_t)sizeof(double) * chunk * npad; }
  else if (strcmp(name, "partial") == 0) { src = h->partial; size = (int64_t)sizeof(double) * (npad / TILE) * chunk; }
  else if (strcmp(name, "kssv") == 0) { src = h->kssv; size = (int64_t)sizeof(double) * chunk; }
  else if (strncmp(name, "ts_", 3) == 0) {
    if (h->ts_ws == nullptr) { set_error("debug_copy '%s': no Thompson-sampling workspace is set", name); return -1; }
    const int64_t mbp = h->ts_mb;
    if (strcmp(name, "ts_Cov") == 0) { src = h->ts_Cov; size = (int64_t)sizeof(double) * mbp * mbp; }
    else if (strcmp(name, "ts_T") == 0) { src = h->ts_T; size = (int64_t)sizeof(double) * (2 * mbp + TILE) * mbp; }
    else { set_error("unknown debug_copy buffer '%s'", name); return -1; }
  }
  else if (strcmp(name, "js_Cov") == 0) {
    if (h->js_ws == nullptr) { set_error("debug_copy '%s': no joint workspace is set", name); return -1; }
    src = h->js_Cov; size = (int64_t)sizeof(double) * h->js_mb * h->js_mb;
  }
  else { set_error("unknown debug_copy buffer '%s'", name); return -1; }
  if (bytes != size) {
    set_error("debug_copy '%s': %lld bytes requested, the buffer has %lld", name, (long long)bytes, (long long)size);
    return -1;
  }
  if (size == 0) return 0;
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_CUDA_OK(cudaMemcpyAsync(dst_dev, src, (size_t)size, cudaMemcpyDeviceToDevice, h->stream));
  DFB_CUDA_OK(cudaStreamSynchronize(h->stream));
  return 0;
}

int dfb_query(dfb_handle* h, const char* name, double* out) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (name == nullptr || out == nullptr) { set_error("bad query arguments"); return -1; }
  const dfb_kernel_desc& desc = active_kernel(h).desc;
  if (strcmp(name, "i8_sigma2_bound") == 0) { *out = h->i8_ready ? i8_sigma2_bound(h, desc) : -1.0; return 0; }
  if (strcmp(name, "last_used_i8") == 0) { *out = (double)h->last_used_i8; return 0; }
  if (strcmp(name, "last_shortlist") == 0) { *out = (double)h->last_shortlist; return 0; }
  if (strcmp(name, "last_selfcheck_violations") == 0) { *out = (double)h->last_selfcheck_violations; return 0; }
  if (strcmp(name, "last_selfcheck_ratio") == 0) { *out = h->last_selfcheck_ratio; return 0; }
  if (strcmp(name, "last_survivors") == 0) { *out = (double)h->last_survivors; return 0; }
  if (strcmp(name, "last_pruned_candidates") == 0) { *out = (double)h->last_pruned; return 0; }
  if (strcmp(name, "chunk") == 0) { *out = (double)h->chunk; return 0; }
  if (strcmp(name, "npad") == 0) { *out = (double)h->npad; return 0; }
  if (strcmp(name, "last_c2_group") == 0) { *out = (double)h->last_c2_group; return 0; }
  if (strcmp(name, "i8_bound_limit") == 0) { *out = I8_BOUND_LIMIT; return 0; }
  if (strcmp(name, "score_impl") == 0) { *out = (double)h->score_impl; return 0; }
  if (strcmp(name, "i8_ready") == 0) { *out = h->i8_ready ? 1.0 : 0.0; return 0; }
  if (strcmp(name, "i8_impl") == 0) { *out = 2.0; return 0; }     // bench.py reads it; the digit scheme is option i8_radix
  if (strcmp(name, "i8_radix256") == 0) { *out = (double)h->i8_radix256; return 0; }
  set_error("unknown query '%s'", name);
  return -1;
}

int dfb_set_option(dfb_handle* h, const char* name, int64_t value) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (name == nullptr) { set_error("option name is NULL"); return -1; }
  if (strcmp(name, "gemm_impl") == 0) {
    if (value != 0 && value != 1) { set_error("gemm_impl must be 0 (cp.async) or 1 (TMA)"); return -1; }
    h->gemm_impl = (int)value;
    return prepare_scoring(h, false, true);
  }
  if (strcmp(name, "kstar_fast") == 0) { h->kstar_fast = value ? 1 : 0; return 0; }
  if (strcmp(name, "lookahead") == 0) { h->lookahead = value ? 1 : 0; return 0; }
  if (strcmp(name, "small_eval") == 0) { h->small_eval = value ? 1 : 0; return 0; }
  if (strcmp(name, "i8_fuse") == 0) { h->i8_fuse = value ? 1 : 0; return 0; }
  if (strcmp(name, "kstar_seg") == 0) { h->kstar_seg = value ? 1 : 0; return 0; }
  if (strcmp(name, "kstar_rows64") == 0) { h->kstar_rows64 = value ? 1 : 0; return 0; }
  if (strcmp(name, "prune") == 0) { h->prune = value ? 1 : 0; return 0; }
  if (strcmp(name, "i8_unguarded") == 0) { h->i8_unguarded = value ? 1 : 0; return 0; }
  if (strcmp(name, "i8_radix") == 0) {
    if (value < -1 || value > 1) { set_error("i8_radix must be -1 (auto), 0 (radix 128) or 1 (radix 256)"); return -1; }
    h->i8_radix_opt = (int)value;
    if (h->i8_ready) { DFB_CUDA_OK(cudaSetDevice(h->device)); DFB_TRY(prepare_i8(h)); }
    return 0;
  }
  if (strcmp(name, "tma_cb_group") == 0 && value >= 1) { h->tma_cb_group = (int)value; return 0; }
  if (strcmp(name, "i8_c2_group") == 0 && value >= 0) { h->i8_c2_group = (int)value; return 0; }
  if (strcmp(name, "score_impl") == 0) {
    if (value < 0 || value > 2) { set_error("score_impl must be 0 (fp64 DMMA), 1 (int8-slice wgmma) or 2 (auto)"); return -1; }
    h->score_impl = (int)value;
    return prepare_scoring(h, true, false);
  }
  set_error("unknown option '%s'", name);
  return -1;
}

int dfb_profile_enable(dfb_handle* h, int on) {
  DFB_TRY(need(h, false, false, false, false, false));
  DFB_CUDA_OK(cudaSetDevice(h->device));
  if (on && h->prof == nullptr) {
    h->prof = new (std::nothrow) ProfClass[PROF_CLASSES];
    if (h->prof == nullptr) { set_error("out of host memory"); return -2; }
  }
  h->prof_on = (on != 0);
  return 0;
}

int dfb_profile_read(dfb_handle* h, int cls, double* ms_total, int64_t* launches, double* units) {
  DFB_TRY(need(h, false, false, false, false, false));
  if (cls < 0 || cls >= PROF_CLASSES || h->prof == nullptr) { set_error("profiling not enabled / bad class"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(h->device));
  DFB_TRY(prof_flush(h, cls));
  ProfClass& pc = h->prof[cls];
  if (ms_total) *ms_total = pc.acc_ms;
  if (launches) *launches = pc.acc_launches;
  if (units) *units = pc.acc_units;
  pc.acc_ms = 0.0; pc.acc_units = 0.0; pc.acc_launches = 0;
  return 0;
}

}  // extern "C"
