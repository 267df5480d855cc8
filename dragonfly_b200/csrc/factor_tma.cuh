// The panel solve and the trailing update of the blocked factorisation of the tall matrix [A ; I ; y^T]
// (api.cu: factorise_tall), on Hopper's TMA and mbarriers:
//   panel     P <- P inv(L_kk)^T        in place, for every structurally non-zero row block of column block `step`
//   trailing  T_rj <- T_rj - P_r P_j^T   for every structurally non-zero tile of column blocks [j0, j1)
//
//   * Compact tile list: blockIdx.x indexes the non-zero 128 x 128 tiles only (fu_* below), each split into
//     sub-tiles of BM x BN, so no CTA starts without work.  A panel tile is read and written in place: each output
//     row reads all 128 columns of its own input row, so panel sub-tiles split rows only (BN = 128).
//   * Operands by TMA (SWIZZLE_128B boxes of BM or BN rows x 16 doubles) into a 4-stage full/empty mbarrier ring:
//     one producer lane, four DMMA consumer warps.  A CTA owns one sub-tile and exits, so the high-priority chain
//     launches find an SM as soon as a bulk CTA retires; two bulk CTAs share an SM, so one's loads and DMMA overlap
//     the other's C read and D store.
//   * Two shapes, chosen by the launch site: the chain shape 32 x 128 (warp tile 32 x 32) spreads the ~41 tiles of
//     panel(k) and next(k) over ~160 CTAs; the bulk shape 128 x 64 (warp tile 64 x 32) runs the rest.
//
// Arithmetic: for every output element, the DMMA.8x8x4 sequence of gemm_tn_kernel -- accumulators from 0, k-slabs
// of 16 in ascending order, DMMA kk = 0..3 of a slab contracting k = 16 kt + 4 kk + fk on quad lane fk -- and the
// epilogue alpha * acc, then + C.  The factor is bit for bit the one gemm_tn_kernel's tiles produce (and the one
// lml_batch_kernel mirrors).  Element (r, k) of a swizzled box row sits in 16-byte chunk (k >> 1) ^ (r & 7); with
// the quad lanes on k = 4 kk + fk a warp's 32 loads hit 16 distinct 8-byte slots twice each: two wavefronts, the
// minimum for 256 bytes.
#pragma once
#include "gemm_tma.cuh"

namespace dfb {

constexpr int FU_STAGES = 4;
constexpr int FU_CONSUMER_WARPS = 4;
constexpr int FU_THREADS = (FU_CONSUMER_WARPS + 1) * 32;
constexpr int FU_CHAIN_BM = 32, FU_CHAIN_BN = 128;       // panel(k), next(k)
constexpr int FU_BULK_BM = 128, FU_BULK_BN = 64;         // rest(k), the single-stream trailing update

constexpr size_t fu_smem_bytes(int bm, int bn) {
  return (size_t)FU_STAGES * (bm + bn) * GEMM_BK * sizeof(double) + 1024 /*align*/ + 2 * FU_STAGES * 8 /*barriers*/;
}

// Row blocks of the tall matrix that are structurally non-zero in column block `step`, in the order the panel
// visits them: top rows step+1 .. nb-1, L^-T rows nb .. nb+step (absent with skip_bottom), the y row block 2 nb.
__host__ __device__ inline int fu_panel_rows(const FactorArgs& g) {
  return (g.nb - g.step - 1) + (g.skip_bottom ? 0 : g.step + 1) + 1;
}
__device__ __forceinline__ int fu_panel_row(const FactorArgs& g, int t) {
  const int top = g.nb - g.step - 1;
  if (t < top) return g.step + 1 + t;
  t -= top;
  return (!g.skip_bottom && t <= g.step) ? g.nb + t : 2 * g.nb;
}

// Non-zero tiles of the trailing update of column blocks [j0, j1): the rows that are full in every column (L^-T
// rows nb .. nb+step, the y row block) first, row by row, then the top's lower triangle (row blocks j .. nb-1 of
// column j) column by column.
__host__ __device__ inline int fu_trail_tiles(const FactorArgs& g) {
  const int nc = g.j1 - g.j0;
  const int full = (g.skip_bottom ? 0 : g.step + 1) + 1;
  return full * nc + nc * g.nb - (g.j0 + g.j1 - 1) * nc / 2;
}
__device__ __forceinline__ void fu_trail_tile(const FactorArgs& g, int t, int& rbk, int& j) {
  const int nc = g.j1 - g.j0;
  const int full = (g.skip_bottom ? 0 : g.step + 1) + 1;
  if (t < full * nc) {
    const int r = t / nc;
    j = g.j0 + (t - r * nc);
    rbk = (r < full - 1) ? g.nb + r : 2 * g.nb;
    return;
  }
  t -= full * nc;
  j = g.j0;
  while (t >= g.nb - j) { t -= g.nb - j; j++; }
  rbk = j + t;
}

// tmA: the tall matrix in boxes of BM rows.  tmB: the panel's inv(L_kk)^T (Dinv, boxes of 128 rows) or the tall
// matrix in boxes of BN rows (the trailing update's P_j).
template <int WM, int WN, int WARPS_M, int WARPS_N, int MIN_BLOCKS>
__global__ void __launch_bounds__(FU_THREADS, MIN_BLOCKS)
factor_update_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const FactorArgs g) {
  constexpr int BM = WM * WARPS_M, BN = WN * WARPS_N;
  constexpr int MI = WM / 8, NI = WN / 8;
  constexpr int SR = TILE / BM, SC = TILE / BN;
  constexpr int A_BYTES = BM * GEMM_BK * 8, STAGE_BYTES = (BM + BN) * GEMM_BK * 8;
  constexpr int NK = TILE / GEMM_BK;
  static_assert(WARPS_M * WARPS_N == FU_CONSUMER_WARPS, "four consumer warps");
  static_assert(TILE % BM == 0 && TILE % BN == 0 && BM % 8 == 0, "sub-tiles of a 128 x 128 tile");
  extern __shared__ unsigned char smem_raw[];
  // One decision per CTA: chol_diag on the other stream may set *info while this CTA starts, and a producer or
  // consumer warp that left on its own would leave the others waiting on the ring forever.
  if (__syncthreads_or(threadIdx.x == 0 && g.info != nullptr && *g.info != 0)) return;

  // SWIZZLE_128B atoms are 1024 B: align the ring
  unsigned char* tiles = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + (size_t)FU_STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + FU_STAGES;

  const int t = blockIdx.x / (SR * SC), sub = blockIdx.x - t * (SR * SC);
  const int sr = sub / SC, sc = sub - sr * SC;
  int rbk, j;
  if (g.panel) { rbk = fu_panel_row(g, t); j = g.step; }
  else fu_trail_tile(g, t, rbk, j);
  const int row0 = rbk * TILE + sr * BM;          // rows of A and D
  const int col0 = j * TILE + sc * BN;            // columns of D; rows of B in the trailing update
  const int k0 = g.step * TILE;                   // column of A (and of the trailing update's B) where k starts
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < FU_STAGES; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], FU_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp == FU_CONSUMER_WARPS) {
    // ---------------- producer: one lane feeds the ring ------------------------------------------
    if (lane == 0) {
      const int bk0 = g.panel ? 0 : k0, brow = g.panel ? 0 : col0;
      for (int kt = 0; kt < NK; kt++) {
        const int s = kt % FU_STAGES;
        const unsigned n = (unsigned)(kt / FU_STAGES);
        mbar_wait(&empty_bar[s], (n & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (unsigned)STAGE_BYTES);
        unsigned char* dst = tiles + (size_t)s * STAGE_BYTES;
        tma_load_2d(dst, &tmA, k0 + kt * GEMM_BK, row0, &full_bar[s]);
        tma_load_2d(dst + A_BYTES, &tmB, bk0 + kt * GEMM_BK, brow, &full_bar[s]);
      }
    }
    return;
  }

  // ---------------- consumers: DMMA on swizzled tiles, gemm_tn_kernel's k order ---------------------
  const int wm = warp / WARPS_N, wn = warp - wm * WARPS_N;
  const int fr = lane >> 2, fk = lane & 3;
  double c[MI][NI][2];
#pragma unroll
  for (int mi = 0; mi < MI; mi++)
#pragma unroll
    for (int ni = 0; ni < NI; ni++) { c[mi][ni][0] = 0.0; c[mi][ni][1] = 0.0; }

  // byte offset of k = 4 kk + fk inside a row whose index is fr mod 8: chunk (2 kk + (fk >> 1)) ^ fr, half fk & 1
  int koff[4];
#pragma unroll
  for (int kk = 0; kk < 4; kk++) koff[kk] = (((2 * kk + (fk >> 1)) ^ fr) << 4) + ((fk & 1) << 3);
  const int a_row0 = (wm * WM + fr) * 128;
  const int b_row0 = A_BYTES + (wn * WN + fr) * 128;

#pragma unroll 1
  for (int kt = 0; kt < NK; kt++) {
    const int s = kt % FU_STAGES;
    const unsigned n = (unsigned)(kt / FU_STAGES);
    mbar_wait(&full_bar[s], n & 1u);
    const unsigned char* St = tiles + (size_t)s * STAGE_BYTES;
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      double a[MI], b[NI];
#pragma unroll
      for (int mi = 0; mi < MI; mi++)
        a[mi] = *reinterpret_cast<const double*>(St + a_row0 + mi * 8 * 128 + koff[kk]);
#pragma unroll
      for (int ni = 0; ni < NI; ni++)
        b[ni] = *reinterpret_cast<const double*>(St + b_row0 + ni * 8 * 128 + koff[kk]);
#pragma unroll
      for (int mi = 0; mi < MI; mi++)
#pragma unroll
        for (int ni = 0; ni < NI; ni++) dmma884(c[mi][ni][0], c[mi][ni][1], a[mi], b[ni]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

  // ---------------- epilogue: D = alpha * acc (+ C), C = D = the tile itself in the trailing update ----------
  // C comes from L2 (ld.global.cg), not L1: the other stream's launches rewrite these tiles, and a CTA on the same SM
  // may have left a line of a tile's older value in L1.  The compiler keeps such loads behind earlier stores, so each
  // fragment row loads all its C before it stores.
  const double alpha = g.panel ? 1.0 : -1.0;
  double* D = g.T + (int64_t)row0 * g.ld + col0;
#pragma unroll
  for (int mi = 0; mi < MI; mi++) {
    double2* p = reinterpret_cast<double2*>(D + (int64_t)(wm * WM + mi * 8 + fr) * g.ld + wn * WN + 2 * fk);
    double2 cc[NI];
    if (!g.panel) {
#pragma unroll
      for (int ni = 0; ni < NI; ni++) cc[ni] = __ldcg(p + ni * 4);
    }
#pragma unroll
    for (int ni = 0; ni < NI; ni++) {
      double2 v;
      v.x = alpha * c[mi][ni][0];
      v.y = alpha * c[mi][ni][1];
      if (!g.panel) {
        v.x += cc[ni].x;
        v.y += cc[ni].y;
      }
      p[ni * 4] = v;
    }
  }
}

}  // namespace dfb
