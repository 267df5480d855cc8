// v2 of the dominant kernel: V = W K_*^T fused with |v|^2 per candidate column (MODE_SCORE + SUMSQ of
// gemm.cuh), re-staged with Hopper's TMA and mbarriers:
//   * operand tiles arrive by TMA (cp.async.bulk.tensor.2d, SASS UTMALDG) from two tensor maps
//     (W and the K_* chunk), 128 rows x 16 doubles per box, SWIZZLE_128B so the fragment reads below
//     are bank-conflict free without padding;
//   * a 6-stage ring guarded by full/empty mbarriers replaces the per-slab __syncthreads: one
//     producer warp (one elected lane) issues the TMA loads, eight consumer warps run DMMA.8x8x4 and
//     never rendezvous with each other inside the k-loop, so the FP64 pipe is not drained at stage
//     boundaries;
//   * same tiling as v1 (CTA 128 x 128, warp tile 64 x 32, lower-triangular k-range per row block,
//     heaviest row blocks first) and the same deterministic epilogue.
// DMMA is free to pick which k each quad lane contracts as long as A and B agree; lanes use
// k = 2*kk + (fk & 1) + 8*(fk >> 1), which maps the eight (row, chunk) pairs of a half-warp onto
// eight different 16-byte chunks of the swizzled row.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "gemm.cuh"
#include "gemm_tma.h"

namespace dfb {

constexpr int TMA_STAGES = 6;
constexpr int TMA_CONSUMER_WARPS = 8;
constexpr int TMA_THREADS = (TMA_CONSUMER_WARPS + 1) * 32;
constexpr int TMA_TILE_BYTES = TILE * GEMM_BK * 8;                 // 16 KB per operand per stage
constexpr int TMA_STAGE_BYTES = 2 * TMA_TILE_BYTES;                // A + B
constexpr size_t TMA_SMEM_BYTES = (size_t)TMA_STAGES * TMA_STAGE_BYTES + 1024 /*align*/ +
                                  2 * TILE * sizeof(double) /*red*/ + 2 * TMA_STAGES * 8 /*barriers*/ + 64;

__device__ __forceinline__ unsigned smem_u32(const void* p) {
  return (unsigned)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(void* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ unsigned mbar_try_wait(void* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
__device__ __forceinline__ void mbar_wait(void* bar, unsigned parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1,
                                            void* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

__global__ void __launch_bounds__(TMA_THREADS, 1)
score_tma_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmK,
                 const ScoreTmaArgs g) {
  extern __shared__ unsigned char smem_raw[];
  // SWIZZLE_128B atoms are 1024 B: align the tile ring
  unsigned char* tiles = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  double* red = reinterpret_cast<double*>(tiles + (size_t)TMA_STAGES * TMA_STAGE_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(red + 2 * TILE);
  uint64_t* empty_bar = full_bar + TMA_STAGES;

  // Tile order: groups of `cb_group` candidate tiles, heaviest row blocks first inside a group, so the
  // resident CTAs share a few K_* panels while they sweep W.
  const int bid = blockIdx.x;
  const int per_group = g.cb_group * g.n_rb;
  const int grp = bid / per_group, rem = bid - grp * per_group;
  const int rb = g.n_rb - 1 - rem / g.cb_group;
  const int cb = grp * g.cb_group + rem % g.cb_group;
  if (cb >= g.n_cb) return;                         // ragged last group (uniform per CTA)
  const int k_hi = min(g.K, (rb + 1) * TILE);
  const int nk = k_hi / GEMM_BK;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < TMA_STAGES; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], TMA_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp == TMA_CONSUMER_WARPS) {
    // ---------------- producer: one lane feeds the ring ------------------------------------------
    if (lane == 0) {
      for (int kt = 0; kt < nk; kt++) {
        const int s = kt % TMA_STAGES;
        const unsigned n = (unsigned)(kt / TMA_STAGES);
        mbar_wait(&empty_bar[s], (n & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (unsigned)TMA_STAGE_BYTES);
        unsigned char* dstA = tiles + (size_t)s * TMA_STAGE_BYTES;
        tma_load_2d(dstA, &tmW, kt * GEMM_BK, rb * TILE, &full_bar[s]);
        tma_load_2d(dstA + TMA_TILE_BYTES, &tmK, kt * GEMM_BK, cb * TILE, &full_bar[s]);
      }
    }
    return;
  }

  // ---------------- consumers: DMMA on swizzled tiles ----------------------------------------------
  const int wm = warp >> 2, wn = warp & 3;
  const int fr = lane >> 2, fk = lane & 3;
  double c[8][4][2];
#pragma unroll
  for (int mi = 0; mi < 8; mi++)
#pragma unroll
    for (int ni = 0; ni < 4; ni++) { c[mi][ni][0] = 0.0; c[mi][ni][1] = 0.0; }

  // byte offset of this lane's element inside a row for k-quad kk: chunk (kk + 4*(fk>>1)) ^ fr
  // (rows of a fragment differ by multiples of 8, so row & 7 == fr), 8-byte half (fk & 1)
  int koff[4];
#pragma unroll
  for (int kk = 0; kk < 4; kk++) koff[kk] = (((kk + 4 * (fk >> 1)) ^ fr) << 4) + ((fk & 1) << 3);
  const int a_row0 = (wm * 64 + fr) * 128;                       // bytes
  const int b_row0 = TMA_TILE_BYTES + (wn * 32 + fr) * 128;

  for (int kt = 0; kt < nk; kt++) {
    const int s = kt % TMA_STAGES;
    const unsigned n = (unsigned)(kt / TMA_STAGES);
    mbar_wait(&full_bar[s], n & 1u);
    const unsigned char* St = tiles + (size_t)s * TMA_STAGE_BYTES;
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
      double a[8], b[4];
#pragma unroll
      for (int mi = 0; mi < 8; mi++)
        a[mi] = *reinterpret_cast<const double*>(St + a_row0 + mi * 8 * 128 + koff[kk]);
#pragma unroll
      for (int ni = 0; ni < 4; ni++)
        b[ni] = *reinterpret_cast<const double*>(St + b_row0 + ni * 8 * 128 + koff[kk]);
#pragma unroll
      for (int mi = 0; mi < 8; mi++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++) dmma884(c[mi][ni][0], c[mi][ni][1], a[mi], b[ni]);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  }

  // ---------------- epilogue: column sums of squares (identical to v1) --------------------------------
#pragma unroll
  for (int ni = 0; ni < 4; ni++) {
#pragma unroll
    for (int e = 0; e < 2; e++) {
      double s = 0.0;
#pragma unroll
      for (int mi = 0; mi < 8; mi++) s = fma(c[mi][ni][e], c[mi][ni][e], s);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 16);
      if (fr == 0) red[wm * TILE + wn * 32 + ni * 8 + 2 * fk + e] = s;
    }
  }
  asm volatile("bar.sync 1, %0;\n" ::"n"(TMA_CONSUMER_WARPS * 32) : "memory");   // consumers only
  if (tid < TILE)
    g.partial[(int64_t)rb * g.ld_partial + (int64_t)cb * TILE + tid] = red[tid] + red[TILE + tid];
}

}  // namespace dfb
