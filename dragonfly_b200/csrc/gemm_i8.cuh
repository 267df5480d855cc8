// The scoring contraction on the Hopper tensor cores: an error-bounded integer-slice (Ozaki-style)
// evaluation of V = W K_*^T followed by the fused |v|^2 column reduction.
//
// wgmma has no f64 kind, and the fp64 DMMA path is far below the int8 rate.  Instead both fp64 operands
// are expanded exactly into small signed digits after a power-of-two scaling,
//     W[i,k]  = 2^E_i * sum_s a_s[i,k] r^-s,    K*[m,k] = 2^F * sum_t b_t[m,k] r^-t,
// so that V[i,m] = 2^(E_i+F) sum_d r^-d G_d[i,m] with G_d = sum_{s+t=d} A_s B_t^T (int32, exact).  Two digit
// schemes (chosen per posterior by api.cu from the a-priori error bound):
//   radix 128: six signed 7-bit digits, all 21 products (groups d = 2..7, weight 2^-7d);
//   radix 256: five digits (top digit 7 bits, four balanced bytes: digits_radix256 in kernels.cu), the 15
//              products with s + t <= 6 (groups d = 2..6, weight 2^-(8d-2)); the dropped terms are ~2^-40 of the
//              operands' scale, the order of the digit truncation.  int32 headroom: 5 K 2^14 < 2^31 needs
//              K <= 26214 (api.cu refuses the scheme beyond npad = 24576).
//
// Digit planes are stored pair-interleaved at 32-k granularity: plane p holds digits 2p+1 and 2p+2 (1-based), and
// every 64-byte row segment holds 32 k-values of the first followed by the same 32 k-values of the second.  One
// TMA box (64 B x rows x 3 planes, SWIZZLE_64B) thus brings all digits of a K = 32 block, and the wgmma
// descriptors of the two digits of a plane differ by a 32-byte start offset inside the swizzle atom.
//
// CTA = one 128 (rows of W) x 32 (candidates) output tile, 9 warps:
//   warps 0-7  two consumer warpgroups, 64 rows each: per K = 32 block one wgmma.m64n32k32.s32.s8.s8 per kept digit
//              product, both operands from shared memory, int32 accumulators in registers (one 16-register
//              fragment per digit group); the epilogue recombines the groups in fp64 (smallest weight first),
//              applies the row / column scales, squares and reduces every column over the tile's 128 rows in a
//              fixed order (deterministic `partial`, same layout as the DMMA kernels);
//   warp 8     TMA producer (one lane): full / empty mbarrier ring of I8_STAGES K-blocks.
// W is lower triangular: row block rb only contracts k < 128 (rb + 1).  Tile order: groups of `cb_group` candidate
// tiles; inside a group the heaviest row blocks first, so the CTAs resident at a time share a few K_* digit tiles and
// sweep W.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "gemm_tma.cuh"   // mbarrier / TMA helpers

namespace dfb {

constexpr int I8_S = 6;                        // radix-128 digits per operand
constexpr int I8_R256_DIGITS = 5;              // radix-256 digits per operand
constexpr int I8_BM = 128, I8_BK = 32;          // I8_BN: gemm_tma.h
constexpr int I8_STAGES = 7;
constexpr int I8_A_PLANE = I8_BM * 2 * I8_BK;  // 8192 B: 128 rows x (32 B digit 2p+1 | 32 B digit 2p+2)
constexpr int I8_B_PLANE = I8_BN * 2 * I8_BK;  // 2048 B
constexpr int I8_A_BYTES = 3 * I8_A_PLANE;
constexpr int I8_STAGE_BYTES = I8_A_BYTES + 3 * I8_B_PLANE;   // 30720
constexpr int I8_CONSUMERS = 256;              // two warpgroups
constexpr int I8_THREADS = I8_CONSUMERS + 32;  // + the producer warp
constexpr size_t I8_SMEM_BYTES = (size_t)I8_STAGES * I8_STAGE_BYTES + 1024 + 8 * I8_BN * sizeof(double) +
                                 2 * I8_STAGES * 8 + 64;

struct ScoreI8Args {
  int n_rb, n_cb, K;
  int cb_group;             // candidate tiles per scheduling group
  double* partial;
  int64_t ld_partial;
  const double* rowscale;   // 2^E_i per row of W
  double colscale;          // 2^F
  const int* abort_count;   // the launch is a no-op once *abort_count > abort_cap (the arg-max shortlist overflowed,
  int abort_cap;            // so this int8 pass will be discarded for an fp64 one); may be NULL
};

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2,
                                            void* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// K-major SWIZZLE_64B shared-memory matrix descriptor of wgmma: start >> 4, LBO 1 (unused for swizzled K-major),
// SBO = 512 B (8 rows x 64 B), layout type 2 = SWIZZLE_64B.
__device__ __forceinline__ uint64_t wgmma_desc_sw64(unsigned smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
// D (64 x 32, int32) (+)= A (64 x 32 int8) B^T (32 x 32 int8); accumulate = 0 overwrites D
__device__ __forceinline__ void wgmma_i8_n32(int (&d)[16], uint64_t da, uint64_t db, unsigned accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
__device__ __forceinline__ void wgmma_fence_operands(int (&d)[16]) {
#pragma unroll
  for (int i = 0; i < 16; i++) asm volatile("" : "+r"(d[i])::"memory");
}

template <bool R256>
__global__ void __launch_bounds__(I8_THREADS, 1)
score_i8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const ScoreI8Args g) {
  // uniform over the grid: the counter is only written by earlier kernels of the same stream
  if (g.abort_count != nullptr && *g.abort_count > g.abort_cap) return;
  constexpr int NS = R256 ? I8_R256_DIGITS : I8_S;      // digits per operand
  constexpr int DMAX = R256 ? 6 : 7;                     // largest kept digit group s + t
  constexpr int NG = DMAX - 1;                           // accumulators: groups 2..DMAX
  extern __shared__ unsigned char smem_raw[];
  unsigned char* tiles = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  double* colsum = reinterpret_cast<double*>(tiles + (size_t)I8_STAGES * I8_STAGE_BYTES);   // [8 warps][32]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(colsum + 8 * I8_BN);
  uint64_t* empty_bar = full_bar + I8_STAGES;

  const int bid = blockIdx.x;
  const int G = (g.cb_group > 0 && g.cb_group < g.n_cb) ? g.cb_group : g.n_cb;
  const int per_group = G * g.n_rb;
  const int grp = bid / per_group, rem = bid - grp * per_group;
  const int cb0 = grp * G;
  const int width = min(G, g.n_cb - cb0);               // the last group may be narrower
  const int rb = g.n_rb - 1 - rem / width;
  const int cb = cb0 + rem % width;
  const int nk = min(g.K, (rb + 1) * TILE) / I8_BK;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < I8_STAGES; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], I8_CONSUMERS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  if (warp == I8_CONSUMERS / 32) {
    // ---------------- TMA producer ----------------------------------------------------------------------
    if (lane == 0) {
      for (int kt = 0; kt < nk; kt++) {
        const int s = kt % I8_STAGES;
        const unsigned n = (unsigned)(kt / I8_STAGES);
        mbar_wait(&empty_bar[s], (n & 1u) ^ 1u);
        mbar_expect_tx(&full_bar[s], (unsigned)I8_STAGE_BYTES);
        unsigned char* dst = tiles + (size_t)s * I8_STAGE_BYTES;
        tma_load_3d(dst, &tmA, kt * 2 * I8_BK, rb * I8_BM, 0, &full_bar[s]);
        tma_load_3d(dst + I8_A_BYTES, &tmB, kt * 2 * I8_BK, cb * I8_BN, 0, &full_bar[s]);
      }
    }
    return;
  }

  // ---------------- consumer warpgroups ------------------------------------------------------------------
  const int wg = warp >> 2;                              // rows [64 wg, 64 wg + 64) of the tile
  int acc[NG][16];
#pragma unroll
  for (int a = 0; a < NG; a++)
#pragma unroll
    for (int i = 0; i < 16; i++) acc[a][i] = 0;
  for (int kt = 0; kt < nk; kt++) {
    const int s = kt % I8_STAGES;
    mbar_wait(&full_bar[s], (unsigned)(kt / I8_STAGES) & 1u);
    const unsigned a0 = smem_u32(tiles + (size_t)s * I8_STAGE_BYTES) + (unsigned)(wg * 64 * 2 * I8_BK);
    const unsigned b0 = smem_u32(tiles + (size_t)s * I8_STAGE_BYTES + I8_A_BYTES);
#pragma unroll
    for (int a = 0; a < NG; a++) wgmma_fence_operands(acc[a]);
    wgmma_fence();
#pragma unroll
    for (int d = 2; d <= DMAX; d++) {
      bool lead = true;
#pragma unroll
      for (int sa = 1; sa <= NS; sa++) {
        const int tb = d - sa;
        if (tb < 1 || tb > NS) continue;
        const unsigned aoff = (unsigned)(((sa - 1) >> 1) * I8_A_PLANE + ((sa - 1) & 1) * I8_BK);
        const unsigned boff = (unsigned)(((tb - 1) >> 1) * I8_B_PLANE + ((tb - 1) & 1) * I8_BK);
        wgmma_i8_n32(acc[d - 2], wgmma_desc_sw64(a0 + aoff), wgmma_desc_sw64(b0 + boff),
                     (kt == 0 && lead) ? 0u : 1u);
        lead = false;
      }
    }
    wgmma_commit();
#pragma unroll
    for (int a = 0; a < NG; a++) wgmma_fence_operands(acc[a]);
    // the products of block kt - 1 are complete: release its stage
    wgmma_wait<1>();
    if (kt > 0 && lane == 0) mbar_arrive(&empty_bar[(kt - 1) % I8_STAGES]);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int a = 0; a < NG; a++) wgmma_fence_operands(acc[a]);

  // Accumulator fragment of m64nN: register 4j + e of lane l in warp w (of the warpgroup) holds row
  // 16 w + l / 4 + 8 (e >> 1), column 8 j + 2 (l % 4) + (e & 1).
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const double rs0 = g.rowscale[(int64_t)rb * I8_BM + r0] * g.colscale;
  const double rs1 = g.rowscale[(int64_t)rb * I8_BM + r0 + 8] * g.colscale;
  double cs[8];
#pragma unroll
  for (int i = 0; i < 16; i++) {
    // v = sum_d G_d w_d, smallest weight first
    double v;
    if constexpr (R256) {
      v = (double)acc[4][i] * 0x1p-46;
      v = fma((double)acc[3][i], 0x1p-38, v);
      v = fma((double)acc[2][i], 0x1p-30, v);
      v = fma((double)acc[1][i], 0x1p-22, v);
      v = fma((double)acc[0][i], 0x1p-14, v);
    } else {
      v = (double)acc[NG - 1][i] * 0x1p-49;
      v = fma((double)acc[4][i], 0x1p-42, v);
      v = fma((double)acc[3][i], 0x1p-35, v);
      v = fma((double)acc[2][i], 0x1p-28, v);
      v = fma((double)acc[1][i], 0x1p-21, v);
      v = fma((double)acc[0][i], 0x1p-14, v);
    }
    v *= ((i & 2) ? rs1 : rs0);
    const int c = (i >> 2) * 2 + (i & 1);                // column slot of this thread (0..7)
    if (i & 2) cs[c] += v * v; else cs[c] = v * v;
  }
  // sum each column slot over the 8 row groups of the warp (lanes with equal l % 4): fixed tree
#pragma unroll
  for (int c = 0; c < 8; c++) {
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 4);
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 8);
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 16);
  }
  if (lane < 4) {
#pragma unroll
    for (int c = 0; c < 8; c++) colsum[warp * I8_BN + (c >> 1) * 8 + 2 * lane + (c & 1)] = cs[c];
  }
  asm volatile("bar.sync 1, %0;\n" ::"n"(I8_CONSUMERS) : "memory");
  if (tid < I8_BN) {
    double t = colsum[tid];
#pragma unroll
    for (int w = 1; w < 8; w++) t += colsum[w * I8_BN + tid];
    g.partial[(int64_t)rb * g.ld_partial + (int64_t)cb * I8_BN + tid] = t;
  }
}

}  // namespace dfb
