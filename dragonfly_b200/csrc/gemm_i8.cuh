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
// every 64-byte row segment holds 32 k-values of the first followed by the same 32 k-values of the second.  A TMA box
// of 64 B x rows x planes (SWIZZLE_64B) thus brings both digits of each plane for a K = 32 block, and the wgmma
// descriptors of the two digits of a plane differ by a 32-byte start offset inside the swizzle atom.  Radix 128 loads
// all three planes in one box.  Radix 256 has five digits, so the second half of plane 3 (the sixth slot) is never
// written: planes 1-2 come in one box and digit 5 in a second box of 32 B x rows from plane 3 (SWIZZLE_32B).
//
// CTA = one 128 (rows of W) x BN (candidates) output tile, BN = i8_tile_n(radix256): 64 for radix 256, 32 for
// radix 128 (six accumulator groups of 32 columns would not fit the register file).  12 warps:
//   warps 0-7  two consumer warpgroups, 64 rows each (setmaxnreg 232).  Per K = 32 block each warp loads its 16 x 32
//              slice of every W digit once from shared memory into registers (ldmatrix.x4: the 8-bit A fragment of
//              wgmma), then issues one wgmma.m64nBNk32.s32.s8.s8 per kept digit product with A from those registers
//              and B (K_* digits) from a shared-memory descriptor, into int32 accumulators (one BN/2-register
//              fragment per digit group).  Each W digit is thus read from shared memory once per block rather than
//              once per product it takes part in; the fragments are double-buffered, and a buffer is reloaded only
//              after wgmma.wait_group has retired the products that read it.  The epilogue recombines the groups in
//              fp64 (smallest weight first), applies the row / column scales, squares and reduces every column over
//              the tile's 128 rows in a fixed order (deterministic `partial`, same layout as the DMMA kernels);
//   warps 8-11 the producer warpgroup (setmaxnreg 40): one lane runs the TMA side of a full / empty mbarrier ring of
//              I8Tile::STAGES K-blocks.
// Clusters of I8_CLUSTER CTAs take adjacent candidate tiles of the same row block, so they read the same W digits.
// Each CTA loads 128 / I8_CLUSTER rows of them and multicasts its box into the same stage of every CTA of the
// cluster; a stage is refilled only when the consumers of all of them have released it (each consumer warp arrives on
// the empty barrier of every CTA of the cluster).  Per CTA and K block L2 delivers 10 KB of W and 10 KB of K_* digits
// at radix 256, against 24 + 12 KB for one CTA loading the whole 3-plane W box alone.
// W is lower triangular: row block rb only contracts k < 128 (rb + 1).  Tile order: groups of `cb_group` candidate
// tiles (rounded up to whole clusters); inside a group the heaviest row blocks first, so the CTAs resident at a time
// share a few K_* digit tiles and sweep W.  When I8_CLUSTER does not divide n_cb, the last cluster of each row block
// has CTAs without a tile: they load their share of W for the others and compute on whatever K_* rows lie past the
// last tile (zeros outside the tensor map), but store nothing.
#pragma once
#include <cuda.h>
#include "common.cuh"
#include "gemm_tma.cuh"   // mbarrier / TMA helpers

namespace dfb {

constexpr int I8_S = 6;                        // radix-128 digits per operand
constexpr int I8_R256_DIGITS = 5;              // radix-256 digits per operand
constexpr int I8_BM = 128, I8_BK = 32;
constexpr int I8_CLUSTER = 2;                  // CTAs per cluster, adjacent candidate tiles sharing the W digits
constexpr int I8_WROWS = I8_BM / I8_CLUSTER;   // rows of W each CTA of a cluster loads
constexpr int I8_CONSUMERS = 256;              // two warpgroups
constexpr int I8_THREADS = I8_CONSUMERS + 128; // + the producer warpgroup
constexpr int I8_CONSUMER_REGS = 232, I8_PRODUCER_REGS = 40;   // 2 * 128 * 232 + 128 * 40 <= 65536

// Stage layout: W as I8_CLUSTER slices of I8_WROWS rows (one per loading CTA), then the K_* tile.  An operand slice of
// r rows holds NP planes of r x 64 B (SWIZZLE_64B) and, at radix 256, digit 5 as r x 32 B (SWIZZLE_32B).
template <bool R256>
struct I8Tile {
  static constexpr int BN = i8_tile_n(R256);                   // candidates per tile
  static constexpr int NP = R256 ? 2 : 3;                      // planes loaded whole
  static constexpr int ROW_BYTES = NP * 2 * I8_BK + (R256 ? I8_BK : 0);   // 160 (radix 256) or 192 B per row
  static constexpr int A_SLICE = I8_WROWS * ROW_BYTES;
  static constexpr int A_BYTES = I8_BM * ROW_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + BN * ROW_BYTES; // 30720 for both schemes
  static constexpr int STAGES = 7;
  static constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 + 8 * BN * sizeof(double) +
                                       2 * STAGES * 8 + 64;
  static_assert(A_SLICE % 1024 == 0 && A_BYTES % 1024 == 0 && STAGE_BYTES % 1024 == 0, "swizzle atoms stay aligned");
};

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
// the same box written to the same shared-memory offset of every CTA in cta_mask, each completing bytes on its own
// mbarrier at the offset of bar
__device__ __forceinline__ void tma_load_3d_multicast(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2,
                                                      void* bar, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;\n" ::"r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
  return r;
}
// arrive on the mbarrier at the offset of bar in CTA `cta` of the cluster.  Default (CTA-scope release) semantics: the
// reads this releases have retired (wgmma.wait_group, ldmatrix results consumed), and a cluster-scope release would
// put a fence in the consumer's path every K block.
__device__ __forceinline__ void mbar_arrive_cluster(void* bar, unsigned cta) {
  asm volatile(
      "{\n"
      ".reg .b32 ra;\n"
      "mapa.shared::cluster.u32 ra, %0, %1;\n"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;\n" ::: "memory");
}
// after mbarrier initialisation, which fence.mbarrier_init has already made visible to the cluster
__device__ __forceinline__ void cluster_sync_relaxed() {
  asm volatile("barrier.cluster.arrive.relaxed;\nbarrier.cluster.wait;\n" ::: "memory");
}
// K-major SWIZZLE_64B shared-memory matrix descriptor of wgmma: start >> 4, LBO 1 (unused for swizzled K-major),
// SBO = 512 B (8 rows x 64 B), layout type 2 = SWIZZLE_64B.
__device__ __forceinline__ uint64_t wgmma_desc_sw64(unsigned smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(512 >> 4) << 32) | (2ull << 62);
}
// K-major SWIZZLE_32B: SBO = 256 B (8 rows x 32 B), layout type 3 = SWIZZLE_32B
__device__ __forceinline__ uint64_t wgmma_desc_sw32(unsigned smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(256 >> 4) << 32) | (3ull << 62);
}
// Four 8 x 16-byte matrices; lanes 8q .. 8q + 7 give the row addresses of matrix q, which lands in register q.
__device__ __forceinline__ void ldmatrix_x4(unsigned (&r)[4], unsigned smem_addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_addr)
               : "memory");
}
// D (64 x 32, int32) (+)= A (64 x 32 int8, registers) B^T (32 x 32 int8, shared); accumulate = 0 overwrites D
__device__ __forceinline__ void wgmma_i8_rs(int (&d)[16], const unsigned (&a)[4], uint64_t db, unsigned accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate)
      : "memory");
}
// D (64 x 64, int32) (+)= A (64 x 32 int8, registers) B^T (32 x 64 int8, shared); accumulate = 0 overwrites D
__device__ __forceinline__ void wgmma_i8_rs(int (&d)[32], const unsigned (&a)[4], uint64_t db, unsigned accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
        "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
        "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
        "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads / writes of wgmma operand registers across an asynchronous wgmma
template <typename T, int N>
__device__ __forceinline__ void wgmma_fence_operands(T (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+r"(r[i])::"memory");
}

template <bool R256>
__global__ void __cluster_dims__(I8_CLUSTER, 1, 1) __launch_bounds__(I8_THREADS, 1)
score_i8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA5,
                const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmB5,
                const ScoreI8Args g) {
  // uniform over the grid: the counter is only written by earlier kernels of the same stream
  if (g.abort_count != nullptr && *g.abort_count > g.abort_cap) return;
  using T = I8Tile<R256>;
  constexpr int BN = T::BN, STAGES = T::STAGES, NP = T::NP;
  constexpr int NS = R256 ? I8_R256_DIGITS : I8_S;      // digits per operand
  constexpr int DMAX = R256 ? 6 : 7;                     // largest kept digit group s + t
  constexpr int NG = DMAX - 1;                           // accumulators: groups 2..DMAX
  constexpr int NACC = BN / 2;                           // int32 accumulator registers per group and thread
  constexpr int A_D5 = NP * I8_WROWS * 2 * I8_BK;        // digit 5 inside a W slice (radix 256)
  constexpr int B_D5 = NP * BN * 2 * I8_BK;              // digit 5 inside the K_* tile (radix 256)
  extern __shared__ unsigned char smem_raw[];
  unsigned char* tiles = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  double* colsum = reinterpret_cast<double*>(tiles + (size_t)STAGES * T::STAGE_BYTES);   // [8 warps][BN]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(colsum + 8 * BN);
  uint64_t* empty_bar = full_bar + STAGES;

  // tile of this CTA: cluster c of the grid holds the I8_CLUSTER adjacent candidate tiles of cluster column cc
  const unsigned rank = cluster_ctarank();
  const int cid = blockIdx.x / I8_CLUSTER;
  const int n_cc = (g.n_cb + I8_CLUSTER - 1) / I8_CLUSTER;
  const int G = (g.cb_group > 0 && g.cb_group < g.n_cb) ? g.cb_group : g.n_cb;
  const int Gc = (G + I8_CLUSTER - 1) / I8_CLUSTER;     // cluster columns per group
  const int per_group = Gc * g.n_rb;
  const int grp = cid / per_group, rem = cid - grp * per_group;
  const int cc0 = grp * Gc;
  const int width = min(Gc, n_cc - cc0);                // the last group may be narrower
  const int rb = g.n_rb - 1 - rem / width;
  const int cb = (cc0 + rem % width) * I8_CLUSTER + (int)rank;
  const int nk = min(g.K, (rb + 1) * TILE) / I8_BK;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], I8_CLUSTER * I8_CONSUMERS / 32);   // every consumer warp of the cluster
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  cluster_sync_relaxed();   // the barriers of every CTA are initialised before any multicast or remote arrive

  if (warp >= I8_CONSUMERS / 32) {
    // ---------------- TMA producer ----------------------------------------------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(I8_PRODUCER_REGS));
    if (warp == I8_CONSUMERS / 32 && lane == 0) {
      constexpr uint16_t all = (uint16_t)((1u << I8_CLUSTER) - 1u);
      const int wrow = rb * I8_BM + (int)rank * I8_WROWS;
      for (int kt = 0; kt < nk; kt++) {
        const int s = kt % STAGES;
        const unsigned n = (unsigned)(kt / STAGES);
        mbar_wait(&empty_bar[s], (n & 1u) ^ 1u);
        // the whole stage: every CTA's W slice and this CTA's K_* tile
        mbar_expect_tx(&full_bar[s], (unsigned)T::STAGE_BYTES);
        unsigned char* dst = tiles + (size_t)s * T::STAGE_BYTES;
        unsigned char* wdst = dst + rank * T::A_SLICE;
        tma_load_3d_multicast(wdst, &tmA, kt * 2 * I8_BK, wrow, 0, &full_bar[s], all);
        if constexpr (R256) tma_load_3d_multicast(wdst + A_D5, &tmA5, kt * 2 * I8_BK, wrow, 2, &full_bar[s], all);
        tma_load_3d(dst + T::A_BYTES, &tmB, kt * 2 * I8_BK, cb * BN, 0, &full_bar[s]);
        if constexpr (R256) tma_load_3d(dst + T::A_BYTES + B_D5, &tmB5, kt * 2 * I8_BK, cb * BN, 2, &full_bar[s]);
      }
    }
    __syncwarp();
    cluster_sync();   // no CTA leaves while another can still multicast into it or arrive on its barriers
    return;
  }

  // ---------------- consumer warpgroups ------------------------------------------------------------------
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(I8_CONSUMER_REGS));
  const int wg = warp >> 2;                              // rows [64 wg, 64 wg + 64) of the tile
  // ldmatrix.x4 of a warp's 16 x 32 slice of one W digit: matrices (rows 0-7 | 8-15) x (bytes 0-15 | 16-31) give the
  // four registers of the 8-bit A fragment of wgmma (register q: row l / 4 + 8 (q & 1), bytes 4 (l % 4) + 16 (q >> 1)
  // .. + 3).  Lane l addresses row (l & 7) + 8 ((l >> 3) & 1), 16-byte chunk l >> 4 of the digit's 32 bytes.
  // SWIZZLE_64B (as TMA wrote the planes) stores 16-byte chunk c of the 64-byte row r at chunk c ^ ((r >> 1) & 3),
  // SWIZZLE_32B (digit 5) chunk c of the 32-byte row r at c ^ ((r >> 2) & 1).  The warp's rows start at a multiple of
  // 16 inside a slice, so (r >> 1) & 3 = (l & 7) >> 1 and (r >> 2) & 1 = (l >> 2) & 1.
  const int arow = wg * 64 + (warp & 3) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
  const unsigned a_slice = (unsigned)((arow / I8_WROWS) * T::A_SLICE);
  const unsigned a_lane = a_slice + (unsigned)((arow % I8_WROWS) * 2 * I8_BK);
  const unsigned a_chunk[2] = {(unsigned)(((0 + (lane >> 4)) ^ ((lane & 7) >> 1)) * 16),   // digit 2p+1 of a plane
                               (unsigned)(((2 + (lane >> 4)) ^ ((lane & 7) >> 1)) * 16)};  // digit 2p+2
  const unsigned a_lane5 = a_slice + (unsigned)(A_D5 + (arow % I8_WROWS) * I8_BK +
                                                (((lane >> 4) ^ ((lane >> 2) & 1)) * 16));
  int acc[NG][NACC];
#pragma unroll
  for (int a = 0; a < NG; a++)
#pragma unroll
    for (int i = 0; i < NACC; i++) acc[a][i] = 0;
  unsigned fa0[NS][4], fa1[NS][4];                      // A fragments of the even / odd K blocks

  // one K block: A fragments into fa, all kept digit products, release of the previous block's stage
  auto block = [&](const int kt, unsigned (&fa)[NS][4], unsigned (&fa_prev)[NS][4]) {
    const int s = kt % STAGES;
    mbar_wait(&full_bar[s], (unsigned)(kt / STAGES) & 1u);
    const unsigned st = smem_u32(tiles + (size_t)s * T::STAGE_BYTES);
#pragma unroll
    for (int sa = 1; sa <= NS; sa++) {
      const unsigned plane = (unsigned)(((sa - 1) >> 1) * I8_WROWS * 2 * I8_BK);
      ldmatrix_x4(fa[sa - 1], (R256 && sa == 5) ? st + a_lane5 : st + plane + a_lane + a_chunk[(sa - 1) & 1]);
    }
    const unsigned b0 = st + (unsigned)T::A_BYTES;
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
        const unsigned boff = (unsigned)(((tb - 1) >> 1) * BN * 2 * I8_BK + ((tb - 1) & 1) * I8_BK);
        const uint64_t db = (R256 && tb == 5) ? wgmma_desc_sw32(b0 + (unsigned)B_D5) : wgmma_desc_sw64(b0 + boff);
        wgmma_i8_rs(acc[d - 2], fa[sa - 1], db, (kt == 0 && lead) ? 0u : 1u);
        lead = false;
      }
    }
    wgmma_commit();
#pragma unroll
    for (int a = 0; a < NG; a++) wgmma_fence_operands(acc[a]);
    // the products of block kt - 1 are complete: its stage and its A fragments are free, in every CTA of the cluster
    wgmma_wait<1>();
#pragma unroll
    for (int sa = 0; sa < NS; sa++) wgmma_fence_operands(fa_prev[sa]);
    if (kt > 0 && lane == 0) {
#pragma unroll
      for (int c = 0; c < I8_CLUSTER; c++) mbar_arrive_cluster(&empty_bar[(kt - 1) % STAGES], (unsigned)c);
    }
  };
  for (int kt = 0; kt < nk; kt += 2) {
    block(kt, fa0, fa1);
    if (kt + 1 == nk) break;
    block(kt + 1, fa1, fa0);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int a = 0; a < NG; a++) wgmma_fence_operands(acc[a]);

  // Accumulator fragment of m64nN: register 4j + e of lane l in warp w (of the warpgroup) holds row
  // 16 w + l / 4 + 8 (e >> 1), column 8 j + 2 (l % 4) + (e & 1).
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const double rs0 = g.rowscale[(int64_t)rb * I8_BM + r0] * g.colscale;
  const double rs1 = g.rowscale[(int64_t)rb * I8_BM + r0 + 8] * g.colscale;
  constexpr int NC = BN / 4;                             // column slots of a thread
  double cs[NC];
#pragma unroll
  for (int i = 0; i < NACC; i++) {
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
    const int c = (i >> 2) * 2 + (i & 1);                // column slot of this thread
    if (i & 2) cs[c] += v * v; else cs[c] = v * v;
  }
  // sum each column slot over the 8 row groups of the warp (lanes with equal l % 4): fixed tree
#pragma unroll
  for (int c = 0; c < NC; c++) {
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 4);
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 8);
    cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], 16);
  }
  if (lane < 4) {
#pragma unroll
    for (int c = 0; c < NC; c++) colsum[warp * BN + (c >> 1) * 8 + 2 * lane + (c & 1)] = cs[c];
  }
  asm volatile("bar.sync 1, %0;\n" ::"n"(I8_CONSUMERS) : "memory");
  if (tid < BN && cb < g.n_cb) {                         // a CTA past the last tile stores nothing
    double t = colsum[tid];
#pragma unroll
    for (int w = 1; w < 8; w++) t += colsum[w * BN + tid];
    g.partial[(int64_t)rb * g.ld_partial + (int64_t)cb * BN + tid] = t;
  }
  cluster_sync();
}

}  // namespace dfb
