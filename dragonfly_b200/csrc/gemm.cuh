// fp64 tensor-core (DMMA.8x8x4) "TN" GEMM for sm_90a:
//
//     acc[i][j] = sum_{k in [0, k_hi)} A[i, k] * B[j, k]          (both operands K-contiguous)
//
// One CTA = one 128 x 128 output tile, 8 warps (2 x 4), warp tile 64 x 32, K pipelined in slabs of
// 16 doubles (128 B per row) through a 4-stage cp.async ring in shared memory.  wgmma has no f64
// kind, so the fp64 contraction runs on the warp-level DMMA path (SASS: DMMA.8x8x4), the FP64 tensor
// core rate of the SM (dfb_measure_peak and tools/ubench_fp64.cu measure it).
//
// The same core serves every dense contraction of the path through a `mode` (which tiles exist and
// which k-range each needs) and an epilogue:
//   MODE_SCORE  + EPI_SUMSQ : V = W K_*^T with W = L^-1 lower triangular (k < (rb+1)*128) and the
//                             fused reduction |v|^2 per candidate column -- V is never stored.
//                             Replaces solve_lower_triangular(L, K_tetr.T) + V.T.dot(V) + diag
//                             (dragonfly/gp/gp_core.py:180-187).
//   MODE_GENERIC+ EPI_STORE : plain tiles (posterior covariance / Thompson sampling blocks)
#pragma once
#include "common.cuh"

namespace dfb {

constexpr int GEMM_THREADS = 256;
constexpr int GEMM_STAGES = 4;
constexpr int GEMM_SROW = GEMM_BK + 4;                    // padded smem row: 20 doubles (160 B)
constexpr int GEMM_STAGE_DOUBLES = 2 * TILE * GEMM_SROW;  // A slab + B slab
constexpr size_t GEMM_SMEM_BYTES = (size_t)GEMM_STAGES * GEMM_STAGE_DOUBLES * sizeof(double);

enum { MODE_SCORE = 0, MODE_GENERIC = 1 };
enum { EPI_STORE = 0, EPI_SUMSQ = 1 };

struct GemmArgs {
  const double* A; int64_t lda;
  const double* B; int64_t ldb;
  const double* C; int64_t ldc;     // nullable: D = alpha * acc (+ C)
  double* D; int64_t ldd;
  double alpha;
  int mode;
  int n_rb, n_cb;                   // SCORE / GENERIC: tile grid
  int K;                            // k extent (multiple of 16)
  int tri;                          // GENERIC: 0 full K, 1 A lower-tri (k < (rb+1)*128), 2 B lower-tri,
                                    //   3 both operands UPPER-tri (k >= max(rb, cb)*128): W^T W from L^-T
  int lower_only;                   // GENERIC: skip tiles with cb > rb
  int rb0;                          // GENERIC: global index of row block 0 (A / C / D already point at it): the
                                    //   triangular ranges and lower_only refer to rb0 + rb
  int ksplit;                       // GENERIC: > 1 = split the k-range of every tile over `ksplit` CTAs; slice s writes
  double* part;                     //   alpha * (its partial sum) to part + s * (n_rb*128) * (n_cb*128) (compact tiles grid,
                                    //   ld = n_cb*128) and splitk_reduce_kernel adds the slices in a fixed order (+ C)
  double* partial; int64_t ld_partial;   // SUMSQ output [n_rb][ld_partial]
  const int* info;                  // nullable: do nothing if *info != 0 (failed factorisation)
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_tn_kernel(const GemmArgs g) {
  extern __shared__ __align__(16) double smem[];
  if (g.info != nullptr && *g.info != 0) return;

  // ---- decode which tile this CTA owns ---------------------------------------------------------
  const int bid = blockIdx.x;
  const double* A; const double* B; const double* C = nullptr; double* D = nullptr;
  int rb = 0, cb = 0, k_hi = g.K, k_lo = 0;
  int64_t ldd = g.ldd;
  if (g.mode == MODE_SCORE) {
    rb = g.n_rb - 1 - bid / g.n_cb;          // heaviest (longest k-range) row blocks first
    cb = bid % g.n_cb;
    A = g.A + (int64_t)rb * TILE * g.lda;
    B = g.B + (int64_t)cb * TILE * g.ldb;
    k_hi = min(g.K, (rb + 1) * TILE);
  } else {
    const int ks = g.ksplit > 1 ? g.ksplit : 1;
    const int tile = bid / ks, slice = bid - tile * ks;
    rb = tile / g.n_cb;
    cb = tile % g.n_cb;
    const int rbg = rb + g.rb0;
    if (g.lower_only && cb > rbg) return;
    A = g.A + (int64_t)rb * TILE * g.lda;
    B = g.B + (int64_t)cb * TILE * g.ldb;
    if (g.tri == 1) k_hi = min(g.K, (rbg + 1) * TILE);
    else if (g.tri == 2) k_hi = min(g.K, (cb + 1) * TILE);
    else if (g.tri == 3 && ks == 1) { k_lo = min(g.K, max(rbg, cb) * TILE); A += k_lo; B += k_lo; }
    if (ks > 1) {
      // slice `slice` of this tile's k-range, in multiples of the pipeline stage; empty slices store zeros
      const int chunk = ((k_hi + ks - 1) / ks + GEMM_BK - 1) / GEMM_BK * GEMM_BK;
      k_lo = min(k_hi, slice * chunk);
      k_hi = min(k_hi, k_lo + chunk);
      ldd = (int64_t)g.n_cb * TILE;
      D = g.part + (int64_t)slice * g.n_rb * TILE * ldd + (int64_t)rb * TILE * ldd + (int64_t)cb * TILE;
      A += k_lo; B += k_lo;
    } else {
      if (g.C) C = g.C + (int64_t)rb * TILE * g.ldc + (int64_t)cb * TILE;
      D = g.D + (int64_t)rb * TILE * g.ldd + (int64_t)cb * TILE;
    }
  }
  const int64_t lda = g.lda, ldb = g.ldb, ldc = g.ldc;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 2, wn = warp & 3;
  const int nk = (k_hi - k_lo) / GEMM_BK;

  // ---- global -> shared loader: 8 threads cover one 128 B row slab, 32 rows per pass ------------
  const int ld_row = tid >> 3;
  const int ld_kc = (tid & 7) * 2;
  const double* a_src = A + (int64_t)ld_row * lda + ld_kc;
  const double* b_src = B + (int64_t)ld_row * ldb + ld_kc;
  auto load_stage = [&](int stage, int kt) {
    double* As = smem + stage * GEMM_STAGE_DOUBLES;
    double* Bs = As + TILE * GEMM_SROW;
    const double* a = a_src + kt * GEMM_BK;
    const double* b = b_src + kt * GEMM_BK;
#pragma unroll
    for (int r = 0; r < 4; r++) {
      cp_async16(As + (ld_row + 32 * r) * GEMM_SROW + ld_kc, a + (int64_t)(32 * r) * lda);
      cp_async16(Bs + (ld_row + 32 * r) * GEMM_SROW + ld_kc, b + (int64_t)(32 * r) * ldb);
    }
  };

  double c[8][4][2];
#pragma unroll
  for (int mi = 0; mi < 8; mi++)
#pragma unroll
    for (int ni = 0; ni < 4; ni++) { c[mi][ni][0] = 0.0; c[mi][ni][1] = 0.0; }

  // ---- software pipeline ---------------------------------------------------------------------------
#pragma unroll
  for (int s = 0; s < GEMM_STAGES - 1; s++) {
    if (s < nk) load_stage(s, s);
    cp_async_commit();
  }
  const int fr = lane >> 2, fk = lane & 3;
  const int a_off = (wm * 64 + fr) * GEMM_SROW + fk;
  const int b_off = TILE * GEMM_SROW + (wn * 32 + fr) * GEMM_SROW + fk;
  for (int kt = 0; kt < nk; kt++) {
    cp_async_wait<GEMM_STAGES - 2>();
    __syncthreads();
    {
      const int nxt = kt + GEMM_STAGES - 1;
      if (nxt < nk) load_stage(nxt % GEMM_STAGES, nxt);
      cp_async_commit();
    }
    const double* St = smem + (kt % GEMM_STAGES) * GEMM_STAGE_DOUBLES;
#pragma unroll
    for (int kk = 0; kk < GEMM_BK / 4; kk++) {
      double a[8], b[4];
#pragma unroll
      for (int mi = 0; mi < 8; mi++) a[mi] = St[a_off + mi * 8 * GEMM_SROW + kk * 4];
#pragma unroll
      for (int ni = 0; ni < 4; ni++) b[ni] = St[b_off + ni * 8 * GEMM_SROW + kk * 4];
#pragma unroll
      for (int mi = 0; mi < 8; mi++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++) dmma884(c[mi][ni][0], c[mi][ni][1], a[mi], b[ni]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  // ---- epilogue ----------------------------------------------------------------------------------------
  if (EPI == EPI_SUMSQ) {
    // column sums of squares over this tile's 128 rows -> partial[rb][cb*128 + col]
    double* red = smem;  // [2][128]
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
    __syncthreads();
    if (tid < TILE)
      g.partial[(int64_t)rb * g.ld_partial + (int64_t)cb * TILE + tid] = red[tid] + red[TILE + tid];
  } else {
    const double alpha = g.alpha;
#pragma unroll
    for (int mi = 0; mi < 8; mi++) {
      const int row = wm * 64 + mi * 8 + fr;
#pragma unroll
      for (int ni = 0; ni < 4; ni++) {
        const int col = wn * 32 + ni * 8 + 2 * fk;
        double2 v;
        v.x = alpha * c[mi][ni][0];
        v.y = alpha * c[mi][ni][1];
        if (C != nullptr) {
          const double2 cc = *reinterpret_cast<const double2*>(C + (int64_t)row * ldc + col);
          v.x += cc.x;
          v.y += cc.y;
        }
        *reinterpret_cast<double2*>(D + (int64_t)row * ldd + col) = v;
      }
    }
  }
}

// Host-side launchers (defined in kernels.cu).  launch_gemm_splitk runs a MODE_GENERIC product with every tile's
// k-range split over `ksplit` CTAs (scratch: ksplit * n_rb*128 * n_cb*128 doubles at `part`) followed by the
// fixed-order reduction D = C + sum_s part_s: for the skinny products of dfb_extend_posterior, whose 1..40 tiles
// would otherwise occupy 1..40 of the 132 SMs for a k-depth of ~N.
int launch_gemm(dfb_handle* h, const GemmArgs& g, int epi, int n_blocks);
int launch_gemm_splitk(dfb_handle* h, GemmArgs g, int ksplit, double* part);

}  // namespace dfb
