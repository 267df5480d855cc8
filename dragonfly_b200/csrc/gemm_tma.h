// Host-visible declarations of the TMA kernels (kernel bodies: gemm_tma.cuh, factor_tma.cuh, gemm_i8.cuh, built in
// kernels.cu).
#pragma once
#include <cuda.h>
#include "common.cuh"

namespace dfb {

struct ScoreTmaArgs {
  int n_rb, n_cb, K;
  int cb_group;             // candidate tiles per scheduling group
  double* partial;
  int64_t ld_partial;
};

// fp64 map of a row-major rows x cols matrix (leading dimension cols_ld) in boxes of box_rows x 16 doubles, SWIZZLE_128B
int make_tensor_map_2d_f64(CUtensorMap* out, const double* base, int64_t rows, int64_t cols_ld,
                           int64_t cols, int box_rows = TILE);
int launch_score_tma(dfb_handle* h, const CUtensorMap& tmW, const CUtensorMap& tmK,
                     const ScoreTmaArgs& g);

// One launch of factor_update_kernel (factor_tma.cuh) on the tall matrix T (ld x (2 ld + 128)) of a factorisation, or
// with top_only on the square ld x ld alone.
struct FactorArgs {
  double* T; int64_t ld;
  int step, nb;
  int skip_bottom;          // the L^-T rows are absent (LML-only build)
  int top_only;             // factor only: neither the L^-T rows nor the y row exist (T is ld x ld)
  int panel;                // 1: panel solve of column block `step`; 0: trailing update of column blocks [j0, j1)
  int j0, j1;
  const int* info;          // nullable: do nothing if *info != 0 (failed factorisation)
};
// The tensor maps the launches of one factorisation read: T (rows x npad) in boxes of 32, 64 and 128 rows,
// inv(L_kk)^T.
struct FactorMaps {
  CUtensorMap t32, t64, t128, dinv;
};
int make_factor_maps(FactorMaps* out, const double* T, int64_t rows, int64_t npad, const double* Dinv);
// chain = true: the 32 x 128 sub-tiles of the critical path (panel(k), next(k)); false: the 128 x 64 bulk shape.
// Panel launches take the chain shape only.
int launch_factor_update(dfb_handle* h, const FactorMaps& m, const FactorArgs& g, bool chain);

struct ScoreI8Args;
// candidates per tile of the int8 contraction (gemm_i8.cuh) and rows of its K_* TMA box, per digit scheme
constexpr int i8_tile_n(bool radix256) { return radix256 ? 64 : 32; }
int make_tensor_map_3d_u8(CUtensorMap* out, const void* base, int64_t cols, int64_t rows, int64_t planes,
                          int64_t row_ld_bytes, int64_t plane_stride_bytes, int box_cols, int box_rows,
                          int box_planes);
// Maps of one operand of score_i8_kernel: three pair-interleaved planes of rows x 2K bytes each, back to back.  W
// (w_operand) is read in boxes of the rows one CTA of a cluster loads, K_* in boxes of one candidate tile.
int make_i8_maps(I8Maps* out, const void* planes, int64_t K, int64_t rows, bool w_operand, bool radix256);
int launch_row_exponent(dfb_handle* h, const double* M, int64_t ld, int64_t rows, int64_t cols,
                        double* rowscale, double* rowinv);
int launch_slice_i8(dfb_handle* h, const double* M, int64_t ld, int64_t rows, int64_t cols,
                    const double* rowinv, double inv_const, void* out, int64_t plane_bytes,
                    int64_t out_ld_bytes);
// radix256 selects the digit scheme of the planes behind tmA / tmB (the scoring path passes h->i8_radix256)
int launch_score_i8_args(dfb_handle* h, bool radix256, const I8Maps& tmA, const I8Maps& tmB, int n_rb,
                         int n_cb, int K, double* partial, int64_t ld_partial, const double* rowscale, double colscale,
                         const int* abort_count = nullptr);

}  // namespace dfb
