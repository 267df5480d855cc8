// Host-visible declarations of the TMA scoring kernel (kernel body: gemm_tma.cuh, built in kernels.cu).
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

int make_tensor_map_2d_f64(CUtensorMap* out, const double* base, int64_t rows, int64_t cols_ld,
                           int64_t cols);
int launch_score_tma(dfb_handle* h, const CUtensorMap& tmW, const CUtensorMap& tmK,
                     const ScoreTmaArgs& g);

struct ScoreI8Args;
constexpr int I8_BN = 32;    // candidates per tile of the int8 contraction (gemm_i8.cuh)
int make_tensor_map_3d_u8(CUtensorMap* out, const void* base, int64_t cols, int64_t rows, int64_t planes,
                          int64_t row_ld_bytes, int64_t plane_stride_bytes, int box_cols, int box_rows,
                          int box_planes);
int launch_row_exponent(dfb_handle* h, const double* M, int64_t ld, int64_t rows, int64_t cols,
                        double* rowscale, double* rowinv);
int launch_slice_i8(dfb_handle* h, const double* M, int64_t ld, int64_t rows, int64_t cols,
                    const double* rowinv, double inv_const, void* out, int64_t plane_bytes,
                    int64_t out_ld_bytes);
int launch_score_i8_args(dfb_handle* h, const CUtensorMap& tmA, const CUtensorMap& tmB, int n_rb, int n_cb, int K,
                         double* partial, int64_t ld_partial, const double* rowscale, double colscale,
                         const int* abort_count = nullptr);

}  // namespace dfb
