// Live roofline denominators for bench.py (dfb_measure_peak): the issue rate of int8 wgmma and of fp64 DMMA.8x8x4 on the
// device the bench runs on, measured in the same process as the timed step instead of being quoted from an earlier
// run.  Not on the product path.
#include "common.cuh"

namespace dfb {

__device__ __forceinline__ unsigned ub_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// One CTA per SM, two warpgroups; operands are whatever sits in shared memory (SWIZZLE_128B K-major descriptors), each
// warpgroup issues 8 x iters wgmma.m64n256k32.s32.s8.s8 into one register accumulator and waits for them at the end.
__global__ void __launch_bounds__(256, 1) ub_i8_rate_kernel(int iters, int* sink) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* tiles = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const unsigned a0 = ub_smem_u32(tiles), b0 = a0 + 8192;     // A: 64 rows x 128 B, B: 256 rows x 128 B
  const uint64_t HI = ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
  int d[128];
#pragma unroll
  for (int i = 0; i < 128; i++) d[i] = 0;
  asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory");
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const uint64_t da = HI | (uint64_t)((((a0 + (j & 3) * 32) & 0x3FFFFu) >> 4) | 0x10000u);
      const uint64_t db = HI | (uint64_t)((((b0 + (j & 3) * 32) & 0x3FFFFu) >> 4) | 0x10000u);
      asm volatile(
          "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 "
          "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,"
          "%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,"
          "%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,"
          "%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,"
          "%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, 1;\n"
          : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
            "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
            "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
            "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
            "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
            "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
            "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
            "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]),
            "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]),
            "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]),
            "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]),
            "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]),
            "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]),
            "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
            "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]),
            "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]),
            "+r"(d[126]), "+r"(d[127])
          : "l"(da), "l"(db)
          : "memory");
    }
  }
  asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory");
  asm volatile("wgmma.wait_group.sync.aligned 0;\n" ::: "memory");
  int x = 0;
#pragma unroll
  for (int i = 0; i < 128; i++) x ^= d[i];
  sink[blockIdx.x * blockDim.x + threadIdx.x] = x;
}

// 16 warps per SM, 8 independent DMMA.8x8x4 accumulators per thread
__global__ void ub_dmma_rate_kernel(double* out, int iters) {
  double c[8][2];
#pragma unroll
  for (int i = 0; i < 8; i++) { c[i][0] = 0; c[i][1] = 0; }
  const double av = 1.0 + threadIdx.x * 1e-9, bv = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < 8; i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(av), "d"(bv));
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

}  // namespace dfb

using namespace dfb;

extern "C" int dfb_measure_peak(int device, int what, double* out) {
  if (out == nullptr || (what != DFB_PEAK_I8 && what != DFB_PEAK_DMMA_F64)) { set_error("bad measure_peak arguments"); return -1; }
  DFB_CUDA_OK(cudaSetDevice(device));
  int sms = 0;
  DFB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  cudaEvent_t e0, e1;
  DFB_CUDA_OK(cudaEventCreate(&e0));
  DFB_CUDA_OK(cudaEventCreate(&e1));
  void* scratch = nullptr;
  DFB_CUDA_OK(cudaMalloc(&scratch, sizeof(double) * (size_t)sms * 512 + 4096));
  float best = 1e30f;
  double work = 0.0;
  if (what == DFB_PEAK_I8) {
    const size_t smem = 8192 + 32768 + 1024;
    DFB_CUDA_OK(cudaFuncSetAttribute(ub_i8_rate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int iters = 8000;
    ub_i8_rate_kernel<<<sms, 256, smem>>>(200, (int*)scratch);
    DFB_CUDA_OK(cudaDeviceSynchronize());
    for (int rep = 0; rep < 3; rep++) {
      DFB_CUDA_OK(cudaEventRecord(e0));
      ub_i8_rate_kernel<<<sms, 256, smem>>>(iters, (int*)scratch);
      DFB_CUDA_OK(cudaEventRecord(e1));
      DFB_CUDA_OK(cudaEventSynchronize(e1));
      float ms = 0.f;
      DFB_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
      if (ms < best) best = ms;
    }
    work = 2.0 * 2 * 64.0 * 256.0 * 32.0 * 8.0 * iters * sms;     // int8 ops (2 per MAC), two warpgroups
  } else {
    const int iters = 8000, threads = 512;
    ub_dmma_rate_kernel<<<sms, threads>>>((double*)scratch, 100);
    DFB_CUDA_OK(cudaDeviceSynchronize());
    for (int rep = 0; rep < 3; rep++) {
      DFB_CUDA_OK(cudaEventRecord(e0));
      ub_dmma_rate_kernel<<<sms, threads>>>((double*)scratch, iters);
      DFB_CUDA_OK(cudaEventRecord(e1));
      DFB_CUDA_OK(cudaEventSynchronize(e1));
      float ms = 0.f;
      DFB_CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
      if (ms < best) best = ms;
    }
    work = 2.0 * 256.0 * 8.0 * (double)iters * (threads / 32) * sms;   // flops
  }
  cudaFree(scratch);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *out = work / (best * 1e-3) * 1e-12;       // TOP/s or TFLOP/s
  return 0;
}
