// Micro-benchmark: fp64 DMMA.8x8x4 vs DFMA issue rate on H100 (sm_90a).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_fp64 ubench_fp64.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("CUDA error %s at %d\n",cudaGetErrorString(e),__LINE__); return 1;}}while(0)

template<int NACC>
__global__ void dmma_kernel(double* out, int iters) {
  double c[NACC][2];
#pragma unroll
  for (int i=0;i<NACC;i++){c[i][0]=0;c[i][1]=0;}
  double av = 1.0 + threadIdx.x*1e-9, bv = 1.0 - threadIdx.x*1e-9;
  for (int it=0; it<iters; it++) {
#pragma unroll
    for (int i=0;i<NACC;i++)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(av), "d"(bv));
  }
  double s=0;
#pragma unroll
  for (int i=0;i<NACC;i++) s+=c[i][0]+c[i][1];
  out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
template<int NACC>
__global__ void dfma_kernel(double* out, int iters) {
  double c[NACC];
#pragma unroll
  for (int i=0;i<NACC;i++) c[i]=i;
  double av = 1.0 + threadIdx.x*1e-9, bv = 1e-9*threadIdx.x;
  for (int it=0; it<iters; it++) {
#pragma unroll
    for (int i=0;i<NACC;i++) c[i] = fma(c[i], av, bv);
  }
  double s=0;
#pragma unroll
  for (int i=0;i<NACC;i++) s+=c[i];
  out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
// mixed: DMMA + DFMA interleaved, to see whether they share a pipe
template<int NACC>
__global__ void mixed_kernel(double* out, int iters) {
  double c[NACC][2]; double f[NACC];
#pragma unroll
  for (int i=0;i<NACC;i++){c[i][0]=0;c[i][1]=0;f[i]=i;}
  double av = 1.0 + threadIdx.x*1e-9, bv = 1.0 - threadIdx.x*1e-9;
  for (int it=0; it<iters; it++) {
#pragma unroll
    for (int i=0;i<NACC;i++) {
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(av), "d"(bv));
      f[i] = fma(f[i], av, bv);
    }
  }
  double s=0;
#pragma unroll
  for (int i=0;i<NACC;i++) s+=c[i][0]+c[i][1]+f[i];
  out[blockIdx.x*blockDim.x+threadIdx.x]=s;
}
int main(){
  int dev=0; CK(cudaSetDevice(dev));
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p,dev));
  int clk=0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, dev);
  printf("device %s SMs %d clock %d kHz\n", p.name, p.multiProcessorCount, clk);
  double* out; CK(cudaMalloc(&out, sizeof(double)*1024*1024*8));
  cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int sms=p.multiProcessorCount;
  for (int warps=4; warps<=32; warps*=2) {
    int threads=warps*32; int blocks=sms; int iters=20000;
    float ms;
    dmma_kernel<8><<<blocks,threads>>>(out,100); CK(cudaDeviceSynchronize());
    cudaEventRecord(e0); dmma_kernel<8><<<blocks,threads>>>(out,iters); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms,e0,e1);
    double flops = 2.0*256*8*(double)iters*warps*blocks;
    printf("DMMA  warps/SM=%2d: %.3f ms  %.2f TFLOP/s  (%.1f FMA/clk/SM @1.965GHz)\n", warps, ms, flops/ms*1e-9, flops/2/(ms*1e-3)/sms/1.965e9);
    dfma_kernel<8><<<blocks,threads>>>(out,100); CK(cudaDeviceSynchronize());
    cudaEventRecord(e0); dfma_kernel<8><<<blocks,threads>>>(out,iters); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms,e0,e1);
    flops = 2.0*32*8*(double)iters*warps*blocks;
    printf("DFMA  warps/SM=%2d: %.3f ms  %.2f TFLOP/s  (%.1f FMA/clk/SM @1.965GHz)\n", warps, ms, flops/ms*1e-9, flops/2/(ms*1e-3)/sms/1.965e9);
    mixed_kernel<8><<<blocks,threads>>>(out,100); CK(cudaDeviceSynchronize());
    cudaEventRecord(e0); mixed_kernel<8><<<blocks,threads>>>(out,iters); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms,e0,e1);
    flops = 2.0*(256+32)*8*(double)iters*warps*blocks;
    printf("MIXED warps/SM=%2d: %.3f ms  %.2f TFLOP/s\n", warps, ms, flops/ms*1e-9);
  }
  return 0;
}
