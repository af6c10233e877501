// Microbenchmark: FP64 issue rates on H100 (DFMA vs DMMA shapes) -- decides the condensation kernel design.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -Ihiop_b200/csrc -o tools/microbench_fp64 tools/microbench_fp64.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "hb_ptx.cuh"

#define CK(x) do { cudaError_t e = (x); if(e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while(0)

__global__ void k_dfma(double* out, int iters, double a, double b)
{
  double c[16];
#pragma unroll
  for(int i = 0; i < 16; i++) c[i] = threadIdx.x + i;
  for(int it = 0; it < iters; it++) {
#pragma unroll
    for(int i = 0; i < 16; i++) c[i] = fma(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for(int i = 0; i < 16; i++) s += c[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma884(double* out, int iters, double a, double b)
{
  double c[8][2];
#pragma unroll
  for(int i = 0; i < 8; i++) { c[i][0] = threadIdx.x; c[i][1] = i; }
  for(int it = 0; it < iters; it++) {
#pragma unroll
    for(int i = 0; i < 8; i++)
      hb_dmma884(c[i][0], c[i][1], a, b);
  }
  double s = 0;
#pragma unroll
  for(int i = 0; i < 8; i++) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma1688(double* out, int iters, double a, double b)
{
  double c[8][4];
  const double fa[4] = {a, b, a, b}, fb[2] = {a, b};
#pragma unroll
  for(int i = 0; i < 8; i++) { c[i][0] = threadIdx.x; c[i][1] = i; c[i][2] = 1; c[i][3] = 2; }
  for(int it = 0; it < iters; it++) {
#pragma unroll
    for(int i = 0; i < 8; i++) hb_dmma1688(c[i], fa, fb);
  }
  double s = 0;
#pragma unroll
  for(int i = 0; i < 8; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma16816(double* out, int iters, double a, double b)
{
  double c[8][4];
  const double fa[8] = {a, b, a, b, a, b, a, b}, fb[4] = {a, b, a, b};
#pragma unroll
  for(int i = 0; i < 8; i++) { c[i][0] = threadIdx.x; c[i][1] = i; c[i][2] = 1; c[i][3] = 2; }
  for(int it = 0; it < iters; it++) {
#pragma unroll
    for(int i = 0; i < 8; i++) hb_dmma16816(c[i], fa, fb);
  }
  double s = 0;
#pragma unroll
  for(int i = 0; i < 8; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_copy(const double4* __restrict__ in, double4* __restrict__ out, size_t n4)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for(; i < n4; i += stride) out[i] = in[i];
}
__global__ void k_read(const double4* __restrict__ in, double* out, size_t n4)
{
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  double s = 0;
  for(; i < n4; i += stride) { double4 v = in[i]; s += v.x + v.y + v.z + v.w; }
  if(s == 1.2345) out[0] = s;
}

int main()
{
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  printf("device %s SMs %d clock %d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  int nsm = p.multiProcessorCount;
  double* out; CK(cudaMalloc(&out, sizeof(double) * nsm * 8 * 1024));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 20000;
  float ms;
  for(int wpb = 4; wpb <= 16; wpb *= 2) {
    int threads = wpb * 32, blocks = nsm * (wpb >= 16 ? 2 : 4);
    // DFMA
    k_dfma<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaEventRecord(e0); k_dfma<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("DFMA      warps/blk %2d blocks %4d: %.2f TFLOP/s\n", wpb, blocks, 2.0 * 16 * iters * (double)threads * blocks / ms / 1e9);
    k_dmma884<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaEventRecord(e0); k_dmma884<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("DMMA 884  warps/blk %2d blocks %4d: %.2f TFLOP/s\n", wpb, blocks, 2.0 * 8 * 256 * iters * (double)wpb * blocks / ms / 1e9);
    k_dmma1688<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaEventRecord(e0); k_dmma1688<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("DMMA 1688 warps/blk %2d blocks %4d: %.2f TFLOP/s\n", wpb, blocks, 2.0 * 8 * 1024 * iters * (double)wpb * blocks / ms / 1e9);
    k_dmma16816<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaEventRecord(e0); k_dmma16816<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("DMMA 16816 warps/blk %2d blocks %4d: %.2f TFLOP/s\n", wpb, blocks, 2.0 * 8 * 2048 * iters * (double)wpb * blocks / ms / 1e9);
  }
  // HBM
  size_t bytes = (size_t)4 << 30;
  double4 *a, *b; CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes));
  CK(cudaMemset(a, 0, bytes)); CK(cudaMemset(b, 0, bytes));
  size_t n4 = bytes / sizeof(double4);
  for(int rep = 0; rep < 3; rep++) {
    cudaEventRecord(e0); k_copy<<<nsm * 16, 512>>>(a, b, n4); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("copy 4GiB: %.1f GB/s (r+w)\n", 2.0 * bytes / ms / 1e6);
    cudaEventRecord(e0); k_read<<<nsm * 16, 512>>>(a, out, n4); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    cudaEventElapsedTime(&ms, e0, e1);
    printf("read 4GiB: %.1f GB/s\n", 1.0 * bytes / ms / 1e6);
  }
  return 0;
}
