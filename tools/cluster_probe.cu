// Probe: cost of one "post to all CTAs of a 16-CTA cluster + synchronise" round on H100, three ways:
//   (a) st.shared::cluster (generic DSM store) + cluster.sync()  (barrier.cluster.arrive.release / wait.acquire)
//   (b) st.async ... mbarrier::complete_tx to every CTA + local mbarrier wait (no cluster barrier, no fence)
//   (c) cluster.sync() alone, and __syncthreads alone, for reference
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -Ihiop_b200/csrc -o tools/cluster_probe tools/cluster_probe.cu
#include <cooperative_groups.h>
#include <cstdio>
#include <cuda_runtime.h>
#include "hb_ptx.cuh"
namespace cg = cooperative_groups;
constexpr int CS = 16;

__global__ void __cluster_dims__(CS, 1, 1) k_probe(int iters, int mode, long long* out)
{
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = cluster.block_rank(), tid = threadIdx.x;
  __shared__ double box[2][CS];
  __shared__ unsigned long long bar[2];
  if(tid == 0) {
    for(int p = 0; p < 2; p++) hb_mbar_init(&bar[p], 1);
    hb_mbar_init_fence();
  }
  __syncthreads();
  cluster.sync();
  double acc = 0.0;
  unsigned phase[2] = {0, 0};
  const long long t0 = clock64();
  for(int it = 0; it < iters; it++) {
    const int p = it & 1;
    if(mode == 0) {
      if(tid < CS) cluster.map_shared_rank(&box[p][0], tid)[rank] = (double)(it + rank);
      cluster.sync();
    } else if(mode == 1) {
      if(tid == 0) hb_mbar_arrive_expect_tx(&bar[p], CS * 8);
      if(tid < CS) {
        const double v = (double)(it + rank);
        hb_st_async_b64(hb_mapa(&box[p][rank], tid), __double_as_longlong(v), hb_mapa(&bar[p], tid));
      }
      while(!hb_mbar_try_wait(&bar[p], phase[p])) {}
      phase[p] ^= 1;
    } else if(mode == 2) {
      cluster.sync();
    } else {
      __syncthreads();
    }
    acc += box[p][(tid + it) & (CS - 1)];
  }
  const long long t1 = clock64();
  cluster.sync();
  if(tid == 0 && rank == 0) { out[0] = t1 - t0; out[1] = (long long)acc; }
}

int main()
{
  long long* d;
  cudaMalloc(&d, 16);
  cudaFuncSetAttribute(k_probe, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
  const char* names[] = {"DSM store + cluster.sync", "st.async + mbarrier wait", "cluster.sync only", "__syncthreads only"};
  for(int threads : {128, 512, 1024})
    for(int mode = 0; mode < 4; mode++) {
      const int iters = 2000;
      k_probe<<<CS, threads>>>(iters, mode, d);
      cudaError_t e = cudaDeviceSynchronize();
      long long h[2] = {0, 0};
      cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
      printf("threads %4d  %-28s %8.1f cycles/round  (%s)\n", threads, names[mode], (double)h[0] / iters, cudaGetErrorString(e));
    }
  return 0;
}
