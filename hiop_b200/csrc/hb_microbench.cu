// In-run peak measurements for bench.py's roofline denominators:
//   * FP64 tensor pipe: mma.sync.m8n8k4.f64 (SASS DMMA.8x8x4, which = 0) or mma.sync.m16n8k16.f64 (SASS DMMA.16x8x16, which = 2)
//     issued back to back from registers by every warp of every SM. On sm_90a the two are different instructions, and
//     16x8x16 is the one the condensation kernel k_syrk_ws runs; 0 stays the 8x8x4 rate that bench.py has always reported.
//   * INT8 wgmma: wgmma.mma_async m64n256k32 s8 issued back to back by two warpgroups per SM on resident shared-memory operands
//     (no loads in the loop): the integer tensor-core rate k_oz_gemm draws on.
// Both are timed with CUDA events on the context stream over a few milliseconds, after a warm-up launch.
#include "hb_common.cuh"
#include "hb_ptx.cuh"

namespace {

// 8 independent accumulators per warp; SHAPE 0 = m8n8k4 (2 doubles each), 2 = m16n8k16 (4 doubles each)
template <int SHAPE>
__global__ void __launch_bounds__(256)
k_peak_dmma(double* __restrict__ out, int iters, double a, double b)
{
  double c[8][4];
  const double fa[8] = {a, b, a, b, a, b, a, b}, fb[4] = {a, b, a, b};
#pragma unroll
  for(int i = 0; i < 8; i++) { c[i][0] = threadIdx.x; c[i][1] = i; c[i][2] = 1; c[i][3] = 2; }
  for(int it = 0; it < iters; it++) {
#pragma unroll
    for(int i = 0; i < 8; i++) {
      if constexpr(SHAPE == 0) hb_dmma884(c[i][0], c[i][1], a, b);
      else hb_dmma16816(c[i], fa, fb);
    }
  }
  double s = 0;
#pragma unroll
  for(int i = 0; i < 8; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// best of 3 timed launches of k_peak_dmma<SHAPE> over 4 CTAs of 8 warps per SM, after a warm-up launch
template <int SHAPE>
int peak_dmma(hb_ctx* c, hb_event& e0, hb_event& e1, double* best)
{
  const int blocks = c->num_sms * 4, iters = 4000;
  const double mma_flop = SHAPE == 0 ? 2.0 * 8 * 8 * 4 : 2.0 * 16 * 8 * 16;
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (size_t)blocks * 256));
  k_peak_dmma<SHAPE><<<blocks, 256, 0, c->stream>>>((double*)c->ws, 100, 1.0000001, 1e-9);
  HB_LAUNCHED();
  float ms = 0.f;
  for(int rep = 0; rep < 3; rep++) {
    HB_CUDA(cudaEventRecord(e0, c->stream));
    k_peak_dmma<SHAPE><<<blocks, 256, 0, c->stream>>>((double*)c->ws, iters, 1.0000001, 1e-9);
    HB_LAUNCHED();
    HB_CUDA(cudaEventRecord(e1, c->stream));
    HB_CUDA(cudaEventSynchronize(e1));
    HB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
    const double tf = mma_flop * 8 * (double)iters * 8 * blocks / (ms * 1e-3) / 1e12; // 8 MMAs per warp per iteration, 8 warps
    if(tf > *best) *best = tf;
  }
  return HB_OK;
}

// one CTA per SM, two warpgroups: 16 KB A tile (128 rows x 128 B, 64 rows per warpgroup) + 32 KB B tile (256 rows x 128 B) in the
// SWIZZLE_128B K-major layout (contents do not matter for the rate), one m64n256 register accumulator per warpgroup
__global__ void __launch_bounds__(256, 1)
k_peak_i8(int iters, int* __restrict__ sink)
{
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024 - (hb_smem_addr(smem_raw) & 1023)) & 1023);
  const int tid = threadIdx.x, wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  for(int i = tid; i < (16 + 32) * 1024 / 4; i += 256) reinterpret_cast<uint32_t*>(smem)[i] = 0x01010101u * (i & 3);
  hb_fence_proxy_async_shared(); // generic-proxy writes of the operands -> visible to the tensor core
  __syncthreads();
  uint32_t acc[128];
#pragma unroll
  for(int i = 0; i < 128; i++) acc[i] = 0u;
  const uint32_t sa = hb_smem_addr(smem) + wg * 64 * 128, sb = hb_smem_addr(smem + 16 * 1024);
  for(int it = 0; it < iters; it++) {
    hb_wgmma_fence();
#pragma unroll
    for(int ks = 0; ks < 4; ks++) hb_wgmma_s8<8>(acc, hb_wgmma_desc_sw128(sa + ks * 32), hb_wgmma_desc_sw128(sb + ks * 32), 1);
    hb_wgmma_commit();
    hb_wgmma_wait<1>();
  }
  hb_wgmma_wait<0>();
  int s = 0;
#pragma unroll
  for(int i = 0; i < 128; i++) s += (int)acc[i];
  if(s == 0x7fffffff) sink[blockIdx.x] = s; // keeps the MMAs live
  if(tid == 0) sink[blockIdx.x] = iters;
}

constexpr int PEAK_I8_SMEM = 48 * 1024 + 1024; // + alignment slack

} // namespace

int hb_microbench_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_peak_i8, cudaFuncAttributeMaxDynamicSharedMemorySize, PEAK_I8_SMEM));
  return HB_OK;
}

// which: 0 = FP64 DMMA m8n8k4 (TFLOP/s), 1 = INT8 wgmma (TOP/s, 2 ops per MAC), 2 = FP64 DMMA m16n8k16 (TFLOP/s)
extern "C" int hb_microbench_peak(hb_ctx* c, int which, double* result_host)
{
  HB_REQUIRE(c && result_host && (which == 0 || which == 1 || which == 2), "hb_microbench_peak: bad arguments");
  HB_CUDA(cudaSetDevice(c->device));
  hb_event e0, e1;
  HB_CHECK(e0.create(cudaEventDefault));
  HB_CHECK(e1.create(cudaEventDefault));
  float ms = 0.f;
  double best = 0.0;
  if(which == 0) {
    HB_CHECK(peak_dmma<0>(c, e0, e1, &best));
  } else if(which == 2) {
    HB_CHECK(peak_dmma<2>(c, e0, e1, &best));
  } else {
    const int blocks = c->num_sms, iters = 20000;
    const int smem = PEAK_I8_SMEM;
    HB_CHECK(hb_ws_reserve(c, sizeof(int) * (size_t)blocks));
    k_peak_i8<<<blocks, 256, smem, c->stream>>>(200, (int*)c->ws.get());
    HB_LAUNCHED();
    for(int rep = 0; rep < 3; rep++) {
      HB_CUDA(cudaEventRecord(e0, c->stream));
      k_peak_i8<<<blocks, 256, smem, c->stream>>>(iters, (int*)c->ws.get());
      HB_LAUNCHED();
      HB_CUDA(cudaEventRecord(e1, c->stream));
      HB_CUDA(cudaEventSynchronize(e1));
      HB_CUDA(cudaEventElapsedTime(&ms, e0, e1));
      const double tops = 2.0 * 128 * 256 * 32 * 4.0 * (double)iters * blocks / (ms * 1e-3) / 1e12;
      if(tops > best) best = tops;
    }
  }
  *result_host = best;
  return HB_OK;
}
