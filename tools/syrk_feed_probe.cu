// Probe: where does the time of the FP64 condensation kernel (k_syrk_ws, hiop_b200/csrc/hb_syrk.cu) go at the bench shape?
// Times the same warp-specialised structure (8 MMA warps, 4 producer warps, 3-stage full/empty mbarrier ring, 128x128 tiles,
// 32-column K chunks) in four variants:
//   full      as shipped: producers stream, MMA warps compute
//   mma-only  the MMA warps loop over one resident stage; the producers issue nothing
//   feed-only the producers stream; the MMA warps only release the stages
//   disjoint  feed-only, but every CTA reads data no other CTA reads (no L2 reuse: the DRAM-fed rate)
// for both K schedules: "streamk" (one contiguous range of the tile-major (tile, k) space per CTA) and "lanes" (CTAs grouped in
// K lanes so that all tiles of a lane read the same K window at the same time; the stream-K remainder as in hb_syrk.cu).
// Reports TFLOP/s executed and bytes/s moved from L2 into shared memory, the SM clock derived from clock64() over the kernel's
// duration, and the FP64 DMMA peaks of the library measured in the same process: m16n8k16 (hb_microbench_peak(2), the shape the
// kernel runs, against which "% of peak" is given) and m8n8k4 (hb_microbench_peak(0)).
// Build (after make -C hiop_b200/csrc):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Iinclude -Ihiop_b200/csrc -o tools/syrk_feed_probe tools/syrk_feed_probe.cu \
//        -Lhiop_b200 -lhiopb200 -Xlinker -rpath,'$ORIGIN/../hiop_b200'
// Run: tools/syrk_feed_probe [M=1012] [K=1000000]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "hiopb200.h"
#include "hb_ptx.cuh"

#define CK(x) do { cudaError_t e = (x); if(e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while(0)

namespace {
constexpr int BM = 128, WBK = 32, WSTAGES = 3, WLDS = WBK + 4, WTILE_D = BM * WLDS, WPROD = 128, WTHREADS = 256 + WPROD;
struct WStage { double a[WTILE_D]; double b[WTILE_D]; double d[WBK]; };
constexpr size_t WSMEM_BYTES = sizeof(WStage) * WSTAGES + 2 * BM * sizeof(const double*) + 2 * WSTAGES * sizeof(unsigned long long);
struct Seg { int ti, tj, k_begin, k_count, slot; };
enum { FULL = 0, MMA_ONLY = 1, FEED_ONLY = 2 };

template <int MODE>
__global__ void __launch_bounds__(WTHREADS, 1)
k_probe(const double* const* __restrict__ rowptr, int M, long long K, const double* __restrict__ dvec, const Seg* __restrict__ segs,
        const int* __restrict__ cta_seg_begin, double* __restrict__ ws, long long* __restrict__ cycles)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WStage* stages = reinterpret_cast<WStage*>(smem_raw);
  const double** srow = reinterpret_cast<const double**>(smem_raw + sizeof(WStage) * WSTAGES);
  unsigned long long* full = reinterpret_cast<unsigned long long*>(srow + 2 * BM);
  unsigned long long* empty = full + WSTAGES;
  const long long t0 = clock64();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if(MODE == MMA_ONLY)
    for(int e = tid; e < (int)(sizeof(WStage) / sizeof(double)); e += WTHREADS) reinterpret_cast<double*>(stages)[e] = 1e-3 * (e & 7);
  if(tid == 0) {
    for(int s = 0; s < WSTAGES; s++) { hb_mbar_init(&full[s], WPROD); hb_mbar_init(&empty[s], 8); }
    hb_mbar_init_fence();
  }
  __syncthreads();
  const int sb = cta_seg_begin[blockIdx.x], se = cta_seg_begin[blockIdx.x + 1];
  int stage = 0;
  unsigned phase = 0;
  if(warp >= 8) {
    hb_setmaxnreg_dec<40>();
    if(MODE == MMA_ONLY) return;
    const int p = tid - 256, kc = p & 15, r0 = p >> 4;
    for(int si = sb; si < se; si++) {
      const Seg sg = segs[si];
      const bool diag = sg.ti == sg.tj;
      hb_bar_sync<1, WPROD>();
      for(int r = p; r < 2 * BM; r += WPROD) {
        const int grow = (r < BM ? sg.ti * BM + r : sg.tj * BM + (r - BM));
        srow[r] = grow < M ? rowptr[grow] : nullptr;
      }
      hb_bar_sync<1, WPROD>();
      for(int it = 0; it < sg.k_count; it++) {
        const long long k = ((long long)sg.k_begin + it) * WBK + kc * 2;
        const long long rem = K - k;
        const int nb = rem >= 2 ? 16 : (rem == 1 ? 8 : 0);
        const long long koff = nb ? k : 0;
        hb_mbar_wait(&empty[stage], phase ^ 1);
        WStage& st = stages[stage];
#pragma unroll 4
        for(int j = 0; j < 16; j++) {
          const int row = r0 + 8 * j;
          const double* pa = srow[row];
          hb_cp_async16(&st.a[row * WLDS + kc * 2], pa ? pa + koff : (const double*)rowptr, pa ? nb : 0);
          if(!diag) {
            const double* pb = srow[BM + row];
            hb_cp_async16(&st.b[row * WLDS + kc * 2], pb ? pb + koff : (const double*)rowptr, pb ? nb : 0);
          }
        }
        if(p < 16 && dvec) hb_cp_async16(&st.d[kc * 2], nb ? dvec + k : (const double*)rowptr, nb);
        hb_mbar_arrive_cp_async(&full[stage]);
        if(++stage == WSTAGES) { stage = 0; phase ^= 1; }
      }
    }
    hb_cp_async_wait_all();
  } else {
    hb_setmaxnreg_inc<232>();
    const int warp_m = warp & 1, warp_n = warp >> 1, g = lane >> 2, t4 = lane & 3;
    for(int si = sb; si < se; si++) {
      const Seg sg = segs[si];
      const bool diag = sg.ti == sg.tj;
      double acc[4][4][4];
#pragma unroll
      for(int i = 0; i < 4; i++)
#pragma unroll
        for(int j = 0; j < 4; j++)
#pragma unroll
          for(int e = 0; e < 4; e++) acc[i][j][e] = 0.0;
      for(int it = 0; it < sg.k_count; it++) {
        if(MODE != MMA_ONLY) hb_mbar_wait(&full[stage], phase);
        if(MODE != FEED_ONLY) {
          const WStage& st = stages[MODE == MMA_ONLY ? 0 : stage];
          const double* sA = st.a + (warp_m * 64 + g) * WLDS + t4;
          const double* sB = (diag ? st.a : st.b) + (warp_n * 32 + g) * WLDS + t4;
#pragma unroll
          for(int kk = 0; kk < WBK; kk += 16) {
            double bf[4][4];
#pragma unroll
            for(int q = 0; q < 4; q++) {
              const double dv = st.d[kk + 4 * q + t4];
#pragma unroll
              for(int j = 0; j < 4; j++) bf[j][q] = sB[j * 8 * WLDS + kk + 4 * q] * dv;
            }
#pragma unroll
            for(int i = 0; i < 4; i++) {
              double af[8];
#pragma unroll
              for(int q = 0; q < 8; q++) af[q] = sA[(i * 16 + 8 * (q & 1)) * WLDS + kk + 4 * (q >> 1)];
#pragma unroll
              for(int j = 0; j < 4; j++) hb_dmma16816(acc[i][j], af, bf[j]);
            }
          }
        }
        if(MODE != MMA_ONLY) {
          __syncwarp();
          if(lane == 0) hb_mbar_arrive(&empty[stage]);
          if(++stage == WSTAGES) { stage = 0; phase ^= 1; }
        }
      }
      double* slot = ws + (size_t)sg.slot * (BM * BM);
#pragma unroll
      for(int i = 0; i < 4; i++)
#pragma unroll
        for(int h = 0; h < 2; h++)
#pragma unroll
          for(int j = 0; j < 4; j++)
            *reinterpret_cast<double2*>(slot + (warp_m * 64 + i * 16 + 8 * h + g) * BM + warp_n * 32 + j * 8 + t4 * 2) =
                make_double2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
    }
  }
  if(blockIdx.x == 0 && tid == 0) *cycles = clock64() - t0;
}

__global__ void k_fill(double* x, size_t n, unsigned seed)
{
  for(size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    unsigned h = (unsigned)i * 2654435761u ^ seed;
    h ^= h >> 13; h *= 0x5bd1e995u; h ^= h >> 15;
    x[i] = (double)(h & 0xffffff) * (1.0 / 16777216.0) + 0.5;
  }
}

struct Sched { std::vector<Seg> segs; std::vector<int> begin; long long bytes = 0, flops = 0; };

long long part(long long n, int p, int i) { return n / p * i + (i < n % p ? i : n % p); }

// kind 0: stream-K over the tile-major (tile, k) space; kind 1: K lanes + stream-K remainder (hb_syrk.cu's build_schedule);
// kind 2: disjoint -- one off-diagonal tile per CTA, CTAs sharing a panel read different K windows
Sched make_sched(int kind, int M, long long K, int G)
{
  const int T = (M + BM - 1) / BM, ntiles = T * (T + 1) / 2;
  const long long kiters = (K + WBK - 1) / WBK, total = (long long)ntiles * kiters;
  std::vector<int2> tij;
  for(int i = 0; i < T; i++)
    for(int j = i; j < T; j++) tij.push_back(make_int2(i, j));
  Sched S;
  auto push = [&](int tile, long long k0, long long cnt) {
    if(cnt > 0) S.segs.push_back(Seg{tij[tile].x, tij[tile].y, (int)k0, (int)cnt, (int)S.segs.size()});
  };
  auto streamk = [&](int cta0, int nct, long long kfirst) { // the (tile, k in [kfirst, kiters)) space over CTAs cta0..cta0+nct-1
    const long long w = kiters - kfirst, tot = (long long)ntiles * w;
    for(int c = 0; c < nct; c++) {
      S.begin[cta0 + c] = (int)S.segs.size();
      for(long long it = part(tot, nct, c), end = part(tot, nct, c + 1); it < end;) {
        const int tile = (int)(it / w);
        const long long kk0 = it % w, cnt = std::min(w - kk0, end - it);
        push(tile, kfirst + kk0, cnt);
        it += cnt;
      }
    }
  };
  S.begin.assign(G + 1, 0);
  if(kind == 2) {
    const long long w = kiters / G;
    for(int c = 0; c < G; c++) {
      S.begin[c] = (int)S.segs.size();
      int tile = c % ntiles;
      while(tij[tile].x == tij[tile].y) tile = (tile + 1) % ntiles;
      push(tile, (long long)c * w, w);
    }
  } else if(kind == 1 && G / ntiles >= 1 && total / G >= 1) {
    const int L = G / ntiles, R = G - L * ntiles;
    const long long w = R ? total / G : kiters / L;
    for(int lane = 0; lane < L; lane++)
      for(int t = 0; t < ntiles; t++) {
        const int c = lane * ntiles + t;
        S.begin[c] = (int)S.segs.size();
        const long long k0 = R ? lane * w : part(kiters, L, lane), k1 = R ? k0 + w : part(kiters, L, lane + 1);
        push(t, k0, k1 - k0);
      }
    if(R) streamk(L * ntiles, R, L * w);
  } else {
    streamk(0, G, 0);
  }
  S.begin[G] = (int)S.segs.size();
  for(const Seg& s : S.segs) {
    S.bytes += (long long)s.k_count * ((s.ti == s.tj ? 1 : 2) * BM * WBK + WBK) * 8;
    S.flops += (long long)s.k_count * BM * BM * WBK * 2;
  }
  return S;
}
} // namespace

int main(int argc, char** argv)
{
  const int M = argc > 1 ? atoi(argv[1]) : 1012;
  const long long K = argc > 2 ? atoll(argv[2]) : 1000000;
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  const int G = prop.multiProcessorCount;
  printf("device %s, %d SMs, M = %d, K = %lld\n", prop.name, G, M, K);
  hb_ctx* hc = nullptr;
  double peak = 0;
  double peak884 = 0;
  if(hb_ctx_create(0, &hc) != HB_OK || hb_microbench_peak(hc, 0, &peak884) != HB_OK || hb_microbench_peak(hc, 2, &peak) != HB_OK) {
    printf("hb_microbench_peak: %s\n", hb_last_error());
    return 1;
  }
  printf("FP64 DMMA peaks: m16n8k16 (hb_microbench_peak(2)) %.1f TFLOP/s, m8n8k4 (hb_microbench_peak(0)) %.1f TFLOP/s\n", peak, peak884);

  double *J, *d;
  CK(cudaMalloc(&J, sizeof(double) * (size_t)M * K));
  CK(cudaMalloc(&d, sizeof(double) * K));
  k_fill<<<G * 8, 256>>>(J, (size_t)M * K, 1u);
  k_fill<<<G * 8, 256>>>(d, (size_t)K, 2u);
  std::vector<const double*> rp(M);
  for(int i = 0; i < M; i++) rp[i] = J + (size_t)i * K;
  const double** rowptr; CK(cudaMalloc(&rowptr, sizeof(double*) * M));
  CK(cudaMemcpy(rowptr, rp.data(), sizeof(double*) * M, cudaMemcpyHostToDevice));
  long long* cyc; CK(cudaMalloc(&cyc, sizeof(long long)));
  CK(cudaFuncSetAttribute(k_probe<FULL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WSMEM_BYTES));
  CK(cudaFuncSetAttribute(k_probe<MMA_ONLY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WSMEM_BYTES));
  CK(cudaFuncSetAttribute(k_probe<FEED_ONLY>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WSMEM_BYTES));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);

  const char* sname[3] = {"streamk", "lanes", "disjoint"};
  for(int kind = 0; kind < 3; kind++) {
    Sched S = make_sched(kind, M, K, G);
    Seg* dsegs; int* dbeg; double* ws;
    CK(cudaMalloc(&dsegs, sizeof(Seg) * S.segs.size()));
    CK(cudaMalloc(&dbeg, sizeof(int) * S.begin.size()));
    CK(cudaMalloc(&ws, sizeof(double) * BM * BM * S.segs.size()));
    CK(cudaMemcpy(dsegs, S.segs.data(), sizeof(Seg) * S.segs.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dbeg, S.begin.data(), sizeof(int) * S.begin.size(), cudaMemcpyHostToDevice));
    const char* vname[3] = {"full", "mma-only", "feed-only"};
    for(int v = 0; v < 3; v++) {
      if(kind == 2 && v != FEED_ONLY) continue;
      auto launch = [&]() {
        if(v == FULL) k_probe<FULL><<<G, WTHREADS, WSMEM_BYTES>>>(rowptr, M, K, d, dsegs, dbeg, ws, cyc);
        if(v == MMA_ONLY) k_probe<MMA_ONLY><<<G, WTHREADS, WSMEM_BYTES>>>(rowptr, M, K, d, dsegs, dbeg, ws, cyc);
        if(v == FEED_ONLY) k_probe<FEED_ONLY><<<G, WTHREADS, WSMEM_BYTES>>>(rowptr, M, K, d, dsegs, dbeg, ws, cyc);
      };
      const int reps = kind == 2 ? 20 : 3;
      launch();
      CK(cudaDeviceSynchronize());
      float best = 1e30f, sum = 0;
      long long cycles = 0;
      for(int r = 0; r < reps; r++) {
        cudaEventRecord(e0); launch(); cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        sum += ms; best = ms < best ? ms : best;
        CK(cudaMemcpy(&cycles, cyc, sizeof(long long), cudaMemcpyDeviceToHost));
      }
      const float ms = sum / reps;
      printf("%-8s %-9s  %8.2f ms (best %8.2f)  SM clock %4.0f MHz", sname[kind], vname[v], ms, best, cycles / (ms * 1e3));
      if(v != FEED_ONLY) printf("  %5.1f TFLOP/s executed (%.0f%% of peak)", S.flops / (ms * 1e9), 100.0 * S.flops / (ms * 1e9) / peak);
      if(v != MMA_ONLY) printf("  %5.2f TB/s into SMs (%.1f GB)", S.bytes / (ms * 1e9), S.bytes / 1e9);
      printf("\n");
    }
    cudaFree(dsegs); cudaFree(dbeg); cudaFree(ws);
  }
  cudaFree(J); cudaFree(d); cudaFree(rowptr); cudaFree(cyc);
  hb_ctx_destroy(hc);
  return 0;
}
