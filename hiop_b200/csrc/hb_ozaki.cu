// C = A diag(d) A^T on the Hopper tensor cores (wgmma.mma_async s8 x s8 -> s32, accumulators in registers, operands by TMA):
// FP64 emulation by integer slicing (Ozaki scheme).
//
//   B = A diag(sqrt(d));   row i:  b_ik = 2^{e_i} * sum_p q_p(i,k) 2^{-(6+7p)} + O(2^{e_i - 6 - 7S}),  q_p int8, |q_p| <= 64
//   C_ij = 2^{e_i+e_j} * sum_{t=0}^{S-1} 2^{-(12+7t)} T_t(i,j),     T_t = sum_{p+q=t} Q_p Q_q^T   (exact int32)
//
// wgmma has no f64 kind; this is the only way the K ~ 1e6, M ~ 1e3 condensation can use the integer tensor pipe. Every
// integer product and accumulation is exact (K is cut into chunks so that (t+1)*Kc*2^12 < 2^31); the only error is the
// truncation of b after 6+7(S-1) bits relative to each row's largest entry (S=7: 2^-48, S=8: 2^-55) plus the final FP64
// recombination. The exact FP64 DMMA kernel (hb_syrk.cu) stays as the reference path and as the fallback.
//
// Pipeline of k_oz_gemm (384 threads, one CTA per SM, 128x32 output tiles, split-K):
//   warp 8 (1 thread)  TMA producer (its warpgroup hands its registers to the consumers with setmaxnreg): per 128-byte K block one box {128 B x 32 rows x S slices} (B) and S boxes
//                      {128 B x 128 rows} (A) from the 3-D tensor map (k, row, slice), SWIZZLE_128B, mbarrier completion
//   warps 0-7          two consumer warpgroups, rows 0-63 and 64-127 of the tile: wgmma m64n32k32 per slice pair,
//                      S register accumulators of 64x32 int32 (one per t = p+q, 16 registers a thread each); at
//                      every K-chunk boundary they recombine them in FP64 and accumulate into the CTA's FP64 partial tile
//                      (workspace, L2 resident)
// The 128x32 tile keeps the S = 8 accumulators at 128 registers a thread (a 64-column tile would need 256); the consumers run
// with 232 registers, the producer warpgroup with 40.
// A last kernel sums the split-K partials in fixed order, applies 2^{e_i+e_j} and mirrors the tile (deterministic).
#include "hb_common.cuh"
#include "hb_ptx.cuh"
#include <cuda.h>
#include <cstdlib>

namespace {

constexpr int TM = 128, TN = 32;
constexpr int KS = 128;           // bytes of K per block (one SWIZZLE_128B row = four MMA K steps)
constexpr int A_TILE = TM * KS;   // 16 KB per slice
constexpr int B_TILE = TN * KS;   // 4 KB per slice
constexpr int OZ_CONSUMERS = 256; // two warpgroups
constexpr int OZ_THREADS = OZ_CONSUMERS + 128; // + the producer warpgroup
constexpr unsigned OZ_SUSPEND_NS = 10000000u;  // suspend-time hint of every mbarrier wait of k_oz_gemm (its SASS differs without it)

// ---------------------------------------------------------------------------------------------------------------------
// slicing
// ---------------------------------------------------------------------------------------------------------------------
// row maxima of |a_ik| * sd_k  (sd = sqrt(d) or 1): integer atomicMax on the bit pattern of a non-negative double
__global__ void __launch_bounds__(256)
k_oz_rowmax(const double* const* __restrict__ rowptr, int M, long long K, const double* __restrict__ sd, unsigned long long* __restrict__ mx)
{
  const int row = blockIdx.y;
  const double* a = rowptr[row];
  double m = 0.0;
  const long long stride = (long long)gridDim.x * 256;
  for(long long k = (long long)blockIdx.x * 256 + threadIdx.x; k < K; k += stride) m = fmax(m, fabs(a[k]) * (sd ? sd[k] : 1.0));
  m = hb_warp_max(m);
  if((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(&mx[row], (unsigned long long)__double_as_longlong(m));
}
// Row maxima AND the row dot products with t = d .* x in the same pass over the rows (a5/a13: J (H+Dx)^-1-weighted rhs, step 2 of
// solveCompressed, costs no second sweep over J when the condensation is pending anyway). A CTA owns RD_COLS columns: each lane keeps
// the sqrt(d) and d.*x values of its columns in registers and the 16 warps stream the rows past them, RD_ROWS rows in flight per warp.
// partial[chunk][row] is combined in a fixed order by k_oz_dot_final; the maxima go through the same order-independent atomicMax.
constexpr int RD_THREADS = 512, RD_COLS = 256, RD_ROWS = 4;
template <bool VEC>
__global__ void __launch_bounds__(RD_THREADS)
k_oz_rowmax_dot(const double* const* __restrict__ rowptr, int M, long long K, const double* __restrict__ d, const double* __restrict__ x,
                unsigned long long* __restrict__ mx, double* __restrict__ partial)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long k0 = (long long)blockIdx.x * RD_COLS;
  const int len = (int)min((long long)RD_COLS, K - k0);
  double sd[8], w[8];
  // slot p of a lane: VEC -> the pair of columns 2*(lane + 32*(p/2)) + (p&1); scalar -> column lane + 32*p (relative to k0)
#define RD_OFF(p) (VEC ? 2 * (lane + 32 * ((p) >> 1)) + ((p) & 1) : lane + 32 * (p))
#pragma unroll
  for(int p = 0; p < 8; p++) {
    const int off = RD_OFF(p);
    if(off < len) {
      const double dv = d ? d[k0 + off] : 1.0;
      sd[p] = d ? sqrt(dv) : 1.0;
      w[p] = dv * x[k0 + off];
    } else {
      sd[p] = 0.0;
      w[p] = 0.0;
    }
  }
  const int wstride = (RD_THREADS / 32) * gridDim.y;
  for(int i0 = warp + (RD_THREADS / 32) * blockIdx.y; i0 < M; i0 += wstride * RD_ROWS) {
    double v[RD_ROWS][8];
#pragma unroll
    for(int r = 0; r < RD_ROWS; r++) {
      const int i = i0 + r * wstride;
      const double* row = i < M ? rowptr[i] + k0 : nullptr;
#pragma unroll
      for(int p = 0; p < (VEC ? 4 : 8); p++) {
        if(VEC) {
          double2 t = make_double2(0.0, 0.0);
          if(row && RD_OFF(2 * p) < len) t = *reinterpret_cast<const double2*>(row + RD_OFF(2 * p));
          v[r][2 * p] = t.x;
          v[r][2 * p + 1] = t.y;
        } else {
          v[r][p] = (row && RD_OFF(p) < len) ? row[RD_OFF(p)] : 0.0;
        }
      }
    }
#pragma unroll
    for(int r = 0; r < RD_ROWS; r++) {
      const int i = i0 + r * wstride;
      double mm = 0.0, acc = 0.0;
#pragma unroll
      for(int p = 0; p < 8; p++) {
        mm = fmax(mm, fabs(v[r][p]) * sd[p]);
        acc += v[r][p] * w[p];
      }
      mm = hb_warp_max(mm);
      acc = hb_warp_sum(acc);
      if(lane == 0 && i < M) {
        if(mm > 0.0) atomicMax(&mx[i], (unsigned long long)__double_as_longlong(mm));
        partial[(size_t)blockIdx.x * M + i] = acc;
      }
    }
  }
#undef RD_OFF
}
// out[i] = sum_chunks partial[c][i]: 32 rows x 8 chunk classes per CTA, fixed-order combine
__global__ void __launch_bounds__(256)
k_oz_dot_final(int M, int nchunks, const double* __restrict__ partial, double* __restrict__ out)
{
  __shared__ double sm[8][33];
  const int ri = threadIdx.x & 31, part = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + ri;
  double s = 0.0;
  if(i < M)
    for(int c = part; c < nchunks; c += 8) s += partial[(size_t)c * M + i];
  sm[part][ri] = s;
  __syncthreads();
  if(part == 0 && i < M) {
    double t = 0.0;
#pragma unroll
    for(int p = 0; p < 8; p++) t += sm[p][ri];
    out[i] = t;
  }
}
__global__ void k_oz_exponents(int M, const unsigned long long* __restrict__ mx, int* __restrict__ e)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= M) return;
  const double m = __longlong_as_double((long long)mx[i]);
  int ex = 0;
  if(m > 0.0) frexp(m, &ex); // m = f * 2^ex, f in [0.5, 1)  ->  |b| / 2^ex < 1
  e[i] = ex;
}
__global__ void k_sqrt(long long n, const double* __restrict__ d, double* __restrict__ sd)
{
  const long long stride = (long long)gridDim.x * blockDim.x;
  for(long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) sd[i] = sqrt(d[i]);
}

// Q[p][row][k] (int8, row pitch Kpad bytes, slice pitch Mpad*Kpad). One thread = 8 consecutive k of one row: a warp reads
// 2 KB of the FP64 row with 16-byte loads and writes 256 contiguous bytes per slice.
//
// Digits without the conversion pipe: with b = a*sd / 2^e (|b| < 1), hi = rint(b * 2^27) carries the first four slices
// (6+7+7+7 bits) and lo = rint((b*2^27 - hi) * 2^(7(S-4))) the remaining S-4. Both roundings use the 1.5*2^52 magic-number
// add (two DADDs at full FP64 rate; the integer is the low word of the sum -- no F2I/FRND, which issue at 1/4 rate and would
// make this kernel conversion-bound). Each 32-bit integer is then cut into balanced
// base-128 digits d in [-64, 63] from the least significant end; the leading digit of either word is bounded by 64.
// sum_p q_p 2^-(6+7p) = b rounded to the last slice's grid, exactly.
template <int ND>
__device__ __forceinline__ void oz_digits(int v, int (&d)[ND])
{
#pragma unroll
  for(int j = ND - 1; j > 0; j--) {
    d[j] = ((v + 64) & 127) - 64;
    v = (v - d[j]) >> 7;
  }
  d[0] = v;
}
template <int S>
__global__ void __launch_bounds__(256)
k_oz_slice(const double* const* __restrict__ rowptr, int M, int Mpad, long long K, long long Kpad, const double* __restrict__ sd,
           const int* __restrict__ e, int8_t* __restrict__ Q, int vec_ok)
{
  static_assert(S >= 5 && S <= 8, "slices");
  constexpr int NLO = S - 4;
  const int row = blockIdx.y;
  const long long k0 = ((long long)blockIdx.x * 256 + threadIdx.x) * 8;
  if(k0 >= Kpad) return;
  double x[8];
#pragma unroll
  for(int j = 0; j < 8; j++) x[j] = 0.0;
  if(row < M) {
    const double* a = rowptr[row];
    // 2^(27 - e) overflows for e <= -997 (row maximum below 2^-997): such a row is scaled by 2^(27 - e - 512), then by 2^512. Both
    // products are exact (the first stays below 2^-485, the second below 2^27), so every row gets exactly b * 2^(27 - e).
    const int es = 27 - e[row];
    const double sc = ldexp(1.0, es > 1023 ? es - 512 : es);
    if(vec_ok && k0 + 7 < K) {
#pragma unroll
      for(int j = 0; j < 8; j += 2) {
        const double2 av = *reinterpret_cast<const double2*>(a + k0 + j);
        double2 sv = make_double2(1.0, 1.0);
        if(sd) sv = *reinterpret_cast<const double2*>(sd + k0 + j);
        x[j] = __dmul_rn(__dmul_rn(av.x, sv.x), sc);
        x[j + 1] = __dmul_rn(__dmul_rn(av.y, sv.y), sc);
      }
    } else {
#pragma unroll
      for(int j = 0; j < 8; j++)
        if(k0 + j < K) x[j] = __dmul_rn(__dmul_rn(a[k0 + j], sd ? sd[k0 + j] : 1.0), sc);
    }
    if(es > 1023) {
#pragma unroll
      for(int j = 0; j < 8; j++) x[j] = __dmul_rn(x[j], 0x1p512);
    }
  }
  const double MAGIC = 6755399441055744.0; // 1.5 * 2^52
  unsigned w[S][2];
#pragma unroll
  for(int h = 0; h < 2; h++) {
    int dh[4][4], dl[4][NLO];
#pragma unroll
    for(int j = 0; j < 4; j++) {
      const double xs = x[4 * h + j];
      const double t = __dadd_rn(xs, MAGIC);
      const int hi = __double2loint(t);
      const double rem = __dsub_rn(xs, __dsub_rn(t, MAGIC));                       // exact, |rem| <= 0.5
      const int lo = __double2loint(__fma_rn(rem, (double)(1 << (7 * NLO)), MAGIC));
      oz_digits<4>(hi, dh[j]);
      oz_digits<NLO>(lo, dl[j]);
    }
#pragma unroll
    for(int p = 0; p < 4; p++)
      w[p][h] = __byte_perm(__byte_perm(dh[0][p], dh[1][p], 0x0040), __byte_perm(dh[2][p], dh[3][p], 0x0040), 0x5410);
#pragma unroll
    for(int p = 0; p < NLO; p++)
      w[4 + p][h] = __byte_perm(__byte_perm(dl[0][p], dl[1][p], 0x0040), __byte_perm(dl[2][p], dl[3][p], 0x0040), 0x5410);
  }
#pragma unroll
  for(int p = 0; p < S; p++) *reinterpret_cast<uint2*>(Q + ((size_t)p * Mpad + row) * Kpad + k0) = make_uint2(w[p][0], w[p][1]);
}

// ---------------------------------------------------------------------------------------------------------------------
// the wgmma GEMM
// ---------------------------------------------------------------------------------------------------------------------
struct OzItem
{
  int bi, bj;       // 128-row block, 32-column block
  int k_begin;      // first K stage (units of KS bytes)
  int k_count;
  int slot;         // FP64 partial tile (TM x TN doubles)
};

template <int S>
struct OzCfg
{
  static constexpr int B_BLOCK = S * B_TILE;                              // all S slices of the 32 B-rows for one K block
  static constexpr int RING = (227 * 1024 - 2 * B_BLOCK - 1536) / A_TILE; // A tiles in flight (11 / 10 / 10 for S = 6 / 7 / 8)
  static constexpr int SMEM = 2 * B_BLOCK + RING * A_TILE + 512 + 1024;   // + barriers + alignment slack
};

// K is swept in blocks of KS = 128 bytes (one SWIZZLE_128B row). Per K block the B operand (S slices x 32 rows, 4S KB) is
// double-buffered and stays resident while the S A tiles (16 KB each) stream through a ring; slice p is multiplied against the
// slices 0..S-1-p of B, one m64n32k32 MMA per slice pair (p, q) into the accumulator of t = p+q. One wgmma group (the four K steps
// of one A tile) stays in flight while the next is issued; a slot is handed back to the producer when the group that read it has
// completed. (Stacking the B slices into one MMA of N = 32 (S-p) gives MMAs whose accumulator ranges overlap with different
// widths, and ptxas then serialises every wgmma.)
template <int S>
__global__ void __launch_bounds__(OZ_THREADS, 1)
k_oz_gemm(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const OzItem* __restrict__ items, int n_items,
          int chunk_blocks, double* __restrict__ partial)
{
  using Cfg = OzCfg<S>;
  constexpr int RING = Cfg::RING;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles must start on a 1024-byte boundary
  uint8_t* smem = smem_raw + ((1024 - (hb_smem_addr(smem_raw) & 1023)) & 1023);
  uint8_t* bbuf = smem;                       // 2 x B_BLOCK
  uint8_t* aring = smem + 2 * Cfg::B_BLOCK;   // RING x A_TILE
  unsigned long long* bfull = reinterpret_cast<unsigned long long*>(aring + RING * A_TILE);
  unsigned long long* bempty = bfull + 2;
  unsigned long long* afull = bempty + 2;
  unsigned long long* aempty = afull + RING;
  // warp index through a shuffle: provably warp-uniform, so the consumer branch is not a divergent path for wgmma
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  if(tid == 0) {
    for(int s = 0; s < 2; s++) { hb_mbar_init(&bfull[s], 1); hb_mbar_init(&bempty[s], 2); }
    for(int s = 0; s < RING; s++) { hb_mbar_init(&afull[s], 1); hb_mbar_init(&aempty[s], 2); }
    hb_mbar_init_fence();
  }
  __syncthreads();

  if(warp >= OZ_CONSUMERS / 32) {
    // ================= TMA producer =================
    hb_setmaxnreg_dec<40>();
    if(warp != OZ_CONSUMERS / 32 || lane != 0) return;
    int bs = 0, as = 0;
    unsigned bph = 0, aph = 0;
    for(int w = blockIdx.x; w < n_items; w += gridDim.x) {
      const OzItem itm = items[w];
      for(int it = 0; it < itm.k_count; it++) {
        const int kc = (itm.k_begin + it) * KS;
        hb_mbar_wait<OZ_SUSPEND_NS>(&bempty[bs], bph ^ 1);
        hb_mbar_arrive_expect_tx(&bfull[bs], Cfg::B_BLOCK);
        hb_tma_load_3d(bbuf + bs * Cfg::B_BLOCK, &mapB, kc, itm.bj * TN, 0, &bfull[bs]); // box {128 B, 32 rows, S slices}
        if(++bs == 2) { bs = 0; bph ^= 1; }
#pragma unroll 1
        for(int p = 0; p < S; p++) {
          hb_mbar_wait<OZ_SUSPEND_NS>(&aempty[as], aph ^ 1);
          hb_mbar_arrive_expect_tx(&afull[as], A_TILE);
          hb_tma_load_3d(aring + as * A_TILE, &mapA, kc, itm.bi * TM, p, &afull[as]);    // box {128 B, 128 rows, 1 slice}
          if(++as == RING) { as = 0; aph ^= 1; }
        }
      }
    }
    return;
  }

  // ================= consumer warpgroups: MMA + epilogue =================
  hb_setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const bool leader = (tid & 127) == 0;
  // accumulator fragment of m64nNk32: register 4j + 2h + c of a 32-column block holds row 16*(warp%4) + lane/4 + 8h, column 8j + 2*(lane%4) + c
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
  // only wgmma writes the accumulators (a chunk's first MMA overwrites them): no register copies while MMAs are in flight
  uint32_t acc[S * 16];
#pragma unroll
  for(int i = 0; i < S * 16; i++) acc[i] = 0u;
  int bs = 0, as = 0, pend_a = -1, pend_b = -1;
  unsigned bph = 0, aph = 0;
  for(int w = blockIdx.x; w < n_items; w += gridDim.x) {
    const OzItem itm = items[w];
    double* tile = partial + (size_t)itm.slot * (TM * TN);
    int in_chunk = 0, chunk = 0;
    for(int it = 0; it < itm.k_count; it++) {
      hb_mbar_wait<OZ_SUSPEND_NS>(&bfull[bs], bph);
      const uint32_t sb = hb_smem_addr(bbuf + bs * Cfg::B_BLOCK);
      const int chunk_start = in_chunk == 0;
#pragma unroll
      for(int p = 0; p < S; p++) {
        hb_mbar_wait<OZ_SUSPEND_NS>(&afull[as], aph);
        const uint32_t sa = hb_smem_addr(aring + as * A_TILE) + wg * (64 * KS);
#pragma unroll
        for(int i = 0; i < S * 16; i++) hb_wgmma_fence_operand(acc[i]);
        hb_wgmma_fence();
#pragma unroll
        for(int ks = 0; ks < KS / 32; ks++)
#pragma unroll
          for(int q = 0; q < S - p; q++)
            hb_wgmma_s8<1>(acc + 16 * (p + q), hb_wgmma_desc_sw128(sa + ks * 32), hb_wgmma_desc_sw128(sb + q * B_TILE + ks * 32),
                           (chunk_start && p == 0 && ks == 0) ? 0 : 1);
        hb_wgmma_commit();
        hb_wgmma_wait<1>();
        if(leader) {
          if(pend_a >= 0) hb_mbar_arrive(&aempty[pend_a]);
          if(pend_b >= 0) hb_mbar_arrive(&bempty[pend_b]);
        }
        pend_a = as;
        pend_b = p == S - 1 ? bs : -1;
        if(++as == RING) { as = 0; aph ^= 1; }
      }
      if(++bs == 2) { bs = 0; bph ^= 1; }
      if(++in_chunk == chunk_blocks || it == itm.k_count - 1) {
        hb_wgmma_wait<0>();
#pragma unroll
        for(int i = 0; i < S * 16; i++) hb_wgmma_fence_operand(acc[i]);
        if(leader) {
          hb_mbar_arrive(&aempty[pend_a]);
          hb_mbar_arrive(&bempty[pend_b]);
        }
        pend_a = pend_b = -1;
#pragma unroll
        for(int j = 0; j < TN / 8; j++) {
#pragma unroll
          for(int h = 0; h < 2; h++) {
            double v[2];
#pragma unroll
            for(int cc = 0; cc < 2; cc++) {
              double s = 0.0;
#pragma unroll
              for(int t = S - 1; t >= 0; t--) s += (double)(int)acc[16 * t + 4 * j + 2 * h + cc] * ldexp(1.0, -(12 + 7 * t)); // smallest weights first
              v[cc] = s;
            }
            double2* dst = reinterpret_cast<double2*>(tile + (size_t)(row0 + 8 * h) * TN + 8 * j + col0);
            if(chunk == 0) {
              *dst = make_double2(v[0], v[1]);
            } else {
              double2 o = *dst;
              o.x += v[0];
              o.y += v[1];
              *dst = o;
            }
          }
        }
        in_chunk = 0;
        chunk++;
      }
    }
  }
}

// C(i,j) = 2^{e_i+e_j} * sum over splits of the partial tiles; upper part computed, mirrored.
__global__ void __launch_bounds__(256)
k_oz_fixup(int M, int n_tiles, const int2* __restrict__ tile_ij, int splits, const double* __restrict__ partial, const int* __restrict__ e,
           double* __restrict__ C, int ldc)
{
  const int t = blockIdx.x;
  const int2 ij = tile_ij[t];
  for(int el = threadIdx.x; el < TM * TN; el += 256) {
    const int r = el / TN, c = el % TN;
    const int gi = ij.x * TM + r, gj = ij.y * TN + c;
    if(gi >= M || gj >= M || gj < gi) continue;
    double v = 0.0;
    for(int s = 0; s < splits; s++) v += partial[((size_t)(t * splits + s)) * (TM * TN) + el];
    v = ldexp(v, e[gi] + e[gj]);
    C[(size_t)gi * ldc + gj] = v;
    C[(size_t)gj * ldc + gi] = v;
  }
}

void put_item(void* dst, int bi, int bj, int, int k_begin, int k_count, int slot)
{
  const OzItem it = {bi, bj, k_begin, k_count, slot};
  memcpy(dst, &it, sizeof(it));
}

// Default: one wave, splits = SMs / tiles (every CTA gets one item). Where that leaves the machine badly filled (144 tiles at m = 1000
// or 1024 on 132 SMs: two waves, 55 % busy) several waves of the persistent CTAs are searched (hb_split_search): e.g. 11 splits = 1584
// items = 12 full waves -> 1.091 of one tile's full-K time, the ideal 144/132.
int oz_splits(const hb_ctx* c, long long nt, long long kstages, int max_splits, size_t tile_bytes)
{
  int splits = (int)(c->num_sms / (nt > 0 ? nt : 1));
  if(splits < 1) splits = 1;
  if(splits > kstages) splits = (int)(kstages > 0 ? kstages : 1);
  const long long items0 = nt * splits;
  const long long waves0 = (items0 + c->num_sms - 1) / c->num_sms;
  const double util0 = nt > 0 ? (double)items0 / (double)(waves0 * c->num_sms) : 1.0;
  if(util0 < 0.7) splits = hb_split_search(c, nt, kstages, max_splits, tile_bytes, splits, (double)waves0 / splits);
  if(splits > kstages) splits = (int)(kstages > 0 ? kstages : 1);
  return splits;
}

} // namespace

// Step 1 of both int8 condensations: the launches and bits are those the slice path has always made
int hb_row_exponents(hb_ctx* c, hb_rowscale& rs, int M, int Mpad, long long K, const double* const* rowptr_dev, bool rows_aligned16,
                     const double* d, const double* dot_x, double* dot_out, const double** sd_out)
{
  HB_CHECK(rs.sd.reserve(c, K, "sqrt(d)"));
  HB_CHECK(rs.mx.reserve(c, Mpad, "row maxima"));
  HB_CHECK(rs.e.reserve(c, Mpad, "row exponents"));
  const double* sd = nullptr;
  if(d) {
    k_sqrt<<<c->num_sms * 8, 256, 0, c->stream>>>(K, d, rs.sd);
    HB_LAUNCHED();
    sd = rs.sd;
  }
  HB_CUDA(cudaMemsetAsync(rs.mx, 0, sizeof(unsigned long long) * Mpad, c->stream));
  if(dot_x && dot_out && K > 0) {
    const int nchunks = (int)((K + RD_COLS - 1) / RD_COLS);
    HB_CHECK(rs.dot_partial.reserve(c, (size_t)nchunks * M, "fused row-dot partials"));
    int rsplit = (2 * c->num_sms + nchunks - 1) / nchunks; // short shards: split the rows of a chunk over several CTAs
    rsplit = rsplit < 1 ? 1 : (rsplit > 8 ? 8 : rsplit);
    // pairs of columns need 16-byte aligned rows AND an even first column per lane (RD_COLS is even)
    if(rows_aligned16 && (K & 1) == 0)
      k_oz_rowmax_dot<true><<<dim3(nchunks, rsplit), RD_THREADS, 0, c->stream>>>(rowptr_dev, M, K, d, dot_x, rs.mx, rs.dot_partial);
    else
      k_oz_rowmax_dot<false><<<dim3(nchunks, rsplit), RD_THREADS, 0, c->stream>>>(rowptr_dev, M, K, d, dot_x, rs.mx, rs.dot_partial);
    HB_LAUNCHED();
    k_oz_dot_final<<<(M + 31) / 32, 256, 0, c->stream>>>(M, nchunks, rs.dot_partial, dot_out);
    HB_LAUNCHED();
  } else {
    long long gx = (K + 256 * 64 - 1) / (256 * 64);
    if(gx < 1) gx = 1;
    if(gx > 64) gx = 64;
    k_oz_rowmax<<<dim3((unsigned)gx, M), 256, 0, c->stream>>>(rowptr_dev, M, K, sd, rs.mx);
    HB_LAUNCHED();
  }
  k_oz_exponents<<<(Mpad + 127) / 128, 128, 0, c->stream>>>(M, rs.mx, rs.e);
  HB_LAUNCHED();
  hb_phase_mark(c, HB_PH_OZ_ROWMAX);
  *sd_out = sd;
  return HB_OK;
}

void hb_delete(hb_int8_state* p) { delete p; }

int hb_int8_empty(hb_ctx* c, int M, double* C, int ldc)
{
  if(M > 0) HB_CUDA(cudaMemset2DAsync(C, sizeof(double) * ldc, 0, sizeof(double) * M, M, c->stream));
  return HB_OK;
}

int hb_split_search(const hb_ctx* c, long long units, long long kstages, int max_splits, size_t tile_bytes, int splits, double best)
{
  for(int sp = 1; sp <= max_splits; sp++) {
    if(sp > 1 && (kstages / sp < 64 || (size_t)units * sp * tile_bytes > ((size_t)1 << 30))) break;
    const double cost = (double)((units * sp + c->num_sms - 1) / c->num_sms) / sp;
    if(cost < best * (1.0 - 1e-3)) { best = cost; splits = sp; }
  }
  return splits;
}

int hb_int8_prepare(hb_ctx* c, hb_state<hb_int8_state>& slot, const hb_int8_layout& L, int M, long long K, hb_int8_state** out)
{
  if(!slot) slot.reset(new hb_int8_state);
  hb_int8_state& st = *slot;
  if(!st.encode) {
    cudaDriverEntryPointQueryResult qres;
    HB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void**)&st.encode, cudaEnableDefault, &qres));
    if(!st.encode) return hb_fail(HB_ERR_CUDA, "cuTensorMapEncodeTiled is not available in this driver%s", "");
  }
  const int Mpad = ((M + L.tm - 1) / L.tm) * L.tm;
  const long long Kpad = ((K + KS - 1) / KS) * KS;
  const size_t qbytes = (size_t)L.planes * Mpad * Kpad;
  if(!st.Q || st.Q.capacity() < qbytes) {
    st.M = -1; // the tensor maps hold the address of Q
    HB_CHECK(st.Q.reserve(c, qbytes, "the int8 planes"));
  }
  const char* env = getenv(L.split_env);
  const int max_splits = env ? atoi(env) : 16;
  if(st.M != M || st.K != K || st.planes != L.planes || st.max_splits != max_splits) {
    st.M = -1;
    HB_CUDA(cudaStreamSynchronize(c->stream));
    const int nbi = Mpad / L.tm, nbj = Mpad / L.tn;
    std::vector<int2> tiles;
    for(int bi = 0; bi < nbi; bi++)
      for(int bj = (L.tm / L.tn) * bi; bj < nbj; bj++)
        if(bj * L.tn < M) tiles.push_back(make_int2(bi, bj));
    const int nt = (int)tiles.size();
    const long long kstages = Kpad / KS;
    const int splits = L.splits(c, (long long)nt * L.groups, kstages, max_splits, L.tile_bytes);
    // split-major: the CTAs running at once sweep the same K window (of the same plane) -> operand reuse in L2
    const int n_items = splits * L.groups * nt;
    std::vector<unsigned char> items((size_t)n_items * L.item_bytes);
    unsigned char* it = items.data();
    for(int s = 0; s < splits; s++)
      for(int g = 0; g < L.groups; g++)
        for(int t = 0; t < nt; t++, it += L.item_bytes) {
          const long long b = hb_part_begin(kstages, splits, s), e = hb_part_begin(kstages, splits, s + 1);
          L.put_item(it, tiles[t].x, tiles[t].y, g, (int)b, (int)(e - b), (t * L.groups + g) * splits + s);
        }
    HB_CHECK(st.items.reserve(c, items.size(), "the int8 work list"));
    HB_CHECK(st.tiles.reserve(c, nt, "the int8 tile list"));
    HB_CUDA(cudaMemcpy(st.items, items.data(), items.size(), cudaMemcpyHostToDevice));
    HB_CUDA(cudaMemcpy(st.tiles, tiles.data(), sizeof(int2) * nt, cudaMemcpyHostToDevice));
    const cuuint64_t dims[3] = {(cuuint64_t)Kpad, (cuuint64_t)Mpad, (cuuint64_t)L.planes};
    const cuuint64_t strides[2] = {(cuuint64_t)Kpad, (cuuint64_t)Kpad * Mpad};
    const cuuint32_t es[3] = {1, 1, 1};
    for(int i = 0; i < L.n_maps; i++)
      if(st.encode(&st.maps[i], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, st.Q, dims, strides, L.box[i], es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return hb_fail(HB_ERR_CUDA, "cuTensorMapEncodeTiled failed%s", "");
    st.M = M; st.K = K; st.planes = L.planes; st.max_splits = max_splits;
    st.Mpad = Mpad; st.Kpad = Kpad; st.splits = splits; st.n_tiles = nt; st.n_items = n_items;
  }
  HB_CHECK(hb_ws_reserve(c, L.tile_bytes * st.n_items));
  *out = &st;
  return HB_OK;
}

int hb_ozaki_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_oz_gemm<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OzCfg<6>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_oz_gemm<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OzCfg<7>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_oz_gemm<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OzCfg<8>::SMEM));
  return HB_OK;
}

// Same contract as hb_syrk_rows (C = A diag(d) A^T, both triangles), computed with S int8 slices on the integer tensor cores
int hb_syrk_rows_ozaki(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool rows_aligned16, const double* d, double* C, int ldc, int S,
                       const double* dot_x, double* dot_out)
{
  HB_REQUIRE(c && M >= 0 && K >= 0 && ldc >= M && (S == 6 || S == 7 || S == 8), "hb_syrk_rows_ozaki: bad arguments");
  if(M == 0 || K == 0) return hb_int8_empty(c, M, C, ldc);
  // 128 x 32 tiles; one item per (tile, K range) multiplies all S slices: per K stage one box of A per slice, one of B with all S
  const hb_int8_layout L = {S, TM, TN, 1, sizeof(double) * TM * TN, sizeof(OzItem), put_item, oz_splits, "HB_OZ_MAX_SPLITS",
                            2, {{KS, TM, 1}, {KS, TN, (cuuint32_t)S}}};
  hb_int8_state* st;
  HB_CHECK(hb_int8_prepare(c, c->oz, L, M, K, &st));
  const int Mpad = st->Mpad;
  const long long Kpad = st->Kpad;
  // 1. sqrt(d), row maxima, exponents, slices
  const double* sd;
  HB_CHECK(hb_row_exponents(c, st->rs, M, Mpad, K, rowptr_dev, rows_aligned16, d, dot_x, dot_out, &sd));
  const unsigned sx = (unsigned)((Kpad / 8 + 255) / 256);
  const int vec_ok = rows_aligned16 ? 1 : 0;
  if(S == 6) k_oz_slice<6><<<dim3(sx, Mpad), 256, 0, c->stream>>>(rowptr_dev, M, Mpad, K, Kpad, sd, st->rs.e, st->Q, vec_ok);
  else if(S == 7) k_oz_slice<7><<<dim3(sx, Mpad), 256, 0, c->stream>>>(rowptr_dev, M, Mpad, K, Kpad, sd, st->rs.e, st->Q, vec_ok);
  else k_oz_slice<8><<<dim3(sx, Mpad), 256, 0, c->stream>>>(rowptr_dev, M, Mpad, K, Kpad, sd, st->rs.e, st->Q, vec_ok);
  HB_LAUNCHED();
  hb_phase_mark(c, HB_PH_OZ_SLICE);
  // 2. wgmma GEMM into FP64 partial tiles
  // (t+1) * Kc * 2^12 < 2^31 with t+1 <= S  ->  Kc <= 2^19 / S columns
  int chunk_stages = (int)((524288 / S) / KS);
  // strict: S products of |q q'| <= 2^12 per column must stay BELOW 2^31 (S = 8 gives exactly 2^31 with 512 stages of 128 columns when
  // every digit is -64, see tests/test_cpu_oz_model.py)
  while((long long)S * chunk_stages * KS * 4096 >= (1LL << 31)) chunk_stages--;
  const int G = st->n_items < c->num_sms ? st->n_items : c->num_sms;
  const OzItem* items = (const OzItem*)st->items.get();
  HB_CHECK(hb_timed_syrk(c, [&] {
    if(S == 6) k_oz_gemm<6><<<G, OZ_THREADS, OzCfg<6>::SMEM, c->stream>>>(st->maps[0], st->maps[1], items, st->n_items, chunk_stages, (double*)c->ws);
    else if(S == 7) k_oz_gemm<7><<<G, OZ_THREADS, OzCfg<7>::SMEM, c->stream>>>(st->maps[0], st->maps[1], items, st->n_items, chunk_stages, (double*)c->ws);
    else k_oz_gemm<8><<<G, OZ_THREADS, OzCfg<8>::SMEM, c->stream>>>(st->maps[0], st->maps[1], items, st->n_items, chunk_stages, (double*)c->ws);
    HB_LAUNCHED();
    return HB_OK;
  }));
  // 3. split-K reduction, row scales, symmetrisation
  k_oz_fixup<<<st->n_tiles, 256, 0, c->stream>>>(M, st->n_tiles, st->tiles, st->splits, (const double*)c->ws, st->rs.e, C, ldc);
  HB_LAUNCHED();
  return HB_OK;
}
