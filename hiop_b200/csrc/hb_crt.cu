// C = A diag(d) A^T on the Hopper int8 tensor cores by Chinese remaindering (Ozaki scheme II: Ozaki, Uchino and Imamura, 2025).
//
//   B = A diag(sqrt(d)), e_i = frexp exponent of row i's exact maximum, t = t(K) = min(53, floor((126 - ceil(log2 K)) / 2)):
//   q_ik = rint(b_ik 2^(t - e_i)), |q| <= 2^t, and X = q q^T is an exact integer matrix with |X| <= K 2^(2t) <= 2^126.
//   For the N = N(K) first moduli p_m of a fixed list of pairwise-coprime integers <= 256 (product P/2 > K 2^(2t)):
//     r_m = q mod p_m, balanced into [-floor(p/2), ceil(p/2) - 1] (int8);  X mod p_m = r_m r_m^T mod p_m  (one int8 GEMM each)
//   X follows from its N residues (Garner's mixed radix with balanced digits, summed in wrapping 128-bit arithmetic), and
//   C_ij = ldexp(RN(X_ij), e_i + e_j - 2t): the correctly rounded value of an exactly known integer.
//
// Residues add exactly in any order, so the K splits, the int32 chunks and the tile schedule cannot change a bit of C: it is a
// function of (A, d) alone. The only errors are the rounding of b to t bits below each row's exponent and the final rounding.
// Compared with the slices of hb_ozaki.cu (S(S+1)/2 = 36 products for S = 8, S accumulators per tile), each modulus is one plain
// product with one accumulator, so the tiles are 128 x 128 with m64n128k32, and N = 16 or 17 products cover K up to 2^20.
// Memory: the residue planes take N Mpad Kpad bytes (17.4 GB at n = 1e6, m + 2l = 1012; the 8 slices take 8.2 GB), and the context
// workspace one int32 residue tile (64 KB) per work item: tiles * N * splits * 64 KB, 40 MB at that size but 3.5 GB at m = 10000 with
// one split (the split search keeps it below 1 GB only when it splits).
//
// Pipeline:
//   k_crt_residues  one thread = 8 consecutive k of one row: q, then N residue bytes each, in the (k, row, plane) layout of the
//                   slice buffer (row pitch Kpad, plane pitch Mpad Kpad, zeros in the padding)
//   k_crt_gemm      persistent CTAs over (tile, modulus, K range) items; warp 8 (one thread) is the TMA producer of a ring of
//                   {128 B x 128 rows} boxes of both operands (one box on a diagonal tile), warps 0-7 are two consumer warpgroups
//                   (rows 0-63 / 64-127) with one int32 m64n128k32 accumulator each. Every CRT_CHUNK K stages the accumulator
//                   is reduced mod p into a running residue; the item's residue tile goes to the context workspace.
//   k_crt_fixup     per output tile (grid x) and 1024-element range of it (grid y), per element: the split residues summed mod p, Garner, the 128-bit sum, RN to double, ldexp,
//                   mirror.
#include "hb_common.cuh"
#include "hb_ptx.cuh"
#include <cuda.h>

namespace {

constexpr int CT = 128;                         // output tile: 128 x 128
constexpr int KS = 128;                         // bytes of K per stage (one SWIZZLE_128B row = four MMA K steps)
constexpr int BOX = CT * KS;                    // 16 KB: one operand box of one stage
constexpr int RING = 6;                         // stages in flight (2 boxes each)
constexpr int CRT_SMEM = RING * 2 * BOX + 256 + 1024; // + barriers + alignment slack
constexpr int CRT_CONSUMERS = 256;
constexpr int CRT_THREADS = CRT_CONSUMERS + 128;
constexpr unsigned CRT_SUSPEND_NS = 10000000u;
// K stages per exact int32 chunk: 1023 * 128 columns * 2^14 (|r| <= 128) = 2^31 - 2^21 < 2^31
constexpr int CRT_CHUNK = 1023;
constexpr int CRT_FIXUP_PARTS = 16; // CTAs per output tile of k_crt_fixup (1024 elements each)
constexpr int CRT_MAX = 17; // moduli in the table: N(K) <= 17 for every K below 2^31
constexpr double MAGIC = 6755399441055744.0; // 1.5 * 2^52: x + MAGIC rounds x (|x| < 2^51) to an integer held in the low word

// The moduli (greedy pairwise-coprime from 256 down), the inverses and the mixed-radix weights of Garner's conversion:
//   W_j = p_0 ... p_{j-1} (W_0 = 1; kept mod 2^128), wmod[j][m] = W_j mod p_m, winv[m] = W_m^{-1} mod p_m.
struct CrtTable
{
  int p[CRT_MAX];
  int winv[CRT_MAX];
  int wmod[CRT_MAX][CRT_MAX];
  unsigned long long wlo[CRT_MAX], whi[CRT_MAX];
};

constexpr int crt_inv(int a, int p) // a^{-1} mod p, gcd(a, p) = 1
{
  int r = 1;
  for(int x = 1; x < p; x++)
    if((a * x) % p == 1) r = x;
  return r;
}
constexpr CrtTable crt_table()
{
  CrtTable T{};
  const int P[CRT_MAX] = {256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191};
  unsigned __int128 W = 1;
  for(int j = 0; j < CRT_MAX; j++) {
    T.p[j] = P[j];
    T.wlo[j] = (unsigned long long)W;
    T.whi[j] = (unsigned long long)(W >> 64);
    for(int m = 0; m < CRT_MAX; m++) T.wmod[j][m] = 0;
    W *= (unsigned)P[j];
  }
  for(int m = 0; m < CRT_MAX; m++) {
    int w = 1; // W_m mod p_m
    for(int j = 0; j < CRT_MAX; j++) {
      if(j < m) T.wmod[j][m] = w;
      if(j < m) w = (w * P[j]) % P[m];
    }
    T.winv[m] = m == 0 ? 1 : crt_inv(w, P[m]);
  }
  return T;
}
constexpr CrtTable CRT_HOST = crt_table();
__constant__ CrtTable c_crt = crt_table();

// x mod p into [-floor(p/2), ceil(p/2) - 1] for |x| < 2^31
__device__ __forceinline__ int crt_bal(int x, int p)
{
  int r = x % p;
  if(r > (p - 1) / 2) r -= p;
  else if(r < -(p / 2)) r += p;
  return r;
}

// ---------------------------------------------------------------------------------------------------------------------
// residues
// ---------------------------------------------------------------------------------------------------------------------
// R[m][row][k] = q_{row,k} mod p_m (balanced int8). q = rint(b 2^(t-e)) is an integer-valued double with |q| <= 2^t <= 2^53;
// k = rint(q / p) by one multiplication with fl(1/p) and the magic-number add (|q / p| < 2^46), r = fma(-p, k, q) is exact (q and
// p k are exact and the result is a small integer), and one correction brings it into the balanced range (|q/p - k| <= 0.51).
__global__ void __launch_bounds__(256)
k_crt_residues(const double* const* __restrict__ rowptr, int M, int Mpad, long long K, long long Kpad, const double* __restrict__ sd,
               const int* __restrict__ e, int t, int nmod, int8_t* __restrict__ R, int vec_ok)
{
  const int row = blockIdx.y;
  const long long k0 = ((long long)blockIdx.x * 256 + threadIdx.x) * 8;
  if(k0 >= Kpad) return;
  double q[8];
#pragma unroll
  for(int j = 0; j < 8; j++) q[j] = 0.0;
  if(row < M) {
    const double* a = rowptr[row];
    // 2^(t - e) overflows for e <= t - 1024: such a row is scaled by 2^(t - e - 512), then by 2^512, both exactly (as k_oz_slice)
    const int es = t - e[row];
    const double sc = ldexp(1.0, es > 1023 ? es - 512 : es);
    if(vec_ok && k0 + 7 < K) {
#pragma unroll
      for(int j = 0; j < 8; j += 2) {
        const double2 av = *reinterpret_cast<const double2*>(a + k0 + j);
        double2 sv = make_double2(1.0, 1.0);
        if(sd) sv = *reinterpret_cast<const double2*>(sd + k0 + j);
        q[j] = __dmul_rn(__dmul_rn(av.x, sv.x), sc);
        q[j + 1] = __dmul_rn(__dmul_rn(av.y, sv.y), sc);
      }
    } else {
#pragma unroll
      for(int j = 0; j < 8; j++)
        if(k0 + j < K) q[j] = __dmul_rn(__dmul_rn(a[k0 + j], sd ? sd[k0 + j] : 1.0), sc);
    }
#pragma unroll
    for(int j = 0; j < 8; j++) q[j] = rint(es > 1023 ? __dmul_rn(q[j], 0x1p512) : q[j]);
  }
  for(int m = 0; m < nmod; m++) {
    const int p = c_crt.p[m];
    const double pd = (double)p, pinv = 1.0 / pd;
    int r[8];
#pragma unroll
    for(int j = 0; j < 8; j++) {
      const double k = __dsub_rn(__dadd_rn(__dmul_rn(q[j], pinv), MAGIC), MAGIC);
      int v = __double2loint(__dadd_rn(__fma_rn(-pd, k, q[j]), MAGIC));
      if(v > (p - 1) / 2) v -= p;
      else if(v < -(p / 2)) v += p;
      r[j] = v;
    }
    const unsigned lo = __byte_perm(__byte_perm(r[0], r[1], 0x0040), __byte_perm(r[2], r[3], 0x0040), 0x5410);
    const unsigned hi = __byte_perm(__byte_perm(r[4], r[5], 0x0040), __byte_perm(r[6], r[7], 0x0040), 0x5410);
    *reinterpret_cast<uint2*>(R + ((size_t)m * Mpad + row) * Kpad + k0) = make_uint2(lo, hi);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// the wgmma GEMM: one residue tile per (tile, modulus, K range)
// ---------------------------------------------------------------------------------------------------------------------
struct CrtItem
{
  int bi, bj;   // 128-row blocks (bi <= bj)
  int plane;    // modulus index
  int k_begin;  // first K stage (units of KS bytes)
  int k_count;
  int slot;     // int32 residue tile (CT x CT) in the workspace
};

__global__ void __launch_bounds__(CRT_THREADS, 1)
k_crt_gemm(const __grid_constant__ CUtensorMap map, const CrtItem* __restrict__ items, int n_items, int* __restrict__ out)
{
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024 - (hb_smem_addr(smem_raw) & 1023)) & 1023); // SWIZZLE_128B boxes start on 1024-byte boundaries
  unsigned long long* full = reinterpret_cast<unsigned long long*>(smem + RING * 2 * BOX);
  unsigned long long* empty = full + RING;
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  if(tid == 0) {
    for(int s = 0; s < RING; s++) { hb_mbar_init(&full[s], 1); hb_mbar_init(&empty[s], 2); }
    hb_mbar_init_fence();
  }
  __syncthreads();

  if(warp >= CRT_CONSUMERS / 32) {
    // ================= TMA producer =================
    hb_setmaxnreg_dec<40>();
    if(warp != CRT_CONSUMERS / 32 || lane != 0) return;
    int s = 0;
    unsigned ph = 0;
    for(int w = blockIdx.x; w < n_items; w += gridDim.x) {
      const CrtItem itm = items[w];
      const bool diag = itm.bi == itm.bj;
      for(int it = 0; it < itm.k_count; it++) {
        const int kc = (itm.k_begin + it) * KS;
        uint8_t* dst = smem + s * 2 * BOX;
        hb_mbar_wait<CRT_SUSPEND_NS>(&empty[s], ph ^ 1);
        hb_mbar_arrive_expect_tx(&full[s], diag ? BOX : 2 * BOX);
        hb_tma_load_3d(dst, &map, kc, itm.bi * CT, itm.plane, &full[s]);
        if(!diag) hb_tma_load_3d(dst + BOX, &map, kc, itm.bj * CT, itm.plane, &full[s]);
        if(++s == RING) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ================= consumer warpgroups =================
  hb_setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const bool leader = (tid & 127) == 0;
  // accumulator fragment of m64n128k32: register 4j + 2h + c holds row 16*(warp%4) + lane/4 + 8h, column 8j + 2*(lane%4) + c
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), col0 = 2 * (lane & 3);
  uint32_t acc[64];
  int res[64];
#pragma unroll
  for(int i = 0; i < 64; i++) acc[i] = 0u;
  int s = 0, pend = -1;
  unsigned ph = 0;
  for(int w = blockIdx.x; w < n_items; w += gridDim.x) {
    const CrtItem itm = items[w];
    const bool diag = itm.bi == itm.bj;
    const double pd = (double)c_crt.p[itm.plane], pinv = 1.0 / pd;
#pragma unroll
    for(int i = 0; i < 64; i++) res[i] = 0;
    // One inner loop per exact int32 chunk: nothing reads the accumulator inside it, so one MMA group stays in flight while the next
    // stage is issued (a read of acc on any path through the loop body makes ptxas drain every group before the next).
    for(int c0 = 0; c0 < itm.k_count; c0 += CRT_CHUNK) {
      const int cn = min(CRT_CHUNK, itm.k_count - c0);
      for(int it = 0; it < cn; it++) {
        hb_mbar_wait<CRT_SUSPEND_NS>(&full[s], ph);
        const uint32_t sa = hb_smem_addr(smem + s * 2 * BOX);
        const uint32_t sb = diag ? sa : sa + BOX;
#pragma unroll
        for(int i = 0; i < 64; i++) hb_wgmma_fence_operand(acc[i]);
        hb_wgmma_fence();
#pragma unroll
        for(int ks = 0; ks < KS / 32; ks++)
          hb_wgmma_s8<4>(acc, hb_wgmma_desc_sw128(sa + wg * (64 * KS) + ks * 32), hb_wgmma_desc_sw128(sb + ks * 32), (it == 0 && ks == 0) ? 0 : 1);
        hb_wgmma_commit();
        hb_wgmma_wait<1>();
        if(leader && pend >= 0) hb_mbar_arrive(&empty[pend]);
        pend = s;
        if(++s == RING) { s = 0; ph ^= 1; }
      }
      hb_wgmma_wait<0>();
#pragma unroll
      for(int i = 0; i < 64; i++) hb_wgmma_fence_operand(acc[i]);
      if(leader) hb_mbar_arrive(&empty[pend]);
      pend = -1;
      // running residue: res + acc (|.| < 2^31 - 2^21 + 2^8, exact in FP64), minus p rint((res + acc) / p), |result| <= 0.51 p
#pragma unroll
      for(int i = 0; i < 64; i++) {
        const double x = (double)res[i] + (double)(int)acc[i];
        const double k = __dsub_rn(__dadd_rn(__dmul_rn(x, pinv), MAGIC), MAGIC);
        res[i] = __double2loint(__dadd_rn(__fma_rn(-pd, k, x), MAGIC));
      }
    }
    int* tile = out + (size_t)itm.slot * (CT * CT);
#pragma unroll
    for(int j = 0; j < CT / 8; j++)
#pragma unroll
      for(int h = 0; h < 2; h++)
        *reinterpret_cast<int2*>(tile + (size_t)(row0 + 8 * h) * CT + 8 * j + col0) = make_int2(res[4 * j + 2 * h], res[4 * j + 2 * h + 1]);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// fix-up: split residues, Garner, correctly rounded conversion, row scales, mirror
// ---------------------------------------------------------------------------------------------------------------------
// ws[((tile * nmod + m) * splits + s) * CT^2 + el]. X = sum_m d_m W_m with balanced digits d_m; |X| < 2^127, so the sum taken mod 2^128
// and read as a signed 128-bit integer is X itself (P exceeds 2^128 for 17 moduli: X is never compared with P/2).
template <int NMOD>
__device__ __forceinline__ __int128 crt_garner(const int* __restrict__ ws, size_t el_base, int splits)
{
  int d[NMOD];
  unsigned __int128 X = 0;
#pragma unroll
  for(int m = 0; m < NMOD; m++) {
    const int p = c_crt.p[m];
    int r = 0;
    for(int s = 0; s < splits; s++) r += ws[el_base + (size_t)(m * splits + s) * (CT * CT)];
    int acc = 0;
#pragma unroll
    for(int j = 0; j < m; j++) acc += d[j] * c_crt.wmod[j][m];
    d[m] = crt_bal(((r - acc) % p) * c_crt.winv[m], p);
    const unsigned __int128 W = ((unsigned __int128)c_crt.whi[m] << 64) | c_crt.wlo[m];
    X += (unsigned __int128)(__int128)d[m] * W;
  }
  return (__int128)X;
}

// RN(X) for |X| < 2^127: |X| normalised to 64 bits with a sticky bit, then one correctly rounded conversion (exact power-of-two scale)
__device__ __forceinline__ double crt_round(__int128 X)
{
  const bool neg = X < 0;
  const unsigned __int128 u = neg ? (unsigned __int128)(-X) : (unsigned __int128)X;
  const unsigned long long hi = (unsigned long long)(u >> 64), lo = (unsigned long long)u;
  double v;
  if(hi == 0) {
    v = __ull2double_rn(lo);
  } else {
    const int sh = 64 - __clzll((long long)hi); // 1 .. 63
    const unsigned long long top = (unsigned long long)(u >> sh) | ((lo & ((1ull << sh) - 1)) != 0 ? 1ull : 0ull);
    v = ldexp(__ull2double_rn(top), sh);
  }
  return neg ? -v : v;
}

template <int NMOD>
__global__ void __launch_bounds__(256)
k_crt_fixup(int M, const int2* __restrict__ tile_ij, int splits, const int* __restrict__ ws, const int* __restrict__ e, int t,
            double* __restrict__ C, int ldc)
{
  const int tt = blockIdx.x;
  constexpr int PART = CT * CT / CRT_FIXUP_PARTS;
  const int2 ij = tile_ij[tt];
  for(int el = blockIdx.y * PART + threadIdx.x; el < (blockIdx.y + 1) * PART; el += 256) {
    const int r = el / CT, cc = el % CT;
    const int gi = ij.x * CT + r, gj = ij.y * CT + cc;
    if(gi >= M || gj >= M || gj < gi) continue;
    const double v = ldexp(crt_round(crt_garner<NMOD>(ws, (size_t)tt * NMOD * splits * (CT * CT) + el, splits)), e[gi] + e[gj] - 2 * t);
    C[(size_t)gi * ldc + gj] = v;
    C[(size_t)gj * ldc + gi] = v;
  }
}

// t(K) = min(53, floor((126 - ceil(log2 K)) / 2)): K 2^(2t) <= 2^126
int crt_bits(long long K)
{
  int lg = 0;
  while((1LL << lg) < K) lg++;
  const int t = (126 - lg) / 2;
  return t < 53 ? t : 53;
}
// N(K): the fewest moduli whose product P satisfies P / 2 > K 2^(2t), i.e. P > K 2^(2t+1) (<= 2^127)
int crt_moduli(long long K, int t)
{
  const unsigned __int128 need = (unsigned __int128)K << (2 * t + 1);
  unsigned __int128 P = 1;
  int n = 0;
  while(P <= need) {
    if(P > ~(unsigned __int128)0 / (unsigned)CRT_HOST.p[n]) return n + 1; // the product passes 2^128 > need
    P *= (unsigned)CRT_HOST.p[n++];
  }
  return n;
}

void put_item(void* dst, int bi, int bj, int plane, int k_begin, int k_count, int slot)
{
  const CrtItem it = {bi, bj, plane, k_begin, k_count, slot};
  memcpy(dst, &it, sizeof(it));
}

// K splits: the count of at most 16 (HB_CRT_MAX_SPLITS) with the shortest makespan, searched from one split (hb_split_search). The
// bits do not depend on it.
int crt_splits(const hb_ctx* c, long long pairs, long long kstages, int max_splits, size_t tile_bytes)
{
  return hb_split_search(c, pairs, kstages, max_splits, tile_bytes, 1, (double)((pairs + c->num_sms - 1) / c->num_sms));
}

} // namespace

int hb_crt_init_attrs(hb_ctx* c)
{
  (void)c;
  HB_CUDA(cudaFuncSetAttribute(k_crt_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, CRT_SMEM));
  return HB_OK;
}

// Same contract as hb_syrk_rows (C = A diag(d) A^T, both triangles), as the correctly rounded value of the exact integer Gram of the
// rows rounded to t(K) bits
int hb_syrk_rows_crt(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool rows_aligned16, const double* d, double* C, int ldc,
                     const double* dot_x, double* dot_out)
{
  HB_REQUIRE(c && M >= 0 && K >= 0 && K < (1LL << 31) && ldc >= M, "hb_syrk_rows_crt: bad arguments");
  if(M == 0 || K == 0) return hb_int8_empty(c, M, C, ldc);
  const int t = crt_bits(K), nmod = crt_moduli(K, t);
  HB_REQUIRE(nmod >= 14 && nmod <= CRT_MAX, "hb_syrk_rows_crt: the reconstruction covers 14 to 17 moduli");
  // 128 x 128 tiles, one item per (tile, modulus, K range): per K stage one box of each operand from the same map
  const hb_int8_layout L = {nmod, CT, CT, nmod, sizeof(int) * CT * CT, sizeof(CrtItem), put_item, crt_splits, "HB_CRT_MAX_SPLITS",
                            1, {{KS, CT, 1}}};
  hb_int8_state* st;
  HB_CHECK(hb_int8_prepare(c, c->crt, L, M, K, &st));
  const int Mpad = st->Mpad;
  const long long Kpad = st->Kpad;
  // 1. sqrt(d), row maxima, exponents (shared with the slice path), residues
  const double* sd;
  HB_CHECK(hb_row_exponents(c, st->rs, M, Mpad, K, rowptr_dev, rows_aligned16, d, dot_x, dot_out, &sd));
  k_crt_residues<<<dim3((unsigned)((Kpad / 8 + 255) / 256), Mpad), 256, 0, c->stream>>>(rowptr_dev, M, Mpad, K, Kpad, sd, st->rs.e, t, nmod, st->Q,
                                                                                       rows_aligned16 ? 1 : 0);
  HB_LAUNCHED();
  hb_phase_mark(c, HB_PH_OZ_SLICE);
  // 2. one exact int8 GEMM per modulus into int32 residue tiles
  int* ws = (int*)c->ws.get();
  HB_CHECK(hb_timed_syrk(c, [&] {
    const int G = st->n_items < c->num_sms ? st->n_items : c->num_sms;
    k_crt_gemm<<<G, CRT_THREADS, CRT_SMEM, c->stream>>>(st->maps[0], (const CrtItem*)st->items.get(), st->n_items, ws);
    HB_LAUNCHED();
    return HB_OK;
  }));
  // 3. split residues, reconstruction, rounding, row scales, symmetrisation
  const dim3 fg(st->n_tiles, CRT_FIXUP_PARTS);
  switch(nmod) {
  case 14: k_crt_fixup<14><<<fg, 256, 0, c->stream>>>(M, st->tiles, st->splits, ws, st->rs.e, t, C, ldc); break; // K <= 8
  case 15: k_crt_fixup<15><<<fg, 256, 0, c->stream>>>(M, st->tiles, st->splits, ws, st->rs.e, t, C, ldc); break;
  case 16: k_crt_fixup<16><<<fg, 256, 0, c->stream>>>(M, st->tiles, st->splits, ws, st->rs.e, t, C, ldc); break;
  case 17: k_crt_fixup<17><<<fg, 256, 0, c->stream>>>(M, st->tiles, st->splits, ws, st->rs.e, t, C, ldc); break;
  }
  HB_LAUNCHED();
  return HB_OK;
}
