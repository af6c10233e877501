// Large-N dense symmetric factorizations and solves (the B1 plug-in at MDS / sweep sizes, N up to a few 10^4).
//
// Roles: hiopLinSolverSymDenseLapack::matrixChanged / solve (src/LinAlg/hiopLinSolverSymDenseLapack.hpp:75-192) and the MAGMA twins
// magma_dsytrf_nopiv_gpu / magma_dpotrf (src/LinAlg/hiopLinSolverSymDenseMagma.cpp:349, 455) + their triangular solves (:250, :420).
//
// Storage convention as in hb_dense.cu: N x N row-major with the UPPER triangle valid = column-major LOWER, Lc(i,j) = A[j*lda + i].
//
// Factorization (Cholesky LL^T and no-pivot LDL^T), block size 128, right-looking with one block of look-ahead on two streams:
//   panel stream  : k_diag128   one CTA factors the 128 x 128 diagonal block in shared memory (16-wide sub-panels) and also emits the
//                               INVERSE of its triangular factor (kept: the solves use it),
//                   k_gemm_pq<128,STORE>   L21 = A21 * L11^-T as a DMMA GEMM against that inverse (LDL^T: W21 = A21 L11^-T, L21 = W21 D^-1)
//   update stream : k_gemm_pq<64,SUB>      A22 -= W21 * L21^T on 128 x 64 tiles of the lower triangle: first the 128 columns of the next
//                                          panel (the panel stream continues as soon as these are done), then the rest.
//   k_gemm_pq: operands are "p-major" (P[p][i], i contiguous = a column of the factor), 16 x tile chunks through a 4-stage cp.async ring,
//   mma.sync.m8n8k4.f64 (SASS DMMA), 8 warps, 2 CTAs per SM for the update tiles so that one tile's read-modify-write epilogue overlaps
//   the other's MMA loop; the epilogue goes through shared memory so that the global accesses run down the (contiguous) columns.
//
// Solves (all three modes incl. Bunch-Kaufman in permuted form): one launch per 256 rows per sweep. Forward step (left-looking):
// the CTAs compute partial products of block-row k against the already solved part, the LAST CTA to finish (ticket) adds them in a
// fixed order and applies the stored 128 x 128 inverses -- deterministic, no atomics on the data. Backward step likewise with the
// rows below. N = 8192: 2 x 32 launches.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include "hb_ptx.cuh"

namespace {

constexpr int BB = 128;  // factorization block = size of the stored diagonal-block inverses
constexpr int KC = 16;   // operand rows per pipeline stage
constexpr int GST = 4;   // pipeline stages
constexpr int TM = 128;  // tile rows (i)
constexpr int PLD = TM + 4;
constexpr int CLD = TM + 2;

// EPI_SUB_CYC: EPI_SUB on a block-cyclic C (the distributed factorization, hb_symdense_dist.cu): blockIdx.z picks the local block
// q = cyc_q0 + z of global block k = q * cyc_p + cyc_r, whose 128 columns C + q * 128 * ldc holds; its tiles start at (k*128, k*128)
enum { EPI_SUB = 0, EPI_STORE = 1, EPI_STORE_LDL = 2, EPI_SUB_CYC = 3 };

struct GemmArgs
{
  const double* P;   // P[p*ldp + i], absolute row index i
  long long ldp;
  const double* Q;   // Q[p*ldq + (j - qsub)]
  long long ldq;
  int qsub;
  int kb;            // number of operand rows (K), <= 128
  double* C;         // C[j*ldc + i]
  long long ldc;
  int i_base, j_base, i_end, j_end;
  int tj0;           // first column tile of this launch
  double* W2;        // EPI_STORE_LDL: W2[(j - j_base)*ldw2 + i] = acc
  long long ldw2;
  const double* dinv; // EPI_STORE_LDL: C = acc * dinv[j - j_base]
  const int* state;   // pivoted panels: k0 = state[0], kb = state[1] read on the device (Q = C + k0*ldc, origin k0 + kb)
  int cyc_p, cyc_r, cyc_q0; // EPI_SUB_CYC
};

template <int TN>
struct GemmCfg
{
  static constexpr int QLD = TN + 4;
  static constexpr int STAGE_D = KC * PLD + KC * QLD;
  static constexpr size_t SMEM = sizeof(double) * ((size_t)GST * STAGE_D > (size_t)TN * CLD ? (size_t)GST * STAGE_D : (size_t)TN * CLD);
};

template <int TN, int EPI>
__global__ void __launch_bounds__(256, (TN == 64 ? 2 : 1)) k_gemm_pq(const GemmArgs g)
{
  extern __shared__ __align__(16) unsigned char gsm_raw[];
  double* sm = reinterpret_cast<double*>(gsm_raw);
  constexpr int QLD = GemmCfg<TN>::QLD;
  constexpr int STAGE_D = GemmCfg<TN>::STAGE_D;
  constexpr int NJ = TN / 16; // 8-wide n fragments per warp (2 warps along j)

  int kb = g.kb, i_base = g.i_base, j_base = g.j_base;
  int jmin = g.j_base;
  const double* Q = g.Q;
  if(g.state) {
    const int k0 = g.state[0];
    kb = g.state[1];
    if(kb <= 0) return;
    jmin = k0 + kb;
    i_base = j_base = jmin & ~1; // tile origins stay even (16-byte accesses); the column below the origin is masked out
    Q = g.C + (size_t)k0 * g.ldc;
  }
  constexpr bool SUB = EPI == EPI_SUB || EPI == EPI_SUB_CYC;
  double* C = g.C;
  int i0 = i_base + TM * blockIdx.x;
  int j0 = j_base + TN * (g.tj0 + blockIdx.y);
  if(EPI == EPI_SUB_CYC) {
    const int q = g.cyc_q0 + blockIdx.z, k0 = (q * g.cyc_p + g.cyc_r) * BB;
    C = g.C + (ptrdiff_t)(q * BB - k0) * g.ldc;
    i0 = k0 + TM * blockIdx.x;
    j0 = k0 + TN * blockIdx.y;
    jmin = k0;
  }
  if(i0 >= g.i_end || j0 >= g.j_end) return;
  if(SUB && i0 + TM - 1 < j0) return; // tile entirely above the diagonal

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 3, wn = warp >> 2;
  const int gq = lane >> 2, t4 = lane & 3;
  const int nch = (kb + KC - 1) / KC;
  const double* P = g.P;

  auto load_chunk = [&](int ch) {
    double* sP = sm + (size_t)(ch % GST) * STAGE_D;
    double* sQ = sP + KC * PLD;
#pragma unroll
    for(int q = 0; q < (KC * TM / 2) / 256; q++) {
      const int idx = tid + 256 * q;
      const int p = idx >> 6, ic = idx & 63;
      const int pp = ch * KC + p, i = i0 + 2 * ic;
      const bool v = pp < kb && i < g.i_end;
      hb_cp_async16(&sP[p * PLD + 2 * ic], v ? P + (size_t)pp * g.ldp + i : P, v ? 16 : 0);
    }
#pragma unroll
    for(int q = 0; q < (KC * TN / 2) / 256; q++) {
      const int idx = tid + 256 * q;
      const int p = idx / (TN / 2), jc = idx % (TN / 2);
      const int pp = ch * KC + p, j = j0 + 2 * jc;
      const bool v = pp < kb && j < g.j_end;
      hb_cp_async16(&sQ[p * QLD + 2 * jc], v ? Q + (size_t)pp * g.ldq + (j - g.qsub) : Q, v ? 16 : 0);
    }
  };

  double acc[4][NJ][2];
#pragma unroll
  for(int a = 0; a < 4; a++)
#pragma unroll
    for(int b = 0; b < NJ; b++) acc[a][b][0] = acc[a][b][1] = 0.0;

  if(SUB) {
    // the read-modify-write epilogue stalled on HBM latency (24% of the stall samples): pull the C tile into L2 now, the reads then
    // overlap the MMA loop and the epilogue loads hit L2. One 128-byte line per request: TN columns x (TM*8/128) lines.
    for(int e = tid; e < TN * (TM * 8 / 128); e += 256) {
      const int jl = e / (TM * 8 / 128), seg = e % (TM * 8 / 128);
      const int gj = j0 + jl, gi = i0 + seg * 16;
      if(gj < g.j_end && gi < g.i_end && gi + 15 >= gj) hb_prefetch_l2(&LC(C, g.ldc, gi, gj));
    }
  }

#pragma unroll
  for(int s = 0; s < GST - 1; s++) {
    if(s < nch) load_chunk(s);
    hb_cp_async_commit();
  }
  for(int it = 0; it < nch; it++) {
    hb_cp_async_wait<GST - 2>();
    __syncthreads();
    {
      const int nx = it + GST - 1;
      if(nx < nch) load_chunk(nx);
      hb_cp_async_commit();
    }
    const double* sP = sm + (size_t)(it % GST) * STAGE_D;
    const double* sQ = sP + KC * PLD;
#pragma unroll
    for(int kk = 0; kk < KC / 4; kk++) {
      double af[4], bf[NJ];
#pragma unroll
      for(int a = 0; a < 4; a++) af[a] = sP[(kk * 4 + t4) * PLD + wm * 32 + a * 8 + gq];
#pragma unroll
      for(int b = 0; b < NJ; b++) bf[b] = sQ[(kk * 4 + t4) * QLD + wn * (TN / 2) + b * 8 + gq];
#pragma unroll
      for(int a = 0; a < 4; a++)
#pragma unroll
        for(int b = 0; b < NJ; b++) hb_dmma884(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
  }
  hb_cp_async_wait<0>();
  __syncthreads();
  // ---- epilogue: accumulators -> shared (column-major tile, stride CLD) -> global, running down the columns ----
  double* sC = sm;
#pragma unroll
  for(int a = 0; a < 4; a++)
#pragma unroll
    for(int b = 0; b < NJ; b++)
#pragma unroll
      for(int h = 0; h < 2; h++) sC[(wn * (TN / 2) + b * 8 + t4 * 2 + h) * CLD + wm * 32 + a * 8 + gq] = acc[a][b][h];
  __syncthreads();
  constexpr int ITEMS = TM * TN / 2 / 256; // double2 items per thread
  constexpr int BATCH = 8;
#pragma unroll 1
  for(int b0 = 0; b0 < ITEMS; b0 += BATCH) {
    double2 cur[BATCH];
    if(SUB) {
#pragma unroll
      for(int s = 0; s < BATCH; s++) {
        const int e = tid + (b0 + s) * 256;
        const int jl = e >> 6, il = (e & 63) * 2;
        const int gi = i0 + il, gj = j0 + jl;
        cur[s] = make_double2(0.0, 0.0);
        if(gj < g.j_end && gj >= jmin && gi + 1 >= gj && gi < g.i_end) {
          if(gi >= gj && gi + 1 < g.i_end) cur[s] = *reinterpret_cast<const double2*>(&LC(C, g.ldc, gi, gj));
          else {
            if(gi >= gj) cur[s].x = LC(C, g.ldc, gi, gj);
            if(gi + 1 < g.i_end) cur[s].y = LC(C, g.ldc, gi + 1, gj);
          }
        }
      }
    }
#pragma unroll
    for(int s = 0; s < BATCH; s++) {
      const int e = tid + (b0 + s) * 256;
      const int jl = e >> 6, il = (e & 63) * 2;
      const int gi = i0 + il, gj = j0 + jl;
      if(gj >= g.j_end || gj < jmin || gi >= g.i_end) continue;
      const double2 v = *reinterpret_cast<const double2*>(&sC[jl * CLD + il]);
      if(SUB) {
        if(gi + 1 < gj) continue;
        if(gi >= gj && gi + 1 < g.i_end) *reinterpret_cast<double2*>(&LC(C, g.ldc, gi, gj)) = make_double2(cur[s].x - v.x, cur[s].y - v.y);
        else {
          if(gi >= gj) LC(C, g.ldc, gi, gj) = cur[s].x - v.x;
          if(gi + 1 < g.i_end) LC(C, g.ldc, gi + 1, gj) = cur[s].y - v.y;
        }
      } else {
        const bool two = gi + 1 < g.i_end;
        double2 o = v;
        if(EPI == EPI_STORE_LDL) {
          const int c = gj - j_base;
          if(two) *reinterpret_cast<double2*>(&g.W2[(size_t)c * g.ldw2 + gi]) = v;
          else g.W2[(size_t)c * g.ldw2 + gi] = v.x;
          const double r = g.dinv[c];
          o.x *= r; o.y *= r;
        }
        if(two) *reinterpret_cast<double2*>(&LC(C, g.ldc, gi, gj)) = o;
        else LC(C, g.ldc, gi, gj) = o.x;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// 128 x 128 diagonal block: factor (LL^T or LDL^T without pivoting) + inverse of the triangular factor, one CTA.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int DSB = BB + 4; // 132: the m8n8k4 fragment reads (4 k-rows x 8 consecutive entries) are bank-conflict free
constexpr int TLD = 116;
constexpr int DTHREADS = 512;
struct DiagSmem
{
  double D[BB * DSB];        // D[j*DSB + i] = element (i,j), i >= j; the slots i < j receive the strictly lower part of the inverse:
                             // Inv(r,c), r > c, lives at D[r*DSB + c]
  double Inv16[8 * 16 * 17]; // inverses of the eight 16 x 16 diagonal triangles
  double Tt[16 * TLD];
  double idg[BB];            // diagonal of the inverse (1/L_rr; 1 for the unit factor of LDL^T)
  double dv[BB];             // LDL^T: d_j
  double rdv[BB];            // LDL^T: 1/d_j
};

// Factors the 128 x 128 block in S.D (16-wide sub-panels). Per sub-panel: warp 0 factors the 16 x 16 diagonal triangle in registers
// and inverts it; the rows below and the rank-16 update of the rest run on the DMMA pipe straight out of shared memory (the first
// version did them with scalar FMAs on 2 x 2 register tiles and was bound by shared-memory wavefronts: 86 us per block).
// InvG (global, column-major 128 x 128, zero above the diagonal from allocation): receives the 16 x 16 diagonal inverses here and the
// off-diagonal blocks in invert_block128.
// ---- pieces of the 128 x 128 block factorization (16-wide sub-panels) ----
// warp 0: factor the 16 x 16 diagonal triangle of sub-panel kb in registers (lane = row, shuffles for the pivot row) and invert it
template <bool LDL>
__device__ __forceinline__ void subpanel_diag(DiagSmem& S, int kb, int k0, int* info, double* __restrict__ InvG)
{
  const int lane = threadIdx.x & 31;
  const int c0 = kb * 16;
  double a[16];
  double myr = 1.0;
#pragma unroll
  for(int c = 0; c < 16; c++) a[c] = (lane < 16 && c <= lane) ? S.D[(c0 + c) * DSB + c0 + lane] : 0.0;
  // spelled out per column (a rolled 16 x 15 nest would put a[] in local memory)
#define BIG_CHOL_COL(j)                                                                          \
  {                                                                                              \
    const double d = __shfl_sync(0xffffffffu, a[j], j);                                          \
    if(!(d > 0.0) && lane == 0 && info) atomicCAS(info, 0, k0 + c0 + j + 1);                     \
    const double r = rsqrt(d);                                                                   \
    if(lane == j) { a[j] = d * r; myr = r; }                                                     \
    else if(lane > j) a[j] *= r;                                                                 \
    _Pragma("unroll") for(int c = j + 1; c < 16; c++) {                                          \
      const double lc = __shfl_sync(0xffffffffu, a[j], c);                                       \
      if(lane >= c) a[c] -= a[j] * lc;                                                           \
    }                                                                                            \
  }
#define BIG_LDL_COL(j)                                                                           \
  {                                                                                              \
    const double d = __shfl_sync(0xffffffffu, a[j], j);                                          \
    if((d == 0.0 || d != d) && lane == 0 && info) atomicCAS(info, 0, k0 + c0 + j + 1);           \
    const double r = 1.0 / d;                                                                    \
    const double wj = a[j];                                                                      \
    if(lane > j) a[j] = wj * r;                                                                  \
    _Pragma("unroll") for(int c = j + 1; c < 16; c++) {                                          \
      const double wc = __shfl_sync(0xffffffffu, wj, c);                                         \
      if(lane >= c) a[c] -= a[j] * wc;                                                           \
    }                                                                                            \
  }
  if(LDL) {
    BIG_LDL_COL(0) BIG_LDL_COL(1) BIG_LDL_COL(2) BIG_LDL_COL(3) BIG_LDL_COL(4) BIG_LDL_COL(5) BIG_LDL_COL(6) BIG_LDL_COL(7)
    BIG_LDL_COL(8) BIG_LDL_COL(9) BIG_LDL_COL(10) BIG_LDL_COL(11) BIG_LDL_COL(12) BIG_LDL_COL(13) BIG_LDL_COL(14) BIG_LDL_COL(15)
  } else {
    BIG_CHOL_COL(0) BIG_CHOL_COL(1) BIG_CHOL_COL(2) BIG_CHOL_COL(3) BIG_CHOL_COL(4) BIG_CHOL_COL(5) BIG_CHOL_COL(6) BIG_CHOL_COL(7)
    BIG_CHOL_COL(8) BIG_CHOL_COL(9) BIG_CHOL_COL(10) BIG_CHOL_COL(11) BIG_CHOL_COL(12) BIG_CHOL_COL(13) BIG_CHOL_COL(14) BIG_CHOL_COL(15)
  }
#undef BIG_CHOL_COL
#undef BIG_LDL_COL
#pragma unroll
  for(int c = 0; c < 16; c++)
    if(lane < 16 && c <= lane) S.D[(c0 + c) * DSB + c0 + lane] = a[c];
  if(lane < 16) {
    S.idg[c0 + lane] = myr;
    if(LDL) {
      double dl = 0.0;
#pragma unroll
      for(int c = 0; c < 16; c++)
        if(c == lane) dl = a[c];
      S.dv[c0 + lane] = dl;
      S.rdv[c0 + lane] = 1.0 / dl;
    }
  }
  __syncwarp();
  // column `lane` of X = T^-1 (T = the 16 x 16 triangle, unit diagonal for LDL^T), right-looking
  double* inv = S.Inv16 + kb * 16 * 17;
  double x[16], sacc[16];
#pragma unroll
  for(int r = 0; r < 16; r++) { x[r] = 0.0; sacc[r] = 0.0; }
#pragma unroll
  for(int q = 0; q < 16; q++) {
    const double rq = __shfl_sync(0xffffffffu, myr, q);
    if(q == lane) x[q] = rq;
    else if(q > lane) x[q] = -sacc[q] * rq;
#pragma unroll
    for(int r = q + 1; r < 16; r++) sacc[r] += S.D[(c0 + q) * DSB + c0 + r] * x[q];
  }
  if(lane < 16) {
#pragma unroll
    for(int r = 0; r < 16; r++) {
      inv[r * 17 + lane] = x[r];
      if(r > lane) S.D[(c0 + r) * DSB + c0 + lane] = x[r]; // strictly lower part of the inverse -> the unused upper slots
      if(InvG && r >= lane) InvG[(size_t)(c0 + lane) * BB + c0 + r] = x[r];
    }
  }
}

// rows below the 16 x 16 triangle: X = A(:, c0:c0+16) T^-T [ D^-1 ] on the DMMA pipe; 8 rows x 16 columns per warp (both column
// tiles, so the in-place write is safe)
template <bool LDL>
__device__ __forceinline__ void subpanel_rows(DiagSmem& S, int kb)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int gq = lane >> 2, t4 = lane & 3;
  const int c0 = kb * 16, below = BB - c0 - 16;
  const double* inv = S.Inv16 + kb * 16 * 17;
  for(int rg = warp; rg < below / 8; rg += nwarps) {
    const int r0 = c0 + 16 + rg * 8;
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
    for(int kk = 0; kk < 4; kk++) {
      const double af = S.D[(c0 + 4 * kk + t4) * DSB + r0 + gq];
#pragma unroll
      for(int nt = 0; nt < 2; nt++) hb_dmma884(acc[nt][0], acc[nt][1], af, inv[(nt * 8 + gq) * 17 + 4 * kk + t4]);
    }
    __syncwarp();
#pragma unroll
    for(int nt = 0; nt < 2; nt++)
#pragma unroll
      for(int h = 0; h < 2; h++) {
        const int c = nt * 8 + 2 * t4 + h;
        double v = acc[nt][h];
        if(LDL) v *= S.rdv[c0 + c];
        S.D[(c0 + c) * DSB + r0 + gq] = v;
      }
  }
}

// one 8 x 8 tile of the rank-16 update with sub-panel kb: C(i0.., j0..) -= L(i0.., c0:c0+16) [D] L(j0.., c0:c0+16)^T, lower part only
template <bool LDL>
__device__ __forceinline__ void rank16_tile(DiagSmem& S, int c0, int i0, int j0)
{
  const int lane = threadIdx.x & 31;
  const int gq = lane >> 2, t4 = lane & 3;
  double u0 = 0.0, u1 = 0.0;
#pragma unroll
  for(int kk = 0; kk < 4; kk++) {
    const double af = S.D[(c0 + 4 * kk + t4) * DSB + i0 + gq];
    double bf = S.D[(c0 + 4 * kk + t4) * DSB + j0 + gq];
    if(LDL) bf *= S.dv[c0 + 4 * kk + t4];
    hb_dmma884(u0, u1, af, bf);
  }
  const int i = i0 + gq, j = j0 + 2 * t4;
  if(i >= j) S.D[j * DSB + i] -= u0;
  if(i >= j + 1) S.D[(j + 1) * DSB + i] -= u1;
}

// Factors the 128 x 128 block in S.D. Per 16-wide sub-panel: warp 0 factors and inverts the 16 x 16 diagonal triangle (the serial
// part, ~5000 cycles); the rows below and the rank-16 update run on the DMMA pipe straight out of shared memory (the first version did
// them with scalar FMAs on 2 x 2 register tiles and was bound by shared-memory wavefronts: 86 us per block). The update is split:
// the 16 columns of the NEXT sub-panel first (all warps), then warp 0 already factors the next triangle while the other warps
// finish the rest of the update.
template <bool LDL>
__device__ void factor_block128(DiagSmem& S, int k0, int* info, double* __restrict__ InvG, long long* prof)
{
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  long long q0 = prof ? clock64() : 0;
#define QP(slot) if(prof && threadIdx.x == 0) { const long long q1 = clock64(); prof[slot] += q1 - q0; q0 = q1; }
  if(warp == 0) subpanel_diag<LDL>(S, 0, k0, info, InvG);
  __syncthreads();
  QP(1);
  for(int kb = 0; kb < BB / 16; kb++) {
    const int c0 = kb * 16, below = BB - c0 - 16, nt8 = below / 8;
    subpanel_rows<LDL>(S, kb);
    __syncthreads();
    QP(2);
    if(nt8 == 0) break;
    // strip: the two 8-column tile columns of the next sub-panel
    for(int t = warp; t < 2 * nt8 - 1; t += nwarps) {
      const int tjc = t < nt8 ? 0 : 1, ti = t < nt8 ? t : t - nt8 + 1;
      rank16_tile<LDL>(S, c0, c0 + 16 + 8 * ti, c0 + 16 + 8 * tjc);
    }
    __syncthreads();
    QP(3);
    if(warp == 0) {
      subpanel_diag<LDL>(S, kb + 1, k0, info, InvG);
    } else {
      const int m = nt8 - 2; // tile columns 2.. : lower triangle of order m
      for(int t = warp - 1; t < m * (m + 1) / 2; t += nwarps - 1) {
        int ti = 0, rem = t;
        while(rem > ti) { rem -= ti + 1; ti++; }
        rank16_tile<LDL>(S, c0, c0 + 16 + 8 * (ti + 2), c0 + 16 + 8 * (rem + 2));
      }
    }
    __syncthreads();
    QP(1);
  }
#undef QP
}

// Off-diagonal 16 x 16 blocks of the 128 x 128 inverse from the factor (lower slots of S.D) and the 16 x 16 diagonal inverses:
// block row a: Inv_ab = -Inv_aa * sum_{q=b}^{a-1} L_aq Inv_qb -- two small DMMA products per block row.
__device__ void invert_block128(DiagSmem& S, double* __restrict__ InvG)
{
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int gq = lane >> 2, t4 = lane & 3;
  for(int a = 1; a < BB / 16; a++) {
    const int ncol = 16 * a;
    for(int t = warp; t < 4 * a; t += nwarps) { // T (16 x ncol) = L_a * InvLower: tile (rt, ct)
      const int rt = t & 1, n0 = (t >> 1) * 8;
      double u0 = 0.0, u1 = 0.0;
      for(int q0 = n0; q0 < ncol; q0 += 4) {
        const int q = q0 + t4, c = n0 + gq;
        const double af = S.D[q * DSB + ncol + 8 * rt + gq];
        const double bf = q > c ? S.D[q * DSB + c] : (q == c ? S.idg[c] : 0.0);
        hb_dmma884(u0, u1, af, bf);
      }
      S.Tt[(8 * rt + gq) * TLD + n0 + 2 * t4] = u0;
      S.Tt[(8 * rt + gq) * TLD + n0 + 2 * t4 + 1] = u1;
    }
    __syncthreads();
    const double* inv = S.Inv16 + a * 16 * 17;
    for(int t = warp; t < 4 * a; t += nwarps) { // Inv_a,: = -Inv16_a * T
      const int rt = t & 1, n0 = (t >> 1) * 8;
      double u0 = 0.0, u1 = 0.0;
#pragma unroll
      for(int k4 = 0; k4 < 16; k4 += 4) hb_dmma884(u0, u1, inv[(8 * rt + gq) * 17 + k4 + t4], S.Tt[(k4 + t4) * TLD + n0 + gq]);
      const int ra = ncol + 8 * rt + gq, c = n0 + 2 * t4;
      S.D[ra * DSB + c] = -u0;
      S.D[ra * DSB + c + 1] = -u1;
      InvG[(size_t)c * BB + ra] = -u0;
      InvG[(size_t)(c + 1) * BB + ra] = -u1;
    }
    __syncthreads();
  }
}

template <bool LDL>
__global__ void __launch_bounds__(DTHREADS, 1)
k_diag128(double* __restrict__ A, long long lda, int N, int k0, double* __restrict__ inv16G, double* __restrict__ dinvG, int* __restrict__ info,
          long long* __restrict__ prof /* NULL, or 8 cycle counters of thread 0: load, 16x16 factor+inverse, rows below, rank-16 update, store, inversion */)
{
  long long t0 = prof ? clock64() : 0;
#define DP(slot) if(prof && threadIdx.x == 0) { const long long t1 = clock64(); prof[slot] += t1 - t0; t0 = t1; }
  extern __shared__ __align__(16) unsigned char dsm_raw[];
  DiagSmem& S = *reinterpret_cast<DiagSmem*>(dsm_raw);
  const int tid = threadIdx.x;
  const int nb = min(BB, N - k0);
  for(int e0 = tid; e0 < BB * BB; e0 += DTHREADS * 8) { // 8 independent loads in flight per thread
    double v[8];
#pragma unroll
    for(int q = 0; q < 8; q++) {
      const int e = e0 + q * DTHREADS;
      const int j = e / BB, i = e % BB;
      v[q] = (i == j) ? 1.0 : 0.0;
      if(i < nb && j < nb && i >= j) v[q] = LC(A, lda, k0 + i, k0 + j);
    }
#pragma unroll
    for(int q = 0; q < 8; q++) {
      const int e = e0 + q * DTHREADS;
      S.D[(e / BB) * DSB + e % BB] = v[q];
    }
  }
  __syncthreads();
  DP(0);
  factor_block128<LDL>(S, k0, info, nullptr, prof);
  if(prof) t0 = clock64();
  for(int e = tid; e < nb * nb; e += DTHREADS) {
    const int j = e / nb, i = e % nb;
    if(i >= j) LC(A, lda, k0 + i, k0 + j) = S.D[j * DSB + i];
  }
  if(LDL && tid < BB) dinvG[tid] = S.rdv[tid];
  for(int e = tid; e < 8 * 16 * 17; e += DTHREADS) inv16G[e] = S.Inv16[e]; // the panel solve below the block uses the 16 x 16 inverses
  DP(4);
#undef DP
}

// ---------------------------------------------------------------------------------------------------------------------
// Panel solve below a factored diagonal block: X = A21 L11^-T by BLOCK SUBSTITUTION with the 16 x 16 diagonal inverses
// (half the flops of a product with the explicit 128 x 128 inverse, and that inverse leaves the critical path: it is only needed by
// the solves and is built for all blocks at once after the factorization). One CTA per 64 rows; warp w owns rows 8w..8w+7 for all
// eight column blocks, so the whole recurrence needs no CTA-wide barrier. LDL^T: X = W = L21 D; L21 = W D^-1 is formed on the way out.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int XROWS = 64;
constexpr int XS = XROWS + 4;
struct TrsmSmem
{
  double L[BB * DSB];     // L[q*DSB + r] = L11(r, q)
  double Inv16[8 * 16 * 17];
  double X[BB * XS];      // X[c*XS + r] = element (row r of the tile, column c)
};

template <bool LDL>
__global__ void __launch_bounds__(256, 1)
k_trsm_panel(double* __restrict__ A, long long lda, int N, int k0, const double* __restrict__ inv16G, const double* __restrict__ dinvG,
             double* __restrict__ W2, long long ldw2)
{
  extern __shared__ __align__(16) unsigned char tsm_raw[];
  TrsmSmem& S = *reinterpret_cast<TrsmSmem*>(tsm_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, t4 = lane & 3;
  const int r0g = k0 + BB;                    // first row below the block
  const int i0 = r0g + XROWS * blockIdx.x;    // first row of this tile
  // ---- loads (16-byte cp.async, all in flight at once): L11, the 16 x 16 inverses, the A21 tile. The upper part of L11 is copied as
  //      it lies in memory (never read: the recurrence only touches entries strictly below the 16 x 16 diagonal blocks). ----
  for(int e = tid; e < BB * BB / 2; e += 256) {
    const int j = e / (BB / 2), i = (e % (BB / 2)) * 2;
    hb_cp_async16(&S.L[j * DSB + i], &LC(A, lda, k0 + i, k0 + j), 16);
  }
  for(int e = tid; e < BB * XROWS / 2; e += 256) {
    const int c = e / (XROWS / 2), r = (e % (XROWS / 2)) * 2;
    const bool v = i0 + r < N;
    hb_cp_async16(&S.X[c * XS + r], v ? &LC(A, lda, i0 + r, k0 + c) : &LC(A, lda, k0, k0), v ? 16 : 0); // (a valid address either way)
  }
  for(int e = tid; e < 8 * 16 * 17; e += 256) S.Inv16[e] = inv16G[e];
  hb_cp_async_commit();
  hb_cp_async_wait<0>();
  __syncthreads();
  const int rw = warp * 8; // my 8 rows
  for(int jb = 0; jb < BB / 16; jb++) {
    const int cb = 16 * jb;
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    for(int q0 = 0; q0 < cb; q0 += 4) {
      const double af = S.X[(q0 + t4) * XS + rw + gq];
#pragma unroll
      for(int nt = 0; nt < 2; nt++) hb_dmma884(acc[nt][0], acc[nt][1], af, S.L[(q0 + t4) * DSB + cb + 8 * nt + gq]);
    }
    // Y = A - sum (my C-fragment elements), in place
#pragma unroll
    for(int nt = 0; nt < 2; nt++)
#pragma unroll
      for(int h = 0; h < 2; h++) {
        double* px = &S.X[(cb + 8 * nt + 2 * t4 + h) * XS + rw + gq];
        *px = *px - acc[nt][h];
      }
    __syncwarp();
    const double* inv = S.Inv16 + jb * 16 * 17;
    double ac2[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
    for(int kk = 0; kk < 4; kk++) {
      const double af = S.X[(cb + 4 * kk + t4) * XS + rw + gq];
#pragma unroll
      for(int nt = 0; nt < 2; nt++) hb_dmma884(ac2[nt][0], ac2[nt][1], af, inv[(nt * 8 + gq) * 17 + 4 * kk + t4]);
    }
    __syncwarp();
#pragma unroll
    for(int nt = 0; nt < 2; nt++)
#pragma unroll
      for(int h = 0; h < 2; h++) S.X[(cb + 8 * nt + 2 * t4 + h) * XS + rw + gq] = ac2[nt][h];
    __syncwarp();
  }
  __syncthreads();
  for(int e = tid; e < BB * XROWS; e += 256) {
    const int c = e / XROWS, r = e % XROWS;
    const int i = i0 + r;
    if(i >= N) continue;
    const double x = S.X[c * XS + r];
    if(LDL) {
      W2[(size_t)c * ldw2 + i] = x;
      LC(A, lda, i, k0 + c) = x * dinvG[c];
    } else {
      LC(A, lda, i, k0 + c) = x;
    }
  }
}

// Inverses of the 128 x 128 diagonal triangles of an EXISTING factor (paths that do not run k_diag128: cooperative Cholesky,
// Bunch-Kaufman). unit: the factor has an implicit unit diagonal (the stored diagonal holds D and is ignored).
__global__ void __launch_bounds__(DTHREADS, 1)
k_block_inverses(const double* __restrict__ F, long long ldf, int N, int unit, double* __restrict__ InvAll)
{
  extern __shared__ __align__(16) unsigned char dsm_raw[];
  DiagSmem& S = *reinterpret_cast<DiagSmem*>(dsm_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k0 = blockIdx.x * BB;
  const int nb = min(BB, N - k0);
  double* InvG = InvAll + (size_t)blockIdx.x * BB * BB;
  for(int e = tid; e < BB * BB; e += DTHREADS) {
    const int j = e / BB, i = e % BB;
    double v = 0.0;
    if(i < nb && j < nb && i > j) v = LC(F, ldf, k0 + i, k0 + j);
    if(i == j) v = (i < nb && !unit) ? LC(F, ldf, k0 + i, k0 + i) : 1.0;
    S.D[j * DSB + i] = v;
  }
  __syncthreads();
  if(tid < BB) S.idg[tid] = 1.0 / S.D[tid * DSB + tid];
  __syncthreads();
  // 16 x 16 diagonal inverses: warp w < 8 handles triangle w, lane = column of the inverse
  if(warp < 8) {
    const int c0 = warp * 16;
    double x[16], sacc[16];
#pragma unroll
    for(int r = 0; r < 16; r++) { x[r] = 0.0; sacc[r] = 0.0; }
#pragma unroll
    for(int q = 0; q < 16; q++) {
      const double rq = S.idg[c0 + q];
      if(q == lane) x[q] = rq;
      else if(q > lane) x[q] = -sacc[q] * rq;
#pragma unroll
      for(int r = q + 1; r < 16; r++) sacc[r] += S.D[(c0 + q) * DSB + c0 + r] * x[q];
    }
    __syncwarp();
    if(lane < 16) {
      double* inv = S.Inv16 + warp * 16 * 17;
#pragma unroll
      for(int r = 0; r < 16; r++) {
        inv[r * 17 + lane] = x[r];
        if(r > lane) S.D[(c0 + r) * DSB + c0 + lane] = x[r];
        if(r >= lane) InvG[(size_t)(c0 + lane) * BB + c0 + r] = x[r];
      }
    }
  }
  __syncthreads();
  invert_block128(S, InvG);
}

// ---------------------------------------------------------------------------------------------------------------------
// Blocked solves. SB rows per launch; the stored inverses make the in-block solves matrix-vector products.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int SB = 128; // rows per step = one stored inverse
constexpr int ST = 1024;

struct StepSmem
{
  double xs[64];
  double red[ST];
  double y[SB];
};

// Every step is one launch of G + 1 CTAs. CTAs 1..G compute the partial products against the part of the vector that is already
// solved; CTA 0 (the "tail") first pulls the 128 x 128 inverse of its block into REGISTERS (those loads do not depend on the
// partials, so their latency overlaps the main phase), then waits for the ticket counter, adds the partials in a fixed order and
// finishes the step with register / shared-memory products only. (Letting the LAST main CTA do the tail of a 256-row step instead
// puts a chain of dependent L2 round trips on every step.)
__device__ __forceinline__ void wait_counter(int* counter, int G)
{
  if(threadIdx.x == 0) {
    volatile int* vc = counter;
    while(*vc < G) __nanosleep(40);
    __threadfence();
  }
  __syncthreads();
}

// y[0..127] = xk - sum of the G partial vectors (fixed order); 1024 threads = 128 rows x 8 groups
__device__ __forceinline__ void gather_partials(StepSmem& S, const double* __restrict__ partial, int G, int nrows, double xk_own)
{
  const int tid = threadIdx.x, r = tid & 127, gsel = tid >> 7;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  int c = gsel;
  for(; c + 24 < G; c += 32) {
    a0 += __ldcg(&partial[(size_t)c * SB + r]);
    a1 += __ldcg(&partial[(size_t)(c + 8) * SB + r]);
    a2 += __ldcg(&partial[(size_t)(c + 16) * SB + r]);
    a3 += __ldcg(&partial[(size_t)(c + 24) * SB + r]);
  }
  for(; c < G; c += 8) a0 += __ldcg(&partial[(size_t)c * SB + r]);
  S.red[tid] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if(tid < SB) {
    double t = 0.0;
#pragma unroll
    for(int q = 0; q < 8; q++) t += S.red[q * 128 + tid];
    S.y[tid] = tid < nrows ? xk_own - t : 0.0;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(ST, 1)
k_solve_fwd_step(const double* __restrict__ F, long long ldf, int N, int k0, const double* __restrict__ InvAll, double* __restrict__ x,
                 double* __restrict__ partial, int* __restrict__ counter)
{
  __shared__ StepSmem S;
  const int tid = threadIdx.x, G = gridDim.x - 1;
  const int nrows = min(SB, N - k0);
  const int r = tid & 127, gsel = tid >> 7; // 8 groups
  // programmatic dependent launch: the next step's grid may start now (its CTAs prefetch the factor / inverse, which no step writes)
  // and blocks in griddepcontrol.wait until this grid has completed before it touches x, the partials or the counter
  hb_griddep_launch_dependents();
  if(blockIdx.x != 0) {
    // ---- main: partial[b][r] = sum_{j in 64-column chunk b} L(k0 + r, j) x_j ----
    const int b = blockIdx.x - 1;
    const int jb = b * 64;
    double v[8];
#pragma unroll
    for(int q = 0; q < 8; q++) {
      const int j = jb + gsel * 8 + q;
      v[q] = (r < nrows && j < k0) ? LC(F, ldf, k0 + r, j) : 0.0;
    }
    hb_griddep_wait();
    // x is written by the tail CTA of EARLIER steps (other SMs, overlapping grids under programmatic dependent launch): read it from L2,
    // never from a line this SM's L1 may still hold from before (a vector that is not 128-byte aligned lets a line straddle k0)
    if(tid < 64) S.xs[tid] = (jb + tid < k0) ? __ldcg(x + jb + tid) : 0.0;
    __syncthreads();
    double acc = 0.0;
#pragma unroll
    for(int q = 0; q < 8; q++) acc += v[q] * S.xs[gsel * 8 + q];
    S.red[tid] = acc;
    __syncthreads();
    if(tid < SB) {
      double t = 0.0;
#pragma unroll
      for(int q = 0; q < 8; q++) t += S.red[q * 128 + tid];
      partial[(size_t)b * SB + tid] = t;
    }
    __threadfence();
    __syncthreads();
    if(tid == 0) atomicAdd(counter, 1);
    return;
  }
  // ---- tail CTA: x_k = Inv_k (b_k - partials); thread (r, gsel) holds Inv(r, gsel + 8 q) ----
  const double* Inv = InvAll + (size_t)(k0 / BB) * BB * BB;
  double inv[16];
#pragma unroll
  for(int q = 0; q < 16; q++) {
    const int cc = gsel + 8 * q;
    inv[q] = cc <= r ? Inv[cc * BB + r] : 0.0;
  }
  hb_griddep_wait();
  const double xk = (tid < nrows) ? __ldcg(x + k0 + tid) : 0.0;
  wait_counter(counter, G);
  gather_partials(S, partial, G, nrows, xk);
  double acc = 0.0;
#pragma unroll
  for(int q = 0; q < 16; q++) acc += inv[q] * S.y[gsel + 8 * q];
  S.red[tid] = acc;
  __syncthreads();
  if(tid < nrows) {
    double t = 0.0;
#pragma unroll
    for(int q = 0; q < 8; q++) t += S.red[q * 128 + tid];
    x[k0 + tid] = t;
  }
  if(tid == 0) *counter = 0;
}

// backward: rows [k0, k0+nrows) of L^T x = z; rows >= k1 = k0 + nrows are solved already
__global__ void __launch_bounds__(ST, 1)
k_solve_bwd_step(const double* __restrict__ F, long long ldf, int N, int k0, const double* __restrict__ InvAll, double* __restrict__ x,
                 double* __restrict__ partial, int* __restrict__ counter)
{
  __shared__ StepSmem S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x - 1;
  const int nrows = min(SB, N - k0);
  const int k1 = k0 + nrows;
  hb_griddep_launch_dependents();
  if(blockIdx.x != 0) {
    // ---- main: partial[b][j] = sum_{i in 64-row chunk b below the step} L(i, k0 + j) x_i ----
    const int b = blockIdx.x - 1;
    const int il = tid & 63, cg = tid >> 6; // 64 rows x 16 column groups of 8
    const int i = k1 + b * 64 + il;
    double v[8];
#pragma unroll
    for(int q = 0; q < 8; q++) {
      const int jl = cg * 8 + q;
      v[q] = (i < N && jl < nrows) ? LC(F, ldf, i, k0 + jl) : 0.0;
    }
    hb_griddep_wait();
    const double xi = i < N ? __ldcg(x + i) : 0.0;
#pragma unroll
    for(int q = 0; q < 8; q++) v[q] = hb_warp_sum(v[q] * xi);
    if(lane == 0) {
#pragma unroll
      for(int q = 0; q < 8; q++) S.red[warp * 8 + q] = v[q];
    }
    __syncthreads();
    if(tid < SB) { // column tid: group tid/8 -> warps 2*(tid/8), 2*(tid/8)+1
      const int cgi = tid >> 3, q = tid & 7;
      partial[(size_t)b * SB + tid] = S.red[(2 * cgi) * 8 + q] + S.red[(2 * cgi + 1) * 8 + q];
    }
    __threadfence();
    __syncthreads();
    if(tid == 0) atomicAdd(counter, 1);
    return;
  }
  // ---- tail CTA: x_k = Inv_k^T y; warp w owns columns w + 32 t (t < 4), lane owns rows lane + 32 u (u < 4) ----
  const double* Inv = InvAll + (size_t)(k0 / BB) * BB * BB;
  double it[16];
#pragma unroll
  for(int t = 0; t < 4; t++)
#pragma unroll
    for(int u = 0; u < 4; u++) {
      const int cc = warp + 32 * t, rr = lane + 32 * u;
      it[t * 4 + u] = rr >= cc ? Inv[cc * BB + rr] : 0.0;
    }
  hb_griddep_wait();
  const double xk = (tid < nrows) ? __ldcg(x + k0 + tid) : 0.0;
  wait_counter(counter, G);
  gather_partials(S, partial, G, nrows, xk);
#pragma unroll
  for(int t = 0; t < 4; t++) {
    double acc = 0.0;
#pragma unroll
    for(int u = 0; u < 4; u++) acc += it[t * 4 + u] * S.y[lane + 32 * u];
    acc = hb_warp_sum(acc);
    const int cc = warp + 32 * t;
    if(lane == 0 && cc < nrows) x[k0 + cc] = acc;
  }
  if(tid == 0) *counter = 0;
}

// diagonal solve between the sweeps of the no-pivot LDL^T (the Bunch-Kaufman block diagonal lives in hb_bk_cluster.cu)
__global__ void k_dsolve(const double* __restrict__ F, long long ldf, int N, double* __restrict__ x)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if(k < N) x[k] = x[k] / LC(F, ldf, k, k);
}

__global__ void k_gather(int N, const int* __restrict__ perm, const double* __restrict__ in, double* __restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < N) out[i] = in[perm[i]];
}
__global__ void k_scatter(int N, const int* __restrict__ perm, const double* __restrict__ in, double* __restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < N) out[perm[i]] = in[i];
}

} // namespace

// ---------------------------------------------------------------------------------------------------------------------
// internal API (hb_dense.cuh)
// ---------------------------------------------------------------------------------------------------------------------
int hb_big_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_gemm_pq<64, EPI_SUB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GemmCfg<64>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_gemm_pq<64, EPI_SUB_CYC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GemmCfg<64>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_gemm_pq<128, EPI_STORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GemmCfg<128>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_gemm_pq<128, EPI_STORE_LDL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GemmCfg<128>::SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_diag128<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DiagSmem)));
  HB_CUDA(cudaFuncSetAttribute(k_diag128<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DiagSmem)));
  HB_CUDA(cudaFuncSetAttribute(k_block_inverses, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DiagSmem)));
  HB_CUDA(cudaFuncSetAttribute(k_trsm_panel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TrsmSmem)));
  HB_CUDA(cudaFuncSetAttribute(k_trsm_panel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TrsmSmem)));
  return HB_OK;
}

int hb_big_init(hb_ctx* c, hb_big* b)
{
  if(!b->panel_stream) {
    int lo = 0, hi = 0;
    HB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    HB_CHECK(b->panel_stream.create(cudaStreamNonBlocking, hi));
  }
  HB_CHECK(b->ev_panel.create(cudaEventDisableTiming));
  HB_CHECK(b->ev_upd.create(cudaEventDisableTiming));
  HB_CHECK(b->ev_upd2.create(cudaEventDisableTiming));
  return HB_OK;
}

int hb_big_reserve(hb_ctx* c, hb_big* b, int N, bool need_w)
{
  HB_CHECK(hb_big_init(c, b));
  const size_t inv = (size_t)((N + BB - 1) / BB) * BB * BB;
  if(!b->InvAll || b->InvAll.capacity() < inv) {
    HB_CHECK(b->InvAll.reserve(c, inv, "diagonal-block inverses"));
    HB_CUDA(cudaMemsetAsync(b->InvAll, 0, sizeof(double) * b->InvAll.capacity(), c->stream)); // the kernels only write the lower triangles
  }
  HB_CHECK(b->partial.reserve(c, (size_t)(N / 64 + 2) * SB, "blocked-solve partials"));
  HB_CHECK(b->xtmp.reserve(c, (size_t)(N + 2), "permuted rhs"));
  HB_CHECK(b->dinv.reserve(c, BB + 8 * 16 * 17, "diagonal-block scratch"));
  if(!b->counter) {
    HB_CHECK(b->counter.reserve(c, 4, "blocked-solve ticket"));
    HB_CUDA(cudaMemsetAsync(b->counter, 0, sizeof(int) * 4, c->stream));
  }
  if(b->capN < N) b->capN = N;
  if(need_w) {
    const size_t ldw = (size_t)((N + 7) & ~7);
    HB_CHECK(b->W[0].reserve(c, ldw * 2 * BB, "LDL panel scratch"));
    HB_CHECK(b->W[1].reserve(c, ldw * 2 * BB, "LDL panel scratch"));
  }
  return HB_OK;
}

// Cholesky (ldl = false) or no-pivot LDL^T (ldl = true) of the column-major-lower triangle; lda must be even and A 16-byte aligned.
// info_dev: 0 ok, k > 0 = breakdown at column k (1-based). The diagonal-block inverses land in b->InvAll.
//
// Schedule: blocks of 128 columns are factored in PAIRS. Inside a pair the first panel updates only the 128 columns of the second
// (K = 128); the rest of the matrix receives both panels at once (K = 256), which halves the read-modify-write passes over the trailing
// matrix and the per-tile prologue/epilogue share of the update kernel. Two streams: the panel stream runs
//   diag(2a) trsm(2a) U1(2a -> block 2a+1) diag(2a+1) trsm(2a+1)
// while the update stream still applies pair a-1 to the columns beyond; the update stream applies pair a first to the two column
// blocks the next pair needs (events E_UA, E_UBa release the panel stream one block at a time), then to everything else.
int hb_big_factor(hb_ctx* c, hb_big* b, int N, double* A, long long lda, bool ldl, bool pairs, int* info_dev)
{
  HB_REQUIRE((lda & 1) == 0 && (reinterpret_cast<uintptr_t>(A) & 15u) == 0, "hb_big_factor: needs an even leading dimension and a 16-byte aligned matrix");
  HB_CHECK(hb_big_reserve(c, b, N, ldl));
  const long long ldw = (N + 7) & ~7;
  cudaStream_t su = c->stream, sp = b->panel_stream;
  HB_CUDA(cudaMemsetAsync(info_dev, 0, sizeof(int), su));
  HB_CUDA(cudaEventRecord(b->ev_upd, su));  // E_UA : the first block of the next pair has received everything
  HB_CUDA(cudaEventRecord(b->ev_upd2, su)); // E_UBa: so has its second block
  const int nblk = (N + BB - 1) / BB;
  double* inv16 = b->dinv + BB;
  auto panel = [&](int blk, double* Wb) -> int { // diagonal block + panel solve of block blk on the panel stream
    return hb_big_panel(N, A, lda, blk * BB, ldl, inv16, b->dinv, Wb, ldw, info_dev, sp);
  };
  auto update = [&](cudaStream_t st, const double* P, long long ldp, int kq0, int kb, int r0, int tj0, int ntj) -> int {
    // A(i,j) -= sum_p P[p][i] * L(j, kq0 + p) on the lower triangle from row/column r0 on, column tiles [tj0, tj0 + ntj) of 64
    GemmArgs g{};
    g.P = P; g.ldp = ldp;
    g.Q = A + (size_t)kq0 * lda; g.ldq = lda; g.qsub = 0;
    g.kb = kb;
    g.C = A; g.ldc = lda;
    g.i_base = r0; g.j_base = r0; g.i_end = N; g.j_end = N; g.tj0 = tj0;
    const int nti = (N - r0 + TM - 1) / TM;
    k_gemm_pq<64, EPI_SUB><<<dim3(nti, ntj), 256, GemmCfg<64>::SMEM, st>>>(g);
    HB_LAUNCHED();
    return HB_OK;
  };
  const int GW = pairs ? 2 : 1; // blocks per group
  for(int a = 0; GW * a < nblk; a++) {
    const int b0 = GW * a, b1 = GW == 2 ? 2 * a + 1 : nblk; // b1 >= nblk: no second block
    const int k0 = b0 * BB;                                   // first column of the group
    double* Wp = ldl ? b->W[a & 1].get() : nullptr;           // W = L*D of the group's panels, p-major rows
    // ---- panel stream ----
    HB_CUDA(cudaStreamWaitEvent(sp, b->ev_upd, 0));
    HB_CHECK(panel(b0, Wp));
    if(b1 < nblk) {
      HB_CUDA(cudaStreamWaitEvent(sp, b->ev_upd2, 0));
      const int r0 = k0 + BB;
      const int ntj = (N - r0 + 63) / 64;
      HB_CHECK(update(sp, ldl ? Wp : A + (size_t)k0 * lda, ldl ? ldw : lda, k0, BB, r0, 0, ntj < 2 ? ntj : 2)); // panel b0 -> columns of block b1
      HB_CHECK(panel(b1, ldl ? Wp + (size_t)BB * ldw : nullptr));
    }
    HB_CUDA(cudaEventRecord(b->ev_panel, sp));
    HB_CUDA(cudaStreamWaitEvent(su, b->ev_panel, 0));
    // ---- update stream: the group's panels (K = 128 or 256) on everything beyond it ----
    const int r0 = k0 + GW * BB;
    if(r0 < N) {
      const int ntj = (N - r0 + 63) / 64;
      const double* P = ldl ? Wp : A + (size_t)k0 * lda;
      const long long ldp = ldl ? ldw : lda;
      HB_CHECK(update(su, P, ldp, k0, GW * BB, r0, 0, ntj < 2 ? ntj : 2));
      HB_CUDA(cudaEventRecord(b->ev_upd, su));
      if(GW == 2) {
        if(ntj > 2) HB_CHECK(update(su, P, ldp, k0, GW * BB, r0, 2, ntj - 2 < 2 ? ntj - 2 : 2));
        HB_CUDA(cudaEventRecord(b->ev_upd2, su));
        if(ntj > 4) HB_CHECK(update(su, P, ldp, k0, GW * BB, r0, 4, ntj - 4));
      } else if(ntj > 2) {
        HB_CHECK(update(su, P, ldp, k0, GW * BB, r0, 2, ntj - 2));
      }
    }
  }
  // the 128 x 128 inverses of the diagonal triangles (for the solves), all blocks at once
  k_block_inverses<<<nblk, DTHREADS, sizeof(DiagSmem), su>>>(A, lda, N, ldl ? 1 : 0, b->InvAll);
  HB_LAUNCHED();
  b->inv_valid = true;
  return HB_OK;
}

// One block step of the factorization on the caller's operands: k_diag128 on the diagonal block at (k0, k0), then k_trsm_panel on the
// rows below it. LC(A, lda, i, j) must address element (i, j) for the columns of this block (global indices); nothing else of A is
// touched. inv16: 8 * 16 * 17 doubles of scratch; dinv: receives 1/d of the block (LDL^T); W: LDL^T only, W[c * ldw + i] = the row i >= k0 + 128
// of column c of W = L D (absolute i).
int hb_big_panel(int N, double* A, long long lda, int k0, bool ldl, double* inv16, double* dinv, double* W, long long ldw, int* info_dev, cudaStream_t st)
{
  const int nb = N - k0 < BB ? N - k0 : BB, r0 = k0 + nb;
  if(ldl) k_diag128<true><<<1, DTHREADS, sizeof(DiagSmem), st>>>(A, lda, N, k0, inv16, dinv, info_dev, nullptr);
  else k_diag128<false><<<1, DTHREADS, sizeof(DiagSmem), st>>>(A, lda, N, k0, inv16, dinv, info_dev, nullptr);
  HB_LAUNCHED();
  if(r0 < N) { // nb == 128 here (only the last block can be partial)
    const int ntile = (N - r0 + XROWS - 1) / XROWS;
    if(ldl) k_trsm_panel<true><<<ntile, 256, sizeof(TrsmSmem), st>>>(A, lda, N, k0, inv16, dinv, W, ldw);
    else k_trsm_panel<false><<<ntile, 256, sizeof(TrsmSmem), st>>>(A, lda, N, k0, inv16, dinv, nullptr, 0);
    HB_LAUNCHED();
  }
  return HB_OK;
}

// The trailing update of hb_big_factor (K = 128, 128 x 64 tiles of the lower triangle) on a block-cyclic matrix: C holds the 128-column
// blocks k = q * nranks + rank (local block q at C + q * 128 * ldc); the local blocks q0 .. q0 + nq - 1 receive
// C(i, j) -= sum_p P[p * ldp + i] Q[p * ldq + j - qsub], i >= j. Every entry sees the same operands in the same order as in hb_big_factor.
int hb_big_update_cyclic(int N, const double* P, long long ldp, const double* Q, long long ldq, int qsub, double* C, long long ldc, int nranks, int rank,
                         int q0, int nq, cudaStream_t st)
{
  if(nq <= 0) return HB_OK;
  GemmArgs g{};
  g.P = P; g.ldp = ldp;
  g.Q = Q; g.ldq = ldq; g.qsub = qsub;
  g.kb = BB;
  g.C = C; g.ldc = ldc;
  g.i_end = N; g.j_end = N;
  g.cyc_p = nranks; g.cyc_r = rank; g.cyc_q0 = q0;
  const int nti = (N - (q0 * nranks + rank) * BB + TM - 1) / TM; // rows of the first (largest) block column
  k_gemm_pq<64, EPI_SUB_CYC><<<dim3(nti, BB / 64, nq), 256, GemmCfg<64>::SMEM, st>>>(g);
  HB_LAUNCHED();
  return HB_OK;
}

// diagnostics: cycle counters of the phases of one k_diag128 launch on the block at k0 (the matrix is modified like in the factorization)
int hb_big_diag_profile(hb_ctx* c, hb_big* b, int N, double* A, long long lda, int k0, bool ldl, long long* prof_host8)
{
  HB_CHECK(hb_big_reserve(c, b, N, false));
  hb_dev<long long> prof;
  hb_dev<int> info;
  HB_CHECK(prof.reserve(c, 8, "profile counters"));
  HB_CHECK(info.reserve(c, 1, "profile info word"));
  HB_CUDA(cudaMemsetAsync(prof, 0, sizeof(long long) * 8, c->stream));
  HB_CUDA(cudaMemsetAsync(info, 0, sizeof(int), c->stream));
  if(ldl) k_diag128<true><<<1, DTHREADS, sizeof(DiagSmem), c->stream>>>(A, lda, N, k0, b->dinv + BB, b->dinv, info, prof);
  else k_diag128<false><<<1, DTHREADS, sizeof(DiagSmem), c->stream>>>(A, lda, N, k0, b->dinv + BB, b->dinv, info, prof);
  HB_LAUNCHED();
  HB_CUDA(cudaMemcpyAsync(prof_host8, prof, sizeof(long long) * 8, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}

// trailing update of a pivoted panel whose origin / width live in device memory (state[0] = k0, state[1] = kb): A22 -= W21 L21^T
int hb_big_trailing_from_state(hb_ctx* c, int N, double* A, long long lda, const double* W, long long ldw, const int* state_dev, int r0_min, cudaStream_t st)
{
  if(r0_min >= N) return HB_OK;
  GemmArgs g{};
  g.P = W; g.ldp = ldw; g.Q = nullptr; g.ldq = lda; g.qsub = 0; g.kb = 0;
  g.C = A; g.ldc = lda;
  g.i_base = g.j_base = r0_min; g.i_end = N; g.j_end = N; g.tj0 = 0;
  g.state = state_dev;
  const int org = r0_min & ~1; // the kernel rounds its tile origin down to an even row
  const int nti = (N - org + TM - 1) / TM, ntj = (N - org + 63) / 64;
  k_gemm_pq<64, EPI_SUB><<<dim3(nti, ntj), 256, GemmCfg<64>::SMEM, st>>>(g);
  HB_LAUNCHED();
  return HB_OK;
}

// 128 x 128 diagonal-block inverses of a factor produced by another path
int hb_big_block_inverses(hb_ctx* c, hb_big* b, int N, const double* F, long long ldf, bool unit)
{
  HB_CHECK(hb_big_reserve(c, b, N, false));
  const int nblk = (N + BB - 1) / BB;
  const int u = unit ? 1 : 0;
  k_block_inverses<<<nblk, DTHREADS, sizeof(DiagSmem), c->stream>>>(F, ldf, N, u, b->InvAll);
  HB_LAUNCHED();
  b->inv_valid = true;
  return HB_OK;
}

// x <- solution of (L [D] L^T) x = x with the factor F (+ b->InvAll). dmode: 0 = Cholesky (no D), 1 = D from the diagonal (LDL^T),
// 2 = Bunch-Kaufman block diagonal (ipiv_dev, dsub_dev), perm_dev (may be NULL): x is gathered through it first and scattered back at the end.
int hb_big_solve(hb_ctx* c, hb_big* b, int N, const double* F, long long ldf, int dmode, const int* ipiv_dev, const double* dsub_dev, const int* perm_dev,
                 double* x)
{
  HB_REQUIRE(b->inv_valid && b->capN >= N, "hb_big_solve: no block inverses for this factor");
  if(N == 0) return HB_OK;
  cudaStream_t st = c->stream;
  double* v = x;
  if(perm_dev) {
    k_gather<<<(N + 255) / 256, 256, 0, st>>>(N, perm_dev, x, b->xtmp);
    HB_LAUNCHED();
    v = b->xtmp;
  }
  // every step is launched with programmatic stream serialization: its CTAs start while the previous step still runs, prefetch what
  // does not depend on it, and wait (griddepcontrol.wait) for its completion before the first dependent access
  cudaLaunchAttribute pdl[1];
  pdl[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(ST);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cfg.attrs = pdl;
  cfg.numAttrs = 1;
  const double* InvAll = b->InvAll;
  double* partial = b->partial;
  int* counter = b->counter;
  for(int k0 = 0; k0 < N; k0 += SB) {
    const int G = (k0 + 63) / 64;
    cfg.gridDim = dim3(G + 1);
    cfg.numAttrs = k0 == 0 ? 0 : 1; // the first step follows foreign kernels (factorization, inverses, gather): plain stream order
    HB_CUDA(cudaLaunchKernelEx(&cfg, k_solve_fwd_step, F, ldf, N, k0, InvAll, v, partial, counter));
    HB_LAUNCHED();
  }
  if(dmode == 1) {
    k_dsolve<<<(N + 127) / 128, 128, 0, st>>>(F, ldf, N, v);
    HB_LAUNCHED();
  } else if(dmode == 2) {
    HB_CHECK(hb_bkc_dsolve(c, N, F, ldf, ipiv_dev, dsub_dev, v));
  }
  const int last = ((N - 1) / SB) * SB;
  for(int k0 = last; k0 >= 0; k0 -= SB) {
    const int nrows = N - k0 < SB ? N - k0 : SB;
    const int below = N - (k0 + nrows);
    const int G = (below + 63) / 64;
    cfg.gridDim = dim3(G + 1);
    cfg.numAttrs = (k0 == last && dmode != 0) ? 0 : 1; // after the diagonal solve kernel: plain stream order
    HB_CUDA(cudaLaunchKernelEx(&cfg, k_solve_bwd_step, F, ldf, N, k0, InvAll, v, partial, counter));
    HB_LAUNCHED();
  }
  if(perm_dev) {
    k_scatter<<<(N + 255) / 256, 256, 0, st>>>(N, perm_dev, b->xtmp, x);
    HB_LAUNCHED();
  }
  return HB_OK;
}
