// Single-launch blocked Cholesky for the small condensed systems (64 < N <= 2048) -- the latency-bound part of every KKT step.
//
// The multi-launch path of hb_dense.cu needs two kernels per 64-column panel and keeps 4 SMs busy in its panel kernel.
// Here ONE cooperative kernel walks the panels with two grid barriers per panel:
//   (1) every CTA factors the 64 x 64 diagonal block redundantly in shared memory (16-wide sub-panels; the inverse of each
//       16 x 16 triangle is kept so that all solves against it become small dense products with full thread parallelism),
//   (2) every CTA computes its few rows of L21 = A21 L11^-T from those inverses,            -- grid barrier --
//   (3) the 64 x 64 tiles of the trailing update are dealt round-robin to the CTAs.         -- grid barrier --
// Reference semantics: DPOTRF('L') on the column-major-lower view (hiopKKTLinSys.cpp:1228-1290 via DPOSVX; hiopDualsUpdater.cpp
// :717); info = first non-positive pivot (1-based), 0 if none.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace {

constexpr int CB = 64;   // panel width
constexpr int CT = 256;  // threads per CTA
constexpr int DS = CB + 1;
constexpr int PS = CB + 2; // stride of the P/Q tiles (16-byte aligned rows)
constexpr int XR = 32;     // rows of L21 a CTA handles per pass

struct CoopSmem
{
  double D[CB * DS];       // D[j*DS + i] = element (i, j) of the diagonal block / of L11
  double Inv[4 * 16 * 17]; // Inv[s][r*17 + c] = (T_s^-1)(r, c), T_s = s-th 16 x 16 diagonal triangle of L11
  double P[CB * PS];       // trailing update: P[p*PS + i];  L21 pass: X[r*DS + j]
  double Q[CB * PS];
};

// Right-looking Cholesky of the 64 x 64 diagonal block in shared memory, 16-wide sub-panels. Everything on the critical path is
// written to keep dependent FP64 chains short (one warp owns it; the first version spent 67 us here per panel, 75% of the kernel):
//   * pivots use rsqrt + multiply (no sqrt followed by a divide); 1/L_jj is kept for the triangular inverses,
//   * T^-1 is built right-looking (two dependent operations per column instead of a 16-term dot product + divide),
//   * the products against T^-1 and the rank-16 update accumulate in four independent partial sums.
__device__ void factor_diag(CoopSmem& S, int k0, int* info, bool report, long long* prof)
{
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long q0 = prof ? clock64() : 0;
#define QP(slot) if(prof) { const long long q1 = clock64(); prof[slot] += q1 - q0; q0 = q1; }
  for(int kb = 0; kb < CB; kb += 16) {
    if(warp == 0) {
      double a[16];
      double myr = 0.0; // 1 / L(lane, lane)
#pragma unroll
      for(int c = 0; c < 16; c++) a[c] = (lane < 16 && c <= lane) ? S.D[(kb + c) * DS + kb + lane] : 0.0;
      // spelled out per column: left to the unroller the 16 x 15 nest stayed rolled with a[] in local memory (LDL/STL on the
      // critical path, 960 cycles per column)
#define CHOL_COL(j)                                                                              \
  {                                                                                              \
    const double d = __shfl_sync(0xffffffffu, a[j], j);                                          \
    if(!(d > 0.0) && lane == 0 && report) atomicCAS(info, 0, k0 + kb + j + 1);                   \
    const double r = rsqrt(d);                                                                   \
    if(lane == j) { a[j] = d * r; myr = r; }                                                     \
    else if(lane > j) a[j] *= r;                                                                 \
    _Pragma("unroll") for(int c = j + 1; c < 16; c++) {                                          \
      const double lc = __shfl_sync(0xffffffffu, a[j], c);                                       \
      if(lane >= c) a[c] -= a[j] * lc;                                                           \
    }                                                                                            \
  }
      CHOL_COL(0) CHOL_COL(1) CHOL_COL(2) CHOL_COL(3) CHOL_COL(4) CHOL_COL(5) CHOL_COL(6) CHOL_COL(7)
      CHOL_COL(8) CHOL_COL(9) CHOL_COL(10) CHOL_COL(11) CHOL_COL(12) CHOL_COL(13) CHOL_COL(14) CHOL_COL(15)
#undef CHOL_COL
#pragma unroll
      for(int c = 0; c < 16; c++)
        if(lane < 16 && c <= lane) S.D[(kb + c) * DS + kb + lane] = a[c];
      __syncwarp();
      QP(6);
      // column `lane` of X = T^-1, right-looking: once x[q] is final every later partial sum is updated independently
      {
        double* inv = S.Inv + (kb / 16) * 16 * 17;
        double x[16], sacc[16];
#pragma unroll
        for(int r = 0; r < 16; r++) { x[r] = 0.0; sacc[r] = 0.0; }
#pragma unroll
        for(int q = 0; q < 16; q++) {
          const double rq = __shfl_sync(0xffffffffu, myr, q); // 1 / T(q, q)
          if(q == lane) x[q] = rq;
          else if(q > lane) x[q] = -sacc[q] * rq;
#pragma unroll
          for(int r = q + 1; r < 16; r++) sacc[r] += S.D[(kb + q) * DS + kb + r] * x[q];
        }
        if(lane < 16) {
#pragma unroll
          for(int r = 0; r < 16; r++) inv[r * 17 + lane] = x[r];
        }
      }
    }
    __syncthreads();
    QP(7);
    const int below = CB - kb - 16;
    {
      // rows below inside the block: L[r][kb+c] = sum_{q<=c} A[r][kb+q] * Tinv[c][q]
      const double* inv = S.Inv + (kb / 16) * 16 * 17;
      double y[3];
#pragma unroll
      for(int s = 0; s < 3; s++) {
        const int e = tid + s * CT;
        y[s] = 0.0;
        if(e < below * 16) {
          const int r = kb + 16 + e % below, c = e / below;
          double acc[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
          for(int q = 0; q < 16; q++)
            if(q <= c) acc[q & 3] += S.D[(kb + q) * DS + r] * inv[c * 17 + q];
          y[s] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
        }
      }
      __syncthreads();
#pragma unroll
      for(int s = 0; s < 3; s++) {
        const int e = tid + s * CT;
        if(e < below * 16) S.D[(kb + e / below) * DS + kb + 16 + e % below] = y[s];
      }
    }
    __syncthreads();
    QP(8);
    // rank-16 update of the remaining lower triangle: 2 x 2 register tiles over the (below/2)^2 grid, lower tiles only
    {
      const int hb2 = below / 2; // below is 48, 32, 16, 0
      for(int e = tid; e < hb2 * hb2; e += CT) {
        const int tc = e / hb2, ti = e % hb2;
        if(ti < tc) continue;
        const int c = kb + 16 + 2 * tc, i = kb + 16 + 2 * ti;
        double s00 = 0.0, s01 = 0.0, s10 = 0.0, s11 = 0.0;
#pragma unroll
        for(int p = 0; p < 16; p++) {
          const double li0 = S.D[(kb + p) * DS + i], li1 = S.D[(kb + p) * DS + i + 1];
          const double lc0 = S.D[(kb + p) * DS + c], lc1 = S.D[(kb + p) * DS + c + 1];
          s00 += li0 * lc0; s10 += li1 * lc0; s01 += li0 * lc1; s11 += li1 * lc1;
        }
        S.D[c * DS + i] -= s00;
        S.D[c * DS + i + 1] -= s10;
        S.D[(c + 1) * DS + i + 1] -= s11;
        if(ti > tc) S.D[(c + 1) * DS + i] -= s01; // (i, c+1) is above the diagonal when ti == tc
      }
    }
    __syncthreads();
    QP(9);
  }
#undef QP
}

__global__ void __launch_bounds__(CT, 1)
k_chol_coop(double* __restrict__ A, int lda, int N, int* __restrict__ info, double* __restrict__ invd /* may be NULL: 16 x 16 inverses per panel */,
            long long* __restrict__ prof /* may be NULL: 10 cycle counters of CTA 0 */)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  CoopSmem& S = *reinterpret_cast<CoopSmem*>(smem_raw);
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, G = gridDim.x, b = blockIdx.x;
  long long t0 = 0;
  const bool timing = prof && b == 0 && tid == 0;
#define PROF(slot)                      \
  if(timing) {                          \
    const long long t1 = clock64();     \
    prof[slot] += t1 - t0;              \
    t0 = t1;                            \
  }
  if(timing) t0 = clock64();
  for(int k0 = 0; k0 < N; k0 += CB) {
    const int nb = min(CB, N - k0);
    // ---- (1) diagonal block ----
    for(int e = tid; e < CB * CB; e += CT) {
      const int j = e / CB, i = e % CB;
      double v = (i == j) ? 1.0 : 0.0;
      if(i < nb && j < nb && i >= j) v = LC(A, lda, k0 + i, k0 + j);
      S.D[j * DS + i] = v;
    }
    __syncthreads();
    PROF(0);
    factor_diag(S, k0, info, b == 0, timing ? prof : nullptr);
    PROF(1);
    // CTA 0 stores the factored block -- but only after the next grid barrier: every CTA loaded the UNFACTORED block at the top of this
    // iteration and nothing orders a slow CTA's load before an in-place store made right here (the factor stays in S.D until then)
    auto store_diag = [&]() {
      if(b == 0) {
        for(int e = tid; e < nb * nb; e += CT) {
          const int j = e / nb, i = e % nb;
          if(i >= j) LC(A, lda, k0 + i, k0 + j) = S.D[j * DS + i];
        }
        if(invd)
          for(int e = tid; e < 4 * 16 * 17; e += CT) invd[(size_t)(k0 / CB) * (4 * 16 * 17) + e] = S.Inv[e];
      }
    };
    const int r0 = k0 + nb;
    const int R = N - r0;
    if(R <= 0) {
      grid.sync();
      store_diag();
      break;
    }
    // ---- (2) my rows of L21 = A21 L11^-T ----
    {
      const int per = (R + G - 1) / G;
      const int first = r0 + b * per, last = min(N, first + per);
      double* X = S.P; // X[r*DS + j]
      for(int c0 = first; c0 < last; c0 += XR) {
        const int rows = min(XR, last - c0);
        __syncthreads();
        for(int e = tid; e < rows * CB; e += CT) {
          const int j = e / rows, r = e % rows;
          X[r * DS + j] = j < nb ? LC(A, lda, c0 + r, k0 + j) : 0.0;
        }
        __syncthreads();
        for(int jb = 0; jb < CB; jb += 16) {
          const double* inv = S.Inv + (jb / 16) * 16 * 17;
          double y[2];
#pragma unroll
          for(int s = 0; s < 2; s++) { // rows * 16 <= 512 outputs
            const int e = tid + s * CT;
            y[s] = 0.0;
            if(e < rows * 16) {
              const int r = e % rows, c = e / rows;
              double acc = 0.0;
#pragma unroll
              for(int q = 0; q < 16; q++)
                if(q <= c) acc += X[r * DS + jb + q] * inv[c * 17 + q];
              y[s] = acc;
            }
          }
          __syncthreads();
#pragma unroll
          for(int s = 0; s < 2; s++) {
            const int e = tid + s * CT;
            if(e < rows * 16) X[(e % rows) * DS + jb + e / rows] = y[s];
          }
          __syncthreads();
          const int rem = CB - jb - 16;
          for(int e = tid; e < rows * rem; e += CT) {
            const int r = e % rows, c2 = jb + 16 + e / rows;
            double acc = 0.0;
#pragma unroll
            for(int q = 0; q < 16; q++) acc += X[r * DS + jb + q] * S.D[(jb + q) * DS + c2];
            X[r * DS + c2] -= acc;
          }
          __syncthreads();
        }
        for(int e = tid; e < rows * nb; e += CT) {
          const int j = e / rows, r = e % rows;
          LC(A, lda, c0 + r, k0 + j) = X[r * DS + j];
        }
      }
    }
    PROF(2);
    grid.sync();
    store_diag();
    PROF(3);
    // ---- (3) trailing update: Lc(i,j) -= sum_p L21[i][p] L21[j][p] on the lower triangle, 64 x 64 tiles round-robin ----
    {
      const int nt = (R + CB - 1) / CB;
      const int ntiles = nt * (nt + 1) / 2;
      const int ty = tid / 16, tx = tid % 16;
      for(int t = b; t < ntiles; t += G) {
        // t -> (ti >= tj)
        int ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
        while((ti + 1) * (ti + 2) / 2 <= t) ti++;
        while(ti * (ti + 1) / 2 > t) ti--;
        const int tj = t - ti * (ti + 1) / 2;
        const int ri = r0 + ti * CB, rj = r0 + tj * CB;
        __syncthreads();
        for(int e = tid; e < CB * CB; e += CT) {
          const int p = e / CB, i = e % CB;
          S.P[p * PS + i] = (p < nb && ri + i < N) ? LC(A, lda, ri + i, k0 + p) : 0.0;
          S.Q[p * PS + i] = (p < nb && rj + i < N) ? LC(A, lda, rj + i, k0 + p) : 0.0;
        }
        __syncthreads();
        // thread (ty, tx) owns rows ty*4..+3 and the INTERLEAVED columns tx, tx+16, tx+32, tx+48: the Q reads of a warp are 16
        // consecutive doubles (conflict-free, shared by its two ty values), the P reads two broadcast addresses -- with 4
        // consecutive columns per thread the loop was bound by shared-memory wavefronts at 2x the FP64 issue time
        double acc[4][4];
#pragma unroll
        for(int a = 0; a < 4; a++)
#pragma unroll
          for(int q = 0; q < 4; q++) acc[a][q] = 0.0;
#pragma unroll 8
        for(int p = 0; p < CB; p++) {
          const double2 p0 = *reinterpret_cast<const double2*>(&S.P[p * PS + ty * 4]);
          const double2 p1 = *reinterpret_cast<const double2*>(&S.P[p * PS + ty * 4 + 2]);
          const double pi[4] = {p0.x, p0.y, p1.x, p1.y};
          double qj[4];
#pragma unroll
          for(int q = 0; q < 4; q++) qj[q] = S.Q[p * PS + tx + 16 * q];
#pragma unroll
          for(int a = 0; a < 4; a++)
#pragma unroll
            for(int q = 0; q < 4; q++) acc[a][q] += pi[a] * qj[q];
        }
        // stage the 64 x 64 product through shared memory so that the read-modify-write of A runs down the columns (contiguous
        // in memory); writing it from the register tiles touched 32 sectors per warp instruction and made this phase 2.5x slower
        __syncthreads();
#pragma unroll
        for(int q = 0; q < 4; q++)
#pragma unroll
          for(int a = 0; a < 4; a++) S.P[(tx + 16 * q) * PS + ty * 4 + a] = acc[a][q];
        __syncthreads();
        {
          double cur[CB * CB / CT];
#pragma unroll
          for(int s = 0; s < CB * CB / CT; s++) {
            const int e = tid + s * CT;
            const int j = rj + e / CB, i = ri + e % CB;
            cur[s] = (i < N && j < N && i >= j) ? LC(A, lda, i, j) : 0.0;
          }
#pragma unroll
          for(int s = 0; s < CB * CB / CT; s++) {
            const int e = tid + s * CT;
            const int j = rj + e / CB, i = ri + e % CB;
            if(i < N && j < N && i >= j) LC(A, lda, i, j) = cur[s] - S.P[(e / CB) * PS + e % CB];
          }
        }
      }
    }
    PROF(4);
    grid.sync();
    PROF(5);
  }
#undef PROF
}


// ---------------------------------------------------------------------------------------------------------------------
// Cooperative SPD solve with the factor above: x = S F^-T F^-1 S rhs, then the residual check against the unscaled matrix and
// up to max_refine corrections (hiopKKTLinSysLowRank::solveWithRefin, hiopKKTLinSys.cpp:1192-1350: ||rhs - N x||_inf < tol).
// The one-CTA version streamed the 8 MB factor twice + N once through a single SM. Here every CTA solves
// the 64-entry diagonal block redundantly from the stored 16 x 16 inverses and updates only its own slice of the remaining
// vector (rows in the forward sweep, columns in the backward sweep); one grid barrier per block.
// ---------------------------------------------------------------------------------------------------------------------
struct SolveSmem
{
  double z[CB];
  double y[16];
  double Inv[4 * 16 * 17];
  double L[CB * DS]; // L[j*DS + i] = element (i, j) of the diagonal block of the factor
  double red[32];
};

// in-block solve with the lower triangle (trans = false: L z' = z; true: L^T z' = z), result in S.z
__device__ void block_solve(SolveSmem& S, bool trans)
{
  const int tid = threadIdx.x;
  for(int step = 0; step < 4; step++) {
    const int sb = trans ? 3 - step : step;
    const double* inv = S.Inv + sb * 16 * 17;
    if(tid < 16) {
      double acc = 0.0;
#pragma unroll
      for(int q = 0; q < 16; q++) {
        // (T^-1 z)_c = sum_{q<=c} inv[c][q] z[q];   (T^-T z)_c = sum_{q>=c} inv[q][c] z[q]
        const double w = trans ? (q >= tid ? inv[q * 17 + tid] : 0.0) : (q <= tid ? inv[tid * 17 + q] : 0.0);
        acc += w * S.z[sb * 16 + q];
      }
      S.y[tid] = acc;
    }
    __syncthreads();
    if(tid < 16) S.z[sb * 16 + tid] = S.y[tid];
    // eliminate the solved 16 unknowns from the rest of the block
    if(!trans) {
      const int r = (sb + 1) * 16 + tid - 16; // rows below: tid 16.. -> r = (sb+1)*16 ..
      if(tid >= 16 && r < CB) {
        double acc = 0.0;
#pragma unroll
        for(int q = 0; q < 16; q++) acc += S.L[(sb * 16 + q) * DS + r] * S.y[q];
        S.z[r] -= acc;
      }
    } else {
      const int cidx = tid - 16; // columns before: c < sb*16
      if(tid >= 16 && cidx < sb * 16) {
        double acc = 0.0;
#pragma unroll
        for(int q = 0; q < 16; q++) acc += S.L[cidx * DS + sb * 16 + q] * S.y[q];
        S.z[cidx] -= acc;
      }
    }
    __syncthreads();
  }
}

// v is updated by other CTAs between the grid barriers of coop_potrs: no read-only promise on it, loads go to L2
__device__ void load_block(SolveSmem& S, const double* __restrict__ F, int ldf, int N, const double* __restrict__ invd, const double* v, int k0)
{
  const int tid = threadIdx.x;
  const int nb = min(CB, N - k0);
  for(int e = tid; e < 4 * 16 * 17; e += CT) S.Inv[e] = invd[(size_t)(k0 / CB) * (4 * 16 * 17) + e];
  for(int e = tid; e < CB * CB; e += CT) {
    const int j = e / CB, i = e % CB;
    S.L[j * DS + i] = (i < nb && j < nb && i >= j) ? LC(F, ldf, k0 + i, k0 + j) : 0.0;
  }
  if(tid < CB) S.z[tid] = tid < nb ? __ldcg(v + k0 + tid) : 0.0;
  __syncthreads();
}

// v <- F^-T F^-1 v (v, w in global memory, length N; w is scratch).
// Every CTA reads the current 64-entry block, solves it redundantly and updates its slice of the remaining entries; ONE CTA stores the
// solved block. That store must not land where a slower CTA may still be reading the unsolved block of the same step (there is no grid
// barrier between the read and the store): the forward sweep therefore reads v and stores its solved blocks into w, the backward sweep
// reads w and stores into v. (The first version stored in place; a late CTA then occasionally loaded already-solved entries, the first
// solve came out wrong and the refinement loop repaired it -- one extra correction and last-bit differences from run to run.)
__device__ void coop_potrs(SolveSmem& S, cg::grid_group& grid, const double* __restrict__ F, int ldf, int N, const double* __restrict__ invd,
                           double* v, double* w)
{
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x, b = blockIdx.x;
  const int nblk = (N + CB - 1) / CB;
  for(int kb = 0; kb < nblk; kb++) { // forward: L z = v
    const int k0 = kb * CB, nb = min(CB, N - k0);
    load_block(S, F, ldf, N, invd, v, k0);
    block_solve(S, false);
    const int r0 = k0 + nb, R = N - r0;
    if(R > 0) {
      const int per = (R + G - 1) / G;
      const int first = r0 + b * per, last = min(N, first + per);
      for(int r = first + warp; r < last; r += CT / 32) { // one warp per row: v[r] -= L[r, k0:k0+nb] . z
        double acc = 0.0;
        for(int q = lane; q < nb; q += 32) acc += LC(F, ldf, r, k0 + q) * S.z[q];
        acc = hb_warp_sum(acc);
        if(lane == 0) v[r] = __ldcg(v + r) - acc;
      }
    }
    if(b == 0 && tid < nb) w[k0 + tid] = S.z[tid];
    grid.sync();
  }
  for(int kb = nblk - 1; kb >= 0; kb--) { // backward: L^T x = z (z in w)
    const int k0 = kb * CB, nb = min(CB, N - k0);
    load_block(S, F, ldf, N, invd, w, k0);
    block_solve(S, true);
    if(k0 > 0) {
      const int per = (k0 + G - 1) / G;
      const int first = b * per, last = min(k0, first + per);
      for(int cix = first + warp; cix < last; cix += CT / 32) { // one warp per column: w[c] -= L[k0:k0+nb, c] . x_k (contiguous)
        double acc = 0.0;
        for(int q = lane; q < nb; q += 32) acc += LC(F, ldf, k0 + q, cix) * S.z[q];
        acc = hb_warp_sum(acc);
        if(lane == 0) w[cix] = __ldcg(w + cix) - acc;
      }
    }
    if(b == 0 && tid < nb) v[k0 + tid] = S.z[tid];
    grid.sync();
  }
}

__global__ void __launch_bounds__(CT, 1)
k_spd_solve_coop(const double* __restrict__ F, int ldf, int N, const double* __restrict__ invd, const double* __restrict__ s,
                 const double* __restrict__ Nref, int ldn, const double* __restrict__ rhs, double* __restrict__ x, double* __restrict__ work /* 2N+2 */,
                 double tol, int max_refine, double* __restrict__ stats)
{
  __shared__ SolveSmem S;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x, b = blockIdx.x;
  const int gtid = b * CT + tid, gthreads = G * CT;
  double* v = work;     // vector being solved (scaled)
  double* r = work + N; // residual
  unsigned long long* nrm_bits = reinterpret_cast<unsigned long long*>(work + 2 * N); // two slots, used alternately
  for(int i = gtid; i < N; i += gthreads) v[i] = rhs[i] * s[i];
  if(gtid < 2) nrm_bits[gtid] = 0ull;
  grid.sync();
  coop_potrs(S, grid, F, ldf, N, invd, v, r); // r is free until the first residual
  for(int i = gtid; i < N; i += gthreads) x[i] = __ldcg(v + i) * s[i];
  grid.sync();
  int nref = 0;
  double nrm = 0.0;
  while(true) {
    // r = rhs - Nref x, one warp per row; ||r||_inf through an integer max on the bit pattern (r >= 0)
    unsigned long long* slot = nrm_bits + (nref & 1);
    double wmax = 0.0;
    for(int i = b * (CT / 32) + warp; i < N; i += G * (CT / 32)) {
      double acc = 0.0;
      const double* row = Nref + (size_t)i * ldn;
      for(int j = lane; j < N; j += 32) acc += row[j] * __ldcg(x + j);
      acc = hb_warp_sum(acc);
      const double ri = rhs[i] - acc;
      if(lane == 0) r[i] = ri;
      wmax = hb_nan_max(wmax, fabs(ri));
    }
    if(lane == 0) {
      const double m = wmax == wmax ? wmax : __longlong_as_double(0x7ff0000000000000LL); // NaN -> +inf so that it wins the max
      atomicMax(slot, (unsigned long long)__double_as_longlong(m));
    }
    grid.sync();
    nrm = __longlong_as_double((long long)*slot);
    if(isinf(nrm) || !(nrm >= tol) || nref >= max_refine) break; // a residual that is not finite stops the loop (reported as NaN)
    if(gtid == 0) nrm_bits[(nref + 1) & 1] = 0ull; // the other slot is idle until the next round's barrier
    for(int i = gtid; i < N; i += gthreads) v[i] = __ldcg(r + i) * s[i];
    grid.sync();
    coop_potrs(S, grid, F, ldf, N, invd, v, r); // the residual has been consumed (v = r .* s above)
    for(int i = gtid; i < N; i += gthreads) x[i] += __ldcg(v + i) * s[i];
    grid.sync();
    nref++;
  }
  if(gtid == 0) {
    stats[0] = (double)nref;
    stats[1] = isinf(nrm) ? __longlong_as_double(0x7ff8000000000000LL) : nrm;
  }
}

// 16 x 16 inverses of the diagonal triangles of an existing factor (the multi-launch Cholesky for N > 2048 does not produce them):
// one CTA per 64-block, thread (sb, c) builds column c of T_sb^-1 right-looking like factor_diag does.
__global__ void __launch_bounds__(64)
k_diag_inverses(const double* __restrict__ F, int ldf, int N, double* __restrict__ invd)
{
  __shared__ double T[4][16][17];
  const int k0 = blockIdx.x * CB, tid = threadIdx.x, sb = tid >> 4, c = tid & 15;
  for(int e = tid; e < 4 * 256; e += 64) {
    const int s = e >> 8, r = (e >> 4) & 15, q = e & 15;
    const int gi = k0 + s * 16 + r, gj = k0 + s * 16 + q;
    T[s][r][q] = (gi < N && gj < N && r >= q) ? LC(F, ldf, gi, gj) : (r == q ? 1.0 : 0.0); // identity beyond N, as the padded panels
  }
  __syncthreads();
  double x[16], sacc[16];
#pragma unroll
  for(int r = 0; r < 16; r++) { x[r] = 0.0; sacc[r] = 0.0; }
#pragma unroll
  for(int q = 0; q < 16; q++) {
    const double rq = 1.0 / T[sb][q][q];
    if(q == c) x[q] = rq;
    else if(q > c) x[q] = -sacc[q] * rq;
#pragma unroll
    for(int r = q + 1; r < 16; r++) sacc[r] += T[sb][r][q] * x[q];
  }
  double* inv = invd + (size_t)blockIdx.x * (4 * 16 * 17) + sb * 16 * 17;
#pragma unroll
  for(int r = 0; r < 16; r++) inv[r * 17 + c] = x[r];
}

} // namespace

int hb_chol_coop_init(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_chol_coop, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSmem)));
  int coop = 0, occ = 0, occ_solve = 0;
  HB_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, c->device));
  HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_chol_coop, CT, sizeof(CoopSmem)));
  HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_solve, k_spd_solve_coop, CT, 0));
  // every CTA of a cooperative launch must be resident at once; one per SM (the solve never launches more than one per SM either)
  c->coop_ctas = (coop && occ >= 1 && occ_solve >= 1) ? c->num_sms : 0;
  return HB_OK;
}

int hb_dense_chol_coop(hb_ctx* c, int N, double* A, int lda, int* info_dev, double* invd, long long* prof)
{
  // one CTA per trailing tile of the first panel (the widest step), never more than fit on the device at once
  const int nt0 = (N - CB + CB - 1) / CB;
  int G = nt0 * (nt0 + 1) / 2;
  if(G > c->coop_ctas) G = c->coop_ctas;
  if(G < 1) G = 1;
  HB_CUDA(cudaMemsetAsync(info_dev, 0, sizeof(int), c->stream));
  void* args[] = {&A, &lda, &N, &info_dev, &invd, &prof};
  HB_CUDA(cudaLaunchCooperativeKernel((const void*)k_chol_coop, dim3(G), dim3(CT), args, sizeof(CoopSmem), c->stream));
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_chol_diag_inverses(hb_ctx* c, int N, const double* F, int ldf, double* invd)
{
  if(N <= 0) return HB_OK;
  k_diag_inverses<<<(N + CB - 1) / CB, 64, 0, c->stream>>>(F, ldf, N, invd);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_spd_solve_coop(hb_ctx* c, int N, const double* F, int ldf, const double* invd, const double* s, const double* Nref, int ldn,
                            const double* rhs, double* x, double* work, double tol, int max_refine, double* stats_dev)
{
  int G = (N + 7) / 8; // ~8 rows / columns per CTA in the widest sweep step, one row of the residual per warp
  if(G > c->coop_ctas) G = c->coop_ctas;
  void* args[] = {&F, &ldf, &N, &invd, &s, &Nref, &ldn, &rhs, &x, &work, &tol, &max_refine, &stats_dev};
  HB_CUDA(cudaLaunchCooperativeKernel((const void*)k_spd_solve_coop, dim3(G), dim3(CT), args, 0, c->stream));
  HB_LAUNCHED();
  return HB_OK;
}
