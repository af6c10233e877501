// Dense symmetric factorizations and solves on device (FP64):
//   * blocked Cholesky LL^T and no-pivot LDL^T  (DPOTRF / magma_dsytrf_nopiv_gpu roles)
//   * Bunch-Kaufman LDL^T with the LAPACK pivoting rule (DSYTRF / magma_dsytrf_gpu roles) + DSYTRS
//   * inertia from the 1x1 / 2x2 pivots with the reference's dsidi rule and +-1e-14 thresholds
//     (src/LinAlg/hiopLinSolverSymDenseLapack.hpp:127-167)
//   * equilibrated SPD solve with device-side residual-driven refinement (hiopKKTLinSysLowRank::solveWithRefin,
//     src/Optimization/hiopKKTLinSys.cpp:1192-1350)
//
// Storage convention of the whole file: the system matrix is N x N ROW-major with its UPPER triangle valid
// (hiopKKTLinSysMDS.cpp:196-206). Read column-major that is the LOWER triangle, which is how LAPACK sees it
// (uplo='L', hiopLinSolverSymDenseLapack.hpp:84) and how the kernels index it:  Lc(i,j) = A[j*lda + i], i >= j.
// Column j of the factor is therefore contiguous in memory -> coalesced along i.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include "hb_ptx.cuh"

namespace {

constexpr int NB = 64;             // panel width of the blocked factorizations
constexpr int PANEL_THREADS = 256; // one row of the slab per thread

// ---------------------------------------------------------------------------------------------------------
// Panel kernel: every CTA factors the nb x nb diagonal block in shared memory (redundantly -- it is 64^3/3 flops),
// CTA 0 writes it back, and each CTA then computes its 256-row slab of L21 by forward substitution, one row per
// thread. LDL variant also emits W = L21*D (needed by the trailing update) into Wout (nb rows of length ldw).
// ---------------------------------------------------------------------------------------------------------
template <bool LDL>
__global__ void __launch_bounds__(PANEL_THREADS)
k_panel(double* __restrict__ A, int lda, int N, int k0, int nb, double* __restrict__ Wout, int ldw, int* __restrict__ info)
{
  __shared__ double D[NB][NB + 1];
  __shared__ double dinv[NB];
  const int tid = threadIdx.x;
  // load the lower part of the diagonal block; pad to identity beyond nb
  {
    double v[NB * NB / PANEL_THREADS];
#pragma unroll
    for(int q = 0; q < NB * NB / PANEL_THREADS; q++) { // all loads first (independent), then the stores
      const int e = tid + q * PANEL_THREADS;
      const int j = e / NB, i = e % NB;
      v[q] = (i == j) ? 1.0 : 0.0;
      if(i < nb && j < nb && i >= j) v[q] = LC(A, lda, k0 + i, k0 + j);
    }
#pragma unroll
    for(int q = 0; q < NB * NB / PANEL_THREADS; q++) {
      const int e = tid + q * PANEL_THREADS;
      D[e / NB][e % NB] = v[q]; // D[j][i] holds element (i,j)
    }
  }
  __syncthreads();
  if(!LDL) {
    // Blocked right-looking Cholesky of the 64x64 diagonal block in shared memory, 16-wide sub-panels, 3 barriers per
    // sub-panel (12 in total instead of 2-3 per column):
    //   (1) warp 0 factors the 16x16 diagonal sub-block in registers (lane r holds row r) with shuffles,
    //   (2) one thread per row below solves its 16 entries against it,
    //   (3) all threads apply the rank-16 update to the remaining lower triangle.
    // D beyond nb is the identity, so a partial last panel needs no special casing.
    const int lane = tid & 31, warp = tid >> 5;
    for(int kb = 0; kb < NB; kb += 16) {
      if(warp == 0) {
        double a[16];
#pragma unroll
        for(int c = 0; c < 16; c++) a[c] = (lane < 16 && c <= lane) ? D[kb + c][kb + lane] : 0.0;
        // spelled out per column: the 16 x 15 nest does not get fully unrolled otherwise and a[] lands in local memory
#define PANEL_CHOL_COL(j)                                                                      \
  {                                                                                            \
    const double d = __shfl_sync(0xffffffffu, a[j], j);                                        \
    if(!(d > 0.0) && lane == 0 && blockIdx.x == 0) atomicCAS(info, 0, k0 + kb + j + 1);       \
    const double l = sqrt(d);                                                                  \
    if(lane == j) a[j] = l;                                                                    \
    else if(lane > j) a[j] = a[j] / l;                                                         \
    _Pragma("unroll") for(int c = j + 1; c < 16; c++) {                                        \
      const double lc = __shfl_sync(0xffffffffu, a[j], c);                                     \
      if(lane >= c) a[c] -= a[j] * lc;                                                         \
    }                                                                                          \
  }
        PANEL_CHOL_COL(0) PANEL_CHOL_COL(1) PANEL_CHOL_COL(2) PANEL_CHOL_COL(3) PANEL_CHOL_COL(4) PANEL_CHOL_COL(5) PANEL_CHOL_COL(6)
        PANEL_CHOL_COL(7) PANEL_CHOL_COL(8) PANEL_CHOL_COL(9) PANEL_CHOL_COL(10) PANEL_CHOL_COL(11) PANEL_CHOL_COL(12) PANEL_CHOL_COL(13)
        PANEL_CHOL_COL(14) PANEL_CHOL_COL(15)
#undef PANEL_CHOL_COL
#pragma unroll
        for(int c = 0; c < 16; c++)
          if(lane < 16 && c <= lane) D[kb + c][kb + lane] = a[c];
      }
      __syncthreads();
      const int below = NB - kb - 16;
      if(tid < below) {
        const int r = kb + 16 + tid;
        double x[16];
#pragma unroll
        for(int c = 0; c < 16; c++) x[c] = D[kb + c][r];
#pragma unroll
        for(int j = 0; j < 16; j++) {
          x[j] /= D[kb + j][kb + j];
          const double xj = x[j];
#pragma unroll
          for(int q = j + 1; q < 16; q++) x[q] -= xj * D[kb + j][kb + q];
        }
#pragma unroll
        for(int c = 0; c < 16; c++) D[kb + c][r] = x[c];
      }
      __syncthreads();
      for(int e = tid; e < below * below; e += PANEL_THREADS) {
        const int c = kb + 16 + e / below, i = kb + 16 + e % below;
        if(i >= c) {
          double s = 0.0;
#pragma unroll
          for(int p = 0; p < 16; p++) s += D[kb + p][i] * D[kb + p][c];
          D[c][i] -= s;
        }
      }
      __syncthreads();
    }
  } else {
  for(int j = 0; j < nb; j++) {
    const double ajj = D[j][j];
    {
      if(ajj == 0.0 || ajj != ajj) {
        if(tid == 0 && blockIdx.x == 0) atomicCAS(info, 0, k0 + j + 1);
      }
      const double r = 1.0 / ajj;
      const int rem = nb - j - 1;
      __syncthreads();
      // trailing uses w = column j (unscaled) and l = w / d
      for(int e = tid; e < rem * rem; e += PANEL_THREADS) {
        const int c = j + 1 + e / rem, i = j + 1 + e % rem;
        if(i >= c) D[c][i] -= D[j][i] * r * D[j][c];
      }
      __syncthreads();
      for(int i = j + 1 + tid; i < nb; i += PANEL_THREADS) D[j][i] *= r;
      if(tid == 0) dinv[j] = r;
      __syncthreads();
    }
  }
  }
  if(blockIdx.x == 0) {
    for(int e = tid; e < nb * nb; e += PANEL_THREADS) {
      const int j = e / nb, i = e % nb;
      if(i >= j) LC(A, lda, k0 + i, k0 + j) = D[j][i];
    }
  }
  // slab rows
  const int i = k0 + nb + blockIdx.x * PANEL_THREADS + tid;
  if(i < N) {
    double x[NB];
#pragma unroll
    for(int j = 0; j < NB; j++) x[j] = j < nb ? LC(A, lda, i, k0 + j) : 0.0;
    // right-looking forward substitution: once x[j] is final, all later entries are updated independently (ILP 63..1
    // instead of a dependent chain per entry)
#pragma unroll
    for(int j = 0; j < NB; j++) {
      if(!LDL) x[j] /= D[j][j];
      const double xj = x[j];
#pragma unroll
      for(int q = j + 1; q < NB; q++) x[q] -= xj * D[j][q]; // element (q,j) of L11
    }
    if(LDL) {
#pragma unroll
      for(int j = 0; j < NB; j++)
        if(j < nb) {
          Wout[(size_t)j * ldw + i] = x[j];
          LC(A, lda, i, k0 + j) = x[j] * dinv[j];
        }
    } else {
#pragma unroll
      for(int j = 0; j < NB; j++)
        if(j < nb) LC(A, lda, i, k0 + j) = x[j];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Trailing update on the DMMA pipe: for i >= j >= r0:  Lc(i,j) -= sum_p P[p][i] * Q[p][j],  p < kb.
// P, Q are kb "row-contiguous" panels: P[p][i] = Pbase[p*ldp + i] (for Cholesky P = Q = the factor panel rows,
// for LDL^T P = W = L*D, Q = L). 64x64 output tiles, 4 warps (2x2), warp tile 32x32. P feeds the A fragments, Q the B fragments:
// swapping the two would change the rounding of every product.
// FROM_STATE (blocked Bunch-Kaufman): the panel's origin k0 and width kb are read from the device state word (state[0], state[1]),
// r0 = k0 + kb, P = L21 (the panel's columns of A) and Q = W21; the grid covers the widest remainder the panel can leave.
// ---------------------------------------------------------------------------------------------------------
constexpr int TT = 64;
constexpr int TLD = TT + 4; // padded: fragment reads (p = lane%4, i = lane/4) are bank-conflict free
template <bool FROM_STATE>
__global__ void __launch_bounds__(128)
k_trailing(double* __restrict__ A, int lda, int N, int r0, const double* __restrict__ P, long long ldp, const double* __restrict__ Q,
           long long ldq, int kb, const int* __restrict__ state)
{
  extern __shared__ __align__(16) unsigned char trailing_smem[];
  double (*sP)[TLD] = reinterpret_cast<double (*)[TLD]>(trailing_smem);
  double (*sQ)[TLD] = sP + NB;
  if(FROM_STATE) {
    const int k0 = state[0];
    kb = state[1];
    r0 = k0 + kb;
    if(kb == 0 || r0 >= N) return;
    P = A + (size_t)k0 * lda;
    ldp = lda;
  }
  // linear tile id -> (ti >= tj)
  int t = blockIdx.x, ti = 0;
  while(t >= ti + 1) { t -= ti + 1; ti++; }
  const int tj = t;
  if(FROM_STATE && ti >= (N - r0 + TT - 1) / TT) return;
  const int i0 = r0 + ti * TT, j0 = r0 + tj * TT;
  const int tid = threadIdx.x;
  {
    // all 8-byte copies of the two operand tiles are issued back to back (one L2 latency for the whole tile instead of
    // one per loop iteration); columns beyond N and the K padding are zero-filled through the src-size operand
    const int kpad = ((kb + 3) / 4) * 4;
    for(int e = tid; e < kpad * TT; e += 128) {
      const int p = e / TT, c = e % TT;
      const bool vp = (p < kb) && (i0 + c < N), vq = (p < kb) && (j0 + c < N);
      const double* gp = vp ? P + (size_t)p * ldp + i0 + c : P;
      const double* gq = vq ? Q + (size_t)p * ldq + j0 + c : Q;
      hb_cp_async8(&sP[p][c], gp, vp ? 8 : 0);
      hb_cp_async8(&sQ[p][c], gq, vq ? 8 : 0);
    }
    hb_cp_async_wait_all();
  }
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5;
  const int wi = warp & 1, wj = warp >> 1;
  const int g = lane >> 2, t4 = lane & 3;
  double acc[4][4][2];
#pragma unroll
  for(int a = 0; a < 4; a++)
#pragma unroll
    for(int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.0;
  const int ksteps = (kb + 3) / 4;
  for(int kk = 0; kk < ksteps; kk++) {
    double af[4], bf[4];
#pragma unroll
    for(int a = 0; a < 4; a++) af[a] = sP[kk * 4 + t4][wi * 32 + a * 8 + g];
#pragma unroll
    for(int b = 0; b < 4; b++) bf[b] = sQ[kk * 4 + t4][wj * 32 + b * 8 + g];
#pragma unroll
    for(int a = 0; a < 4; a++)
#pragma unroll
      for(int b = 0; b < 4; b++) hb_dmma884(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
  }
  // epilogue: all loads of the C tile first, then all stores (a load->sub->store chain per element would serialise on
  // L2 latency because the compiler must assume the stores alias the following loads)
  double cv[4][4][2];
#pragma unroll
  for(int a = 0; a < 4; a++) {
    const int i = i0 + wi * 32 + a * 8 + g;
#pragma unroll
    for(int b = 0; b < 4; b++)
#pragma unroll
      for(int h = 0; h < 2; h++) {
        const int j = j0 + wj * 32 + b * 8 + t4 * 2 + h;
        cv[a][b][h] = (i < N && j < N && i >= j) ? LC(A, lda, i, j) : 0.0;
      }
  }
#pragma unroll
  for(int a = 0; a < 4; a++) {
    const int i = i0 + wi * 32 + a * 8 + g;
#pragma unroll
    for(int b = 0; b < 4; b++)
#pragma unroll
      for(int h = 0; h < 2; h++) {
        const int j = j0 + wj * 32 + b * 8 + t4 * 2 + h;
        if(i < N && j < N && i >= j) LC(A, lda, i, j) = cv[a][b][h] - acc[a][b][h];
      }
  }
}

// ---------------------------------------------------------------------------------------------------------
// CTA-wide triangular solves with a column-major-lower factor (1024 threads). x lives in global memory.
// unit_diag: LDL^T factors (L has an implicit unit diagonal).
// ---------------------------------------------------------------------------------------------------------
constexpr int SOLVE_THREADS = 1024;

// sd: 32 x 33 doubles of shared memory holding the current diagonal block (sd[c][r] = L(j0+r, j0+c)): one coalesced
// load instead of 32 dependent L2 round trips inside the sequential part.
__device__ void dev_forward(const double* __restrict__ A, int lda, int N, double* x, bool unit_diag, double (*sd)[33])
{
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for(int j0 = 0; j0 < N; j0 += 32) {
    const int nb = min(32, N - j0);
    {
      const int c = tid >> 5, r = tid & 31; // 1024 threads = one 32x32 block
      if(c < nb && r < nb && r >= c) sd[c][r] = LC(A, lda, j0 + r, j0 + c);
    }
    __syncthreads();
    if(warp == 0) {
      double b = lane < nb ? x[j0 + lane] : 0.0;
      for(int c = 0; c < nb; c++) {
        double yc = __shfl_sync(0xffffffffu, b, c);
        if(!unit_diag) yc /= sd[c][c];
        if(lane == c) b = yc;
        if(lane > c && lane < nb) b -= sd[c][lane] * yc;
      }
      if(lane < nb) x[j0 + lane] = b;
    }
    __syncthreads();
    for(int i = j0 + nb + tid; i < N; i += SOLVE_THREADS) {
      double s = x[i];
#pragma unroll 8
      for(int c = 0; c < nb; c++) s -= LC(A, lda, i, j0 + c) * x[j0 + c];
      x[i] = s;
    }
    __syncthreads();
  }
}

__device__ void dev_backward(const double* __restrict__ A, int lda, int N, double* x, bool unit_diag, double* sm32 /* 32 doubles */,
                             double (*sd)[33])
{
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nblk = (N + 31) / 32;
  for(int bi = nblk - 1; bi >= 0; bi--) {
    const int j0 = bi * 32;
    const int nb = min(32, N - j0);
    {
      const int c = tid >> 5, r = tid & 31;
      if(c < nb && r < nb && r >= c) sd[c][r] = LC(A, lda, j0 + r, j0 + c);
    }
    // each warp: dot of column (j0+warp) below the block with the already solved tail of x
    if(warp < nb) {
      double s = 0.0;
#pragma unroll 8
      for(int i = j0 + nb + lane; i < N; i += 32) s += LC(A, lda, i, j0 + warp) * x[i];
      s = hb_warp_sum(s);
      if(lane == 0) sm32[warp] = s;
    }
    __syncthreads();
    if(warp == 0) {
      double b = lane < nb ? x[j0 + lane] - sm32[lane] : 0.0;
      for(int c = nb - 1; c >= 0; c--) {
        // x_c = (b_c - sum_{t>c} L(t,c) x_t) / L(c,c)
        double part = (lane > c && lane < nb) ? sd[c][lane] * b : 0.0;
        part = hb_warp_sum(part);
        if(lane == c) {
          b = b - part;
          if(!unit_diag) b /= sd[c][c];
        }
      }
      if(lane < nb) x[j0 + lane] = b;
    }
    __syncthreads();
  }
}

// One-CTA SPD solve with equilibration scaling s and device-side refinement against the unscaled matrix Nref
// (full symmetric storage, row-major, ld = ldn). stats: [0]=#refinements, [1]=last residual inf-norm, [2]=info.
__global__ void __launch_bounds__(SOLVE_THREADS)
k_spd_solve_refine(const double* __restrict__ F, int ldf, int N, const double* __restrict__ s, const double* __restrict__ Nref, int ldn,
                   const double* __restrict__ rhs, double* __restrict__ x, double* __restrict__ work /* 2N */, double tol, int max_refine,
                   double* __restrict__ stats)
{
  __shared__ double sm[32];
  __shared__ double sd[32][33];
  __shared__ double s_nrm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* r = work;       // residual / correction
  double* z = work + N;   // scaled rhs
  for(int i = tid; i < N; i += SOLVE_THREADS) z[i] = rhs[i] * s[i];
  __syncthreads();
  dev_forward(F, ldf, N, z, false, sd);
  dev_backward(F, ldf, N, z, false, sm, sd);
  for(int i = tid; i < N; i += SOLVE_THREADS) x[i] = z[i] * s[i];
  __syncthreads();
  int nref = 0;
  double nrm = 0.0;
  while(true) {
    // r = rhs - Nref*x : one warp per row (rows are contiguous)
    double wmax = 0.0;
    for(int i = warp; i < N; i += SOLVE_THREADS / 32) {
      double acc = 0.0;
      const double* row = Nref + (size_t)i * ldn;
      for(int j = lane; j < N; j += 32) acc += row[j] * x[j];
      acc = hb_warp_sum(acc);
      const double ri = rhs[i] - acc;
      if(lane == 0) r[i] = ri;
      wmax = fmax(wmax, fabs(ri));
    }
    __syncthreads();
    if(lane == 0) sm[warp] = wmax;
    __syncthreads();
    if(tid == 0) {
      double m = 0.0;
      for(int w = 0; w < SOLVE_THREADS / 32; w++) m = fmax(m, sm[w]);
      s_nrm = m;
    }
    __syncthreads();
    nrm = s_nrm;
    if(!(nrm >= tol) || nref >= max_refine) break; // also leaves on NaN
    for(int i = tid; i < N; i += SOLVE_THREADS) r[i] *= s[i];
    __syncthreads();
    dev_forward(F, ldf, N, r, false, sd);
    dev_backward(F, ldf, N, r, false, sm, sd);
    for(int i = tid; i < N; i += SOLVE_THREADS) x[i] += r[i] * s[i];
    __syncthreads();
    nref++;
  }
  if(tid == 0) {
    stats[0] = (double)nref;
    stats[1] = nrm;
  }
}

// s_i = 1/sqrt(A_ii); F(i,j) = s_i A(i,j) s_j on the column-major-lower triangle (equilibration of DPOSVX('E'):
// always applied here -- a symmetric diagonal scaling never changes the exact solution).
__global__ void k_equilibrate(const double* __restrict__ Nfull, int ldn, int N, double* __restrict__ F, int ldf, double* __restrict__ s)
{
  const long long total = (long long)N * N;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e / N), i = (int)(e % N);
    const double sj = 1.0 / sqrt(Nfull[(size_t)j * ldn + j]);
    if(i == j) s[j] = sj;
    if(i >= j) {
      const double si = 1.0 / sqrt(Nfull[(size_t)i * ldn + i]);
      LC(F, ldf, i, j) = si * Nfull[(size_t)j * ldn + i] * sj;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Unblocked Bunch-Kaufman (DSYTF2 'L' logic, bit-compatible pivot choices with LAPACK) in one CTA.
// Used for the 2l x 2l matrix V of the compact BFGS inverse and for small KKT systems; the blocked variant for
// large N is k_lasyf_panel + k_trailing below.
// ---------------------------------------------------------------------------------------------------------
constexpr int BK_THREADS = 1024;
__global__ void __launch_bounds__(BK_THREADS)
k_sytf2(double* __restrict__ A, int lda, int N, int* __restrict__ ipiv, int* __restrict__ info)
{
  __shared__ ArgMax sm[32];
  const int tid = threadIdx.x;
  const int big = 0x7fffffff;
  int k = 0;
  int linfo = 0;
  while(k < N) {
    int kstep = 1, kp = k;
    const double absakk = fabs(LC(A, lda, k, k));
    int imax = k;
    double colmax = 0.0;
    if(k < N - 1) {
      ArgMax a{-1.0, big};
      for(int i = k + 1 + tid; i < N; i += BK_THREADS) a = argmax_comb(a, ArgMax{fabs(LC(A, lda, i, k)), i});
      a = cta_argmax(a, sm);
      imax = a.i;
      colmax = a.v;
    }
    if(fmax(absakk, colmax) == 0.0 || absakk != absakk) {
      if(linfo == 0) linfo = k + 1;
      kp = k;
    } else {
      if(absakk >= BK_ALPHA * colmax) {
        kp = k;
      } else {
        ArgMax a{-1.0, big};
        for(int j = k + tid; j < imax; j += BK_THREADS) a = argmax_comb(a, ArgMax{fabs(LC(A, lda, imax, j)), j});
        for(int i = imax + 1 + tid; i < N; i += BK_THREADS) a = argmax_comb(a, ArgMax{fabs(LC(A, lda, i, imax)), i});
        a = cta_argmax(a, sm);
        const double rowmax = a.v;
        if(absakk >= BK_ALPHA * colmax * (colmax / rowmax)) kp = k;
        else if(fabs(LC(A, lda, imax, imax)) >= BK_ALPHA * rowmax) kp = imax;
        else { kp = imax; kstep = 2; }
      }
      const int kk = k + kstep - 1;
      __syncthreads();
      if(kp != kk) {
        for(int i = kp + 1 + tid; i < N; i += BK_THREADS) {
          const double t = LC(A, lda, i, kk);
          LC(A, lda, i, kk) = LC(A, lda, i, kp);
          LC(A, lda, i, kp) = t;
        }
        for(int i = kk + 1 + tid; i < kp; i += BK_THREADS) {
          const double t = LC(A, lda, i, kk);
          LC(A, lda, i, kk) = LC(A, lda, kp, i);
          LC(A, lda, kp, i) = t;
        }
        if(tid == 0) {
          double t = LC(A, lda, kk, kk);
          LC(A, lda, kk, kk) = LC(A, lda, kp, kp);
          LC(A, lda, kp, kp) = t;
          if(kstep == 2) {
            t = LC(A, lda, k + 1, k);
            LC(A, lda, k + 1, k) = LC(A, lda, kp, k);
            LC(A, lda, kp, k) = t;
          }
        }
        __syncthreads();
      }
      if(kstep == 1) {
        if(k < N - 1) {
          const double d11 = 1.0 / LC(A, lda, k, k);
          const int rem = N - k - 1;
          // A(i,j) -= d11 * x_i * x_j, k < j <= i
          for(long long e = tid; e < (long long)rem * rem; e += BK_THREADS) {
            const int j = k + 1 + (int)(e / rem), i = k + 1 + (int)(e % rem);
            if(i >= j) LC(A, lda, i, j) -= d11 * LC(A, lda, i, k) * LC(A, lda, j, k);
          }
          __syncthreads();
          for(int i = k + 1 + tid; i < N; i += BK_THREADS) LC(A, lda, i, k) *= d11;
          __syncthreads();
        }
      } else {
        if(k < N - 2) {
          double d21 = LC(A, lda, k + 1, k);
          const double d11 = LC(A, lda, k + 1, k + 1) / d21;
          const double d22 = LC(A, lda, k, k) / d21;
          const double t = 1.0 / (d11 * d22 - 1.0);
          d21 = t / d21;
          const int rem = N - k - 2;
          for(long long e = tid; e < (long long)rem * rem; e += BK_THREADS) {
            const int j = k + 2 + (int)(e / rem), i = k + 2 + (int)(e % rem);
            if(i >= j) {
              const double wk = d21 * (d11 * LC(A, lda, j, k) - LC(A, lda, j, k + 1));
              const double wkp1 = d21 * (d22 * LC(A, lda, j, k + 1) - LC(A, lda, j, k));
              LC(A, lda, i, j) = LC(A, lda, i, j) - LC(A, lda, i, k) * wk - LC(A, lda, i, k + 1) * wkp1;
            }
          }
          __syncthreads();
          for(int j = k + 2 + tid; j < N; j += BK_THREADS) {
            const double ajk = LC(A, lda, j, k), ajk1 = LC(A, lda, j, k + 1);
            LC(A, lda, j, k) = d21 * (d11 * ajk - ajk1);
            LC(A, lda, j, k + 1) = d21 * (d22 * ajk1 - ajk);
          }
          __syncthreads();
        }
      }
    }
    if(tid == 0) {
      if(kstep == 1) ipiv[k] = kp + 1;
      else { ipiv[k] = -(kp + 1); ipiv[k + 1] = -(kp + 1); }
    }
    k += kstep;
    __syncthreads();
  }
  if(tid == 0) *info = linfo;
}

// ---------------------------------------------------------------------------------------------------------
// Blocked Bunch-Kaufman (DSYTRF 'L' structure: DLASYF panels + rank-kb trailing updates). The panel (<= 64 columns) is factorized by
// ONE CTA with LAPACK's pivot rule (same pivots as DSYTF2), keeping W = L*D of the panel in a scratch buffer; the trailing matrix is
// then updated A22 -= L21 * W21^T by k_trailing<true>. No host synchronisation inside the loop: the number of columns a panel managed
// to factorize (63 or 64, a 2x2 pivot may not straddle the panel edge) lives in a device-side state word that the next kernels read.
// ---------------------------------------------------------------------------------------------------------
#define WC(W, ldw, i, c) (W)[(size_t)(c) * (ldw) + (i)]

// state[0] = k0 of the current panel, state[1] = kb factorized by the last panel, state[2] = info (first zero pivot, 1-based)
__global__ void __launch_bounds__(BK_THREADS)
k_lasyf_panel(double* __restrict__ A, int lda, int N, double* __restrict__ W, int ldw, int* __restrict__ ipiv, int* __restrict__ state)
{
  __shared__ ArgMax sm[32];
  __shared__ double wrow[NB];
  const int tid = threadIdx.x;
  const int big = 0x7fffffff;
  const int k0 = state[0];
  if(k0 >= N) {
    if(tid == 0) state[1] = 0;
    return;
  }
  const int ns = N - k0;
  const bool last = ns <= NB;
  int linfo = 0;
  int k = k0;
  while(true) {
    const int kl = k - k0;
    if(k >= N) break;
    if(!last && kl >= NB - 1) break;
    // --- W(k:N,kl) = A(k:N,k) - A(k:N,k0:k-1) * W(k,0:kl-1)^T
    __syncthreads();
    for(int c = tid; c < kl; c += BK_THREADS) wrow[c] = WC(W, ldw, k, c);
    __syncthreads();
    for(int i = k + tid; i < N; i += BK_THREADS) {
      double v = LC(A, lda, i, k), v1 = 0.0, v2 = 0.0, v3 = 0.0;
      int c = 0;
#pragma unroll 2
      for(; c + 4 <= kl; c += 4) { // four independent accumulators: the loads of a batch are in flight together
        v -= LC(A, lda, i, k0 + c) * wrow[c];
        v1 -= LC(A, lda, i, k0 + c + 1) * wrow[c + 1];
        v2 -= LC(A, lda, i, k0 + c + 2) * wrow[c + 2];
        v3 -= LC(A, lda, i, k0 + c + 3) * wrow[c + 3];
      }
      for(; c < kl; c++) v -= LC(A, lda, i, k0 + c) * wrow[c];
      WC(W, ldw, i, kl) = (v + v1) + (v2 + v3);
    }
    __syncthreads();
    int kstep = 1, kp = k;
    const double absakk = fabs(WC(W, ldw, k, kl));
    int imax = k;
    double colmax = 0.0;
    if(k < N - 1) {
      ArgMax a{-1.0, big};
      for(int i = k + 1 + tid; i < N; i += BK_THREADS) a = argmax_comb(a, ArgMax{fabs(WC(W, ldw, i, kl)), i});
      a = cta_argmax(a, sm);
      imax = a.i;
      colmax = a.v;
    }
    if(fmax(absakk, colmax) == 0.0 || absakk != absakk) {
      if(linfo == 0) linfo = k + 1;
      kp = k;
    } else {
      if(absakk >= BK_ALPHA * colmax) {
        kp = k;
      } else {
        // column imax (updated) into W(:,kl+1)
        __syncthreads();
        for(int c = tid; c < kl; c += BK_THREADS) wrow[c] = WC(W, ldw, imax, c);
        __syncthreads();
        for(int i = k + tid; i < N; i += BK_THREADS) {
          double v = i < imax ? LC(A, lda, imax, i) : LC(A, lda, i, imax), v1 = 0.0, v2 = 0.0, v3 = 0.0;
          int c = 0;
#pragma unroll 2
          for(; c + 4 <= kl; c += 4) {
            v -= LC(A, lda, i, k0 + c) * wrow[c];
            v1 -= LC(A, lda, i, k0 + c + 1) * wrow[c + 1];
            v2 -= LC(A, lda, i, k0 + c + 2) * wrow[c + 2];
            v3 -= LC(A, lda, i, k0 + c + 3) * wrow[c + 3];
          }
          for(; c < kl; c++) v -= LC(A, lda, i, k0 + c) * wrow[c];
          WC(W, ldw, i, kl + 1) = (v + v1) + (v2 + v3);
        }
        __syncthreads();
        ArgMax a{-1.0, big};
        for(int i = k + tid; i < N; i += BK_THREADS)
          if(i != imax) a = argmax_comb(a, ArgMax{fabs(WC(W, ldw, i, kl + 1)), i});
        a = cta_argmax(a, sm);
        const double rowmax = a.v;
        if(absakk >= BK_ALPHA * colmax * (colmax / rowmax)) {
          kp = k;
        } else if(fabs(WC(W, ldw, imax, kl + 1)) >= BK_ALPHA * rowmax) {
          kp = imax;
          __syncthreads();
          for(int i = k + tid; i < N; i += BK_THREADS) WC(W, ldw, i, kl) = WC(W, ldw, i, kl + 1);
          __syncthreads();
        } else {
          kp = imax;
          kstep = 2;
        }
      }
      const int kk = k + kstep - 1, kkl = kk - k0;
      __syncthreads();
      if(kp != kk) {
        // copy the non-updated column kk into position kp of the trailing submatrix
        if(tid == 0) LC(A, lda, kp, kp) = LC(A, lda, kk, kk);
        for(int i = kk + 1 + tid; i < kp; i += BK_THREADS) LC(A, lda, kp, i) = LC(A, lda, i, kk);
        for(int i = kp + 1 + tid; i < N; i += BK_THREADS) LC(A, lda, i, kp) = LC(A, lda, i, kk);
        // swap rows kk and kp in the panel's finished columns of A and in W(.,0:kkl)
        for(int c = tid; c < kl; c += BK_THREADS) {
          const double t = LC(A, lda, kk, k0 + c);
          LC(A, lda, kk, k0 + c) = LC(A, lda, kp, k0 + c);
          LC(A, lda, kp, k0 + c) = t;
        }
        for(int c = tid; c <= kkl; c += BK_THREADS) {
          const double t = WC(W, ldw, kk, c);
          WC(W, ldw, kk, c) = WC(W, ldw, kp, c);
          WC(W, ldw, kp, c) = t;
        }
        __syncthreads();
      }
      if(kstep == 1) {
        const double akk = WC(W, ldw, k, kl);
        const double r1 = 1.0 / akk;
        for(int i = k + tid; i < N; i += BK_THREADS) {
          const double w = WC(W, ldw, i, kl);
          LC(A, lda, i, k) = (i == k) ? w : w * r1;
        }
      } else {
        if(k < N - 2) {
          double d21 = WC(W, ldw, k + 1, kl);
          const double d11 = WC(W, ldw, k + 1, kl + 1) / d21;
          const double d22 = WC(W, ldw, k, kl) / d21;
          const double t = 1.0 / (d11 * d22 - 1.0);
          d21 = t / d21;
          for(int j = k + 2 + tid; j < N; j += BK_THREADS) {
            const double wj0 = WC(W, ldw, j, kl), wj1 = WC(W, ldw, j, kl + 1);
            LC(A, lda, j, k) = d21 * (d11 * wj0 - wj1);
            LC(A, lda, j, k + 1) = d21 * (d22 * wj1 - wj0);
          }
        }
        if(tid == 0) {
          LC(A, lda, k, k) = WC(W, ldw, k, kl);
          LC(A, lda, k + 1, k) = WC(W, ldw, k + 1, kl);
          LC(A, lda, k + 1, k + 1) = WC(W, ldw, k + 1, kl + 1);
        }
      }
    }
    if(tid == 0) {
      if(kstep == 1) ipiv[k] = kp + 1;
      else { ipiv[k] = -(kp + 1); ipiv[k + 1] = -(kp + 1); }
    }
    k += kstep;
    __syncthreads();
  }
  if(tid == 0) {
    state[1] = k - k0;
    if(linfo != 0 && state[2] == 0) state[2] = linfo;
  }
}

// Puts L21 of the finished panel in LAPACK's standard form (partial undo of the row interchanges, DLASYF label 120)
// and advances the state to the next panel.
__global__ void k_lasyf_finish(double* __restrict__ A, int lda, int N, const int* __restrict__ ipiv, int* __restrict__ state)
{
  const int k0 = state[0], kb = state[1];
  if(kb == 0) return;
  const int kend = k0 + kb;
  int j = kend - 1;
  while(j >= k0) {
    const int jj = j;
    int jp = ipiv[j];
    if(jp < 0) { jp = -jp; j -= 1; }
    jp -= 1;
    j -= 1;
    const int ncols = j - k0 + 1;
    if(jp != jj && ncols >= 1) {
      for(int c = threadIdx.x; c < ncols; c += blockDim.x) {
        const double t = LC(A, lda, jp, k0 + c);
        LC(A, lda, jp, k0 + c) = LC(A, lda, jj, k0 + c);
        LC(A, lda, jj, k0 + c) = t;
      }
    }
    __syncthreads();
    if(j <= k0) break;
  }
  __syncthreads();
  if(threadIdx.x == 0) state[0] = kend;
}

// DSYTRS 'L': one thread per right-hand side (rhs r = B + r*ldb, contiguous N doubles). Used for V^{-1}[S1^T;Y1^T]
// (many rhs, tiny N) and for single-rhs solves with small N.
__global__ void k_sytrs_per_rhs(const double* __restrict__ A, int lda, int N, const int* __restrict__ ipiv, double* __restrict__ B, int ldb,
                                int nrhs)
{
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if(r >= nrhs) return;
  double* b = B + (size_t)r * ldb;
  int k = 0;
  while(k < N) {
    if(ipiv[k] > 0) {
      const int kp = ipiv[k] - 1;
      if(kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
      const double bk = b[k];
      for(int i = k + 1; i < N; i++) b[i] -= LC(A, lda, i, k) * bk;
      b[k] = bk / LC(A, lda, k, k);
      k += 1;
    } else {
      const int kp = -ipiv[k] - 1;
      if(kp != k + 1) { const double t = b[k + 1]; b[k + 1] = b[kp]; b[kp] = t; }
      const double bk0 = b[k], bk1 = b[k + 1];
      for(int i = k + 2; i < N; i++) b[i] -= LC(A, lda, i, k) * bk0 + LC(A, lda, i, k + 1) * bk1;
      const double akm1k = LC(A, lda, k + 1, k);
      const double akm1 = LC(A, lda, k, k) / akm1k;
      const double ak = LC(A, lda, k + 1, k + 1) / akm1k;
      const double denom = akm1 * ak - 1.0;
      const double bkm1 = bk0 / akm1k, bkk = bk1 / akm1k;
      b[k] = (ak * bkm1 - bkk) / denom;
      b[k + 1] = (akm1 * bkk - bkm1) / denom;
      k += 2;
    }
  }
  k = N - 1;
  while(k >= 0) {
    if(ipiv[k] > 0) {
      double s = b[k];
      for(int i = k + 1; i < N; i++) s -= LC(A, lda, i, k) * b[i];
      b[k] = s;
      const int kp = ipiv[k] - 1;
      if(kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
      k -= 1;
    } else {
      double s0 = b[k], s1 = b[k - 1];
      for(int i = k + 1; i < N; i++) {
        s0 -= LC(A, lda, i, k) * b[i];
        s1 -= LC(A, lda, i, k - 1) * b[i];
      }
      b[k] = s0;
      b[k - 1] = s1;
      const int kp = -ipiv[k] - 1;
      if(kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
      k -= 2;
    }
  }
}

// DSYTRS 'L' for ONE right-hand side with the whole CTA cooperating on each column sweep (large N).
__global__ void __launch_bounds__(SOLVE_THREADS)
k_sytrs_cta(const double* __restrict__ A, int lda, int N, const int* __restrict__ ipiv, double* __restrict__ b)
{
  __shared__ double sm[64];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int k = 0;
  while(k < N) {
    const int pv = ipiv[k];
    if(pv > 0) {
      const int kp = pv - 1;
      if(tid == 0 && kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
      __syncthreads();
      const double bk = b[k];
      for(int i = k + 1 + tid; i < N; i += SOLVE_THREADS) b[i] -= LC(A, lda, i, k) * bk;
      __syncthreads();
      if(tid == 0) b[k] = bk / LC(A, lda, k, k);
      k += 1;
    } else {
      const int kp = -pv - 1;
      if(tid == 0 && kp != k + 1) { const double t = b[k + 1]; b[k + 1] = b[kp]; b[kp] = t; }
      __syncthreads();
      const double bk0 = b[k], bk1 = b[k + 1];
      for(int i = k + 2 + tid; i < N; i += SOLVE_THREADS) b[i] -= LC(A, lda, i, k) * bk0 + LC(A, lda, i, k + 1) * bk1;
      __syncthreads();
      if(tid == 0) {
        const double akm1k = LC(A, lda, k + 1, k);
        const double akm1 = LC(A, lda, k, k) / akm1k;
        const double ak = LC(A, lda, k + 1, k + 1) / akm1k;
        const double denom = akm1 * ak - 1.0;
        const double bkm1 = bk0 / akm1k, bkk = bk1 / akm1k;
        b[k] = (ak * bkm1 - bkk) / denom;
        b[k + 1] = (akm1 * bkk - bkm1) / denom;
      }
      k += 2;
    }
    __syncthreads();
  }
  k = N - 1;
  while(k >= 0) {
    const int pv = ipiv[k];
    const int ncol = pv > 0 ? 1 : 2;
    double s0 = 0.0, s1 = 0.0;
    for(int i = k + 1 + tid; i < N; i += SOLVE_THREADS) {
      const double bi = b[i];
      s0 += LC(A, lda, i, k) * bi;
      if(ncol == 2) s1 += LC(A, lda, i, k - 1) * bi;
    }
    s0 = hb_warp_sum(s0);
    s1 = hb_warp_sum(s1);
    __syncthreads();
    if(lane == 0) { sm[warp] = s0; sm[32 + warp] = s1; }
    __syncthreads();
    if(tid == 0) {
      double t0 = 0.0, t1 = 0.0;
      for(int w = 0; w < SOLVE_THREADS / 32; w++) { t0 += sm[w]; t1 += sm[32 + w]; }
      b[k] -= t0;
      if(ncol == 2) b[k - 1] -= t1;
      const int kp = (pv > 0 ? pv : -pv) - 1;
      if(kp != k) { const double t = b[k]; b[k] = b[kp]; b[kp] = t; }
    }
    __syncthreads();
    k -= ncol;
  }
}

// Inertia sweep: BK factor -> LINPACK dsidi rule; no-pivot LDL^T / Cholesky -> signs of the diagonal.
// out = {neg, null, pos}
__global__ void __launch_bounds__(1024)
k_inertia(const double* __restrict__ A, int lda, int N, const int* __restrict__ ipiv, int mode, int* __restrict__ out, double* __restrict__ scratch)
{
  // scratch: 2N doubles (diagonal, sub-diagonal), gathered by all threads (strided loads in parallel)
  double* dg = scratch;
  double* sub = scratch + N;
  for(int k = threadIdx.x; k < N; k += blockDim.x) {
    dg[k] = LC(A, lda, k, k);
    sub[k] = (k + 1 < N) ? LC(A, lda, k + 1, k) : 0.0;
  }
  __syncthreads();
  if(threadIdx.x != 0) return;
  int neg = 0, nul = 0, pos = 0;
  double t = 0.0;
  for(int k = 0; k < N; k++) {
    double d = dg[k];
    if(mode == HB_FACT_BUNCH_KAUFMAN && ipiv[k] <= 0) {
      if(t == 0.0) {
        if(k + 1 < N) {
          t = fabs(sub[k]);
          d = (d / t) * dg[k + 1] - t;
        }
      } else {
        d = t;
        t = 0.0;
      }
    }
    if(d < -1e-14) neg++;
    else if(d < 1e-14) nul++;
    else pos++;
  }
  out[0] = neg; out[1] = nul; out[2] = pos;
}

// LDL^T (no pivoting) single-rhs solve: forward (unit L), D, backward.
__global__ void __launch_bounds__(SOLVE_THREADS)
k_ldl_solve(const double* __restrict__ F, int ldf, int N, double* __restrict__ x)
{
  __shared__ double sm[32];
  __shared__ double sd[32][33];
  dev_forward(F, ldf, N, x, true, sd);
  for(int i = threadIdx.x; i < N; i += SOLVE_THREADS) x[i] /= LC(F, ldf, i, i);
  __syncthreads();
  dev_backward(F, ldf, N, x, true, sm, sd);
}
__global__ void __launch_bounds__(SOLVE_THREADS)
k_chol_solve(const double* __restrict__ F, int ldf, int N, double* __restrict__ x)
{
  __shared__ double sm[32];
  __shared__ double sd[32][33];
  dev_forward(F, ldf, N, x, false, sd);
  dev_backward(F, ldf, N, x, false, sm, sd);
}

} // namespace

// ---------------------------------------------------------------------------------------------------------
// internal API (hb_dense.cuh): each entry point runs one path; hb_symdense.cu decides which
// ---------------------------------------------------------------------------------------------------------
constexpr size_t TRAILING_SMEM = sizeof(double) * 2 * NB * TLD;

int hb_dense_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_trailing<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TRAILING_SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_trailing<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TRAILING_SMEM));
  return HB_OK;
}

int hb_dense_factor_panel(hb_ctx* c, int N, double* A, int lda, bool ldl, double* Wpanel /* NB*N doubles if ldl */, int* info_dev)
{
  HB_CUDA(cudaMemsetAsync(info_dev, 0, sizeof(int), c->stream));
  for(int k0 = 0; k0 < N; k0 += NB) {
    const int nb = N - k0 < NB ? N - k0 : NB;
    const int rest = N - k0 - nb;
    int blocks = (rest + PANEL_THREADS - 1) / PANEL_THREADS;
    if(blocks < 1) blocks = 1;
    if(ldl) k_panel<true><<<blocks, PANEL_THREADS, 0, c->stream>>>(A, lda, N, k0, nb, Wpanel, N, info_dev);
    else k_panel<false><<<blocks, PANEL_THREADS, 0, c->stream>>>(A, lda, N, k0, nb, nullptr, 0, info_dev);
    HB_LAUNCHED();
    if(rest > 0) {
      const int nt = (rest + TT - 1) / TT;
      const int ntiles = nt * (nt + 1) / 2;
      const double* Q = A + (size_t)k0 * lda; // factor panel rows: Q[p][i] = Lc(i, k0+p)
      const double* P = ldl ? Wpanel : Q;
      k_trailing<false><<<ntiles, 128, TRAILING_SMEM, c->stream>>>(A, lda, N, k0 + nb, P, ldl ? (long long)N : (long long)lda, Q, lda, nb,
                                                                     nullptr);
      HB_LAUNCHED();
    }
  }
  return HB_OK;
}

int hb_dense_sytf2(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, int* info_dev)
{
  if(N == 0) return HB_OK;
  k_sytf2<<<1, BK_THREADS, 0, c->stream>>>(A, lda, N, ipiv_dev, info_dev);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_sytrf_blocked(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, double* Wpanel, int* info_dev)
{
  if(N == 0) return HB_OK;
  // device state word (k0, kb, info) in the workspace
  HB_CHECK(hb_ws_reserve(c, 64));
  int* state = reinterpret_cast<int*>(c->ws.get());
  HB_CUDA(cudaMemsetAsync(state, 0, sizeof(int) * 4, c->stream));
  const int max_panels = (N + (NB - 1) - 1) / (NB - 1) + 1;
  for(int p = 0; p < max_panels; p++) {
    const int k0_min = p * (NB - 1); // a panel advances by at least NB-1 columns
    if(k0_min >= N) break;
    k_lasyf_panel<<<1, BK_THREADS, 0, c->stream>>>(A, lda, N, Wpanel, N, ipiv_dev, state);
    HB_LAUNCHED();
    const int rest_max = N - k0_min - (NB - 1);
    if(rest_max > 0) {
      const int nt = (rest_max + TT - 1) / TT;
      k_trailing<true><<<nt * (nt + 1) / 2, 128, TRAILING_SMEM, c->stream>>>(A, lda, N, 0, nullptr, 0, Wpanel, N, 0, state);
      HB_LAUNCHED();
    }
    k_lasyf_finish<<<1, 64, 0, c->stream>>>(A, lda, N, ipiv_dev, state);
    HB_LAUNCHED();
  }
  HB_CUDA(cudaMemcpyAsync(info_dev, state + 2, sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
  return HB_OK;
}

int hb_dense_sytrs(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs, bool cta_per_rhs)
{
  if(N == 0 || nrhs == 0) return HB_OK;
  if(!cta_per_rhs) {
    k_sytrs_per_rhs<<<(nrhs + 63) / 64, 64, 0, c->stream>>>(A, lda, N, ipiv_dev, B, ldb, nrhs);
    HB_LAUNCHED();
  } else {
    for(int r = 0; r < nrhs; r++) {
      k_sytrs_cta<<<1, SOLVE_THREADS, 0, c->stream>>>(A, lda, N, ipiv_dev, B + (size_t)r * ldb);
      HB_LAUNCHED();
    }
  }
  return HB_OK;
}

int hb_dense_inertia_ipiv(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, int* out3_dev)
{
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * 2 * (size_t)(N > 0 ? N : 1) + 256));
  k_inertia<<<1, 1024, 0, c->stream>>>(A, lda, N, ipiv_dev, HB_FACT_BUNCH_KAUFMAN, out3_dev,
                                       reinterpret_cast<double*>(reinterpret_cast<char*>(c->ws.get()) + 256));
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_tri_solve(hb_ctx* c, int N, const double* F, int ldf, bool ldl, double* x)
{
  if(N == 0) return HB_OK;
  if(ldl) k_ldl_solve<<<1, SOLVE_THREADS, 0, c->stream>>>(F, ldf, N, x);
  else k_chol_solve<<<1, SOLVE_THREADS, 0, c->stream>>>(F, ldf, N, x);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_equilibrate(hb_ctx* c, int N, const double* Nfull, int ldn, double* F, int ldf, double* s)
{
  if(N == 0) return HB_OK;
  k_equilibrate<<<hb_grid(c, (long long)N * N), 256, 0, c->stream>>>(Nfull, ldn, N, F, ldf, s);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_spd_solve_refine(hb_ctx* c, int N, const double* F, int ldf, const double* s, const double* Nref, int ldn, const double* rhs,
                              double* x, double* work2N, double tol, int max_refine, double* stats_dev)
{
  if(N == 0) return HB_OK;
  k_spd_solve_refine<<<1, SOLVE_THREADS, 0, c->stream>>>(F, ldf, N, s, Nref, ldn, rhs, x, work2N, tol, max_refine, stats_dev);
  HB_LAUNCHED();
  return HB_OK;
}
