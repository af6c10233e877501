// hiopKKTLinSysLowRank + hiopHessianLowRank on device (the quasi-Newton KKT path).
// Reference: src/Optimization/hiopKKTLinSys.cpp:1031-1350, src/Optimization/hiopHessianLowRank.cpp:221-630, 974-1059,
// hiopKKTLinSysCompressedXYcYd::computeDirections hiopKKTLinSys.cpp:585-691, compute_directions_for_full_space :218-309.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include "hb_lowrank.cuh"
#include <cstdlib>

namespace {

constexpr int ET = 256; // elementwise / streaming kernels

// ---- a1: Dx, DhInv in one pass (hiopKKTLinSys.cpp:1073-1078 + hiopHessianLowRank.cpp:223-229; 7 passes there) ----------
// Same operation order as the reference so the result is bit-identical: Dx = 0 + zl/sxl (+ zu/sxu); DhInv = 1/(sigma + Dx).
__global__ void __launch_bounds__(ET)
k_update_x(long long n, const double* __restrict__ zl, const double* __restrict__ sxl, const double* __restrict__ zu,
           const double* __restrict__ sxu, const double* __restrict__ ixl, const double* __restrict__ ixu, double sigma,
           double* __restrict__ Dx, double* __restrict__ DhInv)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    double d = 0.0;
    if(ixl[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(zl[i], sxl[i]));
    if(ixu[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(zu[i], sxu[i]));
    Dx[i] = d;
    if(DhInv) DhInv[i] = __ddiv_rn(1.0, __dadd_rn(sigma, d));
  }
}
// d-side: Dd = vl/sdl|idl + vu/sdu|idu, Dd_inv = 1/Dd (hiopKKTLinSys.cpp:1081-1088)
__global__ void k_update_d(int mi, const double* __restrict__ vl, const double* __restrict__ sdl, const double* __restrict__ vu,
                           const double* __restrict__ sdu, const double* __restrict__ idl, const double* __restrict__ idu,
                           double* __restrict__ Dd, double* __restrict__ Dd_inv)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < mi; i += gridDim.x * blockDim.x) {
    double d = 0.0;
    if(idl[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vl[i], sdl[i]));
    if(idu[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vu[i], sdu[i]));
    Dd[i] = d;
    Dd_inv[i] = __ddiv_rn(1.0, d);
  }
}

// ---- a8: V from the blocks of C_aug = [J;S;Y] DhInv [J;S;Y]^T (updateInternalBFGSRepresentation, :400-485) ----------------
// V, M and U are written with explicit roundings (no FMA contraction), so each entry is a fixed function of its inputs that
// oracle/lowrank_model.py restates bit for bit.
__global__ void k_build_V(int m, int l, double sigma, const double* __restrict__ C, int ldc, const double* __restrict__ SSt,
                          const double* __restrict__ L, const double* __restrict__ D, double* __restrict__ V)
{
  const int n2 = 2 * l;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < n2 * n2; e += gridDim.x * blockDim.x) {
    const int a = e / n2, b = e % n2;
    double v;
    if(a < l && b < l) v = __dsub_rn(__dmul_rn(__dmul_rn(sigma, sigma), C[(size_t)(m + a) * ldc + m + b]), __dmul_rn(sigma, SSt[a * l + b]));
    else if(a < l && b >= l) v = __dsub_rn(__dmul_rn(sigma, C[(size_t)(m + a) * ldc + m + b]), L[a * l + (b - l)]);
    else if(a >= l && b < l) v = __dsub_rn(__dmul_rn(sigma, C[(size_t)(m + b) * ldc + m + a]), L[b * l + (a - l)]);
    else v = __dadd_rn(C[(size_t)(m + a) * ldc + m + b], a == b ? D[a - l] : 0.0);
    V[a * n2 + b] = v;
  }
}
// M = [[sigma S^T S, L],[L^T, -D]] of the compact (direct) BFGS representation, used by hess_times_vec
__global__ void k_build_Mdirect(int l, double sigma, const double* __restrict__ SSt, const double* __restrict__ L,
                                const double* __restrict__ D, double* __restrict__ Mm)
{
  const int n2 = 2 * l;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < n2 * n2; e += gridDim.x * blockDim.x) {
    const int a = e / n2, b = e % n2;
    double v;
    if(a < l && b < l) v = __dmul_rn(sigma, SSt[a * l + b]);
    else if(a < l && b >= l) v = L[a * l + (b - l)];
    else if(a >= l && b < l) v = L[b * l + (a - l)];
    else v = (a == b ? -D[a - l] : 0.0);
    Mm[a * n2 + b] = v;
  }
}
// U = [S1 Y1] (m x 2l): S1 = sigma * C[0:m, m:m+l], Y1 = C[0:m, m+l:m+2l]; Z = copy of U (rhs of the V solve)
__global__ void k_build_U(int m, int l, double sigma, const double* __restrict__ C, int ldc, double* __restrict__ U, double* __restrict__ Z)
{
  const int n2 = 2 * l;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < m * n2; e += gridDim.x * blockDim.x) {
    const int i = e / n2, q = e % n2;
    double v = C[(size_t)i * ldc + m + q];
    if(q < l) v = __dmul_rn(sigma, v);
    U[e] = v;
    Z[e] = v;
  }
}
// N = W0 - U Z^T + blkdiag(0, Dd_inv) (hiopHessianLowRank.cpp:608-618 + hiopKKTLinSys.cpp:1135); computed for i <= j, mirrored.
__global__ void k_form_N(int m, int meq, int l, const double* __restrict__ C, int ldc, const double* __restrict__ U, const double* __restrict__ Z,
                         const double* __restrict__ Dd_inv, double* __restrict__ Nm)
{
  const int n2 = 2 * l;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < (long long)m * m; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / m), j = (int)(e % m);
    if(j < i) continue;
    double v = C[(size_t)i * ldc + j];
    double corr = 0.0;
    for(int q = 0; q < n2; q++) corr += U[(size_t)i * n2 + q] * Z[(size_t)j * n2 + q];
    v -= corr;
    if(i == j && i >= meq) v += Dd_inv[i - meq];
    Nm[(size_t)i * m + j] = v;
    Nm[(size_t)j * m + i] = v;
  }
}

// ---- all-reduce of the symmetric C_aug as its packed upper triangle (hiopHessianLowRank.cpp:590-591 sends the full m x m buffer) ----
__global__ void k_pack_upper(int M, const double* __restrict__ C, int ldc, double* __restrict__ tri)
{
  const long long tot = (long long)M * (M + 1) / 2;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    // row i of the upper triangle starts at i*M - i(i-1)/2
    int i = (int)((2.0 * M + 1.0 - sqrt((2.0 * M + 1.0) * (2.0 * M + 1.0) - 8.0 * (double)e)) * 0.5);
    while((long long)i * M - (long long)i * (i - 1) / 2 > e) i--;
    while((long long)(i + 1) * M - (long long)(i + 1) * i / 2 <= e) i++;
    const int j = i + (int)(e - ((long long)i * M - (long long)i * (i - 1) / 2));
    tri[e] = C[(size_t)i * ldc + j];
  }
}
__global__ void k_unpack_upper(int M, double* __restrict__ C, int ldc, const double* __restrict__ tri)
{
  const long long tot = (long long)M * (M + 1) / 2;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    int i = (int)((2.0 * M + 1.0 - sqrt((2.0 * M + 1.0) * (2.0 * M + 1.0) - 8.0 * (double)e)) * 0.5);
    while((long long)i * M - (long long)i * (i - 1) / 2 > e) i--;
    while((long long)(i + 1) * M - (long long)(i + 1) * i / 2 <= e) i++;
    const int j = i + (int)(e - ((long long)i * M - (long long)i * (i - 1) / 2));
    const double v = tri[e];
    C[(size_t)i * ldc + j] = v;
    C[(size_t)j * ldc + i] = v;
  }
}

// ---- multi-dot: out[q] = sum_k R_q[k] * w[k] * x[k] * scale_q, q < nq rows (two-stage, deterministic) ------------------------
// rows q < l come from S (scale sigma_s), rows q >= l from Y (scale 1). w may be null (=1).
constexpr int MD_CH = 8;
__global__ void __launch_bounds__(ET)
k_multidot_partial(long long n, int l, const double* __restrict__ S, const double* __restrict__ Y, long long ld, const double* __restrict__ w,
                   const double* __restrict__ x, int q0, double* __restrict__ partial /* [grid][2l] */)
{
  __shared__ double sm[ET / 32];
  const int n2 = 2 * l;
  double acc[MD_CH];
#pragma unroll
  for(int c = 0; c < MD_CH; c++) acc[c] = 0.0;
  const long long stride = (long long)gridDim.x * ET;
  for(long long k = (long long)blockIdx.x * ET + threadIdx.x; k < n; k += stride) {
    const double t = w ? w[k] * x[k] : x[k];
#pragma unroll
    for(int c = 0; c < MD_CH; c++) {
      const int q = q0 + c;
      if(q < n2) {
        const double* row = q < l ? S + (size_t)q * ld : Y + (size_t)(q - l) * ld;
        acc[c] += row[k] * t;
      }
    }
  }
#pragma unroll
  for(int c = 0; c < MD_CH; c++) {
    const double r = hb_block_sum<ET>(acc[c], sm);
    if(threadIdx.x == 0 && q0 + c < n2) partial[(size_t)blockIdx.x * n2 + q0 + c] = r;
  }
}
// one CTA per output: 128 threads stride over the per-CTA partials, fixed-order block reduction (a single thread walking
// all ~1200 partials is a long serial chain)
__global__ void __launch_bounds__(128)
k_multidot_final(int np, int l, double sigma_s, const double* __restrict__ partial, double* __restrict__ out)
{
  __shared__ double sm[4];
  const int n2 = 2 * l;
  const int q = blockIdx.x;
  double s = 0.0;
  for(int p = threadIdx.x; p < np; p += 128) s += partial[(size_t)p * n2 + q];
  s = hb_block_sum<128>(s, sm);
  if(threadIdx.x == 0) out[q] = q < l ? s * sigma_s : s;
}
// x[k] = w[k] * (r[k] - sigma*sum_q S_q[k] p_q - sum_q Y_q[k] p_{l+q})   (hiopHessianLowRank::solve steps 4-5, :526-535)
// general form: out = beta*out + alpha*( base[k]*r[k] ... ) handled by flags below
__global__ void __launch_bounds__(ET)
k_lowrank_apply(long long n, int l, double sigma, const double* __restrict__ S, const double* __restrict__ Y, long long ld,
                const double* __restrict__ p /* 2l */, const double* __restrict__ w /* n or null */, const double* __restrict__ r,
                double diag_scale, const double* __restrict__ diag_add /* n or null */, double beta, double alpha, double* __restrict__ out)
{
  // t = (diag_scale + diag_add[k]) * r[k]  (when w == null)   or   t = r[k] (when w != null)
  // v = t - (sigma*S^T p_s + Y^T p_y)[k];   if w: v *= w[k];   out = beta*out + alpha*v
  extern __shared__ double sp[];
  for(int q = threadIdx.x; q < 2 * l; q += ET) sp[q] = p[q];
  __syncthreads();
  const long long stride = (long long)gridDim.x * ET;
  for(long long k = (long long)blockIdx.x * ET + threadIdx.x; k < n; k += stride) {
    double ss = 0.0, sy = 0.0;
    for(int q = 0; q < l; q++) {
      ss += S[(size_t)q * ld + k] * sp[q];
      sy += Y[(size_t)q * ld + k] * sp[l + q];
    }
    const double corr = sigma * ss + sy;
    double v;
    if(w) v = w[k] * (r[k] - corr);
    else v = (diag_scale + (diag_add ? diag_add[k] : 0.0)) * r[k] - corr;
    out[k] = (beta == 0.0 ? 0.0 : beta * out[k]) + alpha * v;
  }
}

// ---- a13: J*x (rows) and J^T*y (columns) -----------------------------------------------------------------------------------
constexpr int GR_THREADS = 512;
constexpr int GR_CHUNK = 2048; // columns per CTA
__global__ void __launch_bounds__(GR_THREADS)
k_gemv_rows_partial(int m, long long n, const double* __restrict__ A, long long lda, const double* __restrict__ x,
                    double* __restrict__ partial /* [nchunks][m] */)
{
  __shared__ double sx[GR_CHUNK];
  const long long k0 = (long long)blockIdx.x * GR_CHUNK;
  const int len = (int)min((long long)GR_CHUNK, n - k0);
  for(int k = threadIdx.x; k < GR_CHUNK; k += GR_THREADS) sx[k] = k < len ? x[k0 + k] : 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool vec = ((lda & 1) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15u) == 0) && ((k0 & 1) == 0);
  // blockIdx.y interleaves the rows among gridDim.y CTAs of the same column chunk (short local column ranges)
  for(int i = warp + (GR_THREADS / 32) * blockIdx.y; i < m; i += (GR_THREADS / 32) * gridDim.y) {
    const double* row = A + (size_t)i * lda + k0;
    double acc = 0.0;
    if(vec) {
      const double2* r2 = reinterpret_cast<const double2*>(row);
      const int len2 = len >> 1;
#pragma unroll 8
      for(int k = lane; k < len2; k += 32) {
        const double2 v = r2[k];
        acc += v.x * sx[2 * k] + v.y * sx[2 * k + 1];
      }
      if((len & 1) && lane == 0) acc += row[len - 1] * sx[len - 1];
    } else {
#pragma unroll 8
      for(int k = lane; k < len; k += 32) acc += row[k] * sx[k];
    }
    acc = hb_warp_sum(acc);
    if(lane == 0) partial[(size_t)blockIdx.x * m + i] = acc;
  }
}
// y[i] = beta*y[i] + alpha*sum_chunks partial[c][i]: 32 rows x 8 chunk-classes per CTA (coalesced along i), fixed-order combine
__global__ void __launch_bounds__(256)
k_gemv_rows_final(int m, int nchunks, const double* __restrict__ partial, double beta, double* __restrict__ y, double alpha)
{
  __shared__ double sm[8][33];
  const int ri = threadIdx.x & 31, part = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + ri;
  double s = 0.0;
  if(i < m)
    for(int c = part; c < nchunks; c += 8) s += partial[(size_t)c * m + i];
  sm[part][ri] = s;
  __syncthreads();
  if(part == 0 && i < m) {
    double t = 0.0;
#pragma unroll
    for(int p = 0; p < 8; p++) t += sm[p][ri];
    y[i] = (beta == 0.0 ? 0.0 : beta * y[i]) + alpha * t;
  }
}

// y[k] = beta*y[k] + alpha*sum_i A[i][k]*x[i]; each thread owns two adjacent columns. With RG > 1 the CTA covers ET/RG column
// pairs and its RG thread groups take interleaved rows (combined in a fixed order through shared memory): short local column
// ranges (a rank's shard of n) still fill the machine.
constexpr int GC_ROWS = 1024; // rows of x staged per pass
template <int RG>
__global__ void __launch_bounds__(ET)
k_gemv_cols(int m, long long n, const double* __restrict__ A, long long lda, const double* __restrict__ x, double beta,
            double* __restrict__ y, double alpha)
{
  constexpr int CP = ET / RG; // column pairs per CTA
  __shared__ double sx[GC_ROWS];
  __shared__ double2 red[RG > 1 ? ET : 1];
  const bool vec = ((lda & 1) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15u) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15u) == 0);
  const int cp = threadIdx.x % CP, rg = threadIdx.x / CP;
  const long long k = ((long long)blockIdx.x * CP + cp) * 2;
  double a0 = 0.0, a1 = 0.0;
  for(int i0 = 0; i0 < m; i0 += GC_ROWS) {
    const int nr = min(GC_ROWS, m - i0);
    __syncthreads();
    for(int i = threadIdx.x; i < nr; i += ET) sx[i] = x[i0 + i];
    __syncthreads();
    if(k < n) {
      const double* col = A + (size_t)i0 * lda + k;
      if(vec && k + 1 < n) {
#pragma unroll 8
        for(int i = rg; i < nr; i += RG) {
          const double2 v = *reinterpret_cast<const double2*>(col + (size_t)i * lda);
          a0 += v.x * sx[i];
          a1 += v.y * sx[i];
        }
      } else {
#pragma unroll 4
        for(int i = rg; i < nr; i += RG) {
          a0 += col[(size_t)i * lda] * sx[i];
          if(k + 1 < n) a1 += col[(size_t)i * lda + 1] * sx[i];
        }
      }
    }
  }
  if(RG > 1) {
    red[threadIdx.x] = make_double2(a0, a1);
    __syncthreads();
    if(rg != 0) return;
    a0 = 0.0, a1 = 0.0;
#pragma unroll
    for(int g = 0; g < RG; g++) {
      a0 += red[g * CP + cp].x;
      a1 += red[g * CP + cp].y;
    }
  }
  if(k < n) {
    y[k] = (beta == 0.0 ? 0.0 : beta * y[k]) + alpha * a0;
    if(k + 1 < n) y[k + 1] = (beta == 0.0 ? 0.0 : beta * y[k + 1]) + alpha * a1;
  }
}

// ---- a5: rhs reduction + back-substitution (computeDirections / compute_directions_for_full_space) ---------------------------
// Operation order follows the reference exactly (intrinsics forbid FMA contraction) so that rx_tilde etc. are bit-identical.
// out = r0 + (pl? (rsl - dl*rl)/sl) - (pu? (rsu - du*ru)/su)
__global__ void __launch_bounds__(ET)
k_reduce_rhs(long long n, const double* __restrict__ r0, const double* __restrict__ rsl, const double* __restrict__ dl, const double* __restrict__ rl,
             const double* __restrict__ sl, const double* __restrict__ pl, const double* __restrict__ rsu, const double* __restrict__ du,
             const double* __restrict__ ru, const double* __restrict__ su, const double* __restrict__ pu, double* __restrict__ out)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    double v = r0[i];
    if(pl[i] == 1.0) v = __dadd_rn(v, __ddiv_rn(__dsub_rn(rsl[i], __dmul_rn(dl[i], rl[i])), sl[i]));
    if(pu[i] == 1.0) v = __dsub_rn(v, __ddiv_rn(__dsub_rn(rsu[i], __dmul_rn(du[i], ru[i])), su[i]));
    out[i] = v;
  }
}
// ds_l = pl ? r_l + dvar : 0 ; dz_l = pl ? (rs_l - dual_l*ds_l)/s_l : 0 ; ds_u = pu ? r_u - dvar : 0 ; dz_u = pu ? (rs_u - dual_u*ds_u)/s_u : 0
__global__ void __launch_bounds__(ET)
k_recover_slack_duals(long long n, const double* __restrict__ dvar, const double* __restrict__ rl, const double* __restrict__ rsl,
                      const double* __restrict__ dual_l, const double* __restrict__ sl, const double* __restrict__ pl,
                      const double* __restrict__ ru, const double* __restrict__ rsu, const double* __restrict__ dual_u,
                      const double* __restrict__ su, const double* __restrict__ pu, double* __restrict__ dsl, double* __restrict__ dzl,
                      double* __restrict__ dsu, double* __restrict__ dzu)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double dv = dvar[i];
    double a = 0.0, b = 0.0, c = 0.0, d = 0.0;
    if(pl[i] != 0.0) {
      a = __dadd_rn(rl[i], dv);
      b = __ddiv_rn(__dsub_rn(rsl[i], __dmul_rn(dual_l[i], a)), sl[i]);
    }
    if(pu[i] != 0.0) {
      c = __dsub_rn(ru[i], dv);
      d = __ddiv_rn(__dsub_rn(rsu[i], __dmul_rn(dual_u[i], c)), su[i]);
    }
    dsl[i] = a; dzl[i] = b; dsu[i] = c; dzu[i] = d;
  }
}
// ryd_tilde = ryd + ryd2*Dd_inv
__global__ void k_axzpy_small(int n, double* __restrict__ out, const double* __restrict__ y, const double* __restrict__ x, const double* __restrict__ z)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = __dadd_rn(y[i], __dmul_rn(x[i], z[i]));
}
// dd = (ryd2 + dyd)*Dd_inv
__global__ void k_recover_dd(int n, double* __restrict__ dd, const double* __restrict__ ryd2, const double* __restrict__ dyd, const double* __restrict__ Ddinv)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dd[i] = __dmul_rn(__dadd_rn(ryd2[i], dyd[i]), Ddinv[i]);
}
// rhs[i] = t[i] - r[i] for the stacked [ryc; ryd]
__global__ void k_sub_stacked(int meq, int mineq, double* __restrict__ rhs, const double* __restrict__ ryc, const double* __restrict__ ryd)
{
  const int m = meq + mineq;
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) rhs[i] -= (i < meq ? ryc[i] : ryd[i - meq]);
}

// rhs[i] = tdot[i] - sum_q Z[i][q] p[q] - ry[i],  p = [sigma*tdot[m..m+l); tdot[m+l..m+2l)]   (fused steps 1-2 of solveCompressed)
__global__ void k_fused_rhs(int m, int meq, int l, double sigma, const double* __restrict__ tdot, const double* __restrict__ Z,
                            const double* __restrict__ ryc, const double* __restrict__ ryd, double* __restrict__ rhs)
{
  const int n2 = 2 * l;
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    double corr = 0.0;
    for(int q = 0; q < n2; q++) corr += Z[(size_t)i * n2 + q] * (q < l ? sigma * tdot[m + q] : tdot[m + q]);
    rhs[i] = (tdot[i] - corr) - (i < meq ? ryc[i] : ryd[i - meq]);
  }
}

} // namespace

// =============================================================================================================
// p = V^{-1} [sigma*S (w.x); Y (w.x)] style multi-dot into k->p2l (device), all-reduced
int multidot(hb_lowrank* k, const double* w, const double* x, double sigma_s)
{
  hb_ctx* c = k->ctx;
  const int n2 = 2 * k->l;
  if(n2 == 0) return HB_OK;
  const int g = k->md_grid;
  for(int q0 = 0; q0 < n2; q0 += MD_CH) {
    k_multidot_partial<<<g, ET, 0, c->stream>>>(k->n, k->l, k->St, k->Yt, k->n, w, x, q0, k->md_partial);
    HB_LAUNCHED();
  }
  k_multidot_final<<<n2, 128, 0, c->stream>>>(g, k->l, sigma_s, k->md_partial, k->p2l);
  HB_LAUNCHED();
  HB_CHECK(hb_allreduce_sum(c, k->p2l, n2));
  return HB_OK;
}

namespace {

// the per-2048-column partials of A x (A: m x n) into partial[chunk][m]
int gemv_rows_partial(hb_ctx* c, int m, long long n, const double* A, long long lda, const double* x, double* partial)
{
  const int nchunks = (int)((n + GR_CHUNK - 1) / GR_CHUNK);
  if(nchunks == 0) return HB_OK;
  int rsplit = (4 * c->num_sms + nchunks - 1) / nchunks; // at least ~4 CTAs per SM in flight
  rsplit = rsplit < 1 ? 1 : (rsplit > 8 ? 8 : rsplit);
  k_gemv_rows_partial<<<dim3(nchunks, rsplit), GR_THREADS, 0, c->stream>>>(m, n, A, lda, x, partial);
  HB_LAUNCHED();
  return HB_OK;
}

// y = beta*y + alpha * (the partials of all chunks of n columns), all-reduced
int gemv_rows_final(hb_ctx* c, int m, long long n, const double* partial, double beta, double* y, double alpha)
{
  const int nchunks = (int)((n + GR_CHUNK - 1) / GR_CHUNK);
  // beta*y only on rank 0 before the reduction (hiopMatrixDenseRowMajor.cpp:464-467)
  k_gemv_rows_final<<<(m + 31) / 32, 256, 0, c->stream>>>(m, nchunks, partial, c->rank == 0 ? beta : 0.0, y, alpha);
  HB_LAUNCHED();
  return hb_allreduce_sum(c, y, m);
}

// row groups of k_gemv_cols for an m x n matrix: a short column range still fills the machine
int gemv_cols_groups(const hb_ctx* c, int m, long long n)
{
  const long long ctas1 = ((n + 1) / 2 + ET - 1) / ET;
  if(ctas1 >= 8LL * c->num_sms || m < 64) return 1;
  return ctas1 >= 2LL * c->num_sms ? 4 : 8;
}

int gemv_cols_launch(hb_ctx* c, int rg, int m, long long n, const double* A, long long lda, double beta, double* y, double alpha, const double* x)
{
  if(n == 0) return HB_OK;
  const long long pairs = (n + 1) / 2;
  if(rg == 1) k_gemv_cols<1><<<(unsigned)((pairs + ET - 1) / ET), ET, 0, c->stream>>>(m, n, A, lda, x, beta, y, alpha);
  else if(rg == 4) k_gemv_cols<4><<<(unsigned)((pairs + ET / 4 - 1) / (ET / 4)), ET, 0, c->stream>>>(m, n, A, lda, x, beta, y, alpha);
  else k_gemv_cols<8><<<(unsigned)((pairs + ET / 8 - 1) / (ET / 8)), ET, 0, c->stream>>>(m, n, A, lda, x, beta, y, alpha);
  HB_LAUNCHED();
  return HB_OK;
}

// ---- the Jacobian in column chunks --------------------------------------------------------------------------------------------

// timing-enabled cudaEventRecord between the kernels serialises the compute stream against the copy engine (with
// hb_ctx_enable_timing the first kernel starts only when the last copy has ended): off while chunks are copied
struct timing_off
{
  hb_ctx* c;
  bool saved;
  timing_off(hb_ctx* ctx, bool off) : c(ctx), saved(ctx->timing) { c->timing = saved && !off; }
  ~timing_off() { c->timing = saved; }
};

// Calls consume(q, c0, w, P, ld) on the context stream for every chunk q of k->jl: columns c0 .. c0+w-1, m rows at P with leading
// dimension ld. A layout with host rows copies chunk q on k->copy_stream first, `lookahead` chunks ahead of the consumers. Copies are
// submitted only that far ahead: if the two streams ever share a hardware work queue (CUDA_DEVICE_MAX_CONNECTIONS) commands run in
// submission order, and "all copies, then all kernels" would serialise. A reused slot is overwritten only after the context stream
// has finished with the chunk it held (lookahead <= slots - 1); the copy events are reused four chunks apart (lookahead <= 3).
template <class F>
int stream_chunks(hb_lowrank* k, F&& consume)
{
  hb_ctx* c = k->ctx;
  const hb_jac_layout& L = k->jl;
  const long long n = k->n;
  const int meq = k->meq, mi = k->mineq;
  const bool copy = L.from_host();
  const int lookahead = std::max(1, std::min(3, L.slots - 1));
  auto width = [&](int q) { return q * L.csz + L.csz <= n ? L.csz : n - q * L.csz; };
  auto submit_copy = [&](int q) -> int {
    const long long c0 = q * L.csz, w = width(q);
    double* P = const_cast<double*>(L.chunk(q));
    if(q >= L.slots) HB_CUDA(cudaStreamWaitEvent(k->copy_stream, k->slot_free[q % L.slots], 0));
    if(meq)
      HB_CUDA(cudaMemcpy2DAsync(P, sizeof(double) * L.ld, L.Jc + c0, sizeof(double) * n, sizeof(double) * w, meq, cudaMemcpyHostToDevice, k->copy_stream));
    if(mi)
      HB_CUDA(cudaMemcpy2DAsync(P + (size_t)meq * L.ld, sizeof(double) * L.ld, L.Jd + c0, sizeof(double) * n, sizeof(double) * w, mi,
                                cudaMemcpyHostToDevice, k->copy_stream));
    HB_CUDA(cudaEventRecord(k->chunk_ev[q % 4], k->copy_stream));
    return HB_OK;
  };
  if(copy) {
    HB_CHECK(k->copy_stream.create(cudaStreamNonBlocking));
    HB_CHECK(k->copy_start.create(cudaEventDisableTiming));
    for(hb_event& e : k->chunk_ev) HB_CHECK(e.create(cudaEventDisableTiming));
    if(L.slots < L.nch)
      for(hb_event& e : k->slot_free) HB_CHECK(e.create(cudaEventDisableTiming));
    // the copies start after everything enqueued so far on the context stream: its uploads, and the last reads of the slots
    HB_CUDA(cudaEventRecord(k->copy_start, c->stream));
    HB_CUDA(cudaStreamWaitEvent(k->copy_stream, k->copy_start, 0));
    for(int q = 0; q < L.nch && q < lookahead; q++) HB_CHECK(submit_copy(q));
  }
  timing_off off(c, copy);
  for(int q = 0; q < L.nch; q++) {
    if(copy) HB_CUDA(cudaStreamWaitEvent(c->stream, k->chunk_ev[q % 4], 0));
    HB_CHECK(consume(q, q * L.csz, width(q), L.chunk(q), L.ld));
    if(copy && q + L.slots < L.nch) HB_CUDA(cudaEventRecord(k->slot_free[q % L.slots], c->stream));
    if(copy && q + lookahead < L.nch) HB_CHECK(submit_copy(q + lookahead));
  }
  return HB_OK;
}

// The rows of [J; S; Y] restricted to the columns of each chunk of k->jl (nch x (m + 2 l) pointers). A rebuild costs a host
// synchronisation, so the tables of the last two layouts are kept: hb_lowrank_kkt_system_host condenses a staged upload and then
// runs on the device J it leaves.
int jac_table(hb_lowrank* k, const hb_rowtab** out)
{
  hb_ctx* c = k->ctx;
  const hb_jac_layout& L = k->jl;
  const int m = k->m, l = k->l, Ma = m + 2 * l;
  const long long key[9] = {(long long)(uintptr_t)L.base, L.stride, L.slots, L.ld, L.csz, L.nch, l, (long long)(uintptr_t)k->St,
                            (long long)(uintptr_t)k->Yt};
  if(memcmp(key, k->rows[0].key, sizeof(key))) std::swap(k->rows[0], k->rows[1]);
  hb_rowtab& t = k->rows[0];
  if(memcmp(key, t.key, sizeof(key))) { // neither: the older table is rebuilt
    memset(t.key, 0, sizeof(t.key));
    HB_CHECK(t.dev.reserve(c, (size_t)L.nch * Ma, "row pointers"));
    HB_CHECK(t.host.reserve(c, (size_t)L.nch * Ma, "row pointers"));
    bool al = true;
    for(int q = 0; q < L.nch; q++) {
      const long long c0 = q * L.csz;
      const double** row = t.host + (size_t)q * Ma;
      for(int i = 0; i < m; i++) row[i] = L.chunk(q) + (size_t)i * L.ld;
      for(int j = 0; j < l; j++) {
        row[m + j] = k->St + (size_t)j * k->n + c0;
        row[m + l + j] = k->Yt + (size_t)j * k->n + c0;
      }
      for(int i = 0; i < Ma; i++) al = al && ((reinterpret_cast<uintptr_t>(row[i]) & 15u) == 0);
    }
    HB_CUDA(cudaMemcpyAsync(t.dev, t.host, sizeof(double*) * (size_t)L.nch * Ma, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream)); // the host table is rewritten by a later rebuild
    t.aligned = al;
    memcpy(t.key, key, sizeof(key));
  }
  *out = &t;
  return HB_OK;
}

// ---- the condensation modes: HB_CONDENSE_AUTO (-1), HB_CONDENSE_FP64_DMMA (0), int8 slices (6, 7, 8), HB_CONDENSE_INT8_CRT ----
// AUTO runs the FP64 kernel: on H100 it is faster than either int8 mode at the sizes measured (DESIGN.md section 3). The int8 modes
// need the row maxima of the whole J before their first GEMM, so they need J whole on the device.
bool mode_valid(int mode) { return mode == HB_CONDENSE_AUTO || mode == HB_CONDENSE_FP64_DMMA || (mode >= 6 && mode <= 8) || mode == HB_CONDENSE_INT8_CRT; }
int mode_resolved(int mode) { return mode == HB_CONDENSE_AUTO ? HB_CONDENSE_FP64_DMMA : mode; }
bool mode_needs_whole_J(int mode) { return mode_resolved(mode) != HB_CONDENSE_FP64_DMMA; }
// HB_CONDENSE = oz6 | oz7 | oz8 | crt | dmma (anything starting with 'd'): the mode of a new handle; other values leave `mode`
int mode_from_env(int mode)
{
  if(const char* e = getenv("HB_CONDENSE")) {
    if(e[0] == 'o' && e[1] == 'z' && e[2] >= '6' && e[2] <= '8') return e[2] - '0';
    if(strcmp(e, "crt") == 0) return HB_CONDENSE_INT8_CRT;
    if(e[0] == 'd') return HB_CONDENSE_FP64_DMMA;
  }
  return mode;
}
// jac_whole for an int8 mode, the refusal naming the entry point `who` and the mode
int mode_whole_J(hb_lowrank* k, const char* who, int mode, const hb_rowtab** rows)
{
  char what[256];
  snprintf(what, sizeof(what), "%s: the %s (AUTO and 0 condense in FP64)", who,
           mode == HB_CONDENSE_INT8_CRT ? "int8 Chinese-remainder condensation of mode 100" : "int8-slice condensation of modes 6-8");
  return jac_whole(k, what, nullptr, rows);
}

} // namespace

bool jac_set(const hb_lowrank* k) { return k->m == 0 || k->jl.base; }

int jac_whole(hb_lowrank* k, const char* who, const double** J, const hb_rowtab** rows)
{
  if(k->jl.from_host()) {
    snprintf(g_hb_err, sizeof(g_hb_err), "%s needs the whole Jacobian on the device (hb_lowrank_set_jacobian); this one is streamed from host memory",
             who);
    return HB_ERR_INVALID;
  }
  if(J) *J = k->jl.base;
  return rows ? jac_table(k, rows) : HB_OK;
}

int jac_rows(hb_lowrank* k, double beta, double* y, double alpha, const double* x)
{
  hb_ctx* c = k->ctx;
  const int m = k->m;
  if(m == 0) return HB_OK;
  // every chunk starts at a multiple of GR_CHUNK columns: its partials are the ones of the same columns of the whole J, written in place
  const long long nchunks = (k->n + GR_CHUNK - 1) / GR_CHUNK;
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (size_t)(nchunks > 0 ? nchunks : 1) * m));
  double* partial = c->ws;
  HB_CHECK(stream_chunks(k, [&](int, long long c0, long long w, const double* P, long long ld) -> int {
    return gemv_rows_partial(c, m, w, P, ld, x + c0, partial + (size_t)(c0 / GR_CHUNK) * m);
  }));
  return gemv_rows_final(c, m, k->n, partial, beta, y, alpha);
}

int jac_cols(hb_lowrank* k, double beta, double* y, double alpha, const double* x)
{
  hb_ctx* c = k->ctx;
  const int m = k->m;
  // the row groups the whole J selects: each column then sums its rows in the same order
  const int rg = gemv_cols_groups(c, m, k->n);
  return stream_chunks(k, [&](int, long long c0, long long w, const double* P, long long ld) -> int {
    return gemv_cols_launch(c, rg, m, w, P, ld, beta, y + c0, alpha, x);
  });
}

// C = R diag(d) R^T, R = the first M rows of [J; S; Y], chunk by chunk: the partial products of later chunks (and their fused row
// dots) are added in chunk order, so the result does not depend on timing
int jac_syrk(hb_lowrank* k, int M, const double* d, double* C, const double* fuse_rx, double* tdot)
{
  hb_ctx* c = k->ctx;
  const size_t Mmax = (size_t)k->m + 2 * k->lmax;
  if(k->jl.nch > 1) HB_CHECK(k->Ctmp.reserve(c, Mmax * Mmax + Mmax, "partial C_aug"));
  const hb_rowtab* rows;
  HB_CHECK(jac_table(k, &rows));
  const int Ma = k->m + 2 * k->l;
  double* Ct = k->Ctmp;
  double* tt = Ct ? Ct + (size_t)M * M : nullptr;
  return stream_chunks(k, [&](int q, long long c0, long long w, const double*, long long) -> int {
    // every chunk starts at a multiple of 64 columns: its rows keep the 16-byte alignment of the whole rows
    HB_CHECK(hb_syrk_rows(c, M, w, rows->dev + (size_t)q * Ma, rows->aligned, d ? d + c0 : nullptr, q == 0 ? C : Ct, M,
                          fuse_rx ? fuse_rx + c0 : nullptr, tdot ? (q == 0 ? tdot : tt) : nullptr));
    if(q > 0) {
      HB_CHECK(hb_vec_axpy(c, (long long)M * M, C, 1.0, Ct));
      if(tdot) HB_CHECK(hb_vec_axpy(c, M, tdot, 1.0, tt));
    }
    return HB_OK;
  });
}

int jac_gram(hb_lowrank* k, const char* who, int M, const double* d, double* C, const double* fuse_rx, double* tdot, bool* fused)
{
  const int mode = mode_resolved(k->condense_mode);
  const bool fuse = fuse_rx && k->m > 0 &&
                    (mode != HB_CONDENSE_FP64_DMMA || (hb_syrk_extra_row_is_free(M) && (reinterpret_cast<uintptr_t>(fuse_rx) & 15u) == 0));
  if(!fuse) {
    fuse_rx = nullptr;
    tdot = nullptr;
  }
  if(mode == HB_CONDENSE_FP64_DMMA) HB_CHECK(jac_syrk(k, M, d, C, fuse_rx, tdot));
  else {
    const hb_rowtab* rows;
    HB_CHECK(mode_whole_J(k, who, mode, &rows));
    if(tdot && k->n == 0) HB_CUDA(cudaMemsetAsync(tdot, 0, sizeof(double) * M, k->ctx->stream)); // no row-maximum pass then
    if(mode == HB_CONDENSE_INT8_CRT) HB_CHECK(hb_syrk_rows_crt(k->ctx, M, k->n, rows->dev, rows->aligned, d, C, M, fuse_rx, tdot));
    else HB_CHECK(hb_syrk_rows_ozaki(k->ctx, M, k->n, rows->dev, rows->aligned, d, C, M, mode, fuse_rx, tdot));
  }
  if(fused) *fused = fuse;
  return HB_OK;
}

namespace {

// x = (B_k + D_x)^{-1} rhs
int hess_solve(hb_lowrank* k, const double* rhs, double* x)
{
  hb_ctx* c = k->ctx;
  if(k->n == 0) return HB_OK;
  if(k->l > 0) {
    HB_CHECK(multidot(k, k->DhInv, rhs, k->sigma)); // [sigma*S*(DhInv rhs); Y*(DhInv rhs)]
    HB_CHECK(hb_dense_bk_small_solve(c, 2 * k->l, k->V, 2 * k->l, k->ipivV, k->p2l, 2 * k->l, 1));
  }
  k_lowrank_apply<<<hb_grid(c, k->n, ET), ET, sizeof(double) * 2 * (k->l > 0 ? k->l : 1), c->stream>>>(
      k->n, k->l, k->sigma, k->St, k->Yt, k->n, k->p2l, k->DhInv, rhs, 0.0, nullptr, 0.0, 1.0, x);
  HB_LAUNCHED();
  return HB_OK;
}

int condense_enqueue(hb_lowrank* k, const double* fuse_rx = nullptr);
int condense_finish(hb_lowrank* k);


// Enqueues the whole condensation (C_aug, all-reduce, V, N, equilibrated Cholesky) without touching the host. The info words are
// copied to pinned memory; condense_check() looks at them after a stream synchronisation.
int do_condense_async(hb_lowrank* k, const double* fuse_rx = nullptr)
{
  HB_REQUIRE(k->have_update, "hb_lowrank_condense: call hb_lowrank_update first");
  HB_REQUIRE(jac_set(k), "hb_lowrank_condense: Jacobian not set");
  HB_CHECK(condense_enqueue(k, fuse_rx));
  k->check_pending = true;
  k->cond_valid = true; // optimistic: a failure is reported by the next synchronous call (hb_lowrank_check / hb_lowrank_condense)
  return HB_OK;
}

int condense_check(hb_lowrank* k)
{
  hb_ctx* c = k->ctx;
  if(!k->check_pending) return HB_OK;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  k->check_pending = false;
  if(k->info_host[0] != 0) {
    k->cond_valid = false;
    return hb_fail(HB_ERR_NUMERIC, "hb_lowrank_condense: V is singular (BFGS inner matrix)%s", "");
  }
  if(k->info_host[1] != 0) {
    k->cond_valid = false;
    snprintf(g_hb_err, sizeof(g_hb_err), "hb_lowrank_condense: condensed matrix N is not SPD (leading minor %d)", k->info_host[1]);
    return HB_ERR_NUMERIC;
  }
  return HB_OK;
}

// synchronous condensation: reports breakdowns now
int do_condense(hb_lowrank* k)
{
  HB_CHECK(do_condense_async(k));
  return condense_check(k);
}

// fuse_rx (optional): the x-block of the right-hand side the caller is about to solve for; jac_gram leaves tdot = [J; S; Y] (DhInv .* rx)
// where that costs no extra pass over J, from which step 2 of solveCompressed follows without reading J again (see solve_compressed)
int condense_enqueue(hb_lowrank* k, const double* fuse_rx)
{
  const int Ma = k->m + 2 * k->l;
  k->tdot_valid = false;
  if(Ma > 0) {
    HB_CHECK(jac_gram(k, "hb_lowrank_condense", Ma, k->DhInv, k->Caug, fuse_rx, k->tdot, &k->tdot_valid));
    k->condense_used = mode_resolved(k->condense_mode);
  }
  return condense_finish(k);
}

// everything after C_aug = [J;S;Y] DhInv [J;S;Y]^T (local columns) is in k->Caug
int condense_finish(hb_lowrank* k)
{
  hb_ctx* c = k->ctx;
  const int m = k->m, l = k->l, Ma = m + 2 * l;
  HB_CUDA(cudaMemsetAsync(k->info, 0, sizeof(int) * 4, c->stream));
  hb_phase_mark(c, HB_PH_CAUG);
  if(Ma > 0 && c->nranks > 1) {
    // the symmetric C_aug travels as its packed upper triangle: Ma(Ma+1)/2 doubles instead of Ma^2
    const long long tot = (long long)Ma * (Ma + 1) / 2;
    HB_CHECK(k->tri.reserve(c, (size_t)(k->m + 2 * k->lmax) * (k->m + 2 * k->lmax + 1) / 2 + (size_t)(k->m + 2 * k->lmax), "packed C_aug"));
    const int g = hb_grid(c, tot);
    k_pack_upper<<<g, 256, 0, c->stream>>>(Ma, k->Caug, Ma, k->tri);
    HB_LAUNCHED();
    // the fused row dots ride behind the triangle in the same reduction
    if(k->tdot_valid) HB_CUDA(cudaMemcpyAsync(k->tri + tot, k->tdot, sizeof(double) * Ma, cudaMemcpyDeviceToDevice, c->stream));
    HB_CHECK(hb_allreduce_sum(c, k->tri, tot + (k->tdot_valid ? Ma : 0)));
    k_unpack_upper<<<g, 256, 0, c->stream>>>(Ma, k->Caug, Ma, k->tri);
    HB_LAUNCHED();
    if(k->tdot_valid) HB_CUDA(cudaMemcpyAsync(k->tdot, k->tri + tot, sizeof(double) * Ma, cudaMemcpyDeviceToDevice, c->stream));
  }
  hb_phase_mark(c, HB_PH_ALLREDUCE);
  if(l > 0) {
    k_build_V<<<(4 * l * l + 127) / 128, 128, 0, c->stream>>>(m, l, k->sigma, k->Caug, Ma, k->SSt, k->Ld, k->Dd_sec, k->V);
    HB_LAUNCHED();
    HB_CHECK(hb_dense_bk_small_factor(c, 2 * l, k->V, 2 * l, k->ipivV, k->info + 0));
    if(m > 0) {
      k_build_U<<<(m * 2 * l + 127) / 128, 128, 0, c->stream>>>(m, l, k->sigma, k->Caug, Ma, k->U, k->Z);
      HB_LAUNCHED();
      HB_CHECK(hb_dense_bk_small_solve(c, 2 * l, k->V, 2 * l, k->ipivV, k->Z, 2 * l, m));
    }
  }
  if(m > 0) {
    const long long tot = (long long)m * m;
    k_form_N<<<hb_grid(c, tot), 256, 0, c->stream>>>(m, k->meq, l, k->Caug, Ma, k->U, k->Z, k->Dd_inv, k->Nmat);
    HB_LAUNCHED();
    HB_CHECK(hb_dense_equilibrate(c, m, k->Nmat, m, k->F, m, k->svec));
    hb_phase_mark(c, HB_PH_VN);
    HB_CHECK(hb_dense_condensed_factor(c, &k->big, m, k->F, m, k->Finv, k->info + 1));
    hb_phase_mark(c, HB_PH_CHOL);
  }
  HB_CUDA(cudaMemcpyAsync(k->info_host, k->info, sizeof(int) * 4, cudaMemcpyDeviceToHost, c->stream));
  return HB_OK;
}

// a device J: one chunk of all n columns at J (ld n)
hb_jac_layout device_layout(long long n, const double* J)
{
  hb_jac_layout L;
  L.csz = L.ld = n;
  L.base = J;
  return L;
}

} // namespace

extern "C" int hb_lowrank_create(hb_ctx* c, long long n_local, int m_eq, int m_ineq, int l_max, hb_lowrank** out)
{
  HB_REQUIRE(c && out && n_local >= 0 && m_eq >= 0 && m_ineq >= 0 && l_max >= 0 && l_max <= 256, "hb_lowrank_create: bad arguments");
  HB_CUDA(cudaSetDevice(c->device));
  std::unique_ptr<hb_lowrank> k(new hb_lowrank);
  k->ctx = c; k->n = n_local; k->meq = m_eq; k->mineq = m_ineq; k->m = m_eq + m_ineq; k->lmax = l_max;
  k->jl = device_layout(n_local, nullptr);
  k->condense_mode = mode_from_env(k->condense_mode);
  const int m = k->m, Mamax = m + 2 * l_max, l2 = 2 * l_max;
  HB_CHECK(k->Dx.reserve(c, n_local, "Dx")); HB_CHECK(k->DhInv.reserve(c, n_local, "DhInv"));
  HB_CHECK(k->Dd.reserve(c, m_ineq, "Dd")); HB_CHECK(k->Dd_inv.reserve(c, m_ineq, "Dd_inv"));
  HB_CHECK(k->Caug.reserve(c, (size_t)Mamax * Mamax, "C_aug"));
  HB_CHECK(k->SSt.reserve(c, (size_t)l_max * l_max, "S S^T")); HB_CHECK(k->Ld.reserve(c, (size_t)l_max * l_max, "L")); HB_CHECK(k->Dd_sec.reserve(c, l_max, "D"));
  HB_CHECK(k->V.reserve(c, (size_t)l2 * l2, "V")); HB_CHECK(k->Mdir.reserve(c, (size_t)l2 * l2, "M"));
  HB_CHECK(k->U.reserve(c, (size_t)m * l2, "U")); HB_CHECK(k->Z.reserve(c, (size_t)m * l2, "Z"));
  HB_CHECK(k->Nmat.reserve(c, (size_t)m * m, "N")); HB_CHECK(k->F.reserve(c, (size_t)m * m, "the factor of N"));
  HB_CHECK(k->svec.reserve(c, m, "the scaling of N")); HB_CHECK(k->rhs.reserve(c, m, "rhs")); HB_CHECK(k->dy.reserve(c, m, "dy"));
  HB_CHECK(k->work.reserve(c, 2 * (size_t)m + 2, "refinement scratch"));
  HB_CHECK(k->Finv.reserve(c, HB_CHOL_INV_DOUBLES(m > 0 ? m : 1), "diagonal-block inverses of N"));
  HB_CHECK(k->stats.reserve(c, 4, "solve statistics"));
  HB_CHECK(k->nv1.reserve(c, n_local, "n-vector scratch")); HB_CHECK(k->nv2.reserve(c, n_local, "n-vector scratch"));
  HB_CHECK(k->tdot.reserve(c, (size_t)Mamax, "fused row dots"));
  HB_CHECK(k->p2l.reserve(c, l2, "multi-dot result"));
  k->md_grid = hb_grid(c, n_local, ET);
  HB_CHECK(k->md_partial.reserve(c, (size_t)k->md_grid * (l2 > 0 ? l2 : 1), "multi-dot partials"));
  HB_CHECK(k->mi1.reserve(c, m_ineq, "m_ineq scratch")); HB_CHECK(k->mi2.reserve(c, m_ineq, "m_ineq scratch"));
  HB_CHECK(k->ipivV.reserve(c, (size_t)l2 + 1, "pivots of V")); HB_CHECK(k->ipivM.reserve(c, (size_t)l2 + 1, "pivots of M"));
  HB_CHECK(k->info.reserve(c, 4, "info words"));
  HB_CHECK(k->sst_rows.dev.reserve(c, l_max, "row pointers")); HB_CHECK(k->sst_rows.host.reserve(c, l_max, "row pointers"));
  HB_CHECK(k->info_host.reserve(c, 4, "info words"));
  HB_CHECK(k->stats_host.reserve(c, 4, "solve statistics"));
  *out = k.release();
  return HB_OK;
}

extern "C" int hb_lowrank_destroy(hb_lowrank* k)
{
  if(!k) return HB_OK;
  cudaSetDevice(k->ctx->device);
  cudaStreamSynchronize(k->ctx->stream);
  delete k;
  return HB_OK;
}

extern "C" int hb_lowrank_set_patterns(hb_lowrank* k, const double* ixl, const double* ixu, const double* idl, const double* idu)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE((ixl && ixu) || k->n == 0, "hb_lowrank_set_patterns: null x pattern");
  HB_REQUIRE((idl && idu) || k->mineq == 0, "hb_lowrank_set_patterns: null d pattern");
  k->ixl = ixl; k->ixu = ixu; k->idl = idl; k->idu = idu;
  k->cond_valid = false;
  return HB_OK;
}

extern "C" int hb_lowrank_set_jacobian(hb_lowrank* k, const double* Jc, const double* Jd)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE((Jc || k->meq == 0) && (Jd || k->mineq == 0), "hb_lowrank_set_jacobian: null Jacobian");
  hb_ctx* c = k->ctx;
  if(k->ring) { // back from a host-resident Jacobian: its slots are no longer needed
    HB_CUDA(cudaStreamSynchronize(c->stream));
    k->ring.reset();
  }
  const double* J;
  if(k->meq == 0) J = Jd;
  else if(k->mineq == 0 || Jd == Jc + (size_t)k->meq * k->n) J = Jc;
  else {
    HB_CHECK(k->Jpack.reserve(c, (size_t)k->m * k->n, "the packed Jacobian"));
    HB_CUDA(cudaMemcpyAsync(k->Jpack, Jc, sizeof(double) * (size_t)k->meq * k->n, cudaMemcpyDeviceToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(k->Jpack + (size_t)k->meq * k->n, Jd, sizeof(double) * (size_t)k->mineq * k->n, cudaMemcpyDeviceToDevice, c->stream));
    J = k->Jpack;
  }
  k->jl = device_layout(k->n, J);
  k->cond_valid = false;
  return HB_OK;
}

namespace {
// page-locked (hb_malloc_host / cudaHostRegister) host memory: the only kind a copy engine reads asynchronously
bool is_page_locked(const void* p)
{
  cudaPointerAttributes a;
  if(cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}
} // namespace

extern "C" int hb_lowrank_set_jacobian_host(hb_lowrank* k, const double* Jc_host, const double* Jd_host, long long panel_cols)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE((Jc_host || k->meq == 0) && (Jd_host || k->mineq == 0), "hb_lowrank_set_jacobian_host: null Jacobian");
  HB_REQUIRE((k->meq == 0 || is_page_locked(Jc_host)) && (k->mineq == 0 || is_page_locked(Jd_host)),
             "hb_lowrank_set_jacobian_host: Jc and Jd must be page-locked host memory (hb_malloc_host or cudaHostRegister)");
  hb_ctx* c = k->ctx;
  const long long n = k->n, m = k->m;
  // default: panels of about 128 MB, so that a large J takes several and the copies overlap the kernels. Always a multiple of
  // GR_CHUNK columns, so that every panel starts on a J x partial boundary (and at a 16-byte aligned column); never wider than J.
  long long P = panel_cols > 0 ? panel_cols : (((long long)128 << 20) / (8 * (m > 0 ? m : 1)));
  P = (P + GR_CHUNK - 1) / GR_CHUNK * GR_CHUNK;
  const long long Pmax = (n + GR_CHUNK - 1) / GR_CHUNK * GR_CHUNK;
  if(P > Pmax) P = Pmax > 0 ? Pmax : GR_CHUNK;
  hb_jac_layout L;
  L.csz = P;
  L.nch = (int)((n + P - 1) / P);
  L.slots = std::min(HB_PANEL_RING, L.nch);
  // the leading dimension has the parity of n: the gemv kernels then take the same (vector or scalar) path on a panel as on a device
  // J. The slots share one allocation, each starting 16-byte aligned, as the vector paths of the gemvs and k_syrk_ws require.
  L.ld = P + (n & 1);
  L.stride = (m * L.ld + 1) & ~1LL;
  L.Jc = Jc_host;
  L.Jd = Jd_host;
  const size_t need = (size_t)L.slots * L.stride;
  if(k->ring.capacity() > need) { // fewer or narrower slots than before: hold only these
    HB_CUDA(cudaStreamSynchronize(c->stream));
    k->ring.reset();
  }
  HB_CHECK(k->ring.reserve(c, need, "the Jacobian panels"));
  L.base = k->ring;
  k->jl = L;
  k->cond_valid = false;
  return HB_OK;
}

extern "C" int hb_lowrank_set_secant(hb_lowrank* k, int l, double sigma, const double* St, const double* Yt, const double* L_host,
                                     const double* D_host)
{
  HB_REQUIRE(k && l >= 0 && l <= k->lmax, "hb_lowrank_set_secant: bad memory length");
  HB_REQUIRE(l == 0 || (St && Yt && L_host && D_host), "hb_lowrank_set_secant: null argument");
  hb_ctx* c = k->ctx;
  k->l = l; k->sigma = sigma; k->St = St; k->Yt = Yt;
  k->cond_valid = false;
  k->mdir_valid = false;
  k->have_update = false; // DhInv depends on sigma
  if(l > 0) {
    HB_CUDA(cudaMemcpyAsync(k->Ld, L_host, sizeof(double) * l * l, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(k->Dd_sec, D_host, sizeof(double) * l, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream)); // L_host / D_host are caller-owned pageable memory
    // S S^T (l x l) -- depends only on the secant memory, not on the barrier diagonal; over whole rows, wherever J is
    hb_rowtab& t = k->sst_rows;
    bool al = true;
    for(int q = 0; q < l; q++) {
      t.host[q] = St + (size_t)q * k->n;
      al = al && ((reinterpret_cast<uintptr_t>(t.host[q]) & 15u) == 0);
    }
    HB_CUDA(cudaMemcpyAsync(t.dev, t.host, sizeof(double*) * l, cudaMemcpyHostToDevice, c->stream));
    HB_CHECK(hb_syrk_rows(c, l, k->n, t.dev, al, nullptr, k->SSt, l));
    HB_CHECK(hb_allreduce_sum(c, k->SSt, (long long)l * l));
    HB_CUDA(cudaStreamSynchronize(c->stream));
  }
  return HB_OK;
}

extern "C" int hb_lowrank_update(hb_lowrank* k, const double* zl, const double* sxl, const double* zu, const double* sxu, const double* vl,
                                 const double* sdl, const double* vu, const double* sdu)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE(k->n == 0 || (zl && sxl && zu && sxu), "hb_lowrank_update: null x-side iterate block");
  HB_REQUIRE(k->mineq == 0 || (vl && sdl && vu && sdu), "hb_lowrank_update: null d-side iterate block");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_lowrank_update: patterns not set");
  hb_ctx* c = k->ctx;
  k->zl = zl; k->sxl = sxl; k->zu = zu; k->sxu = sxu; k->vl = vl; k->sdl = sdl; k->vu = vu; k->sdu = sdu;
  hb_phase_mark(c, HB_PH_START);
  if(k->n > 0) {
    k_update_x<<<hb_grid(c, k->n, ET), ET, 0, c->stream>>>(k->n, zl, sxl, zu, sxu, k->ixl, k->ixu, k->sigma, k->Dx, k->DhInv);
    HB_LAUNCHED();
  }
  if(k->mineq > 0) {
    k_update_d<<<(k->mineq + 127) / 128, 128, 0, c->stream>>>(k->mineq, vl, sdl, vu, sdu, k->idl, k->idu, k->Dd, k->Dd_inv);
    HB_LAUNCHED();
  }
  hb_phase_mark(c, HB_PH_UPDATE);
  k->have_update = true;
  k->cond_valid = false;
  return HB_OK;
}

extern "C" int hb_lowrank_set_condense_mode(hb_lowrank* k, int mode)
{
  HB_REQUIRE(k && mode_valid(mode), "hb_lowrank_set_condense_mode: mode must be -1, 0, 6, 7, 8 or 100");
  if(mode_needs_whole_J(mode)) HB_CHECK(mode_whole_J(k, "hb_lowrank_set_condense_mode", mode, nullptr));
  k->condense_mode = mode;
  k->cond_valid = false;
  return HB_OK;
}

extern "C" int hb_lowrank_get_condense_mode(hb_lowrank* k) { return k ? k->condense_used : 0; }

extern "C" int hb_lowrank_condense(hb_lowrank* k)
{
  HB_REQUIRE(k, "null handle");
  return do_condense(k);
}

extern "C" int hb_lowrank_condense_async(hb_lowrank* k)
{
  HB_REQUIRE(k, "null handle");
  return do_condense_async(k);
}
extern "C" int hb_lowrank_check(hb_lowrank* k)
{
  HB_REQUIRE(k, "null handle");
  return condense_check(k);
}

extern "C" int hb_lowrank_hess_solve(hb_lowrank* k, const double* rhs, double* x)
{
  HB_REQUIRE(k && (k->n == 0 || (rhs && x)), "hb_lowrank_hess_solve: null argument");
  if(!k->cond_valid) HB_CHECK(do_condense_async(k));
  return hess_solve(k, rhs, x);
}

extern "C" int hb_lowrank_solve_compressed(hb_lowrank* k, double* rx, const double* ryc, const double* ryd, double* dx, double* dyc, double* dyd)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE(k->n == 0 || (rx && dx), "hb_lowrank_solve_compressed: null x block");
  HB_REQUIRE((k->meq == 0 || (ryc && dyc)) && (k->mineq == 0 || (ryd && dyd)), "hb_lowrank_solve_compressed: null dual block");
  hb_ctx* c = k->ctx;
  const int m = k->m;
  // A pending condensation is enqueued here (breakdowns surface at the next synchronous call, hb_lowrank_check). With the int8-slice
  // kernel its row-maximum sweep over [J; S; Y] also produces tdot = [J; S; Y] (DhInv .* rx), and steps 1-2 collapse to
  //   J (H+Dx)^{-1} rx = tdot_J - Z [sigma*tdot_S; tdot_Y],   Z = U V^{-1}  (U = [sigma J DhInv S^T, J DhInv Y^T], kept from the condensation)
  // which is the same product with the low-rank correction applied on the m side: J is not read a second time.
  bool fused = false;
  if(!k->cond_valid) {
    HB_CHECK(do_condense_async(k, rx));
    fused = k->tdot_valid;
    k->tdot_valid = false; // tied to this rx
  }
  k->rhs_fused = fused;
  if(fused) {
    hb_phase_mark(c, HB_PH_HSOLVE1);
    k_fused_rhs<<<(m + 127) / 128, 128, 0, c->stream>>>(m, k->meq, k->l, k->sigma, k->tdot, k->Z, ryc, ryd, k->rhs);
    HB_LAUNCHED();
    hb_phase_mark(c, HB_PH_JX);
  } else {
    // 1. dx_tmp = (H+Dx)^{-1} rx                                  hiopKKTLinSys.cpp:1146
    HB_CHECK(hess_solve(k, rx, dx));
    hb_phase_mark(c, HB_PH_HSOLVE1);
    if(m > 0) {
      // 2. rhs = J*dx_tmp - [ryc; ryd]                              :1154-1157
      HB_CHECK(jac_rows(k, 0.0, k->rhs, 1.0, dx));
      hb_phase_mark(c, HB_PH_JX);
      k_sub_stacked<<<(m + 127) / 128, 128, 0, c->stream>>>(k->meq, k->mineq, k->rhs, ryc, ryd);
      HB_LAUNCHED();
    }
  }
  if(m > 0) {
    // 3. N dy = rhs with residual-driven refinement               :1169, 1192-1350
    HB_CHECK(hb_dense_condensed_solve(c, m, k->F, m, k->Finv, k->svec, k->Nmat, m, k->rhs, k->dy, k->work, 1e-8, 3, k->stats));
    hb_phase_mark(c, HB_PH_SPDSOLVE);
    if(k->meq) HB_CUDA(cudaMemcpyAsync(dyc, k->dy, sizeof(double) * k->meq, cudaMemcpyDeviceToDevice, c->stream));
    if(k->mineq) HB_CUDA(cudaMemcpyAsync(dyd, k->dy + k->meq, sizeof(double) * k->mineq, cudaMemcpyDeviceToDevice, c->stream));
    // 4. rx = rx - J^T dy                                          :1178
    HB_CHECK(jac_cols(k, 1.0, rx, -1.0, k->dy));
    hb_phase_mark(c, HB_PH_JTY);
    HB_CUDA(cudaMemcpyAsync(k->stats_host, k->stats, sizeof(double) * 2, cudaMemcpyDeviceToHost, c->stream));
  }
  // 5. dx = (H+Dx)^{-1} rx                                        :1180
  HB_CHECK(hess_solve(k, rx, dx));
  hb_phase_mark(c, HB_PH_HSOLVE2);
  return HB_OK;
}

extern "C" int hb_lowrank_last_solve_stats(hb_lowrank* k, int* n_refine, double* resid_inf)
{
  HB_REQUIRE(k, "null handle");
  HB_CHECK(condense_check(k));
  HB_CUDA(cudaStreamSynchronize(k->ctx->stream));
  if(n_refine) *n_refine = k->m > 0 ? (int)k->stats_host[0] : 0;
  if(resid_inf) *resid_inf = k->m > 0 ? k->stats_host[1] : 0.0;
  return HB_OK;
}

extern "C" int hb_lowrank_compute_directions(hb_lowrank* k, const double* const* res, double* const* dir)
{
  HB_REQUIRE(k && res && dir, "hb_lowrank_compute_directions: null argument");
  HB_REQUIRE(k->have_update, "hb_lowrank_compute_directions: call hb_lowrank_update first");
  hb_ctx* c = k->ctx;
  enum { RX, RD, RYC, RYD, RXL, RXU, RDL, RDU, RSZL, RSZU, RSVL, RSVU };
  enum { DX, DD, DYC, DYD, DSXL, DSXU, DSDL, DSDU, DZL, DZU, DVL, DVU };
  const long long n = k->n;
  const int mi = k->mineq;
  double* rx_tilde = k->nv1;
  double* ryd2 = k->mi1;
  double* ryd_tilde = k->mi2;
  if(n > 0) {
    k_reduce_rhs<<<hb_grid(c, n, ET), ET, 0, c->stream>>>(n, res[RX], res[RSZL], k->zl, res[RXL], k->sxl, k->ixl, res[RSZU], k->zu, res[RXU], k->sxu,
                                                          k->ixu, rx_tilde);
    HB_LAUNCHED();
  }
  if(mi > 0) {
    k_reduce_rhs<<<hb_grid(c, mi, ET), ET, 0, c->stream>>>(mi, res[RD], res[RSVL], k->vl, res[RDL], k->sdl, k->idl, res[RSVU], k->vu, res[RDU],
                                                           k->sdu, k->idu, ryd2);
    HB_LAUNCHED();
    k_axzpy_small<<<(mi + 127) / 128, 128, 0, c->stream>>>(mi, ryd_tilde, res[RYD], ryd2, k->Dd_inv);
    HB_LAUNCHED();
  }
  HB_CHECK(hb_lowrank_solve_compressed(k, rx_tilde, res[RYC], ryd_tilde, dir[DX], dir[DYC], dir[DYD]));
  if(mi > 0) {
    k_recover_dd<<<(mi + 127) / 128, 128, 0, c->stream>>>(mi, dir[DD], ryd2, dir[DYD], k->Dd_inv);
    HB_LAUNCHED();
    k_recover_slack_duals<<<hb_grid(c, mi, ET), ET, 0, c->stream>>>(mi, dir[DD], res[RDL], res[RSVL], k->vl, k->sdl, k->idl, res[RDU], res[RSVU],
                                                                    k->vu, k->sdu, k->idu, dir[DSDL], dir[DVL], dir[DSDU], dir[DVU]);
    HB_LAUNCHED();
  }
  if(n > 0) {
    k_recover_slack_duals<<<hb_grid(c, n, ET), ET, 0, c->stream>>>(n, dir[DX], res[RXL], res[RSZL], k->zl, k->sxl, k->ixl, res[RXU], res[RSZU], k->zu,
                                                                   k->sxu, k->ixu, dir[DSXL], dir[DZL], dir[DSXU], dir[DZU]);
    HB_LAUNCHED();
  }
  return HB_OK;
}

extern "C" int hb_lowrank_hess_times_vec(hb_lowrank* k, double beta, double* y, double alpha, const double* x, int add_log_term)
{
  HB_REQUIRE(k && (k->n == 0 || (x && y)), "hb_lowrank_hess_times_vec: null argument");
  HB_REQUIRE(!add_log_term || k->have_update, "hb_lowrank_hess_times_vec: Dx not available (call update)");
  hb_ctx* c = k->ctx;
  const int l = k->l;
  if(k->n == 0) return HB_OK;
  if(l > 0) {
    if(!k->mdir_valid) {
      HB_CUDA(cudaMemsetAsync(k->info + 2, 0, sizeof(int), c->stream));
      k_build_Mdirect<<<(4 * l * l + 127) / 128, 128, 0, c->stream>>>(l, k->sigma, k->SSt, k->Ld, k->Dd_sec, k->Mdir);
      HB_LAUNCHED();
      HB_CHECK(hb_dense_bk_small_factor(c, 2 * l, k->Mdir, 2 * l, k->ipivM, k->info + 2));
      k->mdir_valid = true;
    }
    HB_CHECK(multidot(k, nullptr, x, k->sigma)); // [sigma S x; Y x]
    HB_CHECK(hb_dense_bk_small_solve(c, 2 * l, k->Mdir, 2 * l, k->ipivM, k->p2l, 2 * l, 1));
  }
  k_lowrank_apply<<<hb_grid(c, k->n, ET), ET, sizeof(double) * 2 * (l > 0 ? l : 1), c->stream>>>(
      k->n, l, k->sigma, k->St, k->Yt, k->n, k->p2l, nullptr, x, k->sigma, add_log_term ? k->Dx.get() : nullptr, beta, alpha, y);
  HB_LAUNCHED();
  return HB_OK;
}

extern "C" const double* hb_lowrank_Dx(hb_lowrank* k) { return k ? k->Dx.get() : nullptr; }
extern "C" const double* hb_lowrank_DhInv(hb_lowrank* k) { return k ? k->DhInv.get() : nullptr; }
extern "C" const double* hb_lowrank_Dd_inv(hb_lowrank* k) { return k ? k->Dd_inv.get() : nullptr; }
extern "C" const double* hb_lowrank_N(hb_lowrank* k) { return k ? k->Nmat.get() : nullptr; }
extern "C" const double* hb_lowrank_tdot(hb_lowrank* k) { return k ? k->tdot.get() : nullptr; }

extern "C" int hb_debug_lowrank_state(hb_lowrank* k, double* Caug, double* SSt, double* V_built, double* V_factor, int* ipivV, double* U, double* Z,
                                      double* M_built, double* M_factor, int* ipivM, double* p2l, double* rhs, double* tdot, int* info4)
{
  HB_REQUIRE(k, "null handle");
  hb_ctx* c = k->ctx;
  const int m = k->m, l = k->l, n2 = 2 * l, Ma = m + n2;
  auto get = [&](void* dst, const void* src, size_t bytes) -> int {
    if(dst && bytes) HB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    return HB_OK;
  };
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if((V_built || M_built) && l > 0) {
    // rebuilt from the handle's current inputs into scratch: the production path keeps no unfactored copy
    HB_CHECK(hb_ws_reserve(c, sizeof(double) * (size_t)n2 * n2));
    double* W = (double*)c->ws;
    if(V_built) {
      k_build_V<<<(4 * l * l + 127) / 128, 128, 0, c->stream>>>(m, l, k->sigma, k->Caug, Ma, k->SSt, k->Ld, k->Dd_sec, W);
      HB_LAUNCHED();
      HB_CHECK(get(V_built, W, sizeof(double) * n2 * n2));
      HB_CUDA(cudaStreamSynchronize(c->stream));
    }
    if(M_built) {
      k_build_Mdirect<<<(4 * l * l + 127) / 128, 128, 0, c->stream>>>(l, k->sigma, k->SSt, k->Ld, k->Dd_sec, W);
      HB_LAUNCHED();
      HB_CHECK(get(M_built, W, sizeof(double) * n2 * n2));
    }
  }
  HB_CHECK(get(Caug, k->Caug, sizeof(double) * Ma * Ma));
  HB_CHECK(get(SSt, k->SSt, sizeof(double) * l * l));
  HB_CHECK(get(V_factor, k->V, sizeof(double) * n2 * n2));
  HB_CHECK(get(ipivV, k->ipivV, sizeof(int) * n2));
  HB_CHECK(get(U, k->U, sizeof(double) * m * n2));
  HB_CHECK(get(Z, k->Z, sizeof(double) * m * n2));
  HB_CHECK(get(M_factor, k->Mdir, sizeof(double) * n2 * n2));
  HB_CHECK(get(ipivM, k->ipivM, sizeof(int) * n2));
  HB_CHECK(get(p2l, k->p2l, sizeof(double) * n2));
  HB_CHECK(get(rhs, k->rhs, sizeof(double) * m));
  HB_CHECK(get(tdot, k->tdot, sizeof(double) * Ma));
  HB_CHECK(get(info4, k->info, sizeof(int) * 3));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if(info4) info4[3] = k->rhs_fused ? 1 : 0;
  return HB_OK;
}

// ---- one whole KKT system from host buffers ----------------------------------------------------------------------------
extern "C" int hb_lowrank_kkt_system_host(hb_lowrank* k, const double* Jc_host, const double* Jd_host, const double* zl, const double* sxl,
                                          const double* zu, const double* sxu, const double* vl, const double* sdl, const double* vu,
                                          const double* sdu, const double* rx, const double* ryc, const double* ryd, double* dx, double* dyc,
                                          double* dyd)
{
  HB_REQUIRE(k, "null handle");
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int meq = k->meq, mi = k->mineq;
  // device staging: 0..3 x-side iterate, 4..7 d-side iterate, 8 rx, 9 ryc, 10 ryd, 11 dx, 12 dyc, 13 dyd
  const size_t sz[14] = {(size_t)n, (size_t)n, (size_t)n, (size_t)n, (size_t)mi, (size_t)mi, (size_t)mi, (size_t)mi, (size_t)n, (size_t)meq, (size_t)mi,
                         (size_t)n, (size_t)meq, (size_t)mi};
  for(int i = 0; i < 14; i++) HB_CHECK(k->hbuf[i].reserve(c, sz[i], "host-call staging"));
  const double* src[11] = {zl, sxl, zu, sxu, vl, sdl, vu, sdu, rx, ryc, ryd};
  for(int i = 0; i < 11; i++)
    if(sz[i]) {
      HB_REQUIRE(src[i], "hb_lowrank_kkt_system_host: null host input");
      HB_CUDA(cudaMemcpyAsync(k->hbuf[i], src[i], sizeof(double) * sz[i], cudaMemcpyHostToDevice, c->stream));
    }
  const int m = k->m, Ma = m + 2 * k->l;
  const bool have_J = Jc_host || Jd_host;
  // The 8 m n bytes of J dominate this call (PCIe). From 256 MiB on, J is uploaded in column chunks on a second stream and each chunk
  // is condensed (exact FP64 DMMA kernel, which needs no global row scaling) while the next one is in flight; the partial C_aug are
  // added in chunk order, so the result does not depend on timing.
  constexpr size_t chunk_min_bytes = (size_t)256 << 20;
  const bool chunked = have_J && Ma > 0 && !mode_needs_whole_J(k->condense_mode) && (size_t)m * n * sizeof(double) >= chunk_min_bytes && n >= 2048;
  if(have_J) HB_CHECK(k->hJ.reserve(c, (size_t)k->m * n, "the staged Jacobian"));
  if(have_J && !chunked) {
    if(meq) HB_CUDA(cudaMemcpyAsync(k->hJ, Jc_host, sizeof(double) * (size_t)meq * n, cudaMemcpyHostToDevice, c->stream));
    if(mi) HB_CUDA(cudaMemcpyAsync(k->hJ + (size_t)meq * n, Jd_host, sizeof(double) * (size_t)mi * n, cudaMemcpyHostToDevice, c->stream));
  }
  if(have_J) HB_CHECK(hb_lowrank_set_jacobian(k, k->hJ, k->hJ + (size_t)meq * n));
  HB_CHECK(hb_lowrank_update(k, k->hbuf[0], k->hbuf[1], k->hbuf[2], k->hbuf[3], k->hbuf[4], k->hbuf[5], k->hbuf[6], k->hbuf[7]));
  // Not chunked: the condensation stays pending so that solve_compressed below runs it with rx fused, exactly as a device-side
  // update + solveCompressed does; breakdowns are reported after the solve.
  if(chunked) {
    // the staged layout for this one condensation: 16 chunks of a multiple of 64 columns, each copied into its own columns of k->hJ;
    // J is then whole on the device for the solve
    constexpr int NCH = 16;
    hb_jac_layout staged;
    staged.csz = staged.stride = ((n + NCH - 1) / NCH + 63) & ~63LL;
    staged.nch = staged.slots = (int)((n + staged.csz - 1) / staged.csz);
    staged.base = k->hJ;
    staged.ld = n;
    staged.Jc = Jc_host;
    staged.Jd = Jd_host;
    std::swap(k->jl, staged);
    const int rc = do_condense_async(k);
    std::swap(k->jl, staged);
    HB_CHECK(rc);
    HB_CHECK(condense_check(k));
  }
  HB_CHECK(hb_lowrank_solve_compressed(k, k->hbuf[8], k->hbuf[9], k->hbuf[10], k->hbuf[11], k->hbuf[12], k->hbuf[13]));
  HB_CHECK(condense_check(k));
  if(n) HB_CUDA(cudaMemcpyAsync(dx, k->hbuf[11], sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
  if(meq) HB_CUDA(cudaMemcpyAsync(dyc, k->hbuf[12], sizeof(double) * meq, cudaMemcpyDeviceToHost, c->stream));
  if(mi) HB_CUDA(cudaMemcpyAsync(dyd, k->hbuf[13], sizeof(double) * mi, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}

// ---- public gemv (hiopMatrixDenseRowMajor::timesVec / transTimesVec) ----------------------------------------------------
extern "C" int hb_mat_times_vec(hb_ctx* c, int m, long long n, const double* A, long long lda, double beta, double* y, double alpha, const double* x)
{
  HB_REQUIRE(c && m >= 0 && n >= 0 && lda >= n, "hb_mat_times_vec: bad arguments");
  if(m == 0) return HB_OK;
  const int nchunks = (int)((n + GR_CHUNK - 1) / GR_CHUNK);
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (size_t)(nchunks > 0 ? nchunks : 1) * m));
  HB_CHECK(gemv_rows_partial(c, m, n, A, lda, x, (double*)c->ws));
  return gemv_rows_final(c, m, n, (const double*)c->ws, beta, y, alpha);
}
extern "C" int hb_mat_trans_times_vec(hb_ctx* c, int m, long long n, const double* A, long long lda, double beta, double* y, double alpha,
                                      const double* x)
{
  HB_REQUIRE(c && m >= 0 && n >= 0 && lda >= n, "hb_mat_trans_times_vec: bad arguments");
  return gemv_cols_launch(c, gemv_cols_groups(c, m, n), m, n, A, lda, beta, y, alpha, x);
}
