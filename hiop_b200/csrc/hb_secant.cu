// Secant-memory bookkeeping of the quasi-Newton Hessian on the device (SURVEY 8 a11).
//
// Reference: hiopHessianLowRank::update   src/Optimization/hiopHessianLowRank.cpp:262-388
//            growL / growD / updateL / updateD                                      :779-867
//            hiopMatrixDenseRowMajor::appendRow / shiftRows / replaceRow  src/LinAlg/hiopMatrixDenseRowMajor.cpp:129-137, 238-284
//
// The reference keeps x_prev, grad_f_prev and BOTH previous Jacobians on the host, runs four J^T gemvs (32 GB of traffic at
// n=1e6, m=1000) and then copies the two Jacobians (16 GB more). Here the secant pair is formed with one fused pass:
//   y += (J - J_prev)^T [yc; yd]   while   J_prev <- J                (24 GB: read J, read + write J_prev)
// and S_t, Y_t live in HBM, so nothing but the l x l matrix L, the vector D and sigma ever crosses PCIe.
#include "hb_lowrank.cuh"
#include "../../include/hiopb200.h"
#include <cmath>
#include <limits>
#include <cstring>

namespace {

constexpr int ET = 256;
constexpr int GC_ROWS = 512;

// y[c] += sum_i (J[i][c] - Jp[i][c]) * w[i];   Jp[i][c] = J[i][c]
__global__ void __launch_bounds__(ET)
k_gemv_cols_diff_store(int m, long long n, const double* __restrict__ J, double* __restrict__ Jp, const double* __restrict__ w, double* __restrict__ y)
{
  __shared__ double sw[GC_ROWS];
  const bool vec = ((n & 1) == 0) && ((reinterpret_cast<uintptr_t>(J) & 15u) == 0) && ((reinterpret_cast<uintptr_t>(Jp) & 15u) == 0);
  const long long k = ((long long)blockIdx.x * ET + threadIdx.x) * 2;
  double a0 = 0.0, a1 = 0.0;
  for(int i0 = 0; i0 < m; i0 += GC_ROWS) {
    const int nr = min(GC_ROWS, m - i0);
    __syncthreads();
    for(int i = threadIdx.x; i < nr; i += ET) sw[i] = w[i0 + i];
    __syncthreads();
    if(k < n) {
      const size_t base = (size_t)i0 * n + k;
      if(vec && k + 1 < n) {
#pragma unroll 4
        for(int i = 0; i < nr; i++) {
          const double2 v = *reinterpret_cast<const double2*>(J + base + (size_t)i * n);
          const double2 p = *reinterpret_cast<const double2*>(Jp + base + (size_t)i * n);
          a0 += (v.x - p.x) * sw[i];
          a1 += (v.y - p.y) * sw[i];
          *reinterpret_cast<double2*>(Jp + base + (size_t)i * n) = v;
        }
      } else {
        for(int i = 0; i < nr; i++) {
          const double v0 = J[base + (size_t)i * n];
          a0 += (v0 - Jp[base + (size_t)i * n]) * sw[i];
          Jp[base + (size_t)i * n] = v0;
          if(k + 1 < n) {
            const double v1 = J[base + (size_t)i * n + 1];
            a1 += (v1 - Jp[base + (size_t)i * n + 1]) * sw[i];
            Jp[base + (size_t)i * n + 1] = v1;
          }
        }
      }
    }
  }
  if(k < n) {
    y[k] += a0;
    if(k + 1 < n) y[k + 1] += a1;
  }
}

// s = x - x_prev, y = g - g_prev (same single rounding as copyFrom + axpy(-1) in the reference)
__global__ void __launch_bounds__(ET)
k_secant_pair(long long n, const double* __restrict__ x, const double* __restrict__ xp, const double* __restrict__ g, const double* __restrict__ gp,
              double* __restrict__ s, double* __restrict__ y)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    s[i] = __dsub_rn(x[i], xp[i]);
    y[i] = __dsub_rn(g[i], gp[i]);
  }
}

int install(hb_lowrank* k)
{
  const int l = k->sec_lcurr > 0 ? k->sec_lcurr : 0;
  // sigma changes DhInv and the cached condensation; hb_lowrank_set_secant invalidates both and recomputes S S^T
  return hb_lowrank_set_secant(k, l, k->sigma, k->sec_S, k->sec_Y, k->sec_L, k->sec_D);
}

} // namespace

extern "C" int hb_lowrank_secant_reset(hb_lowrank* k, double sigma0, int sigma_strategy)
{
  HB_REQUIRE(k, "null handle");
  HB_REQUIRE(sigma_strategy >= 1 && sigma_strategy <= 5, "hb_lowrank_secant_reset: sigma strategy must be 1..5");
  HB_REQUIRE(k->lmax <= 64, "hb_lowrank_secant_reset: secant_memory_len > 64 is not supported by the device-side bookkeeping");
  k->sec_lcurr = -1;
  k->sec_strategy = sigma_strategy;
  k->sec_sigma0 = sigma0;
  k->sigma = sigma0;
  hb_ctx* c = k->ctx;
  HB_CHECK(k->sec_S.reserve(c, (size_t)k->lmax * k->n, "secant memory S"));
  HB_CHECK(k->sec_Y.reserve(c, (size_t)k->lmax * k->n, "secant memory Y"));
  HB_CHECK(k->sec_xprev.reserve(c, (size_t)k->n, "previous iterate"));
  HB_CHECK(k->sec_gprev.reserve(c, (size_t)k->n, "previous gradient"));
  return hb_lowrank_set_secant(k, 0, sigma0, k->sec_S, k->sec_Y, k->sec_L, k->sec_D);
}

extern "C" int hb_lowrank_secant_update(hb_lowrank* k, const double* x, const double* grad_f, const double* yc, const double* yd,
                                        int jacobian_is_constant, int* status)
{
  HB_REQUIRE(k && (k->n == 0 || (x && grad_f)), "hb_lowrank_secant_update: null argument");
  HB_REQUIRE(k->sec_S, "hb_lowrank_secant_update: call hb_lowrank_secant_reset first");
  HB_REQUIRE(jac_set(k), "hb_lowrank_secant_update: register the current Jacobian with hb_lowrank_set_jacobian first");
  HB_REQUIRE((k->meq == 0 || yc) && (k->mineq == 0 || yd), "hb_lowrank_secant_update: null multiplier block");
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int m = k->m, lmax = k->lmax;
  const bool needJ = m > 0 && !jacobian_is_constant;
  const double* J = nullptr;
  if(needJ) HB_CHECK(jac_whole(k, "hb_lowrank_secant_update with jacobian_is_constant == 0 (J_prev is a device copy of J)", &J));
  int st = 0;
  if(needJ) HB_CHECK(k->sec_Jprev.reserve(c, (size_t)m * n, "previous Jacobian"));
  if(k->sec_lcurr < 0) {
    // first optimization iterate: only remember it                                     hiopHessianLowRank.cpp:372-381
    k->sec_lcurr = 0;
    if(needJ) HB_CUDA(cudaMemcpyAsync(k->sec_Jprev, J, sizeof(double) * (size_t)m * n, cudaMemcpyDeviceToDevice, c->stream));
  } else {
    double* s = k->nv1;
    double* y = k->nv2;
    if(n > 0) {
      k_secant_pair<<<hb_grid(c, n, ET), ET, 0, c->stream>>>(n, x, k->sec_xprev, grad_f, k->sec_gprev, s, y);
      HB_LAUNCHED();
    }
    if(needJ) {
      // y += (J - J_prev)^T [yc; yd], J_prev <- J in the same pass                       :291-297, 366-367
      HB_CHECK(hb_ws_reserve(c, sizeof(double) * (size_t)m));
      HB_CHECK(hb_stack(c, k->meq, yc, k->mineq, yd, (double*)c->ws));
      if(n > 0) {
        const long long pairs = (n + 1) / 2;
        k_gemv_cols_diff_store<<<(unsigned)((pairs + ET - 1) / ET), ET, 0, c->stream>>>(m, n, J, k->sec_Jprev, (const double*)c->ws, y);
        HB_LAUNCHED();
      }
    }
    double s_inf = 0.0;
    HB_CHECK(hb_vec_infnorm(c, n, s, &s_inf));
    const double eps = std::numeric_limits<double>::epsilon();
    if(s_inf >= 100 * eps) { // :284
      double sTy = 0.0, s_nrm2 = 0.0, y_nrm2 = 0.0;
      HB_CHECK(hb_vec_dot(c, n, s, y, &sTy));
      HB_CHECK(hb_vec_twonorm(c, n, s, &s_nrm2));
      HB_CHECK(hb_vec_twonorm(c, n, y, &y_nrm2));
      if(sTy > s_nrm2 * y_nrm2 * std::sqrt(eps)) { // :305
        st = 1;
        if(lmax > 0) {
          const int l = k->sec_lcurr;
          double yts[64];
          if(l > 0) { // Y^T s with the memory as it is before the new pair enters          :309-310
            HB_CHECK(multidot(k, nullptr, s, 1.0));
            HB_CUDA(cudaMemcpyAsync(yts, k->p2l + l, sizeof(double) * l, cudaMemcpyDeviceToHost, c->stream));
            HB_CUDA(cudaStreamSynchronize(c->stream));
          }
          if(l < lmax) {
            // appendRow + growL + growD                                                    :313-318, 779-823
            HB_CUDA(cudaMemcpyAsync(k->sec_S + (size_t)l * n, s, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
            HB_CUDA(cudaMemcpyAsync(k->sec_Y + (size_t)l * n, y, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
            double Ln[64 * 64];
            for(int i = 0; i < l; i++)
              for(int j = 0; j < l; j++) Ln[i * (l + 1) + j] = k->sec_L[i * l + j];
            for(int j = 0; j < l; j++) Ln[l * (l + 1) + j] = yts[j];
            for(int i = 0; i < l + 1; i++) Ln[i * (l + 1) + l] = 0.0;
            std::memcpy(k->sec_L, Ln, sizeof(double) * (l + 1) * (l + 1));
            k->sec_D[l] = sTy;
            k->sec_lcurr = l + 1;
          } else {
            // shiftRows(-1) + replaceRow(l-1) + updateL + updateD                           :320-327, 825-867
            for(int q = 0; q + 1 < l; q++) { // rows move one at a time: source and destination rows never overlap
              HB_CUDA(cudaMemcpyAsync(k->sec_S + (size_t)q * n, k->sec_S + (size_t)(q + 1) * n, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
              HB_CUDA(cudaMemcpyAsync(k->sec_Y + (size_t)q * n, k->sec_Y + (size_t)(q + 1) * n, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
            }
            HB_CUDA(cudaMemcpyAsync(k->sec_S + (size_t)(l - 1) * n, s, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
            HB_CUDA(cudaMemcpyAsync(k->sec_Y + (size_t)(l - 1) * n, y, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
            const int lm1 = l - 1;
            double* L = k->sec_L;
            for(int i = 1; i < lm1; i++)
              for(int j = 0; j < i; j++) L[i * l + j] = L[(i + 1) * l + j + 1];
            for(int j = 0; j < lm1; j++) L[lm1 * l + j] = yts[j + 1];
            L[lm1 * l + lm1] = 0.0;
            for(int i = 0; i < l - 1; i++) k->sec_D[i] = k->sec_D[i + 1];
            k->sec_D[l - 1] = sTy;
          }
        }
        double sg;
        switch(k->sec_strategy) { // :335-355
          case 1: sg = sTy / (s_nrm2 * s_nrm2); break;
          case 2: sg = y_nrm2 * y_nrm2 / sTy; break;
          case 3: sg = std::sqrt(s_nrm2 * s_nrm2 / y_nrm2 / y_nrm2); break;
          case 4: sg = 0.5 * (sTy / (s_nrm2 * s_nrm2) + y_nrm2 * y_nrm2 / sTy); break;
          default: sg = k->sec_sigma0; break;
        }
        k->sigma = std::fmax(std::fmin(1e+8, sg), 1e-8); // :357-358
      } else {
        st = 3;
      }
    } else {
      st = 2;
    }
    if(needJ && n == 0) { /* nothing to store */ }
  }
  // remember the iterate (J_prev was refreshed by the fused pass)                        :364-367
  if(n > 0) {
    HB_CUDA(cudaMemcpyAsync(k->sec_xprev, x, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(k->sec_gprev, grad_f, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
  }
  if(status) *status = st;
  if(st == 1 || st == 0) HB_CHECK(install(k));
  return HB_OK;
}

extern "C" int hb_lowrank_secant_state(hb_lowrank* k, int* l, double* sigma, const double** St, const double** Yt, double* L_host, double* D_host)
{
  HB_REQUIRE(k, "null handle");
  const int ll = k->sec_lcurr > 0 ? k->sec_lcurr : 0;
  if(l) *l = ll;
  if(sigma) *sigma = k->sigma;
  if(St) *St = k->sec_S;
  if(Yt) *Yt = k->sec_Y;
  if(L_host) std::memcpy(L_host, k->sec_L, sizeof(double) * ll * ll);
  if(D_host) std::memcpy(D_host, k->sec_D, sizeof(double) * ll);
  return HB_OK;
}
