// hiopIterate / hiopLogBarProblem vector pipeline on the device (SURVEY 8 f1, second piece): the line-search side of one IPM iteration.
//
// Reference: hiopIterate::fractionToTheBdry                      src/Optimization/hiopIterate.cpp:326-363   (8 reductions + 1 all-reduce)
//            hiopIterate::takeStep_primals / takeStep_duals                                    :366-390   (16 vector calls)
//            hiopIterate::evalLogBarrier, addLogBarGrad_x/_d, linearDampingTerm, addLinearDampingTermToGrad_x/_d  :522-588
//            hiopLogBarProblem::updateWithNlpInfo / updateWithNlpInfo_trial_funcOnly  src/Optimization/hiopLogBarProblem.hpp:83-132
//            hiopVectorPar::fractionToTheBdry_w_pattern_local :1038-1061, logBarrier_local :863-881, linearDampingTerm_local :907-925
// One fused kernel per primal block (x-side over n_local, d-side over m_ineq) and call; scalars come back after a fixed-order second
// stage. Elementwise results (gradients, steps) are bit-identical to the reference; sums agree to rounding (the reference uses Kahan
// summation for the barrier, here a fixed-order tree).
#include "hb_lowrank.cuh"
#include "../../include/hiopb200.h"
#include <cmath>

namespace {

constexpr int ET = 256;
enum { X, D, YC, YD, SXL, SXU, SDL, SDU, ZL, ZU, VL, VU };

__device__ __forceinline__ double ftb(double x, double dx, double sel, double tau) // hiopVectorPar.cpp:1038-1061
{
  return (dx >= 0 || sel == 0.0) ? 1.0 : fmin(1.0, -tau * x / dx);
}

// partial[b] = {min over the block's slacks (primal step), min over its bound duals (dual step)}
__global__ void __launch_bounds__(ET)
k_ftb_block(long long n, double tau, const double* __restrict__ sl, const double* __restrict__ dsl, const double* __restrict__ su,
            const double* __restrict__ dsu, const double* __restrict__ zl, const double* __restrict__ dzl, const double* __restrict__ zu,
            const double* __restrict__ dzu, const double* __restrict__ il, const double* __restrict__ iu, double* __restrict__ partial)
{
  __shared__ double sm[ET / 32];
  double ap = 1.0, ad = 1.0;
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double l = il[i], u = iu[i];
    ap = fmin(ap, fmin(ftb(sl[i], dsl[i], l, tau), ftb(su[i], dsu[i], u, tau)));
    ad = fmin(ad, fmin(ftb(zl[i], dzl[i], l, tau), ftb(zu[i], dzu[i], u, tau)));
  }
  double v = hb_block_reduce<HB_MIN, ET>(ap, sm);
  if(threadIdx.x == 0) partial[2 * blockIdx.x] = v;
  v = hb_block_reduce<HB_MIN, ET>(ad, sm);
  if(threadIdx.x == 0) partial[2 * blockIdx.x + 1] = v;
}

// log-barrier pieces of one primal block: partial[b] = {sum log(sl)|il + sum log(su)|iu, sum sl|(il & !iu) + sum su|(iu & !il)};
// optionally the gradient g = ((g0 - mu/sl|il) + mu/su|iu) [then 1*g + ct (il - iu)]   hiopIterate.cpp:539-551, 568-588
__global__ void __launch_bounds__(ET)
k_logbar_block(long long n, const double* __restrict__ sl, const double* __restrict__ su, const double* __restrict__ il, const double* __restrict__ iu,
               double mu, double ct, bool damp, const double* __restrict__ g0 /* NULL = 0 */, double* __restrict__ g /* NULL: function only */,
               double* __restrict__ partial)
{
  __shared__ double sm[ET / 32];
  double bl = 0.0, dt = 0.0;
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double l = il[i], u = iu[i], a = sl[i], b = su[i];
    if(l != 0.0) bl += log(a);
    if(u != 0.0) bl += log(b);
    if(l == 1.0 && u == 0.0) dt += a;
    if(u == 1.0 && l == 0.0) dt += b;
    if(g) {
      double v = g0 ? g0[i] : 0.0;
      if(l == 1.0) v = __dadd_rn(v, __ddiv_rn(-mu, a));
      if(u == 1.0) v = __dadd_rn(v, __ddiv_rn(mu, b));
      if(damp) v = __dadd_rn(__dmul_rn(1.0, v), __dmul_rn(ct, __dsub_rn(l, u)));
      g[i] = v;
    }
  }
  double v = hb_block_sum<ET>(bl, sm);
  if(threadIdx.x == 0) partial[2 * blockIdx.x] = v;
  v = hb_block_sum<ET>(dt, sm);
  if(threadIdx.x == 0) partial[2 * blockIdx.x + 1] = v;
}

// out = a + alpha * d (copyFrom + axpy), for up to 6 blocks in one launch
struct StepArgs
{
  const double* a[6];
  const double* d[6];
  double* out[6];
  long long len[6];
  double alpha[6];
  int count;
};
__global__ void __launch_bounds__(ET)
k_take_step(StepArgs A)
{
  for(int q = 0; q < A.count; q++) {
    const long long stride = (long long)gridDim.x * ET;
    for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < A.len[q]; i += stride)
      A.out[q][i] = __dadd_rn(A.a[q][i], __dmul_rn(A.alpha[q], A.d[q][i]));
  }
}

// hiopVectorPar::adjustDuals_plh (src/LinAlg/hiopVectorPar.cpp:1117-1148): keep z within [mu/(kappa s), kappa mu/s] on the pattern
__device__ __forceinline__ double adjust_plh(double z, double s, double sel, double mu, double kappa)
{
  if(sel != 1.0) return z;
  double a = __ddiv_rn(mu, s);
  const double b = __ddiv_rn(a, kappa);
  a = __dmul_rn(a, kappa);
  if(z < b) return b;
  if(a <= b) return b;
  return a < z ? a : z;
}
__global__ void __launch_bounds__(ET)
k_adjust_duals(long long n, double mu, double kappa, const double* __restrict__ sl, const double* __restrict__ su, const double* __restrict__ il,
               const double* __restrict__ iu, double* __restrict__ zl, double* __restrict__ zu)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    zl[i] = adjust_plh(zl[i], sl[i], il[i], mu, kappa);
    zu[i] = adjust_plh(zu[i], su[i], iu[i], mu, kappa);
  }
}

// hiopIterate::adjust_small_slacks for one slack block (hiopIterate.cpp:413-479), the reference's chain of ~20 vector calls per element,
// same operations in the same order (bit-identical); cnt counts the entries whose shifted slack was negative (numOfElemsLessThan).
__global__ void __launch_bounds__(ET)
k_adjust_small_slack(long long n, double mu, double small_val, double scale_fact, const double* __restrict__ bound, const double* __restrict__ dual,
                     const double* __restrict__ sel, double* __restrict__ slack, int* __restrict__ cnt)
{
  int local = 0;
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double s = slack[i];
    const bool on = sel[i] == 1.0;
    double a1 = s;
    if(on) a1 = __dadd_rn(a1, -small_val);
    if(a1 > 0.0) a1 = 0.0;
    if(a1 < 0.0) local++;
    a1 = __dmul_rn((double)((0.0 < a1) - (a1 < 0.0)), -1.0);
    const double s0 = s < 0.0 ? 0.0 : s;
    double a2 = on ? __ddiv_rn(mu, dual[i]) : 0.0;
    const double a3 = on ? small_val : 0.0;
    if(a2 < a3) a2 = a3;
    a2 = __dadd_rn(a2, __dmul_rn(-1.0, s0));
    a1 = __dmul_rn(a1, a2);
    a1 = __dadd_rn(a1, __dmul_rn(1.0, s0));
    double b2 = on ? 1.0 : 0.0;
    const double b3 = fabs(bound[i]);
    if(b2 < b3) b2 = b3;
    b2 = __dmul_rn(b2, scale_fact);
    b2 = __dadd_rn(b2, __dmul_rn(1.0, s0));
    if(a1 > b2) a1 = b2;
    slack[i] = a1;
  }
  if(local) atomicAdd(cnt, local);
}

} // namespace

extern "C" int hb_iterate_fraction_to_bdry(hb_lowrank* k, const double* const* it, const double* const* dir, double tau, double* alpha_primal,
                                           double* alpha_dual)
{
  HB_REQUIRE(k && it && dir && alpha_primal && alpha_dual, "hb_iterate_fraction_to_bdry: null argument");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_iterate_fraction_to_bdry: patterns not set");
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int mi = k->mineq;
  const int gx = hb_grid(c, n, ET), gd = hb_grid(c, mi, ET);
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (2 * (size_t)(gx + gd) + 4)));
  double* px = (double*)c->ws;
  double* pd = px + 2 * (size_t)gx;
  double* out = pd + 2 * (size_t)gd; // {x primal, x dual, d primal, d dual}
  k_ftb_block<<<gx, ET, 0, c->stream>>>(n, tau, it[SXL], dir[SXL], it[SXU], dir[SXU], it[ZL], dir[ZL], it[ZU], dir[ZU], k->ixl, k->ixu, px);
  HB_LAUNCHED();
  HB_CHECK(hb_reduce_slots(c, gx, px, out, {HB_MIN, HB_MIN}));
  if(c->nranks > 1) HB_CHECK(hb_allreduce_op(c, out, 2, HB_MIN)); // x-side blocks are sharded: MPI_MIN of the reference (:356-360)
  k_ftb_block<<<gd, ET, 0, c->stream>>>(mi, tau, it[SDL], dir[SDL], it[SDU], dir[SDU], it[VL], dir[VL], it[VU], dir[VU], k->idl, k->idu, pd);
  HB_LAUNCHED();
  HB_CHECK(hb_reduce_slots(c, gd, pd, out + 2, {HB_MIN, HB_MIN}));
  double h[4];
  HB_CUDA(cudaMemcpyAsync(h, out, sizeof(double) * 4, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  *alpha_primal = fmin(10.0, fmin(h[0], h[2])); // the reference starts from 10 (:329); every term is <= 1
  *alpha_dual = fmin(10.0, fmin(h[1], h[3]));
  return HB_OK;
}

extern "C" int hb_iterate_take_step(hb_lowrank* k, const double* const* it, const double* const* dir, double alpha_primal, double alpha_dual,
                                    int which /* 1 = primals (x, d), 2 = duals (yc, yd, zl, zu, vl, vu), 3 = both */, double* const* out)
{
  HB_REQUIRE(k && it && dir && out, "hb_iterate_take_step: null argument");
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int me = k->meq, mi = k->mineq;
  auto launch = [&](const int* ids, const double* al, int cnt) -> int {
    StepArgs A;
    A.count = 0;
    long long mx = 1;
    for(int q = 0; q < cnt; q++) {
      const int b = ids[q];
      const long long len = (b == X || b == ZL || b == ZU) ? n : (b == YC ? me : mi);
      if(len == 0) continue;
      A.a[A.count] = it[b]; A.d[A.count] = dir[b]; A.out[A.count] = out[b]; A.len[A.count] = len; A.alpha[A.count] = al[q];
      A.count++;
      if(len > mx) mx = len;
    }
    if(A.count == 0) return HB_OK;
    k_take_step<<<hb_grid(c, mx, ET), ET, 0, c->stream>>>(A);
    HB_LAUNCHED();
    return HB_OK;
  };
  if(which & 1) { // takeStep_primals :366-372
    const int ids[2] = {X, D};
    const double al[2] = {alpha_primal, alpha_primal};
    HB_CHECK(launch(ids, al, 2));
  }
  if(which & 2) { // takeStep_duals :374-390 (yc, yd move with the PRIMAL step length)
    const int ids[6] = {YD, YC, ZL, ZU, VL, VU};
    const double al[6] = {alpha_primal, alpha_primal, alpha_dual, alpha_dual, alpha_dual, alpha_dual};
    HB_CHECK(launch(ids, al, 6));
  }
  return HB_OK;
}

extern "C" int hb_iterate_adjust_duals_plh(hb_lowrank* k, double* const* it, double mu, double kappa_sigma)
{
  HB_REQUIRE(k && it, "hb_iterate_adjust_duals_plh: null argument");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_iterate_adjust_duals_plh: patterns not set");
  hb_ctx* c = k->ctx;
  if(k->n > 0) {
    k_adjust_duals<<<hb_grid(c, k->n, ET), ET, 0, c->stream>>>(k->n, mu, kappa_sigma, it[SXL], it[SXU], k->ixl, k->ixu, it[ZL], it[ZU]);
    HB_LAUNCHED();
  }
  if(k->mineq > 0) {
    k_adjust_duals<<<hb_grid(c, k->mineq, ET), ET, 0, c->stream>>>(k->mineq, mu, kappa_sigma, it[SDL], it[SDU], k->idl, k->idu, it[VL], it[VU]);
    HB_LAUNCHED();
  }
  return HB_OK;
}

extern "C" int hb_iterate_adjust_small_slacks(hb_lowrank* k, double* const* it, const double* const* it_curr, double mu, const double* xl,
                                              const double* xu, const double* dl, const double* du, int* num_adjusted)
{
  HB_REQUIRE(k && it && it_curr, "hb_iterate_adjust_small_slacks: null argument");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_iterate_adjust_small_slacks: patterns not set");
  hb_ctx* c = k->ctx;
  const double eps = 2.220446049250313e-16;
  const double small_val = eps * fmin(1.0, mu);
  const double scale_fact = pow(eps, 0.75);
  HB_CHECK(hb_ws_reserve(c, 64));
  int* cnt = (int*)c->ws.get();
  HB_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int), c->stream));
  struct Blk { int s, z; const double* bound; const double* sel; long long len; };
  const Blk blks[4] = {{SXL, ZL, xl, k->ixl, k->n}, {SXU, ZU, xu, k->ixu, k->n}, {SDL, VL, dl, k->idl, (long long)k->mineq},
                       {SDU, VU, du, k->idu, (long long)k->mineq}};
  for(const Blk& b : blks) {
    if(b.len == 0) continue;
    double smin = 0.0;
    HB_CHECK(hb_vec_min_w_pattern(c, b.len, it[b.s], b.sel, &smin)); // slack.min_w_pattern(select) :432
    if(!(smin < small_val)) continue;
    k_adjust_small_slack<<<hb_grid(c, b.len, ET), ET, 0, c->stream>>>(b.len, mu, small_val, scale_fact, b.bound, it_curr[b.z], b.sel, it[b.s], cnt);
    HB_LAUNCHED();
  }
  int h = 0;
  HB_CUDA(cudaMemcpyAsync(&h, cnt, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if(num_adjusted) *num_adjusted = h;
  return HB_OK;
}

extern "C" int hb_iterate_logbar(hb_lowrank* k, const double* const* it, double f, double mu, double kappa_d, const double* grad_f, double* grad_x_logbar,
                                 double* grad_d_logbar, double* f_logbar)
{
  HB_REQUIRE(k && it && f_logbar, "hb_iterate_logbar: null argument");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_iterate_logbar: patterns not set");
  HB_REQUIRE((grad_x_logbar == nullptr) == (grad_d_logbar == nullptr) || k->mineq == 0 || k->n == 0, "hb_iterate_logbar: pass both gradients or none");
  HB_REQUIRE(!grad_x_logbar || grad_f || k->n == 0, "hb_iterate_logbar: grad_f needed for the gradient");
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int mi = k->mineq;
  const int gx = hb_grid(c, n, ET), gd = hb_grid(c, mi, ET);
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (2 * (size_t)(gx + gd) + 4)));
  double* px = (double*)c->ws;
  double* pd = px + 2 * (size_t)gx;
  double* out = pd + 2 * (size_t)gd;
  const double ct = kappa_d * mu * 1.0;
  const bool damp = kappa_d > 0.0;
  k_logbar_block<<<gx, ET, 0, c->stream>>>(n, it[SXL], it[SXU], k->ixl, k->ixu, mu, ct, damp, grad_f, grad_x_logbar, px);
  HB_LAUNCHED();
  HB_CHECK(hb_reduce_slots(c, gx, px, out, {HB_SUM, HB_SUM}));
  if(c->nranks > 1) HB_CHECK(hb_allreduce_op(c, out, 2, HB_SUM)); // :529-533, :561-565
  k_logbar_block<<<gd, ET, 0, c->stream>>>(mi, it[SDL], it[SDU], k->idl, k->idu, mu, ct, damp, nullptr, grad_d_logbar, pd);
  HB_LAUNCHED();
  HB_CHECK(hb_reduce_slots(c, gd, pd, out + 2, {HB_SUM, HB_SUM}));
  double h[4];
  HB_CUDA(cudaMemcpyAsync(h, out, sizeof(double) * 4, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  const double barrier = h[0] + h[2];
  double fl = f + (-mu * barrier); // hiopLogBarProblem.hpp:95-96
  if(damp) {
    double tx = h[1]; tx *= mu; tx *= kappa_d;
    double td = h[3]; td *= mu; td *= kappa_d;
    fl += tx + td; // :107
  }
  *f_logbar = fl;
  return HB_OK;
}
