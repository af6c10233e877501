// Residual of the (log-barrier) KKT conditions on the device (SURVEY 8 f1, first piece of the vector pipeline around the KKT solve).
//
// Reference: hiopResidual::update   src/Optimization/hiopResidual.cpp:154-368  (≈ 60 hiopVector calls + 20 norms)
//            linear damping terms   src/Optimization/hiopLogBarProblem.hpp:135-145, hiopIterate.cpp:568-588,
//                                   hiopVectorPar::addLinearDampingTerm src/LinAlg/hiopVectorPar.cpp:927-944
// Here: one J^T [yc; yd] pass, ONE fused elementwise kernel per primal block (x-side, d-side) that writes its five residual blocks
// and accumulates the six norms it feeds, one small kernel for the constraint rows, a fixed-order second reduction stage.
// Elementwise results are bit-identical to the reference (same operation order, no FMA contraction).
#include "hb_lowrank.cuh"
#include "../../include/hiopb200.h"
#include <cmath>

namespace {

constexpr int ET = 256;
constexpr int NP = 6; // per-block partials: max|r0|, sum|r0|, max|r|, sum|r|, max complem (nlp), max complem (barrier)
const std::initializer_list<hb_op> NORM_OPS = {HB_MAX, HB_SUM, HB_MAX, HB_SUM, HB_MAX, HB_MAX};

// XSIDE: r0 = (t - zl) + zu with t = grad + J^T y (already in r_opt), damping beta = +1, then negated     hiopResidual.cpp:176-190
// else : r0 = (yd + vl) - vu,                                           damping beta = -1, not negated   :192-201
// bound rows: rl = il ? (p - sl) - lo : 0;  ru = iu ? (XSIDE ? (up - p) - su : (up - su) - p) : 0         :239-278
// complementarity: rz = i ? -(s z) [+ mu] : 0                                                             :285-345
// 4 CTAs per SM (at most 64 registers): without the bound the six block reductions push the kernel past 64 registers and 3 CTAs
template <bool XSIDE>
__global__ void __launch_bounds__(ET, 4)
k_resid_block(long long n, const double* tin /* may alias r_opt */, const double* __restrict__ p, const double* __restrict__ sl, const double* __restrict__ su,
              const double* __restrict__ zl, const double* __restrict__ zu, const double* __restrict__ il, const double* __restrict__ iu,
              const double* __restrict__ lo, const double* __restrict__ up, double mu, double ct, bool damp, double* r_opt,
              double* __restrict__ rl, double* __restrict__ ru, double* __restrict__ rzl, double* __restrict__ rzu, double* __restrict__ partial)
{
  __shared__ double sm[ET / 32];
  double m0 = 0.0, s0 = 0.0, m1 = 0.0, s1 = 0.0, c0 = 0.0, c1 = 0.0;
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double l = il[i], u = iu[i], zlo = zl[i], zup = zu[i], pp = p[i], slo = sl[i], sup = su[i];
    double r0 = XSIDE ? __dadd_rn(__dsub_rn(tin[i], zlo), zup) : __dsub_rn(__dadd_rn(tin[i], zlo), zup);
    m0 = fmax(m0, fabs(r0));
    s0 += fabs(r0);
    if(damp) r0 = __dadd_rn(__dmul_rn(1.0, r0), __dmul_rn(ct, __dsub_rn(l, u)));
    if(XSIDE) r0 = -r0;
    m1 = fmax(m1, fabs(r0));
    s1 += fabs(r0);
    r_opt[i] = r0;
    rl[i] = l == 0.0 ? 0.0 : __dsub_rn(__dsub_rn(pp, slo), lo[i]);
    ru[i] = u == 0.0 ? 0.0 : (XSIDE ? __dsub_rn(__dsub_rn(up[i], pp), sup) : __dsub_rn(__dsub_rn(up[i], sup), pp));
    double a = l == 0.0 ? 0.0 : __dsub_rn(0.0, __dmul_rn(slo, zlo));
    double b = u == 0.0 ? 0.0 : __dsub_rn(0.0, __dmul_rn(sup, zup));
    c0 = fmax(c0, fmax(fabs(a), fabs(b)));
    if(l == 1.0) a = __dadd_rn(a, mu);
    if(u == 1.0) b = __dadd_rn(b, mu);
    c1 = fmax(c1, fmax(fabs(a), fabs(b)));
    rzl[i] = a;
    rzu[i] = b;
  }
  double v;
  v = hb_block_reduce<HB_MAX, ET>(m0, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 0] = v;
  v = hb_block_sum<ET>(s0, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 1] = v;
  v = hb_block_reduce<HB_MAX, ET>(m1, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 2] = v;
  v = hb_block_sum<ET>(s1, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 3] = v;
  v = hb_block_reduce<HB_MAX, ET>(c0, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 4] = v;
  v = hb_block_reduce<HB_MAX, ET>(c1, sm); if(threadIdx.x == 0) partial[(size_t)blockIdx.x * NP + 5] = v;
}

// constraint rows (one CTA): ryc = crhs - c, ryd = d_it - d; out = {max|ryc|, sum|ryc|, max|ryd|, sum|ryd|, viol_dl, viol_du}   :203-237
__global__ void __launch_bounds__(ET)
k_resid_cons(int me, int mi, const double* __restrict__ crhs, const double* __restrict__ cv, const double* __restrict__ dit, const double* __restrict__ dv,
             const double* __restrict__ dl, const double* __restrict__ du, const double* __restrict__ idl, const double* __restrict__ idu,
             double* __restrict__ ryc, double* __restrict__ ryd, double* __restrict__ out)
{
  __shared__ double sm[ET / 32];
  double mc = 0.0, sc = 0.0, md = 0.0, sd = 0.0, vl = 0.0, vu = 0.0;
  for(int i = threadIdx.x; i < me; i += ET) {
    const double r = __dsub_rn(crhs[i], cv[i]);
    ryc[i] = r;
    mc = fmax(mc, fabs(r));
    sc += fabs(r);
  }
  for(int i = threadIdx.x; i < mi; i += ET) {
    const double r = __dsub_rn(dit[i], dv[i]);
    ryd[i] = r;
    md = fmax(md, fabs(r));
    sd += fabs(r);
    if(idl[i] == 1.0) vl = fmax(vl, -__dsub_rn(dv[i], dl[i])); // -(min over pattern of d - dl) when negative
    if(idu[i] == 1.0) vu = fmax(vu, -__dsub_rn(du[i], dv[i]));
  }
  double v;
  v = hb_block_reduce<HB_MAX, ET>(mc, sm); if(threadIdx.x == 0) out[0] = v;
  v = hb_block_sum<ET>(sc, sm); if(threadIdx.x == 0) out[1] = v;
  v = hb_block_reduce<HB_MAX, ET>(md, sm); if(threadIdx.x == 0) out[2] = v;
  v = hb_block_sum<ET>(sd, sm); if(threadIdx.x == 0) out[3] = v;
  v = hb_block_reduce<HB_MAX, ET>(vl, sm); if(threadIdx.x == 0) out[4] = v;
  v = hb_block_reduce<HB_MAX, ET>(vu, sm); if(threadIdx.x == 0) out[5] = v;
}
} // namespace

extern "C" int hb_lowrank_residual_update(hb_lowrank* k, const double* const* it, const double* cvals, const double* dvals, const double* grad_f,
                                          double mu, double kappa_d, const double* xl, const double* xu, const double* dl, const double* du,
                                          const double* crhs, double* const* res, double* norms_host)
{
  HB_REQUIRE(k && it && res && norms_host, "hb_lowrank_residual_update: null argument");
  HB_REQUIRE(k->n == 0 || k->ixl, "hb_lowrank_residual_update: patterns not set");
  HB_REQUIRE(jac_set(k), "hb_lowrank_residual_update: register the Jacobian with hb_lowrank_set_jacobian first");
  enum { X, D, YC, YD, SXL, SXU, SDL, SDU, ZL, ZU, VL, VU };
  enum { RX, RD, RYC, RYD, RXL, RXU, RDL, RDU, RSZL, RSZU, RSVL, RSVU };
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int me = k->meq, mi = k->mineq, m = k->m;
  const double ct = kappa_d * mu * 1.0;
  const int gx = hb_grid(c, n, ET), gd = hb_grid(c, mi, ET);
  // workspace: partials of the two blocks, 6 + 6 + 6 results, stacked multipliers
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * ((size_t)(gx + gd) * NP + 18 + (size_t)m + 8)));
  double* px = (double*)c->ws;
  double* pd = px + gx * NP;
  double* outx = pd + (size_t)gd * NP;
  double* outd = outx + 6;
  double* outc = outd + 6;
  double* ystk = outc + 6;
  HB_CUDA(cudaMemsetAsync(outx, 0, sizeof(double) * 18, c->stream));
  if(n > 0) {
    // rx <- grad_f + Jc^T yc + Jd^T yd                                                          :176-178
    HB_CUDA(cudaMemcpyAsync(res[RX], grad_f, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
    if(m > 0) {
      HB_CHECK(hb_stack(c, me, it[YC], mi, it[YD], ystk));
      HB_CHECK(jac_cols(k, 1.0, res[RX], 1.0, ystk));
    }
    k_resid_block<true><<<gx, ET, 0, c->stream>>>(n, res[RX], it[X], it[SXL], it[SXU], it[ZL], it[ZU], k->ixl, k->ixu, xl, xu, mu, ct, kappa_d > 0.0,
                                                       res[RX], res[RXL], res[RXU], res[RSZL], res[RSZU], px);
    HB_LAUNCHED();
    HB_CHECK(hb_reduce_slots(c, gx, px, outx, NORM_OPS));
  }
  if(c->nranks > 1) { // x-side blocks are sharded: combine the partial norms (d-side and constraint rows are replicated)
    // layout outx = {max, sum, max, sum, max, max}: reduce sums and maxima separately
    double* tmp = ystk + m;
    HB_CUDA(cudaMemcpyAsync(tmp, outx, sizeof(double) * 6, cudaMemcpyDeviceToDevice, c->stream));
    HB_CHECK(hb_allreduce_op(c, outx, 6, HB_MAX)); // max of everything ...
    HB_CHECK(hb_allreduce_op(c, tmp, 6, HB_SUM));  // ... and sum of everything; pick per slot below
    HB_CUDA(cudaMemcpyAsync(outx + 1, tmp + 1, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    HB_CUDA(cudaMemcpyAsync(outx + 3, tmp + 3, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  }
  if(mi > 0) {
    k_resid_block<false><<<gd, ET, 0, c->stream>>>(mi, it[YD], it[D], it[SDL], it[SDU], it[VL], it[VU], k->idl, k->idu, dl, du, mu, -ct, kappa_d > 0.0,
                                                   res[RD], res[RDL], res[RDU], res[RSVL], res[RSVU], pd);
    HB_LAUNCHED();
    HB_CHECK(hb_reduce_slots(c, gd, pd, outd, NORM_OPS));
  }
  if(m > 0) {
    k_resid_cons<<<1, ET, 0, c->stream>>>(me, mi, crhs, cvals, it[D], dvals, dl, du, k->idl, k->idu, res[RYC], res[RYD], outc);
    HB_LAUNCHED();
  }
  double h[18];
  HB_CUDA(cudaMemcpyAsync(h, outx, sizeof(double) * 18, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  const double *hx = h, *hd = h + 6, *hc = h + 12;
  norms_host[0] = fmax(hx[0], hd[0]);                 // nrmInf_nlp_optim
  norms_host[1] = fmax(hc[0], hc[2]);                 // nrmInf_nlp_feasib
  norms_host[2] = fmax(hx[4], hd[4]);                 // nrmInf_nlp_complem
  norms_host[3] = fmax(hx[2], hd[2]);                 // nrmInf_bar_optim
  norms_host[4] = norms_host[1];                      // nrmInf_bar_feasib                        :281
  norms_host[5] = fmax(hx[5], hd[5]);                 // nrmInf_bar_complem
  norms_host[6] = hc[1] + hc[3];                      // nrmOne_nlp_feasib
  norms_host[7] = norms_host[6];                      // nrmOne_bar_feasib
  norms_host[8] = hx[1] + hd[1];                      // nrmOne_nlp_optim
  norms_host[9] = hx[3] + hd[3];                      // nrmOne_bar_optim
  norms_host[10] = fmax(hc[0], fmax(hc[4], hc[5]));   // nrmInf_cons_violation                    :210-226
  return HB_OK;
}
