// Outer iterative refinement of the quasi-Newton KKT step on device (SURVEY 8 a19 / f3).
//
// Reference: hiopKKTLinSys::compute_directions_w_IR  src/Optimization/hiopKKTLinSys.cpp:909-960
//            hiopBiCGStabSolver::solve               src/LinAlg/hiopKrylovSolver.cpp:399-700
//            hiopMatVecKKTFullOpr::times_vec         src/Optimization/hiopKKTLinSys.cpp:1619-1733   (operator, 12 x 12 blocks)
//            hiopPrecondKKTOpr::times_vec            src/Optimization/hiopKKTLinSys.cpp:1900-1909   (= computeDirections)
//            hiopVectorCompoundPD                    src/LinAlg/hiopVectorCompoundPD.cpp:99-255     (block order)
//
// The reference runs every compound-vector operation as 12 hiopVector calls and every KKT product as ~45 of them; here a
// compound vector is ONE contiguous buffer (n-sized blocks first, then the m-sized ones), so copy/axpy/scale/dot/norm are one
// kernel each and the operator is two fused elementwise kernels + one J pass per direction. Scalars of the recurrence come
// back to the host (the same branch structure as the reference decides convergence, stagnation and breakdown).
#include "hb_lowrank.cuh"
#include "../../include/hiopb200.h"
#include <cmath>
#include <limits>
#include <algorithm>

namespace {

constexpr int ET = 256;

// block ids in the reference's compound order (hiopVectorCompoundPD.cpp:228-255)
enum { PX, PD, PYC, PYD, PSXL, PSXU, PSDL, PSDU, PZL, PZU, PVL, PVU, NPART };

struct Layout
{
  long long off[NPART];
  long long len[NPART];
  long long n_span; // doubles covered by the n-sized blocks (sharded across ranks)
  long long total;  // whole compound vector
};

Layout make_layout(const hb_lowrank* k)
{
  Layout L;
  const long long n = k->n, mi = k->mineq, me = k->meq;
  const long long np = (n + 1) & ~1LL, mip = (mi + 1) & ~1LL, mep = (me + 1) & ~1LL; // 16-byte aligned blocks, pads stay 0
  const int order_n[5] = {PX, PSXL, PSXU, PZL, PZU};
  long long o = 0;
  for(int q : order_n) { L.off[q] = o; L.len[q] = n; o += np; }
  L.n_span = o;
  const int order_m[7] = {PD, PYC, PYD, PSDL, PSDU, PVL, PVU};
  for(int q : order_m) { L.off[q] = o; L.len[q] = (q == PYC) ? me : mi; o += (q == PYC) ? mep : mip; }
  L.total = o;
  return L;
}

// One primal block (x with its bound slacks/duals, or d with its): the rows of hiopMatVecKKTFullOpr::times_vec that are
// elementwise (hiopKKTLinSys.cpp:1672-1730), same operation order:
//   y0   = (y0 - dzl) + dzu                 y0 arrives holding H dx + J^T dy  (x block)  or  -dyd  (d block)
//   yrl  = ixl ? dsl - dp : 0               yru = ixu ? dsu + dp : 0
//   yrzl = sl*dzl + zl*dsl                  yrzu = su*dzu + zu*dsu
__global__ void __launch_bounds__(ET)
k_kkt_full_block(long long n, const double* __restrict__ dp, const double* __restrict__ dsl, const double* __restrict__ dsu,
                 const double* __restrict__ dzl, const double* __restrict__ dzu, const double* __restrict__ sl, const double* __restrict__ zl,
                 const double* __restrict__ su, const double* __restrict__ zu, const double* __restrict__ il, const double* __restrict__ iu,
                 double* __restrict__ y0, double* __restrict__ yrl, double* __restrict__ yru, double* __restrict__ yrzl, double* __restrict__ yrzu)
{
  const long long stride = (long long)gridDim.x * ET;
  for(long long i = (long long)blockIdx.x * ET + threadIdx.x; i < n; i += stride) {
    const double p = dp[i], a = dsl[i], b = dsu[i], zl_ = dzl[i], zu_ = dzu[i];
    y0[i] = __dadd_rn(__dsub_rn(y0[i], zl_), zu_);
    yrl[i] = il[i] == 0.0 ? 0.0 : __dsub_rn(a, p);
    yru[i] = iu[i] == 0.0 ? 0.0 : __dadd_rn(b, p);
    yrzl[i] = __dadd_rn(__dmul_rn(sl[i], zl_), __dmul_rn(zl[i], a));
    yrzu[i] = __dadd_rn(__dmul_rn(su[i], zu_), __dmul_rn(zu[i], b));
  }
}
__global__ void k_neg(int n, double* __restrict__ y, const double* __restrict__ x)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < n) y[i] = -x[i];
}
// yryc = (J dx)[0:me];  yryd = (J dx)[me:] - dd
__global__ void k_split_jdx(int me, int mi, const double* __restrict__ jdx, const double* __restrict__ dd, double* __restrict__ yryc,
                            double* __restrict__ yryd)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < me) yryc[i] = jdx[i];
  else if(i < me + mi) yryd[i - me] = __dsub_rn(jdx[i], dd[i - me]);
}

constexpr int KRY_EXTRA = 4 * 2048 + 64;

int ensure_ws(hb_lowrank* k, const Layout& L, int nvec)
{
  if(!k->kry) {
    HB_CHECK(k->kry.reserve(k->ctx, (size_t)L.total * nvec, "the BiCGStab workspace"));
    HB_CUDA(cudaMemsetAsync(k->kry, 0, sizeof(double) * (size_t)L.total * nvec, k->ctx->stream));
  }
  // 2 m-vectors + the device scalars and per-CTA partial sums of the recurrence (KRY_EXTRA doubles)
  return k->kry_m.reserve(k->ctx, (size_t)(2 * k->m + 2 + KRY_EXTRA), "the BiCGStab m-workspace");
}

// y = K x on compound buffers (y and x must not alias)
int full_times_vec(hb_lowrank* k, const Layout& L, double* y, const double* x)
{
  hb_ctx* c = k->ctx;
  const long long n = k->n;
  const int me = k->meq, mi = k->mineq, m = k->m;
  auto X = [&](int q) { return x + L.off[q]; };
  auto Y = [&](int q) { return y + L.off[q]; };
  double* dy = k->kry_m;      // [dyc; dyd] stacked
  double* jdx = k->kry_m + m; // J dx
  // rx = H dx + Jc^T dyc + Jd^T dyd - dzl + dzu                                         :1672-1678 (all deltas are 0: QN path)
  HB_CHECK(hb_lowrank_hess_times_vec(k, 0.0, Y(PX), 1.0, X(PX), 0));
  if(m > 0) {
    HB_CHECK(hb_stack(c, me, X(PYC), mi, X(PYD), dy));
    HB_CHECK(jac_cols(k, 1.0, Y(PX), 1.0, dy));
    // ryc = Jc dx; ryd = Jd dx - dd                                                      :1687-1694
    HB_CHECK(jac_rows(k, 0.0, jdx, 1.0, X(PX)));
    k_split_jdx<<<(m + 127) / 128, 128, 0, c->stream>>>(me, mi, jdx, X(PD), Y(PYC), Y(PYD));
    HB_LAUNCHED();
  }
  if(n > 0) {
    k_kkt_full_block<<<hb_grid(c, n, ET), ET, 0, c->stream>>>(n, X(PX), X(PSXL), X(PSXU), X(PZL), X(PZU), k->sxl, k->zl, k->sxu, k->zu, k->ixl, k->ixu, Y(PX),
                                                        Y(PSXL), Y(PSXU), Y(PZL), Y(PZU));
    HB_LAUNCHED();
  }
  if(mi > 0) {
    // rd = -dyd - dvl + dvu                                                              :1680-1685
    k_neg<<<(mi + 127) / 128, 128, 0, c->stream>>>(mi, Y(PD), X(PYD));
    HB_LAUNCHED();
    k_kkt_full_block<<<hb_grid(c, mi, ET), ET, 0, c->stream>>>(mi, X(PD), X(PSDL), X(PSDU), X(PVL), X(PVU), k->sdl, k->vl, k->sdu, k->vu, k->idl, k->idu,
                                                         Y(PD), Y(PSDL), Y(PSDU), Y(PVL), Y(PVU));
    HB_LAUNCHED();
  }
  return HB_OK;
}

int precond(hb_lowrank* k, const Layout& L, double* y, const double* x)
{
  const double* res[NPART];
  double* dir[NPART];
  for(int q = 0; q < NPART; q++) { res[q] = x + L.off[q]; dir[q] = y + L.off[q]; }
  return hb_lowrank_compute_directions(k, res, dir);
}

// reductions over a compound buffer: n-sized blocks are sharded, m-sized ones replicated -> ranks != 0 leave the latter out
// before the all-reduce (the reference reduces each block in its own communicator, hiopVectorCompoundPD.cpp:438-461)
struct Cv
{
  hb_lowrank* k;
  const Layout& L;
  long long red_len() const { return (k->ctx->nranks > 1 && k->ctx->rank != 0) ? L.n_span : L.total; }
  int dot(const double* a, const double* b, double* out) const { return hb_vec_dot(k->ctx, red_len(), a, b, out); }
  int nrm2(const double* a, double* out) const { return hb_vec_twonorm(k->ctx, red_len(), a, out); }
  int copy(double* y, const double* x) const { return hb_vec_copy(k->ctx, L.total, y, x); }
  int axpy(double* y, double a, const double* x) const { return hb_vec_axpy(k->ctx, L.total, y, a, x); }
  int scale(double* y, double a) const { return hb_vec_scale(k->ctx, L.total, y, a); }
  // r = b - K x
  int resid(double* r, const double* b, const double* x) const
  {
    HB_CHECK(full_times_vec(k, L, r, x));
    HB_CHECK(axpy(r, -1.0, b));
    return scale(r, -1.0);
  }
};

int gather(hb_lowrank* k, const Layout& L, double* buf, const double* const* parts)
{
  for(int q = 0; q < NPART; q++)
    if(L.len[q]) HB_CUDA(cudaMemcpyAsync(buf + L.off[q], parts[q], sizeof(double) * L.len[q], cudaMemcpyDeviceToDevice, k->ctx->stream));
  return HB_OK;
}
int scatter(hb_lowrank* k, const Layout& L, const double* buf, double* const* parts)
{
  for(int q = 0; q < NPART; q++)
    if(L.len[q]) HB_CUDA(cudaMemcpyAsync(parts[q], buf + L.off[q], sizeof(double) * L.len[q], cudaMemcpyDeviceToDevice, k->ctx->stream));
  return HB_OK;
}

constexpr int NVEC = 11; // b, xk, xmin, res, pk, ph, v, sk, t, rt, io

// ---------------------------------------------------------------------------------------------------------------------------------
// Device-driven recurrence. The scalars of BiCGStab (rho, alpha, omega, beta, the norms) live in a small device block; the vector
// updates read them there, every group of inner products of a half-iteration is ONE pass (fused with the vector update that produces
// the vector being measured), and the host looks at the scalars once per half-iteration to take the reference's exit decisions
// (hiopKrylovSolver.cpp:470-660) -- two stream synchronisations per iteration instead of twelve, 5 passes over the compound vectors
// instead of 14. With a communicator each group is one all-reduce of 4 doubles.
// ---------------------------------------------------------------------------------------------------------------------------------
enum { SC_RHO = 0, SC_RHO1, SC_ALPHA, SC_OMEGA, SC_BETA, SC_RTV, SC_NPH2, SC_NXK2, SC_NRM2, SC_TT, SC_TS, SC_BAD, SC_NEWRHO, SC_COUNT = 16 };
enum { KM_P = 0, KM_A, KM_B, KM_D3, KM_D4 };
constexpr int KT = 256;

// One fused pass over the compound vectors. `len` elements are updated, the inner products run over the first `red_len` only (ranks
// other than 0 leave the replicated m-sized tail out of the sums). partial[blockIdx.x*4 + q].
template <int MODE>
__global__ void __launch_bounds__(KT)
k_kry_pass(long long len, long long red_len, const double* __restrict__ sc, int first, double* __restrict__ xk, double* __restrict__ pk,
           const double* __restrict__ ph, double* __restrict__ r, const double* __restrict__ v, double* __restrict__ sk, const double* __restrict__ t,
           const double* __restrict__ rt, double* __restrict__ partial)
{
  __shared__ double sm[KT / 32];
  const bool bad = sc[SC_BAD] != 0.0;
  const double alpha = sc[SC_ALPHA], omega = sc[SC_OMEGA], beta = sc[SC_BETA];
  double d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0;
  const long long stride = (long long)gridDim.x * KT;
  for(long long i = (long long)blockIdx.x * KT + threadIdx.x; i < len; i += stride) {
    const bool in = i < red_len;
    if(MODE == KM_P) {
      if(!bad) pk[i] = first ? r[i] : fma(1.0, r[i], fma(-omega, v[i], pk[i]) * beta); // axpy(pk,-omega,v); scale(beta); axpy(pk,1,r)
    } else if(MODE == KM_A) {
      if(!bad) {
        xk[i] = fma(alpha, ph[i], xk[i]);
        const double s = fma(-alpha, v[i], r[i]);
        sk[i] = s;
        if(in) d0 += s * s;
      }
    } else if(MODE == KM_B) {
      if(!bad) {
        xk[i] = fma(omega, ph[i], xk[i]);
        const double rr = fma(-omega, t[i], sk[i]);
        r[i] = rr;
        if(in) { d0 += rr * rr; d1 += rt[i] * rr; }
      }
    } else if(MODE == KM_D3) {
      if(in) { d0 += rt[i] * v[i]; d1 += ph[i] * ph[i]; d2 += xk[i] * xk[i]; }
    } else {
      if(in) { const double tv = t[i]; d0 += tv * tv; d1 += tv * sk[i]; d2 += ph[i] * ph[i]; d3 += xk[i] * xk[i]; }
    }
  }
  if(MODE == KM_P) return;
  const double r0 = hb_block_sum<KT>(d0, sm), r1 = hb_block_sum<KT>(d1, sm), r2 = hb_block_sum<KT>(d2, sm), r3 = hb_block_sum<KT>(d3, sm);
  if(threadIdx.x == 0) {
    partial[blockIdx.x * 4 + 0] = r0; partial[blockIdx.x * 4 + 1] = r1; partial[blockIdx.x * 4 + 2] = r2; partial[blockIdx.x * 4 + 3] = r3;
  }
}
// the scalar recurrences and breakdown guards (hiopKrylovSolver.cpp:476-486, 505-513, 576-590), one thread
__global__ void k_kry_scalars(int op, int ii, double* __restrict__ sc, const double* __restrict__ sums)
{
  if(threadIdx.x != 0 || blockIdx.x != 0) return;
  if(op == 0) { // start of an iteration: rho1 <- rho, rho <- <rt, r>, beta
    sc[SC_RHO1] = sc[SC_RHO];
    const double rho = sc[SC_NEWRHO];
    sc[SC_RHO] = rho;
    if(rho == 0.0 || fabs(rho) > 1e40) sc[SC_BAD] = 1.0;
    if(ii > 0) {
      const double beta = rho / sc[SC_RHO1] * (sc[SC_ALPHA] / sc[SC_OMEGA]);
      sc[SC_BETA] = beta;
      if(beta == 0.0 || fabs(beta) > 1e40) sc[SC_BAD] = 1.0;
    }
  } else if(op == 1) { // alpha
    sc[SC_RTV] = sums[0]; sc[SC_NPH2] = sums[1]; sc[SC_NXK2] = sums[2];
    if(sc[SC_BAD] == 0.0) {
      const double rtv = sums[0];
      if(rtv == 0.0 || fabs(rtv) > 1e40) sc[SC_BAD] = 1.0;
      const double alpha = sc[SC_RHO] / rtv;
      sc[SC_ALPHA] = alpha;
      if(fabs(alpha) > 1e20) sc[SC_BAD] = 1.0;
    }
  } else if(op == 2) { // ||sk||^2
    sc[SC_NRM2] = sums[0];
  } else if(op == 3) { // omega
    sc[SC_TT] = sums[0]; sc[SC_TS] = sums[1]; sc[SC_NPH2] = sums[2]; sc[SC_NXK2] = sums[3];
    if(sc[SC_BAD] == 0.0) {
      const double tt = sums[0];
      if(tt == 0.0 || fabs(tt) > 1e20) sc[SC_BAD] = 1.0;
      const double omega = sums[1] / tt;
      sc[SC_OMEGA] = omega;
      if(fabs(omega) > 1e20) sc[SC_BAD] = 1.0;
    }
  } else { // ||r||^2 and the next rho
    sc[SC_NRM2] = sums[0];
    sc[SC_NEWRHO] = sums[1];
  }
}

} // namespace

extern "C" int hb_lowrank_kkt_full_times_vec(hb_lowrank* k, const double* const* x, double* const* y)
{
  HB_REQUIRE(k && x && y, "hb_lowrank_kkt_full_times_vec: null argument");
  HB_REQUIRE(k->have_update, "hb_lowrank_kkt_full_times_vec: call hb_lowrank_update first");
  const Layout L = make_layout(k);
  HB_CHECK(ensure_ws(k, L, NVEC));
  double* xin = k->kry + 9 * L.total;
  double* yout = k->kry + 10 * L.total;
  HB_CHECK(gather(k, L, xin, x));
  HB_CHECK(full_times_vec(k, L, yout, xin));
  return scatter(k, L, yout, y);
}

extern "C" int hb_lowrank_compute_directions_w_ir(hb_lowrank* k, const double* const* res, double* const* dir, double tol, int maxit, double* info)
{
  HB_REQUIRE(k && res && dir, "hb_lowrank_compute_directions_w_ir: null argument");
  HB_REQUIRE(k->have_update, "hb_lowrank_compute_directions_w_ir: call hb_lowrank_update first");
  if(maxit <= 0) { // hiopKKTLinSys.cpp:914-917
    if(info) { info[0] = 0; info[1] = 0; info[2] = 0; info[3] = 0; }
    return hb_lowrank_compute_directions(k, res, dir);
  }
  const Layout L = make_layout(k);
  HB_CHECK(ensure_ws(k, L, NVEC));
  const Cv cv{k, L};
  double* W = k->kry;
  double *b = W, *xk = W + L.total, *xmin = W + 2 * L.total, *r = W + 3 * L.total, *pk = W + 4 * L.total, *ph = W + 5 * L.total,
         *v = W + 6 * L.total, *sk = W + 7 * L.total, *t = W + 8 * L.total, *rt = W + 9 * L.total;
  HB_CHECK(gather(k, L, b, res));

  int flag = 1;
  double iter = 0.0, abs_resid = 0.0, rel_resid = 0.0;
  auto finish = [&](const double* sol) -> int {
    if(info) { info[0] = flag; info[1] = iter; info[2] = abs_resid; info[3] = rel_resid; }
    return scatter(k, L, sol, dir);
  };

  double n2b;
  HB_CHECK(cv.nrm2(b, &n2b));
  if(n2b == 0.0) { // rhs = 0 -> solution = 0                                             hiopKrylovSolver.cpp:402-412
    flag = 0;
    HB_CUDA(cudaMemsetAsync(xk, 0, sizeof(double) * L.total, k->ctx->stream));
    return finish(xk);
  }
  HB_CUDA(cudaMemsetAsync(xk, 0, sizeof(double) * L.total, k->ctx->stream)); // set_x0(0.0), hiopKKTLinSys.cpp:939
  const double tolb = tol * n2b;
  double imin = 0.0;
  HB_CHECK(cv.copy(xmin, xk));
  HB_CHECK(cv.resid(r, b, xk));
  double normr;
  HB_CHECK(cv.nrm2(r, &normr));
  abs_resid = normr;
  if(normr <= tolb) { // :451-461
    flag = 0;
    rel_resid = normr / n2b;
    return finish(xk);
  }
  HB_CHECK(cv.copy(rt, r));
  double normrmin = normr;
  int stagsteps = 0, moresteps = 0;
  const double eps = std::numeric_limits<double>::epsilon();
  const int maxmsteps = 100, maxstagsteps = 3;
  bool returned_xk = false; // the two "tol is too small" exits copy xk into b before the closing min-residual test (:546, :623)
  // device scalar block + per-CTA partial sums live behind the m-workspace; the host mirror is the pinned stats buffer of the handle
  hb_ctx* c = k->ctx;
  int kg = hb_grid(c, L.total, KT);
  if(kg > 2048) kg = 2048;
  double* partial = k->kry_m + (size_t)(2 * k->m + 2); // (the context workspace is used by the kernels inside precond / K)
  double* sc = partial + (size_t)kg * 4;
  double* sums = sc + SC_COUNT;
  double sc_host[SC_COUNT];
  const long long red_len = cv.red_len();
  auto group = [&](int op, int ii_) -> int { // partials -> 4 sums (all-reduced) -> scalar program
    HB_CHECK(hb_reduce_slots(c, kg, partial, sums, {HB_SUM, HB_SUM, HB_SUM, HB_SUM}));
    HB_CHECK(hb_allreduce_sum(c, sums, 4));
    k_kry_scalars<<<1, 32, 0, c->stream>>>(op, ii_, sc, sums);
    HB_LAUNCHED();
    return HB_OK;
  };
  auto poll = [&]() -> int {
    HB_CUDA(cudaMemcpyAsync(sc_host, sc, sizeof(double) * SC_COUNT, cudaMemcpyDeviceToHost, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
    return HB_OK;
  };
  {
    // rho = 1, omega = 1, alpha = 0 (hiopKrylovSolver.cpp:466-468); the first <rt, r> = ||r||^2 is already known
    double init[SC_COUNT] = {0};
    init[SC_RHO] = 1.0; init[SC_OMEGA] = 1.0; init[SC_NEWRHO] = 0.0;
    HB_CUDA(cudaMemcpyAsync(sc, init, sizeof(double) * SC_COUNT, cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream)); // init[] is a stack array
    double rho0;
    HB_CHECK(cv.dot(rt, r, &rho0));
    HB_CUDA(cudaMemcpyAsync(sc + SC_NEWRHO, &rho0, sizeof(double), cudaMemcpyHostToDevice, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
  }
  int ii = 0;
  for(; ii < maxit; ++ii) {
    // ---------------- first half: p, ph = M^-1 p, v = K ph, alpha, x += alpha ph, s = r - alpha v ----------------
    k_kry_scalars<<<1, 32, 0, c->stream>>>(0, ii, sc, sums);
    HB_LAUNCHED();
    k_kry_pass<KM_P><<<kg, KT, 0, c->stream>>>(L.total, red_len, sc, ii == 0 ? 1 : 0, xk, pk, ph, r, v, sk, t, rt, partial);
    HB_LAUNCHED();
    HB_CHECK(precond(k, L, ph, pk));
    HB_CHECK(full_times_vec(k, L, v, ph));
    k_kry_pass<KM_D3><<<kg, KT, 0, c->stream>>>(L.total, red_len, sc, 0, xk, pk, ph, r, v, sk, t, rt, partial);
    HB_LAUNCHED();
    HB_CHECK(group(1, ii));
    k_kry_pass<KM_A><<<kg, KT, 0, c->stream>>>(L.total, red_len, sc, 0, xk, pk, ph, r, v, sk, t, rt, partial);
    HB_LAUNCHED();
    HB_CHECK(group(2, ii));
    HB_CHECK(poll());
    {
      const double rho = sc_host[SC_RHO], beta = sc_host[SC_BETA], rtv = sc_host[SC_RTV], alpha = sc_host[SC_ALPHA];
      if(rho == 0.0 || std::fabs(rho) > 1e40) { flag = 4; iter = ii + 1 - 0.5; break; }
      if(ii > 0 && (beta == 0.0 || std::fabs(beta) > 1e40)) { flag = 4; iter = ii + 1 - 0.5; break; }
      if(rtv == 0.0 || std::fabs(rtv) > 1e40) { flag = 4; iter = ii + 1 - 0.5; break; }
      if(std::fabs(alpha) > 1e20) { flag = 4; iter = ii + 1 - 0.5; break; }
      if(std::sqrt(sc_host[SC_NPH2]) * std::fabs(alpha) < eps * std::sqrt(sc_host[SC_NXK2])) stagsteps++; else stagsteps = 0;
      normr = std::sqrt(sc_host[SC_NRM2]);
    }
    abs_resid = normr;
    if(normr <= tolb || stagsteps >= maxstagsteps || moresteps) {
      HB_CHECK(cv.resid(sk, b, xk));
      HB_CHECK(cv.nrm2(sk, &abs_resid));
      if(abs_resid <= tolb) { flag = 0; iter = ii + 1 - 0.5; break; }
      if(stagsteps >= maxstagsteps && moresteps == 0) stagsteps = 0;
      moresteps++;
      if(moresteps >= maxmsteps) { returned_xk = true; flag = 3; iter = ii + 1 - 0.5; break; }
    }
    if(stagsteps >= maxstagsteps) { iter = ii + 1 - 0.5; flag = 3; break; }
    if(abs_resid < normrmin) { normrmin = abs_resid; HB_CHECK(cv.copy(xmin, xk)); imin = ii + 1 - 0.5; }

    // ---------------- second half: ph = M^-1 s, t = K ph, omega, x += omega ph, r = s - omega t, next rho ----------------
    HB_CHECK(precond(k, L, ph, sk));
    HB_CHECK(full_times_vec(k, L, t, ph));
    k_kry_pass<KM_D4><<<kg, KT, 0, c->stream>>>(L.total, red_len, sc, 0, xk, pk, ph, r, v, sk, t, rt, partial);
    HB_LAUNCHED();
    HB_CHECK(group(3, ii));
    k_kry_pass<KM_B><<<kg, KT, 0, c->stream>>>(L.total, red_len, sc, 0, xk, pk, ph, r, v, sk, t, rt, partial);
    HB_LAUNCHED();
    HB_CHECK(group(4, ii));
    HB_CHECK(poll());
    {
      const double tt = sc_host[SC_TT], omega = sc_host[SC_OMEGA];
      if(tt == 0.0 || std::fabs(tt) > 1e20) { iter = ii + 1; flag = 4; break; }
      if(std::fabs(omega) > 1e20) { iter = ii + 1; flag = 4; break; }
      if(std::sqrt(sc_host[SC_NPH2]) * std::fabs(omega) < eps * std::sqrt(sc_host[SC_NXK2])) stagsteps++; else stagsteps = 0;
      normr = std::sqrt(sc_host[SC_NRM2]);
    }
    abs_resid = normr;
    if(normr <= tolb || stagsteps >= maxstagsteps || moresteps) {
      HB_CHECK(cv.resid(r, b, xk));
      HB_CHECK(cv.nrm2(r, &abs_resid));
      if(abs_resid <= tolb) { flag = 0; iter = ii + 1; break; }
      if(stagsteps >= maxstagsteps && moresteps == 0) stagsteps = 0;
      moresteps++;
      if(moresteps >= maxmsteps) { returned_xk = true; flag = 3; iter = ii + 1; break; }
      // r was replaced by the true residual: the next rho must be taken against it
      double rho_next;
      HB_CHECK(cv.dot(rt, r, &rho_next));
      HB_CUDA(cudaMemcpyAsync(sc + SC_NEWRHO, &rho_next, sizeof(double), cudaMemcpyHostToDevice, c->stream));
      HB_CUDA(cudaStreamSynchronize(c->stream));
    }
    if(abs_resid < normrmin) { normrmin = abs_resid; HB_CHECK(cv.copy(xmin, xk)); imin = ii + 1; }
    if(stagsteps >= maxstagsteps) { iter = ii + 1 - 0.5; flag = 3; break; }
  }

  if(flag == 0) { // :663-668
    rel_resid = abs_resid / n2b;
    return finish(xk);
  }
  // not converged: the iterate with the smaller true residual of {xmin, xk} is returned                     :669-697
  // (after a "tol is too small" exit the reference has already overwritten b with xk, so its closing residual is taken
  //  against that vector; the outcome of its comparison is reproduced by evaluating it against the same data)
  const double* rhs_for_test = b;
  if(returned_xk) {
    HB_CHECK(cv.copy(b, xk));
  }
  HB_CHECK(cv.resid(r, rhs_for_test, xmin));
  double normr_comp;
  HB_CHECK(cv.nrm2(r, &normr_comp));
  if(normr_comp <= abs_resid) {
    iter = imin + 1;
    abs_resid = normr_comp;
    rel_resid = normr_comp / n2b;
    return finish(xmin);
  }
  iter = ii + 1;
  rel_resid = abs_resid / n2b;
  return finish(xk);
}
