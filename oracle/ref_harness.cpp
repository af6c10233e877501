// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or called from the product (hiop_b200/).
//
// Flat C wrapper around the UNMODIFIED reference classes compiled into oracle/_ref/libhiop_ref.a
// (recipe: oracle/Makefile). It lets tests / golden-vector generators / the CPU-baseline leg of bench.py
// replay one KKT system through the reference's own code on plain host arrays:
//
//   ref_qn_*        hiopKKTLinSysLowRank::update + solveCompressed      src/Optimization/hiopKKTLinSys.cpp:1057-1190
//                   hiopHessianLowRank::{updateLogBarrierDiagonal,solve,symMatTimesInverseTimesMatTrans,timesVec}
//                                                                        src/Optimization/hiopHessianLowRank.cpp:221-630
//                   hiopKKTLinSysCompressedXYcYd::computeDirections      src/Optimization/hiopKKTLinSys.cpp:585-691
//   ref_symdense_*  hiopLinSolverSymDenseLapack::{matrixChanged,solve}   src/LinAlg/hiopLinSolverSymDenseLapack.hpp:75-192
//   ref_vec_op      hiopVectorPar elementwise ops and reductions         src/LinAlg/hiopVectorPar.cpp
//   ref_mat_*       hiopMatrixDenseRowMajor / hiopMatrixSparseTriplet assembly ops used by the MDS KKT build
//
// Compiled with -fno-access-control because the quasi-Newton state (S_t, Y_t, L, D, sigma) is private in
// hiopHessianLowRank (hiopHessianLowRank.hpp:128-160) and the residual blocks are private in hiopResidual.
#include "hiopInterface.hpp"
#include "hiopNlpFormulation.hpp"
#include "hiopIterate.hpp"
#include "hiopResidual.hpp"
#include "hiopHessianLowRank.hpp"
#include "hiopKKTLinSys.hpp"
#include "hiopLinSolverSymDenseLapack.hpp"
#include "hiopVectorPar.hpp"
#include "hiopMatrixDenseRowMajor.hpp"
#include "hiopMatrixSparseTriplet.hpp"
#include "hiopPDPerturbation.hpp"
#include "hiopVectorCompoundPD.hpp"
#include "hiopKrylovSolver.hpp"
#include "hiopKKTLinSysDense.hpp"
#include "hiopDualsUpdater.hpp"
#include "hiopCSR_IO.hpp"
#include "hiopLogBarProblem.hpp"
#include <unistd.h>
#include "LinAlgFactory.hpp"

#include <chrono>
#include <iostream>
#include <locale>
#include <cstring>
#include <vector>
#include <cmath>

using namespace hiop;

// libstdc++ is linked statically into this .so in this image: make sure its stream/locale machinery is initialised before the
// reference formats numbers into std::stringstream (hiopBiCGStabSolver::solve builds its convergence report that way).
static std::ios_base::Init s_ios_init;

namespace {

/// Synthetic dense-constraints NLP whose only job is to expose sizes and bound patterns to hiopNlpDenseConstraints.
class SynthDenseCons : public hiopInterfaceDenseConstraints
{
public:
  SynthDenseCons(int n, int m_eq, int m_ineq, const double* ixl, const double* ixu, const double* idl, const double* idu)
    : n_(n), meq_(m_eq), mineq_(m_ineq), ixl_(ixl, ixl + n), ixu_(ixu, ixu + n), idl_(idl, idl + m_ineq), idu_(idu, idu + m_ineq)
  {}
  bool get_prob_sizes(size_type& n, size_type& m) { n = n_; m = meq_ + mineq_; return true; }
  bool get_vars_info(const size_type& n, double* xlow, double* xupp, NonlinearityType* type)
  {
    for(int i = 0; i < n; i++) {
      xlow[i] = ixl_[i] == 1.0 ? 0.0 : -1e20;
      xupp[i] = ixu_[i] == 1.0 ? 10.0 : 1e20;
      type[i] = hiopNonlinear;
    }
    return true;
  }
  bool get_cons_info(const size_type& m, double* clow, double* cupp, NonlinearityType* type)
  {
    for(int i = 0; i < meq_; i++) { clow[i] = cupp[i] = 1.0; type[i] = hiopNonlinear; }
    for(int i = 0; i < mineq_; i++) {
      clow[meq_ + i] = idl_[i] == 1.0 ? 0.0 : -1e20;
      cupp[meq_ + i] = idu_[i] == 1.0 ? 10.0 : 1e20;
      type[meq_ + i] = hiopNonlinear;
    }
    return true;
  }
  bool eval_f(const size_type&, const double*, bool, double& f) { f = 0.; return true; }
  bool eval_grad_f(const size_type& n, const double*, bool, double* g) { memset(g, 0, n * sizeof(double)); return true; }
  bool eval_cons(const size_type&, const size_type&, const size_type& nc, const index_type*, const double*, bool, double* c)
  { memset(c, 0, nc * sizeof(double)); return true; }
  bool eval_Jac_cons(const size_type& n, const size_type&, const size_type& nc, const index_type*, const double*, bool, double* J)
  { memset(J, 0, sizeof(double) * n * nc); return true; }
  bool get_vecdistrib_info(size_type, index_type*) { return false; }

private:
  int n_, meq_, mineq_;
  std::vector<double> ixl_, ixu_, idl_, idu_;
};

double now_s()
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct QnCtx
{
  SynthDenseCons* iface;
  hiopNlpDenseConstraints* nlp;
  hiopIterate* it;
  hiopHessianLowRank* hess;
  hiopKKTLinSysLowRank* kkt;
  hiopMatrixDense *Jc, *Jd;
  hiopVector* gradf;
  hiopPDPerturbationNull* pert = nullptr;
  int n, meq, mineq, lmax;
};

void set_vec(hiopVector* v, const double* src) { if(v->get_size() > 0) memcpy(v->local_data(), src, sizeof(double) * v->get_size()); }
void get_vec(const hiopVector* v, double* dst) { if(v->get_size() > 0) memcpy(dst, v->local_data_const(), sizeof(double) * v->get_size()); }

} // namespace

extern "C" {

void* ref_qn_create(int n, int m_eq, int m_ineq, int lmax, const double* ixl, const double* ixu, const double* idl, const double* idu)
{
  QnCtx* c = new QnCtx;
  c->n = n; c->meq = m_eq; c->mineq = m_ineq; c->lmax = lmax;
  c->iface = new SynthDenseCons(n, m_eq, m_ineq, ixl, ixu, idl, idu);
  c->nlp = new hiopNlpDenseConstraints(*c->iface);
  c->nlp->options->SetIntegerValue("verbosity_level", 0);
  c->nlp->options->SetIntegerValue("secant_memory_len", lmax);
  c->nlp->options->SetStringValue("fixed_var", "relax");
  c->nlp->finalizeInitialization();
  c->it = new hiopIterate(c->nlp);
  c->hess = new hiopHessianLowRank(c->nlp, lmax);
  c->kkt = new hiopKKTLinSysLowRank(c->nlp);
  c->Jc = c->nlp->alloc_Jac_c();
  c->Jd = c->nlp->alloc_Jac_d();
  c->gradf = c->nlp->alloc_primal_vec();
  c->gradf->setToZero();
  return c;
}

void ref_qn_destroy(void* h)
{
  QnCtx* c = (QnCtx*)h;
  delete c->pert;
  delete c->gradf; delete c->Jd; delete c->Jc; delete c->kkt; delete c->hess; delete c->it; delete c->nlp; delete c->iface;
  delete c;
}

/// sizes as the formulation sees them (sanity check for the eq/ineq split): out = {n, m_eq, m_ineq, n_low, n_upp}
void ref_qn_sizes(void* h, int* out)
{
  QnCtx* c = (QnCtx*)h;
  out[0] = c->nlp->n(); out[1] = c->nlp->m_eq(); out[2] = c->nlp->m_ineq();
  out[3] = c->nlp->n_low_local(); out[4] = c->nlp->n_upp_local();
}

void ref_qn_set_iterate(void* h, const double* sxl, const double* sxu, const double* zl, const double* zu,
                        const double* sdl, const double* sdu, const double* vl, const double* vu)
{
  QnCtx* c = (QnCtx*)h;
  set_vec(c->it->sxl, sxl); set_vec(c->it->sxu, sxu); set_vec(c->it->zl, zl); set_vec(c->it->zu, zu);
  set_vec(c->it->sdl, sdl); set_vec(c->it->sdu, sdu); set_vec(c->it->vl, vl); set_vec(c->it->vu, vu);
  c->it->x->setToZero(); c->it->d->setToZero(); c->it->yc->setToZero(); c->it->yd->setToZero();
}

void ref_qn_set_jac(void* h, const double* Jc, const double* Jd)
{
  QnCtx* c = (QnCtx*)h;
  if(c->meq) memcpy(c->Jc->local_data(), Jc, sizeof(double) * (size_t)c->meq * c->n);
  if(c->mineq) memcpy(c->Jd->local_data(), Jd, sizeof(double) * (size_t)c->mineq * c->n);
}

/// Plants the compact-BFGS state: S_t,Y_t are l x n row-major, L is l x l (strictly lower = s_i^T y_j), D is l.
void ref_qn_set_secant(void* h, int l, double sigma, const double* St, const double* Yt, const double* L, const double* D)
{
  QnCtx* c = (QnCtx*)h;
  hiopHessianLowRank* H = c->hess;
  H->alloc_for_limited_mem(l);
  H->l_curr = l;
  H->sigma = sigma;
  if(l > 0) {
    memcpy(H->St_->local_data(), St, sizeof(double) * (size_t)l * c->n);
    memcpy(H->Yt_->local_data(), Yt, sizeof(double) * (size_t)l * c->n);
    memcpy(H->L_->local_data(), L, sizeof(double) * l * l);
    memcpy(H->D_->local_data(), D, sizeof(double) * l);
  }
  H->matrixChanged = true;
}

/// hiopKKTLinSysLowRank::update -> Dx, DhInv, Dd_inv. times[0] = seconds.
void ref_qn_update(void* h, double* Dx, double* DhInv, double* Dd_inv, double* times)
{
  QnCtx* c = (QnCtx*)h;
  double t0 = now_s();
  c->kkt->update(c->it, c->gradf, c->Jc, c->Jd, c->hess);
  times[0] = now_s() - t0;
  if(Dx) get_vec(c->kkt->Dx_, Dx);
  if(DhInv) get_vec(c->hess->DhInv, DhInv);
  if(Dd_inv) get_vec(c->kkt->Dd_inv_, Dd_inv);
}

/// N = J (B+Dx)^{-1} J^T + blkdiag(0, Dd_inv), as formed at hiopKKTLinSys.cpp:1124-1135. Nout is m x m row-major.
void ref_qn_condense(void* h, double* Nout, double* times)
{
  QnCtx* c = (QnCtx*)h;
  int m = c->meq + c->mineq;
  hiopMatrixDense* J = c->nlp->alloc_multivector_primal(m);
  hiopMatrixDense* N = LinearAlgebraFactory::create_matrix_dense("DEFAULT", m, m);
  double t0 = now_s();
  J->copyRowsFrom(*c->Jc, c->meq, 0);
  J->copyRowsFrom(*c->Jd, c->mineq, c->meq);
  c->hess->symMatTimesInverseTimesMatTrans(0.0, *N, 1.0, *J);
  N->addSubDiagonal(1., c->meq, *c->kkt->Dd_inv_);
  times[0] = now_s() - t0;
  memcpy(Nout, N->local_data(), sizeof(double) * (size_t)m * m);
  delete N; delete J;
}

/// hiopKKTLinSysLowRank::solveCompressed. rx is clobbered by the reference (hiopKKTLinSys.cpp:1178); we pass a copy.
int ref_qn_solve_compressed(void* h, const double* rx, const double* ryc, const double* ryd,
                            double* dx, double* dyc, double* dyd, double* times)
{
  QnCtx* c = (QnCtx*)h;
  hiopVector* vrx = c->nlp->alloc_primal_vec(); hiopVector* vdx = c->nlp->alloc_primal_vec();
  hiopVector* vryc = c->nlp->alloc_dual_eq_vec(); hiopVector* vdyc = c->nlp->alloc_dual_eq_vec();
  hiopVector* vryd = c->nlp->alloc_dual_ineq_vec(); hiopVector* vdyd = c->nlp->alloc_dual_ineq_vec();
  set_vec(vrx, rx); set_vec(vryc, ryc); set_vec(vryd, ryd);
  double t0 = now_s();
  bool ok = c->kkt->solveCompressed(*vrx, *vryc, *vryd, *vdx, *vdyc, *vdyd);
  times[0] = now_s() - t0;
  get_vec(vdx, dx); get_vec(vdyc, dyc); get_vec(vdyd, dyd);
  delete vrx; delete vdx; delete vryc; delete vdyc; delete vryd; delete vdyd;
  return ok ? 0 : -1;
}

/// hiopHessianLowRank::solve: x = (B_k + D_x)^{-1} rhs
void ref_qn_hess_solve(void* h, const double* rhs, double* x)
{
  QnCtx* c = (QnCtx*)h;
  hiopVector* r = c->nlp->alloc_primal_vec(); hiopVector* xx = c->nlp->alloc_primal_vec();
  set_vec(r, rhs);
  c->hess->solve(*r, *xx);
  get_vec(xx, x);
  delete r; delete xx;
}

/// hiopHessianLowRank::timesVec (recursive BFGS product; addLogTerm as used by the full-KKT operator)
void ref_qn_hess_times_vec(void* h, double beta, double* y, double alpha, const double* x, int add_log_term)
{
  QnCtx* c = (QnCtx*)h;
  hiopVector* vy = c->nlp->alloc_primal_vec(); hiopVector* vx = c->nlp->alloc_primal_vec();
  set_vec(vy, y); set_vec(vx, x);
  c->hess->timesVecCmn(beta, *vy, alpha, *vx, add_log_term != 0);
  get_vec(vy, y);
  delete vy; delete vx;
}

/// hiopKKTLinSysCompressedXYcYd::computeDirections on the 12 residual blocks -> 12 direction blocks.
/// res/dir order: x, d, yc, yd, sxl, sxu, sdl, sdu, zl, zu, vl, vu  (n, mi, me, mi, n, n, mi, mi, n, n, mi, mi)
/// residual order: rx, rd, ryc, ryd, rxl, rxu, rdl, rdu, rszl, rszu, rsvl, rsvu
int ref_qn_compute_directions(void* h, const double* const* res, double* const* dir)
{
  QnCtx* c = (QnCtx*)h;
  hiopResidual r(c->nlp);
  hiopIterate d(c->nlp);
  set_vec(r.rx, res[0]); set_vec(r.rd, res[1]); set_vec(r.ryc, res[2]); set_vec(r.ryd, res[3]);
  set_vec(r.rxl, res[4]); set_vec(r.rxu, res[5]); set_vec(r.rdl, res[6]); set_vec(r.rdu, res[7]);
  set_vec(r.rszl, res[8]); set_vec(r.rszu, res[9]); set_vec(r.rsvl, res[10]); set_vec(r.rsvu, res[11]);
  bool ok = c->kkt->computeDirections(&r, &d);
  get_vec(d.x, dir[0]); get_vec(d.d, dir[1]); get_vec(d.yc, dir[2]); get_vec(d.yd, dir[3]);
  get_vec(d.sxl, dir[4]); get_vec(d.sxu, dir[5]); get_vec(d.sdl, dir[6]); get_vec(d.sdu, dir[7]);
  get_vec(d.zl, dir[8]); get_vec(d.zu, dir[9]); get_vec(d.vl, dir[10]); get_vec(d.vu, dir[11]);
  return ok ? 0 : -1;
}

/// hiopHessianLowRank::update (hiopHessianLowRank.cpp:262-388) with the iterate (x, yc, yd), grad_f and the Jacobians given as
/// plain arrays. Reads back the secant memory afterwards: out_l = rows of S_t/Y_t; St, Yt (lmax x n, first out_l rows valid),
/// L (lmax x lmax row-major, leading out_l x out_l block valid, packed with stride out_l), D (out_l), sigma.
int ref_qn_hess_update(void* h, const double* x, const double* grad_f, const double* yc, const double* yd, const double* Jc, const double* Jd,
                       int* out_l, double* St, double* Yt, double* L, double* D, double* sigma)
{
  QnCtx* c = (QnCtx*)h;
  set_vec(c->it->x, x); set_vec(c->it->yc, yc); set_vec(c->it->yd, yd);
  set_vec(c->gradf, grad_f);
  ref_qn_set_jac(h, Jc, Jd);
  bool ok = c->hess->update(*c->it, *c->gradf, *c->Jc, *c->Jd);
  hiopHessianLowRank* H = c->hess;
  const int l = H->St_->m();
  *out_l = l;
  *sigma = H->sigma;
  if(l > 0) {
    memcpy(St, H->St_->local_data_const(), sizeof(double) * (size_t)l * c->n);
    memcpy(Yt, H->Yt_->local_data_const(), sizeof(double) * (size_t)l * c->n);
    memcpy(L, H->L_->local_data_const(), sizeof(double) * l * l);
    memcpy(D, H->D_->local_data_const(), sizeof(double) * l);
  }
  return ok ? 0 : -1;
}

/// sigma_update_strategy 1..5 = sty, sty_inv, snrm_ynrm, sty_srnm_ynrm, sigma0 (hiopHessianLowRank.cpp:49-53, 124-136); also
/// resets sigma to sigma0 like the constructor does (:120-121).
void ref_qn_set_sigma_strategy(void* h, int strategy, double sigma0)
{
  QnCtx* c = (QnCtx*)h;
  c->hess->sigma_update_strategy = strategy;
  c->hess->sigma0 = sigma0;
  c->hess->sigma = sigma0;
}

/// hiopDualsLsqUpdateLinsysRedDenseSymPD::do_lsq_update (hiopDualsUpdater.cpp:232-332, DPOTRF/DPOTRS :690-735): the LSQ
/// multipliers yc, yd from [Jc Jc^T, Jc Jd^T; ., Jd Jd^T + I] y = -[Jc vx; Jd vx + vd], vx = grad_f - zl + zu, vd = vl - vu.
/// Uses the Jacobians and zl, zu, vl, vu already planted by ref_qn_set_jac / ref_qn_set_iterate.
int ref_qn_lsq_duals(void* h, const double* grad_f, double* yc, double* yd)
{
  QnCtx* c = (QnCtx*)h;
  set_vec(c->gradf, grad_f);
  hiopDualsLsqUpdateLinsysRedDenseSymPD lsq(c->nlp);
  hiopDualsLsqUpdateLinsysRedDense* base = &lsq;
  bool ok = base->do_lsq_update(*c->it, *c->gradf, *c->Jc, *c->Jd);
  get_vec(c->it->yc, yc); get_vec(c->it->yd, yd);
  return ok ? 0 : -1;
}

/// hiopResidual::update (src/Optimization/hiopResidual.cpp:154-368) with the log-barrier proxy hiopLogBarProblem (mu, kappa_d).
/// iter: 12 blocks in the order x, d, yc, yd, sxl, sxu, sdl, sdu, zl, zu, vl, vu; bounds xl, xu (n), dl, du (m_ineq), crhs (m_eq)
/// overwrite the formulation's own. res: 12 blocks (rx, rd, ryc, ryd, rxl, rxu, rdl, rdu, rszl, rszu, rsvl, rsvu). norms (11):
/// nrmInf nlp {optim, feasib, complem}, nrmInf bar {optim, feasib, complem}, nrmOne nlp_feasib, bar_feasib, nlp_optim, bar_optim,
/// nrmInf_cons_violation. Uses the Jacobians planted by ref_qn_set_jac.
int ref_qn_residual_update(void* h, const double* const* iter, const double* cvals, const double* dvals, const double* grad, double mu,
                           double kappa_d, const double* xl, const double* xu, const double* dl, const double* du, const double* crhs,
                           double* const* res, double* norms)
{
  QnCtx* c = (QnCtx*)h;
  hiopIterate& it = *c->it;
  set_vec(it.x, iter[0]); set_vec(it.d, iter[1]); set_vec(it.yc, iter[2]); set_vec(it.yd, iter[3]);
  set_vec(it.sxl, iter[4]); set_vec(it.sxu, iter[5]); set_vec(it.sdl, iter[6]); set_vec(it.sdu, iter[7]);
  set_vec(it.zl, iter[8]); set_vec(it.zu, iter[9]); set_vec(it.vl, iter[10]); set_vec(it.vu, iter[11]);
  set_vec(c->nlp->xl_, xl); set_vec(c->nlp->xu_, xu); set_vec(c->nlp->dl_, dl); set_vec(c->nlp->du_, du); set_vec(c->nlp->c_rhs_, crhs);
  hiopVector* cv = c->nlp->alloc_dual_eq_vec();
  hiopVector* dv = c->nlp->alloc_dual_ineq_vec();
  set_vec(cv, cvals); set_vec(dv, dvals); set_vec(c->gradf, grad);
  hiopLogBarProblem lp(c->nlp);
  lp.mu = mu; lp.kappa_d = kappa_d; lp.iter = &it;
  hiopResidual r(c->nlp);
  r.update(it, 0.0, *cv, *dv, *c->gradf, *c->Jc, *c->Jd, lp);
  get_vec(r.rx, res[0]); get_vec(r.rd, res[1]); get_vec(r.ryc, res[2]); get_vec(r.ryd, res[3]);
  get_vec(r.rxl, res[4]); get_vec(r.rxu, res[5]); get_vec(r.rdl, res[6]); get_vec(r.rdu, res[7]);
  get_vec(r.rszl, res[8]); get_vec(r.rszu, res[9]); get_vec(r.rsvl, res[10]); get_vec(r.rsvu, res[11]);
  norms[0] = r.nrmInf_nlp_optim; norms[1] = r.nrmInf_nlp_feasib; norms[2] = r.nrmInf_nlp_complem;
  norms[3] = r.nrmInf_bar_optim; norms[4] = r.nrmInf_bar_feasib; norms[5] = r.nrmInf_bar_complem;
  norms[6] = r.nrmOne_nlp_feasib; norms[7] = r.nrmOne_bar_feasib; norms[8] = r.nrmOne_nlp_optim; norms[9] = r.nrmOne_bar_optim;
  norms[10] = r.nrmInf_cons_violation;
  delete dv; delete cv;
  return 0;
}

namespace {
void plant_iterate(hiopIterate& it, const double* const* b)
{
  set_vec(it.x, b[0]); set_vec(it.d, b[1]); set_vec(it.yc, b[2]); set_vec(it.yd, b[3]);
  set_vec(it.sxl, b[4]); set_vec(it.sxu, b[5]); set_vec(it.sdl, b[6]); set_vec(it.sdu, b[7]);
  set_vec(it.zl, b[8]); set_vec(it.zu, b[9]); set_vec(it.vl, b[10]); set_vec(it.vu, b[11]);
}
} // namespace

/// hiopLogBarProblem::updateWithNlpInfo (hiopLogBarProblem.hpp:83-120): log-barrier function value and gradients at the iterate.
int ref_qn_logbar_update(void* h, const double* const* iter, double f, double mu, double kappa_d, const double* grad, double* gx, double* gd,
                         double* f_logbar)
{
  QnCtx* c = (QnCtx*)h;
  plant_iterate(*c->it, iter);
  set_vec(c->gradf, grad);
  hiopVector* cv = c->nlp->alloc_dual_eq_vec();
  hiopVector* dv = c->nlp->alloc_dual_ineq_vec();
  hiopLogBarProblem lp(c->nlp);
  lp.kappa_d = kappa_d;
  lp.updateWithNlpInfo(*c->it, mu, f, *cv, *dv, *c->gradf, *c->Jc, *c->Jd);
  get_vec(lp._grad_x_logbar, gx); get_vec(lp._grad_d_logbar, gd);
  *f_logbar = lp.f_logbar;
  delete dv; delete cv;
  return 0;
}

/// hiopIterate::adjustDuals_primalLogHessian (hiopIterate.cpp:508-521): zl, zu, vl, vu clamped in place, returned through out[0..3].
int ref_qn_adjust_duals(void* h, const double* const* iter, double mu, double kappa, double* const* out)
{
  QnCtx* c = (QnCtx*)h;
  plant_iterate(*c->it, iter);
  c->it->adjustDuals_primalLogHessian(mu, kappa);
  get_vec(c->it->zl, out[0]); get_vec(c->it->zu, out[1]); get_vec(c->it->vl, out[2]); get_vec(c->it->vu, out[3]);
  return 0;
}

/// hiopIterate::adjust_small_slacks (hiopIterate.cpp:481-505) on the slacks of `iter` with the duals of `iter_curr`, bounds as given.
/// out[0..3] = sxl, sxu, sdl, sdu afterwards; returns the number of adjusted slacks.
int ref_qn_adjust_small_slacks(void* h, const double* const* iter, const double* const* iter_curr, double mu, const double* xl, const double* xu,
                               const double* dl, const double* du, double* const* out)
{
  QnCtx* c = (QnCtx*)h;
  plant_iterate(*c->it, iter);
  hiopIterate cur(c->nlp);
  plant_iterate(cur, iter_curr);
  set_vec(c->nlp->xl_, xl); set_vec(c->nlp->xu_, xu); set_vec(c->nlp->dl_, dl); set_vec(c->nlp->du_, du);
  const int n = c->it->adjust_small_slacks(cur, mu);
  get_vec(c->it->sxl, out[0]); get_vec(c->it->sxu, out[1]); get_vec(c->it->sdl, out[2]); get_vec(c->it->sdu, out[3]);
  return n;
}

/// hiopIterate::fractionToTheBdry (hiopIterate.cpp:326-363): largest primal / dual step lengths keeping slacks and duals positive.
int ref_qn_fraction_to_bdry(void* h, const double* const* iter, const double* const* dir, double tau, double* alpha_primal, double* alpha_dual)
{
  QnCtx* c = (QnCtx*)h;
  plant_iterate(*c->it, iter);
  hiopIterate d(c->nlp);
  plant_iterate(d, dir);
  c->it->fractionToTheBdry(d, tau, *alpha_primal, *alpha_dual);
  return 0;
}

namespace {
void ensure_pert(QnCtx* c)
{
  if(c->pert) return;
  // the quasi-Newton driver installs the all-zero perturbation object (hiopAlgFilterIPM.cpp:1052-1059)
  c->pert = new hiopPDPerturbationNull();
  c->pert->initialize(c->nlp);
  c->kkt->set_PD_perturb_calc(c->pert);
}
void set_resid(hiopResidual& r, const double* const* res)
{
  set_vec(r.rx, res[0]); set_vec(r.rd, res[1]); set_vec(r.ryc, res[2]); set_vec(r.ryd, res[3]);
  set_vec(r.rxl, res[4]); set_vec(r.rxu, res[5]); set_vec(r.rdl, res[6]); set_vec(r.rdu, res[7]);
  set_vec(r.rszl, res[8]); set_vec(r.rszu, res[9]); set_vec(r.rsvl, res[10]); set_vec(r.rsvu, res[11]);
}
void get_iter(const hiopIterate& d, double* const* dir)
{
  get_vec(d.x, dir[0]); get_vec(d.d, dir[1]); get_vec(d.yc, dir[2]); get_vec(d.yd, dir[3]);
  get_vec(d.sxl, dir[4]); get_vec(d.sxu, dir[5]); get_vec(d.sdl, dir[6]); get_vec(d.sdu, dir[7]);
  get_vec(d.zl, dir[8]); get_vec(d.zu, dir[9]); get_vec(d.vl, dir[10]); get_vec(d.vu, dir[11]);
}
} // namespace

/// hiopKKTLinSys::compute_directions_w_IR (hiopKKTLinSys.cpp:909-960): BiCGStab on the full KKT system, preconditioned by
/// computeDirections. mu sets the tolerance min(mu*ir_outer_tol_factor, ir_outer_tol_min); info = {flag, iter, abs, rel}.
int ref_qn_compute_directions_w_IR(void* h, const double* const* res, double* const* dir, double mu, int maxit, double* info)
{
  QnCtx* c = (QnCtx*)h;
  ensure_pert(c);
  c->nlp->options->SetIntegerValue("ir_outer_maxit", maxit);
  c->kkt->set_logbar_mu(mu);
  hiopResidual r(c->nlp);
  hiopIterate d(c->nlp);
  set_resid(r, res);
  bool ok = c->kkt->compute_directions_w_IR(&r, &d);
  get_iter(d, dir);
  if(info && c->kkt->bicgIR_) {
    info[0] = c->kkt->bicgIR_->flag_;
    info[1] = c->kkt->bicgIR_->get_sol_num_iter();
    info[2] = c->kkt->bicgIR_->get_sol_abs_resid();
    info[3] = c->kkt->bicgIR_->get_sol_rel_resid();
  }
  return ok ? 0 : -1;
}

/// y = K x with hiopMatVecKKTFullOpr::times_vec (hiopKKTLinSys.cpp:1619-1733); x/y in the compound order of dir/res.
int ref_qn_kkt_full_times_vec(void* h, const double* const* x, double* const* y)
{
  QnCtx* c = (QnCtx*)h;
  ensure_pert(c);
  hiopIterate xi(c->nlp), yi(c->nlp);
  set_vec(xi.x, x[0]); set_vec(xi.d, x[1]); set_vec(xi.yc, x[2]); set_vec(xi.yd, x[3]);
  set_vec(xi.sxl, x[4]); set_vec(xi.sxu, x[5]); set_vec(xi.sdl, x[6]); set_vec(xi.sdu, x[7]);
  set_vec(xi.zl, x[8]); set_vec(xi.zu, x[9]); set_vec(xi.vl, x[10]); set_vec(xi.vu, x[11]);
  hiopVectorCompoundPD xv(&xi), yv(&yi);
  hiopMatVecKKTFullOpr opr(c->kkt, c->it);
  bool ok = opr.times_vec(yv, xv);
  get_iter(yi, y);
  return ok ? 0 : -1;
}

/// hiopBiCGStabSolver::solve (hiopKrylovSolver.cpp:399-700) on a dense n x n system A x = b with a dense left preconditioner
/// Minv (both row-major), x0 = 0: pins the recurrence, the exit rules and the minimal-residual fallback of the restatement
/// on systems that need many iterations. b is overwritten with the solution; info = {flag, iter, abs_resid, rel_resid}.
int ref_bicgstab_dense(int n, const double* A, const double* Minv, double* b, double tol, int maxit, double* info)
{
  hiopMatrixDense* Am = LinearAlgebraFactory::create_matrix_dense("DEFAULT", n, n);
  hiopMatrixDense* Mm = LinearAlgebraFactory::create_matrix_dense("DEFAULT", n, n);
  memcpy(Am->local_data(), A, sizeof(double) * (size_t)n * n);
  memcpy(Mm->local_data(), Minv, sizeof(double) * (size_t)n * n);
  hiopMatVecOpr Aop(Am), Mop(Mm);
  hiopVector* bv = LinearAlgebraFactory::create_vector("DEFAULT", n);
  set_vec(bv, b);
  bool ok;
  {
    hiopBiCGStabSolver solver(n, &Aop, &Mop, nullptr, nullptr);
    solver.set_max_num_iter(maxit);
    solver.set_tol(tol);
    solver.set_x0(0.0);
    ok = solver.solve(bv);
    info[0] = solver.flag_;
    info[1] = solver.get_sol_num_iter();
    info[2] = solver.get_sol_abs_resid();
    info[3] = solver.get_sol_rel_resid();
  }
  get_vec(bv, b);
  delete bv; delete Mm; delete Am;
  return ok ? 0 : 1;
}

/// hiopKKTLinSysDenseXYcYd / XDYcYd::build_kkt_matrix (hiopKKTLinSysDense.hpp:85-172, 249-330) on plain arrays.
/// form 0 = XYcYd (N = nx+neq+nineq), 1 = XDYcYd (N = nx+neq+2 nineq). H is nx x nx row-major (upper triangle used).
/// deltas = {delta_wx (nx), delta_wd (nineq), delta_cc (neq), delta_cd (nineq)}. Mout is N x N row-major (upper triangle valid).
int ref_densekkt_build(int form, int nx, int neq, int nineq, const double* H, const double* Jc, const double* Jd, const double* ixl,
                       const double* ixu, const double* idl, const double* idu, const double* zl, const double* sxl, const double* zu,
                       const double* sxu, const double* vl, const double* sdl, const double* vu, const double* sdu, const double* const* deltas,
                       double* Mout)
{
  SynthDenseCons iface(nx, neq, nineq, ixl, ixu, idl, idu);
  hiopNlpDenseConstraints nlp(iface);
  nlp.options->SetIntegerValue("verbosity_level", 0);
  nlp.options->SetStringValue("fixed_var", "relax");
  nlp.finalizeInitialization();
  hiopIterate it(&nlp);
  set_vec(it.zl, zl); set_vec(it.sxl, sxl); set_vec(it.zu, zu); set_vec(it.sxu, sxu);
  set_vec(it.vl, vl); set_vec(it.sdl, sdl); set_vec(it.vu, vu); set_vec(it.sdu, sdu);
  hiopMatrixDense* Hm = LinearAlgebraFactory::create_matrix_dense("DEFAULT", nx, nx);
  memcpy(Hm->local_data(), H, sizeof(double) * (size_t)nx * nx);
  hiopMatrixDense* Jcm = nlp.alloc_Jac_c();
  hiopMatrixDense* Jdm = nlp.alloc_Jac_d();
  if(neq) memcpy(Jcm->local_data(), Jc, sizeof(double) * (size_t)neq * nx);
  if(nineq) memcpy(Jdm->local_data(), Jd, sizeof(double) * (size_t)nineq * nx);
  hiopPDPerturbationNull pert;
  pert.initialize(&nlp);
  set_vec(pert.delta_wx_curr_, deltas[0]); set_vec(pert.delta_wd_curr_, deltas[1]);
  set_vec(pert.delta_cc_curr_, deltas[2]); set_vec(pert.delta_cd_curr_, deltas[3]);
  auto fill = [&](hiopKKTLinSysCompressed* kkt) {
    kkt->iter_ = &it; kkt->Hess_ = Hm; kkt->Jac_c_ = Jcm; kkt->Jac_d_ = Jdm;
    kkt->set_PD_perturb_calc(&pert);
    // the barrier diagonals as update() computes them (hiopKKTLinSys.cpp:560-566, 793-803)
    kkt->Dx_->setToZero();
    kkt->Dx_->axdzpy_w_pattern(1.0, *it.zl, *it.sxl, nlp.get_ixl());
    kkt->Dx_->axdzpy_w_pattern(1.0, *it.zu, *it.sxu, nlp.get_ixu());
  };
  int N;
  if(form == 0) {
    hiopKKTLinSysDenseXYcYd kkt(&nlp);
    fill(&kkt);
    kkt.build_kkt_matrix(pert);
    hiopMatrixDense& M = dynamic_cast<hiopLinSolverSymDense*>(kkt.linSys_)->sysMatrix();
    N = M.m();
    memcpy(Mout, M.local_data(), sizeof(double) * (size_t)N * N);
  } else {
    hiopKKTLinSysDenseXDYcYd kkt(&nlp);
    fill(&kkt);
    kkt.Dd_->setToZero();
    kkt.Dd_->axdzpy_w_pattern(1.0, *it.vl, *it.sdl, nlp.get_idl());
    kkt.Dd_->axdzpy_w_pattern(1.0, *it.vu, *it.sdu, nlp.get_idu());
    kkt.build_kkt_matrix(pert);
    hiopMatrixDense& M = dynamic_cast<hiopLinSolverSymDense*>(kkt.linSys_)->sysMatrix();
    N = M.m();
    memcpy(Mout, M.local_data(), sizeof(double) * (size_t)N * N);
  }
  delete Jdm; delete Jcm; delete Hm;
  return N;
}

/// hiopCSR_IO::writeMatToFile + writeRhsToFile + writeSolToFile (src/Utils/hiopCSR_IO.hpp:44-155): writes
/// <dir>/kkt_linsys_<counter>.iajaaa for the N x N row-major matrix M (upper triangle) and one rhs/solution pair.
int ref_write_iajaaa(const char* dir, int counter, int N, const double* M, int nx, int meq, int mineq, const double* rhs, const double* sol)
{
  static const double one = 1.0;
  SynthDenseCons iface(1, 0, 0, &one, &one, &one, &one);
  hiopNlpDenseConstraints nlp(iface);
  nlp.options->SetIntegerValue("verbosity_level", 0);
  hiopMatrixDense* Mm = LinearAlgebraFactory::create_matrix_dense("DEFAULT", N, N);
  memcpy(Mm->local_data(), M, sizeof(double) * (size_t)N * N);
  hiopVector* r = LinearAlgebraFactory::create_vector("DEFAULT", N);
  hiopVector* x = LinearAlgebraFactory::create_vector("DEFAULT", N);
  set_vec(r, rhs); set_vec(x, sol);
  char cwd[4096];
  if(!getcwd(cwd, sizeof(cwd)) || chdir(dir) != 0) return -1; // the reference writes into the current directory
  {
    hiopCSR_IO io(&nlp);
    io.writeMatToFile(*Mm, counter, nx, meq, mineq);
    io.writeRhsToFile(*r, counter);
    io.writeSolToFile(*x, counter);
  }
  int rc = chdir(cwd);
  delete x; delete r; delete Mm;
  return rc;
}

// ---------------------------------------------------------------------------------------------------------
// hiopLinSolverSymDenseLapack (B1). M is N x N row-major with the UPPER triangle valid (hiopKKTLinSysMDS.cpp:196-206).
// Returns matrixChanged()'s value: #negative eigenvalues, or -1 when singular. rhs (nrhs vectors) solved in place.
// ---------------------------------------------------------------------------------------------------------
int ref_symdense_factor_solve(int N, const double* M, int nrhs, double* rhs, double* factor_out, double* times)
{
  static const double one = 1.0;
  SynthDenseCons iface(1, 0, 0, &one, &one, &one, &one);
  hiopNlpDenseConstraints nlp(iface);
  nlp.options->SetIntegerValue("verbosity_level", 0);
  hiopLinSolverSymDenseLapack ls(N, &nlp);
  memcpy(ls.sysMatrix().local_data(), M, sizeof(double) * (size_t)N * N);
  double t0 = now_s();
  int ret = ls.matrixChanged();
  if(times) times[0] = now_s() - t0;
  if(factor_out) memcpy(factor_out, ls.sysMatrix().local_data(), sizeof(double) * (size_t)N * N);
  t0 = now_s();
  if(ret >= 0 || ret == -1) {
    for(int k = 0; k < nrhs; k++) {
      hiopVectorPar x(N);
      memcpy(x.local_data(), rhs + (size_t)k * N, sizeof(double) * N);
      bool ok = ls.solve(x);
      (void)ok;
      memcpy(rhs + (size_t)k * N, x.local_data(), sizeof(double) * N);
    }
  }
  if(times) times[1] = now_s() - t0;
  return ret;
}

// ---------------------------------------------------------------------------------------------------------
// hiopVectorPar ops. y is in/out; returns the scalar result for reductions (0 otherwise).
// ---------------------------------------------------------------------------------------------------------
enum {
  OP_AXDZPY_W_PATTERN = 1,   // y += alpha*x/z where sel==1            hiopVectorPar.cpp:767-790
  OP_AXZPY = 2,              // y += alpha*x*z                          :710-734
  OP_AXDZPY = 3,             // y += alpha*x/z                          :736-765
  OP_COMPONENT_MULT = 4,     // y *= x                                  :564-572
  OP_COMPONENT_DIV = 5,      // y /= x                                  :574-582
  OP_COMPONENT_DIV_W_SEL = 6,// y = sel ? y/x : 0                       :584-592
  OP_INVERT = 7,             // y = 1/y                                 :852-860
  OP_SELECT_PATTERN = 8,     // y = sel ? y : 0                         :1063-1071
  OP_ADD_CONSTANT = 9,       // y += alpha                              :793-797
  OP_ADD_CONSTANT_W_SEL = 10,// y += alpha where sel==1                 :799-804
  OP_SCALE = 11,             // y *= alpha
  OP_AXPY = 12,              // y += alpha*x
  OP_ADD_LOGBAR_GRAD = 13,   // y += alpha/x where sel==1               :893-905
  OP_ADD_LIN_DAMPING = 14,   // y = alpha*y + beta*(ixl-ixu)  (x=ixl,z=ixu)   :927-944
  OP_TWONORM = 20, OP_DOT = 21, OP_INFNORM = 22, OP_ONENORM = 23,
  OP_LOGBARRIER = 24,        // sum log(y_i) where sel==1 (Kahan)       :863-881
  OP_LIN_DAMPING_TERM = 25,  // sum y_i where x(ixl)==1 && z(ixu)==0, times alpha(mu)*beta(kappa_d)  :907-925
  OP_MIN_W_PATTERN = 26,     // min y_i where sel==1                    :821-839
  OP_FRAC_TO_BDRY = 27,      // fractionToTheBdry_local(y=x, x=dx, alpha=tau)            :1017-1036
  OP_FRAC_TO_BDRY_W_SEL = 28,// fractionToTheBdry_w_pattern_local(y=x, x=dx, alpha=tau, sel)  :1038-1061
  OP_SUM = 29,
};

double ref_vec_op(int op, int n, double* y, const double* x, const double* z, const double* sel, double alpha, double beta)
{
  hiopVectorPar vy(n), vx(n), vz(n), vs(n);
  if(n > 0) {
    memcpy(vy.local_data(), y, sizeof(double) * n);
    if(x) memcpy(vx.local_data(), x, sizeof(double) * n);
    if(z) memcpy(vz.local_data(), z, sizeof(double) * n);
    if(sel) memcpy(vs.local_data(), sel, sizeof(double) * n);
  }
  double ret = 0.;
  switch(op) {
    case OP_AXDZPY_W_PATTERN: vy.axdzpy_w_pattern(alpha, vx, vz, vs); break;
    case OP_AXZPY: vy.axzpy(alpha, vx, vz); break;
    case OP_AXDZPY: vy.axdzpy(alpha, vx, vz); break;
    case OP_COMPONENT_MULT: vy.componentMult(vx); break;
    case OP_COMPONENT_DIV: vy.componentDiv(vx); break;
    case OP_COMPONENT_DIV_W_SEL: vy.componentDiv_w_selectPattern(vx, vs); break;
    case OP_INVERT: vy.invert(); break;
    case OP_SELECT_PATTERN: vy.selectPattern(vs); break;
    case OP_ADD_CONSTANT: vy.addConstant(alpha); break;
    case OP_ADD_CONSTANT_W_SEL: vy.addConstant_w_patternSelect(alpha, vs); break;
    case OP_SCALE: vy.scale(alpha); break;
    case OP_AXPY: vy.axpy(alpha, vx); break;
    case OP_ADD_LOGBAR_GRAD: vy.addLogBarrierGrad(alpha, vx, vs); break;
    case OP_ADD_LIN_DAMPING: vy.addLinearDampingTerm(vx, vz, alpha, beta); break;
    case OP_TWONORM: ret = vy.twonorm(); break;
    case OP_DOT: ret = vy.dotProductWith(vx); break;
    case OP_INFNORM: ret = vy.infnorm(); break;
    case OP_ONENORM: ret = vy.onenorm(); break;
    case OP_LOGBARRIER: ret = vy.logBarrier_local(vs); break;
    case OP_LIN_DAMPING_TERM: ret = vy.linearDampingTerm_local(vx, vz, alpha, beta); break;
    case OP_MIN_W_PATTERN: ret = vy.min_w_pattern(vs); break;
    case OP_FRAC_TO_BDRY: ret = vy.fractionToTheBdry_local(vx, alpha); break;
    case OP_FRAC_TO_BDRY_W_SEL: ret = vy.fractionToTheBdry_w_pattern_local(vx, alpha, vs); break;
    case OP_SUM: ret = vy.sum_local(); break;
    default: return NAN;
  }
  if(n > 0) memcpy(y, vy.local_data(), sizeof(double) * n);
  return ret;
}

// ---------------------------------------------------------------------------------------------------------
// hiopMatrixDenseRowMajor ops used on the path (a13/a14)
// ---------------------------------------------------------------------------------------------------------
/// y = beta*y + alpha*A*x, A m x n row-major                                  hiopMatrixDenseRowMajor.cpp:436-470
void ref_mat_times_vec(int m, int n, const double* A, double beta, double* y, double alpha, const double* x)
{
  hiopMatrixDenseRowMajor M(m, n);
  memcpy(M.local_data(), A, sizeof(double) * (size_t)m * n);
  hiopVectorPar vy(m), vx(n);
  memcpy(vy.local_data(), y, sizeof(double) * m); memcpy(vx.local_data(), x, sizeof(double) * n);
  M.timesVec(beta, vy, alpha, vx);
  memcpy(y, vy.local_data(), sizeof(double) * m);
}
/// y = beta*y + alpha*A^T*x                                                   :494-528
void ref_mat_trans_times_vec(int m, int n, const double* A, double beta, double* y, double alpha, const double* x)
{
  hiopMatrixDenseRowMajor M(m, n);
  memcpy(M.local_data(), A, sizeof(double) * (size_t)m * n);
  hiopVectorPar vy(n), vx(m);
  memcpy(vy.local_data(), y, sizeof(double) * n); memcpy(vx.local_data(), x, sizeof(double) * m);
  M.transTimesVec(beta, vy, alpha, vx);
  memcpy(y, vy.local_data(), sizeof(double) * n);
}
/// W(Nw x Nw, upper) block starting (row_start, col_start) += alpha * A^T, A m x n      :779-798
void ref_mat_trans_add_to_sym_upper(int m, int n, const double* A, int row_start, int col_start, double alpha, int Nw, double* W)
{
  hiopMatrixDenseRowMajor M(m, n), Wm(Nw, Nw);
  memcpy(M.local_data(), A, sizeof(double) * (size_t)m * n);
  memcpy(Wm.local_data(), W, sizeof(double) * (size_t)Nw * Nw);
  M.transAddToSymDenseMatrixUpperTriangle(row_start, col_start, alpha, Wm);
  memcpy(W, Wm.local_data(), sizeof(double) * (size_t)Nw * Nw);
}
/// W's diagonal block starting at diag_start += alpha * triu(A), A n x n                   :810-829
void ref_mat_add_upper_to_sym_upper(int n, const double* A, int diag_start, double alpha, int Nw, double* W)
{
  hiopMatrixDenseRowMajor M(n, n), Wm(Nw, Nw);
  memcpy(M.local_data(), A, sizeof(double) * (size_t)n * n);
  memcpy(Wm.local_data(), W, sizeof(double) * (size_t)Nw * Nw);
  M.addUpperTriangleToSymDenseMatrixUpperTriangle(diag_start, alpha, Wm);
  memcpy(W, Wm.local_data(), sizeof(double) * (size_t)Nw * Nw);
}
/// W[start+i, start+i] += alpha*d[i]                                                        :719-737
void ref_mat_add_sub_diagonal(int Nw, double* W, int start, double alpha, int nd, const double* d)
{
  hiopMatrixDenseRowMajor Wm(Nw, Nw);
  memcpy(Wm.local_data(), W, sizeof(double) * (size_t)Nw * Nw);
  hiopVectorPar vd(nd);
  memcpy(vd.local_data(), d, sizeof(double) * nd);
  Wm.addSubDiagonal(alpha, start, vd);
  memcpy(W, Wm.local_data(), sizeof(double) * (size_t)Nw * Nw);
}

// ---------------------------------------------------------------------------------------------------------
// hiopMatrixSparseTriplet Schur terms of the MDS KKT build (a14)
// ---------------------------------------------------------------------------------------------------------
/// W diag block at (start,start) += alpha * M * D^{-1} * M^T (upper triangle only)     hiopMatrixSparseTriplet.cpp:390-441
void ref_sp_add_MDinvMtrans(int m, int n, int nnz, const int* iRow, const int* jCol, const double* vals,
                            int start, double alpha, const double* D, int Nw, double* W)
{
  hiopMatrixSparseTriplet M(m, n, nnz);
  memcpy(M.i_row(), iRow, sizeof(int) * nnz); memcpy(M.j_col(), jCol, sizeof(int) * nnz); memcpy(M.M(), vals, sizeof(double) * nnz);
  hiopMatrixDenseRowMajor Wm(Nw, Nw);
  memcpy(Wm.local_data(), W, sizeof(double) * (size_t)Nw * Nw);
  hiopVectorPar vd(n);
  memcpy(vd.local_data(), D, sizeof(double) * n);
  M.addMDinvMtransToDiagBlockOfSymDeMatUTri(start, alpha, vd, Wm);
  memcpy(W, Wm.local_data(), sizeof(double) * (size_t)Nw * Nw);
}
/// W block at (row_start,col_start) += alpha * M1 * D^{-1} * M2^T                        :447-525
void ref_sp_add_MDinvNtrans(int m1, int n, int nnz1, const int* iRow1, const int* jCol1, const double* vals1,
                            int m2, int nnz2, const int* iRow2, const int* jCol2, const double* vals2,
                            int row_start, int col_start, double alpha, const double* D, int Nw, double* W)
{
  hiopMatrixSparseTriplet M1(m1, n, nnz1), M2(m2, n, nnz2);
  memcpy(M1.i_row(), iRow1, sizeof(int) * nnz1); memcpy(M1.j_col(), jCol1, sizeof(int) * nnz1); memcpy(M1.M(), vals1, sizeof(double) * nnz1);
  memcpy(M2.i_row(), iRow2, sizeof(int) * nnz2); memcpy(M2.j_col(), jCol2, sizeof(int) * nnz2); memcpy(M2.M(), vals2, sizeof(double) * nnz2);
  hiopMatrixDenseRowMajor Wm(Nw, Nw);
  memcpy(Wm.local_data(), W, sizeof(double) * (size_t)Nw * Nw);
  hiopVectorPar vd(n);
  memcpy(vd.local_data(), D, sizeof(double) * n);
  M1.addMDinvNtransToSymDeMatUTri(row_start, col_start, alpha, vd, M2, Wm);
  memcpy(W, Wm.local_data(), sizeof(double) * (size_t)Nw * Nw);
}
/// y = beta*y + alpha * M * x (trans = 0) or alpha * M^T * x (trans = 1), M m x n sparse triplet   :73-89, :110-126
void ref_sp_times_vec(int trans, int m, int n, int nnz, const int* iRow, const int* jCol, const double* vals, double beta, double* y,
                      double alpha, const double* x)
{
  hiopMatrixSparseTriplet M(m, n, nnz);
  memcpy(M.i_row(), iRow, sizeof(int) * nnz); memcpy(M.j_col(), jCol, sizeof(int) * nnz); memcpy(M.M(), vals, sizeof(double) * nnz);
  const int ny = trans ? n : m, nx = trans ? m : n;
  hiopVectorPar vy(ny), vx(nx);
  memcpy(vy.local_data(), y, sizeof(double) * ny); memcpy(vx.local_data(), x, sizeof(double) * nx);
  if(trans) M.transTimesVec(beta, vy, alpha, vx);
  else M.timesVec(beta, vy, alpha, vx);
  memcpy(y, vy.local_data(), sizeof(double) * ny);
}

} // extern "C"
