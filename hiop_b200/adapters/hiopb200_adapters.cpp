// Implementation of the HiOp-side adapter classes over the C-ABI (include/hiopb200.h).
#include "hiopb200_hooks.hpp"
#include "hiopLinSolverSymDenseB200.hpp"
#include "hiopKKTLinSysLowRankB200.hpp"
#include "hiopHessianLowRankB200.hpp"
#include "hiopLinSolverSymDenseLapack.hpp"
#include "hiopNlpFormulation.hpp"
#include "hiopIterate.hpp"
#include "hiopResidual.hpp"
#include "LinAlgFactory.hpp"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <chrono>

namespace hiop
{
namespace
{
// One engine context per process. A failure (no sm_90 device, ...) is NOT fatal here: the adapters remember it and answer with the
// reference's own failure values -- update() / solve() false, matrixChanged() -1 -- so that the driver escalates exactly as it does for a
// failed factorization (hiopAlgFilterIPM.cpp:1216-1229); nothing in this file calls exit().
hb_ctx* shared_ctx()
{
  static hb_ctx* ctx = nullptr;
  static bool tried = false;
  if(!tried) {
    tried = true;
    const char* dev = getenv("HIOP_B200_DEVICE");
    if(hb_ctx_create(dev ? atoi(dev) : 0, &ctx) != HB_OK) {
      fprintf(stderr, "hiop-b200: %s\n", hb_last_error());
      ctx = nullptr;
    }
  }
  return ctx;
}
// records the first engine error of an adapter object; returns true when rc is HB_OK
bool ok(int rc, const char* what, bool* healthy)
{
  if(rc == HB_OK) return true;
  fprintf(stderr, "hiop-b200: %s failed: %s\n", what, hb_last_error());
  if(healthy) *healthy = false;
  return false;
}
// 64-bit FNV-1a over the raw bytes: constant-Jacobian detection for problems that do not declare themselves linear (small J only)
unsigned long long fnv1a(const void* p, size_t bytes)
{
  const unsigned long long* w = static_cast<const unsigned long long*>(p);
  unsigned long long h = 1469598103934665603ull;
  for(size_t i = 0; i < bytes / 8; i++) { h ^= w[i]; h *= 1099511628211ull; }
  return h;
}
} // namespace

bool hiop_b200_enabled()
{
  const char* e = getenv("HIOP_B200");
  return e && atoi(e) != 0;
}

hiopKKTLinSysLowRank* hiop_b200_new_lowrank_kkt(hiopNlpFormulation* nlp)
{
  if(hiop_b200_enabled()) return new hiopKKTLinSysLowRankB200(nlp);
  return new hiopKKTLinSysLowRank(nlp);
}

hiopLinSolverSymDense* hiop_b200_new_symdense_solver(int n, hiopNlpFormulation* nlp, const bool* safe_mode)
{
  if(hiop_b200_enabled()) return new hiopLinSolverSymDenseB200(n, nlp, safe_mode);
  return new hiopLinSolverSymDenseLapack(n, nlp);
}

hiopMatrix* hiop_b200_new_hessian_lowrank(hiopNlpDenseConstraints* nlp, int max_memory_length)
{
  if(hiop_b200_enabled()) return new hiopHessianLowRankB200(nlp, max_memory_length);
  return new hiopHessianLowRank(nlp, max_memory_length);
}

// ---------------------------------------------------------------------------------------------------------
hiopHessianLowRankB200::hiopHessianLowRankB200(hiopNlpDenseConstraints* nlp, int max_memory_length)
  : hiopHessianLowRank(nlp, max_memory_length), device_mode_(false), pending_(0)
{
  const char* e = getenv("HIOP_B200_SECANT");
  const char* ir = getenv("HIOP_B200_IR");
  // the host-side BiCGStab of HIOP_B200_IR=host applies this object's timesVec, which needs S_t / Y_t on the host
  device_mode_ = e && !strcmp(e, "device") && !(ir && !strcmp(ir, "host")) && max_memory_length <= 64;
}

bool hiopHessianLowRankB200::update(const hiopIterate& x_curr, const hiopVector& grad_f_curr, const hiopMatrix& Jac_c_curr,
                                    const hiopMatrix& Jac_d_curr)
{
  if(!device_mode_) return hiopHessianLowRank::update(x_curr, grad_f_curr, Jac_c_curr, Jac_d_curr);
  pending_++; // carried out by hiopKKTLinSysLowRankB200::update, which is called with the same iterate next (hiopAlgFilterIPM.cpp:1215-1216)
  pending_grad_f_ = &grad_f_curr;
  pending_it_ = &x_curr;
  return true;
}

double hiopHessianLowRankB200::sigma0_value() const { return sigma0; }
int hiopHessianLowRankB200::sigma_strategy_value() const { return sigma_update_strategy; }

void hiopHessianLowRankB200::mirror(int l, double sigma_new, const double* L_host, const double* D_host)
{
  sigma = sigma_new;
  l_curr = l;
  // L_ (l x l) and D_ (l) are resized by the base class as the memory grows (growL / growD, hiopHessianLowRank.cpp:779-823); here they
  // are re-created at the mirrored size
  if(L_->m() != l) {
    delete L_;
    delete D_;
    L_ = LinearAlgebraFactory::create_matrix_dense("DEFAULT", l, l);
    D_ = LinearAlgebraFactory::create_vector("DEFAULT", l);
  }
  if(l > 0) {
    memcpy(L_->local_data(), L_host, sizeof(double) * (size_t)l * l);
    memcpy(D_->local_data(), D_host, sizeof(double) * (size_t)l);
  }
}

// ---------------------------------------------------------------------------------------------------------
hiopLinSolverSymDenseB200::hiopLinSolverSymDenseB200(int n, hiopNlpFormulation* nlp, const bool* safe_mode)
  : hiopLinSolverSymDense(n, nlp), ctx_(shared_ctx()), h_(nullptr), safe_mode_(safe_mode), healthy_(true)
{
  if(!ctx_) { healthy_ = false; return; }
  ok(hb_symdense_create(ctx_, n, &h_), "hb_symdense_create", &healthy_);
}
hiopLinSolverSymDenseB200::~hiopLinSolverSymDenseB200() { if(h_) hb_symdense_destroy(h_); }

int hiopLinSolverSymDenseB200::matrixChanged()
{
  if(!healthy_) return -1;
  // The factorization follows the KKT object's CURRENT safe mode (read through the pointer on every call): Bunch-Kaufman when
  // safe_mode is on (MagmaBuKa role), LDL^T without pivoting otherwise (MagmaNopiv role). The non-MAGMA build of the reference
  // never re-creates linSys_ when safe_mode flips (hiopKKTLinSysMDS.cpp:405-430 does so only under HIOP_USE_MAGMA), so a mode
  // frozen at construction would lose the reference's stability fallback.
  int mode = (safe_mode_ == nullptr || *safe_mode_) ? HB_FACT_BUNCH_KAUFMAN : HB_FACT_NOPIV;
  // "bk" | "nopiv": overrides the safe_mode choice; "rbt": the random-butterfly safe mode wherever Bunch-Kaufman would run
  const char* force = getenv("HIOP_B200_LINSOL");
  if(force && !strcmp(force, "bk")) mode = HB_FACT_BUNCH_KAUFMAN;
  if(force && !strcmp(force, "nopiv")) mode = HB_FACT_NOPIV;
  if(force && !strcmp(force, "rbt") && mode == HB_FACT_BUNCH_KAUFMAN) mode = HB_FACT_RBT_NOPIV;
  nlp_->runStats.linsolv.tmFactTime.start();
  // M_ lives in host memory (mem_space=default): upload + factorize (the MAGMA twin does the same H2D per factorization,
  // hiopLinSolverSymDenseMagma.cpp:139-146)
  const int ret = hb_symdense_matrix_changed_host(h_, M_->local_data(), mode);
  nlp_->runStats.linsolv.tmFactTime.stop();
  if(ret < -1) {
    nlp_->log->printf(hovError, "hiopLinSolverSymDenseB200: %s\n", hb_last_error());
    return -1;
  }
  return ret;
}

bool hiopLinSolverSymDenseB200::solve(hiopVector& x)
{
  if(!healthy_) return false;
  nlp_->runStats.linsolv.tmTriuSolves.start();
  const int rc = hb_symdense_solve_host(h_, x.local_data(), 1);
  nlp_->runStats.linsolv.tmTriuSolves.stop();
  return rc == 1;
}

// ---------------------------------------------------------------------------------------------------------
hiopKKTLinSysLowRankB200::hiopKKTLinSysLowRankB200(hiopNlpFormulation* nlp)
  : hiopKKTLinSysLowRank(nlp), ctx_(shared_ctx()), h_(nullptr), dJ_(nullptr), dSt_(nullptr), dYt_(nullptr), healthy_(true)
{
  for(int i = 0; i < 12; i++) dres_[i] = ddir_[i] = nullptr;
  for(auto*& p : dpat_) p = nullptr;
  for(auto*& p : dit_) p = nullptr;
  for(auto*& p : drhs_) p = nullptr;
  for(auto*& p : dsol_) p = nullptr;
  const char* ir = getenv("HIOP_B200_IR");
  ir_on_device_ = !(ir && !strcmp(ir, "host"));
  n_ = nlp_->n_local();
  meq_ = nlp_->m_eq();
  mineq_ = nlp_->m_ineq();
  lmax_ = nlp_->options->GetInteger("secant_memory_len");
  if(!ctx_) { healthy_ = false; return; }
#ifdef HIOP_USE_MPI
  if(nlp_->get_num_ranks() > 1) {
    // the engine context of this adapter is single-GPU: with an MPI-distributed HiOp the condensed matrix, the multi-dots and J dx
    // would be reduced over the local columns only. (The C-ABI itself shards over NCCL, hb_comm_init; bootstrapping its id over MPI is
    // the missing piece.) Refuse instead of computing wrong directions.
    fprintf(stderr, "hiop-b200: hiopKKTLinSysLowRankB200 does not support MPI-distributed problems (%d ranks); use the reference classes\n",
            nlp_->get_num_ranks());
    healthy_ = false;
    return;
  }
#endif
  if(!ok(hb_lowrank_create(ctx_, n_, meq_, mineq_, lmax_ > 0 ? lmax_ : 1, &h_), "hb_lowrank_create", &healthy_)) return;
  const size_t m = (size_t)meq_ + mineq_;
  const char* jac = getenv("HIOP_B200_JAC");
  jac_host_ = jac && !strcmp(jac, "host");
  bool a = jac_host_ || ok(hb_malloc(ctx_, sizeof(double) * m * n_, (void**)&dJ_), "hb_malloc(J)", &healthy_);
  a = a && ok(hb_malloc(ctx_, sizeof(double) * (size_t)(lmax_ > 0 ? lmax_ : 1) * n_, (void**)&dSt_), "hb_malloc(S)", &healthy_);
  a = a && ok(hb_malloc(ctx_, sizeof(double) * (size_t)(lmax_ > 0 ? lmax_ : 1) * n_, (void**)&dYt_), "hb_malloc(Y)", &healthy_);
  const size_t psz[4] = {(size_t)n_, (size_t)n_, (size_t)mineq_, (size_t)mineq_};
  for(int i = 0; i < 4 && a; i++) a = ok(hb_malloc(ctx_, sizeof(double) * psz[i], (void**)&dpat_[i]), "hb_malloc(pattern)", &healthy_);
  const size_t isz[8] = {(size_t)n_, (size_t)n_, (size_t)n_, (size_t)n_, (size_t)mineq_, (size_t)mineq_, (size_t)mineq_, (size_t)mineq_};
  for(int i = 0; i < 8 && a; i++) a = ok(hb_malloc(ctx_, sizeof(double) * isz[i], (void**)&dit_[i]), "hb_malloc(iterate)", &healthy_);
  const size_t rsz[3] = {(size_t)n_, (size_t)meq_, (size_t)mineq_};
  for(int i = 0; i < 3 && a; i++) {
    a = ok(hb_malloc(ctx_, sizeof(double) * rsz[i], (void**)&drhs_[i]), "hb_malloc(rhs)", &healthy_);
    a = a && ok(hb_malloc(ctx_, sizeof(double) * rsz[i], (void**)&dsol_[i]), "hb_malloc(sol)", &healthy_);
  }
  if(!a) return;
  // patterns are fixed for the lifetime of the formulation
  upload(dpat_[0], nlp_->get_ixl().local_data_const(), n_);
  upload(dpat_[1], nlp_->get_ixu().local_data_const(), n_);
  upload(dpat_[2], nlp_->get_idl().local_data_const(), mineq_);
  upload(dpat_[3], nlp_->get_idu().local_data_const(), mineq_);
  ok(hb_lowrank_set_patterns(h_, dpat_[0], dpat_[1], dpat_[2], dpat_[3]), "hb_lowrank_set_patterns", &healthy_);
}

hiopKKTLinSysLowRankB200::~hiopKKTLinSysLowRankB200()
{
  if(getenv("HIOP_B200_STATS") && n_updates_ > 0) {
    // per-iteration KKT time of the engine path, next to the reference's own tmSolverInternal / time_kkt output
    fprintf(stderr, "hiop-b200 stats: updates %d, Jacobian uploads %d (first %.0f bytes, after the first %.0f bytes), KKT update+condense %.3f ms/it, "
            "directions %.3f ms/call (%d calls), secant updates on the device %d\n", n_updates_, n_jac_uploads_, jac_bytes_first_, jac_bytes_later_,
            1e3 * t_update_ / n_updates_, n_dirs_ ? 1e3 * t_dirs_ / n_dirs_ : 0.0, n_dirs_, n_secant_dev_);
  }
  if(h_) hb_lowrank_destroy(h_);
  if(!ctx_) return;
  for(void* p : jac_pinned_) if(p) hb_host_unregister(ctx_, p);
  hb_free(ctx_, dJ_); hb_free(ctx_, dSt_); hb_free(ctx_, dYt_);
  for(auto* p : dsec_) if(p) hb_free(ctx_, p);
  for(auto* p : dpat_) hb_free(ctx_, p);
  for(auto* p : dit_) hb_free(ctx_, p);
  for(auto* p : drhs_) hb_free(ctx_, p);
  for(auto* p : dsol_) hb_free(ctx_, p);
  for(auto* p : dres_) if(p) hb_free(ctx_, p);
  for(auto* p : ddir_) if(p) hb_free(ctx_, p);
}

bool hiopKKTLinSysLowRankB200::upload(double* dst, const double* src, size_t count)
{
  if(count == 0) return true;
  return ok(hb_memcpy_h2d(ctx_, dst, src, sizeof(double) * count), "hb_memcpy_h2d", &healthy_);
}

bool hiopKKTLinSysLowRankB200::update(const hiopIterate* iter, const hiopVector* grad_f, const hiopMatrixDense* Jac_c,
                                      const hiopMatrixDense* Jac_d, hiopHessianLowRank* Hess)
{
  if(!healthy_) return false;
  // host bookkeeping of the reference (Dx_, Dd_inv_, DhInv are still read by the inherited computeDirections and by the
  // full-KKT operator of the outer BiCGStab refinement, hiopKKTLinSys.cpp:1619-1733)
  if(!hiopKKTLinSysLowRank::update(iter, grad_f, Jac_c, Jac_d, Hess)) return false;
  nlp_->runStats.tmSolverInternal.start();
  const auto t0 = std::chrono::steady_clock::now();
  // Jacobian [Jc;Jd] -> device (the user callbacks write host memory, hiopNlpFormulation.cpp:1499-1533), but ONLY when it changed:
  //  * the formulation re-evaluates the Jacobian of a problem declared linear / quadratic once (hiopNlpFormulation.cpp:1548-1551,
  //    1586-1589): its evaluation counters tell whether the callback ran since the last upload;
  //  * small Jacobians (<= 64 MB) are additionally fingerprinted, which catches constant Jacobians of problems that do not declare
  //    themselves linear (the bundled NlpDenseConsEx1/Ex2 re-evaluate theirs every iteration with identical values).
  const size_t jbytes = sizeof(double) * ((size_t)meq_ + mineq_) * n_;
  if(jac_host_) {
    // HIOP_B200_JAC=host: the engine reads [Jc; Jd] where HiOp's callbacks write it, streaming it through device panels on every pass.
    // Its buffers are page-locked once (and again only if the formulation ever hands over different ones).
    const double* src[2] = {Jac_c->local_data_const(), Jac_d->local_data_const()};
    const size_t bytes[2] = {sizeof(double) * (size_t)meq_ * n_, sizeof(double) * (size_t)mineq_ * n_};
    bool reg = false;
    for(int i = 0; i < 2; i++) {
      void* p = bytes[i] ? const_cast<double*>(src[i]) : nullptr;
      if(p == jac_pinned_[i]) continue;
      if(jac_pinned_[i]) hb_host_unregister(ctx_, jac_pinned_[i]);
      jac_pinned_[i] = nullptr;
      if(p && !ok(hb_host_register(ctx_, p, bytes[i]), "hb_host_register(J)", &healthy_)) return false;
      jac_pinned_[i] = p;
      reg = true;
    }
    if(reg || n_jac_uploads_ == 0) {
      if(!ok(hb_lowrank_set_jacobian_host(h_, src[0], src[1], 0), "hb_lowrank_set_jacobian_host", &healthy_)) return false;
      n_jac_uploads_++;
    }
  }
  const long long evals = (long long)nlp_->runStats.nEvalJac_con_eq + nlp_->runStats.nEvalJac_con_ineq;
  bool changed = !jac_host_ && ((n_jac_uploads_ == 0) || (evals != jac_evals_seen_));
  unsigned long long hash = 0;
  if(changed && n_jac_uploads_ > 0 && jbytes <= ((size_t)64 << 20)) {
    hash = fnv1a(Jac_c->local_data_const(), sizeof(double) * (size_t)meq_ * n_) ^ (fnv1a(Jac_d->local_data_const(), sizeof(double) * (size_t)mineq_ * n_) * 31);
    if(hash == jac_hash_) changed = false;
  } else if(n_jac_uploads_ == 0 && jbytes <= ((size_t)64 << 20)) {
    hash = fnv1a(Jac_c->local_data_const(), sizeof(double) * (size_t)meq_ * n_) ^ (fnv1a(Jac_d->local_data_const(), sizeof(double) * (size_t)mineq_ * n_) * 31);
  }
  jac_evals_seen_ = evals;
  if(changed) {
    upload(dJ_, Jac_c->local_data_const(), (size_t)meq_ * n_);
    upload(dJ_ + (size_t)meq_ * n_, Jac_d->local_data_const(), (size_t)mineq_ * n_);
    if(n_jac_uploads_ == 0) jac_bytes_first_ += (double)jbytes; else jac_bytes_later_ += (double)jbytes;
    n_jac_uploads_++;
    jac_hash_ = hash;
    if(!ok(hb_lowrank_set_jacobian(h_, dJ_, dJ_ + (size_t)meq_ * n_), "hb_lowrank_set_jacobian", &healthy_)) return false;
  }
  hiopHessianLowRankB200* hdev = dynamic_cast<hiopHessianLowRankB200*>(Hess);
  static const bool trace = getenv("HIOP_B200_TRACE") != nullptr;
#define TR(msg) do { if(trace) { fprintf(stderr, "hiop-b200 trace: %s\n", msg); fflush(stderr); } } while(0)
  TR("update: secant stage");
  if(hdev && hdev->device_mode()) {
    // a11 on the device: the iterate(s) hiopHessianLowRankB200::update noted are applied here, with the Jacobian registered just above
    if(!secant_ready_) {
      if(!ok(hb_lowrank_secant_reset(h_, hdev->sigma0_value(), hdev->sigma_strategy_value()), "hb_lowrank_secant_reset", &healthy_)) return false;
      for(int i = 0; i < 2; i++)
        if(!ok(hb_malloc(ctx_, sizeof(double) * (size_t)(n_ > 0 ? n_ : 1), (void**)&dsec_[i]), "hb_malloc(secant)", &healthy_)) return false;
      if(!ok(hb_malloc(ctx_, sizeof(double) * (size_t)(meq_ > 0 ? meq_ : 1), (void**)&dsec_[2]), "hb_malloc(secant)", &healthy_)) return false;
      if(!ok(hb_malloc(ctx_, sizeof(double) * (size_t)(mineq_ > 0 ? mineq_ : 1), (void**)&dsec_[3]), "hb_malloc(secant)", &healthy_)) return false;
      secant_ready_ = true;
      TR("secant reset done");
    }
    const int pend = hdev->take_pending();
    if(pend > 0) {
      const hiopIterate* its = hdev->pending_iterate();
      const hiopVector* gs = hdev->pending_grad_f();
      if(!its || !gs) {
        nlp_->log->printf(hovError, "hiopKKTLinSysLowRankB200::update: the quasi-Newton update did not leave its iterate / gradient\n");
        return false;
      }
      upload(dsec_[0], its->x->local_data_const(), n_);
      upload(dsec_[1], gs->local_data_const(), n_);
      upload(dsec_[2], its->yc->local_data_const(), meq_);
      upload(dsec_[3], its->yd->local_data_const(), mineq_);
      int status = 0;
      TR("secant uploads done");
      if(!ok(hb_lowrank_secant_update(h_, dsec_[0], dsec_[1], dsec_[2], dsec_[3], 0, &status), "hb_lowrank_secant_update", &healthy_)) return false;
      TR("secant update done");
      int l = 0;
      double sg = 0.0, Lh[64 * 64], Dh[64];
      if(!ok(hb_lowrank_secant_state(h_, &l, &sg, nullptr, nullptr, Lh, Dh), "hb_lowrank_secant_state", &healthy_)) return false;
      TR("secant state read");
      hdev->mirror(l, sg, Lh, Dh);
      TR("mirrored");
      n_secant_dev_++;
    }
  } else {
    // secant memory as hiopHessianLowRank::update left it on the host (hiopHessianLowRank.cpp:262-388)
    const int l = Hess->St_->m();
    if(l > 0) {
      upload(dSt_, Hess->St_->local_data_const(), (size_t)l * n_);
      upload(dYt_, Hess->Yt_->local_data_const(), (size_t)l * n_);
    }
    if(!ok(hb_lowrank_set_secant(h_, l, Hess->sigma, dSt_, dYt_, l ? Hess->L_->local_data_const() : nullptr, l ? Hess->D_->local_data_const() : nullptr),
           "hb_lowrank_set_secant", &healthy_))
      return false;
  }
  TR("update: iterate upload");
  const hiopVector* blocks[8] = {iter->zl, iter->sxl, iter->zu, iter->sxu, iter->vl, iter->sdl, iter->vu, iter->sdu};
  for(int i = 0; i < 8; i++) upload(dit_[i], blocks[i]->local_data_const(), blocks[i]->get_size());
  if(!healthy_) return false;
  if(!ok(hb_lowrank_update(h_, dit_[0], dit_[1], dit_[2], dit_[3], dit_[4], dit_[5], dit_[6], dit_[7]), "hb_lowrank_update", &healthy_)) return false;
  // N and its factor depend only on the state set above: condense ONCE per update(); every preconditioner apply of the
  // outer BiCGStab then reuses it (the reference rebuilds and refactorizes N on each solveCompressed call).
  // HB_ERR_NUMERIC (V singular / N not SPD; the engine does not retry) is the reference's "update failed": return false and let
  // the driver escalate (hiopAlgFilterIPM.cpp:1216-1229); the adapter stays usable.
  TR("update: condense");
  const int rc = hb_lowrank_condense(h_);
  TR("update: condensed");
  t_update_ += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  n_updates_++;
  nlp_->runStats.tmSolverInternal.stop();
  if(rc != HB_OK) {
    nlp_->log->printf(hovError, "hiopKKTLinSysLowRankB200::update: %s\n", hb_last_error());
    return false;
  }
  return true;
}

#undef TR

bool hiopKKTLinSysLowRankB200::solveCompressed(hiopVector& rx, hiopVector& ryc, hiopVector& ryd, hiopVector& dx, hiopVector& dyc,
                                               hiopVector& dyd)
{
  if(!healthy_) return false;
  upload(drhs_[0], rx.local_data_const(), n_);
  upload(drhs_[1], ryc.local_data_const(), meq_);
  upload(drhs_[2], ryd.local_data_const(), mineq_);
  const int rc = hb_lowrank_solve_compressed(h_, drhs_[0], drhs_[1], drhs_[2], dsol_[0], dsol_[1], dsol_[2]);
  if(rc != HB_OK) {
    nlp_->log->printf(hovError, "hiopKKTLinSysLowRankB200::solveCompressed: %s\n", hb_last_error());
    return false;
  }
  bool a = true;
  if(n_) a = a && ok(hb_memcpy_d2h(ctx_, dx.local_data(), dsol_[0], sizeof(double) * n_), "d2h", &healthy_);
  if(meq_) a = a && ok(hb_memcpy_d2h(ctx_, dyc.local_data(), dsol_[1], sizeof(double) * meq_), "d2h", &healthy_);
  if(mineq_) a = a && ok(hb_memcpy_d2h(ctx_, dyd.local_data(), dsol_[2], sizeof(double) * mineq_), "d2h", &healthy_);
  // like the reference, rx is overwritten with rx - J^T [dyc;dyd] (hiopKKTLinSys.cpp:1178)
  if(n_) a = a && ok(hb_memcpy_d2h(ctx_, rx.local_data(), drhs_[0], sizeof(double) * n_), "d2h", &healthy_);
  a = a && ok(hb_ctx_sync(ctx_), "hb_ctx_sync", &healthy_);
  return a;
}

bool hiopKKTLinSysLowRankB200::compute_directions_w_IR(const hiopResidual* resid, hiopIterate* dir)
{
  const int maxit = nlp_->options->GetInteger("ir_outer_maxit");
  if(!healthy_) return false;
  if(!ir_on_device_ || maxit <= 0) return hiopKKTLinSys::compute_directions_w_IR(resid, dir);
  nlp_->runStats.tmSolverInternal.start();
  const auto t0 = std::chrono::steady_clock::now();
  // compound order of hiopVectorCompoundPD (hiopVectorCompoundPD.cpp:228-255)
  const hiopVector* rb[12] = {resid->rx, resid->rd, resid->ryc, resid->ryd, resid->rxl, resid->rxu, resid->rdl, resid->rdu,
                              resid->rszl, resid->rszu, resid->rsvl, resid->rsvu};
  hiopVector* db[12] = {dir->x, dir->d, dir->yc, dir->yd, dir->sxl, dir->sxu, dir->sdl, dir->sdu, dir->zl, dir->zu, dir->vl, dir->vu};
  for(int i = 0; i < 12; i++) {
    const size_t sz = (size_t)rb[i]->get_size();
    if(!dres_[i]) {
      if(!ok(hb_malloc(ctx_, sizeof(double) * sz, (void**)&dres_[i]), "hb_malloc(residual)", &healthy_) ||
         !ok(hb_malloc(ctx_, sizeof(double) * sz, (void**)&ddir_[i]), "hb_malloc(direction)", &healthy_)) {
        nlp_->runStats.tmSolverInternal.stop();
        return false;
      }
    }
    upload(dres_[i], rb[i]->local_data_const(), sz);
  }
  const double tol = std::min(mu_ * nlp_->options->GetNumeric("ir_outer_tol_factor"), nlp_->options->GetNumeric("ir_outer_tol_min"));
  double info[4] = {0, 0, 0, 0};
  const int rc = hb_lowrank_compute_directions_w_ir(h_, dres_, ddir_, tol, maxit, info);
  if(rc != HB_OK) {
    nlp_->log->printf(hovError, "hiopKKTLinSysLowRankB200::compute_directions_w_IR: %s\n", hb_last_error());
    nlp_->runStats.tmSolverInternal.stop();
    return false;
  }
  bool a = true;
  for(int i = 0; i < 12; i++) {
    const size_t sz = (size_t)db[i]->get_size();
    if(sz) a = a && ok(hb_memcpy_d2h(ctx_, db[i]->local_data(), ddir_[i], sizeof(double) * sz), "d2h", &healthy_);
  }
  a = a && ok(hb_ctx_sync(ctx_), "hb_ctx_sync", &healthy_);
  t_dirs_ += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  n_dirs_++;
  if(!a) {
    nlp_->runStats.tmSolverInternal.stop();
    return false;
  }
  nlp_->runStats.kkt.nIterRefinInner += info[1];
  if(info[0] != 0.0)  // the step is accepted whatever BiCGStab reports (hiopKKTLinSys.cpp:950-953)
    nlp_->log->printf(hovWarning, "BiCGStab (device) did NOT converge: flag %d after %g iters, abs res %g, rel res %g\n", (int)info[0], info[1],
                      info[2], info[3]);
  else
    nlp_->log->printf(hovScalars, "BiCGStab (device) converged: actual normResid=%g relResid=%g iter=%g\n", info[2], info[3], info[1]);
  nlp_->runStats.tmSolverInternal.stop();
  return true;
}

} // namespace hiop
