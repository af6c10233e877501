// hiopKKTLinSysLowRankB200 -- drop-in for hiopKKTLinSysLowRank (src/Optimization/hiopKKTLinSys.hpp:385-460) whose
// update() / solveCompressed() run on the B200 engine. The rhs reduction and the back-substitution stay in the
// inherited hiopKKTLinSysCompressedXYcYd::computeDirections (src/Optimization/hiopKKTLinSys.cpp:585-691), i.e. the
// boundary is exactly the pure-virtual solveCompressed() of the reference (B2 in SURVEY.md section 8b).
//
// Needs read access to the compact-BFGS state of hiopHessianLowRank (S_t, Y_t, L, D, sigma are private,
// src/Optimization/hiopHessianLowRank.hpp:128-160): upstream this is one more `friend class` line next to the existing
// ones; in this repo the adapter translation unit is compiled with -fno-access-control instead.
#pragma once
#include "hiopKKTLinSys.hpp"
#include "hiopHessianLowRank.hpp"
#include "hiopb200.h"

namespace hiop
{
class hiopKKTLinSysLowRankB200 : public hiopKKTLinSysLowRank
{
public:
  hiopKKTLinSysLowRankB200(hiopNlpFormulation* nlp);
  virtual ~hiopKKTLinSysLowRankB200();

  bool update(const hiopIterate* iter, const hiopVector* grad_f, const hiopMatrixDense* Jac_c, const hiopMatrixDense* Jac_d,
              hiopHessianLowRank* Hess) override;
  bool solveCompressed(hiopVector& rx, hiopVector& ryc, hiopVector& ryd, hiopVector& dx, hiopVector& dyc, hiopVector& dyd) override;
  /// Outer BiCGStab refinement (hiopKKTLinSys.cpp:909-960) on the device: one upload of the 12 residual blocks, one download
  /// of the 12 direction blocks; operator, preconditioner and all reductions stay in HBM. HIOP_B200_IR=host keeps the
  /// reference's host-side BiCGStab (which then calls solveCompressed() above for every preconditioner apply).
  bool compute_directions_w_IR(const hiopResidual* resid, hiopIterate* direction) override;

private:
  bool upload(double* dst, const double* src, size_t count);
  hb_ctx* ctx_;
  hb_lowrank* h_;
  long long n_;
  int meq_, mineq_, lmax_;
  // device mirrors
  double *dJ_, *dSt_, *dYt_;
  // HIOP_B200_JAC=host: HiOp's Jacobian buffers are page-locked in place and streamed from the host (no dJ_)
  bool jac_host_ = false;
  void* jac_pinned_[2] = {nullptr, nullptr};
  double* dsec_[4] = {nullptr, nullptr, nullptr, nullptr}; // x, grad_f, yc, yd of the iterate handed to the device-side secant update
  bool secant_ready_ = false;
  int n_secant_dev_ = 0;
  double *dpat_[4], *dit_[8], *drhs_[3], *dsol_[3];
  double *dres_[12], *ddir_[12]; // allocated on the first device-side refinement
  bool ir_on_device_;
  bool healthy_;   // false after an engine error: every entry point then answers false (the reference's failure value), nothing aborts
  // Jacobian traffic and timing (HIOP_B200_STATS=1 prints them when the object dies)
  int n_updates_ = 0, n_jac_uploads_ = 0, n_dirs_ = 0;
  long long jac_evals_seen_ = -1;
  unsigned long long jac_hash_ = 0;
  double jac_bytes_first_ = 0.0, jac_bytes_later_ = 0.0, t_update_ = 0.0, t_dirs_ = 0.0;
};
} // namespace hiop
