// The quasi-Newton KKT handle and the helpers of hb_lowrank.cu that the other files of the IPM vector path call.
#pragma once
#include "hb_common.cuh"
#include "hb_dense.cuh"

constexpr int HB_PANEL_RING = 3; // device panels of a host-resident Jacobian

struct hb_lowrank
{
  hb_ctx* ctx = nullptr;
  long long n = 0;
  int meq = 0, mineq = 0, m = 0, lmax = 0, l = 0;
  double sigma = 1.0;
  // borrowed
  const double *ixl = nullptr, *ixu = nullptr, *idl = nullptr, *idu = nullptr;
  const double *J = nullptr, *St = nullptr, *Yt = nullptr;
  const double *zl = nullptr, *sxl = nullptr, *zu = nullptr, *sxu = nullptr, *vl = nullptr, *sdl = nullptr, *vu = nullptr, *sdu = nullptr;
  // owned
  hb_dev<double> Dx, DhInv, Dd, Dd_inv;
  hb_dev<double> Jpack;
  hb_dev<const double*> rowptr_dev;
  hb_pinned<const double*> rowptr_host;
  bool rows_aligned = false, rowptr_dirty = true;
  hb_dev<double> Caug, SSt, Ld, Dd_sec, V, Mdir, U, Z;
  hb_dev<int> ipivV, ipivM, info; // info[0]: V, info[1]: N chol, info[2]: M
  hb_dev<double> Nmat, F, svec, rhs, dy, work, stats;
  hb_dev<double> nv1, nv2; // n-vector scratch
  hb_dev<double> p2l, md_partial;
  hb_dev<double> mi1, mi2; // m_ineq scratch
  int md_grid = 0;
  bool have_update = false, cond_valid = false, mdir_valid = false;
  int condense_mode = -1; // -1 = auto, 0 = FP64 DMMA, 6/7/8 = INT8-slice wgmma
  int condense_used = 0;
  bool check_pending = false; // an asynchronous condensation left its info words unchecked
  hb_dev<double> tri;  // packed upper triangle of C_aug for the all-reduce
  hb_dev<double> tdot; // [J; S; Y] (DhInv .* rx) from the fused row-maximum sweep of an int8-slice condensation (m + 2 lmax)
  bool tdot_valid = false;
  // host staging (hb_lowrank_kkt_system_host)
  hb_dev<double> hbuf[14];
  hb_dev<double> hJ;
  hb_pinned<int> info_host;     // 4 ints
  hb_pinned<double> stats_host; // 4 doubles
  // BiCGStab workspace (hb_krylov.cu), allocated on first use
  hb_dev<double> kry;
  hb_dev<double> kry_m; // 2 m-vectors
  // secant memory owned by the engine (hb_secant.cu): S_t, Y_t (lmax x n), previous iterate / gradient / Jacobian
  hb_dev<double> sec_S, sec_Y, sec_xprev, sec_gprev, sec_Jprev;
  double sec_L[64 * 64] = {0}, sec_D[64] = {0}; // host copies of L (row-major, stride l) and D; lmax <= 64 in this mode
  // host-resident Jacobian (hb_lowrank_set_jacobian_host): borrowed page-locked rows of Jc and Jd (ld = n), streamed through a ring of
  // device panels of panel_cols columns (leading dimension panel_ld); panel_cols == 0: J is on the device (k->J)
  const double *Jc_host = nullptr, *Jd_host = nullptr;
  long long panel_cols = 0, panel_ld = 0;
  hb_dev<double> panel[HB_PANEL_RING];
  hb_event panel_free[HB_PANEL_RING]; // the context stream is done with a ring slot
  // column chunks of J copied on a second stream while the context stream consumes earlier ones: the condensation of
  // hb_lowrank_kkt_system_host and every pass over a host-resident J
  hb_stream copy_stream;
  hb_event copy_start, chunk_ev[4];
  hb_dev<double> Ctmp; // partial C_aug (+ partial fused row dots) of one chunk
  hb_dev<const double*> chunk_rowptr_dev;
  hb_pinned<const double*> chunk_rowptr_host; // rows of [J; S; Y] per chunk (chunks x (m + 2 l))
  long long chunk_key[8] = {0};               // what chunk_rowptr_dev was built for
  bool chunk_rows_aligned = false;
  hb_dev<double> Finv;  // 16 x 16 inverses of the diagonal of F (cooperative Cholesky / solve)
  hb_big big;           // look-ahead Cholesky of large condensed systems: panel stream, events, scratch
  hb_dev<double> lsq_M; // m x m LSQ matrix / Cholesky factor + 2 m-vectors (hb_lsq.cu)
  int sec_lcurr = -1, sec_strategy = 1;
  double sec_sigma0 = 1.0;
};

// The Jacobian gemvs (hb_lowrank.cu) for an m x n row-major A with leading dimension lda (elements), n = the local columns.
// y = beta*y + alpha*A x, summed over the ranks (beta*y on rank 0 only)
int gemv_rows(hb_ctx* c, int m, long long n, const double* A, long long lda, double beta, double* y, double alpha, const double* x);
// y = beta*y + alpha*A^T x over the local columns (no reduction)
int gemv_cols(hb_ctx* c, int m, long long n, const double* A, long long lda, double beta, double* y, double alpha, const double* x);
// The registered Jacobian J = [Jc; Jd] of a handle, on the device or streamed from the host in column panels (same results: the J x
// partials are kept per 2048 columns and summed in one fixed order, each column of J^T y depends on its own column only).
bool jac_set(const hb_lowrank* k); // a Jacobian is registered (or m == 0)
// y (m) = beta*y + alpha*J x, all-reduced like gemv_rows
int jac_rows(hb_lowrank* k, double beta, double* y, double alpha, const double* x);
// y (n) = beta*y + alpha*J^T x
int jac_cols(hb_lowrank* k, double beta, double* y, double alpha, const double* x);
// C (M x M, ldc = M) = R diag(d) R^T over the local columns, R = the first M rows of [J; S; Y]; FP64 DMMA (hb_syrk_rows), with its
// fused extra row when fuse_rx is given (tdot, M doubles)
int jac_syrk(hb_lowrank* k, int M, const double* d, double* C, const double* fuse_rx = nullptr, double* tdot = nullptr);
// k->p2l (device, 2l doubles) = [sigma_s * S (w.*x); Y (w.*x)], all-reduced; w may be NULL
int multidot(hb_lowrank* k, const double* w, const double* x, double sigma_s);
// device table of row pointers [J rows (m); S rows (l); Y rows (l)] -> k->rowptr_dev, k->rows_aligned
int refresh_rowptr(hb_lowrank* k);
