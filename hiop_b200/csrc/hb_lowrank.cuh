// The quasi-Newton KKT handle and the helpers of hb_lowrank.cu that the other files of the IPM vector path call.
#pragma once
#include "hb_common.cuh"
#include "hb_dense.cuh"

constexpr int HB_PANEL_RING = 3; // device slots of a host-resident Jacobian

// Where the columns of J = [Jc; Jd] (m x n) are during a pass over them: nch chunks of csz columns (the last one may be narrower).
// Chunk q is read from slot q % slots at base + (q % slots) * stride, leading dimension ld. With host rows Jc, Jd (ld n), every pass
// copies chunk q into its slot first; without, the slots hold J itself.
//   device J (hb_lowrank_set_jacobian):          one chunk of all n columns, the slot is J, ld n
//   host J (hb_lowrank_set_jacobian_host):       P columns per chunk, HB_PANEL_RING slots of one allocation, ld P + (n mod 2)
//   staged upload (hb_lowrank_kkt_system_host): slot q at hJ + q csz, ld n, for its condensation; a device J on hJ after it
struct hb_jac_layout
{
  long long csz = 0, stride = 0, ld = 0;
  int nch = 1, slots = 1;
  const double* base = nullptr;
  const double *Jc = nullptr, *Jd = nullptr;
  bool from_host() const { return Jc || Jd; }
  const double* chunk(int q) const { return base + (q % slots) * stride; }
};

// a device table of row pointers (hb_syrk_rows) and what it was built from
struct hb_rowtab
{
  hb_dev<const double*> dev;
  hb_pinned<const double*> host;
  long long key[9] = {0};
  bool aligned = false; // every row is 16-byte aligned
};

struct hb_lowrank
{
  hb_ctx* ctx = nullptr;
  long long n = 0;
  int meq = 0, mineq = 0, m = 0, lmax = 0, l = 0;
  double sigma = 1.0;
  // borrowed
  const double *ixl = nullptr, *ixu = nullptr, *idl = nullptr, *idu = nullptr;
  const double *St = nullptr, *Yt = nullptr;
  const double *zl = nullptr, *sxl = nullptr, *zu = nullptr, *sxu = nullptr, *vl = nullptr, *sdl = nullptr, *vu = nullptr, *sdu = nullptr;
  // owned
  hb_dev<double> Dx, DhInv, Dd, Dd_inv;
  // the Jacobian: where its columns are, and what the handle holds of it (the packed copy of a device J given as separate Jc and Jd,
  // the staged upload of hb_lowrank_kkt_system_host, the slots of a host J)
  hb_jac_layout jl;
  hb_dev<double> Jpack, hJ, ring;
  hb_rowtab rows[2]; // the [J; S; Y] tables of the last two layouts, the last one used first (jac_table)
  hb_rowtab sst_rows; // the l rows of S, for S S^T
  // a pass that copies J from the host: the copy stream, its events, the partial C_aug (+ partial fused row dots) of one chunk
  hb_stream copy_stream;
  hb_event copy_start, chunk_ev[4], slot_free[HB_PANEL_RING];
  hb_dev<double> Ctmp;
  hb_dev<double> Caug, SSt, Ld, Dd_sec, V, Mdir, U, Z;
  hb_dev<int> ipivV, ipivM, info; // info[0]: V, info[1]: N chol, info[2]: M
  hb_dev<double> Nmat, F, svec, rhs, dy, work, stats;
  hb_dev<double> nv1, nv2; // n-vector scratch
  hb_dev<double> p2l, md_partial;
  hb_dev<double> mi1, mi2; // m_ineq scratch
  int md_grid = 0;
  bool have_update = false, cond_valid = false, mdir_valid = false;
  int condense_mode = -1; // -1 = auto, 0 = FP64 DMMA, 6/7/8 = INT8-slice wgmma, 100 = INT8 Chinese remaindering
  int condense_used = 0;
  bool check_pending = false; // an asynchronous condensation left its info words unchecked
  hb_dev<double> tri;  // packed upper triangle of C_aug for the all-reduce
  hb_dev<double> tdot; // [J; S; Y] (DhInv .* rx) from the fused row-maximum sweep of an int8-slice condensation (m + 2 lmax)
  bool tdot_valid = false;
  bool rhs_fused = false; // the last solve_compressed formed rhs from tdot (k_fused_rhs)
  // host staging (hb_lowrank_kkt_system_host)
  hb_dev<double> hbuf[14];
  hb_pinned<int> info_host;     // 4 ints
  hb_pinned<double> stats_host; // 4 doubles
  // BiCGStab workspace (hb_krylov.cu), allocated on first use
  hb_dev<double> kry;
  hb_dev<double> kry_m; // 2 m-vectors
  // secant memory owned by the engine (hb_secant.cu): S_t, Y_t (lmax x n), previous iterate / gradient / Jacobian
  hb_dev<double> sec_S, sec_Y, sec_xprev, sec_gprev, sec_Jprev;
  double sec_L[64 * 64] = {0}, sec_D[64] = {0}; // host copies of L (row-major, stride l) and D; lmax <= 64 in this mode
  hb_dev<double> Finv;  // 16 x 16 inverses of the diagonal of F (cooperative Cholesky / solve)
  hb_big big;           // look-ahead Cholesky of large condensed systems: panel stream, events, scratch
  hb_dev<double> lsq_M; // m x m LSQ matrix / Cholesky factor + 2 m-vectors (hb_lsq.cu)
  int sec_lcurr = -1, sec_strategy = 1;
  double sec_sigma0 = 1.0;
};

// The registered Jacobian J = [Jc; Jd] of a handle: every pass runs over the chunks of k->jl, one for a device J (same results for any
// chunking: the J x partials are kept per 2048 columns and summed in one fixed order, each column of J^T y depends on its own column).
bool jac_set(const hb_lowrank* k); // a Jacobian is registered (or m == 0)
// y (m) = beta*y + alpha*J x, summed over the ranks (beta*y on rank 0 only)
int jac_rows(hb_lowrank* k, double beta, double* y, double alpha, const double* x);
// y (n) = beta*y + alpha*J^T x over the local columns (no reduction)
int jac_cols(hb_lowrank* k, double beta, double* y, double alpha, const double* x);
// C (M x M, ldc = M) = R diag(d) R^T over the local columns, R = the first M rows of [J; S; Y]; FP64 DMMA (hb_syrk_rows), with its
// fused extra row when fuse_rx is given (tdot, M doubles)
int jac_syrk(hb_lowrank* k, int M, const double* d, double* C, const double* fuse_rx = nullptr, double* tdot = nullptr);
// The same C by the handle's condensation mode (hb_lowrank_set_condense_mode): jac_syrk, or an int8 kernel over the whole J (refused
// for a J streamed from host memory, the error naming the entry point `who`). With fuse_rx, tdot (M doubles) = R (d .* fuse_rx) where
// that costs no extra pass over J, and *fused tells whether it did: always for the int8 modes, which sweep all rows for their maxima
// anyway; in FP64 only when the extra SYRK row fits in the padding of the last 128-row tile (a whole tile row would cost more than the
// sweep it saves) and fuse_rx is 16-byte aligned (the fast kernel needs it). Never fused for a handle without Jacobian rows (m == 0).
int jac_gram(hb_lowrank* k, const char* who, int M, const double* d, double* C, const double* fuse_rx = nullptr, double* tdot = nullptr,
             bool* fused = nullptr);
// The whole J on the device, for the passes that cannot run chunk by chunk: the int8-slice condensation and LSQ matrix (a global
// row-maximum pass comes first) and the J_prev update of the secant (a device copy of J). *J (m x n, ld n) and *rows (the table of
// [J rows (m); S rows (l); Y rows (l)]) as asked for; HB_ERR_INVALID, naming `who`, for a J streamed from host memory.
int jac_whole(hb_lowrank* k, const char* who, const double** J = nullptr, const hb_rowtab** rows = nullptr);
// k->p2l (device, 2l doubles) = [sigma_s * S (w.*x); Y (w.*x)], all-reduced; w may be NULL
int multidot(hb_lowrank* k, const double* w, const double* x, double sigma_s);
