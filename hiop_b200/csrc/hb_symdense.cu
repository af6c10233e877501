// Dense symmetric factorizations / solves: which kernels run for every caller, and hiopLinSolverSymDense on device (B1): matrixChanged() /
// solve() semantics of src/LinAlg/hiopLinSolverSymDenseLapack.hpp:75-192 and the MAGMA twins hiopLinSolverSymDenseMagma.cpp:120-270, 324-476.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include <cstdlib>

// ---------------------------------------------------------------------------------------------------------------------------------------
// The dispatch, in one place. N = order; "coop" = the single-launch cooperative kernels of hb_chol_coop.cu, "panels" = 64-wide panel +
// trailing-update launches (hb_dense.cu), "look-ahead" = hb_dense_big.cu, "blocked solve" = hb_big_solve with 128 x 128 inverses.
//
//   caller        mode   N                                 factor                                 solve                          inertia
//   symdense      BK     >= bk_cluster_min (385), fits     cluster BK (odd N: padded copy)        blocked, permuted              parallel, ipiv + dsub
//                 BK     96 .. cluster                     one-CTA DLASYF panels + trailing       DSYTRS                         serial, LAPACK ipiv
//                 BK     < 96                              DSYTF2, one CTA                        DSYTRS                         serial, LAPACK ipiv
//                 NOPIV  >= big_min_ldl (257)              look-ahead LDL^T (odd N: padded copy)  blocked                        parallel, diagonal
//                 NOPIV  < big_min_ldl                     panels                                 blocked from 257, else one CTA parallel, diagonal
//                 RBT    any                               k_rbt_fused (hb_rbt.cu), then NOPIV's   U^T, NOPIV's, refinement, U    NOPIV's
//                 CHOL   >= big_min_chol (1025)            look-ahead (odd N: padded copy)        blocked                        parallel, diagonal
//                 CHOL   65 .. 2048 and < big_min_chol     coop                                   blocked from 257, else one CTA parallel, diagonal
//                 CHOL   other                             panels                                 blocked from 257, else one CTA parallel, diagonal
//   condensed N   CHOL   65 .. 2048                        coop + 16 x 16 inverses                coop up to 16384, else one-CTA refinement
//   (hb_lowrank)  CHOL   > 2048, even ld, aligned          look-ahead + 16 x 16 inverses          idem
//                 CHOL   other                             panels (+ 16 x 16 inverses if > 64)    idem (one-CTA refinement if <= 64)
//   LSQ duals     CHOL   65 .. 2048                        coop                                   one CTA
//                 CHOL   other                             panels                                 one CTA
//   V, Mdir       BK     any                               DSYTF2                                 DSYTRS
//
// RBT (safe mode) is NOPIV's plan on A' = U^T A U: the fused transform reads the upper triangle of M once and writes A' into the factor
// buffer (M in place for N != 1 mod 4, the padded copy for odd N on the look-ahead path) and into a kept full copy for the refinement.
// DSYTRS sweeps each rhs with one CTA when nrhs < 8 and N > 64, else one thread per rhs. The look-ahead factorizations take their
// 128-column blocks in pairs from pair_min on. Without cooperative launches (unsupported, or HB_CHOL_COOP=0) no "coop" path runs: the
// factor takes the panels and the condensed solve the one-CTA refinement (and no 16 x 16 inverses are formed).
// ---------------------------------------------------------------------------------------------------------------------------------------
namespace {
constexpr int BLOCKED_BK_MIN_N = 96;   // below: the one-CTA DSYTF2 kernel beats panel + trailing launches
constexpr int BIG_SOLVE_MIN_N = 257;   // Cholesky / no-pivot LDL^T factored by the smaller paths: the blocked multi-CTA solve from here on
constexpr int COOP_MIN_N = 65;         // cooperative factor / solve: COOP_MIN_N <= N <= COOP_FACTOR_MAX_N / COOP_SOLVE_MAX_N
constexpr int COOP_FACTOR_MAX_N = 2048;
constexpr int COOP_SOLVE_MAX_N = 16384;
constexpr int CONDENSED_BIG_MIN_N = 2049; // condensed N: the look-ahead Cholesky (it needs an even ld and a 16-byte aligned matrix)
constexpr int SYTRS_CTA_MIN_N = 65, SYTRS_CTA_MAX_NRHS = 7;

enum Factor { F_SYTF2, F_SYTRF_BLOCKED, F_BK_CLUSTER, F_PANEL_CHOL, F_PANEL_LDL, F_COOP_CHOL, F_BIG_CHOL, F_BIG_LDL };
enum Solve { S_SYTRS, S_ONE_CTA, S_BIG, S_COOP_REFINE, S_ONE_CTA_REFINE };
enum Inertia { I_IPIV, I_BLOCKDIAG, I_DIAG };
struct Plan
{
  Factor f;
  Solve s;
  Inertia in;
  bool pairs; // look-ahead factorization: 128-column blocks in pairs
};

bool coop_factor(const hb_ctx* c, int N) { return c->coop_ctas > 0 && N >= COOP_MIN_N && N <= COOP_FACTOR_MAX_N; }

Plan symdense_plan(const hb_ctx* c, int mode, int N)
{
  if(mode == HB_FACT_BUNCH_KAUFMAN) {
    if(N >= c->bk_cluster_min && hb_bkc_supported(N)) return {F_BK_CLUSTER, S_BIG, I_BLOCKDIAG, false};
    return {N >= BLOCKED_BK_MIN_N ? F_SYTRF_BLOCKED : F_SYTF2, S_SYTRS, I_IPIV, false};
  }
  const bool ldl = mode == HB_FACT_NOPIV;
  if(N >= (ldl ? c->big_min_ldl : c->big_min_chol)) return {ldl ? F_BIG_LDL : F_BIG_CHOL, S_BIG, I_DIAG, N >= c->pair_min};
  const Factor f = ldl ? F_PANEL_LDL : coop_factor(c, N) ? F_COOP_CHOL : F_PANEL_CHOL;
  return {f, N >= BIG_SOLVE_MIN_N ? S_BIG : S_ONE_CTA, I_DIAG, false};
}

// The condensed N (second block of the table): the factor path, the solve with refinement, whether the 16 x 16 diagonal inverses of the
// cooperative solve are formed after a factor that does not produce them itself, and the look-ahead pairing.
struct CondensedPlan
{
  Factor f;
  Solve s;
  bool inverses;
  bool pairs;
};

CondensedPlan condensed_plan(const hb_ctx* c, int N, int ldf, const double* F)
{
  const Solve s = c->coop_ctas > 0 && N >= COOP_MIN_N && N <= COOP_SOLVE_MAX_N ? S_COOP_REFINE : S_ONE_CTA_REFINE;
  if(coop_factor(c, N)) return {F_COOP_CHOL, s, false, false};
  const bool inv = N >= COOP_MIN_N && c->coop_ctas > 0;
  if(N >= CONDENSED_BIG_MIN_N && (ldf & 1) == 0 && (reinterpret_cast<uintptr_t>(F) & 15u) == 0) return {F_BIG_CHOL, s, inv, N >= c->pair_min};
  return {F_PANEL_CHOL, s, inv, false};
}

int bk_sytrs(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs)
{
  return hb_dense_sytrs(c, N, A, lda, ipiv_dev, B, ldb, nrhs, nrhs <= SYTRS_CTA_MAX_NRHS && N >= SYTRS_CTA_MIN_N);
}
} // namespace

int hb_dense_init(hb_ctx* c)
{
  HB_CHECK(hb_dense_init_attrs(c));
  HB_CHECK(hb_big_init_attrs(c));
  HB_CHECK(hb_rows_init_attrs());
  HB_CHECK(hb_bkc_init_attrs(c));
  HB_CHECK(hb_chol_coop_init(c));
  // Thresholds of the symdense caller, with the environment overrides benchmarks use (a negative order keeps the default).
  // Look-ahead factorization from big_min_{chol,ldl} on; HB_DENSE_BIG_MIN sets both.
  const char* e = getenv("HB_DENSE_BIG_MIN");
  const int big = e ? atoi(e) : -1;
  c->big_min_chol = big >= 0 ? big : 1025;
  c->big_min_ldl = big >= 0 ? big : 257;
  // cluster Bunch-Kaufman from this order on (below: one-CTA DLASYF panels / DSYTF2)
  e = getenv("HB_BK_CLUSTER_MIN");
  const int bkc = e ? atoi(e) : -1;
  c->bk_cluster_min = bkc >= 0 ? bkc : 385;
  // pairing the look-ahead blocks pays once the update dominates the panel chain (not re-measured on H100)
  e = getenv("HB_DENSE_PAIR_MIN");
  c->pair_min = e ? atoi(e) : 6144;
  e = getenv("HB_CHOL_COOP");
  if(e && e[0] == '0') c->coop_ctas = 0;
  return HB_OK;
}

int hb_dense_bk_small_factor(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, int* info_dev)
{
  return hb_dense_sytf2(c, N, A, lda, ipiv_dev, info_dev);
}
int hb_dense_bk_small_solve(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs)
{
  return bk_sytrs(c, N, A, lda, ipiv_dev, B, ldb, nrhs);
}

int hb_dense_condensed_factor(hb_ctx* c, hb_big* big, int N, double* F, int ldf, double* invd, int* info_dev)
{
  const CondensedPlan p = condensed_plan(c, N, ldf, F);
  switch(p.f) {
  case F_COOP_CHOL: HB_CHECK(hb_dense_chol_coop(c, N, F, ldf, info_dev, invd, nullptr)); break;
  case F_BIG_CHOL: HB_CHECK(hb_big_factor(c, big, N, F, ldf, false, p.pairs, info_dev)); break;
  default: HB_CHECK(hb_dense_factor_panel(c, N, F, ldf, false, nullptr, info_dev)); break;
  }
  if(p.inverses) HB_CHECK(hb_dense_chol_diag_inverses(c, N, F, ldf, invd));
  return HB_OK;
}

int hb_dense_condensed_solve(hb_ctx* c, int N, const double* F, int ldf, const double* invd, const double* s, const double* Nref, int ldn,
                             const double* rhs, double* x, double* work, double tol, int max_refine, double* stats_dev)
{
  if(N == 0) return HB_OK;
  if(condensed_plan(c, N, ldf, F).s == S_COOP_REFINE)
    return hb_dense_spd_solve_coop(c, N, F, ldf, invd, s, Nref, ldn, rhs, x, work, tol, max_refine, stats_dev);
  return hb_dense_spd_solve_refine(c, N, F, ldf, s, Nref, ldn, rhs, x, work, tol, max_refine, stats_dev);
}

int hb_dense_lsq_factor(hb_ctx* c, int N, double* A, int lda, int* info_dev)
{
  if(coop_factor(c, N)) return hb_dense_chol_coop(c, N, A, lda, info_dev, nullptr, nullptr);
  return hb_dense_factor_panel(c, N, A, lda, false, nullptr, info_dev);
}
int hb_dense_lsq_solve(hb_ctx* c, int N, const double* F, int ldf, double* x) { return hb_dense_tri_solve(c, N, F, ldf, false, x); }

struct hb_symdense : hb_dense_result // mode, factored, the inertia counts and the safe mode's statistics
{
  hb_ctx* ctx = nullptr;
  int N = 0;
  hb_dev<double> M;         // N x N row-major, upper triangle valid on entry, factor in place
  hb_dev<double> W;         // panel scratch (lazy)
  hb_dev<double> xbuf;      // staging for the *_host variants (lazy)
  hb_dev<double> Fpad;      // odd N: copy of M with an even leading dimension (the large-N kernels use 16-byte accesses)
  double* F = nullptr;      // where the current factor lives (M or Fpad)
  long long ldf = 0;
  hb_big big;               // large-N path: streams, diagonal-block inverses, solve scratch
  Plan plan{};              // the paths of the current factor
  // cluster Bunch-Kaufman (hb_bk_cluster.cu): permuted factor P A P^T = L D L^T
  hb_dev<double> dsub;      // sub-diagonal of the 2x2 blocks of D
  hb_dev<int> perm;         // gather order of the right-hand side
  hb_dev<int> bk_state;     // device: k0, kb, info, -
  hb_dev<int> swaplog;
  hb_dev<double> Wp;        // W = L*D of the current panel
  hb_dev<int> ipiv;
  hb_dev<int> info;         // device: [0] info, [1..3] inertia
  hb_pinned<int> info_host;
  int bk_widths = 0;        // cluster Bunch-Kaufman: OR of the panel widths (8 / 16 / 32 / 64) the last factorization launched (no order)
  // HB_FACT_RBT_NOPIV, allocated by the first RBT factorization: A' (N x N, full), the butterfly diagonals (2 N), row-sum scratch and
  // ||A'||_inf; the solve adds the rows of x and b', the residual and per-rhs norms
  hb_dev<double> Ak, rbt_f, rbt_part, rbt_nrm, rbt_xw, rbt_b, rbt_r, rbt_col;
  hb_pinned<double> rbt_nrm_host;
  hb_event ev_rbt[2];
};

extern "C" int hb_symdense_create(hb_ctx* c, int N, hb_symdense** out)
{
  HB_REQUIRE(c && out && N >= 0, "hb_symdense_create: bad arguments");
  HB_CUDA(cudaSetDevice(c->device));
  std::unique_ptr<hb_symdense> s(new hb_symdense);
  s->ctx = c;
  s->N = N;
  HB_CHECK(s->M.reserve(c, (size_t)N * N, "the N x N system matrix"));
  HB_CHECK(s->ipiv.reserve(c, (size_t)N + 1, "pivots"));
  HB_CHECK(s->info.reserve(c, 4, "info words"));
  HB_CHECK(s->info_host.reserve(c, 4, "info words"));
  HB_CUDA(cudaMemsetAsync(s->M, 0, sizeof(double) * s->M.capacity(), c->stream));
  *out = s.release();
  return HB_OK;
}

extern "C" int hb_symdense_destroy(hb_symdense* s)
{
  if(!s) return HB_OK;
  cudaSetDevice(s->ctx->device);
  cudaStreamSynchronize(s->ctx->stream);
  delete s;
  return HB_OK;
}

extern "C" double* hb_symdense_matrix(hb_symdense* s) { return s ? s->M.get() : nullptr; }

// the RBT buffers, on the first RBT factorization of the handle
static int rbt_reserve(hb_symdense* s)
{
  if(s->Ak) return HB_OK;
  hb_ctx* c = s->ctx;
  const int N = s->N;
  HB_CHECK(s->rbt_f.reserve(c, (size_t)2 * N, "butterfly diagonals"));
  HB_CHECK(s->rbt_part.reserve(c, hb_rbt_part_doubles(N), "row sums of |A'|"));
  HB_CHECK(s->rbt_nrm.reserve(c, 1, "norm of A'"));
  HB_CHECK(s->rbt_nrm_host.reserve(c, 3, "norms"));
  for(int e = 0; e < 2; e++) HB_CHECK(s->ev_rbt[e].create(cudaEventDefault));
  HB_CHECK(hb_rbt_table(c, N, s->rbt_f));
  return s->Ak.reserve(c, (size_t)N * N, "the transformed matrix A'"); // last: its presence marks the set complete
}

// A' = U^T A U from the upper triangle of M into the factor buffer s->F (upper triangle) and s->Ak (full), ||A'||_inf into rbt_anorm
static int rbt_transform(hb_symdense* s)
{
  hb_ctx* c = s->ctx;
  const int N = s->N;
  const bool direct = s->F != s->M.get() || hb_rbt_in_place(N);
  HB_CUDA(cudaEventRecord(s->ev_rbt[0], c->stream));
  HB_CHECK(hb_rbt_fused(c, N, s->rbt_f, s->M, N, direct ? s->F : nullptr, s->ldf, s->Ak, N, s->rbt_part, s->rbt_nrm));
  HB_CUDA(cudaEventRecord(s->ev_rbt[1], c->stream));
  if(!direct) HB_CUDA(cudaMemcpyAsync(s->M, s->Ak, sizeof(double) * N * N, cudaMemcpyDeviceToDevice, c->stream)); // small N only
  HB_CUDA(cudaMemcpyAsync(s->rbt_nrm_host, s->rbt_nrm, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  s->rbt_anorm = s->rbt_nrm_host[0];
  HB_CUDA(cudaEventElapsedTime(&s->rbt_ms, s->ev_rbt[0], s->ev_rbt[1]));
  return HB_OK;
}

// where the factor of a plan lives: M, or for odd N on the look-ahead and cluster paths a copy with an even leading dimension (the
// 16-byte operand copies)
static int factor_buffer(hb_symdense* s, const Plan& p, bool copy)
{
  hb_ctx* c = s->ctx;
  const int N = s->N;
  s->F = s->M; s->ldf = N;
  const bool big = p.f == F_BIG_CHOL || p.f == F_BIG_LDL;
  if((big || p.f == F_BK_CLUSTER) && (N & 1)) {
    const long long ld = (N + 7) & ~7LL;
    if(!s->Fpad) {
      HB_CHECK(s->Fpad.reserve(c, (size_t)ld * N, "the padded factor"));
      HB_CUDA(cudaMemsetAsync(s->Fpad, 0, sizeof(double) * (size_t)ld * N, c->stream));
    }
    if(copy)
      HB_CUDA(cudaMemcpy2DAsync(s->Fpad, sizeof(double) * ld, s->M, sizeof(double) * N, sizeof(double) * N, N, cudaMemcpyDeviceToDevice, c->stream));
    s->F = s->Fpad; s->ldf = ld;
  }
  return HB_OK;
}

extern "C" int hb_symdense_matrix_changed(hb_symdense* s, int mode)
{
  HB_REQUIRE(s, "null handle");
  HB_REQUIRE(mode == HB_FACT_BUNCH_KAUFMAN || mode == HB_FACT_NOPIV || mode == HB_FACT_CHOLESKY || mode == HB_FACT_RBT_NOPIV,
             "hb_symdense_matrix_changed: bad mode");
  hb_ctx* c = s->ctx;
  const int N = s->N;
  const bool rbt = mode == HB_FACT_RBT_NOPIV;
  s->mode = mode;
  s->factored = false;
  if(N == 0) { const int none[3] = {0, 0, 0}; return s->finish(none, 0); }
  HB_CUDA(cudaMemsetAsync(s->info, 0, sizeof(int) * 4, c->stream));
  s->big.inv_valid = false;
  const Plan p = symdense_plan(c, rbt ? HB_FACT_NOPIV : mode, N);
  s->plan = p;
  s->bk_widths = 0;
  const bool big = p.f == F_BIG_CHOL || p.f == F_BIG_LDL;
  HB_CHECK(factor_buffer(s, p, !rbt));
  if(rbt) {
    HB_CHECK(rbt_reserve(s));
    HB_CHECK(rbt_transform(s));
  }
  const long long ldw = (N + 7) & ~7LL;
  if(p.f == F_BK_CLUSTER) {
    HB_CHECK(s->dsub.reserve(c, (size_t)N + 2, "Bunch-Kaufman sub-diagonal"));
    HB_CHECK(s->perm.reserve(c, (size_t)N + 2, "Bunch-Kaufman permutation"));
    HB_CHECK(s->bk_state.reserve(c, 4, "Bunch-Kaufman state"));
    HB_CHECK(s->swaplog.reserve(c, HB_BKC_SWAPLOG_INTS(N), "Bunch-Kaufman swap log"));
    HB_CHECK(s->Wp.reserve(c, HB_BKC_W_DOUBLES(ldw), "Bunch-Kaufman panel scratch"));
  }
  if(p.f == F_PANEL_LDL || p.f == F_SYTRF_BLOCKED) HB_CHECK(s->W.reserve(c, (size_t)2 * 64 * N, "panel scratch"));
  switch(p.f) {
  case F_SYTF2: HB_CHECK(hb_dense_sytf2(c, N, s->M, N, s->ipiv, s->info)); break;
  case F_SYTRF_BLOCKED: HB_CHECK(hb_dense_sytrf_blocked(c, N, s->M, N, s->ipiv, s->W, s->info)); break;
  case F_BK_CLUSTER:
    HB_CHECK(hb_bkc_factor(c, &s->big, N, s->F, s->ldf, s->ipiv, s->dsub, s->perm, s->Wp, ldw, s->bk_state, s->swaplog, s->info,
                           &s->bk_widths));
    break;
  case F_PANEL_CHOL:
  case F_PANEL_LDL: HB_CHECK(hb_dense_factor_panel(c, N, s->M, N, p.f == F_PANEL_LDL, s->W, s->info)); break;
  case F_COOP_CHOL: HB_CHECK(hb_dense_chol_coop(c, N, s->M, N, s->info, nullptr, nullptr)); break;
  case F_BIG_CHOL:
  case F_BIG_LDL: HB_CHECK(hb_big_factor(c, &s->big, N, s->F, s->ldf, p.f == F_BIG_LDL, p.pairs, s->info)); break;
  }
  // the blocked solve needs the 128 x 128 diagonal inverses; only the look-ahead factorization forms them itself
  if(p.s == S_BIG && !big) HB_CHECK(hb_big_block_inverses(c, &s->big, N, s->F, s->ldf, mode != HB_FACT_CHOLESKY));
  switch(p.in) {
  case I_IPIV: HB_CHECK(hb_dense_inertia_ipiv(c, N, s->F, (int)s->ldf, s->ipiv, s->info + 1)); break;
  case I_BLOCKDIAG: HB_CHECK(hb_dense_inertia_blockdiag(c, N, s->F, s->ldf, s->ipiv, s->dsub, s->info + 1)); break;
  case I_DIAG: HB_CHECK(hb_dense_inertia_diag(c, N, s->F, s->ldf, s->info + 1)); break;
  }
  HB_CUDA(cudaMemcpyAsync(s->info_host, s->info, sizeof(int) * 4, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return s->finish(s->info_host + 1, s->info_host[0]);
}

extern "C" int hb_symdense_inertia(hb_symdense* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  return s->inertia(n_neg, n_null, n_pos);
}

// the sweeps of the current factor on nrhs right-hand sides stored one after the other, in place
static int plan_sweeps(hb_symdense* s, double* x, int nrhs)
{
  hb_ctx* c = s->ctx;
  switch(s->plan.s) {
  case S_BIG: {
    const bool bkc = s->plan.f == F_BK_CLUSTER;
    const int dmode = bkc ? 2 : (s->mode == HB_FACT_CHOLESKY ? 0 : 1);
    for(int r = 0; r < nrhs; r++)
      HB_CHECK(hb_big_solve(c, &s->big, s->N, s->F, s->ldf, dmode, s->ipiv, s->dsub, bkc ? s->perm.get() : nullptr, x + (size_t)r * s->N));
    break;
  }
  case S_SYTRS: HB_CHECK(bk_sytrs(c, s->N, s->M, s->N, s->ipiv, x, s->N, nrhs)); break;
  case S_ONE_CTA:
    for(int r = 0; r < nrhs; r++) HB_CHECK(hb_dense_tri_solve(c, s->N, s->M, s->N, s->mode != HB_FACT_CHOLESKY, x + (size_t)r * s->N));
    break;
  }
  return HB_OK;
}

// RBT: hb_rbt_solve on the rows of x (row-major N x nrhs), the sweeps of the NOPIV plan on columns, the residual against the kept A'
// with its ||A'||_inf, or (tests: hb_debug_symdense_rbt_solve) against a full N x N Aref with anorm
static int rbt_solve(hb_symdense* s, double* x, int nrhs, hb_rbt_trace* trace = nullptr, const double* Aref = nullptr, double anorm = 0.0)
{
  hb_ctx* c = s->ctx;
  const int N = s->N;
  const size_t n = (size_t)N * nrhs;
  HB_CHECK(s->rbt_xw.reserve(c, n, "solve rows"));
  HB_CHECK(s->rbt_b.reserve(c, n, "transformed rhs"));
  HB_CHECK(s->rbt_r.reserve(c, n + 3 * (size_t)nrhs, "residual and norms"));
  HB_CHECK(s->rbt_nrm_host.reserve(c, 3 * (size_t)nrhs, "norms"));
  if(nrhs > 1) HB_CHECK(s->rbt_col.reserve(c, n, "solve columns"));
  auto sweeps = [&](double* v) -> int {
    if(nrhs == 1) return plan_sweeps(s, v, 1); // one rhs: rows and columns are the same array
    HB_CHECK(hb_rbt_to_rows(c, N, nrhs, s->rbt_col, v, true));
    HB_CHECK(plan_sweeps(s, s->rbt_col, nrhs));
    return hb_rbt_to_rows(c, N, nrhs, s->rbt_col, v, false);
  };
  const double* Ar = Aref ? Aref : s->Ak.get();
  auto residual = [&](const double* xr, const double* b, double* r) { return hb_rbt_rows(c, N, 1, 0, N, Ar, N, nrhs, xr, b, r); };
  HB_CHECK(hb_rbt_to_rows(c, N, nrhs, x, s->rbt_xw, false));
  const int ok = hb_rbt_solve(c, N, nrhs, s->rbt_f, Aref ? anorm : s->rbt_anorm, s->rbt_xw, s->rbt_b, s->rbt_r, s->rbt_nrm_host, sweeps, residual,
                              &s->rbt_corr, &s->rbt_berr, trace);
  if(ok < 0) return ok;
  HB_CHECK(hb_rbt_to_rows(c, N, nrhs, x, s->rbt_xw, true));
  return ok;
}

extern "C" int hb_symdense_solve(hb_symdense* s, double* x, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_solve: bad arguments");
  if(const int rc = s->solve_ready(s->N, x, nrhs, "hb_symdense"); rc != HB_OK) return rc;
  if(s->mode == HB_FACT_RBT_NOPIV) return rbt_solve(s, x, nrhs);
  HB_CHECK(plan_sweeps(s, x, nrhs));
  return 1;
}

extern "C" int hb_symdense_rbt_stats(hb_symdense* s, int* corrections, double* backward_error, float* transform_ms)
{
  HB_REQUIRE(s, "null handle");
  return s->rbt_stats(corrections, backward_error, transform_ms);
}

// diagnostics (tests): the RBT transform of the upper triangle of M without factoring; A' (full) and the factor buffer's upper triangle
extern "C" int hb_debug_symdense_rbt(hb_symdense* s, double* Ak_host, double* F_host)
{
  HB_REQUIRE(s, "null handle");
  if(s->N == 0) return HB_OK;
  hb_ctx* c = s->ctx;
  const int N = s->N;
  HB_CUDA(cudaSetDevice(c->device));
  s->factored = false;
  s->plan = symdense_plan(c, HB_FACT_NOPIV, N);
  HB_CHECK(factor_buffer(s, s->plan, false));
  HB_CHECK(rbt_reserve(s));
  HB_CHECK(rbt_transform(s));
  if(Ak_host) HB_CUDA(cudaMemcpyAsync(Ak_host, s->Ak, sizeof(double) * N * N, cudaMemcpyDeviceToHost, c->stream));
  if(F_host)
    HB_CUDA(cudaMemcpy2DAsync(F_host, sizeof(double) * N, s->F, sizeof(double) * s->ldf, sizeof(double) * N, N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}

// diagnostics (tests): one refined RBT solve of x, traced, with the residual and ||.||_inf of Aref / anorm instead of the kept A' when
// Aref is given (the kept A' is not touched)
extern "C" int hb_debug_symdense_rbt_solve(hb_symdense* s, double* x, int nrhs, const double* Aref, double anorm, int* ret_host, int* passes_host,
                                           double* anorm_host, double* norms_host, double* xp_host, double* bp_host)
{
  HB_REQUIRE(s && x && nrhs > 0 && s->N > 0, "hb_debug_symdense_rbt_solve: bad arguments");
  auto solve = [&](hb_rbt_trace* t) -> int {
    HB_CUDA(cudaSetDevice(s->ctx->device));
    return rbt_solve(s, x, nrhs, t, Aref, anorm);
  };
  return hb_rbt_traced_solve(*s, "hb_debug_symdense_rbt_solve", solve, ret_host, passes_host, anorm_host, norms_host, xp_host, bp_host);
}

extern "C" int hb_symdense_matrix_changed_host(hb_symdense* s, const double* M_host, int mode)
{
  HB_REQUIRE(s && (M_host || s->N == 0), "hb_symdense_matrix_changed_host: null matrix");
  if(s->N) HB_CUDA(cudaMemcpyAsync(s->M, M_host, sizeof(double) * (size_t)s->N * s->N, cudaMemcpyHostToDevice, s->ctx->stream));
  return hb_symdense_matrix_changed(s, mode);
}

extern "C" int hb_symdense_solve_host(hb_symdense* s, double* x_host, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_solve_host: bad arguments");
  if(s->N == 0 || nrhs == 0) return 1;
  HB_REQUIRE(x_host, "hb_symdense_solve_host: null rhs");
  hb_ctx* c = s->ctx;
  const size_t need = (size_t)s->N * nrhs;
  HB_CHECK(s->xbuf.reserve(c, need, "rhs staging"));
  HB_CUDA(cudaMemcpyAsync(s->xbuf, x_host, sizeof(double) * need, cudaMemcpyHostToDevice, c->stream));
  int rc = hb_symdense_solve(s, s->xbuf, nrhs);
  if(rc != 1) return rc;
  HB_CUDA(cudaMemcpyAsync(x_host, s->xbuf, sizeof(double) * need, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return 1;
}

// diagnostics (tools/prof_diag.py): phase cycle counters of the 128 x 128 diagonal-block kernel on the leading block of M
extern "C" int hb_debug_diag128_profile(hb_symdense* s, int ldl, long long* prof_host8)
{
  HB_REQUIRE(s && prof_host8 && s->N >= 128 && (s->N & 1) == 0, "hb_debug_diag128_profile: needs an even N >= 128");
  return hb_big_diag_profile(s->ctx, &s->big, s->N, s->M, s->N, 0, ldl != 0, prof_host8);
}
// diagnostics (tests): what the last hb_symdense_matrix_changed chose and computed. Every output pointer may be NULL.
extern "C" int hb_debug_symdense_factor(hb_symdense* s, int* plan4, int* bk_widths, double* F_host, int* ipiv_host, int* perm_host,
                                        double* dsub_host)
{
  HB_REQUIRE(s && s->N > 0 && s->F, "hb_debug_symdense_factor: no factorization of a non-empty matrix yet");
  hb_ctx* c = s->ctx;
  const int N = s->N;
  if(plan4) { plan4[0] = s->plan.f; plan4[1] = s->plan.s; plan4[2] = s->plan.in; plan4[3] = s->plan.pairs; }
  if(bk_widths) *bk_widths = s->bk_widths;
  HB_CUDA(cudaSetDevice(c->device));
  if(F_host)
    HB_CUDA(cudaMemcpy2DAsync(F_host, sizeof(double) * N, s->F, sizeof(double) * s->ldf, sizeof(double) * N, N, cudaMemcpyDeviceToHost, c->stream));
  const bool bk = s->plan.f == F_SYTF2 || s->plan.f == F_SYTRF_BLOCKED || s->plan.f == F_BK_CLUSTER;
  HB_REQUIRE(bk || !ipiv_host, "hb_debug_symdense_factor: ipiv exists only for the Bunch-Kaufman factors");
  if(ipiv_host) HB_CUDA(cudaMemcpyAsync(ipiv_host, s->ipiv, sizeof(int) * N, cudaMemcpyDeviceToHost, c->stream));
  const bool bkc = s->plan.f == F_BK_CLUSTER;
  HB_REQUIRE(bkc || (!perm_host && !dsub_host), "hb_debug_symdense_factor: perm / dsub exist only for the cluster Bunch-Kaufman factor");
  if(perm_host) HB_CUDA(cudaMemcpyAsync(perm_host, s->perm, sizeof(int) * N, cudaMemcpyDeviceToHost, c->stream));
  if(dsub_host) HB_CUDA(cudaMemcpyAsync(dsub_host, s->dsub, sizeof(double) * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}
extern "C" int hb_debug_bk_profile(hb_ctx* c, int on, long long* prof_host8)
{
  HB_REQUIRE(c, "null ctx");
  return hb_bkc_profile(c, on, prof_host8);
}

// diagnostics (tests): the condensed-N sequence of hb_lowrank (equilibrate, factor, solve with refinement) on caller matrices, with
// scratch allocated like the handle's (ld N, one allocation per buffer).
extern "C" int hb_debug_condensed_solve(hb_ctx* c, int N, const double* Nfact, const double* Nref, int ldn, const double* rhs, double* x,
                                        double tol, int max_refine, int* plan4, double* s_host, double* Aeq_host, double* F_host,
                                        double* stats_host, int* info_host)
{
  HB_REQUIRE(c && N > 0 && ldn >= N && Nfact && Nref && rhs && x && max_refine >= 0, "hb_debug_condensed_solve: bad arguments");
  HB_CUDA(cudaSetDevice(c->device));
  hb_big big;
  hb_dev<double> F, s, invd, work, stats;
  hb_dev<int> info;
  HB_CHECK(F.reserve(c, (size_t)N * N, "the factor of N"));
  HB_CHECK(s.reserve(c, N, "the scaling of N"));
  HB_CHECK(work.reserve(c, 2 * (size_t)N + 2, "refinement scratch"));
  HB_CHECK(invd.reserve(c, HB_CHOL_INV_DOUBLES(N), "diagonal-block inverses of N"));
  HB_CHECK(stats.reserve(c, 4, "solve statistics"));
  HB_CHECK(info.reserve(c, 1, "info word"));
  const CondensedPlan p = condensed_plan(c, N, N, F);
  if(plan4) { plan4[0] = p.f; plan4[1] = p.s; plan4[2] = p.inverses; plan4[3] = p.pairs; }
  HB_CUDA(cudaMemsetAsync(info, 0, sizeof(int), c->stream));
  HB_CHECK(hb_dense_equilibrate(c, N, Nfact, ldn, F, N, s));
  if(Aeq_host) HB_CUDA(cudaMemcpyAsync(Aeq_host, F, sizeof(double) * (size_t)N * N, cudaMemcpyDeviceToHost, c->stream));
  if(s_host) HB_CUDA(cudaMemcpyAsync(s_host, s, sizeof(double) * N, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  HB_CHECK(hb_dense_condensed_factor(c, &big, N, F, N, invd, info));
  HB_CHECK(hb_dense_condensed_solve(c, N, F, N, invd, s, Nref, ldn, rhs, x, work, tol, max_refine, stats));
  if(F_host) HB_CUDA(cudaMemcpyAsync(F_host, F, sizeof(double) * (size_t)N * N, cudaMemcpyDeviceToHost, c->stream));
  if(stats_host) HB_CUDA(cudaMemcpyAsync(stats_host, stats, sizeof(double) * 2, cudaMemcpyDeviceToHost, c->stream));
  if(info_host) HB_CUDA(cudaMemcpyAsync(info_host, info, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  return HB_OK;
}
