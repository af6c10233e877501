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
enum Solve { S_SYTRS, S_ONE_CTA, S_BIG };
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

int bk_sytrs(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs)
{
  return hb_dense_sytrs(c, N, A, lda, ipiv_dev, B, ldb, nrhs, nrhs <= SYTRS_CTA_MAX_NRHS && N >= SYTRS_CTA_MIN_N);
}
} // namespace

int hb_dense_init(hb_ctx* c)
{
  HB_CHECK(hb_dense_init_attrs(c));
  HB_CHECK(hb_big_init_attrs(c));
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
  if(coop_factor(c, N)) return hb_dense_chol_coop(c, N, F, ldf, info_dev, invd, nullptr);
  if(N >= CONDENSED_BIG_MIN_N && (ldf & 1) == 0 && (reinterpret_cast<uintptr_t>(F) & 15u) == 0)
    HB_CHECK(hb_big_factor(c, big, N, F, ldf, false, N >= c->pair_min, info_dev));
  else
    HB_CHECK(hb_dense_factor_panel(c, N, F, ldf, false, nullptr, info_dev));
  if(N >= COOP_MIN_N && c->coop_ctas > 0) HB_CHECK(hb_dense_chol_diag_inverses(c, N, F, ldf, invd)); // for the cooperative solve
  return HB_OK;
}

int hb_dense_condensed_solve(hb_ctx* c, int N, const double* F, int ldf, const double* invd, const double* s, const double* Nref, int ldn,
                             const double* rhs, double* x, double* work, double tol, int max_refine, double* stats_dev)
{
  if(N == 0) return HB_OK;
  if(c->coop_ctas > 0 && N >= COOP_MIN_N && N <= COOP_SOLVE_MAX_N)
    return hb_dense_spd_solve_coop(c, N, F, ldf, invd, s, Nref, ldn, rhs, x, work, tol, max_refine, stats_dev);
  return hb_dense_spd_solve_refine(c, N, F, ldf, s, Nref, ldn, rhs, x, work, tol, max_refine, stats_dev);
}

int hb_dense_lsq_factor(hb_ctx* c, int N, double* A, int lda, int* info_dev)
{
  if(coop_factor(c, N)) return hb_dense_chol_coop(c, N, A, lda, info_dev, nullptr, nullptr);
  return hb_dense_factor_panel(c, N, A, lda, false, nullptr, info_dev);
}
int hb_dense_lsq_solve(hb_ctx* c, int N, const double* F, int ldf, double* x) { return hb_dense_tri_solve(c, N, F, ldf, false, x); }

struct hb_symdense
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
  int mode = -1;
  int bk_widths = 0;        // cluster Bunch-Kaufman: OR of the panel widths (8 / 16 / 32 / 64) the last factorization launched (no order)
  bool factored = false;
  int n_neg = 0, n_null = 0, n_pos = 0;
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

extern "C" int hb_symdense_matrix_changed(hb_symdense* s, int mode)
{
  HB_REQUIRE(s, "null handle");
  HB_REQUIRE(mode == HB_FACT_BUNCH_KAUFMAN || mode == HB_FACT_NOPIV || mode == HB_FACT_CHOLESKY, "hb_symdense_matrix_changed: bad mode");
  hb_ctx* c = s->ctx;
  const int N = s->N;
  s->mode = mode;
  s->factored = false;
  if(N == 0) { s->factored = true; s->n_neg = s->n_null = s->n_pos = 0; return 0; }
  HB_CUDA(cudaMemsetAsync(s->info, 0, sizeof(int) * 4, c->stream));
  s->F = s->M; s->ldf = N; s->big.inv_valid = false;
  const Plan p = symdense_plan(c, mode, N);
  s->plan = p;
  s->bk_widths = 0;
  const bool big = p.f == F_BIG_CHOL || p.f == F_BIG_LDL;
  if((big || p.f == F_BK_CLUSTER) && (N & 1)) { // even leading dimension for the 16-byte operand copies
    const long long ld = (N + 7) & ~7LL;
    if(!s->Fpad) {
      HB_CHECK(s->Fpad.reserve(c, (size_t)ld * N, "the padded factor"));
      HB_CUDA(cudaMemsetAsync(s->Fpad, 0, sizeof(double) * (size_t)ld * N, c->stream));
    }
    HB_CUDA(cudaMemcpy2DAsync(s->Fpad, sizeof(double) * ld, s->M, sizeof(double) * N, sizeof(double) * N, N, cudaMemcpyDeviceToDevice, c->stream));
    s->F = s->Fpad; s->ldf = ld;
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
  s->n_neg = s->info_host[1]; s->n_null = s->info_host[2]; s->n_pos = s->info_host[3];
  if(s->info_host[0] != 0) return -1; // zero pivot / not SPD: "matrix is singular" (hiopLinSolverSymDenseLapack.hpp:109-116)
  s->factored = true;
  if(s->n_null > 0) return -1;        // :166
  return s->n_neg;
}

extern "C" int hb_symdense_inertia(hb_symdense* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  if(n_neg) *n_neg = s->n_neg;
  if(n_null) *n_null = s->n_null;
  if(n_pos) *n_pos = s->n_pos;
  return HB_OK;
}

extern "C" int hb_symdense_solve(hb_symdense* s, double* x, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_solve: bad arguments");
  if(s->N == 0 || nrhs == 0) return 1;
  HB_REQUIRE(x, "hb_symdense_solve: null rhs");
  if(!s->factored) return hb_fail(HB_ERR_STATE, "hb_symdense_solve: no valid factorization (call hb_symdense_matrix_changed)%s", "");
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
    for(int r = 0; r < nrhs; r++) HB_CHECK(hb_dense_tri_solve(c, s->N, s->M, s->N, s->mode == HB_FACT_NOPIV, x + (size_t)r * s->N));
    break;
  }
  return 1;
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
