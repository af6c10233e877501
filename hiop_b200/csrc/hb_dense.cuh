// Internal API of the dense symmetric factorizations / solves on device: the device helpers their kernel files share, the entry points
// of each kernel file (each runs one path, no fall-back), and the per-caller dispatch of hb_symdense.cu that chooses between them.
#pragma once
#include <functional>
#include "hb_common.cuh"

// ---- device helpers ----
// Storage convention: N x N row-major with the upper triangle valid = column-major lower triangle, Lc(i,j) = A[j*lda + i], i >= j.
#define LC(A, lda, i, j) (A)[(size_t)(j) * (lda) + (i)]
#define BK_ALPHA 0.6403882032022076 /* (1+sqrt(17))/8: Bunch-Kaufman pivot threshold */

struct ArgMax
{
  double v;
  int i;
};
// IDAMAX semantics: first index of the maximum absolute value. A total order on (|v|, i), so every reduction order gives the same pivot.
__device__ __forceinline__ ArgMax argmax_comb(ArgMax a, ArgMax b)
{
  if(b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
  return a;
}
// CTA-wide arg-max, every thread gets the result; sm: 32 entries of shared memory
__device__ inline ArgMax cta_argmax(ArgMax a, ArgMax* sm)
{
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, a.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, a.i, o);
    a = argmax_comb(a, b);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if(lane == 0) sm[warp] = a;
  __syncthreads();
  // second stage by shuffles in every warp (a loop over the 32 partials in all 1024 threads cost ~2500 cycles of LDS traffic per column)
  ArgMax r{-1.0, 0x7fffffff};
  if(lane < (int)(blockDim.x >> 5)) r = sm[lane];
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, r.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, r.i, o);
    r = argmax_comb(r, b);
  }
  return r;
}

// The inertia rule of the reference's dsidi sweep (hiopLinSolverSymDenseLapack.hpp:127-167) for one diagonal value of a factor: negative
// below -1e-14, null up to 1e-14, positive otherwise (NaN included)
__device__ __forceinline__ void hb_inertia_count(double d, int& neg, int& nul, int& pos)
{
  if(d < -1e-14) neg++; else if(d < 1e-14) nul++; else pos++;
}

struct hb_big;

// ---- the outcome of a factorization, as hb_symdense, hb_symdense_dist and hb_symdense_host report it ----
// The mode and result of the last matrix_changed with its inertia counts, and the statistics of the safe mode (HB_FACT_RBT_NOPIV):
// ||A'||_inf and the transform time of the last factorization, the corrections and the backward error of the last solve.
struct hb_dense_result
{
  int mode = -1;
  bool factored = false;
  int n_neg = 0, n_null = 0, n_pos = 0;
  double rbt_anorm = 0.0, rbt_berr = 0.0;
  int rbt_corr = 0;
  float rbt_ms = 0.f;
  // the end of matrix_changed, from the counts {neg, null, pos}: -1 after a breakdown (info != 0), which leaves no factorization
  // ("matrix is singular", hiopLinSolverSymDenseLapack.hpp:109-116); else factored, and -1 with a null pivot (:166) or n_neg
  template <typename T> int finish(const T* counts, int info)
  {
    n_neg = (int)counts[0]; n_null = (int)counts[1]; n_pos = (int)counts[2];
    factored = info == 0;
    return info != 0 || n_null > 0 ? -1 : n_neg;
  }
  // the *_inertia and *_rbt_stats getters; every output may be NULL
  int inertia(int* neg, int* null, int* pos) const
  {
    if(neg) *neg = n_neg;
    if(null) *null = n_null;
    if(pos) *pos = n_pos;
    return HB_OK;
  }
  int rbt_stats(int* corrections, double* backward_error, float* transform_ms) const
  {
    if(corrections) *corrections = rbt_corr;
    if(backward_error) *backward_error = rbt_berr;
    if(transform_ms) *transform_ms = rbt_ms;
    return HB_OK;
  }
  // the precondition of <who>_solve: 1 when there is nothing to solve, HB_OK to go on, else the error
  int solve_ready(int N, const void* x, int nrhs, const char* who) const
  {
    if(N == 0 || nrhs == 0) return 1;
    if(!x) {
      snprintf(g_hb_err, sizeof(g_hb_err), "%s_solve: null rhs (%s:%d)", who, __FILE__, __LINE__);
      return HB_ERR_INVALID;
    }
    if(!factored) {
      snprintf(g_hb_err, sizeof(g_hb_err), "%s_solve: no valid factorization (call %s_matrix_changed)", who, who);
      return HB_ERR_STATE;
    }
    return HB_OK;
  }
  // a solve in groups of right-hand sides reports the most corrections and the largest omega of its groups (a NaN wins)
  void merge_rbt(int corr, double berr)
  {
    rbt_corr = corr > rbt_corr ? corr : rbt_corr;
    if(rbt_berr == rbt_berr && (berr != berr || berr > rbt_berr)) rbt_berr = berr;
  }
};

// ---- dispatch by caller (hb_symdense.cu; the hb_symdense_* C-ABI is the fourth caller) ----
// The 2l x 2l matrices of the compact BFGS inverse (V, Mdir): Bunch-Kaufman
int hb_dense_bk_small_factor(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, int* info_dev);
int hb_dense_bk_small_solve(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs);
// The equilibrated condensed matrix N of the quasi-Newton KKT system: Cholesky (+ the 16 x 16 diagonal inverses the cooperative solve
// uses, invd: HB_CHOL_INV_DOUBLES(N) doubles) and the SPD solve with device-side refinement against Nref (work: 2N+2 doubles).
// big: the caller's look-ahead state.
#define HB_CHOL_INV_DOUBLES(N) ((size_t)(((N) + 63) / 64) * (4 * 16 * 17))
int hb_dense_condensed_factor(hb_ctx* c, hb_big* big, int N, double* F, int ldf, double* invd, int* info_dev);
int hb_dense_condensed_solve(hb_ctx* c, int N, const double* F, int ldf, const double* invd, const double* s, const double* Nref, int ldn,
                             const double* rhs, double* x, double* work, double tol, int max_refine, double* stats_dev);
// J J^T + I of the least-squares duals: Cholesky and one solve
int hb_dense_lsq_factor(hb_ctx* c, int N, double* A, int lda, int* info_dev);
int hb_dense_lsq_solve(hb_ctx* c, int N, const double* F, int ldf, double* x);

// ---- hb_dense.cu: 64-wide panels, one-CTA kernels ----
int hb_dense_init_attrs(hb_ctx* c);
// LL^T (ldl=false) or no-pivot LDL^T (ldl=true), 64-wide panel + trailing-update launches. Wpanel: 64*N doubles of scratch when ldl.
// info_dev: 0 ok, k>0 = breakdown at column k (1-based).
int hb_dense_factor_panel(hb_ctx* c, int N, double* A, int lda, bool ldl, double* Wpanel, int* info_dev);
// Bunch-Kaufman: unblocked single-CTA kernel (DSYTF2 logic)
int hb_dense_sytf2(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, int* info_dev);
// Bunch-Kaufman: blocked (one-CTA DLASYF panels + DMMA trailing updates); Wpanel: 2*64*N doubles of scratch
int hb_dense_sytrf_blocked(hb_ctx* c, int N, double* A, int lda, int* ipiv_dev, double* Wpanel, int* info_dev);
// DSYTRS with a LAPACK-format factor: one thread per rhs, or (cta_per_rhs) one CTA sweeping each rhs
int hb_dense_sytrs(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, double* B, int ldb, int nrhs, bool cta_per_rhs);
// inertia of a LAPACK-format Bunch-Kaufman factor (serial dsidi sweep)
int hb_dense_inertia_ipiv(hb_ctx* c, int N, const double* A, int lda, const int* ipiv_dev, int* out3_dev);
// one-CTA triangular solves (Cholesky, or unit L + D for ldl)
int hb_dense_tri_solve(hb_ctx* c, int N, const double* F, int ldf, bool ldl, double* x);
int hb_dense_equilibrate(hb_ctx* c, int N, const double* Nfull, int ldn, double* F, int ldf, double* s);
// one-CTA SPD solve with equilibration scaling s and refinement against Nref; work2N: 2N doubles
int hb_dense_spd_solve_refine(hb_ctx* c, int N, const double* F, int ldf, const double* s, const double* Nref, int ldn, const double* rhs,
                              double* x, double* work2N, double tol, int max_refine, double* stats_dev);

// ---- hb_chol_coop.cu: single-launch cooperative Cholesky and SPD solve (64 < N) ----
// sets the kernels' attributes and c->coop_ctas (0 when the device cannot launch them cooperatively)
int hb_chol_coop_init(hb_ctx* c);
// invd (may be NULL): receives the 16 x 16 diagonal inverses; prof (may be NULL): 10 cycle counters of CTA 0
int hb_dense_chol_coop(hb_ctx* c, int N, double* A, int lda, int* info_dev, double* invd, long long* prof);
// the 16 x 16 diagonal inverses of a factor produced by another Cholesky path
int hb_dense_chol_diag_inverses(hb_ctx* c, int N, const double* F, int ldf, double* invd);
// cooperative solve + refinement with the factor and its invd; work: 2N+2 doubles
int hb_dense_spd_solve_coop(hb_ctx* c, int N, const double* F, int ldf, const double* invd, const double* s, const double* Nref, int ldn,
                            const double* rhs, double* x, double* work, double tol, int max_refine, double* stats_dev);

// ---- large-N path (hb_dense_big.cu): blocked Cholesky / no-pivot LDL^T with look-ahead, 128 x 128 diagonal-block inverses, blocked solves ----
struct hb_big
{
  hb_stream panel_stream;
  hb_event ev_panel, ev_upd, ev_upd2;
  hb_dev<double> InvAll;  // ceil(N/128) inverses of the 128 x 128 diagonal triangles of the factor (column-major, zeros above)
  hb_dev<double> W[2];    // LDL^T: W = L*D of the current PAIR of panels, 256 p-major rows (double-buffered across the look-ahead)
  hb_dev<double> dinv;
  hb_dev<double> partial; // solve: per-CTA partial products
  hb_dev<int> counter;    // solve: ticket of the "last CTA finishes the step" pattern (self-resetting)
  hb_dev<double> xtmp;    // permuted rhs (Bunch-Kaufman)
  int capN = 0;
  bool inv_valid = false;
  // the panel stream may still run the last panel of a factorization when its owner is destroyed
  ~hb_big()
  {
    if(panel_stream) cudaStreamSynchronize(panel_stream);
  }
};
int hb_big_init_attrs(hb_ctx* c);
int hb_big_init(hb_ctx* c, hb_big* b);
int hb_big_reserve(hb_ctx* c, hb_big* b, int N, bool need_w);
// pairs: factor the 128-column blocks in pairs (K = 256 trailing updates)
int hb_big_factor(hb_ctx* c, hb_big* b, int N, double* A, long long lda, bool ldl, bool pairs, int* info_dev);
// the per-block pieces of hb_big_factor, for the block-row step loop (hb_blockrow.cu): one panel step (k_diag128 +
// k_trsm_panel) and the K = 128 trailing update on a block-cyclic matrix
int hb_big_panel(int N, double* A, long long lda, int k0, bool ldl, double* inv16, double* dinv, double* W, long long ldw, int* info_dev, cudaStream_t st);
int hb_big_update_cyclic(int N, const double* P, long long ldp, const double* Q, long long ldq, int qsub, double* C, long long ldc, int nranks, int rank,
                         int q0, int nq, cudaStream_t st);
int hb_big_diag_profile(hb_ctx* c, hb_big* b, int N, double* A, long long lda, int k0, bool ldl, long long* prof_host8);
int hb_big_trailing_from_state(hb_ctx* c, int N, double* A, long long lda, const double* W, long long ldw, const int* state_dev, int r0_min, cudaStream_t st);
int hb_big_block_inverses(hb_ctx* c, hb_big* b, int N, const double* F, long long ldf, bool unit);
int hb_big_solve(hb_ctx* c, hb_big* b, int N, const double* F, long long ldf, int dmode, const int* ipiv_dev, const double* dsub_dev, const int* perm_dev,
                 double* x);

// ---- cluster Bunch-Kaufman (hb_bk_cluster.cu) ----
int hb_bkc_init_attrs(hb_ctx* c);
bool hb_bkc_supported(int N);
int hb_bkc_factor(hb_ctx* c, hb_big* b, int N, double* A, long long lda, int* ipiv_dev, double* dsub_dev, int* perm_dev, double* Wp, long long ldw,
                  int* state_dev, int* swaplog_dev, int* info_dev, int* widths_host);
int hb_bkc_dsolve(hb_ctx* c, int N, const double* F, long long ldf, const int* ipiv_dev, const double* dsub_dev, double* x);
int hb_bkc_profile(hb_ctx* c, int on, long long* prof_host8);
#define HB_BKC_SWAPLOG_INTS(N) ((size_t)((N) / 7 + 4) * 132)
#define HB_BKC_W_DOUBLES(ldw) ((size_t)(ldw) * (64 + 128)) /* W = L*D of a panel (<= 64 columns) + staging rows of the interchange kernel */
// inertia {neg, null, pos} of a cluster Bunch-Kaufman factor with the dsidi rule, all rows in parallel (1x1 / 2x2 blocks marked by
// ipiv, off-diagonal in dsub)
int hb_dense_inertia_blockdiag(hb_ctx* c, int N, const double* F, long long ldf, const int* ipiv_dev, const double* dsub_dev, int* out3_dev);

// ---- random butterfly transform (HB_FACT_RBT_NOPIV, hb_rbt.cu): A' = U^T A U, U = B2 B1, shared by hb_symdense and hb_symdense_dist ----
// oracle/rbt_model.py states every expression; both handles produce the same bits of A', b' and x for a given N.
constexpr double HB_RBT_C = 0.7071067811865476; // the double nearest 1/sqrt(2)
constexpr double HB_RBT_EPS = 0x1p-52;          // refinement target of the backward error
constexpr int HB_RBT_MAX_CORR = 3;

// the entries of column i of a level's butterfly: rows lo and hi (lo = hi = i when unpaired), sign s of the hi side (+1 on the lo side)
struct rbt_pos
{
  int lo, hi;
  double s;
  bool paired;
};
__host__ __device__ __forceinline__ rbt_pos rbt_at(int N, int level, int i)
{
  int o = 0, n = N;
  if(level == 2) {
    const int h = (N + 1) / 2;
    if(i >= h) o = h, n = N - h;
    else n = h;
  }
  const int hh = (n + 1) / 2, t = i - o;
  if(t < n - hh) return {i, i + hh, 1.0, true};
  if(t >= hh) return {i - hh, i, -1.0, true};
  return {i, i, 1.0, false};
}

// out(i, j) of one level, B^T a B, from a(lo_i, lo_j), a(hi_i, hi_j), a(lo_i, hi_j), a(hi_i, lo_j): (f_i f_j) (t w) in the model's order
__device__ __forceinline__ double rbt_entry(double all, double ahh, double alh, double ahl, const rbt_pos& pi, const rbt_pos& pj, double fi, double fj)
{
  const double ss = pi.s * pj.s;
  double t, w;
  if(pi.paired && pj.paired) {
    t = __dadd_rn(__dadd_rn(all, __dmul_rn(ss, ahh)), __dadd_rn(__dmul_rn(pj.s, alh), __dmul_rn(pi.s, ahl)));
    w = 0.5;
  } else if(pi.paired || pj.paired) {
    t = __dadd_rn(all, __dmul_rn(ss, ahh));
    w = HB_RBT_C;
  } else {
    t = all;
    w = 1.0;
  }
  return __dmul_rn(__dmul_rn(fi, fj), __dmul_rn(t, w));
}

// ---- block rows (hb_blockrow.cu): the step loop and the solve sweeps of hb_symdense_dist and hb_symdense_host ----
// Block row k (rows k0 = 128 k .. of the row-major upper triangle) is block column k of the lower view. A handle holds some on the device;
// the others reach it through its transport (another rank's broadcast, or a copy from page-locked host memory).
constexpr int HB_ROWS_DB = 128;  // block size (hb_big_factor's)
constexpr int HB_ROWS_HDR = 136; // step header: 1/d (128 doubles), the breakdown word as the int at slot 128, pad to 16 bytes
enum { HB_ROWS_PH_PANEL = 0, HB_ROWS_PH_MOVE, HB_ROWS_PH_UPDATE, HB_ROWS_PH_COUNT }; // profiled: panel chain, transport + fold, update
int hb_rows_init_attrs();

// What a block-row handle owns for the loop, besides the outcome of its last factorization. The update stream is the context's.
struct hb_rows : hb_dense_result
{
  hb_stream sp;                                     // panel stream (high priority)
  hb_event ev_bc[2], ev_free[2], ev_ahead, ev_join; // per step parity: panel ready, operands free; look-ahead done; panel stream joined
  int create();
};

// Where step k's panel lives on this rank: its header, and its rows from `sub` on (pan[p * ldp + i - sub]: row i of column k0 + p). A
// local panel's rows >= k0 + 128 go there unless pan is null (LDL^T: W = L D; Cholesky: L, copied from A); a received one arrives there
// (LDL^T: W, and L is formed into L with the same layout; Cholesky: L).
struct hb_rows_panel { double* hdr; double* pan; long long ldp; int sub; double* L; };

// Steps 0 .. nsteps-1 of the factorization of the local block columns, hb_big_factor's K = 128 schedule. Block k is local iff k % P ==
// rank and k / P >= q0; local block q = k / P holds global columns k0 .. at A + q * 128 * ld. Per step k:
//   panel stream : wait for ev_free[k & 1]; at(k, local, b); local: zero the header's breakdown word, the panel into b; move(k, local,
//                  b) makes the panel's operands ready; fold the breakdown into *info; received LDL^T: form L (k_trsm_panel's
//                  multiplication; a local panel's L is read from A); ev_bc[k & 1]; block k+1 first when it is local (look-ahead)
//   update stream: behind ev_bc[k & 1], the other local blocks beyond k; then behind the look-ahead, ev_free[k & 1]
// So ev_free[k & 1] is recorded only when every reader of step k's operands, on both streams, is done: a transport reuses its buffers
// of parity k & 1 by waiting for ev_free[k & 1] on the stream that writes them. Every entry of A gets the panels 0, 1, ... in ascending
// order, from the same kernel on the same operand bits. prof: null, or 2 * HB_ROWS_PH_COUNT events per step (begin, end of each phase).
int hb_rows_factor(hb_ctx* c, hb_rows& r, int N, double* A, long long ld, int P, int rank, int q0, int nsteps, bool ldl, double* inv16, int* info,
                   const std::function<int(int k, bool local, hb_rows_panel& b)>& at,
                   const std::function<int(int k, bool local, const hb_rows_panel& b)>& move, hb_event* prof = nullptr);
// out3 = {neg, null, pos} of the diagonal entries A[e * ld + k0 + t] (e = q * 128 + t of the nloc owned blocks) with hb_inertia_count,
// as doubles (the counts the distributed handle all-reduces)
int hb_rows_inertia(const double* A, long long ld, int N, int P, int rank, int nloc, double* out3, cudaStream_t st);
// the same for the whole diagonal of a Cholesky / no-pivot LDL^T factor F (P = 1, A = F, ld = ldf, nloc = ceil(N / 128)), as ints
int hb_dense_inertia_diag(hb_ctx* c, int N, const double* F, long long ldf, int* out3_dev);
// The forward steps on the row-major N x nrhs xw (y_k = L_kk^-1 b_k, b_>k -= L_>k,k y_k, LDL^T: z_k = y_k / d_k) in ascending block order,
// then the backward steps (x_k = L_kk^-T (z_k - L_>k,k^T x_>k)) in descending order. rows(k, &Ak): block row k addressed like the factor
// (Ak[(k0 + p) * ld + i] = L(i, k0 + p)), or null when another rank computes it; after(k, forward) runs after each. ybuf, tdot: 128 nrhs.
int hb_rows_sweeps(int N, long long ld, bool ldl, double* xw, int nrhs, double* ybuf, double* tdot, cudaStream_t st,
                   const std::function<int(int k, const double** Ak)>& rows, const std::function<int(int k, bool forward)>& after);

// global row of local row y of rank `rank` in the block-cyclic layout (P = 1: y)
__host__ __device__ __forceinline__ int rbt_global_row(int y, int P, int rank) { return ((y / HB_ROWS_DB) * P + rank) * HB_ROWS_DB + y % HB_ROWS_DB; }

// Which rows of A a handle holds for the transform: local row y is global row global(y) (-1: none), global row g is local row local(g)
// (-1: not held). rows == nullptr: the block-cyclic rows of rank `rank` of P (hb_symdense_dist); else the explicit map rows[y], pos[g]
// (hb_symdense_host: the window of a strip).
struct hb_rbt_rowmap
{
  const int* rows;
  const int* pos;
  int P, rank;
  __device__ __forceinline__ int global(int y) const { return rows ? rows[y] : rbt_global_row(y, P, rank); }
  __device__ __forceinline__ int local(int g) const
  {
    if(pos) return pos[g];
    return (g / HB_ROWS_DB) % P == rank ? (g / HB_ROWS_DB / P) * HB_ROWS_DB + g % HB_ROWS_DB : -1;
  }
};
// the mirror of the upper triangle: every local row y >= ybeg (of nrows) with global row r gets dst(y, j) = src(j, r) for the columns
// q0 <= j < q0 + nq, j < r, where src holds rows q0 .. (ld doubles each, column r at src[(j - q0) * ld + r])
int hb_rbt_mirror(hb_ctx* c, int N, hb_rbt_rowmap m, int nrows, int ybeg, const double* src, long long ld, int q0, int nq, double* dst);
// one level B^T A B on full rows (ld): for each of the nsrc source rows q (local row x of `in`, global m.global(x); or, with src, global
// row q0 + x held at src + x ld), its partner r, when held (m.local(r) >= 0), gets its whole output row from rows r and q in `out`, at
// the same local row as in `in`. Every output entry is rbt_entry on the model's operands, so it does not depend on the map.
int hb_rbt_level(hb_ctx* c, int N, int level, const double* f, const double* in, long long ld, hb_rbt_rowmap m, int nsrc, const double* src, int q0,
                 double* out);

// f[(level - 1) * N + i]: the diagonal entry of column i at level 1 (B1) and 2 (B2), a function of N alone (2 N doubles)
int hb_rbt_table(hb_ctx* c, int N, double* f);
// x (N x nrhs, one rhs after the other) -> xw (row-major N x nrhs), or back
int hb_rbt_to_rows(hb_ctx* c, int N, int nrhs, double* x, double* xw, bool back);
// rows of a row-major A' (full rows, ld; the nrows local rows of rank `rank` of P in the block-cyclic layout): x == NULL: out[y] =
// sum_j |A'(y, j)| per local row y; else out[r * nrhs + q] = b'(r, q) - sum_j A'(r, j) x'(j, q) per global row r (x, b row-major)
int hb_rbt_rows(hb_ctx* c, int N, int P, int rank, int nrows, const double* A, long long ld, int nrhs, const double* x, const double* b, double* out);
// out[0] = max_i |v(i)| over n entries (NaN kept): ||A'||_inf from the row sums
int hb_rbt_max1(hb_ctx* c, int n, const double* v, double* out);
// The refined RBT solve on the row-major N x nrhs xw (b in, x out): b' = U^T b (kept in bp), sweeps(xw), then while the stopping rule
// allows: residual(x', b', r) forms r = b' - A' x' in rw, sweeps(rw), x' += r; finally x = U x'. omega = max over the rhs of
// ||r||_inf / (anorm ||x'||_inf + ||b'||_inf), NaN for a column where one of the three norms or anorm is not finite, +inf where the
// denominator is 0 and r is not, 0 for a zero column (a NaN wins the max); correct while omega is finite, omega > HB_RBT_EPS, fewer than
// HB_RBT_MAX_CORR corrections were made and omega is at most half its value before the last correction. rw: N nrhs + 3 nrhs doubles,
// nrm_host: 3 nrhs pinned doubles. Returns 1, 0 when omega is not finite, or an HB_ERR_* code; *corr and *berr receive the corrections
// and the last omega. trace (tests only, NULL otherwise) receives what the loop read: it adds copies to the host, never a kernel.
struct hb_rbt_trace
{
  double anorm = 0.0;
  std::vector<double> norms; // per pass: max |r|, max |x'|, max |b'| of every rhs (3 nrhs), then omega
  std::vector<double> x;     // per pass: x' (row-major N x nrhs) before its residual
  std::vector<double> b;     // b' (row-major N x nrhs)
};
int hb_rbt_solve(hb_ctx* c, int N, int nrhs, const double* f, double anorm, double* xw, double* bp, double* rw, double* nrm_host,
                 const std::function<int(double*)>& sweeps, const std::function<int(const double*, const double*, double*)>& residual, int* corr,
                 double* berr, hb_rbt_trace* trace = nullptr);
// The traced solve of the debug entries hb_debug_symdense_rbt_solve / hb_debug_symdense_dist_rbt_solve (who): HB_ERR_STATE without an
// RBT factorization in r; else solve(trace), its return value into *ret_host and what the trace read into the host buffers (every one
// may be NULL)
int hb_rbt_traced_solve(const hb_dense_result& r, const char* who, const std::function<int(hb_rbt_trace*)>& solve, int* ret_host, int* passes,
                        double* anorm, double* norms, double* xp, double* bp);
// One GPU: A' from the upper triangle of A (ld lda; the other triangle is not read) in one pass (k_rbt_fused): the upper triangle of A'
// into F (ldf; may be A itself when hb_rbt_in_place(N), NULL for none), the full A' into Ak (ldk), ||A'||_inf into nrm_dev[0].
// part: hb_rbt_part_doubles(N) doubles of row-sum scratch.
bool hb_rbt_in_place(int N);
size_t hb_rbt_part_doubles(int N);
int hb_rbt_fused(hb_ctx* c, int N, const double* f, const double* A, long long lda, double* F, long long ldf, double* Ak, long long ldk, double* part,
                 double* nrm_dev);
// The strips of the out-of-core transform (hb_symdense_host): strip [s0, s1) of the butterfly slots produces the rows at those slots in
// each of the four quarters of k_rbt_fused's schedule, and reads its window: the same slots (N != 1 mod 4), or one slot more on each side
// plus the three fixed rows (N = 1 mod 4), laid out as k_rbt_fused lays out a tile's window with s1 - s0 slots per quarter.
struct hb_rbt_window
{
  int N, slots, s0, s1, W, wr; // slots: of the longest quarter; W: window slots per quarter; wr: window positions
  int ext, qs[4], qlen[4], sp[3];
};
hb_rbt_window hb_rbt_window_of(int N, int s0, int s1);
// the window's positions: rows[k] = the global row held at position k (-1: none, or held at an earlier position); pos_win[g] = the
// position of global row g (-1: outside), pos_out[g] = the same for the strip's own rows only (-1 elsewhere)
int hb_rbt_window_map(hb_ctx* c, const hb_rbt_window& w, int* rows, int* pos_win, int* pos_out);
// host side of the same: position k of the window (-1: none or a repeat), and whether global row g is one of the strip's rows
int hb_rbt_window_row(const hb_rbt_window& w, int k);
bool hb_rbt_window_out(const hb_rbt_window& w, int g);
