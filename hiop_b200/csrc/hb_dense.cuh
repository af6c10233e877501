// Internal API of the dense symmetric factorizations / solves on device: the device helpers their kernel files share, the entry points
// of each kernel file (each runs one path, no fall-back), and the per-caller dispatch of hb_symdense.cu that chooses between them.
#pragma once
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

struct hb_big;

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
// inertia {neg, null, pos} from the diagonal with the dsidi thresholds, all rows in parallel: of a cluster Bunch-Kaufman factor
// (1x1 / 2x2 blocks marked by ipiv, off-diagonal in dsub), or of a Cholesky / no-pivot LDL^T factor (signs of the diagonal)
int hb_dense_inertia_blockdiag(hb_ctx* c, int N, const double* F, long long ldf, const int* ipiv_dev, const double* dsub_dev, int* out3_dev);
int hb_dense_inertia_diag(hb_ctx* c, int N, const double* F, long long ldf, int* out3_dev);
