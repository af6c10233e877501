// hiopMatrixDenseRowMajor primitives that round 1 only had fused inside the KKT assembly kernels, as standalone entry points
// (B3 / SURVEY 8 a13), and the curvature test of the inertia-free Newton path (a17):
//   timesMatTrans_local   src/LinAlg/hiopMatrixDenseRowMajor.cpp:646-674   (DGEMM: C = beta C + alpha A B^T)
//   addDiagonal           :703-718     addSubDiagonal :719-764 (three overloads)     addMatrix :766-776 (DAXPY)
//   copyRowsFrom          :169-197     copyBlockFromMatrix / copyFromMatrixBlock :200-236
//   transAddToSymDenseMatrixUpperTriangle :779-798     addUpperTriangleToSymDenseMatrixUpperTriangle :810-829
//   hiopKKTLinSysCompressed::test_direction   src/Optimization/hiopKKTLinSys.cpp:455-509
// All matrices row-major with an explicit leading dimension (elements), FP64. One launch each; they are O(size) streaming kernels.
#include "hb_common.cuh"
#include "hb_lowrank.cuh"

namespace {

constexpr int MT = 256;

// C(i,j) = beta C(i,j) + alpha sum_k A(i,k) B(j,k): one warp per output entry, lanes along k (rows are contiguous)
__global__ void __launch_bounds__(MT)
k_times_mat_trans(int m, int kk, long long n, const double* __restrict__ A, long long lda, const double* __restrict__ B, long long ldb, double beta,
                  double* __restrict__ C, long long ldc, double alpha)
{
  const int lane = threadIdx.x & 31;
  const long long nout = (long long)m * kk;
  for(long long o = (long long)blockIdx.x * (MT / 32) + (threadIdx.x >> 5); o < nout; o += (long long)gridDim.x * (MT / 32)) {
    const int i = (int)(o / kk), j = (int)(o % kk);
    const double* a = A + (size_t)i * lda;
    const double* b = B + (size_t)j * ldb;
    double s = 0.0;
    for(long long q = lane; q < n; q += 32) s += a[q] * b[q];
    s = hb_warp_sum(s);
    if(lane == 0) C[(size_t)i * ldc + j] = (beta == 0.0 ? 0.0 : beta * C[(size_t)i * ldc + j]) + alpha * s;
  }
}
// M[dst0+i][dst0+i] += alpha * (d ? d[src0+i] : 1)
__global__ void k_add_sub_diag(double* __restrict__ M, long long ld, int dst0, int num, double alpha, const double* __restrict__ d, int src0)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < num; i += gridDim.x * blockDim.x) {
    double* q = &M[(size_t)(dst0 + i) * ld + dst0 + i];
    *q = __dadd_rn(*q, d ? __dmul_rn(alpha, d[src0 + i]) : alpha); // product rounded before the add, like the host loops
  }
}
// Y(i,j) += alpha X(i,j)
__global__ void k_add_matrix(int m, int n, double* __restrict__ Y, long long ldy, double alpha, const double* __restrict__ X, long long ldx)
{
  const long long tot = (long long)m * n;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / n), j = (int)(e % n);
    Y[(size_t)i * ldy + j] = __dadd_rn(Y[(size_t)i * ldy + j], __dmul_rn(alpha, X[(size_t)i * ldx + j]));
  }
}
// dst(i, j) = src(rows ? rows[i] : i + i0, j0 + j) for an m x n block
__global__ void k_copy_block(int m, int n, double* __restrict__ dst, long long ldd, int di0, int dj0, const double* __restrict__ src, long long lds,
                             const int* __restrict__ rows, int si0, int sj0)
{
  const long long tot = (long long)m * n;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / n), j = (int)(e % n);
    const int si = rows ? rows[i] : si0 + i;
    dst[(size_t)(di0 + i) * ldd + dj0 + j] = src[(size_t)si * lds + sj0 + j];
  }
}
// W(row_start + j, col_start + i) += alpha A(i,j)   (A m x n; the block must lie in W's upper triangle)
__global__ void k_trans_add_upper(int m, int n, const double* __restrict__ A, long long lda, int row_start, int col_start, double alpha,
                                  double* __restrict__ W, long long ldw)
{
  const long long tot = (long long)m * n;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e / m), i = (int)(e % m); // i fastest: contiguous writes along W's row (row_start + j)
    double* q = &W[(size_t)(row_start + j) * ldw + col_start + i];
    *q = __dadd_rn(*q, __dmul_rn(alpha, A[(size_t)i * lda + j]));
  }
}
// W(diag_start + i, diag_start + j) += alpha A(i,j) for j >= i
__global__ void k_add_upper_to_upper(int n, const double* __restrict__ A, long long lda, int diag_start, double alpha, double* __restrict__ W, long long ldw)
{
  const long long tot = (long long)n * n;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / n), j = (int)(e % n);
    if(j >= i) {
      double* q = &W[(size_t)(diag_start + i) * ldw + diag_start + j];
      *q = __dadd_rn(*q, __dmul_rn(alpha, A[(size_t)i * lda + j]));
    }
  }
}
// partial[blk] = {sum (w[i] + dw[i]) x[i]^2, sum x[i]^2}
__global__ void __launch_bounds__(MT)
k_curv_sums(long long n, const double* __restrict__ x, const double* __restrict__ w, const double* __restrict__ dw, double* __restrict__ partial)
{
  __shared__ double sm[MT / 32];
  double a = 0.0, b = 0.0;
  for(long long i = (long long)blockIdx.x * MT + threadIdx.x; i < n; i += (long long)gridDim.x * MT) {
    const double xi = x[i];
    a += ((w ? w[i] : 0.0) + (dw ? dw[i] : 0.0)) * xi * xi;
    b += xi * xi;
  }
  const double ra = hb_block_sum<MT>(a, sm), rb = hb_block_sum<MT>(b, sm);
  if(threadIdx.x == 0) { partial[2 * blockIdx.x] = ra; partial[2 * blockIdx.x + 1] = rb; }
}

} // namespace

extern "C" int hb_mat_times_mat_trans(hb_ctx* c, int m, int k, long long n, const double* A, long long lda, const double* B, long long ldb, double beta,
                                      double* C, long long ldc, double alpha)
{
  HB_REQUIRE(c && m >= 0 && k >= 0 && n >= 0 && lda >= n && ldb >= n && ldc >= k, "hb_mat_times_mat_trans: bad arguments");
  if(m == 0 || k == 0) return HB_OK;
  k_times_mat_trans<<<hb_grid(c, (long long)m * k * 32, MT), MT, 0, c->stream>>>(m, k, n, A, lda, B, ldb, beta, C, ldc, alpha);
  HB_LAUNCHED();
  if(c->nranks > 1) return hb_fail(HB_ERR_INVALID, "hb_mat_times_mat_trans: local (non-reduced) product only%s", "");
  return HB_OK;
}
extern "C" int hb_mat_add_sub_diagonal(hb_ctx* c, double* M, long long ld, int start_on_dest_diag, int num_elems, double alpha, const double* d,
                                       int start_on_src_vec)
{
  HB_REQUIRE(c && M && start_on_dest_diag >= 0 && num_elems >= 0 && start_on_src_vec >= 0, "hb_mat_add_sub_diagonal: bad arguments");
  if(num_elems == 0) return HB_OK;
  k_add_sub_diag<<<(num_elems + 127) / 128, 128, 0, c->stream>>>(M, ld, start_on_dest_diag, num_elems, alpha, d, start_on_src_vec);
  HB_LAUNCHED();
  return HB_OK;
}
extern "C" int hb_mat_add_matrix(hb_ctx* c, int m, int n, double* Y, long long ldy, double alpha, const double* X, long long ldx)
{
  HB_REQUIRE(c && m >= 0 && n >= 0 && ldy >= n && ldx >= n, "hb_mat_add_matrix: bad arguments");
  if(m == 0 || n == 0) return HB_OK;
  k_add_matrix<<<hb_grid(c, (long long)m * n, MT), MT, 0, c->stream>>>(m, n, Y, ldy, alpha, X, ldx);
  HB_LAUNCHED();
  return HB_OK;
}
extern "C" int hb_mat_copy_rows_from(hb_ctx* c, int n_rows, int n_cols, double* dst, long long ldd, const double* src, long long lds, const int* rows_idx_dev)
{
  HB_REQUIRE(c && n_rows >= 0 && n_cols >= 0 && (rows_idx_dev || n_rows == 0), "hb_mat_copy_rows_from: bad arguments");
  if(n_rows == 0 || n_cols == 0) return HB_OK;
  k_copy_block<<<hb_grid(c, (long long)n_rows * n_cols, MT), MT, 0, c->stream>>>(n_rows, n_cols, dst, ldd, 0, 0, src, lds, rows_idx_dev, 0, 0);
  HB_LAUNCHED();
  return HB_OK;
}
extern "C" int hb_mat_copy_block(hb_ctx* c, int m, int n, double* dst, long long ldd, int dst_i, int dst_j, const double* src, long long lds, int src_i,
                                 int src_j)
{
  HB_REQUIRE(c && m >= 0 && n >= 0 && dst_i >= 0 && dst_j >= 0 && src_i >= 0 && src_j >= 0, "hb_mat_copy_block: bad arguments");
  if(m == 0 || n == 0) return HB_OK;
  k_copy_block<<<hb_grid(c, (long long)m * n, MT), MT, 0, c->stream>>>(m, n, dst, ldd, dst_i, dst_j, src, lds, nullptr, src_i, src_j);
  HB_LAUNCHED();
  return HB_OK;
}
extern "C" int hb_mat_trans_add_to_sym_upper(hb_ctx* c, int m, int n, const double* A, long long lda, int row_start, int col_start, double alpha, double* W,
                                             long long ldw)
{
  HB_REQUIRE(c && m >= 0 && n >= 0 && row_start >= 0 && col_start >= row_start, "hb_mat_trans_add_to_sym_upper: the block must lie in the upper triangle");
  if(m == 0 || n == 0) return HB_OK;
  k_trans_add_upper<<<hb_grid(c, (long long)m * n, MT), MT, 0, c->stream>>>(m, n, A, lda, row_start, col_start, alpha, W, ldw);
  HB_LAUNCHED();
  return HB_OK;
}
extern "C" int hb_mat_add_upper_to_sym_upper(hb_ctx* c, int n, const double* A, long long lda, int diag_start, double alpha, double* W, long long ldw)
{
  HB_REQUIRE(c && n >= 0 && diag_start >= 0, "hb_mat_add_upper_to_sym_upper: bad arguments");
  if(n == 0) return HB_OK;
  k_add_upper_to_upper<<<hb_grid(c, (long long)n * n, MT), MT, 0, c->stream>>>(n, A, lda, diag_start, alpha, W, ldw);
  HB_LAUNCHED();
  return HB_OK;
}

// hiopKKTLinSysCompressed::test_direction for the quasi-Newton / low-rank Hessian: dWd = dx^T (B + Dx + delta_wx) dx + dd^T (Dd + delta_wd) dd
// against neg_curv_test_fact * (||dx||^2 + ||dd||^2). out_host = {dWd, xs_nrmsq}; returns 1 (positive curvature, accept), 0 (negative), <0 error.
extern "C" int hb_lowrank_test_direction(hb_lowrank* k, const double* dx, const double* dd, const double* delta_wx, const double* delta_wd,
                                         double neg_curv_test_fact, double* out_host2)
{
  HB_REQUIRE(k && (dx || k->n == 0) && (dd || k->mineq == 0), "hb_lowrank_test_direction: null argument");
  HB_REQUIRE(k->have_update, "hb_lowrank_test_direction: call hb_lowrank_update first");
  hb_ctx* c = k->ctx;
  double bxx = 0.0;
  if(k->n > 0) {
    HB_CHECK(hb_lowrank_hess_times_vec(k, 0.0, k->nv2, 1.0, dx, 0)); // B dx (compact form)
    HB_CHECK(hb_vec_dot(c, k->n, k->nv2, dx, &bxx));                  // all-reduced
  }
  const int g1 = hb_grid(c, k->n, MT), g2 = hb_grid(c, k->mineq, MT);
  HB_CHECK(hb_ws_reserve(c, sizeof(double) * (2 * (size_t)(g1 + g2) + 8)));
  double* p1 = (double*)c->ws;
  double* p2 = p1 + 2 * g1;
  double* out = p2 + 2 * g2;
  k_curv_sums<<<g1, MT, 0, c->stream>>>(k->n, dx, k->Dx, delta_wx, p1);
  HB_LAUNCHED();
  k_curv_sums<<<g2, MT, 0, c->stream>>>(k->mineq, dd, k->Dd, delta_wd, p2);
  HB_LAUNCHED();
  HB_CHECK(hb_reduce_slots(c, g1, p1, out, {HB_SUM, HB_SUM}));
  HB_CHECK(hb_reduce_slots(c, g2, p2, out + 2, {HB_SUM, HB_SUM}));
  if(c->nranks > 1) {
    // the x-sized sums are sharded, the d-sized ones replicated: only rank 0 contributes the latter
    if(c->rank != 0) HB_CUDA(cudaMemsetAsync(out + 2, 0, 2 * sizeof(double), c->stream));
    HB_CHECK(hb_allreduce_sum(c, out, 4));
  }
  double h[4];
  HB_CUDA(cudaMemcpyAsync(h, out, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  const double dWd = bxx + h[0] + h[2], xs = h[1] + h[3];
  if(out_host2) { out_host2[0] = dWd; out_host2[1] = xs; }
  return dWd < xs * neg_curv_test_fact ? 0 : 1;
}
