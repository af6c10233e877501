// The dense symmetric system factored across the ranks of the context's communicator: Cholesky LL^T and no-pivot LDL^T on a 1-D
// block-cyclic layout, with NCCL broadcasts of the panels (hb_symdense_dist_*, include/hiopb200.h).
//
// Layout. Block size 128 (that of hb_big_factor). Block row k of the N x N row-major upper triangle (rows k*128 .. min(N, k*128+128)-1,
// full width) is block column k of the column-major lower view the kernels use (hb_dense.cuh). It belongs to rank k mod P and is
// stored as local block q = k div P: the owned block rows are stacked in order, each 128 rows of ld doubles.
//
// Factorization, step k (all ranks run the same host sequence, so every rank issues the same collectives in the same order):
//   owner of k, panel stream : k_diag128 + k_trsm_panel of block k (hb_big_panel) into the broadcast buffer: header [1/d (128), info]
//                              + the panel rows >= (k+1)*128 (Cholesky: L; LDL^T: W = L D, as hb_big_factor uses them)
//   every rank, panel stream : ncclBroadcast of that buffer from the owner; fold the header's info word; LDL^T: L = W * (1/d)
//   owner of k+1, panel stream: look-ahead, the panel applied to block k+1 first, so that its panel chain runs under the others' update
//   every rank, update stream: the panel applied to every other owned block column beyond k (k_gemm_pq, block-cyclic epilogue)
// Each entry sees the same k_diag128 / k_trsm_panel / k_gemm_pq arithmetic in the same k order as hb_big_factor with K = 128, so the
// factor is bit-identical to hb_symdense's look-ahead path (unpaired blocks) for every P. Broadcast buffers are double-buffered across
// steps. A breakdown (the first failing column, like hb_big_factor's info word) travels in the header of its step, so every rank
// returns the same value; like the single-GPU path, the factorization runs to its last block either way.
//
// Solves (x replicated on every rank): forward sweep, owner of block k: y_k = L_kk^-1 b_k, b_>k -= L_>k,k y_k, z_k = y_k (/ d_k), then
// the broadcast of rows k*128 .. N; backward sweep, owner of block k: x_k = L_kk^-T (z_k - L_>k,k^T x_>k), broadcast of its rows. Every
// block is computed by its owner in the same order for every P, so the solution does not depend on P.
//
// Safe mode (HB_FACT_RBT_NOPIV): A' = U^T A U with a depth-2 random butterfly U = B2 B1 (rbt_transform: the mirror of the upper
// triangle, then one pass per level, each output row formed from its row and its partner row), the no-pivot LDL^T above on A', and
// solves refined against a kept copy of A' (rbt_solve, the refinement loop of hb_rbt.cu). Every entry of A' is a fixed expression of oracle/rbt_model.py and the random
// diagonals depend on N alone, so A', the factor and the solution do not depend on P either.
#include "hb_common.cuh"
#include "hb_dense.cuh"

namespace {

constexpr int DB = HB_DIST_DB;   // block size = hb_big_factor's
constexpr int HDR = 136;         // broadcast header: 1/d (128 doubles), info word (as the first int of slot 128), pad to 16 bytes
constexpr int SOLVE_RHS = 4;     // right-hand sides per CTA of the diagonal-block solves
constexpr int DLD = DB + 1;      // shared-memory stride of the diagonal block
constexpr size_t DIAG_SMEM = sizeof(double) * ((size_t)DB * DLD + SOLVE_RHS * DB);

// fold the breakdown of a received step into the factorization's info word (the first one stays, as in hb_big_factor); LDL^T: form
// L = W * (1/d) of the received panel with the operation k_trsm_panel uses, so that L is bit-identical to the owner's
__global__ void k_dist_recv(const double* __restrict__ hdr, const double* __restrict__ W, long long ldb, int rows, int ldl, double* __restrict__ L,
                            int* __restrict__ info)
{
  if(blockIdx.x == 0 && threadIdx.x == 0) {
    const int step = *reinterpret_cast<const int*>(hdr + DB);
    if(*info == 0 && step != 0) *info = step;
  }
  if(!ldl) return;
  const long long total = (long long)DB * ldb;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e / ldb), i = (int)(e % ldb);
    if(i < rows) L[e] = W[e] * hdr[c];
  }
}

// {neg, null, pos} of the owned diagonal entries with the +-1e-14 rule of the I_DIAG sweep (hb_dense_inertia_diag)
__global__ void __launch_bounds__(1024) k_dist_inertia(const double* __restrict__ A, long long ld, int N, int P, int rank, int nloc, double* __restrict__ out3)
{
  __shared__ int cnt[3];
  if(threadIdx.x < 3) cnt[threadIdx.x] = 0;
  __syncthreads();
  int neg = 0, nul = 0, pos = 0;
  for(int e = threadIdx.x; e < nloc * DB; e += blockDim.x) {
    const int q = e / DB, t = e % DB, k0 = (q * P + rank) * DB;
    if(k0 + t >= N) continue;
    const double d = A[(size_t)e * ld + k0 + t];
    if(d < -1e-14) neg++; else if(d < 1e-14) nul++; else pos++;
  }
  atomicAdd(&cnt[0], neg); atomicAdd(&cnt[1], nul); atomicAdd(&cnt[2], pos);
  __syncthreads();
  if(threadIdx.x < 3) out3[threadIdx.x] = (double)cnt[threadIdx.x];
}

// the nb x nb diagonal block of block column k0 into shared memory: S[j * DLD + i] = L(k0 + i, k0 + j), i >= j
__device__ __forceinline__ void load_diag(const double* __restrict__ A, long long ld, int k0, int nb, double* S)
{
  for(int e = threadIdx.x; e < nb * nb; e += blockDim.x) {
    const int j = e / nb, i = e % nb;
    if(i >= j) S[j * DLD + i] = A[(size_t)(k0 + j) * ld + k0 + i];
  }
  __syncthreads();
}

// forward: y = L_kk^-1 b_k for SOLVE_RHS rhs per CTA (thread = row i, rhs cl); y -> ybuf, z = y (LDL^T: y / d) -> xw
__global__ void __launch_bounds__(DB * SOLVE_RHS) k_dist_fwd_diag(const double* __restrict__ A, long long ld, int k0, int nb, int ldl, double* __restrict__ xw,
                                                                  int nrhs, double* __restrict__ ybuf)
{
  extern __shared__ double dsm[];
  double* S = dsm;
  double* ys = dsm + DB * DLD;
  load_diag(A, ld, k0, nb, S);
  const int i = threadIdx.x % DB, cl = threadIdx.x / DB, c = blockIdx.x * SOLVE_RHS + cl;
  const bool live = i < nb && c < nrhs;
  double b = live ? xw[(size_t)(k0 + i) * nrhs + c] : 0.0;
  for(int j = 0; j < nb; j++) {
    if(i == j) ys[cl * DB + j] = ldl ? b : b / S[j * DLD + j];
    __syncthreads();
    if(i > j) b -= S[j * DLD + i] * ys[cl * DB + j];
  }
  if(live) {
    const double y = ys[cl * DB + i];
    ybuf[(size_t)i * nrhs + c] = y;
    xw[(size_t)(k0 + i) * nrhs + c] = ldl ? y / S[i * DLD + i] : y;
  }
}

// forward: b_i -= sum_p L(i, k0 + p) y_p for the rows i >= k0 + 128
__global__ void k_dist_fwd_panel(const double* __restrict__ A, long long ld, int N, int k0, double* __restrict__ xw, int nrhs, const double* __restrict__ ybuf)
{
  const int i = k0 + DB + blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= N) return;
  for(int c = 0; c < nrhs; c++) {
    double acc = 0.0;
    for(int p = 0; p < DB; p++) acc += A[(size_t)(k0 + p) * ld + i] * ybuf[(size_t)p * nrhs + c];
    xw[(size_t)i * nrhs + c] -= acc;
  }
}

// backward: t[p][c] = sum_{i >= k0 + 128} L(i, k0 + p) x_i (one CTA per p, fixed-order block reduction)
__global__ void __launch_bounds__(256) k_dist_bwd_dots(const double* __restrict__ A, long long ld, int N, int k0, const double* __restrict__ xw, int nrhs,
                                                       double* __restrict__ t)
{
  __shared__ double red[8];
  const int p = blockIdx.x;
  const double* col = A + (size_t)(k0 + p) * ld;
  for(int c = 0; c < nrhs; c++) {
    double acc = 0.0;
    for(int i = k0 + DB + threadIdx.x; i < N; i += 256) acc += col[i] * xw[(size_t)i * nrhs + c];
    acc = hb_block_sum<256>(acc, red);
    if(threadIdx.x == 0) t[(size_t)p * nrhs + c] = acc;
  }
}

// backward: x_k = L_kk^-T (z_k - t) (unit diagonal for LDL^T) in place in xw
__global__ void __launch_bounds__(DB * SOLVE_RHS) k_dist_bwd_diag(const double* __restrict__ A, long long ld, int k0, int nb, int ldl, double* __restrict__ xw,
                                                                  int nrhs, const double* __restrict__ t)
{
  extern __shared__ double dsm[];
  double* S = dsm;
  double* xs = dsm + DB * DLD;
  load_diag(A, ld, k0, nb, S);
  const int i = threadIdx.x % DB, cl = threadIdx.x / DB, c = blockIdx.x * SOLVE_RHS + cl;
  const bool live = i < nb && c < nrhs;
  double v = live ? xw[(size_t)(k0 + i) * nrhs + c] : 0.0;
  if(live && t) v -= t[(size_t)i * nrhs + c];
  for(int j = nb - 1; j >= 0; j--) {
    if(i == j) xs[cl * DB + j] = ldl ? v : v / S[j * DLD + j];
    __syncthreads();
    if(i < j) v -= S[i * DLD + j] * xs[cl * DB + j];
  }
  if(live) xw[(size_t)(k0 + i) * nrhs + c] = xs[cl * DB + i];
}

// ---- random butterfly transform (HB_FACT_RBT_NOPIV): A' = U^T A U, U = B2 B1 (oracle/rbt_model.py states every expression; the
// diagonals, the vector and row kernels and the refined solve are shared with hb_symdense in hb_rbt.cu) ------------------------------
constexpr int RBT_COLS = 1024;               // columns per CTA of k_rbt_level (256 threads x 4)

// mirror: every owned row r gets dst(r, j) = src(j, r) for the columns q0 <= j < q0 + nq, j < r, where src holds the rows q0 .. of the
// upper triangle (ld doubles each). 32 x 32 tiles through shared memory: rows y0 .. of the owned rows, starting at local row ybeg.
__global__ void __launch_bounds__(256) k_rbt_mirror(int N, int P, int rank, int nrows, int ybeg, const double* __restrict__ src, long long ld, int q0,
                                                    int nq, double* __restrict__ dst)
{
  __shared__ double tile[32][33];
  const int y0 = ybeg + blockIdx.y * 32, j0 = q0 + blockIdx.x * 32, tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  for(int jj = ty; jj < 32; jj += 8) {
    const int y = y0 + tx, j = j0 + jj;
    const int r = rbt_global_row(y, P, rank);
    tile[jj][tx] = (y < nrows && r < N && j < q0 + nq && j < r) ? src[(size_t)(j - q0) * ld + r] : 0.0;
  }
  __syncthreads();
  for(int yy = ty; yy < 32; yy += 8) {
    const int y = y0 + yy, j = j0 + tx;
    const int r = rbt_global_row(y, P, rank);
    if(y < nrows && r < N && j < q0 + nq && j < r) dst[(size_t)y * ld + j] = tile[tx][yy];
  }
}

// one level B^T A B on full rows. CTA x = a source row q: local row x of `in` (src == nullptr: every partner is local) or row x of src
// (global rows q0 .. q0 + nq, the owner's broadcast). Its partner r (q itself when unpaired), when this rank owns it, gets its whole
// output row from rows r and q: out(r, j) = (f_r f_j) (t w) with t and w of oracle/rbt_model.py, in that operation order.
__global__ void __launch_bounds__(256) k_rbt_level(int N, int level, const double* __restrict__ f, const double* __restrict__ in, long long ld, int P,
                                                   int rank, const double* __restrict__ src, int q0, double* __restrict__ out)
{
  const int q = src ? q0 + blockIdx.x : rbt_global_row(blockIdx.x, P, rank);
  if(q >= N) return;
  const double* rowq = src ? src + (size_t)blockIdx.x * ld : in + (size_t)blockIdx.x * ld;
  const rbt_pos pq = rbt_at(N, level, q);
  const int r = pq.lo == q ? pq.hi : pq.lo;
  if((r / DB) % P != rank) return;
  const size_t lr = (size_t)(r / DB / P) * DB + r % DB;
  const double* rowr = in + lr * ld;
  const rbt_pos pr = rbt_at(N, level, r);
  const double* RL = pr.lo == r ? rowr : rowq;
  const double* RH = pr.hi == r ? rowr : rowq;
  const double* fl = f + (size_t)(level - 1) * N;
  const double fi = fl[r];
  double* o = out + lr * ld;
  const int jend = min(N, (int)(blockIdx.y + 1) * RBT_COLS);
  for(int j = blockIdx.y * RBT_COLS + threadIdx.x; j < jend; j += 256) {
    const rbt_pos pj = rbt_at(N, level, j);
    o[j] = rbt_entry(RL[pj.lo], RH[pj.hi], RL[pj.hi], RH[pj.lo], pr, pj, fi, fl[j]);
  }
}

enum { PH_PANEL = 0, PH_BCAST, PH_UPDATE, PH_COUNT };

// Every rank's local result rc (HB_OK or an HB_ERR_* code) made common before the next collective, so that a rank whose allocation
// failed never leaves the others waiting in a broadcast: all ranks return the most severe code (their own when they failed).
int agree(hb_ctx* c, int rc)
{
  if(c->nranks == 1) return rc;
  c->red_host[0] = -(double)rc;
  HB_CUDA(cudaMemcpyAsync(c->red_dev, c->red_host, sizeof(double), cudaMemcpyHostToDevice, c->stream));
  HB_CHECK(hb_allreduce_op(c, c->red_dev, 1, HB_MAX));
  HB_CUDA(cudaMemcpyAsync(c->red_host, c->red_dev, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  const int worst = -(int)c->red_host[0];
  if(rc != HB_OK || worst == HB_OK) return rc;
  snprintf(g_hb_err, sizeof(g_hb_err), "hb_symdense_dist: another rank failed with code %d", worst);
  return worst;
}

} // namespace

// ---- the per-block kernels above, for this file and the host-resident handle (hb_symdense_host.cu) ----
int hb_dist_init_attrs()
{
  HB_CUDA(cudaFuncSetAttribute(k_dist_fwd_diag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DIAG_SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_dist_bwd_diag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DIAG_SMEM));
  return HB_OK;
}

int hb_dist_form_l(hb_ctx* c, const double* hdr, const double* W, long long ldb, int rows, double* L, int* info, cudaStream_t st)
{
  k_dist_recv<<<hb_grid(c, DB * ldb), 256, 0, st>>>(hdr, W, ldb, rows, 1, L, info);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dist_inertia(const double* A, long long ld, int N, int P, int rank, int nloc, double* out3, cudaStream_t st)
{
  k_dist_inertia<<<1, 1024, 0, st>>>(A, ld, N, P, rank, nloc, out3);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dist_fwd_block(const double* Ak, long long ld, int N, int k0, bool ldl, double* xw, int nrhs, double* ybuf, cudaStream_t st)
{
  const int nb = N - k0 < DB ? N - k0 : DB, rows = N - k0 - nb, ctas = (nrhs + SOLVE_RHS - 1) / SOLVE_RHS;
  k_dist_fwd_diag<<<ctas, DB * SOLVE_RHS, DIAG_SMEM, st>>>(Ak, ld, k0, nb, ldl ? 1 : 0, xw, nrhs, ybuf);
  HB_LAUNCHED();
  if(rows > 0) {
    k_dist_fwd_panel<<<(rows + 255) / 256, 256, 0, st>>>(Ak, ld, N, k0, xw, nrhs, ybuf);
    HB_LAUNCHED();
  }
  return HB_OK;
}

int hb_dist_bwd_block(const double* Ak, long long ld, int N, int k0, bool ldl, double* xw, int nrhs, double* tdot, cudaStream_t st)
{
  const int nb = N - k0 < DB ? N - k0 : DB, rows = N - k0 - nb, ctas = (nrhs + SOLVE_RHS - 1) / SOLVE_RHS;
  if(rows > 0) {
    k_dist_bwd_dots<<<nb, 256, 0, st>>>(Ak, ld, N, k0, xw, nrhs, tdot);
    HB_LAUNCHED();
  }
  k_dist_bwd_diag<<<ctas, DB * SOLVE_RHS, DIAG_SMEM, st>>>(Ak, ld, k0, nb, ldl ? 1 : 0, xw, nrhs, rows > 0 ? tdot : nullptr);
  HB_LAUNCHED();
  return HB_OK;
}

struct hb_symdense_dist
{
  hb_ctx* ctx = nullptr;
  int N = 0, P = 1, rank = 0, nblk = 0, nloc = 0;
  long long ld = 0;
  hb_dev<double> A;           // nloc * 128 rows of ld doubles: the owned block rows, in order
  hb_dev<double> bbuf[2];     // broadcast buffers: [ld doubles of slack | header | 128 x ldb panel]
  hb_dev<double> Lbuf[2];     // LDL^T: L of the received panel (allocated with the handle: no allocation between collectives)
  hb_dev<double> inv16;       // k_diag128 scratch
  hb_dev<int> info;           // [0]: the first breakdown column (1-based, 0: none)
  hb_dev<double> red;         // inertia counts, all-reduced
  hb_pinned<double> red_host;
  hb_pinned<int> info_host;
  hb_dev<double> xw, ybuf, tdot; // solve
  hb_stream sp;               // panel stream
  hb_event ev_bc[2], ev_free[2], ev_join;
  // per-phase timing (hb_symdense_dist_profile): begin / end events of each phase of each step
  bool profile = false;
  std::unique_ptr<hb_event[]> ev_prof;
  float phase_ms[PH_COUNT] = {0.f, 0.f, 0.f};
  int mode = -1;
  bool factored = false;
  int n_neg = 0, n_null = 0, n_pos = 0;
  // HB_FACT_RBT_NOPIV, allocated by the first RBT factorization: A' (full rows, owned like A), the butterfly diagonals (2 N), the row
  // sums of |A'| and norm scratch; the solve adds b', the residual and the per-rhs norms
  bool rbt_ready = false;
  hb_dev<double> Ak, rbt_f, rbt_rows, rbt_nrm, rbt_b, rbt_r;
  hb_pinned<double> rbt_nrm_host;
  hb_event ev_rbt[2];
  double rbt_anorm = 0.0, rbt_berr = 0.0;
  int rbt_corr = 0;
  float rbt_ms = 0.f;
  ~hb_symdense_dist()
  {
    if(sp) cudaStreamSynchronize(sp);
  }
};

extern "C" int hb_symdense_dist_create(hb_ctx* c, int N, hb_symdense_dist** out)
{
  HB_REQUIRE(c && out, "hb_symdense_dist_create: null argument");
  HB_CUDA(cudaSetDevice(c->device));
  if(c->nranks > 1) {
    // every rank must see the same order, and be able to broadcast, before any rank allocates or enters a broadcast: all refuse
    // together otherwise
    if(!c->nccl_comm) return hb_fail(HB_ERR_COMM, "hb_symdense_dist_create: communicator not initialised%s", "");
    const int ready = hb_broadcast_ready(c);
    c->red_host[0] = N;
    c->red_host[1] = -(double)N;
    c->red_host[2] = -(double)ready;
    HB_CUDA(cudaMemcpyAsync(c->red_dev, c->red_host, sizeof(double) * 3, cudaMemcpyHostToDevice, c->stream));
    HB_CHECK(hb_allreduce_op(c, c->red_dev, 3, HB_MAX));
    HB_CUDA(cudaMemcpyAsync(c->red_host, c->red_dev, sizeof(double) * 3, cudaMemcpyDeviceToHost, c->stream));
    HB_CUDA(cudaStreamSynchronize(c->stream));
    HB_REQUIRE(c->red_host[0] == -c->red_host[1], "hb_symdense_dist_create: the ranks passed different orders N");
    if(c->red_host[2] != 0.0) return ready != HB_OK ? ready : hb_fail(HB_ERR_COMM, "hb_symdense_dist_create: another rank cannot broadcast%s", "");
  }
  HB_REQUIRE(N >= 0, "hb_symdense_dist_create: negative order");
  std::unique_ptr<hb_symdense_dist> s(new hb_symdense_dist);
  s->ctx = c;
  s->N = N;
  s->P = c->nranks;
  s->rank = c->rank;
  s->nblk = (N + DB - 1) / DB;
  s->nloc = s->nblk > s->rank ? (s->nblk - s->rank + s->P - 1) / s->P : 0;
  s->ld = N > 0 ? ((N + 7) & ~7LL) : 8;
  auto allocate = [&]() -> int {
    HB_CHECK(s->A.reserve(c, (size_t)s->nloc * DB * s->ld, "the owned block rows"));
    HB_CUDA(cudaMemsetAsync(s->A, 0, sizeof(double) * s->A.capacity(), c->stream));
    for(int b = 0; b < 2; b++) {
      HB_CHECK(s->bbuf[b].reserve(c, (size_t)s->ld + HDR + (size_t)DB * s->ld, "panel broadcast buffer"));
      HB_CHECK(s->Lbuf[b].reserve(c, (size_t)DB * s->ld, "received panel"));
    }
    HB_CHECK(s->inv16.reserve(c, 8 * 16 * 17, "diagonal-block scratch"));
    HB_CHECK(s->info.reserve(c, 4, "info words"));
    HB_CHECK(s->info_host.reserve(c, 4, "info words"));
    HB_CHECK(s->red.reserve(c, 4, "inertia counts"));
    HB_CHECK(s->red_host.reserve(c, 4, "inertia counts"));
    int lo = 0, hi = 0;
    HB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    HB_CHECK(s->sp.create(cudaStreamNonBlocking, hi));
    for(int b = 0; b < 2; b++) {
      HB_CHECK(s->ev_bc[b].create(cudaEventDisableTiming));
      HB_CHECK(s->ev_free[b].create(cudaEventDisableTiming));
    }
    HB_CHECK(s->ev_join.create(cudaEventDisableTiming));
    HB_CHECK(hb_dist_init_attrs());
    HB_CUDA(cudaStreamSynchronize(c->stream));
    return HB_OK;
  };
  HB_CHECK(agree(c, allocate()));
  *out = s.release();
  return HB_OK;
}

extern "C" int hb_symdense_dist_destroy(hb_symdense_dist* s)
{
  if(!s) return HB_OK;
  cudaSetDevice(s->ctx->device);
  cudaStreamSynchronize(s->ctx->stream);
  delete s;
  return HB_OK;
}

extern "C" int hb_symdense_dist_local(hb_symdense_dist* s, double** A_local, long long* ld, int* n_blocks)
{
  HB_REQUIRE(s, "null handle");
  if(A_local) *A_local = s->A.get();
  if(ld) *ld = s->ld;
  if(n_blocks) *n_blocks = s->nloc;
  return HB_OK;
}

extern "C" int hb_symdense_dist_order(hb_symdense_dist* s) { return s ? s->N : -1; }

extern "C" int hb_symdense_dist_profile(hb_symdense_dist* s, int on, float* ms3)
{
  HB_REQUIRE(s, "null handle");
  if(on) {
    if(!s->ev_prof) {
      s->ev_prof.reset(new hb_event[(size_t)2 * PH_COUNT * (s->nblk > 0 ? s->nblk : 1)]);
      for(int e = 0; e < 2 * PH_COUNT * s->nblk; e++) HB_CHECK(s->ev_prof[e].create(cudaEventDefault));
    }
    for(float& m : s->phase_ms) m = 0.f;
    s->profile = true;
    return HB_OK;
  }
  s->profile = false;
  if(ms3)
    for(int p = 0; p < PH_COUNT; p++) ms3[p] = s->phase_ms[p];
  return HB_OK;
}

// the RBT buffers, on the first RBT factorization of the handle (every rank calls it, then agree())
static int rbt_reserve(hb_symdense_dist* s)
{
  if(s->rbt_ready) return HB_OK;
  hb_ctx* c = s->ctx;
  HB_CHECK(s->Ak.reserve(c, (size_t)s->nloc * DB * s->ld, "the transformed matrix A'"));
  HB_CHECK(s->rbt_f.reserve(c, (size_t)2 * s->N, "butterfly diagonals"));
  HB_CHECK(s->rbt_rows.reserve(c, (size_t)s->nloc * DB, "row sums of |A'|"));
  HB_CHECK(s->rbt_nrm.reserve(c, 4, "norm of A'"));
  for(int e = 0; e < 2; e++) HB_CHECK(s->ev_rbt[e].create(cudaEventDefault));
  HB_CHECK(hb_rbt_table(c, s->N, s->rbt_f));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  s->rbt_ready = true;
  return HB_OK;
}

// true when every row's partner at `level` is owned by the rank that owns the row, decided from N and P alone (every rank agrees): all
// pairing distances are multiples of 128 P
static bool rbt_level_local(int N, int P, int level)
{
  if(P == 1) return true;
  auto ok = [&](int n) { const int hh = (n + 1) / 2; return n - hh == 0 || hh % (DB * P) == 0; };
  if(level == 1) return ok(N);
  const int h = (N + 1) / 2;
  return ok(h) && ok(N - h);
}

// the first `stages` steps of A' = U^T A U on the owned rows: the mirror of the upper triangle into the lower part of every row, then
// B2^T A B2 (stage 1) and B1^T (.) B1 (stage 2). The result is left in A; after stage 2 it is also kept in Ak, with ||A'||_inf in
// rbt_anorm. Every rank issues the same broadcasts: the owner of block k sends its rows from its own buffer, the others receive them in
// the first panel broadcast buffer.
static int rbt_transform(hb_symdense_dist* s, int stages)
{
  hb_ctx* c = s->ctx;
  const int N = s->N, P = s->P, rank = s->rank, nrows = s->nloc * DB;
  const long long ld = s->ld;
  cudaStream_t st = c->stream;
  double* recv = s->bbuf[0];
  if(s->profile) HB_CUDA(cudaEventRecord(s->ev_rbt[0], st));
  // mirror
  for(int k = 0; k < s->nblk; k++) {
    const int owner = k % P, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
    double* src = P == 1 ? s->A.get() : (owner == rank ? s->A.get() + (size_t)(k / P) * DB * ld : recv);
    if(P > 1) HB_CHECK(hb_broadcast(c, src, (long long)nb * ld, owner, st));
    const int q0 = P == 1 ? 0 : k0, nq = P == 1 ? N : nb;
    const int qa = k <= rank ? 0 : (k - rank + P - 1) / P; // first owned block at or after k
    if(nrows > qa * DB) {
      k_rbt_mirror<<<dim3((nq + 31) / 32, (nrows - qa * DB + 31) / 32), 256, 0, st>>>(N, P, rank, nrows, qa * DB, src, ld, q0, nq, s->A);
      HB_LAUNCHED();
    }
    if(P == 1) break;
  }
  // the two levels: A -> Ak (B2), Ak -> A (B1)
  const int chunks = (N + RBT_COLS - 1) / RBT_COLS;
  for(int st_i = 0; st_i < stages; st_i++) {
    const int level = st_i == 0 ? 2 : 1;
    const double* in = st_i == 0 ? s->A.get() : s->Ak.get();
    double* out = st_i == 0 ? s->Ak.get() : s->A.get();
    if(rbt_level_local(N, P, level)) {
      if(nrows > 0) {
        k_rbt_level<<<dim3(nrows, chunks), 256, 0, st>>>(N, level, s->rbt_f, in, ld, P, rank, nullptr, 0, out);
        HB_LAUNCHED();
      }
      continue;
    }
    for(int k = 0; k < s->nblk; k++) {
      const int owner = k % P, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
      double* src = owner == rank ? const_cast<double*>(in) + (size_t)(k / P) * DB * ld : recv;
      HB_CHECK(hb_broadcast(c, src, (long long)nb * ld, owner, st));
      k_rbt_level<<<dim3(nb, chunks), 256, 0, st>>>(N, level, s->rbt_f, in, ld, P, rank, src, k0, out);
      HB_LAUNCHED();
    }
  }
  if(stages == 1) HB_CUDA(cudaMemcpyAsync(s->A, s->Ak, sizeof(double) * nrows * ld, cudaMemcpyDeviceToDevice, st));
  if(s->profile) HB_CUDA(cudaEventRecord(s->ev_rbt[1], st));
  if(stages == 2) {
    HB_CUDA(cudaMemcpyAsync(s->Ak, s->A, sizeof(double) * nrows * ld, cudaMemcpyDeviceToDevice, st));
    HB_CHECK(hb_rbt_rows(c, N, P, rank, nrows, s->Ak, ld, 0, nullptr, nullptr, s->rbt_rows));
    HB_CHECK(hb_rbt_max1(c, nrows, s->rbt_rows, s->rbt_nrm));
    HB_CHECK(hb_allreduce_op(c, s->rbt_nrm, 1, HB_MAX));
    HB_CUDA(cudaMemcpyAsync(s->red_host, s->rbt_nrm, sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  HB_CUDA(cudaStreamSynchronize(st));
  if(stages == 2) s->rbt_anorm = s->red_host[0];
  s->rbt_ms = 0.f;
  if(s->profile) HB_CUDA(cudaEventElapsedTime(&s->rbt_ms, s->ev_rbt[0], s->ev_rbt[1]));
  return HB_OK;
}

extern "C" int hb_debug_symdense_dist_rbt(hb_symdense_dist* s, int stages)
{
  HB_REQUIRE(s && stages >= 0 && stages <= 2, "hb_debug_symdense_dist_rbt: bad arguments");
  if(s->N == 0) return HB_OK;
  HB_CUDA(cudaSetDevice(s->ctx->device));
  HB_CHECK(agree(s->ctx, rbt_reserve(s)));
  s->factored = false;
  return rbt_transform(s, stages);
}

extern "C" int hb_symdense_dist_rbt_stats(hb_symdense_dist* s, int* corrections, double* backward_error, float* transform_ms)
{
  HB_REQUIRE(s, "null handle");
  if(corrections) *corrections = s->rbt_corr;
  if(backward_error) *backward_error = s->rbt_berr;
  if(transform_ms) *transform_ms = s->rbt_ms;
  return HB_OK;
}

extern "C" int hb_symdense_dist_matrix_changed(hb_symdense_dist* s, int mode)
{
  HB_REQUIRE(s, "null handle");
  if(mode == HB_FACT_BUNCH_KAUFMAN)
    return hb_fail(HB_ERR_INVALID, "hb_symdense_dist_matrix_changed: Bunch-Kaufman is not distributed (its pivot search needs every column); use hb_symdense "
                                   "or HB_FACT_RBT_NOPIV%s", "");
  HB_REQUIRE(mode == HB_FACT_NOPIV || mode == HB_FACT_CHOLESKY || mode == HB_FACT_RBT_NOPIV, "hb_symdense_dist_matrix_changed: bad mode");
  hb_ctx* c = s->ctx;
  const int N = s->N, P = s->P, rank = s->rank;
  const bool ldl = mode != HB_FACT_CHOLESKY;
  s->mode = mode;
  s->factored = false;
  if(N == 0) { s->factored = true; s->n_neg = s->n_null = s->n_pos = 0; return 0; }
  HB_CUDA(cudaSetDevice(c->device));
  if(mode == HB_FACT_RBT_NOPIV) {
    HB_CHECK(agree(c, rbt_reserve(s)));
    HB_CHECK(rbt_transform(s, 2));
  }
  cudaStream_t su = c->stream, sp = s->sp;
  const long long ld = s->ld;
  double* A = s->A;
  HB_CUDA(cudaMemsetAsync(s->info, 0, sizeof(int) * 4, su));
  HB_CUDA(cudaEventRecord(s->ev_free[0], su));
  HB_CUDA(cudaEventRecord(s->ev_free[1], su));
  auto mark = [&](int k, int ph, int end, cudaStream_t st) -> int {
    if(s->profile) HB_CUDA(cudaEventRecord(s->ev_prof[((size_t)k * PH_COUNT + ph) * 2 + end], st));
    return HB_OK;
  };
  for(int k = 0; k < s->nblk; k++) {
    const int owner = k % P, sl = k & 1;
    const int k0 = k * DB, r0 = k0 + DB < N ? k0 + DB : N, rows = N - r0;
    const long long ldb = (rows + 1) & ~1;
    double* hdr = s->bbuf[sl] + ld; // the slack in front keeps pan - r0 inside the allocation
    double* pan = hdr + HDR;
    int* info_step = reinterpret_cast<int*>(hdr + DB);
    HB_CUDA(cudaStreamWaitEvent(sp, s->ev_free[sl], 0)); // the update of step k-2 (this buffer, and block k's last update) is done
    HB_CHECK(mark(k, PH_PANEL, 0, sp));
    if(owner == rank) {
      double* Ak = A + (ptrdiff_t)((k / P) * DB - k0) * ld; // LC(Ak, ld, i, j) = element (i, j) for the columns of block k
      HB_CUDA(cudaMemsetAsync(info_step, 0, sizeof(double), sp));
      HB_CHECK(hb_big_panel(N, Ak, ld, k0, ldl, s->inv16, hdr, ldl ? pan - r0 : nullptr, ldb, info_step, sp));
      if(!ldl && rows > 0)
        HB_CUDA(cudaMemcpy2DAsync(pan, sizeof(double) * ldb, Ak + (size_t)k0 * ld + r0, sizeof(double) * ld, sizeof(double) * rows, DB,
                                  cudaMemcpyDeviceToDevice, sp));
    }
    HB_CHECK(mark(k, PH_PANEL, 1, sp));
    HB_CHECK(mark(k, PH_BCAST, 0, sp));
    HB_CHECK(hb_broadcast(c, hdr, HDR + DB * ldb, owner, sp));
    k_dist_recv<<<ldl ? hb_grid(c, DB * ldb) : 1, 256, 0, sp>>>(hdr, pan, ldb, rows, ldl ? 1 : 0, ldl ? s->Lbuf[sl].get() : nullptr, s->info);
    HB_LAUNCHED();
    HB_CHECK(mark(k, PH_BCAST, 1, sp));
    HB_CUDA(cudaEventRecord(s->ev_bc[sl], sp));
    if(rows == 0) continue;
    const double* Pop = pan - r0;                     // P[p * ldb + i], absolute row i
    const double* Qop = ldl ? s->Lbuf[sl].get() : pan; // Q[p * ldb + j - r0]
    const bool ahead = k + 1 < s->nblk && (k + 1) % P == rank;
    if(ahead) {
      HB_CUDA(cudaStreamWaitEvent(sp, s->ev_free[sl ^ 1], 0)); // block k+1 has received the panels up to k-1
      HB_CHECK(hb_big_update_cyclic(N, Pop, ldb, Qop, ldb, r0, A, ld, P, rank, (k + 1) / P, 1, sp));
    }
    const int first = ahead ? k + 2 : k + 1;         // first global block the update stream takes
    const int qa = first <= rank ? 0 : (first - rank + P - 1) / P;
    HB_CUDA(cudaStreamWaitEvent(su, s->ev_bc[sl], 0));
    HB_CHECK(mark(k, PH_UPDATE, 0, su));
    HB_CHECK(hb_big_update_cyclic(N, Pop, ldb, Qop, ldb, r0, A, ld, P, rank, qa, s->nloc - qa, su));
    HB_CHECK(mark(k, PH_UPDATE, 1, su));
    HB_CUDA(cudaEventRecord(s->ev_free[sl], su));
  }
  HB_CUDA(cudaEventRecord(s->ev_join, sp));
  HB_CUDA(cudaStreamWaitEvent(su, s->ev_join, 0));
  HB_CHECK(hb_dist_inertia(A, ld, N, P, rank, s->nloc, s->red, su));
  HB_CHECK(hb_allreduce_op(c, s->red, 3, HB_SUM));
  HB_CUDA(cudaMemcpyAsync(s->red_host, s->red, sizeof(double) * 3, cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaMemcpyAsync(s->info_host, s->info, sizeof(int), cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaStreamSynchronize(su));
  if(s->profile) {
    for(int k = 0; k < s->nblk; k++)
      for(int ph = 0; ph < PH_COUNT; ph++) {
        if(ph == PH_UPDATE && k + 1 == s->nblk) continue; // the last block has no trailing update
        float ms = 0.f;
        HB_CUDA(cudaEventElapsedTime(&ms, s->ev_prof[((size_t)k * PH_COUNT + ph) * 2], s->ev_prof[((size_t)k * PH_COUNT + ph) * 2 + 1]));
        s->phase_ms[ph] += ms;
      }
  }
  s->n_neg = (int)s->red_host[0]; s->n_null = (int)s->red_host[1]; s->n_pos = (int)s->red_host[2];
  if(s->info_host[0] != 0) return -1; // zero pivot / not SPD, as hb_symdense_matrix_changed
  s->factored = true;
  if(s->n_null > 0) return -1;
  return s->n_neg;
}

extern "C" int hb_symdense_dist_inertia(hb_symdense_dist* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  if(n_neg) *n_neg = s->n_neg;
  if(n_null) *n_null = s->n_null;
  if(n_pos) *n_pos = s->n_pos;
  return HB_OK;
}

// the forward and backward sweeps of the factor on the replicated row-major N x nrhs vectors xw, in place
static int dist_sweeps(hb_symdense_dist* s, double* xw, int nrhs)
{
  hb_ctx* c = s->ctx;
  const int N = s->N, P = s->P, rank = s->rank;
  const bool ldl = s->mode != HB_FACT_CHOLESKY;
  const long long ld = s->ld;
  cudaStream_t st = c->stream;
  for(int k = 0; k < s->nblk; k++) {
    const int owner = k % P, k0 = k * DB;
    if(owner == rank) HB_CHECK(hb_dist_fwd_block(s->A.get() + (ptrdiff_t)((k / P) * DB - k0) * ld, ld, N, k0, ldl, xw, nrhs, s->ybuf, st));
    HB_CHECK(hb_broadcast(c, xw + (size_t)k0 * nrhs, (long long)(N - k0) * nrhs, owner, st));
  }
  for(int k = s->nblk - 1; k >= 0; k--) {
    const int owner = k % P, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
    if(owner == rank) HB_CHECK(hb_dist_bwd_block(s->A.get() + (ptrdiff_t)((k / P) * DB - k0) * ld, ld, N, k0, ldl, xw, nrhs, s->tdot, st));
    HB_CHECK(hb_broadcast(c, xw + (size_t)k0 * nrhs, (long long)nb * nrhs, owner, st));
  }
  return HB_OK;
}

// RBT solve on the row-major xw (b in, x out): hb_rbt_solve with the sweeps above, and residual rows formed by the owner of each block
// row and broadcast, so that the stopping rule reads only replicated values and every rank makes the same decisions.
static int rbt_solve(hb_symdense_dist* s, double* xw, int nrhs, hb_rbt_trace* trace)
{
  hb_ctx* c = s->ctx;
  const int N = s->N, P = s->P, rank = s->rank, nrows = s->nloc * DB;
  auto sweeps = [&](double* v) { return dist_sweeps(s, v, nrhs); };
  auto residual = [&](const double* x, const double* b, double* r) -> int {
    HB_CHECK(hb_rbt_rows(c, N, P, rank, nrows, s->Ak, s->ld, nrhs, x, b, r));
    for(int k = 0; k < s->nblk; k++) {
      const int k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
      HB_CHECK(hb_broadcast(c, r + (size_t)k0 * nrhs, (long long)nb * nrhs, k % P, c->stream));
    }
    return HB_OK;
  };
  return hb_rbt_solve(c, N, nrhs, s->rbt_f, s->rbt_anorm, xw, s->rbt_b, s->rbt_r, s->rbt_nrm_host, sweeps, residual, &s->rbt_corr, &s->rbt_berr,
                      trace);
}

static int dist_solve(hb_symdense_dist* s, double* x, int nrhs, hb_rbt_trace* trace)
{
  hb_ctx* c = s->ctx;
  const int N = s->N;
  const bool rbt = s->mode == HB_FACT_RBT_NOPIV;
  HB_CUDA(cudaSetDevice(c->device));
  auto reserve = [&]() -> int {
    HB_CHECK(s->xw.reserve(c, (size_t)N * nrhs, "solve rows"));
    HB_CHECK(s->ybuf.reserve(c, (size_t)DB * nrhs, "solve block"));
    HB_CHECK(s->tdot.reserve(c, (size_t)DB * nrhs, "solve block products"));
    if(rbt) {
      HB_CHECK(s->rbt_b.reserve(c, (size_t)N * nrhs, "transformed rhs"));
      HB_CHECK(s->rbt_r.reserve(c, (size_t)N * nrhs + 3 * nrhs, "residual and norms"));
      HB_CHECK(s->rbt_nrm_host.reserve(c, 3 * (size_t)nrhs, "norms"));
    }
    return HB_OK;
  };
  HB_CHECK(agree(c, reserve()));
  double* xw = s->xw;
  HB_CHECK(hb_rbt_to_rows(c, N, nrhs, x, xw, false));
  int ok = 1;
  if(rbt) {
    ok = rbt_solve(s, xw, nrhs, trace);
    if(ok < 0) return ok;
  } else {
    HB_CHECK(dist_sweeps(s, xw, nrhs));
  }
  HB_CHECK(hb_rbt_to_rows(c, N, nrhs, x, xw, true));
  return ok;
}

extern "C" int hb_symdense_dist_solve(hb_symdense_dist* s, double* x, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_dist_solve: bad arguments");
  if(s->N == 0 || nrhs == 0) return 1;
  HB_REQUIRE(x, "hb_symdense_dist_solve: null rhs");
  if(!s->factored) return hb_fail(HB_ERR_STATE, "hb_symdense_dist_solve: no valid factorization (call hb_symdense_dist_matrix_changed)%s", "");
  return dist_solve(s, x, nrhs, nullptr);
}

// diagnostics (tests): hb_symdense_dist_solve after HB_FACT_RBT_NOPIV, traced (collective)
extern "C" int hb_debug_symdense_dist_rbt_solve(hb_symdense_dist* s, double* x, int nrhs, int* ret_host, int* passes_host, double* anorm_host,
                                                double* norms_host, double* xp_host, double* bp_host)
{
  HB_REQUIRE(s && x && nrhs > 0 && s->N > 0, "hb_debug_symdense_dist_rbt_solve: bad arguments");
  if(!s->factored || s->mode != HB_FACT_RBT_NOPIV)
    return hb_fail(HB_ERR_STATE, "hb_debug_symdense_dist_rbt_solve: no valid RBT factorization%s", "");
  hb_rbt_trace t;
  const int ok = dist_solve(s, x, nrhs, &t);
  if(ok < 0) return ok;
  if(ret_host) *ret_host = ok;
  hb_rbt_trace_out(t, passes_host, anorm_host, norms_host, xp_host, bp_host);
  return HB_OK;
}
