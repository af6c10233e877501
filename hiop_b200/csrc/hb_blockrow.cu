// Block rows (hb_dense.cuh): the factorization step loop and the solve sweeps that hb_symdense_dist (block rows of other ranks, NCCL
// broadcasts) and hb_symdense_host (block rows in page-locked host memory, a copy stream) share, with their per-block kernels. Each handle
// keeps only how a panel travels and its own bookkeeping.
#include <algorithm>
#include "hb_common.cuh"
#include "hb_dense.cuh"

namespace {

constexpr int DB = HB_ROWS_DB;
constexpr int SOLVE_RHS = 4; // right-hand sides per CTA of the diagonal-block solves
constexpr int DLD = DB + 1;  // shared-memory stride of the diagonal block
constexpr size_t DIAG_SMEM = sizeof(double) * ((size_t)DB * DLD + SOLVE_RHS * DB);

// fold the breakdown of a step into the factorization's info word (the first one stays, as in hb_big_factor); a received LDL^T panel:
// form L = W * (1/d) with the operation k_trsm_panel uses, so that L is bit-identical to the one its owner holds
__global__ void k_rows_recv(const double* __restrict__ hdr, const double* __restrict__ W, long long ldb, int rows, int ldl, double* __restrict__ L,
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

// {neg, null, pos} of the owned diagonal entries (hb_rows_inertia): doubles for the block-row handles, ints for hb_symdense's info words
template <typename T>
__global__ void __launch_bounds__(1024) k_rows_inertia(const double* __restrict__ A, long long ld, int N, int P, int rank, int nloc, T* __restrict__ out3)
{
  __shared__ int cnt[3];
  if(threadIdx.x < 3) cnt[threadIdx.x] = 0;
  __syncthreads();
  int neg = 0, nul = 0, pos = 0;
  for(int e = threadIdx.x; e < nloc * DB; e += blockDim.x) {
    const int q = e / DB, t = e % DB, k0 = (q * P + rank) * DB;
    if(k0 + t >= N) continue;
    hb_inertia_count(A[(size_t)e * ld + k0 + t], neg, nul, pos);
  }
  atomicAdd(&cnt[0], neg); atomicAdd(&cnt[1], nul); atomicAdd(&cnt[2], pos);
  __syncthreads();
  if(threadIdx.x < 3) out3[threadIdx.x] = (T)cnt[threadIdx.x];
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
__global__ void __launch_bounds__(DB * SOLVE_RHS) k_rows_fwd_diag(const double* __restrict__ A, long long ld, int k0, int nb, int ldl, double* __restrict__ xw,
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
__global__ void k_rows_fwd_panel(const double* __restrict__ A, long long ld, int N, int k0, double* __restrict__ xw, int nrhs, const double* __restrict__ ybuf)
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
__global__ void __launch_bounds__(256) k_rows_bwd_dots(const double* __restrict__ A, long long ld, int N, int k0, const double* __restrict__ xw, int nrhs,
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
__global__ void __launch_bounds__(DB * SOLVE_RHS) k_rows_bwd_diag(const double* __restrict__ A, long long ld, int k0, int nb, int ldl, double* __restrict__ xw,
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

} // namespace

int hb_rows_init_attrs()
{
  HB_CUDA(cudaFuncSetAttribute(k_rows_fwd_diag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DIAG_SMEM));
  HB_CUDA(cudaFuncSetAttribute(k_rows_bwd_diag, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DIAG_SMEM));
  return HB_OK;
}

int hb_rows::create()
{
  int lo = 0, hi = 0;
  HB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  HB_CHECK(sp.create(cudaStreamNonBlocking, hi));
  for(hb_event* e : {&ev_bc[0], &ev_bc[1], &ev_free[0], &ev_free[1], &ev_ahead, &ev_join}) HB_CHECK(e->create(cudaEventDisableTiming));
  return HB_OK;
}

int hb_rows_factor(hb_ctx* c, hb_rows& r, int N, double* A, long long ld, int P, int rank, int q0, int nsteps, bool ldl, double* inv16, int* info,
                   const std::function<int(int k, bool local, hb_rows_panel& b)>& at,
                   const std::function<int(int k, bool local, const hb_rows_panel& b)>& move, hb_event* prof)
{
  cudaStream_t su = c->stream, sp = r.sp;
  const int qend = nsteps > rank ? (nsteps - rank + P - 1) / P : 0; // local blocks q0 .. qend-1
  auto local = [&](int k) { return k < nsteps && k % P == rank && k / P >= q0; };
  auto mark = [&](int k, int ph, int end, cudaStream_t st) -> int {
    if(prof) HB_CUDA(cudaEventRecord(prof[((size_t)k * HB_ROWS_PH_COUNT + ph) * 2 + end], st));
    return HB_OK;
  };
  for(hb_event& e : r.ev_free) HB_CUDA(cudaEventRecord(e, su));
  for(int k = 0; k < nsteps; k++) {
    const int sl = k & 1, k0 = k * DB, r0 = k0 + DB < N ? k0 + DB : N;
    const bool mine = local(k);
    double* Ak = A + (ptrdiff_t)((k / P) * DB - k0) * ld; // LC(Ak, ld, i, j) = element (i, j) for the columns of block k, when local
    HB_CUDA(cudaStreamWaitEvent(sp, r.ev_free[sl], 0));   // the readers of step k-2's operands are done, and block k has its update
    hb_rows_panel b{};
    HB_CHECK(at(k, mine, b));
    HB_CHECK(mark(k, HB_ROWS_PH_PANEL, 0, sp));
    if(mine) {
      HB_CUDA(cudaMemsetAsync(b.hdr + DB, 0, sizeof(double), sp));
      HB_CHECK(hb_big_panel(N, Ak, ld, k0, ldl, inv16, b.hdr, ldl && b.pan ? b.pan - b.sub : nullptr, b.ldp, reinterpret_cast<int*>(b.hdr + DB), sp));
      if(!ldl && b.pan && r0 < N)
        HB_CUDA(cudaMemcpy2DAsync(b.pan, sizeof(double) * b.ldp, Ak + (size_t)k0 * ld + r0, sizeof(double) * ld, sizeof(double) * (N - r0), DB,
                                  cudaMemcpyDeviceToDevice, sp));
    }
    HB_CHECK(mark(k, HB_ROWS_PH_PANEL, 1, sp));
    HB_CHECK(mark(k, HB_ROWS_PH_MOVE, 0, sp));
    HB_CHECK(move(k, mine, b));
    const bool form = ldl && !mine;
    k_rows_recv<<<form ? hb_grid(c, DB * b.ldp) : 1, 256, 0, sp>>>(b.hdr, b.pan, b.ldp, N - b.sub, form ? 1 : 0, b.L, info);
    HB_LAUNCHED();
    HB_CHECK(mark(k, HB_ROWS_PH_MOVE, 1, sp));
    HB_CUDA(cudaEventRecord(r.ev_bc[sl], sp));
    if(r0 == N) continue;
    // the operands P[p * ldp + i] (absolute row i) and Q[p * ldq + j - qsub]: the received panel (and its L), or W and L of a local one
    const double* Lk = Ak + (size_t)k0 * ld;
    const double* Pp = mine && !ldl ? Lk : b.pan - b.sub;
    const double* Qp = mine ? Lk : ldl ? b.L : b.pan;
    const long long ldp = mine && !ldl ? ld : b.ldp, ldq = mine ? ld : b.ldp;
    const int qsub = mine ? 0 : b.sub;
    const bool ahead = local(k + 1);
    if(ahead) {
      HB_CUDA(cudaStreamWaitEvent(sp, r.ev_free[sl ^ 1], 0)); // block k+1 has received the panels up to k-1
      HB_CHECK(hb_big_update_cyclic(N, Pp, ldp, Qp, ldq, qsub, A, ld, P, rank, (k + 1) / P, 1, sp));
      HB_CUDA(cudaEventRecord(r.ev_ahead, sp));
    }
    const int first = ahead ? k + 2 : k + 1; // first global block the update stream takes
    const int qa = std::max(q0, first <= rank ? 0 : (first - rank + P - 1) / P);
    HB_CUDA(cudaStreamWaitEvent(su, r.ev_bc[sl], 0));
    HB_CHECK(mark(k, HB_ROWS_PH_UPDATE, 0, su));
    HB_CHECK(hb_big_update_cyclic(N, Pp, ldp, Qp, ldq, qsub, A, ld, P, rank, qa, qend - qa, su));
    HB_CHECK(mark(k, HB_ROWS_PH_UPDATE, 1, su));
    if(ahead) HB_CUDA(cudaStreamWaitEvent(su, r.ev_ahead, 0));
    HB_CUDA(cudaEventRecord(r.ev_free[sl], su));
  }
  HB_CUDA(cudaEventRecord(r.ev_join, sp));
  HB_CUDA(cudaStreamWaitEvent(su, r.ev_join, 0));
  return HB_OK;
}

int hb_rows_inertia(const double* A, long long ld, int N, int P, int rank, int nloc, double* out3, cudaStream_t st)
{
  k_rows_inertia<<<1, 1024, 0, st>>>(A, ld, N, P, rank, nloc, out3);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_inertia_diag(hb_ctx* c, int N, const double* F, long long ldf, int* out3_dev)
{
  k_rows_inertia<<<1, 1024, 0, c->stream>>>(F, ldf, N, 1, 0, (N + DB - 1) / DB, out3_dev);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rows_sweeps(int N, long long ld, bool ldl, double* xw, int nrhs, double* ybuf, double* tdot, cudaStream_t st,
                   const std::function<int(int k, const double** Ak)>& rows, const std::function<int(int k, bool forward)>& after)
{
  const int nblk = (N + DB - 1) / DB, ctas = (nrhs + SOLVE_RHS - 1) / SOLVE_RHS;
  for(int fwd = 1; fwd >= 0; fwd--)
    for(int i = 0; i < nblk; i++) {
      const int k = fwd ? i : nblk - 1 - i, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB, below = N - k0 - nb;
      const double* Ak = nullptr;
      HB_CHECK(rows(k, &Ak));
      if(Ak && fwd) {
        k_rows_fwd_diag<<<ctas, DB * SOLVE_RHS, DIAG_SMEM, st>>>(Ak, ld, k0, nb, ldl ? 1 : 0, xw, nrhs, ybuf);
        HB_LAUNCHED();
        if(below > 0) {
          k_rows_fwd_panel<<<(below + 255) / 256, 256, 0, st>>>(Ak, ld, N, k0, xw, nrhs, ybuf);
          HB_LAUNCHED();
        }
      } else if(Ak) {
        if(below > 0) {
          k_rows_bwd_dots<<<nb, 256, 0, st>>>(Ak, ld, N, k0, xw, nrhs, tdot);
          HB_LAUNCHED();
        }
        k_rows_bwd_diag<<<ctas, DB * SOLVE_RHS, DIAG_SMEM, st>>>(Ak, ld, k0, nb, ldl ? 1 : 0, xw, nrhs, below > 0 ? tdot : nullptr);
        HB_LAUNCHED();
      }
      HB_CHECK(after(k, fwd != 0));
    }
  return HB_OK;
}
