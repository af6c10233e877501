// hiopKKTLinSysCompressedMDSXYcYd on device (mixed dense-sparse Newton KKT): dense (n_d + m) x (n_d + m) system assembly
// including the sparse Schur terms -J_s (H_s + D_xs + delta_wx)^{-1} J_s^T, Haynsworth inertia counts of the eliminated
// diagonal block, and the compressed solve around the dense factorization (hb_symdense).
// Reference: src/Optimization/hiopKKTLinSysMDS.cpp:78-110 (factorizeWithCurvCheck), :172-305 (build_kkt_matrix),
// :307-403 (solveCompressed); matrix kernels src/LinAlg/hiopMatrixDenseRowMajor.cpp:719-829 and
// src/LinAlg/hiopMatrixSparseTriplet.cpp:390-525. The sparse block stays on ONE GPU (north star).
#include "hb_common.cuh"

struct hb_mds
{
  hb_ctx* ctx = nullptr;
  int nxs = 0, nxd = 0, neq = 0, nineq = 0, nnz_c = 0, nnz_d = 0;
  // stacked sparse Jacobian Js = [Jcs; Jds] ((neq+nineq) x nxs): CSR (values in triplet order) + CSC (gather map)
  hb_dev<int> csr_ptr, csr_col;
  hb_dev<int> csc_ptr, csc_row, csc_src;
  hb_dev<double> vals; // nnz_c + nnz_d
  hb_dev<double> Dx, Hxs, Dd_inv, rhs, rxs;
  hb_dev<int> counts;          // device: [neg, zero]
  hb_pinned<int> counts_host;
  bool have_structure = false, have_update = false, built = false;
};

namespace {

constexpr int T = 256;

__global__ void __launch_bounds__(T)
k_mds_update(long long n, const double* __restrict__ zl, const double* __restrict__ sxl, const double* __restrict__ zu,
             const double* __restrict__ sxu, const double* __restrict__ ixl, const double* __restrict__ ixu, double* __restrict__ Dx)
{
  const long long stride = (long long)gridDim.x * T;
  for(long long i = (long long)blockIdx.x * T + threadIdx.x; i < n; i += stride) {
    double d = 0.0;
    if(ixl[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(zl[i], sxl[i]));
    if(ixu[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(zu[i], sxu[i]));
    Dx[i] = d;
  }
}

// Hxs = Dx[0:nxs] + delta_wx[0:nxs] + diag(H_s)   (hiopKKTLinSysMDS.cpp:223-231);  counts for Haynsworth (:90-91)
__global__ void k_mds_hxs(int nxs, const double* __restrict__ Dx, const double* __restrict__ dwx, const double* __restrict__ Hs,
                          double* __restrict__ Hxs, int* __restrict__ counts)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < nxs; i += gridDim.x * blockDim.x) {
    const double v = __dadd_rn(__dadd_rn(Dx[i], dwx[i]), Hs[i]);
    Hxs[i] = v;
    if(v < -1e-14) atomicAdd(&counts[0], 1);
    if(fabs(v) < 1e-14) atomicAdd(&counts[1], 1);
  }
}
// Dd_inv = 1/(delta_wd + vl/sdl|idl + vu/sdu|idu)     (:280-286)
__global__ void k_mds_ddinv(int mi, const double* __restrict__ dwd, const double* __restrict__ vl, const double* __restrict__ sdl,
                            const double* __restrict__ vu, const double* __restrict__ sdu, const double* __restrict__ idl,
                            const double* __restrict__ idu, double* __restrict__ Dd_inv)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < mi; i += gridDim.x * blockDim.x) {
    double d = dwd[i];
    if(idl[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vl[i], sdl[i]));
    if(idu[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vu[i], sdu[i]));
    Dd_inv[i] = __ddiv_rn(1.0, d);
  }
}

// One thread per upper-triangle entry (r <= c) of Msys (N x N row-major). Each entry is produced with the reference's
// order of additions (Msys starts from zero there, :196) so the assembled matrix is bit-identical:
//   (1,1) r,c < nxd        : 0 + Hd[r][c]  (+ Dx[nxs+r] + delta_wx[nxs+r] on the diagonal)                 :204,213,215
//   (1,2),(1,3)            : 0 + Jcd[c-nxd][r]   /  0 + Jdd[c-nxd-neq][r]                                    :205-206
//   (2,2),(2,3),(3,3)      : 0 + (-1)*sum_k Js[i,k]/Hxs[k]*Js[j,k]  (merge-join of two sorted sparse rows)    :239,268,276
//                            then  - delta_cc  |  - Dd_inv - delta_cd  on the diagonal                         :245,289-290
// The explicit 0 + is not a no-op: it turns -0.0 into +0.0, as the reference's `W += alpha*x` does. Without it a pair of sparse
// rows that shares no column (acc = 0, -1 * acc = -0.0) and every -0.0 entry of Hd / Jcd / Jdd would keep the wrong sign bit.
struct MdsBuildArgs
{
  int nxs, nxd, neq, nineq;
  const double *Hd, *Jcd, *Jdd, *Dx, *dwx;
  const int *ptr, *col;
  const double *vals, *Hxs, *dcc, *Dd_inv, *dcd;
};

__device__ __forceinline__ double mds_entry(const MdsBuildArgs& a, int r, int c)
{
  const int nxd = a.nxd, neq = a.neq;
  double v;
  if(r < nxd) {
    if(c < nxd) {
      v = __dadd_rn(0.0, a.Hd[(size_t)r * nxd + c]);
      if(r == c) {
        v = __dadd_rn(v, a.Dx[a.nxs + r]);
        v = __dadd_rn(v, a.dwx[a.nxs + r]);
      }
    } else if(c < nxd + neq) {
      v = __dadd_rn(0.0, a.Jcd[(size_t)(c - nxd) * nxd + r]);
    } else {
      v = __dadd_rn(0.0, a.Jdd[(size_t)(c - nxd - neq) * nxd + r]);
    }
  } else {
    const int i = r - nxd, j = c - nxd;
    int ki = a.ptr[i], kj = a.ptr[j];
    const int ei = a.ptr[i + 1], ej = a.ptr[j + 1];
    double acc = 0.0;
    while(ki < ei && kj < ej) {
      const int ci = a.col[ki], cj = a.col[kj];
      if(ci == cj) {
        acc = __dadd_rn(acc, __dmul_rn(__ddiv_rn(a.vals[ki], a.Hxs[ci]), a.vals[kj]));
        ki++; kj++;
      } else if(ci < cj) ki++;
      else kj++;
    }
    v = __dadd_rn(0.0, __dmul_rn(-1.0, acc));
    if(i == j) {
      if(i < neq) v = __dsub_rn(v, a.dcc[i]);
      else {
        v = __dsub_rn(v, a.Dd_inv[i - neq]);
        v = __dsub_rn(v, a.dcd[i - neq]);
      }
    }
  }
  return v;
}

// The upper-triangle entries of the first `rows` rows one rank owns in hb_symdense_dist's block-cyclic layout: local row lr holds
// global row (lr / 128 * P + rank) * 128 + lr % 128, ld doubles per row. P = 1, rank = 0, ld = rows = N is the N x N matrix.
// `rows` must not reach past global row N - 1.
__global__ void __launch_bounds__(T) k_mds_build(const MdsBuildArgs a, int P, int rank, int rows, double* __restrict__ M, long long ld)
{
  const int N = a.nxd + a.neq + a.nineq;
  const long long total = (long long)rows * N;
  for(long long e = (long long)blockIdx.x * T + threadIdx.x; e < total; e += (long long)gridDim.x * T) {
    const int lr = (int)(e / N), c = (int)(e % N);
    const int r = (lr / 128 * P + rank) * 128 + lr % 128;
    if(c < r) continue;
    M[(size_t)lr * ld + c] = mds_entry(a, r, c);
  }
}

// rxs = rx[0:nxs]/Hxs
__global__ void k_mds_rxs(int nxs, const double* __restrict__ rx, const double* __restrict__ Hxs, double* __restrict__ rxs)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < nxs; i += gridDim.x * blockDim.x) rxs[i] = __ddiv_rn(rx[i], Hxs[i]);
}
// rhs = [ rx[nxs:], ryc - Jcs*rxs, ryd - Jds*rxs ]   (:337-357)
__global__ void k_mds_pack_rhs(int nxs, int nxd, int neq, int nineq, const double* __restrict__ rx, const double* __restrict__ ryc,
                               const double* __restrict__ ryd, const int* __restrict__ ptr, const int* __restrict__ col,
                               const double* __restrict__ vals, const double* __restrict__ rxs, double* __restrict__ rhs)
{
  const int N = nxd + neq + nineq;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < N; e += gridDim.x * blockDim.x) {
    if(e < nxd) {
      rhs[e] = rx[nxs + e];
    } else {
      const int i = e - nxd;
      double y = i < neq ? ryc[i] : ryd[i - neq];
      for(int k = ptr[i]; k < ptr[i + 1]; k++) y = __dadd_rn(y, __dmul_rn(__dmul_rn(-1.0, rxs[col[k]]), vals[k])); // y += alpha*x*v
      rhs[e] = y;
    }
  }
}
// dx[nxs:] = sol[0:nxd]; dyc, dyd = sol[nxd:]; dxs = (rx[0:nxs] - Jcs^T dyc - Jds^T dyd)/Hxs   (:383-395)
__global__ void k_mds_unpack(int nxs, int nxd, int neq, int nineq, const double* __restrict__ sol, const double* __restrict__ rx,
                             const int* __restrict__ cptr, const int* __restrict__ crow, const int* __restrict__ csrc,
                             const double* __restrict__ vals, const double* __restrict__ Hxs, double* __restrict__ dx, double* __restrict__ dyc,
                             double* __restrict__ dyd)
{
  const int total = nxs + nxd + neq + nineq;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    if(e < nxs) {
      double y = rx[e];
      for(int k = cptr[e]; k < cptr[e + 1]; k++) y = __dadd_rn(y, __dmul_rn(__dmul_rn(-1.0, sol[nxd + crow[k]]), vals[csrc[k]]));
      dx[e] = __ddiv_rn(y, Hxs[e]);
    } else if(e < nxs + nxd) {
      dx[e] = sol[e - nxs];
    } else if(e < nxs + nxd + neq) {
      dyc[e - nxs - nxd] = sol[nxd + (e - nxs - nxd)];
    } else {
      dyd[e - nxs - nxd - neq] = sol[nxd + neq + (e - nxs - nxd - neq)];
    }
  }
}

} // namespace

extern "C" int hb_mds_create(hb_ctx* c, int nxs, int nxd, int neq, int nineq, hb_mds** out)
{
  HB_REQUIRE(c && out && nxs >= 0 && nxd >= 0 && neq >= 0 && nineq >= 0, "hb_mds_create: bad arguments");
  HB_CUDA(cudaSetDevice(c->device));
  std::unique_ptr<hb_mds> h(new hb_mds);
  h->ctx = c; h->nxs = nxs; h->nxd = nxd; h->neq = neq; h->nineq = nineq;
  HB_CHECK(h->Dx.reserve(c, (size_t)nxs + nxd, "hb_mds Dx"));
  HB_CHECK(h->Hxs.reserve(c, nxs, "hb_mds Hxs"));
  HB_CHECK(h->rxs.reserve(c, nxs, "hb_mds rxs"));
  HB_CHECK(h->Dd_inv.reserve(c, nineq, "hb_mds Dd_inv"));
  HB_CHECK(h->rhs.reserve(c, (size_t)nxd + neq + nineq, "hb_mds rhs"));
  HB_CHECK(h->counts.reserve(c, 2, "hb_mds inertia counts"));
  HB_CHECK(h->counts_host.reserve(c, 2, "hb_mds inertia counts"));
  *out = h.release();
  return HB_OK;
}

extern "C" int hb_mds_destroy(hb_mds* h)
{
  if(!h) return HB_OK;
  cudaSetDevice(h->ctx->device);
  cudaStreamSynchronize(h->ctx->stream);
  delete h;
  return HB_OK;
}

extern "C" int hb_mds_set_sparsity(hb_mds* h, int nnz_c, const int* iRow_c, const int* jCol_c, int nnz_d, const int* iRow_d, const int* jCol_d)
{
  HB_REQUIRE(h && nnz_c >= 0 && nnz_d >= 0, "hb_mds_set_sparsity: bad arguments");
  HB_REQUIRE((nnz_c == 0 || (iRow_c && jCol_c)) && (nnz_d == 0 || (iRow_d && jCol_d)), "hb_mds_set_sparsity: null index array");
  hb_ctx* c = h->ctx;
  const int m = h->neq + h->nineq, nnz = nnz_c + nnz_d;
  std::vector<int> ptr(m + 1, 0), col(nnz ? nnz : 1), row(nnz ? nnz : 1);
  for(int k = 0; k < nnz; k++) {
    const int r = k < nnz_c ? iRow_c[k] : h->neq + iRow_d[k - nnz_c];
    const int cc = k < nnz_c ? jCol_c[k] : jCol_d[k - nnz_c];
    HB_REQUIRE(r >= 0 && r < m && cc >= 0 && cc < h->nxs, "hb_mds_set_sparsity: index out of range");
    if(k > 0 && k != nnz_c) {
      const bool sorted = (row[k - 1] < r) || (row[k - 1] == r && col[k - 1] < cc);
      HB_REQUIRE(sorted, "hb_mds_set_sparsity: triplets must be sorted by (row, col) like hiopMatrixSparseTriplet requires");
    }
    row[k] = r; col[k] = cc;
    ptr[r + 1]++;
  }
  for(int r = 0; r < m; r++) ptr[r + 1] += ptr[r];
  // CSC with ascending rows inside each column (counting sort keeps the triplet order)
  std::vector<int> cptr(h->nxs + 1, 0), crow(nnz ? nnz : 1), csrc(nnz ? nnz : 1);
  for(int k = 0; k < nnz; k++) cptr[col[k] + 1]++;
  for(int j = 0; j < h->nxs; j++) cptr[j + 1] += cptr[j];
  std::vector<int> fill(cptr.begin(), cptr.end() - 1);
  for(int k = 0; k < nnz; k++) {
    const int p = fill[col[k]]++;
    crow[p] = row[k];
    csrc[p] = k;
  }
  h->have_structure = false;
  HB_CHECK(h->csr_ptr.reserve(c, (size_t)m + 1, "hb_mds CSR pointers")); HB_CHECK(h->csr_col.reserve(c, nnz, "hb_mds CSR columns"));
  HB_CHECK(h->csc_ptr.reserve(c, (size_t)h->nxs + 1, "hb_mds CSC pointers")); HB_CHECK(h->csc_row.reserve(c, nnz, "hb_mds CSC rows"));
  HB_CHECK(h->csc_src.reserve(c, nnz, "hb_mds CSC gather map")); HB_CHECK(h->vals.reserve(c, nnz, "hb_mds Jacobian values"));
  HB_CUDA(cudaStreamSynchronize(c->stream)); // the synchronous uploads below must not overwrite arrays a queued kernel still reads
  HB_CUDA(cudaMemcpy(h->csr_ptr, ptr.data(), sizeof(int) * (m + 1), cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(h->csc_ptr, cptr.data(), sizeof(int) * (h->nxs + 1), cudaMemcpyHostToDevice));
  if(nnz) {
    HB_CUDA(cudaMemcpy(h->csr_col, col.data(), sizeof(int) * nnz, cudaMemcpyHostToDevice));
    HB_CUDA(cudaMemcpy(h->csc_row, crow.data(), sizeof(int) * nnz, cudaMemcpyHostToDevice));
    HB_CUDA(cudaMemcpy(h->csc_src, csrc.data(), sizeof(int) * nnz, cudaMemcpyHostToDevice));
  }
  h->nnz_c = nnz_c; h->nnz_d = nnz_d;
  h->have_structure = true;
  h->built = false;
  return HB_OK;
}

extern "C" int hb_mds_update(hb_mds* h, const double* zl, const double* sxl, const double* zu, const double* sxu, const double* ixl,
                             const double* ixu)
{
  HB_REQUIRE(h, "null handle");
  const long long n = (long long)h->nxs + h->nxd;
  HB_REQUIRE(n == 0 || (zl && sxl && zu && sxu && ixl && ixu), "hb_mds_update: null argument");
  hb_ctx* c = h->ctx;
  if(n > 0) {
    k_mds_update<<<hb_grid(c, n, T), T, 0, c->stream>>>(n, zl, sxl, zu, sxu, ixl, ixu, h->Dx);
    HB_LAUNCHED();
  }
  h->have_update = true;
  h->built = false;
  return HB_OK;
}

namespace {
// everything of build_kkt_matrix before the entries: the sparse values, Hxs (+ its Haynsworth counts), Dd_inv; the arguments of the entries
int mds_prepare(hb_mds* h, const double* Hd, const double* Hs_diag, const double* Jcd, const double* Jdd, const double* Jcs_vals, const double* Jds_vals,
                const double* vl, const double* sdl, const double* vu, const double* sdu, const double* idl, const double* idu, const double* delta_wx,
                const double* delta_wd, const double* delta_cc, const double* delta_cd, MdsBuildArgs* args)
{
  HB_REQUIRE(h->have_structure && h->have_update, "hb_mds_build_kkt_matrix: call hb_mds_set_sparsity and hb_mds_update first");
  HB_REQUIRE((h->nxd == 0 || Hd) && (h->nxs == 0 || Hs_diag) && (h->nxs + h->nxd == 0 || delta_wx), "hb_mds_build_kkt_matrix: null Hessian block");
  HB_REQUIRE(h->nineq == 0 || (vl && sdl && vu && sdu && idl && idu && delta_wd && delta_cd), "hb_mds_build_kkt_matrix: null d-side block");
  HB_REQUIRE(h->neq == 0 || delta_cc, "hb_mds_build_kkt_matrix: null delta_cc");
  hb_ctx* c = h->ctx;
  if(h->nnz_c) HB_CUDA(cudaMemcpyAsync(h->vals, Jcs_vals, sizeof(double) * h->nnz_c, cudaMemcpyDeviceToDevice, c->stream));
  if(h->nnz_d) HB_CUDA(cudaMemcpyAsync(h->vals + h->nnz_c, Jds_vals, sizeof(double) * h->nnz_d, cudaMemcpyDeviceToDevice, c->stream));
  HB_CUDA(cudaMemsetAsync(h->counts, 0, sizeof(int) * 2, c->stream));
  if(h->nxs) {
    k_mds_hxs<<<hb_grid(c, h->nxs, T), T, 0, c->stream>>>(h->nxs, h->Dx, delta_wx, Hs_diag, h->Hxs, h->counts);
    HB_LAUNCHED();
  }
  if(h->nineq) {
    k_mds_ddinv<<<hb_grid(c, h->nineq, T), T, 0, c->stream>>>(h->nineq, delta_wd, vl, sdl, vu, sdu, idl, idu, h->Dd_inv);
    HB_LAUNCHED();
  }
  *args = MdsBuildArgs{h->nxs, h->nxd, h->neq, h->nineq, Hd, Jcd, Jdd, h->Dx, delta_wx, h->csr_ptr, h->csr_col, h->vals, h->Hxs, delta_cc, h->Dd_inv,
                       delta_cd};
  return HB_OK;
}
} // namespace

extern "C" int hb_mds_build_kkt_matrix(hb_mds* h, const double* Hd, const double* Hs_diag, const double* Jcd, const double* Jdd,
                                       const double* Jcs_vals, const double* Jds_vals, const double* vl, const double* sdl, const double* vu,
                                       const double* sdu, const double* idl, const double* idu, const double* delta_wx, const double* delta_wd,
                                       const double* delta_cc, const double* delta_cd, double* Msys)
{
  HB_REQUIRE(h && Msys, "hb_mds_build_kkt_matrix: null argument");
  MdsBuildArgs a;
  HB_CHECK(mds_prepare(h, Hd, Hs_diag, Jcd, Jdd, Jcs_vals, Jds_vals, vl, sdl, vu, sdu, idl, idu, delta_wx, delta_wd, delta_cc, delta_cd, &a));
  hb_ctx* c = h->ctx;
  const int N = h->nxd + h->neq + h->nineq;
  if(N > 0) {
    k_mds_build<<<hb_grid(c, (long long)N * N, T), T, 0, c->stream>>>(a, 1, 0, N, Msys, N);
    HB_LAUNCHED();
  }
  h->built = true;
  return HB_OK;
}

extern "C" int hb_mds_build_kkt_matrix_dist(hb_mds* h, const double* Hd, const double* Hs_diag, const double* Jcd, const double* Jdd,
                                            const double* Jcs_vals, const double* Jds_vals, const double* vl, const double* sdl, const double* vu,
                                            const double* sdu, const double* idl, const double* idu, const double* delta_wx, const double* delta_wd,
                                            const double* delta_cc, const double* delta_cd, hb_symdense_dist* s)
{
  HB_REQUIRE(h && s, "hb_mds_build_kkt_matrix_dist: null argument");
  const int N = h->nxd + h->neq + h->nineq;
  double* M = nullptr;
  long long ld = 0;
  int nloc = 0;
  HB_CHECK(hb_symdense_dist_local(s, &M, &ld, &nloc));
  HB_REQUIRE(hb_symdense_dist_order(s) == N, "hb_mds_build_kkt_matrix_dist: the handle's order is not nxd + neq + nineq");
  MdsBuildArgs a;
  HB_CHECK(mds_prepare(h, Hd, Hs_diag, Jcd, Jdd, Jcs_vals, Jds_vals, vl, sdl, vu, sdu, idl, idu, delta_wx, delta_wd, delta_cc, delta_cd, &a));
  hb_ctx* c = h->ctx;
  if(nloc > 0) {
    // every owned block has 128 rows but the matrix's last one
    const int last = ((nloc - 1) * c->nranks + c->rank) * 128, rows = (nloc - 1) * 128 + std::min(128, N - last);
    k_mds_build<<<hb_grid(c, (long long)rows * N, T), T, 0, c->stream>>>(a, c->nranks, c->rank, rows, M, ld);
    HB_LAUNCHED();
  }
  h->built = true;
  return HB_OK;
}

extern "C" int hb_mds_hxs_inertia(hb_mds* h, int* n_neg, int* n_zero)
{
  HB_REQUIRE(h && h->built, "hb_mds_hxs_inertia: build the KKT matrix first");
  hb_ctx* c = h->ctx;
  HB_CUDA(cudaMemcpyAsync(h->counts_host, h->counts, sizeof(int) * 2, cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  if(n_neg) *n_neg = h->counts_host[0];
  if(n_zero) *n_zero = h->counts_host[1];
  return HB_OK;
}

extern "C" const double* hb_mds_Dx(hb_mds* h) { return h ? h->Dx.get() : nullptr; }
extern "C" const double* hb_mds_Hxs(hb_mds* h) { return h ? h->Hxs.get() : nullptr; }
extern "C" const double* hb_mds_Dd_inv(hb_mds* h) { return h ? h->Dd_inv.get() : nullptr; }

namespace {
// solveCompressed around a dense solve of the packed rhs (in place, h->rhs): pack, solve, unpack
template <typename Solve>
int mds_solve(hb_mds* h, const double* rx, const double* ryc, const double* ryd, double* dx, double* dyc, double* dyd, Solve&& solve)
{
  HB_REQUIRE(h->built, "hb_mds_solve_compressed: build + factorize the KKT matrix first");
  hb_ctx* c = h->ctx;
  const int N = h->nxd + h->neq + h->nineq;
  if(h->nxs) {
    k_mds_rxs<<<hb_grid(c, h->nxs, T), T, 0, c->stream>>>(h->nxs, rx, h->Hxs, h->rxs);
    HB_LAUNCHED();
  }
  if(N) {
    k_mds_pack_rhs<<<hb_grid(c, N, T), T, 0, c->stream>>>(h->nxs, h->nxd, h->neq, h->nineq, rx, ryc, ryd, h->csr_ptr, h->csr_col, h->vals, h->rxs, h->rhs);
    HB_LAUNCHED();
    const int rc = solve(h->rhs.get());
    if(rc != 1) return rc < 0 ? rc : hb_fail(HB_ERR_NUMERIC, "hb_mds_solve_compressed: dense solve failed%s", "");
  }
  const int total = h->nxs + h->nxd + h->neq + h->nineq;
  if(total) {
    k_mds_unpack<<<hb_grid(c, total, T), T, 0, c->stream>>>(h->nxs, h->nxd, h->neq, h->nineq, h->rhs, rx, h->csc_ptr, h->csc_row, h->csc_src, h->vals,
                                                      h->Hxs, dx, dyc, dyd);
    HB_LAUNCHED();
  }
  return HB_OK;
}
} // namespace

extern "C" int hb_mds_solve_compressed(hb_mds* h, hb_symdense* s, const double* rx, const double* ryc, const double* ryd, double* dx, double* dyc,
                                       double* dyd)
{
  HB_REQUIRE(h && s, "hb_mds_solve_compressed: null handle");
  return mds_solve(h, rx, ryc, ryd, dx, dyc, dyd, [&](double* b) { return hb_symdense_solve(s, b, 1); });
}

extern "C" int hb_mds_solve_compressed_dist(hb_mds* h, hb_symdense_dist* s, const double* rx, const double* ryc, const double* ryd, double* dx,
                                            double* dyc, double* dyd)
{
  HB_REQUIRE(h && s, "hb_mds_solve_compressed_dist: null handle");
  HB_REQUIRE(hb_symdense_dist_order(s) == h->nxd + h->neq + h->nineq, "hb_mds_solve_compressed_dist: the handle's order is not nxd + neq + nineq");
  return mds_solve(h, rx, ryc, ryd, dx, dyc, dyd, [&](double* b) { return hb_symdense_dist_solve(s, b, 1); });
}

// =====================================================================================================================
// Dense-Newton KKT classes (SURVEY 8 a16): hiopKKTLinSysDenseXYcYd / hiopKKTLinSysDenseXDYcYd
// src/Optimization/hiopKKTLinSysDense.hpp:85-207, 249-370. Same addition order per entry as the reference's sequence of
// addUpperTriangle / transAdd / addSubDiagonal calls -> bit-identical upper triangle; the lower triangle is zero like after
// the reference's Msys.setToZero(). Copied entries of H, Jc and Jd start from 0 + like the reference's `+=` (-0.0 -> +0.0).
// =====================================================================================================================
namespace {

// Dd = vl/sdl|idl + vu/sdu|idu (hiopKKTLinSys.cpp:799-803);  form 0 stores 1/(delta_wd + Dd) instead (hiopKKTLinSysDense.hpp:142-149)
__global__ void k_dense_dd(int nineq, int form, const double* __restrict__ dwd, const double* __restrict__ vl, const double* __restrict__ sdl,
                           const double* __restrict__ vu, const double* __restrict__ sdu, const double* __restrict__ idl, const double* __restrict__ idu,
                           double* __restrict__ out)
{
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < nineq; i += gridDim.x * blockDim.x) {
    double d = form == 0 ? dwd[i] : 0.0;
    if(idl[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vl[i], sdl[i]));
    if(idu[i] == 1.0) d = __dadd_rn(d, __ddiv_rn(vu[i], sdu[i]));
    out[i] = form == 0 ? __ddiv_rn(1.0, d) : d;
  }
}

__global__ void __launch_bounds__(T)
k_densekkt_build(int form, int nx, int neq, int nineq, const double* __restrict__ H, const double* __restrict__ Jc, const double* __restrict__ Jd,
                 const double* __restrict__ Dx, const double* __restrict__ dwx, const double* __restrict__ dwd, const double* __restrict__ dcd,
                 const double* __restrict__ Dd, double* __restrict__ M)
{
  const int N = nx + neq + nineq + (form ? nineq : 0);
  const long long total = (long long)N * N;
  const int yc0 = nx + (form ? nineq : 0), yd0 = yc0 + neq;
  for(long long e = (long long)blockIdx.x * T + threadIdx.x; e < total; e += (long long)gridDim.x * T) {
    const int i = (int)(e / N), j = (int)(e % N);
    double v = 0.0;
    if(j >= i) {
      if(i < nx) {
        if(j < nx) {
          v = __dadd_rn(0.0, H[(size_t)i * nx + j]);
          if(i == j) v = __dadd_rn(__dadd_rn(v, Dx[i]), dwx[i]);
        } else if(j >= yc0 && j < yd0) {
          v = __dadd_rn(0.0, Jc[(size_t)(j - yc0) * nx + i]);
        } else if(j >= yd0) {
          v = __dadd_rn(0.0, Jd[(size_t)(j - yd0) * nx + i]);
        }
      } else if(form == 0) {
        if(i == j) {
          if(i >= yd0) v = __dadd_rn(0.0, -Dd[i - yd0]);                                 // addSubDiagonal(-1, nx+neq, Dd_inv)      :151-152
          if(i < nx + nineq) v = __dadd_rn(v, -dcd[i - nx]);               // addSubDiagonal(-1, nx, delta_cd)        :157 (starts at nx)
        }
      } else {
        if(i == j) {
          if(i < yc0) v = __dadd_rn(Dd[i - nx], dwd[i - nx]);              // Dd + delta_wd                            :293-294
          else if(i < yc0 + nineq) v = __dadd_rn(0.0, -dcd[i - yc0]);                     // addSubDiagonal(-1, nx+nineq, delta_cd)  :312
        } else if(i < yc0 && j >= yd0 && j - yd0 == i - nx) {
          v = -1.0;                                                        // the -I block                            :296-305
        }
      }
    }
    M[e] = v;
  }
}

} // namespace

extern "C" int hb_densekkt_build(hb_ctx* c, int form, int nx, int neq, int nineq, const double* H, const double* Jc, const double* Jd,
                                 const double* zl, const double* sxl, const double* zu, const double* sxu, const double* ixl, const double* ixu,
                                 const double* vl, const double* sdl, const double* vu, const double* sdu, const double* idl, const double* idu,
                                 const double* delta_wx, const double* delta_wd, const double* delta_cc, const double* delta_cd, double* Dx,
                                 double* Dd, double* Msys)
{
  (void)delta_cc; // the reference reads it but never adds it in these two classes (hiopKKTLinSysDense.hpp:157, 312 use delta_cd)
  HB_REQUIRE(c && (form == 0 || form == 1) && nx >= 0 && neq >= 0 && nineq >= 0, "hb_densekkt_build: bad arguments");
  HB_REQUIRE(nx == 0 || (H && zl && sxl && zu && sxu && ixl && ixu && delta_wx && Dx), "hb_densekkt_build: null x block");
  HB_REQUIRE(nineq == 0 || (Jd && vl && sdl && vu && sdu && idl && idu && delta_wd && delta_cd && Dd), "hb_densekkt_build: null d block");
  HB_REQUIRE((neq == 0 || Jc) && Msys, "hb_densekkt_build: null argument");
  HB_CUDA(cudaSetDevice(c->device));
  if(nx) {
    k_mds_update<<<hb_grid(c, nx, T), T, 0, c->stream>>>(nx, zl, sxl, zu, sxu, ixl, ixu, Dx);
    HB_LAUNCHED();
  }
  if(nineq) {
    k_dense_dd<<<hb_grid(c, nineq, T), T, 0, c->stream>>>(nineq, form, delta_wd, vl, sdl, vu, sdu, idl, idu, Dd);
    HB_LAUNCHED();
  }
  const long long N = nx + neq + nineq + (form ? nineq : 0);
  if(N) {
    k_densekkt_build<<<hb_grid(c, N * N, T), T, 0, c->stream>>>(form, nx, neq, nineq, H, Jc, Jd, Dx, delta_wx, delta_wd, delta_cd, Dd, Msys);
    HB_LAUNCHED();
  }
  return HB_OK;
}

extern "C" int hb_densekkt_solve_compressed(hb_ctx* c, hb_symdense* s, int form, int nx, int neq, int nineq, const double* rx, const double* rd,
                                            const double* ryc, const double* ryd, double* dx, double* dd, double* dyc, double* dyd, double* work)
{
  HB_REQUIRE(c && s && work && (form == 0 || form == 1), "hb_densekkt_solve_compressed: bad arguments");
  HB_REQUIRE(form == 0 || nineq == 0 || (rd && dd), "hb_densekkt_solve_compressed: XDYcYd needs rd / dd");
  // rhs = [rx; (rd); ryc; ryd] -> solve in place -> split                                  hiopKKTLinSysDense.hpp:174-207, 332-370
  const size_t B = sizeof(double);
  const int o_d = nx, o_yc = nx + (form ? nineq : 0), o_yd = o_yc + neq;
  auto cp = [&](double* dst, const double* src, int n) -> int {
    if(n) HB_CUDA(cudaMemcpyAsync(dst, src, B * n, cudaMemcpyDeviceToDevice, c->stream));
    return HB_OK;
  };
  HB_CHECK(cp(work, rx, nx));
  if(form) HB_CHECK(cp(work + o_d, rd, nineq));
  HB_CHECK(cp(work + o_yc, ryc, neq));
  HB_CHECK(cp(work + o_yd, ryd, nineq));
  const int rc = hb_symdense_solve(s, work, 1);
  if(rc != 1) return rc < 0 ? rc : hb_fail(HB_ERR_NUMERIC, "hb_densekkt_solve_compressed: dense solve failed%s", "");
  HB_CHECK(cp(dx, work, nx));
  if(form) HB_CHECK(cp(dd, work + o_d, nineq));
  HB_CHECK(cp(dyc, work + o_yc, neq));
  HB_CHECK(cp(dyd, work + o_yd, nineq));
  return HB_OK;
}
