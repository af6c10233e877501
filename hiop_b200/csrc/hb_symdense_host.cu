// The dense symmetric system of one GPU with the matrix in page-locked host memory (hb_symdense_host_*, include/hiopb200.h): Cholesky
// LL^T and no-pivot LDL^T of matrices larger than the device memory, streamed through HBM. A block row kept in host memory is to time
// what a block row of another rank is to space in hb_symdense_dist.
//
// Layout. The block rows of hb_blockrow.cu at one rank: block row k is rows k*128 .. min(N, k*128+128)-1 of the caller's N x N row-major
// matrix (upper triangle valid), i.e. block column k of the column-major lower view the kernels use (hb_dense.cuh). A slab is a run of
// H consecutive block rows; H comes from the device budget alone (make_plan). On the device, slab rows keep their full width ld, so the
// kernels address an entry of the slab by its global (row, column) through a shifted base pointer.
//
// Factorization, left-looking over the slabs; slab s holds the block rows b0 .. b1-1 (rows c0 = b0*128 ..). The copy stream brings the
// slab in, one copy per block row from its diagonal column to N - 1 (the strictly lower entries of the diagonal blocks ride along and go
// back unchanged). Then the step loop of hb_blockrow.cu runs steps 0 .. b1-1, the slab's blocks local, ring slot k & 1 the transport:
//   k < b0 : the copy stream, behind the slot's ev_free, brings columns c0 .. N-1 of block row k into the slot (LDL^T: of W = L D,
//            which the slab of block k left in pinned host memory)
//   k >= b0: the panel writes W into the slot (LDL^T), and the copy stream takes block row k, now final, back to the host, and W to
//            pinned host memory when a later slab streams it
// So the factor, the return value and the inertia are bit-identical to hb_symdense_dist at P = 1 for every slab plan. H2D traffic per
// factorization: the matrix once plus, per slab, 128 b0 (N - c0) doubles of panels; D2H: the factor once (LDL^T with several slabs:
// plus the W rows of every block a later slab streams).
//
// Solves: the sweeps of hb_blockrow.cu (hb_rows_sweeps) on row-major groups of at most RHS right-hand sides. With one slab the factor
// stays resident and the sweeps read it there; otherwise every sweep streams block row k (columns k0 .. N-1) through the ring, about
// 8 N^2 bytes per group.
#include "hb_common.cuh"
#include "hb_dense.cuh"

namespace {

constexpr int DB = HB_ROWS_DB, HDR = HB_ROWS_HDR; // one step header per block: its 1/d are read again by every later slab
constexpr int RHS = 16;         // right-hand sides per pass of a solve (the size of the solve scratch)
constexpr size_t ALIGN_D = 32;  // every part of the device allocation starts on a 256-byte boundary
enum { B_PEAK = 0, B_H2D, B_D2H_CHOL, B_D2H_LDL, B_SOLVE_H2D, B_COUNT };

size_t up(size_t d) { return (d + ALIGN_D - 1) / ALIGN_D * ALIGN_D; }

// The device memory of a handle is one allocation: the panel ring (two slots, each 128 rows of W or L and 128 rows of the formed L), the
// per-block 1/d, the 16 x 16 diagonal inverses of k_diag128, the diagonal of the factor (inertia), the solve scratch for RHS
// right-hand sides, the counts and the info word, then the slab. Offsets in doubles.
struct plan_t
{
  int N = 0, nblk = 0, H = 0, nslab = 0;
  long long ld = 8;
  size_t ring = 0, hdr = 0, inv16 = 0, diag = 0, xw = 0, ybuf = 0, tdot = 0, red = 0, info = 0, slab = 0, total = 0;
  long long bytes[B_COUNT] = {0, 0, 0, 0, 0};
};

int make_plan(int N, size_t budget, plan_t& p)
{
  p = plan_t{};
  if(N < 0) return hb_fail(HB_ERR_INVALID, "hb_symdense_host: negative order%s", "");
  p.N = N;
  if(N == 0) return HB_OK;
  p.nblk = (N + DB - 1) / DB;
  p.ld = (N + 7) & ~7LL;
  size_t o = 0;
  auto part = [&](size_t n) { const size_t at = o; o += up(n); return at; };
  p.ring = part((size_t)4 * DB * p.ld);
  p.hdr = part((size_t)p.nblk * HDR);
  p.inv16 = part(8 * 16 * 17);
  p.diag = part((size_t)p.nblk * DB);
  p.xw = part((size_t)N * RHS);
  p.ybuf = part((size_t)DB * RHS);
  p.tdot = part((size_t)DB * RHS);
  p.red = part(4);
  p.info = part(4);
  p.slab = o;
  const size_t fixed = sizeof(double) * o, row = sizeof(double) * p.ld, first = (size_t)(N < DB ? N : DB);
  if(budget < fixed + first * row) {
    snprintf(g_hb_err, sizeof(g_hb_err), "hb_symdense_host: a device budget of %zu bytes is below the minimum %zu for N = %d (one block row, the panel ring "
             "and the scratch)", budget, fixed + first * row, N);
    return HB_ERR_INVALID;
  }
  const size_t fit = (budget - fixed) / row; // rows of the slab
  p.H = fit >= (size_t)N ? p.nblk : (int)(fit / DB);
  p.nslab = (p.nblk + p.H - 1) / p.H;
  const size_t srows = (size_t)p.H * DB < (size_t)N ? (size_t)p.H * DB : (size_t)N;
  p.total = o + srows * p.ld;
  // traffic: the matrix in and the factor out once, block row by block row from its diagonal column
  long long io = 0, panels = 0, wout = 0;
  for(int k = 0; k < p.nblk; k++) {
    const long long k0 = (long long)k * DB, nb = N - k0 < DB ? N - k0 : DB;
    io += nb * (N - k0);
  }
  for(int s = 0; s < p.nslab; s++) {
    const long long b0 = (long long)s * p.H;
    panels += b0 * DB * (N - b0 * DB);
  }
  for(long long k = 0; k < (long long)(p.nslab - 1) * p.H; k++) wout += (long long)DB * (N - (k + 1) * DB);
  p.bytes[B_PEAK] = (long long)(sizeof(double) * p.total);
  p.bytes[B_H2D] = 8 * (io + panels);
  p.bytes[B_D2H_CHOL] = 8 * io;
  p.bytes[B_D2H_LDL] = 8 * (io + wout);
  p.bytes[B_SOLVE_H2D] = p.nslab > 1 ? 16 * io : 0;
  return HB_OK;
}

// page-locked (hb_malloc_host / hb_host_register) host memory: the only kind a copy engine reads and writes asynchronously
bool page_locked(const void* p)
{
  unsigned flags = 0;
  if(cudaHostGetFlags(&flags, const_cast<void*>(p)) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return true;
}

} // namespace

struct hb_symdense_host : hb_rows // the panel stream, the step loop's events, mode, factored and the inertia counts
{
  hb_ctx* ctx = nullptr;
  plan_t p;
  hb_dev<double> mem;          // the plan's device allocation
  hb_pinned<double> Wh;        // LDL^T with several slabs: W = L D of the blocks a later slab streams, block k at woff[k], N - (k+1)*128 per row
  std::vector<size_t> woff;
  hb_pinned<double> host;      // landing slots: inertia counts (3 doubles), info word
  double* M = nullptr;         // the caller's page-locked matrix (borrowed)
  long long ldh = 0;
  hb_stream sc;                // copy stream
  hb_event ev_in[2], ev_read[2], ev_out[2], ev_a, ev_b, ev_panel;
  bool resident = false;
  double* at(size_t off) const { return mem.get() + off; }
  double* slot(int j) const { return mem.get() + p.ring + (size_t)j * 2 * DB * p.ld; } // W or L rows; the formed L follows at + 128 ld
  ~hb_symdense_host()
  {
    if(sc) cudaStreamSynchronize(sc);
    if(sp) cudaStreamSynchronize(sp);
  }
};

extern "C" int hb_symdense_host_plan_view(int N, size_t device_bytes, int* dims, int* slab_first_block_host, long long* bytes_host)
{
  HB_REQUIRE(device_bytes > 0, "hb_symdense_host_plan_view: device_bytes must be given (0 asks the device, which this host-only view does not)");
  plan_t p;
  HB_CHECK(make_plan(N, device_bytes, p));
  if(dims) {
    dims[0] = p.nslab;
    dims[1] = p.nblk;
    dims[2] = p.H;
  }
  if(slab_first_block_host) {
    for(int s = 0; s < p.nslab; s++) slab_first_block_host[s] = s * p.H;
    slab_first_block_host[p.nslab] = p.nblk;
  }
  if(bytes_host)
    for(int b = 0; b < B_COUNT; b++) bytes_host[b] = p.bytes[b];
  return HB_OK;
}

extern "C" int hb_symdense_host_create(hb_ctx* c, int N, size_t device_bytes, hb_symdense_host** out)
{
  HB_REQUIRE(c && out, "hb_symdense_host_create: null argument");
  HB_REQUIRE(N >= 0, "hb_symdense_host_create: negative order");
  HB_CUDA(cudaSetDevice(c->device));
  if(device_bytes == 0) { // what is free, less 5 % (at least 256 MiB) for the context and the caller
    size_t free_b = 0, total_b = 0;
    HB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t margin = free_b / 20 > ((size_t)256 << 20) ? free_b / 20 : ((size_t)256 << 20);
    device_bytes = free_b > margin ? free_b - margin : 1;
  }
  std::unique_ptr<hb_symdense_host> s(new hb_symdense_host);
  s->ctx = c;
  HB_CHECK(make_plan(N, device_bytes, s->p));
  if(N > 0) HB_CHECK(s->mem.reserve(c, s->p.total, "slab, panel ring and scratch"));
  HB_CHECK(s->host.reserve(c, 4, "inertia counts and info word"));
  HB_CHECK(s->create());
  HB_CHECK(s->sc.create(cudaStreamNonBlocking));
  for(int j = 0; j < 2; j++)
    for(hb_event* e : {&s->ev_in[j], &s->ev_read[j], &s->ev_out[j]}) HB_CHECK(e->create(cudaEventDisableTiming));
  for(hb_event* e : {&s->ev_a, &s->ev_b, &s->ev_panel}) HB_CHECK(e->create(cudaEventDisableTiming));
  *out = s.release();
  return HB_OK;
}

extern "C" int hb_symdense_host_destroy(hb_symdense_host* s)
{
  if(!s) return HB_OK;
  cudaSetDevice(s->ctx->device);
  cudaStreamSynchronize(s->ctx->stream);
  delete s;
  return HB_OK;
}

extern "C" int hb_symdense_host_set_matrix(hb_symdense_host* s, double* M_host, long long ld)
{
  HB_REQUIRE(s, "null handle");
  const int N = s->p.N;
  s->factored = s->resident = false;
  s->M = nullptr;
  if(N == 0) return HB_OK;
  HB_REQUIRE(M_host && ld >= N, "hb_symdense_host_set_matrix: null matrix or ld < N");
  HB_REQUIRE(page_locked(M_host) && page_locked(M_host + (size_t)(N - 1) * ld + N - 1),
             "hb_symdense_host_set_matrix: the matrix must be page-locked host memory (hb_malloc_host or hb_host_register)");
  s->M = M_host;
  s->ldh = ld;
  return HB_OK;
}

namespace {

// block rows kb .. ke-1 of the slab starting at block row b0 between the caller's matrix and the device, on the copy stream, each from
// its diagonal column to N - 1
int slab_copy(hb_symdense_host* s, int b0, int kb, int ke, bool in)
{
  const plan_t& p = s->p;
  const int N = p.N;
  const long long ld = p.ld, ldh = s->ldh;
  double* S = s->at(p.slab);
  for(int k = kb; k < ke; k++) {
    const long long k0 = (long long)k * DB, nb = N - k0 < DB ? N - k0 : DB;
    double* d = S + (size_t)(k0 - (long long)b0 * DB) * ld + k0;
    double* h = s->M + (size_t)k0 * ldh + k0;
    if(in) HB_CUDA(cudaMemcpy2DAsync(d, sizeof(double) * ld, h, sizeof(double) * ldh, sizeof(double) * (N - k0), nb, cudaMemcpyHostToDevice, s->sc));
    else HB_CUDA(cudaMemcpy2DAsync(h, sizeof(double) * ldh, d, sizeof(double) * ld, sizeof(double) * (N - k0), nb, cudaMemcpyDeviceToHost, s->sc));
  }
  return HB_OK;
}

// `rows` rows of `width` doubles from the host (pitch hld) into ring slot j (pitch ld) on the copy stream, once `free` (the slot's last
// reader is done) has passed; the stream `use` then waits for the copy
int ring_in(hb_symdense_host* s, int j, const double* src, long long hld, long long width, long long rows, cudaEvent_t free, cudaStream_t use)
{
  cudaStream_t sc = s->sc;
  HB_CUDA(cudaStreamWaitEvent(sc, free, 0));
  HB_CUDA(cudaMemcpy2DAsync(s->slot(j), sizeof(double) * s->p.ld, src, sizeof(double) * hld, sizeof(double) * width, rows, cudaMemcpyHostToDevice, sc));
  HB_CUDA(cudaEventRecord(s->ev_in[j], sc));
  HB_CUDA(cudaStreamWaitEvent(use, s->ev_in[j], 0));
  return HB_OK;
}

// the compute stream's work so far before the copy stream's next copy (from == su), or the copy stream's before the compute stream's
int order(hb_symdense_host* s, bool compute_first)
{
  cudaStream_t su = s->ctx->stream, sc = s->sc;
  hb_event& e = compute_first ? s->ev_a : s->ev_b;
  HB_CUDA(cudaEventRecord(e, compute_first ? su : sc));
  HB_CUDA(cudaStreamWaitEvent(compute_first ? sc : su, e, 0));
  return HB_OK;
}

int factor(hb_symdense_host* s, bool ldl)
{
  hb_ctx* c = s->ctx;
  const plan_t& p = s->p;
  const int N = p.N;
  const long long ld = p.ld;
  cudaStream_t su = c->stream, sc = s->sc, sp = s->sp;
  double* S = s->at(p.slab);
  double* hdr = s->at(p.hdr);
  int* info = reinterpret_cast<int*>(s->at(p.info));
  const int wlast = (p.nslab - 1) * p.H; // the blocks before this one are streamed by a later slab
  HB_CUDA(cudaMemsetAsync(info, 0, sizeof(int), su));
  HB_CHECK(order(s, true)); // the slab and the ring may still be read by an earlier solve
  for(int sl = 0; sl < p.nslab; sl++) {
    const int b0 = sl * p.H, b1 = b0 + p.H < p.nblk ? b0 + p.H : p.nblk, c0 = b0 * DB, c1 = b1 * DB < N ? b1 * DB : N;
    HB_CHECK(slab_copy(s, b0, b0, b1, true));
    HB_CHECK(order(s, false));
    // the transport of step k, ring slot k & 1: a block before the slab arrives from the host (its columns c0 .. N-1; LDL^T: of W);
    // a block of the slab writes W there (LDL^T, when a block follows) and goes back to the host once its panel is done
    auto at = [&](int k, bool local, hb_rows_panel& b) -> int {
      const int r0 = (k + 1) * DB < N ? (k + 1) * DB : N;
      double* R = s->slot(k & 1);
      b = local ? hb_rows_panel{hdr + (size_t)k * HDR, ldl && r0 < N ? R : nullptr, ld, r0, nullptr}
                : hb_rows_panel{hdr + (size_t)k * HDR, R, ld, c0, R + (size_t)DB * ld};
      if(local && b.pan) HB_CUDA(cudaStreamWaitEvent(sp, s->ev_out[k & 1], 0)); // W goes into the slot once its last copy to the host is done
      return HB_OK;
    };
    auto move = [&](int k, bool local, const hb_rows_panel&) -> int {
      const int j = k & 1, r0 = (k + 1) * DB < N ? (k + 1) * DB : N;
      if(!local && ldl) return ring_in(s, j, s->Wh.get() + s->woff[k] + (c0 - r0), N - r0, N - c0, DB, s->ev_free[j], sp);
      if(!local) return ring_in(s, j, s->M + (size_t)k * DB * s->ldh + c0, s->ldh, N - c0, DB, s->ev_free[j], sp);
      // block row k is final: back to the host under the rest of the slab's updates
      HB_CUDA(cudaEventRecord(s->ev_panel, sp));
      HB_CUDA(cudaStreamWaitEvent(sc, s->ev_panel, 0));
      HB_CHECK(slab_copy(s, b0, k, k + 1, false));
      if(ldl && r0 < N && k < wlast) {
        HB_CUDA(cudaMemcpy2DAsync(s->Wh.get() + s->woff[k], sizeof(double) * (N - r0), s->slot(j), sizeof(double) * ld, sizeof(double) * (N - r0), DB,
                                  cudaMemcpyDeviceToHost, sc));
        HB_CUDA(cudaEventRecord(s->ev_out[j], sc));
      }
      return HB_OK;
    };
    HB_CHECK(hb_rows_factor(c, *s, N, S - (ptrdiff_t)c0 * ld, ld, 1, 0, b0, b1, ldl, s->at(p.inv16), info, at, move));
    // the slab's diagonal (inertia); the next slab's copy waits for the compute stream to be done with this one
    HB_CUDA(cudaMemcpy2DAsync(s->at(p.diag) + c0, sizeof(double), S + c0, sizeof(double) * (ld + 1), sizeof(double), c1 - c0, cudaMemcpyDeviceToDevice, su));
    HB_CHECK(order(s, true));
  }
  HB_CHECK(order(s, false));
  HB_CHECK(hb_rows_inertia(s->at(p.diag), 0, N, 1, 0, p.nblk, s->at(p.red), su));
  HB_CUDA(cudaMemcpyAsync(s->host, s->at(p.red), sizeof(double) * 3, cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaMemcpyAsync(s->host.get() + 3, info, sizeof(int), cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaStreamSynchronize(su));
  return HB_OK;
}

} // namespace

extern "C" int hb_symdense_host_matrix_changed(hb_symdense_host* s, int mode)
{
  HB_REQUIRE(s, "null handle");
  if(mode == HB_FACT_BUNCH_KAUFMAN)
    return hb_fail(HB_ERR_INVALID, "hb_symdense_host_matrix_changed: Bunch-Kaufman needs up-to-date columns for its pivot search; use hb_symdense%s", "");
  if(mode == HB_FACT_RBT_NOPIV)
    return hb_fail(HB_ERR_INVALID, "hb_symdense_host_matrix_changed: the random butterfly needs partner rows and both triangles; for the safe mode beyond "
                                   "one GPU use hb_symdense_dist%s", "");
  HB_REQUIRE(mode == HB_FACT_NOPIV || mode == HB_FACT_CHOLESKY, "hb_symdense_host_matrix_changed: bad mode");
  const plan_t& p = s->p;
  const int N = p.N;
  const bool ldl = mode == HB_FACT_NOPIV;
  if(N > 0 && !s->M) return hb_fail(HB_ERR_STATE, "hb_symdense_host_matrix_changed: no matrix (call hb_symdense_host_set_matrix)%s", "");
  s->mode = mode;
  s->factored = s->resident = false;
  if(N == 0) { const double none[3] = {0.0, 0.0, 0.0}; return s->finish(none, 0); }
  HB_CUDA(cudaSetDevice(s->ctx->device));
  if(ldl && p.nslab > 1 && !s->Wh) {
    const int wlast = (p.nslab - 1) * p.H;
    std::vector<size_t> off(wlast);
    size_t tot = 0;
    for(int k = 0; k < wlast; k++) {
      off[k] = tot;
      tot += (size_t)DB * (N - (size_t)(k + 1) * DB);
    }
    HB_CHECK(s->Wh.reserve(s->ctx, tot, "W = L D rows of the streamed block rows"));
    s->woff.swap(off);
  }
  HB_CHECK(factor(s, ldl));
  s->resident = p.nslab == 1;
  return s->finish(s->host, *reinterpret_cast<const int*>(s->host.get() + 3));
}

extern "C" int hb_symdense_host_inertia(hb_symdense_host* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  if(n_neg) *n_neg = s->n_neg;
  if(n_null) *n_null = s->n_null;
  if(n_pos) *n_pos = s->n_pos;
  return HB_OK;
}

extern "C" int hb_symdense_host_solve(hb_symdense_host* s, double* x, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_host_solve: bad arguments");
  const plan_t& p = s->p;
  const int N = p.N;
  if(N == 0 || nrhs == 0) return 1;
  HB_REQUIRE(x, "hb_symdense_host_solve: null rhs");
  if(!s->factored) return hb_fail(HB_ERR_STATE, "hb_symdense_host_solve: no valid factorization (call hb_symdense_host_matrix_changed)%s", "");
  hb_ctx* c = s->ctx;
  HB_CUDA(cudaSetDevice(c->device));
  cudaStream_t su = c->stream;
  const bool ldl = s->mode == HB_FACT_NOPIV;
  const long long ld = p.ld;
  double* xw = s->at(p.xw);
  long long t = 0;
  int j = 0;
  // block row k on the device: the resident factor, or columns k0 .. N-1 of the host's block row streamed into ring slot j, which is
  // free again once the block's step is done
  auto rows = [&](int k, const double** Ak) -> int {
    const long long k0 = (long long)k * DB;
    if(s->resident) {
      *Ak = s->at(p.slab);
      return HB_OK;
    }
    j = (int)(t++ & 1);
    HB_CHECK(ring_in(s, j, s->M + (size_t)k0 * s->ldh + k0, s->ldh, N - k0, N - k0 < DB ? N - k0 : DB, s->ev_read[j], su));
    *Ak = s->slot(j) - (ptrdiff_t)(k0 * ld + k0);
    return HB_OK;
  };
  auto after = [&](int, bool) -> int {
    if(!s->resident) HB_CUDA(cudaEventRecord(s->ev_read[j], su));
    return HB_OK;
  };
  for(int g0 = 0; g0 < nrhs; g0 += RHS) {
    const int ng = nrhs - g0 < RHS ? nrhs - g0 : RHS;
    double* xg = x + (size_t)g0 * N;
    HB_CHECK(hb_rbt_to_rows(c, N, ng, xg, xw, false));
    HB_CHECK(hb_rows_sweeps(N, ld, ldl, xw, ng, s->at(p.ybuf), s->at(p.tdot), su, rows, after));
    HB_CHECK(hb_rbt_to_rows(c, N, ng, xg, xw, true));
  }
  if(!s->resident) HB_CUDA(cudaStreamSynchronize(s->sc)); // the last read of the host matrix is done when the solve returns
  return 1;
}
