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
//
// Safe mode (HB_FACT_RBT_NOPIV, with a kept copy registered): A' = U^T A U strip by strip into the kept copy (rbt_transform: each strip's
// window assembled from the matrix's upper triangle, then the level kernels of hb_rbt.cu on an explicit row map), the factorization
// above with the slabs copied in from A' (the caller's strictly lower diagonal blocks merged back), and solves refined against A' with
// hb_rbt_solve, the residual streaming the block rows of A' through the ring. All bit-identical to hb_symdense_dist at P = 1.
#include <algorithm>
#include <vector>
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

// The safe mode (HB_FACT_RBT_NOPIV) in the same allocation. The transform runs strips of T butterfly slots: the window rows of A (X) and
// their level-2 rows (Y) take the part from hdr to the end, which holds nothing the transform needs; the ring slots bring the mirrored
// columns in their first 128 rows, and their second halves (the formed L, idle outside a factorization) hold the row sums of |A'|, the
// diagonals, ||A'||_inf and the window's row maps. A solve keeps the diagonals, b' and the residual there. So the factorization runs the
// plain plan, and a budget that takes a plain factorization takes this one.
enum { R_PEAK = 0, R_XFORM_H2D, R_XFORM_D2H, R_FACTOR_H2D, R_RESID_H2D, R_COUNT };

struct rbt_plan_t
{
  int slots = 0, T = 0, nstrip = 0, wr = 0;
  size_t Y = 0; // offset of Y from X (doubles)
  long long bytes[R_COUNT] = {0, 0, 0, 0, 0};
};

// a run of consecutive window rows g0 .. g1-1 at window positions pos ..
struct rbt_run { int g0, g1, pos; };

// the runs of a strip's window (upper parts copied from the host, lower parts mirrored) or, out, of its own rows
std::vector<rbt_run> strip_runs(const hb_rbt_window& w, bool out)
{
  std::vector<rbt_run> r;
  for(int a = 0; a < 4; a++) {
    const int lo = out ? w.s0 : std::max(0, w.s0 - w.ext), hi = std::min(w.qlen[a], out ? w.s1 : w.s1 + w.ext);
    if(lo < hi) r.push_back({w.qs[a] + lo, w.qs[a] + hi, a * w.W + lo - (w.s0 - w.ext)});
  }
  if(!out)
    for(int k = 4 * w.W; k < w.wr; k++) {
      const int g = hb_rbt_window_row(w, k);
      if(g >= 0) r.push_back({g, g + 1, k});
    }
  return r;
}

// the block rows k0 .. k0+nb-1 carry the mirrored columns of run u from lo on (lo >= g1: none)
int mirror_lo(const rbt_run& u, long long k0) { return (int)std::max<long long>(u.g0, k0 + 1); }

int make_rbt_plan(const plan_t& p, rbt_plan_t& r)
{
  r = rbt_plan_t{};
  const int N = p.N;
  if(N == 0) return HB_OK;
  const hb_rbt_window w1 = hb_rbt_window_of(N, 0, 1);
  r.slots = w1.slots;
  const size_t region = p.total - p.hdr;
  auto need = [&](int T) { return 2 * up((size_t)hb_rbt_window_of(N, 0, T).wr * p.ld); };
  if(need(1) > region) {
    snprintf(g_hb_err, sizeof(g_hb_err), "hb_symdense_host: the device budget of this handle holds no transform strip for N = %d (%zu bytes needed)", N,
             sizeof(double) * (p.hdr + need(1)));
    return HB_ERR_INVALID;
  }
  int lo = 1, hi = r.slots; // the largest T that fits
  while(lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if(need(mid) <= region) lo = mid;
    else hi = mid - 1;
  }
  r.T = lo;
  r.nstrip = (r.slots + r.T - 1) / r.T;
  const hb_rbt_window wT = hb_rbt_window_of(N, 0, r.T);
  r.wr = wT.wr;
  r.Y = up((size_t)r.wr * p.ld);
  // traffic: per strip the window's rows from their first column of the run, and the window's columns of every block row above them
  long long h2d = 0, diag = 0;
  for(int t = 0; t < r.nstrip; t++) {
    const hb_rbt_window w = hb_rbt_window_of(N, t * r.T, std::min(r.slots, (t + 1) * r.T));
    const std::vector<rbt_run> runs = strip_runs(w, false);
    for(const rbt_run& u : runs) {
      h2d += (long long)(u.g1 - u.g0) * (N - u.g0);
      for(int k = 0; k < p.nblk; k++) {
        const long long k0 = (long long)k * DB, nb = N - k0 < DB ? N - k0 : DB;
        const int lo_c = mirror_lo(u, k0);
        if(lo_c < u.g1) h2d += nb * (u.g1 - lo_c);
      }
    }
  }
  for(int k = 0; k < p.nblk; k++) {
    const long long nb = N - (long long)k * DB < DB ? N - (long long)k * DB : DB;
    diag += nb * nb;
  }
  r.bytes[R_PEAK] = p.bytes[B_PEAK];
  r.bytes[R_XFORM_H2D] = 8 * h2d;
  r.bytes[R_XFORM_D2H] = 8LL * N * N;
  r.bytes[R_FACTOR_H2D] = p.bytes[B_H2D] + 8 * diag;
  r.bytes[R_RESID_H2D] = 8LL * N * N;
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

// the strictly lower part of a diagonal block (nb x nb, pitch ld) from T into D: the caller's entries that ride along with a block row of A'
__global__ void k_keep_lower(int nb, const double* __restrict__ T, long long ld, double* __restrict__ D)
{
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < nb * nb; e += gridDim.x * blockDim.x) {
    const int i = e / nb, j = e % nb;
    if(j < i) D[(size_t)i * ld + j] = T[(size_t)i * ld + j];
  }
}

} // namespace

struct hb_symdense_host : hb_rows // the panel stream, the step loop's events and the outcome record
{
  hb_ctx* ctx = nullptr;
  plan_t p;
  hb_dev<double> mem;          // the plan's device allocation
  hb_pinned<double> Wh;        // LDL^T with several slabs: W = L D of the blocks a later slab streams, block k at woff[k], N - (k+1)*128 per row
  std::vector<size_t> woff;
  hb_pinned<double> host;      // landing slots: inertia counts (3 doubles), info word, ||A'||_inf, the solve's norms (3 RHS)
  double* M = nullptr;         // the caller's page-locked matrix (borrowed)
  long long ldh = 0;
  double* K = nullptr;         // HB_FACT_RBT_NOPIV: the caller's page-locked buffer for A' (borrowed)
  long long ldk = 0;
  rbt_plan_t rp;
  hb_stream sc;                // copy stream
  hb_event ev_in[2], ev_read[2], ev_out[2], ev_a, ev_b, ev_panel, ev_t[2];
  bool resident = false;
  double* at(size_t off) const { return mem.get() + off; }
  double* slot(int j) const { return mem.get() + p.ring + (size_t)j * 2 * DB * p.ld; } // W or L rows; the formed L follows at + 128 ld
  double* half(int j) const { return slot(j) + (size_t)DB * p.ld; }                    // that second half
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
  HB_CHECK(s->host.reserve(c, 8 + 3 * RHS, "inertia counts, info word and norms"));
  HB_CHECK(s->create());
  HB_CHECK(s->sc.create(cudaStreamNonBlocking));
  for(int j = 0; j < 2; j++)
    for(hb_event* e : {&s->ev_in[j], &s->ev_read[j], &s->ev_out[j]}) HB_CHECK(e->create(cudaEventDisableTiming));
  for(hb_event* e : {&s->ev_a, &s->ev_b, &s->ev_panel}) HB_CHECK(e->create(cudaEventDisableTiming));
  for(hb_event& e : s->ev_t) HB_CHECK(e.create(cudaEventDefault));
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
// its diagonal column to N - 1. HB_FACT_RBT_NOPIV brings A' in from the kept copy; the strictly lower part of its diagonal block is then
// the caller's again (from M through the second half of ring slot 1, which no step uses before the slab's loop), so that it goes back
// unchanged.
int slab_copy(hb_symdense_host* s, int b0, int kb, int ke, bool in)
{
  const plan_t& p = s->p;
  const int N = p.N;
  const long long ld = p.ld, ldh = s->ldh;
  const bool kept = in && s->mode == HB_FACT_RBT_NOPIV;
  double* S = s->at(p.slab);
  for(int k = kb; k < ke; k++) {
    const long long k0 = (long long)k * DB, nb = N - k0 < DB ? N - k0 : DB;
    double* d = S + (size_t)(k0 - (long long)b0 * DB) * ld + k0;
    double* h = s->M + (size_t)k0 * ldh + k0;
    if(kept) {
      HB_CUDA(cudaMemcpy2DAsync(d, sizeof(double) * ld, s->K + (size_t)k0 * s->ldk + k0, sizeof(double) * s->ldk, sizeof(double) * (N - k0), nb,
                                cudaMemcpyHostToDevice, s->sc));
      HB_CUDA(cudaMemcpy2DAsync(s->half(1), sizeof(double) * ld, h, sizeof(double) * ldh, sizeof(double) * nb, nb, cudaMemcpyHostToDevice, s->sc));
      k_keep_lower<<<(int)((nb * nb + 255) / 256), 256, 0, s->sc>>>((int)nb, s->half(1), ld, d);
      HB_LAUNCHED();
    } else if(in) HB_CUDA(cudaMemcpy2DAsync(d, sizeof(double) * ld, h, sizeof(double) * ldh, sizeof(double) * (N - k0), nb, cudaMemcpyHostToDevice, s->sc));
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

// the device scratch of the safe mode in the second halves of the ring slots (see rbt_plan_t)
struct rbt_scratch
{
  double *rsum, *f, *nrm, *bp, *rw;
  int *rows, *pos_win, *pos_out;
};
rbt_scratch scratch(const hb_symdense_host* s)
{
  const int N = s->p.N;
  const size_t ints = up(((size_t)s->rp.wr + 1) / 2) * 2; // window positions, in ints, rounded to the alignment
  rbt_scratch r;
  r.f = s->half(0);
  r.rsum = r.f + up(2 * (size_t)N);
  r.nrm = r.rsum + up(N);
  r.bp = r.rsum; // a solve: b' after the diagonals
  r.rw = s->half(1);
  r.rows = reinterpret_cast<int*>(s->half(1));
  r.pos_win = r.rows + ints;
  r.pos_out = r.pos_win + up(((size_t)N + 1) / 2) * 2;
  return r;
}

// A' = U^T A U into the kept copy, strip by strip (hb_rbt_window), and ||A'||_inf into s->rbt_anorm. M is only read.
//   copy stream: the window rows of A, each run from its first column on, into X; then, for every block row above the window's last
//                row, its columns at the window rows into ring slot t & 1; finally the strip's rows of A' from X to the kept copy
//   compute    : the mirror of each slot into the lower parts of X; level 2 (X -> Y) on the window, level 1 (Y -> X) on the strip's
//                rows; their row sums of |A'|
int rbt_transform(hb_symdense_host* s)
{
  hb_ctx* c = s->ctx;
  const plan_t& p = s->p;
  const rbt_plan_t& rp = s->rp;
  const int N = p.N;
  const long long ld = p.ld, ldh = s->ldh;
  cudaStream_t su = c->stream, sc = s->sc;
  const rbt_scratch r = scratch(s);
  double* X = s->at(p.hdr);
  double* Y = X + rp.Y;
  long long t = 0;
  HB_CUDA(cudaEventRecord(s->ev_t[0], su));
  HB_CHECK(hb_rbt_table(c, N, r.f));
  for(int st = 0; st < rp.nstrip; st++) {
    const hb_rbt_window w = hb_rbt_window_of(N, st * rp.T, std::min(rp.slots, (st + 1) * rp.T));
    const std::vector<rbt_run> runs = strip_runs(w, false), outs = strip_runs(w, true);
    const hb_rbt_rowmap win{r.rows, r.pos_win, 1, 0}, own{r.rows, r.pos_out, 1, 0};
    HB_CHECK(hb_rbt_window_map(c, w, r.rows, r.pos_win, r.pos_out));
    HB_CHECK(order(s, true)); // the last strip's kernels are done with X and Y
    int last = 0;
    for(const rbt_run& u : runs) {
      HB_CUDA(cudaMemcpy2DAsync(X + (size_t)u.pos * ld + u.g0, sizeof(double) * ld, s->M + (size_t)u.g0 * ldh + u.g0, sizeof(double) * ldh,
                                sizeof(double) * (N - u.g0), u.g1 - u.g0, cudaMemcpyHostToDevice, sc));
      last = std::max(last, u.g1 - 1);
    }
    for(long long k0 = 0; k0 < last; k0 += DB) {
      const long long nb = N - k0 < DB ? N - k0 : DB;
      const int j = (int)(t++ & 1);
      HB_CUDA(cudaStreamWaitEvent(sc, s->ev_read[j], 0));
      for(const rbt_run& u : runs) {
        const int lo = mirror_lo(u, k0);
        if(lo < u.g1)
          HB_CUDA(cudaMemcpy2DAsync(s->slot(j) + lo, sizeof(double) * ld, s->M + (size_t)k0 * ldh + lo, sizeof(double) * ldh, sizeof(double) * (u.g1 - lo),
                                    nb, cudaMemcpyHostToDevice, sc));
      }
      HB_CUDA(cudaEventRecord(s->ev_in[j], sc));
      HB_CUDA(cudaStreamWaitEvent(su, s->ev_in[j], 0));
      HB_CHECK(hb_rbt_mirror(c, N, win, w.wr, 0, s->slot(j), ld, (int)k0, (int)nb, X));
      HB_CUDA(cudaEventRecord(s->ev_read[j], su));
    }
    HB_CHECK(order(s, false));
    HB_CHECK(hb_rbt_level(c, N, 2, r.f, X, ld, win, w.wr, nullptr, 0, Y));
    HB_CHECK(hb_rbt_level(c, N, 1, r.f, Y, ld, own, w.wr, nullptr, 0, X));
    for(const rbt_run& u : outs) HB_CHECK(hb_rbt_rows(c, N, 1, 0, u.g1 - u.g0, X + (size_t)u.pos * ld, ld, 0, nullptr, nullptr, r.rsum + u.g0));
    HB_CHECK(order(s, true));
    for(const rbt_run& u : outs)
      HB_CUDA(cudaMemcpy2DAsync(s->K + (size_t)u.g0 * s->ldk, sizeof(double) * s->ldk, X + (size_t)u.pos * ld, sizeof(double) * ld, sizeof(double) * N,
                                u.g1 - u.g0, cudaMemcpyDeviceToHost, sc));
  }
  HB_CHECK(hb_rbt_max1(c, N, r.rsum, r.nrm));
  HB_CHECK(order(s, false)); // the kept copy is complete
  HB_CUDA(cudaEventRecord(s->ev_t[1], su));
  HB_CUDA(cudaMemcpyAsync(s->host.get() + 4, r.nrm, sizeof(double), cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaStreamSynchronize(su));
  s->rbt_anorm = s->host.get()[4];
  HB_CUDA(cudaEventElapsedTime(&s->rbt_ms, s->ev_t[0], s->ev_t[1]));
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

// whether the N x N buffers a (ld lda) and b (ld ldb) share memory
bool overlaps(const double* a, long long lda, const double* b, long long ldb, int N)
{
  const double *a1 = a + (size_t)(N - 1) * lda + N, *b1 = b + (size_t)(N - 1) * ldb + N;
  return a < b1 && b < a1;
}

} // namespace

extern "C" int hb_symdense_host_set_rbt_copy(hb_symdense_host* s, double* K_host, long long ld)
{
  HB_REQUIRE(s, "null handle");
  const int N = s->p.N;
  s->factored = s->resident = false;
  s->K = nullptr;
  if(!K_host || N == 0) return HB_OK;
  HB_REQUIRE(ld >= N, "hb_symdense_host_set_rbt_copy: ld < N");
  HB_REQUIRE(page_locked(K_host) && page_locked(K_host + (size_t)(N - 1) * ld + N - 1),
             "hb_symdense_host_set_rbt_copy: the copy must be page-locked host memory (hb_malloc_host or hb_host_register)");
  HB_REQUIRE(!s->M || !overlaps(K_host, ld, s->M, s->ldh, N), "hb_symdense_host_set_rbt_copy: the copy overlaps the matrix");
  HB_CHECK(make_rbt_plan(s->p, s->rp));
  s->K = K_host;
  s->ldk = ld;
  return HB_OK;
}

extern "C" int hb_symdense_host_matrix_changed(hb_symdense_host* s, int mode)
{
  HB_REQUIRE(s, "null handle");
  if(mode == HB_FACT_BUNCH_KAUFMAN)
    return hb_fail(HB_ERR_INVALID, "hb_symdense_host_matrix_changed: Bunch-Kaufman needs up-to-date columns for its pivot search; use hb_symdense%s", "");
  const plan_t& p = s->p;
  const int N = p.N;
  const bool rbt = mode == HB_FACT_RBT_NOPIV;
  if(rbt && N > 0 && !s->K)
    return hb_fail(HB_ERR_INVALID, "hb_symdense_host_matrix_changed: the random butterfly keeps A' in a second page-locked buffer; register one with "
                                   "hb_symdense_host_set_rbt_copy%s", "");
  HB_REQUIRE(mode == HB_FACT_NOPIV || mode == HB_FACT_CHOLESKY || rbt, "hb_symdense_host_matrix_changed: bad mode");
  const bool ldl = mode != HB_FACT_CHOLESKY;
  if(N > 0 && !s->M) return hb_fail(HB_ERR_STATE, "hb_symdense_host_matrix_changed: no matrix (call hb_symdense_host_set_matrix)%s", "");
  HB_REQUIRE(!rbt || N == 0 || !overlaps(s->K, s->ldk, s->M, s->ldh, N), "hb_symdense_host_matrix_changed: the copy of A' overlaps the matrix");
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
  if(rbt) HB_CHECK(rbt_transform(s));
  HB_CHECK(factor(s, ldl));
  s->resident = p.nslab == 1;
  return s->finish(s->host.get(), *reinterpret_cast<const int*>(s->host.get() + 3));
}

extern "C" int hb_symdense_host_inertia(hb_symdense_host* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  return s->inertia(n_neg, n_null, n_pos);
}

extern "C" int hb_symdense_host_solve(hb_symdense_host* s, double* x, int nrhs)
{
  HB_REQUIRE(s && nrhs >= 0, "hb_symdense_host_solve: bad arguments");
  const plan_t& p = s->p;
  const int N = p.N;
  if(const int rc = s->solve_ready(N, x, nrhs, "hb_symdense_host"); rc != HB_OK) return rc;
  hb_ctx* c = s->ctx;
  HB_CUDA(cudaSetDevice(c->device));
  cudaStream_t su = c->stream;
  const bool ldl = s->mode != HB_FACT_CHOLESKY, rbt = s->mode == HB_FACT_RBT_NOPIV;
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
  int ok = 1;
  const rbt_scratch r = scratch(s);
  if(rbt) {
    HB_CHECK(hb_rbt_table(c, N, r.f));
    s->rbt_corr = 0;
    s->rbt_berr = 0.0;
  }
  for(int g0 = 0; g0 < nrhs; g0 += RHS) {
    const int ng = nrhs - g0 < RHS ? nrhs - g0 : RHS;
    double* xg = x + (size_t)g0 * N;
    HB_CHECK(hb_rbt_to_rows(c, N, ng, xg, xw, false));
    if(!rbt) {
      HB_CHECK(hb_rows_sweeps(N, ld, ldl, xw, ng, s->at(p.ybuf), s->at(p.tdot), su, rows, after));
    } else {
      // refined against the kept A': the residual rows of each block row of A', streamed through the ring like a factor row
      auto sweeps = [&](double* v) { return hb_rows_sweeps(N, ld, true, v, ng, s->at(p.ybuf), s->at(p.tdot), su, rows, after); };
      auto residual = [&](const double* xv, const double* b, double* out) -> int {
        for(int k = 0; k < p.nblk; k++) {
          const long long k0 = (long long)k * DB, nb = N - k0 < DB ? N - k0 : DB;
          const int jr = (int)(t++ & 1);
          HB_CHECK(ring_in(s, jr, s->K + (size_t)k0 * s->ldk, s->ldk, N, nb, s->ev_read[jr], su));
          HB_CHECK(hb_rbt_rows(c, N, 1, 0, (int)nb, s->slot(jr), ld, ng, xv, b + (size_t)k0 * ng, out + (size_t)k0 * ng));
          HB_CUDA(cudaEventRecord(s->ev_read[jr], su));
        }
        return HB_OK;
      };
      int corr = 0;
      double berr = 0.0;
      const int rc = hb_rbt_solve(c, N, ng, r.f, s->rbt_anorm, xw, r.bp, r.rw, s->host.get() + 8, sweeps, residual, &corr, &berr);
      if(rc < 0) return rc;
      ok &= rc;
      s->merge_rbt(corr, berr);
    }
    HB_CHECK(hb_rbt_to_rows(c, N, ng, xg, xw, true));
  }
  if(!s->resident || rbt) HB_CUDA(cudaStreamSynchronize(s->sc)); // the last read of the host buffers is done when the solve returns
  return ok;
}

extern "C" int hb_symdense_host_rbt_stats(hb_symdense_host* s, int* corrections, double* backward_error, float* transform_ms)
{
  HB_REQUIRE(s, "null handle");
  return s->rbt_stats(corrections, backward_error, transform_ms);
}

extern "C" int hb_symdense_host_rbt_plan_view(int N, size_t device_bytes, int* dims, int* strip_first_slot_host, long long* bytes_host)
{
  HB_REQUIRE(device_bytes > 0, "hb_symdense_host_rbt_plan_view: device_bytes must be given (0 asks the device, which this host-only view does not)");
  plan_t p;
  rbt_plan_t r;
  HB_CHECK(make_plan(N, device_bytes, p));
  HB_CHECK(make_rbt_plan(p, r));
  if(dims) {
    dims[0] = r.nstrip;
    dims[1] = r.T;
    dims[2] = r.slots;
    dims[3] = r.wr;
    dims[4] = p.nslab;
    dims[5] = p.H;
  }
  if(strip_first_slot_host) {
    for(int t = 0; t < r.nstrip; t++) strip_first_slot_host[t] = t * r.T;
    strip_first_slot_host[r.nstrip] = r.slots;
  }
  if(bytes_host)
    for(int b = 0; b < R_COUNT; b++) bytes_host[b] = r.bytes[b];
  return HB_OK;
}
