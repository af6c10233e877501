// The dense symmetric system factored across the ranks of the context's communicator: Cholesky LL^T and no-pivot LDL^T on a 1-D
// block-cyclic layout, with NCCL broadcasts of the panels (hb_symdense_dist_*, include/hiopb200.h).
//
// Layout. The block rows of hb_blockrow.cu: block row k belongs to rank k mod P and is stored as local block q = k div P, the owned
// block rows stacked in order, each 128 rows of ld doubles.
//
// Factorization: the step loop of hb_blockrow.cu over every block. All ranks run the same host sequence, so every rank issues the same
// collectives in the same order. Step k's transport: the owner's panel (the header [1/d, breakdown word] and the rows >= (k+1)*128,
// Cholesky: L, LDL^T: W = L D) is broadcast from buffer k & 1, where the others receive it. The loop's look-ahead lets the owner of block
// k+1 run its panel chain and broadcast under the others' update. The factor is bit-identical to hb_symdense's look-ahead path
// (unpaired blocks) for every P. The breakdown travels in its step's header, so every rank returns the same value.
//
// Solves (x replicated on every rank): the sweeps of hb_blockrow.cu, block k computed by its owner, which broadcasts the rows it changed
// (forward: rows k*128 .. N, backward: its block). Every block is computed in the same order for every P, so x does not depend on P.
//
// Safe mode (HB_FACT_RBT_NOPIV): A' = U^T A U with a depth-2 random butterfly U = B2 B1 (rbt_transform: the mirror of the upper
// triangle, then one pass per level, each output row formed from its row and its partner row; the kernels live in hb_rbt.cu), the
// no-pivot LDL^T above on A', and solves refined against a kept copy of A' (rbt_solve, the refinement loop of hb_rbt.cu). Every entry of A' is a fixed expression of oracle/rbt_model.py and the random
// diagonals depend on N alone, so A', the factor and the solution do not depend on P either.
#include "hb_common.cuh"
#include "hb_dense.cuh"

namespace {

constexpr int DB = HB_ROWS_DB, HDR = HB_ROWS_HDR;

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

struct hb_symdense_dist : hb_rows // the panel stream, the step loop's events and the outcome record
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
  // per-phase timing (hb_symdense_dist_profile): begin / end events of each phase of each step
  bool profile = false;
  std::unique_ptr<hb_event[]> ev_prof;
  float phase_ms[HB_ROWS_PH_COUNT] = {0.f, 0.f, 0.f};
  // HB_FACT_RBT_NOPIV, allocated by the first RBT factorization: A' (full rows, owned like A), the butterfly diagonals (2 N), the row
  // sums of |A'| and norm scratch; the solve adds b', the residual and the per-rhs norms
  bool rbt_ready = false;
  hb_dev<double> Ak, rbt_f, rbt_rows, rbt_nrm, rbt_b, rbt_r;
  hb_pinned<double> rbt_nrm_host;
  hb_event ev_rbt[2];
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
    HB_CHECK(s->create());
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
      s->ev_prof.reset(new hb_event[(size_t)2 * HB_ROWS_PH_COUNT * (s->nblk > 0 ? s->nblk : 1)]);
      for(int e = 0; e < 2 * HB_ROWS_PH_COUNT * s->nblk; e++) HB_CHECK(s->ev_prof[e].create(cudaEventDefault));
    }
    for(float& m : s->phase_ms) m = 0.f;
    s->profile = true;
    return HB_OK;
  }
  s->profile = false;
  if(ms3)
    for(int p = 0; p < HB_ROWS_PH_COUNT; p++) ms3[p] = s->phase_ms[p];
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
  const hb_rbt_rowmap cyclic{nullptr, nullptr, P, rank};
  if(s->profile) HB_CUDA(cudaEventRecord(s->ev_rbt[0], st));
  // mirror
  for(int k = 0; k < s->nblk; k++) {
    const int owner = k % P, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
    double* src = P == 1 ? s->A.get() : (owner == rank ? s->A.get() + (size_t)(k / P) * DB * ld : recv);
    if(P > 1) HB_CHECK(hb_broadcast(c, src, (long long)nb * ld, owner, st));
    const int q0 = P == 1 ? 0 : k0, nq = P == 1 ? N : nb;
    const int qa = k <= rank ? 0 : (k - rank + P - 1) / P; // first owned block at or after k
    if(nrows > qa * DB) {
      HB_CHECK(hb_rbt_mirror(c, N, cyclic, nrows, qa * DB, src, ld, q0, nq, s->A));
    }
    if(P == 1) break;
  }
  // the two levels: A -> Ak (B2), Ak -> A (B1)
  for(int st_i = 0; st_i < stages; st_i++) {
    const int level = st_i == 0 ? 2 : 1;
    const double* in = st_i == 0 ? s->A.get() : s->Ak.get();
    double* out = st_i == 0 ? s->Ak.get() : s->A.get();
    if(rbt_level_local(N, P, level)) {
      HB_CHECK(hb_rbt_level(c, N, level, s->rbt_f, in, ld, cyclic, nrows, nullptr, 0, out));
      continue;
    }
    for(int k = 0; k < s->nblk; k++) {
      const int owner = k % P, k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
      double* src = owner == rank ? const_cast<double*>(in) + (size_t)(k / P) * DB * ld : recv;
      HB_CHECK(hb_broadcast(c, src, (long long)nb * ld, owner, st));
      HB_CHECK(hb_rbt_level(c, N, level, s->rbt_f, in, ld, cyclic, nb, src, k0, out));
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
  return s->rbt_stats(corrections, backward_error, transform_ms);
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
  if(N == 0) { const double none[3] = {0.0, 0.0, 0.0}; return s->finish(none, 0); }
  HB_CUDA(cudaSetDevice(c->device));
  if(mode == HB_FACT_RBT_NOPIV) {
    HB_CHECK(agree(c, rbt_reserve(s)));
    HB_CHECK(rbt_transform(s, 2));
  }
  cudaStream_t su = c->stream;
  const long long ld = s->ld;
  HB_CUDA(cudaMemsetAsync(s->info, 0, sizeof(int) * 4, su));
  // the transport: the owner's panel goes out from the header and panel rows of broadcast buffer k & 1, the others receive it there
  auto at = [&](int k, bool, hb_rows_panel& b) -> int { // the slack of ld doubles in front keeps pan - r0 inside the allocation
    const int r0 = (k + 1) * DB < N ? (k + 1) * DB : N;
    b = {s->bbuf[k & 1] + ld, s->bbuf[k & 1] + ld + HDR, (N - r0 + 1) & ~1, r0, s->Lbuf[k & 1]};
    return HB_OK;
  };
  auto move = [&](int k, bool, const hb_rows_panel& b) { return hb_broadcast(c, b.hdr, HDR + DB * b.ldp, k % P, s->sp); };
  HB_CHECK(hb_rows_factor(c, *s, N, s->A, ld, P, rank, 0, s->nblk, ldl, s->inv16, s->info, at, move, s->profile ? s->ev_prof.get() : nullptr));
  HB_CHECK(hb_rows_inertia(s->A, ld, N, P, rank, s->nloc, s->red, su));
  HB_CHECK(hb_allreduce_op(c, s->red, 3, HB_SUM));
  HB_CUDA(cudaMemcpyAsync(s->red_host, s->red, sizeof(double) * 3, cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaMemcpyAsync(s->info_host, s->info, sizeof(int), cudaMemcpyDeviceToHost, su));
  HB_CUDA(cudaStreamSynchronize(su));
  if(s->profile) {
    for(int k = 0; k < s->nblk; k++)
      for(int ph = 0; ph < HB_ROWS_PH_COUNT; ph++) {
        if(ph == HB_ROWS_PH_UPDATE && k + 1 == s->nblk) continue; // the last block has no trailing update
        float ms = 0.f;
        HB_CUDA(cudaEventElapsedTime(&ms, s->ev_prof[((size_t)k * HB_ROWS_PH_COUNT + ph) * 2], s->ev_prof[((size_t)k * HB_ROWS_PH_COUNT + ph) * 2 + 1]));
        s->phase_ms[ph] += ms;
      }
  }
  return s->finish(s->red_host.get(), s->info_host[0]);
}

extern "C" int hb_symdense_dist_inertia(hb_symdense_dist* s, int* n_neg, int* n_null, int* n_pos)
{
  HB_REQUIRE(s, "null handle");
  return s->inertia(n_neg, n_null, n_pos);
}

// the forward and backward sweeps of the factor on the replicated row-major N x nrhs vectors xw, in place: the owner of block k computes
// it, then broadcasts the rows it changed (forward: k0 .. N-1, backward: its block)
static int dist_sweeps(hb_symdense_dist* s, double* xw, int nrhs)
{
  const int N = s->N, P = s->P;
  auto rows = [&](int k, const double** Ak) {
    *Ak = k % P == s->rank ? s->A.get() + (ptrdiff_t)((k / P) * DB - k * DB) * s->ld : nullptr;
    return HB_OK;
  };
  auto after = [&](int k, bool forward) {
    const int k0 = k * DB, nb = N - k0 < DB ? N - k0 : DB;
    return hb_broadcast(s->ctx, xw + (size_t)k0 * nrhs, (long long)(forward ? N - k0 : nb) * nrhs, k % P, s->ctx->stream);
  };
  return hb_rows_sweeps(N, s->ld, s->mode != HB_FACT_CHOLESKY, xw, nrhs, s->ybuf, s->tdot, s->ctx->stream, rows, after);
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
  if(const int rc = s->solve_ready(s->N, x, nrhs, "hb_symdense_dist"); rc != HB_OK) return rc;
  return dist_solve(s, x, nrhs, nullptr);
}

// diagnostics (tests): hb_symdense_dist_solve after HB_FACT_RBT_NOPIV, traced (collective)
extern "C" int hb_debug_symdense_dist_rbt_solve(hb_symdense_dist* s, double* x, int nrhs, int* ret_host, int* passes_host, double* anorm_host,
                                                double* norms_host, double* xp_host, double* bp_host)
{
  HB_REQUIRE(s && x && nrhs > 0 && s->N > 0, "hb_debug_symdense_dist_rbt_solve: bad arguments");
  auto solve = [&](hb_rbt_trace* t) { return dist_solve(s, x, nrhs, t); };
  return hb_rbt_traced_solve(*s, "hb_debug_symdense_dist_rbt_solve", solve, ret_host, passes_host, anorm_host, norms_host, xp_host, bp_host);
}
