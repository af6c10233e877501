// Shared internals of libhiopb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/hiopb200.h"

#define HB_NUM_SMS_DEFAULT 132

extern thread_local char g_hb_err[512];
extern long long g_hb_launches;

inline int hb_fail(int code, const char* fmt, const char* a = "", int line = 0)
{
  snprintf(g_hb_err, sizeof(g_hb_err), fmt, a, line);
  return code;
}

#define HB_CUDA(call)                                                                              \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if(e__ != cudaSuccess) {                                                                       \
      snprintf(g_hb_err, sizeof(g_hb_err), "%s at %s:%d", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return HB_ERR_CUDA;                                                                          \
    }                                                                                              \
  } while(0)

#define HB_CHECK(expr)                                                                             \
  do {                                                                                             \
    int rc__ = (expr);                                                                             \
    if(rc__ != HB_OK) return rc__;                                                                 \
  } while(0)

#define HB_REQUIRE(cond, msg)                                                                      \
  do {                                                                                             \
    if(!(cond)) {                                                                                  \
      snprintf(g_hb_err, sizeof(g_hb_err), "%s (%s:%d)", msg, __FILE__, __LINE__);                 \
      return HB_ERR_INVALID;                                                                       \
    }                                                                                              \
  } while(0)

// count a launch and check for launch errors
#define HB_LAUNCHED()                                                                              \
  do {                                                                                             \
    g_hb_launches++;                                                                               \
    cudaError_t e__ = cudaGetLastError();                                                          \
    if(e__ != cudaSuccess) {                                                                       \
      snprintf(g_hb_err, sizeof(g_hb_err), "launch failed: %s at %s:%d", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return HB_ERR_CUDA;                                                                          \
    }                                                                                              \
  } while(0)

// ---- ownership ----------------------------------------------------------------------------------------------------------
// Every device buffer, pinned buffer, stream and event the engine keeps is held by one of the owners below, and every handle is an
// aggregate of owners: deleting a handle releases what it holds, and a failed allocation leaves the owner empty, so the next call
// simply allocates it again. Owners release without synchronising; each *_destroy entry point synchronises the context stream first.
// g_hb_live counts what the owners hold (hb_debug_live_resources).
extern std::atomic<long long> g_hb_live;
struct hb_ctx;

// count elements of elem bytes, in pinned host memory or on the device. On failure *p stays null, the runtime error is cleared and
// the result is HB_ERR_ALLOC with a message naming `what` and the byte count.
int hb_mem_alloc(void** p, size_t count, size_t elem, bool pinned, const char* what);
void hb_mem_free(void* p, bool pinned);

template <typename T, bool PINNED>
class hb_array
{
public:
  hb_array() = default;
  hb_array(hb_array&& o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
  hb_array& operator=(hb_array&& o) noexcept
  {
    std::swap(p_, o.p_);
    std::swap(cap_, o.cap_);
    return *this;
  }
  ~hb_array() { reset(); }
  operator T*() const { return p_; }
  T* get() const { return p_; }
  size_t capacity() const { return cap_; }
  void reset()
  {
    if(p_) hb_mem_free(p_, PINNED);
    p_ = nullptr;
    cap_ = 0;
  }
  // Holds at least max(count, 1) elements afterwards, or nothing when the allocation fails (HB_ERR_ALLOC). Growing waits for the
  // context stream, frees the old array and then allocates: the contents are not kept.
  int reserve(hb_ctx* c, size_t count, const char* what);

private:
  T* p_ = nullptr;
  size_t cap_ = 0;
};
template <typename T> using hb_dev = hb_array<T, false>;
template <typename T> using hb_pinned = hb_array<T, true>;

// an owned cudaStream_t (hb_stream) or cudaEvent_t (hb_event)
template <typename H>
class hb_handle
{
public:
  hb_handle() = default;
  hb_handle(const hb_handle&) = delete;
  hb_handle& operator=(const hb_handle&) = delete;
  ~hb_handle();
  operator H() const { return h_; }
  int create(unsigned flags, int priority = 0); // no-op while one is held; the priority applies to streams

private:
  H h_ = nullptr;
};
using hb_stream = hb_handle<cudaStream_t>;
using hb_event = hb_handle<cudaEvent_t>;

// per-context state: of each int8 condensation (hb_int8_state, below; released in hb_ozaki.cu), the SYRK schedule cache (hb_syrk.cu)
struct hb_int8_state;
struct ScheduleCache;
void hb_delete(hb_int8_state* p);
void hb_delete(ScheduleCache* p);
struct hb_deleter
{
  template <typename S> void operator()(S* p) const { hb_delete(p); }
};
template <typename S> using hb_state = std::unique_ptr<S, hb_deleter>;

// phase marks of the quasi-Newton step (ids are the HB_PH_* below); a no-op unless hb_ctx_phase_timeline switched them on
enum { HB_PH_START = 0, HB_PH_UPDATE, HB_PH_OZ_ROWMAX, HB_PH_OZ_SLICE, HB_PH_CAUG, HB_PH_ALLREDUCE, HB_PH_VN, HB_PH_CHOL, HB_PH_HSOLVE1, HB_PH_JX, HB_PH_SPDSOLVE, HB_PH_JTY, HB_PH_HSOLVE2, HB_PH_COUNT };

struct hb_ctx
{
  int device = 0;
  int num_sms = HB_NUM_SMS_DEFAULT;
  hb_stream stream;
  // scratch for reductions: per-CTA partials + a pinned host landing slot
  hb_dev<double> red_dev;     // RED_SLOTS doubles
  hb_pinned<double> red_host; // 64 doubles
  // generic workspace (grown on demand by hb_ws_reserve)
  hb_dev<double> ws;
  // optional kernel timing (roofline reporting)
  bool timing = false;
  hb_event ev_syrk0, ev_syrk1;
  bool syrk_timed = false;
  // phase timeline (hb_ctx_phase_timeline): events recorded at fixed points of one update + condense + solve when enabled
  bool phases = false;
  hb_event ev_phase[HB_PH_COUNT];
  unsigned phase_mask = 0;
  // per-context state of the int8-slice condensation (hb_ozaki.cu: the slice buffer) and of the Chinese-remainder condensation
  // (hb_crt.cu: the residue planes), side by side
  hb_state<hb_int8_state> oz, crt;
  // schedule cache of the FP64 condensation (hb_syrk.cu)
  hb_state<ScheduleCache> syrk_sched;
  // dense symmetric solvers: size thresholds (with their environment overrides, set by hb_dense_init in hb_symdense.cu) and the
  // number of CTAs of the cooperative Cholesky resident at once (0: no cooperative kernels -- unsupported, or HB_CHOL_COOP=0)
  int bk_cluster_min = 0, big_min_chol = 0, big_min_ldl = 0, pair_min = 0;
  int coop_ctas = 0;
  hb_dev<long long> bkc_prof; // diagnostics: 8 cycle counters of the cluster Bunch-Kaufman panel while profiling is on
  // NCCL (destroyed by hb_ctx_destroy)
  void* nccl_comm = nullptr;
  int nranks = 1, rank = 0;
};

template <typename T, bool PINNED>
int hb_array<T, PINNED>::reserve(hb_ctx* c, size_t count, const char* what)
{
  if(p_ && count <= cap_) return HB_OK;
  if(p_) {
    HB_CUDA(cudaStreamSynchronize(c->stream));
    reset();
  }
  const size_t n = count ? count : 1;
  void* q = nullptr;
  HB_CHECK(hb_mem_alloc(&q, n, sizeof(T), PINNED, what));
  p_ = static_cast<T*>(q);
  cap_ = n;
  return HB_OK;
}

static constexpr int HB_RED_SLOTS = 4096;

// c->ws holds at least `bytes` afterwards
int hb_ws_reserve(hb_ctx* ctx, size_t bytes);

// grid of a grid-stride streaming kernel: one thread per item, at most 8 CTAs per SM, at least one CTA
inline int hb_grid(const hb_ctx* c, long long items, int threads = 256)
{
  const long long g = (items + threads - 1) / threads, cap = (long long)c->num_sms * 8;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// reduction operations; the values are NCCL's op codes (ncclSum, ncclMax, ncclMin)
enum hb_op { HB_SUM = 0, HB_MAX = 2, HB_MIN = 3 };

// in-place all-reduce of `count` doubles over the context's ranks, on the context stream (nothing to do on one rank)
int hb_allreduce_op(hb_ctx* c, double* buf, long long count, hb_op op);

// Second stage of the per-CTA reductions: out[q] = ops[q] over partial[b * slots + q], b < nblocks, slots = ops.size() <= 8. Fixed
// order: warp q owns slot q, lane l combines b = l, l + 32, ... in turn, then the warp combines its lanes with an xor tree.
int hb_reduce_slots(hb_ctx* c, int nblocks, const double* partial, double* out, std::initializer_list<hb_op> ops);
// out = [a (na doubles); b (nb doubles)]
int hb_stack(hb_ctx* c, int na, const double* a, int nb, const double* b, double* out);

// C = A diag(d) A^T over the rows of a device row-pointer table: FP64 DMMA (hb_syrk.cu), int8 slices (hb_ozaki.cu), int8 Chinese
// remaindering (hb_crt.cu). Optional dot_out[i] = sum_k row_i[k] d[k] dot_x[k] from the int8 row-maximum pass (none when K == 0).
int hb_syrk_rows(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool aligned16, const double* d, double* C, int ldc,
                 const double* fuse_rx = nullptr, double* tdot = nullptr);
bool hb_syrk_extra_row_is_free(int M);
int hb_syrk_rows_ozaki(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool rows_aligned16, const double* d, double* C, int ldc, int S,
                       const double* dot_x, double* dot_out);
// the correctly rounded value of an exact integer Gram
int hb_syrk_rows_crt(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool rows_aligned16, const double* d, double* C, int ldc,
                     const double* dot_x, double* dot_out);

// Runs launch(), which launches the GEMM kernel of a condensation, between the two events hb_ctx_last_syrk_ms reads when timing is on
template <typename F>
int hb_timed_syrk(hb_ctx* c, F&& launch)
{
  if(c->timing) HB_CUDA(cudaEventRecord(c->ev_syrk0, c->stream));
  HB_CHECK(launch());
  if(c->timing) {
    HB_CUDA(cudaEventRecord(c->ev_syrk1, c->stream));
    c->syrk_timed = true;
  }
  return HB_OK;
}

// The host driver of both int8 condensations (hb_ozaki.cu). Step 1: sd = sqrt(d) (when d is given), the exact row maxima of |a_ik| sd_k and their frexp exponents e_i, and optionally
// dot_out[i] = sum_k a_ik d_k dot_x_k from the same sweep. Marks HB_PH_OZ_ROWMAX.
struct hb_rowscale
{
  hb_dev<double> sd;
  hb_dev<unsigned long long> mx;
  hb_dev<int> e;
  hb_dev<double> dot_partial; // [chunks][M] partial row dots of the fused row-maximum pass
};
int hb_row_exponents(hb_ctx* c, hb_rowscale& rs, int M, int Mpad, long long K, const double* const* rowptr_dev, bool rows_aligned16,
                     const double* d, const double* dot_x, double* dot_out, const double** sd_out);

// How a scheme lays out its work. Rows are padded to tm, K to 128-byte stages; plane p of the int8 buffer holds row r at
// Q + (p Mpad + r) Kpad. The tiles (bi, bj) with bj >= (tm / tn) bi and bj tn < M cover the upper triangle. Work items are listed
// split-major, then by group, then by tile; the item of tile t, group g and split s owns workspace tile (t groups + g) splits + s.
struct hb_int8_layout
{
  int planes;         // int8 planes of every row: S slices, or N(K) moduli
  int tm, tn;         // output tile
  int groups;         // work items per tile and K range: 1 (each item runs all planes) or one per plane
  size_t tile_bytes;  // workspace of one item
  size_t item_bytes;  // the work item the GEMM kernel reads, written by put_item
  void (*put_item)(void* dst, int bi, int bj, int group, int k_begin, int k_count, int slot);
  // K splits for `units` items per split, max_splits read from the environment variable split_env (default 16) on every call
  int (*splits)(const hb_ctx* c, long long units, long long kstages, int max_splits, size_t tile_bytes);
  const char* split_env;
  int n_maps;
  cuuint32_t box[2][3]; // TMA box of each tensor map over (k bytes, row, plane)
};
// per-context state of one scheme: its planes, row scales, work list, tile list and tensor maps
struct hb_int8_state
{
  int M = -1, planes = 0, max_splits = 0; // (M, K, planes, max_splits): what the work list and tensor maps were built for
  long long K = -1, Kpad = 0;
  int Mpad = 0, splits = 0, n_tiles = 0, n_items = 0;
  hb_dev<int8_t> Q;
  hb_rowscale rs;
  hb_dev<unsigned char> items;
  hb_dev<int2> tiles;
  CUtensorMap maps[2];
  PFN_cuTensorMapEncodeTiled encode = nullptr; // resolved on first use
};
// Clears C for K == 0; nothing to do for M == 0
int hb_int8_empty(hb_ctx* c, int M, double* C, int ldc);
// The state of `slot` ready for M rows of K columns (M, K > 0): plane buffer, work list and tensor maps (rebuilt when the key changed),
// and a context workspace of one tile per item
int hb_int8_prepare(hb_ctx* c, hb_state<hb_int8_state>& slot, const hb_int8_layout& L, int M, long long K, hb_int8_state** st);
// The K-split search of both schemes: of at most max_splits splits (>= 64 stages and <= 1 GB of workspace, not asked of one split), the
// count with the shortest makespan ceil(units splits / SMs) / splits that beats `best`, the cost of `splits`, by 0.1 %; ties go lower
int hb_split_search(const hb_ctx* c, long long units, long long kstages, int max_splits, size_t tile_bytes, int splits, double best);

// set once by hb_ctx_create: the dynamic-shared-memory / cluster attributes of each kernel file's kernels (function attributes are
// per device) and the dense solvers' thresholds
int hb_syrk_init_attrs(hb_ctx* c);
int hb_ozaki_init_attrs(hb_ctx* c);
int hb_crt_init_attrs(hb_ctx* c);
int hb_microbench_init_attrs(hb_ctx* c);
int hb_dense_init(hb_ctx* c);

inline void hb_phase_mark(hb_ctx* c, int id)
{
  if(c->phases && c->ev_phase[id]) {
    cudaEventRecord(c->ev_phase[id], c->stream);
    c->phase_mask |= 1u << id;
  }
}

// ---- small device helpers ---------------------------------------------------------------------------------
__device__ __forceinline__ double hb_warp_sum(double v)
{
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double hb_warp_max(double v)
{
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double hb_warp_min(double v)
{
#pragma unroll
  for(int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <hb_op OP>
__device__ __forceinline__ double hb_identity()
{
  return OP == HB_SUM ? 0.0 : (OP == HB_MAX ? -INFINITY : INFINITY);
}
template <hb_op OP>
__device__ __forceinline__ double hb_combine(double a, double b)
{
  return OP == HB_SUM ? a + b : (OP == HB_MAX ? fmax(a, b) : fmin(a, b));
}
template <hb_op OP>
__device__ __forceinline__ double hb_warp_reduce(double v)
{
  return OP == HB_SUM ? hb_warp_sum(v) : (OP == HB_MAX ? hb_warp_max(v) : hb_warp_min(v));
}

// Block-wide reduction in a FIXED order (warp xor trees, then warp 0 runs one over the per-warp values) -> deterministic for a fixed
// launch geometry. Starts with a barrier, so `sm` may be reused by consecutive calls.
template <hb_op OP, int THREADS>
__device__ __forceinline__ double hb_block_reduce(double v, double* sm /* >= THREADS/32 doubles */)
{
  v = hb_warp_reduce<OP>(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if(l == 0) sm[w] = v;
  __syncthreads();
  double r = hb_identity<OP>();
  if(w == 0) r = hb_warp_reduce<OP>((l < THREADS / 32) ? sm[l] : hb_identity<OP>());
  return r; // valid on warp 0 (all lanes)
}
template <int THREADS>
__device__ __forceinline__ double hb_block_sum(double v, double* sm)
{
  return hb_block_reduce<HB_SUM, THREADS>(v, sm);
}

// stream-K style even split of `total` items over `parts`
__host__ __device__ inline long long hb_part_begin(long long total, int parts, int p)
{
  return (total / parts) * p + (p < (int)(total % parts) ? p : (total % parts));
}
