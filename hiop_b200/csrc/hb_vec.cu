// hiopVector elementwise ops and reductions (oracle: src/LinAlg/hiopVectorPar.cpp in the reference tree).
// All kernels are pure HBM streams: 128-bit loads/stores (double2) when every pointer is 16-byte aligned,
// grid = num_SMs x 8 CTAs of 256 threads, grid-stride. Reductions are two-stage with a fixed summation order
// (deterministic for a given n), never atomics. The second reduction stage of the other kernel files (hb_reduce_slots) and the
// [a; b] stacking of the two multiplier blocks (hb_stack) live here too.
#include "hb_common.cuh"

namespace {

constexpr int VT = 256;

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- elementwise: y[i] = f(y[i], x[i], z[i], s[i]) --------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(VT) k_ew2(long long n2, double2* __restrict__ y, const double2* __restrict__ x,
                                           const double2* __restrict__ z, const double2* __restrict__ s, F f)
{
  const long long stride = (long long)gridDim.x * VT;
  for(long long i = (long long)blockIdx.x * VT + threadIdx.x; i < n2; i += stride) {
    double2 yy = y[i];
    double2 xx = x ? x[i] : make_double2(0., 0.);
    double2 zz = z ? z[i] : make_double2(0., 0.);
    double2 ss = s ? s[i] : make_double2(0., 0.);
    yy.x = f(yy.x, xx.x, zz.x, ss.x);
    yy.y = f(yy.y, xx.y, zz.y, ss.y);
    y[i] = yy;
  }
}
template <class F>
__global__ void __launch_bounds__(VT) k_ew1(long long n, long long start, double* __restrict__ y, const double* __restrict__ x,
                                           const double* __restrict__ z, const double* __restrict__ s, F f)
{
  const long long stride = (long long)gridDim.x * VT;
  for(long long i = start + (long long)blockIdx.x * VT + threadIdx.x; i < n; i += stride) {
    y[i] = f(y[i], x ? x[i] : 0., z ? z[i] : 0., s ? s[i] : 0.);
  }
}

template <class F>
int ew(hb_ctx* c, long long n, double* y, const double* x, const double* z, const double* s, F f)
{
  HB_REQUIRE(c && n >= 0, "vector op: bad arguments");
  if(n == 0) return HB_OK;
  HB_REQUIRE(y != nullptr, "vector op: null y");
  const bool v2 = aligned16(y) && (!x || aligned16(x)) && (!z || aligned16(z)) && (!s || aligned16(s));
  long long n2 = v2 ? n / 2 : 0;
  if(n2 > 0) {
    k_ew2<<<hb_grid(c, n2, VT), VT, 0, c->stream>>>(n2, (double2*)y, (const double2*)x, (const double2*)z, (const double2*)s, f);
    HB_LAUNCHED();
  }
  if(2 * n2 < n) {
    k_ew1<<<hb_grid(c, n - 2 * n2, VT), VT, 0, c->stream>>>(n, 2 * n2, y, x, z, s, f);
    HB_LAUNCHED();
  }
  return HB_OK;
}

// ---- reductions ------------------------------------------------------------------------------------------
template <hb_op OP, class F>
__global__ void __launch_bounds__(VT) k_red1(long long n, const double* __restrict__ a, const double* __restrict__ b,
                                            const double* __restrict__ s, F f, double* __restrict__ partial)
{
  __shared__ double sm[VT / 32];
  double acc = hb_identity<OP>();
  const long long stride = (long long)gridDim.x * VT;
  for(long long i = (long long)blockIdx.x * VT + threadIdx.x; i < n; i += stride)
    acc = hb_combine<OP>(acc, f(a[i], b ? b[i] : 0., s ? s[i] : 0.));
  double r = hb_block_reduce<OP, VT>(acc, sm);
  if(threadIdx.x == 0) partial[blockIdx.x] = r;
}
template <hb_op OP>
__global__ void __launch_bounds__(VT) k_red2(int np, const double* __restrict__ partial, double* __restrict__ out)
{
  __shared__ double sm[VT / 32];
  double acc = hb_identity<OP>();
  for(int i = threadIdx.x; i < np; i += VT) acc = hb_combine<OP>(acc, partial[i]);
  double r = hb_block_reduce<OP, VT>(acc, sm);
  if(threadIdx.x == 0) out[0] = r;
}

template <hb_op OP, class F>
int reduce(hb_ctx* c, long long n, const double* a, const double* b, const double* s, F f, double* out_host, bool sqrt_after = false,
           double scale = 1.0)
{
  HB_REQUIRE(c && out_host && n >= 0, "reduction: bad arguments");
  int g = hb_grid(c, n, VT);
  if(g > HB_RED_SLOTS - 8) g = HB_RED_SLOTS - 8;
  double* res = c->red_dev + (HB_RED_SLOTS - 8);
  k_red1<OP><<<g, VT, 0, c->stream>>>(n, a, b, s, f, c->red_dev);
  HB_LAUNCHED();
  k_red2<OP><<<1, VT, 0, c->stream>>>(g, c->red_dev, res);
  HB_LAUNCHED();
  HB_CHECK(hb_allreduce_op(c, res, 1, OP));
  HB_CUDA(cudaMemcpyAsync(c->red_host, res, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  HB_CUDA(cudaStreamSynchronize(c->stream));
  double v = c->red_host[0];
  if(sqrt_after) v = sqrt(v);
  *out_host = v * scale;
  return HB_OK;
}

// ---- second reduction stage and stacking for the other kernel files ------------------------------------------------------------
constexpr int MAX_SLOTS = 8;
struct SlotOps
{
  hb_op op[MAX_SLOTS];
};
template <hb_op OP>
__device__ __forceinline__ double fold_slot(int nblocks, int slots, int q, const double* __restrict__ partial)
{
  double v = hb_identity<OP>();
  for(int b = threadIdx.x & 31; b < nblocks; b += 32) v = hb_combine<OP>(v, partial[(size_t)b * slots + q]);
  return hb_warp_reduce<OP>(v);
}
__global__ void __launch_bounds__(32 * MAX_SLOTS) k_reduce_slots(int nblocks, int slots, const double* __restrict__ partial, SlotOps ops,
                                                                 double* __restrict__ out)
{
  const int q = threadIdx.x >> 5;
  const hb_op op = ops.op[q];
  const double v = op == HB_SUM ? fold_slot<HB_SUM>(nblocks, slots, q, partial)
                                : (op == HB_MAX ? fold_slot<HB_MAX>(nblocks, slots, q, partial) : fold_slot<HB_MIN>(nblocks, slots, q, partial));
  if((threadIdx.x & 31) == 0) out[q] = v;
}

__global__ void k_concat(int na, const double* __restrict__ a, int nb, const double* __restrict__ b, double* __restrict__ out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < na) out[i] = a[i];
  else if(i < na + nb) out[i] = b[i - na];
}

} // namespace

int hb_reduce_slots(hb_ctx* c, int nblocks, const double* partial, double* out, std::initializer_list<hb_op> ops)
{
  HB_REQUIRE(ops.size() >= 1 && ops.size() <= MAX_SLOTS, "hb_reduce_slots: 1 to 8 slots");
  SlotOps so{};
  int slots = 0;
  for(hb_op op : ops) so.op[slots++] = op;
  k_reduce_slots<<<1, 32 * slots, 0, c->stream>>>(nblocks, slots, partial, so, out);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_stack(hb_ctx* c, int na, const double* a, int nb, const double* b, double* out)
{
  if(na + nb == 0) return HB_OK;
  k_concat<<<(na + nb + 127) / 128, 128, 0, c->stream>>>(na, a, nb, b, out);
  HB_LAUNCHED();
  return HB_OK;
}

// ---- elementwise API -------------------------------------------------------------------------------------------
extern "C" int hb_vec_set(hb_ctx* c, long long n, double* y, double cst)
{
  return ew(c, n, y, nullptr, nullptr, nullptr, [cst] __device__(double, double, double, double) { return cst; });
}
extern "C" int hb_vec_copy(hb_ctx* c, long long n, double* y, const double* x)
{
  HB_REQUIRE(c && n >= 0, "hb_vec_copy: bad arguments");
  if(n) HB_CUDA(cudaMemcpyAsync(y, x, sizeof(double) * n, cudaMemcpyDeviceToDevice, c->stream));
  return HB_OK;
}
extern "C" int hb_vec_scale(hb_ctx* c, long long n, double* y, double alpha)
{
  return ew(c, n, y, nullptr, nullptr, nullptr, [alpha] __device__(double y, double, double, double) { return y * alpha; });
}
extern "C" int hb_vec_axpy(hb_ctx* c, long long n, double* y, double alpha, const double* x)
{
  return ew(c, n, y, x, nullptr, nullptr, [alpha] __device__(double y, double x, double, double) { return y + alpha * x; });
}
extern "C" int hb_vec_axzpy(hb_ctx* c, long long n, double* y, double alpha, const double* x, const double* z)
{
  // the reference special-cases alpha = +-1 only to skip a multiply (hiopVectorPar.cpp:720-733); (alpha*x)*z then +y, each
  // rounded separately (no FMA contraction) so the result is bit-identical to the CPU path
  return ew(c, n, y, x, z, nullptr, [alpha] __device__(double y, double x, double z, double) { return __dadd_rn(y, __dmul_rn(__dmul_rn(alpha, x), z)); });
}
extern "C" int hb_vec_axdzpy(hb_ctx* c, long long n, double* y, double alpha, const double* x, const double* z)
{
  // reference order for general alpha: x/z*alpha (hiopVectorPar.cpp:761)
  return ew(c, n, y, x, z, nullptr, [alpha] __device__(double y, double x, double z, double) { return __dadd_rn(y, __dmul_rn(__ddiv_rn(x, z), alpha)); });
}
extern "C" int hb_vec_axdzpy_w_pattern(hb_ctx* c, long long n, double* y, double alpha, const double* x, const double* z,
                                       const double* sel)
{
  HB_REQUIRE(sel || n == 0, "axdzpy_w_pattern: null pattern");
  // masked-out lanes may hold z == 0 (tests/LinAlg/vectorTests.hpp:1187-1191): the division is not evaluated there
  return ew(c, n, y, x, z, sel,
            [alpha] __device__(double y, double x, double z, double s) { return s == 1.0 ? __dadd_rn(y, __ddiv_rn(__dmul_rn(alpha, x), z)) : y; });
}
extern "C" int hb_vec_component_mult(hb_ctx* c, long long n, double* y, const double* x)
{
  return ew(c, n, y, x, nullptr, nullptr, [] __device__(double y, double x, double, double) { return y * x; });
}
extern "C" int hb_vec_component_div(hb_ctx* c, long long n, double* y, const double* x)
{
  return ew(c, n, y, x, nullptr, nullptr, [] __device__(double y, double x, double, double) { return y / x; });
}
extern "C" int hb_vec_component_div_w_pattern(hb_ctx* c, long long n, double* y, const double* x, const double* sel)
{
  HB_REQUIRE(sel || n == 0, "component_div_w_pattern: null pattern");
  // masked-out entries are set to 0, not kept (hiopVectorPar.cpp:588-591)
  return ew(c, n, y, x, nullptr, sel, [] __device__(double y, double x, double, double s) { return s == 0.0 ? 0.0 : y / x; });
}
extern "C" int hb_vec_invert(hb_ctx* c, long long n, double* y)
{
  return ew(c, n, y, nullptr, nullptr, nullptr, [] __device__(double y, double, double, double) { return 1.0 / y; });
}
extern "C" int hb_vec_select_pattern(hb_ctx* c, long long n, double* y, const double* sel)
{
  HB_REQUIRE(sel || n == 0, "select_pattern: null pattern");
  return ew(c, n, y, nullptr, nullptr, sel, [] __device__(double y, double, double, double s) { return s == 0.0 ? 0.0 : y; });
}
extern "C" int hb_vec_add_constant(hb_ctx* c, long long n, double* y, double cst)
{
  return ew(c, n, y, nullptr, nullptr, nullptr, [cst] __device__(double y, double, double, double) { return y + cst; });
}
extern "C" int hb_vec_add_constant_w_pattern(hb_ctx* c, long long n, double* y, double cst, const double* sel)
{
  HB_REQUIRE(sel || n == 0, "add_constant_w_pattern: null pattern");
  return ew(c, n, y, nullptr, nullptr, sel, [cst] __device__(double y, double, double, double s) { return s == 1.0 ? y + cst : y; });
}
extern "C" int hb_vec_add_log_barrier_grad(hb_ctx* c, long long n, double* y, double alpha, const double* x, const double* sel)
{
  HB_REQUIRE((sel && x) || n == 0, "add_log_barrier_grad: null argument");
  return ew(c, n, y, x, nullptr, sel, [alpha] __device__(double y, double x, double, double s) { return s == 1.0 ? __dadd_rn(y, __ddiv_rn(alpha, x)) : y; });
}
extern "C" int hb_vec_add_linear_damping_term(hb_ctx* c, long long n, double* y, const double* ixl, const double* ixu, double alpha,
                                              double ct)
{
  HB_REQUIRE((ixl && ixu) || n == 0, "add_linear_damping_term: null pattern");
  return ew(c, n, y, ixl, ixu, nullptr, [alpha, ct] __device__(double y, double l, double u, double) { return __dadd_rn(__dmul_rn(alpha, y), __dmul_rn(ct, __dsub_rn(l, u))); });
}

// ---- reductions API --------------------------------------------------------------------------------------------
extern "C" int hb_vec_dot(hb_ctx* c, long long n, const double* x, const double* y, double* out)
{
  return reduce<HB_SUM>(c, n, x, y, nullptr, [] __device__(double a, double b, double) { return a * b; }, out);
}
extern "C" int hb_vec_twonorm(hb_ctx* c, long long n, const double* x, double* out)
{
  return reduce<HB_SUM>(c, n, x, nullptr, nullptr, [] __device__(double a, double, double) { return a * a; }, out, true);
}
extern "C" int hb_vec_infnorm(hb_ctx* c, long long n, const double* x, double* out)
{
  int rc = reduce<HB_MAX>(c, n, x, nullptr, nullptr, [] __device__(double a, double, double) { return fabs(a); }, out);
  if(rc == HB_OK && n == 0) *out = 0.0;
  return rc;
}
extern "C" int hb_vec_onenorm(hb_ctx* c, long long n, const double* x, double* out)
{
  return reduce<HB_SUM>(c, n, x, nullptr, nullptr, [] __device__(double a, double, double) { return fabs(a); }, out);
}
extern "C" int hb_vec_min_w_pattern(hb_ctx* c, long long n, const double* x, const double* sel, double* out)
{
  HB_REQUIRE(sel || n == 0, "min_w_pattern: null pattern");
  // the reference starts from 1e100 (hiopVectorPar.cpp:826)
  int rc = reduce<HB_MIN>(c, n, x, nullptr, sel, [] __device__(double a, double, double s) { return s == 1.0 ? a : 1e100; }, out);
  if(rc == HB_OK && *out > 1e100) *out = 1e100;
  return rc;
}
extern "C" int hb_vec_log_barrier(hb_ctx* c, long long n, const double* x, const double* sel, double* out)
{
  HB_REQUIRE(sel || n == 0, "log_barrier: null pattern");
  return reduce<HB_SUM>(c, n, x, nullptr, sel, [] __device__(double a, double, double s) { return s != 0.0 ? log(a) : 0.0; }, out);
}
extern "C" int hb_vec_linear_damping_term(hb_ctx* c, long long n, const double* x, const double* ixl, const double* ixu, double mu,
                                          double kappa_d, double* out)
{
  HB_REQUIRE((ixl && ixu) || n == 0, "linear_damping_term: null pattern");
  int rc = reduce<HB_SUM>(c, n, x, ixl, ixu, [] __device__(double a, double l, double u) { return (l == 1.0 && u == 0.0) ? a : 0.0; }, out);
  if(rc == HB_OK) {
    double t = *out;
    t *= mu;
    t *= kappa_d;
    *out = t;
  }
  return rc;
}
extern "C" int hb_vec_fraction_to_bdry(hb_ctx* c, long long n, const double* x, const double* dx, double tau, const double* sel,
                                       double* out)
{
  HB_REQUIRE((x && dx) || n == 0, "fraction_to_bdry: null argument");
  int rc;
  if(sel)
    rc = reduce<HB_MIN>(c, n, x, dx, sel,
                       [tau] __device__(double xx, double d, double s) { return (d >= 0 || s == 0.0) ? 1.0 : fmin(1.0, -tau * xx / d); }, out);
  else
    rc = reduce<HB_MIN>(c, n, x, dx, nullptr, [tau] __device__(double xx, double d, double) { return d >= 0 ? 1.0 : fmin(1.0, -tau * xx / d); },
                       out);
  if(rc == HB_OK && n == 0) *out = 1.0;
  return rc;
}
