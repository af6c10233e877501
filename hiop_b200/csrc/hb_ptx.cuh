// Every inline PTX instruction of the library (sm_90a), one __device__ __forceinline__ function each; the kernel files and the probes
// in tools/ call these and write no asm of their own. The comment on each function states what a caller may rely on. Every wait and
// fence carries a "memory" clobber: the compiler neither moves a load or store across it nor keeps a value read before it in a
// register past it. Issuing an asynchronous copy orders nothing by itself; its wait does.
#pragma once
#include <cuda.h>
#include <cstdint>

// the 32-bit shared-window address of a generic pointer into this CTA's shared memory, as the PTX operands below take it
__device__ __forceinline__ uint32_t hb_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- cp.async: 16 (8) bytes global -> shared; the src_bytes read (0, 8 or 16) are followed by zeros. The data are defined to the
// issuing thread after the wait of its group (to other threads after that wait and a barrier) or through hb_mbar_arrive_cp_async.
__device__ __forceinline__ void hb_cp_async16(void* smem, const void* gmem, int src_bytes)
{
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(hb_smem_addr(smem)), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void hb_cp_async8(void* smem, const void* gmem, int src_bytes)
{
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(hb_smem_addr(smem)), "l"(gmem), "r"(src_bytes));
}
// closes the group of this thread's cp.async issued since the last commit
__device__ __forceinline__ void hb_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
// returns once at most N of this thread's committed groups are still in flight
template <int N> __device__ __forceinline__ void hb_cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
// returns once all of this thread's cp.async, committed or not, have landed
__device__ __forceinline__ void hb_cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// ---- mbarrier: an 8-byte barrier object in shared memory
// sets the barrier to expect `count` arrivals per phase; other threads may use it only after hb_mbar_init_fence and a CTA barrier
__device__ __forceinline__ void hb_mbar_init(unsigned long long* bar, unsigned count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(hb_smem_addr(bar)), "r"(count) : "memory");
}
// makes the preceding inits visible to the async proxy and to the other CTAs of the cluster (release)
__device__ __forceinline__ void hb_mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
// one arrival, with release semantics: the thread's earlier accesses happen before the phase completes
__device__ __forceinline__ void hb_mbar_arrive(unsigned long long* bar)
{
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(hb_smem_addr(bar)) : "memory");
}
// one arrival that also makes the current phase wait for `bytes` more bytes of asynchronous writes (TMA, st.async) to complete
__device__ __forceinline__ void hb_mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(hb_smem_addr(bar)), "r"(bytes) : "memory");
}
// one arrival (counted in the init count: noinc) once all earlier cp.async of this thread have landed
__device__ __forceinline__ void hb_mbar_arrive_cp_async(unsigned long long* bar)
{
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(hb_smem_addr(bar)) : "memory");
}
// Blocks until the phase of the given parity has completed (acquire: what was released into that phase is visible afterwards). The
// retry loop lives inside the asm, so to the compiler the wait is straight-line code and a warpgroup stays converged for wgmma.
// SUSPEND_NS != 0 lets each try suspend the thread for up to that many nanoseconds before it fails.
template <unsigned SUSPEND_NS = 0>
__device__ __forceinline__ void hb_mbar_wait(unsigned long long* bar, unsigned parity)
{
  if constexpr(SUSPEND_NS == 0)
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra.uni DONE_%=;\nbra.uni WAIT_%=;\nDONE_%=:\n}\n"
                 ::"r"(hb_smem_addr(bar)), "r"(parity) : "memory");
  else
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n@p bra.uni DONE_%=;\nbra.uni WAIT_%=;\nDONE_%=:\n}\n"
                 ::"r"(hb_smem_addr(bar)), "r"(parity), "r"(SUSPEND_NS) : "memory");
}
// one non-blocking test of the phase of the given parity: true, with hb_mbar_wait's acquire, once it has completed
__device__ __forceinline__ bool hb_mbar_try_wait(unsigned long long* bar, unsigned parity)
{
  unsigned ok;
  asm volatile("{\n.reg .pred q;\nmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\nselp.u32 %0, 1, 0, q;\n}\n" : "=r"(ok) : "r"(hb_smem_addr(bar)), "r"(parity) : "memory");
  return ok != 0;
}

// ---- thread-block clusters
// the shared::cluster address of the same location in the shared memory of CTA `rank`
__device__ __forceinline__ uint32_t hb_mapa(const void* p, unsigned rank)
{
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(hb_smem_addr(p)), "r"(rank));
  return r;
}
// 8 bytes to shared::cluster address `dst` (hb_mapa), completing 8 transaction bytes of the barrier at `bar` in the same CTA; a
// reader of that CTA sees them after its wait on the barrier. No other ordering, not even among the posts of one thread.
__device__ __forceinline__ void hb_st_async_b64(uint32_t dst, unsigned long long bits, uint32_t bar)
{
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];\n" ::"r"(dst), "l"(bits), "r"(bar) : "memory");
}
// TMA: the box at (c0, c1, c2) of a 3-D tensor map -> dst, completing its bytes on `bar` (armed by hb_mbar_arrive_expect_tx); dst is
// readable after the wait on that barrier
__device__ __forceinline__ void hb_tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, unsigned long long* bar)
{
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n"
               ::"r"(hb_smem_addr(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(hb_smem_addr(bar)) : "memory");
}

// ---- programmatic dependent launch
// blocks until the grids this one depends on have completed and their memory operations are visible
__device__ __forceinline__ void hb_griddep_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
// lets the dependent grid start launching; orders none of this grid's memory accesses (the dependent's hb_griddep_wait does)
__device__ __forceinline__ void hb_griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

// a hint to pull the line holding p into L2; no ordering
__device__ __forceinline__ void hb_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];\n" ::"l"(p)); }
// this thread's earlier generic-proxy writes to shared memory become visible to later async-proxy reads (wgmma, TMA)
__device__ __forceinline__ void hb_fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
// the warpgroup's per-thread register budget rises (inc) or falls (dec) to N; all four warps of the warpgroup execute it together
template <int N> __device__ __forceinline__ void hb_setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void hb_setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N) : "memory"); }
// named barrier ID over NTHREADS threads (a multiple of 32) of the CTA, ordering their memory accesses as __syncthreads does
template <int ID, int NTHREADS> __device__ __forceinline__ void hb_bar_sync() { asm volatile("bar.sync %0, %1;\n" ::"n"(ID), "n"(NTHREADS) : "memory"); }

// ---- FP64 MMA (SASS DMMA), registers only. On sm_90a each shape is its own instruction (DMMA.8x8x4, DMMA.16x8x8, DMMA.16x8x16), and
// 8x8x4 issues at half the rate of the other two.
// c[0..1] += a * b: one m8n8k4 fragment per thread
__device__ __forceinline__ void hb_dmma884(double& c0, double& c1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
// the m16n8k8 and m16n8k16 shapes, fragments as in the PTX ISA (k_syrk_ws runs m16n8k16). For m16n8k16 with g = lane / 4, t = lane % 4:
// a[i] = A(g + 8 (i % 2), t + 4 (i / 2)), b[i] = B(t + 4 i, g), c = C(g, 2t), C(g, 2t + 1), C(g + 8, 2t), C(g + 8, 2t + 1)
__device__ __forceinline__ void hb_dmma1688(double (&c)[4], const double (&a)[4], const double (&b)[2])
{
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void hb_dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4])
{
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
               : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// ---- wgmma.mma_async m64nNk32 s32 += s8 * s8 (both operands K-major in shared memory, by descriptor), N = 32 * NQ.
// d holds the warpgroup's N/2 accumulators per thread; the 16 registers d[16q .. 16q+15] are output columns 32q .. 32q+31.
// scale_d = 0 overwrites d with the product, 1 accumulates.
// K-major SWIZZLE_128B operand descriptor of sm_90 (rows 128 B apart, 8-row groups 1024 B apart; layout type 1 = SWIZZLE_128B in
// bits 62-63). K steps of 32 bytes inside the 128-byte swizzle row advance the start address.
__device__ __forceinline__ uint64_t hb_wgmma_desc_sw128(uint32_t smem_addr)
{
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)((1024 >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// orders the warpgroup's earlier register and shared-memory accesses before the wgmma that follow
__device__ __forceinline__ void hb_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
// closes the group of the warpgroup's wgmma issued since the last commit
__device__ __forceinline__ void hb_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
// keeps the compiler from moving accumulator reads or writes across the asynchronous MMAs that own the register
__device__ __forceinline__ void hb_wgmma_fence_operand(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }
// returns once at most N of the warpgroup's committed groups are in flight: their accumulators and shared operands are free again
template <int N> __device__ __forceinline__ void hb_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }

template <int NQ>
__device__ __forceinline__ void hb_wgmma_s8(uint32_t* d, uint64_t da, uint64_t db, int scale_d);

template <>
__device__ __forceinline__ void hb_wgmma_s8<1>(uint32_t* d, uint64_t da, uint64_t db, int scale_d)
{
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
               : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void hb_wgmma_s8<4>(uint32_t* d, uint64_t da, uint64_t db, int scale_d)
{
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
               : "l"(da), "l"(db), "r"(scale_d));
}

template <>
__device__ __forceinline__ void hb_wgmma_s8<8>(uint32_t* d, uint64_t da, uint64_t db, int scale_d)
{
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n}\n"
               : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
               : "l"(da), "l"(db), "r"(scale_d));
}
