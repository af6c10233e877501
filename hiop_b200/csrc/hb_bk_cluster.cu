// Bunch-Kaufman LDL^T for large N: the panel is factorized by ONE THREAD-BLOCK CLUSTER of 16 CTAs with the panel resident in their
// (distributed) shared memory.
//
// Role: hiopLinSolverSymDenseLapack::matrixChanged's DSYTRF (src/LinAlg/hiopLinSolverSymDenseLapack.hpp:90-102) and
// hiopLinSolverSymDenseMagmaBuKa's magma_dsytrf_gpu (src/LinAlg/hiopLinSolverSymDenseMagma.cpp:151): same pivot rule as LAPACK's
// DSYTF2 / DLASYF ('L'), same inertia. oracle/bk_model.py is the numpy statement of exactly this organisation (tested against DSYTRF).
//
// Why a cluster: the pivot search needs the maximum of the whole current column once per column -- N global reductions per
// factorization. A grid-wide barrier per column adds up over thousands of columns, the one-CTA DLASYF panel of hb_dense.cu streams the panel through
// one SM. A cluster barrier is far cheaper (tools/cluster_probe.cu) and 16 SMs hold a 32-column panel of 13000 rows in shared memory.
//
//   * CTA r owns a contiguous slab of rows; slab[c][row] is kept RIGHT-LOOKING inside the panel (after each pivot the remaining
//     panel columns are updated in shared memory), so the current column is always up to date: no matrix-vector product per column.
//   * one cluster barrier per column on the common path: every CTA posts its column maximum and CTA 0 (owner of the panel's top rows)
//     posts the pivot column's top entries to all 16 CTAs through DSM, barrier, then everybody takes the same decision and updates
//     its rows with no further communication. A failed first test (|a_kk| < alpha colmax) costs two more barriers: the owner of row
//     imax posts that row, all CTAs build their part of the candidate column (entries outside the panel are updated on demand from
//     the finished slab columns), post its maximum, barrier, decide 1x1 / interchange / 2x2.
//   * the trailing matrix outside the panel stays non-updated in global memory and receives the interchanges as DLASYF's copies;
//     every global element is only ever touched by the CTA that owns its row index, so no inter-CTA ordering is needed there.
//   * L (and W = L*D for the trailing update) are written once per panel; the interchanges are logged and applied to the previous
//     columns by k_bk_apply_swaps on a side stream -> the stored factor is the fully permuted  P A P^T = L D L^T  (one permutation
//     vector, unit L with zeros below the diagonal of 2x2 blocks, d21 in dsub), which the blocked solves of hb_dense_big.cu consume.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include "hb_ptx.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace {

constexpr int CS = 16;     // CTAs per cluster
constexpr int PT = 1024;   // threads per CTA
constexpr int NBMAX = 64;  // widest panel (used when the slab of 64 columns fits in the cluster's shared memory)

// the 16 per-CTA candidates of a mailbox -> the cluster-wide maximum (every warp by shuffles)
template <typename IT>
__device__ __forceinline__ ArgMax mailbox_argmax(const double* v, const IT* idx)
{
  const int lane = threadIdx.x & 31;
  ArgMax r{-1.0, 0x7fffffff};
  if(lane < CS) { r.v = v[lane]; r.i = (int)idx[lane]; }
#pragma unroll
  for(int o = 8; o > 0; o >>= 1) {
    ArgMax b;
    b.v = __shfl_xor_sync(0xffffffffu, r.v, o);
    b.i = __shfl_xor_sync(0xffffffffu, r.i, o);
    r = argmax_comb(r, b);
  }
  r.v = __shfl_sync(0xffffffffu, r.v, 0);
  r.i = __shfl_sync(0xffffffffu, r.i, 0);
  return r;
}

// 8 bytes to the same shared-memory location of CTA `rank`, completing 8 bytes of that CTA's mailbox barrier
__device__ __forceinline__ void bk_post(const void* local_dst, unsigned long long bits, const void* local_bar, unsigned rank)
{
  hb_st_async_b64(hb_mapa(local_dst, rank), bits, hb_mapa(local_bar, rank));
}

// replicated per-step mailbox (one per parity); every CTA of the cluster holds a copy that the others write through DSM
struct BkStep
{
  double cand_v[CS];
  long long cand_i[CS];
  double coltop[NBMAX];      // column k at the panel's top rows: coltop[c] = T(k0+c, k), c >= kl                (from CTA 0, every step)
  double coltop1[NBMAX];     // column k+1 at the top rows, c >= kl+1                                            (from CTA 0, fail path)
  double colimax_top[NBMAX]; // column imax at the top rows below imax (imax inside the panel)                   (from CTA 0, fail path)
  double rowk[NBMAX];        // row k of the slab, all columns                                                   (from CTA 0, fail path)
  double rowk1[NBMAX];       // row k+1 of the slab                                                              (from CTA 0, fail path)
  double rowimax[NBMAX];     // row imax of the slab, all columns                                                (from its owner, fail path)
  double cand2_v[CS];
  int cand2_i[CS];
  double diag_imax;          // updated T(imax, imax)                                                            (from the owner of imax)
};

struct BkShared
{
  ArgMax am[32];
  int dtype[NBMAX]; // 0 = not factored, 1 = 1x1, 2 = first column of a 2x2 block, 3 = second column
  double d11[NBMAX], d21[NBMAX], d22[NBMAX];
  double ptop1[NBMAX], ptop2[NBMAX], ctop[NBMAX], vld[NBMAX];
  int swaps[2 * NBMAX];
  unsigned long long mbar[2]; // per-parity mailbox barriers: the step's posts arrive as st.async ... complete_tx (no cluster barrier, no fence)
  int piv[NBMAX];      // ipiv / dsub of the panel's columns, written to global memory once per panel (a global store per column sat in
  double sub[NBMAX];   // front of every cluster barrier: its release fence waits for all outstanding stores)
};

// swap log of one panel (global): [0] = number of interchanges, [1] = k0, [2] = kb, then (kk, kp) pairs
constexpr int SWAPLOG_STRIDE = 4 + 2 * NBMAX;

template <bool PROF>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(PT, 1)
k_bk_panel(double* __restrict__ A, long long lda, int N, double* __restrict__ W, long long ldw, int NB, int S, int* __restrict__ ipiv,
           double* __restrict__ dsub, int* __restrict__ state, int* __restrict__ swaplog_all, int panel_index,
           long long* __restrict__ prof /* NULL or 8 cycle counters (CTA 0, thread 0): load, column max, barrier 1, fail path, interchange, pivot, write-back */)
{
  long long pt0 = PROF ? clock64() : 0;
#define PP(slot) if(PROF && threadIdx.x == 0 && rank == 0) { const long long pt1 = clock64(); prof[slot] += pt1 - pt0; pt0 = pt1; }
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) unsigned char bk_smem[];
  double* slab = reinterpret_cast<double*>(bk_smem);          // [NB][S]
  double* ccol = slab + (size_t)NB * S;                       // [S] candidate column (own rows)
  BkStep* bc = reinterpret_cast<BkStep*>(ccol + S);           // [2]
  __shared__ BkShared sh;
  const int tid = threadIdx.x, nthr = blockDim.x;
  int* swaplog = swaplog_all + (size_t)panel_index * SWAPLOG_STRIDE;
  const int k0 = state[0];
  if(k0 >= N) {
    if(rank == 0 && tid == 0) { state[1] = 0; swaplog[0] = 0; swaplog[1] = k0; swaplog[2] = 0; }
    return; // uniform over the cluster: nobody reaches a cluster barrier
  }
  const int rows = N - k0;
  const bool last = rows <= NB;
  const int nbp = min(NB, rows);
  const int lo = k0 + rank * S;
  const int big = 0x7fffffff;
  // ---- load the slab (lower part of the panel columns; zeros elsewhere) ----
  for(int rl = tid; rl < S; rl += nthr) {
    const int i = lo + rl;
    for(int c0 = 0; c0 < nbp; c0 += 8) { // 8 independent loads in flight per thread
      double v[8];
#pragma unroll
      for(int q = 0; q < 8; q++) {
        const int c = c0 + q;
        v[q] = (c < nbp && i < N && i >= k0 + c) ? LC(A, lda, i, k0 + c) : 0.0;
      }
#pragma unroll
      for(int q = 0; q < 8; q++)
        if(c0 + q < nbp) slab[(size_t)(c0 + q) * S + rl] = v[q];
    }
  }
  if(tid < NBMAX) sh.dtype[tid] = 0;
  if(tid == 0) {
    hb_mbar_init(&sh.mbar[0], 1);
    hb_mbar_init(&sh.mbar[1], 1);
    hb_mbar_init_fence();
  }
  __syncthreads();
  cluster.sync();
  PP(0);

  int k = k0, nsw = 0, linfo = 0, step = 0;
  while(k < N && (last || (k - k0) < NB - 1)) {
    const int kl = k - k0;
    const int par = step & 1;
    BkStep* my = &bc[par];
    unsigned long long* mb = &sh.mbar[par];
    const unsigned mphase = (unsigned)((step >> 1) & 1); // each parity's barrier completes once every second step
    step++;
    // ---- S1: column maximum over my rows i > k, posted to every CTA; CTA 0 posts the top of column k ----
    {
      ArgMax a{-1.0, big};
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        if(i < N && i > k) a = argmax_comb(a, ArgMax{fabs(slab[(size_t)kl * S + rl]), i});
      }
      a = cta_argmax(a, sh.am);
      // this step's mail: 16 candidates (value + index) from the 16 CTAs and the top of column k from CTA 0
      if(tid == 0) hb_mbar_arrive_expect_tx(mb, CS * 16 + nbp * 8);
      if(tid < CS) {
        bk_post(&my->cand_v[rank], (unsigned long long)__double_as_longlong(a.v), mb, tid);
        bk_post(&my->cand_i[rank], (unsigned long long)(long long)a.i, mb, tid);
      }
      if(rank == 0)
        for(int e = tid; e < CS * nbp; e += nthr) {
          const int dst = e / nbp, c = e % nbp;
          bk_post(&my->coltop[c], (unsigned long long)__double_as_longlong(slab[(size_t)kl * S + c]), mb, dst);
        }
    }
    PP(1);
    while(!hb_mbar_try_wait(mb, mphase)) {}
    PP(2);
    const ArgMax cm = mailbox_argmax(my->cand_v, my->cand_i);
    const double absakk = fabs(my->coltop[kl]);
    double colmax = 0.0;
    int imax = k;
    if(k < N - 1) { colmax = cm.v; imax = cm.i; }
    int kstep = 1, kp = k;
    bool have_cand = false, zero_col = false;
    if(fmax(absakk, colmax) == 0.0 || absakk != absakk) {
      if(linfo == 0) linfo = k + 1; // DSYTF2: column is zero (or NaN): info = k, no elimination
      zero_col = true;
    } else if(absakk < BK_ALPHA * colmax) {
      // =================== fail path: candidate column = row/column imax of the updated trailing matrix ===================
      have_cand = true;
      const int il = imax - k0;                 // panel-local index of imax (>= nbp: outside the panel)
      const int owner = (imax - k0) / S;        // CTA that owns row imax
      const bool inpanel = il < nbp;
      // F1: owner posts row imax of the slab; CTA 0 posts rows k, k+1, the top of column k+1 and (inside the panel) of column imax
      if(rank == owner)
        for(int e = tid; e < CS * nbp; e += nthr) {
          const int dst = e / nbp, c = e % nbp;
          cluster.map_shared_rank(my, dst)->rowimax[c] = slab[(size_t)c * S + (imax - lo)];
        }
      if(rank == 0)
        for(int e = tid; e < CS * nbp; e += nthr) {
          const int dst = e / nbp, c = e % nbp;
          BkStep* r = cluster.map_shared_rank(my, dst);
          r->rowk[c] = slab[(size_t)c * S + kl];
          r->rowk1[c] = (kl + 1 < S) ? slab[(size_t)c * S + kl + 1] : 0.0;
          r->coltop1[c] = (kl + 1 < nbp && c >= kl + 1) ? slab[(size_t)(kl + 1) * S + c] : 0.0;
          r->colimax_top[c] = (inpanel && c > il) ? slab[(size_t)il * S + c] : 0.0;
        }
      cluster.sync();
      // v = (L D)(imax, c) for the finished columns (everybody, from the posted row and the replicated D blocks)
      if(tid < NBMAX) {
        double v = 0.0;
        const int c = tid;
        if(c < kl) {
          if(sh.dtype[c] == 1) v = my->rowimax[c] * sh.d11[c];
          else if(sh.dtype[c] == 2) v = my->rowimax[c] * sh.d11[c] + my->rowimax[c + 1] * sh.d21[c];
          else if(sh.dtype[c] == 3) v = my->rowimax[c - 1] * sh.d21[c - 1] + my->rowimax[c] * sh.d22[c - 1];
        }
        sh.vld[c] = v;
      }
      __syncthreads();
      // F2: my part of the candidate column
      ArgMax a2{-1.0, big};
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        double cv = 0.0;
        if(i < N && i >= k) {
          if(i - k0 < nbp && i < imax) cv = my->rowimax[i - k0];          // row piece inside the panel columns (slab row imax)
          else if(inpanel) cv = slab[(size_t)il * S + rl];                // i >= imax, column imax of the slab
          else {
            const double raw = i < imax ? __ldcg(&LC(A, lda, imax, i)) : __ldcg(&LC(A, lda, i, imax));
            double acc = 0.0;
            for(int c = 0; c < kl; c++) acc += slab[(size_t)c * S + rl] * sh.vld[c];
            cv = raw - acc;
          }
          if(i != imax) a2 = argmax_comb(a2, ArgMax{fabs(cv), i});
        }
        ccol[rl] = cv;
      }
      a2 = cta_argmax(a2, sh.am);
      if(tid < CS) {
        BkStep* r = cluster.map_shared_rank(my, tid);
        r->cand2_v[rank] = a2.v;
        r->cand2_i[rank] = a2.i;
        if(rank == owner) r->diag_imax = ccol[imax - lo];
      }
      cluster.sync();
      const double rowmax = fmax(0.0, mailbox_argmax(my->cand2_v, my->cand2_i).v);
      if(absakk >= BK_ALPHA * colmax * (colmax / rowmax)) kp = k;
      else if(fabs(my->diag_imax) >= BK_ALPHA * rowmax) kp = imax;
      else { kp = imax; kstep = 2; }
    }
    const int kk = k + kstep - 1, kkl = kk - k0;
    const bool swap = (kp != kk);
    PP(3);
    if(have_cand && (kp == imax)) {
      // candidate column at the panel's top rows (replicated): ctop[c] = T(k0+c, imax)-or-T(imax, k0+c)
      if(tid < NBMAX) {
        const int c = tid, i = k0 + c;
        double v = 0.0;
        if(c < nbp) {
          if(i < imax) v = my->rowimax[c];
          else if(i == imax) v = my->diag_imax;
          else v = my->colimax_top[c];
        }
        sh.ctop[c] = v;
      }
      __syncthreads();
    }
    if(swap) {
      const int kpl = kp - k0;
      const int owner = (kp - k0) / S;
      const int nfin = kl + (kstep == 2 ? 1 : 0);
      const double* oldtop_kk = (kk == k) ? my->coltop : my->coltop1;   // old column kk at the top rows
      const double* oldrow_kk = (kk == k) ? my->rowk : my->rowk1;
      // ---- global (non-updated) trailing matrix: DLASYF's copies of column kk into position kp (row owners only) ----
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        if(i < N) {
          if(i > kp) LC(A, lda, i, kp) = __ldcg(&LC(A, lda, i, kk));
          else if(i > kk && i < kp) LC(A, lda, kp, i) = __ldcg(&LC(A, lda, i, kk));
          else if(i == kp) LC(A, lda, kp, kp) = __ldcg(&LC(A, lda, kk, kk));
        }
      }
      // ---- slab: column kp (inside the panel) takes the old column kk below kp ----
      if(kpl < nbp) {
        for(int rl = tid; rl < S; rl += nthr) {
          const int i = lo + rl;
          if(i < N && i > kp) slab[(size_t)kpl * S + rl] = slab[(size_t)kkl * S + rl];
        }
        if(rank == 0 && tid == 0) slab[(size_t)kpl * S + kpl] = oldtop_kk[kkl];
      }
      __syncthreads();
      // ---- slab: rows kk <-> kp in the finished columns; row kp of the unfinished panel columns between kk and kp ----
      if(rank == 0 && tid < nfin) slab[(size_t)tid * S + kkl] = my->rowimax[tid];
      if(rank == owner && tid < nbp) {
        const int c = tid;
        if(c < nfin) slab[(size_t)c * S + (kp - lo)] = oldrow_kk[c];
        else if(c > kkl && k0 + c < kp) slab[(size_t)c * S + (kp - lo)] = oldtop_kk[c];
      }
      // ---- slab: new column kk = candidate column with the entries at positions kk and kp exchanged ----
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        if(i < N && i >= kk) {
          double v = ccol[rl];
          if(i == kk) v = my->diag_imax;
          else if(i == kp) v = my->rowimax[kkl];
          slab[(size_t)kkl * S + rl] = v;
        }
      }
      if(tid == 0) {
        sh.swaps[2 * nsw] = kk;
        sh.swaps[2 * nsw + 1] = kp;
      }
      nsw++;
      __syncthreads();
    }
    PP(4);
    // =================== pivot ===================
    if(kstep == 1) {
      double d;
      const bool plain = (!have_cand || kp == k); // the pivot column is column k as it stands: its top entries are in the mailbox
      const double* ptop = my->coltop;
      if(!plain) {
        if(tid < NBMAX) { // interchange: candidate column with positions kkl and kpl exchanged
          const int c = tid;
          double v = 0.0;
          if(c < nbp) {
            const int kpl = kp - k0;
            v = sh.ctop[c];
            if(c == kkl) v = my->diag_imax;
            else if(c == kpl) v = sh.ctop[kkl];
          }
          sh.ptop1[c] = v;
        }
        __syncthreads();
        ptop = sh.ptop1;
      }
      d = plain ? my->coltop[kl] : my->diag_imax;
      const double r1 = 1.0 / d;
      if(tid == 0) { sh.dtype[kl] = 1; sh.d11[kl] = d; }
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        if(i < N && i > k && !zero_col) {
          const double w = slab[(size_t)kl * S + rl];
          const double l = w * r1;
          const int cend = min(nbp - 1, i - k0);
          for(int c0 = kl + 1; c0 <= cend; c0 += 8) { // loads first, then the FMAs, then the stores (no dependent LDS/STS chain)
            double v[8], pt[8];
#pragma unroll
            for(int q = 0; q < 8; q++) {
              const int c = min(c0 + q, nbp - 1);
              v[q] = slab[(size_t)c * S + rl];
              pt[q] = ptop[c];
            }
#pragma unroll
            for(int q = 0; q < 8; q++)
              if(c0 + q <= cend) slab[(size_t)(c0 + q) * S + rl] = v[q] - l * pt[q];
          }
          slab[(size_t)kl * S + rl] = l;
        }
      }
      if(rank == 0 && tid == 0) {
        slab[(size_t)kl * S + kl] = d;
        sh.piv[kl] = kp + 1;
        sh.sub[kl] = 0.0;
      }
    } else {
      // 2x2 pivot on columns k, k+1 (kk = k+1 now holds the candidate column, rows already interchanged)
      const int kpl = kp - k0;
      if(tid < NBMAX) {
        const int c = tid;
        double v1 = 0.0, v2 = 0.0;
        if(c < nbp) {
          // column k at the top rows, with the interchange k+1 <-> kp applied to the row index
          v1 = my->coltop[c];
          if(swap) {
            if(c == kl + 1) v1 = my->rowimax[kl];          // T'(k+1, k) = T(kp, k)
            else if(c == kpl) v1 = my->coltop[kl + 1];     // T'(kp, k) = T(k+1, k)
          }
          // column k+1 = candidate column (positions k+1 and kp exchanged); without interchange imax == k+1: the slab column itself
          if(swap) {
            v2 = sh.ctop[c];
            if(c == kl + 1) v2 = my->diag_imax;
            else if(c == kpl) v2 = sh.ctop[kl + 1];
          } else {
            v2 = (c >= kl + 1) ? my->coltop1[c] : 0.0;
          }
        }
        sh.ptop1[c] = v1;
        sh.ptop2[c] = v2;
      }
      __syncthreads();
      const double a11 = sh.ptop1[kl], a21 = sh.ptop1[kl + 1], a22 = sh.ptop2[kl + 1];
      // LAPACK's scaled inverse of the 2x2 block (DSYTF2)
      const double e11 = a22 / a21, e22 = a11 / a21;
      const double t = 1.0 / (e11 * e22 - 1.0);
      const double s2 = t / a21;
      if(tid == 0) {
        sh.dtype[kl] = 2; sh.dtype[kl + 1] = 3;
        sh.d11[kl] = a11; sh.d21[kl] = a21; sh.d22[kl] = a22;
      }
      for(int rl = tid; rl < S; rl += nthr) {
        const int i = lo + rl;
        if(i < N && i > k + 1) {
          const double w1 = slab[(size_t)kl * S + rl], w2 = slab[(size_t)(kl + 1) * S + rl];
          const double l1 = s2 * (e11 * w1 - w2);
          const double l2 = s2 * (e22 * w2 - w1);
          const int cend = min(nbp - 1, i - k0);
          for(int c0 = kl + 2; c0 <= cend; c0 += 4) {
            double v[4], p1[4], p2[4];
#pragma unroll
            for(int q = 0; q < 4; q++) {
              const int c = min(c0 + q, nbp - 1);
              v[q] = slab[(size_t)c * S + rl];
              p1[q] = sh.ptop1[c];
              p2[q] = sh.ptop2[c];
            }
#pragma unroll
            for(int q = 0; q < 4; q++)
              if(c0 + q <= cend) slab[(size_t)(c0 + q) * S + rl] = v[q] - (l1 * p1[q] + l2 * p2[q]);
          }
          slab[(size_t)kl * S + rl] = l1;
          slab[(size_t)(kl + 1) * S + rl] = l2;
        }
      }
      if(rank == 0 && tid == 0) {
        slab[(size_t)kl * S + kl] = a11;
        slab[(size_t)kl * S + kl + 1] = 0.0; // L(k+1, k) = 0; d21 lives in dsub
        slab[(size_t)(kl + 1) * S + kl + 1] = a22;
        sh.piv[kl] = -(kp + 1);
        sh.piv[kl + 1] = -(kp + 1);
        sh.sub[kl] = a21;
        sh.sub[kl + 1] = 0.0;
      }
    }
    k += kstep;
    // no CTA barrier here: the next column maximum reads only the thread's own rows, and cta_argmax synchronises before anything
    // written by other threads (the top of the next column, sh.dtype ...) is read
    PP(5);
  }
  __syncthreads();
  // ---- write back L for the factored columns, W = L*D for the rows below the panel ----
  const int kb = k - k0;
  const int r0 = k0 + kb;
  for(int rl = tid; rl < S; rl += nthr) {
    const int i = lo + rl;
    if(i >= N) continue;
    for(int c = 0; c < kb; c++) {
      if(i < k0 + c) continue;
      const double l = slab[(size_t)c * S + rl];
      LC(A, lda, i, k0 + c) = l;
      if(i >= r0) {
        double w;
        const int ty = sh.dtype[c];
        if(ty == 1) w = l * sh.d11[c];
        else if(ty == 2) w = l * sh.d11[c] + slab[(size_t)(c + 1) * S + rl] * sh.d21[c];
        else w = slab[(size_t)(c - 1) * S + rl] * sh.d21[c - 1] + l * sh.d22[c - 1];
        W[(size_t)c * ldw + i] = w;
      }
    }
  }
  if(rank == 0) {
    for(int e = tid; e < kb; e += nthr) { ipiv[k0 + e] = sh.piv[e]; dsub[k0 + e] = sh.sub[e]; }
    for(int e = tid; e < 2 * nsw; e += nthr) swaplog[4 + e] = sh.swaps[e];
    if(tid == 0) {
      swaplog[0] = nsw; swaplog[1] = k0; swaplog[2] = kb;
      state[1] = kb;
      if(linfo != 0 && state[2] == 0) state[2] = linfo;
    }
  }
  PP(6);
#undef PP
}

// advances the panel origin after the trailing update has consumed (k0, kb)
__global__ void k_bk_advance(int* __restrict__ state)
{
  if(threadIdx.x == 0 && blockIdx.x == 0) state[0] += state[1];
}

// The interchanges of one panel applied to the rows of all PREVIOUS columns (fully permuted L) and to the permutation vector.
// The <= 32 swaps touch <= 64 rows: each thread (one column) reads all affected entries, then writes them to their final places --
// independent loads, no chain of dependent swaps.
__global__ void __launch_bounds__(256)
k_bk_apply_swaps(double* __restrict__ A, long long lda, int N, const int* __restrict__ swaplog_all, int panel_index, int* __restrict__ perm,
                 double* __restrict__ scratch /* 2*NBMAX x ldscr */, long long ldscr)
{
  __shared__ int rows[2 * NBMAX], src[2 * NBMAX];
  __shared__ int nrow;
  const int* swaplog = swaplog_all + (size_t)panel_index * SWAPLOG_STRIDE;
  const int nsw = swaplog[0], k0 = swaplog[1];
  if(nsw == 0) return;
  if(threadIdx.x == 0) {
    int n = 0;
    for(int s = 0; s < nsw; s++) {
      const int a = swaplog[4 + 2 * s], b = swaplog[4 + 2 * s + 1];
      int ia = -1, ib = -1;
      for(int q = 0; q < n; q++) { if(rows[q] == a) ia = q; if(rows[q] == b) ib = q; }
      if(ia < 0) { ia = n; rows[n] = a; src[n] = a; n++; }
      if(ib < 0) { ib = n; rows[n] = b; src[n] = b; n++; }
      const int t = src[ia]; src[ia] = src[ib]; src[ib] = t; // current row a now holds what was in row b
    }
    nrow = n;
  }
  __syncthreads();
  const int n = nrow;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if(j < k0) {
    // all affected entries of column j are staged (reads independent of each other), then written to their final rows
    for(int q0 = 0; q0 < n; q0 += 8) {
      double v[8];
#pragma unroll
      for(int q = 0; q < 8; q++) v[q] = q0 + q < n ? LC(A, lda, src[q0 + q], j) : 0.0;
#pragma unroll
      for(int q = 0; q < 8; q++)
        if(q0 + q < n) scratch[(size_t)(q0 + q) * ldscr + j] = v[q];
    }
    for(int q0 = 0; q0 < n; q0 += 8) {
      double v[8];
#pragma unroll
      for(int q = 0; q < 8; q++) v[q] = q0 + q < n ? scratch[(size_t)(q0 + q) * ldscr + j] : 0.0;
#pragma unroll
      for(int q = 0; q < 8; q++)
        if(q0 + q < n && src[q0 + q] != rows[q0 + q]) LC(A, lda, rows[q0 + q], j) = v[q];
    }
  }
  if(blockIdx.x == 0 && threadIdx.x == 0) {
    int pv[2 * NBMAX];
    for(int q = 0; q < n; q++) pv[q] = perm[src[q]];
    for(int q = 0; q < n; q++) perm[rows[q]] = pv[q];
  }
}

__global__ void k_iota(int N, int* __restrict__ perm, double* __restrict__ dsub)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < N) { perm[i] = i; dsub[i] = 0.0; }
}

// block-diagonal solve with D (1x1 and 2x2 blocks: dsub[k] != 0 marks the first row of a 2x2 block [[d_k, s],[s, d_k+1]])
__global__ void k_bk_dsolve(const double* __restrict__ F, long long ldf, int N, const int* __restrict__ ipiv, const double* __restrict__ dsub,
                            double* __restrict__ x)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if(k >= N) return;
  if(ipiv[k] > 0) { x[k] = x[k] / LC(F, ldf, k, k); return; }
  const double s = dsub[k];
  if(s == 0.0) return; // second row of a block (or handled by the first)
  const double akm1 = LC(F, ldf, k, k) / s, ak = LC(F, ldf, k + 1, k + 1) / s;
  const double denom = akm1 * ak - 1.0;
  const double bkm1 = x[k] / s, bk = x[k + 1] / s;
  x[k] = (ak * bkm1 - bk) / denom;
  x[k + 1] = (akm1 * bk - bkm1) / denom;
}

// inertia from the block diagonal with the reference's dsidi rule and thresholds (hiopLinSolverSymDenseLapack.hpp:127-167), all rows in
// parallel: a 1x1 pivot contributes the sign of d; the first row of a 2x2 block (dsub != 0) contributes (d_k/t) d_k+1 - t and t = |dsub|.
// ipiv == NULL: plain diagonal (no-pivot LDL^T / Cholesky factors).
__global__ void __launch_bounds__(1024)
k_inertia_par(const double* __restrict__ F, long long ldf, int N, const int* __restrict__ ipiv, const double* __restrict__ dsub, int* __restrict__ out)
{
  __shared__ int cnt[3];
  if(threadIdx.x < 3) cnt[threadIdx.x] = 0;
  __syncthreads();
  int neg = 0, nul = 0, pos = 0;
  for(int k = threadIdx.x; k < N; k += blockDim.x) {
    const double dk = LC(F, ldf, k, k);
    if(!ipiv || ipiv[k] > 0) {
      if(dk < -1e-14) neg++; else if(dk < 1e-14) nul++; else pos++;
    } else {
      const double s = dsub[k];
      if(s != 0.0) {
        const double t = fabs(s);
        const double d1 = (dk / t) * LC(F, ldf, k + 1, k + 1) - t;
        if(d1 < -1e-14) neg++; else if(d1 < 1e-14) nul++; else pos++;
        if(t < 1e-14) nul++; else pos++;
      }
    }
  }
  atomicAdd(&cnt[0], neg); atomicAdd(&cnt[1], nul); atomicAdd(&cnt[2], pos);
  __syncthreads();
  if(threadIdx.x < 3) out[threadIdx.x] = cnt[threadIdx.x];
}

} // namespace

// geometry of one cluster panel with `rows` active rows: rows per CTA (S), panel width (NB: the widest of 64/32/16/8 whose slab fits),
// dynamic shared memory
int hb_bkc_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_bk_panel<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  HB_CUDA(cudaFuncSetAttribute(k_bk_panel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  HB_CUDA(cudaFuncSetAttribute(k_bk_panel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  HB_CUDA(cudaFuncSetAttribute(k_bk_panel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  return HB_OK;
}

static void bkc_geometry(int rows, int* S, int* NB, size_t* smem)
{
  int s = (rows + CS - 1) / CS;
  if(s < NBMAX) s = NBMAX;
  s = (s + 31) & ~31;
  // 64 columns halve the passes of the trailing update over the matrix but lengthen the in-panel update of every column step:
  // break-even taken at 3000 active rows (not re-measured on H100)
  int nb = rows >= 3000 ? NBMAX : 32;
  const size_t budget = 200 * 1024;
  while(nb > 8 && ((size_t)nb * s + s) * sizeof(double) + 2 * sizeof(BkStep) > budget) nb >>= 1;
  *S = s; *NB = nb;
  *smem = ((size_t)nb * s + s) * sizeof(double) + 2 * sizeof(BkStep);
}

bool hb_bkc_supported(int N)
{
  int S, NB;
  size_t smem;
  bkc_geometry(N, &S, &NB, &smem);
  return smem <= 215 * 1024 && S >= NB;
}

// Bunch-Kaufman factorization P A P^T = L D L^T of the column-major-lower triangle (lda even). Outputs: unit L strictly below the
// diagonal (zeros below 2x2 blocks), D on the diagonal + dsub, ipiv (sign marks 2x2 blocks), perm (gather order for the right-hand
// side), info_dev (first exactly-zero pivot column, 1-based), widths_host (OR of the panel widths launched, in no order; the last launch
// may find no column left when the device k0 has already reached N). Wp: NB x ldw doubles of scratch (W = L*D of the current panel).
int hb_bkc_factor(hb_ctx* c, hb_big* b, int N, double* A, long long lda, int* ipiv_dev, double* dsub_dev, int* perm_dev, double* Wp, long long ldw,
                  int* state_dev /* 4 ints */, int* swaplog_dev, int* info_dev, int* widths_host)
{
  *widths_host = 0;
  double* swap_scratch = Wp + (size_t)NBMAX * ldw; // Wp holds NBMAX columns of W followed by 2*NBMAX rows of staging for the interchanges
  HB_REQUIRE((lda & 1) == 0, "hb_bkc_factor: needs an even leading dimension");
  HB_CHECK(hb_big_init(c, b));
  cudaStream_t st = c->stream, side = b->panel_stream;
  HB_CUDA(cudaMemsetAsync(state_dev, 0, sizeof(int) * 4, st));
  k_iota<<<(N + 255) / 256, 256, 0, st>>>(N, perm_dev, dsub_dev);
  HB_LAUNCHED();
  // The origin k0 of a panel is only known on the device (a panel factors NB or NB-1 columns); the host tracks its bounds
  // k0_min <= k0 <= k0_max to size the launches: rows per CTA and panel width from the rows that are certainly left at most.
  int k0_min = 0, k0_max = 0;
  for(int p = 0; k0_min < N; p++) {
    int S, NB;
    size_t smem;
    bkc_geometry(N - k0_min, &S, &NB, &smem);
    *widths_host |= NB;
    int threads = S < PT ? S : PT; // one row per thread where possible: fewer idle warps in every barrier / shuffle stage
    if(threads < 128) threads = 128;
    if(c->bkc_prof) k_bk_panel<true><<<CS, threads, smem, st>>>(A, lda, N, Wp, ldw, NB, S, ipiv_dev, dsub_dev, state_dev, swaplog_dev, p, c->bkc_prof);
    else k_bk_panel<false><<<CS, threads, smem, st>>>(A, lda, N, Wp, ldw, NB, S, ipiv_dev, dsub_dev, state_dev, swaplog_dev, p, nullptr);
    HB_LAUNCHED();
    // the interchanges on the previous columns and on the permutation run beside the trailing update (disjoint data)
    HB_CUDA(cudaEventRecord(b->ev_upd, st));
    HB_CUDA(cudaStreamWaitEvent(side, b->ev_upd, 0));
    {
      const int kmax = k0_max < N ? k0_max : N;
      k_bk_apply_swaps<<<kmax > 0 ? (kmax + 255) / 256 : 1, 256, 0, side>>>(A, lda, N, swaplog_dev, p, perm_dev, swap_scratch, ldw);
      HB_LAUNCHED();
    }
    const int r0_min = k0_min + (NB - 1);
    if(r0_min < N) HB_CHECK(hb_big_trailing_from_state(c, N, A, lda, Wp, ldw, state_dev, r0_min, st));
    k_bk_advance<<<1, 32, 0, st>>>(state_dev);
    HB_LAUNCHED();
    k0_min += NB - 1;
    k0_max += NB;
  }
  HB_CUDA(cudaEventRecord(b->ev_panel, side));
  HB_CUDA(cudaStreamWaitEvent(st, b->ev_panel, 0));
  HB_CUDA(cudaMemcpyAsync(info_dev, state_dev + 2, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return HB_OK;
}

int hb_dense_inertia_blockdiag(hb_ctx* c, int N, const double* F, long long ldf, const int* ipiv_dev, const double* dsub_dev, int* out3_dev)
{
  k_inertia_par<<<1, 1024, 0, c->stream>>>(F, ldf, N, ipiv_dev, dsub_dev, out3_dev);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_dense_inertia_diag(hb_ctx* c, int N, const double* F, long long ldf, int* out3_dev)
{
  return hb_dense_inertia_blockdiag(c, N, F, ldf, nullptr, nullptr, out3_dev);
}

int hb_bkc_dsolve(hb_ctx* c, int N, const double* F, long long ldf, const int* ipiv_dev, const double* dsub_dev, double* x)
{
  k_bk_dsolve<<<(N + 127) / 128, 128, 0, c->stream>>>(F, ldf, N, ipiv_dev, dsub_dev, x);
  HB_LAUNCHED();
  return HB_OK;
}

// diagnostics: switch the phase counters of k_bk_panel on (allocates / zeroes them) and read them back
int hb_bkc_profile(hb_ctx* c, int on, long long* prof_host8)
{
  if(on) {
    HB_CHECK(c->bkc_prof.reserve(c, 8, "Bunch-Kaufman profile counters"));
    HB_CUDA(cudaMemsetAsync(c->bkc_prof, 0, sizeof(long long) * 8, c->stream));
  } else if(c->bkc_prof) {
    if(prof_host8) {
      HB_CUDA(cudaMemcpyAsync(prof_host8, c->bkc_prof, sizeof(long long) * 8, cudaMemcpyDeviceToHost, c->stream));
      HB_CUDA(cudaStreamSynchronize(c->stream));
    }
    c->bkc_prof.reset();
  }
  return HB_OK;
}
