// C = A * diag(d) * A^T in FP64 on the sm_90a DMMA pipe -- the condensation kernel.
//
// Replaces the reference's scalar triple loops symmMatTimesDiagTimesMatTrans_local / matTimesDiagTimesMatTrans_local
// (src/Optimization/hiopHessianLowRank.cpp:1079-1154) which stream J m/2 times from DRAM. Here the augmented row set
// A = [J; S_t; Y_t] (M = m + 2l rows, K = n_local columns, K-contiguous rows living in several buffers -> a device
// table of row pointers) is read ONCE per output tile pair and all of W = J D J^T, S1, Y1 and the three l x l
// blocks of V come out of the same pass.
//
// Why DMMA and not the integer tensor path: wgmma has no f64 kind; mma.sync.*.f64 (SASS DMMA) is the FP64 tensor path of sm_90a. The
// kernel k_syrk_ws issues m16n8k16 (DMMA.16x8x16); m8n8k4 lowers to DMMA.8x8x4, which runs at half that rate on H100.
//
// Work decomposition: 128x128 output tiles (upper triangle of the tile grid only). k_syrk_ws sweeps K in 32-column chunks through a
// 3-stage ring filled by producer warps (see below), for every row alignment: rows that are only 8-byte aligned (every odd n_local)
// differ from 16-byte aligned ones in the producers' copy width alone.
// The diagonal tiles run in pairs on their upper triangles (see pair_cell_row). The (tile or pair, K-range) space is cut into one
// K window per CTA in K lanes, plus stream-K ranges for the CTAs left over (see plan_schedule): every SM is busy for the same time
// whatever M is, and the units of a lane start at the same columns. Each CTA writes its partial 128x128 tile to a workspace
// slot; a second kernel sums the slots of each tile in a FIXED order and mirrors the result, so the output is
// bit-reproducible run to run (no atomics).
#include "hb_common.cuh"
#include "hb_ptx.cuh"

#include <algorithm>

namespace {

constexpr int BM = 128;          // tile rows = tile cols

struct Seg
{
  int ti, tj;      // tile coordinates, ti <= tj; with slot_j >= 0 the two diagonal tiles (ti, ti) and (tj, tj)
  int k_begin;     // first K iteration (units of WBK columns)
  int k_count;     // number of K iterations
  int slot;        // workspace slot receiving the partial tile (ti, tj), or (ti, ti) of a diagonal pair
  int slot_j;      // diagonal pair: slot receiving the upper triangle of (tj, tj); -1 otherwise
};

// Diagonal pair: a CTA loads tile row ti into stage.a and tile row tj into stage.b as for the off-diagonal tile (ti, tj), and its MMA
// warps compute only the 16x16 cells on and above the diagonal of (ti, ti) (warps 0-3, from a x a) and of (tj, tj) (warps 4-7, from
// b x b): 2 x 36 cells, 144 of the 256 m16n8 fragments of two full diagonal tiles. Warp w takes the cells of block rows p = w & 3 and
// 7 - p: 8 - p cells in row p and p + 1 in row 7 - p, 9 in all, so every warp issues the same 18 m16n8k16 per 16 columns of K and
// warps w and w + 4 (the same tensor sub-partition) do equal work. Cell k (0..8) of block row p is (r, c) in 16-row blocks, in column
// order: columns p .. 6 - p hold row p alone, columns 7 - p .. 7 rows p and 7 - p, which then share one B fragment.
constexpr int PAIR_CELLS = 9;
__host__ __device__ constexpr int pair_cell_row(int p, int k) { return k < 7 - 2 * p || (k - (7 - 2 * p)) % 2 == 0 ? p : 7 - p; }
__host__ __device__ constexpr int pair_cell_col(int p, int k) { return k < 7 - 2 * p ? p + k : 7 - p + (k - (7 - 2 * p)) / 2; }

// ---------------------------------------------------------------------------------------------------------------------
// Warp-specialised kernel: 8 MMA warps + 4 producer warps, mbarrier full/empty ring.
// The producers issue cp.async copies (zero-filling rows beyond M and the K tail through the src-size operand)
// and signal the stage's mbarrier with cp.async.mbarrier.arrive.noinc; the MMA warps never execute a CTA-wide barrier
// and never compute a global address, so they drift out of phase and keep the FP64 tensor pipe busy during refills.
// Each MMA warp owns a 64x32 block of the tile: 4 x 4 m16n8k16 accumulators, 64 doubles per thread. With one A and four B fragments
// that does not fit the 168 registers of 384 threads, so the producer warpgroup gives its registers to the MMA warpgroups (setmaxnreg
// 40 / 232). d scales the B fragment in registers: each product is rounded twice.
// ALIGN16 (rows, d, the extra row and the row table 16-byte aligned): 16 producer threads per row, 16 bytes per copy. Otherwise
// (every odd n_local: the packed rows of J then start on alternating 8-byte boundaries) 32 threads per row, 8 bytes per copy. The
// copy width is the only difference: the shared layout, the MMA warps and so the summation order are the same.
// (A first version staged rows with 256-byte cp.async.bulk copies from one producer warp: 288 bulk copies per stage
// made the producer the bottleneck.)
// ---------------------------------------------------------------------------------------------------------------------
constexpr int WBK = 32;                 // doubles per K chunk
constexpr int WSTAGES = 3;
constexpr int WLDS = WBK + 4;           // 36 doubles = 288 B row stride (288 mod 128 = 32 -> conflict-free LDS.64 fragment reads)
constexpr int WTILE_D = BM * WLDS;
constexpr int WPROD = 128;              // producer threads (4 warps)
constexpr int WTHREADS = 256 + WPROD;
struct WStage
{
  double a[WTILE_D];
  double b[WTILE_D];
  double d[WBK];
};
constexpr size_t WSMEM_BYTES = sizeof(WStage) * WSTAGES + 2 * BM * sizeof(const double*) + 2 * WSTAGES * sizeof(unsigned long long);

// a cp.async of 16 (ALIGN16) or 8 bytes, of which the first src_bytes are read and the rest zero-filled
template <bool ALIGN16>
__device__ __forceinline__ void cp_async_chunk(double* smem, const double* gmem, int src_bytes)
{
  if constexpr(ALIGN16) hb_cp_async16(smem, gmem, src_bytes);
  else hb_cp_async8(smem, gmem, src_bytes);
}

// One segment of a full 128x128 tile on the 8 MMA warps (a diagonal tile multiplies stage.a by itself): the warp owns a 64x32 block.
__device__ __forceinline__ void mma_tile_seg(const Seg& sg, const WStage* stages, unsigned long long* full, unsigned long long* empty,
                                             int& stage, unsigned& phase, bool unit_d, int warp, int lane, double* ws)
{
  const int warp_m = warp & 1, warp_n = warp >> 1;
  const int g = lane >> 2, t4 = lane & 3;
  const bool diag = sg.ti == sg.tj;
  double acc[4][4][4]; // [16-row block i][8-column block j]: rows g, g, g+8, g+8; columns 2*t4, 2*t4+1, 2*t4, 2*t4+1
#pragma unroll
  for(int i = 0; i < 4; i++)
#pragma unroll
    for(int j = 0; j < 4; j++)
#pragma unroll
      for(int e = 0; e < 4; e++) acc[i][j][e] = 0.0;
  for(int it = 0; it < sg.k_count; it++) {
    hb_mbar_wait(&full[stage], phase);
    const WStage& st = stages[stage];
    const double* sA = st.a + (warp_m * 64 + g) * WLDS + t4;
    const double* sB = (diag ? st.a : st.b) + (warp_n * 32 + g) * WLDS + t4;
#pragma unroll
    for(int kk = 0; kk < WBK; kk += 16) {
      // m16n8k16 fragments: B element q at (k = t4 + 4q, column g), A element q at (row g + 8*(q&1), k = t4 + 4*(q>>1))
      double bf[4][4];
#pragma unroll
      for(int q = 0; q < 4; q++) {
        const double dv = unit_d ? 1.0 : st.d[kk + 4 * q + t4];
#pragma unroll
        for(int j = 0; j < 4; j++) bf[j][q] = sB[j * 8 * WLDS + kk + 4 * q] * dv;
      }
#pragma unroll
      for(int i = 0; i < 4; i++) {
        double af[8];
#pragma unroll
        for(int q = 0; q < 8; q++) af[q] = sA[(i * 16 + 8 * (q & 1)) * WLDS + kk + 4 * (q >> 1)];
#pragma unroll
        for(int j = 0; j < 4; j++) hb_dmma16816(acc[i][j], af, bf[j]);
      }
    }
    __syncwarp();
    if(lane == 0) hb_mbar_arrive(&empty[stage]);
    if(++stage == WSTAGES) { stage = 0; phase ^= 1; }
  }
  double* slot = ws + (size_t)sg.slot * (BM * BM);
#pragma unroll
  for(int i = 0; i < 4; i++) {
#pragma unroll
    for(int h = 0; h < 2; h++) {
      const int row = warp_m * 64 + i * 16 + 8 * h + g;
#pragma unroll
      for(int j = 0; j < 4; j++) {
        const int col = warp_n * 32 + j * 8 + t4 * 2;
        *reinterpret_cast<double2*>(slot + row * BM + col) = make_double2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
      }
    }
  }
}

// One segment of a diagonal pair on the warps of block row P (see pair_cell_row): 9 cells of 16x16, 72 accumulators per thread, the
// two A fragments and one B fragment at a time; within the 232 registers without spills only because P is a template parameter, so that
// each cell's fragments are known at compile time. As in a full tile, A is the block row of the lower-indexed rows and d scales the B fragment, so each product
// is rounded as it is there.
template <int P>
__device__ __forceinline__ void mma_pair_seg(const Seg& sg, const WStage* stages, unsigned long long* full, unsigned long long* empty,
                                             int& stage, unsigned& phase, bool unit_d, int warp, int lane, double* ws)
{
  const int g = lane >> 2, t4 = lane & 3;
  double acc[PAIR_CELLS][2][4]; // [cell][8-column half]: rows g, g, g+8, g+8; columns 2*t4, 2*t4+1, 2*t4, 2*t4+1
#pragma unroll
  for(int k = 0; k < PAIR_CELLS; k++)
#pragma unroll
    for(int h = 0; h < 2; h++)
#pragma unroll
      for(int e = 0; e < 4; e++) acc[k][h][e] = 0.0;
  for(int it = 0; it < sg.k_count; it++) {
    hb_mbar_wait(&full[stage], phase);
    const WStage& st = stages[stage];
    const double* sX = (warp < 4 ? st.a : st.b) + g * WLDS + t4;
#pragma unroll
    for(int kk = 0; kk < WBK; kk += 16) {
      double dv[4], alo[8], ahi[8], bf[2][4];
#pragma unroll
      for(int q = 0; q < 4; q++) dv[q] = unit_d ? 1.0 : st.d[kk + 4 * q + t4];
#pragma unroll
      for(int q = 0; q < 8; q++) {
        const int off = 8 * (q & 1) * WLDS + kk + 4 * (q >> 1);
        alo[q] = sX[P * 16 * WLDS + off];
        ahi[q] = sX[(7 - P) * 16 * WLDS + off];
      }
#pragma unroll
      for(int k = 0; k < PAIR_CELLS; k++) {
        const int r = pair_cell_row(P, k), c = pair_cell_col(P, k);
        if(k == 0 || c != pair_cell_col(P, k - 1)) {
#pragma unroll
          for(int h = 0; h < 2; h++)
#pragma unroll
            for(int q = 0; q < 4; q++) bf[h][q] = sX[(c * 16 + 8 * h) * WLDS + kk + 4 * q] * dv[q];
        }
        hb_dmma16816(acc[k][0], r == P ? alo : ahi, bf[0]);
        hb_dmma16816(acc[k][1], r == P ? alo : ahi, bf[1]);
      }
    }
    __syncwarp();
    if(lane == 0) hb_mbar_arrive(&empty[stage]);
    if(++stage == WSTAGES) { stage = 0; phase ^= 1; }
  }
  double* slot = ws + (size_t)(warp < 4 ? sg.slot : sg.slot_j) * (BM * BM);
#pragma unroll
  for(int k = 0; k < PAIR_CELLS; k++) {
    const int r = pair_cell_row(P, k), c = pair_cell_col(P, k);
#pragma unroll
    for(int h = 0; h < 2; h++) {
      const int row = r * 16 + 8 * h + g;
#pragma unroll
      for(int j = 0; j < 2; j++) {
        const int col = c * 16 + j * 8 + t4 * 2;
        *reinterpret_cast<double2*>(slot + row * BM + col) = make_double2(acc[k][j][2 * h], acc[k][j][2 * h + 1]);
      }
    }
  }
}

template <bool ALIGN16>
__global__ void __launch_bounds__(WTHREADS, 1)
k_syrk_ws(const double* const* __restrict__ rowptr, int M, long long K, const double* __restrict__ dvec, const double* __restrict__ extra_row,
          const Seg* __restrict__ segs, const int* __restrict__ cta_seg_begin, double* __restrict__ ws)
{
  extern __shared__ __align__(128) unsigned char smem_raw[];
  WStage* stages = reinterpret_cast<WStage*>(smem_raw);
  const double** srow = reinterpret_cast<const double**>(smem_raw + sizeof(WStage) * WSTAGES); // [2*BM] row pointers (producers only)
  unsigned long long* full = reinterpret_cast<unsigned long long*>(srow + 2 * BM);
  unsigned long long* empty = full + WSTAGES;

  const int tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  if(tid == 0) {
#pragma unroll
    for(int s = 0; s < WSTAGES; s++) {
      hb_mbar_init(&full[s], WPROD); // every producer thread arrives once its copies of the stage have landed
      hb_mbar_init(&empty[s], 8);    // one arrival per MMA warp
    }
    hb_mbar_init_fence();
  }
  __syncthreads();

  const int sb = cta_seg_begin[blockIdx.x], se = cta_seg_begin[blockIdx.x + 1];
  int stage = 0;
  unsigned phase = 0;

  if(warp >= 8) {
    // ================= producer warps =================
    hb_setmaxnreg_dec<40>();
    constexpr int CW = ALIGN16 ? 2 : 1;     // doubles per copy
    constexpr int LOG_LPR = ALIGN16 ? 4 : 5; // producer threads per row: WBK / CW
    constexpr int RSTEP = WPROD >> LOG_LPR;  // rows per pass: 8 or 4
    const int p = tid - 256;          // 0..127
    const int kc = p & ((1 << LOG_LPR) - 1); // copy within the 256-byte row segment
    const int r0 = p >> LOG_LPR;      // rows r0 + RSTEP*j
    for(int si = sb; si < se; si++) {
      const Seg sg = segs[si];
      const bool diag = sg.ti == sg.tj;
      hb_bar_sync<1, WPROD>(); // all producers done with the previous segment's row table
      for(int r = p; r < 2 * BM; r += WPROD) {
        const int grow = (r < BM ? sg.ti * BM + r : sg.tj * BM + (r - BM));
        srow[r] = grow < M ? rowptr[grow] : (grow == M ? extra_row : nullptr);
      }
      hb_bar_sync<1, WPROD>();
      for(int it = 0; it < sg.k_count; it++) {
        const long long k = ((long long)sg.k_begin + it) * WBK + kc * CW;
        const long long rem = K - k;
        const int nb = rem >= CW ? 8 * CW : (rem == 1 ? 8 : 0); // bytes read: the K tail fills half of a 16-byte copy
        const long long koff = nb ? k : 0;
        hb_mbar_wait(&empty[stage], phase ^ 1);
        WStage& st = stages[stage];
        // the zero-byte copies read from rowptr: a valid address aligned to the copy width (hb_syrk_rows checks 16 bytes for ALIGN16)
#pragma unroll 4
        for(int j = 0; j < BM / RSTEP; j++) {
          const int row = r0 + RSTEP * j;
          const double* pa = srow[row];
          cp_async_chunk<ALIGN16>(&st.a[row * WLDS + kc * CW], pa ? pa + koff : (const double*)rowptr, pa ? nb : 0);
          if(!diag) {
            const double* pb = srow[BM + row];
            cp_async_chunk<ALIGN16>(&st.b[row * WLDS + kc * CW], pb ? pb + koff : (const double*)rowptr, pb ? nb : 0);
          }
        }
        if(p < (1 << LOG_LPR) && dvec) cp_async_chunk<ALIGN16>(&st.d[kc * CW], nb ? dvec + k : (const double*)rowptr, nb);
        hb_mbar_arrive_cp_async(&full[stage]);
        if(++stage == WSTAGES) { stage = 0; phase ^= 1; }
      }
    }
    hb_cp_async_wait_all();
  } else {
    // ================= 8 MMA warps =================
    hb_setmaxnreg_inc<232>(); // 64 (72 in a diagonal pair) accumulators + the A and B fragments of m16n8k16 per thread
    const bool unit_d = (dvec == nullptr);
    for(int si = sb; si < se; si++) {
      const Seg sg = segs[si];
      if(sg.slot_j < 0) mma_tile_seg(sg, stages, full, empty, stage, phase, unit_d, warp, lane, ws);
      else if((warp & 3) == 0) mma_pair_seg<0>(sg, stages, full, empty, stage, phase, unit_d, warp, lane, ws);
      else if((warp & 3) == 1) mma_pair_seg<1>(sg, stages, full, empty, stage, phase, unit_d, warp, lane, ws);
      else if((warp & 3) == 2) mma_pair_seg<2>(sg, stages, full, empty, stage, phase, unit_d, warp, lane, ws);
      else mma_pair_seg<3>(sg, stages, full, empty, stage, phase, unit_d, warp, lane, ws);
    }
  }
}

// Sums the partial slots of each tile in schedule order and writes C (both triangles); with an extra row (tdot != NULL) its products
// with rows 0..M-1 (column M of the result) go to tdot.
__global__ void __launch_bounds__(256)
k_syrk_fixup(int M, const int2* __restrict__ tile_ij, const int* __restrict__ tile_slot_begin, const int* __restrict__ tile_slots,
             const double* __restrict__ ws, double* __restrict__ C, int ldc, double* __restrict__ tdot)
{
  const int t = blockIdx.x;
  const int2 ij = tile_ij[t];
  const int s0 = tile_slot_begin[t], s1 = tile_slot_begin[t + 1];
  const int r0 = blockIdx.y * 16; // 8 row-chunks of 16 rows
  for(int e = threadIdx.x; e < 16 * BM; e += 256) {
    const int r = r0 + e / BM, c = e % BM;
    const int gi = ij.x * BM + r, gj = ij.y * BM + c;
    if(gi >= M || gj > M || (gj == M && !tdot)) continue;
    if(ij.x == ij.y && c < r) continue; // diagonal tile: use the upper part and mirror it (exact symmetry)
    double v = 0.0;
    for(int s = s0; s < s1; s++) v += ws[(size_t)tile_slots[s] * (BM * BM) + r * BM + c];
    if(gj == M) {
      tdot[gi] = v;
      continue;
    }
    C[(size_t)gi * ldc + gj] = v;
    C[(size_t)gj * ldc + gi] = v;
  }
}

struct Schedule
{
  int M = -1;      // (M, K, G): the key this way was built for, M = -1 while it holds none
  long long K = -1;
  int G = 0;       // SM count the schedule was built for
  int Gl = 0;      // CTAs to launch
  long long stamp = 0;
  int ntiles = 0, nslots = 0;
  hb_dev<int> d_cta_seg_begin, d_tile_slot_begin, d_tile_slots;
  hb_dev<int2> d_tile_ij;
  hb_dev<Seg> d_segs;
};
constexpr int SCHED_WAYS = 4;

} // namespace

struct ScheduleCache // per context (c->syrk_sched), small LRU cache keyed by (M, K)
{
  Schedule ways[SCHED_WAYS];
  long long clock = 0;
};
void hb_delete(ScheduleCache* p) { delete p; }

namespace {

constexpr int FRAGS_TILE = 8 * 16; // m16n8 fragments of a full tile per 16 columns of K
// Schedule cost of one K iteration, in full-tile fragments: a tile costs its 128 fragments. A diagonal pair issues 144 (8 * 2 *
// PAIR_CELLS) but runs them more slowly than a tile runs 128: its warps load more shared-memory fragments per MMA (one B fragment per
// 2 or 4 MMAs, against one per 4) and hold 72 accumulators. So a pair is costed at 162 (9/8 of its 144). Measured on an H100 80GB HBM3
// at 700 W (n = 1e6, 1013 rows): with a pair cost of 144 (equal DMMA counts per SM) k_syrk_ws ran only 1.5 % faster than with full
// diagonal tiles; costs of 162 to 176 gave the same, fastest time, 150 and 156 slower ones.
constexpr int COST_TILE = FRAGS_TILE, COST_PAIR = 162;

// The schedule of one (M, K, G), built on the host alone. The work is cut in units: an off-diagonal tile (COST_TILE per K step), a
// pair of diagonal tiles (2p, 2p + 1) (COST_PAIR, see pair_cell_row) and, for odd T, the last diagonal tile alone (the full tile,
// COST_TILE). Units are cut over the CTAs by cost, so that every SM is busy for the same time whatever M is.
struct SchedulePlan
{
  int G = 0;                          // CTAs to launch
  int ntiles = 0;
  std::vector<int2> tij;              // tile t = (tile row, tile column), ti <= tj
  std::vector<Seg> segs;
  std::vector<int> cta_begin;         // the segments of CTA b are segs[cta_begin[b] .. cta_begin[b + 1])
  std::vector<int> slot_tile;         // the tile each workspace slot belongs to
  std::vector<int> tile_slot_begin, tile_slots; // the slots of tile t, in the fixed order k_syrk_fixup sums them
};

void plan_schedule(int M, long long K, int G, SchedulePlan& P)
{
  const int T = (M + BM - 1) / BM;
  const int ntiles = T * (T + 1) / 2;
  const long long kiters = (K + WBK - 1) / WBK;
  auto tile_of = [T](int i, int j) { return i * T - i * (i - 1) / 2 + (j - i); };
  P = SchedulePlan();
  P.ntiles = ntiles;
  P.tij.resize(ntiles);
  for(int i = 0; i < T; i++)
    for(int j = i; j < T; j++) P.tij[tile_of(i, j)] = make_int2(i, j);
  struct Unit
  {
    int ti, tj, cost;
    bool pair;
  };
  std::vector<Unit> units; // in tile-row order: consecutive units of a stream-K range share rows
  for(int i = 0; i < T; i++)
    for(int j = i; j < T; j++) {
      if(i < j) units.push_back({i, j, COST_TILE, false});
      else if(i % 2 == 0) units.push_back(i + 1 < T ? Unit{i, i + 1, COST_PAIR, true} : Unit{i, i, COST_TILE, false});
    }
  const int nu = (int)units.size();
  const long long total = (long long)nu * kiters;
  if(total < G) G = (int)(total > 0 ? total : 1);
  long long work = 0; // cost-iterations
  bool uniform = true;
  for(const Unit& u : units) {
    work += u.cost * kiters;
    uniform = uniform && u.cost == units[0].cost;
  }
  P.G = G;
  P.cta_begin.assign(G + 1, 0);
  auto push = [&](int u, long long k0, long long cnt) {
    const Unit& U = units[u];
    Seg s{U.ti, U.tj, (int)k0, (int)cnt, (int)P.slot_tile.size(), -1};
    P.slot_tile.push_back(tile_of(U.ti, U.pair ? U.ti : U.tj));
    if(U.pair) {
      s.slot_j = (int)P.slot_tile.size();
      P.slot_tile.push_back(tile_of(U.tj, U.tj));
    }
    P.segs.push_back(s);
  };
  // stream-K: CTAs cta0 .. cta0+nct-1 take contiguous ranges of the unit-major space (unit u, k in [kfirst[u], kiters)) holding equal
  // shares of its cost: a CTA runs the iterations whose cost starts in its share.
  auto stream_k = [&](int cta0, int nct, const std::vector<long long>& kfirst) {
    long long tot = 0;
    for(int u = 0; u < nu; u++) tot += units[u].cost * (kiters - kfirst[u]);
    int u = 0;
    long long k = kfirst[0], pos = 0;
    for(int cta = 0; cta < nct; cta++) {
      P.cta_begin[cta0 + cta] = (int)P.segs.size();
      const long long end = hb_part_begin(tot, nct, cta + 1);
      while(pos < end) {
        while(k == kiters) k = kfirst[++u];
        const long long f = units[u].cost;
        const long long cnt = std::min((end - pos + f - 1) / f, kiters - k);
        push(u, k, cnt);
        k += cnt;
        pos += cnt * f;
      }
    }
  };
  // K lanes: when every unit can have a CTA of its own (G >= nu), CTA lane*nu + u runs unit u over the K window of its lane, so the
  // units of a lane read nearly the same columns of [J; S; Y] at the same time and each panel chunk comes from DRAM about once per
  // lane (with stream-K alone the CTAs of the tiles that share a panel sit at unrelated K offsets, and J is re-read from DRAM).
  // - "lanes, R = 0": equal weights (T = 1) and G a multiple of nu: the lanes split K evenly and there is nothing left over.
  // - "lanes, R > 0" and "L = 1": a lane CTA runs about work / G / cost iterations of its unit (a pair's window is 64/81 of a tile's),
  //   and the R = G - L*nu CTAs left over take the rest of every unit stream-K style. With unequal weights and R = 0, the last lane's
  //   CTAs take the rest instead.
  // - "stream-K" (G < nu) and "reduced G" (fewer unit iterations than SMs): stream-K over all of K.
  const int L = G / nu, R = G - L * nu;
  std::vector<long long> kfirst(nu, 0);
  if(L >= 1 && R == 0 && uniform) {
    for(int lane = 0; lane < L; lane++)
      for(int u = 0; u < nu; u++) {
        P.cta_begin[lane * nu + u] = (int)P.segs.size();
        const long long k0 = hb_part_begin(kiters, L, lane), k1 = hb_part_begin(kiters, L, lane + 1);
        push(u, k0, k1 - k0);
      }
  } else {
    const int Ll = R ? L : L - 1, Rr = G - Ll * nu;
    std::vector<long long> w(nu, 0);
    // lane windows of at most t cost-iterations each; returns the work they leave to the Rr other CTAs
    auto windows = [&](long long t) {
      long long rest = work;
      for(int u = 0; u < nu; u++) {
        w[u] = std::min(t / units[u].cost, kiters / Ll);
        rest -= Ll * w[u] * units[u].cost;
      }
      return rest;
    };
    // the least t whose leftover is at most t per other CTA: every CTA then runs between t - COST_PAIR and about t (rounding each lane CTA
    // down to whole iterations with t = work / G would leave the up to G lane CTAs' shortfall to the few others)
    long long lo = 0, hi = work;
    while(Ll >= 1 && lo < hi) {
      const long long mid = lo + (hi - lo) / 2;
      if(windows(mid) <= mid * Rr) hi = mid;
      else lo = mid + 1;
    }
    bool lanes = Ll >= 1;
    if(lanes) windows(lo);
    for(int u = 0; lanes && u < nu; u++) lanes = w[u] >= 1;
    if(lanes) {
      for(int lane = 0; lane < Ll; lane++)
        for(int u = 0; u < nu; u++) {
          P.cta_begin[lane * nu + u] = (int)P.segs.size();
          push(u, lane * w[u], w[u]);
        }
      for(int u = 0; u < nu; u++) kfirst[u] = Ll * w[u];
      stream_k(Ll * nu, G - Ll * nu, kfirst);
    } else {
      stream_k(0, G, kfirst);
    }
  }
  P.cta_begin[G] = (int)P.segs.size();
  P.tile_slot_begin.assign(ntiles + 1, 0);
  for(int t : P.slot_tile) P.tile_slot_begin[t + 1]++;
  for(int t = 0; t < ntiles; t++) P.tile_slot_begin[t + 1] += P.tile_slot_begin[t];
  P.tile_slots.resize(P.slot_tile.size());
  std::vector<int> fill(P.tile_slot_begin.begin(), P.tile_slot_begin.end() - 1);
  for(int s = 0; s < (int)P.slot_tile.size(); s++) P.tile_slots[fill[P.slot_tile[s]]++] = s;
}

int build_schedule(hb_ctx* c, Schedule*& Sout, int M, long long K)
{
  if(!c->syrk_sched) c->syrk_sched.reset(new ScheduleCache);
  ScheduleCache& sc = *c->syrk_sched;
  Schedule* ways = sc.ways;
  int victim = 0;
  for(int w = 0; w < SCHED_WAYS; w++) {
    if(ways[w].M == M && ways[w].K == K && ways[w].G == c->num_sms) {
      ways[w].stamp = ++sc.clock;
      Sout = &ways[w];
      return HB_OK;
    }
    if(ways[w].stamp < ways[victim].stamp) victim = w;
  }
  Schedule& S = ways[victim];
  Sout = &S;
  S.stamp = ++sc.clock;
  S.M = -1;
  HB_CUDA(cudaStreamSynchronize(c->stream));
  SchedulePlan P;
  plan_schedule(M, K, c->num_sms, P);
  const int G = P.G, ntiles = P.ntiles, nslots = (int)P.slot_tile.size();
  if(P.tile_slots.empty()) P.tile_slots.push_back(0);
  if(P.segs.empty()) P.segs.push_back(Seg{0, 0, 0, 0, 0, -1});
  HB_CHECK(S.d_cta_seg_begin.reserve(c, (size_t)G + 1, "SYRK schedule"));
  HB_CHECK(S.d_tile_slot_begin.reserve(c, (size_t)ntiles + 1, "SYRK schedule"));
  HB_CHECK(S.d_tile_slots.reserve(c, P.tile_slots.size(), "SYRK schedule"));
  HB_CHECK(S.d_tile_ij.reserve(c, ntiles, "SYRK schedule"));
  HB_CHECK(S.d_segs.reserve(c, P.segs.size(), "SYRK schedule"));
  HB_CUDA(cudaMemcpy(S.d_cta_seg_begin, P.cta_begin.data(), sizeof(int) * (G + 1), cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(S.d_tile_slot_begin, P.tile_slot_begin.data(), sizeof(int) * (ntiles + 1), cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(S.d_tile_slots, P.tile_slots.data(), sizeof(int) * P.tile_slots.size(), cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(S.d_tile_ij, P.tij.data(), sizeof(int2) * ntiles, cudaMemcpyHostToDevice));
  HB_CUDA(cudaMemcpy(S.d_segs, P.segs.data(), sizeof(Seg) * P.segs.size(), cudaMemcpyHostToDevice));
  S.M = M; S.K = K; S.G = c->num_sms; S.Gl = G; S.ntiles = ntiles; S.nslots = nslots;
  return HB_OK;
}

} // namespace

int hb_syrk_init_attrs(hb_ctx* c)
{
  HB_CUDA(cudaFuncSetAttribute(k_syrk_ws<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WSMEM_BYTES));
  HB_CUDA(cudaFuncSetAttribute(k_syrk_ws<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WSMEM_BYTES));
  return HB_OK;
}

// true when an (M+1)-th row adds no tile row to the SYRK of M rows (hb_syrk_rows' fuse_rx costs no extra MMA)
bool hb_syrk_extra_row_is_free(int M) { return (M + BM) / BM == (M + BM - 1) / BM; }

// rowptr: DEVICE table of M row pointers (each row K doubles, K-contiguous). d: length K (device) or NULL (= ones).
// C: M x M (ldc), both triangles written. `aligned16`: every row pointer is 16-byte aligned; with d, fuse_rx and the table itself
// also 16-byte aligned, k_syrk_ws copies 16 bytes at a time, else 8.
// fuse_rx (optional, device, length K): swept as row M of the same pass; tdot[i] = sum_k row_i[k] d[k] fuse_rx[k] for i < M. It costs
// no extra MMA when M + 1 rows need no more 128-row tiles than M.
int hb_syrk_rows(hb_ctx* c, int M, long long K, const double* const* rowptr_dev, bool aligned16, const double* d, double* C, int ldc,
                 const double* fuse_rx, double* tdot)
{
  HB_REQUIRE(c && M >= 0 && K >= 0 && ldc >= M && (fuse_rx == nullptr) == (tdot == nullptr), "hb_syrk_rows: bad arguments");
  if(M == 0) return HB_OK;
  if(K == 0) {
    HB_CUDA(cudaMemset2DAsync(C, sizeof(double) * ldc, 0, sizeof(double) * M, M, c->stream));
    if(tdot) HB_CUDA(cudaMemsetAsync(tdot, 0, sizeof(double) * M, c->stream));
    return HB_OK;
  }
  const bool align16 = aligned16 && ((reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(fuse_rx) | reinterpret_cast<uintptr_t>(rowptr_dev)) & 15u) == 0;
  Schedule* Sp = nullptr;
  HB_CHECK(build_schedule(c, Sp, M + (fuse_rx ? 1 : 0), K));
  Schedule& S = *Sp;
  HB_CHECK(hb_ws_reserve(c, (size_t)S.nslots * BM * BM * sizeof(double)));
  const int G = S.Gl;
  HB_CHECK(hb_timed_syrk(c, [&] {
    if(align16)
      k_syrk_ws<true><<<G, WTHREADS, WSMEM_BYTES, c->stream>>>(rowptr_dev, M, K, d, fuse_rx, S.d_segs, S.d_cta_seg_begin, (double*)c->ws);
    else
      k_syrk_ws<false><<<G, WTHREADS, WSMEM_BYTES, c->stream>>>(rowptr_dev, M, K, d, fuse_rx, S.d_segs, S.d_cta_seg_begin, (double*)c->ws);
    HB_LAUNCHED();
    return HB_OK;
  }));
  k_syrk_fixup<<<dim3(S.ntiles, BM / 16), 256, 0, c->stream>>>(M, S.d_tile_ij, S.d_tile_slot_begin, S.d_tile_slots, (const double*)c->ws, C, ldc, tdot);
  HB_LAUNCHED();
  return HB_OK;
}

// The schedule hb_syrk_rows would run for M rows (the fused rhs row included) and K columns on G SMs, built on the host: see hiopb200.h.
extern "C" int hb_syrk_schedule_view(int M, long long K, int G, int cap, int* nslots, long long* slots, unsigned char* frags)
{
  HB_REQUIRE(M >= 1 && K >= 1 && G >= 1 && cap >= 0 && nslots && (cap == 0 || (slots && frags)), "hb_syrk_schedule_view: bad arguments");
  SchedulePlan P;
  plan_schedule(M, K, G, P);
  *nslots = (int)P.slot_tile.size();
  for(int b = 0; b < P.G; b++)
    for(int si = P.cta_begin[b]; si < P.cta_begin[b + 1]; si++) {
      const Seg& sg = P.segs[si];
      for(int half = 0; half < (sg.slot_j >= 0 ? 2 : 1); half++) {
        const int s = half ? sg.slot_j : sg.slot;
        if(s >= cap) continue;
        const int2 ij = P.tij[P.slot_tile[s]];
        long long* rec = slots + 5 * (size_t)s;
        rec[0] = b; rec[1] = ij.x; rec[2] = ij.y; rec[3] = sg.k_begin; rec[4] = sg.k_count;
        unsigned char* f = frags + (size_t)FRAGS_TILE * s;
        if(sg.slot_j < 0) {
          std::fill(f, f + FRAGS_TILE, (unsigned char)1);
          continue;
        }
        std::fill(f, f + FRAGS_TILE, (unsigned char)0);
        for(int warp = 4 * half; warp < 4 * half + 4; warp++) // mma_pair_seg: warps 0-3 write slot, 4-7 slot_j
          for(int k = 0; k < PAIR_CELLS; k++) {
            const int r = pair_cell_row(warp & 3, k), c = pair_cell_col(warp & 3, k);
            f[r * 16 + 2 * c]++;
            f[r * 16 + 2 * c + 1]++;
          }
      }
    }
  return HB_OK;
}
