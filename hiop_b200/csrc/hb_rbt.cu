// The random butterfly transform of the safe mode (HB_FACT_RBT_NOPIV), shared by hb_symdense (one GPU), hb_symdense_dist and
// hb_symdense_host: the butterfly diagonals, U^T b and U x on row-major N x nrhs vectors, the rows of b' - A' x' and of |A'|, the
// refined solve, the row-wise transform of the distributed and host-resident handles (k_rbt_mirror, k_rbt_level on a row map: the
// block-cyclic rows of a rank, or the window of a strip), the strips' windows, and the one-pass transform of the one-GPU handle
// (k_rbt_fused). oracle/rbt_model.py states every expression.
//
// k_rbt_fused. A'(i, j) reads B2^T A B2 at rows {i, p1(i)} and columns {j, p1(j)}, which reads A at rows {i, p2(i), p1(i), p2(p1(i))}
// (p1, p2: the level-1 and level-2 partners), and alike for j. Split [0, N) into four quarters Q0 = [0, ha), Q1 = [ha, h), Q2 = [h, h + hb),
// Q3 = [h + hb, N) (h = ceil(N/2), ha = ceil(h/2), hb = ceil((N - h)/2)): level 2 pairs Q0 with Q1 and Q2 with Q3 at the same offset
// ("slot"), and for N != 1 (mod 4) level 1 pairs Q0 with Q2 and Q1 with Q3 at the same slot too. Then the 4-row groups of one slot are
// closed under both pairings, and a tile of RBT_T slots (4 RBT_T rows) needs nothing but itself. A CTA takes the tile pair (bi <= bj):
// it reads the window of A it needs (rows of tile bi x columns of tile bj, upper triangle, each entry from HBM once), forms B2^T A B2
// in shared memory, then A'(i, j) for i in tile bi, j in tile bj, and writes them twice: Ak (i, j) and (j, i), and the upper triangle
// of F once. For N = 1 (mod 4) level 1 pairs Q1 slot t with Q3 slot t + 1 and Q0 slot m with Q3 slot 0 (m = (N - 1) / 4): the window
// grows by one slot on each side and three fixed rows {m, 2m + 1, 3m + 1}, 75 rows instead of 64, so at most (75/64)^2 = 1.37 times
// the reads. The tile schedule is __host__ __device__ code that hb_rbt_schedule_view runs on the host for the tests.
#include "hb_common.cuh"
#include "hb_dense.cuh"
#include <algorithm>

namespace {

constexpr unsigned long long RBT_SEED = 0x5EED2011B7F10001ull, RBT_GOLDEN = 0x9E3779B97F4A7C15ull;

// r_t of butterfly `half` of `level`: 1 + (k - 2^19) / 2^23, k = the top 20 bits of splitmix64 of the counter (stream << 32 | t)
__device__ __forceinline__ double rbt_diag(int level, int half, int t)
{
  unsigned long long z = RBT_SEED + RBT_GOLDEN * ((((unsigned long long)(2 * level + half)) << 32 | (unsigned)t) + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)((1LL << 23) + (long long)(z >> 44) - (1LL << 19)) / (double)(1 << 23);
}

__global__ void k_rbt_table(int N, double* __restrict__ f)
{
  const int h = (N + 1) / 2;
  for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    f[i] = rbt_diag(1, 0, i);
    f[N + i] = i < h ? rbt_diag(2, 0, i) : rbt_diag(2, 1, i - h);
  }
}

__global__ void k_rbt_to_rows(int N, int nrhs, double* __restrict__ x, double* __restrict__ xw, int back)
{
  const long long total = (long long)N * nrhs;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long i = e / nrhs, c = e % nrhs;
    if(back) x[c * N + i] = xw[e];
    else xw[e] = x[c * N + i];
  }
}

// one level on the row-major vectors (N x nrhs): B^T v (trans) or B v
__global__ void k_rbt_vec(int N, int nrhs, int level, const double* __restrict__ f, const double* __restrict__ in, double* __restrict__ out, int trans)
{
  const double* fl = f + (size_t)(level - 1) * N;
  const long long total = (long long)N * nrhs;
  for(long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / nrhs), c = (int)(e % nrhs);
    const rbt_pos p = rbt_at(N, level, i);
    const double vl = in[(size_t)p.lo * nrhs + c], vh = in[(size_t)p.hi * nrhs + c];
    double v;
    if(!p.paired) v = __dmul_rn(fl[i], vl);
    else if(trans) v = __dmul_rn(fl[i], __dmul_rn(__dadd_rn(vl, __dmul_rn(p.s, vh)), HB_RBT_C));
    else v = __dmul_rn(__dadd_rn(__dmul_rn(fl[p.lo], vl), __dmul_rn(p.s, __dmul_rn(fl[p.hi], vh))), HB_RBT_C);
    out[e] = v;
  }
}

// CTA per local row y of A' (full rows): out_y = sum_j |A'(y, j)| (norm) or r_r = b'_r - sum_j A'(r, j) x'_j per rhs, in a fixed order
__global__ void __launch_bounds__(256) k_rbt_rows(int N, int P, int rank, const double* __restrict__ A, long long ld, int nrhs, const double* __restrict__ x,
                                                  const double* __restrict__ b, double* __restrict__ out)
{
  __shared__ double red[8];
  const int r = rbt_global_row(blockIdx.x, P, rank);
  if(r >= N) {
    if(!x && threadIdx.x == 0) out[blockIdx.x] = 0.0;
    return;
  }
  const double* row = A + (size_t)blockIdx.x * ld;
  if(!x) {
    double acc = 0.0;
    for(int j = threadIdx.x; j < N; j += 256) acc += fabs(row[j]);
    acc = hb_block_sum<256>(acc, red);
    if(threadIdx.x == 0) out[blockIdx.x] = acc;
    return;
  }
  for(int c = 0; c < nrhs; c++) {
    double acc = 0.0;
    for(int j = threadIdx.x; j < N; j += 256) acc += row[j] * x[(size_t)j * nrhs + c];
    acc = hb_block_sum<256>(acc, red);
    if(threadIdx.x == 0) out[(size_t)r * nrhs + c] = b[(size_t)r * nrhs + c] - acc;
    __syncthreads();
  }
}

// one CTA per column c: out[c * 3 + k] = max_i |v_k(i, c)| over the N rows of the row-major N x ncols arrays v_0, v_1, v_2 (0 for an
// absent one), NaN kept, in a fixed order
__global__ void __launch_bounds__(256) k_rbt_max(int N, int ncols, const double* __restrict__ v0, const double* __restrict__ v1, const double* __restrict__ v2,
                                                 double* __restrict__ out)
{
  __shared__ double sm[3][256];
  const double* v[3] = {v0, v1, v2};
  const int c = blockIdx.x;
  for(int k = 0; k < 3; k++) {
    double m = 0.0;
    if(v[k])
      for(int i = threadIdx.x; i < N; i += 256) m = hb_nan_max(m, fabs(v[k][(size_t)i * ncols + c]));
    sm[k][threadIdx.x] = m;
  }
  __syncthreads();
  if(threadIdx.x < 3) {
    double m = 0.0;
    for(int t = 0; t < 256; t++) m = hb_nan_max(m, sm[threadIdx.x][t]);
    out[(size_t)c * 3 + threadIdx.x] = m;
  }
}

// ---- the row-wise transform of the distributed and host-resident handles: the mirror, then one pass per level ----------------------
constexpr int RBT_COLS = 1024; // columns per CTA of k_rbt_level (256 threads x 4)

// mirror: every held row r gets dst(y, j) = src(j, r) for the columns q0 <= j < q0 + nq, j < r, where src holds the rows q0 .. of the
// upper triangle (ld doubles each). 32 x 32 tiles through shared memory: local rows y0 .., starting at local row ybeg.
__global__ void __launch_bounds__(256) k_rbt_mirror(int N, hb_rbt_rowmap m, int nrows, int ybeg, const double* __restrict__ src, long long ld, int q0,
                                                    int nq, double* __restrict__ dst)
{
  __shared__ double tile[32][33];
  const int y0 = ybeg + blockIdx.y * 32, j0 = q0 + blockIdx.x * 32, tx = threadIdx.x % 32, ty = threadIdx.x / 32;
  for(int jj = ty; jj < 32; jj += 8) {
    const int y = y0 + tx, j = j0 + jj;
    const int r = y < nrows ? m.global(y) : N;
    tile[jj][tx] = (r < N && j < q0 + nq && j < r) ? src[(size_t)(j - q0) * ld + r] : 0.0;
  }
  __syncthreads();
  for(int yy = ty; yy < 32; yy += 8) {
    const int y = y0 + yy, j = j0 + tx;
    const int r = y < nrows ? m.global(y) : N;
    if(r < N && j < q0 + nq && j < r) dst[(size_t)y * ld + j] = tile[tx][yy];
  }
}

// one level B^T A B on full rows. CTA x = a source row q: local row x of `in` (src == nullptr: every partner is held) or row x of src
// (global rows q0 .. q0 + nq, the owner's broadcast). Its partner r (q itself when unpaired), when held, gets its whole output row from
// rows r and q: out(r, j) = (f_r f_j) (t w) with t and w of oracle/rbt_model.py, in that operation order.
__global__ void __launch_bounds__(256) k_rbt_level(int N, int level, const double* __restrict__ f, const double* __restrict__ in, long long ld,
                                                   hb_rbt_rowmap m, const double* __restrict__ src, int q0, double* __restrict__ out)
{
  const int q = src ? q0 + blockIdx.x : m.global(blockIdx.x);
  if(q < 0 || q >= N) return;
  const double* rowq = src ? src + (size_t)blockIdx.x * ld : in + (size_t)blockIdx.x * ld;
  const rbt_pos pq = rbt_at(N, level, q);
  const int r = pq.lo == q ? pq.hi : pq.lo;
  const int lr = m.local(r);
  if(lr < 0) return;
  const double* rowr = in + (size_t)lr * ld;
  const rbt_pos pr = rbt_at(N, level, r);
  const double* RL = pr.lo == r ? rowr : rowq;
  const double* RH = pr.hi == r ? rowr : rowq;
  const double* fl = f + (size_t)(level - 1) * N;
  const double fi = fl[r];
  double* o = out + (size_t)lr * ld;
  const int jend = min(N, (int)(blockIdx.y + 1) * RBT_COLS);
  for(int j = blockIdx.y * RBT_COLS + threadIdx.x; j < jend; j += 256) {
    const rbt_pos pj = rbt_at(N, level, j);
    o[j] = rbt_entry(RL[pj.lo], RH[pj.hi], RL[pj.hi], RH[pj.lo], pr, pj, fi, fl[j]);
  }
}

// ---- the one-pass transform of the one-GPU handle ----------------------------------------------------------------------------------
constexpr int RBT_T = 16;                        // slots per tile: 4 RBT_T output rows
constexpr int RBT_OR = 4 * RBT_T;                // output rows of a tile
constexpr int RBT_WMAX = 4 * (RBT_T + 2) + 3;    // window rows of a tile, N = 1 (mod 4)
constexpr int RBT_SLD = RBT_WMAX + 1;            // shared-memory stride of the window

struct rbt_quarters
{
  int N, s[4], len[4], nt, W, ext, wr, sp[3];
  bool closed;
};

__host__ __device__ inline rbt_quarters rbt_quarters_of(int N)
{
  rbt_quarters q;
  const int h = (N + 1) / 2, m1 = N - h, ha = (h + 1) / 2, hb = (m1 + 1) / 2;
  q.N = N;
  q.s[0] = 0; q.s[1] = ha; q.s[2] = h; q.s[3] = h + hb;
  q.len[0] = ha; q.len[1] = h - ha; q.len[2] = hb; q.len[3] = m1 - hb;
  q.nt = (ha + RBT_T - 1) / RBT_T;
  q.closed = (N & 3) != 1;
  q.ext = q.closed ? 0 : 1;
  q.W = RBT_T + 2 * q.ext;
  q.wr = 4 * q.W + (q.closed ? 0 : 3);
  const int m = (N - 1) / 4;
  q.sp[0] = q.closed ? -1 : m;
  q.sp[1] = q.closed || 2 * m + 1 >= N ? -1 : 2 * m + 1;
  q.sp[2] = q.closed || 3 * m + 1 >= N ? -1 : 3 * m + 1;
  return q;
}

// the tile pair (bi <= bj) of CTA b, in the order (0,0), (0,1), (1,1), (0,2), ...
__host__ __device__ inline void rbt_cta_tiles(int b, int& bi, int& bj)
{
  int j = (int)((sqrt(8.0 * b + 1.0) - 1.0) * 0.5);
  while(j * (j + 1) / 2 > b) j--;
  while((j + 1) * (j + 2) / 2 <= b) j++;
  bj = j;
  bi = b - j * (j + 1) / 2;
}

// output row k (0 .. RBT_OR-1) of tile b: quarter k / RBT_T, slot b RBT_T + k % RBT_T; -1 past the quarter
__host__ __device__ inline int rbt_out_row(const rbt_quarters& q, int b, int k)
{
  const int a = k / RBT_T, slot = b * RBT_T + k % RBT_T;
  return slot < q.len[a] ? q.s[a] + slot : -1;
}

// window row k (0 .. q.wr-1) of the tile or strip whose first slot is `first`: the slots first - ext .. first + q.W - ext - 1 of each
// quarter, then the three fixed rows of N = 1 (mod 4); -1 where there is none
__host__ __device__ inline int rbt_window_row(const rbt_quarters& q, int first, int k)
{
  if(k < 4 * q.W) {
    const int a = k / q.W, slot = first - q.ext + k % q.W;
    return slot >= 0 && slot < q.len[a] ? q.s[a] + slot : -1;
  }
  k -= 4 * q.W;
  return k < 3 ? q.sp[k] : -1;
}

// the first window position of the tile or strip starting at slot `first` that holds row g, -1 if none
__host__ __device__ inline int rbt_window_pos(const rbt_quarters& q, int first, int g)
{
  const int a = g >= q.s[3] ? 3 : g >= q.s[2] ? 2 : g >= q.s[1] ? 1 : 0;
  const int w = g - q.s[a] - (first - q.ext);
  if(w >= 0 && w < q.W) return a * q.W + w;
  for(int e = 0; e < 3; e++)
    if(q.sp[e] == g) return 4 * q.W + e;
  return -1;
}

// the row the kernel reads into window position k: rbt_window_row unless an earlier position holds it already (-1)
__host__ __device__ inline int rbt_window_held(const rbt_quarters& q, int first, int k)
{
  const int g = k < q.wr ? rbt_window_row(q, first, k) : -1;
  return g >= 0 && rbt_window_pos(q, first, g) == k ? g : -1;
}

__global__ void __launch_bounds__(256) k_rbt_fused(int N, const double* __restrict__ f, const double* A, long long lda, double* F, long long ldf,
                                                   double* __restrict__ Ak, long long ldk, double* __restrict__ part)
{
  __shared__ double S[RBT_WMAX * RBT_SLD];
  __shared__ int rw[RBT_WMAX], cw[RBT_WMAX];
  __shared__ double red[RBT_OR][2];
  __shared__ rbt_quarters q; // in shared memory: the schedule functions index its arrays
  if(threadIdx.x == 0) q = rbt_quarters_of(N);
  __syncthreads();
  int bi, bj;
  rbt_cta_tiles(blockIdx.x, bi, bj);
  const int wr = q.wr, tid = threadIdx.x;
  const bool diag = bi == bj;
  for(int k = tid; k < wr; k += 256) {
    rw[k] = rbt_window_held(q, bi * RBT_T, k);
    cw[k] = rbt_window_held(q, bj * RBT_T, k);
  }
  __syncthreads();
  // the window of A from its upper triangle: entries on or above the diagonal along rows, the others along columns (coalesced both)
  for(int e = tid; e < wr * wr; e += 256) {
    const int k = e / wr, l = e % wr, r = rw[k], c = cw[l];
    if(r >= 0 && c >= 0 && r <= c) S[k * RBT_SLD + l] = A[(size_t)r * lda + c];
  }
  if(!diag)
    for(int e = tid; e < wr * wr; e += 256) {
      const int l = e / wr, k = e % wr, r = rw[k], c = cw[l];
      if(r >= 0 && c >= 0 && r > c) S[k * RBT_SLD + l] = A[(size_t)c * lda + r];
    }
  __syncthreads();
  if(diag) { // same rows and columns: the lower entries from the upper ones already read
    for(int e = tid; e < wr * wr; e += 256) {
      const int k = e / wr, l = e % wr, r = rw[k], c = cw[l];
      if(r >= 0 && c >= 0 && r > c) S[k * RBT_SLD + l] = S[l * RBT_SLD + k];
    }
    __syncthreads();
  }
  // B2^T A B2 in place: the lo corner of every 2 x 2 block of partners computes the block
  const double* f2 = f + N;
  for(int e = tid; e < wr * wr; e += 256) {
    const int k = e / wr, l = e % wr, r = rw[k], c = cw[l];
    if(r < 0 || c < 0) continue;
    const rbt_pos pr = rbt_at(N, 2, r), pc = rbt_at(N, 2, c);
    if(pr.lo != r || pc.lo != c) continue;
    const int k2 = pr.paired ? rbt_window_pos(q, bi * RBT_T, pr.hi) : k, l2 = pc.paired ? rbt_window_pos(q, bj * RBT_T, pc.hi) : l;
    if(k2 < 0 || l2 < 0) continue;
    const double all = S[k * RBT_SLD + l], ahh = S[k2 * RBT_SLD + l2], alh = S[k * RBT_SLD + l2], ahl = S[k2 * RBT_SLD + l];
    const rbt_pos ph = rbt_at(N, 2, pr.hi), qh = rbt_at(N, 2, pc.hi);
    S[k * RBT_SLD + l] = rbt_entry(all, ahh, alh, ahl, pr, pc, f2[r], f2[c]);
    if(pc.paired) S[k * RBT_SLD + l2] = rbt_entry(all, ahh, alh, ahl, pr, qh, f2[r], f2[pc.hi]);
    if(pr.paired) S[k2 * RBT_SLD + l] = rbt_entry(all, ahh, alh, ahl, ph, pc, f2[pr.hi], f2[c]);
    if(pr.paired && pc.paired) S[k2 * RBT_SLD + l2] = rbt_entry(all, ahh, alh, ahl, ph, qh, f2[pr.hi], f2[pc.hi]);
  }
  __syncthreads();
  // B1^T (.) B1 for the output rows of tile bi x those of tile bj; pass 0 writes rows i along j, pass 1 (bi < bj) rows j along i.
  // Row sums of |A'| over the tile into part[(other tile) * N + row], each in a fixed order.
  const int tx = tid & (RBT_OR - 1), ty = tid / RBT_OR, lane = tid & 31;
  for(int pass = 0; pass < (diag ? 1 : 2); pass++) {
    const int bo = pass ? bj : bi, bx = pass ? bi : bj; // rows of the pass from tile bo, along tile bx
    const int x = rbt_out_row(q, bx, tx);
    rbt_pos px{};
    int x1 = -1, x2 = -1;
    if(x >= 0) {
      px = rbt_at(N, 1, x);
      x1 = rbt_window_pos(q, bx * RBT_T, px.lo);
      x2 = rbt_window_pos(q, bx * RBT_T, px.hi);
    }
    for(int ro = ty; ro < RBT_OR; ro += 256 / RBT_OR) {
      const int y = rbt_out_row(q, bo, ro);
      double v = 0.0;
      if(x >= 0 && y >= 0) {
        const rbt_pos py = rbt_at(N, 1, y);
        const int y1 = rbt_window_pos(q, bo * RBT_T, py.lo), y2 = rbt_window_pos(q, bo * RBT_T, py.hi);
        // S is indexed [row of tile bi][column of tile bj]
        const int i = pass ? x : y, j = pass ? y : x;
        const int k1 = pass ? x1 : y1, k2 = pass ? x2 : y2, l1 = pass ? y1 : x1, l2 = pass ? y2 : x2;
        const rbt_pos pi = pass ? px : py;
        const rbt_pos pj = pass ? py : px;
        if(k1 >= 0 && k2 >= 0 && l1 >= 0 && l2 >= 0) {
          v = rbt_entry(S[k1 * RBT_SLD + l1], S[k2 * RBT_SLD + l2], S[k1 * RBT_SLD + l2], S[k2 * RBT_SLD + l1], pi, pj, f[i], f[j]);
          Ak[(size_t)y * ldk + x] = v;
          if(F && y <= x) F[(size_t)y * ldf + x] = v;
        }
      }
      double a = fabs(v);
#pragma unroll
      for(int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if(lane == 0) red[ro][(tid >> 5) & 1] = a;
    }
    __syncthreads();
    if(tid < RBT_OR) {
      const int y = rbt_out_row(q, bo, tid);
      if(y >= 0) part[(size_t)bx * N + y] = red[tid][0] + red[tid][1];
    }
    __syncthreads();
  }
}

// rows[r] = sum over the column tiles c (in order) of part[c * N + r]
__global__ void k_rbt_rowsum(int N, int nt, const double* __restrict__ part, double* __restrict__ rows)
{
  for(int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
    double acc = 0.0;
    for(int c = 0; c < nt; c++) acc += part[(size_t)c * N + r];
    rows[r] = acc;
  }
}

// the quarters of order N with the window of a strip of `slots` slots per quarter (k_rbt_fused's layout with RBT_T -> slots)
__host__ __device__ inline rbt_quarters rbt_strip_quarters(int N, int slots)
{
  rbt_quarters q = rbt_quarters_of(N);
  q.W = slots + 2 * q.ext;
  q.wr = 4 * q.W + (q.closed ? 0 : 3);
  return q;
}

__global__ void k_rbt_window_map(rbt_quarters q, int s0, int s1, int* __restrict__ rows, int* __restrict__ pos_win, int* __restrict__ pos_out)
{
  const int n = q.N > q.wr ? q.N : q.wr;
  for(int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    if(e < q.wr) rows[e] = rbt_window_held(q, s0, e);
    if(e < q.N) {
      const int w = rbt_window_pos(q, s0, e), a = e >= q.s[3] ? 3 : e >= q.s[2] ? 2 : e >= q.s[1] ? 1 : 0, slot = e - q.s[a];
      pos_win[e] = w;
      pos_out[e] = slot >= s0 && slot < s1 ? w : -1;
    }
  }
}

} // namespace

int hb_rbt_mirror(hb_ctx* c, int N, hb_rbt_rowmap m, int nrows, int ybeg, const double* src, long long ld, int q0, int nq, double* dst)
{
  if(nrows <= ybeg || nq <= 0) return HB_OK;
  k_rbt_mirror<<<dim3((nq + 31) / 32, (nrows - ybeg + 31) / 32), 256, 0, c->stream>>>(N, m, nrows, ybeg, src, ld, q0, nq, dst);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_level(hb_ctx* c, int N, int level, const double* f, const double* in, long long ld, hb_rbt_rowmap m, int nsrc, const double* src, int q0,
                 double* out)
{
  if(nsrc <= 0) return HB_OK;
  k_rbt_level<<<dim3(nsrc, (N + RBT_COLS - 1) / RBT_COLS), 256, 0, c->stream>>>(N, level, f, in, ld, m, src, q0, out);
  HB_LAUNCHED();
  return HB_OK;
}

hb_rbt_window hb_rbt_window_of(int N, int s0, int s1)
{
  const rbt_quarters q = rbt_strip_quarters(N, s1 - s0);
  hb_rbt_window w{};
  w.N = N; w.slots = q.len[0]; w.s0 = s0; w.s1 = s1; w.W = q.W; w.wr = q.wr; w.ext = q.ext;
  for(int a = 0; a < 4; a++) { w.qs[a] = q.s[a]; w.qlen[a] = q.len[a]; }
  for(int e = 0; e < 3; e++) w.sp[e] = q.sp[e];
  return w;
}

int hb_rbt_window_map(hb_ctx* c, const hb_rbt_window& w, int* rows, int* pos_win, int* pos_out)
{
  const rbt_quarters q = rbt_strip_quarters(w.N, w.s1 - w.s0);
  k_rbt_window_map<<<hb_grid(c, w.N > w.wr ? w.N : w.wr), 256, 0, c->stream>>>(q, w.s0, w.s1, rows, pos_win, pos_out);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_window_row(const hb_rbt_window& w, int k) { return rbt_window_held(rbt_strip_quarters(w.N, w.s1 - w.s0), w.s0, k); }

bool hb_rbt_window_out(const hb_rbt_window& w, int g)
{
  const int a = g >= w.qs[3] ? 3 : g >= w.qs[2] ? 2 : g >= w.qs[1] ? 1 : 0, slot = g - w.qs[a];
  return slot >= w.s0 && slot < w.s1;
}

int hb_rbt_table(hb_ctx* c, int N, double* f)
{
  if(N == 0) return HB_OK;
  k_rbt_table<<<hb_grid(c, N), 256, 0, c->stream>>>(N, f);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_to_rows(hb_ctx* c, int N, int nrhs, double* x, double* xw, bool back)
{
  k_rbt_to_rows<<<hb_grid(c, (long long)N * nrhs), 256, 0, c->stream>>>(N, nrhs, x, xw, back ? 1 : 0);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_rows(hb_ctx* c, int N, int P, int rank, int nrows, const double* A, long long ld, int nrhs, const double* x, const double* b, double* out)
{
  if(nrows <= 0) return HB_OK;
  k_rbt_rows<<<nrows, 256, 0, c->stream>>>(N, P, rank, A, ld, nrhs, x, b, out);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_max1(hb_ctx* c, int n, const double* v, double* out)
{
  k_rbt_max<<<1, 256, 0, c->stream>>>(n, 1, v, nullptr, nullptr, out);
  HB_LAUNCHED();
  return HB_OK;
}

int hb_rbt_solve(hb_ctx* c, int N, int nrhs, const double* f, double anorm, double* xw, double* bp, double* rw, double* nrm_host,
                 const std::function<int(double*)>& sweeps, const std::function<int(const double*, const double*, double*)>& residual, int* corr_out,
                 double* berr_out, hb_rbt_trace* trace)
{
  cudaStream_t st = c->stream;
  const int tg = hb_grid(c, (long long)N * nrhs);
  const size_t n = (size_t)N * nrhs;
  double* nrm = rw + n; // per rhs: max |r|, max |x'|, max |b'|
  auto to_trace = [&](std::vector<double>& v, const double* d, size_t count) -> int {
    const size_t at = v.size();
    v.resize(at + count);
    HB_CUDA(cudaMemcpyAsync(v.data() + at, d, sizeof(double) * count, cudaMemcpyDeviceToHost, st));
    HB_CUDA(cudaStreamSynchronize(st));
    return HB_OK;
  };
  k_rbt_vec<<<tg, 256, 0, st>>>(N, nrhs, 2, f, xw, rw, 1);
  HB_LAUNCHED();
  k_rbt_vec<<<tg, 256, 0, st>>>(N, nrhs, 1, f, rw, bp, 1);
  HB_LAUNCHED();
  HB_CUDA(cudaMemcpyAsync(xw, bp, sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
  HB_CHECK(sweeps(xw));
  if(trace) {
    *trace = hb_rbt_trace{};
    trace->anorm = anorm;
    HB_CHECK(to_trace(trace->b, bp, n));
  }
  double om = 0.0, prev = INFINITY;
  int corr = 0;
  for(;;) {
    if(trace) HB_CHECK(to_trace(trace->x, xw, n));
    HB_CHECK(residual(xw, bp, rw));
    k_rbt_max<<<nrhs, 256, 0, st>>>(N, nrhs, rw, xw, bp, nrm);
    HB_LAUNCHED();
    HB_CUDA(cudaMemcpyAsync(nrm_host, nrm, sizeof(double) * 3 * nrhs, cudaMemcpyDeviceToHost, st));
    HB_CUDA(cudaStreamSynchronize(st));
    om = 0.0;
    for(int q = 0; q < nrhs; q++) {
      const double* m3 = nrm_host + 3 * q;
      const double den = anorm * m3[1] + m3[2];
      double w;
      if(!std::isfinite(m3[0]) || !std::isfinite(m3[1]) || !std::isfinite(m3[2]) || !std::isfinite(anorm)) w = NAN;
      else w = den > 0.0 ? m3[0] / den : (m3[0] == 0.0 ? 0.0 : INFINITY);
      om = (w > om || w != w) ? w : om;
    }
    if(trace) {
      trace->norms.insert(trace->norms.end(), nrm_host, nrm_host + 3 * nrhs);
      trace->norms.push_back(om);
    }
    if(!(std::isfinite(om) && corr < HB_RBT_MAX_CORR && om > HB_RBT_EPS && om <= 0.5 * prev)) break;
    HB_CHECK(sweeps(rw));
    HB_CHECK(hb_vec_axpy(c, (long long)N * nrhs, xw, 1.0, rw));
    corr++;
    prev = om;
  }
  *corr_out = corr;
  *berr_out = om;
  k_rbt_vec<<<tg, 256, 0, st>>>(N, nrhs, 1, f, xw, rw, 0);
  HB_LAUNCHED();
  k_rbt_vec<<<tg, 256, 0, st>>>(N, nrhs, 2, f, rw, xw, 0);
  HB_LAUNCHED();
  return std::isfinite(om) ? 1 : 0;
}

int hb_rbt_traced_solve(const hb_dense_result& r, const char* who, const std::function<int(hb_rbt_trace*)>& solve, int* ret_host, int* passes,
                        double* anorm, double* norms, double* xp, double* bp)
{
  if(!r.factored || r.mode != HB_FACT_RBT_NOPIV) return hb_fail(HB_ERR_STATE, "%s: no valid RBT factorization", who);
  hb_rbt_trace t;
  const int ok = solve(&t);
  if(ok < 0) return ok;
  if(ret_host) *ret_host = ok;
  if(passes) *passes = (int)(t.b.empty() ? 0 : t.x.size() / t.b.size());
  if(anorm) *anorm = t.anorm;
  if(norms) std::copy(t.norms.begin(), t.norms.end(), norms);
  if(xp) std::copy(t.x.begin(), t.x.end(), xp);
  if(bp) std::copy(t.b.begin(), t.b.end(), bp);
  return HB_OK;
}

bool hb_rbt_in_place(int N) { return rbt_quarters_of(N).closed; }

size_t hb_rbt_part_doubles(int N) { return (size_t)(rbt_quarters_of(N).nt + 1) * N; }

int hb_rbt_fused(hb_ctx* c, int N, const double* f, const double* A, long long lda, double* F, long long ldf, double* Ak, long long ldk, double* part,
                 double* nrm_dev)
{
  if(N == 0) return HB_OK;
  const rbt_quarters q = rbt_quarters_of(N);
  HB_REQUIRE(F != A || q.closed, "hb_rbt_fused: in place only when the slot groups are closed (N != 1 mod 4)");
  k_rbt_fused<<<q.nt * (q.nt + 1) / 2, 256, 0, c->stream>>>(N, f, A, lda, F, ldf, Ak, ldk, part);
  HB_LAUNCHED();
  double* rows = part + (size_t)q.nt * N;
  k_rbt_rowsum<<<hb_grid(c, N), 256, 0, c->stream>>>(N, q.nt, part, rows);
  HB_LAUNCHED();
  return hb_rbt_max1(c, N, rows, nrm_dev);
}

// The tile schedule of k_rbt_fused for order N, run on the host: see hiopb200.h.
extern "C" int hb_rbt_schedule_view(int N, int cap, int* dims4, int* ctas_host, int* window_host, int* out_host)
{
  HB_REQUIRE(N >= 1 && cap >= 0 && dims4 && (cap == 0 || (ctas_host && window_host && out_host)), "hb_rbt_schedule_view: bad arguments");
  const rbt_quarters q = rbt_quarters_of(N);
  const int nctas = q.nt * (q.nt + 1) / 2;
  dims4[0] = q.nt; dims4[1] = nctas; dims4[2] = RBT_WMAX; dims4[3] = RBT_OR;
  for(int b = 0; b < nctas && b < cap; b++) rbt_cta_tiles(b, ctas_host[2 * b], ctas_host[2 * b + 1]);
  for(int t = 0; t < q.nt && t < cap; t++) {
    for(int k = 0; k < RBT_WMAX; k++) window_host[(size_t)t * RBT_WMAX + k] = rbt_window_held(q, t * RBT_T, k);
    for(int k = 0; k < RBT_OR; k++) out_host[(size_t)t * RBT_OR + k] = rbt_out_row(q, t, k);
  }
  return HB_OK;
}

// One strip of the out-of-core transform of order N, run on the host: see hiopb200.h.
extern "C" int hb_rbt_strip_view(int N, int s0, int s1, int* wr_host, int* window_host, int* out_host)
{
  HB_REQUIRE(N >= 1 && s0 >= 0 && s1 > s0 && wr_host, "hb_rbt_strip_view: bad arguments");
  const hb_rbt_window w = hb_rbt_window_of(N, s0, s1);
  HB_REQUIRE(s1 <= w.slots, "hb_rbt_strip_view: the strip ends past the last slot");
  *wr_host = w.wr;
  if(window_host)
    for(int k = 0; k < w.wr; k++) window_host[k] = hb_rbt_window_row(w, k);
  if(out_host)
    for(int a = 0; a < 4; a++)
      for(int t = s0; t < s1; t++) out_host[a * (s1 - s0) + t - s0] = t < w.qlen[a] ? w.qs[a] + t : -1;
  return HB_OK;
}
