"""CPU model of the int8-slice (Ozaki-scheme) condensation of hiop_b200/csrc/hb_ozaki.cu -- TEST INFRASTRUCTURE ONLY.

Restates what the device path does, bit for bit, so that its output can be predicted exactly and its exactness claims checked without
a GPU:
- row exponents from the exact row maximum (k_oz_rowmax / k_oz_rowmax_dot / k_oz_exponents);
- digits from two magic-number roundings and balanced base-128 extraction (k_oz_slice);
- the host schedule of hb_syrk_rows_ozaki: tiles, K splits (with its multi-wave split search) and K chunks (schedule);
- exact integer anti-diagonal sums T_t = sum_{p+q=t} Q_p Q_q^T per K chunk, recombined in FP64 in the kernel's order: t = S-1 .. 0
  inside a chunk (k_oz_gemm's epilogue), the chunks of a split in K order, the splits in order, then 2^{e_i + e_j} (k_oz_fixup)
  (condense_bits);
- an a-priori bound on the result's distance from the exact B B^T (truncation_bound).

The integer sums are formed with FP64 GEMMs: every partial sum is an integer below 2^31, so any summation order is exact. They run in
numpy, or in torch on a device for the large shapes. The model is not used by the product."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

MAGIC = 6755399441055744.0  # 1.5 * 2^52
TM, TN, KS = 128, 32, 128   # k_oz_gemm's output tile (rows x columns) and K stage (columns)
U = 2.0 ** -53


def row_exponents(B: np.ndarray) -> np.ndarray:
    """e_i with max_k |b_ik| = f * 2^e_i, f in [0.5, 1) (frexp); 0 for an all-zero row."""
    mx = np.abs(B).max(axis=1, initial=0.0)
    e = np.zeros(B.shape[0], dtype=np.int64)
    nz = mx > 0
    e[nz] = np.frexp(mx[nz])[1]
    return e


def _digits(v: np.ndarray, nd: int) -> list[np.ndarray]:
    """Balanced base-128 digits of the integers v, least significant extracted first, leading digit = what is left."""
    v = v.astype(np.int64)
    d = [None] * nd
    for j in range(nd - 1, 0, -1):
        d[j] = ((v + 64) & 127) - 64
        v = (v - d[j]) >> 7
    d[0] = v
    return d


def slices(B: np.ndarray, e: np.ndarray, S: int, rows_per_block: int = 64) -> np.ndarray:
    """Q[p] (int8): sum_p Q[p] 2^-(6+7p) = B / 2^e rounded to the last slice's grid. Rows are done in blocks to bound the memory of the
    FP64 temporaries at large K."""
    assert 5 <= S <= 8
    nlo = S - 4
    M, K = B.shape
    Q = np.empty((S, M, K), dtype=np.int8)
    for r0 in range(0, M, rows_per_block):
        r1 = min(r0 + rows_per_block, M)
        xs = np.ldexp(B[r0:r1], (27 - e[r0:r1])[:, None])   # exact, |xs| < 2^27 (also for rows below 2^-997)
        t = xs + MAGIC
        hi = t - MAGIC                                        # rint(xs), exact
        rem = xs - hi                                         # exact, |rem| <= 0.5
        lo = (rem * float(1 << (7 * nlo)) + MAGIC) - MAGIC
        for p, d in enumerate(_digits(hi.astype(np.int64), 4) + _digits(lo.astype(np.int64), nlo)):
            Q[p, r0:r1] = d
    return Q


def digits(B: np.ndarray, S: int):
    """(e, Q): the row exponents and int8 slices k_oz_slice produces from B = A diag(sqrt(d))."""
    e = row_exponents(B)
    return e, slices(B, e, S)


# ---- the host schedule of hb_syrk_rows_ozaki ------------------------------------------------------------------------------------

def chunk_stages(S: int) -> int:
    """K stages per chunk: (t+1) * Kc * 2^12 < 2^31 for every t <= S-1, strictly (S = 8: 511 stages, not 512)."""
    cs = (524288 // S) // KS
    while S * cs * KS * 4096 >= 2 ** 31:
        cs -= 1
    return cs


def part_begin(total: int, parts: int, p: int) -> int:
    """hb_part_begin (hb_common.cuh): start of part p when total items are cut into parts as even as possible."""
    return (total // parts) * p + min(p, total % parts)


BRANCHES = ("splits = G // tiles", "splits clamped to kstages", "search picks sp > 1", "search keeps 1",
            "one split, several chunks", "several splits, several chunks")


@dataclass
class Schedule:
    M: int
    K: int
    S: int
    num_sms: int
    Mpad: int
    Kpad: int
    kstages: int
    tiles: list
    splits: int
    items: list              # (bi, bj, k_begin, k_count, slot), split-major
    chunk_stages: int
    clamped: bool            # G // tiles exceeded the K stages
    searched: bool           # the one-wave split count filled less than 70 % of the machine: the multi-wave search ran
    branch: str = field(default="")

    def split_chunks(self):
        """Per split (in order), its K chunks (in order) as column ranges [c0, c1) of the unpadded K."""
        out = []
        for s in range(self.splits):
            b, e = part_begin(self.kstages, self.splits, s), part_begin(self.kstages, self.splits, s + 1)
            out.append([(c * KS, min(min(c + self.chunk_stages, e) * KS, self.K)) for c in range(b, e, self.chunk_stages)])
        return out

    @property
    def max_chunks(self) -> int:
        return max(len(c) for c in self.split_chunks())

    @property
    def chain(self) -> int:
        """Longest chain of FP64 additions behind one entry: S terms in the epilogue, the later chunks of a split, the splits."""
        return self.S + self.max_chunks - 1 + self.splits


def schedule(M: int, K: int, S: int, num_sms: int, max_splits: int = 16) -> Schedule:
    """hb_syrk_rows_ozaki's work list, restated (max_splits: HB_OZ_MAX_SPLITS)."""
    assert M >= 1 and K >= 1
    G = num_sms
    Mpad = -(-M // TM) * TM
    Kpad = -(-K // KS) * KS
    nbi, nbj = Mpad // TM, Mpad // TN
    tiles = [(bi, bj) for bi in range(nbi) for bj in range((TM // TN) * bi, nbj) if bj * TN < M]
    nt = len(tiles)
    kstages = Kpad // KS
    splits = max(G // max(nt, 1), 1)
    clamped = splits > kstages
    if clamped:
        splits = kstages if kstages > 0 else 1
    items0 = nt * splits
    waves0 = -(-items0 // G)
    util0 = items0 / (waves0 * G) if nt > 0 else 1.0
    searched = util0 < 0.7
    if searched:
        best = waves0 / splits
        for sp in range(1, max_splits + 1):
            if sp > 1 and (kstages // sp < 64 or nt * sp * TM * TN * 8 > (1 << 30)):
                break
            cost = (-(-(nt * sp) // G)) / sp
            if cost < best * (1.0 - 1e-3):
                best, splits = cost, sp
    if splits > kstages:
        splits = kstages if kstages > 0 else 1
    items = []
    for s in range(splits):
        b, e = part_begin(kstages, splits, s), part_begin(kstages, splits, s + 1)
        for t, (bi, bj) in enumerate(tiles):
            items.append((bi, bj, b, e - b, t * splits + s))
    sch = Schedule(M=M, K=K, S=S, num_sms=G, Mpad=Mpad, Kpad=Kpad, kstages=kstages, tiles=tiles, splits=splits, items=items,
                   chunk_stages=chunk_stages(S), clamped=clamped, searched=searched)
    if clamped:
        sch.branch = "splits clamped to kstages"
    elif searched:
        sch.branch = "search picks sp > 1" if splits > 1 else "search keeps 1"
    elif sch.max_chunks > 1:
        sch.branch = "several splits, several chunks" if splits > 1 else "one split, several chunks"
    else:
        sch.branch = "splits = G // tiles"
    return sch


# (branch, preferred M, K, S): on 132 SMs every preferred M lands in its branch; find_shape moves M on other SM counts
BRANCH_CASES = [
    ("splits = G // tiles", 100, 20000, 8), ("splits = G // tiles", 100, 20000, 6), ("splits = G // tiles", 300, 60001, 7),
    ("splits clamped to kstages", 100, 1000, 8), ("splits clamped to kstages", 1, 5000, 7),
    ("search picks sp > 1", 1000, 200001, 8), ("search picks sp > 1", 1000, 20000, 6),
    ("search keeps 1", 1000, 12000, 8),
    ("one split, several chunks", 1260, 140001, 8), ("one split, several chunks", 1260, 140001, 6),
    ("several splits, several chunks", 300, 470001, 8),
]


def find_shape(branch: str, M0: int, K: int, S: int, num_sms: int, max_splits: int = 16) -> int:
    """The M nearest M0 (ties to the smaller) whose schedule on num_sms SMs is `branch`."""
    for M in sorted(range(1, 2049), key=lambda m: (abs(m - M0), m)):
        if schedule(M, K, S, num_sms, max_splits).branch == branch:
            return M
    raise AssertionError(f"no M puts K = {K}, S = {S} in the branch '{branch}' on {num_sms} SMs")


# ---- the exact integer sums and the FP64 recombination --------------------------------------------------------------------------

def _pair_products(Qc: np.ndarray, pairs, device=None) -> dict:
    """{(p, q): Q_p Q_q^T} over the columns of Qc (S x M x k, int8), exact (FP64 GEMMs of integers with sums below 2^53)."""
    if device is None:
        F = Qc.astype(np.float64)
        return {pq: F[pq[0]] @ F[pq[1]].T for pq in pairs}
    import torch
    F = torch.from_numpy(np.ascontiguousarray(Qc)).to(device).to(torch.float64)
    return {pq: (F[pq[0]] @ F[pq[1]].T).cpu().numpy() for pq in pairs}


def _antidiag_sums(Qc: np.ndarray, S: int, device=None) -> list[np.ndarray]:
    """T_t = sum_{p+q=t} Q_p Q_q^T for t = 0..S-1 (the products k_oz_gemm keeps), exact."""
    P = _pair_products(Qc, [(p, t - p) for t in range(S) for p in range(t + 1)], device)
    return [sum(P[(p, t - p)] for p in range(t + 1)) for t in range(S)]


def _recombine(Q: np.ndarray, e: np.ndarray, S: int, split_chunks, device=None, drop_t=None):
    """The device's FP64 arithmetic over the integer sums: per chunk s = 0; s += T_t 2^-(12+7t) for t = S-1..0; the first chunk of a
    split is stored, the later ones added; the splits summed in order from 0.0; then ldexp(e_i + e_j). Returns (C, max |T_t|).
    drop_t: an anti-diagonal left out (for mutation tests only)."""
    M = Q.shape[1]
    max_acc = 0
    tot = np.zeros((M, M))
    for chunks in split_chunks:
        tile = None
        for c0, c1 in chunks:
            T = _antidiag_sums(Q[:, :, c0:c1], S, device)
            max_acc = max(max_acc, max(int(np.abs(t).max(initial=0)) for t in T))
            v = np.zeros((M, M))
            for t in range(S - 1, -1, -1):
                if t != drop_t:
                    v = v + T[t] * 2.0 ** (-(12 + 7 * t))
            tile = v if tile is None else tile + v
        tot = tot + tile
    return np.ldexp(tot, e[:, None] + e[None, :]), max_acc


def condense_bits(B: np.ndarray, S: int, sched: Schedule, device=None, dig=None, drop_t=None, split_order=None) -> np.ndarray:
    """The exact output C of hb_syrk_rows_ozaki for B = A diag(sqrt(d)) (both triangles) under the schedule `sched`.
    dig: (e, Q) from digits(B, S) when already computed. drop_t / split_order: mutations of the kernel (tests only)."""
    assert sched.M == B.shape[0] and sched.K == B.shape[1] and sched.S == S
    e, Q = dig if dig is not None else digits(B, S)
    sc = sched.split_chunks()
    if split_order is not None:
        sc = [sc[s] for s in split_order]
    return _recombine(Q, e, S, sc, device, drop_t)[0]


def gram(B: np.ndarray, S: int, chunk_cols: int | None = None):
    """C ~= B B^T from the slices, as one split cut into K chunks of chunk_cols columns (default: the device's chunk of
    chunk_stages(S) stages, 65408 columns for S = 8). Returns (C, info) with info = dict(max_abs_digit, max_abs_int32_accumulator)."""
    M, K = B.shape
    e, Q = digits(B, S)
    Kc = chunk_cols or chunk_stages(S) * KS
    C, max_acc = _recombine(Q, e, S, [[(k0, min(k0 + Kc, K)) for k0 in range(0, K, Kc)]])
    return C, dict(max_abs_digit=int(np.abs(Q.astype(np.int64)).max(initial=0)), max_abs_int32_accumulator=max_acc, exponents=e, Q=Q)




# ---- the a-priori bound and an exact reference --------------------------------------------------------------------------------

COL_BLOCK = 32768   # columns per block of the bound and reference GEMMs (bounds the FP64 temporaries at large K)


def _dev(x, device):
    """x as an FP64 array where the GEMMs run: numpy (device None) or a torch tensor on `device`"""
    x = np.ascontiguousarray(x, dtype=np.float64)
    if device is None:
        return x
    import torch
    return torch.from_numpy(x).to(device)


def _host(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def truncation_bound(B: np.ndarray, S: int, chain: int | None = None, device=None, dig=None):
    """A-priori bound R (M x M) with |C - B B^T|_ij <= R_ij 2^{e_i + e_j} + 2^-1075 for the slices' result C; returns (R, e).

    With beta = B / 2^e (|beta| < 1), q its rounding to the grid g = 2^-(6+7(S-1)) (what the digits represent), Z = [beta != 0] and
    w_p = 2^-(6+7p), the three terms are:
    - operand rounding: |q_i.q_j - beta_i.beta_j| <= g/2 (Z |beta|^T + |beta| Z^T) + (g/2)^2 Z Z^T;
    - the dropped products p + q >= S: at most sum_{p+q>=S} |Q_p| |Q_q|^T w_p w_q;
    - the FP64 recombination: a chain of `chain` additions (Schedule.chain; default: one split cut into the device's chunks) over
      terms whose absolute values sum to at most D D^T, D = sum_p |Q_p| w_p: gamma_chain D D^T.
    The integer sums are exact, and the scaling by 2^{e_i + e_j} is exact unless the result is subnormal (the 2^-1075 term). The bound
    is itself evaluated in FP64 from non-negative terms (sums of K products): the factor 1 + gamma_{K+3S} covers that."""
    M, K = B.shape
    e, Q = dig if dig is not None else digits(B, S)
    if chain is None:
        chain = S + -(-K // (chunk_stages(S) * KS))
    g = 2.0 ** (-(6 + 7 * (S - 1)))
    w = [2.0 ** (-(6 + 7 * p)) for p in range(S)]
    op = drop = rec = 0.0
    for k0 in range(0, K, COL_BLOCK):
        beta = np.ldexp(B[:, k0:k0 + COL_BLOCK], -e[:, None])
        A, Z = _dev(np.abs(beta), device), _dev(beta != 0, device)
        op = op + 0.5 * g * (Z @ A.T + A @ Z.T) + (0.5 * g) ** 2 * (Z @ Z.T)
        del A, Z
        Qa = [_dev(np.abs(Q[p, :, k0:k0 + COL_BLOCK]), device) for p in range(S)]
        drop = drop + sum((Qa[p] @ Qa[q].T) * (w[p] * w[q]) for p in range(S) for q in range(S) if p + q >= S)
        D = sum(Qa[p] * w[p] for p in range(S))
        rec = rec + D @ D.T
    gam = lambda c: c * U / (1.0 - c * U)
    R = (_host(op) + _host(drop) + gam(chain) * _host(rec)) * (1.0 + gam(K + 3 * S))
    return R, e


def exact_gram(B: np.ndarray, device=None):
    """(G, err): G = B B^T to within err entrywise.

    Each row is scaled by 2^-e (its frexp exponent) and cut into P integer pieces of w bits (trunc), w chosen so that K products of two
    pieces sum exactly in FP64 (K 2^{2w} <= 2^53); the P^2 piece products are exact GEMMs, summed with the compensated cascade Sum2
    (Ogita, Rump and Oishi, SIAM J. Sci. Comput. 26 (2005)): |G_rel - exact| <= u |exact| + gamma_{2P^2}^2 sum |terms|. The bits below
    2^-(w P) of each scaled row (P w >= 80) are dropped and counted in err, and so is the rounding of the final scaling (2^-1074)."""
    M, K = B.shape
    e = row_exponents(B)
    w = (53 - int(K).bit_length()) // 2
    P = -(-80 // w)
    pairs = [(p, q) for p in range(P) for q in range(P)]
    prods = {pq: 0.0 for pq in pairs}
    tailterm = 0.0
    tail = 2.0 ** (-w * P)
    for k0 in range(0, K, COL_BLOCK):
        r = np.ldexp(B[:, k0:k0 + COL_BLOCK], -e[:, None])
        A, Z = _dev(np.abs(r), device), _dev(r != 0, device)
        tailterm = tailterm + tail * (Z @ A.T + A @ Z.T + tail * (Z @ Z.T))
        del A, Z
        pieces = []
        for p in range(P):
            x = np.trunc(np.ldexp(r, w * (p + 1)))
            pieces.append(_dev(x, device))
            r = r - np.ldexp(x, -w * (p + 1))
        for p, q in pairs:
            prods[(p, q)] = prods[(p, q)] + pieces[p] @ pieces[q].T     # integers below 2^53: exact in any order
    s = c = asum = 0.0
    for (p, q) in sorted(pairs, key=lambda pq: -(pq[0] + pq[1])):   # smallest terms first
        t = np.ldexp(_host(prods[(p, q)]), -w * (p + q + 2))
        asum = asum + np.abs(t)
        z = s + t
        bb = z - s
        c = c + ((s - (z - bb)) + (t - bb))
        s = z
    G_rel = s + c
    g2 = (2 * len(pairs) * U / (1 - 2 * len(pairs) * U)) ** 2
    err_rel = U * np.abs(G_rel) + g2 * asum + _host(tailterm)
    ee = e[:, None] + e[None, :]
    return np.ldexp(G_rel, ee), np.ldexp(err_rel * (1.0 + 8 * U), ee) + 2.0 ** -1074
