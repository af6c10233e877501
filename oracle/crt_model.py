"""CPU model of the Chinese-remainder int8 condensation of hiop_b200/csrc/hb_crt.cu -- TEST INFRASTRUCTURE ONLY.

The device result is C_ij = ldexp(RN(X_ij), e_i + e_j - 2t) with X = q q^T an exact integer matrix, so it does not depend on the tile
schedule, the K splits or the int32 chunks, and the model needs none of them. It restates:
- t(K) and the modulus count N(K) (bits, n_moduli; switch_points prints the table);
- q = rint(b 2^(t - e)) with the row exponents of the slice path (quantize);
- the balanced residues by the kernel's formula r = q - p rint(q fl(1/p)) plus one correction (residues);
- X mod p per modulus with FP64 GEMMs of the residues, exact while K 2^14 < 2^53 (numpy, or torch on a device for large shapes);
- balanced Garner in Python integers, float(int) for the correctly rounded conversion, then np.ldexp (condense_bits);
- the a-priori bound of the result's distance from B B^T (bound), and a brute-force X in Python integers (brute_force_x).
The model is not used by the product."""
from __future__ import annotations

from math import gcd, prod

import numpy as np

from .oz_model import row_exponents

MODULI = (256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191)
MAGIC = 6755399441055744.0   # 1.5 * 2^52
KS = 128                      # columns per K stage
CHUNK_STAGES = 1023           # K stages per exact int32 chunk of k_crt_gemm
U = 2.0 ** -53


def bits(K: int) -> int:
    """t(K) = min(53, floor((126 - ceil(log2 K)) / 2)): K 2^(2t) <= 2^126."""
    return min(53, (126 - (int(K) - 1).bit_length()) // 2)


def n_moduli(K: int, t: int | None = None) -> int:
    """The fewest leading moduli whose product P satisfies P/2 > K 2^(2t)."""
    t = bits(K) if t is None else t
    n = 0
    while prod(MODULI[:n]) <= int(K) << (2 * t + 1):
        n += 1
    return n


def switch_points(Kmax: int = 1 << 31) -> list[tuple[int, int, int]]:
    """(K, t, N) at every K below Kmax where (t(K), N(K)) changes."""
    out, K = [], 1
    while True:
        cur = (bits(K), n_moduli(K))
        step = 1
        while K + step < Kmax and (bits(K + step), n_moduli(K + step)) == cur:
            step *= 2
        if K + step >= Kmax:
            return out
        lo, hi = K, K + step
        while lo + 1 < hi:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if (bits(mid), n_moduli(mid)) == cur else (lo, mid)
        out.append((hi, bits(hi), n_moduli(hi)))
        K = hi


def balanced_range(p: int) -> tuple[int, int]:
    return -(p // 2), (p - 1) // 2


def quantize(B: np.ndarray):
    """(e, t, q): row exponents, the bit count and q = rint(b 2^(t - e)) as integer-valued doubles (|q| <= 2^t)."""
    e = row_exponents(B)
    t = bits(B.shape[1])
    q = np.rint(np.ldexp(B, (t - e)[:, None]))
    return e, t, q


def residues(q: np.ndarray, p: int) -> np.ndarray:
    """The kernel's residue of the integer-valued doubles q: k = rint(q fl(1/p)) (FP64 product, magic-number rounding), r = q - p k
    (exact: the device's FMA rounds an exact small integer), then one correction into the balanced range. int64."""
    k = (q * (1.0 / p) + MAGIC) - MAGIC
    r = q.astype(np.int64) - p * k.astype(np.int64)
    lo, hi = balanced_range(p)
    r = np.where(r > hi, r - p, r)
    return np.where(r < lo, r + p, r)


def _bal(x, p: int):
    lo, hi = balanced_range(p)
    r = np.mod(x, p)
    return np.where(r > hi, r - p, r)


def residue_grams(q: np.ndarray, n: int, device=None) -> list[np.ndarray]:
    """[X mod p_m (balanced, int64) for m < n] from FP64 GEMMs of the residues (exact: |sum| <= K 2^14 < 2^53). With a torch device the
    residues (the same IEEE operations as residues()) and the GEMMs run there."""
    if device is None:
        return [_bal((lambda R: R @ R.T)(residues(q, p).astype(np.float64)).astype(np.int64), p) for p in MODULI[:n]]
    import torch
    qt = torch.from_numpy(np.ascontiguousarray(q)).to(device)
    qi = qt.to(torch.int64)
    out = []
    for p in MODULI[:n]:
        k = (qt * (1.0 / p) + MAGIC) - MAGIC
        r = qi - p * k.to(torch.int64)
        lo, hi = balanced_range(p)
        r = torch.where(r > hi, r - p, r)
        R = torch.where(r < lo, r + p, r).to(torch.float64)
        out.append(_bal((R @ R.T).cpu().numpy().astype(np.int64), p))
    return out


def garner(res: list[np.ndarray], balanced: bool = True) -> np.ndarray:
    """X (object array of Python ints) from its residues: mixed-radix digits d_m (balanced unless told otherwise), X = sum d_m W_m."""
    n = len(res)
    d, X, W = [], np.zeros(res[0].shape, dtype=object), 1
    for m in range(n):
        p = MODULI[m]
        s = np.zeros(res[0].shape, dtype=np.int64)
        Wj = 1
        for j in range(m):
            s = s + d[j] * (Wj % p)
            Wj *= MODULI[j]
        dm = np.mod((res[m] - s) * pow(Wj % p, -1, p) if m else res[m], p)
        if balanced:
            dm = _bal(dm, p)
        d.append(dm.astype(np.int64))
        X = X + dm.astype(object) * W
        W *= p
    return X


def round_scale(X: np.ndarray, e: np.ndarray, t: int) -> np.ndarray:
    """ldexp(RN(X_ij), e_i + e_j - 2t): float(int) rounds to nearest, ties to even."""
    v = np.vectorize(float, otypes=[np.float64])(X) if X.size else np.zeros(X.shape)
    return np.ldexp(v, (e[:, None] + e[None, :] - 2 * t))


def condense_bits(B: np.ndarray, device=None, n: int | None = None, t: int | None = None, balanced: bool = True) -> np.ndarray:
    """The exact output C of hb_syrk_rows_crt for B = A diag(sqrt(d)) (both triangles). n / t / balanced: mutations (tests only)."""
    M, K = B.shape
    e = row_exponents(B)
    tt = bits(K) if t is None else t
    q = np.rint(np.ldexp(B, (tt - e)[:, None]))
    nn = n_moduli(K, bits(K)) if n is None else n
    return round_scale(garner(residue_grams(q, nn, device), balanced), e, tt)


def brute_force_x(B: np.ndarray) -> np.ndarray:
    """X = q q^T in Python integers (small shapes only)."""
    _, _, q = quantize(B)
    Q = q.astype(np.int64).astype(object)
    return Q.dot(Q.T)


def bound(B: np.ndarray, C: np.ndarray, device=None) -> np.ndarray:
    """A-priori bound on |C - B B^T|: sum_k (|b_ik| 2^(e_j-t-1) + |b_jk| 2^(e_i-t-1) + 2^(e_i+e_j-2t-2)) + u |C|, evaluated in FP64 from
    non-negative terms (the factor 1 + 4u covers that), plus 2^-1074 for a result that lands below the normal range."""
    M, K = B.shape
    e = row_exponents(B)
    t = bits(K)
    if device is None:
        a = np.abs(B).sum(axis=1)
    else:
        import torch
        a = torch.from_numpy(np.abs(B)).to(device).sum(dim=1).cpu().numpy()
    nz = (B != 0).any(axis=1)
    g = np.where(nz, np.ldexp(1.0, e - t - 1), 0.0)   # half the grid of row i (zero rows are exact)
    R = a[:, None] * g[None, :] + g[:, None] * a[None, :] + K * np.outer(g, g)
    return R * (1.0 + 4 * U) + U * np.abs(C) + 2.0 ** -1074


def round_sticky64(x: int) -> float:
    """The kernel's RN(X): |X| < 2^127 normalised to 64 bits with a sticky bit, then one rounding of a 64-bit integer (numpy's uint64
    conversion rounds to nearest even), then an exact power-of-two scale."""
    neg, u = x < 0, abs(x)
    if u < 1 << 64:
        v = float(np.uint64(u).astype(np.float64))
    else:
        sh = u.bit_length() - 64
        top = (u >> sh) | (1 if u & ((1 << sh) - 1) else 0)
        v = float(np.ldexp(np.uint64(top).astype(np.float64), sh))
    return -v if neg else v


def pairwise_coprime() -> bool:
    return all(gcd(a, b) == 1 for i, a in enumerate(MODULI) for b in MODULI[i + 1:])
