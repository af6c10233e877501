"""TEST INFRASTRUCTURE (never imported by hiop_b200/): numpy model of the symmetric random butterfly transform of hb_symdense_dist.cu
(HB_FACT_RBT_NOPIV, include/hiopb200.h), which the device matches bit for bit.

Depth 2 (Baboulin, Becker, Bosilca, Danalis, Dongarra 2014): U = B2 B1, A' = U^T A U = B1^T (B2^T A B2) B1.
  * B1 is one butterfly of order N; B2 = diag(butterfly of order h, butterfly of order N - h), h = ceil(N / 2).
  * A butterfly of order n (hh = ceil(n / 2), m = n - hh) is [R0 R1; R0 -R1] / sqrt(2) with the random diagonal R = diag(r_0 .. r_n-1):
    local row t < m pairs with t + hh. For odd n the middle row t = hh - 1 is unpaired and only scaled by r_t.
  * Column i of a butterfly has its entries in rows lo_i and hi_i (lo_i = hi_i when unpaired) with coefficients f_i c and s_i f_i c:
    f_i = r_t, s_i = +1 on the lo side (and when unpaired), -1 on the hi side, c = 1 / sqrt(2) (1 when unpaired).
  * r_t = 1 + (k - 2^19) / 2^23 with k the top 20 bits of splitmix64(SEED, stream, t), stream = 2 * level + half: dyadic, in
    [15/16, 17/16), exact in FP64 and a function of N alone (never of the number of ranks).

Every entry is one fixed expression in IEEE double (no fused multiply-add), which hb_symdense_dist.cu writes with __dmul_rn /
__dadd_rn in the same order:
    t = (a(lo_i, lo_j) + s_i s_j a(hi_i, hi_j)) + (s_j a(lo_i, hi_j) + s_i a(hi_i, lo_j))     both paired
    t = a(lo_i, lo_j) + s_i s_j a(hi_i, hi_j)                                                  one unpaired
    t = a(i, j)                                                                                both unpaired
    out(i, j) = (f_i f_j) (t w),  w = 1/2 (both paired: the two 1/sqrt(2) combine exactly), C = fl(1/sqrt(2)) (one), 1 (none).
Both sums are commutative under a swap of i and j, so out is exactly symmetric when a is."""
import numpy as np

SEED = 0x5EED_2011_B7F1_0001
GOLDEN = 0x9E37_79B9_7F4A_7C15
C = 0.7071067811865476        # the double nearest 1/sqrt(2)
EPS = 2.0 ** -52              # refinement target: backward error <= EPS
MAX_CORRECTIONS = 3
M64 = (1 << 64) - 1


def _splitmix64(z):
    z = z.astype(np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def diagonal(level: int, half: int, n: int) -> np.ndarray:
    """r_0 .. r_n-1 of butterfly `half` (0 or 1) of level 1 (B1, half 0) or level 2 (B2)"""
    stream = 2 * level + half
    ctr = (np.uint64(stream) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(SEED) + np.uint64(GOLDEN) * (ctr + np.uint64(1))
    k = (_splitmix64(z) >> np.uint64(44)).astype(np.int64)
    return (float(1 << 23) + (k - (1 << 19)).astype(np.float64)) / float(1 << 23)


def segments(N: int, level: int):
    """(offset, order, half) of the butterflies of a level"""
    if level == 1:
        return [(0, N, 0)]
    h = (N + 1) // 2
    return [(0, h, 0), (h, N - h, 1)]


def level_maps(N: int, level: int):
    """per global index i: lo, hi (= i when unpaired), s (+1 / -1), paired (bool), f"""
    lo, hi = np.arange(N), np.arange(N)
    s, f = np.ones(N), np.ones(N)
    paired = np.zeros(N, dtype=bool)
    for o, n, half in segments(N, level):
        if n == 0:
            continue
        hh = (n + 1) // 2
        m = n - hh
        t = np.arange(n)
        f[o:o + n] = diagonal(level, half, n)
        a = t < m
        hi[o + t[a]] = o + t[a] + hh
        b = t >= hh
        lo[o + t[b]] = o + t[b] - hh
        s[o + t[b]] = -1.0
        paired[o + t[a | b]] = True
    return lo, hi, s, paired, f


def partner(N: int, level: int) -> np.ndarray:
    """the row each row combines with at a level (itself when unpaired): an involution"""
    lo, hi, _, _, _ = level_maps(N, level)
    return np.where(lo == np.arange(N), hi, lo)


def two_sided(A: np.ndarray, level: int) -> np.ndarray:
    """B^T A B for the butterfly level (A full, N x N)"""
    N = A.shape[0]
    lo, hi, s, p, f = level_maps(N, level)
    all_ = A[np.ix_(lo, lo)]
    ahh = A[np.ix_(hi, hi)]
    alh = A[np.ix_(lo, hi)]
    ahl = A[np.ix_(hi, lo)]
    ss = s[:, None] * s[None, :]
    pp = p[:, None] & p[None, :]
    one = p[:, None] ^ p[None, :]
    t = np.where(pp | one, all_ + ss * ahh, all_)
    t = np.where(pp, t + (s[None, :] * alh + s[:, None] * ahl), t)
    w = np.where(pp, 0.5, np.where(one, C, 1.0))
    return (f[:, None] * f[None, :]) * (t * w)


def mirror(Aupper: np.ndarray) -> np.ndarray:
    """the full symmetric matrix from the upper triangle (what the mirror step writes into the lower part of every row)"""
    U = np.triu(Aupper)
    return U + np.triu(U, 1).T


def transform(A: np.ndarray, stages: int = 2) -> np.ndarray:
    """A' = U^T A U from the upper triangle of A; stages = 1 stops after B2^T A B2"""
    out = mirror(A)
    for level in (2, 1)[:stages]:
        out = two_sided(out, level)
    return out


def _apply_T(v, level):
    """B^T v (v: N or N x nrhs)"""
    N = v.shape[0]
    lo, hi, s, p, f = level_maps(N, level)
    v2 = v.reshape(N, -1)
    sc, fc = s[:, None], f[:, None]
    out = np.where(p[:, None], fc * ((v2[lo] + sc * v2[hi]) * C), fc * v2)
    return out.reshape(v.shape)


def _apply(v, level):
    """B v"""
    N = v.shape[0]
    lo, hi, s, p, f = level_maps(N, level)
    v2 = v.reshape(N, -1)
    sc = s[:, None]
    out = np.where(p[:, None], (f[lo][:, None] * v2[lo] + sc * (f[hi][:, None] * v2[hi])) * C, f[:, None] * v2)
    return out.reshape(v.shape)


def apply_UT(b):
    """b' = U^T b = B1^T (B2^T b)"""
    return _apply_T(_apply_T(np.asarray(b, dtype=np.float64), 2), 1)


def apply_U(x):
    """x = U x' = B2 (B1 x')"""
    return _apply(_apply(np.asarray(x, dtype=np.float64), 1), 2)


def U_matrix(N: int) -> np.ndarray:
    return apply_U(np.eye(N))


def nopiv_ldlt(A: np.ndarray, nb: int = 128):
    """LDL^T without pivoting of a full symmetric A: (L, d, ret) with ret the value hb_symdense_dist_matrix_changed gives (number of
    negative pivots, -1 for a zero or non-finite pivot or |d| < 1e-14). Right-looking in blocks of nb: the columns of a block one by one
    (with the block's rows), then one product L S for the trailing matrix, S the block's rows of the Schur complement.""" 
    N = A.shape[0]
    S = np.array(A, dtype=np.float64)
    L = np.eye(N)
    d = np.zeros(N)
    for k0 in range(0, N, nb):
        k1 = min(k0 + nb, N)
        for k in range(k0, k1):
            d[k] = S[k, k]
            if d[k] == 0.0 or not np.isfinite(d[k]):
                return L, d, -1
            L[k + 1:, k] = S[k + 1:, k] / d[k]
            S[k + 1:, k + 1:k1] -= np.outer(L[k + 1:, k], S[k, k + 1:k1])
            S[k + 1:k1, k1:] -= np.outer(L[k + 1:k1, k], S[k, k1:])
        S[k1:, k1:] -= L[k1:, k0:k1] @ S[k0:k1, k1:]
    return L, d, inertia_ret(d)


def inertia_counts(d):
    d = np.asarray(d)
    return int((d < -1e-14).sum()), int(((d >= -1e-14) & (d < 1e-14)).sum()), int((d >= 1e-14).sum())


def inertia_ret(d):
    neg, nul, _ = inertia_counts(d)
    return -1 if nul else neg


def dsytrf_inertia(A: np.ndarray):
    """(neg, null, pos) from LAPACK's Bunch-Kaufman DSYTRF with LINPACK dsidi's rule: 1 x 1 pivots by sign (|d| < 1e-14 null), a 2 x 2
    block [[a, b], [b, c]] by its determinant (negative: one of each sign; positive: two of the sign of a)"""
    from scipy.linalg import lapack
    N = A.shape[0]
    ldu, piv, info = lapack.dsytrf(np.asfortranarray(np.tril(A)), lower=1)
    neg = nul = pos = 0
    k = 0
    while k < N:
        if piv[k] > 0:
            dk = ldu[k, k]
            if dk < -1e-14:
                neg += 1
            elif dk < 1e-14:
                nul += 1
            else:
                pos += 1
            k += 1
        else:
            a, b, c = ldu[k, k], ldu[k + 1, k], ldu[k + 1, k + 1]
            det = (a / abs(b)) * c - abs(b)
            if det < 0:
                neg, pos = neg + 1, pos + 1
            elif det > 0:
                neg, pos = (neg + 2, pos) if a < 0 else (neg, pos + 2)
            else:
                nul += 2
            k += 2
    return neg, nul, pos


def column_omegas(nA, num, xn, bn):
    """the stopping rule's quotient per column from ||A||_inf and the per-column max |r|, max |x|, max |b|: num / (nA xn + bn), NaN where
    one of the four is not finite, +inf where the denominator is 0 and num is not, 0 for a zero column"""
    num, xn, bn = (np.asarray(v, dtype=np.float64) for v in (num, xn, bn))
    finite = np.isfinite(num) & np.isfinite(xn) & np.isfinite(bn) & np.isfinite(nA)
    with np.errstate(divide="ignore", invalid="ignore"):
        den = nA * xn + bn
        w = np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num == 0, 0.0, np.inf))
    return np.where(finite, w, np.nan)


def nan_max(w) -> float:
    """the largest entry, NaN if there is one, 0 for none"""
    w = np.asarray(w, dtype=np.float64)
    return float(np.max(w)) if w.size else 0.0


def backward_error(A, x, b, nA=None) -> float:
    """||b - A x||_inf / (||A||_inf ||x||_inf + ||b||_inf), the largest over the columns of x, b (column_omegas; a NaN wins). nA replaces
    ||A||_inf."""
    x2, b2 = x.reshape(A.shape[0], -1), b.reshape(A.shape[0], -1)
    if nA is None:
        nA = np.abs(A).sum(axis=1).max(initial=0.0)
    with np.errstate(invalid="ignore", over="ignore"):
        r = b2 - A @ x2
    return nan_max(column_omegas(nA, np.abs(r).max(axis=0), np.abs(x2).max(axis=0), np.abs(b2).max(axis=0)))


def solve(A: np.ndarray, b: np.ndarray):
    """A x = b through A' = U^T A U, its no-pivot LDL^T and refinement against A' with the rule of hb_symdense_solve /
    hb_symdense_dist_solve (refine). Returns (x, corrections, backward error against A')."""
    return refine(A, b)[:3]


def refine(A: np.ndarray, b: np.ndarray, Aref=None, anorm=None, Ap=None, factor=None):
    """solve with every exit of the refinement visible: correct while omega is finite, omega > EPS, fewer than MAX_CORRECTIONS
    corrections were made and the last correction at least halved it. The residuals and omegas are against A' and ||A'||_inf, or against
    Aref (full, in the transformed basis) and anorm when given (anorm defaults to ||Aref||_inf). Ap, factor: A' and nopiv_ldlt(A') when the
    caller has them already. Returns (x, corrections, omega, omegas, ret): omegas = every omega the rule read, ret = 1 when the last one
    is finite, else 0."""
    Ap = transform(A) if Ap is None else Ap
    L, d, ret = nopiv_ldlt(Ap) if factor is None else factor
    assert ret >= 0, ret
    from scipy.linalg import solve_triangular
    Ar = Ap if Aref is None else Aref
    nA = np.abs(Ar).sum(axis=1).max(initial=0.0) if anorm is None else anorm

    def ldl_solve(v):
        y = solve_triangular(L, v, lower=True, unit_diagonal=True, check_finite=False)
        return solve_triangular(L.T, y / (d if y.ndim == 1 else d[:, None]), lower=False, unit_diagonal=True, check_finite=False)

    bp = apply_UT(b)
    with np.errstate(invalid="ignore", over="ignore"):
        xp = ldl_solve(bp)
        om, prev, corr = backward_error(Ar, xp, bp, nA), np.inf, 0
        oms = [om]
        while np.isfinite(om) and corr < MAX_CORRECTIONS and om > EPS and om <= 0.5 * prev:
            xp = xp + ldl_solve(bp - Ar @ xp)
            corr += 1
            prev, om = om, backward_error(Ar, xp, bp, nA)
            oms.append(om)
        x = apply_U(xp)
    return x, corr, om, oms, int(np.isfinite(om))
