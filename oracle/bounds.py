"""TEST INFRASTRUCTURE ONLY -- exact references and rigorous floating-point error bounds for the kernel tests.

A kernel that sums in a different order than numpy cannot be held to a fixed relative tolerance without either hiding real errors (the
tolerance is set by the largest entry, as in |N - N_ref| <= 1e-12 max|N|) or failing on benign reorderings. The helpers here give the
standard a-priori bounds (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., ch. 3-4) so each test can state what its
kernel is allowed to get wrong:

- a sum or dot product evaluated with any bracketing whose longest chain of additions (the depth of the summation tree, plus one for
  the multiplication) is c has |fl(s) - s| <= gamma_c * sum |terms|, gamma_c = c u / (1 - c u), u = 2^-53;
- C = A diag(d) A^T through any order of K-term sums: |fl(C) - C| <= gamma_{K+2} * (|A| diag(d) |A|^T), entrywise (syrk_bound).

The exact references (exact_dot and friends) use Dekker / Veltkamp TwoProduct and math.fsum: the result is the correctly rounded value
of the mathematically exact dot product, so the only error left in a comparison is the kernel's own.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -53                 # unit roundoff of IEEE binary64 (round to nearest)
_SPLIT = 2.0 ** 27 + 1.0       # Veltkamp splitter for 53-bit significands


def gamma(c: float) -> float:
    """gamma_c = c u / (1 - c u)."""
    c = float(c)
    assert c * U < 1.0
    return c * U / (1.0 - c * U)


def _split(a):
    t = _SPLIT * a
    hi = t - (t - a)
    return hi, a - hi


def two_product(a, b):
    """Error-free product, vectorised: a*b = p + e exactly (no overflow / underflow assumed; |a|, |b| < 2^996)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_sum(v) -> float:
    """Correctly rounded sum of the entries of v (math.fsum)."""
    return math.fsum(np.asarray(v, dtype=np.float64).ravel().tolist())


def exact_dot(a, b) -> float:
    """Correctly rounded value of the exact dot product sum_i a_i b_i."""
    p, e = two_product(np.ravel(a), np.ravel(b))
    return math.fsum(p.tolist() + e.tolist())


def exact_rows(A, x):
    """y_i = exact_dot(A[i, :], x) for every row (the reference of y = A x)."""
    A = np.asarray(A, dtype=np.float64)
    return np.array([exact_dot(A[i], x) for i in range(A.shape[0])])


def exact_cols(A, x):
    """y_k = sum_i A[i, k] x_i for every column (the reference of y = A^T x), vectorised over the columns.

    TwoProduct per term, then the compensated cascade Sum2 (Ogita, Rump and Oishi, SIAM J. Sci. Comput. 26 (2005), alg. 4.4) down the
    rows: the result is as accurate as if computed in twice the working precision, |y - y_exact| <= u |y_exact| + gamma_{2m}^2 sum |terms|
    (cols_ref_error gives that bound). Not correctly rounded, but 1e-15 below any kernel bound used with it."""
    A = np.asarray(A, dtype=np.float64)
    x = np.asarray(x, dtype=np.float64)
    s = np.zeros(A.shape[1])
    c = np.zeros(A.shape[1])
    for i in range(A.shape[0]):
        p, e = two_product(A[i], x[i])
        for t in (p, e):
            z = s + t                      # TwoSum(s, t)
            bb = z - s
            c += (s - (z - bb)) + (t - bb)
            s = z
    return s + c


def cols_ref_error(m: int, y_ref, abs_terms):
    """Bound on |exact_cols - exact| for m rows (see exact_cols)."""
    return U * np.abs(y_ref) + gamma(2 * m) ** 2 * abs_terms


def syrk_bound(A, d):
    """B = |A| diag(d) |A|^T, the entrywise scale of the rounding error of A diag(d) A^T (d >= 0 not required)."""
    Aa = np.abs(np.asarray(A, dtype=np.float64))
    return (Aa * np.abs(d)) @ Aa.T


def syrk_tol(B, K: int, N_ref, c_kernel: int | None = None):
    """Componentwise tolerance for a condensed N = A diag(d) A^T (+ a diagonal) from a kernel against a numpy FP64 reference.

    Both sides are within gamma_{K+2} B of the exact product (K products each rounded twice, d folded into one factor first, summed in
    any order); c_kernel replaces K + 2 for the kernel when its chain is longer (partial tiles added in a fix-up pass). The 2 u |N| term
    covers the rounding of the diagonal addition (Dd_inv) on each side."""
    ck = K + 2 if c_kernel is None else c_kernel
    return (gamma(ck) + gamma(K + 2)) * B + 2.0 * U * np.abs(N_ref)


TAU_DIAG = 1e-12   # diagonal-scaled criterion for N with secant rows (l > 0): |N - N_ref| <= TAU_DIAG sqrt(N_ii N_jj)


def condensed_error_ratio(N, N_ref, J, DhInv, l: int, num_sms: int, tau: float = TAU_DIAG) -> float:
    """max entrywise error of a condensed N against a reference, over its tolerance (<= 1 passes; 1 / ratio is the margin).

    l = 0: N = J DhInv J^T + blkdiag(0, Dd_inv) exactly, held to syrk_tol with the FP64 DMMA kernel's chain (K products, then the K
    windows of at most num_sms CTAs added in the fix-up pass). l > 0: N also carries the low-rank correction through a 2l x 2l
    solve, whose error scales with the diagonal of N rather than with |J| DhInv |J|^T: |N - N_ref| <= tau sqrt(N_ii N_jj)."""
    N = np.asarray(N)
    if l == 0:
        K = np.asarray(J).shape[1]
        tol = syrk_tol(syrk_bound(J, DhInv), K, N_ref, c_kernel=K + 2 + num_sms)
    else:
        d = np.abs(np.diag(N_ref))
        tol = tau * np.sqrt(np.outer(d, d))
    return float((np.abs(N - N_ref) / np.maximum(tol, np.finfo(np.float64).tiny)).max())


def reduction_chain(n: int, grid: int, threads: int = 256, second_threads: int = 256) -> int:
    """Longest serial addition chain of the two-stage reductions (hb_vec.cu k_red1 + k_red2): each thread strides over
    ceil(n / (grid * threads)) items, a warp xor tree (5), a block tree over the warp sums (5), then the second stage over the grid
    partials: ceil(grid / second_threads) per thread, warp tree (5), block tree (5)."""
    per = -(-n // (grid * threads))
    return per + 5 + 5 + (-(-grid // second_threads)) + 5 + 5


def slots_chain(n: int, grid: int, threads: int = 256) -> int:
    """Longest addition chain of a block-partial kernel finished by hb_reduce_slots (hb_vec.cu): ceil(n / (grid * threads)) items per
    thread, a warp tree (5) and a block tree (5), then one warp per slot over the grid partials: ceil(grid / 32) per lane and a warp tree
    (5)."""
    return -(-n // (grid * threads)) + 5 + 5 + (-(-grid // 32)) + 5


def stream_grid(items: int, num_sms: int, threads: int = 256) -> int:
    """hb_grid (hb_common.cuh): ceil(items / threads) CTAs, clamped to [1, 8 num_sms]."""
    return max(1, min(-(-items // threads), 8 * num_sms))
