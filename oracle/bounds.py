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


# ---- dense symmetric factorizations and solves (Higham ch. 8, 10, 11, 14) ----------------------------------------------------------
#
# Every kernel factor is written as P A P^T = L D L^T: L unit lower triangular (zeros below the diagonal of a 2 x 2 pivot block), D block
# diagonal with 1 x 1 and 2 x 2 blocks (d on the diagonal, the off-diagonal of the 2 x 2 block starting at column k in dsub[k]). Cholesky is
# the case L = R^T, D = I, P = I. The helpers take numpy arrays or torch FP64 tensors (CPU or CUDA) and compute in the same place.

FACTOR_C = 3          # kernel term of the factor bound: theta * gamma(FACTOR_C * N + 3), see factor_backward_ratio
SOLVE_C = 7           # kernel term of the solve bound:  theta * gamma(SOLVE_C * N + 3), see solve_backward_ratio


def _xp(a):
    import torch
    return torch if isinstance(a, torch.Tensor) else np


def ld_product(L, d, dsub=None):
    """L D (D block diagonal from d and dsub), as a dense array."""
    LD = L * d[None, :]
    if dsub is not None:
        k = np.nonzero(dsub)[0] if _xp(L) is np else dsub.nonzero().flatten()
        LD[:, k] += L[:, k + 1] * dsub[k][None, :]
        LD[:, k + 1] += L[:, k] * dsub[k][None, :]
    return LD


def lapack_to_permuted(ldu, ipiv):
    """LAPACK dsytrf ('L') output -> (L, d, dsub, perm) with A[perm][:, perm] = L D L^T.

    LAPACK keeps each column of L in the row order of its own step; the later interchanges are applied here to the earlier columns (what
    dsyconv does), which is the fully permuted form the cluster Bunch-Kaufman kernel stores."""
    N = ldu.shape[0]
    Lo = np.tril(ldu)
    d = np.diag(Lo).copy()
    L = np.tril(Lo, -1)
    dsub = np.zeros(N)
    perm = np.arange(N)
    k = 0
    while k < N:
        if ipiv[k] > 0:
            kk, kp, step = k, ipiv[k] - 1, 1
        else:
            kk, kp, step = k + 1, -ipiv[k] - 1, 2
            dsub[k] = L[k + 1, k]
            L[k + 1, k] = 0.0
        if kp != kk:
            L[[kk, kp], :k] = L[[kp, kk], :k]
            perm[[kk, kp]] = perm[[kp, kk]]
        k += step
    return L + np.eye(N), d, dsub, perm


def perm_from_ipiv(ipiv):
    """The gather order of P A P^T implied by a pivot vector in LAPACK's convention (1-based; a negative pair marks a 2 x 2 block whose
    second row was exchanged)."""
    ipiv = np.asarray(ipiv)
    N = ipiv.shape[0]
    perm = np.arange(N)
    k = 0
    while k < N:
        step = 1 if ipiv[k] > 0 else 2
        kk, kp = k + step - 1, abs(int(ipiv[k])) - 1
        perm[[kk, kp]] = perm[[kp, kk]]
        k += step
    return perm


def bk_cluster_to_lapack(ipiv, perm, dsub):
    """The cluster Bunch-Kaufman output as LAPACK's ipiv. The kernel writes ipiv in LAPACK's convention already; what can be wrong is
    the rest of the output agreeing with it: perm must be the product of the interchanges ipiv records and dsub must be non-zero exactly
    at the first column of each 2 x 2 block. Raises AssertionError where they disagree."""
    ipiv = np.asarray(ipiv).astype(np.int64)
    N = ipiv.shape[0]
    assert np.array_equal(np.asarray(perm), perm_from_ipiv(ipiv)), "perm is not the product of the interchanges in ipiv"
    first = np.zeros(N, dtype=bool)
    k = 0
    while k < N:
        if ipiv[k] < 0:
            assert k + 1 < N and ipiv[k + 1] == ipiv[k], f"2 x 2 block at {k} not marked on both rows"
            first[k] = True
            k += 2
        else:
            k += 1
    assert np.all((np.asarray(dsub) != 0.0) <= first), "dsub set outside the first column of a 2 x 2 block"
    return ipiv


def block_theta(L, b):
    """theta = max_k || |T_kk^-1| |T_kk| ||_inf over the b x b diagonal blocks T_kk of the (unit or Cholesky) lower triangle L: the factor
    by which multiplying by an explicit inverse instead of substituting can enlarge the rounding error (Higham ch. 14, eq. (14.3)-(14.4):
    the computed inverse X of a triangular T has |X T - I| <= c_b u |X| |T|)."""
    from scipy.linalg import solve_triangular
    import torch
    N = L.shape[0]
    th = 1.0
    for k0 in range(0, N, b):
        T = L[k0:k0 + b, k0:k0 + b]
        T = T.cpu().numpy() if isinstance(T, torch.Tensor) else np.asarray(T)
        X = solve_triangular(T, np.eye(T.shape[0]), lower=True)
        th = max(th, float((np.abs(X) @ np.abs(T)).sum(axis=1).max()))
    return th


def factor_backward_ratio(PAP, L, d, dsub=None, theta=1.0):
    """max_ij |P A P^T - L D L^T|_ij / tol_ij (<= 1 passes; 1 / ratio is the margin), with

        tol = theta gamma(3N + 3) (|P A P^T| + |L||D||L^T|) + gamma(N + 3) |L||D||L^T|.

    Kernel term. Entry (i, j) of the Schur complement receives at most N rank-1 (or rank-2) updates, each formed as a product w l with
    w = l d (L D for a 2 x 2 block) rounded once, then multiplied and subtracted: Higham's proof of Thm 10.3 (Cholesky) and Thm 11.3
    (block LDL^T, Bunch-Kaufman) gives |Delta A| <= gamma(N + 3) (|A| + |L||D||L^T|) for that chain. The columns of L are then obtained
    by a triangular solve with the pivot block; where the kernel multiplies by an explicit inverse of a b x b diagonal block (b = 16 in
    k_trsm_panel and the cooperative paths, 128 in the look-ahead and blocked-solve paths) the solve adds a b-term dot product (gamma_b)
    and the inverse's own residual c_b u |X||T| with c_b <= b (Higham ch. 14, column-by-column substitution), both scaled by theta: at
    most theta gamma(2N). gamma(N + 3) + theta gamma(2N) <= theta gamma(3N + 3): the constant in front of N u is 3.
    Check term. The product L D L^T is formed here in FP64 with at most N + 2 roundings per entry and the difference with one more:
    gamma(N + 3) |L||D||L^T| (Higham Lemma 3.5)."""
    xp = _xp(L)
    N = L.shape[0]
    LD = ld_product(L, d, dsub)
    aL = xp.abs(L)
    aLD = ld_product(aL, xp.abs(d), None if dsub is None else xp.abs(dsub))
    ratio = 0.0
    for i0 in range(0, N, 4096):          # row blocks: the temporaries stay 4096 x N at large N
        rows = slice(i0, i0 + 4096)
        absprod = aLD[rows] @ aL.T
        tol = theta * gamma(FACTOR_C * N + 3) * (xp.abs(PAP[rows]) + absprod) + gamma(N + 3) * absprod
        err = xp.abs(PAP[rows] - LD[rows] @ L.T)
        ratio = max(ratio, float((err / xp.clip(tol, np.finfo(np.float64).tiny, None)).max()))
    return ratio


EXACT_RESIDUAL_MAX_N = 320    # above: the residual in FP64 with its evaluation bound (exact_rows takes ~1 s per rhs at N = 4000)


def solve_backward_ratio(A, x, b, L, d, dsub=None, theta=1.0, extra=0.0):
    """Backward error of a solve A x = b through the factor P A P^T = L D L^T (one rhs per column of x, b), against its bound:
    returns (ratio, omega). omega is the Oettli-Prager backward error max_i |b - A x|_i / (|A||x| + |b|)_i (Higham Thm 7.3); ratio is
    max_i |b - A x|_i / tol_i with

        tol = theta gamma(7N + 3) ((|A| + P^T |L||D||L^T| P) |x| + |b|) + eval,

    Higham Thm 10.4 / 11.4: (A + Delta A) x = b with |Delta A| <= p(N) u (|A| + P^T|L||D||L^T|P): the factor term of
    factor_backward_ratio (theta gamma(3N + 3)) plus one triangular solve per factor of L (gamma(N) each, Thm 8.5), each doubled by the
    explicit diagonal-block inverses of the blocked solves (theta gamma(2N) each): theta gamma(7N + 3). A, L: full arrays in the permuted
    order given by perm on the caller's side; pass A = P A P^T, x, b permuted alike. eval = 0 when the residual is evaluated exactly
    (numpy arrays, N <= EXACT_RESIDUAL_MAX_N), else gamma(N + 1)(|A||x| + |b|) for the FP64 evaluation. extra (>= 0, broadcast to b):
    a bound on how far the right-hand side the kernel solved with is from b, added to tol (a b formed by a reduction)."""
    xp = _xp(A)
    N = A.shape[0]
    x = x.reshape(N, -1)
    b = b.reshape(N, -1)
    if xp is np and N <= EXACT_RESIDUAL_MAX_N:
        r = np.stack([b[:, j] - exact_rows(A, x[:, j]) for j in range(x.shape[1])], axis=1)
        ev = 0.0
    else:
        r = b - A @ x
        ev = 1.0
    aA = xp.abs(A)
    ax = xp.abs(x)
    op = aA @ ax + xp.abs(b)
    aL = xp.abs(L)
    ldl = ld_product(aL, xp.abs(d), None if dsub is None else xp.abs(dsub)) @ (aL.T @ ax)
    tol = theta * gamma(SOLVE_C * N + 3) * (op + ldl) + ev * gamma(N + 1) * op + extra
    tiny = np.finfo(np.float64).tiny
    ratio = float((xp.abs(r) / xp.clip(tol, tiny, None)).max())
    omega = float((xp.abs(r) / xp.clip(op, tiny, None)).max())
    return ratio, omega


def known_inertia_matrix(N, n_two, n_neg1, seed, reflectors=3, device="cpu"):
    """A symmetric N x N matrix with inertia known by construction, built with torch FP64 (on `device`): returns (M, (neg, 0, pos)).

    B = n_two 2 x 2 blocks [[e, b], [b, e']] with |b| in [0.5, 2] and |e|, |e'| <= 1e-3 |b| (one negative and one positive eigenvalue
    each, both of modulus about |b|), then N - 2 n_two 1 x 1 blocks of modulus in [0.5, 2], n_neg1 of them negative; a random symmetric
    permutation P scatters the two rows of every 2 x 2 block far apart; `reflectors` Householder reflectors H_k = I - 2 v v^T mix it:
    M = Q P B P^T Q^T with Q = H_1 ... H_k orthogonal. Sylvester's law of inertia: inertia(M) = inertia(B) = (n_two + n_neg1, 0,
    n_two + N - 2 n_two - n_neg1), and the eigenvalues of M are those of B, at least ~0.5 in modulus. The mixing leaves the diagonal of
    the 2 x 2 rows at about 1 / N against off-diagonals of about 1, so Bunch-Kaufman takes 2 x 2 pivots there, with partners anywhere."""
    import torch
    assert 2 * n_two <= N and n_neg1 <= N - 2 * n_two
    r = np.random.default_rng(seed)
    n1 = N - 2 * n_two
    diag = np.zeros(N)
    off = np.zeros(max(N - 1, 0))
    bb = r.uniform(0.5, 2.0, n_two) * r.choice([-1.0, 1.0], n_two)
    diag[0:2 * n_two:2] = r.uniform(-1e-3, 1e-3, n_two) * np.abs(bb)
    diag[1:2 * n_two:2] = r.uniform(-1e-3, 1e-3, n_two) * np.abs(bb)
    off[0:2 * n_two:2] = bb
    v1 = r.uniform(0.5, 2.0, n1)
    v1[:n_neg1] *= -1.0
    diag[2 * n_two:] = v1
    p = r.permutation(N)
    V = r.standard_normal((reflectors, N))
    dev = torch.device(device)
    t = lambda a: torch.as_tensor(a, dtype=torch.float64, device=dev)
    pt = torch.as_tensor(p, device=dev)
    M = torch.zeros((N, N), dtype=torch.float64, device=dev)
    M[pt, pt] = t(diag)
    if N > 1:
        i = torch.arange(0, 2 * n_two, 2, device=dev)
        M[pt[i], pt[i + 1]] = t(off[0:2 * n_two:2])
        M[pt[i + 1], pt[i]] = t(off[0:2 * n_two:2])
    for k in range(reflectors):
        v = t(V[k] / np.linalg.norm(V[k]))
        Mv = M @ v
        c = v @ Mv
        # H M H = M - 2 v (M v)^T - 2 (M v) v^T + 4 (v^T M v) v v^T
        M -= 2.0 * (torch.outer(v, Mv) + torch.outer(Mv, v)) - 4.0 * c * torch.outer(v, v)
    M = 0.5 * (M + M.T)
    neg = n_two + n_neg1
    return M, (neg, 0, N - neg)
