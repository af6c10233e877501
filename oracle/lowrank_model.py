"""TEST INFRASTRUCTURE ONLY -- the compact-BFGS stages that follow C_aug (hb_lowrank.cu), restated in numpy, with an error bound per stage.

Every stage is checked against the exact operation applied to that stage's own inputs as read back from the device, so no bound depends
on how well conditioned V is:

- k_build_V, k_build_Mdirect and k_build_U round every operation explicitly: build_V, build_M and build_U give their bits;
- the factors of V and M: LAPACK's pivots (dsytrf with lwork = N runs the unblocked DSYTF2 that k_sytf2 restates) and
  bounds.factor_backward_ratio; Z = U V^-1 and the 2l-vector p of each low-rank solve: bounds.solve_backward_ratio;
- N = W - U Z^T + blkdiag(0, Dd_inv), the fused rhs and the x-side applications: sums of products, held to gamma_c of their chain
  against a compensated reference (sum2);
- the multi-dot q = [sigma S (w.x); Y (w.x)] that feeds a low-rank solve: the two-stage reduction's chain (multidot_chain).
"""
from __future__ import annotations

import numpy as np

from . import bounds
from .bounds import U, gamma


# ---- the builders (explicit roundings, so numpy's elementwise FP64 operations give the same bits) --------------------------------------
def build_V(C, m: int, l: int, sigma: float, SSt, L, D, mutate: str | None = None):
    """k_build_V: V = [[sigma^2 C_SS - sigma S S^T, sigma C_SY - L], [(sigma C_SY - L)^T, C_YY + diag(D)]] as the kernel forms it from
    C_aug (Ma x Ma), S S^T, L (L_ij = s_i^T y_j, i > j) and D. mutate="L" puts L^T where the kernel reads L (a test of the test)."""
    s = np.float64(sigma)
    CSS = C[m:m + l, m:m + l]
    CSY = C[m:m + l, m + l:m + 2 * l]
    CYY = C[m + l:m + 2 * l, m + l:m + 2 * l]
    LSY = L.T if mutate == "L" else L          # V[a][l + j] = sigma C[m+a][m+l+j] - L[a][j]
    V = np.empty((2 * l, 2 * l))
    V[:l, :l] = (s * s) * CSS - s * SSt
    V[:l, l:] = s * CSY - LSY
    V[l:, :l] = (s * C[m:m + l, m + l:m + 2 * l] - LSY).T
    V[l:, l:] = CYY + np.diag(D)
    return V


def build_M(l: int, sigma: float, SSt, L, D):
    """k_build_Mdirect: M = [[sigma S S^T, L], [L^T, -diag(D)]]."""
    M = np.zeros((2 * l, 2 * l))
    M[:l, :l] = np.float64(sigma) * SSt
    M[:l, l:] = L
    M[l:, :l] = L.T
    M[np.arange(l, 2 * l), np.arange(l, 2 * l)] = -np.asarray(D)
    return M


def build_U(C, m: int, l: int, sigma: float, drop_sigma: bool = False):
    """k_build_U: U = [sigma C_JS, C_JY] (m x 2l). drop_sigma: the S1 block without sigma (a test of the test)."""
    Ub = C[:m, m:m + 2 * l].copy()
    if not drop_sigma:
        Ub[:, :l] = np.float64(sigma) * Ub[:, :l]
    return Ub


# ---- compensated reference of a sum of products -----------------------------------------------------------------------------------------
def sum2(terms):
    """sum_t a_t * b_t, elementwise over the broadcast shape of the pairs (a_t, b_t): TwoProduct per term and a compensated cascade
    (Ogita, Rump and Oishi, alg. 4.4), as accurate as twice the working precision. Returns (value, bound on its own error):
    |value - exact| <= u |value| + gamma(2T)^2 sum |a||b| (bounds.cols_ref_error with 2T terms)."""
    s = c = mag = None
    for a, b in terms:
        p, e = bounds.two_product(*np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)))
        if s is None:
            s, c, mag = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
        mag = mag + np.abs(p)
        for t in (p, e):
            z = s + t
            bb = z - s
            c = c + ((s - (z - bb)) + (t - bb))
            s = z
    v = s + c
    T = max(len(terms), 1)
    return v, U * np.abs(v) + gamma(2 * T) ** 2 * mag * (1 + 4 * U)


def _ratio(err, tol):
    return float((np.abs(err) / np.maximum(tol, np.finfo(np.float64).tiny)).max(initial=0.0))


# ---- stage bounds ---------------------------------------------------------------------------------------------------------------------
def factor_check(A, F_colmajor, ipiv):
    """The Bunch-Kaufman factor of A as k_sytf2 leaves it (LAPACK's lower layout): (factor_backward_ratio, number of 2 x 2 pivots,
    the permuted form (L, d, dsub, perm))."""
    L, d, dsub, perm = bounds.lapack_to_permuted(np.tril(F_colmajor), np.asarray(ipiv))
    PAP = A[np.ix_(perm, perm)]
    r = bounds.factor_backward_ratio(PAP, L, d, dsub)
    return r, int((np.asarray(ipiv) < 0).sum()) // 2, (L, d, dsub, perm)


def solve_ratio(A, fac, x, b, extra=0.0):
    """bounds.solve_backward_ratio for A x = b through fac = (L, d, dsub, perm) from factor_check; x, b: N or N x k (one rhs per column);
    extra: bound on the error of the rhs the kernel solved with (N or N x 1)."""
    L, d, dsub, perm = fac
    N = A.shape[0]
    x = np.asarray(x).reshape(N, -1)[perm]
    b = np.asarray(b).reshape(N, -1)[perm]
    ex = np.asarray(extra, dtype=np.float64)
    if ex.ndim:
        ex = ex.reshape(N, -1)[perm]
    return bounds.solve_backward_ratio(A[np.ix_(perm, perm)], x, b, L, d, dsub, extra=ex)


def n_ratio(N, W, Ub, Z, Dd_inv, meq: int):
    """k_form_N on the upper triangle against W - U Z^T + blkdiag(0, Dd_inv):
    |N - ref| <= gamma(2l + 2) (|W| + |U||Z|^T) + u |Dd_inv| (+ the reference's own error)."""
    m, n2 = Ub.shape
    dd = np.zeros(m)
    dd[meq:] = Dd_inv
    terms = [(W, 1.0)] + [(Ub[:, q:q + 1], -Z[None, :, q]) for q in range(n2)] + [(np.diag(dd), 1.0)]
    ref, ref_err = sum2(terms)
    tol = gamma(n2 + 2) * (np.abs(W) + np.abs(Ub) @ np.abs(Z).T) + U * np.diag(np.abs(dd)) + ref_err
    iu = np.triu_indices(m)
    return _ratio((N - ref)[iu], tol[iu])


def fused_rhs_ratio(rhs, tdot, Z, sigma: float, ry, m: int, l: int):
    """k_fused_rhs: rhs_i = tdot_i - sum_q Z_iq p_q - ry_i, p = [fl(sigma tdot_S); tdot_Y] as the kernel forms it:
    |rhs - ref| <= gamma(2l + 2) (|tdot_J| + |Z||p| + |ry|)."""
    p = np.concatenate([np.float64(sigma) * tdot[m:m + l], tdot[m + l:m + 2 * l]])
    terms = [(tdot[:m], 1.0), (ry, -1.0)] + [(Z[:, q], -p[q]) for q in range(2 * l)]
    ref, ref_err = sum2(terms)
    tol = gamma(2 * l + 2) * (np.abs(tdot[:m]) + np.abs(Z) @ np.abs(p) + np.abs(ry)) + ref_err
    return _ratio(rhs - ref, tol)


def multidot_chain(n: int, grid: int) -> int:
    """Longest rounding chain of multidot (hb_lowrank.cu): w x rounded, one product and ceil(n / (grid 256)) additions per thread, the
    256-thread block sum, then k_multidot_final's 128 threads over the grid partials and its block sum, then the scale by sigma."""
    return bounds.reduction_chain(n, grid, 256, 128) + 3


def multidot_exact(S, Y, w, x, sigma: float):
    """q = [sigma S t; Y t] with t = fl(w x) (as the kernel rounds it; w None means 1), from exact dots, and the magnitudes
    [sigma |S||t|; |Y||t|] its error bound scales with."""
    t = x if w is None else w * x
    rows = np.vstack([S, Y])
    q = bounds.exact_rows(rows, t)
    mag = np.abs(rows) @ np.abs(t)
    l = S.shape[0]
    q[:l] *= sigma
    mag[:l] *= sigma
    return q, mag


def apply_ratio(out, r, S, Y, p, sigma: float, w=None, diag=None, beta: float = 0.0, y0=None, alpha: float = 1.0, p_sigma: bool = True):
    """k_lowrank_apply against the exact operation on the read-back p:
        w given:  out = w (r - sigma S^T p_S - Y^T p_Y)                                       (hess_solve)
        else:     out = beta y0 + alpha ((sigma + diag) r - sigma S^T p_S - Y^T p_Y)          (hess_times_vec, diag = Dx or 0)
    |out - ref| <= gamma(l + 6) (|beta y0| + |alpha| |w| (|c r| + sigma |S|^T|p_S| + |Y|^T|p_Y|)). p_sigma=False drops sigma from the
    reference's S term (a test of the test)."""
    l = S.shape[0]
    sg = np.float64(sigma)
    ps = sg * p[:l] if p_sigma else p[:l]
    corr_terms = [(S[q], -ps[q]) for q in range(l)] + [(Y[q], -p[l + q]) for q in range(l)]
    mag = sg * (np.abs(S).T @ np.abs(p[:l])) + np.abs(Y).T @ np.abs(p[l:])
    if w is not None:
        inner, e1 = sum2([(r, 1.0)] + corr_terms)
        ref = w * inner
        tol = gamma(l + 6) * np.abs(w) * (np.abs(r) + mag) + np.abs(w) * e1 + U * np.abs(ref)
    else:
        dg = np.zeros_like(r) if diag is None else diag
        inner, e1 = sum2([(r, sg), (r, dg)] + corr_terms)
        by = beta * y0 if beta != 0.0 else np.zeros_like(r)
        ref = by + alpha * inner
        tol = gamma(l + 6) * (np.abs(by) + abs(alpha) * ((sg + dg) * np.abs(r) + mag)) + abs(alpha) * e1 + 2 * U * np.abs(ref)
    return _ratio(out - ref, tol)
