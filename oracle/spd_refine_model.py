"""TEST INFRASTRUCTURE ONLY -- the condensed SPD solve of the quasi-Newton KKT path in numpy: what its equilibration computes to the bit,
when its refinement loop stops, and how far each of its stages may be from exact (Higham, Accuracy and Stability of Numerical Algorithms,
2nd ed., ch. 3, 10, 12, 14; the conventions of oracle/bounds.py).

The device sequence (hb_dense_equilibrate, hb_dense_condensed_factor, hb_dense_condensed_solve: k_spd_solve_coop or k_spd_solve_refine) is

    s = 1 / sqrt(diag(Nfact)),  Aeq_ij = (s_i Nfact_ij) s_j,  Aeq = R R^T
    x_0 = s .* solve(Aeq, s .* rhs)
    loop:  r_k = rhs - Nref x_k (one warp per row),  rho_k = ||r_k||_inf
           stop with rho_k reported as NaN when rho_k is not finite, else stop when rho_k < tol or k == max_refine
           x_{k+1} = x_k + s .* solve(Aeq, s .* r_k)

The handle passes Nfact = Nref = N, tol = 1e-8, max_refine = 3 (HiOp's solveWithRefin). A test that passes Nfact = (1 + eps) N makes the
loop a stationary iteration whose error contracts by eps / (1 + eps) per correction, so every exit can be placed with a margin of ~1 / eps.

Stage bound. Stage k solves Aeq y = s .* r_{k-1} (r_{-1} = rhs, exact); the test sees y only through x_k - x_{k-1}, and r_{k-1} only
exactly (rhs - Nref x_{k-1} evaluated in extended precision here). With y~ = fl(fl(x_k - x_{k-1}) / s):

    |s .* r - Aeq y~| <= theta gamma(7N+3) ((|Aeq| + |R||R^T|) |y| + |z|) + |Aeq| E_y + |s| e_r + u |z|,   z = fl(s .* r^),
    |y| <= |y~| + E_y,   E_y = gamma(4) (|y~| + |x_k| / |s|),   e_r = gamma(c + 1) |Nref| |x_{k-1}| + u |r|,  c = ceil(N / 32) + 6

theta gamma(7N+3) is the solve bound of bounds.solve_backward_ratio (factor, two triangular solves, explicit diagonal-block inverses);
E_y covers the three roundings between y and y~ (s .* y, the addition to x_{k-1}, the division here); e_r is the residual the kernel
computed against the exact one: each lane sums ceil(N / 32) products, a 5-level xor tree adds the lanes, rhs_i minus that sum rounds once.
The reported rho is within max_i e_r of the exact ||rhs - Nref x||_inf.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.bounds import U, gamma

LD = np.longdouble
U_LD = float(np.finfo(LD).eps) / 2.0    # unit roundoff of the extended-precision evaluation (x87: 2^-64; binary128: 2^-113)
ROW_BLOCK = 1024                         # rows per extended-precision block (the temporaries stay ROW_BLOCK x N)


def gamma_ld(c: float) -> float:
    return c * U_LD / (1.0 - c * U_LD)


# ---- bits ---------------------------------------------------------------------------------------------------------------------------
def equilibrate(Nfact):
    """(s, Aeq) as k_equilibrate computes them: s_i = 1 / sqrt(Nfact_ii), Aeq_ij = (s_i Nfact_ij) s_j on the upper triangle (row-major;
    the strict lower triangle of Aeq is zero here and not written by the kernel)."""
    Nfact = np.asarray(Nfact, dtype=np.float64)
    s = 1.0 / np.sqrt(np.diag(Nfact))
    return s, np.triu((s[None, :] * Nfact) * s[:, None])


def residual_chain(N: int) -> int:
    """longest addition chain of one residual entry: ceil(N / 32) products per lane, 5-level xor tree, 1 for the product"""
    return -(-N // 32) + 6


def inf_norm(r, drop_nan=False) -> float:
    """||r||_inf as the kernels take it: NaN when any entry is NaN. drop_nan: fmax's rule (a NaN operand is skipped), the old kernels'."""
    a = np.abs(np.asarray(r, dtype=np.float64))
    if drop_nan:
        a = a[~np.isnan(a)]
        return float(a.max(initial=0.0))
    return float(a.max(initial=0.0)) if not np.isnan(a).any() else math.nan


# ---- the loop -------------------------------------------------------------------------------------------------------------------------
MUTATIONS = ("unscaled_correction", "residual_vs_aeq", "strict_tol", "extra_correction", "missing_correction", "nan_dropped")


def refine(solve_eq, Aeq_full, Nref, rhs, s, tol, max_refine, mutation=None):
    """The device loop with solve_eq(z) solving Aeq y = z. Returns (xs, rhos, nref, rho_reported): xs[k] is x after k corrections,
    rhos[k] its residual norm as computed here. mutation (one of MUTATIONS): a planted mistake, for the test that the checks see it."""
    assert mutation in (None,) + MUTATIONS
    Nref = np.asarray(Nref, dtype=np.float64)
    A_res = Aeq_full if mutation == "residual_vs_aeq" else Nref
    scale = (lambda v: v) if mutation == "unscaled_correction" else (lambda v: v * s)
    limit = max_refine + (1 if mutation == "extra_correction" else -1 if mutation == "missing_correction" else 0)
    x = solve_eq(rhs * s) * s
    xs, rhos = [x], []
    nref = 0
    while True:
        r = rhs - A_res @ x
        rho = inf_norm(r, drop_nan=mutation == "nan_dropped")
        rhos.append(rho)
        if not math.isfinite(rho):
            return xs, rhos, nref, math.nan
        done = rho <= tol if mutation == "strict_tol" else rho < tol
        if done or nref >= limit:
            return xs, rhos, nref, rho
        x = x + scale(solve_eq(scale(r)))
        xs.append(x)
        nref += 1


def expected_exit(rhos, tol, max_refine):
    """(nref, reported rho) the exit rule gives for the residual norms rho_0, rho_1, ... of the iterates"""
    for k, rho in enumerate(rhos):
        if not math.isfinite(rho):
            return k, math.nan
        if rho < tol or k == max_refine:
            return k, rho
    raise AssertionError("the residual norms end before the loop does")


# ---- residuals in extended precision -------------------------------------------------------------------------------------------------
def _matvec_ld(A, x):
    """A x in extended precision, and the bound gamma_ld(n + 1) |A| |x| of its evaluation (A float64, x float64 or long double)"""
    A = np.asarray(A)
    x = np.asarray(x, dtype=LD)
    y = np.empty(A.shape[0], dtype=LD)
    for i0 in range(0, A.shape[0], ROW_BLOCK):
        y[i0:i0 + ROW_BLOCK] = A[i0:i0 + ROW_BLOCK].astype(LD) @ x
    return y


def residual_ld(Nref, rhs, x):
    """(r, err): r = rhs - Nref x in extended precision with |r - exact| <= err, and |Nref| |x| (float64, rounded up by the bound)"""
    ax = np.abs(Nref) @ np.abs(x)
    r = np.asarray(rhs, dtype=LD) - _matvec_ld(Nref, x)
    err = gamma_ld(Nref.shape[0] + 2) * (ax + np.abs(rhs)) * (1.0 + 4 * U)
    return r, err, ax


# ---- stage bounds ---------------------------------------------------------------------------------------------------------------------
def stage_ratio(Aeq_full, R, theta, s, Nref, rhs, x_prev, x_new):
    """max_i |s .* r - Aeq y~|_i / tol_i for one stage (<= 1 passes; 1 / ratio is the margin), see the module docstring.
    x_prev = None: the first solve (r = rhs exactly). Aeq_full: both triangles; R: the lower Cholesky factor the kernel computed."""
    N = Aeq_full.shape[0]
    if x_prev is None:
        r, r_err = np.asarray(rhs, dtype=LD), np.zeros(N)
        e_r = np.zeros(N)
        x_prev = np.zeros(N)
    else:
        r, r_err, ax = residual_ld(Nref, rhs, x_prev)
        e_r = gamma(residual_chain(N) + 1) * ax + U * np.abs(r.astype(np.float64))
    y = (x_new - x_prev) / s
    ay = np.abs(y)
    E_y = gamma(4) * (ay + np.abs(x_new) / np.abs(s))
    ay_up = ay + E_y
    aA = np.abs(Aeq_full)
    aR = np.abs(R)
    sr = np.abs(s) * np.abs(r.astype(np.float64))
    az = (sr + np.abs(s) * e_r) * (1.0 + U)                              # |s .* r^| rounded to z
    tol = theta * gamma(7 * N + 3) * (aA @ ay_up + aR @ (aR.T @ ay_up) + az) + aA @ E_y + np.abs(s) * e_r + U * az
    lhs = np.asarray(s, dtype=LD) * r - _matvec_ld(Aeq_full, y)
    ev = np.abs(s) * r_err + gamma_ld(N + 3) * (sr + aA @ ay)          # the extended-precision evaluation here, rounded up below
    tol = tol + ev * (1.0 + 4 * U)
    return float((np.abs(lhs).astype(np.float64) / np.maximum(tol, np.finfo(np.float64).tiny)).max())


def rho_ratio(Nref, rhs, x, rho_hat):
    """|rho^ - ||rhs - Nref x||_inf| over its bound max_i e_r,i (plus the evaluation here): <= 1 passes"""
    N = Nref.shape[0]
    r, r_err, ax = residual_ld(Nref, rhs, x)
    ar = np.abs(r)
    rho = ar.max()
    e_r = gamma(residual_chain(N) + 1) * ax + U * np.abs(r.astype(np.float64))
    tol = float((e_r + r_err).max()) * (1.0 + 4 * U) + float(r_err.max())
    return float(abs(LD(rho_hat) - rho)) / max(tol, np.finfo(np.float64).tiny)
