"""The exact references and error bounds of oracle/bounds.py: exact_dot is the correctly rounded exact dot product, the componentwise
SYRK bound accepts a correct FP64 condensation computed in another order, and it rejects the kinds of wrong kernels that the old
tolerance |N - N_ref| <= 1e-12 max|N| lets through on the synthetic problems (whose all-ones row 0 makes max|N| about 1e4 while every
other entry is about 0.3)."""
from fractions import Fraction

import numpy as np
import pytest

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko


def _frac_dot(a, b):
    return sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0))


@pytest.mark.parametrize("seed", range(6))
def test_exact_dot_is_correctly_rounded(seed):
    r = np.random.default_rng(seed)
    n = int(r.integers(1, 400))
    a = r.standard_normal(n) * 10.0 ** r.uniform(-8, 8, n)
    b = r.standard_normal(n) * 10.0 ** r.uniform(-8, 8, n)
    if seed % 2:
        # heavy cancellation: the exact result is many orders below sum |a_i b_i|
        a = np.concatenate([a, -a, [1e-3]])
        b = np.concatenate([b, b, [3.0]])
    want = _frac_dot(a, b)
    got = bounds.exact_dot(a, b)
    assert got == float(want)          # Fraction -> float rounds to nearest
    assert bounds.exact_sum(a) == float(sum((Fraction(float(v)) for v in a), Fraction(0)))


def test_exact_rows_and_cols_against_fractions():
    r = np.random.default_rng(7)
    A = r.standard_normal((9, 37)) * 10.0 ** r.uniform(-5, 5, (9, 37))
    x, y = r.standard_normal(37), r.standard_normal(9)
    rows = bounds.exact_rows(A, x)
    for i in range(9):
        assert rows[i] == float(_frac_dot(A[i], x))
    cols = bounds.exact_cols(A, y)
    terms = (np.abs(A) * np.abs(y)[:, None]).sum(axis=0)
    for k in range(37):
        exact = float(_frac_dot(A[:, k], y))
        assert abs(cols[k] - exact) <= bounds.cols_ref_error(9, exact, terms[k]), k


def test_gamma_and_reduction_chain():
    assert bounds.gamma(1) == pytest.approx(bounds.U, rel=1e-15)
    assert bounds.gamma(1000) > 1000 * bounds.U
    # hb_grid clamp at 132 SMs: 1056 CTAs of 256 threads; one item per thread below it
    assert bounds.stream_grid(540672, 132) == 1056 and bounds.stream_grid(270336, 132) == 1056 and bounds.stream_grid(1, 132) == 1
    assert bounds.reduction_chain(270336, 1056) == 1 + 10 + 5 + 10
    assert bounds.reduction_chain(270337, 1056) == 2 + 10 + 5 + 10


def _condensation_inputs(n, m):
    P = synth.make_qn_problem(n, m, 0, seed=3 + n % 89)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    return P.J, DhInv


def _w_reordered(J, d, parts=5):
    """J diag(d) J^T summed over column blocks in reverse order: a different but equally valid FP64 evaluation."""
    K = J.shape[1]
    edges = np.linspace(0, K, parts + 1).astype(int)
    W = np.zeros((J.shape[0], J.shape[0]))
    for q in reversed(range(parts)):
        s = slice(edges[q], edges[q + 1])
        W += (J[:, s] * d[s]) @ J[:, s].T
    return W


@pytest.fixture(scope="module")
def case():
    n, m = 20003, 251
    J, d = _condensation_inputs(n, m)
    W = (J * d) @ J.T
    return dict(n=n, m=m, J=J, d=d, W=W, B=bounds.syrk_bound(J, d))


def _ratio(Wt, case):
    """max over the entries outside the 128 x 128 tile holding row / column 0 of |Wt - W| / bound"""
    tol = bounds.syrk_tol(case["B"], case["n"], case["W"], c_kernel=case["n"] + 2 + 132)
    r = np.abs(Wt - case["W"]) / tol
    return float(r[128:, 128:].max())


def test_bound_accepts_fp64_in_another_order(case):
    W2 = _w_reordered(case["J"], case["d"])
    tol = bounds.syrk_tol(case["B"], case["n"], case["W"], c_kernel=case["n"] + 2 + 132)
    ratio = float((np.abs(W2 - case["W"]) / tol).max())
    print(f"reordered FP64 W: error / bound = {ratio:.2e}")
    assert ratio <= 1.0


def test_bound_rejects_the_simulated_kernel_mutations(case):
    J, d, W, m = case["J"], case["d"], case["W"], case["m"]
    old_tol = 1e-12 * np.abs(W).max()
    # (1) DhInv rounded to FP32 in the tiles that do not hold row 0 (tile rows ti >= 1: rows and columns from 128 on)
    d32 = d.astype(np.float32).astype(np.float64)
    W1 = W.copy()
    W1[128:, 128:] = (J[128:] * d32) @ J[128:].T
    # (2) the result stored through a float in those tiles
    W2 = W.copy()
    W2[128:, 128:] = W2[128:, 128:].astype(np.float32).astype(np.float64)
    # (3) one K column dropped in those tiles
    k = case["n"] // 2
    W3 = W.copy()
    drop = np.outer(J[:, k], J[:, k]) * d[k]
    W3[128:, 128:] -= drop[128:, 128:]
    for name, Wm, factor in (("fp32 DhInv", W1, 100.0), ("fp32 store", W2, 100.0), ("dropped column", W3, 1e7)):
        err = np.abs(Wm - W)
        r = _ratio(Wm, case)
        print(f"{name}: error / bound = {r:.2e}; old check {'passes' if err.max() <= old_tol else 'fails'}")
        assert r > factor, (name, r)
    # the gap the componentwise bound closes: the old check cannot see the FP32 DhInv
    assert np.abs(W1 - W).max() <= old_tol


# ---- dense symmetric factorizations: the bounds accept LAPACK's factors and solves and reject wrong ones ----------------------------
from scipy.linalg import lapack  # noqa: E402

from oracle import bk_model  # noqa: E402


def _spd(N, seed):
    r = np.random.default_rng(seed)
    G = r.standard_normal((N, N // 2 + 1))
    return G @ G.T / N + np.diag(r.uniform(0.5, 2.0, N))


def _family(N, seed, n_two=None):
    M, inertia = bounds.known_inertia_matrix(N, N // 3 if n_two is None else n_two, N // 7, seed)
    return M.numpy(), inertia


def _sytrf(M):
    ldu, ipiv, info = lapack.dsytrf(np.asfortranarray(np.tril(M)), lower=1)
    assert info == 0
    return ldu, ipiv


def _bk_inertia(d, dsub):
    """inertia of D: a 2 x 2 block [[a, s], [s, c]] has det < 0 (one of each sign) under Bunch-Kaufman's choice of it"""
    neg = pos = 0
    k = 0
    while k < d.shape[0]:
        if k + 1 < d.shape[0] and dsub[k] != 0.0:
            det = d[k] * d[k + 1] - dsub[k] ** 2
            ev = np.linalg.eigvalsh(np.array([[d[k], dsub[k]], [dsub[k], d[k + 1]]]))
            assert det < 0
            neg += int((ev < 0).sum())
            pos += int((ev > 0).sum())
            k += 2
        else:
            neg += int(d[k] < 0)
            pos += int(d[k] > 0)
            k += 1
    return neg, 0, pos


@pytest.mark.parametrize("N", [97, 256])
def test_known_inertia_family(N):
    """inertia by construction equals the eigenvalue count and the inertia of dsytrf's D; at least N/4 2 x 2 pivots, interchange
    partners far outside any panel, and 2 x 2 blocks across 32- and 64-column boundaries"""
    M, inertia = _family(N, seed=N)
    ev = np.linalg.eigvalsh(M)
    assert (int((ev < 0).sum()), 0, int((ev > 0).sum())) == inertia
    assert np.abs(ev).min() > 0.3
    ldu, ipiv = _sytrf(M)
    L, d, dsub, perm = bounds.lapack_to_permuted(ldu, ipiv)
    assert _bk_inertia(d, dsub) == inertia
    two = np.nonzero(dsub)[0]
    assert two.size >= N // 4
    assert (np.abs(np.abs(ipiv) - 1 - np.arange(N)) > min(64, N // 3)).sum() >= N // 8
    assert any(k % 32 == 31 for k in two) and (N < 128 or any(k % 64 == 63 for k in two))


@pytest.mark.parametrize("N", [1, 2, 40, 161])
def test_lapack_to_permuted_and_perm_from_ipiv(N):
    M, _ = _family(N, seed=3 * N + 1)
    ldu, ipiv = _sytrf(M)
    L, d, dsub, perm = bounds.lapack_to_permuted(ldu, ipiv)
    assert np.array_equal(perm, bounds.perm_from_ipiv(ipiv))
    assert bounds.factor_backward_ratio(M[np.ix_(perm, perm)], L, d, dsub) <= 1.0
    # the numpy model of the cluster kernel (same output form) maps onto the same LAPACK pivots
    Lm, dm, dsubm, permm, ipivm, info = bk_model.factor(M, NB=32)
    assert info == 0
    assert np.array_equal(bounds.bk_cluster_to_lapack(ipivm, permm, dsubm), ipiv)
    assert np.array_equal(permm, perm)
    if N > 2:
        bad = permm.copy()
        bad[[0, 1]] = bad[[1, 0]]
        with pytest.raises(AssertionError):
            bounds.bk_cluster_to_lapack(ipivm, bad, dsubm)


def test_bounds_accept_lapack_factors_and_solves():
    """dpotrf / dpotrs and dsytrf / dsytrs through the helpers, CPU and torch FP64 evaluation alike"""
    import torch
    for N in (33, 300):
        A = _spd(N, N)
        R, info = lapack.dpotrf(A, lower=1)
        assert info == 0
        L = np.tril(R)
        one = np.ones(N)
        fr = bounds.factor_backward_ratio(A, L, one)
        b = np.random.default_rng(1).standard_normal((N, 3))
        x, info = lapack.dpotrs(R, b, lower=1)
        sr, om = bounds.solve_backward_ratio(A, x, b, L, one)
        tA, tL, tx, tb = (torch.from_numpy(np.ascontiguousarray(v)) for v in (A, L, x, b))
        sr_t, _ = bounds.solve_backward_ratio(tA, tx, tb, tL, torch.ones(N, dtype=torch.float64))
        print(f"dpotrf N={N}: factor {fr:.2e}, solve {sr:.2e} (torch {sr_t:.2e}), omega {om:.1e}")
        assert fr <= 1.0 and sr <= 1.0 and sr_t <= 1.0 and om < 10 * N * bounds.U
        M, _ = _family(N, seed=N + 5)
        ldu, ipiv = _sytrf(M)
        Lb, d, dsub, perm = bounds.lapack_to_permuted(ldu, ipiv)
        PAP = M[np.ix_(perm, perm)]
        x, info = lapack.dsytrs(ldu, ipiv, b, lower=1)
        assert info == 0
        sr, om = bounds.solve_backward_ratio(PAP, x[perm], b[perm], Lb, d, dsub)
        fr = bounds.factor_backward_ratio(PAP, Lb, d, dsub)
        print(f"dsytrf N={N}: factor {fr:.2e}, solve {sr:.2e}, omega {om:.1e}")
        assert fr <= 1.0 and sr <= 1.0


def test_theta_of_explicit_inverses():
    assert bounds.block_theta(np.eye(70), 16) == 1.0
    L = np.tril(np.random.default_rng(2).uniform(-1, 1, (64, 64)), -1) + np.eye(64)
    assert bounds.block_theta(L, 16) > bounds.block_theta(L, 1) == 1.0


# margins the factor bound must reject by (ratio = error / bound); measured values are printed
MUTATION_MARGINS = {"L entry off by 1e3 u": 3.0, "tile without its last 16-column K chunk": 1e6, "2x2 dsub with the wrong sign": 1e6,
                    "two adjacent ipiv entries swapped": 1e6}


def test_factor_bound_rejects_mutations():
    ratios = {}
    # (1) one entry of a Cholesky factor off by 1e3 u relative (column 0, where L L^T carries that entry alone)
    N = 32
    A = _spd(N, 4)
    R, _ = lapack.dpotrf(A, lower=1)
    L = np.tril(R)
    Lm = L.copy()
    i = int(np.argmax(np.abs(L[1:, 0]))) + 1
    Lm[i, 0] *= 1.0 + 1e3 * bounds.U
    assert bounds.factor_backward_ratio(A, L, np.ones(N)) <= 1.0
    ratios["L entry off by 1e3 u"] = bounds.factor_backward_ratio(A, Lm, np.ones(N))
    # (2) a trailing-update tile (rows 64..127 x columns 0..63 of the Schur complement after 32 columns) that skips the last 16-column K
    # chunk of the update: the factor is then an exact factor of A plus that chunk's contribution on the tile
    N = 192
    A = _spd(N, 5)
    R, _ = lapack.dpotrf(A, lower=1)
    L = np.tril(R)
    E = np.zeros((N, N))
    rows, cols, ks = slice(96, 160), slice(32, 96), slice(16, 32)
    E[rows, cols] = L[rows, ks] @ L[cols, ks].T
    E = np.tril(E, -1)
    E = E + E.T
    Rm, info = lapack.dpotrf(A + E, lower=1)
    assert info == 0
    ratios["tile without its last 16-column K chunk"] = bounds.factor_backward_ratio(A, np.tril(Rm), np.ones(N))
    # (3) / (4) a Bunch-Kaufman factor with one 2 x 2 off-diagonal negated, or with two adjacent 1 x 1 interchanges swapped
    N = 200
    M, _ = _family(N, seed=9)
    ldu, ipiv = _sytrf(M)
    Lb, d, dsub, perm = bounds.lapack_to_permuted(ldu, ipiv)
    k = int(np.nonzero(dsub)[0][0])
    ds = dsub.copy()
    ds[k] = -ds[k]
    ratios["2x2 dsub with the wrong sign"] = bounds.factor_backward_ratio(M[np.ix_(perm, perm)], Lb, d, ds)
    one = [j for j in range(N - 1) if ipiv[j] > 0 and ipiv[j + 1] > 0 and ipiv[j] != ipiv[j + 1]
           and (j == 0 or ipiv[j - 1] > 0 or ipiv[j - 2] < 0)]
    assert one
    j = one[0]
    ip = ipiv.copy()
    ip[[j, j + 1]] = ip[[j + 1, j]]
    Lw, dw, dsubw, permw = bounds.lapack_to_permuted(ldu, ip)
    ratios["two adjacent ipiv entries swapped"] = bounds.factor_backward_ratio(M[np.ix_(permw, permw)], Lw, dw, dsubw)
    for name, r in ratios.items():
        print(f"mutation {name}: error / bound = {r:.3g} (must exceed {MUTATION_MARGINS[name]:g})")
    for name, r in ratios.items():
        assert r > MUTATION_MARGINS[name], (name, r)
