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
