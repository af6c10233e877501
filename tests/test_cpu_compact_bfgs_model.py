"""The compact-BFGS stage model (oracle/lowrank_model.py) on the CPU: every stage bound holds on a numpy run of the stages and is not
vacuous, and each of five planted mistakes breaks a bound or the builders' bits. The GPU side is tests/test_gpu_compact_bfgs.py."""
import numpy as np
import pytest
from scipy.linalg import lapack

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko
from oracle import lowrank_model as lm


def _stages(n=600, m=6, l=5, dx0=False, sigma=1.0, seed=3):
    """One condensation and both low-rank solves, stage by stage in numpy / LAPACK (the device's operations, other rounding)."""
    P = synth.make_qn_problem(n, m, l, sigma=sigma, seed=seed)
    if dx0:
        P.ixl[:] = 0.0
        P.ixu[:] = 0.0
    Dx, DhInv, _, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, sigma)
    R = np.vstack([P.J, P.St, P.Yt])
    C = (R * DhInv) @ R.T
    C = np.triu(C) + np.triu(C, 1).T                          # symmetric, as the device's C_aug
    SSt = P.St @ P.St.T
    V = lm.build_V(C, m, l, sigma, SSt, P.L, P.D)
    F, ipiv, info = lapack.dsytrf(V, lower=1, lwork=2 * l)
    assert info == 0
    Ub = lm.build_U(C, m, l, sigma)
    Z, info = lapack.dsytrs(F, ipiv, Ub.T.copy(), lower=1)
    Z = np.ascontiguousarray(Z.T)
    N = C[:m, :m] - Ub @ Z.T
    N[np.arange(P.m_eq, m), np.arange(P.m_eq, m)] += Dd_inv
    N = np.triu(N) + np.triu(N, 1).T
    r = np.random.default_rng(seed).standard_normal(n)
    q, _ = lm.multidot_exact(P.St, P.Yt, DhInv, r, sigma)
    p, _ = lapack.dsytrs(F, ipiv, q, lower=1)
    x = DhInv * (r - sigma * (P.St.T @ p[:l]) - P.Yt.T @ p[l:])
    return dict(P=P, DhInv=DhInv, Dd_inv=Dd_inv, C=C, SSt=SSt, V=V, F=F, ipiv=ipiv, Ub=Ub, Z=Z, N=N, r=r, q=q, p=p, x=x, sigma=sigma,
                m=m, l=l)


def _ipiv0(ipiv):
    """scipy returns LAPACK's 1-based pivots as given: keep them (lapack_to_permuted reads that convention)"""
    return np.asarray(ipiv)


@pytest.mark.parametrize("dx0", [False, True])
def test_stage_bounds_hold_and_are_not_vacuous(dx0):
    s = _stages(dx0=dx0)
    P, m, l = s["P"], s["m"], s["l"]
    rf, n22, fac = lm.factor_check(s["V"], s["F"], _ipiv0(s["ipiv"]))
    rz, _ = lm.solve_ratio(s["V"], fac, s["Z"].T, s["Ub"].T)
    rn = lm.n_ratio(s["N"], s["C"][:m, :m], s["Ub"], s["Z"], s["Dd_inv"], P.m_eq)
    rp, _ = lm.solve_ratio(s["V"], fac, s["p"], s["q"])
    rx = lm.apply_ratio(s["x"], s["r"], P.St, P.Yt, s["p"], s["sigma"], w=s["DhInv"])
    ratios = dict(factor=rf, Z=rz, N=rn, p=rp, x=rx)
    print(f"dx0={dx0}: 2x2 pivots {n22}, margins " + ", ".join(f"{kk} {1 / max(v, 1e-300):.3g}" for kk, v in ratios.items()))
    for kk, v in ratios.items():
        assert v <= 1.0, (kk, v)
    # the summation stages are held to gamma of their chain: a numpy run reaches at least 1 % of that
    assert rn >= 1e-2 and rx >= 1e-2, ratios
    if dx0:
        # V_SS is pure cancellation (rounding noise): the first pivot cannot be V_11 in place. Bunch-Kaufman takes the large diagonal of
        # V_YY by an interchange instead (|V_YY,aa| >= D_a = s_a^T y_a >= alpha |V_SY| entries of that row here), so no 2 x 2 pivot
        assert _ipiv0(s["ipiv"])[0] != 1


def test_builders_restate_the_formulas():
    s = _stages()
    P, m, l, sg = s["P"], s["m"], s["l"], s["sigma"]
    V = s["V"]
    assert np.array_equal(V, V.T)
    # against the reference's one-Gram form, up to rounding
    Vref = ko.build_V(P.St, P.Yt, P.L, P.D, sg, s["DhInv"])
    iu = np.triu_indices(2 * l)
    assert np.abs(V - Vref)[iu].max() <= 1e-12 * np.abs(Vref).max()
    M = lm.build_M(l, sg, s["SSt"], P.L, P.D)
    assert np.array_equal(M, M.T) and np.array_equal(np.diag(M)[l:], -P.D)


def test_mutations_break_a_bound_or_the_bits():
    s = _stages(dx0=True)
    P, m, l, sg = s["P"], s["m"], s["l"], 1.0
    C = s["C"]
    # L in place of L^T in V_SY
    assert not np.array_equal(lm.build_V(C, m, l, sg, s["SSt"], P.L, P.D, mutate="L"), s["V"])
    # sigma dropped from S1 (needs sigma != 1 to show)
    s2 = _stages(sigma=3.0)
    assert not np.array_equal(lm.build_U(s2["C"], m, l, 3.0, drop_sigma=True), s2["Ub"])
    # one skipped 2 x 2 interchange, on a matrix whose factorization is made of them
    A = bounds.known_inertia_matrix(40, 16, 3, seed=5)[0].numpy()
    F, ipiv, info = lapack.dsytrf(A, lower=1, lwork=40)
    assert info == 0 and lm.factor_check(A, F, ipiv)[0] <= 1.0
    ipiv = _ipiv0(ipiv).copy()
    k = next(i for i in range(0, 39) if ipiv[i] < 0 and -ipiv[i] - 1 != i + 1)
    ipiv[k] = ipiv[k + 1] = -(k + 2)
    assert lm.factor_check(A, F, ipiv)[0] > 1.0
    # the last column of U Z^T dropped
    Nbad = s["C"][:m, :m] - s["Ub"][:, :-1] @ s["Z"][:, :-1].T
    Nbad[np.arange(P.m_eq, m), np.arange(P.m_eq, m)] += s["Dd_inv"]
    assert lm.n_ratio(Nbad, s["C"][:m, :m], s["Ub"], s["Z"], s["Dd_inv"], P.m_eq) > 1.0
    # p_S applied without sigma (sigma != 1)
    assert lm.apply_ratio(s2["x"], s2["r"], s2["P"].St, s2["P"].Yt, s2["p"], 3.0, w=s2["DhInv"], p_sigma=False) > 1.0


def test_sum2_is_twice_working_precision():
    r = np.random.default_rng(0)
    a, b = r.standard_normal(500), r.standard_normal(500)
    v, err = lm.sum2([(a[i], b[i]) for i in range(500)])
    assert abs(v - bounds.exact_dot(a, b)) <= err
