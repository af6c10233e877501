"""The numpy model of the random butterfly transform of hb_symdense_dist's safe mode (oracle/rbt_model.py): its pairing, the
conditioning and exact symmetry of U^T A U, diagonals that depend on N alone, and the inertia the no-pivot LDL^T of A' gives against
numpy's eigenvalues and LAPACK's Bunch-Kaufman DSYTRF, with the refined solve on every family."""
import pathlib

import numpy as np
import pytest

from oracle import rbt_model as rbt

GOLDEN = pathlib.Path(__file__).parent / "golden"
COND_U_MAX = 3.0     # butterflies are orthogonal up to the diagonals in [15/16, 17/16) and an unpaired row's missing 1/sqrt(2)


@pytest.mark.parametrize("N", [1, 2, 3, 127, 128, 129, 4099])
def test_pairing_covers_every_row_once_per_level(N):
    for level in (1, 2):
        lo, hi, s, paired, f = rbt.level_maps(N, level)
        p = rbt.partner(N, level)
        assert np.array_equal(p[p], np.arange(N))                         # an involution
        seen = np.zeros(N, dtype=int)
        for i in range(N):
            if lo[i] == i:
                seen[i] += 1
                if hi[i] != i:
                    seen[hi[i]] += 1
        assert (seen == 1).all()
        unpaired = np.nonzero(~paired)[0]
        odd = [(o, n) for o, n, _ in rbt.segments(N, level) if n % 2 == 1]
        assert sorted(unpaired.tolist()) == sorted(o + (n + 1) // 2 - 1 for o, n in odd)
        assert (s[paired & (lo != np.arange(N))] == -1.0).all() and (s[lo == np.arange(N)] == 1.0).all()


@pytest.mark.parametrize("N", [1, 2, 3, 127, 128, 129, 300])
def test_U_nonsingular_and_well_conditioned(N):
    U = rbt.U_matrix(N)
    assert np.linalg.cond(U) < COND_U_MAX
    # U^T as the model applies it to vectors is the transpose of U
    assert np.allclose(rbt.apply_UT(np.eye(N)), U.T, rtol=0, atol=1e-15)


@pytest.mark.parametrize("N", [1, 2, 3, 127, 128, 129, 300])
def test_transform_is_exactly_symmetric_and_is_UT_A_U(N):
    r = np.random.default_rng(N)
    A = r.standard_normal((N, N))
    A = A + A.T
    Ap = rbt.transform(np.triu(A))                   # only the upper triangle is read
    assert np.array_equal(Ap.view(np.uint64), Ap.T.view(np.uint64))
    U = rbt.U_matrix(N)
    assert np.abs(Ap - U.T @ A @ U).max() <= 1e-13 * max(1.0, np.abs(A).max())


@pytest.mark.parametrize("N", [1, 2, 3, 128, 129, 4099])
def test_diagonals_depend_on_N_only_and_are_dyadic(N):
    for level in (1, 2):
        a, b = rbt.level_maps(N, level)[4], rbt.level_maps(N, level)[4]
        assert np.array_equal(a, b)
        assert ((a >= 15 / 16) & (a < 17 / 16)).all()
        assert np.array_equal(a * 2.0 ** 23, np.round(a * 2.0 ** 23))
    # the first butterfly of a level depends on its order only through its length: a prefix of a longer one
    assert np.array_equal(rbt.diagonal(1, 0, N), rbt.diagonal(1, 0, N + 77)[:N])


def random_indefinite(N, seed):
    """Q diag(lam) Q^T with |lam| in [1e-3, 10], about a third negative"""
    r = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(r.standard_normal((N, N)))
    lam = np.exp(r.uniform(np.log(1e-3), np.log(10.0), N)) * np.where(r.random(N) < 0.35, -1.0, 1.0)
    A = (Q * lam) @ Q.T
    return 0.5 * (A + A.T)


def golden(name, key):
    M = np.load(GOLDEN / name)[key]
    U = np.triu(M)
    return U + np.triu(U, 1).T


def saddle(n, m, seed, zeros):
    """[[H, J^T], [J, 0]] with H symmetric and `zeros` exact zeros on its diagonal, the first at (0, 0)"""
    r = np.random.default_rng(seed)
    H = r.standard_normal((n, n))
    H = H + H.T
    H[np.diag_indices(n)] += 2.0
    idx = np.concatenate([[0], r.choice(np.arange(1, n), zeros - 1, replace=False)])
    H[idx, idx] = 0.0
    J = r.standard_normal((m, n))
    return np.block([[H, J.T], [J, np.zeros((m, m))]])


def families():
    for N, seed in ((40, 1), (97, 2), (150, 3), (260, 4)):
        yield f"random{N}", random_indefinite(N, seed)
    yield "mds_golden", golden("mds_nxs50_nxd20.npz", "ref_M")
    yield "densekkt_M0", golden("densekkt_nx30.npz", "ref_M0")
    yield "densekkt_M1", golden("densekkt_nx30.npz", "ref_M1")
    for n, m, seed, z in ((30, 10, 5, 4), (90, 40, 6, 20), (129, 60, 7, 40)):
        yield f"saddle{n}_{m}", saddle(n, m, seed, z)


FAMILIES = dict(families())


@pytest.mark.parametrize("name", list(FAMILIES))
def test_model_inertia_matches_eigenvalues_and_dsytrf(name):
    A = FAMILIES[name]
    lam = np.linalg.eigvalsh(A)
    assert np.abs(lam).min() > 1e-8 * np.abs(lam).max()           # the family is nonsingular: the counts below are well defined
    neg = int((lam < 0).sum())
    assert rbt.dsytrf_inertia(A) == (neg, 0, A.shape[0] - neg)
    _, d, ret = rbt.nopiv_ldlt(rbt.transform(A))
    assert ret == neg and rbt.inertia_counts(d) == (neg, 0, A.shape[0] - neg)
    if name.startswith("saddle"):
        assert rbt.nopiv_ldlt(A)[2] == -1                           # the plain no-pivot LDL^T meets the zero at (0, 0)


@pytest.mark.parametrize("name", list(FAMILIES))
def test_model_solve_reaches_the_refinement_rule(name):
    A = FAMILIES[name]
    N = A.shape[0]
    b = np.random.default_rng(N).standard_normal((N, 2))
    x, corr, om = rbt.solve(A, b)
    assert corr <= rbt.MAX_CORRECTIONS
    assert om <= 4 * rbt.EPS, (corr, om)
    assert rbt.backward_error(A, x, b) <= 1e-14


@pytest.mark.parametrize("name", list(FAMILIES))
def test_model_refine_records_what_solve_returns(name):
    """refine's omega history ends in solve's omega after solve's corrections, and its x is solve's, bit for bit"""
    A = FAMILIES[name]
    N = A.shape[0]
    b = np.random.default_rng(N).standard_normal((N, 2))
    x, corr, om = rbt.solve(A, b)
    x2, corr2, om2, oms, ret = rbt.refine(A, b)
    assert np.array_equal(x.view(np.uint64), x2.view(np.uint64)) and (corr2, om2) == (corr, om)
    assert ret == 1 and len(oms) == corr + 1 and oms[-1] == om


# ---- the stopping rule of the refinement on non-finite values and at every exit --------------------------------------------------------
def test_column_omegas_on_non_finite_and_zero_columns():
    nan, inf = np.nan, np.inf
    w = rbt.column_omegas(2.0, [1.0, 0.0, nan, 1.0, 1.0, 1.0, inf, 3.0], [1.0, 0.0, 1.0, nan, inf, 1.0, 1.0, 0.0],
                          [2.0, 0.0, 1.0, 1.0, 1.0, inf, 1.0, 0.0])
    assert w[0] == 0.25 and w[1] == 0.0                                # a finite column; a zero column stays 0
    assert np.isnan(w[2:7]).all()                                      # any non-finite norm: NaN, never 0 or +inf
    assert w[7] == np.inf                                              # zero denominator under a non-zero residual
    assert np.isnan(rbt.column_omegas(inf, [1.0, 0.0], [1.0, 0.0], [1.0, 0.0])).all()   # ||A||_inf overflowed: NaN, not "converged"
    assert np.isnan(rbt.nan_max([0.5, nan, 1.0])) and rbt.nan_max([0.5, inf]) == inf and rbt.nan_max([]) == 0.0
    A = np.eye(3)
    assert np.isnan(rbt.backward_error(A, np.array([1.0, nan, 0.0]), np.ones(3)))
    assert rbt.backward_error(A, np.zeros((3, 2)), np.zeros((3, 2))) == 0.0


CAP_RATIO = 1.0 + 2.0 ** -8       # Aref = A' (1 + 2^-8): each correction contracts the error by 2^-8
DIVERGE_RATIO = 2.0 + 2.0 ** -4   # Aref = A' (2 + 2^-4): the error grows by 17/16, and omega by about 17 in the first correction
PLACED_MIN_N = 129                # below, ||A'|| ||x'|| / ||b'|| is too small for stagnation and divergence to clear 0.5 omega by 10x


def placed_reference(Ap, case):
    """(Aref, anorm) of a placed exit on the model's A': anorm is ||Aref||_inf, or +inf for the overflow case"""
    if case == "overflow":
        return Ap, np.inf
    Aref = Ap * {"cap": CAP_RATIO, "stagnation": 2.0, "divergence": DIVERGE_RATIO}[case]
    return Aref, float(np.abs(Aref).sum(axis=1).max())


def placed_rhs(N, nrhs, case, seed):
    """the right-hand side of a placed exit: zero; a NaN or +Inf in column 1 of a 3-column b; else standard normal"""
    b = np.random.default_rng(seed).standard_normal((N, nrhs))
    if case == "zero":
        return np.zeros((N, nrhs))
    if case in ("nan", "inf"):
        b[N // 2, 1] = np.nan if case == "nan" else np.inf
    return b


# every placed exit: corrections, return value, and what the last omega is
PLACED = {"zero": (0, 1, "zero"), "cap": (3, 1, "finite"), "stagnation": (1, 1, "finite"), "divergence": (1, 1, "finite"),
          "nan": (0, 0, "nan"), "inf": (0, 0, "nan"), "overflow": (0, 0, "nan")}


def assert_placed(case, corr, ret, oms):
    """the exit of `case` from a solve's corrections, return value and omega sequence, with the sequence at least a factor 10 away from
    EPS and from 0.5 omega_prev wherever the rule compares them"""
    want_corr, want_ret, last = PLACED[case]
    assert (corr, ret, len(oms)) == (want_corr, want_ret, want_corr + 1), (case, corr, ret, oms)
    if last == "zero":
        assert oms == [0.0]
    elif last == "nan":
        assert np.isnan(oms[-1])
    for k, om in enumerate(oms if last == "finite" else []):
        assert om >= 10 * rbt.EPS, (case, k, oms)
        if k:
            assert om >= 10 * 0.5 * oms[k - 1] or om <= 0.1 * 0.5 * oms[k - 1], (case, k, oms)
    if case == "cap":
        assert all(oms[k] <= 0.1 * 0.5 * oms[k - 1] for k in (1, 2, 3))
    if case in ("stagnation", "divergence"):
        assert oms[1] > 10 * 0.5 * oms[0] and oms[1] > oms[0]


@pytest.mark.parametrize("case,N", [(c, N) for c in PLACED for N in (1, 2, 3, 129, 1000)
                                    if N >= PLACED_MIN_N or c not in ("stagnation", "divergence")])
def test_model_places_every_exit(case, N):
    A = known_matrix(N)
    Ap = rbt.transform(A)
    nrhs = 3 if case in ("nan", "inf") else 1 + (N % 2) * 2
    b = placed_rhs(N, nrhs, case, seed=N)
    Aref, anorm = placed_reference(Ap, case) if case in ("cap", "stagnation", "divergence", "overflow") else (None, None)
    x, corr, om, oms, ret = rbt.refine(A, b, Aref=Aref, anorm=anorm, Ap=Ap)
    assert_placed(case, corr, ret, oms)
    assert om == oms[-1] or (np.isnan(om) and np.isnan(oms[-1]))
    if case == "zero":
        assert np.array_equal(x, np.zeros_like(x))
    if case == "divergence":
        assert_corrected_x(A, b, x)


def assert_corrected_x(A, b, x):
    """divergence returns the corrected x: x'_1 = x'_0 + A'^-1 (b' - c A' x'_0) = (2 - c) x'_0, 16 times smaller than the first solve's.
    The first solve is ~1e-8 from A^-1 b (the growth of the no-pivot factor of A'); an uncorrected x would be 15/16 of |x| away."""
    xs = np.linalg.solve(A, b)
    assert np.abs(x - (2.0 - DIVERGE_RATIO) * xs).max() <= 1e-6 * np.abs(xs).max()


def known_matrix(N):
    """the matrix of order N of the placed exits and the GPU refinement tests"""
    from oracle import bounds
    return bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
