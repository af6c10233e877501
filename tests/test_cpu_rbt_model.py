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
