"""oracle/spd_refine_model.py on a numpy run: its stage bounds hold on a run of the loop with scipy's Cholesky, and every planted mistake
in the loop (MUTATIONS) breaks a stage bound, the exit rule or the NaN report. The GPU test (test_gpu_condensed_refine.py) holds the device
kernels to the same checks."""
import math

import numpy as np
import pytest
from scipy.linalg import cho_factor, cho_solve

from oracle import spd_refine_model as m

N = 200
EPS = 1e-3


def _problem(seed=0, spread=3.0):
    """SPD Nref with a diagonal spread over 10^(+-spread) (s far from 1), Nfact = (1 + EPS) Nref, rhs"""
    r = np.random.default_rng(seed)
    G = r.standard_normal((N, N // 2))
    B = G @ G.T / N + np.diag(r.uniform(0.5, 2.0, N))
    d = 10.0 ** r.uniform(-spread, spread, N)
    Nref = (B * np.sqrt(d)[:, None]) * np.sqrt(d)[None, :]
    Nref = 0.5 * (Nref + Nref.T)
    Nfact = (1.0 + EPS) * Nref
    rhs = r.standard_normal(N) * np.sqrt(d)
    return Nref, Nfact, rhs


def _setup(Nfact):
    s, Aeq = m.equilibrate(Nfact)
    Afull = np.triu(Aeq) + np.triu(Aeq, 1).T
    cf = cho_factor(Afull, lower=True)
    R = np.tril(cf[0])
    return s, Afull, R, (lambda z: cho_solve(cf, z))


def _stage_ratios(xs, Afull, R, s, Nref, rhs):
    return [m.stage_ratio(Afull, R, 1.0, s, Nref, rhs, xs[k - 1] if k else None, xs[k]) for k in range(len(xs))]


def test_equilibration_bits():
    Nref, Nfact, _ = _problem()
    s, Aeq = m.equilibrate(Nfact)
    for i, j in ((0, 0), (3, 17), (N - 1, N - 1), (5, N - 1)):
        si, sj = 1.0 / math.sqrt(Nfact[i, i]), 1.0 / math.sqrt(Nfact[j, j])
        assert s[i] == si and Aeq[i, j] == (si * Nfact[i, j]) * sj
    assert np.all(np.tril(Aeq, -1) == 0.0)
    assert np.abs(np.diag(Aeq) - 1.0).max() <= 4 * m.U


def test_stage_bounds_hold_and_are_not_vacuous():
    Nref, Nfact, rhs = _problem()
    s, Afull, R, solve = _setup(Nfact)
    xs, rhos, nref, rho = m.refine(solve, Afull, Nref, rhs, s, 0.0, 3)
    assert nref == 3 and len(xs) == 4
    ratios = _stage_ratios(xs, Afull, R, s, Nref, rhs)
    rho_r = m.rho_ratio(Nref, rhs, xs[-1], rho)
    print("stage ratios", [f"{x:.3g}" for x in ratios], f"rho ratio {rho_r:.3g}", "rhos", [f"{x:.3g}" for x in rhos])
    assert max(ratios) <= 1.0 and rho_r <= 1.0
    # the bounds are within 100x of what the numpy run's stages actually get wrong
    assert max(ratios) >= 1e-2
    # the contraction: each correction divides the residual by ~1 / EPS
    for k in range(2):
        assert 0.1 / EPS <= rhos[k] / rhos[k + 1] <= 10.0 / EPS


def test_exit_rule():
    Nref, Nfact, rhs = _problem(1)
    s, Afull, R, solve = _setup(Nfact)
    _, rhos, _, _ = m.refine(solve, Afull, Nref, rhs, s, 0.0, 3)
    cases = [(math.inf, 3, 0), (0.0, 0, 0), (0.0, 1, 1), (0.0, 3, 3), (math.sqrt(rhos[0] * rhos[1]), 3, 1), (math.sqrt(rhos[1] * rhos[2]), 3, 2),
             (rhos[1], 3, 2), (np.nextafter(rhos[1], math.inf), 3, 1)]
    for tol, mr, k in cases:
        xs, _, nref, rho = m.refine(solve, Afull, Nref, rhs, s, tol, mr)
        assert (nref, rho) == (k, rhos[k]) == m.expected_exit(rhos, tol, mr), (tol, mr, nref, k)


@pytest.mark.parametrize("mutation", m.MUTATIONS)
def test_every_mutation_is_seen(mutation):
    Nref, Nfact, rhs = _problem(2)
    s, Afull, R, solve = _setup(Nfact)
    _, rhos, _, _ = m.refine(solve, Afull, Nref, rhs, s, 0.0, 3)
    seen = []
    # stages of a run to max_refine = 3 with tol = 0
    xs, _, nref, rho = m.refine(solve, Afull, Nref, rhs, s, 0.0, 3, mutation=mutation)
    ratios = _stage_ratios(xs, Afull, R, s, Nref, rhs)
    if max(ratios) > 1.0:
        seen.append(f"stage bound {max(ratios):.3g}")
    # every exit of test_exit_rule
    for tol, mr in ((0.0, 0), (0.0, 1), (0.0, 3), (math.sqrt(rhos[0] * rhos[1]), 3), (rhos[1], 3), (np.nextafter(rhos[1], math.inf), 3)):
        _, _, nref, rho = m.refine(solve, Afull, Nref, rhs, s, tol, mr, mutation=mutation)
        if (nref, rho) != m.expected_exit(rhos, tol, mr):
            seen.append(f"exit at tol {tol:.3g}, max_refine {mr}")
    # a NaN in the rhs: 0 corrections, NaN reported
    for i in (0, N - 1):
        bad = rhs.copy()
        bad[i] = math.nan
        with np.errstate(invalid="ignore"):
            _, _, nref, rho = m.refine(lambda z: np.linalg.solve(Afull, z), Afull, Nref, bad, s, 1e-8, 3, mutation=mutation)
        if not (nref == 0 and math.isnan(rho)):
            seen.append(f"NaN at {i}: {nref} corrections, rho {rho}")
    print(mutation, seen)
    assert seen, mutation


def test_unmutated_nan_and_inf():
    Nref, Nfact, rhs = _problem(3)
    s, Afull, R, solve = _setup(Nfact)
    for v in (math.nan, math.inf):
        bad = rhs.copy()
        bad[N // 2] = v
        with np.errstate(invalid="ignore"):
            _, _, nref, rho = m.refine(lambda z: np.linalg.solve(Afull, z), Afull, Nref, bad, s, 1e-8, 3)
        assert nref == 0 and math.isnan(rho)
    assert math.isnan(m.inf_norm([1.0, math.nan, 2.0])) and m.inf_norm([1.0, math.nan, 2.0], drop_nan=True) == 2.0
