"""The dense solver dispatch (hb_symdense.cu) at every order where it switches kernels: factor + solve of the B1 solver in all three modes,
the condensed SPD system of the quasi-Newton KKT path, against LAPACK through numpy / the oracle; and the per-handle look-ahead state of
the condensed Cholesky (two contexts on one device)."""
import numpy as np
import pytest

from hiop_b200 import synth
from oracle import kkt_oracle as ko
from test_gpu_parity import ctx, _setup_kkt, _as_dict, _run_solve, _relerr  # noqa: F401

pytestmark = pytest.mark.gpu

EDGES = [1, 10, 64, 65, 95, 96, 256, 257, 384, 385, 1024, 1025, 2048, 2049, 2501]


def _matrix(mode, N):
    from hiop_b200.engine import LinSolverSymDense
    if mode == LinSolverSymDense.CHOLESKY:
        r = np.random.default_rng(N)
        A = r.standard_normal((N, N // 2 + 1))
        return A @ A.T + np.diag(r.uniform(0.5, 2.0, N)), 0
    m = N // 3
    return synth.make_kkt_like(N - m, m, seed=N), m


@pytest.mark.parametrize("N", EDGES)
@pytest.mark.parametrize("mode", ["BUNCH_KAUFMAN", "NOPIV", "CHOLESKY"])
def test_symdense_at_threshold_edges(ctx, mode, N):
    from hiop_b200.engine import LinSolverSymDense
    mode = getattr(LinSolverSymDense, mode)
    K, neg = _matrix(mode, N)
    s = LinSolverSymDense(ctx, N, mode)
    s.set_matrix(ctx.to_device(np.triu(K) + np.tril(np.full((N, N), np.nan), -1)))  # the lower part must never be read
    assert s.matrixChanged() == neg
    assert s.inertia() == (neg, 0, N - neg)
    tol = 1e-9 if mode == LinSolverSymDense.CHOLESKY else 1e-8
    for nrhs in (1, 8):
        rhs = np.random.default_rng(nrhs).standard_normal((nrhs, N))
        x = ctx.to_device(rhs.copy())
        assert s.solve(x)
        ctx.sync()
        ref = np.linalg.solve(K, rhs.T).T
        assert np.abs(x.cpu().numpy() - ref).max() <= tol * np.abs(ref).max()
    s.close()


@pytest.mark.parametrize("m", [1, 64, 65, 2048, 2049, 2050])
def test_condensed_solve_at_threshold_edges(ctx, m):
    P = synth.make_qn_problem(max(600, 3 * m), m, 4, seed=77 + m)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    dxo, dyco, dydo, _ = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    p = _as_dict(P)
    k, _ = _setup_kkt(ctx, p)
    dx, dyc, dyd = _run_solve(ctx, k, p)
    assert _relerr(dx, dxo) <= 1e-8 and _relerr(dyc, dyco) <= 1e-8 and _relerr(dyd, dydo) <= 1e-8
    k.close()


def test_two_contexts_own_their_lookahead_state():
    """m = 2050 takes the look-ahead Cholesky; each handle owns its panel stream and scratch, so two contexts on one device that solve
    back to back without a synchronisation give the bits of one handle alone"""
    from hiop_b200.engine import Context
    P = synth.make_qn_problem(6000, 2050, 4, seed=2050)
    p = _as_dict(P)

    def start(c):
        k, T = _setup_kkt(c, p)
        rx, ryc, ryd = c.to_device(P.rx), c.to_device(P.ryc), c.to_device(P.ryd)
        out = (c.zeros(P.n), c.zeros(P.m_eq), c.zeros(P.m_ineq))
        return k, T, (rx, ryc, ryd), out

    c0, c1 = Context(0), Context(0)
    k, T, r, out = start(c0)
    assert k.solveCompressed(*r, *out)
    c0.sync()
    alone = [v.cpu().numpy() for v in out]
    k.close()
    runs = [start(c0), start(c1)]
    for (k, T, r, out), c in zip(runs, (c0, c1)):
        c.sync()                              # inputs in place; the two solves below then run with no synchronisation between them
    for k, T, r, out in runs:
        assert k.solveCompressed(*r, *out)
    c0.sync()
    c1.sync()
    for k, T, r, out in runs:
        for a, b in zip(alone, out):
            assert np.array_equal(a, b.cpu().numpy())
        k.close()
    c0.close()
    c1.close()
