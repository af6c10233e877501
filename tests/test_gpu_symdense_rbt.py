"""The random-butterfly safe mode on one GPU (hb_symdense, HB_FACT_RBT_NOPIV): the one-pass transform bit for bit against
oracle/rbt_model.py, the factor bit for bit against hb_symdense's no-pivot factor of the model's A', inertia against Bunch-Kaufman, the
refined solve against LAPACK and against the distributed handle at P = 1, failure and resources, the mixed dense-sparse step with
linSys.mode = RBT_NOPIV, and the drop-in MDS driver with HIOP_B200_LINSOL=rbt."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import bounds
from oracle import rbt_model as rbt
from dense_handles import K128, MDS_FIELDS, SOLVE_REL, bk_single, golden_mds, gpu_families, orig_backward_error, rbt_dist, readback, upper_nan
from dense_handles import make_ctx  # noqa: F401 (a fixture)
from test_gpu_dropin_drivers import REF, ROW, _compare, _tables_agree

pytestmark = pytest.mark.gpu
RBT, NOPIV, BK = 3, 1, 0


def dev(ctx, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)


def rbt_single(ctx, A, rhs=None, mode=RBT):
    """factor A (numpy, full; the lower triangle handed over as NaN) on a LinSolverSymDense in `mode`; solve rhs (N x nrhs) when given.
    Returns rc, inertia, x, stats"""
    from hiop_b200.engine import LinSolverSymDense
    N = A.shape[0]
    s = LinSolverSymDense(ctx, N, mode)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(dev(ctx, A)))
    ctx.sync()
    rc = s.matrixChanged()
    inr = s.inertia()
    x = stats = None
    if rhs is not None and rc >= 0:
        xd = ctx.to_device(np.ascontiguousarray(rhs.T))
        assert s.solve(xd)
        ctx.sync()
        x = xd.cpu().numpy().T.copy()
        stats = s.rbt_stats()
    s.close()
    return rc, inr, x, stats


def _bits_equal(a, b, what):
    if not np.array_equal(a.view(np.uint64), b.view(np.uint64)):
        bad = np.argwhere(a.view(np.uint64) != b.view(np.uint64))
        pytest.fail(f"{what}: {len(bad)} entries differ, first at {tuple(bad[0])}: {a[tuple(bad[0])]!r} vs {b[tuple(bad[0])]!r}")


@pytest.mark.parametrize("N", [1, 2, 3, 127, 128, 129, 300, 1000, 2049, 4097, 4099])
def test_transform_bit_identical_to_the_model(make_ctx, N):
    """A' kept in full and the upper triangle in the factor buffer (M in place, or the padded copy for odd N), the lower triangle NaN on
    input; N = 2049 and 4097 are 1 (mod 4), where the 4-row groups do not close"""
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx()
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    want = rbt.transform(A, 2)
    s = LinSolverSymDense(ctx, N, RBT)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(dev(ctx, A)))
    ctx.sync()
    Ak, F = np.empty((N, N)), np.empty((N, N))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert ctx.L.hb_debug_symdense_rbt(s.h, p(Ak), p(F)) == 0
    _bits_equal(Ak, want, f"A' N={N}")
    iu = np.triu_indices(N)
    _bits_equal(F[iu], want[iu], f"factor buffer N={N}")
    s.close()


@pytest.mark.parametrize("N", [300, 1001, 4099, 6200])
def test_factor_bit_identical_to_nopiv_on_the_model(make_ctx, N):
    """the factor, the plan and the inertia are hb_symdense NOPIV's on the model's A'; N = 6200 takes the paired look-ahead blocks"""
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx()
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    out = []
    for mode, M in ((RBT, A), (NOPIV, rbt.transform(A, 2))):
        s = LinSolverSymDense(ctx, N, mode)
        torch.cuda.synchronize()
        s.set_matrix(upper_nan(dev(ctx, M)))
        ctx.sync()
        rc = s.matrixChanged()
        out.append((rc, s.inertia(), readback(s)))
        s.close()
    (rc1, in1, rb1), (rc2, in2, rb2) = out
    neg = N // 8 + N // 3
    assert rc1 == rc2 == neg and in1 == in2 == (neg, 0, N - neg)
    assert rb1["plan"] == rb2["plan"] and rb1["plan"][3] == (N >= 6144), rb1["plan"]
    iu = np.triu_indices(N)
    _bits_equal(rb1["F"][iu], rb2["F"][iu], f"factor N={N}")
    torch.cuda.empty_cache()


def test_inertia_equals_bunch_kaufman_and_solve_is_refined(make_ctx):
    ctx = make_ctx()
    for name, A in gpu_families():
        N = A.shape[0]
        rc_bk, in_bk = bk_single(ctx, A)
        b = np.random.default_rng(N).standard_normal((N, 3))
        rc, inr, x, (corr, om, ms) = rbt_single(ctx, A, b)
        assert rc == rc_bk >= 0 and inr == in_bk, (name, rc, rc_bk, inr, in_bk)
        assert corr <= 3 and ms > 0.0, (name, corr, ms)
        assert orig_backward_error(A, x, b) <= 1e-14, (name, orig_backward_error(A, x, b), om)
        xlu = np.linalg.solve(A, b)
        cond = np.linalg.cond(A, np.inf)
        assert np.abs(x - xlu).max() <= SOLVE_REL * cond * np.abs(xlu).max(), name
        # three right-hand sides at once give the columns of three single solves, up to the corrections: the stopping rule takes the
        # largest omega over the right-hand sides, so a column may be corrected once more or less than alone
        for q in range(3):
            xq = rbt_single(ctx, A, b[:, q:q + 1])[2]
            assert np.abs(xq[:, 0] - x[:, q]).max() <= SOLVE_REL * cond * np.abs(x[:, q]).max(), (name, q)
        # the distributed handle at P = 1 (another factor schedule below N = 257): both backward stable
        xd = rbt_dist(ctx, A, b)[3]
        assert np.abs(xd - x).max() <= SOLVE_REL * cond * np.abs(x).max(), name
        if name.startswith("saddle"):
            assert rbt_single(ctx, A, mode=NOPIV)[0] == -1, name     # the plain no-pivot LDL^T breaks down where RBT does not
    torch.cuda.empty_cache()


@pytest.mark.parametrize("N", [300, 1000, 4099])
def test_solution_agrees_with_the_distributed_handle(make_ctx, N):
    """on well-conditioned matrices (cond_inf ~ 150) with the same factor schedule (look-ahead, blocks unpaired): 1e-14 relative"""
    ctx = make_ctx(**K128)
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    b = np.random.default_rng(N).standard_normal((N, 2))
    rc, inr, x, (corr, om, _) = rbt_single(ctx, A, b)
    rcd, ind, _, xd, _ = rbt_dist(ctx, A, b)
    neg = N // 8 + N // 3
    assert rc == rcd == neg and inr == ind == (neg, 0, N - neg)
    assert corr <= 3 and om <= 4 * rbt.EPS, (corr, om)
    assert np.abs(xd - x).max() <= 1e-14 * np.abs(x).max(), np.abs(xd - x).max() / np.abs(x).max()
    torch.cuda.empty_cache()


def test_zero_row_fails_and_the_handle_stays_usable(make_ctx):
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx()
    live0 = int(ctx.L.hb_debug_live_resources())
    N = 700
    A = 1e-3 * bounds.known_inertia_matrix(N, 0, 200, seed=4)[0].numpy()
    Z = A.copy()
    Z[300, :] = 0.0
    Z[:, 300] = 0.0
    s = LinSolverSymDense(ctx, N, RBT)
    s.set_matrix(dev(ctx, Z))
    assert s.matrixChanged() == -1
    s.set_matrix(dev(ctx, A))
    assert s.matrixChanged() == 200 and s.inertia() == (200, 0, N - 200)
    x = ctx.to_device(np.ones(N))
    assert s.solve(x)
    ctx.sync()
    assert orig_backward_error(A, x.cpu().numpy(), np.ones(N)) <= 1e-14
    S = dev(ctx, np.eye(N) * 2.0)
    for mode in (BK, NOPIV):                                          # the other modes on the same handle, after a failure
        s.mode = RBT
        s.set_matrix(dev(ctx, Z))
        assert s.matrixChanged() == -1
        s.mode = mode
        s.set_matrix(S)
        assert s.matrixChanged() == 0
        x = ctx.to_device(np.ones(N))
        assert s.solve(x)
        ctx.sync()
        assert np.allclose(x.cpu().numpy(), 0.5, rtol=4 * rbt.EPS, atol=0.0)
    s.close()
    assert int(ctx.L.hb_debug_live_resources()) == live0


def test_mds_step_golden_in_rbt_mode(make_ctx):
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd
    from test_gpu_mds import _full_residual
    ctx = make_ctx()
    p = golden_mds()
    T = {f: ctx.to_device(np.asarray(getattr(p, f), dtype=np.float64)) for f in ("zl", "sxl", "zu", "sxu", "ixl", "ixu", "rx", "ryc", "ryd") + MDS_FIELDS}
    torch.cuda.synchronize()
    k = KKTLinSysCompressedMDSXYcYd(ctx, p.nxs, p.nxd, p.neq, p.nineq, safe_mode=True)
    k.linSys.mode = k.linSys.RBT_NOPIV
    k.set_sparsity(p.iRow_c, p.jCol_c, p.iRow_d, p.jCol_d)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
    k.build_kkt_matrix(*[T[f] for f in MDS_FIELDS])
    ret = k.factorizeWithCurvCheck()
    dx, dyc, dyd = ctx.zeros(p.nxs + p.nxd), ctx.zeros(p.neq), ctx.zeros(p.nineq)
    assert ret == p.neq + p.nineq, ret
    assert k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
    ctx.sync()
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "mds_nxs50_nxd20.npz"))
    assert _full_residual(p, g["ref_Dx"], g["ref_Dd_inv"], dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy()) <= 1e-8
    k.close()


def test_mds_step_at_n5000_in_rbt_mode(make_ctx):
    import bench
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd
    ctx = make_ctx()
    nxs, nxd, neq, nineq = 50_000, 4000, 500, 500
    with ctx:
        T = bench.make_mds_device_problem(torch, ctx, nxs, nxd, neq, nineq, nnz_row=max(1, round(5.0 * nxs / (neq + nineq))))
        args = [T[f] for f in ("Hd", "Hs", "Jcd", "Jdd", "Jcs", "Jds", "vl", "sdl", "vu", "sdu", "idl", "idu", "dwx", "dwd", "dcc", "dcd")]
        k = KKTLinSysCompressedMDSXYcYd(ctx, nxs, nxd, neq, nineq, safe_mode=True)
        k.linSys.mode = k.linSys.RBT_NOPIV
        k.set_sparsity(T["iRc"], T["jCc"], T["iRd"], T["jCd"])
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
        k.build_kkt_matrix(*args)
        ret = k.factorizeWithCurvCheck()
        dx, dyc, dyd = ctx.zeros(nxs + nxd), ctx.zeros(neq), ctx.zeros(nineq)
        assert ret == neq + nineq, ret
        assert k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        ctx.sync()
        res = bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd)
        k.close()
    assert res <= 1e-8, res
    torch.cuda.empty_cache()


def test_mds1_driver_with_rbt():
    os.environ["HIOP_B200_LINSOL"] = "rbt"
    try:
        worst, nit, out = _compare("mds1_b200.exe", ["400", "100", "0", "-selfcheck"])
    finally:
        os.environ.pop("HIOP_B200_LINSOL", None)
    assert "selfcheck passed" in out
    assert worst <= 1e-5, worst


def test_mds1_driver_with_rbt_in_speculative_mode(tmp_path):
    """linsol_mode speculative: no-pivot LDL^T while safe mode is off, RBT whenever HiOp turns it on"""
    path = os.path.join(REF, "mds1_b200.exe")
    if not os.path.exists(path):
        pytest.skip("mds1_b200.exe not built")
    (tmp_path / "hiop.options").write_text("linsol_mode speculative\n")
    tabs = []
    for b200 in (False, True):
        env = dict(os.environ)
        for k in ("HIOP_B200", "HIOP_B200_LINSOL"):
            env.pop(k, None)
        if b200:
            env.update(HIOP_B200="1", HIOP_B200_LINSOL="rbt")
        p = subprocess.run([path, "400", "100", "0", "-selfcheck"], capture_output=True, text=True, env=env, timeout=600, cwd=str(tmp_path))
        assert p.returncode == 0 and "selfcheck passed" in p.stdout, p.stdout[-1500:]
        tabs.append([[float(x) for x in m.groups()] for m in (ROW.match(line) for line in p.stdout.splitlines()) if m])
    assert _tables_agree([r + [0.0] for r in tabs[1]], [r + [0.0] for r in tabs[0]])[0] <= 1e-5
