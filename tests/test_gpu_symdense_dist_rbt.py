"""The safe mode of the distributed dense factorization (HB_FACT_RBT_NOPIV): the random butterfly transform bit for bit against
oracle/rbt_model.py, its factor bit for bit against hb_symdense's no-pivot factor of the model's A', inertia against hb_symdense's
Bunch-Kaufman, the refined solve, failure and resources, the mixed dense-sparse step in stable mode, and P = 2, 4 against P = 1.

Single-rank cases run on one GPU. Multi-rank cases spawn one process per GPU and skip when fewer GPUs are present."""
import numpy as np
import pytest
import torch

from hiop_b200 import sharding, synth
from oracle import bounds
from oracle import rbt_model as rbt
from multirank import run_ranks
from dense_handles import (GOLDEN, K128, MDS_FIELDS, SOLVE_REL, bk_single, factor_parts_from_rows, factor_single, golden_mds, gpu_families,
                           local_rows, orig_backward_error, rbt_dist, same_rows, upper_nan)
from dense_handles import make_ctx  # noqa: F401 (a fixture)

RBT, NOPIV, CHOL, BK = 3, 1, 2, 0


# ---- one rank -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 127, 128, 129, 300, 1000, 4099])
def test_transform_and_factor_bit_identical_to_the_model(make_ctx, N):
    from hiop_b200.engine import LinSolverSymDenseDist
    ctx = make_ctx(**K128)
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    want = [rbt.mirror(A), rbt.transform(A, 1), rbt.transform(A, 2)]
    s = LinSolverSymDenseDist(ctx, N)
    for stage in range(3):
        torch.cuda.synchronize()
        s.set_matrix(upper_nan(torch.from_numpy(A).to(ctx.device)))
        assert ctx.L.hb_debug_symdense_dist_rbt(s.h, stage) == 0
        for r, v in local_rows(s).items():
            if not np.array_equal(v.view(np.uint64), want[stage][r].view(np.uint64)):
                bad = np.nonzero(v.view(np.uint64) != want[stage][r].view(np.uint64))[0]
                pytest.fail(f"stage {stage} N={N}: row {r}, {bad.size} entries differ, first at {bad[0]}: {v[bad[0]]!r} vs {want[stage][r][bad[0]]!r}")
    s.close()
    # the factor: hb_symdense's no-pivot LDL^T (look-ahead, K = 128) of the model's A', bit for bit, and within the backward-error bound
    Ap = want[2]
    rc1, in1, F = factor_single(ctx, NOPIV, torch.from_numpy(Ap).to(ctx.device))
    b = np.random.default_rng(N).standard_normal((N, 2))
    rc, inr, rows, x, (corr, om, _) = rbt_dist(ctx, A, b)
    same_rows(rows, F, f"rbt N={N}")
    neg = N // 8 + N // 3
    assert rc == rc1 == neg and inr == in1 == (neg, 0, N - neg)
    L, d = factor_parts_from_rows(rows, N, NOPIV)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)
    th = max(bounds.block_theta(t(L), 16), bounds.block_theta(t(L), 128))
    assert bounds.factor_backward_ratio(t(Ap), t(L), t(d), None, th) <= 1.0
    # the refined solve
    assert corr <= 3 and om <= 4 * rbt.EPS, (corr, om)
    assert orig_backward_error(A, x, b) <= 1e-14
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_inertia_equals_bunch_kaufman_and_solve_is_refined(make_ctx):
    ctx = make_ctx()
    for name, A in gpu_families():
        N = A.shape[0]
        rc_bk, in_bk = bk_single(ctx, A)
        b = np.random.default_rng(N).standard_normal((N, 3))
        rc, inr, _, x, (corr, om, _) = rbt_dist(ctx, A, b)
        assert rc == rc_bk >= 0 and inr == in_bk, (name, rc, rc_bk, inr, in_bk)
        assert corr <= 3, (name, corr)
        assert orig_backward_error(A, x, b) <= 1e-14, (name, orig_backward_error(A, x, b), om)
        xbk = np.linalg.solve(A, b)     # LAPACK's LU on the host: the reference solution for the forward error
        cond = np.linalg.cond(A, np.inf)
        assert np.abs(x - xbk).max() <= SOLVE_REL * cond * np.abs(xbk).max(), name
        if name.startswith("saddle"):
            assert rbt_dist(ctx, A, mode=NOPIV)[0] == -1, name     # the plain no-pivot LDL^T on the same handle type breaks down
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_zero_row_fails_and_the_handle_stays_usable(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseDist
    ctx = make_ctx(**K128)
    live0 = int(ctx.L.hb_debug_live_resources())
    N = 700
    A = 1e-3 * bounds.known_inertia_matrix(N, 0, 200, seed=4)[0].numpy()
    Z = A.copy()
    Z[300, :] = 0.0
    Z[:, 300] = 0.0
    s = LinSolverSymDenseDist(ctx, N)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(ctx.device)
    s.set_matrix(dev(Z))
    assert s.matrixChanged(RBT) == -1
    s.set_matrix(dev(A))
    assert s.matrixChanged(RBT) == 200 and s.inertia() == (200, 0, N - 200)
    x = ctx.to_device(np.ones(N))
    assert s.solve(x)
    ctx.sync()
    assert orig_backward_error(A, x.cpu().numpy(), np.ones(N)) <= 1e-14
    S = dev(np.eye(N) * 2.0)
    for mode in (CHOL, NOPIV):                                       # the other modes on the same handle, after a failure
        s.set_matrix(dev(Z))
        assert s.matrixChanged(RBT) == -1
        s.set_matrix(S)
        assert s.matrixChanged(mode) == 0
        x = ctx.to_device(np.ones(N))
        assert s.solve(x)
        ctx.sync()
        assert np.allclose(x.cpu().numpy(), 0.5, rtol=4 * rbt.EPS, atol=0.0)
    s.close()
    assert int(ctx.L.hb_debug_live_resources()) == live0


# ---- mixed dense-sparse in stable mode ------------------------------------------------------------------------------------------------
def mds_stable(ctx, p):
    """single-GPU KKTLinSysCompressedMDSXYcYd(safe_mode=True) and factorizeWithCurvCheck_dist(safe_mode=True) on the same inputs"""
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd, LinSolverSymDenseDist
    T = {f: ctx.to_device(np.asarray(getattr(p, f), dtype=np.float64)) for f in ("zl", "sxl", "zu", "sxu", "ixl", "ixu", "rx", "ryc", "ryd") + MDS_FIELDS}
    torch.cuda.synchronize()
    out = []
    for dist in (False, True):
        k = KKTLinSysCompressedMDSXYcYd(ctx, p.nxs, p.nxd, p.neq, p.nineq, safe_mode=True)
        k.set_sparsity(p.iRow_c, p.jCol_c, p.iRow_d, p.jCol_d)
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
        dx, dyc, dyd = ctx.zeros(p.nxs + p.nxd), ctx.zeros(p.neq), ctx.zeros(p.nineq)
        if dist:
            d = LinSolverSymDenseDist(ctx, p.nxd + p.neq + p.nineq)
            k.build_kkt_matrix_dist(d, *[T[f] for f in MDS_FIELDS])
            ret = k.factorizeWithCurvCheck_dist(d, safe_mode=True)
            ok = ret >= 0 and k.solveCompressed_dist(d, T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        else:
            k.build_kkt_matrix(*[T[f] for f in MDS_FIELDS])
            ret = k.factorizeWithCurvCheck()
            ok = ret >= 0 and k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        ctx.sync()
        out.append((ret, ok, dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy()))
        if dist:
            d.close()
        k.close()
    return out


MDS_REL = 1e-9      # both are backward-stable solves of a system of moderate condition


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["golden", "small", "medium"])
def test_mds_stable_mode_matches_single_gpu(make_ctx, name):
    from test_gpu_mds import _full_residual
    ctx = make_ctx()
    if name == "golden":
        p = golden_mds()
    else:
        nxs, nxd, neq, nineq, nnz, seed = {"small": (3000, 150, 60, 50, 12, 11), "medium": (20000, 600, 150, 150, 20, 13)}[name]
        p = synth.make_mds_problem(nxs, nxd, neq, nineq, nnz_per_row=nnz, seed=seed)
    (r1, ok1, dx1, dyc1, dyd1), (r2, ok2, dx2, dyc2, dyd2) = mds_stable(ctx, p)
    assert r1 == r2 >= 0 and ok1 and ok2, (r1, r2, ok1, ok2)
    scale = max(1.0, np.abs(dx1).max(), np.abs(dyc1).max(initial=0.0), np.abs(dyd1).max(initial=0.0))
    err = max(np.abs(dx2 - dx1).max(), np.abs(dyc2 - dyc1).max(initial=0.0), np.abs(dyd2 - dyd1).max(initial=0.0)) / scale
    assert err <= MDS_REL, err
    if name == "golden":
        g = np.load(GOLDEN / "mds_nxs50_nxd20.npz")
        assert _full_residual(p, g["ref_Dx"], g["ref_Dd_inv"], dx2, dyc2, dyd2) <= 1e-8


@pytest.mark.gpu
def test_mds_stable_mode_at_n5000_inertia_and_residual(make_ctx):
    """a synthetic MDS system with N = nxd + neq + nineq = 5 000 built with hb_mds_build_kkt_matrix_dist: the return value equals the
    single-GPU Bunch-Kaufman step's, and the uncondensed residual with bench.py's independent operators is below 1e-8"""
    import bench
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd, LinSolverSymDenseDist
    ctx = make_ctx()
    nxs, nxd, neq, nineq = 50_000, 4000, 500, 500
    with ctx:
        T = bench.make_mds_device_problem(torch, ctx, nxs, nxd, neq, nineq, nnz_row=max(1, round(5.0 * nxs / (neq + nineq))))
        args = [T[f] for f in ("Hd", "Hs", "Jcd", "Jdd", "Jcs", "Jds", "vl", "sdl", "vu", "sdu", "idl", "idu", "dwx", "dwd", "dcc", "dcd")]
        k = KKTLinSysCompressedMDSXYcYd(ctx, nxs, nxd, neq, nineq, safe_mode=True)
        k.set_sparsity(T["iRc"], T["jCc"], T["iRd"], T["jCd"])
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
        k.build_kkt_matrix(*args)
        ret1 = k.factorizeWithCurvCheck()
        dist = LinSolverSymDenseDist(ctx, nxd + neq + nineq)
        k.build_kkt_matrix_dist(dist, *args)
        ret = k.factorizeWithCurvCheck_dist(dist, safe_mode=True)
        dx, dyc, dyd = ctx.zeros(nxs + nxd), ctx.zeros(neq), ctx.zeros(nineq)
        assert ret == ret1 == neq + nineq, (ret, ret1)
        assert k.solveCompressed_dist(dist, T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        ctx.sync()
        res = bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd)
        dist.close()
        k.close()
    assert res <= 1e-8, res
    torch.cuda.empty_cache()


# ---- several ranks -------------------------------------------------------------------------------------------------------------------------
def _case(N):
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    return A, np.random.default_rng(N).standard_normal((N, 2))


def _rank_worker(rank, world, uid, out, sizes):
    import os
    from hiop_b200.engine import Context
    torch.cuda.set_device(rank)
    os.environ["HB_DENSE_PAIR_MIN"] = str(1 << 30)
    ctx = Context(rank)
    try:
        ctx.init_comm(world, rank, uid)
        for N in sizes:
            A, b = _case(N)
            rc, inr, rows, x, stats = rbt_dist(ctx, A, b)
            out[(rank, N)] = (rc, inr, rows, x, stats[0])
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,sizes", [(2, [4099]), (4, [300, 1000])], ids=["p2", "p4"])
def test_ranks_match_one_rank_bit_for_bit(make_ctx, world, sizes):
    """every owned row of the factor, the inertia, the solution and the number of corrections are those of P = 1; at N = 300 and P = 4
    rank 3 owns no block and still takes part in every collective"""
    out = run_ranks(_rank_worker, world, (sizes,), comm="nccl")
    ctx = make_ctx(HB_DENSE_PAIR_MIN=1 << 30)
    for N in sizes:
        A, b = _case(N)
        rc, inr, rows, x, (corr, _, _) = rbt_dist(ctx, A, b)
        for rank in range(world):
            rrc, rin, rrows, rx, rcorr = out[(rank, N)]
            assert (rrc, rin, rcorr) == (rc, inr, corr), (world, rank, N)
            assert set(rrows) == {r for bb, e in sharding.block_rows(N, world, rank) for r in range(bb, e)}
            for r, v in rrows.items():
                assert np.array_equal(v[r:].view(np.uint64), rows[r][r:].view(np.uint64)), (world, rank, N, r)
            assert np.array_equal(rx.view(np.uint64), x.view(np.uint64)), (world, rank, N)
