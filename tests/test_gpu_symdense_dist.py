"""The dense symmetric system factored across ranks (hb_symdense_dist, LinSolverSymDenseDist): its block-cyclic layout, the factor
bit for bit against hb_symdense's look-ahead path at K = 128 and across P, the backward-error bounds and inertia of
test_gpu_symdense_paths.py, failure and misuse, and the mixed dense-sparse path on top of it.

Single-rank cases run on one GPU. Multi-rank cases spawn one process per GPU (multirank.run_ranks) and skip when fewer GPUs are
present."""
import ctypes

import numpy as np
import pytest
import torch

from hiop_b200 import sharding, synth
from oracle import bounds
from multirank import run_ranks
from dense_handles import K128, MDS_FIELDS, factor_dist, factor_parts_from_rows, factor_single, local_rows, matrix, rhs, same_rows
from dense_handles import make_ctx  # noqa: F401 (a fixture)

CHOL, NOPIV, BK = 2, 1, 0
ERR_INVALID, ERR_STATE = -1, -5                              # HB_ERR_* of include/hiopb200.h


# ---- layout (CPU) -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,world", [(0, 1), (1, 1), (127, 2), (128, 2), (129, 2), (300, 4), (1000, 4), (4099, 2), (22000, 8), (5, 8)])
def test_block_rows_cover_every_row_once_block_cyclic(N, world):
    seen = np.zeros(N, dtype=int)
    for rank in range(world):
        rows = sharding.block_rows(N, world, rank)
        assert rows == sorted(rows)
        for b, e in rows:
            assert b % 128 == 0 and (b // 128) % world == rank and 0 < e - b <= 128 and (e - b == 128 or e == N)
            seen[b:e] += 1
    assert (seen == 1).all()


# ---- single rank -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [CHOL, NOPIV], ids=["chol", "nopiv"])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1000, 4099, 8192])
def test_one_rank_bit_identical_to_symdense_and_within_bounds(make_ctx, mode, N):
    ctx = make_ctx(**K128)
    dev = ctx.device
    M, inertia = matrix(mode, N, seed=N + mode, device=dev)
    rc1, in1, F = factor_single(ctx, mode, M)
    bs = [rhs(N, N, 1), rhs(N, N + 1, 3)]
    rc, inr, rows, sols = factor_dist(ctx, mode, M, bs)
    same_rows(rows, F, f"{('', 'nopiv', 'chol')[mode]} N={N}")
    assert rc == rc1 == inertia[0] and inr == in1 == inertia, (rc, rc1, inr, in1, inertia)
    # the factor and every solve within the backward-error bounds of test_gpu_symdense_paths.py
    L, d = factor_parts_from_rows(rows, N, mode)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    th = max(bounds.block_theta(t(L), 16), bounds.block_theta(t(L), 128))
    fr = bounds.factor_backward_ratio(M, t(L), t(d), None, th)
    assert fr <= 1.0, fr
    for b, x in zip(bs, sols):
        if N <= bounds.EXACT_RESIDUAL_MAX_N:
            sr, _ = bounds.solve_backward_ratio(M.cpu().numpy(), x.T.copy(), b.T.copy(), L, d, None, th)
        else:
            sr, _ = bounds.solve_backward_ratio(M, t(x.T), t(b.T), t(L), t(d), None, th)
        assert sr <= 1.0, sr
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_nopiv_inertia_equals_symdense_on_quasidefinite(make_ctx):
    """the KKT-like quasi-definite family test_gpu_symdense_paths.py uses for the no-pivot LDL^T: inertia (m, 0, N - m)"""
    ctx = make_ctx(**K128)
    N, m = 2049, 683
    M = torch.from_numpy(synth.make_kkt_like(N - m, m, seed=5)).to(ctx.device)
    rc1, in1, F = factor_single(ctx, NOPIV, M)
    rc, inr, rows, _ = factor_dist(ctx, NOPIV, M, [])
    same_rows(rows, F, "quasi-definite")
    assert rc == rc1 == m and inr == in1 == (m, 0, N - m)


@pytest.mark.gpu
def test_failure_and_misuse(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseDist
    ctx = make_ctx(**K128)
    live0 = int(ctx.L.hb_debug_live_resources())
    N = 700
    s = LinSolverSymDenseDist(ctx, N)
    x = ctx.to_device(rhs(N, 1, 1))
    assert ctx.L.hb_symdense_dist_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE   # solve before any factorization
    M, _ = matrix(CHOL, N, 3, ctx.device)
    s.set_matrix(M)
    assert ctx.L.hb_symdense_dist_matrix_changed(s.h, BK) == ERR_INVALID                        # Bunch-Kaufman is not distributed
    with pytest.raises(Exception, match="Bunch-Kaufman is not distributed"):                     # the wrapper does not let it read as -1
        s.matrixChanged(BK)
    # not SPD: a negative diagonal entry in block row 3 -> -1, then the handle factors an SPD matrix
    Mb = M.clone()
    Mb[3 * 128 + 5, 3 * 128 + 5] = -1.0
    s.set_matrix(Mb)
    assert s.matrixChanged(CHOL) == -1
    assert ctx.L.hb_symdense_dist_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE
    s.set_matrix(M)
    assert s.matrixChanged(CHOL) == 0 and s.inertia() == (0, 0, N)
    assert s.solve(x)
    # a zero pivot under the no-pivot LDL^T
    Z = torch.eye(N, dtype=torch.float64, device=ctx.device)
    Z[200, 200] = 0.0
    s.set_matrix(Z)
    assert s.matrixChanged(NOPIV) == -1
    ctx.sync()
    s.close()
    assert int(ctx.L.hb_debug_live_resources()) == live0


# ---- mixed dense-sparse, one rank ------------------------------------------------------------------------------------------------------
def mds_run(ctx, p, dist):
    """build (single and distributed), factor the distributed matrix with the no-pivot LDL^T, solve; returns (M, rows, ret, dx, dyc, dyd)"""
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd
    T = {f: ctx.to_device(getattr(p, f)) for f in ("zl", "sxl", "zu", "sxu", "ixl", "ixu", "rx", "ryc", "ryd") + MDS_FIELDS}
    torch.cuda.synchronize()
    k = KKTLinSysCompressedMDSXYcYd(ctx, p.nxs, p.nxd, p.neq, p.nineq, safe_mode=False)
    k.set_sparsity(p.iRow_c, p.jCol_c, p.iRow_d, p.jCol_d)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
    k.build_kkt_matrix(*[T[f] for f in MDS_FIELDS])
    M = k.Msys().copy()
    k.build_kkt_matrix_dist(dist, *[T[f] for f in MDS_FIELDS])
    rows = local_rows(dist)
    ret = dist.matrixChanged(NOPIV)
    dx, dyc, dyd = ctx.zeros(p.nxs + p.nxd), ctx.zeros(p.neq), ctx.zeros(p.nineq)
    ok = ret >= 0 and k.solveCompressed_dist(dist, T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
    ctx.sync()
    out = (M, rows, ret, ok, dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy())
    k.close()
    return out


# N = 260 (three blocks) and N = 900 (seven blocks: more than one per rank at P = 4)
MDS_SHAPES = {"small": (3000, 150, 60, 50, 12, 11), "medium": (20000, 600, 150, 150, 20, 13)}


def mds_problem(name):
    nxs, nxd, neq, nineq, nnz, seed = MDS_SHAPES[name]
    return synth.make_mds_problem(nxs, nxd, neq, nineq, nnz_per_row=nnz, seed=seed)


def mds_problems():
    from test_cpu_mds_model import EDGES, edge_problem
    for name in MDS_SHAPES:
        yield name, mds_problem(name)
    for name, shape, edit in EDGES:
        yield name, edge_problem(name, shape, edit)


@pytest.mark.gpu
def test_mds_dist_build_bit_identical_and_solve_matches_oracle(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseDist
    from oracle import kkt_oracle as ko
    ctx = make_ctx()
    for name, p in mds_problems():
        N = p.nxd + p.neq + p.nineq
        if N == 0:
            continue
        dist = LinSolverSymDenseDist(ctx, N)
        M, rows, ret, ok, dx, dyc, dyd = mds_run(ctx, p, dist)
        dist.close()
        for r, v in rows.items():
            assert np.array_equal(v[r:].view(np.uint64), M[r, r:].view(np.uint64)), (name, r)
        assert name not in MDS_SHAPES or (ret >= 0 and ok), name
        if ret < 0:                                  # an edge whose condensed matrix the no-pivot LDL^T cannot take
            continue
        assert ok, name
        Mo, _, Hxs, _ = ko.mds_build_kkt_matrix(p)
        reto, fac = ko.mds_factorize_with_curv_check(Mo, Hxs)
        if reto >= 0:
            dxo, dyco, dydo = ko.mds_solve_compressed(p, fac, Hxs, p.rx, p.ryc, p.ryd)
            scale = max(1.0, np.abs(dxo).max(initial=0.0), np.abs(dyco).max(initial=0.0), np.abs(dydo).max(initial=0.0))
            err = max(np.abs(dx - dxo).max(initial=0.0), np.abs(dyc - dyco).max(initial=0.0), np.abs(dyd - dydo).max(initial=0.0)) / scale
            assert err <= 1e-8, (name, err)


@pytest.mark.gpu
def test_mds_dist_residual_at_a_medium_size(make_ctx):
    """the uncondensed-system residual of bench.py's independent operators <= 1e-8"""
    import bench
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd, LinSolverSymDenseDist
    ctx = make_ctx()
    nxs, nxd, neq, nineq = 50_000, 1500, 300, 300
    with ctx:
        T = bench.make_mds_device_problem(torch, ctx, nxs, nxd, neq, nineq, nnz_row=max(1, round(5.0 * nxs / (neq + nineq))))
        k = KKTLinSysCompressedMDSXYcYd(ctx, nxs, nxd, neq, nineq, safe_mode=False)
        k.set_sparsity(T["iRc"], T["jCc"], T["iRd"], T["jCd"])
        dist = LinSolverSymDenseDist(ctx, nxd + neq + nineq)
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
        k.build_kkt_matrix_dist(dist, T["Hd"], T["Hs"], T["Jcd"], T["Jdd"], T["Jcs"], T["Jds"], T["vl"], T["sdl"], T["vu"], T["sdu"], T["idl"],
                                T["idu"], T["dwx"], T["dwd"], T["dcc"], T["dcd"])
        assert dist.matrixChanged(NOPIV) == neq + nineq
        dx, dyc, dyd = ctx.zeros(nxs + nxd), ctx.zeros(neq), ctx.zeros(nineq)
        assert k.solveCompressed_dist(dist, T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        ctx.sync()
        res = bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd)
        dist.close()
        k.close()
    assert res <= 1e-8, res


@pytest.mark.gpu
def test_mds_dist_build_bit_identical_at_the_bench_sparse_shape(make_ctx):
    """test_gpu_mds_paths.py's bench shape: n_s = 500 000, m = 2 000 (1 250 sorted columns per row), n_d = 2 000: N = 4 000, 32 blocks"""
    from hiop_b200.engine import LinSolverSymDenseDist
    ctx = make_ctx()
    p = synth.make_mds_problem(500_000, 2000, 1000, 1000, nnz_per_row=1250, seed=42)
    dist = LinSolverSymDenseDist(ctx, 4000)
    M, rows, ret, ok, dx, dyc, dyd = mds_run(ctx, p, dist)
    dist.close()
    assert len(rows) == 4000
    for r, v in rows.items():
        assert np.array_equal(v[r:].view(np.uint64), M[r, r:].view(np.uint64)), r
    torch.cuda.empty_cache()


# ---- several ranks -------------------------------------------------------------------------------------------------------------------------
def _rank_worker(rank, world, uid, out, cases):
    from hiop_b200.engine import Context
    torch.cuda.set_device(rank)
    import os
    os.environ["HB_DENSE_PAIR_MIN"] = str(1 << 30)
    ctx = Context(rank)
    try:
        ctx.init_comm(world, rank, uid)
        for mode, N in cases:
            M, _ = matrix(mode, N, seed=N + mode, device=ctx.device)
            rc, inr, rows, sols = factor_dist(ctx, mode, M, [rhs(N, N, 1), rhs(N, N + 1, 3)])
            out[(rank, mode, N)] = (rc, inr, rows, sols)
        # failure on a block owned by rank 1: the same value on every rank, then an SPD matrix factors
        from hiop_b200.engine import LinSolverSymDenseDist
        N = 700
        s = LinSolverSymDenseDist(ctx, N)
        M, _ = matrix(CHOL, N, 3, ctx.device)
        Mb = M.clone()
        Mb[128 + 7, 128 + 7] = -1.0
        s.set_matrix(Mb)
        r1 = s.matrixChanged(CHOL)
        s.set_matrix(M)
        r2 = s.matrixChanged(CHOL)
        s.close()
        out[(rank, "fail")] = (r1, r2)
        # the mixed dense-sparse path: this rank's rows of the distributed build, and the replicated solution
        for name in MDS_SHAPES:
            p = mds_problem(name)
            dist = LinSolverSymDenseDist(ctx, p.nxd + p.neq + p.nineq)
            _, rows, ret, ok, dx, dyc, dyd = mds_run(ctx, p, dist)
            dist.close()
            out[(rank, "mds", name)] = (rows, ret, ok, dx, dyc, dyd)
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,cases", [(2, [(CHOL, 4099), (NOPIV, 4099)]), (4, [(CHOL, 1000), (NOPIV, 1000), (CHOL, 300), (NOPIV, 300)])],
                         ids=["p2", "p4"])
def test_ranks_match_one_rank_bit_for_bit(make_ctx, world, cases):
    out = run_ranks(_rank_worker, world, (cases,), comm="nccl")
    ctx = make_ctx(HB_DENSE_PAIR_MIN=1 << 30)
    for mode, N in cases:
        M, _ = matrix(mode, N, seed=N + mode, device=ctx.device)
        rc, inr, rows, sols = factor_dist(ctx, mode, M, [rhs(N, N, 1), rhs(N, N + 1, 3)])
        for rank in range(world):
            rrc, rin, rrows, rsols = out[(rank, mode, N)]
            assert (rrc, rin) == (rc, inr)
            assert set(rrows) == {r for b, e in sharding.block_rows(N, world, rank) for r in range(b, e)}
            for r, v in rrows.items():
                assert np.array_equal(v.view(np.uint64), rows[r].view(np.uint64)), (world, rank, mode, N, r)
            for a, b in zip(rsols, sols):
                assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (world, rank, mode, N)
    assert len({out[(rank, "fail")] for rank in range(world)}) == 1 and out[(0, "fail")] == (-1, 0)
    # mixed dense-sparse: each rank's rows are the single-GPU build's rows, the outputs are those of P = 1 on every rank
    from hiop_b200.engine import LinSolverSymDenseDist
    for name in MDS_SHAPES:
        p = mds_problem(name)
        N = p.nxd + p.neq + p.nineq
        dist = LinSolverSymDenseDist(ctx, N)
        M, _, ret, ok, dx, dyc, dyd = mds_run(ctx, p, dist)
        dist.close()
        assert ret >= 0 and ok, name
        for rank in range(world):
            rrows, rret, rok, rdx, rdyc, rdyd = out[(rank, "mds", name)]
            assert set(rrows) == {r for b, e in sharding.block_rows(N, world, rank) for r in range(b, e)}, (name, rank)
            for r, v in rrows.items():
                assert np.array_equal(v[r:].view(np.uint64), M[r, r:].view(np.uint64)), (name, rank, r)
            assert (rret, rok) == (ret, ok), (name, rank)
            for a, b in ((rdx, dx), (rdyc, dyc), (rdyd, dyd)):
                assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (name, rank)
