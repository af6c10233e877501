"""Measures the dense symmetric factorization distributed over P GPUs (hb_symdense_dist) against the single-GPU hb_symdense.

    torchrun --nproc-per-node P tools/bench_dist_symdense.py [--sizes 8192,22000,32768] [--steps 3] [--warmup 1]
    python tools/bench_dist_symdense.py            # P = 1

Prints one JSON line per (N, mode, P) from rank 0: factor and solve ms (device events, maximum over ranks, after warm-up), N^3/3 over
the factor time, the bytes one factorization broadcasts (from the shapes), the per-phase sums of one profiled factorization (maximum
over ranks: panel chain, broadcast including the wait for the owner, trailing update), hb_symdense's time on the same matrix on rank 0
with its default dispatch and with its blocks never paired (K = 128 updates), max |x_dist - x_single| / |x|, and the card's name and power limit.
Mode rbt (the safe mode, HB_FACT_RBT_NOPIV) adds the transform time of one profiled factorization, the corrections and backward error of
the refined solve, and whether its inertia equals hb_symdense's Bunch-Kaufman on rank 0 on the same matrix, and the same for the one-GPU
safe mode (hb_symdense with HB_FACT_RBT_NOPIV) on rank 0. Then one line each for a mixed dense-sparse step in speculative mode (no-pivot
LDL^T) and in stable mode (RBT; update + build + factor + solve) at bench.py's MDS size, distributed against the replicated single-GPU step
(stable: Bunch-Kaufman, and the one-GPU RBT step), with the residual of the uncondensed system (must be <= 1e-8)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHOL, NOPIV, RBT, BK = 2, 1, 3, 0
BLOCK, HDR = 128, 136   # hb_blockrow.cu (HB_ROWS_DB, HB_ROWS_HDR): block size, broadcast step header (doubles)


def card(local_rank):
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local_rank)], capture_output=True, text=True)
    name, _, power = out.stdout.strip().partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def broadcast_bytes(N):
    """one factorization: per block k the header and the 128 panel columns of the rows below it (even row count)"""
    nblk = (N + BLOCK - 1) // BLOCK
    tot = 0
    for k in range(nblk):
        rows = max(0, N - min(N, (k + 1) * BLOCK))
        tot += 8 * (HDR + BLOCK * ((rows + 1) & ~1))
    return tot


def make_matrix(mode, N, dev, seed):
    """diagonally dominant symmetric matrix: SPD (Cholesky) or with N // 3 negative eigenvalues (no-pivot LDL^T)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    R = torch.rand((N, N), generator=g, dtype=torch.float64, device=dev)
    M = R + R.T
    del R
    d = torch.full((N,), 2.0 * N, dtype=torch.float64, device=dev)
    if mode == NOPIV:
        d[: N // 3] = -2.0 * N
    M.diagonal().copy_(d)
    return M


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,22000,32768")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-mds", action="store_true")
    ap.add_argument("--mds-ns", type=int, default=500_000)
    ap.add_argument("--mds-nd", type=int, default=20_000)
    ap.add_argument("--mds-m", type=int, default=2000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dist_symdense needs CUDA devices; nothing is measured without them")
    import torch.distributed as dist
    from hiop_b200.engine import Context, LinSolverSymDense, LinSolverSymDenseDist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("gloo")
    ctx = Context(local_rank)
    if world > 1:
        box = [ctx.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        ctx.init_comm(world, rank, box[0])
    dev = ctx.device
    info = card(local_rank)
    ctx_k128 = None
    if rank == 0:
        # hb_symdense with its 128-column blocks never paired (K = 128 updates, as the distributed factorization runs them): what
        # separates the distributed factor from hb_symdense's default K = 256 updates
        os.environ["HB_DENSE_PAIR_MIN"] = str(1 << 30)
        ctx_k128 = Context(local_rank)
        del os.environ["HB_DENSE_PAIR_MIN"]

    def rmax(v):
        if world == 1:
            return v
        t = torch.tensor([float(x) for x in np.atleast_1d(v)], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.tolist() if np.ndim(v) else float(t[0])

    def timed(fn, steps, c=ctx):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(c.stream)
        for _ in range(steps):
            fn()
        e1.record(c.stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    for N in [int(v) for v in args.sizes.split(",")]:
        for mode in (CHOL, NOPIV):
            M = make_matrix(mode, N, dev, seed=N + mode)
            b = torch.randn(N, generator=torch.Generator(device=dev).manual_seed(7), dtype=torch.float64, device=dev)
            torch.cuda.synchronize()
            s = LinSolverSymDenseDist(ctx, N)
            x = torch.empty_like(b)

            def factor():
                s.set_matrix(M)
                rc = s.matrixChanged(mode)
                assert rc == (N // 3 if mode == NOPIV else 0), rc
            copy_ms = timed(lambda: s.set_matrix(M), 1)
            for _ in range(args.warmup):
                factor()
            f_ms = timed(factor, args.steps) - copy_ms
            s.profile(True)
            factor()
            phases = s.profile(False)

            def solve():
                with torch.cuda.stream(ctx.stream):   # in order with the previous solve, which runs on the engine's stream
                    x.copy_(b)
                assert s.solve(x)
            solve()
            s_ms = timed(solve, args.steps)
            x_dist = x.clone()
            s.close()
            f_ms, s_ms = rmax(f_ms), rmax(s_ms)
            phases = rmax(list(phases))
            single = None
            if rank == 0:
                ss = LinSolverSymDense(ctx, N, mode)

                def sfactor():
                    ss.set_matrix(M)
                    assert ss.matrixChanged() == (N // 3 if mode == NOPIV else 0)
                sfactor()
                c_ms = timed(lambda: ss.set_matrix(M), 1)
                sf_ms = timed(sfactor, args.steps) - c_ms
                xs = b.clone()
                torch.cuda.synchronize()
                assert ss.solve(xs)
                ctx.sync()
                diff = float((x_dist - xs).abs().max() / xs.abs().max())
                ss.close()
                resid = lambda v: float((M @ v - b).abs().max() / b.abs().max())
                su = LinSolverSymDense(ctx_k128, N, mode)

                def ufactor():
                    su.set_matrix(M)
                    assert su.matrixChanged() == (N // 3 if mode == NOPIV else 0)
                ufactor()
                cu_ms = timed(lambda: su.set_matrix(M), 1, ctx_k128)
                uf_ms = timed(ufactor, args.steps, ctx_k128) - cu_ms
                su.close()
                single = {"factor_ms": sf_ms, "tflops": N ** 3 / 3 / (sf_ms * 1e-3) / 1e12, "max_rel_diff_x": diff, "resid_single": resid(xs),
                          "resid_dist": resid(x_dist), "factor_ms_blocks_unpaired_k128": uf_ms}
            del M
            torch.cuda.empty_cache()
            if rank == 0:
                print(json.dumps({"N": N, "mode": "cholesky" if mode == CHOL else "nopiv_ldlt", "P": world, "factor_ms": f_ms, "solve_ms": s_ms,
                                  "tflops": N ** 3 / 3 / (f_ms * 1e-3) / 1e12,
                                  "broadcast_bytes_per_factor": broadcast_bytes(N) if world > 1 else 0,
                                  "phase_ms_max_over_ranks": {"panel_chain": phases[0], "broadcast": phases[1], "trailing_update": phases[2]},
                                  "single_gpu_hb_symdense_rank0": single, **info}), flush=True)

        run_rbt(N, ctx, world, rank, rmax, timed, info)

    if not args.no_mds:
        run_mds(args, ctx, world, rank, rmax, timed, info)
        run_mds(args, ctx, world, rank, rmax, timed, info, stable=True)
    if ctx_k128:
        ctx_k128.close()
    ctx.close()
    if world > 1:
        dist.destroy_process_group()


def run_rbt(N, ctx, world, rank, rmax, timed, info):
    """the safe mode on the no-pivot matrix of make_matrix: factor and solve ms, transform ms, corrections, backward error, inertia check"""
    from hiop_b200.engine import LinSolverSymDense, LinSolverSymDenseDist
    dev = ctx.device
    M = make_matrix(NOPIV, N, dev, seed=N + RBT)
    b = torch.randn(N, generator=torch.Generator(device=dev).manual_seed(7), dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    s = LinSolverSymDenseDist(ctx, N)
    x = torch.empty_like(b)

    def factor():
        s.set_matrix(M)
        rc = s.matrixChanged(RBT)
        assert rc == N // 3, rc
    copy_ms = timed(lambda: s.set_matrix(M), 1)
    factor()
    f_ms = timed(factor, 3) - copy_ms
    s.profile(True)
    factor()
    s.profile(False)
    transform_ms = s.rbt_stats()[2]
    inertia = s.inertia()

    def solve():
        with torch.cuda.stream(ctx.stream):
            x.copy_(b)
        assert s.solve(x)
    solve()
    s_ms = timed(solve, 3)
    corr, berr, _ = s.rbt_stats()
    s.close()
    f_ms, s_ms, transform_ms = rmax(f_ms), rmax(s_ms), rmax(transform_ms)
    same = single = None
    if rank == 0:
        ss = LinSolverSymDense(ctx, N, BK)
        ss.set_matrix(M)
        rc_bk = ss.matrixChanged()
        in_bk = ss.inertia()
        same = rc_bk == N // 3 and in_bk == inertia
        ss.close()
        # the same safe mode on one GPU (hb_symdense): fused transform, NOPIV's plan on A', refined solve
        su = LinSolverSymDense(ctx, N, RBT)

        def sfactor():
            su.set_matrix(M)
            assert su.matrixChanged() == N // 3
        sfactor()
        c_ms = timed(lambda: su.set_matrix(M), 1)
        sf_ms = timed(sfactor, 3) - c_ms
        t_ms = su.rbt_stats()[2]

        def ssolve():
            with torch.cuda.stream(ctx.stream):
                x.copy_(b)
            assert su.solve(x)
        ssolve()
        ss_ms = timed(ssolve, 3)
        scorr, sberr, _ = su.rbt_stats()
        single = {"factor_ms": sf_ms, "transform_ms": t_ms, "solve_ms": ss_ms, "corrections": scorr, "backward_error": sberr,
                  "inertia_equals_bunch_kaufman": rc_bk == N // 3 and su.inertia() == in_bk}
        su.close()
    del M
    torch.cuda.empty_cache()
    if rank == 0:
        print(json.dumps({"N": N, "mode": "rbt", "P": world, "factor_ms": f_ms, "solve_ms": s_ms, "transform_ms": transform_ms,
                          "corrections": corr, "backward_error": berr, "inertia": list(inertia), "inertia_equals_bunch_kaufman_rank0": same,
                          "single_gpu_hb_symdense_rank0": single, **info}), flush=True)


def run_mds(args, ctx, world, rank, rmax, timed, info, stable=False):
    import bench
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd, LinSolverSymDenseDist
    nxs, nxd, m = args.mds_ns, args.mds_nd, args.mds_m
    nineq = m // 2
    neq = m - nineq
    nnz_row = max(1, int(round(5.0 * nxs / max(m, 1))))
    N = nxd + m
    with ctx:
        T = bench.make_mds_device_problem(torch, ctx, nxs, nxd, neq, nineq, nnz_row)
        dx, dyc, dyd = ctx.zeros(nxs + nxd), ctx.zeros(neq), ctx.zeros(nineq)
        k = KKTLinSysCompressedMDSXYcYd(ctx, nxs, nxd, neq, nineq, safe_mode=False)
        k.set_sparsity(T["iRc"], T["jCc"], T["iRd"], T["jCd"])
        blocks = (T["Hd"], T["Hs"], T["Jcd"], T["Jdd"], T["Jcs"], T["Jds"], T["vl"], T["sdl"], T["vu"], T["sdu"], T["idl"], T["idu"], T["dwx"], T["dwd"],
                  T["dcc"], T["dcd"])
        s = LinSolverSymDenseDist(ctx, N)

        def step_dist():
            k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
            k.build_kkt_matrix_dist(s, *blocks)
            if stable:
                assert k.factorizeWithCurvCheck_dist(s, safe_mode=True) == neq + nineq
            else:
                assert s.matrixChanged(NOPIV) == neq + nineq
            assert k.solveCompressed_dist(s, T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
        for _ in range(max(args.warmup, 1)):
            step_dist()
        ms = rmax(timed(step_dist, args.steps))
        resid = bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd)
        dxd = dx.clone()
        s.close()
        single = None
        if rank == 0:
            if stable:       # the single-GPU stable step: Bunch-Kaufman
                k.close()
                k = KKTLinSysCompressedMDSXYcYd(ctx, nxs, nxd, neq, nineq, safe_mode=True)
                k.set_sparsity(T["iRc"], T["jCc"], T["iRd"], T["jCd"])

            def step_single():
                k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
                k.build_kkt_matrix(*blocks)
                assert k.factorizeWithCurvCheck() == neq + nineq
                assert k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
            step_single()
            sms = timed(step_single, args.steps)
            single = {"ms_per_step": sms, "resid": bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd),
                      "max_rel_diff_dx": float((dxd - dx).abs().max() / dx.abs().max())}
            if stable:       # the single-GPU stable step with the random-butterfly safe mode instead of Bunch-Kaufman
                k.linSys.mode = k.linSys.RBT_NOPIV
                step_single()
                single["rbt_ms_per_step"] = timed(step_single, args.steps)
                single["rbt_resid"] = bench.mds_independent_residual(torch, T, nxs, nxd, neq, nineq, dx, dyc, dyd)
                single["rbt_transform_ms"] = k.linSys.rbt_stats()[2]
        k.close()
    assert resid <= 1e-8, resid
    if rank == 0:
        print(json.dumps({"workload": f"mds {'stable' if stable else 'speculative'} step n_s={nxs} n_d={nxd} m={m} (N={N})", "P": world, "ms_per_step": ms,
                          "kkt_residual_rel_independent_operators": resid, "single_gpu_replicated_step_rank0": single, **info}), flush=True)


if __name__ == "__main__":
    main()
