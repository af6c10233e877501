"""Measures the dense symmetric solver with the matrix in page-locked host memory (hb_symdense_host) against hb_symdense in HBM.

    python tools/bench_host_symdense.py [--sizes 22000] [--budget-gib 4,80] [--modes cholesky,nopiv_ldlt,rbt] [--repeats 3] [--warmup 1]

First line: the rate of plain pinned-host <-> device copies of 1 GiB (device events), the ceiling of the streaming. Then one JSON line
per (N, budget, mode): factor ms (host clock around the synchronous call; the median, min and max of the repeats), solve ms for one
right-hand side (host clock around the call and a synchronise), the slab count, the H2D and D2H bytes of one factorization from the plan
and those bytes over the factor time, N^3/3 over the factor time, and, when the matrix fits in HBM, hb_symdense on the same matrix with
its 128-column blocks never paired (the factorization the host-resident one reproduces bit for bit: K = 128 updates), timed the same
way and alternating with the host-resident runs, with max |x_host - x_hbm| (the factors are the same bits; the two solves run
different kernels). The card's name and power limit are read in the same run.

The matrix: uniform [0, 1) entries above the diagonal and 2 N on it (diagonally dominant; the no-pivot LDL^T gets -2 N on the first
N / 3 diagonal entries, hence N / 3 negative eigenvalues). Only the upper triangle is filled; the factorization reads nothing else.

--modes rbt (the safe mode, LinSolverSymDenseHost(rbt=True) on the no-pivot matrix): factor ms (host clock, transform included), the
transform's ms (device events) and its share of the factor, its H2D + D2H bytes from the plan over its time, solve ms of one right-hand
side with its corrections and omega, the strips and slabs, and the bytes of the plan; then the same matrix through hb_symdense_dist RBT
at P = 1 (whose x the host handle reproduces bit for bit: max |x_host - x_dist| is reported) and, when it fits next to the device copy,
through hb_symdense RBT in HBM, timed the same way."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHOL, NOPIV, RBT = 2, 1, 3
MODES = {"cholesky": CHOL, "nopiv_ldlt": NOPIV, "rbt": RBT}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    name, _, power = out.stdout.strip().partition(",")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def copy_rates(dev):
    """GB/s of 1 GiB pinned host -> device and device -> host copies (device events, median of 5)"""
    n = 1 << 27
    h = torch.empty(n, dtype=torch.float64, pin_memory=True).fill_(1.0)
    d = torch.empty(n, dtype=torch.float64, device=dev)
    out = {}
    for name, (dst, src) in (("h2d", (d, h)), ("d2h", (h, d))):
        ms = []
        for _ in range(6):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dst.copy_(src, non_blocking=True)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        out[f"pinned_{name}_GBps"] = 8 * n / (statistics.median(ms[1:]) * 1e-3) / 1e9
    return out


def fill(src, mode, seed):
    """the benchmark matrix into the pinned host tensor src (upper triangle and diagonal)"""
    N = src.shape[0]
    g = torch.Generator().manual_seed(seed)
    torch.rand(src.shape, generator=g, dtype=torch.float64, out=src)
    d = torch.full((N,), 2.0 * N, dtype=torch.float64)
    if mode == NOPIV:
        d[: N // 3] = -2.0 * N
    src.diagonal().copy_(d)


def spread(v):
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def timed(call, sync):
    sync()
    t0 = time.perf_counter()
    out = call()
    sync()
    return (time.perf_counter() - t0) * 1e3, out


def run_rbt(ctx, N, gibs, args, info):
    """one JSON line per budget: the safe mode on the host-resident handle against hb_symdense_dist (P = 1) and hb_symdense in HBM"""
    from hiop_b200.engine import LinSolverSymDense, LinSolverSymDenseDist, LinSolverSymDenseHost
    dev = ctx.device
    src = torch.empty((N, N), dtype=torch.float64, pin_memory=True)
    fill(src, NOPIV, seed=N + RBT)
    b = torch.randn(N, generator=torch.Generator().manual_seed(7), dtype=torch.float64).to(dev)
    sync = ctx.sync

    def measure(setup, factor, solve, stats):
        f_ms, s_ms = [], []
        x = torch.empty_like(b)
        for it in range(args.warmup + args.repeats):
            setup()
            ms, rc = timed(factor, sync)
            with torch.cuda.stream(ctx.stream):
                x.copy_(b)
            ms_s, ok = timed(lambda: solve(x), sync)
            if it >= args.warmup:
                f_ms.append(ms)
                s_ms.append(ms_s)
        corr, om, t_ms = stats()
        return {"rc": rc, "solve_ok": bool(ok), "factor_ms": spread(f_ms), "solve_ms": spread(s_ms), "corrections": corr, "omega": om,
                "transform_ms": t_ms}, x

    ref = {}
    # hb_symdense_dist at P = 1 (A and A' on the device) and hb_symdense (the matrix, A' and the device copy it is filled from)
    free = torch.cuda.mem_get_info(dev)[0]
    if 3.3 * 8 * N * N < free:
        Md = src.to(dev)
        d = LinSolverSymDenseDist(ctx, N)
        d.profile(True)
        r, xd = measure(lambda: d.set_matrix(Md), lambda: d.matrixChanged(RBT), d.solve, d.rbt_stats)
        d.profile(False)
        d.close()
        ref["hb_symdense_dist_p1"] = r
        torch.cuda.empty_cache()
        ss = LinSolverSymDense(ctx, N, RBT)

        def sset():
            ss.set_matrix(Md)
            sync()
        r, _ = measure(sset, ss.matrixChanged, ss.solve, ss.rbt_stats)
        ss.close()
        ref["hb_symdense_in_hbm"] = r
        del Md
        torch.cuda.empty_cache()
    else:
        xd = None
    for gib in gibs:
        budget = int(gib * (1 << 30))
        p = LinSolverSymDenseHost.rbt_plan_view(N, budget)
        s = LinSolverSymDenseHost(ctx, N, budget, rbt=True)
        r, x = measure(lambda: s.matrix().copy_(src), lambda: s.matrixChanged(RBT), s.solve, s.rbt_stats)
        s.close()
        tx = r["transform_ms"]
        print(json.dumps({"N": N, "mode": "rbt", "budget_gib": gib, "strips": p["strips"], "strip_slots": p["strip_slots"], "slabs": p["slabs"],
                          "slab_block_rows": p["slab_blocks"], "peak_device_bytes": p["peak_bytes"], **r,
                          "transform_share_of_factor": tx / r["factor_ms"]["median"],
                          "transform_h2d_bytes": p["transform_h2d_bytes"], "transform_d2h_bytes": p["transform_d2h_bytes"],
                          "transform_h2d_plus_d2h_GBps": (p["transform_h2d_bytes"] + p["transform_d2h_bytes"]) / (tx * 1e-3) / 1e9 if tx else None,
                          "factor_h2d_bytes": p["factor_h2d_bytes"], "residual_h2d_bytes_per_pass": p["residual_h2d_bytes"],
                          "max_abs_diff_x_vs_dist": float((x - xd).abs().max()) if xd is not None else None, **ref, **info}), flush=True)
    del src


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="22000")
    ap.add_argument("--budget-gib", default="4,80")
    ap.add_argument("--modes", default="cholesky", help="comma-separated: cholesky, nopiv_ldlt")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_symdense needs a CUDA device; nothing is measured without one")
    from hiop_b200.engine import Context, LinSolverSymDense, LinSolverSymDenseHost
    ctx = Context(0)
    dev = ctx.device
    os.environ["HB_DENSE_PAIR_MIN"] = str(1 << 30)   # hb_symdense with K = 128 updates, the factorization reproduced here
    ctx_k128 = Context(0)
    del os.environ["HB_DENSE_PAIR_MIN"]
    info = card()
    print(json.dumps({"workload": "pinned copies of 1 GiB", **copy_rates(dev), **info}), flush=True)
    for N in [int(v) for v in args.sizes.split(",")]:
        for mname in args.modes.split(","):
            mode = MODES[mname]
            if mode == RBT:
                run_rbt(ctx, N, [float(v) for v in args.budget_gib.split(",")], args, info)
                continue
            want = N // 3 if mode == NOPIV else 0
            src = torch.empty((N, N), dtype=torch.float64, pin_memory=True)
            fill(src, mode, seed=N + mode)
            b = torch.randn(N, generator=torch.Generator().manual_seed(7), dtype=torch.float64).to(dev)
            free = torch.cuda.mem_get_info(dev)[0]
            fits = 2.2 * 8 * N * N < free                 # hb_symdense's matrix and the device copy it is filled from
            Md = src.to(dev) if fits else None
            for gib in [float(v) for v in args.budget_gib.split(",")]:
                budget = int(gib * (1 << 30))
                p = LinSolverSymDenseHost.plan_view(N, budget)
                s = LinSolverSymDenseHost(ctx, N, budget)
                x = torch.empty_like(b)

                def factor():
                    s.matrix().copy_(src)
                    t0 = time.perf_counter()
                    rc = s.matrixChanged(mode)
                    ms = (time.perf_counter() - t0) * 1e3
                    assert rc == want, rc
                    return ms

                def solve():
                    with torch.cuda.stream(ctx.stream):
                        x.copy_(b)
                    ctx.sync()
                    t0 = time.perf_counter()
                    assert s.solve(x)
                    ctx.sync()
                    return (time.perf_counter() - t0) * 1e3

                ss = None
                if fits:
                    ss = LinSolverSymDense(ctx_k128, N, mode)
                    xs = torch.empty_like(b)

                def sfactor():
                    ss.set_matrix(Md)
                    ctx_k128.sync()
                    t0 = time.perf_counter()
                    assert ss.matrixChanged() == want
                    ctx_k128.sync()
                    return (time.perf_counter() - t0) * 1e3

                def ssolve():
                    with torch.cuda.stream(ctx_k128.stream):
                        xs.copy_(b)
                    ctx_k128.sync()
                    t0 = time.perf_counter()
                    assert ss.solve(xs)
                    ctx_k128.sync()
                    return (time.perf_counter() - t0) * 1e3

                for _ in range(args.warmup):
                    factor()
                    solve()
                    if ss:
                        sfactor()
                        ssolve()
                f_ms, s_ms, sf_ms, ss_ms = [], [], [], []
                for _ in range(args.repeats):              # alternate the two solvers
                    f_ms.append(factor())
                    s_ms.append(solve())
                    if ss:
                        sf_ms.append(sfactor())
                        ss_ms.append(ssolve())
                fmed = statistics.median(f_ms)
                in_hbm = None
                if ss:
                    in_hbm = {"factor_ms": spread(sf_ms), "solve_ms": spread(ss_ms),
                              "tflops": N ** 3 / 3 / (statistics.median(sf_ms) * 1e-3) / 1e12,
                              "max_abs_diff_x": float((x - xs).abs().max())}
                    ss.close()
                s.close()
                d2h = p["d2h_bytes_ldlt"] if mode == NOPIV else p["d2h_bytes_cholesky"]
                print(json.dumps({"N": N, "mode": mname, "budget_gib": gib, "slabs": p["slabs"], "slab_block_rows": p["slab_blocks"],
                                  "peak_device_bytes": p["peak_bytes"], "factor_ms": spread(f_ms), "solve_ms": spread(s_ms),
                                  "tflops": N ** 3 / 3 / (fmed * 1e-3) / 1e12, "h2d_bytes": p["h2d_bytes"], "d2h_bytes": d2h,
                                  "h2d_plus_d2h_GBps_over_factor": (p["h2d_bytes"] + d2h) / (fmed * 1e-3) / 1e9,
                                  "solve_h2d_bytes": p["solve_h2d_bytes"], "hb_symdense_k128_in_hbm": in_hbm, **info}), flush=True)
            del Md, src
            torch.cuda.empty_cache()
    ctx_k128.close()
    ctx.close()


if __name__ == "__main__":
    main()
