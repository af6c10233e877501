"""Condensation modes side by side on one device: exact FP64 DMMA, 8 int8 slices and int8 Chinese remaindering.

One process builds the quasi-Newton workload of bench.py (default n = 1e6, m = 1000, l = 6), warms every mode up, then alternates
dmma / oz8 / crt for --rounds rounds of --steps steps each. Per mode it prints one JSON line: the step time (update + condensation +
solveCompressed, CUDA events), the dominant kernel of each round's last step (k_syrk_ws / k_oz_gemm / k_crt_gemm, hb_ctx_last_syrk_ms, read after the timed
window so that the steps run without a host synchronisation), the phase timeline of one
step, the useful int8 rate of the int8 GEMMs against the measured int8 wgmma peak (hb_microbench_peak(ctx, 1)), and
max|N - N_fp64| / max|N_fp64|. Each line names the device, its power limit and the median SM clock under load (bench.ClockSampler).

    python tools/bench_condense_modes.py [--n 1000000 --m 1000 --l 6 --steps 5 --rounds 3 --warmup 2]

It needs a GPU and fails without one; it writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODES = {"dmma": 0, "oz8": 8, "crt": 100}


def int8_ops(mode, n, Ma):
    """useful int8 tensor operations (2 per MAC) of the upper-triangle tiles the mode's GEMM computes"""
    if mode == "oz8":
        Mpad = -(-Ma // 128) * 128
        tiles = sum(1 for bi in range(Mpad // 128) for bj in range(4 * bi, Mpad // 32) if bj * 32 < Ma)
        return 2.0 * tiles * 128 * 32 * n * 36          # 36 slice products per tile
    if mode == "crt":
        from oracle import crt_model
        nb = -(-Ma // 128)
        return 2.0 * (nb * (nb + 1) // 2) * 128 * 128 * n * crt_model.n_moduli(n)
    return 0.0


def power_limit(idx):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={idx}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return float(out)
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1000000)
    ap.add_argument("--m", type=int, default=1000)
    ap.add_argument("--l", type=int, default=6)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    from bench import ClockSampler, make_device_problem
    from hiop_b200.engine import Context, KKTLinSysLowRank
    if not torch.cuda.is_available():
        raise SystemExit("bench_condense_modes.py needs a GPU")
    n, m, l = args.n, args.m, args.l
    ctx = Context(0)
    T = make_device_problem(ctx, torch, n, n, m, l, 0, 1, None)
    m_eq, m_ineq = T["m_eq"], T["m_ineq"]
    k = KKTLinSysLowRank(ctx, n, m_eq, m_ineq, max(l, 1))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:m_eq], T["J"][m_eq:])
    k.set_secant(1.0, T["St"] if l else None, T["Yt"] if l else None, T["L"], T["D"])
    ctx.enable_timing(True)
    rx_work = ctx.zeros(n)
    dx, dyc, dyd = ctx.zeros(n), ctx.zeros(m_eq), ctx.zeros(m_ineq)
    name = torch.cuda.get_device_name(0)
    plimit = power_limit(0)

    def step():
        rx_work.copy_(T["rx"])
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
        assert k.solveCompressed(rx_work, T["ryc"], T["ryd"], dx, dyc, dyd)

    res = {md: {"ms_step": [], "kernel_ms": [], "clock": []} for md in MODES}
    Nref, dev = {}, {}
    with ctx:
        peak_i8 = ctx.microbench_peak(1)
        for md, code in MODES.items():                 # warm-up of every mode, one phase timeline, N of each mode
            k.set_condense_mode(code)
            for _ in range(args.warmup):
                step()
            k.check()
            ctx.phase_timeline(True)
            step()
            res[md]["phases"] = {ph: round(v, 3) for ph, v in ctx.phase_timeline(False).items()}
            k.check()
            assert k.condense_mode_used() == code
            Nref[md] = k.N()
        for md in MODES:
            dev[md] = float(np.abs(Nref[md] - Nref["dmma"]).max() / np.abs(Nref["dmma"]).max())
        for _ in range(args.rounds):
            for md, code in MODES.items():
                k.set_condense_mode(code)
                step()                                 # the first step after a mode switch re-plans the schedule
                ctx.sync()
                sampler = ClockSampler(0)
                sampler.start()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):                # enqueued back to back: no host synchronisation inside the timed window
                    step()
                e1.record()
                ctx.sync()
                torch.cuda.synchronize()
                k.check()
                ck = sampler.stop()
                res[md]["ms_step"].append(e0.elapsed_time(e1) / args.steps)
                res[md]["kernel_ms"].append(ctx.last_syrk_ms())   # the dominant kernel of the round's last step, read after the window
                if ck.get("sm_mhz"):
                    res[md]["clock"].append(ck["sm_mhz"])
    Ma = m + 2 * l
    for md in MODES:
        r = res[md]
        kms = statistics.median(r["kernel_ms"])
        ops = int8_ops(md, n, Ma)
        print(json.dumps({
            "mode": md, "device": name, "power_limit_w": plimit, "sm_clock_mhz_median": statistics.median(r["clock"]) if r["clock"] else None,
            "n": n, "m": m, "l": l, "rounds": args.rounds, "steps_per_round": args.steps,
            "ms_step_median": round(statistics.median(r["ms_step"]), 3), "ms_step_rounds": [round(x, 3) for x in r["ms_step"]],
            "kernel_ms_median": round(kms, 3), "phase_ms": r["phases"],
            "int8_tops": round(ops / (kms * 1e-3) / 1e12, 1) if ops else None, "int8_peak_tops": round(peak_i8, 1),
            "int8_share_of_peak": round(ops / (kms * 1e-3) / 1e12 / peak_i8, 3) if ops else None,
            "max_dN_over_max_N_vs_fp64": dev[md]}), flush=True)
    k.close()
    ctx.close()


if __name__ == "__main__":
    main()
