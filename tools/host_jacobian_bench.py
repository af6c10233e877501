"""Times one quasi-Newton step with the Jacobian in device memory against the same step with it in page-locked host memory
(hb_lowrank_set_jacobian_host), at a chosen n, m and panel width:

  step = update + condense + solveCompressed (condensation pending, so the fused rhs row applies where it is free), and
  ir   = one compute_directions_w_IR solve (the outer BiCGStab refinement on the full KKT system).

For the host J it reports the H2D rate the step reached, counting 8 m n bytes per pass over J (a step makes two passes: the condensation
and J^T dy). Prints one JSON line with the card name and its power limit.

    python tools/host_jacobian_bench.py --n 1000000 --m 1000 --panel-cols 0 --reps 5 [--no-device]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hiop_b200 import synth  # noqa: E402
from hiop_b200.engine import Context, KKTLinSysLowRank  # noqa: E402
from oracle import kkt_oracle as ko  # noqa: E402

ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


def _power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True,
                             timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def _time(ctx, fn, reps):
    fn()                                        # warm-up: lazy buffers, schedules, the chunk table
    ctx.sync()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        a.record(ctx.stream)
        fn()
        b.record(ctx.stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def run(ctx, P, T, host, panel_cols, reps):
    l = P.l
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, max(l, 1))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    if host:
        Jc, Jd = (torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (P.Jc, P.Jd))
        k.set_jacobian_host(Jc, Jd, panel_cols)
    else:
        J = ctx.to_device(P.J)
        k.set_jacobian(J[:P.m_eq], J[P.m_eq:])
    k.set_secant(P.sigma, T["St"] if l else None, T["Yt"] if l else None, P.L, P.D)
    D = ctx.to_device
    rx0, ryc, ryd = D(P.rx), D(P.ryc), D(P.ryd)
    rx, dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)

    def step():
        k.update(*(T[kk] for kk in ITERATE))
        rx.copy_(rx0)
        k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)

    res = {kk: D(P.res[kk]) for kk in ko.RES_NAMES}
    sizes = dict(x=P.n, d=P.m_ineq, yc=P.m_eq, yd=P.m_ineq, sxl=P.n, sxu=P.n, sdl=P.m_ineq, sdu=P.m_ineq, zl=P.n, zu=P.n, vl=P.m_ineq, vu=P.m_ineq)
    dirs = {kk: ctx.zeros(sizes[kk]) for kk in ko.DIR_NAMES}
    info = []

    def ir():
        info[:] = [k.compute_directions_w_IR(res, dirs, 1e-2, 8)[1]]

    with ctx:
        out = dict(step_ms=_time(ctx, step, reps), ir_ms=_time(ctx, ir, reps))
    out["ir_info"] = list(info[0])
    if host:
        out["h2d_GBps_step"] = 2 * 8 * P.m * P.n / (out["step_ms"] * 1e6)
    k.close()
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--m", type=int, default=1000)
    ap.add_argument("--l", type=int, default=6)
    ap.add_argument("--panel-cols", type=int, default=0, help="0: the default width (about 128 MB per panel)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-device", action="store_true", help="skip the device-J run (J larger than HBM)")
    a = ap.parse_args()
    P = synth.make_qn_problem(a.n, a.m, a.l, seed=5)
    ctx = Context(0)
    T = {name: ctx.to_device(getattr(P, name)) for name in ("ixl", "ixu", "idl", "idu", "zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu", "St", "Yt")}
    result = dict(card=torch.cuda.get_device_name(0), power_limit_w=_power_limit_w(), n=a.n, m=a.m, l=a.l, J_GB=8 * a.m * a.n / 1e9,
                  panel_cols=a.panel_cols)
    if not a.no_device:
        result["device"] = run(ctx, P, T, False, a.panel_cols, a.reps)
    result["host"] = run(ctx, P, T, True, a.panel_cols, a.reps)
    print(json.dumps(result))
    ctx.close()


if __name__ == "__main__":
    main()
