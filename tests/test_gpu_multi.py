"""Two-GPU parity: the column-sharded engine (NCCL all-reduce inside libhiopb200.so) against the single-GPU engine and
the oracle. Needs >= 2 GPUs (gpurun --gpus 2); skipped otherwise."""
import os

import numpy as np
import pytest
import torch

from hiop_b200 import sharding, synth
from oracle import kkt_oracle as ko
from multirank import run_ranks

pytestmark = pytest.mark.gpu


def _worker(rank, world, uid, out, n, m, l):
    from hiop_b200.engine import Context
    torch.cuda.set_device(rank)
    ctx = Context(rank)
    try:
        ctx.init_comm(world, rank, uid)
        _run(ctx, rank, world, n, m, l, out)
    finally:
        ctx.close()


def _run(ctx, rank, world, n, m, l, out):
    from hiop_b200.engine import KKTLinSysLowRank
    P = synth.make_qn_problem(n, m, l, seed=77)
    b, e = sharding.column_range(n, world, rank)
    sl = slice(b, e)
    D = ctx.to_device
    k = KKTLinSysLowRank(ctx, e - b, P.m_eq, P.m_ineq, max(l, 1))
    J = D(np.ascontiguousarray(P.J[:, sl]))
    T = {name: D(np.ascontiguousarray(getattr(P, name)[sl])) for name in ("ixl", "ixu", "zl", "sxl", "zu", "sxu", "rx")}
    T.update({name: D(getattr(P, name)) for name in ("idl", "idu", "vl", "sdl", "vu", "sdu", "ryc", "ryd")})
    St, Yt = D(np.ascontiguousarray(P.St[:, sl])), D(np.ascontiguousarray(P.Yt[:, sl]))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(J[:P.m_eq], J[P.m_eq:])
    k.set_secant(P.sigma, St if l else None, Yt if l else None, P.L, P.D)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    dx, dyc, dyd = ctx.zeros(e - b), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
    ctx.sync()
    out[f"dx{rank}"] = dx.cpu().numpy()
    out[f"dy{rank}"] = np.concatenate([dyc.cpu().numpy(), dyd.cpu().numpy()])
    out[f"N{rank}"] = k.N()
    # the sharded entry points around the solve: device BiCGStab (compound-vector reductions count replicated blocks once),
    # residual norms, fraction-to-the-boundary, LSQ multipliers
    nb = {"x", "sxl", "sxu", "zl", "zu"}
    shard = lambda name, v: np.ascontiguousarray(v[sl]) if name in nb else np.ascontiguousarray(v)
    res = {rk: D(shard(dk, P.res[rk])) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    dirs = {dk: ctx.zeros(res[rk].numel()) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    ok, info = k.compute_directions_w_IR(res, dirs, mu=1e-2, maxit=8)
    assert ok
    ctx.sync()
    out[f"ir_info{rank}"] = tuple(info)
    for dk in ko.DIR_NAMES:
        out[f"ir_{dk}{rank}"] = dirs[dk].cpu().numpy()
    itr, dat = synth.make_iterate(P)
    it_d = {dk: D(shard(dk, v)) for dk, v in itr.items()}
    xl, xu = D(np.ascontiguousarray(dat["xl"][sl])), D(np.ascontiguousarray(dat["xu"][sl]))
    res2 = {rk: ctx.zeros(it_d[dk].numel()) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    nm = k.residual_update(it_d, D(dat["c"]), D(dat["d"]), D(np.ascontiguousarray(dat["grad"][sl])), 0.1, 1e-5, xl, xu, D(dat["dl"]), D(dat["du"]),
                           D(dat["crhs"]), res2)
    out[f"norms{rank}"] = nm
    rng = np.random.default_rng(5)
    direction = {dk: rng.standard_normal(np.asarray(v).size) * np.where(np.asarray(v) != 0, 1.0, 0.0) for dk, v in itr.items()}
    out[f"ftb{rank}"] = k.fraction_to_bdry(it_d, {dk: D(shard(dk, v)) for dk, v in direction.items()}, 0.995)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(D(np.ascontiguousarray(dat["grad"][sl])), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    out[f"lsq{rank}"] = np.concatenate([yc.cpu().numpy(), yd.cpu().numpy()])
    k.close()


@pytest.mark.parametrize("n,m,l", [(40001, 70, 6), (9000, 140, 0)])
def test_two_gpu_sharded_matches_oracle(n, m, l):
    out = run_ranks(_worker, 2, (n, m, l), comm="nccl")
    P = synth.make_qn_problem(n, m, l, seed=77)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    dx, dyc, dyd, N = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    np.testing.assert_array_equal(out["N0"], out["N1"])          # replicated data stays bit-identical across ranks
    np.testing.assert_array_equal(out["dy0"], out["dy1"])
    assert np.abs(out["N0"] - N).max() <= 1e-12 * np.abs(N).max()
    dxs = np.concatenate([out["dx0"], out["dx1"]])
    assert np.abs(dxs - dx).max() <= 1e-8 * np.abs(dx).max()
    assert np.abs(out["dy0"] - np.concatenate([dyc, dyd])).max() <= 1e-8 * max(1.0, np.abs(dyc).max())
    # sharded entry points around the solve
    it = dict(sxl=P.sxl, sxu=P.sxu, zl=P.zl, zu=P.zu, sdl=P.sdl, sdu=P.sdu, vl=P.vl, vu=P.vu)
    pat = dict(ixl=P.ixl, ixu=P.ixu, idl=P.idl, idu=P.idu)
    do, info_o = ko.compute_directions_w_ir(st, it, pat, P.res, 1e-2, 8, Dx=Dx)
    assert out["ir_info0"][0] == out["ir_info1"][0] == info_o[0] and out["ir_info0"][1] == info_o[1]
    nb = {"x", "sxl", "sxu", "zl", "zu"}
    for dk in ko.DIR_NAMES:
        got = np.concatenate([out[f"ir_{dk}0"], out[f"ir_{dk}1"]]) if dk in nb else out[f"ir_{dk}0"]
        if dk not in nb:
            np.testing.assert_array_equal(out[f"ir_{dk}0"], out[f"ir_{dk}1"])
        assert np.abs(got - do[dk]).max(initial=0.0) <= 1e-8 * max(1.0, np.abs(do[dk]).max(initial=0.0)), dk
    itr, dat = synth.make_iterate(P)
    _, no = ko.residual_update(itr, dat["c"], dat["d"], dat["grad"], P.Jc, P.Jd, 0.1, 1e-5, pat, dat["xl"], dat["xu"], dat["dl"], dat["du"], dat["crhs"])
    for kk in ko.NORM_NAMES:
        assert out["norms0"][kk] == out["norms1"][kk]
        assert abs(out["norms0"][kk] - no[kk]) <= 1e-12 * max(1.0, abs(no[kk])), kk
    rng = np.random.default_rng(5)
    direction = {dk: rng.standard_normal(np.asarray(v).size) * np.where(np.asarray(v) != 0, 1.0, 0.0) for dk, v in itr.items()}
    assert out["ftb0"] == out["ftb1"] == ko.iterate_fraction_to_bdry(itr, direction, 0.995, pat)
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, dat["grad"], P.zl, P.zu, P.vl, P.vu)
    np.testing.assert_array_equal(out["lsq0"], out["lsq1"])
    assert np.abs(out["lsq0"] - np.concatenate([yco, ydo])).max() <= 1e-9 * max(1.0, np.abs(np.concatenate([yco, ydo])).max())
