"""The column-sharded quasi-Newton engine (n split over NCCL ranks, m and l replicated, sharding.column_range) held to the same engine on
one GPU, at P = 1, 2 and 4 ranks.

Every output of a sharded run falls in one of three kinds, each checked without a conditioning-dependent tolerance:
  - replicated (m- and l-sized results, scalars): bit-identical on every rank;
  - column-local (elementwise n-sized results): bit-identical to a one-rank handle on that rank's columns;
  - summed (Gram blocks, dots): the one-rank partials of the shards plus the all-reduce -- fl(G0 + G1) bit for bit at P = 2, where the
    single addition is commutative, and within gamma(P - 1) sum |G_r| at P = 4, where NCCL's order is unspecified.
End-to-end results are also held to the oracle. Two defects are pinned here: the adjusted-slack count must be the global one on every
rank, and a failed LSQ factorization must leave the caller's multipliers untouched (on one GPU too).

One multirank.run_ranks call per world size runs every case; each rank writes arrays back through a manager, and a hung collective
fails the test after a timeout with every rank terminated. Skipped when fewer than P GPUs are present."""
import ctypes
import functools
import time

import numpy as np
import pytest
import torch

from hiop_b200 import sharding, synth
from oracle import bounds
from oracle import kkt_oracle as ko
from multirank import run_ranks

pytestmark = pytest.mark.gpu

N_BLOCKS = set(sharding.N_BLOCKS)
SENTINEL = 0.3125                                   # what yc, yd hold before an LSQ call that must not touch them
REPLICATED = ("N", "Z", "V", "p2l", "dy", "ir_info", "ir_m", "norms", "ftb", "flog", "gd", "step_m", "nadj", "lsq", "lsq_bad", "cond_bad",
              "vec_tw", "p2l_hs", "p2l_htv0", "p2l_htv1", "test_dir", "kfull_ry", "dy_pend", "fused", "statuses", "sec_L", "sec_D", "sec_sigma")
COLUMN_LOCAL = ("gx", "step_n", "plh", "mtv_T", "kfull_elem")
SUMMED = ("Caug", "SSt", "vec_dot", "vec_one", "vec_logbar", "mv")
EXTREMAL = {"vec_inf": np.max, "vec_min": np.min, "vec_ftb": np.min}


def _kkt_cases(world, num_sms):
    """(name, (kind, n, m, m_ineq, l, condense mode, seed)); every n is odd, so the split is uneven at P = 2 and 4"""
    wide = world * (8192 * num_sms + 1) + 1            # every rank past the grid clamp of hb_grid
    return [("uneven_fp64", ("kkt", 40001, 70, 35, 6, 0, 77)),
            ("int8_slices_m300", ("kkt", 9001, 300, 150, 1, 8, 5)),
            ("crt_no_ineq_l33", ("kkt", 20001, 70, 0, 33, 100, 9)),
            ("single_row_l0", ("kkt", 5003, 1, 0, 0, 0, 3)),
            ("unconstrained", ("kkt", 3001, 0, 0, 6, 0, 11)),
            ("past_grid_clamp", ("kkt", wide, 4, 2, 2, 0, 13))]


SECANT_CASES = [("secant_lmax3", ("secant", 1001, 4, 3, 3, 0, 31)), ("secant_lmax6", ("secant", 2003, 5, 2, 6, 0, 37))]


@functools.lru_cache(maxsize=2)
def _problem(case):
    _, n, m, mi, l, _, seed = case
    return synth.make_qn_problem(n, m, l, m_ineq=mi, seed=seed)


@functools.lru_cache(maxsize=2)
def _iterate(case, world):
    """iterate, data, a direction, and trial slacks that collapse below eps*min(1, mu) only on rank 0's x columns (and on a few d lanes)"""
    P = _problem(case)
    itr, dat = synth.make_iterate(P)
    pat = dict(ixl=P.ixl, ixu=P.ixu, idl=P.idl, idu=P.idu)
    rng = np.random.default_rng(5)
    direction = {k: rng.standard_normal(np.asarray(v).size) * np.where(np.asarray(v) != 0, 1.0, 0.0) for k, v in itr.items()}
    trial = {k: np.array(v, dtype=np.float64) for k, v in itr.items()}
    e0 = sharding.column_range(P.n, world, 0)[1]
    for s, p in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu")):
        trial[s] = np.where(pat[p] == 1.0, np.abs(trial[s]) + 1e-3, 0.0)
        hit = (rng.random(trial[s].size) < 0.2) & (pat[p] == 1.0)
        if s in N_BLOCKS:
            hit[e0:] = False
        trial[s] = np.where(hit, rng.choice([0.0, -1e-9, 1e-20, 3e-17], size=trial[s].size), trial[s])
    return itr, dat, direction, trial, pat


def _run_kkt(ctx, case, world, rank, single):
    """One rank's outputs of every sharded entry point (single: a one-rank handle on the same columns, the reference of the sharded run)"""
    from hiop_b200.engine import KKTLinSysLowRank
    _, n, m, mi, l, mode, _ = case
    P = _problem(case)
    me = P.m_eq
    b, e = sharding.column_range(n, world, rank)
    nl = e - b
    D = ctx.to_device
    col = lambda v: np.ascontiguousarray(np.asarray(v)[..., b:e])
    shard = lambda k, v: col(v) if k in N_BLOCKS else np.ascontiguousarray(v)
    get = lambda t: t.cpu().numpy()
    r = {}
    k = KKTLinSysLowRank(ctx, nl, me, mi, max(l, 1))
    k.set_condense_mode(mode)
    J = D(col(P.J))
    T = {nm: D(col(getattr(P, nm))) for nm in ("ixl", "ixu", "zl", "sxl", "zu", "sxu")}
    T.update({nm: D(getattr(P, nm)) for nm in ("idl", "idu", "vl", "sdl", "vu", "sdu")})
    St, Yt = D(col(P.St)), D(col(P.Yt))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(J[:me], J[me:])
    k.set_secant(P.sigma, St if l else None, Yt if l else None, P.L, P.D)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    k.condense()
    dx, dyc, dyd = ctx.zeros(nl), ctx.zeros(me), ctx.zeros(mi)
    assert k.solveCompressed(D(col(P.rx)), D(P.ryc), D(P.ryd), dx, dyc, dyd)
    ctx.sync()
    ds = k.debug_state(l)
    r["Caug"] = np.triu(ds["Caug"])                    # the all-reduce carries the packed upper triangle
    r["SSt"] = ds["SSt"]
    r["N"], r["Z"], r["V"], r["p2l"] = k.N(), ds["Z"], ds["V_built"], ds["p2l"]
    r["dx"], r["dy"] = get(dx), np.concatenate([get(dyc), get(dyd)])
    # device BiCGStab refinement over the compound vectors
    res = {rk: D(shard(dk, P.res[rk])) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    dirs = {dk: ctx.zeros(res[rk].numel()) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    ok, info = k.compute_directions_w_IR(res, dirs, mu=1e-2, maxit=8)
    assert ok
    ctx.sync()
    r["ir_info"] = np.array(info, dtype=np.float64)
    r["ir_n"] = {dk: get(dirs[dk]) for dk in ko.DIR_NAMES if dk in N_BLOCKS}
    r["ir_m"] = np.concatenate([get(dirs[dk]) for dk in ko.DIR_NAMES if dk not in N_BLOCKS])
    # residual norms, fraction to the boundary, log barrier, step, dual clamp, small slacks
    itr, dat, direction, trial, pat = _iterate(case, world)
    it_d = {dk: D(shard(dk, v)) for dk, v in itr.items()}
    dir_d = {dk: D(shard(dk, v)) for dk, v in direction.items()}
    xl, xu = D(col(dat["xl"])), D(col(dat["xu"]))
    res2 = {rk: ctx.zeros(it_d[dk].numel()) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    nm = k.residual_update(it_d, D(dat["c"]), D(dat["d"]), D(col(dat["grad"])), 0.1, 1e-5, xl, xu, D(dat["dl"]), D(dat["du"]), D(dat["crhs"]),
                           res2)
    r["norms"] = np.array([nm[kk] for kk in ko.NORM_NAMES])
    ap, ad = k.fraction_to_bdry(it_d, dir_d, 0.995)
    r["ftb"] = np.array([ap, ad])
    gx, gd = ctx.zeros(nl), ctx.zeros(mi)
    r["flog"] = np.array([k.logbar(it_d, 3.25, 0.1, 1e-5, D(col(dat["grad"])), gx, gd)])
    r["gx"], r["gd"] = get(gx), get(gd)
    out_d = {dk: ctx.zeros(v.numel()) for dk, v in it_d.items()}
    k.take_step(it_d, dir_d, 0.75, 0.5, out_d)            # fixed step lengths: the one-rank shard runs find other local alphas
    ctx.sync()
    r["step_n"] = np.concatenate([get(out_d[dk]) for dk in ko.DIR_NAMES if dk in N_BLOCKS])
    r["step_m"] = np.concatenate([get(out_d[dk]) for dk in ko.DIR_NAMES if dk not in N_BLOCKS])
    k.adjust_duals_plh(out_d, 0.1, 10.0)
    ctx.sync()
    r["plh"] = np.concatenate([get(out_d[dk]) for dk in ("zl", "zu", "vl", "vu")])
    tr_d = {dk: D(shard(dk, v)) for dk, v in trial.items()}
    r["nadj"] = np.array([k.adjust_small_slacks(tr_d, it_d, 0.1, xl, xu, D(dat["dl"]), D(dat["du"]))])
    ctx.sync()
    r["slack"] = {s: get(tr_d[s]) for s in ("sxl", "sxu", "sdl", "sdu")}
    # public vector and matrix helpers on the shards
    x, g = it_d["x"], D(col(dat["grad"]))
    r["vec_dot"], r["vec_one"] = np.array([ctx.vec_dot(x, g)]), np.array([ctx.vec_onenorm(x)])
    r["vec_tw"], r["vec_inf"] = np.array([ctx.vec_twonorm(x)]), np.array([ctx.vec_infnorm(x)])
    r["vec_min"] = np.array([ctx.vec_min_w_pattern(it_d["sxl"], T["ixl"])])
    r["vec_logbar"] = np.array([ctx.vec_log_barrier(it_d["sxl"], T["ixl"])])
    r["vec_ftb"] = np.array([ctx.vec_fraction_to_bdry(it_d["sxl"], dir_d["sxl"], 0.995, T["ixl"])])
    if m:
        y = D(np.linspace(-1.0, 1.0, m))
        ctx.mat_times_vec(J, 0.5 if (rank == 0 or not single) else 0.0, y, 1.0, x)     # beta is applied on rank 0 only
        yt = D(col(np.linspace(2.0, -1.0, n)))
        ctx.mat_trans_times_vec(J, 0.5, yt, -1.0, D(np.linspace(-1.0, 3.0, m)))
        ctx.sync()
        r["mv"], r["mtv_T"] = get(y), get(yt)
    # the Hessian alone: (B + Dx)^-1 r, and y = beta y + 0.75 (B + Dx) x for beta in {0, 1}
    xs_ = D(col(P.rx))
    hs = ctx.zeros(nl)
    k.hess_solve(xs_, hs)
    ctx.sync()
    r["hess_solve"], r["p2l_hs"] = get(hs), k.debug_state(l)["p2l"]
    for beta in (0.0, 1.0):
        yv = D(col(np.linspace(-2.0, 2.0, n)))
        k.hess_times_vec(beta, yv, 0.75, D(col(dat["grad"])), True)
        ctx.sync()
        r[f"hess_times_vec{beta:g}"], r[f"p2l_htv{beta:g}"] = get(yv), k.debug_state(l)["p2l"]
    # test_direction: the replicated d-sums enter once (rank 0 only)
    dwx, dwd = D(np.full(nl, 1e-3)), D(np.full(mi, 2e-3))
    td = (ctypes.c_double * 2)()
    rc = ctx.L.hb_lowrank_test_direction(k.h, ctypes.c_void_p(dir_d["x"].data_ptr()), ctypes.c_void_p(dir_d["d"].data_ptr()),
                                         ctypes.c_void_p(dwx.data_ptr()), ctypes.c_void_p(dwd.data_ptr()), 1e-11, td)
    r["test_dir"] = np.array([rc, td[0], td[1]], dtype=np.float64)
    # y = K x of the full KKT operator: blocks without B or J are elementwise
    X = {dk: D(shard(dk, direction[dk])) for dk in ko.DIR_NAMES}
    Y = {rk: ctx.zeros(X[dk].numel()) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    k.kkt_full_times_vec(X, Y)
    ctx.sync()
    r["kfull_elem"] = np.concatenate([get(Y[rk]) for rk in ko.RES_NAMES if rk not in ("rx", "ryc", "ryd")])
    r["kfull_rx"], r["kfull_ry"] = get(Y["rx"]), np.concatenate([get(Y["ryc"]), get(Y["ryd"])])
    # a condensation left pending by update(): solveCompressed runs it with rx fused, and the row dots tdot ride in C_aug's all-reduce
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    dx, dyc, dyd = ctx.zeros(nl), ctx.zeros(me), ctx.zeros(mi)
    assert k.solveCompressed(D(col(P.rx)), D(P.ryc), D(P.ryd), dx, dyc, dyd)
    k.check()
    ctx.sync()
    ds = k.debug_state(l)
    r["dx_pend"], r["dy_pend"] = get(dx), np.concatenate([get(dyc), get(dyd)])
    r["fused"], r["tdot"] = np.array([float(ds["info"][3])]), ds["tdot"]
    if m and mode == 0:
        # the same system from host memory: kkt_system_host (J staged whole), then J registered from pinned memory in column panels
        itn = dict(zl=col(P.zl), sxl=col(P.sxl), zu=col(P.zu), sxu=col(P.sxu), vl=P.vl, sdl=P.sdl, vu=P.vu, sdu=P.sdu)
        hx, hyc, hyd = np.zeros(nl), np.zeros(me), np.zeros(mi)
        k.kkt_system_host(col(P.Jc), col(P.Jd), itn, col(P.rx), np.ascontiguousarray(P.ryc), np.ascontiguousarray(P.ryd), hx, hyc, hyd)
        r["host_sys"] = np.concatenate([hx, hyc, hyd])
        Jc_p, Jd_p = torch.from_numpy(col(P.Jc)).pin_memory(), torch.from_numpy(col(P.Jd)).pin_memory()
        k.set_jacobian_host(Jc_p, Jd_p, 1024)
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
        dx, dyc, dyd = ctx.zeros(nl), ctx.zeros(me), ctx.zeros(mi)
        assert k.solveCompressed(D(col(P.rx)), D(P.ryc), D(P.ryd), dx, dyc, dyd)
        k.check()
        ctx.sync()
        r["host_panels"] = np.concatenate([get(dx), get(dyc), get(dyd)])
        k.set_jacobian(J[:me], J[me:])
    # least-squares multipliers, then the same call on a Jacobian whose equality row 0 is zero in every shard: J J^T + I is singular and
    # yc, yd must keep what they held
    yc, yd = ctx.zeros(me), ctx.zeros(mi)
    assert k.lsq_duals(g, T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    r["lsq"] = np.concatenate([get(yc), get(yd)])
    if me and mode == 0:
        Jb_host = col(P.J)
        Jb_host[0] = 0.0
        Jb = D(Jb_host)
        k.set_jacobian(Jb[:me], Jb[me:])
        yc, yd = D(np.full(me, SENTINEL)), D(np.full(mi, SENTINEL))
        okb = k.lsq_duals(g, T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
        ctx.sync()
        r["lsq_bad"] = np.concatenate([[float(okb)], get(yc), get(yd)])
        # the same zero row makes the condensed N singular: every rank must report the breakdown
        from hiop_b200._lib import EngineError
        k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
        try:
            k.condense()
            r["cond_bad"] = np.array([0.0])
        except EngineError:
            r["cond_bad"] = np.array([1.0])
    k.close()
    return r


def _run_secant(ctx, case, world, rank, single):
    """hiopHessianLowRank::update over synth.make_secant_sequence: first call, appends, shifts past l_max and both skip rules"""
    from hiop_b200.engine import KKTLinSysLowRank
    _, n, me, mi, lmax, _, seed = case
    b, e = sharding.column_range(n, world, rank)
    D = ctx.to_device
    seq = synth.make_secant_sequence(n, me, mi, steps=9, seed=seed)
    k = KKTLinSysLowRank(ctx, e - b, me, mi, lmax)
    k.set_patterns(D(np.ones(e - b)), D(np.zeros(e - b)), D(np.ones(mi)), D(np.zeros(mi)))
    k.secant_reset(1.0, 1)
    statuses = []
    for it in seq:
        J = D(np.ascontiguousarray(np.vstack([it["Jc"], it["Jd"]])[:, b:e]))
        k.set_jacobian(J[:me], J[me:])
        statuses.append(k.secant_update(D(it["x"][b:e]), D(it["grad_f"][b:e]), D(it["yc"]), D(it["yd"])))
    l, sigma, St, Yt, L, Dg = k.secant_state()
    k.close()
    return dict(statuses=np.array(statuses, dtype=np.float64), sec_L=L, sec_D=Dg, sec_sigma=np.array([sigma]), St=St, Yt=Yt)


def _run_case(ctx, case, world, rank, single):
    return (_run_kkt if case[0] == "kkt" else _run_secant)(ctx, case, world, rank, single)


def _worker(rank, world, uid, out, cases):
    from hiop_b200.engine import Context
    torch.cuda.set_device(rank)
    ctx = Context(rank)
    try:
        ctx.init_comm(world, rank, uid)
        for name, case in cases:
            out[f"{name}/{rank}"] = _run_case(ctx, case, world, rank, single=False)
    finally:
        ctx.close()


def _singles(cases, world):
    """the one-GPU engine on each rank's columns: {name: [shard 0's outputs, ...]}"""
    from hiop_b200.engine import Context
    ctx = Context(0)
    try:
        return {name: [_run_case(ctx, case, world, r, single=True) for r in range(world)] for name, case in cases}
    finally:
        ctx.close()


WORLDS = [1, 2, 4]
_CASES1 = _kkt_cases(1, 1)                               # names and shapes other than the widest n, which depends on P and the SM count
KKT_NAMES = [name for name, _ in _CASES1]
BREAKDOWN_NAMES = [name for name, c in _CASES1 if c[2] > c[3] and c[5] == 0]     # an equality row to zero, FP64 condensation
HOST_NAMES = [name for name, c in _CASES1 if c[2] > 0 and c[5] == 0]
FUSED_NAMES = [name for name, c in _CASES1 if c[5] != 0]                        # the int8 modes fuse the row dots into the condensation
SECANT_NAMES = [name for name, _ in SECANT_CASES]
_RUNS = {}


def _results(world):
    """(cases, sharded outputs, one-GPU shard outputs) of world P, computed once per session"""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    if world not in _RUNS:
        cases = _kkt_cases(world, torch.cuda.get_device_properties(0).multi_processor_count) + SECANT_CASES
        try:
            t0 = time.monotonic()
            out = run_ranks(_worker, world, (cases,), comm="nccl")
            S = {name: [out[f"{name}/{r}"] for r in range(world)] for name, _ in cases}
            t1 = time.monotonic()
            G = _singles(cases, world)
            print(f"\nP = {world}: sharded run {t1 - t0:.1f} s, one-GPU shard runs {time.monotonic() - t1:.1f} s")
            _RUNS[world] = (dict(cases), S, G)
        except Exception as exc:
            _RUNS[world] = exc
            raise
    got = _RUNS[world]
    if isinstance(got, Exception):
        pytest.fail(f"the P = {world} run failed: {got!r}")
    return got


def _within(label, err, tol):
    """err <= tol elementwise; prints the largest err / tol"""
    err, tol = np.atleast_1d(np.asarray(err, dtype=np.float64)), np.atleast_1d(np.asarray(tol, dtype=np.float64))
    ratio = float((err / np.where(tol > 0, tol, 1.0)).max(initial=0.0))
    print(f"  {label}: {ratio:.2e} of its bound")
    assert (err <= tol).all(), f"{label}: error {err.max(initial=0.0):.3e} over its bound"


def _rel(label, got, want, rtol):
    _within(label, np.abs(np.asarray(got) - want).max(initial=0.0), rtol * max(1.0, np.abs(want).max(initial=0.0)))


def _summed(name, key, S, G, world):
    """all-reduced S[.][key] against the one-GPU partials G[r][key]: replicated, fl(G0 + G1) at P <= 2, gamma(P - 1) sum |G_r| beyond"""
    for r in range(1, world):
        np.testing.assert_array_equal(S[r][key], S[0][key], err_msg=f"{name}: summed {key} differs on rank {r}")
    parts = [G[r][key] for r in range(world)]
    if world <= 2:
        np.testing.assert_array_equal(S[0][key], parts[0] if world == 1 else parts[0] + parts[1], err_msg=f"{name}: {key} != fl(G0 + G1)")
    else:
        _within(f"{name}: {key} all-reduce", np.abs(S[0][key] - np.sum(parts, axis=0)), bounds.gamma(world - 1) * np.sum(np.abs(parts), axis=0))


def _oracle_state(P):
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    return Dx, Dd, ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)


def _independent_residual(P, dx, dyc, dyd):
    """relative residual of the compressed 3-block KKT system with J and the compact BFGS form of B applied here, outside the engine"""
    Dx = P.zl / P.sxl + np.where(P.ixu == 1.0, P.zu / np.where(P.ixu == 1.0, P.sxu, 1.0), 0.0)
    Dd = P.vl / P.sdl + np.where(P.idu == 1.0, P.vu / np.where(P.idu == 1.0, P.sdu, 1.0), 0.0)
    s, l = P.sigma, P.St.shape[0]
    Bdx = s * dx
    if l:
        M = np.block([[s * (P.St @ P.St.T), P.L], [P.L.T, -np.diag(P.D)]])
        p = np.linalg.solve(M, np.concatenate([s * (P.St @ dx), P.Yt @ dx]))
        Bdx = Bdx - (s * (P.St.T @ p[:l]) + P.Yt.T @ p[l:])
    r1 = Bdx + Dx * dx + P.J.T @ np.concatenate([dyc, dyd]) - P.rx
    Jdx = P.J @ dx
    r2, r3 = Jdx[:P.m_eq] - P.ryc, Jdx[P.m_eq:] - dyd / Dd - P.ryd
    num = max(np.abs(r1).max(), np.abs(r2).max(initial=0.0), np.abs(r3).max(initial=0.0))
    return num / max(np.abs(P.rx).max(), np.abs(P.ryc).max(initial=0.0), np.abs(P.ryd).max(initial=0.0))


@pytest.mark.parametrize("name", KKT_NAMES + SECANT_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_outputs_by_kind(world, name):
    """replicated outputs bit-identical on every rank, column-local ones equal to the one-GPU run on the rank's columns, summed ones
    the shards' partials plus the all-reduce, extremal ones the min / max of the partials"""
    _, S, G = _results(world)
    S, G = S[name], G[name]
    for key in REPLICATED:
        if key in S[0]:
            for r in range(1, world):
                np.testing.assert_array_equal(S[r][key], S[0][key], err_msg=f"{name}: {key} differs on rank {r}")
    for key in COLUMN_LOCAL:
        if key in S[0]:
            for r in range(world):
                np.testing.assert_array_equal(S[r][key], G[r][key], err_msg=f"{name}: {key} of rank {r} != the one-GPU run on its columns")
    for key in SUMMED:
        if key in S[0]:
            _summed(name, key, S, G, world)
    for key, fold in EXTREMAL.items():
        if key in S[0]:
            for r in range(world):
                assert S[r][key][0] == fold([G[q][key][0] for q in range(world)]), f"{name}: {key} on rank {r}"


@pytest.mark.parametrize("name", KKT_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_kkt_path_against_oracle(world, name):
    cases, S, _ = _results(world)
    case, S = cases[name], S[name]
    mode, m, l = case[5], case[2], case[4]
    P = _problem(case)
    Dx, Dd, st = _oracle_state(P)
    cat = lambda key: np.concatenate([s[key] for s in S])
    dxo, dyco, dydo, No = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    _rel(f"{name}: dx", cat("dx"), dxo, 1e-8)
    _rel(f"{name}: dy", S[0]["dy"], np.concatenate([dyco, dydo]), 1e-8)
    _rel(f"{name}: dx (pending condensation)", cat("dx_pend"), dxo, 1e-8)
    if m:
        _rel(f"{name}: N", S[0]["N"], No, 1e-8 if mode else 1e-12)
    me = P.m_eq
    _within(f"{name}: independent-operator KKT residual", _independent_residual(P, cat("dx"), S[0]["dy"][:me], S[0]["dy"][me:]), 1e-8)
    it = dict(sxl=P.sxl, sxu=P.sxu, zl=P.zl, zu=P.zu, sdl=P.sdl, sdu=P.sdu, vl=P.vl, vu=P.vu)
    pat = dict(ixl=P.ixl, ixu=P.ixu, idl=P.idl, idu=P.idu)
    do, info_o = ko.compute_directions_w_ir(st, it, pat, P.res, 1e-2, 8, Dx=Dx)
    assert S[0]["ir_info"][0] == info_o[0] and S[0]["ir_info"][1] == info_o[1]
    for dk in ko.DIR_NAMES:
        if dk in N_BLOCKS:
            _rel(f"{name}: IR {dk}", np.concatenate([s["ir_n"][dk] for s in S]), do[dk], 1e-8)
    _rel(f"{name}: IR m-blocks", S[0]["ir_m"], np.concatenate([do[dk] for dk in ko.DIR_NAMES if dk not in N_BLOCKS]), 1e-8)
    itr, dat, direction, trial, pat_i = _iterate(case, world)
    _, no = ko.residual_update(itr, dat["c"], dat["d"], dat["grad"], P.Jc, P.Jd, 0.1, 1e-5, pat_i, dat["xl"], dat["xu"], dat["dl"], dat["du"],
                               dat["crhs"])
    for q, kk in enumerate(ko.NORM_NAMES):
        _rel(f"{name}: {kk}", S[0]["norms"][q], no[kk], 1e-12)
    assert tuple(S[0]["ftb"]) == ko.iterate_fraction_to_bdry(itr, direction, 0.995, pat_i)
    flo, gxo, gdo = ko.logbar_update(itr, 3.25, 0.1, 1e-5, dat["grad"], pat_i)
    _rel(f"{name}: f_logbar", S[0]["flog"][0], flo, 1e-12)
    np.testing.assert_array_equal(cat("gx"), gxo)
    np.testing.assert_array_equal(S[0]["gd"], gdo)
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, dat["grad"], P.zl, P.zu, P.vl, P.vu)
    _rel(f"{name}: LSQ duals", S[0]["lsq"], np.concatenate([yco, ydo]), 1e-8 if mode else 1e-9)
    # the Hessian alone, and test_direction with the regularisations
    _rel(f"{name}: hess_solve", cat("hess_solve"), ko.hess_solve(st, P.rx), 1e-9)
    for beta in (0.0, 1.0):
        want = ko.hess_times_vec(P.St, P.Yt, P.sigma, Dx, beta, np.linspace(-2.0, 2.0, P.n), 0.75, dat["grad"], True)
        _rel(f"{name}: hess_times_vec beta {beta:g}", cat(f"hess_times_vec{beta:g}"), want, 1e-9)
    dxv, ddv = direction["x"], direction["d"]
    Bdx = ko.hess_times_vec(P.St, P.Yt, P.sigma, Dx, 0.0, np.zeros(P.n), 1.0, dxv, False)
    dWd = Bdx @ dxv + ((Dx + 1e-3) * dxv) @ dxv + ((Dd + 2e-3) * ddv) @ ddv
    xs = dxv @ dxv + ddv @ ddv
    scale = abs(Bdx @ dxv) + ((Dx + 1e-3) * dxv) @ dxv + ((Dd + 2e-3) * ddv) @ ddv
    rc, got_dwd, got_xs = S[0]["test_dir"]
    assert rc == (0 if dWd < xs * 1e-11 else 1)
    _within(f"{name}: test_direction dWd", abs(got_dwd - dWd), 1e-9 * scale)
    _within(f"{name}: test_direction |dx|^2 + |dd|^2 (d part once)", abs(got_xs - xs), 1e-12 * xs)
    yk = ko.kkt_full_times_vec(st, it, pat, direction, Dx)
    _rel(f"{name}: K x, rx block", cat("kfull_rx"), yk["rx"], 1e-11)
    _rel(f"{name}: K x, ryc/ryd blocks", S[0]["kfull_ry"], np.concatenate([yk["ryc"], yk["ryd"]]), 1e-11)
    elem = [rk for rk in ko.RES_NAMES if rk not in ("rx", "ryc", "ryd")]
    nb = {rk for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES) if dk in N_BLOCKS}
    for r, s in enumerate(S):
        b, e = sharding.column_range(P.n, world, r)
        want = np.concatenate([yk[rk][b:e] if rk in nb else yk[rk] for rk in elem])
        np.testing.assert_array_equal(s["kfull_elem"], want, err_msg=f"{name}: elementwise blocks of K x on rank {r}")


@pytest.mark.parametrize("name", KKT_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_adjusted_slack_count_is_global_on_every_rank(world, name):
    """x-slacks collapse on rank 0's columns only; every rank must return the x-side counts summed over the ranks plus the d-side count once"""
    cases, S, _ = _results(world)
    case, S = cases[name], S[name]
    itr, dat, direction, trial, pat = _iterate(case, world)
    want = 0
    for s, p, bnd, dual in (("sxl", "ixl", "xl", "zl"), ("sxu", "ixu", "xu", "zu"), ("sdl", "idl", "dl", "vl"), ("sdu", "idu", "du", "vu")):
        new, cnt = ko.adjust_small_slack(trial[s], dat[bnd], itr[dual], pat[p], 0.1)
        want += cnt
        got = np.concatenate([sr["slack"][s] for sr in S]) if s in N_BLOCKS else S[0]["slack"][s]
        np.testing.assert_array_equal(got, new, err_msg=f"{name}: {s}")
    assert want > 0
    assert [int(sr["nadj"][0]) for sr in S] == [want] * world, f"{name}: adjusted-slack count per rank, want {want} on every rank"


@pytest.mark.parametrize("name", BREAKDOWN_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_failed_lsq_leaves_the_duals_on_every_rank(world, name):
    """equality row 0 zero in every shard: J J^T + I is singular, lsq_duals fails and yc, yd keep what they held"""
    _, S, _ = _results(world)
    for r, sr in enumerate(S[name]):
        assert sr["lsq_bad"][0] == 0.0, f"{name}: lsq_duals reported success on a singular J J^T on rank {r}"
        assert (sr["lsq_bad"][1:] == SENTINEL).all(), f"{name}: a failed lsq_duals overwrote yc/yd on rank {r}"


@pytest.mark.parametrize("name", BREAKDOWN_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_condensation_breakdown_is_reported_on_every_rank(world, name):
    _, S, _ = _results(world)
    assert [sr["cond_bad"][0] for sr in S[name]] == [1.0] * world, f"{name}: N not SPD must fail the condensation on every rank"


@pytest.mark.parametrize("name", FUSED_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_fused_row_dots_ride_the_condensation_all_reduce(world, name):
    """solveCompressed on a pending int8 condensation: tdot = [J; S; Y] (DhInv .* rx) is summed with C_aug's packed triangle"""
    _, S, G = _results(world)
    S, G = S[name], G[name]
    assert [s["fused"][0] for s in S] == [1.0] * world and [g["fused"][0] for g in G] == [1.0] * world, f"{name}: fused path not taken"
    _summed(name, "tdot", S, G, world)


@pytest.mark.parametrize("name", HOST_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_host_jacobian_gives_the_device_bits(world, name):
    """kkt_system_host (J staged whole) solves the same system as the device J bit for bit; a pinned J streamed in 1024-column panels
    condenses panel by panel, so its solution is held to the device one within 1e-12 (as tests/test_gpu_host_jacobian.py does)"""
    _, S, _ = _results(world)
    for r, s in enumerate(S[name]):
        want = np.concatenate([s["dx_pend"], s["dy_pend"]])
        np.testing.assert_array_equal(s["host_sys"], want, err_msg=f"{name}: kkt_system_host on rank {r}")
        _within(f"{name}: set_jacobian_host with panels on rank {r}", np.abs(s["host_panels"] - want).max(), 1e-12 * np.abs(want).max())


@pytest.mark.parametrize("name", SECANT_NAMES)
@pytest.mark.parametrize("world", WORLDS)
def test_secant_memory_against_oracle(world, name):
    cases, S, _ = _results(world)
    _, n, me, mi, lmax, _, seed = cases[name]
    S = S[name]
    seq = synth.make_secant_sequence(n, me, mi, steps=9, seed=seed)
    mem = ko.SecantMemory(n, lmax, 1.0, 1)
    want = [mem.update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"]) for it in seq]
    assert {2, 3} <= set(want) and 1 in want
    for r in range(world):
        assert list(S[r]["statuses"].astype(int)) == want, f"{name}: secant statuses on rank {r}"
    np.testing.assert_array_equal(np.concatenate([s["St"] for s in S], axis=1), mem.St)   # one subtraction per entry
    _rel(f"{name}: Y_t", np.concatenate([s["Yt"] for s in S], axis=1), mem.Yt, 1e-13)
    _within(f"{name}: L", np.abs(np.tril(S[0]["sec_L"], -1) - np.tril(mem.L, -1)).max(initial=0.0), 1e-12)
    _within(f"{name}: D", np.abs(S[0]["sec_D"] - mem.D).max(initial=0.0), 1e-12)
    _rel(f"{name}: sigma", S[0]["sec_sigma"][0], mem.sigma, 1e-12)
