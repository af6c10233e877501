"""A/B check of two builds of libhiopb200.so on every pass over the quasi-Newton Jacobian: device J, host J in panels, and the staged
upload of hb_lowrank_kkt_system_host. Each run loads the library named by HIOPB200_SO (the tree's build if unset), runs the same
seeded cases and writes their outputs and hb_launch_count deltas to one .npz; `compare` then requires bit-identical arrays and equal
launch counts.

    HIOPB200_SO=/path/to/a/libhiopb200.so python tools/jacobian_layout_ab.py run a.npz
    python tools/jacobian_layout_ab.py run b.npz
    python tools/jacobian_layout_ab.py compare a.npz b.npz
"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


def _tensors(ctx, P):
    D = ctx.to_device
    T = {kk: D(getattr(P, kk)) for kk in ("ixl", "ixu", "idl", "idu", "St", "Yt") + ITERATE}
    T["J"] = D(P.J)
    return T


def _handle(ctx, P, T, host_panels=None, Jh=None):
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, max(P.l, 1))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    if host_panels is None:
        k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    else:
        k.set_jacobian_host(Jh[0], Jh[1], host_panels)
    k.set_secant(float(P.sigma), T["St"] if P.l else None, T["Yt"] if P.l else None, P.L, P.D)
    return k


def _update(k, T):
    k.update(*(T[kk] for kk in ITERATE))


def _solve(ctx, k, P):
    D = ctx.to_device
    dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(D(P.rx), D(P.ryc), D(P.ryd), dx, dyc, dyd)
    k.check()
    ctx.sync()
    return {"dx": dx.cpu().numpy(), "dyc": dyc.cpu().numpy(), "dyd": dyd.cpu().numpy()}


def _gemv_consumers(ctx, k, P, T):
    """residual_update, kkt_full_times_vec, compute_directions_w_ir, lsq_duals"""
    from hiop_b200 import synth
    from oracle import kkt_oracle as ko
    D = ctx.to_device
    out = {}
    itr, dat = synth.make_iterate(P)
    it_d = {kk: D(np.ascontiguousarray(v)) for kk, v in itr.items()}
    sizes = {kk: v.size for kk, v in itr.items()}
    args = [D(dat[kk]) for kk in ("c", "d", "grad")] + [0.1, 1e-5] + [D(dat[kk]) for kk in ("xl", "xu", "dl", "du", "crhs")]
    res = {rk: ctx.zeros(sizes[dk]) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    nrm = k.residual_update(it_d, *args, res)
    ctx.sync()
    out.update({"resid_" + rk: v.cpu().numpy() for rk, v in res.items()})
    out["resid_norms"] = np.array(list(nrm.values()))
    rng = np.random.default_rng(5)
    X = {kk: D(rng.standard_normal(sizes[kk])) for kk in ko.DIR_NAMES}
    Y = {rk: ctx.zeros(sizes[dk]) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    k.kkt_full_times_vec(X, Y)
    ctx.sync()
    out.update({"kx_" + rk: v.cpu().numpy() for rk, v in Y.items()})
    _update(k, T)
    R = {kk: D(P.res[kk]) for kk in ko.RES_NAMES}
    dirs = {kk: ctx.zeros(sizes[kk]) for kk in ko.DIR_NAMES}
    ok, info = k.compute_directions_w_IR(R, dirs, 1e-2, 8)
    assert ok
    ctx.sync()
    out.update({"ir_" + kk: v.cpu().numpy() for kk, v in dirs.items()})
    out["ir_info"] = np.array(info, dtype=np.float64)
    return out


def _lsq(ctx, k, P, T):
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(ctx.to_device(np.ones(P.n)), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    return {"yc": yc.cpu().numpy(), "yd": yd.cpu().numpy()}


def cases(ctx):
    """yields (name, function returning a dict of arrays)"""
    import torch
    from hiop_b200 import synth

    def device_solve(n, m, l):
        def f():
            P = synth.make_qn_problem(n, m, l, seed=11)
            T = _tensors(ctx, P)
            k = _handle(ctx, P, T)
            out = {}
            for rep in range(2):  # the second call runs on the cached row-pointer table
                _update(k, T)
                out.update({f"{kk}{rep}": v for kk, v in _solve(ctx, k, P).items()})
            out["N"] = k.N()
            k.close()
            return out
        return f

    def condense(mode):
        def f():
            P = synth.make_qn_problem(36000, 80, 4, seed=9)
            T = _tensors(ctx, P)
            k = _handle(ctx, P, T)
            k.set_condense_mode(mode)
            _update(k, T)
            k.condense()
            out = {"N": k.N(), "used": np.array([k.condense_mode_used()])}
            out.update({"lsq_" + kk: v for kk, v in _lsq(ctx, k, P, T).items()})
            _update(k, T)
            out.update(_solve(ctx, k, P))
            k.close()
            return out
        return f

    big = {}

    def big_problem():
        if not big:
            P = synth.make_qn_problem(200001, 300, 6, seed=97)
            big["P"], big["T"] = P, _tensors(ctx, P)
            big["Jh"] = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in (P.Jc, P.Jd)]
        return big["P"], big["T"], big["Jh"]

    def jac_passes(panels):
        def f():
            P, T, Jh = big_problem()
            k = _handle(ctx, P, T, panels, Jh)
            _update(k, T)
            out = _solve(ctx, k, P)
            _update(k, T)
            k.condense()
            out["N"] = k.N()
            out.update(_gemv_consumers(ctx, k, P, T))
            out.update({"lsq_" + kk: v for kk, v in _lsq(ctx, k, P, T).items()})
            k.close()
            return out
        return f

    def kkt_host(n, m, l):
        def f():
            P = synth.make_qn_problem(n, m, l, seed=6)
            T = _tensors(ctx, P)
            k = _handle(ctx, P, T)
            it = {kk: np.ascontiguousarray(getattr(P, kk)) for kk in ITERATE}
            out = {}
            for rep in range(3):
                hx, hyc, hyd = np.zeros(P.n), np.zeros(P.m_eq), np.zeros(P.m_ineq)
                k.kkt_system_host(np.ascontiguousarray(P.Jc), np.ascontiguousarray(P.Jd), it, P.rx.copy(), P.ryc.copy(), P.ryd.copy(), hx, hyc, hyd)
                out.update({f"dx{rep}": hx, f"dyc{rep}": hyc, f"dyd{rep}": hyd})
            out["N"] = k.N()
            out["used"] = np.array([k.condense_mode_used()])
            # the device J the staged upload leaves behind serves the gemvs
            out.update(_gemv_consumers(ctx, k, P, T))
            k.close()
            return out
        return f

    def secant(constant):
        def f():
            P = synth.make_qn_problem(50001, 40, 4, seed=21)
            T = _tensors(ctx, P)
            k = _handle(ctx, P, T)
            k.secant_reset(1.0, 1)
            D = ctx.to_device
            rng = np.random.default_rng(4)
            out = {}
            for i in range(5):
                if not constant and i:
                    J = D(P.J + 1e-3 * i * rng.standard_normal(P.J.shape))
                    T["J" + str(i)] = J
                    k.set_jacobian(J[:P.m_eq], J[P.m_eq:])
                x, g = D(rng.standard_normal(P.n)), D(rng.standard_normal(P.n))
                yc, yd = D(rng.standard_normal(P.m_eq)), D(rng.standard_normal(P.m_ineq))
                out[f"status{i}"] = np.array([k.secant_update(x, g, yc, yd, jacobian_is_constant=constant)])
                ll, sg, St, Yt, L, Dv = k.secant_state()
                out.update({f"sigma{i}": np.array([sg]), f"St{i}": St, f"Yt{i}": Yt, f"L{i}": L, f"D{i}": Dv})
            k.close()
            return out
        return f

    yield "device_solve_fused", device_solve(20001, 24, 4)       # m + 2l = 32: the fused rhs row is free
    yield "device_solve_unfused", device_solve(20001, 120, 4)    # m + 2l = 128: no padding row, Jx pass
    yield "condense_mode0", condense(0)
    yield "condense_mode8", condense(8)
    yield "device_gemv_consumers", jac_passes(None)
    for name, panels in (("one", 200704), ("two", 100352), ("many", 2048)):
        yield "host_panels_" + name, jac_passes(panels)
    yield "kkt_system_host_small", kkt_host(3000, 24, 4)
    yield "kkt_system_host_chunked", kkt_host(48000, 700, 6)       # 269 MB of J: the staged upload
    yield "secant_constant_J", secant(True)
    yield "secant_changing_J", secant(False)


def run(path):
    from hiop_b200 import _lib
    from hiop_b200.engine import Context
    ctx = Context(0)
    arrays, launches = {}, {}
    for name, f in cases(ctx):
        ctx.sync()
        l0 = ctx.launch_count()
        out = f()
        ctx.sync()
        launches[name] = ctx.launch_count() - l0
        arrays.update({f"{name}::{kk}": np.asarray(v) for kk, v in out.items()})
        print(f"{name}: {len(out)} outputs, {launches[name]} launches", flush=True)
    arrays["__launches__"] = np.array(json.dumps(launches))
    arrays["__library__"] = np.array(_lib.SO_PATH)
    np.savez(path, **arrays)
    ctx.close()


def compare(a_path, b_path):
    a, b = np.load(a_path), np.load(b_path)
    la, lb = json.loads(str(a["__launches__"])), json.loads(str(b["__launches__"]))
    keys = sorted((set(a.files) | set(b.files)) - {"__launches__", "__library__"})
    differ = [kk for kk in keys if kk not in a.files or kk not in b.files or a[kk].shape != b[kk].shape
              or a[kk].tobytes() != b[kk].tobytes()]
    launch_diff = {kk: (la.get(kk), lb.get(kk)) for kk in set(la) | set(lb) if la.get(kk) != lb.get(kk)}
    summary = {"arrays": len(keys), "bit_identical": len(keys) - len(differ), "differ": differ, "launches_a": la,
               "launch_deltas_differ": launch_diff}
    print(json.dumps(summary, indent=1))
    return 0 if not differ and not launch_diff else 1


if __name__ == "__main__":
    if sys.argv[1] == "run":
        run(sys.argv[2])
    else:
        sys.exit(compare(sys.argv[2], sys.argv[3]))
