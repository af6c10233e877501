"""The condensed SPD solve that ends every quasi-Newton step (hb_dense_equilibrate, hb_dense_condensed_factor, hb_dense_condensed_solve)
held to oracle/spd_refine_model.py through hb_debug_condensed_solve, on every row of the condensed dispatch table: the equilibration bit
for bit, the factor to factor_backward_ratio, each stage of the refinement to its bound, every exit of the loop, non-finite residuals,
breakdowns against dpotrf, and the same through the quasi-Newton handle. Each case asserts the plan row it is named after.

Nfact = (1 + EPS) Nref makes the refinement a stationary iteration that divides the residual by ~1 / EPS per correction, so each exit is
placed with a margin of ~1 / EPS."""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.linalg import lapack

from hiop_b200 import synth
from hiop_b200._lib import EngineError, check
from oracle import bounds
from oracle import kkt_oracle as ko
from oracle import spd_refine_model as model
from test_gpu_parity import _as_dict, _setup_kkt

pytestmark = pytest.mark.gpu

# enum order of Factor / Solve in hb_symdense.cu
FACTOR = ("SYTF2", "SYTRF_BLOCKED", "BK_CLUSTER", "PANEL_CHOL", "PANEL_LDL", "COOP_CHOL", "BIG_CHOL", "BIG_LDL")
SOLVE = ("SYTRS", "ONE_CTA", "BIG", "COOP_REFINE", "ONE_CTA_REFINE")
DEV = torch.device("cuda", 0)
EPS = 1e-3
NOCOOP = dict(HB_CHOL_COOP=0)
STAGES_MAX_N = 8192      # above: only the first solve's stage bound (each stage costs two extended-precision products on the host)


@pytest.fixture
def make_ctx(monkeypatch):
    """Context(0) created under the given environment (hb_dense_init reads the knobs once per context)"""
    made = []

    def make(**env):
        from hiop_b200.engine import Context
        for k in ("HB_DENSE_PAIR_MIN", "HB_BK_CLUSTER_MIN", "HB_DENSE_BIG_MIN", "HB_CHOL_COOP"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        c = Context(0)
        made.append(c)
        return c
    yield make
    for c in made:
        c.close()


def _spd(N, seed, spread=2.0):
    """SPD, well conditioned after equilibration, with a diagonal spread over 10^(+-spread) (so s is far from 1)"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randn((N, N // 2 + 1), generator=g, dtype=torch.float64).to(DEV)
    d = torch.rand(N, generator=g, dtype=torch.float64).to(DEV) * 1.5 + 0.5
    sc = 10.0 ** ((torch.rand(N, generator=g, dtype=torch.float64).to(DEV) * 2 - 1) * spread)
    B = G @ G.T / N + torch.diag(d)
    B = 0.5 * (B + B.T)
    return (B * sc.sqrt()[:, None]) * sc.sqrt()[None, :], (torch.randn(N, generator=g, dtype=torch.float64).to(DEV) * sc.sqrt())


def run(ctx, Nfact, Nref, rhs, tol, max_refine, s=False, Aeq=False, F=False):
    """hb_debug_condensed_solve on device tensors; returns plan, x (host), nref, rho, info and the requested read-backs"""
    N = rhs.shape[0]
    torch.cuda.synchronize()
    x = torch.zeros(N, dtype=torch.float64, device=DEV)
    plan = (ctypes.c_int * 4)()
    stats = np.zeros(2)
    info = ctypes.c_int(-7)
    out = dict(s=np.empty(N) if s else None, Aeq=np.empty((N, N)) if Aeq else None, F=np.empty((N, N)) if F else None)
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    check(ctx.L.hb_debug_condensed_solve(ctx.h, N, ctypes.c_void_p(Nfact.data_ptr()), ctypes.c_void_p(Nref.data_ptr()), N,
                                         ctypes.c_void_p(rhs.data_ptr()), ctypes.c_void_p(x.data_ptr()), float(tol), max_refine, plan,
                                         p(out["s"]), p(out["Aeq"]), p(out["F"]), p(stats), ctypes.byref(info)), "hb_debug_condensed_solve")
    out.update(plan=(FACTOR[plan[0]], SOLVE[plan[1]], bool(plan[2]), bool(plan[3])), x=x.cpu().numpy(), nref=int(stats[0]),
               rho=float(stats[1]), info=info.value)
    return out


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


# ---- the rows of the condensed dispatch table ---------------------------------------------------------------------------------------
ROWS = [
    (1, {}, ("PANEL_CHOL", "ONE_CTA_REFINE", False, False)),
    (64, {}, ("PANEL_CHOL", "ONE_CTA_REFINE", False, False)),
    (65, {}, ("COOP_CHOL", "COOP_REFINE", False, False)),
    (1000, {}, ("COOP_CHOL", "COOP_REFINE", False, False)),
    (2048, {}, ("COOP_CHOL", "COOP_REFINE", False, False)),
    (2049, {}, ("PANEL_CHOL", "COOP_REFINE", True, False)),
    (2050, {}, ("BIG_CHOL", "COOP_REFINE", True, False)),
    (6144, {}, ("BIG_CHOL", "COOP_REFINE", True, True)),
    (16384, {}, ("BIG_CHOL", "COOP_REFINE", True, True)),
    (16385, {}, ("PANEL_CHOL", "ONE_CTA_REFINE", True, False)),
    (64, NOCOOP, ("PANEL_CHOL", "ONE_CTA_REFINE", False, False)),
    (65, NOCOOP, ("PANEL_CHOL", "ONE_CTA_REFINE", False, False)),
    (2049, NOCOOP, ("PANEL_CHOL", "ONE_CTA_REFINE", False, False)),
]


def _id(r):
    return f"N{r[0]}" + ("-nocoop" if r[1] else "")


@pytest.mark.parametrize("N,env,expect", ROWS, ids=[_id(r) for r in ROWS])
def test_condensed_row(make_ctx, N, env, expect):
    ctx = make_ctx(**env)
    Nref, rhs = _spd(N, seed=N + len(env))
    Nfact = (1.0 + EPS) * Nref
    # stages: max_refine = k with tol = 0 stops after exactly k corrections
    runs = [run(ctx, Nfact, Nref, rhs, 0.0, k, s=(k == 3), Aeq=(k == 3), F=(k == 3)) for k in range(4)]
    for k, o in enumerate(runs):
        assert o["plan"] == expect, (o["plan"], expect)
        assert o["nref"] == k and o["info"] == 0, (k, o["nref"], o["info"])
    xs = [o["x"] for o in runs]
    rhos = [o["rho"] for o in runs]
    last = runs[3]
    # equilibration, bit for bit
    Nref_h, Nfact_h, rhs_h = Nref.cpu().numpy(), Nfact.cpu().numpy(), rhs.cpu().numpy()
    s_m, Aeq_m = model.equilibrate(Nfact_h)
    assert np.array_equal(_bits(last["s"]), _bits(s_m))
    assert np.array_equal(_bits(np.triu(last["Aeq"])), _bits(Aeq_m))
    # the factor against the equilibrated matrix
    Aeq_full = np.triu(Aeq_m) + np.triu(Aeq_m, 1).T
    R = np.ascontiguousarray(np.tril(last["F"].T))
    del last["F"], last["Aeq"]
    Rt, At = torch.from_numpy(R).to(DEV), torch.from_numpy(Aeq_full).to(DEV)
    th = max(bounds.block_theta(Rt, 16), bounds.block_theta(Rt, 128))
    fr = bounds.factor_backward_ratio(At, Rt, torch.ones(N, dtype=torch.float64, device=DEV), None, th)
    del Rt, At
    torch.cuda.empty_cache()
    # each stage, from the read-back x of the stage before
    n_st = 4 if N <= STAGES_MAX_N else 1
    sr = [model.stage_ratio(Aeq_full, R, th, s_m, Nref_h, rhs_h, xs[k - 1] if k else None, xs[k]) for k in range(n_st)]
    rr = [model.rho_ratio(Nref_h, rhs_h, xs[k], rhos[k]) for k in ((0, 3) if N <= STAGES_MAX_N else (3,))]
    del Aeq_full, R
    # exits
    exits = [(math.inf, 3), (0.0, 0), (0.0, 1), (0.0, 3), (math.sqrt(rhos[0] * rhos[1]), 3), (math.sqrt(rhos[1] * rhos[2]), 3)]
    for k in range(3):
        exits += [(rhos[k], 3), (float(np.nextafter(rhos[k], math.inf)), 3)]
    for tol, mr in exits:
        o = run(ctx, Nfact, Nref, rhs, tol, mr)
        k, rho = model.expected_exit(rhos, tol, mr)
        assert (o["nref"], o["rho"]) == (k, rho), (tol, mr, o["nref"], k)
        assert np.array_equal(_bits(o["x"]), _bits(xs[k])), (tol, mr)
    assert model.expected_exit(rhos, math.sqrt(rhos[0] * rhos[1]), 3)[0] == 1
    assert model.expected_exit(rhos, math.sqrt(rhos[1] * rhos[2]), 3)[0] == 2
    print(f"condensed N={N} {env}: plan {expect}, theta {th:.2f}; factor margin {1 / max(fr, 1e-300):.3g}; stage margins "
          f"{[f'{1 / max(v, 1e-300):.3g}' for v in sr]}; rho margins {[f'{1 / max(v, 1e-300):.3g}' for v in rr]}; "
          f"rho {[f'{v:.3g}' for v in rhos]}")
    assert fr <= 1.0 and max(sr) <= 1.0 and max(rr) <= 1.0
    assert all(rhos[k + 1] < rhos[k] * 10 * EPS for k in range(2))
    torch.cuda.empty_cache()


@pytest.mark.parametrize("spread", [150.0])
def test_equilibration_bits_wide_diagonal(make_ctx, spread):
    ctx = make_ctx()
    N = 1000
    Nref, rhs = _spd(N, seed=3, spread=spread)
    o = run(ctx, Nref, Nref, rhs, 1e-8, 3, s=True, Aeq=True)
    s_m, Aeq_m = model.equilibrate(Nref.cpu().numpy())
    d = np.diag(Nref.cpu().numpy())
    print(f"diagonal from {d.min():.3g} to {d.max():.3g}: {o['nref']} corrections, rho {o['rho']:.3g}")
    assert d.min() < 1e-140 and d.max() > 1e140
    assert np.array_equal(_bits(o["s"]), _bits(s_m)) and np.array_equal(_bits(np.triu(o["Aeq"])), _bits(Aeq_m))


# ---- non-finite residuals ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,env,solve", [(1000, {}, "COOP_REFINE"), (1000, NOCOOP, "ONE_CTA_REFINE"), (64, {}, "ONE_CTA_REFINE")],
                         ids=["coop", "one-cta-nocoop", "one-cta-64"])
@pytest.mark.parametrize("where,value", [(0, math.nan), (-1, math.nan), (None, math.inf)], ids=["nan-first", "nan-last", "inf-mid"])
def test_non_finite_residual(make_ctx, N, env, solve, where, value):
    """0 corrections and a NaN residual norm (a fmax that drops NaN reported a NaN dy as converged)"""
    ctx = make_ctx(**env)
    Nref, rhs = _spd(N, seed=11)
    i = N // 2 if where is None else where % N
    rhs[i] = value
    o = run(ctx, Nref, Nref, rhs, 1e-8, 3)
    print(f"N={N} {solve}: rhs[{i}] = {value}: {o['nref']} corrections, rho {o['rho']}, x finite {np.isfinite(o['x']).sum()} of {N}")
    assert o["plan"][1] == solve
    assert o["nref"] == 0 and math.isnan(o["rho"])


# ---- breakdowns -------------------------------------------------------------------------------------------------------------------------
BREAK_ROWS = [(64, "PANEL_CHOL"), (1000, "COOP_CHOL"), (2049, "PANEL_CHOL"), (2050, "BIG_CHOL"), (6144, "BIG_CHOL")]


@pytest.mark.parametrize("N,factor", BREAK_ROWS, ids=[f"N{r[0]}" for r in BREAK_ROWS])
def test_breakdown_leading_minor(make_ctx, N, factor):
    ctx = make_ctx()
    Nref, rhs = _spd(N, seed=21 + N)
    for col in sorted({c for c in (0, 63, 64, 127, 128, N - 1) if c < N}):
        for kind in ("negative", "indefinite2x2"):
            B = Nref.clone()
            if kind == "negative":
                B[col, col] = -1.0
            else:
                if N < 2:
                    continue
                a, b = (col, col + 1) if col + 1 < N else (col - 1, col)
                for t in (a, b):
                    B[t, :] = 0.0
                    B[:, t] = 0.0
                B[a, a], B[b, b], B[a, b], B[b, a] = 1.0, 1.0, 2.0, 2.0
            o = run(ctx, B, B, rhs, 1e-8, 3)
            lead = min(N, col + 2)
            _, info = lapack.dpotrf(np.ascontiguousarray(B[:lead, :lead].cpu().numpy()), lower=1)
            assert o["plan"][0] == factor
            assert info > 0 and o["info"] == info, (kind, col, o["info"], info)
    torch.cuda.empty_cache()


# ---- through the quasi-Newton handle --------------------------------------------------------------------------------------------------
def test_handle_breakdown_then_recovery_and_rounding_floor(make_ctx):
    """A zero J_d row with v_l < 0 makes Dd_inv < 0: check() reports the leading minor m_eq + i + 1 and the same handle then solves a
    valid iterate. rhs scaled by 1e12 puts the rounding floor above 1e-8: 3 corrections, like the reference's loop"""
    ctx = make_ctx()
    P = synth.make_qn_problem(3000, 40, 4, seed=31)
    p = _as_dict(P)
    i = 5
    bad = dict(p)
    bad["Jd"] = p["Jd"].copy()
    bad["Jd"][i, :] = 0.0
    bad["vl"] = p["vl"].copy()
    bad["vl"][i] = -1e6
    k, T = _setup_kkt(ctx, bad)
    rx, ryc, ryd = ctx.to_device(P.rx), ctx.to_device(P.ryc), ctx.to_device(P.ryd)
    dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
    with pytest.raises(EngineError, match=f"leading minor {P.m_eq + i + 1}\\)"):
        k.check()
    # the same handle, a valid iterate
    T["J"] = ctx.to_device(np.vstack([p["Jc"], p["Jd"]]))
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    vl = ctx.to_device(p["vl"])
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], vl, T["sdl"], T["vu"], T["sdu"])
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    for scale in (1.0, 1e12):
        rx, ryc, ryd = ctx.to_device(P.rx * scale), ctx.to_device(P.ryc * scale), ctx.to_device(P.ryd * scale)
        dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
        assert k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
        k.check()
        ctx.sync()
        nref, resid = k.last_solve_stats()
        dy = np.concatenate([dyc.cpu().numpy(), dyd.cpu().numpy()])
        Nm = k.N()
        rhs = k.debug_state(int(P.l))["rhs"]
        rr = model.rho_ratio(Nm, rhs, dy, resid)
        dxo, dyco, dydo, No = ko.solve_compressed(st, P.rx * scale, P.ryc * scale, P.ryd * scale)
        _, nref_o, resid_o = ko.solve_with_refin(No, rhs)
        err = max(np.abs(dx.cpu().numpy() - dxo).max() / np.abs(dxo).max(), np.abs(dy - np.concatenate([dyco, dydo])).max() / np.abs(dydo).max())
        print(f"handle, rhs x {scale:g}: {nref} corrections (reference {nref_o}), rho {resid:.3g} (reference {resid_o:.3g}), "
              f"rho margin {1 / max(rr, 1e-300):.3g}, rel err vs oracle {err:.2e}")
        assert nref == nref_o == (0 if scale == 1.0 else 3)
        assert rr <= 1.0 and err <= 1e-8
    k.close()
