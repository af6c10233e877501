"""The Chinese-remainder condensation (HB_CONDENSE_INT8_CRT) inside the rest of the quasi-Newton step: a direction with Dx over 16 decades
checked with operators that never see N, the fused rhs row of the row-maximum sweep against its gamma bound, and the
reference's ExM driver with HB_CONDENSE=crt through the C++ adapter."""
import re

import numpy as np
import pytest
import torch

from bench import independent_kkt_residual
from hiop_b200 import synth
from oracle import bounds
from oracle import crt_model as crt
from test_gpu_crt import CRT, DEV, ITERATE, _model, _setup, ctx  # noqa: F401
from test_gpu_dropin_drivers import _run_env, _tables_agree
from test_gpu_ozaki_schedule import RD_COLS, _G, _rsplit

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def _direction_residual(ctx, mode, entry_decades, seed=4242):
    """n = 200001, m = 300, l = 4; Dx = zl/sxl in [1, 1e16] (DhInv over 16 decades) and the Jacobian's columns scaled by 10^U(-d/2, d/2),
    so each row of B = J sqrt(DhInv) spans about d + 8 decades. Returns ||K sol - rhs||_inf / ||rhs||_inf with K applied by torch
    matmuls and the compact BFGS form (bench.independent_kkt_residual): neither N nor its factor takes part."""
    from hiop_b200.engine import KKTLinSysLowRank
    n, m, l = 200001, 300, 4
    P = synth.make_qn_problem(n, m, l, seed=seed)
    r = np.random.default_rng(7)
    P.sxl[:] = 10.0 ** r.uniform(-8.0, 0.0, n)
    P.zl[:] = 10.0 ** r.uniform(0.0, 8.0, n)
    J = np.vstack([P.Jc, P.Jd]) * 10.0 ** r.uniform(-entry_decades / 2, entry_decades / 2, n)[None, :]
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ITERATE + ("ixl", "ixu", "idl", "idu", "St", "Yt", "rx", "ryc", "ryd")}
    T["J"] = D(J)
    k = KKTLinSysLowRank(ctx, n, P.m_eq, P.m_ineq, l)
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    k.set_secant(P.sigma, T["St"], T["Yt"], P.L, P.D)
    k.set_condense_mode(mode)
    k.update(*(T[kk] for kk in ITERATE))
    assert bool((T["ixl"] == 1.0).all())                      # the independent residual takes Dx = zl/sxl on every column
    dx, dyc, dyd = ctx.zeros(n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(T["rx"].clone(), T["ryc"], T["ryd"], dx, dyc, dyd)
    k.check()
    ctx.sync()
    assert k.condense_mode_used() == mode
    T.update(m_eq=P.m_eq, m_ineq=P.m_ineq, L=P.L, D=P.D)
    rel = independent_kkt_residual(torch, None, 1, T, P.sigma, dx, dyc, dyd)
    k.close()
    return rel


def test_direction_with_dx_over_16_decades(ctx):
    """Dx over 16 decades and the Jacobian's entries over 12 (rows of B spanning about 20 decades): the CRT direction meets
    ||K sol - rhs|| / ||rhs|| <= 1e-8. With the entries over 16 decades the system itself is too ill-conditioned for that gate in any
    mode (the exact FP64 condensation lands near 1e-7 there): the CRT direction must then be no worse than 10x the FP64 one."""
    rel = _direction_residual(ctx, CRT, 12)
    print(f"Dx 16 decades, entries 12: crt {rel:.2e}")
    assert rel <= 1e-8, rel
    rc, rf = _direction_residual(ctx, CRT, 16), _direction_residual(ctx, 0, 16)
    print(f"Dx 16 decades, entries 16: crt {rc:.2e}, fp64 {rf:.2e}")
    assert rc <= 10 * rf, (rc, rf)


@pytest.mark.parametrize("variant", ["vec-rsplit1", "scalar-rsplit8"])
def test_fused_rhs_row_meets_the_sweep_bound(ctx, variant):
    """A pending CRT condensation + solveCompressed: the row-maximum sweep (k_oz_rowmax_dot, VEC or scalar, rsplit 1 or 8) leaves
    tdot = J (DhInv .* rx); against the exact dot with w = fl(DhInv .* rx), |tdot - exact| <= gamma_c sum_k |J_ik w_k| + u |exact| with
    c = 8 + 5 + ceil(nchunks / 8) + 8, the bound of the slice path's sweep. N equals the integer model."""
    G = _G()
    vec = variant.startswith("vec")
    K = 2 * G * RD_COLS + 1000 if variant.endswith("rsplit1") else (G // 4) * RD_COLS - 100
    K += 0 if vec else 1
    assert _rsplit(K, G) == (1 if variant.endswith("rsplit1") else 8)
    M = 100
    P = synth.make_qn_problem(K, M, 0, seed=K)
    k, T = _setup(ctx, P)
    D = ctx.to_device
    dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
    assert k.solveCompressed(D(P.rx), D(P.ryc), D(P.ryd), dx, dyc, dyd)
    k.check()
    ctx.sync()
    assert k.condense_mode_used() == CRT
    N, tdot, DhInv, Dd_inv = k.N(), k.tdot(), k.DhInv(), k.Dd_inv()
    k.close()
    Nm, _ = _model(P.J, DhInv, Dd_inv, P.m_eq)
    assert np.array_equal(N, Nm)
    w = DhInv * P.rx
    ref = bounds.exact_rows(P.J, w)
    c = 8 + 5 + -(-(-(-K // RD_COLS)) // 8) + 8
    tol = bounds.gamma(c) * (np.abs(P.J) @ np.abs(w)) + U * np.abs(ref)
    ratio = float((np.abs(tdot - ref) / tol).max())
    print(f"CRT fused {variant}: K={K} t={crt.bits(K)}: N bit-exact, tdot margin {1.0 / max(ratio, 1e-300):.3g}")
    assert ratio <= 1.0, ratio


def test_exM_with_the_crt_condensation():
    """exM_b200.exe 33000 64 with HIOP_B200=1 HB_CONDENSE=crt against the reference build: the 1e-5 rule on every iterate up to the first
    flipped line-search decision, the same optimum (1e-8), iteration counts within 2"""
    n, m = 33000, 64
    rc_r, out_r, _, tab_r = _run_env("exM_b200.exe", [str(n), str(m)], {})
    assert rc_r == 0, out_r[-1500:]
    rc_b, out_b, err_b, tab_b = _run_env("exM_b200.exe", [str(n), str(m)], {"HIOP_B200": "1", "HB_CONDENSE": "crt"})
    assert rc_b == 0, (out_b[-1500:], err_b[-500:])
    worst, rows = _tables_agree(tab_b, tab_r, until_linesearch_differs=True)
    assert worst <= 1e-5, worst
    assert rows >= min(25, len(tab_r)), (rows, len(tab_r))
    assert abs(len(tab_b) - len(tab_r)) <= 2, (len(tab_b), len(tab_r))
    obj_r = float(re.search(r"objective=([-+0-9.e]+)", out_r).group(1))
    obj_b = float(re.search(r"objective=([-+0-9.e]+)", out_b).group(1))
    print(f"exM {n} {m} crt: {len(tab_b)} iterations (reference {len(tab_r)}), {rows} rows within {worst:.1e}, objective {obj_b!r}")
    assert abs(obj_b - obj_r) <= 1e-8 * abs(obj_r), (obj_b, obj_r)
