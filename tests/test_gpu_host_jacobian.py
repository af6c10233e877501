"""The quasi-Newton KKT path on a Jacobian kept in page-locked host memory (hb_lowrank_set_jacobian_host), against the same handle on a
device Jacobian built from the same seeded problem.

Every pass over J streams it through a ring of device panels. J x keeps the per-2048-column partials of the whole J and J^T y sums each
column in the same row order, so the residual and the full-KKT operator (gemvs only) are bit-identical; the condensation adds the panels'
partial products in panel order and is held to the componentwise bound of oracle/bounds.py. n = 200001 leaves a ragged last panel; the
panel widths give one panel, exactly two, four of the default width and 98 of the smallest width (2048 columns)."""
import numpy as np
import pytest
import torch

from hiop_b200 import _lib, synth
from hiop_b200._lib import EngineError
from oracle import bounds
from oracle import kkt_oracle as ko
from test_gpu_krylov import _ir
from test_gpu_parity import _as_dict, _setup_kkt

pytestmark = pytest.mark.gpu

N, M = 200001, 300
GR_CHUNK = 2048
PANELS = {"one": 200704, "two": 100352, "default": 0, "many": GR_CHUNK}  # 0: the default width (about 128 MB: four panels here)
ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


def _panel_count(panel_cols, n=N, m=M):
    P = panel_cols if panel_cols > 0 else (128 << 20) // (8 * m)
    P = min(-(-P // GR_CHUNK) * GR_CHUNK, -(-n // GR_CHUNK) * GR_CHUNK)
    return -(-n // P)


def test_panel_widths_cover_the_cases():
    assert [_panel_count(PANELS[k]) for k in ("one", "two", "default", "many")] == [1, 2, 4, 98]


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _pinned(a):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


@pytest.fixture(scope="module", params=[0, 6], ids=["l0", "l6"])
def case(request, ctx):
    """(problem dict, device handle, its tensors, pinned Jc / Jd, the oracle's N)"""
    l = request.param
    P = synth.make_qn_problem(N, M, l, seed=91 + l)
    p = _as_dict(P)
    kd, T = _setup_kkt(ctx, p)
    kd.set_condense_mode(0)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    N_ref = ko.condense(st)[0]
    yield dict(P=P, p=p, kd=kd, T=T, Jc=_pinned(P.Jc), Jd=_pinned(P.Jd), DhInv=DhInv, N_ref=N_ref)
    kd.close()


def _host_handle(ctx, c, panel_cols):
    """a handle on the same problem as c["kd"], with J registered from pinned host memory"""
    from hiop_b200.engine import KKTLinSysLowRank
    p, T = c["p"], c["T"]
    l = int(p["l"])
    k = KKTLinSysLowRank(ctx, p["n"], p["m_eq"], p["m_ineq"], max(l, 1))
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian_host(c["Jc"], c["Jd"], panel_cols)
    k.set_secant(float(p["sigma"]), T["St"] if l else None, T["Yt"] if l else None, p["L"], p["D"])
    k.update(*(T[kk] for kk in ITERATE))
    return k


def _update(k, T):
    k.update(*(T[kk] for kk in ITERATE))


@pytest.mark.parametrize("panels", list(PANELS))
def test_gemv_consumers_are_bit_identical(ctx, case, panels):
    P, T, kd = case["P"], case["T"], case["kd"]
    kh = _host_handle(ctx, case, PANELS[panels])
    _update(kd, T)
    D = ctx.to_device
    itr, dat = synth.make_iterate(P)
    it_d = {kk: D(np.ascontiguousarray(v)) for kk, v in itr.items()}
    sizes = {kk: v.size for kk, v in itr.items()}
    args = [D(dat[kk]) for kk in ("c", "d", "grad")] + [0.1, 1e-5] + [D(dat[kk]) for kk in ("xl", "xu", "dl", "du", "crhs")]
    out = []
    for k in (kd, kh):
        res = {rk: ctx.zeros(sizes[dk]) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
        nrm = k.residual_update(it_d, *args, res)
        ctx.sync()
        out.append(({rk: v.cpu().numpy() for rk, v in res.items()}, nrm))
    for rk in ko.RES_NAMES:
        np.testing.assert_array_equal(out[1][0][rk], out[0][0][rk], err_msg=rk)
    assert out[1][1] == out[0][1]
    # y = K x on the full KKT system: H x + J^T y blocks and J x blocks
    rng = np.random.default_rng(5)
    X = {kk: D(rng.standard_normal(sizes[kk])) for kk in ko.DIR_NAMES}
    ys = []
    for k in (kd, kh):
        Y = {rk: ctx.zeros(sizes[dk]) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
        k.kkt_full_times_vec(X, Y)
        ctx.sync()
        ys.append({rk: v.cpu().numpy() for rk, v in Y.items()})
    for rk in ko.RES_NAMES:
        np.testing.assert_array_equal(ys[1][rk], ys[0][rk], err_msg=rk)
    kh.close()


@pytest.mark.parametrize("panels", list(PANELS))
def test_condensation_and_solves_agree(ctx, case, panels):
    P, p, T, kd = case["P"], case["p"], case["T"], case["kd"]
    G = torch.cuda.get_device_properties(0).multi_processor_count
    kh = _host_handle(ctx, case, PANELS[panels])
    _update(kd, T)
    kd.condense()
    kh.condense()
    assert kh.condense_mode_used() == 0
    Nd, Nh = kd.N(), kh.N()
    assert np.array_equal(Nh, Nh.T)
    # against the oracle, under the componentwise bound (l = 0) or the diagonal-scaled one (l > 0); the device handle for scale
    ratio_h = bounds.condensed_error_ratio(Nh, case["N_ref"], P.J, case["DhInv"], P.l, G)
    ratio_d = bounds.condensed_error_ratio(Nd, case["N_ref"], P.J, case["DhInv"], P.l, G)
    assert ratio_h <= 1.0 and ratio_d <= 1.0, (ratio_h, ratio_d)
    # and against each other: both are within the bound of the exact N
    assert bounds.condensed_error_ratio(Nh, Nd, P.J, case["DhInv"], P.l, G) <= 2.0
    # solveCompressed, with a pending condensation (the fused rhs row where it applies)
    sol = []
    for k in (kd, kh):
        _update(k, T)
        D = ctx.to_device
        rx, ryc, ryd = D(P.rx), D(P.ryc), D(P.ryd)
        dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
        assert k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
        k.check()
        ctx.sync()
        sol.append([v.cpu().numpy() for v in (dx, dyc, dyd)])
    for a, b in zip(sol[1], sol[0]):
        assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max()
    # the outer BiCGStab refinement on the full KKT system
    dd, info_d = _ir(ctx, kd, p, 1e-2, 8)
    dh, info_h = _ir(ctx, kh, p, 1e-2, 8)
    assert info_h[0] == info_d[0] and info_h[1] == info_d[1], (info_h, info_d)
    for kk in ko.DIR_NAMES:
        assert np.abs(dh[kk] - dd[kk]).max(initial=0.0) <= 1e-10 * max(1.0, np.abs(dd[kk]).max(initial=0.0)), kk
    # the least-squares multipliers: J J^T in panels, then J vx
    ones = ctx.to_device(np.ones(P.n))
    ys = []
    for k in (kd, kh):
        yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
        assert k.lsq_duals(ones, T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
        ys.append(np.concatenate([yc.cpu().numpy(), yd.cpu().numpy()]))
    assert np.abs(ys[1] - ys[0]).max() <= 1e-10 * np.abs(ys[0]).max()
    kh.close()


def _small(ctx, l=4):
    P = synth.make_qn_problem(20001, 30, l, seed=3)
    p = _as_dict(P)
    kd, T = _setup_kkt(ctx, p)
    c = dict(P=P, p=p, kd=kd, T=T, Jc=_pinned(P.Jc), Jd=_pinned(P.Jd))
    return c, _host_handle(ctx, c, GR_CHUNK)


def _solve(ctx, k, P, T):
    _update(k, T)
    D = ctx.to_device
    dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(D(P.rx), D(P.ryc), D(P.ryd), dx, dyc, dyd)
    ctx.sync()
    return dx.cpu().numpy()


def test_refused_combinations_leave_the_handle_usable(ctx):
    c, kh = _small(ctx)
    P, T, kd = c["P"], c["T"], c["kd"]
    ref = _solve(ctx, kd, P, T)
    L = _lib.lib()
    # the int8-slice condensation needs a global row-maximum pass over J
    assert L.hb_lowrank_set_condense_mode(kh.h, 8) == -1
    assert b"int8-slice" in L.hb_last_error()
    assert kh.condense_mode_used() == 0
    assert np.abs(_solve(ctx, kh, P, T) - ref).max() <= 1e-12 * np.abs(ref).max()
    # a changing Jacobian in device-secant mode would need J_prev on the host
    kh.secant_reset(1.0, 1)
    D = ctx.to_device
    x, g, yc, yd = D(np.zeros(P.n)), D(np.ones(P.n)), D(np.zeros(P.m_eq)), D(np.zeros(P.m_ineq))
    with pytest.raises(EngineError, match="jacobian_is_constant"):
        kh.secant_update(x, g, yc, yd, jacobian_is_constant=False)
    assert kh.secant_update(x, g, yc, yd, jacobian_is_constant=True) == 0
    kd.secant_reset(1.0, 1)
    assert kd.secant_update(x, g, yc, yd, jacobian_is_constant=True) == 0
    x2, g2 = D(np.full(P.n, 0.5)), D(np.linspace(1.0, 2.0, P.n))
    assert kh.secant_update(x2, g2, yc, yd, jacobian_is_constant=True) == kd.secant_update(x2, g2, yc, yd, jacobian_is_constant=True)
    assert np.abs(_solve(ctx, kh, P, T) - _solve(ctx, kd, P, T)).max() <= 1e-12 * np.abs(ref).max()
    # pageable host memory cannot be streamed asynchronously
    Jp = np.ascontiguousarray(P.Jc)
    assert L.hb_lowrank_set_jacobian_host(kh.h, Jp.ctypes.data, c["Jd"].data_ptr(), 0) == -1
    # back to the device-resident path
    kh.set_jacobian(c["T"]["Jc"], c["T"]["Jd"])
    kh.set_condense_mode(8)
    kh.set_condense_mode(-1)
    assert np.abs(_solve(ctx, kh, P, T) - _solve(ctx, kd, P, T)).max() <= 1e-12 * np.abs(ref).max()
    kh.close()
    kd.close()


def test_resources_are_released(ctx):
    """the panels, the copy stream and its events go with the handle"""
    live0 = _lib.lib().hb_debug_live_resources()
    c, kh = _small(ctx)
    _solve(ctx, kh, c["P"], c["T"])
    kh.close()
    c["kd"].close()
    ctx.sync()
    assert _lib.lib().hb_debug_live_resources() == live0


def test_device_footprint_stays_within_the_panels(ctx):
    """J of 2.4 GB on the host; the handle's device memory stays within four panels + O(m^2 + n): J is never copied whole."""
    from hiop_b200.engine import KKTLinSysLowRank
    n, m, l, panel_cols = 1_000_001, 300, 2, 65536
    J_bytes = 8 * m * n
    assert J_bytes >= 2 << 30
    me, mi = m // 2, m - m // 2
    # J = randn / sqrt(n) with a row of ones, generated in place in pinned memory
    Jc = torch.empty((me, n), dtype=torch.float64).pin_memory()
    Jd = torch.empty((mi, n), dtype=torch.float64).pin_memory()
    g = torch.Generator().manual_seed(3)
    for t in (Jc, Jd):
        t.normal_(0.0, n ** -0.5, generator=g)
    Jc[0].fill_(1.0)
    rng = np.random.default_rng(12)
    D = ctx.to_device
    U = lambda k: rng.uniform(1e-3, 1.0, k)
    ixl, ixu, idl, idu = D(np.ones(n)), D(np.zeros(n)), D(np.ones(mi)), D(np.zeros(mi))
    it = [D(U(n)), D(U(n)), D(np.zeros(n)), D(np.ones(n)), D(U(mi)), D(U(mi)), D(np.zeros(mi)), D(np.ones(mi))]
    St_h = rng.standard_normal((l, n))
    Yt_h = St_h * rng.uniform(0.5, 2.0, (l, n))
    St, Yt = D(St_h), D(Yt_h)
    Ls, Ds = synth.secant_LD(St_h, Yt_h)
    rx, ryc, ryd = D(rng.standard_normal(n)), D(rng.standard_normal(me)), D(rng.standard_normal(mi))
    dx, dyc, dyd = ctx.zeros(n), ctx.zeros(me), ctx.zeros(mi)
    ctx.sync()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    k = KKTLinSysLowRank(ctx, n, me, mi, l)
    k.set_patterns(ixl, ixu, idl, idu)
    k.set_jacobian_host(Jc, Jd, panel_cols)
    k.set_secant(1.0, St, Yt, Ls, Ds)
    k.update(*it)
    assert k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
    k.check()
    ctx.sync()
    used = free0 - torch.cuda.mem_get_info()[0]
    panel_bytes = 8 * m * panel_cols
    allowance = 4 * panel_bytes + 8 * (16 * (m + 2 * l) ** 2 + 16 * n) + (64 << 20)
    print(f"J {J_bytes / 2**30:.2f} GiB on the host; the handle holds {used / 2**20:.0f} MiB of device memory (allowance {allowance / 2**20:.0f} MiB)")
    assert used <= allowance < J_bytes
    assert np.all(np.isfinite(dx.cpu().numpy()))
    k.close()


def test_dropin_exM_with_the_jacobian_on_the_host():
    """HIOP_B200_JAC=host: the KKT adapter page-locks HiOp's Jacobian buffers and registers them instead of uploading J; the iterate
    table follows the device-resident run under the 1e-5 rule of the drop-in tests."""
    from test_gpu_dropin_drivers import _run_env, _tables_agree
    args = ["20000", "64"]
    rc_d, out_d, err_d, tab_d = _run_env("exM_b200.exe", args, {"HIOP_B200": "1"})
    assert rc_d == 0, (out_d[-1500:], err_d[-500:])
    rc_h, out_h, err_h, tab_h = _run_env("exM_b200.exe", args, {"HIOP_B200": "1", "HIOP_B200_JAC": "host"})
    assert rc_h == 0, (out_h[-1500:], err_h[-500:])
    worst, rows = _tables_agree(tab_h, tab_d, until_linesearch_differs=True)
    assert worst <= 1e-5, worst
    assert rows >= min(25, len(tab_d)), (rows, len(tab_d))
