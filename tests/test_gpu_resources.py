"""Ownership of the engine's device resources: whatever a context and its handles allocate on the way -- every lazily grown buffer,
stream and event -- is released when they are destroyed, and a create that fails part-way releases what it had and leaves the context
usable. hb_debug_live_resources() counts the device buffers, pinned buffers, streams and events held."""
import ctypes

import numpy as np
import pytest

from hiop_b200 import _lib, synth
from oracle import kkt_oracle as ko
from test_gpu_dense_dispatch import _matrix
from test_gpu_krylov import _ir
from test_gpu_mds import _device_run
from test_gpu_parity import _as_dict, _relerr, _run_solve, _setup_kkt

pytestmark = pytest.mark.gpu
HB_ERR_ALLOC = -3
ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


def _live():
    return _lib.lib().hb_debug_live_resources()


def _host_solve(k, P):
    p = _as_dict(P)
    it = {kk: np.ascontiguousarray(p[kk]) for kk in ITERATE}
    out = (np.zeros(P.n), np.zeros(P.m_eq), np.zeros(P.m_ineq))
    k.kkt_system_host(np.ascontiguousarray(P.Jc), np.ascontiguousarray(P.Jd), it, P.rx.copy(), P.ryc.copy(), P.ryd.copy(), *out)
    return out


def test_every_lazy_path_releases_what_it_holds():
    from hiop_b200.engine import Context, LinSolverSymDense
    live0 = _live()
    ctx = Context(0)
    assert _live() > live0
    ctx.enable_timing(True)
    ctx.phase_timeline(True)
    # the condensation in FP64 and with 8 int8 slices, each followed by the fused-rhs solve; BiCGStab, the LSQ duals, the device secant
    P = synth.make_qn_problem(6000, 40, 4, seed=21)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    for mode in (0, 8):
        k.set_condense_mode(mode)
        k.update(*(T[kk] for kk in ITERATE))
        _run_solve(ctx, k, p)
        assert k.condense_mode_used() == mode
    ctx.phase_timeline(False)
    _ir(ctx, k, p, 1e-2, 8)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(ctx.to_device(np.ones(P.n)), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    k.secant_reset(1.0, 1)
    keep = []
    for it in synth.make_secant_sequence(P.n, P.m_eq, P.m_ineq, steps=3):
        keep.append(ctx.to_device(np.vstack([it["Jc"], it["Jd"]])))
        k.set_jacobian(keep[-1][:P.m_eq], keep[-1][P.m_eq:])
        k.secant_update(*(ctx.to_device(it[kk]) for kk in ("x", "grad_f", "yc", "yd")))
    ctx.sync()
    k.close()
    # more (M, K) shapes than the SYRK schedule cache has ways (4), then a condensed system that takes the look-ahead Cholesky
    for n, m in ((1000, 8), (1100, 9), (1200, 10), (1300, 11), (1400, 12), (6000, 2050)):
        p = _as_dict(synth.make_qn_problem(n, m, 2, seed=n))
        k, _ = _setup_kkt(ctx, p)
        _run_solve(ctx, k, p)
        k.close()
    # the whole system from host memory: J uploaded at once, and (m n >= 2^25 doubles, n >= 2048) in chunks on a second stream
    for n, m in ((3000, 24), (1 << 19, 64)):
        P = synth.make_qn_problem(n, m, 4, seed=5)
        k, _ = _setup_kkt(ctx, _as_dict(P))
        assert all(np.all(np.isfinite(v)) for v in _host_solve(k, P))
        k.close()
    # the dense symmetric solver in all three modes: one-CTA, panel and blocked paths, and, at an odd order past the look-ahead and
    # cluster thresholds, the padded copy
    for N in (10, 200, 1025):
        for mode in (LinSolverSymDense.BUNCH_KAUFMAN, LinSolverSymDense.NOPIV, LinSolverSymDense.CHOLESKY):
            K, neg = _matrix(mode, N)
            s = LinSolverSymDense(ctx, N, mode)
            assert s.matrixChanged_host(np.triu(K)) == neg
            b = np.random.default_rng(N).standard_normal(N)
            ref = np.linalg.solve(K, b)
            assert s.solve_host(b)
            assert np.abs(b - ref).max() <= 1e-8 * np.abs(ref).max()
            s.close()
    _device_run(ctx, synth.make_mds_problem(200, 50, 20, 30, seed=9), True)
    ctx.close()
    assert _live() == live0


def test_failed_create_leaves_nothing_behind():
    from hiop_b200.engine import Context
    ctx = Context(0)
    L = _lib.lib()
    live = _live()
    h = ctypes.c_void_p()
    # m = 2^20 needs an 8 TiB C_aug, allocated after the small n- and m_ineq-sized buffers succeeded
    assert L.hb_lowrank_create(ctx.h, 1000, 1 << 20, 0, 6, ctypes.byref(h)) == HB_ERR_ALLOC
    assert h.value is None
    assert b"C_aug" in L.hb_last_error()
    assert _live() == live
    # the same context then solves a normal system
    P = synth.make_qn_problem(3000, 24, 4, seed=5)
    p = _as_dict(P)
    k, _ = _setup_kkt(ctx, p)
    dx, dyc, dyd = _run_solve(ctx, k, p)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    dxo, dyco, dydo, _ = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    assert _relerr(dx, dxo) <= 1e-8 and _relerr(dyc, dyco) <= 1e-8 and _relerr(dyd, dydo) <= 1e-8
    k.close()
    ctx.close()
