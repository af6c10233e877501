"""The dense symmetric solver with the matrix in page-locked host memory (hb_symdense_host, LinSolverSymDenseHost): the factor, the
return value, the inertia and the solutions bit for bit against hb_symdense_dist at P = 1 for one slab, two slabs, one block row per
slab and three slabs with a shorter last one; the backward-error bounds of test_gpu_symdense_dist.py; the strictly lower triangle left
alone; failure, misuse, device footprint and resources."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from dense_handles import K128, assert_lower_untouched, budget_for, budgets, dist_rows_array, factor_dist, matrix, plan, rhs, same_rows, upper_nan
from dense_handles import make_ctx  # noqa: F401 (a fixture)

CHOL, NOPIV, BK, RBT = 2, 1, 0, 3
ERR_INVALID, ERR_STATE = -1, -5


def host_factor(ctx, mode, M, budget, rhs_list):
    """factor M (device, full) with LinSolverSymDenseHost under `budget`; returns rc, inertia, the host buffer after the factorization
    and the solves (NaN below the diagonal going in), and the solutions"""
    from hiop_b200.engine import LinSolverSymDenseHost
    N = M.shape[0]
    s = LinSolverSymDenseHost(ctx, N, budget)
    s.matrix().copy_(upper_nan(M).cpu())
    rc = s.matrixChanged(mode)
    inertia = s.inertia()
    sols = []
    for b in rhs_list:
        x = ctx.to_device(b)
        assert s.solve(x)
        ctx.sync()
        sols.append(x.cpu().numpy())
    F = s.matrix().numpy().copy()
    s.close()
    return rc, inertia, F, sols


def factor_parts(F, mode):
    L = np.triu(F).T.copy()
    if mode == CHOL:
        return L, np.ones(F.shape[0])
    d = np.diag(L).copy()
    np.fill_diagonal(L, 1.0)
    return L, d


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [CHOL, NOPIV], ids=["chol", "nopiv"])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1000, 4099, 8192])
def test_bit_identical_to_dist_for_every_slab_plan_and_within_bounds(make_ctx, mode, N):
    ctx = make_ctx(**K128)
    dev = ctx.device
    M, inertia = matrix(mode, N, seed=N + mode, device=dev)
    bs = [rhs(N, N, 1), rhs(N, N + 1, 3)]
    rc_d, in_d, rows, sols_d = factor_dist(ctx, mode, M, bs)
    Fd = dist_rows_array(rows, N)
    assert rc_d == inertia[0] and in_d == inertia
    for name, budget in budgets(N).items():
        what = f"{('', 'nopiv', 'chol')[mode]} N={N} {name} ({plan(N, budget)['slabs']} slabs)"
        rc, inr, F, sols = host_factor(ctx, mode, M, budget, bs)
        same_rows({r: F[r] for r in range(N)}, Fd, what)
        assert (rc, inr) == (rc_d, in_d), (what, rc, inr)
        for a, b in zip(sols, sols_d):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), what
        assert_lower_untouched(F, M, what)
    # the factor and every solve within the backward-error bounds of test_gpu_symdense_dist.py (one check: all plans gave these bits)
    L, d = factor_parts(F, mode)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    th = max(bounds.block_theta(t(L), 16), bounds.block_theta(t(L), 128))
    fr = bounds.factor_backward_ratio(M, t(L), t(d), None, th)
    assert fr <= 1.0, fr
    for b, x in zip(bs, sols):
        if N <= bounds.EXACT_RESIDUAL_MAX_N:
            sr, _ = bounds.solve_backward_ratio(M.cpu().numpy(), x.T.copy(), b.T.copy(), L, d, None, th)
        else:
            sr, _ = bounds.solve_backward_ratio(M, t(x.T), t(b.T), t(L), t(d), None, th)
        assert sr <= 1.0, sr
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_nopiv_inertia_on_quasidefinite_with_several_slabs(make_ctx):
    """test_gpu_symdense_dist.py's KKT-like quasi-definite family: inertia (m, 0, N - m) with one block row per slab"""
    ctx = make_ctx(**K128)
    N, m = 2049, 683
    M = torch.from_numpy(synth.make_kkt_like(N - m, m, seed=5)).to(ctx.device)
    budget = budget_for(N, -(-N // 128))
    assert plan(N, budget)["slabs"] == 17
    rc, inr, F, _ = host_factor(ctx, NOPIV, M, budget, [])
    assert rc == m and inr == (m, 0, N - m)
    rc_d, in_d, rows, _ = factor_dist(ctx, NOPIV, M, [])
    same_rows({r: F[r] for r in range(N)}, dist_rows_array(rows, N), "quasi-definite")
    assert (rc, inr) == (rc_d, in_d)


@pytest.mark.gpu
def test_breakdown_in_the_third_slab_like_dist(make_ctx):
    ctx = make_ctx(**K128)
    N = 700
    budget = budget_for(N, -(-N // 128))           # one block row per slab: block row 2 is the third slab
    M, _ = matrix(CHOL, N, 3, ctx.device)
    Mb = M.clone()
    Mb[2 * 128 + 5, 2 * 128 + 5] = -1.0            # not SPD
    Z = torch.eye(N, dtype=torch.float64, device=ctx.device)
    Z[2 * 128 + 9, 2 * 128 + 9] = 0.0              # a zero pivot of the no-pivot LDL^T
    for mode, A in ((CHOL, Mb), (NOPIV, Z)):
        rc_d, in_d, _, _ = factor_dist(ctx, mode, A, [])
        rc, inr, F, _ = host_factor(ctx, mode, A, budget, [])
        assert rc == rc_d == -1, (mode, rc, rc_d)
        assert inr == in_d, (mode, inr, in_d)


@pytest.mark.gpu
def test_misuse_refusals_and_resources(make_ctx):
    from hiop_b200.engine import EngineError, LinSolverSymDenseHost
    ctx = make_ctx(**K128)
    L = ctx.L
    live0 = int(L.hb_debug_live_resources())
    N = 700
    budget = budget_for(N, 3)
    s = LinSolverSymDenseHost(ctx, N, budget)
    x = ctx.to_device(rhs(N, 1, 1))
    assert L.hb_symdense_host_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE       # solve before any factorization
    M, inertia = matrix(NOPIV, N, 4, ctx.device)
    s.matrix().copy_(upper_nan(M).cpu())
    assert L.hb_symdense_host_matrix_changed(s.h, BK) == ERR_INVALID
    assert L.hb_symdense_host_matrix_changed(s.h, RBT) == ERR_INVALID
    with pytest.raises(EngineError, match="only CHOLESKY and NOPIV"):
        s.matrixChanged(BK)
    # still usable: the refusals touched neither the buffer nor the handle
    assert s.matrixChanged(NOPIV) == inertia[0] and s.inertia() == inertia
    rc_d, in_d, rows, sols_d = factor_dist(ctx, NOPIV, M, [rhs(N, 2, 1)])
    same_rows({r: s.matrix()[r].numpy() for r in range(N)}, dist_rows_array(rows, N), "after the refusals")
    y = ctx.to_device(rhs(N, 2, 1))
    assert s.solve(y)
    ctx.sync()
    assert np.array_equal(y.cpu().numpy().view(np.uint64), sols_d[0].view(np.uint64))
    # a buffer that is not page-locked is refused, and so is a too short leading dimension
    plain = np.zeros((N, N))
    assert L.hb_symdense_host_set_matrix(s.h, ctypes.c_void_p(plain.ctypes.data), N) == ERR_INVALID
    assert L.hb_symdense_host_set_matrix(s.h, ctypes.c_void_p(s.matrix().data_ptr()), N - 1) == ERR_INVALID
    assert L.hb_symdense_host_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE       # set_matrix dropped the factorization
    # a budget below one block row plus the ring and the scratch
    with pytest.raises(EngineError):
        LinSolverSymDenseHost(ctx, N, budget_for(N, -(-N // 128)) - 1)
    s.close()
    ctx.sync()
    assert int(L.hb_debug_live_resources()) == live0


@pytest.mark.gpu
def test_device_footprint_within_budget_and_factor_bit_identical_at_16384(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseHost
    ctx = make_ctx(**K128)
    dev = ctx.device
    N, budget = 16384, 512 << 20
    p = plan(N, budget)
    assert p["slabs"] >= 4 and p["peak_bytes"] <= budget
    # load the kernels first (lazy module loading takes device memory on a kernel's first launch)
    for mode in (CHOL, NOPIV):
        Mw, _ = matrix(mode, 300, 1, dev)
        host_factor(ctx, mode, Mw, budget_for(300, 3), [rhs(300, 1, 1)])
    M, inertia = matrix(NOPIV, N, 11, dev)
    Mh = upper_nan(M).cpu()
    b = ctx.to_device(rhs(N, 5, 1))
    x = b.clone()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    low = [free0]
    stop = threading.Event()

    def poll():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(dev)[0])
            stop.wait(0.002)
    th = threading.Thread(target=poll)
    th.start()
    try:
        s = LinSolverSymDenseHost(ctx, N, budget)
        s.matrix().copy_(Mh)
        rc = s.matrixChanged(NOPIV)
        inr = s.inertia()
        assert s.solve(x)
        ctx.sync()
    finally:
        stop.set()
        th.join()
    held = free0 - low[0]
    assert 0 < held <= budget, (held, budget)
    assert rc == inertia[0] and inr == inertia
    F = s.matrix().numpy().copy()
    s.close()
    del Mh
    torch.cuda.empty_cache()
    rc_d, in_d, rows, sols_d = factor_dist(ctx, NOPIV, M, [rhs(N, 5, 1)])
    same_rows({r: F[r] for r in range(N)}, dist_rows_array(rows, N), "N=16384 under 512 MiB")
    assert (rc, inr) == (rc_d, in_d)
    assert np.array_equal(x.cpu().numpy().view(np.uint64), sols_d[0].view(np.uint64))
    torch.cuda.empty_cache()
