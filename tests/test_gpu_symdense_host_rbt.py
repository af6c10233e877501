"""The safe mode of the host-resident dense solver (HB_FACT_RBT_NOPIV on hb_symdense_host, LinSolverSymDenseHost(rbt=True)): the kept
A' bit for bit against oracle/rbt_model.py; the factor, the return value, the inertia, the solutions, the corrections and omega bit for
bit against hb_symdense_dist at P = 1 for every slab plan of test_gpu_symdense_host.py and for many transform strips; the strictly lower
triangle of the matrix left alone; the KKT families' inertia against Bunch-Kaufman; failure, misuse, device footprint and resources."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from oracle import bounds
from oracle import rbt_model as rbt
from dense_handles import (K128, assert_lower_untouched, bk_single, budget_for, budgets, dist_rows_array, gpu_families, local_rows, matrix,
                           orig_backward_error, plan, rhs, same_rows, upper_nan)
from dense_handles import make_ctx  # noqa: F401 (a fixture)

RBT, NOPIV = 3, 1
ERR_INVALID, ERR_STATE = -1, -5
NRHS = (1, 3, 16, 17)


def rbt_plan(N, budget):
    from hiop_b200.engine import LinSolverSymDenseHost
    return LinSolverSymDenseHost.rbt_plan_view(N, budget)


def dist_reference(ctx, A, bs):
    """hb_symdense_dist RBT at P = 1 on A (numpy, full): rc, inertia, rows, and per rhs block (nrhs x N) the solution and
    (corrections, omega). A block of 17 is solved as its first 16 and its last one, as the host handle groups them."""
    from hiop_b200.engine import LinSolverSymDenseDist
    N = A.shape[0]
    s = LinSolverSymDenseDist(ctx, N)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(torch.from_numpy(np.ascontiguousarray(A)).to(ctx.device)))
    rc = s.matrixChanged(RBT)
    inr = s.inertia()
    rows = local_rows(s)
    sols = []
    for b in bs:
        parts, stats = [], []
        for lo, hi in ((0, 16), (16, 17)) if len(b) > 16 else ((0, len(b)),):
            x = ctx.to_device(b[lo:hi])
            s.solve(x)
            ctx.sync()
            parts.append(x.cpu().numpy())
            stats.append(s.rbt_stats()[:2])
        sols.append((np.concatenate(parts), stats))
    s.close()
    return rc, inr, rows, sols


def host_rbt(ctx, A, budget, bs):
    """the same on LinSolverSymDenseHost(rbt=True) under `budget`: rc, inertia, the matrix buffer, the kept A', and per rhs block the
    solution, the return value and (corrections, omega)"""
    from hiop_b200.engine import LinSolverSymDenseHost
    N = A.shape[0]
    s = LinSolverSymDenseHost(ctx, N, budget, rbt=True)
    s.matrix().copy_(upper_nan(torch.from_numpy(np.ascontiguousarray(A))))
    rc = s.matrixChanged(RBT)
    inr = s.inertia()
    ms = s.rbt_stats()[2]
    sols = []
    if rc >= 0:
        for b in bs:
            x = ctx.to_device(b)
            ok = s.solve(x)
            ctx.sync()
            sols.append((x.cpu().numpy(), ok, s.rbt_stats()[:2]))
    F, K = s.matrix().numpy().copy(), s.kept().numpy().copy()
    s.close()
    return rc, inr, F, K, sols, ms


def many_strips_budget(N):
    """one block row per slab: the smallest strips the plan makes"""
    return budget_for(N, -(-N // 128))


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.uint64), np.asarray(b).view(np.uint64))


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 2, 3, 127, 128, 129, 300, 1001, 4097, 4099])
def test_kept_copy_factor_and_refined_solves_bit_identical_to_dist(make_ctx, N):
    ctx = make_ctx(**K128)
    A = bounds.known_inertia_matrix(N, N // 8, N // 3, seed=N)[0].numpy()
    Ap = rbt.transform(A, 2)
    bs = [rhs(N, N + q, q) for q in NRHS]
    rc_d, in_d, rows, sols_d = dist_reference(ctx, A, bs)
    neg = N // 8 + N // 3
    assert rc_d == neg and in_d == (neg, 0, N - neg)
    Fd = dist_rows_array(rows, N)
    plans = dict(budgets(N), many_strips=many_strips_budget(N))
    if N >= 1001:
        assert rbt_plan(N, plans["many_strips"])["strips"] >= 4
    M = torch.from_numpy(A)
    for name, budget in plans.items():
        rp = rbt_plan(N, budget)
        what = f"N={N} {name} ({rp['slabs']} slabs, {rp['strips']} strips)"
        rc, inr, F, K, sols, ms = host_rbt(ctx, A, budget, bs)
        assert same_bits(K, Ap), what                         # both triangles of A'
        same_rows({r: F[r] for r in range(N)}, Fd, what)
        assert (rc, inr) == (rc_d, in_d), (what, rc, inr)
        assert ms > 0.0, what
        for q, (x, ok, (corr, om)), (xd, stats_d) in zip(NRHS, sols, sols_d):
            assert ok, (what, q)
            assert same_bits(x, xd), (what, q)
            assert corr == max(c for c, _ in stats_d) and same_bits(om, max(o for _, o in stats_d)), (what, q, corr, om, stats_d)
        assert_lower_untouched(F, M, what)
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_kkt_families_inertia_equals_bunch_kaufman_and_solves_are_refined(make_ctx):
    ctx = make_ctx()
    for name, A in gpu_families():
        N = A.shape[0]
        rc_bk, in_bk = bk_single(ctx, A)
        b = np.random.default_rng(N).standard_normal((N, 3))
        rc, inr, _, _, sols, _ = host_rbt(ctx, A, budget_for(N, 2), [np.ascontiguousarray(b.T)])
        assert rc == rc_bk >= 0 and inr == in_bk, (name, rc, rc_bk, inr, in_bk)
        x, ok, (corr, om) = sols[0]
        assert ok and corr <= 3, (name, corr)
        assert orig_backward_error(A, x.T.copy(), b) <= 1e-14, (name, orig_backward_error(A, x.T.copy(), b), om)
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_zero_row_fails_and_the_handle_then_factors_and_solves(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseHost
    ctx = make_ctx(**K128)
    N = 700
    A = 1e-3 * bounds.known_inertia_matrix(N, 0, 200, seed=4)[0].numpy()
    Z = A.copy()
    Z[300, :] = 0.0
    Z[:, 300] = 0.0
    s = LinSolverSymDenseHost(ctx, N, budget_for(N, 3), rbt=True)
    s.matrix().copy_(upper_nan(torch.from_numpy(Z)))
    assert s.matrixChanged(RBT) == -1
    s.matrix().copy_(upper_nan(torch.from_numpy(A)))
    assert s.matrixChanged(RBT) == 200 and s.inertia() == (200, 0, N - 200)
    x = ctx.to_device(np.ones(N))
    assert s.solve(x)
    ctx.sync()
    assert orig_backward_error(A, x.cpu().numpy(), np.ones(N)) <= 1e-14
    s.close()


@pytest.mark.gpu
def test_misuse_refusals_and_resources(make_ctx):
    from hiop_b200.engine import EngineError, LinSolverSymDenseHost
    ctx = make_ctx(**K128)
    L = ctx.L
    live0 = int(L.hb_debug_live_resources())
    N = 700
    budget = budget_for(N, 3)
    A = bounds.known_inertia_matrix(N, 50, 100, seed=6)[0].numpy()
    Mh = upper_nan(torch.from_numpy(A))
    # without a registered copy the safe mode is refused and the handle goes on
    s = LinSolverSymDenseHost(ctx, N, budget)
    s.matrix().copy_(Mh)
    assert L.hb_symdense_host_matrix_changed(s.h, RBT) == ERR_INVALID
    with pytest.raises(EngineError, match="only CHOLESKY and NOPIV"):
        s.matrixChanged(RBT)
    assert s.matrixChanged(NOPIV) == 150
    s.close()
    # with one: every bad copy is refused, unregisters the copy and drops the factorization
    s = LinSolverSymDenseHost(ctx, N, budget, rbt=True)
    s.matrix().copy_(Mh)
    assert s.matrixChanged(RBT) == 150
    K = s.kept()
    x = ctx.to_device(rhs(N, 1, 1))
    plain = np.zeros((N, N))
    bad = [(ctypes.c_void_p(plain.ctypes.data), N),                              # not page-locked
           (ctypes.c_void_p(K.data_ptr()), N - 1),                               # ld < N
           (ctypes.c_void_p(s.matrix().data_ptr()), N)]                          # the matrix itself
    for ptr, ld in bad:
        assert L.hb_symdense_host_set_rbt_copy(s.h, ptr, ld) == ERR_INVALID
        assert L.hb_symdense_host_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE
        assert L.hb_symdense_host_matrix_changed(s.h, RBT) == ERR_INVALID
        s.matrix().copy_(Mh)
        assert L.hb_symdense_host_set_rbt_copy(s.h, ctypes.c_void_p(K.data_ptr()), N) == 0
        assert s.matrixChanged(RBT) == 150
    # a good copy drops the factorization too; NULL unregisters it
    assert L.hb_symdense_host_set_rbt_copy(s.h, ctypes.c_void_p(K.data_ptr()), N) == 0
    assert L.hb_symdense_host_solve(s.h, ctypes.c_void_p(x.data_ptr()), 1) == ERR_STATE
    assert L.hb_symdense_host_set_rbt_copy(s.h, None, N) == 0
    s.matrix().copy_(Mh)
    assert L.hb_symdense_host_matrix_changed(s.h, RBT) == ERR_INVALID
    assert L.hb_symdense_host_set_rbt_copy(s.h, ctypes.c_void_p(K.data_ptr()), N) == 0
    assert s.matrixChanged(RBT) == 150 and s.solve(x)
    ctx.sync()
    assert L.hb_symdense_host_matrix_changed(s.h, 0) == ERR_INVALID           # Bunch-Kaufman stays refused
    s.close()
    ctx.sync()
    assert int(L.hb_debug_live_resources()) == live0


@pytest.mark.gpu
def test_device_footprint_within_budget_and_bit_identical_at_16384(make_ctx):
    from hiop_b200.engine import LinSolverSymDenseHost
    ctx = make_ctx(**K128)
    dev = ctx.device
    N, budget = 16384, 512 << 20
    rp = rbt_plan(N, budget)
    assert rp["slabs"] >= 4 and rp["strips"] >= 2 and rp["peak_bytes"] <= budget and plan(N, budget)["peak_bytes"] == rp["peak_bytes"]
    # load the kernels first (lazy module loading takes device memory on a kernel's first launch)
    Aw = bounds.known_inertia_matrix(300, 10, 20, seed=1)[0].numpy()
    host_rbt(ctx, Aw, budget_for(300, 3), [rhs(300, 1, 1)])
    M, inertia = matrix(NOPIV, N, 11, dev)
    A = M.cpu().numpy()
    Mh = upper_nan(M).cpu()
    b = rhs(N, 5, 2)
    x = ctx.to_device(b)
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
        s = LinSolverSymDenseHost(ctx, N, budget, rbt=True)
        s.matrix().copy_(Mh)
        rc = s.matrixChanged(RBT)
        inr = s.inertia()
        ok = s.solve(x)
        ctx.sync()
        corr, om, _ = s.rbt_stats()
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
    rc_d, in_d, rows, sols_d = dist_reference(ctx, A, [b])
    same_rows({r: F[r] for r in range(N)}, dist_rows_array(rows, N), "N=16384 under 512 MiB")
    assert (rc, inr) == (rc_d, in_d)
    xd, stats_d = sols_d[0]
    assert ok and same_bits(x.cpu().numpy(), xd) and (corr, om) == stats_d[0]
    torch.cuda.empty_cache()
