"""The refinement loop of the random-butterfly safe mode (hb_rbt_solve, shared by hb_symdense and hb_symdense_dist), read from inside
through hb_debug_symdense_rbt_solve / hb_debug_symdense_dist_rbt_solve: ||A'||_inf on both handles against the exact row sums of the
model's A', every pass's norms, omega and decision against the host and the stopping rule, each correction against a sweep of its
residual, every exit placed with a margin through the one-GPU reference override and matched with oracle/rbt_model.refine, non-finite
right-hand sides on both handles (P = 1 and 2), scale-invariant omegas over several right-hand sides, and the handle after a failed
solve.

Single-rank cases run on one GPU. The P = 2 cases spawn one process per GPU and skip when fewer GPUs are present."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from oracle import bounds
from oracle import rbt_model as rbt
from test_cpu_rbt_model import known_matrix, PLACED, PLACED_MIN_N, assert_corrected_x, assert_placed, placed_reference, placed_rhs
from dense_handles import make_ctx, gpu_families, upper_nan  # noqa: F401 (make_ctx: a fixture)
from multirank import run_ranks

pytestmark = pytest.mark.gpu
RBT = 3
MAX_PASSES = rbt.MAX_CORRECTIONS + 1
SIZES = [1, 2, 3, 129, 1000, 2049, 4099]     # 2049 = 1 (mod 4): the fused transform's window grows; odd N: a padded factor copy


def p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@functools.lru_cache(maxsize=len(SIZES))
def model(N):
    """the test matrix of order N, the model's A' and its no-pivot factor"""
    A = known_matrix(N)
    Ap = rbt.transform(A)
    return A, Ap, rbt.nopiv_ldlt(Ap)


class Trace:
    def __init__(self, ret, passes, anorm, norms, xp, bp, x, stats):
        self.ret, self.passes, self.anorm, self.norms, self.xp, self.bp, self.x, self.stats = ret, passes, anorm, norms, xp, bp, x, stats


def _traced(entry, ctx, h, b, *extra):
    N, nrhs = b.shape
    xd = ctx.to_device(np.ascontiguousarray(b.T))
    ret, passes = ctypes.c_int(-9), ctypes.c_int(-9)
    an = np.full(1, np.nan)
    norms = np.full(MAX_PASSES * (3 * nrhs + 1), np.nan)
    xp = np.full((MAX_PASSES, N, nrhs), np.nan)
    bp = np.full((N, nrhs), np.nan)
    rc = entry(h, ctypes.c_void_p(xd.data_ptr()), nrhs, *extra, ctypes.byref(ret), ctypes.byref(passes), p(an), p(norms), p(xp), p(bp))
    assert rc == 0, ctx.L.hb_last_error().decode()
    ctx.sync()
    P = passes.value
    return Trace(ret.value, P, an[0], norms[:P * (3 * nrhs + 1)].reshape(P, 3 * nrhs + 1), xp[:P], bp, xd.cpu().numpy().T.copy(), None)


def single_handle(ctx, A):
    from hiop_b200.engine import LinSolverSymDense
    s = LinSolverSymDense(ctx, A.shape[0], RBT)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(torch.from_numpy(np.ascontiguousarray(A)).to(ctx.device)))
    ctx.sync()
    assert s.matrixChanged() >= 0
    return s


def dist_handle(ctx, A):
    from hiop_b200.engine import LinSolverSymDenseDist
    s = LinSolverSymDenseDist(ctx, A.shape[0])
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(torch.from_numpy(np.ascontiguousarray(A)).to(ctx.device)))
    assert s.matrixChanged(RBT) >= 0
    return s


def traced_single(ctx, s, b, Aref=None, anorm=0.0):
    """one traced solve on the one-GPU handle; Aref (numpy, full) and anorm replace the kept A' and ||A'||_inf when given"""
    Ad = None if Aref is None else torch.from_numpy(np.ascontiguousarray(Aref)).to(ctx.device)
    torch.cuda.synchronize()
    t = _traced(ctx.L.hb_debug_symdense_rbt_solve, ctx, s.h, b, None if Ad is None else ctypes.c_void_p(Ad.data_ptr()), float(anorm))
    t.stats = s.rbt_stats()
    return t


def traced_dist(ctx, s, b):
    t = _traced(ctx.L.hb_debug_symdense_dist_rbt_solve, ctx, s.h, b)
    t.stats = s.rbt_stats()
    return t


def rule_corrects(k, om, prev):
    """the stopping rule: True when the loop corrects after reading omega `om` with k corrections made and `prev` before the last"""
    return bool(np.isfinite(om) and k < rbt.MAX_CORRECTIONS and om > rbt.EPS and om <= 0.5 * prev)


def check_decisions(t):
    """omega of every pass is the NaN-wins max of the column quotients of the traced norms, each decision is the rule applied to the
    device's own omegas, and the return value and the statistics agree with the last one"""
    nrhs = t.bp.shape[1]
    assert 1 <= t.passes <= MAX_PASSES
    prev = np.inf
    for k in range(t.passes):
        m3 = t.norms[k, :3 * nrhs].reshape(nrhs, 3)
        w = rbt.column_omegas(t.anorm, m3[:, 0], m3[:, 1], m3[:, 2])
        om = t.norms[k, -1]
        want = rbt.nan_max(w)
        assert om == want or (np.isnan(om) and np.isnan(want)), (k, om, want)
        assert rule_corrects(k, om, prev) == (k + 1 < t.passes), (k, om, prev, t.passes)
        prev = om
    last = t.norms[-1, -1]
    assert t.ret == int(np.isfinite(last))
    assert t.stats[0] == t.passes - 1
    assert t.stats[1] == last or (np.isnan(t.stats[1]) and np.isnan(last))


def residual_chain(N):
    """longest addition chain of a row of k_rbt_rows: ceil(N / 256) terms per thread, then the block reduction (warp and block trees)"""
    return -(-N // 256) + 13 + 1


def check_passes(t, Ap, fac, Aref=None):
    """every traced pass against the host: max |x'| and max |b'| exactly, max |r| within the evaluation bounds of the device's and the
    host's residual, and each correction x'_k+1 - x'_k a sweep of r_k within the solve bound of the factor"""
    N, nrhs = t.bp.shape
    Ar = Ap if Aref is None else Aref
    aA = np.abs(Ar)
    ev = bounds.gamma(residual_chain(N)) + bounds.gamma(N + 1)
    L, d, _ = fac
    th = max(bounds.block_theta(L, 16), bounds.block_theta(L, 128))
    for k in range(t.passes):
        xk = t.xp[k]
        m3 = t.norms[k, :3 * nrhs].reshape(nrhs, 3)
        assert np.array_equal(m3[:, 1], np.abs(xk).max(axis=0), equal_nan=True), k
        assert np.array_equal(m3[:, 2], np.abs(t.bp).max(axis=0), equal_nan=True), k
        r = t.bp - Ar @ xk
        scale = aA @ np.abs(xk) + np.abs(t.bp)
        tol = ev * scale.max(axis=0)
        assert (np.abs(m3[:, 0] - np.abs(r).max(axis=0)) <= tol).all(), (k, m3[:, 0], np.abs(r).max(axis=0), tol)
        if k + 1 < t.passes:
            dk = t.xp[k + 1] - xk
            # r_k as the device formed it is within ev |Ar||x_k| + |b'| of r; recovering d_k from x'_k+1 = fl(x'_k + d_k) costs
            # u |x'_k+1| and u |d_k| per entry, through |A'|
            extra = ev * scale + np.abs(Ap) @ (bounds.U * (np.abs(t.xp[k + 1]) + np.abs(dk)))
            ratio, _ = bounds.solve_backward_ratio(Ap, dk, r, L, d, None, th, extra=extra)
            assert ratio <= 1.0, (k, ratio)


# ---- ||A'||_inf ----------------------------------------------------------------------------------------------------------------------
def exact_anorm(Ap):
    return max(bounds.exact_sum(np.abs(row)) for row in Ap)


def fused_chain(N):
    """k_rbt_fused + k_rbt_rowsum: a warp tree and one pair sum over the 64 columns of a tile, then the ceil(ceil(ceil(N/2)/2) / 16) tile
    partials in order"""
    h = (N + 1) // 2
    return 6 + -(-((h + 1) // 2) // 16)


@pytest.mark.parametrize("N", SIZES)
def test_anorm_on_both_handles(make_ctx, N):
    ctx = make_ctx()
    A, Ap, _ = model(N)
    ref = exact_anorm(Ap)
    b = np.random.default_rng(N).standard_normal((N, 1))
    s = single_handle(ctx, A)
    a1 = traced_single(ctx, s, b).anorm
    s.close()
    d = dist_handle(ctx, A)
    a2 = traced_dist(ctx, d, b).anorm
    d.close()
    assert abs(a1 - ref) <= bounds.gamma(fused_chain(N)) * ref, (a1, ref)
    assert abs(a2 - ref) <= bounds.gamma(residual_chain(N)) * ref, (a2, ref)


# ---- every pass against the host ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nrhs", [1, 3])
@pytest.mark.parametrize("N", SIZES)
def test_every_pass_against_the_host(make_ctx, N, nrhs):
    """unperturbed solves on both handles (P = 1): the traced b' is the model's U^T b bit for bit, and every pass, decision and
    correction holds. Convergence after k >= 1 corrections sits on the rounding floor of omega; it is checked here only as a decision."""
    ctx = make_ctx()
    A, Ap, fac = model(N)
    b = np.random.default_rng(N + nrhs).standard_normal((N, nrhs))
    s = single_handle(ctx, A)
    d = dist_handle(ctx, A)
    for t in (traced_single(ctx, s, b), traced_dist(ctx, d, b)):
        assert np.array_equal(t.bp.view(np.uint64), rbt.apply_UT(b).view(np.uint64))
        check_decisions(t)
        check_passes(t, Ap, fac)
        assert t.ret == 1 and rbt.backward_error(A, t.x, b) <= 1e-14
    s.close()
    d.close()
    torch.cuda.empty_cache()


def test_every_pass_on_the_families(make_ctx):
    """the same on the indefinite, saddle-point and KKT matrices of gpu_families(), three right-hand sides"""
    ctx = make_ctx()
    for name, A in gpu_families():
        N = A.shape[0]
        Ap = rbt.transform(A)
        fac = rbt.nopiv_ldlt(Ap)
        b = np.random.default_rng(N).standard_normal((N, 3))
        s = single_handle(ctx, A)
        d = dist_handle(ctx, A)
        for t in (traced_single(ctx, s, b), traced_dist(ctx, d, b)):
            check_decisions(t)
            check_passes(t, Ap, fac)
            assert t.ret == 1 and rbt.backward_error(A, t.x, b) <= 1e-14, name
        s.close()
        d.close()


@pytest.mark.parametrize("N", [129, 1000])
def test_correction_is_a_sweep_of_its_residual(make_ctx, N):
    """with Aref = A' (1 + 2^-8) every correction is large against the rounding floor, so the sweep check of check_passes has teeth"""
    ctx = make_ctx()
    A, Ap, fac = model(N)
    b = placed_rhs(N, 3, "cap", seed=N)
    Aref, anorm = placed_reference(Ap, "cap")
    s = single_handle(ctx, A)
    t = traced_single(ctx, s, b, Aref, anorm)
    s.close()
    assert t.passes == 4
    check_decisions(t)
    check_passes(t, Ap, fac, Aref)


# ---- every exit placed with a margin ------------------------------------------------------------------------------------------------
def _placed_cases():
    for case in PLACED:
        for N in SIZES:
            if case in ("stagnation", "divergence") and N < PLACED_MIN_N:
                continue
            yield case, N


@pytest.mark.parametrize("nrhs", [1, 3])
@pytest.mark.parametrize("case,N", list(_placed_cases()))
def test_every_exit_is_placed_and_matches_the_model(make_ctx, case, N, nrhs):
    if case in ("nan", "inf"):
        nrhs = 3                    # a non-finite column among finite ones
    ctx = make_ctx()
    A, Ap, fac = model(N)
    b = placed_rhs(N, nrhs, case, seed=N + nrhs)
    Aref, anorm = placed_reference(Ap, case) if case in ("cap", "stagnation", "divergence", "overflow") else (None, 0.0)
    _, mcorr, mom, moms, mret = rbt.refine(A, b, Aref=Aref, anorm=None if Aref is None else anorm, Ap=Ap, factor=fac)
    assert_placed(case, mcorr, mret, moms)
    s = single_handle(ctx, A)
    t = traced_single(ctx, s, b, Aref, anorm)
    oms = list(t.norms[:, -1])
    assert_placed(case, t.passes - 1, t.ret, oms)
    check_decisions(t)
    assert (t.passes - 1, t.ret) == (mcorr, mret)
    for k, (om, mo) in enumerate(zip(oms, moms)):
        # the device's and the model's omegas come from different sweeps and residual orders: they agree to the rounding of the
        # residual, far inside the factor-10 margins of the exits
        assert (np.isnan(om) and np.isnan(mo)) or abs(om - mo) <= 1e-3 * abs(mo) + 1e-14, (k, om, mo)
    if case == "zero":
        assert np.array_equal(t.x, np.zeros_like(t.x)) and tuple(t.stats[:2]) == (0, 0.0)
    if case == "divergence":
        assert_corrected_x(A, b, t.x)
    if case in ("cap", "stagnation", "divergence", "overflow"):
        # the override leaves the kept A' and ||A'||_inf alone: the next solve on the handle is a fresh handle's, bit for bit
        b1 = np.random.default_rng(1).standard_normal((N, 1))
        u = traced_single(ctx, s, b1)
        s2 = single_handle(ctx, A)
        v = traced_single(ctx, s2, b1)
        s2.close()
        assert np.array_equal(u.x.view(np.uint64), v.x.view(np.uint64)) and u.anorm == v.anorm and tuple(u.stats[:2]) == tuple(v.stats[:2])
        assert u.ret == 1 and rbt.backward_error(A, u.x, b1) <= 1e-14
    s.close()


@pytest.mark.parametrize("case", ["nan", "inf"])
@pytest.mark.parametrize("N", SIZES)
def test_non_finite_rhs_on_the_distributed_handle(make_ctx, N, case):
    ctx = make_ctx()
    A, _, _ = model(N)
    d = dist_handle(ctx, A)
    t = traced_dist(ctx, d, placed_rhs(N, 3, case, seed=N))
    d.close()
    assert_placed(case, t.passes - 1, t.ret, list(t.norms[:, -1]))
    check_decisions(t)


def _nonfinite_worker(rank, world, uid, out, N):
    from hiop_b200.engine import Context
    torch.cuda.set_device(rank)
    ctx = Context(rank)
    try:
        ctx.init_comm(world, rank, uid)
        A, _, _ = model(N)
        d = dist_handle(ctx, A)
        res = []
        for case in ("nan", "inf", "finite"):
            b = placed_rhs(N, 3, "cap" if case == "finite" else case, seed=N)
            t = traced_dist(ctx, d, b)
            res.append((t.ret, t.passes, t.stats[:2], list(t.norms[:, -1]), t.x if case == "finite" else None, t.anorm))
        d.close()
        out[rank] = res
    finally:
        ctx.close()


@pytest.mark.parametrize("N", [129, 1000])
def test_non_finite_rhs_at_two_ranks(make_ctx, N):
    """every rank returns 0 after no correction with omega NaN (a rank left in a collective would trip run_ranks' deadline), the next
    finite solve agrees on every rank, and ||A'||_inf (each rank's row sums, then an all-reduce max) is within its summation bound"""
    out = run_ranks(_nonfinite_worker, 2, (N,), comm="nccl")
    ref = exact_anorm(model(N)[1])
    for rank in range(2):
        assert abs(out[rank][2][5] - ref) <= bounds.gamma(residual_chain(N)) * ref
        for case, (ret, passes, stats, oms, _, _) in zip(("nan", "inf"), out[rank][:2]):
            assert_placed(case, passes - 1, ret, oms)
            assert np.isnan(stats[1]) and stats[0] == 0
    f0, f1 = out[0][2], out[1][2]
    assert f0[0] == f1[0] == 1 and f0[1] == f1[1] and np.array_equal(f0[4].view(np.uint64), f1[4].view(np.uint64))


# ---- several right-hand sides ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [3, 129, 2049])
def test_column_omegas_are_scale_invariant(make_ctx, N):
    """b = [b0, 2^-600 b0, 2^600 b0]: every operation scales exactly, so every pass's column quotients agree bit for bit, and omega is
    their max; a distinct column of its own scale changes nothing in the others"""
    ctx = make_ctx()
    A, Ap, fac = model(N)
    b0 = np.random.default_rng(N).standard_normal(N)
    b = np.stack([b0, 2.0 ** -600 * b0, 2.0 ** 600 * b0], axis=1)
    s = single_handle(ctx, A)
    d = dist_handle(ctx, A)
    for t in (traced_single(ctx, s, b), traced_dist(ctx, d, b)):
        check_decisions(t)
        for k in range(t.passes):
            m3 = t.norms[k, :9].reshape(3, 3)
            w = rbt.column_omegas(t.anorm, m3[:, 0], m3[:, 1], m3[:, 2])
            assert w[0] == w[1] == w[2] == t.norms[k, -1], (k, w)
        assert np.array_equal(t.x[:, 1], 2.0 ** -600 * t.x[:, 0]) and np.array_equal(t.x[:, 2], 2.0 ** 600 * t.x[:, 0])
    # distinct columns at three scales: omega follows the largest column quotient, checked pass by pass
    bm = np.random.default_rng(N + 1).standard_normal((N, 3)) * np.array([1.0, 2.0 ** -600, 2.0 ** 600])
    t = traced_single(ctx, s, bm)
    check_decisions(t)
    check_passes(t, Ap, fac)
    s.close()
    d.close()


# ---- the handle after a failed solve ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [129, 1000])
def test_failed_solve_leaves_the_handle_as_fresh(make_ctx, N):
    ctx = make_ctx()
    live0 = int(ctx.L.hb_debug_live_resources())
    A, _, _ = model(N)
    b = np.random.default_rng(N).standard_normal((N, 3))
    fresh = single_handle(ctx, A)
    want = traced_single(ctx, fresh, b)
    fresh.close()
    s = single_handle(ctx, A)
    for case in ("nan", "inf"):
        t = traced_single(ctx, s, placed_rhs(N, 3, case, seed=N))
        assert t.ret == 0 and t.passes == 1 and np.isnan(t.stats[1])
    got = traced_single(ctx, s, b)
    assert np.array_equal(got.x.view(np.uint64), want.x.view(np.uint64)) and tuple(got.stats[:2]) == tuple(want.stats[:2])
    # the same through the production entry, which never traces
    x = ctx.to_device(np.ascontiguousarray(b.T))
    assert s.solve(x)
    ctx.sync()
    assert np.array_equal(x.cpu().numpy().T.view(np.uint64), want.x.view(np.uint64)) and tuple(s.rbt_stats()[:2]) == tuple(want.stats[:2])
    s.close()
    torch.cuda.empty_cache()
    assert int(ctx.L.hb_debug_live_resources()) == live0
