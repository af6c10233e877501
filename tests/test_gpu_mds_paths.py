"""The mixed dense-sparse KKT path (hb_mds.cu) held to oracle/mds_model.py bit for bit, at the bench's sparse shape, on every sparsity
edge and on both sides of each dense-solver dispatch row it takes.

The packed rhs and the unpack are observed without any read-back entry point: hb_mds_solve_compressed takes the dense solver handle as
an argument, so the solve runs once on a factored identity of order N. Every operation of an identity's factor and solve is exact, so
dx[nxs:], dyc, dyd are then the packed rhs and dx[:nxs] is the unpack of it; each test first asserts that the identity solve returns a
random vector bit for bit on the dispatch row it uses. With the real factor, the dense part of the step is held to the solve's backward
error bound against the device's own M and the model's rhs, and dx_s to the model's unpack of the device's own dense solution."""
import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from oracle import mds_model as mm
from test_cpu_mds_model import EDGES, edge_problem

pytestmark = pytest.mark.gpu
BK, NOPIV = 0, 1


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def same_bits(a, b, what):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    bad = np.nonzero(u64(a).ravel() != u64(b).ravel())[0]
    if bad.size:
        idx = [np.unravel_index(k, a.shape) for k in bad[:6]]
        neg0 = int(((a.ravel()[bad] == 0.0) & (b.ravel()[bad] == 0.0)).sum())
        pytest.fail(f"{what}: {bad.size} entries differ ({neg0} of them only in the sign of a zero), first {[(i, a[i], b[i]) for i in idx]}")


def sync(ctx):
    torch.cuda.synchronize()         # torch's own stream (tensors made or copied by torch)
    ctx.sync()                       # the engine's stream


_IDENTITY_OK = {}


def identity_solver(ctx, N, mode):
    """a LinSolverSymDense holding the factored identity of order N; asserts (once per order and mode) that its solve returns a random
    vector bit for bit"""
    from hiop_b200.engine import LinSolverSymDense
    s = LinSolverSymDense(ctx, N, mode)
    s.set_matrix(ctx.to_device(np.eye(N)))
    sync(ctx)
    assert s.matrixChanged() == 0
    if (N, mode) not in _IDENTITY_OK:
        b = np.random.default_rng(N).standard_normal(N)
        x = ctx.to_device(b)
        assert s.solve(x)
        sync(ctx)
        same_bits(x.cpu().numpy(), b, f"identity solve N={N} mode={mode}")
        _IDENTITY_OK[(N, mode)] = True
    return s


FIELDS = ("zl", "sxl", "zu", "sxu", "ixl", "ixu", "Hd", "Hs_diag", "Jcd", "Jdd", "Jcs_vals", "Jds_vals", "vl", "sdl", "vu", "sdu", "idl", "idu",
          "delta_wx", "delta_wd", "delta_cc", "delta_cd", "rx", "ryc", "ryd")


class Run:
    """one handle: set_sparsity, update, build, factorizeWithCurvCheck, and solves with the real factor or an identity"""

    def __init__(self, ctx, p, safe=True):
        from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd
        self.ctx, self.p, self.safe = ctx, p, safe
        self.N = p.nxd + p.neq + p.nineq
        self.k = KKTLinSysCompressedMDSXYcYd(ctx, p.nxs, p.nxd, p.neq, p.nineq, safe_mode=safe)
        self.k.set_sparsity(p.iRow_c, p.jCol_c, p.iRow_d, p.jCol_d)

    def build(self, p=None):
        p = p or self.p
        self.p = p
        T = self.T = {f: self.ctx.to_device(getattr(p, f)) for f in FIELDS}
        sync(self.ctx)
        self.k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
        self.k.build_kkt_matrix(*[T[f] for f in FIELDS[6:22]])
        self.M = self.k.Msys().copy()
        self.ret = self.k.factorizeWithCurvCheck()
        return self

    def solve(self, identity):
        from hiop_b200._lib import check
        p, ctx = self.p, self.ctx
        dx, dyc, dyd = ctx.zeros(p.nxs + p.nxd), ctx.zeros(p.neq), ctx.zeros(p.nineq)
        if identity:
            s = identity_solver(ctx, self.N, BK if self.safe else NOPIV)
            from hiop_b200.engine import _ptr
            rc = ctx.L.hb_mds_solve_compressed(self.k.h, s.h, *[_ptr(t) for t in (self.T["rx"], self.T["ryc"], self.T["ryd"], dx, dyc, dyd)])
            check(rc, "hb_mds_solve_compressed")
            sync(ctx)
            s.close()
        else:
            assert self.k.solveCompressed(self.T["rx"], self.T["ryc"], self.T["ryd"], dx, dyc, dyd)
            sync(ctx)
        return dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy()

    def close(self):
        self.k.close()


def check_exact(r, what):
    """assembly, Haynsworth counts, pack and unpack of one built handle against the model, bit for bit; the inputs unchanged"""
    p = r.p
    Dx, Hxs, Dd_inv = mm.diagonals(p)
    M, n_empty = mm.assemble(p, Dx, Hxs, Dd_inv)
    iu = np.triu_indices(r.N)
    same_bits(r.M[iu], M[iu], f"{what}: Msys upper triangle")
    neg, zero = mm.hxs_counts(Hxs)
    assert zero == 0 and r.ret == p.neq + p.nineq + neg, (what, r.ret, neg, zero)
    dx, dyc, dyd = r.solve(identity=True)
    rhs = mm.pack(p, Hxs, p.rx, p.ryc, p.ryd)
    same_bits(np.concatenate([dx[p.nxs:], dyc, dyd]), rhs, f"{what}: packed rhs")
    dxo, _, _ = mm.unpack(p, Hxs, rhs, p.rx)
    same_bits(dx[:p.nxs], dxo[:p.nxs], f"{what}: unpacked dx_s")
    for f in ("rx", "ryc", "ryd"):                        # the device leaves the residuals alone (the reference overwrites ryd)
        same_bits(r.T[f].cpu().numpy(), getattr(p, f), f"{what}: {f} after the solve")
    return n_empty


def check_real_solve(r, what):
    """with the real factor: [dx_d; dyc; dyd] within the solve's backward error bound for the device's M and the model's rhs (factor read
    back), dx_s = the model's unpack of the device's own dense solution, bit for bit"""
    from test_gpu_symdense_paths import readback, factor_parts, theta
    p = r.p
    _, Hxs, _ = mm.diagonals(p)
    dx, dyc, dyd = r.solve(identity=False)
    sol = np.concatenate([dx[p.nxs:], dyc, dyd])
    dxo, _, _ = mm.unpack(p, Hxs, sol, p.rx)
    same_bits(dx[:p.nxs], dxo[:p.nxs], f"{what}: dx_s from the device's dense solution")
    rb = readback(r.k.linSys)
    L, d, dsub, perm = factor_parts(rb)
    A = np.triu(r.M) + np.triu(r.M, 1).T
    b = mm.pack(p, Hxs, p.rx, p.ryc, p.ryd)
    tn = lambda t: None if t is None else t.cpu().numpy()
    ratio, omega = bounds.solve_backward_ratio(A[perm][:, perm], sol[perm], b[perm], tn(L), tn(d), tn(dsub), theta(L))
    print(f"{what}: plan {rb['plan']}, solve margin {1 / max(ratio, 1e-300):.3g} (omega {omega:.2e})")
    assert ratio <= 1.0, (what, ratio)


# ---- the bench's sparse part ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bench_problem():
    """n_s = 500 000, m = 2 000 (neq = nineq = 1 000), 1 250 sorted distinct columns per row, with n_d = 2 000 (N = 4 000)"""
    return synth.make_mds_problem(500_000, 2000, 1000, 1000, nnz_per_row=1250, seed=42)


@pytest.mark.parametrize("safe", [True, False])
def test_bench_sparse_shape_bit_exact(ctx, bench_problem, safe):
    r = Run(ctx, bench_problem, safe).build()
    n_empty = check_exact(r, f"bench shape safe={safe}")
    print(f"bench shape: {n_empty} of {1000 * 2001} Schur pairs share no column (+0.0 in the reference)")
    assert n_empty > 0
    r.close()


# ---- sparsity edges --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,shape,edit", EDGES, ids=[e[0] for e in EDGES])
def test_edges_bit_exact(ctx, name, shape, edit):
    p = edge_problem(name, shape, edit)
    r = Run(ctx, p).build()
    check_exact(r, name)
    check_real_solve(r, name)
    r.close()


def test_empty_columns_give_rx_over_hxs(ctx):
    p = edge_problem(*EDGES[1])
    r = Run(ctx, p).build()
    dx, _, _ = r.solve(identity=False)
    _, Hxs, _ = mm.diagonals(p)
    empty = np.setdiff1d(np.arange(p.nxs), np.concatenate([p.jCol_c, p.jCol_d]))
    same_bits(dx[empty], p.rx[empty] / Hxs[empty], "dx_s on empty columns")
    r.close()


# ---- dispatch rows of the dense solver --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,safe", [(95, True), (96, True), (384, True), (385, True), (256, False), (257, False)])
def test_dispatch_rows(ctx, N, safe):
    neq = N // 5
    nineq = N // 4
    p = synth.make_mds_problem(3 * N, N - neq - nineq, neq, nineq, nnz_per_row=7, seed=N, dwx=1e-6, dcc=1e-8)
    r = Run(ctx, p, safe).build()
    assert r.ret == neq + nineq
    check_exact(r, f"N={N} safe={safe}")
    check_real_solve(r, f"N={N} safe={safe}")
    r.close()


# ---- Haynsworth counts ------------------------------------------------------------------------------------------------------------------
def _haynsworth_problem(seed):
    """no row touches columns 0..9, so whatever Hxs holds there (0, NaN, negative) leaves the dense M finite and its inertia alone"""
    p = synth.make_mds_problem(40, 10, 4, 5, seed=seed)
    r = np.random.default_rng(20)
    cols = [10 + r.choice(30, 4, replace=False) for _ in range(9)]
    return mm.with_pattern(p, cols[:4], cols[4:], seed=seed)


def _hxs_inertia(ctx, r):
    import ctypes
    from hiop_b200._lib import check
    a, b = ctypes.c_int(), ctypes.c_int()
    check(ctx.L.hb_mds_hxs_inertia(r.k.h, ctypes.byref(a), ctypes.byref(b)), "hb_mds_hxs_inertia")
    return a.value, b.value


def test_haynsworth_thresholds(ctx):
    p = _haynsworth_problem(21)
    t = 1e-14
    targets = [-t, t, np.nextafter(-t, -1.0), np.nextafter(-t, 0.0), np.nextafter(t, 0.0), np.nextafter(t, 1.0), 0.0, -0.0, np.nan, -3.0]
    p.ixl[:len(targets)] = 0.0                       # Dx = 0 there, so Hxs = (0 + 0) + Hs = Hs bit for bit (and -0.0 -> +0.0)
    p.ixu[:len(targets)] = 0.0
    p.Hs_diag[:len(targets)] = targets
    _, Hxs, _ = mm.diagonals(p)
    same_bits(Hxs[:8], np.array(targets[:8]) + 0.0, "Hxs at the thresholds")
    neg, zero = mm.hxs_counts(Hxs)
    # strict: -t is not < -t and t is not < t; below -t: its outward neighbour and -3; inside: the two inward neighbours, 0.0, -0.0
    assert (neg, zero) == (2, 4), (neg, zero)
    r = Run(ctx, p).build()
    assert _hxs_inertia(ctx, r) == (neg, zero)
    assert r.ret == -1                               # a null eigenvalue of Hxs, while the dense factor is fine:
    assert r.k.linSys.matrixChanged() == p.neq + p.nineq
    # negative entries only: their count is added to the dense factor's
    q = _haynsworth_problem(22)
    q.ixl[:3] = q.ixu[:3] = 0.0                      # Dx = 0 there: Hxs = Hs
    q.Hs_diag[:3] = -5.0
    assert mm.hxs_counts(mm.diagonals(q)[1]) == (3, 0)
    r.build(q)
    assert _hxs_inertia(ctx, r) == (3, 0) and r.ret == q.neq + q.nineq + 3
    # no negative entries on the same handle: the counters are reset per build
    r.build(_haynsworth_problem(23))
    assert _hxs_inertia(ctx, r) == (0, 0) and r.ret == 4 + 5
    r.close()


# ---- handle reuse -------------------------------------------------------------------------------------------------------------------
def test_handle_reuse_gives_fresh_bits(ctx):
    def prob(nnz, seed):
        return synth.make_mds_problem(500, 40, 20, 30, nnz_per_row=nnz, seed=seed, dwx=1e-5, dcc=1e-7)
    A1, B, A2 = prob(4, 31), prob(40, 32), prob(4, 33)
    A2 = mm.with_pattern(A2, [A1.jCol_c[A1.iRow_c == i] for i in range(20)], [A1.jCol_d[A1.iRow_d == i] for i in range(30)], seed=34)

    def outputs(r):
        return [r.M[np.triu_indices(r.N)], np.array([r.ret])] + list(r.solve(identity=False)) + list(r.solve(identity=True))
    fresh = []
    for q in (A1, B, A2):
        f = Run(ctx, q).build()
        fresh.append(outputs(f))
        f.close()
    r = Run(ctx, A1).build()
    for q, ref in zip((A1, B, A2), fresh):
        if q is not A1:
            r.k.set_sparsity(q.iRow_c, q.jCol_c, q.iRow_d, q.jCol_d)
            r.build(q)
        for a, b in zip(outputs(r), ref):
            same_bits(a, b, "reused handle")
    r.close()
