"""GPU parity tests: the CUDA path (through the C-ABI) against (1) the golden fixtures produced by the unmodified
reference, (2) the oracle on seeded inputs at sizes it finishes in seconds, (3) size-independent properties
(KKT residual of the solution computed with independent operators) at larger sizes.

Tolerances (north_star: 1e-8 relative on the KKT residual; elementwise kernels are bit-exact where the operation
order is the reference's):  elementwise/diagonals: exact;  N: componentwise FP64 bound (2 gamma_K |J| DhInv |J|^T) without
secant memory, 1e-12 sqrt(N_ii N_jj) with it (oracle/bounds.py);  directions: 1e-8 relative."""
import glob
import os

import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _relerr(a, b):
    return float(np.abs(a - b).max() / max(1.0, np.abs(b).max())) if b.size else 0.0


def _setup_kkt(ctx, p, l_max=None):
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, p["n"], p["m_eq"], p["m_ineq"], l_max if l_max is not None else max(int(p["l"]), 1))
    T = {}
    J = np.vstack([p["Jc"], p["Jd"]])
    T["J"] = ctx.to_device(J)
    T["Jc"], T["Jd"] = T["J"][:p["m_eq"]], T["J"][p["m_eq"]:]
    for key in ("ixl", "ixu", "idl", "idu", "sxl", "sxu", "zl", "zu", "sdl", "sdu", "vl", "vu", "St", "Yt"):
        T[key] = ctx.to_device(p[key])
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["Jc"], T["Jd"])
    l = int(p["l"])
    k.set_secant(float(p["sigma"]), T["St"] if l else None, T["Yt"] if l else None, p["L"], p["D"])
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    return k, T


def _as_dict(p: synth.QnProblem):
    d = {k: getattr(p, k) for k in ("n", "m_eq", "m_ineq", "l", "sigma", "Jc", "Jd", "ixl", "ixu", "idl", "idu", "sxl", "sxu", "zl", "zu",
                                    "sdl", "sdu", "vl", "vu", "St", "Yt", "L", "D", "rx", "ryc", "ryd")}
    for kk, v in p.res.items():
        d["res_" + kk] = v
    return d


def _run_solve(ctx, k, p):
    rx = ctx.to_device(p["rx"])
    ryc, ryd = ctx.to_device(p["ryc"]), ctx.to_device(p["ryd"])
    dx, dyc, dyd = ctx.zeros(p["n"]), ctx.zeros(p["m_eq"]), ctx.zeros(p["m_ineq"])
    assert k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
    ctx.sync()
    return dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy()


def _run_dirs(ctx, k, p):
    res = {kk: ctx.to_device(p["res_" + kk]) for kk in ko.RES_NAMES}
    sizes = dict(x=p["n"], d=p["m_ineq"], yc=p["m_eq"], yd=p["m_ineq"], sxl=p["n"], sxu=p["n"], sdl=p["m_ineq"], sdu=p["m_ineq"],
                 zl=p["n"], zu=p["n"], vl=p["m_ineq"], vu=p["m_ineq"])
    dirs = {kk: ctx.zeros(int(sizes[kk])) for kk in ko.DIR_NAMES}
    assert k.computeDirections(res, dirs)
    ctx.sync()
    return {kk: v.cpu().numpy() for kk, v in dirs.items()}


# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(os.path.basename(f) for f in glob.glob(os.path.join(GOLD, "qn_*.npz"))))
def test_qn_against_reference_golden(ctx, name):
    g = dict(np.load(os.path.join(GOLD, name)))
    g = {kk: (v if v.ndim else v.item()) for kk, v in g.items()}
    k, T = _setup_kkt(ctx, g)
    np.testing.assert_array_equal(k.Dx(), g["ref_Dx"])
    np.testing.assert_array_equal(k.DhInv(), g["ref_DhInv"])
    np.testing.assert_array_equal(k.Dd_inv(), g["ref_Dd_inv"])
    k.condense()
    N = k.N()
    J = np.vstack([g["Jc"], g["Jd"]])
    assert bounds.condensed_error_ratio(N, g["ref_N"], J, g["ref_DhInv"], int(g["l"]), _num_sms()) <= 1.0
    assert np.array_equal(N, N.T)
    rhs = ctx.to_device(g["rx"])
    x = ctx.zeros(g["n"])
    k.hess_solve(rhs, x)
    ctx.sync()
    assert _relerr(x.cpu().numpy(), g["ref_hess_solve"]) <= 1e-11
    dx, dyc, dyd = _run_solve(ctx, k, g)
    assert _relerr(dx, g["ref_dx"]) <= 1e-8 and _relerr(dyc, g["ref_dyc"]) <= 1e-8 and _relerr(dyd, g["ref_dyd"]) <= 1e-8
    d = _run_dirs(ctx, k, g)
    for kk in ko.DIR_NAMES:
        assert _relerr(d[kk], g["ref_dir_" + kk]) <= 1e-8, kk
    # compact-form B*x equals the reference's recursive timesVec
    xx, y = ctx.to_device(g["tv_x"]), ctx.zeros(g["n"])
    k.hess_times_vec(0.0, y, 1.0, xx, True)
    ctx.sync()
    assert _relerr(y.cpu().numpy(), g["ref_Bx"]) <= 1e-10
    k.close()


@pytest.mark.parametrize("n,m,l,mz", [
    (20000, 130, 6, True),     # crosses a 128-row tile boundary (m+2l = 142)
    (4099, 37, 3, False),      # odd n: rows are not 16-byte aligned -> 8-byte cp.async path, K tail
    (10000, 1, 6, True),       # NlpDenseConsEx1 shape
    (6000, 260, 0, False),     # empty secant memory, 3x3 tile grid
    (2500, 0, 4, False),       # unconstrained
    (17, 5, 2, True),          # tiny: single partial K chunk
])
def test_qn_against_oracle(ctx, n, m, l, mz):
    P = synth.make_qn_problem(n, m, l, masked_zero_divisors=mz, seed=4321 + n)
    p = _as_dict(P)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    k, T = _setup_kkt(ctx, p)
    np.testing.assert_array_equal(k.Dx(), Dx)
    np.testing.assert_array_equal(k.DhInv(), DhInv)
    if m:
        k.condense()
        No, _, _, _ = ko.condense(st)
        assert bounds.condensed_error_ratio(k.N(), No, st.J, DhInv, l, _num_sms()) <= 1.0
    dxo, dyco, dydo, _ = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    dx, dyc, dyd = _run_solve(ctx, k, p)
    assert _relerr(dx, dxo) <= 1e-8 and _relerr(dyc, dyco) <= 1e-8 and _relerr(dyd, dydo) <= 1e-8
    it = dict(sxl=P.sxl, sxu=P.sxu, zl=P.zl, zu=P.zu, sdl=P.sdl, sdu=P.sdu, vl=P.vl, vu=P.vu)
    pat = dict(ixl=P.ixl, ixu=P.ixu, idl=P.idl, idu=P.idu)
    do = ko.compute_directions(st, it, pat, P.res)
    d = _run_dirs(ctx, k, p)
    for kk in ko.DIR_NAMES:
        assert np.all(np.isfinite(d[kk])), kk
        assert _relerr(d[kk], do[kk]) <= 1e-8, kk
    k.close()


def _kkt_residual(ctx, k, T, p, dx, dyc, dyd):
    """Relative residual of the 3-block compressed KKT system evaluated with operators that are independent of the
    solve path (compact-form B*x, public gemv entry points)."""
    n, meq, mi = p["n"], p["m_eq"], p["m_ineq"]
    dxd, dycd, dydd = ctx.to_device(dx), ctx.to_device(dyc), ctx.to_device(dyd)
    r1 = ctx.to_device(p["rx"])
    r1.mul_(-1.0)
    k.hess_times_vec(1.0, r1, 1.0, dxd, True)                 # (B + Dx) dx - rx
    if meq:
        ctx.mat_trans_times_vec(T["Jc"], 1.0, r1, 1.0, dycd)
    if mi:
        ctx.mat_trans_times_vec(T["Jd"], 1.0, r1, 1.0, dydd)
    out = [ctx.vec_infnorm(r1)]
    if meq:
        r2 = ctx.to_device(p["ryc"])
        ctx.mat_times_vec(T["Jc"], -1.0, r2, 1.0, dxd)         # Jc dx - ryc
        out.append(ctx.vec_infnorm(r2))
    if mi:
        r3 = ctx.to_device(p["ryd"])
        ctx.mat_times_vec(T["Jd"], -1.0, r3, 1.0, dxd)         # Jd dx - ryd - Dd_inv*dyd
        ctx.vec_axzpy(r3, -1.0, ctx.to_device(k.Dd_inv()), dydd)
        out.append(ctx.vec_infnorm(r3))
    scale = max(np.abs(p["rx"]).max(), np.abs(p["ryc"]).max() if meq else 0.0, np.abs(p["ryd"]).max() if mi else 0.0)
    return max(out) / scale


def test_kkt_residual_property_medium(ctx):
    """n = 2e5, m = 512: beyond what the oracle's triple loop does in seconds -> check the defining property."""
    P = synth.make_qn_problem(200000, 512, 6, seed=99)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    dx, dyc, dyd = _run_solve(ctx, k, p)
    nref, resid = k.last_solve_stats()
    assert resid < 1e-8
    assert _kkt_residual(ctx, k, T, p, dx, dyc, dyd) <= 1e-8
    k.close()


def test_kkt_system_host_matches_device_path(ctx):
    P = synth.make_qn_problem(3000, 24, 4, seed=5)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    dx, dyc, dyd = _run_solve(ctx, k, p)
    it = {kk: np.ascontiguousarray(p[kk]) for kk in ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")}
    hx, hyc, hyd = np.zeros(P.n), np.zeros(P.m_eq), np.zeros(P.m_ineq)
    k.kkt_system_host(np.ascontiguousarray(P.Jc), np.ascontiguousarray(P.Jd), it, P.rx.copy(), P.ryc.copy(), P.ryd.copy(), hx, hyc, hyd)
    np.testing.assert_array_equal(hx, dx)
    np.testing.assert_array_equal(hyc, dyc)
    np.testing.assert_array_equal(hyd, dyd)
    k.close()


def test_kkt_system_host_chunked_overlapped_path(ctx):
    """Large J: the host entry point uploads J in column chunks on a second stream and condenses chunk by chunk (FP64 DMMA).
    Same answer as the device-resident path (summation order differs), identical from call to call."""
    P = synth.make_qn_problem(48000, 700, 6, seed=6)             # 269 MB of J -> above the 256 MB chunking threshold
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    k.set_condense_mode(0)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    dx, dyc, dyd = _run_solve(ctx, k, p)
    it = {kk: np.ascontiguousarray(p[kk]) for kk in ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")}
    outs = []
    for rep in range(2):
        hx, hyc, hyd = np.zeros(P.n), np.zeros(P.m_eq), np.zeros(P.m_ineq)
        k.kkt_system_host(np.ascontiguousarray(P.Jc), np.ascontiguousarray(P.Jd), it, P.rx.copy(), P.ryc.copy(), P.ryd.copy(), hx, hyc, hyd)
        outs.append((hx, hyc, hyd))
    for a, b in zip(outs[0], outs[1]):
        np.testing.assert_array_equal(a, b)
    assert _relerr(outs[0][0], dx) <= 1e-9 and _relerr(outs[0][1], dyc) <= 1e-9 and _relerr(outs[0][2], dyd) <= 1e-9
    assert k.condense_mode_used() == 0
    k.close()


def test_condense_is_bit_reproducible(ctx):
    P = synth.make_qn_problem(50000, 200, 6, seed=8)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    k.condense()
    N1 = k.N().copy()
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    k.condense()
    np.testing.assert_array_equal(N1, k.N())
    k.close()


# ----------------------------------------------------------------------------------------------------------------
def test_vector_ops_against_reference_golden(ctx):
    g = dict(np.load(os.path.join(GOLD, "vector_ops.npz")))
    y, x, z, sel, ixu = g["y"], g["x"], g["z"], g["sel"], g["ixu"]
    z0 = z * sel
    D = ctx.to_device

    def run(fn, y0, *a):
        t = D(y0)
        fn(t, *a)
        ctx.sync()
        return t.cpu().numpy()
    for alpha in (1.0, -1.0, 0.37):
        np.testing.assert_array_equal(run(ctx.vec_axdzpy_w_pattern, y, alpha, D(x), D(z0), D(sel)), g[f"axdzpy_w_pattern_{alpha}"])
        np.testing.assert_array_equal(run(ctx.vec_axzpy, y, alpha, D(x), D(z)), g[f"axzpy_{alpha}"])
        np.testing.assert_array_equal(run(ctx.vec_axdzpy, y, alpha, D(x), D(z)), g[f"axdzpy_{alpha}"])
    np.testing.assert_array_equal(run(ctx.vec_component_div_w_pattern, y, D(z0), D(sel)), g["component_div_w_sel"])
    np.testing.assert_array_equal(run(ctx.vec_component_mult, y, D(x)), g["component_mult"])
    np.testing.assert_array_equal(run(ctx.vec_component_div, y, D(z)), g["component_div"])
    np.testing.assert_array_equal(run(ctx.vec_invert, z), g["invert"])
    np.testing.assert_array_equal(run(ctx.vec_select_pattern, y, D(sel)), g["select_pattern"])
    np.testing.assert_array_equal(run(ctx.vec_add_constant, y, 0.25), g["add_constant"])
    np.testing.assert_array_equal(run(ctx.vec_add_constant_w_pattern, y, 0.25, D(sel)), g["add_constant_w_sel"])
    np.testing.assert_array_equal(run(ctx.vec_add_log_barrier_grad, y, 0.1, D(z0), D(sel)), g["add_logbar_grad"])
    np.testing.assert_array_equal(run(ctx.vec_add_linear_damping_term, y, D(sel), D(ixu), 0.9, 1e-6), g["add_lin_damping"])
    tol = 1e-13
    assert abs(ctx.vec_twonorm(D(y)) - g["twonorm"]) <= tol * g["twonorm"]
    assert abs(ctx.vec_dot(D(y), D(x)) - g["dot"]) <= tol * np.abs(y * x).sum()
    assert ctx.vec_infnorm(D(y)) == g["infnorm"]
    assert abs(ctx.vec_onenorm(D(y)) - g["onenorm"]) <= tol * g["onenorm"]
    assert abs(ctx.vec_log_barrier(D(z), D(sel)) - g["logbarrier"]) <= tol * np.abs(np.log(z) * sel).sum()
    assert abs(ctx.vec_linear_damping_term(D(z), D(sel), D(ixu), 0.1, 1e-5) - g["lin_damping_term"]) <= tol * abs(g["lin_damping_term"])
    assert ctx.vec_min_w_pattern(D(y), D(sel)) == g["min_w_pattern"]
    assert ctx.vec_fraction_to_bdry(D(z), D(x), 0.995) == g["frac_to_bdry"]
    assert ctx.vec_fraction_to_bdry(D(z), D(x), 0.995, D(sel)) == g["frac_to_bdry_w_sel"]


def test_vector_ops_ragged_and_empty(ctx):
    r = np.random.default_rng(2)
    for n in (0, 1, 2, 3, 255, 257, 100003):
        y, x = r.standard_normal(n), r.standard_normal(n)
        z = r.uniform(0.5, 2, n)
        sel = (r.random(n) < 0.5).astype(np.float64)
        t = ctx.to_device(y)
        ctx.vec_axdzpy_w_pattern(t, 0.5, ctx.to_device(x), ctx.to_device(z * sel), ctx.to_device(sel))
        ctx.sync()
        np.testing.assert_array_equal(t.cpu().numpy(), ko.axdzpy_w_pattern(y.copy(), 0.5, x, z * sel, sel))
        assert ctx.vec_infnorm(ctx.to_device(y)) == (np.abs(y).max() if n else 0.0)
        assert abs(ctx.vec_dot(ctx.to_device(y), ctx.to_device(x)) - float(y @ x)) <= 1e-12 * max(1.0, np.abs(y * x).sum())
        assert ctx.vec_fraction_to_bdry(ctx.to_device(z), ctx.to_device(x), 0.99) == ko.fraction_to_the_bdry(z, x, 0.99)
    # unaligned views (odd offset) exercise the scalar path
    y = r.standard_normal(1001)
    t = ctx.to_device(y)
    ctx.vec_scale(t[1:], 2.0)
    ctx.sync()
    np.testing.assert_array_equal(t.cpu().numpy()[1:], y[1:] * 2.0)


def test_gemv_against_oracle(ctx):
    r = np.random.default_rng(3)
    for m, n in ((7, 5000), (33, 4097), (1, 1), (130, 2049)):
        A, x, y = r.standard_normal((m, n)), r.standard_normal(n), r.standard_normal(m)
        yt = ctx.to_device(y)
        ctx.mat_times_vec(ctx.to_device(A), 0.5, yt, -2.0, ctx.to_device(x))
        ctx.sync()
        ref = ko.times_vec(A, 0.5, y.copy(), -2.0, x)
        assert np.abs(yt.cpu().numpy() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
        xt = ctx.to_device(x)
        ctx.mat_trans_times_vec(ctx.to_device(A), 1.0, xt, -1.0, ctx.to_device(y))
        ctx.sync()
        ref = ko.trans_times_vec(A, 1.0, x.copy(), -1.0, y)
        assert np.abs(xt.cpu().numpy() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


# ----------------------------------------------------------------------------------------------------------------
def _symdense_check(ctx, K, mode, expect_ret, rhs):
    from hiop_b200.engine import LinSolverSymDense
    N = K.shape[0]
    s = LinSolverSymDense(ctx, N, mode)
    s.set_matrix(ctx.to_device(np.triu(K) + np.tril(np.full((N, N), np.nan), -1)))  # lower part must never be read
    ret = s.matrixChanged()
    assert ret == expect_ret, (ret, expect_ret)
    if ret >= 0 and N:
        x = ctx.to_device(rhs)
        assert s.solve(x)
        ctx.sync()
        xs = x.cpu().numpy()
        Kf = np.triu(K) + np.triu(K, 1).T
        assert np.abs(Kf @ xs - rhs).max() <= 1e-9 * max(1.0, np.abs(rhs).max()) * max(1.0, np.linalg.cond(Kf) * 1e-3)
        return xs
    s.close()
    return None


def test_symdense_against_reference_golden(ctx):
    from hiop_b200.engine import LinSolverSymDense
    g = dict(np.load(os.path.join(GOLD, "symdense.npz")))
    for i in range(int(g["count"])):
        K, rhs, ret, sol = g[f"K{i}"], g[f"rhs{i}"], int(g[f"ret{i}"]), g[f"sol{i}"]
        xs = _symdense_check(ctx, K, LinSolverSymDense.BUNCH_KAUFMAN, ret, rhs)
        if ret >= 0:
            assert _relerr(xs, sol) <= 1e-8, i


@pytest.mark.parametrize("nx,m", [(150, 60), (400, 111), (63, 1), (64, 64), (700, 333)])
def test_symdense_blocked_bk_inertia_and_solve(ctx, nx, m):
    from hiop_b200.engine import LinSolverSymDense
    K = synth.make_kkt_like(nx, m, seed=nx + m)
    rhs = np.random.default_rng(1).standard_normal(nx + m)
    reto, f = ko.symdense_matrix_changed(np.triu(K))
    assert reto == m
    xs = _symdense_check(ctx, K, LinSolverSymDense.BUNCH_KAUFMAN, m, rhs)
    assert _relerr(xs, f.solve(rhs)) <= 1e-8
    # quasi-definite: LDL^T without pivoting is stable and must report the same inertia (magma nopiv mode)
    xs2 = _symdense_check(ctx, K, LinSolverSymDense.NOPIV, m, rhs)
    assert _relerr(xs2, xs) <= 1e-7


def test_symdense_general_indefinite_needs_pivoting(ctx):
    from hiop_b200.engine import LinSolverSymDense
    for N, nneg in ((300, 120), (129, 64)):
        M = synth.make_symmetric_indefinite(N, nneg, seed=N)
        M[np.diag_indices(N)] *= 1e-6   # tiny diagonal: forces 2x2 pivots
        ev = np.linalg.eigvalsh(M)
        rhs = np.random.default_rng(2).standard_normal(N)
        _symdense_check(ctx, M, LinSolverSymDense.BUNCH_KAUFMAN, int((ev < 0).sum()), rhs)


def test_symdense_cholesky_and_singular(ctx):
    from hiop_b200.engine import LinSolverSymDense
    r = np.random.default_rng(4)
    for N in (1, 5, 64, 65, 300):
        A = r.standard_normal((N, N))
        S = A @ A.T + N * np.eye(N)
        _symdense_check(ctx, S, LinSolverSymDense.CHOLESKY, 0, r.standard_normal(N))
    S = -np.eye(10)
    assert _symdense_check(ctx, S, LinSolverSymDense.CHOLESKY, -1, np.ones(10)) is None
    K = synth.make_kkt_like(20, 6, seed=3)
    K[3, :] = 0.0
    K[:, 3] = 0.0
    assert _symdense_check(ctx, K, LinSolverSymDense.BUNCH_KAUFMAN, -1, np.ones(26)) is None
    assert _symdense_check(ctx, np.zeros((0, 0)), LinSolverSymDense.BUNCH_KAUFMAN, 0, np.zeros(0)) is None
