"""Dense-Newton KKT classes on the device (SURVEY 8 a16): hiopKKTLinSysDenseXYcYd / hiopKKTLinSysDenseXDYcYd
(src/Optimization/hiopKKTLinSysDense.hpp) -- assembly bit-identical to the reference's golden matrix, inertia and solution
against the reference's LAPACK result, and against the oracle on seeded shapes incl. neq = 0 / nineq = 0."""
import os

import numpy as np
import pytest

from hiop_b200 import synth
from oracle import kkt_oracle as ko
from test_gpu_parity import ctx  # noqa: F401

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _run(ctx, form, H, Jc, Jd, it, pat, deltas, rhs):
    from hiop_b200.engine import KKTLinSysDense
    nx, neq, nineq = H.shape[0], Jc.shape[0], Jd.shape[0]
    D = ctx.to_device
    k = KKTLinSysDense(ctx, nx, neq, nineq, "XYcYd" if form == 0 else "XDYcYd")
    k.build_kkt_matrix(D(H), D(Jc), D(Jd), {kk: D(v) for kk, v in it.items()}, {kk: D(v) for kk, v in pat.items()}, [D(d) for d in deltas])
    M = k.Msys()
    ret = k.factorize()
    o = [0, nx, nx + (nineq if form else 0), nx + (nineq if form else 0) + neq, k.N]
    rx, ryc, ryd = D(rhs[:nx]), D(rhs[o[2]:o[3]]), D(rhs[o[3]:])
    rd = D(rhs[nx:o[2]]) if form else ctx.zeros(0)
    dx, dd, dyc, dyd = ctx.zeros(nx), ctx.zeros(nineq if form else 0), ctx.zeros(neq), ctx.zeros(nineq)
    ok = k.solveCompressed(rx, rd, ryc, ryd, dx, dd, dyc, dyd)
    ctx.sync()
    sol = np.concatenate([dx.cpu().numpy(), dd.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy()])
    k.close()
    return M, ret, ok, sol


@pytest.mark.parametrize("form", [0, 1])
def test_dense_kkt_against_reference_golden(ctx, form):
    g = dict(np.load(os.path.join(GOLD, "densekkt_nx30.npz")))
    it = {kk: g[kk] for kk in ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")}
    pat = {kk: g[kk] for kk in ("ixl", "ixu", "idl", "idu")}
    M, ret, ok, sol = _run(ctx, form, g["H"], g["Jc"], g["Jd"], it, pat, (g["dwx"], g["dwd"], g["dcc"], g["dcd"]), g[f"rhs{form}"])
    np.testing.assert_array_equal(M.view(np.uint64), g[f"ref_M{form}"].view(np.uint64))
    assert ret == int(g[f"ref_ret{form}"]) and ok
    assert np.abs(sol - g[f"ref_sol{form}"]).max() <= 1e-9 * np.abs(g[f"ref_sol{form}"]).max()


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("nx,neq,nineq,dw,dc", [(200, 40, 60, 0.0, 0.0), (97, 33, 5, 1e-4, 1e-8), (64, 0, 20, 1e-3, 1e-6), (50, 12, 0, 0.0, 0.0)])
def test_dense_kkt_against_oracle(ctx, form, nx, neq, nineq, dw, dc):
    p = synth.make_mds_problem(0, nx, neq, nineq, seed=3 + nx, dwx=dw, dcc=dc)
    it = dict(zl=p.zl, sxl=p.sxl, zu=p.zu, sxu=p.sxu, vl=p.vl, sdl=p.sdl, vu=p.vu, sdu=p.sdu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    deltas = (p.delta_wx, p.delta_wd, p.delta_cc, p.delta_cd)
    Mo, _, _ = ko.dense_build_kkt_matrix(form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas)
    rhs = np.random.default_rng(nx).standard_normal(Mo.shape[0])
    M, ret, ok, sol = _run(ctx, form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas, rhs)
    np.testing.assert_array_equal(M.view(np.uint64), Mo.view(np.uint64))
    ret_o, f = ko.symdense_matrix_changed(Mo)
    assert ret == ret_o == neq + nineq and ok         # inertia the Newton driver requires (hiopAlgFilterIPM.cpp:2084-2096)
    K = np.triu(Mo) + np.triu(Mo, 1).T
    assert np.abs(K @ sol - rhs).max() <= 1e-9 * max(1.0, np.abs(rhs).max())
    assert np.abs(sol - f.solve(rhs)).max() <= 1e-8 * max(1.0, np.abs(sol).max())


def test_write_kkt_from_device(ctx, tmp_path):
    """hb_iajaaa_write_matrix / append_vector download from the device and write the reference's interchange format."""
    import ctypes
    from hiop_b200 import iajaaa
    from hiop_b200.engine import KKTLinSysDense, check
    p = synth.make_mds_problem(0, 40, 6, 9, seed=77)
    it = dict(zl=p.zl, sxl=p.sxl, zu=p.zu, sxu=p.sxu, vl=p.vl, sdl=p.sdl, vu=p.vu, sdu=p.sdu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    D = ctx.to_device
    k = KKTLinSysDense(ctx, 40, 6, 9, "XYcYd")
    k.build_kkt_matrix(D(p.Hd), D(p.Jcd), D(p.Jdd), {kk: D(v) for kk, v in it.items()}, {kk: D(v) for kk, v in pat.items()},
                       [D(d) for d in (p.delta_wx, p.delta_wd, p.delta_cc, p.delta_cd)])
    M = k.Msys()
    f = str(tmp_path / "kkt_linsys_0.iajaaa").encode()
    check(ctx.L.hb_iajaaa_write_matrix(ctx.h, f, k.N, ctypes.c_void_p(k.linSys._mptr), 40, 6, 9), "write")
    rhs = D(np.arange(k.N, dtype=np.float64))
    check(ctx.L.hb_iajaaa_append_vector(ctx.h, f, k.N, ctypes.c_void_p(rhs.data_ptr())), "append")
    check(ctx.L.hb_iajaaa_append_vector(ctx.h, f, k.N, ctypes.c_void_p(rhs.data_ptr())), "append")
    back = iajaaa.read_system(f.decode())
    assert np.abs(back["M"] - np.triu(M)).max() <= 1e-19 + 1e-15 * np.abs(M).max()
    assert np.array_equal(back["pairs"][0][0], np.arange(k.N, dtype=np.float64))
    k.close()


def _dominant_problem(nx, neq, nineq, seed, frac):
    """H diagonally dominant (so any off-diagonal entry may be zeroed), about frac of H's off-diagonal pairs and of Jc, Jd set to -0.0"""
    r = np.random.default_rng(seed)
    p = synth.make_mds_problem(0, nx, neq, nineq, seed=seed, dwx=1e-4, dcc=1e-8)
    H = 0.01 * r.standard_normal((nx, nx)) / np.sqrt(nx)
    H = H + H.T + np.diag(r.uniform(1.0, 2.0, nx))
    Z = np.triu(r.random((nx, nx)) < frac, 1)
    H[Z | Z.T] = -0.0
    Jc, Jd = p.Jcd.copy(), p.Jdd.copy()
    Jc[r.random(Jc.shape) < frac] = -0.0
    Jd[r.random(Jd.shape) < frac] = -0.0
    it = dict(zl=p.zl, sxl=p.sxl, zu=p.zu, sxu=p.sxu, vl=p.vl, sdl=p.sdl, vu=p.vu, sdu=p.sdu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    return H, Jc, Jd, it, pat, (p.delta_wx, p.delta_wd, p.delta_cc, p.delta_cd)


@pytest.mark.parametrize("form", [0, 1])
def test_dense_kkt_negative_zero_inputs(ctx, form):
    """-0.0 in H, Jc and Jd: the reference's `+=` into a zeroed Msys stores +0.0, and so must the device"""
    H, Jc, Jd, it, pat, deltas = _dominant_problem(80, 20, 25, 41, 0.2)
    Mo, _, _ = ko.dense_build_kkt_matrix(form, H, Jc, Jd, it, pat, deltas)
    rhs = np.random.default_rng(42).standard_normal(Mo.shape[0])
    M, ret, ok, _ = _run(ctx, form, H, Jc, Jd, it, pat, deltas, rhs)
    bad = np.nonzero(M.view(np.uint64) != Mo.view(np.uint64))
    assert bad[0].size == 0, f"{bad[0].size} entries differ, first {[(i, j, M[i, j], Mo[i, j]) for i, j in zip(*bad)][:4]}"
    assert np.signbit(Jc).any() and not np.signbit(Mo[Mo == 0.0]).any()
    assert ret == 20 + 25 and ok


def test_dense_kkt_cluster_bunch_kaufman_order(ctx):
    """XDYcYd at N = 600 + 100 + 2 * 150 = 1000, past the cluster Bunch-Kaufman threshold: bit-identical assembly, the inertia, and the
    solve within its backward error bound for the factor read back"""
    from oracle import bounds
    from dense_handles import readback, factor_parts, theta
    from hiop_b200.engine import KKTLinSysDense
    H, Jc, Jd, it, pat, deltas = _dominant_problem(600, 100, 150, 43, 0.05)
    Mo, _, _ = ko.dense_build_kkt_matrix(1, H, Jc, Jd, it, pat, deltas)
    N = Mo.shape[0]
    rhs = np.random.default_rng(44).standard_normal(N)
    D = ctx.to_device
    k = KKTLinSysDense(ctx, 600, 100, 150, "XDYcYd")
    k.build_kkt_matrix(D(H), D(Jc), D(Jd), {kk: D(v) for kk, v in it.items()}, {kk: D(v) for kk, v in pat.items()}, [D(d) for d in deltas])
    M = k.Msys()
    np.testing.assert_array_equal(M.view(np.uint64), Mo.view(np.uint64))
    assert k.factorize() == 100 + 150
    rb = readback(k.linSys)
    assert rb["plan"][0] == "BK_CLUSTER", rb["plan"]
    x = D(rhs)
    assert k.linSys.solve(x)
    ctx.sync()
    sol = x.cpu().numpy()
    k.close()
    L, d, dsub, perm = factor_parts(rb)
    tn = lambda t: None if t is None else t.cpu().numpy()
    A = np.triu(Mo) + np.triu(Mo, 1).T
    ratio, omega = bounds.solve_backward_ratio(A[perm][:, perm], sol[perm], rhs[perm], tn(L), tn(d), tn(dsub), theta(L))
    print(f"dense KKT N={N}: plan {rb['plan']}, solve margin {1 / max(ratio, 1e-300):.3g} (omega {omega:.2e})")
    assert ratio <= 1.0
