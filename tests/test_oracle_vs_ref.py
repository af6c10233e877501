"""Pins the numpy/C restatement (oracle/kkt_oracle.py) against the UNMODIFIED reference (oracle/_ref).
Runs only where oracle/_ref was built (this container); the same tuples are frozen in tests/golden for the GPU box."""
import numpy as np
import pytest

from hiop_b200 import synth
from oracle import kkt_oracle as ko
from oracle import ref

pytestmark = pytest.mark.ref


def _ref_system(p):
    q = ref.RefQn(p.n, p.m_eq, p.m_ineq, max(p.l, 1), p.ixl, p.ixu, p.idl, p.idu)
    q.set_iterate(p.sxl, p.sxu, p.zl, p.zu, p.sdl, p.sdu, p.vl, p.vu)
    q.set_jac(p.Jc, p.Jd)
    q.set_secant(p.sigma, p.St, p.Yt, p.L, p.D)
    return q


def _oracle_state(p):
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(p.zl, p.sxl, p.zu, p.sxu, p.ixl, p.ixu, p.vl, p.sdl, p.vu, p.sdu, p.idl,
                                          p.idu, p.sigma)
    return Dx, ko.QnState(p.Jc, p.Jd, DhInv, Dd_inv, p.St, p.Yt, p.L, p.D, p.sigma)


@pytest.mark.parametrize("n,m,l,mz", [(500, 4, 6, False), (2000, 50, 6, True), (1000, 1, 3, False),
                                       (3000, 64, 0, False), (777, 33, 2, True)])
def test_qn_system_matches_reference(n, m, l, mz):
    p = synth.make_qn_problem(n, m, l, masked_zero_divisors=mz)
    q = _ref_system(p)
    Dx_r, DhInv_r, Ddinv_r = q.update()
    Dx, st = _oracle_state(p)
    np.testing.assert_array_equal(Dx, Dx_r)
    np.testing.assert_array_equal(st.DhInv, DhInv_r)
    np.testing.assert_array_equal(st.Dd_inv, Ddinv_r)
    N_r = q.condense()
    N, W0, S1, Y1 = ko.condense(st)
    scale = np.abs(N_r).max()
    assert np.abs(N - N_r).max() <= 1e-12 * scale
    hs_r = q.hess_solve(p.rx)
    hs = ko.hess_solve(st, p.rx)
    assert np.abs(hs - hs_r).max() <= 1e-11 * np.abs(hs_r).max()
    dx_r, dyc_r, dyd_r = q.solve_compressed(p.rx, p.ryc, p.ryd)
    dx, dyc, dyd, _ = ko.solve_compressed(st, p.rx, p.ryc, p.ryd)
    for a, b in ((dx, dx_r), (dyc, dyc_r), (dyd, dyd_r)):
        if b.size:
            assert np.abs(a - b).max() <= 1e-8 * max(1.0, np.abs(b).max())
    q.close()


def test_compute_directions_matches_reference():
    p = synth.make_qn_problem(1500, 20, 4, masked_zero_divisors=True)
    q = _ref_system(p)
    q.update()
    _, st = _oracle_state(p)
    d_r = q.compute_directions(p.res)
    it = dict(sxl=p.sxl, sxu=p.sxu, zl=p.zl, zu=p.zu, sdl=p.sdl, sdu=p.sdu, vl=p.vl, vu=p.vu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    d = ko.compute_directions(st, it, pat, p.res)
    for k in ko.DIR_NAMES:
        assert np.all(np.isfinite(d_r[k])), k
        assert np.abs(d[k] - d_r[k]).max() <= 1e-8 * max(1.0, np.abs(d_r[k]).max()), k
    q.close()


def test_kkt_full_operator_matches_reference():
    """hiopMatVecKKTFullOpr::times_vec on a random 12-block vector."""
    p = synth.make_qn_problem(700, 12, 4, masked_zero_divisors=True)
    q = _ref_system(p)
    Dx_r, _, _ = q.update()
    _, st = _oracle_state(p)
    rng = np.random.default_rng(17)
    x = {k: rng.standard_normal(np.asarray(p.res[rk]).size) for k, rk in zip(ko.DIR_NAMES, ko.RES_NAMES)}
    it = dict(sxl=p.sxl, sxu=p.sxu, zl=p.zl, zu=p.zu, sdl=p.sdl, sdu=p.sdu, vl=p.vl, vu=p.vu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    y_r = q.kkt_full_times_vec(x)
    y = ko.kkt_full_times_vec(st, it, pat, x, Dx_r)
    for k in ko.RES_NAMES:
        tol = 1e-12 if k in ("rx", "ryc", "ryd") else 0.0          # elementwise rows are bit-identical
        assert np.abs(y[k] - y_r[k]).max(initial=0.0) <= tol * max(1.0, np.abs(y_r[k]).max(initial=0.0)), k
    q.close()


@pytest.mark.parametrize("mu,maxit", [(1e-1, 8), (1e-6, 8), (1e-3, 2), (1.0, 0)])
def test_compute_directions_w_ir_matches_reference(mu, maxit):
    """hiopKKTLinSys::compute_directions_w_IR: BiCGStab on the full KKT system, preconditioned by computeDirections."""
    p = synth.make_qn_problem(1200, 16, 4, masked_zero_divisors=True)
    q = _ref_system(p)
    Dx_r, _, _ = q.update()
    _, st = _oracle_state(p)
    it = dict(sxl=p.sxl, sxu=p.sxu, zl=p.zl, zu=p.zu, sdl=p.sdl, sdu=p.sdu, vl=p.vl, vu=p.vu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    d_r, info_r = q.compute_directions_w_ir(p.res, mu, maxit)
    d, info = ko.compute_directions_w_ir(st, it, pat, p.res, mu, maxit, Dx=Dx_r)
    if maxit > 0:
        assert info[0] == info_r[0] and info[1] == info_r[1], (info, info_r)     # same exit flag, same (half-)iteration count
    for k in ko.DIR_NAMES:
        assert np.all(np.isfinite(d_r[k])), k
        assert np.abs(d[k] - d_r[k]).max(initial=0.0) <= 1e-8 * max(1.0, np.abs(d_r[k]).max(initial=0.0)), k
    # the defining property: the returned direction solves the unreduced system to the BiCGStab tolerance
    if maxit > 0 and info_r[0] == 0:
        y = ko.kkt_full_times_vec(st, it, pat, d, Dx_r)
        rr = np.concatenate([y[k] - np.asarray(p.res[k]) for k in ko.RES_NAMES])
        bb = np.concatenate([np.asarray(p.res[k]) for k in ko.RES_NAMES])
        assert np.linalg.norm(rr) <= min(mu * 1e-2, 1e-6) * np.linalg.norm(bb) * 1.01
    q.close()


@pytest.mark.parametrize("case", ["good_prec", "rough_prec", "no_prec_budget", "singular", "zero_rhs"])
def test_bicgstab_recurrence_matches_reference(case):
    """hiopBiCGStabSolver::solve on dense systems that need several iterations / hit the non-convergence exits."""
    rng = np.random.default_rng(21)
    n = 60
    A = rng.standard_normal((n, n)) + 8.0 * np.eye(n)
    b = rng.standard_normal(n)
    tol, maxit = 1e-10, 40
    if case == "good_prec":
        Minv = np.linalg.inv(A + 1e-3 * rng.standard_normal((n, n)))
    elif case == "rough_prec":
        Minv = np.linalg.inv(A + 0.15 * rng.standard_normal((n, n)))   # ~10 iterations; beyond that BiCGStab trajectories are rounding-chaotic
    elif case == "no_prec_budget":
        Minv, maxit = np.eye(n), 5                 # runs out of iterations -> minimal-residual fallback
    elif case == "singular":
        A = np.outer(rng.standard_normal(n), rng.standard_normal(n))   # rank 1: breakdown / stagnation exits
        Minv = np.eye(n)
    else:
        Minv, b = np.eye(n), np.zeros(n)
    x_r, info_r = ref.bicgstab_dense(A, Minv, b, tol, maxit)
    x, flag, it, a, rel = ko.bicgstab(lambda v: A @ v, lambda v: Minv @ v, b, tol, maxit)
    assert flag == info_r[0] and it == info_r[1], ((flag, it, a, rel), info_r)
    assert np.abs(x - x_r).max(initial=0.0) <= 1e-7 * max(1.0, np.abs(x_r).max(initial=0.0))
    assert abs(a - info_r[2]) <= 1e-3 * abs(info_r[2]) + 1e-13     # residual norms: same digits up to rounding amplification


@pytest.mark.parametrize("strategy", [1, 2, 3, 4, 5])
def test_secant_update_matches_reference(strategy):
    """hiopHessianLowRank::update over a sequence: first call, appends, shifts (l_max = 3), both skip rules, all sigma rules."""
    n, me, mi, lmax = 300, 4, 3, 3
    seq = synth.make_secant_sequence(n, me, mi, steps=8)
    ones = np.ones(n)
    q = ref.RefQn(n, me, mi, lmax, ones, np.zeros(n), np.ones(mi), np.zeros(mi))
    q.set_sigma_strategy(strategy, 1.0)
    mem = ko.SecantMemory(n, lmax, 1.0, strategy)
    statuses = []
    for it in seq:
        l, St, Yt, L, D, sigma = q.hess_update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"])
        statuses.append(mem.update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"]))
        assert mem.St.shape[0] == l
        np.testing.assert_array_equal(mem.St, St)                       # s = x - x_prev: one rounding, same bits
        assert np.abs(mem.Yt - Yt).max(initial=0.0) <= 1e-13 * max(1.0, np.abs(Yt).max(initial=0.0))
        assert np.abs(np.tril(mem.L, -1) - np.tril(L, -1)).max(initial=0.0) <= 1e-12
        assert np.abs(mem.D - D).max(initial=0.0) <= 1e-12
        assert abs(mem.sigma - sigma) <= 1e-12 * sigma
    assert statuses == [0, 1, 1, 2, 1, 3, 1, 1], statuses
    q.close()


@pytest.mark.parametrize("form", [0, 1])
@pytest.mark.parametrize("nx,neq,nineq,dw,dc", [(40, 6, 9, 0.0, 0.0), (25, 10, 4, 1e-4, 1e-8), (12, 0, 5, 1e-3, 1e-6), (9, 3, 0, 0.0, 0.0)])
def test_dense_newton_kkt_matrix_matches_reference(form, nx, neq, nineq, dw, dc):
    """hiopKKTLinSysDenseXYcYd / XDYcYd::build_kkt_matrix incl. non-zero regularisations (delta_cd lands on the first dual
    rows in the reference: reproduced)."""
    p = synth.make_mds_problem(0, nx, neq, nineq, seed=7 + nx, dwx=dw, dcc=dc)
    it = dict(zl=p.zl, sxl=p.sxl, zu=p.zu, sxu=p.sxu, vl=p.vl, sdl=p.sdl, vu=p.vu, sdu=p.sdu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    deltas = (p.delta_wx, p.delta_wd, p.delta_cc, p.delta_cd)
    M_r = ref.densekkt_build(form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas)
    M, _, _ = ko.dense_build_kkt_matrix(form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas)
    np.testing.assert_array_equal(_u64(M), _u64(M_r))          # same additions in the same order: bit-identical, lower triangle zero


@pytest.mark.parametrize("form", [0, 1])
def test_dense_newton_kkt_matrix_negative_zeros_match_reference(form):
    """-0.0 entries of H, Jc and Jd become +0.0 in the reference's Msys (`+=` into a zeroed matrix)"""
    from oracle import mds_model as mm
    p = mm.with_negative_zeros(synth.make_mds_problem(0, 25, 10, 4, seed=8, dwx=1e-4, dcc=1e-8), seed=9)
    it = dict(zl=p.zl, sxl=p.sxl, zu=p.zu, sxu=p.sxu, vl=p.vl, sdl=p.sdl, vu=p.vu, sdu=p.sdu)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    deltas = (p.delta_wx, p.delta_wd, p.delta_cc, p.delta_cd)
    M_r = ref.densekkt_build(form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas)
    M, _, _ = ko.dense_build_kkt_matrix(form, p.Hd, p.Jcd, p.Jdd, it, pat, deltas)
    np.testing.assert_array_equal(_u64(M), _u64(M_r))
    assert np.signbit(p.Jcd).any() and not np.signbit(M_r[M_r == 0.0]).any()


@pytest.mark.parametrize("n,m", [(800, 14), (300, 1), (500, 40)])
def test_lsq_duals_match_reference(n, m):
    """hiopDualsLsqUpdateLinsysRedDenseSymPD::do_lsq_update (initial / recalculated multipliers)."""
    p = synth.make_qn_problem(n, m, 0)
    q = _ref_system(p)
    g = np.random.default_rng(8).standard_normal(n)
    yc_r, yd_r = q.lsq_duals(g)
    yc, yd = ko.lsq_duals(p.Jc, p.Jd, g, p.zl, p.zu, p.vl, p.vu)
    for a, b in ((yc, yc_r), (yd, yd_r)):
        assert np.abs(a - b).max(initial=0.0) <= 1e-10 * max(1.0, np.abs(b).max(initial=0.0))
    q.close()


def test_iajaaa_writer_is_byte_identical_to_reference(tmp_path):
    """write_kkt dumps: the C-ABI writer against hiopCSR_IO (matrix + rhs + solution), then the reader round-trips it."""
    from hiop_b200 import iajaaa
    K = np.triu(synth.make_kkt_like(23, 9, seed=4))
    K[2, 5] = 0.0                       # structural zeros are skipped (|a| <= 1e-25)
    K[7, 7] = 1e-30
    rhs = np.random.default_rng(2).standard_normal(32)
    sol = np.random.default_rng(3).standard_normal(32) * 1e3
    f_ref = ref.write_iajaaa(tmp_path, 7, K, 23, 4, 5, rhs, sol)
    f_own = str(tmp_path / "own.iajaaa")
    iajaaa.write_system(f_own, K, 23, 4, 5, [(rhs, sol)])
    assert open(f_own, "rb").read() == open(f_ref, "rb").read()
    back = iajaaa.read_system(f_ref)
    assert (back["N"], back["nx"], back["meq"], back["mineq"]) == (32, 23, 4, 5)
    Kz = K.copy()
    Kz[np.abs(Kz) <= 1e-25] = 0.0
    assert np.abs(back["M"] - Kz).max() <= 1e-19 + 1e-15 * np.abs(Kz).max()          # "%.20f" text: absolute 1e-20 resolution
    assert np.abs(back["pairs"][0][0] - rhs).max() <= 1e-15 and np.abs(back["pairs"][0][1] - sol).max() <= 1e-12


@pytest.mark.parametrize("n,m,mz,mu,kd", [(900, 14, True, 0.1, 1e-5), (400, 1, False, 1e-4, 0.0), (300, 9, True, 1.0, 1e-5)])
def test_residual_update_matches_reference(n, m, mz, mu, kd):
    """hiopResidual::update: the 12 residual blocks bit for bit (elementwise), J^T y to 1e-13, all 11 norms."""
    p = synth.make_qn_problem(n, m, 0, masked_zero_divisors=mz)
    itr, dat = synth.make_iterate(p)
    q = _ref_system(p)
    r_r, n_r = q.residual_update(itr, dat["c"], dat["d"], dat["grad"], mu, kd, dat["xl"], dat["xu"], dat["dl"], dat["du"], dat["crhs"])
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    r, nm = ko.residual_update(itr, dat["c"], dat["d"], dat["grad"], p.Jc, p.Jd, mu, kd, pat, dat["xl"], dat["xu"], dat["dl"], dat["du"], dat["crhs"])
    for k in ko.RES_NAMES:
        if k == "rx":
            assert np.abs(r[k] - r_r[k]).max(initial=0.0) <= 1e-13 * max(1.0, np.abs(r_r[k]).max(initial=0.0)), k
        else:
            np.testing.assert_array_equal(r[k], r_r[k], err_msg=k)
    for k in ko.NORM_NAMES:
        assert abs(nm[k] - n_r[k]) <= 1e-12 * max(1.0, abs(n_r[k])), (k, nm[k], n_r[k])
    q.close()


@pytest.mark.parametrize("n,m,mz,mu,kd", [(900, 14, True, 0.1, 1e-5), (400, 1, False, 1e-4, 0.0)])
def test_logbar_and_fraction_to_bdry_match_reference(n, m, mz, mu, kd):
    """hiopLogBarProblem::updateWithNlpInfo and hiopIterate::fractionToTheBdry."""
    p = synth.make_qn_problem(n, m, 0, masked_zero_divisors=mz)
    itr, dat = synth.make_iterate(p)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    # slacks must be positive where the pattern is set (log): masked-out entries may be anything
    for s, ptn in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu")):
        itr[s] = np.where(pat[ptn] == 1.0, np.abs(itr[s]) + 1e-3, itr[s])
    q = _ref_system(p)
    fl_r, gx_r, gd_r = q.logbar_update(itr, 3.25, mu, kd, dat["grad"])
    fl, gx, gd = ko.logbar_update(itr, 3.25, mu, kd, dat["grad"], pat)
    assert abs(fl - fl_r) <= 1e-13 * max(1.0, abs(fl_r))
    np.testing.assert_array_equal(gx, gx_r)
    np.testing.assert_array_equal(gd, gd_r)
    rng = np.random.default_rng(12)
    direction = {k: rng.standard_normal(np.asarray(v).size) * np.where(np.asarray(v) != 0, 1.0, 0.0) for k, v in itr.items()}
    # adjustDuals_primalLogHessian: duals scattered over several decades so that every branch of the clamp is taken
    itr2 = dict(itr)
    for zk in ("zl", "zu", "vl", "vu"):
        itr2[zk] = itr[zk] * 10.0 ** rng.integers(-6, 7, size=np.asarray(itr[zk]).size)
    got = ko.iterate_adjust_duals(itr2, pat, mu, 1e10 if kd == 0.0 else 50.0)
    want = q.adjust_duals(itr2, mu, 1e10 if kd == 0.0 else 50.0)
    for a, b in zip(got, want):
        np.testing.assert_array_equal(a, b)
    ap_r, ad_r = q.fraction_to_bdry(itr, direction, 0.995)
    ap, ad = ko.iterate_fraction_to_bdry(itr, direction, 0.995, pat)
    assert ap == ap_r and ad == ad_r, ((ap, ad), (ap_r, ad_r))
    q.close()


@pytest.mark.parametrize("mu", [1e-2, 10.0])
def test_adjust_small_slacks_matches_reference(mu):
    """hiopIterate::adjust_small_slacks: slacks that collapsed to (or below) zero are pushed back; untouched when none is small."""
    p = synth.make_qn_problem(600, 12, 0, masked_zero_divisors=True)
    itr, dat = synth.make_iterate(p)
    pat = dict(ixl=p.ixl, ixu=p.ixu, idl=p.idl, idu=p.idu)
    rng = np.random.default_rng(4)
    q = _ref_system(p)
    for collapse in (True, False):
        trial = {k: np.array(v, dtype=np.float64) for k, v in itr.items()}
        for s_, ptn in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu")):
            trial[s_] = np.where(pat[ptn] == 1.0, np.abs(trial[s_]) + 1e-3, 0.0)
            if collapse:
                hit = (rng.random(trial[s_].size) < 0.2) & (pat[ptn] == 1.0)
                trial[s_] = np.where(hit, rng.choice([0.0, -1e-9, 1e-20, 3e-17], size=trial[s_].size), trial[s_])
        num_r, got_r = q.adjust_small_slacks(trial, itr, mu, dat["xl"], dat["xu"], dat["dl"], dat["du"])
        num = 0
        for (s_, ptn, bnd, dual), want in zip((("sxl", "ixl", "xl", "zl"), ("sxu", "ixu", "xu", "zu"), ("sdl", "idl", "dl", "vl"),
                                                ("sdu", "idu", "du", "vu")), got_r):
            new, k = ko.adjust_small_slack(trial[s_], dat[bnd], itr[dual], pat[ptn], mu)
            num += k
            np.testing.assert_array_equal(new, want, err_msg=s_)
        assert num == num_r and (num > 0) == collapse
    q.close()


def test_hess_times_vec_matches_reference():
    p = synth.make_qn_problem(900, 3, 5)
    q = _ref_system(p)
    Dx_r, _, _ = q.update()
    x = np.random.default_rng(3).standard_normal(p.n)
    y0 = np.random.default_rng(4).standard_normal(p.n)
    for add in (False, True):
        y_r = q.hess_times_vec(0.5, y0, 2.0, x, add)
        y = ko.hess_times_vec(p.St, p.Yt, p.sigma, Dx_r, 0.5, y0, 2.0, x, add)
        assert np.abs(y - y_r).max() <= 1e-10 * np.abs(y_r).max()
    q.close()


@pytest.mark.parametrize("nx,m", [(30, 10), (120, 37), (5, 0), (1, 1)])
def test_symdense_matches_reference(nx, m):
    K = synth.make_kkt_like(nx, m)
    rhs = np.random.default_rng(5).standard_normal(nx + m)
    ret_r, sol_r, _, _ = ref.symdense_factor_solve(np.triu(K), rhs)
    ret, f = ko.symdense_matrix_changed(np.triu(K))
    assert ret == ret_r == m
    sol = f.solve(rhs)
    assert np.abs(sol - sol_r).max() <= 1e-9 * np.abs(sol_r).max()
    assert np.abs(K @ sol - rhs).max() <= 1e-9 * np.abs(rhs).max()


def test_symdense_singular_matches_reference():
    K = synth.make_kkt_like(20, 6)
    K[3, :] = 0.0
    K[:, 3] = 0.0
    ret_r, _, _, _ = ref.symdense_factor_solve(np.triu(K))
    ret, _ = ko.symdense_matrix_changed(np.triu(K))
    assert ret == ret_r == -1


def test_vector_ops_match_reference():
    r = np.random.default_rng(9)
    n = 1000
    y, x = r.standard_normal(n), r.standard_normal(n)
    z = r.uniform(0.5, 2.0, n)
    sel = (r.random(n) < 0.6).astype(np.float64)
    z0 = z * sel  # zero divisors on masked-out lanes
    for alpha in (1.0, -1.0, 0.37):
        yr, _ = ref.vec_op("axdzpy_w_pattern", y, x, z0, sel, alpha)
        np.testing.assert_array_equal(ko.axdzpy_w_pattern(y.copy(), alpha, x, z0, sel), yr)
        yr, _ = ref.vec_op("axzpy", y, x, z, None, alpha)
        np.testing.assert_array_equal(ko.axzpy(y.copy(), alpha, x, z), yr)
    yr, _ = ref.vec_op("component_div_w_sel", y, z0, None, sel)
    np.testing.assert_array_equal(ko.component_div_w_select(y.copy(), z0, sel), yr)
    yr, _ = ref.vec_op("add_logbar_grad", y, z0, None, sel, 0.1)
    np.testing.assert_array_equal(ko.add_log_barrier_grad(y.copy(), 0.1, z0, sel), yr)
    _, lb = ref.vec_op("logbarrier", z, None, None, sel)
    assert lb == ko.log_barrier(z, sel)
    ixu = (r.random(n) < 0.3).astype(np.float64)
    _, ld = ref.vec_op("lin_damping_term", z, sel, ixu, None, 0.1, 1e-5)
    assert ld == ko.linear_damping_term(z, sel, ixu, 0.1, 1e-5)
    yr, _ = ref.vec_op("add_lin_damping", y, sel, ixu, None, 0.9, 1e-6)
    np.testing.assert_array_equal(ko.add_linear_damping_term(y.copy(), sel, ixu, 0.9, 1e-6), yr)
    _, fb = ref.vec_op("frac_to_bdry_w_sel", z, x, None, sel, 0.995)
    assert fb == ko.fraction_to_the_bdry(z, x, 0.995, sel)
    _, fb = ref.vec_op("frac_to_bdry", z, x, None, None, 0.995)
    assert fb == ko.fraction_to_the_bdry(z, x, 0.995)


def test_mds_assembly_ops_match_reference():
    r = np.random.default_rng(21)
    Nw, m, n = 40, 7, 12
    A = r.standard_normal((m, n))
    W = r.standard_normal((Nw, Nw))
    Wr = W.copy()
    ref.lib().ref_mat_trans_add_to_sym_upper(m, n, A.ctypes.data_as(ref.dp), 3, 20, 0.7, Nw, Wr.ctypes.data_as(ref.dp))
    np.testing.assert_array_equal(ko.trans_add_to_sym_upper(A, 3, 20, 0.7, W.copy()), Wr)
    H = r.standard_normal((n, n))
    Wr = W.copy()
    ref.lib().ref_mat_add_upper_to_sym_upper(n, H.ctypes.data_as(ref.dp), 5, -1.3, Nw, Wr.ctypes.data_as(ref.dp))
    np.testing.assert_array_equal(ko.add_upper_to_sym_upper(H, 5, -1.3, W.copy()), Wr)
    # sparse Schur terms: sorted triplets, ~4 nnz per row
    ms, ns = 9, 30
    rows, cols = [], []
    for i in range(ms):
        cs = np.sort(r.choice(ns, 4, replace=False))
        rows += [i] * 4
        cols += list(cs)
    iR, jC = np.array(rows, dtype=np.int32), np.array(cols, dtype=np.int32)
    vals = r.standard_normal(iR.size)
    D = r.uniform(0.5, 2.0, ns)
    Wr = W.copy()
    ref.lib().ref_sp_add_MDinvMtrans(ms, ns, iR.size, iR.ctypes.data_as(ref.ip), jC.ctypes.data_as(ref.ip),
                                     vals.ctypes.data_as(ref.dp), 11, -1.0, D.ctypes.data_as(ref.dp), Nw,
                                     Wr.ctypes.data_as(ref.dp))
    Wo = ko.sp_add_MDinvMtrans(ms, ns, iR, jC, vals, 11, -1.0, D, W.copy())
    assert np.abs(Wo - Wr).max() <= 1e-13 * np.abs(Wr).max()


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _mds_build_with_reference_methods(p):
    """(ko's M, the reference's W, Dx, Hxs, Dd_inv): W from the reference's own matrix methods called in the order of
    hiopKKTLinSysCompressedMDSXYcYd::build_kkt_matrix (src/Optimization/hiopKKTLinSysMDS.cpp:196-290) on a zeroed matrix."""
    M, Dx, Hxs, Dd_inv = ko.mds_build_kkt_matrix(p)
    L, dp, ip = ref.lib(), ref.dp, ref.ip
    N = p.nxd + p.neq + p.nineq
    W = np.zeros((N, N))
    wp = W.ctypes.data_as(dp)

    def D(a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        return a, a.ctypes.data_as(dp)

    def I(a):
        a = np.ascontiguousarray(a, dtype=np.int32)
        return a, a.ctypes.data_as(ip)
    Dx_r, _ = ref.vec_op("axdzpy_w_pattern", np.zeros(p.nxs + p.nxd), p.zl, p.sxl, p.ixl, 1.0)
    Dx_r, _ = ref.vec_op("axdzpy_w_pattern", Dx_r, p.zu, p.sxu, p.ixu, 1.0)
    np.testing.assert_array_equal(Dx, Dx_r)
    a, pa = D(p.Hd); L.ref_mat_add_upper_to_sym_upper(p.nxd, pa, 0, 1.0, N, wp)
    a, pa = D(p.Jcd); L.ref_mat_trans_add_to_sym_upper(p.neq, p.nxd, pa, 0, p.nxd, 1.0, N, wp)
    a, pa = D(p.Jdd); L.ref_mat_trans_add_to_sym_upper(p.nineq, p.nxd, pa, 0, p.nxd + p.neq, 1.0, N, wp)
    a, pa = D(Dx[p.nxs:]); L.ref_mat_add_sub_diagonal(N, wp, 0, 1.0, p.nxd, pa)
    a, pa = D(p.delta_wx[p.nxs:]); L.ref_mat_add_sub_diagonal(N, wp, 0, 1.0, p.nxd, pa)
    hx, phx = D(Hxs)
    ic, pic = I(p.iRow_c); jc, pjc = I(p.jCol_c); vc, pvc = D(p.Jcs_vals)
    idd, pid = I(p.iRow_d); jd, pjd = I(p.jCol_d); vd, pvd = D(p.Jds_vals)
    L.ref_sp_add_MDinvMtrans(p.neq, p.nxs, ic.size, pic, pjc, pvc, p.nxd, -1.0, phx, N, wp)
    a, pa = D(p.delta_cc); L.ref_mat_add_sub_diagonal(N, wp, p.nxd, -1.0, p.neq, pa)
    L.ref_sp_add_MDinvMtrans(p.nineq, p.nxs, idd.size, pid, pjd, pvd, p.nxd + p.neq, -1.0, phx, N, wp)
    L.ref_sp_add_MDinvNtrans(p.neq, p.nxs, ic.size, pic, pjc, pvc, p.nineq, idd.size, pid, pjd, pvd, p.nxd, p.nxd + p.neq, -1.0, phx, N, wp)
    a, pa = D(Dd_inv); L.ref_mat_add_sub_diagonal(N, wp, p.nxd + p.neq, -1.0, p.nineq, pa)
    a, pa = D(p.delta_cd); L.ref_mat_add_sub_diagonal(N, wp, p.nxd + p.neq, -1.0, p.nineq, pa)
    return M, W, Dx, Hxs, Dd_inv


def test_mds_negative_zero_inputs_match_reference_methods():
    """-0.0 in Hd, Jcd, Jdd and the sparse values, empty sparse rows and pairs of rows that share no column: the reference's `+=` into
    a zeroed Msys stores +0.0 for all of them, and ko.mds_build_kkt_matrix must have the same bits."""
    from oracle import mds_model as mm
    p = mm.with_negative_zeros(synth.make_mds_problem(60, 25, 9, 14, dwx=1e-4, dcc=1e-6), seed=3)
    r = np.random.default_rng(4)
    cols = lambda i: [] if i % 3 == 0 else r.choice(60, 3, replace=False)
    mm.with_pattern(p, [cols(i) for i in range(9)], [cols(i + 1) for i in range(14)], seed=5)
    p.Jcs_vals[::4] = -0.0
    M, W, *_ = _mds_build_with_reference_methods(p)
    np.testing.assert_array_equal(_u64(M), _u64(W))
    assert (W == 0.0).sum() > W.size // 2 and not np.signbit(W[W == 0.0]).any()


def test_mds_sparse_mat_vecs_match_reference():
    """ko.mds_pack / ko.mds_unpack's triplet loops against hiopMatrixSparseTriplet::timesVec / transTimesVec (beta = 1, alpha = -1)"""
    if not ref.has_sp_times_vec():
        pytest.skip("oracle/_ref was built before ref_sp_times_vec existed: rebuild it with `make -C oracle ref`")
    n = 300
    p = synth.make_mds_problem(n, 5, 20, 30, nnz_per_row=40, seed=6)
    r = np.random.default_rng(7)
    for iR, jC, v, m in ((p.iRow_c, p.jCol_c, p.Jcs_vals, 20), (p.iRow_d, p.jCol_d, p.Jds_vals, 30)):
        for trans, ny, nx in ((0, m, n), (1, n, m)):
            x, y = r.standard_normal(nx), r.standard_normal(ny)
            y_r = ref.sp_times_vec(trans, m, n, iR, jC, v, y, -1.0, x)
            y_m = (ko.sp_trans_times_vec if trans else ko.sp_times_vec)(iR, jC, v, y.copy(), -1.0, x)
            np.testing.assert_array_equal(_u64(y_m), _u64(y_r))


def test_mds_build_kkt_matrix_matches_reference_methods():
    """ko.mds_build_kkt_matrix against the reference's own matrix methods called in the order of
    hiopKKTLinSysCompressedMDSXYcYd::build_kkt_matrix (src/Optimization/hiopKKTLinSysMDS.cpp:196-290)."""
    p = synth.make_mds_problem(60, 25, 9, 14, dwx=1e-4, dcc=1e-6)
    M, W, Dx, Hxs, Dd_inv = _mds_build_with_reference_methods(p)
    np.testing.assert_array_equal(_u64(M), _u64(W))
    # and the whole system is a valid KKT system: inertia (nxd, 0, neq+nineq) for the dense block
    ret_r, _, _, _ = ref.symdense_factor_solve(W)
    ret, f = ko.mds_factorize_with_curv_check(M, Hxs)
    assert ret == ret_r == p.neq + p.nineq
    dx, dyc, dyd = ko.mds_solve_compressed(p, f, Hxs, p.rx, p.ryc, p.ryd)
    # residual of the full (unreduced) XYcYd system
    import scipy.sparse as sp
    Jc = np.hstack([sp.csr_matrix((p.Jcs_vals, (p.iRow_c, p.jCol_c)), shape=(p.neq, p.nxs)).toarray(), p.Jcd])
    Jd = np.hstack([sp.csr_matrix((p.Jds_vals, (p.iRow_d, p.jCol_d)), shape=(p.nineq, p.nxs)).toarray(), p.Jdd])
    H = np.zeros((p.nxs + p.nxd, p.nxs + p.nxd))
    H[:p.nxs, :p.nxs] = np.diag(p.Hs_diag)
    H[p.nxs:, p.nxs:] = p.Hd
    H += np.diag(Dx + p.delta_wx)
    r1 = H @ dx + Jc.T @ dyc + Jd.T @ dyd - p.rx
    r2 = Jc @ dx - p.delta_cc * dyc - p.ryc
    r3 = Jd @ dx - (Dd_inv + p.delta_cd) * dyd - p.ryd
    assert max(np.abs(r1).max(), np.abs(r2).max(), np.abs(r3).max()) <= 1e-9
