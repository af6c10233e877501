"""Streaming kernels past the launch-grid clamp, and the Jacobian gemvs on every launch-geometry branch.

hb_grid caps a streaming launch at 8 CTAs of 256 threads per SM (270,336 threads on 132 SMs), so every grid-stride loop only takes its
second trip beyond 2048 G items (G = SM count), i.e. beyond 4096 G doubles on the double2 path. The sizes below are derived from G:
4096 G + 1 (odd: the double2 kernel k_ew2 covers its 2048 G pairs in exactly one trip and the last double goes to k_ew1, while the
reductions and the scalar path take a second trip), 8192 G (two full k_ew2 trips) and 8192 G + 1. A view offset by one double takes the
scalar k_ew1 path.

Elementwise ops whose kernels round every operation explicitly are bit-exact against the oracle's restatements; reductions and gemvs
are held to gamma_c * sum|terms| around exact references (oracle/bounds.py), with c the longest serial addition chain of the kernel,
derived from its launch geometry next to each check.

The x side of the quasi-Newton handle runs at n = 8192 G + 1 through update, hess_solve, hess_times_vec, residual_update,
fraction_to_bdry, take_step, logbar, adjust_duals_plh, adjust_small_slacks, kkt_full_times_vec, test_direction, secant_update and the LSQ
multipliers.

Not covered: the d side past the clamp (m_ineq > 2048 G). hb_lowrank_create allocates N and its factor as m x m, which at that size is
more than 580 GB."""
import ctypes

import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko

pytestmark = pytest.mark.gpu
U = bounds.U


def _G():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes():
    G = _G()
    return [4096 * G + 1, 8192 * G, 8192 * G + 1]


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _p(t):
    q = ctypes.c_void_p(t.data_ptr())
    q._keep = t
    return q


@pytest.fixture(scope="module", params=[0, 1, 2], ids=["4096G+1", "8192G", "8192G+1"])
def vecs(request):
    n = _sizes()[request.param]
    r = np.random.default_rng(n)
    sel = (r.random(n) < 0.5).astype(np.float64)
    ixu = (r.random(n) < 0.3).astype(np.float64)
    return dict(n=n, y=r.standard_normal(n), x=r.standard_normal(n), z=r.uniform(0.5, 2.0, n), sel=sel, ixu=ixu)


def _run(ctx, fn, y0, *a, offset=0):
    buf = ctx.to_device(np.concatenate([np.zeros(offset), y0]))
    t = buf[offset:]
    fn(t, *a)
    ctx.sync()
    return t.cpu().numpy()


@pytest.mark.parametrize("offset", [0, 1], ids=["double2", "scalar"])
def test_elementwise_ops_bit_exact_past_the_clamp(ctx, vecs, offset):
    D = ctx.to_device
    y, x, z, sel, ixu = vecs["y"], vecs["x"], vecs["z"], vecs["sel"], vecs["ixu"]
    z0 = z * sel
    xd, zd, z0d, seld, ixud = D(x), D(z), D(z0), D(sel), D(ixu)
    eq = np.testing.assert_array_equal
    for alpha in (1.0, -1.0, 0.37):
        eq(_run(ctx, ctx.vec_axzpy, y, alpha, xd, zd, offset=offset), ko.axzpy(y.copy(), alpha, x, z))
        eq(_run(ctx, ctx.vec_axdzpy_w_pattern, y, alpha, xd, z0d, seld, offset=offset), ko.axdzpy_w_pattern(y.copy(), alpha, x, z0, sel))
    eq(_run(ctx, ctx.vec_axdzpy, y, 0.37, xd, zd, offset=offset), y + (x / z) * 0.37)
    eq(_run(ctx, ctx.vec_set, y, 0.25, offset=offset), np.full_like(y, 0.25))
    eq(_run(ctx, ctx.vec_scale, y, 0.37, offset=offset), y * 0.37)
    eq(_run(ctx, ctx.vec_component_mult, y, xd, offset=offset), y * x)
    eq(_run(ctx, ctx.vec_component_div, y, zd, offset=offset), y / z)
    eq(_run(ctx, ctx.vec_component_div_w_pattern, y, z0d, seld, offset=offset), ko.component_div_w_select(y.copy(), z0, sel))
    eq(_run(ctx, ctx.vec_invert, z, offset=offset), 1.0 / z)
    eq(_run(ctx, ctx.vec_select_pattern, y, seld, offset=offset), ko.select_pattern(y.copy(), sel))
    eq(_run(ctx, ctx.vec_add_constant, y, 0.25, offset=offset), y + 0.25)
    eq(_run(ctx, ctx.vec_add_constant_w_pattern, y, 0.25, seld, offset=offset), np.where(sel == 1.0, y + 0.25, y))
    eq(_run(ctx, ctx.vec_add_log_barrier_grad, y, 0.1, z0d, seld, offset=offset), ko.add_log_barrier_grad(y.copy(), 0.1, z0, sel))
    eq(_run(ctx, ctx.vec_add_linear_damping_term, y, seld, ixud, 0.9, 1e-6, offset=offset), ko.add_linear_damping_term(y.copy(), sel, ixu, 0.9, 1e-6))
    # y + alpha*x may be contracted to one fused multiply-add: either rounding of y + alpha x is within 2u (|y| + |alpha x|)
    got = _run(ctx, ctx.vec_axpy, y, -0.37, xd, offset=offset)
    assert np.all(np.abs(got - (y - 0.37 * x)) <= 2 * U * (np.abs(y) + np.abs(0.37 * x)))
    # every element was visited: a grid-stride loop that skipped the items past the clamp would leave y unchanged there
    assert not np.any(got[-1000:] == y[-1000:])


def test_reductions_against_exact_sums_past_the_clamp(ctx, vecs):
    D = ctx.to_device
    n, y, x, z, sel, ixu = vecs["n"], vecs["y"], vecs["x"], vecs["z"], vecs["sel"], vecs["ixu"]
    G = _G()
    g = bounds.stream_grid(n, G)
    c = bounds.reduction_chain(n, g)
    gam = bounds.gamma(c + 1)          # + 1: the product / square / log of each term
    yd, xd, zd, seld, ixud = D(y), D(x), D(z), D(sel), D(ixu)
    margins = {}

    def check(name, got, exact, tol):
        err = abs(got - exact)
        margins[name] = tol / max(err, 1e-300)
        assert err <= tol, (name, got, exact, err, tol)
    d1 = ctx.vec_dot(yd, xd)
    assert ctx.vec_dot(yd, xd) == d1                      # same bits on a second call
    check("dot", d1, bounds.exact_dot(y, x), gam * np.abs(y * x).sum())
    s2 = bounds.exact_dot(y, y)
    check("twonorm", ctx.vec_twonorm(yd), np.sqrt(s2), (gam + 2 * U) * np.sqrt(s2))
    check("onenorm", ctx.vec_onenorm(yd), bounds.exact_sum(np.abs(y)), gam * np.abs(y).sum())
    # log: at most 1 ulp on the device and in numpy, 2u |log z_i| each
    lg = np.log(z) * (sel != 0)
    check("log_barrier", ctx.vec_log_barrier(zd, seld), bounds.exact_sum(lg), (gam + 4 * U) * np.abs(lg).sum())
    ld = np.where((sel == 1.0) & (ixu == 0.0), z, 0.0)
    exact_ld = bounds.exact_sum(ld) * 0.1 * 1e-5
    check("linear_damping_term", ctx.vec_linear_damping_term(zd, seld, ixud, 0.1, 1e-5), exact_ld, (gam + 3 * U) * ld.sum() * 1e-6)
    assert ctx.vec_infnorm(yd) == np.abs(y).max()
    assert ctx.vec_min_w_pattern(yd, seld) == y[sel == 1.0].min()
    # the extreme entries at the very end, where only the last grid-stride trip reaches
    y2 = y.copy()
    y2[-1] = 50.0
    y2[-2] = -60.0
    assert ctx.vec_infnorm(D(y2)) == 60.0
    assert ctx.vec_min_w_pattern(D(y2), D(np.ones(n))) == -60.0
    assert ctx.vec_fraction_to_bdry(zd, xd, 0.995) == ko.fraction_to_the_bdry(z, x, 0.995)
    assert ctx.vec_fraction_to_bdry(zd, xd, 0.995, seld) == ko.fraction_to_the_bdry(z, x, 0.995, sel)
    print(f"n={n} (grid {g}, chain {c}): margins " + ", ".join(f"{k} {v:.3g}" for k, v in margins.items()))


# ---- Jacobian gemvs ------------------------------------------------------------------------------------------------------------
GR_CHUNK, ET = 2048, 256


def _rows_chain(n):
    """k_gemv_rows_partial: a lane adds 2 products per double2 over a GR_CHUNK / 64 trips, plus an odd tail, then a warp tree (5);
    k_gemv_rows_final: ceil(nchunks / 8) partials per chunk class, 8 classes in a row, then alpha t (1), beta y (1) and the sum (1),
    plus the product rounding (1)."""
    nchunks = -(-n // GR_CHUNK)
    return 2 * (GR_CHUNK // 64) + 1 + 5 + (-(-nchunks // 8)) + 8 + 4


def _cols_rg(m, n, G):
    """row groups of k_gemv_cols (gemv_cols in hb_lowrank.cu)"""
    ctas1 = -(-((n + 1) // 2) // ET)
    return 1 if (ctas1 >= 8 * G or m < 64) else (4 if ctas1 >= 2 * G else 8)


def _cols_chain(m, rg):
    """k_gemv_cols: ceil(m / RG) products per thread, RG group sums in a row, alpha, beta, the sum and the product rounding (4)"""
    return -(-m // rg) + rg + 4


def _matrix(ctx, r, m, n, lda, offset):
    """an m x n matrix with leading dimension lda, starting `offset` doubles into its buffer (offset 1: 8-byte aligned only)"""
    full = r.standard_normal((m, lda))
    full[:, n:] = np.nan                     # padding must never be read
    buf = ctx.to_device(np.concatenate([np.zeros(offset), full.ravel()]))
    return full[:, :n].copy(), buf[offset:]


def _vec(ctx, v, offset):
    buf = ctx.to_device(np.concatenate([np.zeros(offset), v]))
    return buf[offset:]


def _gemv_rows_cases():
    out = []
    for n in (2047, 2048, 2049):
        for i, m in enumerate((1, 63, 64, 130)):
            out.append((m, n, (0, 1, 2)[(i + n) % 3], (i + n) % 2))
    return out


@pytest.mark.parametrize("m,n,lda_extra,offset", _gemv_rows_cases() + [(8, "8192G+1", 1, 0), (5, "8192G+1", 0, 1)])
@pytest.mark.parametrize("beta", [0.0, 0.5])
def test_gemv_rows_componentwise(ctx, m, n, lda_extra, offset, beta):
    """y = beta y + alpha A x (hb_mat_times_vec -> gemv_rows): n around GR_CHUNK (one chunk: 8 row splits), and nchunks >= 4 G (one row
    split); lda in {n, n+1, n+2}, A 8-byte aligned only, beta = 0 over a y full of NaN."""
    G = _G()
    if isinstance(n, str):
        n = 8192 * G + 1
    r = np.random.default_rng(m * 7 + n)
    A, Ad = _matrix(ctx, r, m, n, n + lda_extra, offset)
    x = r.standard_normal(n)
    y0 = np.full(m, np.nan) if beta == 0.0 else r.standard_normal(m)
    alpha = -1.5
    yd = ctx.to_device(y0)
    xd = ctx.to_device(x)
    assert ctx.L.hb_mat_times_vec(ctx.h, m, n, _p(Ad), n + lda_extra, beta, _p(yd), alpha, _p(xd)) == 0
    ctx.sync()
    got = yd.cpu().numpy()
    Ax = bounds.exact_rows(A, x)
    ref = alpha * Ax + (beta * y0 if beta else 0.0)
    scale = abs(alpha) * (np.abs(A) @ np.abs(x)) + (abs(beta) * np.abs(y0) if beta else 0.0)
    tol = bounds.gamma(_rows_chain(n)) * scale + U * np.abs(ref)
    err = np.abs(got - ref)
    assert np.all(np.isfinite(got))
    assert np.all(err <= tol), float((err / tol).max())
    print(f"gemv_rows m={m} n={n} lda=n+{lda_extra} offset={offset} beta={beta}: margin {float((tol / np.maximum(err, 1e-300)).min()):.3g}")


def _gemv_cols_cases(G):
    """(m, n, lda_extra, A offset, y offset, expected row groups)"""
    return [
        (1024, 3001, 1, 0, 0, 8), (1025, 3001, 0, 0, 1, 8), (2049, 2050, 2, 1, 0, 8),    # second and third GC_ROWS staging pass
        (64, 1024 * G - 512, 0, 0, 0, 8), (64, 1024 * G, 0, 0, 0, 4),                     # ctas1 = 2G - 1 / 2G
        (64, 4096 * G - 512, 2, 0, 0, 4), (64, 4096 * G, 0, 0, 1, 1),                     # ctas1 = 8G - 1 / 8G
        (130, 1024 * G + 1, 1, 0, 0, 4), (63, 1024 * G - 511, 0, 1, 0, 1),                # odd n; m < 64 always one row group
    ]


@pytest.mark.parametrize("case", range(9))
@pytest.mark.parametrize("beta", [0.0, -0.5])
def test_gemv_cols_componentwise(ctx, case, beta):
    """y = beta y + alpha A^T x (hb_mat_trans_times_vec -> gemv_cols) on all three row-group variants, at both switch points, with
    more than GC_ROWS = 1024 rows, lda != n, a misaligned A or y, and beta = 0 over a y full of NaN."""
    G = _G()
    m, n, lda_extra, aoff, yoff, rg = _gemv_cols_cases(G)[case]
    assert _cols_rg(m, n, G) == rg
    r = np.random.default_rng(case)
    A, Ad = _matrix(ctx, r, m, n, n + lda_extra, aoff)
    x = r.standard_normal(m)
    y0 = np.full(n, np.nan) if beta == 0.0 else r.standard_normal(n)
    alpha = 0.75
    yd = _vec(ctx, y0, yoff)
    assert ctx.L.hb_mat_trans_times_vec(ctx.h, m, n, _p(Ad), n + lda_extra, beta, _p(yd), alpha, _p(ctx.to_device(x))) == 0
    ctx.sync()
    got = yd.cpu().numpy()
    Atx = bounds.exact_cols(A, x)
    absterms = np.abs(A).T @ np.abs(x)
    ref = alpha * Atx + (beta * y0 if beta else 0.0)
    scale = abs(alpha) * absterms + (abs(beta) * np.abs(y0) if beta else 0.0)
    tol = bounds.gamma(_cols_chain(m, rg)) * scale + abs(alpha) * bounds.cols_ref_error(m, Atx, absterms) + U * np.abs(ref)
    err = np.abs(got - ref)
    assert np.all(np.isfinite(got))
    assert np.all(err <= tol), float((err / tol).max())
    print(f"gemv_cols m={m} n={n} RG={rg} lda=n+{lda_extra} beta={beta}: margin {float((tol / np.maximum(err, 1e-300)).min()):.3g}")


# ---- the x side of the quasi-Newton handle past the clamp ------------------------------------------------------------------------
@pytest.mark.parametrize("l", [4, 5])
def test_lowrank_x_side_past_the_clamp(ctx, l):
    """n = 8192 G + 1, m = 8: update (Dx, DhInv bit-exact), hess_solve and hess_times_vec against the oracle. l = 4 / 5 put 2l = 8 / 10
    rows through k_multidot_partial, i.e. one or two MD_CH = 8 passes."""
    from hiop_b200.engine import KKTLinSysLowRank
    n = 8192 * _G() + 1
    P = synth.make_qn_problem(n, 8, l, seed=l)
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, l)
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ("ixl", "ixu", "idl", "idu", "zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu", "St", "Yt")}
    J = D(P.J)
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(J[:P.m_eq], J[P.m_eq:])
    k.set_secant(P.sigma, T["St"], T["Yt"], P.L, P.D)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    np.testing.assert_array_equal(k.Dx(), Dx)
    np.testing.assert_array_equal(k.DhInv(), DhInv)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    x = D(np.zeros(n))
    k.hess_solve(D(P.rx), x)
    ctx.sync()
    want = ko.hess_solve(st, P.rx)
    assert np.abs(x.cpu().numpy() - want).max() <= 1e-11 * max(1.0, np.abs(want).max())
    v = np.random.default_rng(l).standard_normal(n)
    y = D(np.full(n, np.nan))
    k.hess_times_vec(0.0, y, 1.0, D(v), True)
    ctx.sync()
    want = ko.hess_times_vec(P.St, P.Yt, P.sigma, Dx, 0.0, np.zeros(n), 1.0, v, True)
    got = y.cpu().numpy()
    assert np.all(np.isfinite(got))
    assert np.abs(got - want).max() <= 1e-10 * max(1.0, np.abs(want).max())
    k.close()


@pytest.fixture(scope="module")
def qn_big():
    """n = 8192 G + 1, m = 8, l = 0, with a full iterate around it (synth.make_iterate)"""
    P = synth.make_qn_problem(8192 * _G() + 1, 8, 0, masked_zero_divisors=True, seed=41)
    itr, dat = synth.make_iterate(P)
    pat = dict(ixl=P.ixl, ixu=P.ixu, idl=P.idl, idu=P.idu)
    return P, itr, dat, pat


def test_residual_update_past_the_clamp(ctx, qn_big):
    """hiopResidual::update (k_resid_block<true> on the x side): every block but rx bit-exact; rx (one J^T y sweep of m rows plus four
    elementwise terms on each side) within 2 gamma_{m+8} of its terms; infinity norms exact on the device's own blocks, one-norms within
    the chain bound of the block kernel + hb_reduce_slots. kappa_d = 0 keeps rx before the damping term equal to -rx."""
    from test_gpu_parity import _setup_kkt, _as_dict
    P, itr, dat, pat = qn_big
    n, mu = P.n, 0.1
    k, T = _setup_kkt(ctx, _as_dict(P))
    D = ctx.to_device
    it_d = {kk: D(np.ascontiguousarray(v)) for kk, v in itr.items()}
    res_d = {rk: ctx.zeros(np.asarray(itr[dk]).size) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    nm = k.residual_update(it_d, D(dat["c"]), D(dat["d"]), D(dat["grad"]), mu, 0.0, D(dat["xl"]), D(dat["xu"]), D(dat["dl"]), D(dat["du"]),
                           D(dat["crhs"]), res_d)
    ctx.sync()
    ro, no = ko.residual_update(itr, dat["c"], dat["d"], dat["grad"], P.Jc, P.Jd, mu, 0.0, pat, dat["xl"], dat["xu"], dat["dl"], dat["du"], dat["crhs"])
    r = {rk: res_d[rk].cpu().numpy() for rk in ko.RES_NAMES}
    for rk in ko.RES_NAMES:
        if rk != "rx":
            np.testing.assert_array_equal(r[rk], ro[rk], err_msg=rk)
    scale = np.abs(dat["grad"]) + np.abs(P.Jc).T @ np.abs(itr["yc"]) + np.abs(P.Jd).T @ np.abs(itr["yd"]) + np.abs(itr["zl"]) + np.abs(itr["zu"])
    assert np.all(np.abs(r["rx"] - ro["rx"]) <= 2 * bounds.gamma(P.m + 8) * scale)
    # infinity norms: maxima of the device's own blocks (exact); the rx part is the device's rx
    inf = lambda *vs: max(float(np.abs(v).max(initial=0.0)) for v in vs)   # noqa: E731
    assert nm["inf_nlp_optim"] == nm["inf_bar_optim"] == inf(r["rx"], r["rd"])
    assert nm["inf_nlp_feasib"] == nm["inf_bar_feasib"] == no["inf_nlp_feasib"]
    assert nm["inf_bar_complem"] == inf(r["rszl"], r["rszu"], r["rsvl"], r["rsvu"])
    for kk in ("inf_nlp_complem", "inf_cons_violation"):              # maxima of once-rounded products / differences
        assert abs(nm[kk] - no[kk]) <= 2 * U * abs(no[kk]), kk
    G = _G()
    gam = bounds.gamma(bounds.slots_chain(n, bounds.stream_grid(n, G)) + 2)   # + 2: the host adds the x and d parts
    for kk, blocks in (("one_nlp_optim", ("rx", "rd")), ("one_bar_optim", ("rx", "rd")), ("one_nlp_feasib", ("ryc", "ryd")), ("one_bar_feasib", ("ryc", "ryd"))):
        s = bounds.exact_sum(np.concatenate([np.abs(r[b]) for b in blocks]))
        assert abs(nm[kk] - s) <= gam * s, (kk, nm[kk], s)
    k.close()


def test_line_search_pipeline_past_the_clamp(ctx, qn_big):
    """fraction_to_bdry (exact), take_step (one multiply-add per entry), logbar (log sums within the chain bound, gradients bit-exact),
    adjust_duals_plh and adjust_small_slacks (bit-exact) at n = 8192 G + 1."""
    from test_gpu_parity import _setup_kkt, _as_dict
    P, itr, dat, pat = qn_big
    n, mu = P.n, 0.1
    itr = dict(itr)
    for s, ptn in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu")):
        itr[s] = np.where(pat[ptn] == 1.0, np.abs(itr[s]) + 1e-3, itr[s])
    rng = np.random.default_rng(5)
    direction = {kk: rng.standard_normal(np.asarray(v).size) * np.where(np.asarray(v) != 0, 1.0, 0.0) for kk, v in itr.items()}
    k, T = _setup_kkt(ctx, _as_dict(P))
    D = ctx.to_device
    it_d = {kk: D(np.ascontiguousarray(v)) for kk, v in itr.items()}
    dir_d = {kk: D(np.ascontiguousarray(v)) for kk, v in direction.items()}
    ap, ad = k.fraction_to_bdry(it_d, dir_d, 0.995)
    assert (ap, ad) == ko.iterate_fraction_to_bdry(itr, direction, 0.995, pat)
    out_d = {kk: ctx.zeros(np.asarray(v).size) for kk, v in itr.items()}
    k.take_step(it_d, dir_d, ap, ad, out_d)
    ctx.sync()
    for kk in ko.DIR_NAMES:
        if kk in ("sxl", "sxu", "sdl", "sdu"):
            continue                                 # slacks are recomputed from x, d by the driver
        al = ap if kk in ("x", "d", "yc", "yd") else ad
        y, dd = np.asarray(itr[kk]), direction[kk]
        got = out_d[kk].cpu().numpy()
        assert np.all(np.abs(got - (y + al * dd)) <= 2 * U * (np.abs(y) + np.abs(al * dd))), kk
    gx, gd = ctx.zeros(n), ctx.zeros(P.m_ineq)
    fl = k.logbar(it_d, 3.25, mu, 0.0, D(dat["grad"]), gx, gd)
    flo, gxo, gdo = ko.logbar_update(itr, 3.25, mu, 0.0, dat["grad"], pat)
    ctx.sync()
    np.testing.assert_array_equal(gx.cpu().numpy(), gxo)
    np.testing.assert_array_equal(gd.cpu().numpy(), gdo)
    logs = np.concatenate([np.log(itr[s][pat[p] == 1.0]) for s, p in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu"))])
    exact = 3.25 - mu * bounds.exact_sum(logs)
    c = bounds.slots_chain(n, bounds.stream_grid(n, _G())) + 8           # + the host's sum of the four blocks, the scaling and f
    assert abs(fl - exact) <= (bounds.gamma(c) + 4 * U) * (3.25 + mu * np.abs(logs).sum()), (fl, exact)
    itr2 = dict(itr)
    for zk in ("zl", "zu", "vl", "vu"):
        itr2[zk] = itr[zk] * 10.0 ** rng.integers(-6, 7, size=np.asarray(itr[zk]).size)
    it2_d = {kk: D(np.ascontiguousarray(v)) for kk, v in itr2.items()}
    k.adjust_duals_plh(it2_d, mu, 50.0)
    ctx.sync()
    for name, want in zip(("zl", "zu", "vl", "vu"), ko.iterate_adjust_duals(itr2, pat, mu, 50.0)):
        np.testing.assert_array_equal(it2_d[name].cpu().numpy(), want, err_msg=name)
    trial = {kk: np.array(v, dtype=np.float64) for kk, v in itr.items()}
    for s_, ptn in (("sxl", "ixl"), ("sxu", "ixu"), ("sdl", "idl"), ("sdu", "idu")):
        hit = (rng.random(trial[s_].size) < 0.2) & (pat[ptn] == 1.0)
        trial[s_] = np.where(hit, rng.choice([0.0, -1e-9, 1e-20, 3e-17], size=trial[s_].size), np.where(pat[ptn] == 1.0, trial[s_], 0.0))
    hit_last = trial["sxl"].copy()
    tr_d = {kk: D(np.ascontiguousarray(v)) for kk, v in trial.items()}
    num = k.adjust_small_slacks(tr_d, it_d, mu, *[D(dat[b]) for b in ("xl", "xu", "dl", "du")])
    ctx.sync()
    want_num = 0
    for s_, ptn, bnd, dual in (("sxl", "ixl", "xl", "zl"), ("sxu", "ixu", "xu", "zu"), ("sdl", "idl", "dl", "vl"), ("sdu", "idu", "du", "vu")):
        new, cnt = ko.adjust_small_slack(trial[s_], dat[bnd], itr[dual], pat[ptn], mu)
        want_num += cnt
        np.testing.assert_array_equal(tr_d[s_].cpu().numpy(), new, err_msg=s_)
    assert num == want_num > 0
    assert not np.array_equal(tr_d["sxl"].cpu().numpy()[-1000:], hit_last[-1000:])
    k.close()


def test_full_operator_direction_test_and_lsq_past_the_clamp(ctx, qn_big):
    """kkt_full_times_vec (elementwise blocks bit-exact, the blocks with B x and J sums to 1e-12), test_direction (dx^T (B + Dx) dx and
    ||dx||^2 against exact sums) and the LSQ multipliers at n = 8192 G + 1."""
    from test_gpu_parity import _setup_kkt, _as_dict
    P, itr, dat, pat = qn_big
    n = P.n
    k, T = _setup_kkt(ctx, _as_dict(P))
    D = ctx.to_device
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    it = dict(sxl=P.sxl, sxu=P.sxu, zl=P.zl, zu=P.zu, sdl=P.sdl, sdu=P.sdu, vl=P.vl, vu=P.vu)
    rng = np.random.default_rng(8)
    sizes = dict(x=n, d=P.m_ineq, yc=P.m_eq, yd=P.m_ineq, sxl=n, sxu=n, sdl=P.m_ineq, sdu=P.m_ineq, zl=n, zu=n, vl=P.m_ineq, vu=P.m_ineq)
    xin = {kk: rng.standard_normal(sizes[kk]) for kk in ko.DIR_NAMES}
    X = {kk: D(xin[kk]) for kk in ko.DIR_NAMES}
    Y = {rk: ctx.zeros(sizes[dk]) for rk, dk in zip(ko.RES_NAMES, ko.DIR_NAMES)}
    k.kkt_full_times_vec(X, Y)
    ctx.sync()
    want = ko.kkt_full_times_vec(st, it, pat, xin, Dx)
    for rk in ko.RES_NAMES:
        got = Y[rk].cpu().numpy()
        if rk in ("rd", "rxl", "rxu", "rdl", "rdu", "rszl", "rszu", "rsvl", "rsvu"):
            np.testing.assert_array_equal(got, want[rk], err_msg=rk)
        else:
            assert np.abs(got - want[rk]).max() <= 1e-12 * max(1.0, np.abs(want[rk]).max()), rk
    # test_direction with l = 0: B = sigma I
    dx, dd = rng.standard_normal(n), rng.standard_normal(P.m_ineq)
    out = (ctypes.c_double * 2)()
    dx_d, dd_d = D(dx), D(dd)
    assert ctx.L.hb_lowrank_test_direction(k.h, _p(dx_d), _p(dd_d), None, None, 1e30, out) == 0
    w = P.sigma + Dx
    dWd = bounds.exact_dot(w * dx, dx) + bounds.exact_dot(Dd * dd, dd)
    terms = float((np.abs(w) * dx * dx).sum() + (Dd * dd * dd).sum())
    c = bounds.slots_chain(n, bounds.stream_grid(n, _G())) + 6
    assert abs(out[0] - dWd) <= bounds.gamma(c) * terms, (out[0], dWd)
    xs = bounds.exact_dot(dx, dx) + bounds.exact_dot(dd, dd)
    assert abs(out[1] - xs) <= bounds.gamma(c) * xs, (out[1], xs)
    # LSQ multipliers: J J^T + I from the condensation and J (g - zl + zu) from one row sweep
    g = rng.standard_normal(n)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(D(g), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, g, P.zl, P.zu, P.vl, P.vu)
    for a, b in ((yc.cpu().numpy(), yco), (yd.cpu().numpy(), ydo)):
        assert np.abs(a - b).max() <= 1e-10 * max(1.0, np.abs(b).max())
    k.close()


def test_secant_update_past_the_clamp(ctx):
    """hiopHessianLowRank::update (k_secant_pair and the Jacobian differences) at n = 8192 G + 1 over a sequence with appends and both skip
    rules: S_t bit-exact, Y_t, L, D and sigma as in tests/test_gpu_secant.py."""
    from hiop_b200.engine import KKTLinSysLowRank
    n, me, mi, lmax = 8192 * _G() + 1, 4, 3, 3
    seq = synth.make_secant_sequence(n, me, mi, steps=7)
    k = KKTLinSysLowRank(ctx, n, me, mi, lmax)
    k.set_patterns(ctx.to_device(np.ones(n)), ctx.to_device(np.zeros(n)), ctx.to_device(np.ones(mi)), ctx.to_device(np.zeros(mi)))
    k.secant_reset(1.0, 1)
    mem = ko.SecantMemory(n, lmax, 1.0, 1)
    for it in seq:
        J = ctx.to_device(np.vstack([it["Jc"], it["Jd"]]))
        k.set_jacobian(J[:me], J[me:])
        s = k.secant_update(ctx.to_device(it["x"]), ctx.to_device(it["grad_f"]), ctx.to_device(it["yc"]), ctx.to_device(it["yd"]))
        assert s == mem.update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"])
        l, sigma, St, Yt, L, Dd = k.secant_state()
        assert l == mem.St.shape[0]
        np.testing.assert_array_equal(St, mem.St)
        assert np.abs(Yt - mem.Yt).max(initial=0.0) <= 1e-13 * max(1.0, np.abs(mem.Yt).max(initial=0.0))
        assert np.abs(np.tril(L, -1) - np.tril(mem.L, -1)).max(initial=0.0) <= 1e-12 * max(1.0, np.abs(mem.L).max(initial=0.0))
        assert np.abs(Dd - mem.D).max(initial=0.0) <= 1e-12 * max(1.0, np.abs(mem.D).max(initial=0.0))
        assert abs(sigma - mem.sigma) <= 1e-12 * mem.sigma
    k.close()
