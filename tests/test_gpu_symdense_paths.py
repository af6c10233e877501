"""Every path of the dense symmetric factorizations and solves (hb_symdense.cu dispatch table; hb_dense.cu, hb_dense_big.cu,
hb_bk_cluster.cu, hb_chol_coop.cu) held to componentwise backward-error bounds (oracle/bounds.py, Higham ch. 8, 10, 11, 14): the factor
read back with hb_debug_symdense_factor against |P A P^T - L D L^T| <= theta gamma(3N+3)(|A| + |L||D||L^T|) + check rounding, every solve
against the Oettli-Prager-type bound theta gamma(7N+3)((|A| + |L||D||L^T|)|x| + |b|), the inertia against a matrix family whose inertia is
known by construction, and the Bunch-Kaufman pivots against LAPACK's dsytrf. Each case asserts the plan codes (and cluster panel widths)
the dispatch chose, so a threshold change cannot silently move a case to another path. The branches that are not the default at these
sizes are forced through the environment knobs hb_dense_init reads once per context (HB_DENSE_PAIR_MIN, HB_BK_CLUSTER_MIN,
HB_DENSE_BIG_MIN, HB_CHOL_COOP)."""
import numpy as np
import pytest
import torch
from scipy.linalg import lapack

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko
from test_gpu_parity import _setup_kkt, _as_dict, _kkt_residual
from dense_handles import DEV, factor_parts, make_ctx, readback, theta  # noqa: F401 (make_ctx: fixture)

pytestmark = pytest.mark.gpu

BK, NOPIV, CHOL = 0, 1, 2
DSYTRF_MAX_N = 7001      # pivot sequence and factor compared with scipy's dsytrf up to this order


# ---- matrices -------------------------------------------------------------------------------------------------------------------------
def _spd(N, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = torch.randn((N, N // 2 + 1), generator=g, dtype=torch.float64).to(DEV)
    d = torch.rand(N, generator=g, dtype=torch.float64).to(DEV) * 1.5 + 0.5
    return G @ G.T / N + torch.diag(d), (0, 0, N)


def _indefinite(N, seed):
    return bounds.known_inertia_matrix(N, N // 3, N // 7, seed, device=DEV)


def _quasidefinite(N, seed):
    m = N // 3
    return torch.from_numpy(synth.make_kkt_like(N - m, m, seed=seed)).to(DEV), (m, 0, N - m)


MATRIX = {BK: _indefinite, NOPIV: _quasidefinite, CHOL: _spd}


def _upper_only(M):
    """M with NaN in the strict lower triangle, which hb_symdense_matrix_changed documents as never read"""
    U = M.clone()
    U.masked_fill_(torch.ones(M.shape, dtype=torch.bool, device=M.device).tril_(-1), float("nan"))
    return U


def set_matrix(s, M):
    """s.set_matrix(M) for an M computed by torch. torch wrote M on its own stream and the engine copies it on its non-blocking stream, so
    wait for torch's kernels first, and for the copy before M (or a temporary it came from) can be freed and its memory reused."""
    M = M.contiguous()
    torch.cuda.synchronize()
    s.set_matrix(M)
    s.ctx.sync()


# ---- one factorization, read back -----------------------------------------------------------------------------------------------------
def _same(a, b):
    """bitwise equal, None (no such output for this factor) only with None"""
    return (a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b))


def run_case(ctx, mode, N, seed, expect, widths=None, nrhs_list=(1, 7, 8)):
    """factor + solves on one handle; asserts plan, inertia, factor and solve bounds, pivots. Returns the margins."""
    from hiop_b200.engine import LinSolverSymDense
    M, inertia = MATRIX[mode](N, seed)
    s = LinSolverSymDense(ctx, N, mode)
    set_matrix(s, _upper_only(M))
    ret = s.matrixChanged()
    rb = readback(s)
    assert rb["plan"] == expect, (rb["plan"], expect)
    if widths is not None:
        assert rb["widths"] == widths, (rb["widths"], widths)
    assert ret == inertia[0] and s.inertia() == inertia, (ret, s.inertia(), inertia)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    sols = []
    for nrhs in nrhs_list:
        b = torch.randn((nrhs, N), generator=g, dtype=torch.float64)
        x = ctx.to_device(b.numpy())
        assert s.solve(x)
        ctx.sync()
        sols.append((b.to(DEV), x))
    s.close()
    L, d, dsub, perm = factor_parts(rb)
    if rb["plan"][0] == "BK_CLUSTER":
        bounds.bk_cluster_to_lapack(rb["ipiv"], rb["perm"], rb["dsub"])
    pt = torch.from_numpy(perm).to(DEV)
    Mh = M.cpu().numpy() if mode == BK and N <= DSYTRF_MAX_N else None
    PAP = M[pt][:, pt]
    del M
    th = theta(L)
    fr = bounds.factor_backward_ratio(PAP, L, d, dsub, th)
    sr, om = 0.0, 0.0
    small = N <= bounds.EXACT_RESIDUAL_MAX_N
    for b, x in sols:
        xp, bp = x.T[pt], b.T[pt]
        if small:   # exact residual on the host
            r, o = bounds.solve_backward_ratio(PAP.cpu().numpy(), xp.cpu().numpy(), bp.cpu().numpy(), L.cpu().numpy(), d.cpu().numpy(),
                                               None if dsub is None else dsub.cpu().numpy(), th)
        else:
            r, o = bounds.solve_backward_ratio(PAP, xp, bp, L, d, dsub, th)
        sr, om = max(sr, r), max(om, o)
    msg = (f"{('BK', 'NOPIV', 'CHOL')[mode]} N={N}: plan {rb['plan']} widths {rb['widths']} theta {th:.2f}; factor margin {1 / max(fr, 1e-300):.3g}, "
           f"solve margin {1 / max(sr, 1e-300):.3g} (omega {om:.2e})")
    if mode == BK and N <= DSYTRF_MAX_N:
        ldu, ipiv, info = lapack.dsytrf(np.asfortranarray(np.tril(Mh)), lower=1)
        assert info == 0
        assert np.array_equal(rb["ipiv"], ipiv), np.nonzero(rb["ipiv"] != ipiv)[0][:8]
        if rb["plan"][0] in ("SYTF2", "SYTRF_BLOCKED"):
            # the factor itself against dsytrf's: both factor the same P A P^T within the bound, so within twice it of each other
            Ll, dl, dsubl, _ = bounds.lapack_to_permuted(ldu, ipiv)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
            prod_lapack = bounds.ld_product(t(Ll), t(dl), t(dsubl)) @ t(Ll).T
            rr = bounds.factor_backward_ratio(prod_lapack, L, d, dsub, th) / 2
            msg += f"; vs dsytrf's factor margin {1 / max(rr, 1e-300):.3g}"
            assert rr <= 1.0
        msg += "; ipiv = dsytrf's"
    print(msg)
    assert fr <= 1.0 and sr <= 1.0, msg
    return rb


# ---- the case table ---------------------------------------------------------------------------------------------------------------------
PAIRS = dict(HB_DENSE_PAIR_MIN=0, HB_DENSE_BIG_MIN=0)
BKMIN0 = dict(HB_BK_CLUSTER_MIN=0)
NOCOOP = dict(HB_CHOL_COOP=0)
BIGOFF = dict(HB_DENSE_BIG_MIN=1 << 30)

CASES = [
    # Bunch-Kaufman, default thresholds: DSYTF2 < 96 <= blocked DLASYF < 385 <= cluster
    (BK, 1, {}, ("SYTF2", "SYTRS", "IPIV", False), None),
    (BK, 64, {}, ("SYTF2", "SYTRS", "IPIV", False), None),
    (BK, 95, {}, ("SYTF2", "SYTRS", "IPIV", False), None),
    (BK, 96, {}, ("SYTRF_BLOCKED", "SYTRS", "IPIV", False), None),
    (BK, 200, {}, ("SYTRF_BLOCKED", "SYTRS", "IPIV", False), None),
    (BK, 384, {}, ("SYTRF_BLOCKED", "SYTRS", "IPIV", False), None),
    (BK, 385, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 32),
    (BK, 1001, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 32),
    (BK, 3500, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 64 | 32),
    (BK, 7001, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 32 | 64),
    (BK, 12000, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 16 | 32 | 64),
    (BK, 24000, {}, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 8 | 16 | 32 | 64),
    # cluster Bunch-Kaufman below its default minimum: one CTA row per panel, 2x2 blocks across the NB-1 panel ends, last panel
] + [(BK, n, BKMIN0, ("BK_CLUSTER", "BIG", "BLOCKDIAG", False), 32) for n in (1, 2, 31, 33, 63, 64, 65, 97, 200)] + [
    # no-pivot LDL^T: panels < 257 <= look-ahead; pairs forced from 0 and by default from 6144
    (NOPIV, 64, {}, ("PANEL_LDL", "ONE_CTA", "DIAG", False), None),
    (NOPIV, 256, {}, ("PANEL_LDL", "ONE_CTA", "DIAG", False), None),
    (NOPIV, 300, BIGOFF, ("PANEL_LDL", "BIG", "DIAG", False), None),
    (NOPIV, 257, {}, ("BIG_LDL", "BIG", "DIAG", False), None),
    (NOPIV, 2049, {}, ("BIG_LDL", "BIG", "DIAG", False), None),
] + [(NOPIV, n, PAIRS, ("BIG_LDL", "BIG", "DIAG", True), None) for n in (257, 384, 640, 1153, 2049)] + [
    (NOPIV, 6144, {}, ("BIG_LDL", "BIG", "DIAG", True), None),
    # Cholesky: panels < 65 <= cooperative <= 2048, look-ahead from 1025; without cooperative launches the panels
    (CHOL, 10, {}, ("PANEL_CHOL", "ONE_CTA", "DIAG", False), None),
    (CHOL, 64, {}, ("PANEL_CHOL", "ONE_CTA", "DIAG", False), None),
    (CHOL, 65, {}, ("COOP_CHOL", "ONE_CTA", "DIAG", False), None),
    (CHOL, 256, {}, ("COOP_CHOL", "ONE_CTA", "DIAG", False), None),
    (CHOL, 257, {}, ("COOP_CHOL", "BIG", "DIAG", False), None),
    (CHOL, 1024, {}, ("COOP_CHOL", "BIG", "DIAG", False), None),
    (CHOL, 1025, {}, ("BIG_CHOL", "BIG", "DIAG", False), None),
    (CHOL, 2049, {}, ("BIG_CHOL", "BIG", "DIAG", False), None),
    (CHOL, 2500, BIGOFF, ("PANEL_CHOL", "BIG", "DIAG", False), None),
] + [(CHOL, n, NOCOOP, ("PANEL_CHOL", "ONE_CTA" if n < 257 else "BIG", "DIAG", False), None) for n in (65, 256, 257, 1024)] + [
    (CHOL, n, PAIRS, ("BIG_CHOL", "BIG", "DIAG", True), None) for n in (257, 384, 640, 1153, 2049)] + [
    (CHOL, 6144, {}, ("BIG_CHOL", "BIG", "DIAG", True), None),
]


def _id(c):
    env = ",".join(f"{k[3:].lower()}={v}" for k, v in c[2].items())
    return f"{('bk', 'nopiv', 'chol')[c[0]]}-{c[1]}" + (f"-{env}" if env else "")


@pytest.mark.parametrize("mode,N,env,expect,widths", CASES, ids=[_id(c) for c in CASES])
def test_symdense_path(make_ctx, mode, N, env, expect, widths):
    run_case(make_ctx(**env), mode, N, seed=N + 7 * mode, expect=expect, widths=widths)
    torch.cuda.empty_cache()


# ---- state carried by one handle ------------------------------------------------------------------------------------------------------
def _factor_bits(ctx, s, M, mode, rhs):
    from hiop_b200.engine import LinSolverSymDense  # noqa: F401
    s.mode = mode
    set_matrix(s, M)
    ret = s.matrixChanged()
    rb = readback(s)
    x = ctx.to_device(rhs)
    assert s.solve(x)
    ctx.sync()
    return ret, rb, x.cpu().numpy()


def test_one_handle_through_every_mode_gives_fresh_bits(make_ctx):
    """odd N: BK (cluster, padded) -> NOPIV (look-ahead, padded) -> CHOL (look-ahead, padded) -> BK on one handle, each equal to a fresh
    handle's factor and solution to the bit; Fpad, W / Wp, the inverses and the solve's ticket counter carry nothing over"""
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx(HB_DENSE_BIG_MIN=0)
    N = 1153
    rhs = np.random.default_rng(3).standard_normal((8, N))
    mats = {BK: MATRIX[BK](N, 1)[0], NOPIV: MATRIX[NOPIV](N, 2)[0], CHOL: MATRIX[CHOL](N, 3)[0]}
    s = LinSolverSymDense(ctx, N, BK)
    for mode in (BK, NOPIV, CHOL, BK):
        ret, rb, x = _factor_bits(ctx, s, mats[mode], mode, rhs)
        f = LinSolverSymDense(ctx, N, mode)
        ret_f, rb_f, x_f = _factor_bits(ctx, f, mats[mode], mode, rhs)
        f.close()
        print(f"mode {mode}: plan {rb['plan']}")
        assert rb["plan"] == rb_f["plan"] and rb["plan"][0] in ("BK_CLUSTER", "BIG_LDL", "BIG_CHOL")
        assert ret == ret_f >= 0
        assert np.array_equal(np.triu(rb["F"]), np.triu(rb_f["F"])) and _same(rb["ipiv"], rb_f["ipiv"])
        assert np.array_equal(x, x_f)
        # a second solve on the same factor, and each rhs alone against the 8-rhs batch of the blocked solve
        x2 = ctx.to_device(rhs)
        assert s.solve(x2)
        ctx.sync()
        assert np.array_equal(x, x2.cpu().numpy())
        for j in (0, 5, 7):
            xj = ctx.to_device(rhs[j].copy())
            assert s.solve(xj)
            ctx.sync()
            assert np.array_equal(x[j], xj.cpu().numpy())
    s.close()


@pytest.mark.parametrize("mode,N,env", [(NOPIV, 2049, PAIRS), (CHOL, 1153, PAIRS), (BK, 3500, {})])
def test_bit_reproducible(make_ctx, mode, N, env):
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx(**env)
    M = MATRIX[mode](N, 4)[0]
    rhs = np.random.default_rng(4).standard_normal((1, N))
    outs = []
    for _ in range(2):
        s = LinSolverSymDense(ctx, N, mode)
        outs.append(_factor_bits(ctx, s, M, mode, rhs))
        s.close()
    (r0, b0, x0), (r1, b1, x1) = outs
    assert b0["plan"][3] == (mode != BK) and r0 == r1
    assert np.array_equal(np.triu(b0["F"]), np.triu(b1["F"])) and np.array_equal(x0, x1)


# ---- breakdown ------------------------------------------------------------------------------------------------------------------------
def _broken(mode, M, col):
    B = M.clone()
    if mode == CHOL:
        B[col, col] = -1.0            # leading minor col + 1 not positive definite
    else:
        B[col, :] = 0.0               # exactly zero pivot at col
        B[:, col] = 0.0
    return B


@pytest.mark.parametrize("mode", [NOPIV, CHOL])
@pytest.mark.parametrize("N,col", [(1153, 0), (1153, 15), (1153, 16), (1153, 127), (1153, 128), (640, 200), (1153, 1152), (1100, 1090)])
def test_breakdown_then_recovery(make_ctx, mode, N, col):
    """-1 for a breakdown at column 0, across the 16-column sub-panels of k_diag128, across a 128-column block, in the second block of
    a pair (640: blocks 0-127 and 128-255 form the first pair) and in the last, partial block (1153 = 9 * 128 + 1: column 1152 alone;
    1100 = 8 * 128 + 76: columns 1024-1099); then a good matrix on the same handle
    gives the bits of a fresh handle"""
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx(**PAIRS)
    M = MATRIX[mode](N, 5)[0]
    rhs = np.random.default_rng(5).standard_normal((1, N))
    s = LinSolverSymDense(ctx, N, mode)
    set_matrix(s, _broken(mode, M, col))
    assert s.matrixChanged() == -1
    assert readback(s)["plan"] == ((("BIG_LDL", "BIG_CHOL")[mode == CHOL]), "BIG", "DIAG", True)
    ret, rb, x = _factor_bits(ctx, s, M, mode, rhs)
    s.close()
    f = LinSolverSymDense(ctx, N, mode)
    ret_f, rb_f, x_f = _factor_bits(ctx, f, M, mode, rhs)
    f.close()
    assert ret == ret_f >= 0
    assert np.array_equal(np.triu(rb["F"]), np.triu(rb_f["F"])) and np.array_equal(x, x_f)


@pytest.mark.parametrize("N", [200, 1001])
def test_singular_bunch_kaufman(make_ctx, N):
    from hiop_b200.engine import LinSolverSymDense
    ctx = make_ctx()
    M = MATRIX[BK](N, 6)[0]
    M[N // 2, :] = 0.0
    M[:, N // 2] = 0.0
    s = LinSolverSymDense(ctx, N, BK)
    set_matrix(s, M)
    assert s.matrixChanged() == -1
    assert s.inertia()[1] == 1
    print(f"singular BK N={N}: plan {readback(s)['plan']}, inertia {s.inertia()}")
    s.close()


# ---- the condensed N of the quasi-Newton KKT path and the LSQ duals ----------------------------------------------------------------
@pytest.mark.parametrize("coop", [True, False])
@pytest.mark.parametrize("m", [64, 65, 2048, 2049, 2050, 6144, 6145])
def test_condensed_solve_needs_no_refinement(make_ctx, m, coop):
    """The first solve of N dy = rhs must already be at rounding level: zero refinement steps.

    Bound on the residual r = rhs - N dy of that first solve, row by row: the Cholesky of the equilibrated matrix (unit diagonal) has
    |R^T||R| <= 1 entrywise, so Higham Thm 10.4 gives |r_i| <= theta gamma(7m+3) sum_j sqrt(N_ii N_jj)|dy_j|; the solve evaluates r in
    FP64, adding gamma(m+1)(|N||dy| + |rhs|)_i, and |rhs| <= |N||dy| + |r| moves |r| to the left: divide by 1 - gamma(m+1). The solve
    reports only ||r||_inf, so the check is ||r||_inf <= max_i bound_i (a norm comparison of the componentwise bound).

    Which factorization runs is chosen by m inside the quasi-Newton handle (condensed_plan, dispatch table of hb_symdense.cu): m = 6144
    is the paired look-ahead, 6145 (odd ld) the panels, 2049 / 2050 the panels / look-ahead, up to 2048 the cooperative kernels; without
    cooperative launches the panels and the one-CTA refinement solve. test_gpu_condensed_refine.py asserts those rows through
    hb_debug_condensed_solve, which runs the same plan."""
    ctx = make_ctx(**({} if coop else NOCOOP))
    P = synth.make_qn_problem(max(600, 3 * m), m, 4, seed=77 + m)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    rx, ryc, ryd = ctx.to_device(P.rx), ctx.to_device(P.ryc), ctx.to_device(P.ryd)
    dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(rx, ryc, ryd, dx, dyc, dyd)
    ctx.sync()
    nref, resid = k.last_solve_stats()
    Nm = torch.from_numpy(k.N()).to(DEV)
    dy = torch.cat([dyc, dyd])
    sq = torch.sqrt(torch.diagonal(Nm))
    R = torch.linalg.cholesky(Nm / torch.outer(sq, sq))
    th = max(bounds.block_theta(R, 16), bounds.block_theta(R, 128))
    ndy = torch.abs(Nm) @ torch.abs(dy)
    bound = (th * bounds.gamma(7 * m + 3) * sq * (sq @ torch.abs(dy)) + bounds.gamma(m + 1) * 2 * ndy) / (1 - bounds.gamma(m + 1))
    bound = float(bound.max())
    kres = _kkt_residual(ctx, k, T, p, dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy())
    print(f"condensed m={m} coop={coop}: refinements {nref}, residual {resid:.3e}, bound {bound:.3e} (margin {bound / max(resid, 1e-300):.3g}),"
          f" KKT residual {kres:.2e}")
    k.close()
    assert nref == 0 and resid <= bound
    assert kres <= 1e-8


@pytest.mark.parametrize("coop", [True, False])
@pytest.mark.parametrize("m", [64, 65, 2048, 2049])
def test_lsq_duals_with_and_without_coop(make_ctx, m, coop):
    ctx = make_ctx(**({} if coop else NOCOOP))
    n = max(3000, 3 * m)
    P = synth.make_qn_problem(n, m, 0, seed=5 + m)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    g = np.random.default_rng(9).standard_normal(n)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(ctx.to_device(g), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, g, P.zl, P.zu, P.vl, P.vu)
    for a, b in ((yc.cpu().numpy(), yco), (yd.cpu().numpy(), ydo)):
        assert np.abs(a - b).max(initial=0.0) <= 1e-10 * max(1.0, np.abs(b).max(initial=0.0))
    k.close()

