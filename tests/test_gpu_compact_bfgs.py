"""The quasi-Newton Hessian side (hb_lowrank.cu) held stage by stage, at secant-memory lengths 1 to 256.

Each stage's output is read back (hb_debug_lowrank_state) and compared with the exact operation on that stage's own inputs, also read
back, so that no check needs a tolerance against an end result whose accuracy depends on how well conditioned V is (oracle/lowrank_model.py):

  1. C_aug = [J; S; Y] DhInv [J; S; Y]^T: the FP64 kernel to syrk_tol, the int8 modes (8, 100) to their digit models bit for bit; S S^T
     to syrk_tol;
  2. V, M and U as built: the numpy restatement, bit for bit;
  3. the factors of V and M: LAPACK's DSYTF2 pivots, factor_backward_ratio <= 1, info 0;
  4. Z = U V^-1: solve_backward_ratio <= 1 for every column;
  5. N = W - U Z^T + blkdiag(0, Dd_inv) to gamma(2l + 2), and exactly symmetric;
  6. the fused rhs of solveCompressed to gamma(2l + 2);
  7. hess_solve: the read-back p solves V p = q (q formed exactly, plus the multi-dot's chain), x against DhInv (r - sigma S^T p_S - Y^T p_Y);
  8. hess_times_vec, beta in {0, 1}: the same with M and (sigma + Dx) x.

Every check prints its margin (bound / error). The memory lengths put 2l below 8, at 2l mod 8 in {0, 2} (the multi-dot's launches), at
64 | 66 (k_sytrs_cta from order 65 on) and k_sytf2 at order 512; m = 7 and 8 at l = 33 put the Z solve on both sides of the CTA switch."""
import numpy as np
import pytest
import torch
from scipy.linalg import lapack

from hiop_b200 import synth
from hiop_b200._lib import EngineError
from oracle import bounds
from oracle import crt_model as crt
from oracle import kkt_oracle as ko
from oracle import lowrank_model as lm
from oracle import oz_model as oz

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


def _G():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _problem(n, m, l, regime, seed):
    """default: the synthetic problem; dx0: no bounds on x (Dx = 0, V_SS pure cancellation); sigma_lo / sigma_hi: sigma at its clamps;
    sequence: the pairs, L, D and sigma of a make_secant_sequence run through SecantMemory"""
    sigma = {"sigma_lo": 1e-8, "sigma_hi": 1e8}.get(regime, 1.0)
    P = synth.make_qn_problem(n, m, l, sigma=sigma, seed=seed)
    if regime == "dx0":
        P.ixl[:] = 0.0
        P.ixu[:] = 0.0
    if regime == "sequence":
        mem = ko.SecantMemory(n, l, 1.0, 1)
        for it in synth.make_secant_sequence(n, P.m_eq, P.m_ineq, steps=l + 3, seed=seed):
            mem.update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"])
        assert mem.St.shape[0] == l
        P.St, P.Yt, P.L, P.D, P.sigma = mem.St, mem.Yt, mem.L, mem.D, mem.sigma
    return P


def _setup(ctx, P, l_max, mode=0):
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, l_max)
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ITERATE + ("ixl", "ixu", "idl", "idu", "St", "Yt", "ryc", "ryd")}
    T["J"] = D(P.J)
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    l = P.St.shape[0]
    k.set_secant(P.sigma, T["St"] if l else None, T["Yt"] if l else None, P.L, P.D)
    if mode:
        k.set_condense_mode(mode)
    k.update(*(T[kk] for kk in ITERATE))
    return k, T


def _solve(ctx, k, P, T):
    dx, dyc, dyd = ctx.zeros(P.n), ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.solveCompressed(ctx.to_device(P.rx), T["ryc"], T["ryd"], dx, dyc, dyd)
    k.check()
    return dx.cpu().numpy()


def _bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.int64), np.ascontiguousarray(b).view(np.int64))


def _ratio(err, tol):
    return float((np.abs(err) / np.maximum(tol, np.finfo(np.float64).tiny)).max(initial=0.0))


def _sym_upper(A):
    """the symmetric matrix the factor kernels read: the row-major upper triangle (LAPACK's column-major lower)"""
    return np.triu(A) + np.triu(A, 1).T


def _factor(A, F, ipiv, info, label, what, r):
    """stage 3 for V or M: LAPACK's unblocked pivots, the backward error, info; returns the permuted factor"""
    assert info == 0, (label, what, info)
    ref_ipiv = lapack.dsytrf(A, lower=1, lwork=A.shape[0])[1]
    assert np.array_equal(ipiv, ref_ipiv), (label, what, np.argwhere(ipiv != ref_ipiv)[:5].ravel().tolist())
    rf, n22, fac = lm.factor_check(A, F, ipiv)
    r[f"{what} factor"] = rf
    return fac, n22


# (n, m, l, regime, condensation mode)
CASES = [
    (4099, 8, 1, "default", 0),
    (4096, 7, 4, "default", 0),
    (4099, 1, 5, "dx0", 0),
    (4098, 0, 32, "default", 0),
    (4100, 7, 33, "default", 0),
    (4099, 8, 33, "dx0", 0),
    (8192, 300, 64, "sigma_hi", 0),
    (4099, 7, 64, "sequence", 0),
    (4099, 7, 128, "sigma_lo", 0),
    (4099, 8, 256, "default", 0),
    (4096, 8, 256, "dx0", 0),
    (4099, 8, 33, "default", 8),
    (4099, 300, 5, "default", 8),
    (4099, 7, 33, "sequence", 100),
    (4099, 8, 256, "default", 100),
]


@pytest.mark.parametrize("n,m,l,regime,mode", CASES, ids=[f"n{c[0]}-m{c[1]}-l{c[2]}-{c[3]}-mode{c[4]}" for c in CASES])
def test_stages_against_their_own_inputs(ctx, n, m, l, regime, mode):
    label = f"n={n} m={m} l={l} {regime} mode {mode}"
    G = _G()
    P = _problem(n, m, l, regime, seed=n + 7 * m + 13 * l)
    k, T = _setup(ctx, P, l, mode)
    _solve(ctx, k, P, T)
    st = k.debug_state(l)
    DhInv, Dx, Dd_inv = k.DhInv(), k.Dx(), k.Dd_inv()
    N = k.N() if m else None
    sg, S, Y, meq = P.sigma, P.St, P.Yt, P.m_eq
    Ma = m + 2 * l
    r = {}

    # 1. C_aug and S S^T
    R = np.vstack([P.J, S, Y])
    C = st["Caug"]
    if mode == 0:
        ref = (R * DhInv) @ R.T
        r["C_aug"] = _ratio(C - ref, bounds.syrk_tol(bounds.syrk_bound(R, DhInv), n, ref, c_kernel=n + 2 + G))
    else:
        B = R * np.sqrt(DhInv)
        Cm = oz.condense_bits(B, 8, oz.schedule(Ma, n, 8, G), device="cuda") if mode == 8 else crt.condense_bits(B, device="cuda")
        assert np.array_equal(C, Cm), (label, int((C != Cm).sum()))
    SSt = st["SSt"]
    ref = S @ S.T
    r["SS^T"] = _ratio(SSt - ref, bounds.syrk_tol(bounds.syrk_bound(S, np.ones(n)), n, ref, c_kernel=n + 2 + G))

    # 2. V, M and U as built
    assert _bits(st["V_built"], lm.build_V(C, m, l, sg, SSt, P.L, P.D)), label
    assert _bits(st["M_built"], lm.build_M(l, sg, SSt, P.L, P.D)), label
    if m:
        assert _bits(st["U"], lm.build_U(C, m, l, sg)), label

    # 3. the factor of V
    V = _sym_upper(st["V_built"])
    facV, n22 = _factor(V, st["V_factor"], st["ipivV"], st["info"][0], label, "V", r)
    kappa = np.linalg.cond(V)

    # 4. Z; 5. N; 6. the fused rhs
    if m:
        r["Z"] = lm.solve_ratio(V, facV, st["Z"].T, st["U"].T)[0]
        r["N"] = lm.n_ratio(N, C[:m, :m], st["U"], st["Z"], Dd_inv, meq)
        assert np.array_equal(N, N.T), label
        assert st["info"][1] == 0
        if mode:
            assert st["info"][3] == 1, label          # the int8 modes always fuse the row dots
        if st["info"][3]:
            r["fused rhs"] = lm.fused_rhs_ratio(st["rhs"], st["tdot"], st["Z"], sg, np.concatenate([P.ryc, P.ryd]), m, l)

    # 7. hess_solve
    chain = lm.multidot_chain(n, 1)            # the grid only shortens the chain; 1 CTA is its longest form
    rr = np.random.default_rng(l).standard_normal(n)
    x = ctx.zeros(n)
    k.hess_solve(ctx.to_device(rr), x)
    p = k.debug_state(l)["p2l"]
    q, mag = lm.multidot_exact(S, Y, DhInv, rr, sg)
    r["hess_solve p"] = lm.solve_ratio(V, facV, p, q, extra=bounds.gamma(chain) * mag + U * np.abs(q))[0]
    r["hess_solve x"] = lm.apply_ratio(x.cpu().numpy(), rr, S, Y, p, sg, w=DhInv)

    # 8. hess_times_vec, beta = 0 and 1
    xv = np.random.default_rng(l + 1).standard_normal(n)
    y0 = np.random.default_rng(l + 2).standard_normal(n)
    for beta in (0.0, 1.0):
        y = ctx.to_device(y0)
        k.hess_times_vec(beta, y, 0.75, ctx.to_device(xv), True)
        s3 = k.debug_state(l)
        M = s3["M_built"]
        facM, _ = _factor(M, s3["M_factor"], s3["ipivM"], s3["info"][2], label, "M", r)
        q, mag = lm.multidot_exact(S, Y, None, xv, sg)
        r[f"hess_times_vec p (beta {beta:g})"] = lm.solve_ratio(M, facM, s3["p2l"], q, extra=bounds.gamma(chain) * mag + U * np.abs(q))[0]
        r[f"hess_times_vec y (beta {beta:g})"] = lm.apply_ratio(y.cpu().numpy(), xv, S, Y, s3["p2l"], sg, diag=Dx, beta=beta, y0=y0, alpha=0.75)
    k.close()
    print(f"{label}: kappa(V) {kappa:.3g}, {n22} 2x2 pivots in V, first pivot {int(st['ipivV'][0])}; margins "
          + ", ".join(f"{kk} {1 / max(v, 1e-300):.3g}" for kk, v in r.items()))
    bad = {kk: v for kk, v in r.items() if not v <= 1.0}
    assert not bad, (label, bad)
    if regime == "dx0":
        assert int(st["ipivV"][0]) != 1, label    # V_11 is rounding noise: it is never taken in place


def test_large_lmax_handle_gives_the_same_bits(ctx):
    """A handle created for l_max = 256 running l = 3 computes what a handle for l_max = 3 computes, bit for bit."""
    P = synth.make_qn_problem(4099, 8, 3, seed=77)
    out = []
    for lmax in (256, 3):
        k, T = _setup(ctx, P, lmax)
        dx = _solve(ctx, k, P, T)
        st = k.debug_state(3)
        x = ctx.zeros(P.n)
        k.hess_solve(ctx.to_device(P.rx), x)
        out.append((k.N(), st["Z"], dx, x.cpu().numpy()))
        k.close()
    for a, b in zip(*out):
        assert _bits(a, b)


def test_l256_condensation_is_reproducible(ctx):
    P = synth.make_qn_problem(4099, 8, 256, seed=78)
    k, T = _setup(ctx, P, 256)
    got = []
    for _ in range(2):
        k.update(*(T[kk] for kk in ITERATE))
        k.condense()
        got.append((k.N(), k.debug_state(256)["Z"]))
    k.close()
    assert _bits(got[0][0], got[1][0]) and _bits(got[0][1], got[1][1])


def test_device_secant_memory_fills_and_shifts_at_64(ctx):
    """l_max = 64, the largest the device bookkeeping keeps, over 69 accepted pairs: the memory fills and then shifts five times. S_t is
    bit-exact (one subtraction per entry); L, D and sigma are held to the reduction bounds of their dots on the read-back pairs."""
    from hiop_b200.engine import KKTLinSysLowRank
    n, me, mi, lmax = 2001, 3, 2, 64
    seq = synth.make_secant_sequence(n, me, mi, steps=72, seed=9)
    k = KKTLinSysLowRank(ctx, n, me, mi, lmax)
    k.set_patterns(ctx.to_device(np.ones(n)), ctx.to_device(np.zeros(n)), ctx.to_device(np.ones(mi)), ctx.to_device(np.zeros(mi)))
    k.secant_reset(1.0, 1)
    mem = ko.SecantMemory(n, lmax, 1.0, 1)
    accepted = 0
    for it in seq:
        J = ctx.to_device(np.vstack([it["Jc"], it["Jd"]]))
        k.set_jacobian(J[:me], J[me:])
        s = k.secant_update(ctx.to_device(it["x"]), ctx.to_device(it["grad_f"]), ctx.to_device(it["yc"]), ctx.to_device(it["yd"]))
        assert s == mem.update(it["x"], it["grad_f"], it["yc"], it["yd"], it["Jc"], it["Jd"])
        accepted += s == 1
    l, sigma, St, Yt, L, D = k.secant_state()
    k.close()
    assert accepted > 66 and l == lmax
    assert _bits(St, mem.St)
    c = lm.multidot_chain(n, 1)
    Lref = np.array([[bounds.exact_dot(St[i], Yt[j]) if i > j else 0.0 for j in range(l)] for i in range(l)])
    mag = np.abs(St) @ np.abs(Yt).T
    rL = _ratio(np.tril(L, -1) - Lref, bounds.gamma(c) * np.tril(mag, -1))
    Dref = np.array([bounds.exact_dot(St[i], Yt[i]) for i in range(l)])
    rD = _ratio(D - Dref, bounds.gamma(c) * np.diag(mag))
    s, y = St[-1], Yt[-1]
    sty, ss = bounds.exact_dot(s, y), bounds.exact_dot(s, s)
    sig_ref = sty / ss
    rel = bounds.gamma(c) * float(np.abs(s) @ np.abs(y)) / abs(sty) + 2 * bounds.gamma(c + 3) + 4 * U
    assert 1e-8 < sig_ref < 1e8
    rS = abs(sigma - sig_ref) / (rel * sig_ref)
    print(f"l_max = 64 over {accepted} accepted pairs: margins L {1 / max(rL, 1e-300):.3g}, D {1 / max(rD, 1e-300):.3g}, "
          f"sigma {1 / max(rS, 1e-300):.3g}")
    assert rL <= 1.0 and rD <= 1.0 and rS <= 1.0


def test_device_secant_memory_refuses_65_and_handle_stays_usable(ctx):
    from hiop_b200.engine import KKTLinSysLowRank
    P = synth.make_qn_problem(3001, 6, 3, seed=79)
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, 65)
    with pytest.raises(EngineError, match="64"):
        k.secant_reset(1.0, 1)
    k.close()
    k, T = _setup(ctx, P, 65)
    dx = _solve(ctx, k, P, T)
    k.close()
    k, T = _setup(ctx, P, 3)
    assert _bits(dx, _solve(ctx, k, P, T))
    k.close()


def test_create_refuses_lmax_above_256(ctx):
    from hiop_b200.engine import KKTLinSysLowRank
    with pytest.raises(EngineError):
        KKTLinSysLowRank(ctx, 1000, 2, 2, 257)
    KKTLinSysLowRank(ctx, 1000, 2, 2, 256).close()
