"""The int8-slice (Ozaki) condensation held to its digit model bit for bit, on every branch of its K-split schedule.

With no secant memory (l = 0) the condensed matrix is N = C + blkdiag(0, Dd_inv), C = B B^T from the slices of B = J diag(sqrt(DhInv)),
and k_form_N adds Dd_inv with one rounding. The scheme is deterministic: the digits come from exact scalings and roundings, the integer
products are exact, the row maxima go through an order-independent atomicMax, and the FP64 recombination runs in a fixed order
(t = S-1 .. 0 in k_oz_gemm's epilogue, then the K chunks of a split, then the splits in k_oz_fixup). So oracle/oz_model.condense_bits
predicts N exactly and every case asserts np.array_equal. A kernel that drops one anti-diagonal of products, sums its splits in another
order or cuts K into other chunks fails here, where a tolerance relative to sqrt(N_ii N_jj) would let some of them pass.

Each case also prints its margin against the exact B B^T + blkdiag(0, Dd_inv) (oz_model.exact_gram) under oz_model.truncation_bound.

hb_syrk_rows_ozaki cuts the upper triangle into 128 x 32 tiles and K into splits (one wave of G // tiles splits, clamped to the K stages,
or a multi-wave search when that fills less than 70 % of the machine) and every split into chunks of chunk_stages(S) stages. The
branch cases derive their M from the device's SM count (oz_model.find_shape) and assert the branch they are named after."""
import os

import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from oracle import oz_model as oz

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
DEV = "cuda"


def _G():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _setup(ctx, P, S, J=None):
    """l = 0, condensation mode S; J: the device Jacobian to register (default: a contiguous copy of P.J)"""
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, 1)
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ("ixl", "ixu", "idl", "idu", "zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu", "ryc", "ryd")}
    T["J"] = D(P.J) if J is None else J
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    k.set_secant(P.sigma, None, None, P.L, P.D)
    k.set_condense_mode(S)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    return k, T


def _model(J, DhInv, Dd_inv, meq, S, sch):
    """(N predicted bit for bit, B, digits)"""
    B = J * np.sqrt(DhInv)
    dig = oz.digits(B, S)
    N = oz.condense_bits(B, S, sch, device=DEV, dig=dig)
    i = np.arange(meq, J.shape[0])
    N[i, i] = N[i, i] + Dd_inv
    return N, B, dig


def _margin(N, B, dig, Dd_inv, meq, S, sch):
    """min over the entries of bound / |N - exact|: > 1 when N meets truncation_bound"""
    G, err = oz.exact_gram(B, device=DEV)
    i = np.arange(meq, B.shape[0])
    ref = G.copy()
    ref[i, i] = ref[i, i] + Dd_inv
    R, e = oz.truncation_bound(B, S, sch.chain, device=DEV, dig=dig)
    tol = np.ldexp(R, e[:, None] + e[None, :]) + 2.0 ** -1075 + err + 2 * U * (np.abs(N) + np.abs(ref))
    ratio = float((np.abs(N - ref) / tol).max())
    assert ratio <= 1.0, ratio
    return 1.0 / max(ratio, 1e-300)


def _run(ctx, P, S, sch, label, J=None, mutate=None):
    k, T = _setup(ctx, P, S, J)
    if mutate is not None:
        mutate(k, T)
    k.condense()
    assert k.condense_mode_used() == S
    N = k.N()
    DhInv, Dd_inv = k.DhInv(), k.Dd_inv()
    Jh = T["J"].cpu().numpy()
    k.close()
    Nm, B, dig = _model(Jh, DhInv, Dd_inv, P.m_eq, S, sch)
    bad = np.argwhere(N != Nm)
    assert bad.size == 0, (label, len(bad), bad[:5].tolist(), N[tuple(bad[0])] if bad.size else None, Nm[tuple(bad[0])] if bad.size else None)
    margin = _margin(N, B, dig, Dd_inv, P.m_eq, S, sch)
    print(f"{label}: M={sch.M} K={sch.K} S={S}: {sch.branch}, {sch.splits} splits, {len(sch.items)} items, {sch.max_chunks} chunks "
          f"on {sch.num_sms} SMs; bit-exact, margin {margin:.3g}")
    return N


# ---- every branch of the schedule --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", oz.BRANCH_CASES, ids=[f"{c[0]}-M{c[1]}-K{c[2]}-S{c[3]}" for c in oz.BRANCH_CASES])
def test_condensation_equals_digit_model(ctx, case):
    branch, M0, K, S = case
    G = _G()
    M = oz.find_shape(branch, M0, K, S, G)
    sch = oz.schedule(M, K, S, G)
    assert sch.branch == branch
    P = synth.make_qn_problem(K, M, 0, seed=M + K + S)
    _run(ctx, P, S, sch, branch)


def test_every_oz_branch_is_reached():
    """Every branch of the schedule has a case on this device (restated host arithmetic)."""
    G = _G()
    got = {oz.schedule(oz.find_shape(b, M0, K, S, G), K, S, G).branch for b, M0, K, S in oz.BRANCH_CASES}
    assert got == set(oz.BRANCHES), (G, got)


# ---- edges of M, K and the slicing kernel's paths ------------------------------------------------------------------------------------

# (M, K, S, J offset by one double): M around the 32-column and 128-row tile edges; K mod 128 in {0, 1, 8, 127} and K < 128; odd K
# makes the rows 8-byte aligned (the scalar path of k_oz_slice); a J one double off a 16-byte boundary at even K does too (vec_ok = 0)
EDGES = [(1, 4096, 8, False), (31, 4097, 7, False), (32, 4104, 6, False), (33, 4223, 8, False), (127, 100, 8, False),
         (129, 3001, 7, False), (40, 4096, 8, True), (64, 5000, 6, True)]


@pytest.mark.parametrize("M,K,S,offset", EDGES, ids=[f"M{e[0]}-K{e[1]}-S{e[2]}{'-offset' if e[3] else ''}" for e in EDGES])
def test_edges_equal_digit_model(ctx, M, K, S, offset):
    P = synth.make_qn_problem(K, M, 0, seed=3 * M + K)
    J = None
    if offset:
        buf = torch.zeros(M * K + 1, dtype=torch.float64, device=DEV)
        J = buf[1:].view(M, K)
        J.copy_(torch.from_numpy(P.J))
        assert J.data_ptr() % 16 == 8
    sch = oz.schedule(M, K, S, _G())
    _run(ctx, P, S, sch, f"edge M={M} K={K}{' offset' if offset else ''}", J=J)


# ---- extreme rows ----------------------------------------------------------------------------------------------------------------------

def _entry_hitting(J, DhInv, i, target):
    """Sets one entry of row i of J (host copy) so that fl(J_ik sqrt(DhInv_k)) == target exactly; returns k"""
    sd = np.sqrt(DhInv)
    for k in range(J.shape[1]):
        a0 = target / sd[k]
        for a in (a0, np.nextafter(a0, np.inf), np.nextafter(a0, -np.inf)):
            if a * sd[k] == target:
                J[i, k] = a
                return k
    raise AssertionError("no column reproduces the target")


EXTREME = ["tiny 1e-303", "1e+-150", "zero row", "max a power of two", "leading digit 64"]


@pytest.mark.parametrize("kind", EXTREME)
def test_extreme_rows_equal_digit_model(ctx, kind):
    """Rows whose maximum is below 2^-997 (2^(27 - e) overflows unless it is applied in two steps), rows at 1e+-150, an all-zero row, a
    row whose maximum is a power of two and one whose maximum rounds the first word of digits up to 2^27 (leading digit 64). The small
    rows are inequality rows: Dd_inv keeps N positive definite."""
    M, K, S = 40, 6000, 8
    P = synth.make_qn_problem(K, M, 0, seed=77)
    meq = P.m_eq
    J = P.J.copy()
    if kind == "tiny 1e-303":
        J[meq + 3] *= 1e-303
    elif kind == "1e+-150":
        J[5] *= 1e150
        J[meq + 5] *= 1e-150
    elif kind == "zero row":
        J[meq + 2] = 0.0
    else:
        # DhInv only depends on the iterate: one throw-away update gives the device's values
        k0, _ = _setup(ctx, P, S)
        DhInv = k0.DhInv()
        k0.close()
        J[3] *= 0.25                                          # keeps every other entry of the row below the planted maximum
        if kind == "max a power of two":
            _entry_hitting(J, DhInv, 3, 0.5)
        else:
            _entry_hitting(J, DhInv, 3, 1.0 - 2.0 ** -30)     # beta = 1 - 2^-30: rint(beta 2^27) = 2^27
            e, Q = oz.digits(J[3:4] * np.sqrt(DhInv), S)
            assert Q[0].max() == 64
    P.Jc, P.Jd = np.ascontiguousarray(J[:meq]), np.ascontiguousarray(J[meq:])
    sch = oz.schedule(M, K, S, _G())
    N = _run(ctx, P, S, sch, kind)
    assert np.all(np.isfinite(N))


# ---- the fused sweep: solveCompressed with the condensation pending ----------------------------------------------------------------------

RD_COLS = 256


def _rsplit(K, G):
    nchunks = -(-K // RD_COLS)
    return min(max(-(-2 * G // nchunks), 1), 8)


@pytest.mark.parametrize("variant", ["vec-rsplit1", "scalar-rsplit1", "vec-rsplit8", "scalar-rsplit8"])
def test_fused_sweep_equals_digit_model_and_bounds_tdot(ctx, variant):
    """The row maxima come from k_oz_rowmax_dot (16-byte rows and even K: the paired VEC loads; else scalar), whose rows are split over
    rsplit CTAs per column chunk; N must equal the same model. tdot = J (DhInv .* rx) from the same sweep, against the exact dot with
    w = fl(DhInv .* rx) (the kernel forms the same w): each lane sums its 8 columns (8), a warp tree (5), k_oz_dot_final sums every
    8th chunk (ceil(nchunks / 8)) and then the 8 classes (8): |tdot - exact| <= gamma_c sum_k |J_ik w_k| + u |exact| with
    c = 8 + 5 + ceil(nchunks / 8) + 8."""
    G = _G()
    vec = variant.startswith("vec")
    K = 2 * G * RD_COLS + 1000 if variant.endswith("rsplit1") else (G // 4) * RD_COLS - 100
    K += 0 if vec else 1
    want = 1 if variant.endswith("rsplit1") else 8
    assert _rsplit(K, G) == want
    M, S = 100, 8
    P = synth.make_qn_problem(K, M, 0, seed=K)
    k, T = _setup(ctx, P, S)
    dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
    assert k.solveCompressed(ctx.to_device(P.rx), T["ryc"], T["ryd"], dx, dyc, dyd)
    k.check()
    ctx.sync()
    assert k.condense_mode_used() == S
    N, tdot, DhInv, Dd_inv = k.N(), k.tdot(), k.DhInv(), k.Dd_inv()
    k.close()
    sch = oz.schedule(M, K, S, G)
    Nm, B, dig = _model(P.J, DhInv, Dd_inv, P.m_eq, S, sch)
    assert np.array_equal(N, Nm)
    w = DhInv * P.rx
    ref = bounds.exact_rows(P.J, w)
    c = 8 + 5 + -(-(-(-K // RD_COLS)) // 8) + 8
    tol = bounds.gamma(c) * (np.abs(P.J) @ np.abs(w)) + U * np.abs(ref)
    ratio = float((np.abs(tdot - ref) / tol).max())
    print(f"fused {variant}: K={K} rsplit={want}: N bit-exact, tdot margin {1.0 / max(ratio, 1e-300):.3g}")
    assert ratio <= 1.0, ratio


def test_fp64_fused_row_meets_syrk_chain(ctx):
    """The FP64 condensation folds J (DhInv .* rx) into its SYRK as row M when that row fits in the last tile (M = 128 T - 1):
    k_syrk_fixup sends it to tdot. Against the exact dot with w = fl(DhInv .* rx): the SYRK chain (K products rounded twice, the K
    windows of at most G CTAs) plus the rounding of w, |tdot - exact| <= gamma_{K+3+G} sum_k |J_ik w_k| + u |exact|."""
    G = _G()
    M, K = 127, 12000
    P = synth.make_qn_problem(K, M, 0, seed=5)
    k, T = _setup(ctx, P, 0)
    dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
    assert k.solveCompressed(ctx.to_device(P.rx), T["ryc"], T["ryd"], dx, dyc, dyd)
    k.check()
    ctx.sync()
    tdot, DhInv = k.tdot(), k.DhInv()
    k.close()
    w = DhInv * P.rx
    ref = bounds.exact_rows(P.J, w)
    tol = bounds.gamma(K + 3 + G) * (np.abs(P.J) @ np.abs(w)) + U * np.abs(ref)
    ratio = float((np.abs(tdot - ref) / tol).max())
    print(f"FP64 fused row M={M} K={K}: tdot margin {1.0 / max(ratio, 1e-300):.3g}")
    assert ratio <= 1.0, ratio


# ---- the schedule cache ---------------------------------------------------------------------------------------------------------------

def test_schedule_revisit_and_fresh_context_are_bit_identical(ctx):
    """The context keeps the work list and tensor maps of the last (M, K, S): another shape rebuilds them, the first shape again must
    give the bits of its first visit, and so must a fresh context."""
    from hiop_b200.engine import Context
    S = 8
    shapes = [(300, 20000), (129, 8001), (300, 20000)]
    probs = {s: synth.make_qn_problem(s[1], s[0], 0, seed=s[0]) for s in shapes}
    out = []
    for s in shapes:
        k, _ = _setup(ctx, probs[s], S)
        k.condense()
        out.append(k.N().copy())
        k.close()
    np.testing.assert_array_equal(out[2], out[0])
    c2 = Context(0)
    try:
        k, _ = _setup(c2, probs[shapes[0]], S)
        k.condense()
        np.testing.assert_array_equal(k.N(), out[0])
        k.close()
    finally:
        c2.close()


def test_max_splits_override_in_a_fresh_context():
    """HB_OZ_MAX_SPLITS bounds the multi-wave split search (read on every call, like HB_CRT_MAX_SPLITS), here in a fresh context. With 1
    the search keeps one split where it would pick more, and N equals the model of that schedule (and differs from the default's)."""
    from hiop_b200.engine import Context
    G, S = _G(), 8
    M = oz.find_shape("search picks sp > 1", 1000, 20000, S, G)
    K = 20000
    dflt, capped = oz.schedule(M, K, S, G), oz.schedule(M, K, S, G, max_splits=1)
    assert dflt.splits > 1 and capped.splits == 1
    P = synth.make_qn_problem(K, M, 0, seed=17)
    old = os.environ.get("HB_OZ_MAX_SPLITS")
    os.environ["HB_OZ_MAX_SPLITS"] = "1"
    c2 = Context(0)
    try:
        N = _run(c2, P, S, capped, "HB_OZ_MAX_SPLITS=1")
    finally:
        c2.close()
        if old is None:
            del os.environ["HB_OZ_MAX_SPLITS"]
        else:
            os.environ["HB_OZ_MAX_SPLITS"] = old
    B = P.J * np.sqrt(_dhinv(P))
    assert not np.array_equal(oz.condense_bits(B, S, dflt, device=DEV), oz.condense_bits(B, S, capped, device=DEV))


def _dhinv(P):
    from oracle import kkt_oracle as ko
    return ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)[1]
