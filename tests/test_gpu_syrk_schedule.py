"""The FP64 condensation (hb_syrk.cu) over its schedule branches and kernels, held to the componentwise error bound.

With no secant memory (l = 0) the condensed matrix is N = J DhInv J^T + blkdiag(0, Dd_inv) exactly, so every entry of N can be held to
|N - N_ref| <= (gamma_c + gamma_{K+2}) (|J| DhInv |J|^T) + 2u|N| (oracle/bounds.py) instead of a fraction of max|N|. On the synthetic
problems max|N| is the all-ones row's N_00 ~ 0.3 n, so the old check was an FP32-level check of every other entry.

build_schedule cuts the upper triangle of 128 x 128 output tiles (T tile rows, ntiles = T(T+1)/2) and the K iterations over the G
streaming multiprocessors. Its branches are restated below (schedule_branch) and every case asserts the branch it is named after; the
shapes are derived from the device's SM count, so a 114-SM H100 PCIe reaches the same branches as a 132-SM SXM part. One kernel,
k_syrk_ws, sweeps K in chunks of WBK = 32 columns with two producers: 16-byte copies when the rows are 16-byte aligned ("ws": even K,
or a single row, M = 1, whose row pointer is J itself) and 8-byte copies otherwise ("odd": odd K with two or more packed rows, which
then start on alternating 8-byte boundaries). The "ws" K tails are K mod 32 in {0, 2, 30} and, at M = 1, the 16-byte producer's
8-byte tail {1, 31}; the "odd" cases reach every branch with K mod 32 in {1, 15, 17, 31}."""
import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds

pytestmark = pytest.mark.gpu

BM, WBK = 128, 32


def schedule_branch(M, K, G):
    """build_schedule's decision (hb_syrk.cu), restated: returns (branch, launched CTAs)."""
    T = -(-M // BM)
    ntiles = T * (T + 1) // 2
    kiters = -(-K // WBK)
    total = ntiles * kiters
    Gl = G if total >= G else max(total, 1)
    L = Gl // ntiles
    R = Gl - L * ntiles
    w = 0 if L < 1 else (total // Gl if R else kiters // L)
    if Gl < G:
        kind = "reduced G"
    elif L >= 1 and w >= 1:
        kind = "L = 1" if L == 1 else ("lanes, R = 0" if R == 0 else "lanes, R > 0")
    else:
        kind = "stream-K"
    return kind, Gl


def _G():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _setup(ctx, P):
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, max(P.l, 1))
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ("ixl", "ixu", "idl", "idu", "zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu", "St", "Yt", "ryc", "ryd")}
    T["J"] = D(P.J)
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    k.set_secant(P.sigma, T["St"] if P.l else None, T["Yt"] if P.l else None, P.L, P.D)
    k.set_condense_mode(0)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    return k, T


def _reference(P, DhInv, Dd_inv):
    """numpy FP64 N = J DhInv J^T + blkdiag(0, Dd_inv) and the bound matrix |J| DhInv |J|^T"""
    J = P.J
    N = (J * DhInv) @ J.T
    N[np.arange(P.m_eq, P.m), np.arange(P.m_eq, P.m)] += Dd_inv
    return N, bounds.syrk_bound(J, DhInv)


def _check_N(N, Nref, B, K, G):
    # kernel chain: K products (each rounded twice: d is folded into one factor) summed along the K windows of at most G CTAs
    tol = bounds.syrk_tol(B, K, Nref, c_kernel=K + 2 + G)
    ratio = float((np.abs(N - Nref) / tol).max())
    assert np.array_equal(N, N.T)
    assert ratio <= 1.0, ratio
    return 1.0 / max(ratio, 1e-300)


# (branch, producer, K, rows short of a full last tile, preferred T). The tile-row count T is chosen on the running device: the preferred
# T when it lands in the branch, else the nearest T that does (on 132 SMs every preferred T lands). K tails: K mod 32 in {0, 2, 30} for
# the 16-byte producer with packed rows, {1, 31} for its 8-byte cp.async tail with a single row (M = 1: the row pointer is J itself,
# 16-byte aligned, whatever K), {1, 15, 17, 31} for the 8-byte producer.
CASES = [
    ("lanes, R = 0", "ws", 4126, 0, 2), ("lanes, R = 0", "ws", 6002, 84, 3), ("lanes, R = 0", "ws", 12288, 8, 11),
    ("lanes, R > 0", "ws", 8194, 12, 4), ("lanes, R > 0", "ws", 9214, 0, 6), ("lanes, R > 0", "ws", 12000, 24, 8),
    ("lanes, R > 0", "ws", 12030, 52, 9),
    ("L = 1", "ws", 12002, 36, 12), ("L = 1", "ws", 12030, 20, 15),
    ("stream-K", "ws", 12288, 48, 16), ("stream-K", "ws", 12002, 0, 17),
    ("reduced G", "ws", 1600, 28, 1), ("reduced G", "ws", 1000, 56, 2),
    ("reduced G", "ws", 2017, 127, 1), ("reduced G", "ws", 2015, 127, 1),
    ("lanes, R = 0", "odd", 8193, 1, 3), ("lanes, R = 0", "odd", 4127, 84, 2),
    ("lanes, R > 0", "odd", 12017, 12, 4), ("lanes, R > 0", "odd", 8191, 40, 7),
    ("L = 1", "odd", 12015, 6, 12), ("L = 1", "odd", 12031, 20, 14),
    ("stream-K", "odd", 12001, 1, 16), ("stream-K", "odd", 12017, 0, 17),
    ("reduced G", "odd", 801, 28, 1), ("reduced G", "odd", 1041, 56, 2), ("reduced G", "odd", 783, 100, 1),
]


def case_shape(case, G):
    """(M, K) of a case on G SMs: M = 128 T - short for the T nearest the preferred one whose schedule is the named branch"""
    branch, producer, K, short, T0 = case
    for T in sorted(range(1, 25), key=lambda t: (abs(t - T0), t)):
        M = BM * T - short
        if M >= 1 and schedule_branch(M, K, G)[0] == branch:
            return M, K
    pytest.fail(f"no tile-row count puts K = {K} ({producer}) in the branch '{branch}' on {G} SMs")


@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{c[1]}-K{c[2]}" for c in CASES])
def test_condensation_meets_componentwise_bound(ctx, case):
    G = _G()
    branch, producer = case[0], case[1]
    M, K = case_shape(case, G)
    assert schedule_branch(M, K, G)[0] == branch
    # odd K makes packed rows 8-byte aligned (the 8-byte producer) unless there is a single row
    assert (K % 2 == 1 and M > 1) == (producer == "odd")
    P = synth.make_qn_problem(K, M, 0, seed=M + K)
    k, T = _setup(ctx, P)
    k.condense()
    assert k.condense_mode_used() == 0
    Nref, B = _reference(P, k.DhInv(), k.Dd_inv())
    margin = _check_N(k.N(), Nref, B, K, G)
    print(f"M={M} K={K} {producer}: {branch} ({schedule_branch(M, K, G)[1]} CTAs of {G} SMs), margin {margin:.3g}")
    k.close()


def test_every_schedule_branch_is_reached():
    """Every branch of build_schedule has a case of each producer on this device, and the 8-byte producer's cases cover K mod 32 in
    {1, 15, 17, 31} (restated arithmetic, not the kernels' results)."""
    G = _G()
    for producer in ("ws", "odd"):
        reached = {c[0] for c in CASES if c[1] == producer and case_shape(c, G)}
        assert reached == {"lanes, R = 0", "lanes, R > 0", "L = 1", "stream-K", "reduced G"}, (G, producer, reached)
    assert {c[2] % WBK for c in CASES if c[1] == "odd"} == {1, 15, 17, 31}


def _numpy_direction(P, DhInv, Dd_inv):
    """l = 0: dy = N^-1 (J DhInv rx - [ryc; ryd]), dx = DhInv (rx - J^T dy)"""
    J = P.J
    N = (J * DhInv) @ J.T
    N[np.arange(P.m_eq, P.m), np.arange(P.m_eq, P.m)] += Dd_inv
    rhs = J @ (DhInv * P.rx) - np.concatenate([P.ryc, P.ryd])
    dy = np.linalg.solve(N, rhs)
    return DhInv * (P.rx - J.T @ dy), dy[:P.m_eq], dy[P.m_eq:]


@pytest.mark.parametrize("T", [9, 16])
@pytest.mark.parametrize("extra", ["free", "new tile row"])
def test_fused_rhs_row_at_tile_edges(ctx, T, extra):
    """solveCompressed with the condensation pending folds J DhInv rx into the SYRK as row M when that row fits in the last tile
    (M = 128 T - 1) and takes the two-pass route when it would start a new tile row (M = 128 T). Both against the route with the
    condensation done first and against numpy."""
    M = 128 * T - (1 if extra == "free" else 0)
    P = synth.make_qn_problem(12000, M, 0, seed=T)
    out = {}
    for pending in (True, False):
        k, Td = _setup(ctx, P)
        if not pending:
            k.condense()
        dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
        assert k.solveCompressed(ctx.to_device(P.rx), Td["ryc"], Td["ryd"], dx, dyc, dyd)
        k.check()
        ctx.sync()
        out[pending] = [v.cpu().numpy().copy() for v in (dx, dyc, dyd)]
        DhInv, Dd_inv = k.DhInv(), k.Dd_inv()
        k.close()
    ref = _numpy_direction(P, DhInv, Dd_inv)
    for a, b, r in zip(out[True], out[False], ref):
        s = max(1.0, np.abs(r).max())
        assert np.abs(a - b).max() <= 1e-10 * s
        assert np.abs(a - r).max() <= 1e-9 * s


def test_schedule_cache_revisit_is_bit_identical(ctx):
    """Six distinct (M, K) keys through the 4-way LRU schedule cache, then the first again: bit-identical to its first visit and to a
    fresh context (the evicted way is rebuilt from scratch)."""
    from hiop_b200.engine import Context
    shapes = [(600, 8000), (300, 8002), (700, 6000), (130, 4000), (1000, 3000), (260, 5000)]
    probs = [synth.make_qn_problem(K, M, 0, seed=i) for i, (M, K) in enumerate(shapes)]
    first = None
    for i, P in enumerate(probs + probs[:1]):
        k, _ = _setup(ctx, P)
        k.condense()
        N = k.N().copy()
        k.close()
        if i == 0:
            first = N
    np.testing.assert_array_equal(N, first)
    c2 = Context(0)
    try:
        k, _ = _setup(c2, probs[0])
        k.condense()
        np.testing.assert_array_equal(k.N(), first)
        k.close()
    finally:
        c2.close()


# l > 0 with the S / Y rows across a tile boundary: N also carries the low-rank correction, so the criterion is diagonal-scaled,
# |N - N_oracle| <= TAU_L sqrt(N_ii N_jj). The measured error is printed as the margin TAU_L / err.
TAU_L = bounds.TAU_DIAG


@pytest.mark.parametrize("n,m,l", [(20000, 120, 6), (12002, 250, 4), (9001, 381, 2)])
def test_condensation_with_secant_rows_across_tiles(ctx, n, m, l):
    from oracle import kkt_oracle as ko
    P = synth.make_qn_problem(n, m, l, seed=n % 71)
    k, _ = _setup(ctx, P)
    k.condense()
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    No, _, _, _ = ko.condense(ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma))
    d = np.abs(np.diag(No))
    err = float((np.abs(k.N() - No) / np.sqrt(np.outer(d, d))).max())
    print(f"n={n} m={m} l={l}: diagonal-scaled error {err:.3g}, margin {TAU_L / max(err, 1e-300):.3g}")
    assert err <= TAU_L, err
    k.close()
