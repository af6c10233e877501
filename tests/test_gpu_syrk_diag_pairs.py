"""k_syrk_ws's diagonal pairs, held to exact arithmetic on every tile-row count from 1 to 17.

A CTA of the FP64 condensation computes two diagonal tiles at once, only their 16x16 cells on and above the diagonal, and the schedule
weighs such a pair at 144 fragments against a full tile's 128. With an even tile-row count T every diagonal tile is paired; with an odd
T the last one runs alone as a full tile. With integer J and a power-of-two DhInv (see test_gpu_syrk_dmma16.py) every entry of N and of
the fused rhs dots is exact in any summation order, so a cell of a pair read from the wrong shared-memory rows, written to the wrong
slot or position, or dropped by the schedule shows up as a wrong entry. Odd K runs the 8-byte producer. With secant memory (l > 0) the
S and Y rows start inside a pair: there N carries the low-rank correction and is held to the diagonal-scaled oracle bound."""
import numpy as np
import pytest

from test_gpu_syrk_dmma16 import _exact_problem, _exact_reference, _run
from test_gpu_syrk_schedule import _setup, ctx  # noqa: F401  (ctx is a fixture)
from oracle import bounds

pytestmark = pytest.mark.gpu

BM = 128

# (T, rows short of a full last tile, K): every T from 1 to 17, K tails mod 32 in {0, 1, 2, 15, 17, 30, 31}, K = 200 and 400 leave
# fewer unit iterations than SMs
EXACT = [(1, 28, 4126), (2, 0, 4126), (2, 56, 200), (3, 1, 400), (3, 84, 6001), (4, 12, 8194), (5, 0, 5007), (6, 0, 9214), (7, 40, 8191),
         (8, 11, 6000), (9, 52, 6030), (10, 1, 4097), (11, 8, 4096), (12, 36, 4002), (13, 3, 3001), (14, 20, 4031), (15, 20, 4030),
         (16, 48, 4002), (17, 0, 4015)]


@pytest.mark.parametrize("T,short,K", EXACT, ids=[f"T{t}-M{BM * t - s}-K{k}" for t, s, k in EXACT])
def test_pairs_condensation_is_exact(ctx, T, short, K):
    M = BM * T - short
    P = _exact_problem(M, K, seed=M + K)
    N, _, DhInv, Dd_inv = _run(ctx, P, fused=False)
    Nref, _ = _exact_reference(P, DhInv, Dd_inv)
    bad = np.argwhere(N != Nref)
    assert bad.size == 0, f"M={M} K={K}: {len(bad)} wrong entries, first at {bad[0].tolist()}: {N[tuple(bad[0])]} != {Nref[tuple(bad[0])]}"


# the rhs row as row M: in the paired last tile (M = 1012, M = 128 T - 1 for even T) and in the unpaired one (odd T)
FUSED = [(1012, 6000), (1012, 6001), (BM * 4 - 1, 4002), (BM * 10 - 1, 4017), (BM * 5 - 1, 4030), (BM * 1 - 1, 3001)]


@pytest.mark.parametrize("M,K", FUSED, ids=[f"M{m}-K{k}" for m, k in FUSED])
def test_pairs_fused_row_is_exact(ctx, M, K):
    P = _exact_problem(M, K, seed=K)
    N, tdot, DhInv, Dd_inv = _run(ctx, P, fused=True)
    Nref, tref = _exact_reference(P, DhInv, Dd_inv)
    assert np.array_equal(N, Nref), int((N != Nref).sum())
    assert np.array_equal(tdot[:M], tref), int((tdot[:M] != tref).sum())


def test_pairs_are_bit_identical_run_to_run(ctx):
    from hiop_b200 import synth
    P = synth.make_qn_problem(20001, 1000, 6, seed=3)
    out = []
    for _ in range(2):
        k, _ = _setup(ctx, P)
        k.condense()
        out.append(k.N().copy())
        k.close()
    assert np.array_equal(out[0], out[1])


# m + 2l rows with the secant rows crossing the boundary inside a pair (tiles 2p | 2p + 1) and, at m = 1000, in the paired last tile
@pytest.mark.parametrize("n,m,l", [(12001, 375, 6), (9000, 635, 4), (8002, 1000, 6)])
def test_pairs_with_secant_rows(ctx, n, m, l):
    from hiop_b200 import synth
    from oracle import kkt_oracle as ko
    P = synth.make_qn_problem(n, m, l, seed=n % 67)
    k, _ = _setup(ctx, P)
    k.condense()
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    No, _, _, _ = ko.condense(ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma))
    d = np.abs(np.diag(No))
    err = float((np.abs(k.N() - No) / np.sqrt(np.outer(d, d))).max())
    assert err <= bounds.TAU_DIAG, err
    assert np.array_equal(k.N(), k.N().T)
    k.close()
