"""FP64 DMMA condensation (k_syrk_ws): odd row / column counts through the K-lane schedule, and the right-hand-side row folded into
the same pass (J (H+Dx)^-1 rx without a second sweep over J) against the two-pass route and the oracle."""
import numpy as np
import pytest
import torch

from hiop_b200 import synth
from oracle import bounds
from oracle import kkt_oracle as ko

pytestmark = pytest.mark.gpu


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
    J = D(P.J)
    T = {name: D(getattr(P, name)) for name in ("ixl", "ixu", "idl", "idu", "zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu", "St", "Yt", "ryc", "ryd")}
    T["J"] = J
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(J[:P.m_eq], J[P.m_eq:])
    k.set_secant(P.sigma, T["St"] if P.l else None, T["Yt"] if P.l else None, P.L, P.D)
    k.set_condense_mode(0)
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["vl"], T["sdl"], T["vu"], T["sdu"])
    return k, T


def _oracle_state(P):
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    return ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)


# m + 2l = 1, 7, 127, 128, 129, 257 rows (tile-row boundaries, one to three 128-row tiles) and K = n from 1 column to a ragged tail
@pytest.mark.parametrize("n,m,l", [(1, 1, 0), (31, 7, 0), (33, 9, 0), (300, 127, 0), (4099, 116, 6), (62501, 129, 0), (20003, 251, 3), (7, 3, 2)])
def test_condensation_odd_shapes_match_oracle(ctx, n, m, l):
    P = synth.make_qn_problem(n, m, l, seed=3 + n % 89)
    k, T = _setup(ctx, P)
    k.condense()
    assert k.condense_mode_used() == 0
    N = k.N()
    st = _oracle_state(P)
    No, _, _, _ = ko.condense(st)
    assert np.array_equal(N, N.T)
    # componentwise for l = 0, diagonal-scaled with the secant rows (oracle/bounds.py)
    ratio = bounds.condensed_error_ratio(N, No, st.J, st.DhInv, l, torch.cuda.get_device_properties(0).multi_processor_count)
    assert ratio <= 1.0, ratio
    k.close()


# the shapes of the int8-slice fused-sweep test, plus m + 2l = 128 (the extra row would need a new tile row: two-pass route) and 1023
@pytest.mark.parametrize("n,m,l", [(40000, 90, 4), (33001, 70, 3), (40960, 64, 0), (300, 66, 2), (30000, 116, 6), (20000, 1011, 6)])
@pytest.mark.parametrize("rx_offset", [0, 1])
def test_fused_rhs_row_delivers_the_same_direction(ctx, n, m, l, rx_offset):
    """solveCompressed with a pending FP64 condensation takes J DhInv rx as one more row of the SYRK when that is free (rx 16-byte
    aligned, no extra tile row); with the condensation already done it takes the two-pass route. Same direction either way; a second
    rhs on the same factor does not reuse the dots of the first."""
    P = synth.make_qn_problem(n, m, l, seed=n % 97)
    res = {}
    for pending in (True, False):
        k, T = _setup(ctx, P)
        if not pending:
            k.condense()
        # rx_offset = 1: rx starts 8 bytes into its buffer -> not 16-byte aligned -> never fused
        buf = ctx.to_device(np.concatenate([np.zeros(rx_offset), P.rx]))
        rx = buf[rx_offset:]
        dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
        assert k.solveCompressed(rx, T["ryc"], T["ryd"], dx, dyc, dyd)
        k.check()
        ctx.sync()
        assert k.condense_mode_used() == 0
        res[pending] = [v.cpu().numpy().copy() for v in (dx, dyc, dyd)]
        rx2 = ctx.to_device(P.rx[::-1].copy())
        dx2, dyc2, dyd2 = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
        assert k.solveCompressed(rx2, T["ryc"], T["ryd"], dx2, dyc2, dyd2)
        ctx.sync()
        res[(pending, 2)] = [v.cpu().numpy().copy() for v in (dx2, dyc2, dyd2)]
        k.close()
    for a, b in zip(res[True] + res[(True, 2)], res[False] + res[(False, 2)]):
        assert np.abs(a - b).max() <= 1e-10 * max(1.0, np.abs(b).max())
    dxo, dyco, dydo, _ = ko.solve_compressed(_oracle_state(P), P.rx, P.ryc, P.ryd)
    assert np.abs(res[True][0] - dxo).max() <= 1e-9 * max(1.0, np.abs(dxo).max())
    assert np.abs(res[True][2] - dydo).max() <= 1e-9 * max(1.0, np.abs(dydo).max())
