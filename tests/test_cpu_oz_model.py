"""Exactness claims of the int8-slice condensation (DESIGN.md section 3), checked on a numpy integer model of the device path
(oracle/oz_model.py): digit range, exact reconstruction of the operands, int32 accumulator bound per K chunk, and the error of the
truncated product against the FP64 Gram matrix for 6 / 7 / 8 slices."""
import numpy as np
import pytest

from oracle import oz_model as oz


def _B(M, K, seed, decades=3.0):
    r = np.random.default_rng(seed)
    return r.standard_normal((M, K)) * 10.0 ** r.uniform(-decades, decades, size=(M, 1)) * np.sqrt(10.0 ** r.uniform(-3, 3, size=(1, K)))


@pytest.mark.parametrize("S", [6, 7, 8])
def test_digits_are_int8_and_reconstruct_the_operand(S):
    B = _B(9, 4000, 1)
    B[3] = 0.0                                               # an all-zero row (exponent 0, all digits 0)
    B[5, 7] = np.abs(B[5]).max() * 4                         # the row maximum itself
    e = oz.row_exponents(B)
    Q = oz.slices(B, e, S)
    assert np.abs(Q).max() <= 64                             # |q| <= 64 (the MMA operands are int8)
    assert np.abs(Q[1:]).max() <= 64 and Q[1:].min() >= -64
    rec = sum(Q[p].astype(np.float64) * 2.0 ** (-(6 + 7 * p)) for p in range(S))
    b = np.ldexp(B, -e[:, None])
    grid = 2.0 ** (-(6 + 7 * (S - 1)))
    assert np.abs(rec - b).max() <= 0.5 * grid               # rounded to the last slice's grid ...
    np.testing.assert_array_equal(rec, np.round(b / grid) * grid)   # ... exactly (round-half-even of the magic-number add)
    assert np.all(Q[:, 3, :] == 0)


def test_int32_accumulator_bound_per_chunk():
    # worst case operands: every digit at its extreme -> (t+1) * Kc * 2^12 must stay below 2^31 with Kc = 2^19 / S
    # (hb_ozaki.cu takes chunks of 128-column stages and drops one stage when the product would reach 2^31 exactly: S = 8)
    for S in (6, 7, 8):
        stages = (524288 // S) // 128
        while S * stages * 128 * 4096 >= 2 ** 31:
            stages -= 1
        assert S * stages * 128 * 64 * 64 < 2 ** 31
        assert stages >= (524288 // S) // 128 - 1
    B = _B(4, 3000, 2)
    C, info = oz.gram(B, 8, chunk_cols=700)                  # several chunks: the result must not depend on the chunking
    C1, _ = oz.gram(B, 8, chunk_cols=3000)
    assert info["max_abs_int32_accumulator"] < 2 ** 31
    assert np.abs(C - C1).max() <= 1e-15 * np.abs(C1).max()


@pytest.mark.parametrize("S,tol", [(6, 2e-10), (7, 2e-12), (8, 5e-14)])
def test_truncated_product_error_against_fp64(S, tol):
    # the tolerances are the ones tests/test_gpu_ozaki.py holds the device path to
    B = _B(24, 20000, 3, decades=2.0)
    C, _ = oz.gram(B, S)
    ref = B @ B.T
    assert np.abs(C - ref).max() <= tol * np.abs(ref).max()
    assert np.array_equal(C, C.T)                            # symmetric by construction (same integer products both ways)


def test_fused_sweep_identity_for_step_2_of_solveCompressed():
    """The identity behind k_oz_rowmax_dot (DESIGN 3.3): with t = [J; S; Y] (DhInv .* rx),
    J (H+Dx)^-1 rx = t_J - Z [sigma t_S; t_Y],  Z = U V^-1,  U = [sigma J DhInv S^T, J DhInv Y^T]
    -- checked against the oracle's own hess_solve + J product (hiopKKTLinSys.cpp:1146-1157, hiopHessianLowRank.cpp:495-540)."""
    from hiop_b200 import synth
    from oracle import kkt_oracle as ko
    for n, m, l in ((3000, 25, 5), (1200, 40, 1), (900, 10, 0)):
        P = synth.make_qn_problem(n, m, l, seed=3 + l)
        Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
        st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
        want = st.J @ ko.hess_solve(st, P.rx)
        w = DhInv * P.rx
        t_J = st.J @ w
        got = t_J
        if l:
            _, _, S1, Y1 = ko.condense(st)
            U = np.hstack([S1, Y1])                              # S1 already carries sigma
            Z = st.Vfac.solve(U.T.copy()).T                      # m x 2l
            p = np.concatenate([P.sigma * (P.St @ w), P.Yt @ w])
            got = t_J - Z @ p
        assert np.abs(got - want).max() <= 1e-11 * max(1.0, np.abs(want).max())


# ---- the schedule, the bit-exact model and the a-priori bound (oz_model.schedule / condense_bits / truncation_bound) -----------------

@pytest.mark.parametrize("G", [114, 132])
def test_every_schedule_branch_is_reached(G):
    """H100 PCIe (114 SMs) and SXM (132 SMs): every branch of hb_syrk_rows_ozaki's schedule has a case, and on 132 SMs the preferred
    shapes are the ones the kernel's comments and tests name."""
    got = {}
    for b, M0, K, S in oz.BRANCH_CASES:
        M = oz.find_shape(b, M0, K, S, G)
        got[b] = oz.schedule(M, K, S, G)
        if G == 132:
            assert M == M0, (b, M)
    assert set(got) == set(oz.BRANCHES)
    if G == 132:
        assert oz.schedule(100, 20000, 8, 132).splits == 33
        assert oz.schedule(100, 1000, 8, 132).splits == 8 and oz.schedule(1, 5000, 8, 132).splits == 40
        s = oz.schedule(1000, 200001, 8, 132)
        assert (s.splits, len(s.items)) == (11, 1584)
        assert len(oz.schedule(1000, 12000, 8, 132).items) == 144
        assert oz.schedule(1260, 140001, 8, 132).max_chunks == 3 and oz.schedule(1260, 140001, 6, 132).max_chunks == 2
    assert oz.chunk_stages(8) == 511 and oz.chunk_stages(8) * 128 == 65408


def test_items_cover_every_tile_and_stage_once():
    for M, K, S, G in ((1000, 200001, 8, 132), (300, 470001, 8, 114), (33, 4223, 7, 132), (1, 100, 6, 132)):
        s = oz.schedule(M, K, S, G)
        cover = {}
        for bi, bj, kb, kc, slot in s.items:
            assert kc >= 1 and 0 <= slot < len(s.tiles) * s.splits
            cover.setdefault((bi, bj), []).append((kb, kc))
        assert set(cover) == set(s.tiles)
        for ranges in cover.values():
            ranges.sort()
            assert ranges[0][0] == 0 and sum(c for _, c in ranges) == s.kstages
            assert all(a + c == b for (a, c), (b, _) in zip(ranges, ranges[1:]))


def _adversarial(M, K, seed):
    """rows at 2^-1000 (the row scaling then needs two steps), 1e+-150, an all-zero row, a row with a power-of-two maximum and one whose
    maximum rounds the first digit word up to 2^27, among rows spanning 6 decades"""
    B = _B(M, K, seed)
    B[1] *= 2.0 ** -1000 / np.abs(B[1]).max()
    B[2] *= 1e150
    B[3] *= 1e-150
    B[4] = 0.0
    B[5, 11] = 2.0 ** np.ceil(np.log2(np.abs(B[5]).max()) + 1)
    B[6] *= 0.25 / np.abs(B[6]).max()
    B[6, 7] = 1.0 - 2.0 ** -30
    return B


@pytest.mark.parametrize("S", [6, 7, 8])
def test_truncation_bound_holds_on_adversarial_rows_and_is_not_vacuous(S):
    B = _adversarial(12, 3000, 4)
    e, Q = oz.digits(B, S)
    assert oz.row_exponents(B)[1] == -999 and Q[0, 6].max() == 64
    sch = oz.schedule(12, 3000, S, 132)
    C = oz.condense_bits(B, S, sch, dig=(e, Q))
    assert np.all(np.isfinite(C)) and np.array_equal(C, C.T)
    G, err = oz.exact_gram(B)
    R, _ = oz.truncation_bound(B, S, sch.chain, dig=(e, Q))
    tol = np.ldexp(R, e[:, None] + e[None, :]) + 2.0 ** -1075 + err
    ratio = np.abs(C - G) / tol
    assert ratio.max() <= 1.0, ratio.max()
    # not vacuous: the bound is within 100x of the error somewhere, and dropping the last anti-diagonal breaks it
    assert ratio.max() >= 1e-2, ratio.max()
    Cd = oz.condense_bits(B, S, sch, dig=(e, Q), drop_t=S - 1)
    assert (np.abs(Cd - G) / tol).max() > 1.0
    # the row at 2^-1000 is sliced exactly like any other row: its digits are those of the row scaled to 1
    e1, Q1 = oz.digits(np.ldexp(B[1:2], 1000), S)         # max 2^-1000 = 0.5 2^-999: e = -999 <= -997
    np.testing.assert_array_equal(Q1[:, 0], Q[:, 1])


def test_mutations_change_the_bits():
    """Dropping anti-diagonal S-1, summing the splits in reverse order or cutting K into 65536-column chunks (instead of the device's
    65408) each changes condense_bits on seeded inputs: the bit-exact GPU comparison would catch each of these kernels."""
    B = _B(100, 20000, 5)
    S = 8
    sch = oz.schedule(100, 20000, S, 132)
    assert sch.splits == 33
    dig = oz.digits(B, S)
    C = oz.condense_bits(B, S, sch, dig=dig)
    assert not np.array_equal(C, oz.condense_bits(B, S, sch, dig=dig, drop_t=S - 1))
    assert not np.array_equal(C, oz.condense_bits(B, S, sch, dig=dig, split_order=range(sch.splits - 1, -1, -1)))
    B2 = _B(16, 70000, 6)
    C1, _ = oz.gram(B2, S)
    C2, _ = oz.gram(B2, S, chunk_cols=65536)
    assert not np.array_equal(C1, C2)
    sch2 = oz.schedule(16, 70000, S, 1)                      # one SM: one split, the device's two chunks
    assert sch2.splits == 1 and sch2.max_chunks == 2
    np.testing.assert_array_equal(oz.condense_bits(B2, S, sch2), C1)
