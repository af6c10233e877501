"""The Chinese-remainder int8 condensation (HB_CONDENSE_INT8_CRT, hb_crt.cu) held to its Python-integer model bit for bit.

With no secant memory (l = 0) the condensed matrix is N = C + blkdiag(0, Dd_inv), C = ldexp(RN(X), e_i + e_j - 2t) with X = q q^T the exact
integer Gram of the rows of B = J diag(sqrt(DhInv)) rounded to t(K) bits. X is formed from residues, which add exactly in any order, so
oracle/crt_model.condense_bits predicts N exactly whatever the tile schedule, the K splits or the int32 chunks, and every case asserts
np.array_equal. Each case also prints its margin against the exact B B^T (oz_model.exact_gram) under crt_model.bound."""
import os
from math import prod

import numpy as np
import pytest
import torch

from hiop_b200 import _lib, synth
from oracle import crt_model as crt
from oracle import kkt_oracle as ko
from oracle import oz_model as oz
from test_gpu_parity import _as_dict, _relerr, _run_solve, _setup_kkt

pytestmark = pytest.mark.gpu

CRT = 100
DEV = "cuda"
ITERATE = ("zl", "sxl", "zu", "sxu", "vl", "sdl", "vu", "sdu")


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _setup(ctx, P, J=None, mode=CRT):
    """l = 0, condensation mode `mode`; J: the device Jacobian to register (default: a contiguous copy of P.J)"""
    from hiop_b200.engine import KKTLinSysLowRank
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, 1)
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ITERATE + ("ixl", "ixu", "idl", "idu")}
    T["J"] = D(P.J) if J is None else J
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    k.set_jacobian(T["J"][:P.m_eq], T["J"][P.m_eq:])
    k.set_secant(P.sigma, None, None, P.L, P.D)
    k.set_condense_mode(mode)
    k.update(*(T[kk] for kk in ITERATE))
    return k, T


def _model(J, DhInv, Dd_inv, meq):
    B = J * np.sqrt(DhInv)
    N = crt.condense_bits(B, device=DEV)
    i = np.arange(meq, J.shape[0])
    N[i, i] = N[i, i] + Dd_inv
    return N, B


def _margin(N, B, Dd_inv, meq):
    """min over the entries of bound / |N - exact|: > 1 when N meets crt_model.bound"""
    G, err = oz.exact_gram(B, device=DEV)
    i = np.arange(meq, B.shape[0])
    ref = G.copy()
    ref[i, i] = ref[i, i] + Dd_inv
    C = N.copy()
    C[i, i] = C[i, i] - Dd_inv
    tol = crt.bound(B, C, device=DEV) + err + 2 * 2.0 ** -53 * (np.abs(N) + np.abs(ref))   # + the rounding of k_form_N's Dd_inv add
    ratio = float((np.abs(N - ref) / tol).max())
    assert ratio <= 1.0, ratio
    return 1.0 / max(ratio, 1e-300)


def _run(ctx, P, label, J=None, mutate=None):
    k, T = _setup(ctx, P, J)
    if mutate is not None:
        mutate(k, T)
    k.condense()
    assert k.condense_mode_used() == CRT
    N = k.N()
    DhInv, Dd_inv = k.DhInv(), k.Dd_inv()
    Jh = T["J"].cpu().numpy()
    k.close()
    Nm, B = _model(Jh, DhInv, Dd_inv, P.m_eq)
    bad = np.argwhere(N != Nm)
    assert bad.size == 0, (label, len(bad), bad[:5].tolist(), N[tuple(bad[0])] if bad.size else None, Nm[tuple(bad[0])] if bad.size else None)
    margin = _margin(N, B, Dd_inv, P.m_eq)
    K = B.shape[1]
    print(f"{label}: M={B.shape[0]} K={K} t={crt.bits(K)} N={crt.n_moduli(K)}: bit-exact, margin {margin:.3g}")
    return N


@pytest.fixture
def max_splits():
    """sets HB_CRT_MAX_SPLITS for one test (read when the work list is built)"""
    old = os.environ.get("HB_CRT_MAX_SPLITS")

    def set_(v):
        os.environ["HB_CRT_MAX_SPLITS"] = str(v)
    yield set_
    if old is None:
        os.environ.pop("HB_CRT_MAX_SPLITS", None)
    else:
        os.environ["HB_CRT_MAX_SPLITS"] = old


# ---- shapes: M around the 128-row tile, K around the 128-column stage, one and several splits, fewer items than SMs --------------

@pytest.mark.parametrize("M,K", [(1, 5000), (31, 5000), (127, 5000), (128, 5000), (129, 5000), (1000, 5000),   # M; 1000: one split
                                 (40, 77), (64, 128 * 40), (64, 128 * 40 + 1), (64, 128 * 41 - 1), (33, 9999),   # K < 128, K mod 128, odd
                                 (64, 100000),                                                                  # several splits
                                 (1, 200),                                                                      # 15 items < SMs
                                 (6, 8)])                                                                       # K <= 8: 14 moduli
def test_condensation_equals_integer_model(ctx, M, K):
    _run(ctx, synth.make_qn_problem(K, M, 0, seed=M + K), f"M{M}-K{K}")


def test_unaligned_rows_take_the_scalar_residue_path(ctx):
    P = synth.make_qn_problem(6000, 40, 0, seed=3)
    buf = torch.zeros(P.J.size + 1, dtype=torch.float64, device=DEV)
    J = buf[1:].view(P.J.shape)                                   # one double off a 16-byte boundary
    J.copy_(torch.from_numpy(P.J))
    assert J.data_ptr() % 16 == 8
    _run(ctx, P, "unaligned J", J=J)


@pytest.mark.parametrize("K", [130944, 130945])
def test_k_across_the_int32_chunk_boundary_in_one_split(ctx, max_splits, K):
    """1023 stages of 128 columns are one exact int32 chunk: K = 130945 needs a second chunk (one split forced), and the bits are those
    of the default split count"""
    P = synth.make_qn_problem(K, 64, 0, seed=K)
    max_splits(1)
    N1 = _run(ctx, P, f"one split, K{K}")
    max_splits(16)
    N16 = _run(ctx, P, f"default splits, K{K}")
    assert np.array_equal(N1, N16)


def _top_of_binade(sd):
    """a with fl(a sd) in [1 - 2^-52, 1) in every column (a few ulp steps of a from (1 - 2^-53) / sd, the device's product rounding)"""
    a = (1.0 - 2.0 ** -53) / sd
    for _ in range(16):
        b = a * sd
        a = np.where(b >= 1.0, np.nextafter(a, 0.0), np.where(b < 1.0 - 2.0 ** -52, np.nextafter(a, np.inf), a))
    b = a * sd
    assert np.all((b >= 1.0 - 2.0 ** -52) & (b < 1.0)), int(np.sum((b < 1.0 - 2.0 ** -52) | (b >= 1.0)))
    return a


@pytest.mark.parametrize("K", [340108, 340109])
def test_k_across_the_16_to_17_moduli_switch(ctx, K):
    """Row 0 at the top of its binade in every column: q = 2^53 - 1 or 2^53 - 2, |X_00| ~ K 2^106. At K = 340109 that exceeds P16/2 ~
    340108.65 2^106, so the 17th Garner digit (weight above 2^64) is non-zero and the 128-bit sum wraps; at K = 340108 it does not."""
    assert crt.n_moduli(K) == (16 if K == 340108 else 17)
    P = synth.make_qn_problem(K, 40, 0, seed=K)
    half16 = prod(crt.MODULI[:16]) // 2

    def worst(k, T):
        sd = np.sqrt(k.DhInv())
        a = _top_of_binade(sd)
        T["J"][0] = torch.from_numpy(a).to(DEV)
        X00 = crt.brute_force_x((a * sd)[None, :])[0, 0]
        assert (X00 > half16) == (K == 340109), (X00, half16)
    _run(ctx, P, f"moduli switch K{K}", mutate=worst)


def test_extreme_rows(ctx):
    """the small and zero rows are inequality rows: Dd_inv keeps N positive definite"""
    P = synth.make_qn_problem(20000, 48, 0, seed=17)
    meq = P.m_eq

    def extreme(k, T):
        J = T["J"]
        J[meq + 1] *= 1e-303
        J[2] *= 1e150
        J[meq + 3] *= 1e-150
        J[meq + 4] = 0.0
        # a power-of-two row maximum: b_5k = a_5k sqrt(DhInv_k) = 2^40 exactly in one column (found on the host with the same products)
        sd = np.sqrt(k.DhInv())
        for col in range(len(sd)):
            a = np.ldexp(1.0, 40) / sd[col]
            if a * sd[col] == np.ldexp(1.0, 40):
                J[5, col] = float(a)
                break
        else:
            raise AssertionError("no column gives an exact power of two")
    _run(ctx, P, "extreme rows", mutate=extreme)


# ---- reproducibility --------------------------------------------------------------------------------------------------------------

def test_repeated_calls_second_context_and_revisited_shape_are_bit_identical(ctx):
    from hiop_b200.engine import Context
    P = synth.make_qn_problem(50000, 200, 0, seed=4)
    k, T = _setup(ctx, P)
    k.condense()
    N0 = k.N()
    for _ in range(2):
        k.update(*(T[kk] for kk in ITERATE))
        k.condense()
        assert np.array_equal(k.N(), N0)
    P2 = synth.make_qn_problem(7000, 33, 0, seed=5)                # another shape, then back
    k2, _ = _setup(ctx, P2)
    k2.condense()
    k2.close()
    k.update(*(T[kk] for kk in ITERATE))
    k.condense()
    assert np.array_equal(k.N(), N0)
    k.close()
    c2 = Context(0)
    k3, _ = _setup(c2, P)
    k3.condense()
    assert np.array_equal(k3.N(), N0)
    k3.close()
    c2.close()


# ---- the rest of the quasi-Newton step in CRT mode -------------------------------------------------------------------------------

def test_fused_rhs_row_and_secant_memory(ctx):
    """A pending CRT condensation + solveCompressed (the row-maximum sweep delivers J (H+Dx)^-1 rx), with l = 6: the direction matches
    the oracle, and N matches the FP64 mode within the bound of the rounded operands"""
    P = synth.make_qn_problem(40000, 120, 6, seed=8)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    k.set_condense_mode(CRT)
    k.update(*(T[kk] for kk in ITERATE))
    dx, dyc, dyd = _run_solve(ctx, k, p)
    assert k.condense_mode_used() == CRT
    Nc = k.N()
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    dxo, dyco, dydo, _ = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    errs = (_relerr(dx, dxo), _relerr(dyc, dyco), _relerr(dyd, dydo))
    assert max(errs) <= 1e-8, errs
    k.set_condense_mode(0)
    k.update(*(T[kk] for kk in ITERATE))
    k.condense()
    Nf = k.N()
    k.close()
    # C_aug entries move by at most (|b_i| |b_j| 2^-t + ...) relative to sqrt(C_ii C_jj); N inherits that through V^-1 (well conditioned here)
    d = np.sqrt(np.abs(np.diag(Nf)))
    rel = float((np.abs(Nc - Nf) / np.outer(d, d)).max())
    print(f"l = 6: direction errors {max(errs):.2e}, |N_crt - N_fp64| / sqrt(N_ii N_jj) <= {rel:.2e}")
    assert rel <= 1e-13, rel


def test_lsq_duals_in_crt_mode(ctx):
    P = synth.make_qn_problem(40000, 100, 0, seed=5 + 40000)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    k.set_condense_mode(CRT)
    g = np.random.default_rng(9).standard_normal(P.n)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(ctx.to_device(g), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, g, P.zl, P.zu, P.vl, P.vu)
    for a, b in ((yc.cpu().numpy(), yco), (yd.cpu().numpy(), ydo)):
        assert np.abs(a - b).max(initial=0.0) <= 1e-10 * max(1.0, np.abs(b).max(initial=0.0))
    k.close()


def test_host_jacobian_is_refused_and_the_handle_still_condenses_in_fp64(ctx):
    from hiop_b200.engine import KKTLinSysLowRank
    P = synth.make_qn_problem(5000, 30, 0, seed=2)
    k = KKTLinSysLowRank(ctx, P.n, P.m_eq, P.m_ineq, 1)
    D = ctx.to_device
    T = {name: D(getattr(P, name)) for name in ITERATE + ("ixl", "ixu", "idl", "idu")}
    k.set_patterns(T["ixl"], T["ixu"], T["idl"], T["idu"])
    Jh = torch.from_numpy(np.ascontiguousarray(P.J)).pin_memory()
    k.set_jacobian_host(Jh[:P.m_eq], Jh[P.m_eq:])
    k.set_secant(P.sigma, None, None, P.L, P.D)
    L = _lib.lib()
    assert L.hb_lowrank_set_condense_mode(k.h, CRT) == -1
    assert b"int8" in L.hb_last_error()
    k.update(*(T[kk] for kk in ITERATE))
    k.condense()
    assert k.condense_mode_used() == 0
    DhInv, Dd_inv = k.DhInv(), k.Dd_inv()
    N = k.N()
    k.close()
    ref = (P.J * DhInv) @ P.J.T
    i = np.arange(P.m_eq, P.J.shape[0])
    ref[i, i] += Dd_inv
    assert np.abs(N - ref).max() <= 1e-12 * np.abs(ref).max()


def test_resources_return_to_baseline_after_destroy():
    from hiop_b200.engine import Context
    live0 = _lib.lib().hb_debug_live_resources()
    c = Context(0)
    c.enable_timing(True)
    c.phase_timeline(True)
    P = synth.make_qn_problem(9000, 70, 0, seed=6)
    k, _ = _setup(c, P)
    k.condense()
    c.phase_timeline(False)
    k.close()
    c.close()
    assert _lib.lib().hb_debug_live_resources() == live0
