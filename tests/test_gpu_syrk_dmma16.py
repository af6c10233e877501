"""k_syrk_ws on the m16n8k16 FP64 MMA, held to exact arithmetic and to the instruction it was written for.

With integer rows |J| <= 2^7, DhInv = 1/(sigma + Dx) a power of two (sigma = 1, Dx in {1, 3, 7}), Dd_inv in {1, 1/2, 1/4} and
K < 2^14, every product J_ik DhInv_k J_jk is a multiple of 2^-3 of magnitude at most 2^13, so every partial sum, in any order, is a
multiple of 2^-3 below 2^27 and exact. So N and
the fused row dots tdot = J (DhInv .* rx) (integer rx) must equal the exact result bit for bit, whatever order the tensor core sums in:
an A or B fragment element read from the wrong row, column or K slot, a missed K tail or a lost accumulator shows up as a wrong entry
that a tolerance would hide. The cases reach every branch of build_schedule on the running device with both producers of k_syrk_ws: even
K (16-byte copies, K mod 32 in {0, 2, 16, 30}) and odd K with several rows (8-byte copies, K mod 32 in {1, 15, 17, 31}), diagonal and
off-diagonal tiles, and the fused rhs row at M = 1012.

The SASS check runs without a GPU: both instantiations of k_syrk_ws in the built library issue DMMA.16x8x16 only (DMMA.8x8x4 is the
half-rate shape on sm_90a) and have no local-memory traffic (a register spill would show as LDL / STL); no kernel of hb_syrk.cu
issues DMMA.8x8x4."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from hiop_b200 import synth
from test_gpu_syrk_schedule import _G, _setup, case_shape, ctx, schedule_branch  # noqa: F401  (ctx is a fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (branch, K, rows short of a full last tile, preferred tile-row count T); the T is moved to the nearest one whose schedule is the
# named branch on this device, as in test_gpu_syrk_schedule.py. Odd K (every M here is > 1) runs the 8-byte producer.
CASES = [
    ("lanes, R = 0", 4126, 0, 2), ("lanes, R = 0", 12288, 8, 11),
    ("lanes, R > 0", 8194, 12, 4), ("lanes, R > 0", 12016, 24, 8),
    ("L = 1", 12030, 36, 12), ("L = 1", 12000, 20, 15),
    ("stream-K", 12288, 48, 16), ("stream-K", 12018, 0, 17),
    ("reduced G", 1600, 28, 1), ("reduced G", 1040, 56, 2),
    ("lanes, R = 0", 12001, 0, 2), ("lanes, R > 0", 12015, 24, 8), ("L = 1", 12017, 36, 12),
    ("stream-K", 12031, 0, 17), ("reduced G", 1041, 56, 2), ("reduced G", 1583, 28, 1),
]


def _exact_problem(M, K, seed):
    """l = 0 problem whose condensation is exact in FP64: integer J and rx, power-of-two DhInv, exact Dd_inv"""
    P = synth.make_qn_problem(K, M, 0, seed=seed)
    r = np.random.default_rng(seed + 7)
    J = r.integers(-128, 129, size=(M, K)).astype(np.float64)
    P.Jc, P.Jd = np.ascontiguousarray(J[:P.m_eq]), np.ascontiguousarray(J[P.m_eq:])
    P.ixu = np.zeros(K)
    P.sxl, P.zl = np.ones(K), r.choice([1.0, 3.0, 7.0], K)
    P.sxu, P.zu = np.ones(K), np.zeros(K)
    P.idu = np.zeros(P.m_ineq)
    P.sdl, P.vl = np.ones(P.m_ineq), r.choice([1.0, 2.0, 4.0], P.m_ineq)
    P.sdu, P.vu = np.ones(P.m_ineq), np.zeros(P.m_ineq)
    P.rx = r.integers(-128, 129, size=K).astype(np.float64)
    return P


def _exact_reference(P, DhInv, Dd_inv):
    assert set(np.unique(DhInv)) <= {0.5, 0.25, 0.125}
    assert set(np.unique(Dd_inv)) <= {1.0, 0.5, 0.25}
    J = P.J
    N = (J * DhInv) @ J.T   # exact in any summation order, so BLAS gives the exact result too
    N[np.arange(P.m_eq, P.m), np.arange(P.m_eq, P.m)] += Dd_inv
    return N, J @ (DhInv * P.rx)


def _run(ctx, P, fused):
    """N (and tdot when `fused`: solveCompressed with the condensation pending folds DhInv .* rx into the SYRK as row M)"""
    k, T = _setup(ctx, P)
    tdot = None
    if fused:
        dx, dyc, dyd = [ctx.zeros(s) for s in (P.n, P.m_eq, P.m_ineq)]
        assert k.solveCompressed(ctx.to_device(P.rx), T["ryc"], T["ryd"], dx, dyc, dyd)
        k.check()
        ctx.sync()
        tdot = k.tdot()
    else:
        k.condense()
    assert k.condense_mode_used() == 0
    out = (k.N().copy(), tdot, k.DhInv(), k.Dd_inv())
    k.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-K{c[1]}" for c in CASES])
def test_ws_condensation_is_exact(ctx, case):
    G = _G()
    branch, K, short, T0 = case
    M, K = case_shape((branch, "ws" if K % 2 == 0 else "odd", K, short, T0), G)
    assert schedule_branch(M, K, G)[0] == branch and M > 1
    P = _exact_problem(M, K, seed=M + K)
    N, _, DhInv, Dd_inv = _run(ctx, P, fused=False)
    Nref, _ = _exact_reference(P, DhInv, Dd_inv)
    bad = np.argwhere(N != Nref)
    assert bad.size == 0, f"M={M} K={K}: {len(bad)} wrong entries, first at {bad[0].tolist()}: {N[tuple(bad[0])]} != {Nref[tuple(bad[0])]}"


@pytest.mark.gpu
@pytest.mark.parametrize("K", [12000, 12002, 12016, 12030, 12001, 12031])
def test_ws_fused_row_is_exact(ctx, K):
    """M = 1012: the rhs row is row 1012 of the eighth tile row (no extra tile), its dots go to tdot; odd K runs the 8-byte producer"""
    M = 1012
    P = _exact_problem(M, K, seed=K)
    N, tdot, DhInv, Dd_inv = _run(ctx, P, fused=True)
    Nref, tref = _exact_reference(P, DhInv, Dd_inv)
    assert np.array_equal(N, Nref), int((N != Nref).sum())
    assert np.array_equal(tdot[:M], tref), int((tdot[:M] != tref).sum())


def _library_sass():
    """{mangled kernel name: SASS} of hiop_b200/libhiopb200.so"""
    lib = os.path.join(ROOT, "hiop_b200", "libhiopb200.so")
    out = subprocess.run(["cuobjdump", "-sass", lib], check=True, capture_output=True, text=True).stdout
    blocks = re.split(r"\n\s*Function : ", out)
    return {b.split("\n", 1)[0].strip(): b for b in blocks[1:]}


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_syrk_sass_is_dmma16x8x16_without_spills():
    if not os.path.exists(os.path.join(ROOT, "hiop_b200", "libhiopb200.so")):
        pytest.skip("libhiopb200.so not built")
    sass = _library_sass()
    ws = {name: body for name, body in sass.items() if "k_syrk_wsILb" in name}
    assert sorted(re.search(r"k_syrk_wsILb(\d)", name).group(1) for name in ws) == ["0", "1"], sorted(ws)
    for name, body in ws.items():
        shapes = set(re.findall(r"\bDMMA\.(\w+)", body))
        assert shapes == {"16x8x16"}, (name, shapes)
        assert not re.search(r"\b(LDL|STL)\b", body), name
    assert not [name for name in sass if "k_syrk_diag" in name]
    syrk = {name: body for name, body in sass.items() if "_hb_syrk_cu_" in name}
    assert len(syrk) == 3, sorted(syrk)  # the two k_syrk_ws instantiations and k_syrk_fixup
    assert not [name for name, body in syrk.items() if "DMMA.8x8x4" in body]
