"""GPU parity of the mixed dense-sparse KKT assembly + compressed solve (hiopKKTLinSysCompressedMDSXYcYd role)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp

from hiop_b200 import synth
from oracle import kkt_oracle as ko

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ctx():
    from hiop_b200.engine import Context
    c = Context(0)
    yield c
    c.close()


def _device_run(ctx, p, safe_mode):
    from hiop_b200.engine import KKTLinSysCompressedMDSXYcYd
    D = ctx.to_device
    k = KKTLinSysCompressedMDSXYcYd(ctx, p.nxs, p.nxd, p.neq, p.nineq, safe_mode=safe_mode)
    k.set_sparsity(p.iRow_c, p.jCol_c, p.iRow_d, p.jCol_d)
    T = {name: D(getattr(p, name)) for name in ("zl", "sxl", "zu", "sxu", "ixl", "ixu", "Hd", "Hs_diag", "Jcd", "Jdd", "Jcs_vals", "Jds_vals", "vl",
                                                "sdl", "vu", "sdu", "idl", "idu", "delta_wx", "delta_wd", "delta_cc", "delta_cd", "rx", "ryc", "ryd")}
    k.update(T["zl"], T["sxl"], T["zu"], T["sxu"], T["ixl"], T["ixu"])
    k.build_kkt_matrix(T["Hd"], T["Hs_diag"], T["Jcd"], T["Jdd"], T["Jcs_vals"], T["Jds_vals"], T["vl"], T["sdl"], T["vu"], T["sdu"], T["idl"],
                       T["idu"], T["delta_wx"], T["delta_wd"], T["delta_cc"], T["delta_cd"])
    M = k.Msys().copy()
    ret = k.factorizeWithCurvCheck()
    dx, dyc, dyd = ctx.zeros(p.nxs + p.nxd), ctx.zeros(p.neq), ctx.zeros(p.nineq)
    ok = k.solveCompressed(T["rx"], T["ryc"], T["ryd"], dx, dyc, dyd)
    ctx.sync()
    out = (M, ret, ok, dx.cpu().numpy(), dyc.cpu().numpy(), dyd.cpu().numpy())
    k.close()
    return out


def _full_residual(p, Dx, Dd_inv, dx, dyc, dyd):
    Jc = np.hstack([sp.csr_matrix((p.Jcs_vals, (p.iRow_c, p.jCol_c)), shape=(p.neq, p.nxs)).toarray(), p.Jcd])
    Jd = np.hstack([sp.csr_matrix((p.Jds_vals, (p.iRow_d, p.jCol_d)), shape=(p.nineq, p.nxs)).toarray(), p.Jdd])
    H = np.zeros((p.nxs + p.nxd,) * 2)
    H[:p.nxs, :p.nxs] = np.diag(p.Hs_diag)
    H[p.nxs:, p.nxs:] = p.Hd
    H += np.diag(Dx + p.delta_wx)
    r1 = H @ dx + Jc.T @ dyc + Jd.T @ dyd - p.rx
    r2 = Jc @ dx - p.delta_cc * dyc - p.ryc
    r3 = Jd @ dx - (Dd_inv + p.delta_cd) * dyd - p.ryd
    return max(np.abs(r1).max(), np.abs(r2).max() if p.neq else 0.0, np.abs(r3).max() if p.nineq else 0.0)


def test_mds_against_reference_golden(ctx):
    g = dict(np.load(os.path.join(GOLD, "mds_nxs50_nxd20.npz")))
    p = SimpleNamespace(**{k: (v if v.ndim else v.item()) for k, v in g.items() if not k.startswith("ref_")})
    M, ret, ok, dx, dyc, dyd = _device_run(ctx, p, True)
    N = p.nxd + p.neq + p.nineq
    iu = np.triu_indices(N)
    np.testing.assert_array_equal(M[iu].view(np.uint64), g["ref_M"][iu].view(np.uint64))  # assembly is bit-identical to the reference's methods
    assert ret == int(g["ref_ret"]) == p.neq + p.nineq and ok
    assert _full_residual(p, g["ref_Dx"], g["ref_Dd_inv"], dx, dyc, dyd) <= 1e-9


@pytest.mark.parametrize("nxs,nxd,neq,nineq,safe", [(400, 100, 60, 43, True), (2000, 300, 150, 203, False), (0, 40, 10, 5, True),
                                                      (100, 0, 7, 9, True), (300, 64, 0, 20, True), (5000, 500, 300, 200, True)])
def test_mds_against_oracle(ctx, nxs, nxd, neq, nineq, safe):
    p = synth.make_mds_problem(nxs, nxd, neq, nineq, seed=nxs + nxd, dwx=1e-5, dcc=1e-7)
    Mo, Dx, Hxs, Dd_inv = ko.mds_build_kkt_matrix(p)
    reto, f = ko.mds_factorize_with_curv_check(Mo, Hxs)
    dxo, dyco, dydo = ko.mds_solve_compressed(p, f, Hxs, p.rx, p.ryc, p.ryd)
    M, ret, ok, dx, dyc, dyd = _device_run(ctx, p, safe)
    iu = np.triu_indices(nxd + neq + nineq)
    np.testing.assert_array_equal(M[iu].view(np.uint64), Mo[iu].view(np.uint64))
    assert ret == reto == neq + nineq and ok
    for a, b in ((dx, dxo), (dyc, dyco), (dyd, dydo)):
        if b.size:
            assert np.abs(a - b).max() <= 1e-8 * max(1.0, np.abs(b).max())
    assert _full_residual(p, Dx, Dd_inv, dx, dyc, dyd) <= 1e-8 * max(1.0, np.abs(p.rx).max())


def test_mds_haynsworth_counts_negative_sparse_block(ctx):
    p = synth.make_mds_problem(200, 50, 20, 30, seed=9)
    p.Hs_diag[:7] = -5.0 - p.Hs_diag[:7]      # 7 negative entries that Dx cannot repair everywhere
    Mo, Dx, Hxs, _ = ko.mds_build_kkt_matrix(p)
    reto, _ = ko.mds_factorize_with_curv_check(Mo, Hxs)
    M, ret, ok, *_ = _device_run(ctx, p, True)
    assert ret == reto
    assert ret == int((np.linalg.eigvalsh(np.triu(Mo) + np.triu(Mo, 1).T) < 0).sum()) + int((Hxs < -1e-14).sum())
