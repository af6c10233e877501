"""LSQ multiplier update on the device (SURVEY 8 f2, hiopDualsLsqUpdateLinsysRedDenseSymPD::do_lsq_update) against the oracle
restatement (pinned to the reference by tests/test_oracle_vs_ref.py::test_lsq_duals_match_reference)."""
import numpy as np
import pytest

from hiop_b200 import synth
from oracle import kkt_oracle as ko
from test_gpu_parity import ctx, _setup_kkt, _as_dict  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,m,mode", [(3000, 20, -1), (4099, 37, -1), (10000, 1, -1), (40000, 100, 0), (40000, 100, 8), (2500, 0, -1),
                                      (3000, 64, -1), (3000, 65, -1), (8000, 2049, -1)])  # both sides of the cooperative Cholesky's range
def test_lsq_duals_against_oracle(ctx, n, m, mode):
    P = synth.make_qn_problem(n, m, 0, seed=5 + n)
    p = _as_dict(P)
    k, T = _setup_kkt(ctx, p)
    k.set_condense_mode(mode)
    g = np.random.default_rng(9).standard_normal(n)
    yc, yd = ctx.zeros(P.m_eq), ctx.zeros(P.m_ineq)
    assert k.lsq_duals(ctx.to_device(g), T["zl"], T["zu"], T["vl"], T["vu"], yc, yd)
    ctx.sync()
    yco, ydo = ko.lsq_duals(P.Jc, P.Jd, g, P.zl, P.zu, P.vl, P.vu)
    tol = 1e-8 if mode == 8 else 1e-10
    for a, b in ((yc.cpu().numpy(), yco), (yd.cpu().numpy(), ydo)):
        assert np.abs(a - b).max(initial=0.0) <= tol * max(1.0, np.abs(b).max(initial=0.0))
    # defining property (normal equations of the LSQ problem): J (J^T y + vx) + [0; yd + vd] = 0
    if m:
        y = np.concatenate([yc.cpu().numpy(), yd.cpu().numpy()])
        J = np.vstack([P.Jc, P.Jd])
        r = J @ (J.T @ y + (g - P.zl + P.zu))
        r[P.m_eq:] += y[P.m_eq:] + (P.vl - P.vu)
        assert np.abs(r).max() <= 1e-9 * max(1.0, np.abs(J @ (g - P.zl + P.zu)).max())
    k.close()
