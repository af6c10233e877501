"""What the GPU tests of the dense symmetric handles share (hb_symdense, hb_symdense_dist, hb_symdense_host through LinSolverSymDense,
LinSolverSymDenseDist and LinSolverSymDenseHost): the context fixture, the test matrices and right-hand sides, each handle's factor,
solutions and statistics as host arrays, bitwise comparisons, and the slab plans of the host-resident handle."""
from types import SimpleNamespace
import ctypes
import pathlib

import numpy as np
import pytest
import torch

from oracle import bounds
from oracle import rbt_model as rbt
from test_cpu_rbt_model import FAMILIES

BK, NOPIV, CHOL, RBT = 0, 1, 2, 3                            # HB_FACT_* of include/hiopb200.h
K128 = dict(HB_DENSE_BIG_MIN=0, HB_DENSE_PAIR_MIN=1 << 30)   # hb_symdense: look-ahead factorization, blocks unpaired (K = 128)
SOLVE_REL = 1e3 * 2.0 ** -52     # |x - x_bk|_inf / |x_bk|_inf <= SOLVE_REL * cond_inf(A): both solves are backward stable
MDS_FIELDS = ("Hd", "Hs_diag", "Jcd", "Jdd", "Jcs_vals", "Jds_vals", "vl", "sdl", "vu", "sdu", "idl", "idu", "delta_wx", "delta_wd", "delta_cc",
              "delta_cd")
GOLDEN = pathlib.Path(__file__).parent / "golden"
DEV = torch.device("cuda", 0)
# enum order of Factor / Solve / Inertia in hb_symdense.cu
FACTOR = ("SYTF2", "SYTRF_BLOCKED", "BK_CLUSTER", "PANEL_CHOL", "PANEL_LDL", "COOP_CHOL", "BIG_CHOL", "BIG_LDL")
SOLVE = ("SYTRS", "ONE_CTA", "BIG")
INERTIA = ("IPIV", "BLOCKDIAG", "DIAG")


@pytest.fixture
def make_ctx(monkeypatch):
    """Context(0) created under the given environment (hb_dense_init reads the knobs once per context)"""
    made = []

    def make(**env):
        from hiop_b200.engine import Context
        for k in ("HB_DENSE_PAIR_MIN", "HB_BK_CLUSTER_MIN", "HB_DENSE_BIG_MIN", "HB_CHOL_COOP"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, str(v))
        c = Context(0)
        made.append(c)
        return c
    yield make
    for c in made:
        c.close()


# ---- matrices and right-hand sides ------------------------------------------------------------------------------------------------------
def matrix(mode, N, seed, device):
    """(M, inertia): SPD for Cholesky, a matrix of known inertia with eigenvalues >= 0.5 in modulus for the no-pivot LDL^T"""
    if mode == CHOL:
        g = torch.Generator(device="cpu").manual_seed(seed)
        G = torch.randn((N, N // 2 + 1), generator=g, dtype=torch.float64).to(device)
        d = torch.rand(N, generator=g, dtype=torch.float64).to(device) * 1.5 + 0.5
        return G @ G.T / max(N, 1) + torch.diag(d), (0, 0, N)
    return bounds.known_inertia_matrix(N, 0, N // 3, seed, device=device)


def rhs(N, seed, nrhs):
    return np.random.default_rng(seed).standard_normal((nrhs, N))


def upper_nan(M):
    U = M.clone()
    U.masked_fill_(torch.ones(M.shape, dtype=torch.bool, device=M.device).tril_(-1), float("nan"))
    return U


def gpu_families():
    for name, A in FAMILIES.items():
        yield name, A
    yield "known_2x2_1000", bounds.known_inertia_matrix(1000, 200, 250, seed=9)[0].numpy()
    from test_cpu_rbt_model import saddle
    yield "saddle_1500_500", saddle(1500, 500, 11, 300)


def golden_mds():
    g = dict(np.load(GOLDEN / "mds_nxs50_nxd20.npz"))
    return SimpleNamespace(**{k: (v if v.ndim else v.item()) for k, v in g.items() if not k.startswith("ref_")})


def orig_backward_error(A, x, b):
    return rbt.backward_error(A, x, b)


# ---- hb_symdense ----------------------------------------------------------------------------------------------------------------------
def readback(s):
    N = s.n
    plan = (ctypes.c_int * 4)()
    widths = ctypes.c_int()
    F = np.empty((N, N))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    plan_only = lambda: s.ctx.L.hb_debug_symdense_factor(s.h, plan, ctypes.byref(widths), None, None, None, None)
    from hiop_b200._lib import check
    check(plan_only(), "hb_debug_symdense_factor")
    bkc = FACTOR[plan[0]] == "BK_CLUSTER"
    ipiv = np.empty(N, dtype=np.int32) if FACTOR[plan[0]] in ("SYTF2", "SYTRF_BLOCKED", "BK_CLUSTER") else None   # pivoting factors only
    perm = np.empty(N, dtype=np.int32) if bkc else None
    dsub = np.empty(N) if bkc else None
    check(s.ctx.L.hb_debug_symdense_factor(s.h, None, None, p(F), p(ipiv) if ipiv is not None else None, p(perm) if bkc else None, p(dsub) if bkc else None),
          "hb_debug_symdense_factor")
    return dict(plan=(FACTOR[plan[0]], SOLVE[plan[1]], INERTIA[plan[2]], bool(plan[3])), widths=widths.value, F=F, ipiv=ipiv, perm=perm,
                dsub=dsub)


def factor_parts(rb):
    """(L, d, dsub, perm) of the factor read back, on the device; P A P^T = L D L^T"""
    f = rb["plan"][0]
    N = rb["F"].shape[0]
    if f in ("SYTF2", "SYTRF_BLOCKED"):                          # LAPACK's 'L' storage and pivots
        L, d, dsub, perm = bounds.lapack_to_permuted(rb["F"].T.copy(), rb["ipiv"].astype(np.int64))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
        return t(L), t(d), t(dsub), perm
    Fl = torch.from_numpy(rb["F"]).to(DEV).T.tril()
    if f.endswith("CHOL"):
        return Fl.contiguous(), torch.ones(N, dtype=torch.float64, device=DEV), None, np.arange(N)
    d = torch.diagonal(Fl).clone()
    L = Fl.tril(-1) + torch.eye(N, dtype=torch.float64, device=DEV)
    if f == "BK_CLUSTER":
        return L, d, torch.from_numpy(rb["dsub"]).to(DEV), rb["perm"].astype(np.int64)
    return L, d, None, np.arange(N)


def theta(L):
    """explicit diagonal-block inverses: 16 x 16 (k_trsm_panel, cooperative paths) and 128 x 128 (look-ahead, blocked solves)"""
    return max(bounds.block_theta(L, 16), bounds.block_theta(L, 128))


def factor_single(ctx, mode, M):
    """hb_symdense's factor (row-major, upper valid) of M, its return value and inertia; asserts the look-ahead path at K = 128"""
    from hiop_b200.engine import LinSolverSymDense
    N = M.shape[0]
    s = LinSolverSymDense(ctx, N, mode)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(M).contiguous())
    ctx.sync()
    rc = s.matrixChanged()
    rb = readback(s)
    assert rb["plan"] == ("BIG_CHOL" if mode == CHOL else "BIG_LDL", "BIG", "DIAG", False), rb["plan"]
    inertia = s.inertia()
    s.close()
    return rc, inertia, rb["F"]


def bk_single(ctx, A):
    """hb_symdense Bunch-Kaufman on A (numpy, full): return value and inertia"""
    from hiop_b200.engine import LinSolverSymDense
    N = A.shape[0]
    s = LinSolverSymDense(ctx, N, BK)
    torch.cuda.synchronize()
    s.set_matrix(torch.from_numpy(np.ascontiguousarray(A)).to(ctx.device))
    ctx.sync()
    rc = s.matrixChanged()
    inr = s.inertia()
    s.close()
    return rc, inr


# ---- hb_symdense_dist -----------------------------------------------------------------------------------------------------------------
def local_rows(s):
    """{global row: this rank's stored row (length N)} of a LinSolverSymDenseDist"""
    torch.cuda.synchronize()
    s.ctx.sync()
    loc = s.local()[:, :s.n].cpu().numpy()
    out = {}
    for q, (b, e) in enumerate(s.rows):
        for r in range(b, e):
            out[r] = loc[q * 128 + r - b]
    return out


def factor_dist(ctx, mode, M, rhs_list):
    """factor M (device, full) with LinSolverSymDenseDist and solve each rhs (nrhs x N); returns rc, inertia, rows, solutions"""
    from hiop_b200.engine import LinSolverSymDenseDist
    N = M.shape[0]
    s = LinSolverSymDenseDist(ctx, N)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(M))
    rc = s.matrixChanged(mode)
    inertia = s.inertia()
    rows = local_rows(s)
    sols = []
    for b in rhs_list:
        x = ctx.to_device(b)
        assert s.solve(x)
        ctx.sync()
        sols.append(x.cpu().numpy())
    s.close()
    return rc, inertia, rows, sols


def rbt_dist(ctx, A, rhs=None, mode=RBT):
    """factor A (numpy, full) on a LinSolverSymDenseDist in `mode`; solve rhs (N x nrhs) when given. Returns rc, inertia, rows, x, stats"""
    from hiop_b200.engine import LinSolverSymDenseDist
    N = A.shape[0]
    s = LinSolverSymDenseDist(ctx, N)
    torch.cuda.synchronize()
    s.set_matrix(upper_nan(torch.from_numpy(np.ascontiguousarray(A)).to(ctx.device)))
    rc = s.matrixChanged(mode)
    inr = s.inertia()
    rows = local_rows(s)
    x = stats = None
    if rhs is not None and rc >= 0:
        xd = ctx.to_device(np.ascontiguousarray(rhs.T))
        assert s.solve(xd)
        ctx.sync()
        x = xd.cpu().numpy().T.copy()
        stats = s.rbt_stats()
    s.close()
    return rc, inr, rows, x, stats


def same_rows(rows, F, what):
    for r, v in rows.items():
        a, b = v[r:], F[r, r:]
        if not np.array_equal(a.view(np.uint64), b.view(np.uint64)):
            bad = np.nonzero(a.view(np.uint64) != b.view(np.uint64))[0]
            pytest.fail(f"{what}: row {r}: {bad.size} entries differ, first at column {r + bad[0]}: {a[bad[0]]!r} vs {b[bad[0]]!r}")


def factor_parts_from_rows(rows, N, mode):
    """(L, d) on the host from the stored rows (row r of the row-major upper triangle = column r of L)"""
    Lt = np.zeros((N, N))
    for r, v in rows.items():
        Lt[r, r:] = v[r:]
    L = Lt.T.copy()
    if mode == CHOL:
        return L, np.ones(N)
    d = np.diag(L).copy()
    np.fill_diagonal(L, 1.0)
    return L, d


def dist_rows_array(rows, N):
    F = np.zeros((N, N))
    for r, v in rows.items():
        F[r] = v[:N]
    return F


# ---- hb_symdense_host -----------------------------------------------------------------------------------------------------------------
def plan(N, budget):
    from hiop_b200.engine import LinSolverSymDenseHost
    return LinSolverSymDenseHost.plan_view(N, budget)


def budget_for(N, slabs):
    """the smallest budget whose plan has at most `slabs` slabs (1 << 40: one slab)"""
    lo, hi = 1, 1 << 40
    while hi - lo > 1:
        mid = (lo + hi) // 2
        try:
            ok = plan(N, mid)["slabs"] <= slabs
        except Exception:
            ok = False
        hi, lo = (mid, lo) if ok else (hi, mid)
    return hi


def budget_for_height(N, H):
    """the smallest budget whose plan puts at least H block rows in a slab"""
    lo, hi = 1, 1 << 40
    while hi - lo > 1:
        mid = (lo + hi) // 2
        try:
            ok = plan(N, mid)["slab_blocks"] >= H
        except Exception:
            ok = False
        hi, lo = (mid, lo) if ok else (hi, mid)
    return hi


def budgets(N):
    """{one slab, two slabs, one block row per slab, three slabs with a shorter last one}, each once"""
    nblk = -(-N // 128)
    out = {}
    for name, n in (("one_slab", 1), ("two_slabs", 2), ("row_per_slab", nblk)):
        b = budget_for(N, n)
        if all(plan(N, b)["slabs"] != plan(N, v)["slabs"] for v in out.values()):
            out[name] = b
    # the first slab height that gives three slabs with a remainder, so that the last slab has fewer block rows
    H = next((h for h in range(1, nblk) if -(-nblk // h) == 3 and nblk % h), None)
    if H is not None:
        b = budget_for_height(N, H)
        p = plan(N, b)
        assert p["slabs"] == 3 and p["first"][3] - p["first"][2] < p["first"][1] - p["first"][0], p
        out["three_slabs_short_last"] = b
    return out


def assert_lower_untouched(F, M, what):
    """the strictly lower triangle of the buffer still holds upper_nan's NaNs, bit for bit"""
    low = np.tril(np.ones(F.shape, dtype=bool), -1)
    want = upper_nan(M).cpu().numpy()
    assert np.array_equal(F[low].view(np.uint64), want[low].view(np.uint64)), what
