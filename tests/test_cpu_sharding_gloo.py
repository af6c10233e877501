"""world_size-2 gloo test (CPU): the column-sharded formulation of the condensed KKT system reproduces the single-rank
result. Each rank runs the ORACLE on its column shard, the partial blocks are summed with torch.distributed (gloo) in the
same places where libhiopb200.so calls ncclAllReduce, and the replicated small solves are done redundantly."""
import numpy as np
import pytest
import torch
import torch.distributed as dist

from hiop_b200 import sharding, synth
from oracle import kkt_oracle as ko
from multirank import run_ranks


def _allreduce(a):
    t = torch.from_numpy(np.ascontiguousarray(a))
    dist.all_reduce(t)
    return t.numpy()


def _worker(rank, world, init_method, out, n, m, l):
    dist.init_process_group("gloo", init_method=init_method, rank=rank, world_size=world)
    try:
        P = synth.make_qn_problem(n, m, l, seed=31)
        b, e = sharding.column_range(n, world, rank)
        sl = slice(b, e)
        Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl[sl], P.sxl[sl], P.zu[sl], P.sxu[sl], P.ixl[sl], P.ixu[sl], P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu,
                                              P.sigma)
        J = np.ascontiguousarray(P.J[:, sl])
        St, Yt = np.ascontiguousarray(P.St[:, sl]), np.ascontiguousarray(P.Yt[:, sl])
        # (1) one all-reduce of the augmented Gram matrix [J;S;Y] DhInv [J;S;Y]^T  and of S S^T
        A = np.vstack([J, St, Yt])
        C = _allreduce(ko.symm_mat_diag_mat_trans(A, DhInv))
        SSt = _allreduce(St @ St.T)
        mm, s = m, P.sigma
        V = np.zeros((2 * l, 2 * l))
        V[:l, :l] = s * s * C[mm:mm + l, mm:mm + l] - s * SSt
        V[:l, l:] = s * C[mm:mm + l, mm + l:] - P.L
        V[l:, :l] = V[:l, l:].T
        V[l:, l:] = C[mm + l:, mm + l:] + np.diag(P.D)
        Vf = ko.SymFactor(V)
        U = np.hstack([s * C[:mm, mm:mm + l], C[:mm, mm + l:]])
        N = C[:mm, :mm] - U @ Vf.solve(U.T.copy())
        idx = np.arange(P.m_eq, mm)
        N[idx, idx] += Dd_inv

        def hess_solve(r):   # (2) 2l doubles all-reduced per solve
            t = DhInv * r
            p = Vf.solve(_allreduce(np.concatenate([s * (St @ t), Yt @ t])))
            return DhInv * (r - s * (St.T @ p[:l]) - Yt.T @ p[l:])
        dxt = hess_solve(P.rx[sl])
        # (3) J*dx: partial products summed; the "- [ryc;ryd]" (beta*y) term enters once (rank-0 rule)
        part = J @ dxt - (np.concatenate([P.ryc, P.ryd]) if rank == 0 else 0.0)
        rhs = _allreduce(part)
        dy, _, _ = ko.solve_with_refin(N, rhs)
        dx = hess_solve(P.rx[sl] - J.T @ dy)
        if rank == 0:
            out["N"], out["dy"] = N, dy
        out[f"dx{rank}"] = dx
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n,m,l", [(1001, 12, 3), (640, 5, 0)])
def test_column_sharded_kkt_matches_single_rank(n, m, l):
    out = run_ranks(_worker, 2, (n, m, l), comm="gloo")
    P = synth.make_qn_problem(n, m, l, seed=31)
    Dx, DhInv, Dd, Dd_inv = ko.kkt_update(P.zl, P.sxl, P.zu, P.sxu, P.ixl, P.ixu, P.vl, P.sdl, P.vu, P.sdu, P.idl, P.idu, P.sigma)
    st = ko.QnState(P.Jc, P.Jd, DhInv, Dd_inv, P.St, P.Yt, P.L, P.D, P.sigma)
    dx, dyc, dyd, N = ko.solve_compressed(st, P.rx, P.ryc, P.ryd)
    assert np.abs(out["N"] - N).max() <= 1e-12 * np.abs(N).max()
    assert np.abs(out["dy"] - np.concatenate([dyc, dyd])).max() <= 1e-9 * max(1.0, np.abs(dyc).max())
    dxs = np.concatenate([out["dx0"], out["dx1"]])
    assert np.abs(dxs - dx).max() <= 1e-9 * np.abs(dx).max()


def _worker_compound(rank, world, init_method, out, n, mi, me):
    dist.init_process_group("gloo", init_method=init_method, rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(5)
        sizes = dict(x=n, d=mi, yc=me, yd=mi, sxl=n, sxu=n, sdl=mi, sdu=mi, zl=n, zu=n, vl=mi, vu=mi)
        a = {k: rng.standard_normal(v) for k, v in sizes.items()}
        b = {k: rng.standard_normal(v) for k, v in sizes.items()}
        lo, hi = sharding.column_range(n, world, rank)
        shard = lambda d: {k: (v[lo:hi] if k in sharding.N_BLOCKS else v) for k, v in d.items()}
        sa, sb = shard(a), shard(b)
        # dot product and 2-norm of BiCGStab: one SUM all-reduce each
        dot = _allreduce(np.array([sharding.compound_reduction_contribution(rank, sa, lambda k, v: float(v @ sb[k]))]))[0]
        nrm2 = np.sqrt(_allreduce(np.array([sharding.compound_reduction_contribution(rank, sa, lambda k, v: float(v @ v))]))[0])
        # inf-norms of the residual (hiopResidual.cpp:349-365): MAX all-reduce of the sharded blocks, replicated blocks combined locally
        t = torch.tensor([max(np.abs(sa[k]).max() for k in sharding.N_BLOCKS)], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        inf = max(float(t[0]), max(np.abs(sa[k]).max(initial=0.0) for k in sharding.M_BLOCKS))
        # fraction-to-the-boundary (hiopIterate.cpp:356-360): MIN all-reduce
        tau = 0.995
        ftb = lambda x, dx: float(np.min(np.where(dx < 0, np.minimum(1.0, -tau * np.abs(x) / np.where(dx < 0, dx, -1.0)), 1.0), initial=1.0))
        t = torch.tensor([min(ftb(sa[k], sb[k]) for k in ("sxl", "sxu"))], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        alpha = min(float(t[0]), min(ftb(sa[k], sb[k]) for k in ("sdl", "sdu")))
        out[rank] = (dot, nrm2, inf, alpha)
        if rank == 0:
            fa, fb = np.concatenate([a[k] for k in sizes]), np.concatenate([b[k] for k in sizes])
            out["want"] = (float(fa @ fb), float(np.linalg.norm(fa)), float(np.abs(fa).max()),
                           min(ftb(a[k], b[k]) for k in ("sxl", "sxu", "sdl", "sdu")))
    finally:
        dist.destroy_process_group()


def test_compound_vector_reductions_count_replicated_blocks_once():
    """The reduction rules of the sharded BiCGStab / residual norms / step-length search: every rank ends with the value a single
    rank would compute on the unsharded 12-block vector."""
    out = run_ranks(_worker_compound, 2, (1001, 7, 5), comm="gloo")
    want = out["want"]
    for rank in (0, 1):
        got = out[rank]
        assert abs(got[0] - want[0]) <= 1e-12 * max(1.0, abs(want[0]))
        assert abs(got[1] - want[1]) <= 1e-12 * want[1]
        assert got[2] == want[2] and got[3] == want[3]


def test_column_range_partitions_exactly():
    for n in (0, 1, 7, 1000003):
        for w in (1, 2, 3, 8):
            r = [sharding.column_range(n, w, k) for k in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[k][1] == r[k + 1][0] for k in range(w - 1))
            sizes = [e - b for b, e in r]
            assert max(sizes) - min(sizes) <= 1
    assert sum(c for _, c in sharding.reductions_per_system(1000, 6)) == 36 + 1012 ** 2 + 12 + 1000 + 12
