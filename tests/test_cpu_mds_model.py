"""oracle/mds_model.py, the vectorised restatement of the mixed dense-sparse KKT path (hb_mds.cu), against kkt_oracle's per-entry loops
(ko.mds_build_kkt_matrix, ko.mds_pack, ko.mds_unpack, which test_oracle_vs_ref pins to the compiled reference) as uint64, so -0.0 and
+0.0 differ; and four planted mistakes that must change the model's bits on cases built to expose them."""
import numpy as np
import pytest

from hiop_b200 import synth
from oracle import kkt_oracle as ko
from oracle import mds_model as mm

U64 = np.uint64


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(U64)


# ---- the cases: (nxs, nxd, neq, nineq) and an edit of the sparsity / values ---------------------------------------------------------
def _empty_rows(p):
    """empty rows in J_cs and J_ds, rows with one entry, and columns no row touches"""
    r = np.random.default_rng(3)
    live = np.arange(0, p.nxs, 3)                 # two thirds of the columns stay empty
    cols = lambda i: [] if i % 4 == 1 else ([int(live[i % live.size])] if i % 4 == 2 else r.choice(live, 4, replace=False))
    return mm.with_pattern(p, [cols(i) for i in range(p.neq)], [cols(i + 1) for i in range(p.nineq)], seed=4)


def _shared_column(p):
    """column 0 touched by all m rows; row 0 of J_cs and the last row of J_ds touch all n_s columns"""
    r = np.random.default_rng(5)
    full = list(range(p.nxs))
    some = lambda: [0] + list(1 + r.choice(p.nxs - 1, 3, replace=False))
    cc = [full] + [some() for _ in range(p.neq - 1)]
    cd = [some() for _ in range(p.nineq - 1)] + [full]
    return mm.with_pattern(p, cc, cd, seed=6)


def _no_jcs(p):
    """nnz_c = 0 with neq > 0"""
    r = np.random.default_rng(7)
    return mm.with_pattern(p, [[]] * p.neq, [r.choice(p.nxs, 3, replace=False) for _ in range(p.nineq)], seed=8)


def _no_jds(p):
    """nnz_d = 0 with nineq > 0"""
    r = np.random.default_rng(9)
    return mm.with_pattern(p, [r.choice(p.nxs, 3, replace=False) for _ in range(p.neq)], [[]] * p.nineq, seed=10)


def _negative_zeros(p):
    return mm.with_negative_zeros(p, seed=11)


def _plain(p):
    return p


EDGES = [
    ("plain", (60, 25, 9, 14), _plain),
    ("empty-rows-cols", (90, 12, 11, 9), _empty_rows),
    ("shared-column", (40, 10, 7, 6), _shared_column),
    ("nnz_c=0", (50, 8, 6, 5), _no_jcs),
    ("nnz_d=0", (50, 8, 6, 5), _no_jds),
    ("negative-zeros", (70, 16, 8, 10), _negative_zeros),
    ("nxs=0", (0, 20, 5, 7), _plain),
    ("nxd=0", (80, 0, 6, 9), _plain),
    ("neq=0", (80, 10, 0, 9), _plain),
    ("nineq=0", (80, 10, 6, 0), _plain),
    ("negative-zeros-empty-rows", (90, 12, 11, 9), lambda p: mm.with_negative_zeros(_empty_rows(p), seed=12)),
]


def edge_problem(name, shape, edit, dwx=1e-4, dcc=1e-6):
    nxs, nxd, neq, nineq = shape
    p = synth.make_mds_problem(nxs, nxd, neq, nineq, seed=sum(shape), dwx=dwx, dcc=dcc)
    return edit(p)


def _oracle(p):
    Mo, Dx, Hxs, Dd_inv = ko.mds_build_kkt_matrix(p)
    return Mo, Dx, Hxs, Dd_inv


@pytest.mark.parametrize("name,shape,edit", EDGES, ids=[e[0] for e in EDGES])
def test_model_equals_oracle_bits(name, shape, edit):
    p = edge_problem(name, shape, edit)
    Mo, Dxo, Hxso, Ddo = _oracle(p)
    Dx, Hxs, Dd_inv = mm.diagonals(p)
    for a, b in ((Dx, Dxo), (Hxs, Hxso), (Dd_inv, Ddo)):
        np.testing.assert_array_equal(bits(a), bits(b))
    M, _ = mm.assemble(p, Dx, Hxs, Dd_inv)
    iu = np.triu_indices(M.shape[0])
    bad = np.nonzero(bits(M[iu]) != bits(Mo[iu]))[0]
    assert bad.size == 0, f"{bad.size} entries differ, first {[(iu[0][k], iu[1][k], M[iu][k], Mo[iu][k]) for k in bad[:4]]}"
    if name.startswith("negative-zeros"):                       # the case has something to show
        assert np.signbit(p.Jcd).any() and np.signbit(p.Hd).any() and not np.signbit(M[iu][M[iu] == 0.0]).any()
    r = np.random.default_rng(13)
    rx, ryc, ryd = r.standard_normal(p.nxs + p.nxd), r.standard_normal(p.neq), r.standard_normal(p.nineq)
    np.testing.assert_array_equal(bits(mm.pack(p, Hxs, rx, ryc, ryd)), bits(ko.mds_pack(p, Hxs, rx, ryc, ryd)))
    sol = r.standard_normal(p.nxd + p.neq + p.nineq)
    for a, b in zip(mm.unpack(p, Hxs, sol, rx), ko.mds_unpack(p, Hxs, sol, rx)):
        np.testing.assert_array_equal(bits(a), bits(b))
    if p.nxs:
        assert mm.hxs_counts(Hxs) == (int((Hxs < -1e-14).sum()), int((np.abs(Hxs) < 1e-14).sum()))


def test_empty_columns_give_rx_over_hxs():
    p = edge_problem(*EDGES[1])
    _, Hxs, _ = mm.diagonals(p)
    r = np.random.default_rng(14)
    rx, sol = r.standard_normal(p.nxs + p.nxd), r.standard_normal(p.nxd + p.neq + p.nineq)
    dx, _, _ = mm.unpack(p, Hxs, sol, rx)
    empty = np.setdiff1d(np.arange(p.nxs), np.concatenate([p.jCol_c, p.jCol_d]))
    assert empty.size > p.nxs // 2
    np.testing.assert_array_equal(bits(dx[empty]), bits(rx[empty] / Hxs[empty]))


def test_model_equals_oracle_bits_medium():
    """a shape where pairs share many columns (long merge chains) and some share none"""
    p = synth.make_mds_problem(600, 30, 40, 45, nnz_per_row=60, seed=15, dwx=1e-3, dcc=1e-5)
    Mo, _, Hxs, _ = _oracle(p)
    M, n_empty = mm.assemble(p, *mm.diagonals(p))
    iu = np.triu_indices(M.shape[0])
    np.testing.assert_array_equal(bits(M[iu]), bits(Mo[iu]))
    assert n_empty > 0
    r = np.random.default_rng(16)
    rx, sol = r.standard_normal(p.nxs + p.nxd), r.standard_normal(p.nxd + p.neq + p.nineq)
    np.testing.assert_array_equal(bits(mm.pack(p, Hxs, rx, p.ryc, p.ryd)), bits(ko.mds_pack(p, Hxs, rx, p.ryc, p.ryd)))
    for a, b in zip(mm.unpack(p, Hxs, sol, rx), ko.mds_unpack(p, Hxs, sol, rx)):
        np.testing.assert_array_equal(bits(a), bits(b))


# ---- planted mistakes ------------------------------------------------------------------------------------------------------------------
def _tiny(nxs, neq, nineq, cols_c, cols_d, vals_c, vals_d):
    p = synth.make_mds_problem(nxs, 2, neq, nineq, seed=17)
    mm.with_pattern(p, cols_c, cols_d)
    p.Jcs_vals, p.Jds_vals = np.array(vals_c, dtype=np.float64), np.array(vals_d, dtype=np.float64)
    p.Hs_diag = np.zeros(nxs)
    p.zl, p.zu = np.ones(nxs + 2), np.zeros(nxs + 2)
    p.sxl, p.sxu = np.ones(nxs + 2), np.ones(nxs + 2)
    p.ixl, p.ixu = np.ones(nxs + 2), np.zeros(nxs + 2)      # Dx = 1, so Hxs = 1 exactly
    return p


def test_mutation_descending_merge():
    """row 0 = (1, 1, 1), row 1 = (1, 2^-53, 2^-53) on columns 0, 1, 2: ascending 1 + u + u = 1, descending u + u + 1 = 1 + 2u"""
    u = 2.0 ** -53
    p = _tiny(3, 2, 0, [[0, 1, 2], [0, 1, 2]], [], [1.0, 1.0, 1.0, 1.0, u, u], [])
    D = mm.diagonals(p)
    M, _ = mm.assemble(p, *D)
    Mm, _ = mm.assemble(p, *D, mutate="desc")
    Mo, *_ = _oracle(p)
    assert M[2, 3] == Mo[2, 3] == -1.0 and Mm[2, 3] == -(1.0 + 2 * u)


def test_mutation_swapped_product():
    """(v_i / H) v_j against (v_j / H) v_i: with H = 3, v_i = 1, v_j = 5, fl(1/3) * 5 != fl(5/3) * 1"""
    p = _tiny(1, 2, 0, [[0], [0]], [], [1.0, 5.0], [])
    p.Hs_diag = np.array([2.0])                     # Hxs = 1 + 2 = 3
    D = mm.diagonals(p)
    M, _ = mm.assemble(p, *D)
    Mm, _ = mm.assemble(p, *D, mutate="swap")
    Mo, *_ = _oracle(p)
    assert bits(M[2, 3]) == bits(Mo[2, 3]) != bits(Mm[2, 3])


def test_mutation_jd_before_jc():
    """one column shared by a J_c and a J_d row, rx_s = 1, terms +u (J_c) and -u (J_d): (1 + u) - u = 1 - u, (1 - u) + u = 1"""
    u = 2.0 ** -53
    p = _tiny(1, 1, 1, [[0]], [[0]], [1.0], [1.0])
    D = mm.diagonals(p)
    sol = np.array([0.0, 0.0, -u, u])               # [dx_d (2); dyc; dyd]: the terms are -dyc * 1 and -dyd * 1
    rx = np.array([1.0, 0.0, 0.0])
    dx, _, _ = mm.unpack(p, D[1], sol, rx)
    dxm, _, _ = mm.unpack(p, D[1], sol, rx, mutate="jd_first")
    dxo, _, _ = ko.mds_unpack(p, D[1], sol, rx)
    assert dx[0] == dxo[0] == 1.0 - u and dxm[0] == 1.0


def test_mutation_no_zero_start():
    """two rows that share no column, and -0.0 in Hd / Jcd: the reference stores +0.0, the mutated model -0.0"""
    p = _tiny(4, 2, 0, [[0, 1], [2, 3]], [], [1.0, 2.0, 3.0, 4.0], [])
    p.Hd = np.array([[1.0, -0.0], [-0.0, 1.0]])
    p.Jcd = np.array([[-0.0, 1.0], [1.0, -0.0]])
    D = mm.diagonals(p)
    M, _ = mm.assemble(p, *D)
    Mm, _ = mm.assemble(p, *D, mutate="no_zero_start")
    Mo, *_ = _oracle(p)
    iu = np.triu_indices(4)
    np.testing.assert_array_equal(bits(M[iu]), bits(Mo[iu]))
    for rc in ((2, 3), (0, 1), (0, 2), (1, 3)):
        assert M[rc] == 0.0 and not np.signbit(M[rc]) and np.signbit(Mm[rc]), rc
