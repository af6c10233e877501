"""TEST INFRASTRUCTURE ONLY -- the mixed dense-sparse KKT path of hb_mds.cu (k_mds_hxs, k_mds_ddinv, k_mds_build, k_mds_pack_rhs,
k_mds_unpack) restated in vectorised numpy, in the reference's exact operation order, so that it gives the reference's bits at the
bench's sparse shape (n_s = 5e5, m = 2000, 1250 nonzeros per row) in seconds, where kkt_oracle's per-pair loops cannot go.

Every entry is a fixed chain of correctly rounded FP64 operations, so numpy's elementwise operations give the same bits as the C++
reference (hiopKKTLinSysMDS.cpp, hiopMatrixSparseTriplet.cpp, hiopMatrixDenseRowMajor.cpp), zero signs included:

- Schur blocks (2,2), (2,3), (3,3): for rows i <= j of the stacked J_s = [J_cs; J_ds], acc = 0.0 + sum over the shared columns c in
  ascending order of fl(fl(v_i / Hxs_c) * v_j) (addMDinvMtransToDiagBlockOfSymDeMatUTri / addMDinvNtransToSymDeMatUTri, :390-525),
  stored as 0.0 + (-1 * acc) into the zeroed Msys (`W += alpha*acc`), then - delta_cc, or - Dd_inv and - delta_cd, on the diagonal.
  A pair of rows that shares no column is +0.0.
- Dense blocks: 0.0 + Hd and 0.0 + J_d^T (addUpperTriangle... / transAdd... into the zeroed Msys), + Dx, + delta_wx on the diagonal.
- pack: y = ryc_i (ryd_i), then y = fl(y + fl(fl(-1 * rxs_c) * v)) over row i's triplets (timesVec(1, y, -1, rxs), :73-89).
- unpack: y = rx_c, then the same update with sol over column c's J_c rows ascending, then its J_d rows ascending (two
  transTimesVec calls, :110-126), then y / Hxs_c (componentDiv).

The Schur sums are vectorised by rank within a pair of rows, pack by rank within a row and unpack by rank within a column: the longest
Python loop is the longest row. `mutate` plants one mistake (a test of the test): "desc" sums the shared columns in descending order,
"swap" forms (v_j / Hxs) * v_i, "jd_first" runs J_d's rows before J_c's in unpack, "no_zero_start" drops the 0.0 + start of every
assembled entry (-0.0 where the reference has +0.0).
"""
from __future__ import annotations

import numpy as np

TINY = 1e-14          # factorizeWithCurvCheck's thresholds on Hxs (hiopKKTLinSysMDS.cpp:90-91)


def stacked(p):
    """(ptr, col, vals) of the stacked sparse Jacobian [J_cs; J_ds] in CSR (triplet order within each row), as hb_mds_set_sparsity
    builds it. p: hiop_b200.synth.MdsProblem-like (sorted triplets)."""
    m = p.neq + p.nineq
    rows = np.concatenate([np.asarray(p.iRow_c, np.int64), p.neq + np.asarray(p.iRow_d, np.int64)])
    col = np.concatenate([np.asarray(p.jCol_c, np.int64), np.asarray(p.jCol_d, np.int64)])
    vals = np.concatenate([np.asarray(p.Jcs_vals, np.float64), np.asarray(p.Jds_vals, np.float64)])
    ptr = np.zeros(m + 1, np.int64)
    np.add.at(ptr, rows + 1, 1)
    return np.cumsum(ptr), rows, col, vals


def diagonals(p):
    """(Dx, Hxs, Dd_inv) as k_mds_update, k_mds_hxs and k_mds_ddinv round them: Dx = 0 + zl/sxl|ixl + zu/sxu|ixu,
    Hxs = (Dx + delta_wx) + Hs, Dd_inv = 1 / ((delta_wd + vl/sdl|idl) + vu/sdu|idu)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        Dx = np.zeros(p.nxs + p.nxd)
        Dx = np.where(p.ixl == 1.0, Dx + p.zl / p.sxl, Dx)
        Dx = np.where(p.ixu == 1.0, Dx + p.zu / p.sxu, Dx)
        Hxs = (Dx[:p.nxs] + p.delta_wx[:p.nxs]) + p.Hs_diag
        d = np.array(p.delta_wd, dtype=np.float64)
        if p.nineq:
            d = np.where(p.idl == 1.0, d + p.vl / p.sdl, d)
            d = np.where(p.idu == 1.0, d + p.vu / p.sdu, d)
        Dd_inv = 1.0 / d
    return Dx, Hxs, Dd_inv


def _ranked_sum(start, count, terms, init):
    """acc_g = init_g + terms[start_g] + terms[start_g + 1] + ... (count_g terms), one rounding per addition, in that order"""
    acc = np.array(init, dtype=np.float64, copy=True)
    order = np.argsort(-count, kind="stable")     # groups by decreasing length: the live groups of rank r are a prefix
    cs, ss = count[order], start[order]
    for r in range(int(cs[0]) if cs.size else 0):
        live = int(np.searchsorted(-cs, -r, side="left"))   # groups with count > r
        idx = order[:live]
        acc[idx] = acc[idx] + terms[ss[:live] + r]
    return acc


def schur(p, Hxs, mutate: str | None = None):
    """The upper triangle of -J_s Hxs^-1 J_s^T before the diagonal shifts, (m x m): the sums as the merge-join of two sorted rows
    forms them, stored as 0.0 + (-1 * acc). Also returns the number of pairs i <= j that share no column."""
    m = p.neq + p.nineq
    ptr, rows, col, vals = stacked(p)
    # CSC with ascending rows within each column (stable: triplet order)
    o = np.argsort(col, kind="stable")
    crow, ccol, cval = rows[o], col[o], vals[o]
    cptr = np.searchsorted(ccol, np.arange(p.nxs + 1))
    # every (a <= b) pair of entries of one column: rows crow[a] <= crow[b]
    end = cptr[ccol + 1]
    cnt = end - np.arange(ccol.size)
    A = np.repeat(np.arange(ccol.size), cnt)
    B = A + (np.arange(A.size) - np.repeat(np.cumsum(cnt) - cnt, cnt))
    i, j, c = crow[A], crow[B], ccol[A]
    h = Hxs[c]
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (cval[B] / h) * cval[A] if mutate == "swap" else (cval[A] / h) * cval[B]
    key = i * m + j
    # pairs in (i, j) order, columns ascending within a pair (they come column by column; a stable sort keeps that)
    s = np.argsort(key, kind="stable")
    if mutate == "desc":
        s = np.lexsort((-c, key))
    key, t = key[s], t[s]
    uk, start, count = np.unique(key, return_index=True, return_counts=True)
    acc = _ranked_sum(start, count, t, np.zeros(uk.size))
    S = np.zeros((m, m))
    if mutate == "no_zero_start":                 # -1 * acc stored as is: a pair that shares no column is -1 * 0.0 = -0.0
        S[np.triu_indices(m)] = -0.0
        S[uk // m, uk % m] = -1.0 * acc
    else:                                         # a pair that shares no column stays 0.0 + (-1 * 0.0) = +0.0
        S[uk // m, uk % m] = 0.0 + (-1.0 * acc)
    return S, m * (m + 1) // 2 - uk.size


def assemble(p, Dx, Hxs, Dd_inv, mutate: str | None = None):
    """Msys (N x N, N = nxd + neq + nineq) with the upper triangle as the reference assembles it into a zeroed matrix and the strict
    lower triangle zero. Returns (M, number of Schur pairs that share no column)."""
    nxs, nxd, neq, nineq = p.nxs, p.nxd, p.neq, p.nineq
    N = nxd + neq + nineq
    z = (lambda a: a) if mutate == "no_zero_start" else (lambda a: 0.0 + a)
    M = np.zeros((N, N))
    M[:nxd, :nxd] = np.triu(z(np.asarray(p.Hd, np.float64)))
    dg = np.arange(nxd)
    M[dg, dg] = (M[dg, dg] + Dx[nxs:]) + p.delta_wx[nxs:]
    M[:nxd, nxd:nxd + neq] = z(np.asarray(p.Jcd, np.float64).T)
    M[:nxd, nxd + neq:] = z(np.asarray(p.Jdd, np.float64).T)
    S, n_empty = schur(p, Hxs, mutate)
    if neq:
        q = np.arange(neq)
        S[q, q] = S[q, q] + -1.0 * np.asarray(p.delta_cc, np.float64)
    if nineq:
        q = np.arange(neq, neq + nineq)
        S[q, q] = (S[q, q] + -1.0 * Dd_inv) + -1.0 * np.asarray(p.delta_cd, np.float64)
    M[nxd:, nxd:] = S
    return M, n_empty


def pack(p, Hxs, rx, ryc, ryd):
    """The dense solve's rhs [rx_d; ryc - J_cs rxs; ryd - J_ds rxs], rxs = rx_s / Hxs, in timesVec's order."""
    ptr, _, col, vals = stacked(p)
    with np.errstate(divide="ignore", invalid="ignore"):
        rxs = rx[:p.nxs] / Hxs
    y0 = np.concatenate([np.asarray(ryc, np.float64), np.asarray(ryd, np.float64)])
    with np.errstate(invalid="ignore"):
        terms = (-1.0 * rxs[col]) * vals
    y = _ranked_sum(ptr[:-1], np.diff(ptr), terms, y0)
    return np.concatenate([np.asarray(rx[p.nxs:], np.float64), y])


def unpack(p, Hxs, sol, rx, mutate: str | None = None):
    """(dx, dyc, dyd) from the dense solution sol = [dx_d; dyc; dyd]: dx_s = (rx_s - J_cs^T dyc - J_ds^T dyd) / Hxs with each column's
    J_c rows ascending, then its J_d rows ascending."""
    nxs, nxd, neq = p.nxs, p.nxd, p.neq
    _, rows, col, vals = stacked(p)
    key = np.where(rows >= neq, rows - neq, rows + (1 << 40)) if mutate == "jd_first" else rows
    o = np.lexsort((key, col))
    ccol = col[o]
    cptr = np.searchsorted(ccol, np.arange(nxs + 1))
    with np.errstate(invalid="ignore"):
        terms = (-1.0 * sol[nxd + rows[o]]) * vals[o]
    y = _ranked_sum(cptr[:-1], np.diff(cptr), terms, np.asarray(rx[:nxs], np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        dxs = y / Hxs
    return np.concatenate([dxs, sol[:nxd]]), sol[nxd:nxd + neq].copy(), sol[nxd + neq:].copy()


def with_pattern(p, cols_c, cols_d, seed=0):
    """p with J_cs / J_ds replaced: row i of J_cs has the columns cols_c[i] (sorted here; an empty list is an empty row), likewise
    J_ds, with standard normal values. Returns p."""
    r = np.random.default_rng(seed)

    def trip(rows):
        iR = np.concatenate([np.full(len(cs), i, np.int32) for i, cs in enumerate(rows)] + [np.zeros(0, np.int32)])
        jC = np.concatenate([np.sort(np.asarray(cs, np.int32)) for cs in rows] + [np.zeros(0, np.int32)])
        return iR, jC, r.standard_normal(iR.size)
    assert len(cols_c) == p.neq and len(cols_d) == p.nineq
    p.iRow_c, p.jCol_c, p.Jcs_vals = trip(cols_c)
    p.iRow_d, p.jCol_d, p.Jds_vals = trip(cols_d)
    return p


def with_negative_zeros(p, seed=0, frac=0.25):
    """p with about frac of the entries of Hd, Jcd, Jdd, J_cs and J_ds set to -0.0 (the derivative -x at x = 0). Returns p."""
    r = np.random.default_rng(seed)
    for name in ("Hd", "Jcd", "Jdd", "Jcs_vals", "Jds_vals"):
        a = np.array(getattr(p, name), dtype=np.float64)
        a[r.random(a.shape) < frac] = -0.0
        setattr(p, name, a)
    return p


def hxs_counts(Hxs):
    """(#Hxs < -1e-14, #|Hxs| < 1e-14): the Haynsworth correction and the null test of factorizeWithCurvCheck (NaN counts in neither)"""
    return int(np.count_nonzero(Hxs < -TINY)), int(np.count_nonzero(np.abs(Hxs) < TINY))
