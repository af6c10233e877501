"""The tile schedule of the one-GPU random butterfly transform (k_rbt_fused, hb_rbt.cu), checked on the host through
hb_rbt_schedule_view: no device needed.

CTA b computes A'(i, j) for the output rows i of tile bi and j of tile bj (bi <= bj) from the window of A it reads: rows of tile bi's
window x columns of tile bj's window, entries A(min, max) of the upper triangle (a diagonal tile reads only r <= c and mirrors the rest in
shared memory). It writes Ak(i, j) and Ak(j, i), and the upper-triangle entry F(min(i, j), max(i, j)), on a diagonal tile for i <= j
only. So the transform is right when (1) every upper-triangle entry of A' is written by exactly one CTA, once, and (2) every entry of A
that A'(i, j) depends on (rows {i, p2(i), p1(i), p2(p1(i))} x the same of j, with p1, p2 the partners of oracle/rbt_model.py) is in
the CTA's window. Where the 4-row groups are closed under both pairings (N != 1 mod 4) the window is exactly the output rows, so each
upper-triangle entry of A is read once and F may be A itself; for N = 1 (mod 4) the re-read is bounded."""
import ctypes

import numpy as np
import pytest

from hiop_b200 import _lib
from oracle import rbt_model as rbt


def schedule_view(N):
    """(ctas (C x 2), window rows (T x W), output rows (T x O))"""
    L = _lib.lib()
    dims = (ctypes.c_int * 4)()
    assert L.hb_rbt_schedule_view(N, 0, dims, None, None, None) == _lib.HB_OK
    T, C, W, O = list(dims)
    ctas = np.zeros((C, 2), np.int32)
    win = np.zeros((T, W), np.int32)
    out = np.zeros((T, O), np.int32)
    cap = max(T, C)
    assert L.hb_rbt_schedule_view(N, cap, dims, ctas.ctypes.data, win.ctypes.data, out.ctypes.data) == _lib.HB_OK
    return ctas, win, out


def deps(N):
    """per row i: the rows of A that row i of A' reads, {i, p2(i), p1(i), p2(p1(i))}"""
    p1, p2 = rbt.partner(N, 1), rbt.partner(N, 2)
    i = np.arange(N)
    return np.stack([i, p2[i], p1[i], p2[p1[i]]], axis=1)


def check_structure(N):
    ctas, win, out = schedule_view(N)
    T = win.shape[0]
    # the output rows of the tiles partition 0 .. N-1
    rows = out[out >= 0]
    assert np.array_equal(np.sort(rows), np.arange(N)), N
    # the CTAs take every tile pair bi <= bj exactly once
    assert len(ctas) == T * (T + 1) // 2
    assert len({(int(a), int(b)) for a, b in ctas}) == len(ctas)
    assert np.all(ctas[:, 0] <= ctas[:, 1]) and np.all(ctas >= 0) and np.all(ctas < T)
    # every row a tile's output rows depend on is in its window, held once
    D = deps(N)
    for t in range(T):
        w = win[t][win[t] >= 0]
        assert len(np.unique(w)) == len(w), (N, t)
        o = out[t][out[t] >= 0]
        assert np.isin(D[o].ravel(), w).all(), (N, t)
        if N % 4 != 1:
            assert np.array_equal(np.sort(w), np.sort(o)), (N, t)   # closed: reads exactly what it writes
    return ctas, win, out


def brute_force(N):
    """every upper-triangle entry of A' written once; every upper-triangle entry of A read (summed over CTAs) once when closed"""
    ctas, win, out = check_structure(N)
    writes = np.zeros((N, N), np.int32)
    reads = np.zeros((N, N), np.int32)
    for bi, bj in ctas:
        I, J = out[bi][out[bi] >= 0], out[bj][out[bj] >= 0]
        ii, jj = np.meshgrid(I, J, indexing="ij")
        keep = np.ones_like(ii, bool) if bi < bj else ii <= jj
        np.add.at(writes, (np.minimum(ii, jj)[keep], np.maximum(ii, jj)[keep]), 1)
        R, Cc = win[bi][win[bi] >= 0], win[bj][win[bj] >= 0]
        rr, cc = np.meshgrid(R, Cc, indexing="ij")
        keep = np.ones_like(rr, bool) if bi < bj else rr <= cc
        np.add.at(reads, (np.minimum(rr, cc)[keep], np.maximum(rr, cc)[keep]), 1)
    up = np.triu(np.ones((N, N), bool))
    assert np.all(writes[up] == 1) and np.all(writes[~up] == 0), N
    assert np.all(reads[~up] == 0)
    if N % 4 != 1:
        assert np.all(reads[up] == 1), N
    else:
        assert np.all(reads[up] >= 1), N
        assert reads.sum() <= (75 / 64) ** 2 * up.sum() + 4 * 75 * 75, (N, reads.sum() / up.sum())


@pytest.mark.parametrize("lo,hi", [(1, 151), (151, 301), (301, 451), (451, 601)])
def test_every_entry_written_once_and_every_input_in_the_window(lo, hi):
    for N in range(lo, hi):
        brute_force(N)


@pytest.mark.parametrize("N", [4097, 4099, 22000, 22001])
def test_large_orders(N):
    ctas, win, out = check_structure(N)
    if N % 4 == 1:   # the bounded re-read: window rows over output rows, per tile
        ratio = (win >= 0).sum() / (out >= 0).sum()
        assert ratio <= 75 / 64 + 1e-12, ratio


def test_groups_close_except_one_mod_four():
    """the derivation behind the schedule: the orbits of rows under both pairings have at most 4 rows unless N = 1 (mod 4), where from
    N = 9 on they chain further"""
    for N in range(1, 400):
        p1, p2 = rbt.partner(N, 1), rbt.partner(N, 2)
        seen = np.zeros(N, bool)
        biggest = 0
        for i in range(N):
            if seen[i]:
                continue
            orbit, stack = {i}, [i]
            while stack:
                r = stack.pop()
                for q in (p1[r], p2[r]):
                    if q not in orbit:
                        orbit.add(q)
                        stack.append(q)
            seen[list(orbit)] = True
            biggest = max(biggest, len(orbit))
        assert biggest <= 4 if N % 4 != 1 else (biggest > 4 or N < 9), (N, biggest)


def test_bad_arguments():
    L = _lib.lib()
    dims = (ctypes.c_int * 4)()
    assert L.hb_rbt_schedule_view(0, 0, dims, None, None, None) == -1
    assert L.hb_rbt_schedule_view(10, 4, dims, None, None, None) == -1
