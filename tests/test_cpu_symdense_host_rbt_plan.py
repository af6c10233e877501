"""The plan of the host-resident dense solver's safe mode (HB_FACT_RBT_NOPIV), checked on the host through
hb_symdense_host_rbt_plan_view and hb_rbt_strip_view: no device needed.

The transform runs strips of butterfly slots. Strip [s0, s1) produces the rows at those slots in each of the four quarters of the
one-GPU transform's schedule, and reads its window: for each quarter a run of consecutive rows (the strip's slots, one more on each side
for N = 1 mod 4), then the three fixed rows {m, 2m+1, 3m+1} of N = 4m + 1. Each window row's upper part is copied from the caller's
matrix from the first column of its run, and its lower part comes from the window's columns of every block row above it. The plan must
produce every row of A' once, keep every level-2 and level-1 partner a strip needs in its window, fit the handle's one allocation, and
refuse a budget that cannot hold one block row next to the ring and the scratch."""
import ctypes

import numpy as np
import pytest

from hiop_b200 import _lib
from oracle import rbt_model as rbt

ERR_INVALID = -1
B = 128
SIZES = list(range(1, 601)) + [4097, 4099, 22000, 22001, 120000]


def plain(N, budget):
    """rc and bytes of hb_symdense_host_plan_view"""
    L = _lib.lib()
    dims = (ctypes.c_int * 3)()
    first = (ctypes.c_int * (-(-N // B) + 1))()
    b = (ctypes.c_longlong * 5)()
    rc = L.hb_symdense_host_plan_view(N, budget, dims, first, b)
    return rc, list(dims), list(b)


def rbt_plan(N, budget):
    """(rc, dims, strip first slots, bytes) of hb_symdense_host_rbt_plan_view"""
    L = _lib.lib()
    dims = (ctypes.c_int * 6)(*([-1] * 6))
    first = (ctypes.c_int * (N + 2))()
    b = (ctypes.c_longlong * 5)()
    rc = L.hb_symdense_host_rbt_plan_view(N, budget, dims, first, b)
    if rc != _lib.HB_OK:
        return rc, None, None, None
    return rc, list(dims), [first[i] for i in range(dims[0] + 1)], list(b)


def strip(N, s0, s1):
    """(window rows by position, -1 for none; the rows the strip produces, -1 past a quarter) of hb_rbt_strip_view"""
    L = _lib.lib()
    wr = ctypes.c_int()
    assert L.hb_rbt_strip_view(N, s0, s1, ctypes.byref(wr), None, None) == _lib.HB_OK
    win = (ctypes.c_int * wr.value)()
    out = (ctypes.c_int * (4 * (s1 - s0)))()
    assert L.hb_rbt_strip_view(N, s0, s1, ctypes.byref(wr), win, out) == _lib.HB_OK
    return np.array(win[:], dtype=np.int64), np.array(out[:], dtype=np.int64)


def minimum_budget(N):
    lo, hi = 1, 1 << 40
    while hi - lo > 1:
        mid = (lo + hi) // 2
        hi, lo = (mid, lo) if plain(N, mid)[0] == _lib.HB_OK else (hi, mid)
    return hi


def runs(N, win):
    """the window's runs (first row, end row): per quarter the held rows of its W positions, then each fixed row alone"""
    fixed = 3 if N % 4 == 1 else 0
    W = (len(win) - fixed) // 4
    out = []
    for a in range(4):
        held = win[a * W:(a + 1) * W]
        held = held[held >= 0]
        if held.size:
            assert np.array_equal(held, np.arange(held[0], held[0] + held.size)), "a quarter's window rows are consecutive"
            out.append((int(held[0]), int(held[-1]) + 1))
    out += [(int(g), int(g) + 1) for g in win[4 * W:] if g >= 0]
    return out


def transform_h2d(N, windows):
    """the closed form: per run, its rows from the run's first column, and the run's columns (those past the block row's first row) of
    every block row of 128"""
    k0 = np.arange(0, N, B, dtype=np.int64)
    nb = np.minimum(B, N - k0)
    total = 0
    for win in windows:
        for g0, g1 in runs(N, win):
            total += (g1 - g0) * (N - g0)
            total += int(np.sum(nb * np.clip(g1 - np.maximum(g0, k0 + 1), 0, None)))
    return 8 * total


def budgets_of(N):
    lo = minimum_budget(N)
    full = plain(N, 1 << 40)[2][0]
    return sorted({lo, lo + (full - lo) // 3, full, 1 << 40})


@pytest.mark.parametrize("N", SIZES)
def test_strips_cover_a_prime_once_partners_in_window_fit_and_bytes_match(N):
    p1, p2 = rbt.partner(N, 1), rbt.partner(N, 2)
    ld = (N + 7) & ~7
    nblk = -(-N // B)
    for budget in budgets_of(N):
        rc, dims, first, b = rbt_plan(N, budget)
        assert rc == _lib.HB_OK, (N, budget)
        strips, T, slots, wr, slabs, H = dims
        # the slab plan and the allocation are the plain plan's
        rc0, d0, b0 = plain(N, budget)
        assert (slabs, H) == (d0[0], d0[2]) and b[0] == b0[0] <= budget
        assert slots == (((N + 1) // 2) + 1) // 2
        assert first == [min(slots, t * T) for t in range(strips)] + [slots] and strips == -(-slots // T)
        produced = np.zeros(N, dtype=np.int64)
        windows = []
        for s0, s1 in zip(first[:-1], first[1:]):
            win, out = strip(N, s0, s1)
            assert len(win) <= wr
            windows.append(win)
            rows = out[out >= 0]
            produced[rows] += 1
            held = set(win[win >= 0].tolist())
            assert len(held) == int(np.sum(win >= 0)), "a row is held at one window position"
            # level 1 reads each output row and its partner after level 2, which reads each of them and its own partner
            need = set(rows.tolist()) | set(p1[rows].tolist())
            need |= set(p2[list(need)].tolist())
            assert need <= held, (N, s0, s1, sorted(need - held)[:5])
        assert np.all(produced == 1), (N, np.nonzero(produced != 1)[0][:5])
        # the strips' X and Y next to the ring (4 x 128 rows of ld), in the one allocation; the scratch in the ring's second halves:
        # diagonals, row sums and norm, or diagonals and b' of 16 right-hand sides (slot 0), and the residual of 16 or the row maps (slot 1)
        assert 2 * wr * ld * 8 + 4 * B * ld * 8 <= b[0]
        assert 8 * (2 * N + 16 * N + 64) <= B * ld * 8 and 8 * (16 * N + 48) <= B * ld * 8 and 4 * (wr + 2 * N + 128) <= B * ld * 8
        # bytes: the transform's closed form, A' out once, the plain factorization plus the diagonal blocks, A' once per residual pass
        diag = sum(min(B, N - k * B) ** 2 for k in range(nblk))
        assert b[1] == transform_h2d(N, windows), (N, budget)
        assert b[2] == 8 * N * N and b[4] == 8 * N * N
        assert b[3] == b0[1] + 8 * diag
    # a budget below one block row, the ring and the scratch is refused, as the plain plan refuses it
    assert rbt_plan(N, minimum_budget(N) - 1)[0] == ERR_INVALID


@pytest.mark.parametrize("N", [22000, 120000])
def test_transform_traffic_is_about_twice_the_upper_triangle(N):
    """about 8 N^2 bytes H2D with few strips (the upper triangle as rows and as mirrored columns), at most 1.5 times that with many"""
    for budget in (1 << 40, minimum_budget(N)):
        rc, dims, first, b = rbt_plan(N, budget)
        assert rc == _lib.HB_OK
        ratio = b[1] / (8.0 * N * N)
        assert 0.95 <= ratio <= (1.1 if dims[0] <= 4 else 1.5), (N, budget, dims, ratio)


def test_zero_budget_and_order_zero():
    assert rbt_plan(1000, 0)[0] == ERR_INVALID
    rc, dims, first, b = rbt_plan(0, 1 << 30)
    assert rc == _lib.HB_OK and dims[0] == 0 and first == [0]
