"""The slab plan of the host-resident dense solver (hb_symdense_host.cu), checked on the host through hb_symdense_host_plan_view: no
device needed.

A slab is a run of consecutive 128-row block rows. The factorization copies each slab in and out once, block row by block row from its
diagonal column, and streams columns c0 .. N-1 of every block row before the slab (c0: the slab's first row); LDL^T with several slabs
also copies out the W = L D rows (columns (k+1)*128 .. N-1) of every block row a later slab streams. A solve that does not find the
factor resident streams every block row twice. The plan must put each block row in exactly one slab, in order, stay within the budget,
and refuse a budget that cannot hold one block row next to the ring and the scratch."""
import ctypes

import pytest

from hiop_b200 import _lib

ERR_INVALID = -1
B = 128
SIZES = [0, 1, 127, 128, 129, 1000, 4099, 22000, 120000]


def plan(N, budget):
    """(rc, slabs, first blocks, bytes) of hb_symdense_host_plan_view"""
    L = _lib.lib()
    nblk = -(-N // B)
    dims = (ctypes.c_int * 3)(-1, -1, -1)
    first = (ctypes.c_int * (nblk + 1))()
    b = (ctypes.c_longlong * 5)()
    rc = L.hb_symdense_host_plan_view(N, budget, dims, first, b)
    if rc != _lib.HB_OK:
        return rc, None, None, None
    assert dims[1] == nblk
    return rc, dims[0], [first[i] for i in range(dims[0] + 1)], list(b)


def closed_form(N, first):
    """{h2d, d2h chol, d2h ldl, solve h2d} from the slab boundaries"""
    nblk = -(-N // B)
    io = sum(min(B, N - k * B) * (N - k * B) for k in range(nblk))
    panels = sum(b0 * B * (N - b0 * B) for b0 in first[:-1])
    last = first[-2] if len(first) > 1 else 0
    wout = sum(B * (N - (k + 1) * B) for k in range(last))
    many = len(first) > 2
    return [8 * (io + panels), 8 * io, 8 * (io + wout), 16 * io if many else 0]


def minimum_budget(N):
    """the smallest accepted budget, by bisection (acceptance is monotone in the budget)"""
    hi = 1 << 40
    assert plan(N, hi)[0] == _lib.HB_OK
    lo = 1                    # refused (or, for N = 0, the answer)
    if plan(N, lo)[0] == _lib.HB_OK:
        return lo
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if plan(N, mid)[0] == _lib.HB_OK:
            hi = mid
        else:
            lo = mid
    return hi


@pytest.mark.parametrize("N", SIZES)
def test_every_block_row_in_one_slab_within_budget_and_bytes_match_the_closed_form(N):
    nblk = -(-N // B)
    lo = minimum_budget(N)
    full = plan(N, 1 << 40)[3][0]           # one slab: the peak of the whole factor resident
    budgets = sorted({lo, lo + 1, full - 1, full, full + 4096} | {lo + (full - lo) * i // 13 for i in range(14)})
    prev = None
    for budget in budgets:
        if budget < lo:
            continue
        rc, slabs, first, b = plan(N, budget)
        assert rc == _lib.HB_OK, (N, budget)
        # every block row in exactly one slab, in order; equal heights but the last
        assert first[0] == 0 and first[-1] == nblk and len(first) == slabs + 1
        assert all(first[s] < first[s + 1] for s in range(slabs))
        heights = [first[s + 1] - first[s] for s in range(slabs)]
        assert len(set(heights[:-1])) <= 1 and (not heights or heights[-1] <= heights[0])
        assert b[0] <= budget, (N, budget, b[0])
        assert b[1:] == closed_form(N, first), (N, budget)
        # a larger budget never makes more slabs; the whole factor fits: one slab
        if prev is not None:
            assert slabs <= prev
        prev = slabs
        if budget >= full and N > 0:
            assert slabs == 1 and b[4] == 0
    if N > 0:
        # the minimum is one block row per slab, and one byte less is refused
        rc, slabs, first, b = plan(N, lo)
        assert slabs == nblk and first == list(range(nblk + 1))
        assert plan(N, lo - 1)[0] == ERR_INVALID
        assert b[0] == lo
    else:
        assert plan(N, lo)[1] == 0


def test_minimum_is_one_block_row_the_ring_and_the_scratch():
    """the budget floor grows with N like one block row plus the ring (4 x 128 rows of ld doubles) plus N-sized scratch"""
    for N in (129, 1000, 4099, 22000):
        ld = (N + 7) & ~7
        lo = minimum_budget(N)
        assert 5 * B * ld * 8 <= lo <= 5 * B * ld * 8 + 8 * N * 20 + (1 << 16), (N, lo)


def test_the_paper_estimate_size():
    """N = 120 000 (beyond one 80 GB card) under a 40 GiB budget: three slabs, bytes of the closed form"""
    rc, slabs, first, b = plan(120000, 40 << 30)
    assert rc == _lib.HB_OK and slabs == 3 and b[0] <= 40 << 30
    assert b[1:] == closed_form(120000, first)


def test_zero_budget_and_negative_order_are_refused():
    assert plan(1000, 0)[0] == ERR_INVALID          # 0 means "what is free" to create, which a host-only view cannot know
    assert plan(-1, 1 << 30)[0] == ERR_INVALID
