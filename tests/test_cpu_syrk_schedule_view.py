"""The FP64 condensation's work schedule (hb_syrk.cu), checked on the host through hb_syrk_schedule_view: no device needed.

The Gram pass cuts the upper triangle of 128 x 128 output tiles and the K chunks of 32 columns over the CTAs. A CTA runs one off-diagonal
tile, one pair of diagonal tiles (only their cells on and above the diagonal) or, for an odd tile-row count, the last diagonal tile in
full, over a K window, and writes one workspace slot per tile; k_syrk_fixup sums the slots of a tile in a fixed order and keeps the
upper triangle of a diagonal tile. So the result is right when every m16n8 fragment that k_syrk_fixup reads (all of an off-diagonal
tile, those touching the upper triangle of a diagonal one) is computed exactly once for every K chunk. The componentwise error bound of
test_gpu_syrk_schedule.py also needs each entry to be one K-window chain per slot (at most K products) plus a sum of at most G slots.
The schedule balances the SMs by cost: a diagonal pair issues 144 fragments per 16 columns of K, a full tile 128, and a pair is costed
at 162 because its fragments run more slowly per MMA."""
import ctypes

import numpy as np
import pytest

from hiop_b200 import _lib

BM, WBK = 128, 32


def schedule_view(M, K, G):
    """(slots, frags): slots[s] = (CTA, tile row, tile column, first K chunk, K chunk count), frags[s] = per-fragment multiplicity"""
    L = _lib.lib()
    n = ctypes.c_int(-1)
    assert L.hb_syrk_schedule_view(M, K, G, 0, ctypes.byref(n), None, None) == _lib.HB_OK
    slots = np.zeros((n.value, 5), np.int64)
    frags = np.zeros((n.value, 128), np.uint8)
    assert L.hb_syrk_schedule_view(M, K, G, n.value, ctypes.byref(n), slots.ctypes.data, frags.ctypes.data) == _lib.HB_OK
    return slots, frags


def _needed(i, j):
    """fragments (16-row block r, 8-column block c at 16 r + c) of tile (i, j) that k_syrk_fixup reads"""
    r, c = np.divmod(np.arange(128), 16)
    return np.ones(128, bool) if i < j else c >= 2 * r


def check_schedule(M, K, G):
    slots, frags = schedule_view(M, K, G)
    T = -(-M // BM)
    kiters = -(-K // WBK)
    assert len(slots) > 0
    assert slots[:, 0].min() >= 0 and slots[:, 0].max() < G
    assert (slots[:, 4] >= 1).all() and (slots[:, 3] >= 0).all() and (slots[:, 3] + slots[:, 4] <= kiters).all()
    tiles = {}
    for s, (cta, i, j, k0, cnt) in enumerate(slots):
        assert 0 <= i <= j < T
        tiles.setdefault((int(i), int(j)), []).append(s)
    assert sorted(tiles) == [(i, j) for i in range(T) for j in range(i, T)]
    for (i, j), ss in tiles.items():
        assert len(ss) <= G, (i, j, len(ss))   # the fixed-order sum of k_syrk_fixup has at most G terms
        # a CTA writes one slot per tile: its K window is one accumulation chain
        assert len({int(slots[s, 0]) for s in ss}) == len(ss), (i, j)
        need = _needed(i, j)
        for f in np.flatnonzero(need):
            cover = [s for s in ss if frags[s, f]]
            assert all(frags[s, f] == 1 for s in cover), (i, j, f)
            iv = sorted((int(slots[s, 3]), int(slots[s, 3] + slots[s, 4])) for s in cover)
            assert iv and iv[0][0] == 0 and iv[-1][1] == kiters, (i, j, f, iv[:3])
            assert all(a[1] == b[0] for a, b in zip(iv, iv[1:])), (i, j, f)   # no K chunk twice, none missing
    return slots, frags


def dmma_per_cta(slots, frags, G):
    """DMMA.16x8x16 per CTA: each K chunk of 32 columns is two k16 steps of every fragment the CTA computes"""
    per = np.zeros(G, np.int64)
    np.add.at(per, slots[:, 0], 2 * slots[:, 4] * frags.sum(axis=1).astype(np.int64))
    return per


# (M, K): every tile-row count T from 1 to 17 (even T: diagonal tiles all paired; odd T: one left alone), with K tails and K short
# enough to leave fewer unit iterations than SMs
SHAPES = [(128 * T - s, K) for T, s, K in [
    (1, 0, 4126), (1, 28, 1600), (2, 0, 4126), (2, 56, 1040), (3, 84, 6002), (3, 1, 100), (4, 12, 8194), (5, 0, 5000),
    (6, 0, 9214), (7, 40, 8191), (8, 11, 1000000), (8, 12, 125000), (8, 24, 12000), (9, 52, 12030), (10, 1, 7777), (11, 8, 12288),
    (12, 36, 12002), (13, 3, 3001), (14, 20, 12031), (15, 20, 12030), (16, 48, 12288), (17, 0, 12002), (17, 100, 33)]]


@pytest.mark.parametrize("G", [132, 114])
@pytest.mark.parametrize("M,K", SHAPES, ids=[f"M{m}-K{k}" for m, k in SHAPES])
def test_every_needed_fragment_is_computed_once_per_k_chunk(M, K, G):
    check_schedule(M, K, G)


# schedule cost per K chunk (plan_schedule): a full tile 128, a diagonal pair 162 (its 144 fragments run more slowly per MMA than a
# full tile's 128, measured on H100), so each of the pair's two slots 81
COST_TILE, COST_PAIR = 128, 162


def cost_per_cta(slots, frags, G):
    per = np.zeros(G, np.int64)
    full = frags.sum(axis=1) == 128
    np.add.at(per, slots[:, 0], slots[:, 4] * np.where(full, COST_TILE, COST_PAIR // 2))
    return per


@pytest.mark.parametrize("G", [132, 114])
@pytest.mark.parametrize("K", [1000000, 125000])
def test_sms_are_balanced_by_cost(K, G):
    """M = 1013 (m = 1000, l = 6 and the fused rhs row): no SM runs more than 2 % above the mean cost, and the kernel issues
    28 x 128 + 4 x 144 fragments per 16 columns of K instead of the 36 x 128 of full diagonal tiles. (At 132 SMs the four lanes of an
    off-diagonal tile cover all of its K chunks, so those 112 CTAs cannot take more: the 20 that run the pairs sit 1.1 % (K = 1e6) and
    1.5 % (K = 125 000) above the mean.)"""
    slots, frags = check_schedule(1013, K, G)
    cost = cost_per_cta(slots, frags, G)
    kiters = -(-K // WBK)
    assert cost.min() > 0
    assert cost.sum() == kiters * (28 * COST_TILE + 4 * COST_PAIR)
    assert cost.max() <= 1.02 * cost.sum() / G, (cost.max(), cost.sum() / G)
    per = dmma_per_cta(slots, frags, G)
    assert per.sum() == 2 * kiters * (28 * 128 + 4 * 144)


@pytest.mark.parametrize("T", [2, 3, 8, 9])
def test_diagonal_pairs_compute_upper_triangles_only(T):
    """Paired diagonal tiles compute the 72 fragments of their upper triangle, never the 56 below; an unpaired one the full tile"""
    slots, frags = check_schedule(128 * T, 40000, 132)
    for s, (_, i, j, _, _) in enumerate(slots):
        if i == j:
            want = np.ones(128, np.uint8) if (T % 2 and i == T - 1) else _needed(i, i).astype(np.uint8)
            assert np.array_equal(frags[s], want), (T, i)


def test_view_rejects_bad_arguments():
    L = _lib.lib()
    n = ctypes.c_int(0)
    assert L.hb_syrk_schedule_view(0, 100, 132, 0, ctypes.byref(n), None, None) == -1
    assert L.hb_syrk_schedule_view(100, 100, 132, 4, ctypes.byref(n), None, None) == -1
