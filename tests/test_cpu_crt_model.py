"""Exactness claims of the Chinese-remainder int8 condensation (hb_crt.cu, DESIGN.md section 3), checked on its Python-integer model
(oracle/crt_model.py): the modulus table and N(K), the range of X against the modulus product and 2^127, the residue formula, the
rounding of a 128-bit integer, the int32 chunk rule, and the error bound."""
from math import prod

import numpy as np
import pytest

from oracle import crt_model as crt


def test_moduli_are_pairwise_coprime_and_n_of_k_matches_the_table():
    assert crt.pairwise_coprime()
    assert crt.MODULI == (256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191)
    assert all(p <= 256 for p in crt.MODULI)
    # the table of the header comment: 16 moduli for 1763 <= K <= 340108, 17 up to 2^20 (t = 53), then t drops by one bit per factor 4
    for K, t, n in [(8, 53, 14), (9, 53, 15), (1762, 53, 15), (1763, 53, 16), (340108, 53, 16), (340109, 53, 17), (10 ** 6, 53, 17),
                    (2 ** 20, 53, 17), (2 ** 20 + 1, 52, 16), (1360434, 52, 16), (1360435, 52, 17), (4194304, 52, 17), (4194305, 51, 16)]:
        assert (crt.bits(K), crt.n_moduli(K)) == (t, n), K
    sw = crt.switch_points(1 << 31)
    assert sw[:6] == [(9, 53, 15), (1763, 53, 16), (340109, 53, 17), (1048577, 52, 16), (1360435, 52, 17), (4194305, 51, 16)]
    assert max(n for _, _, n in sw) <= len(crt.MODULI)       # the device table covers every K below 2^31
    print("switch points (K, t, N):", sw)


@pytest.mark.parametrize("K", [8, 9, 1762, 1763, 340108, 340109, 2 ** 20, 2 ** 20 + 1, 4194304, 4194305, 4 * 10 ** 6, 2 ** 31 - 1])
def test_x_stays_inside_the_modulus_range_and_below_2_127(K):
    t, n = crt.bits(K), crt.n_moduli(K)
    P = prod(crt.MODULI[:n])
    assert K * 2 ** (2 * t) < min(P // 2, 2 ** 127)
    assert K * 2 ** (2 * t) >= prod(crt.MODULI[:n - 1]) // 2   # n is the fewest


@pytest.mark.parametrize("K", [8, 1763, 340109])
def test_worst_case_x_round_trips_through_residues_and_garner(K):
    t, n = crt.bits(K), crt.n_moduli(K)
    for sign in (1, -1):
        X = sign * K * 2 ** (2 * t)                          # every q = +-2^t: the largest |X|
        q = np.array([2.0 ** t])
        res = [crt._bal(sign * K * crt.residues(q, p) ** 2, p) for p in crt.MODULI[:n]]   # K terms r^2 (mod p) of the residue GEMM
        assert int(crt.garner(res)[0]) == X


def test_fma_residue_formula_is_balanced_mod_p_on_edge_values():
    for t in (53, 52, 47):
        for p in crt.MODULI:
            lo, hi = crt.balanced_range(p)
            vals = [2 ** t, -2 ** t, 0, 1, -1, p, -p, p // 2, -(p // 2), (p - 1) // 2 + 1]
            for k in (1, 7, 2 ** 20, 2 ** t // p, -(2 ** t // p)):
                vals += [k * p - 1, k * p, k * p + 1, k * p + p // 2, k * p - p // 2, k * p + (p - 1) // 2 + 1]
            vals = [v for v in vals if abs(v) <= 2 ** t]
            r = crt.residues(np.array(vals, dtype=np.float64), p)
            want = [((v - lo) % p) + lo for v in vals]
            assert r.tolist() == want, (p, t)
            assert r.min() >= lo and r.max() <= hi
    assert crt.residues(np.array([-128.0, 128.0, -2.0 ** 53]), 256).tolist() == [-128, -128, 0]
    assert crt.balanced_range(256) == (-128, 127)


def test_rounding_with_a_sticky_bit_equals_float_of_int():
    rng = np.random.default_rng(5)
    for nb in range(1, 128):
        base = [1 << (nb - 1), (1 << nb) - 1]
        if nb > 54:
            s = nb - 54                                      # 54 bits kept: the last is the rounding bit
            for top in (1 << 53) | 1, (1 << 53) | 2, (1 << 54) - 1, (1 << 53):
                h = (top << s)
                base += [h + (1 << (s - 1)), h + (1 << (s - 1)) - 1, h + (1 << (s - 1)) + 1, h - 1]   # ties and near-ties
        base += [int(rng.integers(1 << 62)) << max(0, nb - 62) for _ in range(4)]
        for x in base:
            x = min(x, (1 << 127) - 1)
            for v in (x, -x):
                assert crt.round_sticky64(v) == float(v), (nb, v)


def test_the_int32_chunk_rule_is_strict_at_all_minus_128():
    worst = crt.CHUNK_STAGES * crt.KS * (-128) * (-128)
    assert worst < 2 ** 31
    assert (crt.CHUNK_STAGES + 1) * crt.KS * 128 * 128 >= 2 ** 31   # one stage more would not be exact
    assert worst + 255 < 2 ** 31                               # plus the running residue of the previous chunks


def _B(M, K, seed, decades=3.0):
    r = np.random.default_rng(seed)
    return r.standard_normal((M, K)) * 10.0 ** r.uniform(-decades, decades, size=(M, 1)) * np.sqrt(10.0 ** r.uniform(-3, 3, size=(1, K)))


@pytest.mark.parametrize("M,K", [(5, 7), (9, 300), (12, 2000)])
def test_brute_force_x_equals_the_residue_route(M, K):
    B = _B(M, K, M + K)
    B[2] = 0.0
    B[3, 1] = 2.0 ** 9                                          # a power-of-two row maximum
    e, t, q = crt.quantize(B)
    X = crt.brute_force_x(B)
    Xr = crt.garner(crt.residue_grams(q, crt.n_moduli(K)))
    assert (X == Xr).all()
    C = crt.condense_bits(B)
    np.testing.assert_array_equal(C, crt.round_scale(X, e, t))
    assert np.array_equal(C, C.T)


def test_bound_holds_on_adversarial_rows_and_is_tight():
    K = 3000
    B = np.full((3, K), 0.25 + 2.0 ** -54)                    # each entry rounds down by half a grid step (tie to even)
    B[:, 0] = 0.75                                            # row maximum in [0.5, 1): e = 0
    B[2] = np.random.default_rng(1).standard_normal(K) * 1e-3
    C = crt.condense_bits(B)
    from fractions import Fraction                            # B B^T exactly
    Bf = [[Fraction(float(x)) for x in row] for row in B]
    G = np.array([[sum(a * b for a, b in zip(Bf[i], Bf[j])) for j in range(3)] for i in range(3)], dtype=object)
    err = np.array([[abs(Fraction(float(C[i, j])) - G[i, j]) for j in range(3)] for i in range(3)], dtype=float)
    R = crt.bound(B, C)
    assert (err <= R).all(), (err, R)
    assert R[0, 1] <= 100 * err[0, 1] and R[0, 0] <= 100 * err[0, 0], (R, err)


def test_mutations_change_the_bits():
    B = _B(6, 2500, 11, decades=1.0)
    B[0] = 1.0 - 2.0 ** -53                                   # |X_00| = K (2^53 - 1)^2 needs all 16 moduli (K = 2500 > 1762)
    B[1, 5] = 0.25 + 2.0 ** -30
    C = crt.condense_bits(B)
    K = B.shape[1]
    assert not np.array_equal(C, crt.condense_bits(B, n=crt.n_moduli(K) - 1))    # the last modulus dropped
    assert not np.array_equal(C, crt.condense_bits(B, t=crt.bits(K) + 1))         # one bit more than t(K)
    assert not np.array_equal(C, crt.condense_bits(B, balanced=False))            # unbalanced digits: X lands in [0, P)
