"""The scalar-MAC bounds model (tests/mac_bounds.py) on the CPU: its words against brute force, its gate boundaries as exact integers,
its closed form against a tap-by-tap sum with SEAL's lifts and against the CPU oracle, and the widest all-+-254 dense window the wgmma
planner fits in shared memory (cnhe_debug_mac_plan runs without a GPU)."""
import numpy as np
import pytest

import mac_bounds as B


def test_maximal_words_against_brute_force():
    rng = np.random.default_rng(1)
    for _ in range(200):
        low_bits = int(rng.integers(1, 9))
        q = int(rng.integers((1 << low_bits) + 1, 1 << 12))
        want = max(x for x in range(q) if x & ((1 << low_bits) - 1) == (1 << low_bits) - 1)
        assert B._largest_with_low_ones(q, low_bits) == want, (q, low_bits)
    for bits in (33, 40, 45, 48, 50):
        for q in B.primes(bits, 4096, 2):
            L = B.limbs(bits)
            x = B.maximal_limb_word(q, bits)
            assert x < q <= x + (1 << 8 * (L - 1)) and x.to_bytes(8, "little")[:L - 1] == b"\xff" * (L - 1)
            h = B.maximal_low_half_word(q)
            assert h < q <= h + (1 << 26) and h & 0x3ffffff == 0x3ffffff


def test_gate_boundaries():
    """imma: K = 33155 puts W1 + W2 limb sums at 2,147,449,350 < 2^31; FP64 with |w| = 2^17 - 1: K = 512; int128: 2 maxbits + bits(K) <= 127"""
    assert B.largest(B.imma_admits, 32) == 33155 and not B.imma_admits(33156) and not B.imma_admits(31)
    assert 33155 * 254 * 255 == 2147449350 < 1 << 31 < 33156 * 254 * 255
    assert B.largest(lambda K: B.fp64_admits(K, 131071, 50)) == 512 and not B.fp64_admits(513, 131071, 50)
    assert not B.fp64_admits(1, 131072, 50) and not B.fp64_admits(1, 1, 51)
    assert B.largest(lambda K: B.int128_admits(K, 56)) == 32767 and not B.int128_admits(32768, 56)
    assert B.largest(lambda K: B.int128_admits(K, 60)) == 127 and not B.int128_admits(128, 60)
    assert B.largest(lambda K: B.int128_admits(K, 61)) == 31
    assert B.largest(B.umma_chunks_admitted) == 2072
    r = B.route
    assert [r(33155, 8, b, 254) for b in (40, 48, 50)] == ["imma"] * 3
    assert [r(33156, 8, b, 254) for b in (40, 48, 50)] == ["fp64"] * 3
    assert (r(512, 8, 50, 131071), r(513, 8, 50, 131071), r(512, 8, 50, 131072)) == ("fp64", "int128", "int128")
    assert (r(32, 8, 32, 254), r(32, 8, 33, 254), r(32, 8, 50, 254), r(32, 8, 51, 254)) == ("fp64", "imma", "imma", "int128")
    assert (r(32, 7, 40, 254), r(31, 8, 40, 254), r(32, 8, 40, 254, rows=2)) == ("fp64",) * 3
    assert (r(32767, 8, 56, 1), r(32768, 8, 56, 1), r(127, 8, 60, 1), r(128, 8, 60, 1)) == ("int128", None, "int128", None)


def _lift(w, t, p):
    """SEAL's lift of a plaintext scalar w (a residue mod t) to q_l: values in the upper half of [0, t) are negative"""
    return (w + p - t) % p if w >= (t + 1) // 2 else w % p


@pytest.mark.parametrize("polys", [2, 3])
def test_closed_form_against_tap_by_tap_sum(polys):
    """repeated and padded taps, signed weights as residues mod t and SEAL's scaled bias (Delta m plus q mod t in the upper half)"""
    rng = np.random.default_rng(polys)
    t, q, N, n_in, M, K = 257, [1000003, 998244353], 8, 4, 6, 9
    Q, dl = q[0] * q[1], B.delta(q, t)
    words = np.stack([rng.integers(0, p, (n_in, polys, N), dtype=np.uint64) for p in q], axis=2)
    gather = rng.integers(-1, n_in, (M, K)).astype(np.int32)
    gather[0] = 2
    w = rng.integers(-(t // 2), t // 2 + 1, (M, K))
    bias = rng.integers(-(t // 2), t // 2 + 1, M)
    bias[0] = -(t // 2)
    got = B.mac_closed_form(words, gather, w, bias, q, t)
    wr, br = B.residues(w, t), B.residues(bias, t)
    for m in range(M):
        for l, p in enumerate(q):
            acc = np.zeros((polys, N), dtype=object)
            for kk in range(K):
                if gather[m, kk] >= 0:
                    acc = (acc + words[gather[m, kk], :, l].astype(object) * _lift(int(wr[m, kk]), t, p)) % p
            b = int(br[m])
            acc[0, 0] = (acc[0, 0] + dl * b + (Q % t if b >= (t + 1) // 2 else 0)) % p
            assert np.array_equal(got[m, :, l].astype(object), acc), (m, l)


def test_closed_form_against_oracle():
    """the CPU oracle's 128-bit multiply-accumulate on 50-bit primes, weights up to +-131071 and repeated inputs"""
    from oracle.oracle_py import Oracle
    t, N = 786433, 2048
    q = B.primes(50, N, 2)
    orc = Oracle(t, N, custom_q=q)
    rng = np.random.default_rng(3)
    n_in, M, K = 5, 9, 40
    words = np.stack([rng.integers(0, p, (n_in, 2, N), dtype=np.uint64) for p in q], axis=2)
    words[0] = np.array([B.maximal_low_half_word(p) for p in q], dtype=np.uint64)[None, :, None]
    gather = rng.integers(-1, n_in, (M, K)).astype(np.int32)
    gather[:, :8] = 0
    w = rng.integers(-131071, 131072, (M, K))
    w[0], w[1] = 131071, -131071
    bias = rng.integers(-(t // 2), t // 2 + 1, M)
    want = orc.mac_layer(words.reshape(n_in, -1), gather, B.residues(w, t), B.residues(bias, t), M, K).reshape(M, 2, 2, N)
    assert np.array_equal(B.mac_closed_form(words, gather, w, bias, q, t), want)


# the widest all-+-254 dense window that fits: 2 c chunks of weights (W1 and W2 columns) next to each kernel's rings
WIDEST = {5: 608, 6: 608, 7: 576}


@pytest.mark.parametrize("limbs", [5, 6, 7])
def test_widest_wgmma_window(limbs):
    """K = 32 c taps, every one needing a W2 column: c main chunks plus c scratch chunks; one chunk more has no plan (the layer goes to
    mma.sync).  The window is far inside the int32 bound of the chunk count."""
    K = B.widest_umma_window(limbs)
    plan = B.umma_plan(*B.wide_dense(16, K), limbs)
    c = K // 32
    assert plan == dict(bundles=1, chunks=2 * c, weight_bytes=2 * c * 4096, extra_taps=K)
    assert B.umma_plan(*B.wide_dense(16, K + 32), limbs) is None
    assert B.umma_plan(*B.wide_dense(16, K + 1), limbs) is None  # a partial chunk costs a whole one
    assert B.umma_chunks_admitted(2 * c)
    assert K == WIDEST[limbs]
