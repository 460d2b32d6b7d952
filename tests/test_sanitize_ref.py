"""The sanitisation restatement (tests/sanitize_ref.py) on the CPU: the multi-word flood reduction against Python big integers, the nonce
layout, the noise model's rule and budget, and SanitizeLayer on the Raw backend."""
import os
import sys

import numpy as np
import pytest

import sanitize_ref as sr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from noise_model import Model  # noqa: E402

PRIMES = [1073479681, 1099511480321, 4503599626321921, 1152921504606830593, 2305843009213317121]  # 30 to 61 bits, = 1 mod 2^13


@pytest.mark.parametrize("q", PRIMES)
def test_flood_reduction_equals_big_integers(q):
    q_all = PRIMES
    mx = sr.max_bits(q_all, 65537)
    for b in (0, 1, 63, 64, 65, 127, 128, mx):
        f = sr.flood_integers(99, 12345 + b, 64, b)
        W, _ = sr.flood_words(b)
        words = sr.rng64_many(99, sr.san_stream(sr.PURPOSE_F, 12345 + b), np.arange(64 * W, dtype=np.uint64)).reshape(64, W)
        assert all(-(2 ** b) <= v < 2 ** b for v in f)
        assert [sr.reduce_words(words[x], b, q) for x in range(64)] == [v % q for v in f]
        if b >= 8:
            assert min(f) < 0 < max(f)  # both halves of the range are drawn


def test_vectorised_sampler_and_nonce_layout():
    from compact_ref import rng64
    w = sr.rng64_many(7, sr.san_stream(sr.PURPOSE_U, 3), np.arange(5, dtype=np.uint64))
    assert [int(x) for x in w] == [rng64(7, sr.san_stream(sr.PURPOSE_U, 3), i) for i in range(5)]
    assert sr.san_stream(16, (1 << 32) + 5) == (16 << 48) | (5 << 16) | 1
    assert len({sr.san_stream(p, n) for p in (16, 17, 18, 19) for n in (0, 1, 1 << 32, (1 << 48) - 1)}) == 16
    with pytest.raises(AssertionError):
        sr.san_stream(16, 1 << 48)
    t = sr.ternary(w)
    assert set(t.tolist()) <= {-1, 0, 1}


def test_model_rule_and_budget():
    rec = dict(N=8192, q=PRIMES[:4], primes=[2277377], mtilde_centered=True, dbc=40, dbc_galois=40)
    m = Model(rec, 0)
    assert m.flood_bits(20) == 20 + 40 + 13 and m.flood_bits(5, 30) == 5 + 30 + 13
    assert m.max_flood_bits() == sr.max_bits(PRIMES[:4], 2277377)
    b = 60
    assert m.sanitize(m.max_flood_bits() + 3, 150) is None
    got = m.sanitize(b, 150)
    assert abs(got - (m.logq - np.log2(2277377) - b - 1)) < 0.5


def test_sanitize_layer_is_the_identity_on_raw():
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.layers import SanitizeLayer
    from cryptonets_b200.raw import RawFactory
    imgs = nw.synthetic_mnist(1, seed=6)
    plain, _ = nw.lola_small(RawFactory(8192), imgs)
    plain.PrepareNetwork()
    want = np.asarray(plain.GetNext().Decrypt())
    net, _ = nw.lola_small(RawFactory(8192), imgs)
    san = SanitizeLayer(Source=net, NoiseBits=30)
    san.PrepareNetwork()
    assert san.FloodBits(8192) == 30 + 40 + 13
    assert np.array_equal(np.asarray(san.GetNext().Decrypt()), want)
