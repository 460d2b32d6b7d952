"""The CPU oracle at 57- to 61-bit coefficient primes (no GPU).

Decryption scales and rounds through {t, gamma} with gamma = 0x1fffffffffc80001, and the BEHZ base Bsk is SEAL's m_sk = 0x1fffffffffe00001
and the next 61-bit primes = 1 mod 2^18.  Each of them is a valid coefficient prime for every N, so a q holding one makes the inverse of q
modulo it 0 and decryption or the multiply silently wrong.  context_create refuses such a q; the oracle, which also serves as transform
tables of arbitrary NTT primes, builds the context but refuses the operations that would divide by 0 there.  On a q clear of them
(worst_case_inputs.clear_primes) its decryption equals the exact big-integer rounding round(t [c0 + c1 s]_Q / Q) mod t from its own
secret key, which does not go through gamma."""
import numpy as np
import pytest

import worst_case_inputs as W

GAMMA, M_SK = W.GAMMA, W.M_SK
SEAL_AUX_ALL = [0x1fffffffffb40001, 0x1fffffffff500001, 0x1fffffffff380001, 0x1fffffffff000001, 0x1ffffffffef00001, 0x1ffffffffee80001,
                0x1ffffffffeb40001, 0x1ffffffffe780001]  # SEAL's first auxiliary primes (test_oracle_textbook pins the first five)
SEAL_AUX = SEAL_AUX_ALL[:3]


def test_clear_primes_are_pinned():
    assert W.clear_primes(61, 16384, 8) == [0x1fffffffffe10001, 0x1fffffffffdd0001, 0x1fffffffffd08001, 0x1fffffffffcf8001,
                                            0x1fffffffffab0001, 0x1fffffffffa10001, 0x1fffffffff998001, 0x1fffffffff978001]
    assert W.clear_primes(61, 4096, 3) == [0x1ffffffffffde001, 0x1ffffffffffce001, 0x1ffffffffffa4001]
    assert W.clear_primes(61, 2048) == [0x1ffffffffffed001]
    assert W.clear_primes(30, 2048) == [0x3fff4001]
    assert W.clear_primes(57, 2048) == [0x1ffffffffffb001]
    assert W.clear_primes(60, 2048) == [0xfffffffffffc001]
    # the plain search meets m_sk and gamma among the largest 61-bit primes at N = 16384; the clear one skips them and SEAL's base
    assert W.primes(61, 16384, 8)[1] == M_SK and W.primes(61, 16384, 8)[5] == GAMMA
    for p in W.clear_primes(61, 16384, 8):
        assert (p - 1) % (1 << 18) and p not in (GAMMA, M_SK) and W.is_prime(p) and (p - 1) % 32768 == 0


@pytest.mark.parametrize("q, N", [
    (W.primes(61, 16384, 8), 16384),                     # the eight largest 61-bit primes: m_sk and gamma among them
    ([GAMMA], 4096),
    (W.clear_primes(61, 4096, 2) + [GAMMA], 4096),
    ([M_SK], 2048),
    (W.clear_primes(61, 4096, 2) + [M_SK], 4096),
    ([SEAL_AUX[0]], 4096),                                # Bsk = {aux_0, m_sk} at k = 1
    ([W.clear_primes(61, 4096)[0], SEAL_AUX[0]], 4096),   # the issue's case: q = {m_sk-free prime, aux_0}
    (W.clear_primes(61, 4096, 2) + [SEAL_AUX[2]], 4096),  # the third auxiliary prime is in Bsk at k = 3
], ids=["primes61x8", "gamma", "clear-gamma", "msk", "clear-msk", "aux0", "clear-aux0", "clear-aux2"])
def test_oracle_refuses_gamma_and_its_bsk(q, N):
    """decryption refuses a q holding gamma; the multiply, the square layer and both BEHZ stages refuse a q holding a prime of the
    oracle's Bsk (SEAL's m_sk and first k auxiliary primes); the rest of the context works, and what is not refused is right"""
    from oracle.oracle_py import Oracle
    t = 65537
    o = Oracle(t, N, -1, 60, 60, custom_q=q)
    assert o.q == q and o.bsk == SEAL_AUX_ALL[:len(q)] + [M_SK]
    o.keygen(3)
    vals = np.random.default_rng(0).integers(0, t, N, dtype=np.uint64)
    ct = o.encrypt(o.encode(vals), 1)
    assert np.array_equal(o.ntt(0, o.ntt(0, ct[:N]), inverse=True), ct[:N])
    has_gamma, has_bsk = GAMMA in q, bool(set(q) & set(o.bsk))
    assert has_gamma or has_bsk
    if has_gamma:
        with pytest.raises(RuntimeError, match="gamma"):
            o.decrypt(ct)
    else:
        assert np.array_equal(o.decode(o.decrypt(ct)), vals)
    behz = [lambda: o.multiply(ct, ct), lambda: o.square_layer(ct), lambda: o.behz_lift(ct[: len(q) * N]),
            lambda: o.behz_floor(np.zeros((2 * len(q) + 1) * N, np.uint64))]
    for fn in behz:
        if has_bsk:
            with pytest.raises(RuntimeError, match="Bsk"):
                fn()
        else:
            fn()
    if not has_bsk:
        ct2 = o.relinearize(o.multiply(ct, ct))
        if o.noise_budget(ct2) > 0:  # one 61-bit prime leaves no budget for a product at t = 65537
            dec = o.decode(W.exact_decrypt(ct2, _secret(o), q, t))
            assert np.array_equal(dec, (vals.astype(object) ** 2 % t).astype(np.uint64))


def test_auxiliary_prime_outside_the_base_is_accepted():
    """at k = 1 Bsk is {aux_0, m_sk}: the second auxiliary prime is an ordinary coefficient prime there"""
    from oracle.oracle_py import Oracle
    o = Oracle(40961, 4096, custom_q=[SEAL_AUX[1]])
    assert o.bsk == [SEAL_AUX[0], M_SK]
    o.keygen(3)
    vals = np.random.default_rng(0).integers(0, 40961, 4096, dtype=np.uint64)
    ct = o.encrypt(o.encode(vals), 1)
    assert np.array_equal(o.decode(o.decrypt(ct)), vals)


# t, N, q: every width 57..61, in and out of order
CLEAR = {
    "n4096-61x3": (40961, 4096, W.clear_primes(61, 4096, 3)),
    "n2048-mixed": (40961, 2048, W.clear_primes(61, 2048) + W.clear_primes(30, 2048) + W.clear_primes(57, 2048) + W.clear_primes(60, 2048)),
    "n4096-59x2": (65537, 4096, W.clear_primes(59, 4096, 2)),
}


def _secret(o):
    """the oracle's secret key as {-1, 0, 1} coefficients (its export is in NTT form)"""
    sk = o.secret_key().reshape(o.k, o.N)
    return W.ternary_secret(np.stack([o.ntt(l, sk[l], inverse=True) for l in range(o.k)]), o.q)


@pytest.mark.parametrize("name", list(CLEAR))
def test_decryption_equals_exact_rounding(name):
    from oracle.oracle_py import Oracle
    t, N, q = CLEAR[name]
    o = Oracle(t, N, -1, 20, 20, custom_q=q)
    assert o.q == q and not (set(q) & set(o.bsk)) and GAMMA not in q
    o.keygen(17)
    s = _secret(o)
    assert 0.5 < np.count_nonzero(s) / N < 0.8
    rng = np.random.default_rng(5)
    vals = rng.integers(0, t, N, dtype=np.uint64)
    vals[:3] = [(t - 1) // 2, (t + 1) // 2, t - 1]
    ct = o.encrypt(o.encode(vals), 1)
    plain = o.decrypt(ct)
    assert np.array_equal(plain, W.exact_decrypt(ct, s, q, t))
    assert np.array_equal(o.decode(plain), vals)
    assert o.noise_budget(ct) > 0
    # after a multiply and relinearisation, where the noise fills more of q
    ct2 = o.relinearize(o.multiply(ct, ct))
    assert np.array_equal(o.decrypt(ct2), W.exact_decrypt(ct2, s, q, t))
    assert np.array_equal(o.decode(o.decrypt(ct2)), (vals.astype(object) ** 2 % t).astype(np.uint64))


def test_exact_rounding_reference_on_textbook_cases():
    """the reference itself: the trivial ciphertext (Delta m, 0) rounds to m, and c1 = 1 picks up s"""
    t, N = 40961, 2048
    q = W.clear_primes(61, N) + W.clear_primes(30, N)
    Q = q[0] * q[1]
    rng = np.random.default_rng(1)
    s = rng.integers(-1, 2, N)
    m = rng.integers(0, t, N)
    delta = Q // t
    ct = np.zeros((2, 2, N), np.uint64)
    for l, p in enumerate(q):
        ct[0, l] = [(delta * int(v)) % p for v in m]
    assert np.array_equal(W.exact_decrypt(ct, s, q, t), m.astype(np.uint64))
    ct[1, :, 0] = 1                               # c1 = 1: c0 + s, with s of 0 and +-1 rounding away below Delta / 2
    assert np.array_equal(W.exact_decrypt(ct, s, q, t), m.astype(np.uint64))
    x = np.zeros(N, np.int64)
    x[1] = 1                                      # c1 = x, s = x^(N-1): c1 s = x^N = -1
    s2 = np.zeros(N, np.int64)
    s2[N - 1] = 1
    assert list(W.times_ternary(x.astype(np.uint64), s2, q[0])[:2]) == [q[0] - 1, 0]
