"""The reference modulus switch (tests/mod_switch_ref.py) that the GPU kernel is checked against: its residue formula against big-integer
division, and its effect on textbook-BFV ciphertexts (oracle/textbook_bfv.py).  CPU only."""
import math

import numpy as np
import pytest

import mod_switch_ref as R
import worst_case_inputs as W
from oracle import textbook_bfv as tb

BITS = [30, 36, 41, 45, 50, 53, 56, 59, 61]  # 30..61-bit primes = 1 mod 2N (no 48-bit one: worst_case_inputs.primes skips it)


def _moduli(k, order):
    q = [W.primes(b, 1024)[0] for b in BITS[:k]]
    if order == "mixed":  # widest first, narrowest second: q_j > q_i and q_j < q_i both occur
        q = q[::-1][:1] + q[:k - 1]
    return q


def _words(q, n, rng):
    """[2][k][n] residues of n random integers in [0, Q) and of 0, Q - 1 and x = Q - 1 - floor(q_j/2), floor(q_j/2), floor(q_j/2) + 1 for
    every prime"""
    Q = math.prod(q)
    xs = [0, Q - 1]
    for p in q:
        xs += [p >> 1, (p >> 1) + 1, Q - 1 - (p >> 1), (p >> 1) - 1]
    xs += [int(rng.integers(0, 1 << 62)) * int(rng.integers(0, 1 << 62)) % Q for _ in range(n)]
    w = np.array([[x % p for x in xs] for p in q], dtype=np.uint64)
    return np.stack([w, w[:, ::-1].copy()])


@pytest.mark.parametrize("order", ["increasing", "mixed"])
@pytest.mark.parametrize("k", range(2, 10))
def test_residue_formula_is_rounded_division(k, order):
    q = _moduli(k, order)
    rng = np.random.default_rng(k)
    w = _words(q, 40, rng)
    for k2 in range(1, k):
        got = R.mod_switch(w, q, k2)
        for part in range(2):
            assert np.array_equal(got[part], R.mod_switch_big(w[part], q, k2)), (k, order, k2)
    # dropping several primes at once equals dropping them one at a time
    step = w
    for j in range(k - 1, 0, -1):
        step = R.mod_switch(step, q[:j + 1], j)
        assert np.array_equal(step, R.mod_switch(w, q, j))


# ---------------------------------------------------------------- textbook BFV
N_TB, T_TB = 16, 257
Q_TB = [W.primes(b, N_TB)[0] for b in (40, 36, 31, 30)]


def _poly_mod(p, Q):
    return [v % Q for v in p]


def _encrypt(rng, s, m, Q):
    a = [int(x) for x in rng.integers(0, 1 << 62, N_TB)]
    a = [x * 3 % Q for x in a]
    e = [int(x) for x in rng.integers(-3, 4, N_TB)]
    delta = Q // T_TB
    as_ = tb.negacyclic_mul(a, s)
    c0 = [(delta * mi - x + ei) % Q for mi, x, ei in zip(m, as_, e)]
    return [c0, a]


def _residues(polys, q):
    return np.array([[[v % p for v in poly] for p in q] for poly in polys], dtype=np.uint64)


def _budget(polys, s, Q):
    """SEAL's invariant noise budget: bits(Q) - bits(max |[t c(s)]_Q|) - 1"""
    _, acc = tb.decrypt_exact(polys, s, T_TB, Q)
    norm = max(abs(tb.center(T_TB * v % Q, Q)) for v in acc)
    return max(0, Q.bit_length() - norm.bit_length() - 1)


def _multiply(ca, cb, Q):
    ca = [[tb.center(v, Q) for v in p] for p in ca]
    cb = [[tb.center(v, Q) for v in p] for p in cb]
    add = lambda u, v: [x + y for x, y in zip(u, v)]
    d = [tb.negacyclic_mul(ca[0], cb[0]), add(tb.negacyclic_mul(ca[0], cb[1]), tb.negacyclic_mul(ca[1], cb[0])), tb.negacyclic_mul(ca[1], cb[1])]
    return [[tb.round_div(T_TB * v, Q) % Q for v in p] for p in d]


@pytest.mark.parametrize("multiplied", [False, True])
def test_textbook_ciphertext_decrypts_after_the_switch(multiplied):
    """A fresh ciphertext, and a size-3 product, switched from 4 primes to 3 and to 2 decrypt to the same message.  Budget: the switch
    divides t c(s) by q_j and adds t times the rounding r0 + r1 s (+ r2 s^2), |r_i| <= 1/2 -- so the budget after it is at least the
    smaller of the budget before and the floor log2 q' - log2(t B) - 1, B the worst case of that rounding for this s, less one bit."""
    rng = np.random.default_rng(5 + multiplied)
    Q = math.prod(Q_TB)
    s = [int(x) for x in rng.integers(-1, 2, N_TB)]
    ma = [int(x) for x in rng.integers(0, T_TB, N_TB)]
    mb = [int(x) for x in rng.integers(0, T_TB, N_TB)]
    ct = _encrypt(rng, s, ma, Q)
    want = ma
    if multiplied:
        ct = _multiply(ct, _encrypt(rng, s, mb, Q), Q)
        prod = tb.negacyclic_mul(ma, mb)
        want = [v % T_TB for v in prod]
    assert tb.decrypt_exact(ct, s, T_TB, Q)[0] == want
    before = _budget(ct, s, Q)
    s2 = tb.negacyclic_mul(s, s)
    B = 0.5 * (1 + sum(abs(v) for v in s) + (sum(abs(v) for v in s2) if multiplied else 0))
    words = _residues(ct, Q_TB)
    for k2 in (3, 2):
        sw = R.mod_switch(words, Q_TB, k2)
        q2 = Q_TB[:k2]
        Q2 = math.prod(q2)
        polys = [tb.crt_compose(sw[i], q2)[0] for i in range(len(ct))]
        assert tb.decrypt_exact(polys, s, T_TB, Q2)[0] == want, k2
        floor = math.log2(Q2) - math.log2(T_TB * B) - 1
        assert _budget(polys, s, Q2) >= min(before, floor) - 1, (k2, before, floor)
