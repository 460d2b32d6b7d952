"""The constants of the cubic and quartic activations (cnhe_layer_poly, DESIGN.md section 4.12), restated in Python integers.

Per plaintext prime t, for the leading coefficient A invertible mod t:
  quartic  P(x) = A x^4 + B x^3 + C x^2 + D x + E = A q^2 + D' x + E',               q = x^2 + beta x + gamma
  cubic    P(x) = A x^3 + B x^2 + C x + D         = lambda (q1^2 - x^4) + C' x + D',  q1 = x^2 + x + gamma
checked for every x mod t (small primes) or over a spread of residues (large ones), for the plaintext primes of every shipped network
and for random primes = 1 mod 2N.  A = 0 mod t has no inverse there, and the constants refuse it."""
import numpy as np
import pytest

from cryptonets_b200.networks import (CIFAR_PRIMES, CRYPTONETS_PRIMES, LOLA_DENSE_PRIMES, LOLA_LARGE_PRIMES, LOLA_PRIMES,
                                      LOLA_SMALL_PRIMES)


def quartic_constants(t, A, B, C, D, E):
    """(beta, gamma, D', E') mod t"""
    A, B, C, D, E = (v % t for v in (A, B, C, D, E))
    if A == 0:
        raise ValueError("the leading coefficient is 0 mod %d" % t)
    inv2 = pow(2, -1, t)
    beta = B * pow(2 * A, -1, t) % t
    gamma = (C * pow(A, -1, t) - beta * beta) * inv2 % t
    return beta, gamma, (D - B * gamma) % t, (E - A * gamma * gamma) % t


def cubic_constants(t, A, B, C, D):
    """(lambda, gamma, C', D') mod t"""
    A, B, C, D = (v % t for v in (A, B, C, D))
    if A == 0:
        raise ValueError("the leading coefficient is 0 mod %d" % t)
    inv2 = pow(2, -1, t)
    lam = A * inv2 % t
    gamma = (B * pow(lam, -1, t) - 1) * inv2 % t
    return lam, gamma, (C - A * gamma) % t, (D - lam * gamma * gamma) % t


def _is_prime(n):
    if n < 2:
        return False
    for p in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def _random_primes(rng, count):
    out = []
    while len(out) < count:
        N = int(rng.choice([4096, 8192, 16384]))
        bits = int(rng.integers(14, 41))
        c = int(rng.integers(1 << (bits - 1), 1 << bits)) // (2 * N) * (2 * N) + 1
        if _is_prime(c):
            out.append(c)
    return out


SHIPPED = sorted(set(CRYPTONETS_PRIMES + LOLA_SMALL_PRIMES + LOLA_PRIMES + LOLA_DENSE_PRIMES + CIFAR_PRIMES + LOLA_LARGE_PRIMES))
PRIMES = SHIPPED + _random_primes(np.random.default_rng(11), 8) + [40961, 65537, 12289]


def _xs(t, rng):
    """every residue for t < 2^17; else 0, 1, the ends and middle of the range and 4096 random residues"""
    if t < (1 << 17):
        return np.arange(t, dtype=object)
    fixed = [0, 1, 2, t - 1, t - 2, t // 2, t // 2 + 1]
    return np.array(fixed + [int(v) for v in rng.integers(0, t, 4096, dtype=np.int64)], dtype=object)


def _coeffs(t, rng, n):
    # random residues, and a set with negative values and constants in the upper half of t
    yield [int(v) for v in rng.integers(1, t, n, dtype=np.int64)]
    yield [-3, t // 2 + 7, -1, 5, t - 2][:n]


@pytest.mark.parametrize("t", PRIMES)
def test_quartic_identity(t):
    rng = np.random.default_rng(t % 1000003)
    x = _xs(t, rng)
    for A, B, C, D, E in _coeffs(t, rng, 5):
        beta, gamma, D1, E1 = quartic_constants(t, A, B, C, D, E)
        q = (x * x + beta * x + gamma) % t
        got = (A * q * q + D1 * x + E1) % t
        want = ((((A * x + B) * x + C) * x + D) * x + E) % t
        assert np.array_equal(got, want)


@pytest.mark.parametrize("t", PRIMES)
def test_cubic_identity(t):
    rng = np.random.default_rng(t % 1000003 + 1)
    x = _xs(t, rng)
    for A, B, C, D in _coeffs(t, rng, 4):
        lam, gamma, C1, D1 = cubic_constants(t, A, B, C, D)
        u = x * x % t
        q1 = (u + x + gamma) % t
        got = (lam * (q1 * q1 - u * u) + C1 * x + D1) % t
        want = (((A * x + B) * x + C) * x + D) % t
        assert np.array_equal(got, want)


def test_identity_coefficients_give_zero_constants():
    """(1, 0, 0, 0, 0): q = x^2 and P = q^2, so the quartic is the square taken twice"""
    for t in SHIPPED:
        assert quartic_constants(t, 1, 0, 0, 0, 0) == (0, 0, 0, 0)


@pytest.mark.parametrize("t", [40961] + SHIPPED[:3])
def test_leading_coefficient_zero_mod_t_is_refused(t):
    with pytest.raises(ValueError, match=str(t)):
        quartic_constants(t, t, 1, 2, 3, 4)
    with pytest.raises(ValueError, match=str(t)):
        cubic_constants(t, 2 * t, 1, 2, 3)
    # nonzero mod this prime: accepted
    quartic_constants(t, t + 1, 1, 2, 3, 4)
    cubic_constants(t, t - 1, 1, 2, 3)
