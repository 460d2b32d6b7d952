"""The Python restatement of the value split and CRT join (tests/values_ref.py) against exact rational arithmetic: the split's residues
name the integer nearest v scale (ties to even) modulo B, and the join is that integer centred, correctly rounded, over the scale."""
import math
import random
from fractions import Fraction

import pytest

import values_ref as vr

PLAIN = {
    "p1": [40961],
    "p2_cryptonets": [549764251649, 549764284417],
    "p2_lola": [2277377, 2424833],
    "p3_126bit": [4398046150657, 4398044938241, 4398044577793],
}


def _nearest_even(q):
    """the integer nearest the rational q, ties to even"""
    f = math.floor(q)
    d = q - f
    if d > Fraction(1, 2) or (d == Fraction(1, 2) and f % 2):
        return f + 1
    return f


def _values(ts, rng):
    B = vr.big_factor(ts)
    vals = [rng.uniform(-1e6, 1e6) for _ in range(200)] + [rng.randint(-10 ** 9, 10 ** 9) + 0.5 for _ in range(50)]
    vals += [0.0, -0.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, float(B // 2), -float(B // 2), float(B), -float(B), 3.0 * B, -3.0 * B, 1e38, -1e38]
    return [v for v in vals if abs(v) < 1.4e38]


@pytest.mark.parametrize("name", list(PLAIN))
def test_split_matches_exact_rounding(name):
    ts = PLAIN[name]
    B = vr.big_factor(ts)
    rng = random.Random(7)
    for scale in (1.0, 3.0, 0.25, 1e-3):
        for v in _values(ts, rng):
            r = vr.split_value(v, scale, ts)
            exact = Fraction(v) * Fraction(scale)
            product = Fraction(float(v) * float(scale))  # one IEEE product: within half an ulp of the exact one
            assert abs(product - exact) <= abs(exact) * Fraction(1, 2 ** 53)
            w = _nearest_even(product)
            if not abs(w) < Fraction(1.5e38):
                assert r is None
                continue
            z = w % B  # the non-negative representative: B - (|w| mod B) for negative w
            assert r == [z % t for t in ts]
            # CRT: the residues name z
            assert sum(c * x for c, x in zip(vr.crt_coeffs(ts), r)) % B == z


@pytest.mark.parametrize("name", list(PLAIN))
def test_join_is_correctly_rounded(name):
    ts = PLAIN[name]
    B = vr.big_factor(ts)
    rng = random.Random(11)
    accs = [rng.randrange(B) for _ in range(300)] + [0, 1, B // 2, B // 2 + 1, B - 1]
    if B > 1 << 60:  # values wider than a double's 53 bits, including exact ties of the conversion
        accs += [(1 << 54) + 2, (1 << 54) + 6, (1 << 55) + 4, (1 << 60) + (1 << 7), B - ((1 << 54) + 2), B - ((1 << 60) + (1 << 7) * 3)]
    for scale in (1.0, 3.0, 1e-3):
        for acc in accs:
            r = [acc % t for t in ts]
            centred = acc - B if 2 * acc > B else acc
            got = vr.join_value(r, scale, ts)
            assert got == float(Fraction(float(centred)) / Fraction(scale))
            assert float(centred) == float(Fraction(centred))  # the integer-to-double step is correctly rounded


def test_round_trip_and_refusals():
    ts = PLAIN["p2_cryptonets"]
    vals = [-3.25, 0.0, 7.5, 1234.0]
    assert vr.join(vr.split(vals, 4.0, ts), 4.0, ts) == [-3.25, 0.0, 7.5, 1234.0]
    for bad in (float("nan"), float("inf"), -float("inf"), 1.5e38, -2e38):
        assert vr.split_value(bad, 1.0, ts) is None
    assert vr.split_value(1e38, 2.0, ts) is None
    with pytest.raises(ValueError):
        vr.split([1.0, float("nan")], 1.0, ts)
