"""The exact model of the FP64 accumulators (tests/fp64_accumulators.py) on the shapes tests/test_gpu_fp64_accumulators.py runs: with the
kernels' re-centre after every 8th term every partial sum stays below 2^53 and every word is exact; without it, or with a period of 64,
the sums pass 2^53 and the words change.  No GPU: the closed form of the diagonal product is checked against the CPU oracle's composition
of rotations, multiply_plain and add on a small case."""
import numpy as np
import pytest

import fp64_accumulators as A
import worst_case_inputs as W

T_PLAIN = 65537  # 1 mod 2N for N = 4096 and 8192
WEIGHT = T_PLAIN - 3


def _report(what, peak):
    print("%-48s peak %.4f * 2^53" % (what, peak / A.TWO53))


@pytest.mark.parametrize("N", [4096, 8192])
def test_diagonal_sums_need_their_recentre(N):
    q = W.primes(49, N, 2)
    w = [A.lift_weight(WEIGHT, T_PLAIN, p) for p in q]
    lengths = list(range(116, 129)) if N == 4096 else [128]
    for name, choose in (("(p-3)/2", A.half_operand), ("widest", A.widest_operand)):
        v = [choose(p, wl) for p, wl in zip(q, w)]
        for l, p in enumerate(q):
            r = A.fmodmul(v[l], w[l], p)
            assert int(r) % p == v[l] * w[l] % p and int(r) % 2 == 1 and abs(r) >= (p - 3) / 2
        for period, bounded in ((8, True), (64, False), (None, False)):
            for l, (peak, exact) in enumerate(A.diag_model(q, v, w, lengths, period)):
                _report("N=%d %s q_%d period %s" % (N, name, l, period), peak)
                assert (peak < A.TWO53) == bounded and exact == bounded


def test_fmodmul_bound_on_canonical_operands():
    """fmodmul of canonical operands below 2^49: |r| <= p/2 + a w 2^-52 < 0.625 p, the bound the kernels' comments cite; the widest
    products found here pass p / 2"""
    for p in W.primes(49, 4096, 2):
        w = A.lift_weight(WEIGHT, T_PLAIN, p)
        r = A.fmodmul(A.widest_operand(p, w), w, p)
        assert p / 2 < abs(r) < 0.625 * p
        # 8 such products on top of a re-centred carry: 5.5 p < 2^52
        assert (0.5 + 8 * 0.625) * p < 2 ** 52


@pytest.mark.parametrize("T", [8, 9, 33, 255])
def test_tensor_sums_need_their_recentre(T):
    """k_behz_tensor_mac_fp over T identical terms, on canonical operands and on the lazy ones the forward re-centring may leave (-p)"""
    p = W.primes(49, 4096, 1)[0]
    col, sp = A.tensor_operands(p)
    peak, exact = A.tensor_model(p, col, sp, T, 8, lazy_reps=(0, -p))
    _report("tensor T=%d period 8" % T, peak)
    assert peak < A.TWO53 and exact
    peak, exact = A.tensor_model(p, col, sp, T, None, lazy_reps=(0, -p))
    _report("tensor T=%d no re-centre" % T, peak)
    assert (peak >= A.TWO53) == (T >= 17) and exact == (T < 17)


def test_closed_form_equals_the_oracle_composition():
    """N = 1024, R = dim = N, n1 = 16, three diagonals dropped: the oracle's rotate_columns, rotate_rows, multiply_plain and add
    composition of the trivial constant ciphertext gives the closed form S v w' at coefficient 0"""
    from cryptonets_b200 import diagonal as dg
    from oracle.oracle_py import Oracle
    N, n1, t = 1024, 16, 12289
    q = W.primes(49, N, 2)
    orc = Oracle(t, N, -1, 10, 20, custom_q=q)
    orc.keygen(5)
    dropped = {(1, 3), (0, 40), (1, 511)}
    M = A.diag_matrix(N, t - 3, dropped)
    w = [A.lift_weight(t - 3, t, p) for p in q]
    v = [A.widest_operand(p, wl, tries=200) for p, wl in zip(q, w)]
    ct = A.trivial_ct(q, v, N)
    model = dg.prerotated_diagonals(np.mod(M, t).astype(np.int64), N, n1, t)
    assert len(model) == N - len(dropped)
    kv = orc.rotate_columns(ct)
    assert np.array_equal(kv, ct)
    baby, inner = {}, {}
    for (b, g, h) in sorted(model, key=lambda k: (k[1], k[0], k[2])):
        assert set(model[(b, g, h)].tolist()) == {t - 3}
        if (b, h) not in baby:
            src = kv if b else ct
            baby[(b, h)] = orc.rotate_rows(src, h) if h else src
        term = orc.multiply_plain(baby[(b, h)], orc.encode(model[(b, g, h)].astype(np.uint64)))
        inner[g] = term if g not in inner else orc.add(inner[g], term)
    want = None
    for g in sorted(inner):
        r = orc.rotate_rows(inner[g], n1 * g) if g else inner[g]
        want = r if want is None else orc.add(want, r)
    assert np.array_equal(want, A.diag_closed_form(q, v, w, len(model), N))
