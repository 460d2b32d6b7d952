"""The worst-case operands of tests/worst_case_inputs.py, run through the exact integer model of the lazy FP64 transforms (no GPU).

The model is first checked to be the transform the oracle computes.  Then, for every ring and every modulus the FP64 path serves:
- the constructed forward input reaches at least 90 % of its path's analytic sum, and the constant class drives the inverse sums
  to their doubling bound;
- for each pass (forward) or stage (inverse) where the schedule sets a re-centre bit, the peak with the schedule stays below 2^52,
  and the peak without that one bit reaches the schedule's limit of 0.9 * 2^52 (up to 1 %).  Where the path can go further, as in
  every inverse segment below 49 bits, it exceeds 2^52; the listing says which.
This is what gives tests/test_gpu_worst_case_operands.py its teeth: there, the kernels must return the oracle's words on these
inputs, which a dropped or misplaced re-centre would not."""
import numpy as np
import pytest

import worst_case_inputs as W

RINGS = {  # name: (t, N, coefficient-modulus count, relinearisation dbc[, custom q]) -- the configurations the GPU tests run
    "default4096": (40961, 4096, -1, 10),
    "cryptonets8192": (549764251649, 8192, -1, 10),
    "cifar16384": (957181001729, 16384, 8, 60),
    # tests/test_gpu_ring_and_modulus_edges.py: the largest 36-, 40- and 44-bit primes = 1 mod 2048 (logN = 10), the two largest 49-bit
    # primes = 1 mod 4096 (logN = 11, the widest modulus of the FP64 schedule)
    "n1024-fp": (12289, 1024, -1, 10, [0xfffffd001, 0xffffff7801, 0xfffffffc001]),
    "n2048-fp49": (40961, 2048, -1, 10, [0x1ffffffff9001, 0x1fffffffe7001]),
}


def _is_prime(n):
    if n < 2:
        return False
    for sp in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37):
        if n % sp == 0:
            return n == sp
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


def fast_bsk(q, t, N):
    """the default ("fast") auxiliary base of context_create: 48-bit primes = 1 mod 2N, as many as B*m_sk > 2^8 N t q needs"""
    need = N.bit_length() - 1 + 8 + t.bit_length() + sum(p.bit_length() for p in q)
    count = max((need + 46) // 47, 2)
    out, cand = [], (1 << 48) + 1
    while len(out) < count:
        cand -= 2 * N
        if _is_prime(cand) and cand not in q and cand != t:
            out.append(cand)
    return out[::-1]


_CACHE = {}


def ring(name):
    """oracle, engine-side modulus list [(kind, p, oracle, table id)] of one ring"""
    if name not in _CACHE:
        from oracle.oracle_py import Oracle
        t, N, count, dbc, *custom = RINGS[name]
        orc = Oracle(t, N, count, dbc, dbc, custom_q=custom[0] if custom else None)
        bo = Oracle(t, N, custom_q=fast_bsk(orc.q, t, N))
        mods = [("q", orc.q[i], orc, i) for i in range(orc.k)] + [("bsk", p, bo, j) for j, p in enumerate(bo.q)]
        _CACHE[name] = (orc, mods)
    return _CACHE[name]


def _tables(o, oid, p):
    w, _, iw, _, inv_n = o.ntt_tables(oid)
    return W.centred_table(w, p), W.centred_table(iw, p), inv_n


def _fp_schedules(logN, sch):
    """(name, passes, mask) of every forward schedule an FP64 kernel runs at this size"""
    out = []
    if logN <= 13:
        out.append(("one-CTA", W.FWD_RADICES[logN], sch["fwd_recenter"]))
    if logN >= 12 and sch["split_ok"]:
        out.append(("split", W.split_radices(logN), sch["fwd_recenter_split"]))
    return out


LIMIT = 0.99 * 0.9 * W.TWO52  # the schedule's limit, less 1 % (its bounds carry a rounding term the exact model does not)


def _over(peak):
    return "" if peak > W.TWO52 else " (below 2^52: within the schedule's 10 % margin)"


def _bits(mask):
    return [b for b in range(32) if (mask >> b) & 1]


def _segment_sum(p, rad, mask, i):
    """largest magnitude any input can reach in the segment of forward passes holding pass i under re-centre mask `mask`: the segment
    starts at the input (p - 1) or at a re-centre (p / 2) and adds at most p / 2 per stage"""
    first = max([j for j in range(i + 1) if (mask >> j) & 1], default=0)
    end = min([j for j in range(i + 1, len(rad)) if (mask >> j) & 1], default=len(rad))
    return ((p // 2) if (mask >> first) & 1 else p - 1) + sum(rad[first:end]) * (p // 2)


@pytest.mark.parametrize("name", list(RINGS))
def test_model_is_the_oracle_transform(name):
    orc, mods = ring(name)
    N = orc.N
    logN = N.bit_length() - 1
    rng = np.random.default_rng(3)
    for kind, p, o, oid in (mods[0], mods[-1]):
        wd, iwd, inv_n = _tables(o, oid, p)
        sch = W.fp_schedule(p, logN)
        a = rng.integers(0, p, N, dtype=np.uint64)
        for label, rad, mask in _fp_schedules(logN, sch):
            x, _ = W.lazy_forward(a, p, wd, rad, mask)
            assert np.array_equal(np.array([int(v) % p for v in x], np.uint64), o.ntt(oid, a)), (kind, label)
        y, _ = W.lazy_inverse(a, p, iwd, inv_n, sch["inv_recenter"])
        assert np.array_equal(np.array([int(v) % p for v in y], np.uint64), o.ntt(oid, a, inverse=True)), kind


@pytest.mark.parametrize("name", list(RINGS))
def test_forward_worst_case_reaches_its_bound(name):
    """every constructed path reaches 90 % of its analytic sum; a schedule bit is needed exactly where that sum crosses the limit"""
    orc, mods = ring(name)
    N = orc.N
    logN = N.bit_length() - 1
    lines = []
    for kind, p, o, oid in mods:
        wd, _, _ = _tables(o, oid, p)
        sch = W.fp_schedule(p, logN)
        assert sch["fp_ok"], (kind, p)
        for out_index in W.forward_path_targets(N):
            a = W.forward_worst_case(p, wd, out_index)
            x, peak0 = W.lazy_forward(a, p, wd, W.split_radices(logN), 0)
            assert abs(int(x[out_index])) >= 0.9 * W.forward_path_sum(p, logN), (kind, out_index)
            assert peak0 == abs(int(x[out_index])), "the path is not the peak"
            for label, rad, mask in _fp_schedules(logN, sch):
                _, peak = W.lazy_forward(a, p, wd, rad, mask)
                assert peak < W.TWO52, (kind, label, out_index)
                for b in _bits(mask):
                    _, peak_wo = W.lazy_forward(a, p, wd, rad, mask & ~(1 << b))
                    if peak_wo > LIMIT:
                        note = _over(peak_wo)
                    else:  # then no input reaches the limit without this bit: even the segment's analytic sum stays below 2^52
                        bound = _segment_sum(p, rad, mask & ~(1 << b), b)
                        assert bound < W.TWO52 and peak_wo >= 0.9 * bound, (kind, label, b, out_index, peak_wo / p)
                        note = " (margin: the analytic sum 2^%.2f is below 2^52; the schedule's bound adds the products' rounding)" % np.log2(bound)
                    if out_index == 0:
                        lines.append("N=%d %s %d-bit %s pass %d: peak %.2f p (2^%.2f) with, %.2f p (2^%.2f) without%s" % (
                            N, kind, p.bit_length(), label, b, peak / p, np.log2(peak), peak_wo / p, np.log2(peak_wo), note))
        # digit planes (the fused key switch's forward, built at N = 4096 / 8192): inputs below 2^dbc
        dbc = RINGS[name][3]
        if kind == "q" and dbc < p.bit_length() and logN in (12, 13):
            a = W.forward_worst_case(p, wd, N - 1, dbc)
            assert int(a.max()) < 1 << dbc
            x, _ = W.lazy_forward(a, p, wd, W.split_radices(logN), 0)
            assert abs(int(x[N - 1])) >= 0.9 * W.forward_path_sum(p, logN, dbc) - logN * (p >> dbc), kind
    print("\n".join(lines))


@pytest.mark.parametrize("name", list(RINGS))
def test_inverse_worst_case_reaches_its_bound(name):
    """the constant class doubles the sums of coefficient 0 at every stage: with the schedule they stay below 2^52, and each
    scheduled re-centre is what keeps them there"""
    orc, mods = ring(name)
    N = orc.N
    logN = N.bit_length() - 1
    lines = []
    for kind, p, o, oid in mods:
        _, iwd, inv_n = _tables(o, oid, p)
        sch = W.fp_schedule(p, logN)
        mask = sch["inv_recenter"]
        for a in (np.full(N, p - 1, np.uint64), np.full(N, W.constant_class(p), object)):
            _, peak = W.lazy_inverse(a, p, iwd, inv_n, mask)
            assert peak < W.TWO52, kind
            _, peak_all = W.lazy_inverse(a, p, iwd, inv_n, 0)
            assert peak_all == N * abs(int(a[0])), "the sums do not add up coherently"
        segs = W.inverse_segments(mask, logN)
        reached = 0
        for n, (b, prev) in enumerate(segs):
            a = np.full(N, W.inverse_constant(p, prev), np.uint64)
            _, peak = W.lazy_inverse(a, p, iwd, inv_n, mask)
            _, peak_wo = W.lazy_inverse(a, p, iwd, inv_n, mask & ~(1 << b))
            assert peak < W.TWO52, (kind, b, peak / p)
            # without bit b the constant class's sums double from the re-centre before it to the stage of the next bit
            end = segs[n + 1][0] if n + 1 < len(segs) else logN - 1
            start = (p - 1) if prev < 0 else int(W.TARGET * p)
            assert peak_wo == start << (end - prev), (kind, b)
            if peak_wo > LIMIT:
                reached += 1
                note = _over(peak_wo)
            else:  # the schedule's bound also counts fresh products summed in later stages, which the constant class lacks
                note = " (not reached by the constant class)"
            lines.append("N=%d %s %d-bit inverse stage %d: peak 2^%.2f with, 2^%.2f without%s" % (
                N, kind, p.bit_length(), b, np.log2(peak), np.log2(peak_wo), note))
        assert reached or not segs, (kind, "no scheduled re-centre of this modulus is shown to be needed")
    print("\n".join(lines))


@pytest.mark.parametrize("name", list(RINGS))
def test_square_and_key_constants(name):
    """the impulse v * delta_0 squares to the NTT-domain constant v^2 = +-TARGET p; a key constant K turns the digit constant v into
    K v = TARGET p"""
    orc, mods = ring(name)
    for kind, p, o, oid in mods[:orc.k]:
        v = W.square_root_near_target(p)
        assert 0.44 * p <= abs(W.centred(v * v, p)) <= W.TARGET * p
        d = (1 << 10) - 3
        assert W.key_constant(p, d) * d % p == int(W.TARGET * p)


def test_mont_rq_words():
    orc, _ = ring("cryptonets8192")
    for r in (W.M_TILDE // 2 - 1, W.M_TILDE // 2, W.M_TILDE - 1):
        x = W.mont_rq_word(orc.q, r)
        assert W.mont_rq_r(x, orc.q) == r
    assert W.mont_rq_r(0, orc.q) == 0


def test_auxiliary_base_bound_at_the_all_max_ciphertext():
    """B * m_sk > 2^8 N t q: the all-(q_i - 1) ciphertext's negacyclic square has coefficients near N Q^2, and the fast base covers
    them with the 2^8 margin the BEHZ floor needs"""
    for name, (t, N, *_) in RINGS.items():
        orc, mods = ring(name)
        Q = 1
        for p in orc.q:
            Q *= p
        Bm = 1
        for kind, p, o, oid in mods:
            if kind == "bsk":
                Bm *= p
        assert Bm > (1 << 8) * N * t * Q, name
        # the all-max word lifted to Bsk is about Q, the tensor square's largest coefficient about N Q^2; t times that over Q is
        # what the floor must carry exactly
        assert N * (Q - 1) * t < Bm, name


def test_digit_map_corners():
    orc, _ = ring("default4096")
    q = orc.q
    assert len(W.digit_map(q, max(p.bit_length() for p in q))) == len(q)
    assert len(W.digit_map(q, 5)) == 24
    assert len(W.digit_map(q, 2)) == 55
    with pytest.raises(ValueError, match="more than 64 digits"):
        W.digit_map(q, 1)
