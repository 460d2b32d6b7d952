"""The exact scalar-MAC path over pending squares (DESIGN 4.15) at its edges, on size-3 words chosen through cnhe_raw_import_products:
every digit width it accepts (and the first it refuses), 5-, 6- and 7-limb contexts and one whose residues have different digit counts,
the int32 digit-sum bound on both sides with maximal digits under same-sign weights (and, at w = 13, the planner's limit before it), the layer shapes around the wgmma bundles, and
digit planes that drive the plane-source key switch's forward transform to its worst case at |S| near 2^31.

Every case is checked three ways, word for word: the exact path, the same layer over the same products relinearised by a read, and the
closed form of tests/exact_deferred_ref.py on sampled outputs of every plaintext channel.  The wgmma launcher reports on stderr which mode
served a layer ("[umma digits" is the exact path), and every case asserts it, so a silent decline cannot pass."""
import numpy as np
import pytest

import exact_deferred_ref as R
import worst_case_inputs as W
from cryptonets_b200._lib import CnheError
from cryptonets_b200.engine import DENSE, SPARSE, Engine
from oracle.oracle_py import Oracle

pytestmark = pytest.mark.gpu

KERNEL_ENV = ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT", "CNHE_MUL_FUSED", "CNHE_KS_FUSED", "CNHE_NO_LAZY")
T = {4096: 40961, 8192: 786433}


def _engine(monkeypatch, N=4096, dbc=10, q=None, t=None):
    for var in KERNEL_ENV:
        monkeypatch.delenv(var, raising=False)
    monkeypatch.setenv("CNHE_UMMA_PROF", "1")
    eng = Engine(t or [T[N]], N, dbc, 20, -1, coeff_moduli=q)
    eng.keygen(17)
    return eng


def _products(eng, rng, n, dbc, maximal=lambda j: j % 2 == 0):
    """[P][n][3][k][N] canonical words, random, with c2 maximal (lower digits 2^dbc - 1, top digit largest below q_l) where maximal(j)"""
    q = np.array(eng.q, dtype=np.uint64)[:, None]
    words = (rng.integers(0, 1 << 62, (eng.P, n, 3, eng.k, eng.N), dtype=np.uint64) % q).astype(np.uint64)
    top = R.maximal_c2(eng.q, dbc, eng.N)
    for j in range(n):
        if maximal(j):
            words[:, j, 2] = top
    return words


def _served(capfd):
    err = capfd.readouterr().err
    return "[umma digits" in err, "[umma " in err


def _layer(eng, ins, gather, wv, bias, M, K, capfd):
    capfd.readouterr()
    outs = eng.layer_conv_dense(ins, gather, wv, bias, M, K)
    eng.sync()
    return outs, _served(capfd)


def _plains(eng, w, bias):
    """weights (M x K signed) as sparse plaintexts; bias None, or per output a scalar (constant) or N slot values"""
    wv = [eng.plain(np.asarray(row, np.float64), 1.0, SPARSE) for row in w]
    if bias is None:
        return wv, None
    return wv, [eng.plain(np.broadcast_to(np.asarray(b, np.float64), (eng.N,)).copy(), 1.0, DENSE) for b in bias]


def _closed_forms(eng, words, w, gather, bias, dbc, outputs, keys=None):
    """{(channel, m): (2 x k x N) words} of the closed form, for the relinearisation keys of the engine (or `keys`, channel 0)"""
    out = {}
    for ch, t in enumerate(eng.primes):
        orc = Oracle(t, eng.N, -1, dbc, 20, custom_q=eng.q)
        kk = keys if keys is not None else eng.export_key(ch, 2).reshape(-1, 2, eng.k, eng.N)
        wc = R.centred_weights(np.asarray(w, np.int64) % t, t)
        for m in outputs:
            b = None
            if bias is not None:
                b = R.bias_words(orc, np.broadcast_to(np.asarray(bias[m], np.int64) % t, (eng.N,)).astype(np.uint64))
            out[ch, m] = R.closed_form(orc, words[ch], wc, gather, kk, dbc, m, b)
    return out


def _three_ways(eng, words, w, gather, bias, dbc, capfd, exact=True, outputs=None, keys=None):
    """the layer over imported pending products (served exactly or not, as `exact` says), the layer over the same products relinearised
    by a read, and the closed form on sampled outputs of every channel: all the same words.  Returns the first layer's outputs."""
    n = words.shape[1]
    M, K = w.shape
    a = eng.raw_import_products(words, n)
    b = eng.raw_import_products(words, n)
    b[n - 1].export_raw(0, 0)  # a read relinearises the whole group
    wv, bv = _plains(eng, w, bias)
    outs, (got_exact, _) = _layer(eng, a, gather, wv, bv, M, K, capfd)
    assert got_exact == exact, "exact path served: %s, expected %s" % (got_exact, exact)
    outs2, (eager_exact, _) = _layer(eng, b, gather, wv, bv, M, K, capfd)
    assert not eager_exact
    for ch in range(eng.P):
        for m in range(M):
            assert np.array_equal(outs[m].export_raw(ch, 0), outs2[m].export_raw(ch, 0)), (ch, m)
        for j in sorted({0, n // 2, n - 1}):  # the imported products the layer read: still their eager words
            assert np.array_equal(a[j].export_raw(ch, 0), b[j].export_raw(ch, 0)), (ch, j)
    outputs = sorted(set(outputs or []) | {0, M // 2, M - 1})
    for (ch, m), want in _closed_forms(eng, words, w, gather, bias, dbc, outputs, keys).items():
        assert np.array_equal(outs[m].export_raw(ch, 0).reshape(2, eng.k, eng.N), want), (ch, m)
    return outs


def _dense(rng, M, K, wbound=120, big=True):
    w = rng.integers(-wbound, wbound + 1, (M, K))
    w[:, 0] = np.where(w[:, 0] == 0, 7, w[:, 0])
    if big:  # weights past a signed byte: the plan's W2 columns, whose taps carry maximal digits too
        w[:, 1], w[:, 2] = 254, -254
    return w, np.tile(np.arange(K, dtype=np.int32), (M, 1))


# ------------------------------------------------------------------------------------------------------------------ digit widths
@pytest.mark.parametrize("dbc", [4, 8, 9, 13, 16])
def test_digit_widths(dbc, monkeypatch, capfd):
    """the cut's low and high limb masks (the high one 0 for w <= 8, 0xFF at w = 16) and its grouping of LIMBS / 2 digits per c2 pass
    (5 limbs here: 2 digits a pass, residues of 36 and 37 bits with different digit counts at w = 4 and 9)"""
    eng = _engine(monkeypatch, dbc=dbc)
    try:
        rng = np.random.default_rng(dbc)
        words = _products(eng, rng, 24, dbc)
        w, g = _dense(rng, 16, 24)
        bias = [int(v) for v in rng.integers(-500, 500, 16)]
        _three_ways(eng, words, w, g, bias, dbc, capfd)
    finally:
        eng.close()


def test_digit_width_17_is_refused(monkeypatch, capfd):
    """w = 17 is past the 16-bit digit planes: the raw import refuses it, the square relinearises at once (the oracle's words) and a
    layer over such squares is not served by the exact path"""
    eng = _engine(monkeypatch, dbc=17)
    try:
        rng = np.random.default_rng(17)
        with pytest.raises(CnheError) as e:
            eng.raw_import_products(_products(eng, rng, 4, 17), 4)
        assert e.value.code == -1
        xs = [eng.encrypt(rng.integers(-100, 100, eng.N).astype(np.float64), 1.0, DENSE) for _ in range(12)]
        sq = eng.layer_square(xs)
        w, g = _dense(rng, 8, 12)
        outs, (exact, _) = _layer(eng, sq, g, *_plains(eng, w, None), 8, 12, capfd)
        assert not exact
        orc = Oracle(T[4096], 4096, -1, 17, 20)
        orc.keygen(17)
        for i in (0, 11):
            x = xs[i].export_raw(0, 0)
            assert np.array_equal(sq[i].export_raw(0, 0), orc.relinearize(orc.multiply(x, x))), i
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------ limb counts
CONTEXTS = {  # name: N, q, dbc -- limbs = ceil(max bit length / 8)
    "n8192-40bit-5limbs": (8192, W.primes(40, 8192, 3), 10),
    "n4096-44bit-6limbs": (4096, W.primes(44, 4096, 3), 10),
    "n4096-49bit-7limbs": (4096, W.primes(49, 4096, 3), 10),
    "n8192-49bit-7limbs": (8192, W.primes(49, 8192, 3), 10),
    "n4096-mixed-w10": (4096, W.primes(36, 4096) + W.primes(44, 4096) + W.primes(49, 4096), 10),
    "n4096-mixed-w4": (4096, W.primes(36, 4096) + W.primes(44, 4096) + W.primes(49, 4096), 4),
}


@pytest.mark.parametrize("name", list(CONTEXTS))
def test_limb_counts(name, monkeypatch, capfd):
    """k_mac_umma<5 / 6 / 7, true> and the fused key switch on every one of these moduli (the FP64 schedule model gives fp_ok and split_ok
    for each); the mixed contexts cut 4, 5, 5 digits (w = 10: the 36-bit residue skips the rest of the second 3-digit pass) and 9, 11,
    13 digits (w = 4: its last two passes skipped whole)"""
    N, q, dbc = CONTEXTS[name]
    for p in q:
        s = W.fp_schedule(p, N.bit_length() - 1)
        assert s["fp_ok"] and s["split_ok"], p
    eng = _engine(monkeypatch, N=N, dbc=dbc, q=q)
    try:
        assert eng.q == q
        rng = np.random.default_rng(len(name))
        words = _products(eng, rng, 20, dbc)
        w, g = _dense(rng, 16, 20)
        bias = [int(v) for v in rng.integers(-500, 500, 16)]
        _three_ways(eng, words, w, g, bias, dbc, capfd)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------ the bound
BOUND_CASES = [(16, 254), (14, 127), (13, 254)]  # digit width, largest |W|


@pytest.mark.parametrize("dbc,wmax", BOUND_CASES, ids=["w16", "w14", "w13"])
@pytest.mark.parametrize("sign", [1, -1])
def test_digit_sum_bound_both_sides(dbc, wmax, sign, monkeypatch, capfd):
    """every c2 maximal, every weight of one sign: sum |W| = bound_edge(w) takes the exact path with its digit sums at that value, one
    unit more declines and gives the eager words.  w = 16: 32768 on 130 taps of |W| <= 254, so the plan's W2 taps carry maximal digits
    as well, and the sums reach 32768 * 65535 = 2147450880; w = 14: 131080 on 1033 taps of |W| <= 127 (33 weight chunks).
    w = 13: 262176 needs 1033 taps at 254, whose 66 weight chunks (W1 and W2) pass the wgmma kernel's shared memory, so no plan
    exists and the layer declines on both sides of the bound, with the eager words -- pinned here."""
    eng = _engine(monkeypatch, dbc=dbc)
    try:
        e = R.bound_edge(dbc)
        mags = R.edge_weights(e, wmax)
        assert mags[-1] < wmax
        n = len(mags)
        rng = np.random.default_rng(dbc + sign)
        words = _products(eng, rng, n, dbc, maximal=lambda j: True)
        M = 8
        inside = sign * np.tile(np.array(mags, np.int64), (M, 1))
        outside = inside.copy()
        outside[:, -1] += sign
        g = np.tile(np.arange(n, dtype=np.int32), (M, 1))
        t = eng.primes[0]
        S = R.digit_sums(words[0], R.centred_weights(inside % t, t), g, eng.q, dbc, 0)
        assert int(S[0].min()) == int(S[0].max()) == sign * e * ((1 << dbc) - 1)  # a lower digit: the full sum
        assert abs(int(S[0, 0])) < 1 << 31 <= (e + 1) * ((1 << dbc) - 1)
        a = eng.raw_import_products(words, n)
        wv_in, _ = _plains(eng, inside, None)
        wv_out, _ = _plains(eng, outside, None)
        outs_in, (exact_in, _) = _layer(eng, a, g, wv_in, None, M, n, capfd)
        assert exact_in == (dbc != 13), "exact path served at the bound: %s" % exact_in
        outs_out, (exact_out, _) = _layer(eng, a, g, wv_out, None, M, n, capfd)  # reads (relinearises) the group
        assert not exact_out
        outs_eager, (exact_again, _) = _layer(eng, a, g, wv_in, None, M, n, capfd)
        assert not exact_again
        for m in range(M):
            assert np.array_equal(outs_in[m].export_raw(0, 0), outs_eager[m].export_raw(0, 0)), m
        for wts, outs in ((inside, outs_in), (outside, outs_out)):
            for (ch, m), want in _closed_forms(eng, words, wts, g, None, dbc, [0, M - 1]).items():
                assert np.array_equal(outs[m].export_raw(ch, 0).reshape(2, eng.k, eng.N), want), (m, wts[0, -1])
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------ shapes
SHAPES = ["M8", "M129", "M300", "conv-padded", "slot-bias", "no-bias", "two-primes", "zero-mod-one-prime"]


@pytest.mark.parametrize("shape", SHAPES)
def test_shapes(shape, monkeypatch, capfd):
    """one, two and three 128-row wgmma bundles, the last one ragged (the outputs of one gather row share a bundle, so every 128 outputs
    of the wider dense layers read a row of their own: one tap padded), a sliding convolution with padded taps and W2 weights over
    three bundles, a per-slot bias (the generic add_plain on the 2-polynomial outputs before the plane-source key switch), no bias, two
    plaintext primes; and an output whose weights are all zero modulo one plaintext prime, which the layer refuses, leaving the
    pending products readable as their eager words"""
    two = shape in ("two-primes", "zero-mod-one-prime")
    eng = _engine(monkeypatch, t=[40961, 65537] if two else None)
    try:
        rng = np.random.default_rng(len(shape))
        n = 40 if shape == "conv-padded" else 24
        words = _products(eng, rng, n, 10)
        M = {"M8": 8, "M129": 129, "M300": 300, "conv-padded": 300}.get(shape, 16)
        w, g = _dense(rng, M, n)
        for b in range(1, (M + 127) // 128):
            g[128 * b:, n - b] = -1
        bias = [int(v) for v in rng.integers(-500, 500, M)]
        if shape == "conv-padded":
            K = 9
            g = ((np.arange(M)[:, None] * (n - K)) // (M - 1) + np.arange(K)[None, :]).astype(np.int32)
            g[::3, K - 1] = -1
            g[1::5, 0] = -1
            w = rng.integers(-254, 255, (M, K))
            w[:, 4] = np.where(w[:, 4] == 0, 5, w[:, 4])
        if shape == "slot-bias":
            bias = [rng.integers(-500, 500, eng.N) for _ in range(M)]
        if shape == "no-bias":
            bias = None
        if shape == "zero-mod-one-prime":
            a = eng.raw_import_products(words, n)
            w[3] = 40961  # 0 modulo the first plaintext prime, 40961 modulo the second
            wv, bv = _plains(eng, w, bias)
            with pytest.raises(CnheError):
                eng.layer_conv_dense(a, g, wv, bv, M, n)
            one = np.ones((1, 1), np.int64)
            for j in (0, 7, n - 1):  # still pending, and read now: relinearise(product j) -- the closed form of one weight 1
                want = _closed_forms(eng, words[:, j:j + 1], one, None, None, 10, [0])
                for ch in range(eng.P):
                    assert np.array_equal(a[j].export_raw(ch, 0).reshape(2, eng.k, eng.N), want[ch, 0]), (ch, j)
            return
        _three_ways(eng, words, w, g, bias, 10, capfd, outputs=[1, 127, 128, 255, 256] if M > 256 else [1, 127, 128] if M > 128 else [1])
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------------------------ plane extremes
@pytest.mark.parametrize("N", [4096, 8192])
@pytest.mark.parametrize("M", [64, 10])
def test_plane_source_key_switch_extremes(N, M, monkeypatch, capfd):
    """Digit planes S_md = +-254 b_d, |S| up to 254 * 129 * 65535 (about 2^31 - 2^17): b_d is the forward worst case of digit d under
    modulus d % k with coefficients below 129 * dmax_d + 1 (dmax_d the digit's largest value that keeps every word below q), solved
    against the twiddles times 254 so that 254 b_d is the worst case itself, and cut into 129 digits of 129 inputs whose weights are all
    254 (outputs of even index) or all -254 (odd).  The relinearisation keys are NTT-domain constants (worst_case_inputs.key_constant).
    The fused key switch reads these planes in place of cut digits: the same words as the closed form and as the eager layer."""
    dbc, n = 16, 129
    eng = _engine(monkeypatch, N=N, dbc=dbc)
    try:
        q, k = eng.q, eng.k
        dm = W.digit_map(q, dbc)
        orc = Oracle(T[N], N, -1, dbc, 20, custom_q=q)
        targets = W.forward_path_targets(N)
        words = np.zeros((1, n, 3, k, N), np.uint64)
        rng = np.random.default_rng(N + M)
        words[0, :, :2] = (rng.integers(0, 1 << 62, (n, 2, k, N), dtype=np.uint64) % np.array(q, dtype=np.uint64)[:, None]).astype(np.uint64)
        keys = np.zeros((len(dm), 2, k, N), np.uint64)
        wd = {}
        for d, (i, sh) in enumerate(dm):
            l = d % k
            if l not in wd:
                wd[l] = [int(x) * 254 % q[l] for x in W.centred_table(orc.ntt_tables(l)[0], q[l])]
            top = sh + dbc >= q[i].bit_length()
            dmax = ((q[i] - 1) >> sh) - 1 if top else (1 << dbc) - 1
            b = W.forward_worst_case(q[l], wd[l], targets[d % 4], limit=n * dmax + 1).astype(np.int64)
            x = np.clip(b[None, :] - dmax * np.arange(n)[:, None], 0, dmax).astype(np.uint64)  # n digits summing to b
            assert np.array_equal(x.astype(np.int64).sum(axis=0), b)
            words[0, :, 2, i] |= x << np.uint64(sh)
            for ll, p in enumerate(q):
                keys[d, :, ll, :] = W.key_constant(p, 254 * int(b[0]))
        assert all(int(words[0, :, 2, i].max()) < q[i] for i in range(k))
        eng.import_key(0, 2, keys)
        w = np.where(np.arange(M)[:, None] % 2 == 0, 254, -254) * np.ones((M, n), np.int64)
        g = np.tile(np.arange(n, dtype=np.int32), (M, 1))
        S = R.digit_sums(words[0], w, g, q, dbc, 1)
        assert int(np.abs(S).max()) > (1 << 31) - (1 << 18) and int(S.max()) <= 0  # output 1: all weights negative
        _three_ways(eng, words, w, g, None, dbc, capfd, outputs=[1], keys=keys)
    finally:
        eng.close()
