"""GPU parity at the ring sizes and modulus widths context_create accepts beyond the reference parameter sets: N = 1024 / 2048 (their own
transform instantiations, the non-fused products and the digit-path key switch), one coefficient prime (k = 1 through the digit
decomposition, BEHZ, the gamma decryption and the fused kernels), 49-bit primes at the widest FP64 schedule, 53- and 56-bit primes
next to a 44-bit one (FP64 and integer transforms in one context, 7-limb words), and 30-bit primes (4 limbs).  Every context is an
Engine beside an Oracle of the same t, N and q, keyed with the same seed, compared word for word.

The scalar-MAC cases also pin which kernel serves a layer: the tensor-core kernels join their limb sums in FP64, exact for moduli below
2^50 only, so a context with a wider prime must take the 128-bit integer MAC.  The last test walks the FP64 scalar MAC's gate
(K * max|w| < 2^26) on both sides at maximal words."""
import os

import numpy as np
import pytest

import worst_case_inputs as W

pytestmark = pytest.mark.gpu


_primes = W.primes


# name: t, N, q (None: the default coefficient modulus, cut to `count` primes); fp: FP64 transforms on every q prime; umma: the wgmma
# kernel serves a slab dense layer (every prime of 33..50 bits: 5..7 eight-bit limbs, and the FP64 epilogue exact)
CONTEXTS = {
    "n1024-fp": dict(t=12289, N=1024, q=_primes(36, 1024) + _primes(40, 1024) + _primes(44, 1024), fp=True, umma=True),
    "n2048-fp49": dict(t=40961, N=2048, q=_primes(49, 2048, 2), fp=True, umma=True),
    "n2048-default": dict(t=40961, N=2048, q=None, count=-1, fp=False, umma=False),  # SEAL's one 54-bit prime
    "n4096-k1": dict(t=40961, N=4096, q=None, count=1, fp=True, umma=True),          # one 36-bit prime
    "n4096-mixed": dict(t=40961, N=4096, q=_primes(44, 4096) + _primes(53, 4096) + _primes(56, 4096), fp=False, umma=False),
    "n1024-narrow": dict(t=12289, N=1024, q=_primes(30, 1024, 2), fp=True, umma=False),
}
DBC_R, DBC_G = 10, 20


def test_prime_search_gives_the_listed_primes():
    assert _primes(49, 2048, 2) == [0x1ffffffff9001, 0x1fffffffe7001]
    assert _primes(44, 1024) == [0xfffffffc001]
    assert _primes(30, 1024, 2) == [0x3fff7801, 0x3fff5801]
    assert _primes(53, 4096) == [0x1ffffffffb4001] and _primes(56, 4096) == [0xfffffffffba001]


def _make_pair(name):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONTEXTS[name]
    count = cfg.get("count", -1)
    eng = Engine([cfg["t"]], cfg["N"], DBC_R, DBC_G, count, coeff_moduli=cfg["q"])
    orc = Oracle(cfg["t"], cfg["N"], count, DBC_R, DBC_G, custom_q=cfg["q"])
    assert eng.q == orc.q
    if cfg["q"] is not None:
        assert eng.q == cfg["q"]
    assert not set(eng.bsk) & set(eng.q)
    eng.keygen(1234)
    orc.keygen(1234)
    return eng, orc


@pytest.fixture(scope="module", params=list(CONTEXTS))
def pair(request):
    eng, orc = _make_pair(request.param)
    yield eng, orc, request.param
    eng.close()


def _mod_table(eng, orc):
    """engine modulus id -> (modulus, oracle, oracle table id)"""
    from oracle.oracle_py import Oracle
    bo = Oracle(orc.t, eng.N, custom_q=eng.bsk)
    return [(orc.q[i], orc, i) for i in range(eng.k)] + [(eng.bsk[j], bo, j) for j in range(eng.kb)] + [(orc.t, orc, 2 * orc.k + 1)]


def _fresh_cts(orc, n, seed, nonce0=100):
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, orc.t, (n, orc.N), dtype=np.uint64)
    return vals, np.stack([orc.encrypt(orc.encode(vals[i]), nonce0 + i) for i in range(n)])


def _worst_polys(p, o, oid, N):
    """forward worst cases for every targeted output, then the inverse constant of every scheduled segment (and p - 1)"""
    w, _, _, _, _ = o.ntt_tables(oid)
    wd = W.centred_table(w, p)
    fwd = [W.forward_worst_case(p, wd, j) for j in W.forward_path_targets(N)]
    mask = W.fp_schedule(p, N.bit_length() - 1)["inv_recenter"]
    inv = [np.full(N, W.inverse_constant(p, prev), np.uint64) for _, prev in W.inverse_segments(mask, N.bit_length() - 1)]
    return np.stack(fwd), np.stack([np.full(N, p - 1, np.uint64)] + inv)


def test_fp64_schedule_where_expected(pair):
    """the port of fp_schedule: FP64 transforms on every q prime of the contexts meant for them (and on every 48-bit Bsk prime); in the
    mixed context on the 44-bit prime only"""
    eng, orc, name = pair
    logN = eng.N.bit_length() - 1
    ok = {p: W.fp_schedule(p, logN)["fp_ok"] for p in eng.q + eng.bsk}
    assert all(ok[p] for p in eng.bsk)
    if CONTEXTS[name]["fp"]:
        assert all(ok[p] for p in eng.q), name
    else:
        assert [ok[p] for p in eng.q] == [int(p.bit_length() <= 49) for p in eng.q]
        assert not all(ok[p] for p in eng.q)


def test_ntt_every_modulus(pair):
    """forward and inverse on every modulus id (q, Bsk, t), out of place and in place, rows at 0 and p - 1, and the worst-case operands
    of the FP64 schedule"""
    eng, orc, _ = pair
    rng = np.random.default_rng(1)
    N = eng.N
    for which, (p, o, oid) in enumerate(_mod_table(eng, orc)):
        polys = rng.integers(0, p, (4, N), dtype=np.uint64)
        polys[0, :6] = [0, 1, p - 1, p - 2, p // 2, p // 2 + 1]
        polys[1, :] = p - 1
        polys[2, :] = 0
        fwd, inv = _worst_polys(p, o, oid, N)
        polys = np.concatenate([polys, fwd])
        n = len(polys)
        want = np.stack([o.ntt(oid, a) for a in polys])
        d, out = eng.dev_from(polys), eng.dev_alloc(polys.size)
        eng.raw_ntt(d, out, n, which, 1, False)
        assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), want), (which, "forward out of place")
        eng.raw_ntt(d, d, n, which, 1, False)
        assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), want), (which, "forward in place")
        eng.raw_ntt(out, d, n, which, 1, True)
        assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), polys), (which, "inverse out of place")
        eng.raw_ntt(out, out, n, which, 1, True)
        assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), polys), (which, "inverse in place")
        eng.dev_free(d)
        eng.dev_free(out)
        m = len(inv)
        d, out = eng.dev_from(inv), eng.dev_alloc(inv.size)
        want = np.stack([o.ntt(oid, a, inverse=True) for a in inv])
        eng.raw_ntt(d, out, m, which, 1, True)
        assert np.array_equal(eng.dev_download(out, inv.size).reshape(inv.shape), want), (which, "inverse worst case out of place")
        eng.raw_ntt(d, d, m, which, 1, True)
        assert np.array_equal(eng.dev_download(d, inv.size).reshape(inv.shape), want), (which, "inverse worst case in place")
        eng.dev_free(d)
        eng.dev_free(out)


@pytest.mark.parametrize("in_place", [False, True])
def test_ntt_ragged_batch(pair, in_place):
    """more than 64 * kt polynomials cycling through every q and Bsk modulus, a ragged tail"""
    eng, orc, _ = pair
    rng = np.random.default_rng(2)
    N, kt = eng.N, eng.k + eng.kb
    tab = _mod_table(eng, orc)
    n = 64 * kt + 3
    polys = np.stack([rng.integers(0, tab[b % kt][0], N, dtype=np.uint64) for b in range(n)])
    polys[0, :] = tab[0][0] - 1
    polys[n - 1, :] = 0
    d = eng.dev_from(polys)
    out = d if in_place else eng.dev_alloc(polys.size)
    eng.raw_ntt(d, out, n, 0, kt, False)
    got = eng.dev_download(out, polys.size).reshape(polys.shape)
    for b in [0, 1] + list(range(2, n, 29)) + [n - 2, n - 1]:
        p, o, oid = tab[b % kt]
        assert np.array_equal(got[b], o.ntt(oid, polys[b])), b
    back = d if not in_place else out
    eng.raw_ntt(out, back, n, 0, kt, True)
    assert np.array_equal(eng.dev_download(back, polys.size).reshape(polys.shape), polys)
    eng.dev_free(d)
    if not in_place:
        eng.dev_free(out)


def test_keygen_bit_identical(pair):
    eng, orc, _ = pair
    assert np.array_equal(eng.export_key(0, 0), orc.secret_key())
    assert np.array_equal(eng.export_key(0, 1), orc.public_key())
    assert np.array_equal(eng.export_key(0, 2), orc.relin_keys().ravel())
    assert eng.galois_elts() == orc.galois_elts()
    for elt in eng.galois_elts()[:3] + eng.galois_elts()[-1:]:
        assert np.array_equal(eng.export_key(0, 3, elt), orc.galois_key(elt).ravel()), elt


def test_encrypt_decrypt(pair):
    from cryptonets_b200.engine import DENSE
    eng, orc, _ = pair
    rng = np.random.default_rng(3)
    half = orc.t // 2
    vals = rng.integers(-half, half + 1, eng.N + 17).astype(np.float64)
    vals[:2] = [half, -half]
    v = eng.encrypt(vals, 1.0, DENSE)  # nonces 1, 2 on a fresh context
    assert v.blocks == 2
    lifted = np.where(vals < 0, vals + orc.t, vals).astype(np.uint64)
    want0 = orc.encrypt(orc.encode(lifted[: eng.N]), 1)
    want1 = orc.encrypt(orc.encode(lifted[eng.N:]), 2)
    assert np.array_equal(v.export_raw(0, 0), want0)
    assert np.array_equal(v.export_raw(0, 1), want1)
    assert np.array_equal(eng.decrypt(v), vals)
    assert eng.noise_budget(v, 0, 0) == orc.noise_budget(want0) > 0
    assert eng.noise_budget(v, 0, 1) == orc.noise_budget(want1)


@pytest.mark.parametrize("centered", [0, 1])
def test_products(pair, centered, monkeypatch):
    """multiply, relinearise, multiply + relinearise and the square on 70 ciphertexts drawn from six (the four-per-CTA staged key MAC
    runs on the digit path; a ragged last group), each where it is built fused and separate, against the oracle"""
    eng, orc, name = pair
    eng.set_option("behz_centered_mtilde", centered)
    orc.set_centered_mtilde(centered)
    try:
        N, k = eng.N, eng.k
        m = 70
        vals, few = _fresh_cts(orc, 6, 7, nonce0=3000)
        few[5] = np.tile(np.array(orc.q, dtype=np.uint64) - 1, 2).repeat(N)  # all-maximal words
        src = np.arange(m) % 6
        src[1::2] = np.roll(src[1::2], 1)
        oth = (src + 1) % 6
        want3 = [orc.multiply(few[j], few[(j + 1) % 6]) for j in range(6)]
        want2 = [orc.relinearize(w) for w in want3]
        wantsq = [orc.relinearize(orc.multiply(few[j], few[j])) for j in range(6)]
        a, b = eng.dev_from(few[src]), eng.dev_from(few[oth])
        out3, out2 = eng.dev_alloc(m * 3 * k * N), eng.dev_alloc(m * 2 * k * N)
        results = {}
        for fused in ("1", "0"):  # no effect where the fused kernels are not built
            monkeypatch.setenv("CNHE_KS_FUSED", fused)
            monkeypatch.setenv("CNHE_MUL_FUSED", fused)
            eng.raw_multiply(0, a, b, m, out3)
            got3 = eng.dev_download(out3, m * 3 * k * N).reshape(m, -1)
            for i in range(m):
                assert np.array_equal(got3[i], want3[src[i]]), (fused, "multiply", i)
            eng.raw_relinearize(0, out3, m, out2)
            got2 = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            for i in range(m):
                assert np.array_equal(got2[i], want2[src[i]]), (fused, "relinearize", i)
            eng.raw_multiply_relin(0, a, b, m, out2)
            got2 = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            for i in range(m):
                assert np.array_equal(got2[i], want2[src[i]]), (fused, "multiply_relin", i)
            eng.raw_multiply_relin(0, a, a, m, out2)  # squaring path
            gotsq = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            for i in range(m):
                assert np.array_equal(gotsq[i], wantsq[src[i]]), (fused, "square", i)
            results[fused] = gotsq.copy()
        assert np.array_equal(results["1"], results["0"])
        if orc.noise_budget(want2[0]) > 0:
            dec = orc.decode(orc.decrypt(want2[0]))
            assert np.array_equal(dec, (vals[0].astype(object) * vals[1].astype(object) % orc.t).astype(np.uint64))
        for p in (a, b, out3, out2):
            eng.dev_free(p)
    finally:
        eng.set_option("behz_centered_mtilde", 0)
        orc.set_centered_mtilde(0)


def test_galois_and_rotations(pair):
    eng, orc, _ = pair
    N, k = eng.N, eng.k
    n = 3
    _, cts = _fresh_cts(orc, n, 9)
    cts[2] = np.tile(np.array(orc.q, dtype=np.uint64) - 1, 2).repeat(N)
    a = eng.dev_from(cts)
    out = eng.dev_alloc(n * 2 * k * N)
    for elt in [2 * N - 1, 3, eng.galois_elts()[2], eng.galois_elts()[-1]]:  # 2N - 1: the column rotation
        eng.raw_apply_galois(0, a, n, elt, out)
        got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
        for i in range(n):
            assert np.array_equal(got[i], orc.apply_galois(cts[i], elt)), elt
    assert np.array_equal(orc.apply_galois(cts[0], 2 * N - 1), orc.rotate_columns(cts[0]))
    for steps in [1, -1, N // 8 + 1, -(N // 4 - 3)]:
        eng.raw_rotate_rows(0, a, n, steps, out)
        got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
        for i in range(n):
            assert np.array_equal(got[i], orc.rotate_rows(cts[i], steps)), steps
    eng.dev_free(a)
    eng.dev_free(out)


@pytest.mark.parametrize("feed", ["slab", "gather"])
def test_dense_layer_every_mac_path(pair, feed, capfd):
    """A dense layer of M = 21 outputs over K = 70 taps (three 32-tap chunks, two 64-tap chunks of the scalar MAC): input 0 at all-maximal
    words, weights +-127 and +-254 (beyond a signed byte), an output with one non-zero tap, a bias.  "slab": consecutive ciphertexts of
    one allocation (the wgmma gate), "gather": scattered and permuted with one padded tap (the mma.sync gate).  The default dispatch
    and each forced fall-back must give the oracle's words; wgmma must serve the slab layer exactly where every prime has 33..50 bits."""
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, orc, name = pair
    N = eng.N
    rng = np.random.default_rng(23)
    M, K = 21, 70
    n_in = K + 2
    _, cts = _fresh_cts(orc, n_in, 12, nonce0=900)
    q = np.array(orc.q, dtype=np.uint64)
    cts = cts.reshape(n_in, 2, len(q), N)
    cts[0] = (q - 1)[None, :, None]
    cts[1, :, :, ::2] = (q - 1)[None, :, None]
    cts = cts.reshape(n_in, -1)
    if feed == "slab":
        ins = eng.import_raw_many(cts, n_in, 1, N, 4.0)
        row = np.arange(K, dtype=np.int32)
    else:
        ins = [eng.import_raw(cts[i], 1, N, 4.0) for i in range(n_in)]
        row = (rng.permutation(n_in - 1)[:K] + 1).astype(np.int32)
        row[0] = 0  # input 0 (maximal words) is a real tap
        row[7] = -1
    gather = np.tile(row, (M, 1)).astype(np.int32)
    w = rng.integers(-127, 128, (M, K)).astype(np.float64)
    w[:, 0] = 127
    w[:, 1] = -127
    w[5, 3], w[6, 40], w[20, 69], w[0, 0] = 254, -254, 165, 254
    w[3, :] = 0
    w[3, 2] = 1
    bias = rng.integers(-1000, 1000, M).astype(np.float64)
    wv = [eng.plain(w[i], 1.0, SPARSE) for i in range(M)]
    bv = [eng.plain(np.full(N, bias[i]), 4.0, DENSE) for i in range(M)]
    t = orc.t
    wres = np.where(w < 0, w + t, w).astype(np.uint64)
    bres = np.where(bias * 4 < 0, bias * 4 + t, bias * 4).astype(np.uint64)
    want = orc.mac_layer(cts, gather, wres, bres, M, K, threads=max(4, os.cpu_count() or 1)).reshape(M, -1)
    for forced in (None, "CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA", "CNHE_MAC_INT"):
        os.environ["CNHE_UMMA_PROF"] = "1"  # the wgmma launcher then reports itself on stderr
        if forced:
            os.environ[forced] = "1"
        capfd.readouterr()
        try:
            outs = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
            eng.sync()
        finally:
            del os.environ["CNHE_UMMA_PROF"]
            if forced:
                del os.environ[forced]
        served = "[umma " in capfd.readouterr().err
        for i in range(M):
            assert np.array_equal(outs[i].export_raw(0, 0), want[i]), (forced, served, i)
        assert served == (feed == "slab" and forced is None and CONTEXTS[name]["umma"]), (forced, "wrong kernel served the layer")


def test_fp_mac_gate_edges():
    """N = 8192 CryptoNets context, every input at maximal words (q - 1 and the word whose low 26-bit half is all ones), every weight
    +-131071: K = 511 keeps K * max|w| below 2^26 (the FP64 scalar MAC), K = 513 goes past it (the 128-bit MAC).  Both give the
    oracle's words, and the FP64 MAC equals the one forced onto integers."""
    from cryptonets_b200.engine import Engine, SPARSE
    from oracle.oracle_py import Oracle
    t, N = 549764251649, 8192
    eng = Engine([t], N, 10, 20, -1)
    orc = Oracle(t, N, -1, 10, 20)
    try:
        k = eng.k
        q = np.array(eng.q, dtype=np.uint64)
        low = (((q - np.uint64(1)) >> np.uint64(26)) << np.uint64(26)) | np.uint64((1 << 26) - 1)
        low = np.where(low < q, low, low - np.uint64(1 << 26))
        n_in = 513
        rng = np.random.default_rng(41)
        cts = np.empty((n_in, 2, k, N), np.uint64)
        for i in range(n_in):
            top = (q - 1) if i % 2 == 0 else low
            cts[i] = top[None, :, None]
            if i % 5 == 4:  # some inputs random below their maximum, to keep the sum from being one constant
                cts[i, 1] = rng.integers(0, q[:, None], (k, N), dtype=np.uint64)
        cts = cts.reshape(n_in, -1)
        ins = eng.import_raw_many(cts, n_in, 1, N, 1.0)
        for K in (511, 513):
            assert (K * 131071 < 1 << 26) == (K == 511)
            M = 2
            w = np.full((M, K), 131071.0)
            w[1, 1::3] = -131071.0
            gather = np.tile(np.arange(K, dtype=np.int32), (M, 1))
            wv = [eng.plain(w[i], 1.0, SPARSE) for i in range(M)]
            wres = np.where(w < 0, w + t, w).astype(np.uint64)
            want = orc.mac_layer(cts, gather, wres, None, M, K, threads=max(4, os.cpu_count() or 1)).reshape(M, -1)
            outs = eng.layer_conv_dense(ins, gather, wv, None, M, K)
            os.environ["CNHE_MAC_INT"] = "1"
            try:
                outs_int = eng.layer_conv_dense(ins, gather, wv, None, M, K)
            finally:
                del os.environ["CNHE_MAC_INT"]
            for i in range(M):
                got = outs[i].export_raw(0, 0)
                assert np.array_equal(got, want[i]), (K, i)
                assert np.array_equal(got, outs_int[i].export_raw(0, 0)), (K, i)
    finally:
        eng.close()
