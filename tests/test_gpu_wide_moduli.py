"""GPU parity at 57- to 61-bit coefficient primes, the widest context_create accepts, and at the largest auxiliary base (kb = KBMAX = 12).

Above 49 bits everything takes the integer path: Harvey transforms, the 128-bit sums of the key MAC, the summed tensor products, the
scalar-MAC layer and decryption, the BEHZ lift and floor, the modulus switch and the dyadic diagonal product.  Their bounds depend on how
wide the prime is: at 61 bits a product of two words is close to 2^122, so a 128-bit sum holds at most 64 of them.  Every context is an
Engine beside an Oracle of the same t, N, q and seed, compared word for word; decryption is also checked against the exact big-integer
rounding from the exported secret key, which does not go through gamma.  The q primes come from worst_case_inputs.clear_primes, which
avoids gamma and SEAL's Bsk; q holding one of those is refused (the last tests)."""
import io
import os
import zipfile

import numpy as np
import pytest

import compact_keys_ref as kr
import compact_ref as cr
import fp64_accumulators as A
import mod_switch_ref as R
import worst_case_inputs as W
from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
_cp = W.clear_primes

# name: t, N, q, decomposition bit counts (relin, galois), environment at creation
CONTEXTS = {
    "n4096-61x3": dict(t=40961, N=4096, q=_cp(61, 4096, 3), dbc=(10, 20), env={}),
    "n16384-61x8": dict(t=65537, N=16384, q=_cp(61, 16384, 8), dbc=(60, 60), env={}),
    "n2048-mixed": dict(t=40961, N=2048, q=_cp(61, 2048) + _cp(30, 2048) + _cp(57, 2048) + _cp(60, 2048), dbc=(10, 20), env={}),
    "n4096-61-seal": dict(t=40961, N=4096, q=_cp(61, 4096, 2), dbc=(10, 20), env={"CNHE_AUX_BASE": "seal"}),
}
ENV = ("CNHE_AUX_BASE", "CNHE_NTT_INT", "CNHE_KS_FUSED", "CNHE_MUL_FUSED")
SEED = 1234


def _engine(cfg, q=None, seed=SEED):
    from cryptonets_b200.engine import Engine
    saved = {v: os.environ.pop(v, None) for v in ENV}
    os.environ.update(cfg["env"])
    try:
        eng = Engine([cfg["t"]], cfg["N"], cfg["dbc"][0], cfg["dbc"][1], -1, coeff_moduli=cfg["q"] if q is None else q)
    finally:
        for v, val in saved.items():
            os.environ.pop(v, None)
            if val is not None:
                os.environ[v] = val
    if seed is not None:
        eng.keygen(seed)
    return eng


def _oracle(cfg, q=None, seed=SEED):
    from oracle.oracle_py import Oracle
    o = Oracle(cfg["t"], cfg["N"], -1, cfg["dbc"][0], cfg["dbc"][1], custom_q=cfg["q"] if q is None else q)
    o.keygen(seed)
    return o


@pytest.fixture(scope="module", params=list(CONTEXTS))
def pair(request):
    cfg = CONTEXTS[request.param]
    eng, orc = _engine(cfg), _oracle(cfg)
    yield eng, orc, request.param
    eng.close()


@pytest.fixture(scope="module")
def n4096():
    cfg = CONTEXTS["n4096-61x3"]
    eng, orc = _engine(cfg), _oracle(cfg)
    yield eng, orc
    eng.close()


def _mod_table(eng, orc):
    """engine modulus id -> (modulus, oracle, oracle table id); SEAL's base is the oracle's own Bsk (ids k..2k)"""
    from oracle.oracle_py import Oracle
    tab = [(orc.q[i], orc, i) for i in range(eng.k)]
    if eng.bsk == orc.bsk:
        tab += [(eng.bsk[j], orc, eng.k + j) for j in range(eng.kb)]
    else:
        bo = Oracle(orc.t, eng.N, custom_q=eng.bsk)
        tab += [(eng.bsk[j], bo, j) for j in range(eng.kb)]
    return tab + [(orc.t, orc, 2 * orc.k + 1)]


def _maximal(q, N, n=1):
    """n ciphertexts whose every word is q_l - 1"""
    return np.tile(np.tile(np.array(q, dtype=np.uint64) - 1, 2).repeat(N), (n, 1))


def _fresh_cts(orc, n, seed, nonce0=100):
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, orc.t, (n, orc.N), dtype=np.uint64)
    return vals, np.stack([orc.encrypt(orc.encode(vals[i]), nonce0 + i) for i in range(n)])


def _secret(eng, orc):
    sk = eng.export_key(0, 0).reshape(eng.k, eng.N)
    return W.ternary_secret(np.stack([orc.ntt(l, sk[l], inverse=True) for l in range(eng.k)]), eng.q)


# ---------------------------------------------------------------- 1. parameters
def test_parameters(pair):
    """the pinned primes, the base the exactness bound needs (twelve 48-bit primes at 8 x 61 bits), integer transforms on every q prime and
    no FP64 element-wise or lazy path (the FP64 diagonal MAC never launches)"""
    eng, orc, name = pair
    cfg = CONTEXTS[name]
    assert eng.q == orc.q == cfg["q"]
    assert [p.bit_length() for p in eng.q] == {"n4096-61x3": [61] * 3, "n16384-61x8": [61] * 8, "n2048-mixed": [61, 30, 57, 60],
                                               "n4096-61-seal": [61, 61]}[name]
    if name == "n16384-61x8":
        assert [hex(p) for p in eng.q] == ["0x1fffffffffe10001", "0x1fffffffffdd0001", "0x1fffffffffd08001", "0x1fffffffffcf8001",
                                           "0x1fffffffffab0001", "0x1fffffffffa10001", "0x1fffffffff998001", "0x1fffffffff978001"]
        assert eng.kb == 12 and all(b.bit_length() == 48 for b in eng.bsk)
    if name == "n4096-61-seal":
        assert eng.bsk == orc.bsk == [0x1fffffffffb40001, 0x1fffffffff500001, W.M_SK]
    elif name != "n16384-61x8":
        assert all(b.bit_length() == 48 for b in eng.bsk)
    assert not set(eng.bsk) & set(eng.q) and W.GAMMA not in eng.q
    logN = eng.N.bit_length() - 1
    for p in eng.q:
        assert W.fp_schedule(p, logN)["fp_ok"] == int(p.bit_length() <= 49)
    assert not all(W.fp_schedule(p, logN)["fp_ok"] for p in eng.q)
    row = eng.plain(np.ones(4), 1.0)
    d = eng.diag_prepare([row])
    x = eng.encrypt(np.ones(4), 1.0)
    eng.prof_enable(True)
    eng.prof_collect()
    ys = eng.mat_mul_diagonal(d, [x])
    assert eng.prof_collect()["scalar_mac_layer"]["launches"] == 0
    eng.prof_enable(False)
    d.dispose()
    eng.dispose_many([row, x] + ys)


# ---------------------------------------------------------------- 2. transforms
def test_ntt_every_modulus(pair):
    """forward and inverse on every modulus id (q, Bsk, t), out of place and in place: rows of 0, 1, p - 1, p - 2, p / 2, a row of p - 1"""
    eng, orc, _ = pair
    rng = np.random.default_rng(1)
    N = eng.N
    for which, (p, o, oid) in enumerate(_mod_table(eng, orc)):
        polys = rng.integers(0, p, (4, N), dtype=np.uint64)
        polys[0, :6] = [0, 1, p - 1, p - 2, p // 2, p // 2 + 1]
        polys[1, :] = p - 1
        polys[2, :] = 0
        polys[3, ::2] = p - 1
        want = np.stack([o.ntt(oid, a) for a in polys])
        d, out = eng.dev_from(polys), eng.dev_alloc(polys.size)
        eng.raw_ntt(d, out, 4, which, 1, False)
        assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), want), (which, "forward out of place")
        eng.raw_ntt(d, d, 4, which, 1, False)
        assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), want), (which, "forward in place")
        eng.raw_ntt(out, d, 4, which, 1, True)
        assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), polys), (which, "inverse out of place")
        eng.raw_ntt(out, out, 4, which, 1, True)
        assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), polys), (which, "inverse in place")
        inv_want = np.stack([o.ntt(oid, a, inverse=True) for a in polys])
        eng.dev_upload(d, polys)
        eng.raw_ntt(d, out, 4, which, 1, True)
        assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), inv_want), (which, "inverse of arbitrary words")
        eng.dev_free(d)
        eng.dev_free(out)


@pytest.mark.parametrize("in_place", [False, True])
def test_ntt_ragged_batch(pair, in_place):
    """more than 64 (k + kb) polynomials cycling through every q and Bsk modulus, a ragged tail"""
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
    for b in [0, 1] + list(range(2, n, 37)) + [n - 2, n - 1]:
        p, o, oid = tab[b % kt]
        assert np.array_equal(got[b], o.ntt(oid, polys[b])), b
    back = d if not in_place else out
    eng.raw_ntt(out, back, n, 0, kt, True)
    assert np.array_equal(eng.dev_download(back, polys.size).reshape(polys.shape), polys)
    eng.dev_free(d)
    if not in_place:
        eng.dev_free(out)


# ---------------------------------------------------------------- 3. keys, 4. encrypt and decrypt
def test_keygen_bit_identical(pair):
    eng, orc, _ = pair
    assert np.array_equal(eng.export_key(0, 0), orc.secret_key())
    assert np.array_equal(eng.export_key(0, 1), orc.public_key())
    assert np.array_equal(eng.export_key(0, 2), orc.relin_keys().ravel())
    elts = eng.galois_elts()
    assert elts == orc.galois_elts()
    for elt in (elts[0], elts[2], elts[-1]):
        assert np.array_equal(eng.export_key(0, 3, elt), orc.galois_key(elt).ravel()), elt


def test_encrypt_decrypt_and_exact_rounding(pair):
    from cryptonets_b200.engine import DENSE
    eng, orc, _ = pair
    rng = np.random.default_rng(3)
    t, N, half = orc.t, eng.N, orc.t // 2
    eng.keygen(SEED)  # nonces restart at 1
    vals = rng.integers(-half, half + 1, N + 17).astype(np.float64)
    vals[:4] = [half, -half, 0, -1]
    v = eng.encrypt(vals, 1.0, DENSE)
    lifted = np.where(vals < 0, vals + t, vals).astype(np.uint64)
    want = [orc.encrypt(orc.encode(lifted[:N]), 1), orc.encrypt(orc.encode(lifted[N:]), 2)]
    s = _secret(eng, orc)
    for b in range(2):
        ct = v.export_raw(0, b)
        assert np.array_equal(ct, want[b]), b
        plain = W.exact_decrypt(ct, s, eng.q, t)
        assert np.array_equal(plain, orc.encode(lifted[b * N:(b + 1) * N])), b
        assert np.array_equal(plain, orc.decrypt(ct)), b
        assert eng.noise_budget(v, 0, b) == orc.noise_budget(ct) > 0
    assert np.array_equal(eng.decrypt(v), vals)
    m = eng.pointwise_multiply(v, v)  # decryption after a multiply and relinearisation, where the noise fills more of q
    assert np.array_equal(W.exact_decrypt(m.export_raw(0, 0), s, eng.q, t), orc.encode((lifted[:N].astype(object) ** 2 % t).astype(np.uint64)))
    assert np.array_equal(eng.decrypt(m), np.where(vals ** 2 % t > half, vals ** 2 % t - t, vals ** 2 % t))


# ---------------------------------------------------------------- 5. products, 6. rotations
@pytest.mark.parametrize("centered", [0, 1])
def test_products(pair, centered, monkeypatch):
    """multiply, relinearise, multiply + relinearise and the square on 70 ciphertexts drawn from six, one of them all-maximal, fused and
    separate, against the oracle"""
    eng, orc, name = pair
    eng.set_option("behz_centered_mtilde", centered)
    orc.set_centered_mtilde(centered)
    try:
        N, k = eng.N, eng.k
        m = 70
        vals, few = _fresh_cts(orc, 6, 7, nonce0=3000)
        few[5] = _maximal(orc.q, N)[0]
        src = np.arange(m) % 6
        src[1::2] = np.roll(src[1::2], 1)
        oth = (src + 1) % 6
        want3 = [orc.multiply(few[j], few[(j + 1) % 6]) for j in range(6)]
        want2 = [orc.relinearize(w) for w in want3]
        wantsq = [orc.relinearize(orc.multiply(few[j], few[j])) for j in range(6)]
        a, b = eng.dev_from(few[src]), eng.dev_from(few[oth])
        out3, out2 = eng.dev_alloc(m * 3 * k * N), eng.dev_alloc(m * 2 * k * N)
        for fused in ("1", "0"):
            monkeypatch.setenv("CNHE_KS_FUSED", fused)
            monkeypatch.setenv("CNHE_MUL_FUSED", fused)
            eng.raw_multiply(0, a, b, m, out3)
            got3 = eng.dev_download(out3, m * 3 * k * N).reshape(m, -1)
            eng.raw_relinearize(0, out3, m, out2)
            got2 = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            eng.raw_multiply_relin(0, a, b, m, out2)
            got2b = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            eng.raw_multiply_relin(0, a, a, m, out2)  # squaring path
            gotsq = eng.dev_download(out2, m * 2 * k * N).reshape(m, -1)
            for i in range(m):
                assert np.array_equal(got3[i], want3[src[i]]), (fused, "multiply", i)
                assert np.array_equal(got2[i], want2[src[i]]), (fused, "relinearize", i)
                assert np.array_equal(got2b[i], want2[src[i]]), (fused, "multiply_relin", i)
                assert np.array_equal(gotsq[i], wantsq[src[i]]), (fused, "square", i)
        dec = orc.decode(orc.decrypt(want2[0]))
        assert np.array_equal(dec, (vals[0].astype(object) * vals[1].astype(object) % orc.t).astype(np.uint64))
        for p in (a, b, out3, out2):
            eng.dev_free(p)
    finally:
        eng.set_option("behz_centered_mtilde", 0)
        orc.set_centered_mtilde(0)


def test_rotations(pair):
    eng, orc, _ = pair
    N, k = eng.N, eng.k
    n = 3
    _, cts = _fresh_cts(orc, n, 9)
    cts[2] = _maximal(orc.q, N)[0]
    a = eng.dev_from(cts)
    out = eng.dev_alloc(n * 2 * k * N)
    eng.raw_apply_galois(0, a, n, 2 * N - 1, out)  # the column rotation
    got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
    for i in range(n):
        assert np.array_equal(got[i], orc.rotate_columns(cts[i])), i
    for steps in [1, -1, N // 8 + 1, -(N // 4 - 3)]:
        eng.raw_rotate_rows(0, a, n, steps, out)
        got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
        for i in range(n):
            assert np.array_equal(got[i], orc.rotate_rows(cts[i], steps)), (steps, i)
    eng.dev_free(a)
    eng.dev_free(out)


# ---------------------------------------------------------------- 7. summed tensor products on the integer path
@pytest.mark.parametrize("T", [33, 64])
def test_summed_tensor_products_at_maximal_words(n4096, T):
    """k_behz_tensor_mac sums 128-bit products of (q_l - 1)^2 ~ 2^122: the trivial ciphertexts with coefficient 0 = q_l - 1 are q_l - 1
    at every NTT point (their Bsk lift b - 1), so d1 gains 2 (q_l - 1)^2 per term.  T = 33 puts 66 such products past 2^128 unless the
    kernel reduces in between.  Against the closed form and the oracle's composition."""
    from cryptonets_b200.engine import DENSE, SPARSE
    from test_gpu_encrypted_product_deferred import Restatement
    eng, orc = n4096
    q, N = eng.q, eng.N
    top = [p - 1 for p in q]
    w = A.trivial_ct(q, top, N, top)
    col = eng.import_raw(w, 1, N, 1.0, DENSE)
    sparse = eng.import_raw(np.tile(w, T), T, T, 1.0, SPARSE)
    eng.prof_enable(True)
    eng.prof_collect()
    out = eng.mat_mul_colmajor_sparse_deferred([col] * T, sparse)
    prof = eng.prof_collect()
    eng.prof_enable(False)
    assert prof["behz_elementwise"]["launches"] > 0
    Kc = eng.product_sum_terms()
    assert Kc >= T  # one chunk: the kernel sums all T terms
    R_ = Restatement(orc)
    lifted = R_.lifted(w)  # [2][k + 1 + k][N] NTT words of the lifted ciphertext
    for part in range(2):
        for l, p in enumerate(q):
            assert (lifted[part, l] == p - 1).all()
    assert 2 * T * (q[0] - 1) ** 2 >= 1 << 128  # d1's sum of one residue, were it never reduced
    want = R_.output([w] * T, [w] * T, Kc)
    assert np.array_equal(out.export_raw(0, 0), want)
    eng.dispose_many([col, sparse, out])


# ---------------------------------------------------------------- 8. the scalar-MAC layer at the 128-bit gate
def test_mac_layer_at_the_128_bit_gate(n4096, capfd):
    """K (q - 1)^2 < 2^128 must hold for the 128-bit k_mac_layer: at 61 bits K = 31 passes the gate (and gives the oracle's words on all-
    maximal inputs with weights -1 and (t - 1) / 2, no tensor-core or FP64 kernel serving), K = 32 is refused and the context stays usable"""
    from cryptonets_b200.engine import SPARSE
    eng, orc = n4096
    N, t = eng.N, orc.t
    n_in = 33
    cts = _maximal(orc.q, N, n_in)
    ins = eng.import_raw_many(cts, n_in, 1, N, 1.0)
    M = 9
    for K in (31, 32):
        w = np.full((M, K), -1.0)
        w[1, ::3] = (t - 1) // 2
        w[2, :] = (t - 1) // 2
        gather = np.tile(np.arange(K, dtype=np.int32), (M, 1))
        wv = [eng.plain(w[i], 1.0, SPARSE) for i in range(M)]
        if K == 32:
            with pytest.raises(CnheError) as e:
                eng.layer_conv_dense(ins, gather, wv, None, M, K)
            assert e.value.code == ERR_INVALID and "128-bit" in str(e.value)
            break
        wres = np.where(w < 0, w + t, w).astype(np.uint64)
        want = orc.mac_layer(cts, gather, wres, None, M, K, threads=max(4, os.cpu_count() or 1)).reshape(M, -1)
        os.environ["CNHE_UMMA_PROF"] = "1"
        capfd.readouterr()
        eng.prof_enable(True)
        eng.prof_collect()
        try:
            outs = eng.layer_conv_dense(ins, gather, wv, None, M, K)
            eng.sync()
        finally:
            del os.environ["CNHE_UMMA_PROF"]
        assert eng.prof_collect()["scalar_mac_layer"]["launches"] >= 1
        eng.prof_enable(False)
        assert "[umma " not in capfd.readouterr().err
        for i in range(M):
            assert np.array_equal(outs[i].export_raw(0, 0), want[i]), i
    x = eng.encrypt(np.arange(10.0), 1.0)
    assert np.array_equal(eng.decrypt(eng.pointwise_multiply(x, x))[:10], np.arange(10.0) ** 2)


# ---------------------------------------------------------------- 9. diagonal and folded products on the integer path
@pytest.mark.parametrize("fold", [None, 64])
def test_diagonal_product(n4096, fold):
    """a 6 x 300 matrix: decryption equals the plaintext product, the dyadic integer path (no FP64 diagonal MAC launch); with W rows of
    one weight w over dim = N and trivial all-maximal inputs, every word equals the closed form N v w' masked to the first W slots"""
    eng, orc = n4096
    N, t, q = eng.N, orc.t, eng.q
    rng = np.random.default_rng(6)
    Mx = rng.integers(-(t // 2), t // 2 + 1, (6, 300)).astype(np.float64)
    Mx[0, :] = t // 2
    v = rng.integers(-(t // 2), t // 2 + 1, 300).astype(np.float64)
    rows = [eng.plain(r, 1.0) for r in Mx]
    d = eng.diag_prepare(rows, 0, 0, fold_width=fold)
    eng.dispose_many(rows)
    x = eng.encrypt(v, 1.0)
    eng.prof_enable(True)
    eng.prof_collect()
    y = eng.mat_mul_diagonal(d, [x])[0]
    assert eng.prof_collect()["scalar_mac_layer"]["launches"] == 0
    eng.prof_enable(False)
    want = (Mx.astype(np.int64).astype(object) @ v.astype(np.int64).astype(object)) % t
    got = np.mod(np.rint(eng.decrypt(y)).astype(np.int64), t)
    assert np.array_equal(got, want.astype(np.int64))
    d.dispose()
    eng.dispose_many([x, y])
    # closed form on maximal words
    Wd = fold or N
    wt = t - 3
    row = eng.plain(np.full(N, float(wt - t)), 1.0)
    d = eng.diag_prepare([row] * Wd, 64, 0, fold_width=fold)
    xm = eng.import_raw(A.trivial_ct(q, [p - 1 for p in q], N), 1, N, 1.0)
    ym = eng.mat_mul_diagonal(d, [xm])[0]
    wl = [A.lift_weight(wt, t, p) for p in q]
    closed = A.diag_closed_form(q, [p - 1 for p in q], wl, N, N)
    if fold:
        closed = orc.multiply_plain(closed, orc.encode(np.array([1] * Wd + [0] * (N - Wd), np.uint64)))
    assert np.array_equal(ym.export_raw(0, 0), closed)
    d.dispose()
    eng.dispose_many([row, xm, ym])


# ---------------------------------------------------------------- 10. modulus switch
@pytest.mark.parametrize("name", ["n2048-mixed", "n16384-61x8"])
def test_mod_switch_every_drop(name):
    """every k' < k: the planted words (0, Q - 1 and the half boundaries of every dropped prime) equal the reference's; the derived keys
    equal a seeded context's on q[:k'], the packed relinearisation copy included"""
    cfg = CONTEXTS[name]
    eng = _engine(cfg, seed=5)
    try:
        N, q = eng.N, eng.q
        rng = np.random.default_rng(1)
        src = eng.encrypt_many(rng.integers(0, cfg["t"], (2, N)).astype(np.float64))
        words = eng.export_raw_many(src)[0].reshape(2, 1, 2, eng.k, N)
        Q = 1
        for p in q:
            Q *= p
        planted = [0, Q - 1]
        for p in q[1:]:
            planted += [p >> 1, (p >> 1) + 1, Q - (p >> 1) - 1]
        for c, x in enumerate(planted):
            for part in range(2):
                words[0, 0, part, :, c] = [x % p for p in q]
        vin = [eng.import_raw(words[i][None], 1, N, 1.0) for i in range(2)]
        for k2 in range(1, eng.k):
            lvl = eng.derive_level(k2)
            fresh = _engine(cfg, q=q[:k2], seed=5)
            try:
                out = eng.mod_switch(vin, lvl)
                got = lvl.export_raw_many(out)[0].reshape(2, 1, 2, k2, N)
                assert np.array_equal(got, R.mod_switch(words, q, k2)), k2
                assert np.array_equal(got[0, 0, 0], R.mod_switch_big(words[0, 0, 0], q, k2)), k2
                assert lvl.q == q[:k2] and lvl.bsk == fresh.bsk
                for what in (0, 1, 2):
                    assert np.array_equal(lvl.export_key(0, what), fresh.export_key(0, what)), (k2, what)
                assert _has_packed(lvl) == _has_packed(fresh)  # the 48-bit packed copy exists only where every q_l < 2^48
                if _has_packed(fresh):
                    assert np.array_equal(lvl.export_key(0, 4), fresh.export_key(0, 4)), k2
                elts = fresh.galois_elts()
                for elt in (elts[0], elts[len(elts) // 2], elts[-1]):
                    assert np.array_equal(lvl.export_key(0, 3, elt), fresh.export_key(0, 3, elt)), (k2, elt)
            finally:
                fresh.close()
                lvl.close()
    finally:
        eng.close()


def _has_packed(eng):
    try:
        eng.export_key(0, 4)
        return True
    except CnheError:
        return False


# ---------------------------------------------------------------- 11. compact formats
@pytest.mark.parametrize("name", ["n4096-61x3", "n2048-mixed"])
def test_compact_upload_and_keys(name):
    """residues of 61, 30, 57 and 60 bits straddle 64-bit words at many offsets: the compact upload against its restatement and the
    client's own words, and a server on the compact evaluation keys against the restated keys and the client's results"""
    from cryptonets_b200.engine import Engine
    cfg = CONTEXTS[name]
    eng = _engine(cfg, seed=4242)
    orc = _oracle(cfg, seed=4242)
    try:
        N, q, k = eng.N, eng.q, eng.k
        vals = np.random.default_rng(1).integers(-50, 51, (3, N + 100)).astype(np.float64)
        blob = eng.encrypt_compact(vals, 1.0)
        key = cr.seeded_key(4242, 1)
        hdr = cr.parse(blob)
        assert hdr["q"] == q and hdr["keys"] == [key]
        want = []
        for i in range(3):
            for b in range(2):
                seg = vals[i, b * N: (b + 1) * N].astype(np.int64) % orc.t
                want.append(cr.encrypt_symmetric(orc, 4242, orc.encode(seg.astype(np.uint64)), 1 + 2 * i + b, cr.expand_c1_ct(key, 2 * i + b, q, N)))
        want = np.stack(want)
        for j in range(6):
            assert np.array_equal(cr.unpack_ct_c0(hdr["payload"][0, j], q, N), want[j, : k * N].reshape(k, N)), j
        assert blob == cr.build_header(N, k, 1, 3, 2, N + 100, 1.0, q, [orc.t], [key]) + np.concatenate(
            [cr.pack_ct_c0(want[j, : k * N].reshape(k, N), q, N) for j in range(6)]).astype("<u8").tobytes()
        vecs = eng.import_compact(blob)
        assert np.array_equal(eng.export_raw_many(vecs).reshape(want.shape), want)
        assert np.array_equal(eng.decrypt_many(vecs), vals)
        # compact evaluation keys
        eng.keygen(4242)
        elts = sorted(eng.galois_elts())
        listed = [elts[1], elts[-2]]
        kblob = eng.save_compact_keys(galois=listed)
        want_blob, keys = kr.expected_keys([orc], 4242, kr.SET_PUBLIC | kr.SET_RELIN, listed)
        assert kblob == want_blob
        server = Engine(None, compact_keys=kblob)
        try:
            assert server.q == q and server.bsk == eng.bsk
            assert np.array_equal(server.export_key(0, 1).reshape(keys[0]["pk"].shape), keys[0]["pk"])
            assert np.array_equal(server.export_key(0, 2).reshape(keys[0]["rlk"].shape), keys[0]["rlk"])
            for g in listed:
                assert np.array_equal(server.export_key(0, 3, g).reshape(keys[0]["glk"][g].shape), keys[0]["glk"][g]), g
            raw = eng.export_raw_many(vecs[:2])
            sv = server.import_raw_many(raw, 2, 2, N + 100)
            prod = server.pointwise_multiply(sv[0], sv[1])
            back = eng.import_raw_many(server.export_raw_many([prod]), 1, 2, N + 100)
            assert np.array_equal(eng.decrypt(back[0]), vals[0] * vals[1])
        finally:
            server.close()
    finally:
        eng.close()


# ---------------------------------------------------------------- 12. refusals
def _exact_check_or_fail(eng, what):
    """a context that should not exist: show whether it decrypts (exact rounding from its own secret key, transformed on the GPU)"""
    N, k = eng.N, eng.k
    eng.keygen(SEED)
    sk = eng.dev_from(eng.export_key(0, 0))
    eng.raw_ntt(sk, sk, k, 0, k, True)
    s = W.ternary_secret(eng.dev_download(sk, k * N).reshape(k, N), eng.q)
    eng.dev_free(sk)
    vals = np.random.default_rng(0).integers(-100, 100, N).astype(np.float64)
    v = eng.encrypt(vals, 1.0)
    plain = W.exact_decrypt(v.export_raw(0, 0), s, eng.q, eng.primes[0])
    assert np.array_equal(eng.decrypt(v), vals), "%s: decryption returns wrong values (the exact rounding from its secret key gives %s...)" % (what, plain[:4])
    pytest.fail("%s was accepted" % what)


def test_gamma_in_q_is_refused():
    """the eight largest 61-bit primes = 1 mod 2^15 hold gamma (and m_sk, harmless with the fast base)"""
    q = W.primes(61, 16384, 8)
    assert W.GAMMA in q
    cfg = dict(CONTEXTS["n16384-61x8"], q=q)
    try:
        eng = _engine(cfg, seed=None)
    except CnheError as e:
        assert e.code == ERR_INVALID and "gamma" in str(e)
        return
    try:
        _exact_check_or_fail(eng, "q holding gamma")
    finally:
        eng.close()


@pytest.mark.parametrize("prime", [W.M_SK, 0x1fffffffffb40001], ids=["m_sk", "aux0"])
def test_seal_base_in_q_is_refused(prime):
    cfg = dict(CONTEXTS["n4096-61-seal"], q=[_cp(61, 4096)[0], prime])
    with pytest.raises(CnheError) as e:
        _engine(cfg, seed=None)
    assert e.value.code == ERR_INVALID and "Bsk" in str(e.value)
    eng = _engine(dict(cfg, env={}), seed=None)  # the fast base has no 61-bit prime: the same q is an ordinary modulus there
    try:
        assert prime in eng.q and all(b.bit_length() == 48 for b in eng.bsk)
    finally:
        eng.close()


def test_nine_61_bit_primes_need_too_large_a_base():
    cfg = dict(CONTEXTS["n16384-61x8"], q=_cp(61, 16384, 9))
    with pytest.raises(CnheError) as e:
        _engine(cfg, seed=None)
    assert e.value.code == ERR_INVALID and "auxiliary base" in str(e.value)


def _gamma_blob_q(q):
    """q with its first 61-bit prime replaced by gamma (same width, so every size in a blob stays valid)"""
    i = next(i for i, p in enumerate(q) if p.bit_length() == 61)
    return i, q[:i] + [W.GAMMA] + q[i + 1:]


def test_loaded_contexts_refuse_gamma():
    """the key archive and the compact-key blob carry q in their headers: a blob whose q holds gamma is refused on load, as creation
    refuses it; a derived level of a valid context (a prefix of a valid q) is created as usual"""
    from cryptonets_b200.engine import Engine
    cfg = CONTEXTS["n2048-mixed"]
    eng = _engine(cfg, seed=9)
    try:
        i, bad_q = _gamma_blob_q(eng.q)
        # the compact key blob: q_l at byte 36 + 8 l
        kblob = bytearray(eng.save_compact_keys(galois=[]))
        kblob[36 + 8 * i: 44 + 8 * i] = W.GAMMA.to_bytes(8, "little")
        with pytest.raises(CnheError) as e:
            Engine(None, compact_keys=bytes(kblob))
        assert e.value.code == ERR_INVALID and "gamma" in str(e.value)
        # the key archive: per environment, version byte, N, k, then q_l at byte 17 + 8 l
        zin = zipfile.ZipFile(io.BytesIO(eng.save_keys(False)))
        out = io.BytesIO()
        with zipfile.ZipFile(out, "w", zipfile.ZIP_STORED) as zout:
            for info in zin.infolist():
                data = bytearray(zin.read(info))
                if info.filename.startswith("environment"):
                    assert int.from_bytes(data[17 + 8 * i: 25 + 8 * i], "little") == eng.q[i]
                    data[17 + 8 * i: 25 + 8 * i] = W.GAMMA.to_bytes(8, "little")
                zout.writestr(info.filename, bytes(data))
        with pytest.raises(CnheError) as e:
            Engine(None, archive=out.getvalue())
        assert e.value.code == ERR_INVALID and "gamma" in str(e.value)
        with pytest.raises(CnheError) as e:
            Engine([cfg["t"]], cfg["N"], 10, 20, -1, coeff_moduli=bad_q)
        assert e.value.code == ERR_INVALID and "gamma" in str(e.value)
        # the unpatched blobs load, and every level derives
        Engine(None, archive=eng.save_keys(False)).close()
        for k2 in range(1, eng.k):
            lvl = eng.derive_level(k2)
            assert lvl.q == eng.q[:k2]
            lvl.close()
    finally:
        eng.close()
