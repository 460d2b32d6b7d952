"""GPU parity: every CUDA kernel / device pipeline of libcnhe against the CPU oracle on identical inputs, keys and
parameters -- bit-exact (integer arithmetic).  Calls go through the C ABI (cryptonets_b200.engine -> libcnhe.so)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096, count=-1, dbc_r=10, dbc_g=20),       # IFactory.cs:247-253
    "cryptonets8192": dict(t=549764251649, N=8192, count=-1, dbc_r=10, dbc_g=20),  # CryptoNets.cs:17
    "lola8192": dict(t=2277377, N=8192, count=3, dbc_r=40, dbc_g=40),          # LoLaCryptonets.cs:285
    "cifar16384": dict(t=957181001729, N=16384, count=8, dbc_r=60, dbc_g=60),  # LolaCifarCryptoNet.cs:35
}


def _make_engine(name, aux):
    """aux: 'fast' = 48-bit auxiliary base + FP64 butterflies (the default product configuration);
            'seal' = SEAL 3.2's 61-bit auxiliary base (integer butterflies on those moduli), comparable stage by stage;
            'int'  = fast base but integer butterflies everywhere (CNHE_NTT_INT)."""
    import os
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS[name]
    os.environ.pop("CNHE_AUX_BASE", None)
    os.environ.pop("CNHE_NTT_INT", None)
    if aux == "seal":
        os.environ["CNHE_AUX_BASE"] = "seal"
    if aux == "int":
        os.environ["CNHE_NTT_INT"] = "1"
    try:
        eng = Engine([cfg["t"]], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    finally:
        os.environ.pop("CNHE_AUX_BASE", None)
        os.environ.pop("CNHE_NTT_INT", None)
    return eng


def _make_pair(name, aux):
    """the engine of _make_engine(name, aux) and the oracle of the same parameters, both keyed with seed 1234"""
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[name]
    eng = _make_engine(name, aux)
    orc = Oracle(cfg["t"], cfg["N"], cfg["count"], cfg["dbc_r"], cfg["dbc_g"])
    assert eng.q == orc.q
    if aux == "seal":
        assert eng.bsk == orc.bsk
    eng.keygen(1234)
    orc.keygen(1234)
    return eng, orc


PAIRS = [(n, "fast") for n in CONFIGS] + [("default4096", "seal"), ("cryptonets8192", "seal"), ("cryptonets8192", "int")]


@pytest.fixture(scope="module", params=PAIRS, ids=lambda p: "%s-%s" % p)
def pair(request):
    name, aux = request.param
    eng, orc = _make_pair(name, aux)
    yield eng, orc, name
    eng.close()


@pytest.fixture(scope="module", params=["default4096", "cryptonets8192"])
def seal_pair(request):
    eng, orc = _make_pair(request.param, "seal")
    yield eng, orc, request.param
    eng.close()


def _bsk_oracle(eng, orc):
    """an oracle whose *coefficient* moduli are the engine's Bsk primes, to check NTTs under those primes"""
    from oracle.oracle_py import Oracle
    return Oracle(orc.t, eng.N, custom_q=eng.bsk)


def _mod_table(eng, orc):
    """engine modulus id -> (modulus, oracle, oracle table id)"""
    bo = _bsk_oracle(eng, orc)
    tab = [(orc.q[i], orc, i) for i in range(eng.k)]
    tab += [(eng.bsk[j], bo, j) for j in range(eng.kb)]
    tab += [(orc.t, orc, 2 * orc.k + 1)]
    return tab


def test_ntt_all_moduli(pair):
    eng, orc, _ = pair
    rng = np.random.default_rng(1)
    N = eng.N
    for which, (p, o, oid) in enumerate(_mod_table(eng, orc)):
        polys = rng.integers(0, p, (3, N), dtype=np.uint64)
        polys[0, :6] = [0, 1, p - 1, p - 2, p // 2, p // 2 + 1]
        polys[1, :] = p - 1  # extreme magnitudes through every butterfly
        d = eng.dev_from(polys)
        eng.raw_ntt(d, d, 3, which, 1, False)
        got = eng.dev_download(d, 3 * N).reshape(3, N)
        want = np.stack([o.ntt(oid, polys[i]) for i in range(3)])
        assert np.array_equal(got, want), which
        eng.raw_ntt(d, d, 3, which, 1, True)
        back = eng.dev_download(d, 3 * N).reshape(3, N)
        assert np.array_equal(back, polys), which
        eng.dev_free(d)


def test_ntt_mixed_batch(pair):
    eng, orc, _ = pair
    rng = np.random.default_rng(2)
    N = eng.N
    tab = _mod_table(eng, orc)
    kt = eng.k + eng.kb
    polys = np.stack([rng.integers(0, tab[b % kt][0], N, dtype=np.uint64) for b in range(2 * kt)])
    d = eng.dev_from(polys)
    out = eng.dev_alloc(polys.size)
    eng.raw_ntt(d, out, 2 * kt, 0, kt, False)
    got = eng.dev_download(out, polys.size).reshape(polys.shape)
    for b in range(2 * kt):
        p, o, oid = tab[b % kt]
        assert np.array_equal(got[b], o.ntt(oid, polys[b])), b
    eng.raw_ntt(out, out, 2 * kt, 0, kt, True)
    assert np.array_equal(eng.dev_download(out, polys.size).reshape(polys.shape), polys)
    eng.dev_free(d)
    eng.dev_free(out)


def test_keygen_bit_identical(pair):
    eng, orc, _ = pair
    assert np.array_equal(eng.export_key(0, 0), orc.secret_key())
    assert np.array_equal(eng.export_key(0, 1), orc.public_key())
    assert np.array_equal(eng.export_key(0, 2), orc.relin_keys().ravel())
    assert eng.galois_elts() == orc.galois_elts()
    for elt in eng.galois_elts()[:3] + eng.galois_elts()[-1:]:
        assert np.array_equal(eng.export_key(0, 3, elt), orc.galois_key(elt).ravel()), elt


def _fresh_cts(orc, n, seed, nonce0=100):
    rng = np.random.default_rng(seed)
    vals = rng.integers(0, orc.t, (n, orc.N), dtype=np.uint64)
    return vals, np.stack([orc.encrypt(orc.encode(vals[i]), nonce0 + i) for i in range(n)])


def test_encrypt_decrypt(pair):
    from cryptonets_b200.engine import DENSE
    eng, orc, _ = pair
    rng = np.random.default_rng(3)
    half = orc.t // 2
    vals = rng.integers(-min(half, 2**40), min(half, 2**40), eng.N + 17).astype(np.float64)
    v = eng.encrypt(vals, 1.0, DENSE)  # nonces 1, 2 on a fresh context
    assert v.blocks == 2
    lifted = np.where(vals < 0, vals + orc.t, vals).astype(np.uint64)
    want0 = orc.encrypt(orc.encode(lifted[: eng.N]), 1)
    want1 = orc.encrypt(orc.encode(lifted[eng.N:]), 2)
    assert np.array_equal(v.export_raw(0, 0), want0)
    assert np.array_equal(v.export_raw(0, 1), want1)
    assert np.array_equal(eng.decrypt(v), vals)
    assert eng.noise_budget(v, 0, 0) == orc.noise_budget(want0)


def test_behz_stages(seal_pair):
    eng, orc, _ = seal_pair
    N, k = eng.N, eng.k
    kt = 2 * k + 1
    _, cts = _fresh_cts(orc, 2, 5)
    d = eng.dev_from(cts)
    out = eng.dev_alloc(2 * 2 * kt * N)
    eng.raw_behz_lift(d, 2, out)
    got = eng.dev_download(out, 2 * 2 * kt * N).reshape(2, 2, kt, N)
    for c in range(2):
        for part in range(2):
            poly = cts[c].reshape(2, k, N)[part]
            assert np.array_equal(got[c, part, :k], poly)
            assert np.array_equal(got[c, part, k:].ravel(), orc.behz_lift(poly))
    rng = np.random.default_rng(6)
    dd = np.stack([np.stack([rng.integers(0, orc.modulus_of(l), N, dtype=np.uint64) for l in range(kt)]) for _ in range(3)])
    d2 = eng.dev_from(dd)
    out3 = eng.dev_alloc(3 * k * N)
    eng.raw_behz_floor(0, d2, 1, out3)
    got = eng.dev_download(out3, 3 * k * N).reshape(3, k * N)
    for i in range(3):
        scaled = np.stack([(dd[i, l].astype(object) * orc.t % orc.modulus_of(l)) for l in range(kt)]).astype(np.uint64)
        assert np.array_equal(got[i], orc.behz_floor(scaled)), i
    for p in (d, out, d2, out3):
        eng.dev_free(p)


@pytest.mark.parametrize("centered", [0, 1])
def test_multiply_relinearize(pair, centered):
    eng, orc, name = pair
    eng.set_option("behz_centered_mtilde", centered)
    orc.set_centered_mtilde(centered)
    try:
        N, k = eng.N, eng.k
        n = 3
        vals, cts = _fresh_cts(orc, 2 * n, 7)
        a, b = eng.dev_from(cts[:n]), eng.dev_from(cts[n:])
        out3, out2, outmr, outsq = eng.dev_alloc(n * 3 * k * N), eng.dev_alloc(n * 2 * k * N), eng.dev_alloc(n * 2 * k * N), eng.dev_alloc(n * 2 * k * N)
        eng.raw_multiply(0, a, b, n, out3)
        got3 = eng.dev_download(out3, n * 3 * k * N).reshape(n, -1)
        want3 = np.stack([orc.multiply(cts[i], cts[n + i]) for i in range(n)])
        assert np.array_equal(got3, want3)
        eng.raw_relinearize(0, out3, n, out2)
        got2 = eng.dev_download(out2, n * 2 * k * N).reshape(n, -1)
        want2 = np.stack([orc.relinearize(want3[i]) for i in range(n)])
        assert np.array_equal(got2, want2)
        eng.raw_multiply_relin(0, a, b, n, outmr)
        assert np.array_equal(eng.dev_download(outmr, n * 2 * k * N).reshape(n, -1), want2)
        eng.raw_multiply_relin(0, a, a, n, outsq)  # squaring path (SquareActivation)
        wantsq = np.stack([orc.relinearize(orc.multiply(cts[i], cts[i])) for i in range(n)])
        assert np.array_equal(eng.dev_download(outsq, n * 2 * k * N).reshape(n, -1), wantsq)
        if name != "cifar16384":  # t^2 products need the CRT wrapper there; slots still multiply mod t
            dec = orc.decode(orc.decrypt(want2[0]))
            assert np.array_equal(dec, (vals[0].astype(object) * vals[n].astype(object) % orc.t).astype(np.uint64))
        for p in (a, b, out3, out2, outmr, outsq):
            eng.dev_free(p)
    finally:
        eng.set_option("behz_centered_mtilde", 0)
        orc.set_centered_mtilde(0)


def test_galois_and_rotations(pair):
    eng, orc, _ = pair
    N, k = eng.N, eng.k
    n = 2
    _, cts = _fresh_cts(orc, n, 9)
    a = eng.dev_from(cts)
    out = eng.dev_alloc(n * 2 * k * N)
    for elt in [2 * N - 1, 3, eng.galois_elts()[2]]:
        eng.raw_apply_galois(0, a, n, elt, out)
        got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
        for i in range(n):
            assert np.array_equal(got[i], orc.apply_galois(cts[i], elt)), elt
    for steps in [1, -1, 4, -64, 169, -507, 0]:
        eng.raw_rotate_rows(0, a, n, steps, out)
        got = eng.dev_download(out, n * 2 * k * N).reshape(n, -1)
        for i in range(n):
            assert np.array_equal(got[i], orc.rotate_rows(cts[i], steps)), steps
    eng.dev_free(a)
    eng.dev_free(out)


def test_mac_layer_and_square_layer(pair):
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, orc, name = pair
    N = eng.N
    rng = np.random.default_rng(11)
    n_in, M, K = 12, 10, 5
    vals, cts = _fresh_cts(orc, n_in, 12, nonce0=500)
    ins = [eng.import_raw(cts[i], 1, N, 4.0) for i in range(n_in)]
    gather = rng.integers(-1, n_in, (M, K)).astype(np.int32)
    gather[:, 0] = np.arange(M) % n_in  # at least one real tap per output
    gather[5:] = gather[4]              # outputs 4.. share a gather row (tile reuse path)
    w = rng.integers(-300, 300, (M, K)).astype(np.float64)
    w[:, 0] = np.where(w[:, 0] == 0, 7, w[:, 0])
    w[2, 1] = 0
    bias = rng.integers(-1000, 1000, M).astype(np.float64)
    wv = [eng.plain(w[m], 8.0, SPARSE) for m in range(M)]
    bv = [eng.plain(np.full(N, bias[m]), 32.0, DENSE) for m in range(M)]
    outs = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
    t = orc.t
    wres = np.where(w * 8 < 0, w * 8 + t, w * 8).astype(np.uint64)
    bres = np.where(bias * 32 < 0, bias * 32 + t, bias * 32).astype(np.uint64)
    want = orc.mac_layer(cts, gather, wres, bres, M, K, threads=4).reshape(M, -1)
    for m in range(M):
        assert np.array_equal(outs[m].export_raw(0, 0), want[m]), m
        assert outs[m].scale == 32.0
    # no bias, identity gather == IMatrix.Mul(ColumnMajor, sparse)  (AtomicSealBfvVector.cs:434-521)
    one = eng.mat_mul_colmajor_sparse(ins[:K], wv[0])
    want1 = orc.mac_layer(cts[:K], None, wres[:1], None, 1, K)
    assert np.array_equal(one.export_raw(0, 0), want1)
    sq = eng.layer_square(outs[:4])
    wantsq = orc.square_layer(want[:4], threads=4).reshape(4, -1)
    for i in range(4):
        assert np.array_equal(sq[i].export_raw(0, 0), wantsq[i]), i
        assert sq[i].scale == 32.0 * 32.0


@pytest.mark.parametrize("shape", ["gather-wide-21x43", "slab-wide-21x43", "slab-byte-21x43", "slab-byte-100x70", "slab-byte-128x33"])
def test_dense_layer_on_tensor_cores(pair, shape, capfd):
    """Dense layer (all outputs read the same K inputs): the exact 8-bit-limb integer GEMM must give the same ciphertext words as the
    oracle's 128-bit multiply-accumulate -- odd M and K (padding inside the tiles), zero weights, extreme weights and maximal residues,
    bias on coefficient 0 of c0.  "gather": inputs scattered in memory, permuted, one padded tap -> mma.sync (mac_imma.cu).  "slab": the
    inputs are consecutive ciphertexts of one allocation read in order, as a dense layer is fed by the layer before it -> wgmma with
    register accumulators and TMA loads (mac_umma.cu), up to 128 outputs, several 32-tap chunks, and ("wide", |w| <= 254) the W2 columns as
    extra taps.  Every case is repeated with the wgmma path off and with both tensor-core paths off (FP64 scalar MAC)."""
    import os
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, orc, name = pair
    N = eng.N
    rng = np.random.default_rng(23)
    feed, kind, dims = shape.split("-")
    wide = kind == "wide"
    M, K = [int(x) for x in dims.split("x")]
    n_in = K + 2
    vals, cts = _fresh_cts(orc, n_in, 12, nonce0=900)
    q = np.array(orc.q, dtype=np.uint64)
    cts = np.array(cts, dtype=np.uint64).reshape(n_in, 2, len(q), N)
    cts[0] = (q - 1)[None, :, None]                       # every word of input 0 at its maximum
    cts[1, :, :, ::2] = (q - 1)[None, :, None]
    cts = cts.reshape(n_in, -1)
    if feed == "slab":
        ins = eng.import_raw_many(cts, n_in, 1, N, 4.0)   # one allocation, evenly spaced
        row = np.arange(K, dtype=np.int32)                # taps 0..K-1 in order (input 0: maximal words)
    else:
        ins = [eng.import_raw(cts[i], 1, N, 4.0) for i in range(n_in)]
        row = rng.permutation(n_in)[:K].astype(np.int32)
        row[7] = -1                                       # one padded tap
    gather = np.tile(row, (M, 1)).astype(np.int32)
    w = rng.integers(-127, 128, (M, K)).astype(np.float64)
    w[:, 0] = 127
    w[:, 1] = -127
    if wide:
        w[5, 3], w[6, 40], w[20, 42] = 254, -254, 165  # beyond 8 bits: carried by the residual fragment
    w[3, :] = 0
    w[3, 2] = 1
    bias = rng.integers(-1000, 1000, M).astype(np.float64)
    wv = [eng.plain(w[m], 1.0, SPARSE) for m in range(M)]
    bv = [eng.plain(np.full(N, bias[m]), 4.0, DENSE) for m in range(M)]
    t = orc.t
    wres = np.where(w < 0, w + t, w).astype(np.uint64)
    bres = np.where(bias * 4 < 0, bias * 4 + t, bias * 4).astype(np.uint64)
    want = orc.mac_layer(cts, gather, wres, bres, M, K, threads=max(4, os.cpu_count() or 1)).reshape(M, -1)
    os.environ["CNHE_UMMA_PROF"] = "1"  # the wgmma launcher then reports itself on stderr
    capfd.readouterr()
    try:
        outs = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
        eng.sync()
    finally:
        del os.environ["CNHE_UMMA_PROF"]
    served = "[umma " in capfd.readouterr().err
    assert served == (feed == "slab"), "wrong kernel served the layer"
    for m in range(M):
        assert np.array_equal(outs[m].export_raw(0, 0), want[m]), m
    for off in ("CNHE_MAC_NO_UMMA", "CNHE_MAC_NO_IMMA"):
        os.environ[off] = "1"
        try:
            outs2 = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
        finally:
            del os.environ[off]
        for m in range(M):
            assert np.array_equal(outs2[m].export_raw(0, 0), want[m]), (off, m)


@pytest.mark.parametrize("fwd,inv", [("1", "1"), ("0", "0"), ("1", "0"), ("0", "1")])
def test_persistent_and_per_polynomial_transforms_agree(pair, fwd, inv):
    """At N = 4096 / 8192 the inverse transform runs on persistent CTAs fed by TMA (cp.async.bulk.tensor) with the unit-stride
    twiddles resident in shared memory, the forward one on one CTA per polynomial.  Both must give the oracle's words on a batch that
    gives every CTA several polynomials (ragged tail), the inverse must bring the batch back, and so must the digit-cutting forward
    inside relinearise and the lazy-double variants inside multiply.  fwd / inv = "1": that direction runs in place (src == dst; the
    persistent kernel then overwrites each polynomial of the array it stages the next ones from), "0": out of place.  The other
    rings run the same checks on their own kernels."""
    eng, orc, name = pair
    rng = np.random.default_rng(11)
    N, k, kt = eng.N, eng.k, eng.k + eng.kb
    tab = _mod_table(eng, orc)
    n = 64 * kt + 3  # more polynomials than CTAs x 2 groups for some moduli, ragged tail
    polys = np.stack([rng.integers(0, tab[b % kt][0], N, dtype=np.uint64) for b in range(n)])
    d, out = eng.dev_from(polys), eng.dev_alloc(polys.size)
    f_dst = d if fwd == "1" else out
    eng.raw_ntt(d, f_dst, n, 0, kt, False)
    got = eng.dev_download(f_dst, polys.size).reshape(polys.shape)
    for b in list(range(0, n, 37)) + [n - 1]:
        p, o, oid = tab[b % kt]
        assert np.array_equal(got[b], o.ntt(oid, polys[b])), b
    i_dst = f_dst if inv == "1" else (out if f_dst == d else d)
    eng.raw_ntt(f_dst, i_dst, n, 0, kt, True)
    assert np.array_equal(eng.dev_download(i_dst, polys.size).reshape(polys.shape), polys)
    eng.dev_free(d)
    eng.dev_free(out)
    m = 5
    _, cts = _fresh_cts(orc, m, 21)
    a, o2 = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N)
    eng.raw_multiply_relin(0, a, a, m, o2)
    want = np.stack([orc.relinearize(orc.multiply(cts[i], cts[i])) for i in range(m)])
    assert np.array_equal(eng.dev_download(o2, m * 2 * k * N).reshape(m, -1), want)
    eng.dev_free(a)
    eng.dev_free(o2)


@pytest.mark.parametrize("split", ["1", "0"])
def test_cta_pair_and_whole_polynomial_transforms_agree(pair, split):
    """N = 16384 runs on CTA pairs on the FP64 path (two 8192-point halves, the cross-half stage on the way in / through distributed
    shared memory on the way out) and on one CTA per polynomial on the integer path (moduli of 2^50 and above, CNHE_NTT_INT).  split =
    "1" checks the ring's own engine, "0" an engine of the same parameters on integer butterflies.  Both must give the oracle's words:
    plain transforms out of place and IN PLACE (the pair reads both halves before either writes), the digit-cutting forward and the
    lazy variants inside multiply + relinearise.  The other rings run the same checks on their own kernels."""
    eng, orc, name = pair
    if split == "0":
        eng = _make_engine(name, "int")
        eng.keygen(1234)
    try:
        _check_transforms_and_product(eng, orc)
    finally:
        if split == "0":
            eng.close()


def _check_transforms_and_product(eng, orc):
    rng = np.random.default_rng(12)
    N, k, kt = eng.N, eng.k, eng.k + eng.kb
    tab = _mod_table(eng, orc)
    n = 40 * kt + 5
    polys = np.stack([rng.integers(0, tab[b % kt][0], N, dtype=np.uint64) for b in range(n)])
    polys[0, :] = tab[0][0] - 1  # largest canonical input everywhere: the worst case of the magnitude schedule
    d, out = eng.dev_from(polys), eng.dev_alloc(polys.size)
    eng.raw_ntt(d, out, n, 0, kt, False)
    got = eng.dev_download(out, polys.size).reshape(polys.shape)
    for b in [0] + list(range(1, n, 41)) + [n - 1]:
        p, o, oid = tab[b % kt]
        assert np.array_equal(got[b], o.ntt(oid, polys[b])), b
    eng.raw_ntt(d, d, n, 0, kt, False)  # in place
    assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), got)
    eng.raw_ntt(d, d, n, 0, kt, True)
    assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), polys)
    eng.raw_ntt(out, d, n, 0, kt, True)  # out of place
    assert np.array_equal(eng.dev_download(d, polys.size).reshape(polys.shape), polys)
    eng.dev_free(d)
    eng.dev_free(out)
    m = 3
    _, cts = _fresh_cts(orc, m, 22)
    a, o2 = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N)
    eng.raw_multiply_relin(0, a, a, m, o2)
    want = np.stack([orc.relinearize(orc.multiply(cts[i], cts[i])) for i in range(m)])
    assert np.array_equal(eng.dev_download(o2, m * 2 * k * N).reshape(m, -1), want)
    eng.dev_free(a)
    eng.dev_free(o2)


@pytest.mark.parametrize("wide", [False, True])
def test_convolution_on_tensor_cores(pair, wide, capfd):
    """A strided, padded convolution over a slab of per-pixel ciphertexts (PoolLayer.cs:68-80, 196-227) on the wgmma path: the host
    plan bundles the outputs of one output row (their taps lie in a window of consecutive inputs), interior rows share one weight matrix,
    padded taps carry no weight, and weights beyond a signed byte ("wide") ride on extra taps gathered into a scratch slab.  Same words as
    the oracle's 128-bit multiply-accumulate, and as the FP64 scalar-MAC kernel."""
    import os
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, orc, name = pair
    N = eng.N
    rng = np.random.default_rng(31)
    side, ker, stride, pad, maps = (17 if name == "default4096" else 9), 3, 2, 1, 4  # 256 outputs = two bundles on the smallest ring
    osz = (side + pad - ker) // stride + 1  # upper padding only, as the reference's Upperpadding
    n_in, K = side * side, ker * ker
    M = maps * osz * osz
    vals, cts = _fresh_cts(orc, n_in, 12, nonce0=1500)
    cts = np.array(cts, dtype=np.uint64)
    cts[0, :] = np.tile(np.array(orc.q, dtype=np.uint64) - 1, 2).repeat(N)  # maximal words in the first pixel
    ins = eng.import_raw_many(cts, n_in, 1, N, 4.0)
    gather = np.full((M, K), -1, dtype=np.int32)
    w = np.zeros((M, K))
    kern = rng.integers(-127, 128, (maps, K)).astype(np.float64)
    kern[:, 0] = [127, -127, 1, 0]
    if wide:
        kern[1, 4], kern[2, 8] = 201, -254
    m = 0
    for y in range(osz):          # position-major, maps innermost: outputs of one window are adjacent (PoolLayer's order)
        for x in range(osz):
            for f in range(maps):
                for dy in range(ker):
                    for dx in range(ker):
                        iy, ix = y * stride + dy - pad, x * stride + dx - pad
                        if 0 <= iy < side and 0 <= ix < side:
                            gather[m, dy * ker + dx] = iy * side + ix
                w[m] = kern[f]
                m += 1
    bias = rng.integers(-1000, 1000, M).astype(np.float64)
    wv = [eng.plain(w[i], 1.0, SPARSE) for i in range(M)]
    bv = [eng.plain(np.full(N, bias[i]), 4.0, DENSE) for i in range(M)]
    t = orc.t
    wres = np.where(w < 0, w + t, w).astype(np.uint64)
    bres = np.where(bias * 4 < 0, bias * 4 + t, bias * 4).astype(np.uint64)
    want = orc.mac_layer(cts, gather, wres, bres, M, K, threads=4).reshape(M, -1)
    os.environ["CNHE_UMMA_PROF"] = "1"
    capfd.readouterr()
    try:
        outs = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
        eng.sync()
    finally:
        del os.environ["CNHE_UMMA_PROF"]
    err = capfd.readouterr().err
    assert "[umma bundles=" in err, "the wgmma kernel did not serve the convolution"
    for i in range(M):
        assert np.array_equal(outs[i].export_raw(0, 0), want[i]), i
    os.environ["CNHE_MAC_NO_UMMA"] = "1"
    try:
        outs2 = eng.layer_conv_dense(ins, gather, wv, bv, M, K)
    finally:
        del os.environ["CNHE_MAC_NO_UMMA"]
    for i in range(M):
        assert np.array_equal(outs2[i].export_raw(0, 0), want[i]), i


def test_tensor_core_layers_randomised():
    """Random dense shapes and random strided / padded convolutions (weights up to +-254, random biases, maximal words) through the
    wgmma kernel and through the FP64 scalar-MAC kernel: two independent GPU implementations, bit-identical outputs
    (tools/umma_stress.py; the oracle-checked cases are test_dense_layer_on_tensor_cores / test_convolution_on_tensor_cores)."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("umma_stress", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "umma_stress.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lines = []
    assert mod.run(16, 3, log=lines.append) == 0, "\n".join(lines)
    assert len(lines) >= 12


def test_key_switch_mac_full_waves(pair, monkeypatch):
    """Waves of 64 or more ciphertexts take the digit path's key-switch inner product (lazy FP64 path) through the copy-engine-staged
    kernel (cp.async.bulk ring, four ciphertexts per CTA share the key words); CNHE_KS_FUSED=0 keeps every ring on the digit path.  70
    ciphertexts (a ragged last group of two) drawn from six: multiply + relinearise must match the oracle on all of them, and where
    the fused key switch is built its outputs must equal the digit path's."""
    eng, orc, name = pair
    N, k = eng.N, eng.k
    m = 70
    _, few = _fresh_cts(orc, 6, 21, nonce0=3000)
    src = np.arange(m) % 6
    src[1::2] = np.roll(src[1::2], 1)  # not all groups alike
    cts = np.stack([few[i] for i in src])
    want = [orc.relinearize(orc.multiply(few[j], few[j])) for j in range(6)]
    a, o1, o2 = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N), eng.dev_alloc(m * 2 * k * N)
    monkeypatch.setenv("CNHE_KS_FUSED", "0")
    eng.raw_multiply_relin(0, a, a, m, o1)
    got = eng.dev_download(o1, m * 2 * k * N).reshape(m, -1)
    for i in range(m):
        assert np.array_equal(got[i], want[src[i]]), i
    monkeypatch.setenv("CNHE_KS_FUSED", "1")  # no effect where the fused key switch is not built
    eng.raw_multiply_relin(0, a, a, m, o2)
    assert np.array_equal(eng.dev_download(o2, m * 2 * k * N).reshape(m, -1), got)
    for d in (a, o1, o2):
        eng.dev_free(d)
