"""Compact evaluation keys (cnhe_keys_save_compact / cnhe_context_load_compact) on the GPU: the client's blob byte for byte against the
Python restatement built from the CPU oracle, the server's expanded keys word for word, key sets left out refusing cleanly, key switches
with the server's keys (fused kernel, 48-bit copy, noise budget), CryptoNets and LoLa-small end to end against the Raw backend, secure
mode and malformed blobs."""
import ctypes as C
import struct

import numpy as np
import pytest

import compact_keys_ref as kr

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=[40961], N=4096, count=-1, dbc_r=10, dbc_g=20),
    "lola_small8192": dict(t=[2277377, 2424833], N=8192, count=3, dbc_r=40, dbc_g=40),
}
SEED = 5151


@pytest.fixture(scope="module", params=list(CONFIGS))
def setup(request):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[request.param]
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    eng.keygen(SEED)
    orcs = []
    for c, t in enumerate(cfg["t"]):
        o = Oracle(t, cfg["N"], cfg["count"], cfg["dbc_r"], cfg["dbc_g"])
        o.keygen(SEED + c)
        orcs.append(o)
    yield eng, cfg, orcs
    eng.close()


def _two(eng):
    e = sorted(eng.galois_elts())
    return [e[1], e[-2]]


def _own_keys(eng, elts):
    return [[eng.export_key(c, w) for w in (0, 1, 2)] + [eng.export_key(c, 3, g) for g in elts] for c in range(eng.P)]


def _check_server(server, want, cfg, listed, sets):
    from cryptonets_b200._lib import CnheError
    for c, w in enumerate(want):
        if sets & kr.SET_PUBLIC:
            assert np.array_equal(server.export_key(c, 1).reshape(w["pk"].shape), w["pk"])
        if sets & kr.SET_RELIN:
            assert np.array_equal(server.export_key(c, 2).reshape(w["rlk"].shape), w["rlk"])
        for g in listed:
            assert np.array_equal(server.export_key(c, 3, g).reshape(w["glk"][g].shape), w["glk"][g]), (c, g)
        absent = [(0, 0)] + [(3, g) for g in server.galois_elts() if g not in listed]
        absent += [] if sets & kr.SET_PUBLIC else [(1, 0)]
        absent += [] if sets & kr.SET_RELIN else [(2, 0)]
        for what, arg in absent:
            with pytest.raises(CnheError) as e:
                server.export_key(c, what, arg)
            assert e.value.code == -3


@pytest.mark.parametrize("selection", ["every", "pk_relin", "two"])
def test_blob_and_server_keys_bit_exact(setup, selection):
    from cryptonets_b200.engine import Engine
    eng, cfg, orcs = setup
    eng.keygen(SEED)  # nonces restart at 1
    galois = {"every": None, "pk_relin": [], "two": _two(eng)}[selection]
    listed = sorted(set(eng.galois_elts())) if galois is None else sorted(galois)
    before = _own_keys(eng, listed[:2])
    blob = eng.save_compact_keys(galois=galois)
    # 3. the client's own keys are untouched
    after = _own_keys(eng, listed[:2])
    assert all(np.array_equal(a, b) for x, y in zip(before, after) for a, b in zip(x, y))
    # 1. the blob byte for byte
    sets = kr.SET_PUBLIC | kr.SET_RELIN
    want_blob, want = kr.expected_keys(orcs, SEED, sets, listed)
    h = kr.parse(blob)
    assert (h["N"], h["k"], h["P"], h["dbc_r"], h["dbc_g"], h["sets"], h["elts"]) == (cfg["N"], eng.k, eng.P, cfg["dbc_r"], cfg["dbc_g"], 3,
                                                                                      listed)
    assert h["q"] == eng.q and h["t"] == cfg["t"]
    assert len(blob) == len(want_blob) == kr.blob_size(cfg["N"], eng.q, eng.P, cfg["dbc_r"], cfg["dbc_g"], sets, len(listed))
    assert blob == want_blob
    # 2. the server's keys word for word; no secret key, no unlisted element
    server = Engine(None, compact_keys=blob)
    try:
        assert (server.N, server.k, server.P, server.q, server.primes) == (eng.N, eng.k, eng.P, eng.q, eng.primes)
        _check_server(server, want, cfg, listed, sets)
    finally:
        server.close()


def test_cifar_shape_relin_and_one_element():
    """N = 16384, k = 8 (LoLa-CIFAR): 48- and 49-bit moduli, so 49-bit packing, and no 48-bit copy of the relinearisation keys"""
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    t, N = [957181001729, 957181034497], 16384
    eng = Engine(t, N, 60, 60, 8)
    try:
        eng.keygen(SEED)
        orcs = []
        for c, tc in enumerate(t):
            o = Oracle(tc, N, 8, 60, 60)
            o.keygen(SEED + c)
            orcs.append(o)
        elt = sorted(eng.galois_elts())[3]
        blob = eng.save_compact_keys(public=False, relin=True, galois=[elt])
        want_blob, want = kr.expected_keys(orcs, SEED, kr.SET_RELIN, [elt])
        assert blob == want_blob
        assert {kr.parse(blob)["q"][l].bit_length() for l in range(8)} == {48, 49}
        server = Engine(None, compact_keys=blob)
        try:
            _check_server(server, want, None, [elt], kr.SET_RELIN)
            # the server squares; the client decrypts
            vals = np.random.default_rng(1).integers(-30, 31, (1, N)).astype(np.float64)
            x = eng.encrypt_many(vals, 1.0)
            raw = eng.export_raw_many(x)
            sv = server.import_raw_many(raw, 1, 1, N)
            out = server.export_raw_many([server.pointwise_multiply(sv[0], sv[0])])
        finally:
            server.close()
        back = eng.import_raw_many(out, 1, 1, N)
        assert np.array_equal(eng.decrypt(back[0]), vals[0] * vals[0])
    finally:
        eng.close()


def _roundtrip(eng, server, vecs):
    """vectors computed on the server, exported raw, imported at the client"""
    out = []
    for v in vecs:
        raw = server.export_raw_many([v])
        out.append(eng.import_raw_many(raw, 1, v.blocks, v.dim, v.scale, v.format)[0])
    return out


def test_missing_key_sets_refuse_and_naf_hops(setup):
    from cryptonets_b200._lib import CnheError
    from cryptonets_b200.engine import Engine
    eng, cfg, orcs = setup
    N = cfg["N"]
    vals = np.random.default_rng(4).integers(-40, 41, (2, N)).astype(np.float64)
    x = eng.encrypt_many(vals, 1.0)
    raw = eng.export_raw_many(x)
    hop4, hop_m1 = orcs[0].galois_elt_from_step(4), orcs[0].galois_elt_from_step(-1)
    assert hop4 in eng.galois_elts() and hop_m1 in eng.galois_elts()

    def refuses(fn):
        with pytest.raises(CnheError) as e:
            fn()
        assert e.value.code == -3, str(e.value)

    # no relinearisation keys: a square layer refuses; no public key: encryption refuses
    s1 = Engine(None, compact_keys=eng.save_compact_keys(public=False, relin=False, galois=[hop4, hop_m1]))
    try:
        sv = s1.import_raw_many(raw, 2, 1, N)
        refuses(lambda: s1.layer_square(sv))
        refuses(lambda: s1.encrypt(vals[0]))
        # only the two NAF hops of 3 (4, then -1): rotation by 3 goes through them
        rot = s1.rotate(sv[0], 3)
        got = eng.decrypt(_roundtrip(eng, s1, [rot])[0])
    finally:
        s1.close()
    assert np.array_equal(got, eng.decrypt(eng.rotate(x[0], 3)))
    assert not np.array_equal(got, vals[0])
    # no Galois key at all: a rotation refuses
    s2 = Engine(None, compact_keys=eng.save_compact_keys(galois=[]))
    try:
        sv = s2.import_raw_many(raw, 2, 1, N)
        refuses(lambda: s2.rotate(sv[0], 3))
        refuses(lambda: s2.rotate(sv[0], 1))
        assert np.array_equal(eng.decrypt(_roundtrip(eng, s2, [s2.pointwise_multiply(sv[0], sv[1])])[0]), vals[0] * vals[1])
    finally:
        s2.close()


def _relin(eng, monkeypatch, cts3, fused, key_bytes=None):
    m, k, N = cts3.shape[0], eng.k, eng.N
    monkeypatch.setenv("CNHE_KS_FUSED", fused)
    a, out = eng.dev_from(cts3), eng.dev_alloc(m * 2 * k * N)
    eng.sync()
    eng.prof_enable(True)
    eng.raw_relinearize(0, a, m, out)
    prof = eng.prof_collect()
    eng.prof_enable(False)
    assert (prof["ntt_forward"]["launches"] == 0) == (fused == "1")
    if fused == "1":
        want = 8.0 * N * (m * k + m * 2 * k) + key_bytes * N * eng.relin_digits * 2 * k
        assert prof["keyswitch_mac"]["bytes"] == pytest.approx(want, rel=1e-9)
    got = eng.dev_download(out, m * 2 * k * N).reshape(m, -1).copy()
    eng.dev_free(a)
    eng.dev_free(out)
    return got


def test_server_key_switch(setup, monkeypatch):
    from cryptonets_b200.engine import Engine
    eng, cfg, _ = setup
    N, k = cfg["N"], eng.k
    server = Engine(None, compact_keys=eng.save_compact_keys(galois=[]))
    try:
        # relinearisation of 64+ ciphertexts: fused kernel on the 48-bit copy, equal to the digit path
        q = np.array(eng.q, dtype=np.uint64)
        cts3 = (np.random.default_rng(2).integers(0, 1 << 62, (65, 3, k, N), dtype=np.uint64) % q[None, None, :, None]).astype(np.uint64)
        assert np.array_equal(_relin(server, monkeypatch, cts3, "1", 6), _relin(server, monkeypatch, cts3, "0"))
        monkeypatch.delenv("CNHE_KS_FUSED")
        # 64 products on the server decrypt at the client; the noise budget is within 1 bit of the client's own keys
        vals = np.random.default_rng(3).integers(-60, 61, (128, N)).astype(np.float64)
        x = eng.encrypt_many(vals, 1.0)
        sv = server.import_raw_many(eng.export_raw_many(x), 128, 1, N)
        prods = server.layer_square(sv[:64])
        pm = server.pointwise_multiply(sv[64], sv[65])
        back = _roundtrip(eng, server, list(prods) + [pm])
    finally:
        server.close()
    assert np.array_equal(eng.decrypt_many(back[:64]), vals[:64] ** 2)
    assert np.array_equal(eng.decrypt(back[64]), vals[64] * vals[65])
    own = eng.pointwise_multiply(x[64], x[65])
    for c in range(eng.P):
        b_server, b_own = eng.noise_budget(back[64], c), eng.noise_budget(own, c)
        print("N=%d channel %d: budget after multiply + relinearise, server keys %d bits, own keys %d bits" % (N, c, b_server, b_own))
        assert abs(b_server - b_own) <= 1


def test_malformed_blobs_size_query_and_server_without_secret_key(setup):
    from cryptonets_b200._lib import CnheError, U64P
    from cryptonets_b200.engine import Engine
    eng, cfg, _ = setup
    two = _two(eng)
    need = C.c_size_t()
    arr = np.array(two, dtype=np.uint64)
    assert eng.L.cnhe_keys_save_compact(eng.h, 3, arr.ctypes.data_as(U64P), 2, None, 0, C.byref(need)) == 0
    blob = eng.save_compact_keys(galois=two)
    assert need.value == len(blob)
    # selection errors
    for sets, elts in ((4, two), (3, [two[0], two[0]]), (3, [5])):
        a = np.array(elts, dtype=np.uint64)
        assert eng.L.cnhe_keys_save_compact(eng.h, sets, a.ctypes.data_as(U64P), len(elts), None, 0, C.byref(need)) == -1
    k, P = eng.k, eng.P
    elts_off = 36 + 8 * k + 8 * P

    def bad(b):
        h = C.c_void_p()
        buf = (C.c_ubyte * max(len(b), 1)).from_buffer_copy(bytes(b) or b"\0")
        assert eng.L.cnhe_context_load_compact(buf, len(b), 0, C.byref(h)) == -1
        assert not h.value

    put = lambda off, fmt, v: blob[:off] + struct.pack(fmt, v) + blob[off + struct.calcsize(fmt):]
    bad(blob[:20])                                   # truncated header
    bad(blob[:elts_off])                             # truncated header
    bad(b"CNHC" + blob[4:])                          # magic
    bad(put(4, "<I", 2))                             # version
    bad(blob[:-1])                                   # length
    bad(blob + bytes(8))                             # length
    bad(put(28, "<I", 7))                            # unknown sets bits
    bad(put(elts_off, "<Q", 5))                      # not a standard element
    bad(put(elts_off, "<Q", two[1]))                 # duplicate element
    bad(put(elts_off + 8, "<Q", two[0]))             # duplicate element
    bad(put(elts_off, "<Q", two[1])[:elts_off + 8] + struct.pack("<Q", two[0]) + blob[elts_off + 16:])  # unsorted
    bad(put(8, "<I", cfg["N"] * 2))                  # N: length and elements no longer match
    bad(put(12, "<I", 10))                           # k above the library's limit
    # a server has no secret key: it cannot export a compact key set
    server = Engine(None, compact_keys=blob)
    try:
        with pytest.raises(CnheError) as e:
            server.save_compact_keys()
        assert e.value.code == -3
    finally:
        server.close()


def test_secure_mode_exports_differ():
    from cryptonets_b200.engine import Engine
    t, N = [40961], 4096
    eng = Engine(t, N, 10, 20)
    try:
        eng.keygen(None)
        b1, b2 = eng.save_compact_keys(galois=[]), eng.save_compact_keys(galois=[])
        h1, h2 = kr.parse(b1), kr.parse(b2)
        assert h1["keys"] != h2["keys"] and h1["keys"][0] != bytes(32)
        assert not np.array_equal(h1["payload"], h2["payload"])
        vals = np.random.default_rng(8).integers(-50, 51, (2, N)).astype(np.float64)
        x = eng.encrypt_many(vals, 1.0)
        raw = eng.export_raw_many(x)
        for b in (b1, b2):
            server = Engine(None, compact_keys=b)
            try:
                sv = server.import_raw_many(raw, 2, 1, N)
                got = _roundtrip(eng, server, [server.pointwise_multiply(sv[0], sv[1])])[0]
                enc = server.encrypt(vals[0])  # the server's public key encrypts for the client
                got_enc = _roundtrip(eng, server, [enc])[0]
            finally:
                server.close()
            assert np.array_equal(eng.decrypt(got), vals[0] * vals[1])
            assert np.array_equal(eng.decrypt(got_enc), vals[0])
    finally:
        eng.close()


def _client_scores(client_f, server_f, out):
    from cryptonets_b200.he import B200BfvMatrix, B200BfvVector
    vecs = _roundtrip(client_f.engine, server_f.engine, [v.vec for v in out.vectors])
    return np.asarray(B200BfvMatrix(client_f, [B200BfvVector(client_f, v) for v in vecs], out.Format, CopyVectors=False).Decrypt())


def test_cryptonets_server_from_pk_relin_blob_end_to_end():
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    from test_gpu_compact_upload import _build_network, _forward
    client = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=91)
    server = None
    try:
        keys = client.SaveCompactKeys(galois=[])
        assert round(len(keys) / 1e6, 1) == 11.6
        server = B200BfvFactory(keys)
        layers = _build_network(server)
        imgs = synthetic_mnist(8192, seed=3)
        x = np.rint(imgs / 256.0 * 16.0)
        blob = client.GetEncryptedMatrixCompact(x, EMatrixFormat.ColumnMajor, 1)
        m = server.LoadCompactMatrix(blob, EMatrixFormat.ColumnMajor)
        m.RegisterScale(16.0)
        scores = _client_scores(client, server, _forward(layers, m))
        scores = scores if scores.shape[-1] == 10 else scores.T
        # the client evaluating the same blob with its own keys gets the same scores exactly
        mine = client.LoadCompactMatrix(blob, EMatrixFormat.ColumnMajor)
        mine.RegisterScale(16.0)
        own = np.asarray(_forward(_build_network(client), mine).Decrypt())
        own = own if own.shape[-1] == 10 else own.T
        assert np.array_equal(scores, own)
        # the Raw backend computes in doubles (test_gpu_network: good to ~2^-45 of the largest intermediate) and predicts the same
        raw_net, _ = cryptonets_mnist(RawFactory(8192), imgs, timing=False)
        raw_net.PrepareNetwork()
        want = np.asarray(raw_net.GetNext().Decrypt())
        assert scores.shape == want.shape == (8192, 10)
        assert np.allclose(scores, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
        assert np.array_equal(np.argmax(scores, axis=1), np.argmax(want, axis=1))
    finally:
        if server is not None:
            server.Dispose()
        client.Dispose()


def test_lola_small_server_with_every_element_end_to_end():
    """LoLa-small topology with every Galois element from the blob.  As in the network tests, one coefficient modulus more than the
    reference's SmallModulusCount=3 lets the last layer decrypt."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    client = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
    server = None
    try:
        server = B200BfvFactory(client.SaveCompactKeys())
        imgs = synthetic_mnist(2, seed=6)
        net, _ = lola_small(server, imgs)
        net.PrepareNetwork()
        raw_net, _ = lola_small(RawFactory(8192), imgs)
        raw_net.PrepareNetwork()
        for _ in range(2):
            got = _client_scores(client, server, net.GetNext()).reshape(-1)
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            assert np.array_equal(got, want)
    finally:
        if server is not None:
            server.Dispose()
        client.Dispose()
