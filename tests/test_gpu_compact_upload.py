"""Compact ciphertext upload (cnhe_vecs_encrypt_compact / cnhe_vecs_import_compact) on the GPU: the blob bit for bit against the Python
restatement and a secret-key encryption composed from the CPU oracle, import bit for bit against the restated expansion, a server
without the secret key, CryptoNets end to end, secure mode, malformed blobs and pipelined imports."""
import struct

import numpy as np
import pytest

import compact_ref as cr

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=[40961], N=4096, count=-1, dbc_r=10, dbc_g=20),
    "cryptonets8192": dict(t=[549764251649, 549764284417], N=8192, count=-1, dbc_r=10, dbc_g=20),
    "lola_small8192": dict(t=[2277377, 2424833], N=8192, count=3, dbc_r=40, dbc_g=40),
    "cifar16384": dict(t=[957181001729, 957181034497], N=16384, count=8, dbc_r=60, dbc_g=60),
}
SEED = 4242


@pytest.fixture(scope="module", params=list(CONFIGS))
def setup(request):
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS[request.param]
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    eng.keygen(SEED)
    yield eng, cfg
    eng.close()


def _oracles(cfg):
    from oracle.oracle_py import Oracle
    out = []
    for c, t in enumerate(cfg["t"]):
        o = Oracle(t, cfg["N"], cfg["count"], cfg["dbc_r"], cfg["dbc_g"])
        o.keygen(SEED + c)
        out.append(o)
    return out


def _values(n, dim, seed=1):
    return np.random.default_rng(seed).integers(-50, 51, (n, dim)).astype(np.float64)


def _expected(orcs, vals, N, nonce0=1):
    """[P][n*B][2kN] ciphertexts of the seeded client, composed on the CPU, and the per-channel keys"""
    n, dim = vals.shape
    B = -(-dim // N)
    cts, keys = [], []
    for c, orc in enumerate(orcs):
        key = cr.seeded_key(SEED + c, nonce0)
        keys.append(key)
        row = []
        for i in range(n):
            for b in range(B):
                seg = vals[i, b * N: min((b + 1) * N, dim)].astype(np.int64) % orc.t
                plain = orc.encode(seg.astype(np.uint64))
                a = cr.expand_c1_ct(key, i * B + b, orc.q, N)
                row.append(cr.encrypt_symmetric(orc, SEED + c, plain, nonce0 + i * B + b, a))
        cts.append(np.stack(row))
    return np.stack(cts), keys


def test_blob_and_import_bit_exact(setup):
    eng, cfg = setup
    eng.keygen(SEED)  # nonces restart at 1
    N, n, dim = cfg["N"], 3, cfg["N"] + 100
    vals = _values(n, dim)
    blob = eng.encrypt_compact(vals, 1.0)
    orcs = _oracles(cfg)
    want, keys = _expected(orcs, vals, N)
    k, P = eng.k, eng.P
    hdr = cr.parse(blob)
    assert (hdr["N"], hdr["k"], hdr["P"], hdr["n"], hdr["B"], hdr["dim"], hdr["scale"]) == (N, k, P, n, 2, dim, 1.0)
    assert hdr["q"] == eng.q and hdr["t"] == cfg["t"] and hdr["keys"] == keys
    # 1. the blob: unpacked c0 equals the oracle's secret-key encryption, and the restatement encodes it to the same bytes
    payload = []
    for c in range(P):
        for j in range(n * 2):
            c0 = want[c, j, : k * N].reshape(k, N)
            assert np.array_equal(cr.unpack_ct_c0(hdr["payload"][c, j], eng.q, N), c0), (c, j)
            payload.append(cr.pack_ct_c0(c0, eng.q, N))
    again = cr.build_header(N, k, P, n, 2, dim, 1.0, eng.q, cfg["t"], keys) + np.concatenate(payload).astype("<u8").tobytes()
    assert again == blob
    assert len(blob) == cr.header_size(k, P) + P * n * 2 * cr.packed_words_per_ct(eng.q, N) * 8
    # 2. import: the expanded ciphertexts equal (c0, restated c1); the library and the oracle decrypt them to the input
    vecs = eng.import_compact(blob)
    assert len(vecs) == n and vecs[0].dim == dim and vecs[0].blocks == 2
    got = eng.export_raw_many(vecs)
    assert np.array_equal(got.reshape(want.shape), want)
    assert np.array_equal(eng.decrypt_many(vecs), vals)
    for c, orc in enumerate(orcs):
        dec = orc.decode(orc.decrypt(want[c, 1]))
        assert np.array_equal(dec[:100], (vals[0, N:].astype(np.int64) % orc.t).astype(np.uint64))
    eng.dispose_many(vecs)


def test_server_without_secret_key(setup):
    from cryptonets_b200.engine import Engine
    eng, cfg = setup
    N = cfg["N"]
    vals = _values(2, N, seed=2)
    blob = eng.encrypt_compact(vals, 1.0)
    server = Engine(None, archive=eng.save_keys(False))
    try:
        comp = server.import_compact(blob)
        raw = eng.export_raw_many(eng.import_compact(blob))  # the expanded ciphertexts
        rawv = server.import_raw_many(raw, 2, 1, N)
        prod_c, prod_r = server.pointwise_multiply(comp[0], comp[1]), server.pointwise_multiply(rawv[0], rawv[1])
        rot_c, rot_r = server.rotate(comp[0], 3), server.rotate(rawv[0], 3)
        pc, rc = server.export_raw_many([prod_c, rot_c]), server.export_raw_many([prod_r, rot_r])
        assert np.array_equal(pc, rc)
    finally:
        server.close()
    back = eng.import_raw_many(pc, 2, 1, N)
    assert np.array_equal(eng.decrypt(back[0]), vals[0] * vals[1])
    local = eng.rotate(eng.import_compact(blob)[0], 3)
    assert np.array_equal(eng.decrypt(back[1]), eng.decrypt(local))
    assert not np.array_equal(eng.decrypt(back[1]), vals[0])


def test_malformed_blobs_are_refused(setup):
    eng, cfg = setup
    N, k, P = cfg["N"], eng.k, eng.P
    blob = bytearray(eng.encrypt_compact(_values(2, N, seed=3), 1.0))
    counts0 = len(eng._live)

    def bad(b, cap=None):
        import ctypes as C
        from cryptonets_b200._lib import VECP
        buf = (C.c_ubyte * max(len(b), 1)).from_buffer_copy(bytes(b) or b"\0")
        out, n = (VECP * 4)(), C.c_int()
        rc = eng.L.cnhe_vecs_import_compact(eng.h, buf, len(b), out, 4 if cap is None else cap, C.byref(n))
        assert rc == -1, rc
        assert all(not out[i] for i in range(4))

    def put(off, fmt, v):
        b = bytearray(blob)
        struct.pack_into(fmt, b, off, v)
        return b

    bad(blob[:40])
    bad(blob[:-1])
    bad(blob + b"\0" * 8)
    bad(b"CNHD" + blob[4:])
    bad(put(4, "<I", 2))        # version
    bad(put(8, "<I", N * 2))    # N
    bad(put(12, "<I", k + 1))   # k
    bad(put(16, "<I", P + 1))   # P
    bad(put(20, "<I", 0))       # n
    bad(put(20, "<I", 3))       # n: length mismatch
    bad(put(24, "<I", 0))       # B
    bad(put(24, "<I", 2))       # B against dim
    bad(put(28, "<Q", N + 1))   # dim against B
    bad(put(44, "<Q", eng.q[0] + 2))            # q_0
    bad(put(44 + 8 * (k - 1), "<Q", 97))        # q_{k-1}
    bad(put(44 + 8 * k, "<Q", cfg["t"][0] + 2))  # t_0
    bad(put(20, "<I", 1 << 31))                 # n B >= 2^32
    bad(blob, cap=1)                            # out too small
    assert len(eng._live) == counts0
    # payload residues in [q_l, 2^b_l) import as canonical words
    hdr = cr.parse(blob)
    q0, b0 = eng.q[0], cr.bitlen(eng.q[0])
    c0 = cr.unpack(hdr["payload"][0, 0], b0, N)
    forged = c0.copy()
    forged[:8] = np.uint64(q0) + np.arange(8, dtype=np.uint64)
    forged[8] = np.uint64((1 << b0) - 1)
    words = cr.pack(forged, b0)
    b = bytearray(blob)
    b[cr.header_size(k, P): cr.header_size(k, P) + words.size * 8] = words.astype("<u8").tobytes()
    v = eng.import_compact(bytes(b))
    got = eng.export_raw_many(v)[0, 0, 0][:N]
    assert np.all(got < q0)
    assert np.array_equal(got[:8], np.arange(8, dtype=np.uint64))
    assert int(got[8]) == (1 << b0) - 1 - q0
    assert np.array_equal(got[9:], c0[9:])


def test_missing_secret_key_and_size_query(setup):
    from cryptonets_b200._lib import CnheError
    from cryptonets_b200.engine import Engine
    eng, cfg = setup
    server = Engine(None, archive=eng.save_keys(False))
    try:
        with pytest.raises(CnheError) as e:
            server.encrypt_compact(_values(1, 10), 1.0)
        assert e.value.code == -3 and "secret key is missing" in str(e.value)
    finally:
        server.close()
    import ctypes as C
    a = _values(2, 10)
    need = C.c_size_t()
    from cryptonets_b200._lib import DBLP
    assert eng.L.cnhe_vecs_encrypt_compact(eng.h, a.ctypes.data_as(DBLP), 2, 10, 1.0, None, 0, C.byref(need)) == 0
    assert need.value == cr.header_size(eng.k, eng.P) + eng.P * 2 * cr.packed_words_per_ct(eng.q, cfg["N"]) * 8
    small = (C.c_ubyte * (need.value - 1))()
    assert eng.L.cnhe_vecs_encrypt_compact(eng.h, a.ctypes.data_as(DBLP), 2, 10, 1.0, small, need.value - 1, C.byref(need)) == -1


def test_secure_mode_keys_differ_and_noise_budget(setup):
    from cryptonets_b200.engine import Engine
    _, cfg = setup
    eng = Engine(cfg["t"], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    try:
        eng.keygen(None)
        vals = _values(2, cfg["N"], seed=5)
        c0 = eng.op_counts(reset=True)["Encryption"]
        b1, b2 = eng.encrypt_compact(vals, 1.0), eng.encrypt_compact(vals, 1.0)
        assert eng.op_counts()["Encryption"] == c0 + 4 * eng.P  # counted per plaintext-modulus channel, as cnhe_vecs_encrypt
        h1, h2 = cr.parse(b1), cr.parse(b2)
        assert all(x != y for x, y in zip(h1["keys"], h2["keys"]))
        assert h1["keys"][0] not in (bytes(32),) and len(set(h1["keys"])) == eng.P
        assert not np.array_equal(h1["payload"], h2["payload"])
        v1, v2 = eng.import_compact(b1), eng.import_compact(b2)
        assert np.array_equal(eng.decrypt_many(v1), vals) and np.array_equal(eng.decrypt_many(v2), vals)
        pk = eng.encrypt_many(vals, 1.0)
        for c in range(eng.P):
            bc, bp = eng.noise_budget(v1[0], c), eng.noise_budget(pk[0], c)
            print("%s channel %d: fresh noise budget compact %d bits, public-key %d bits" % (cfg["N"], c, bc, bp))
            assert bc >= bp
    finally:
        eng.close()


@pytest.mark.parametrize("multi_stream", [0, 1])
def test_pipelined_imports(setup, multi_stream):
    eng, cfg = setup
    N = cfg["N"]
    blobs = [eng.encrypt_compact(_values(4, N, seed=10 + i), 1.0) for i in range(5)]
    eng.sync()
    eng.set_option("multi_stream", multi_stream)
    try:
        seq = []
        for b in blobs:  # sequential: import, square, export
            v = eng.import_compact(b)
            sq = eng.layer_square(v)
            seq.append(eng.export_raw_many(sq))
            eng.dispose_many(sq)
            eng.dispose_many(v)
        pipe, nxt = [], eng.import_compact(blobs[0])
        for i in range(len(blobs)):  # batch i + 1 is imported before batch i is exported
            cur = nxt
            sq = eng.layer_square(cur)
            eng.dispose_many(cur)
            if i + 1 < len(blobs):
                nxt = eng.import_compact(blobs[i + 1])
            pipe.append(eng.export_raw_many(sq))
            eng.dispose_many(sq)
        for a, b in zip(seq, pipe):
            assert np.array_equal(a, b)
    finally:
        eng.sync()
        eng.set_option("multi_stream", 1)


def _build_network(factory):
    from cryptonets_b200.layers import PoolLayer, SquareActivation
    from cryptonets_b200.networks import cryptonets_weights, transpose

    class Src:
        Factory = factory

        def GetOutputScale(self):
            return 16.0

        def PrepareNetwork(self):
            pass

    w = cryptonets_weights()
    conv1 = PoolLayer(Source=Src(), InputShape=[28, 28], KernelShape=[5, 5], Upperpadding=[1, 1], Stride=[2, 2], MapCount=[5, 1], WeightsScale=32,
                      Weights=w["Weights_0"])
    act2 = SquareActivation(Source=conv1)
    dense3 = PoolLayer(Source=act2, InputShape=[845], KernelShape=[845], Stride=[1000], MapCount=[100], Weights=transpose(w["Weights_1"], 845, 100),
                       Bias=w["Biases_2"], WeightsScale=1024)
    act4 = SquareActivation(Source=dense3)
    dense5 = PoolLayer(Source=act4, InputShape=[100], KernelShape=[100], Stride=[1000], MapCount=[10], Weights=w["Weights_3"], Bias=w["Biases_3"],
                       WeightsScale=32)
    layers = [conv1, act2, dense3, act4, dense5]
    dense5.PrepareNetwork()
    return layers


def _forward(layers, m):
    for layer in layers:
        nxt = layer.Apply(m)
        if layer is not layers[0]:
            m.Dispose()
        m = nxt
    return m


def test_cryptonets_compact_batch_end_to_end():
    from cryptonets_b200.he import B200BfvFactory, B200BfvMatrix, B200BfvVector
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    try:
        eng = f.engine
        layers = _build_network(f)
        imgs = synthetic_mnist(8192, seed=3)
        x = np.rint(imgs / 256.0 * 16.0)
        blob = f.GetEncryptedMatrixCompact(x, EMatrixFormat.ColumnMajor, 1)
        assert len(blob) == cr.header_size(5, 2) + 2 * 784 * 223232
        mc = f.LoadCompactMatrix(blob, EMatrixFormat.ColumnMajor)
        mc.RegisterScale(16.0)
        raw = eng.export_raw_many([v.vec for v in mc.vectors])
        mr = B200BfvMatrix(f, [B200BfvVector(f, v) for v in eng.import_raw_many(raw, 784, 1, 8192, 16.0)], EMatrixFormat.ColumnMajor,
                           CopyVectors=False)
        out_c, out_r = _forward(layers, mc), _forward(layers, mr)
        assert np.array_equal(eng.export_raw_many([v.vec for v in out_c.vectors]), eng.export_raw_many([v.vec for v in out_r.vectors]))
        scores = np.asarray(out_c.Decrypt())
        scores = scores if scores.shape[-1] == 10 else scores.T
        raw_net, _ = cryptonets_mnist(RawFactory(8192), imgs, timing=False)
        raw_net.PrepareNetwork()
        want = np.asarray(raw_net.GetNext().Decrypt())
        assert np.array_equal(np.argmax(scores, axis=1), np.argmax(want, axis=1))
        assert len(set(np.argmax(scores, axis=1))) > 1
    finally:
        f.Dispose()
