"""Batched forms of the LoLa vector operations for several clients (duplicate, permute, row dot products, interleave, plain products), the
client-by-row plain-product kernel behind them, and LoLa / LoLa-Dense served to several clients in one pass.  Every batched output must
be the ciphertext the single call (or a server holding only that client's keys) computes, word for word."""
import numpy as np
import pytest

from cryptonets_b200._lib import CnheError, check

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
T, N = 2277377, 8192  # one LoLa-small plaintext prime: a single stream


@pytest.fixture(scope="module")
def slots3():
    """A server context with its own keys in slot 0 and two clients' compact keys in slots 1 and 2."""
    from cryptonets_b200.engine import Engine
    server = Engine([T], N, 40, 40, 3)
    server.keygen(100)
    clients, slots = [], [0]
    for j in range(2):
        c = Engine([T], N, 40, 40, 3)
        c.keygen(200 + j)
        clients.append(c)
        slots.append(server.add_client_compact(c.save_compact_keys(public=False)))
    yield server, [server] + clients, slots
    for c in clients:
        c.close()
    server.close()


def _inputs(server, owners, slots, order, rng, dim=N // 2, high=1000):
    """One encrypted vector of `dim` values per entry of `order` (an owner index): encrypted by that owner, uploaded, bound to its slot."""
    vals, vecs = [], []
    for o in order:
        x = rng.integers(0, high, dim).astype(np.float64)
        v = owners[o].encrypt(x)
        if owners[o] is not server:
            raw = owners[o].export_raw_many([v])
            v.dispose()
            v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, dim)
            v.set_key_slot(slots[o])
        vals.append(x)
        vecs.append(v)
    return vals, vecs


def _same(server, got, ref):
    """Word-for-word equality of two vectors, with their metadata and key slot."""
    assert (got.dim, got.scale, got.format, got.blocks, got.key_slot) == (ref.dim, ref.scale, ref.format, ref.blocks, ref.key_slot)
    return np.array_equal(server.export_raw_many([got]), server.export_raw_many([ref]))


def _client_decrypt(client_eng, server_eng, v):
    raw = server_eng.export_raw_many([v])
    w = client_eng.import_raw(np.ascontiguousarray(raw[:, 0]), v.blocks, v.dim, v.scale, v.format)
    out = client_eng.decrypt(w)
    w.dispose()
    return out


# ------------------------------------------------------------------------------------------------ entry points against single calls
@pytest.mark.parametrize("dim,count", [(1000, 8), (300, 4), (4096, 2)])
def test_duplicate_batch_matches_single_calls(slots3, dim, count):
    """Counts whose copies reach the second half of the slots (1024 x 8, 4096 x 2) take the column rotation; 512 x 4 does not."""
    server, owners, slots = slots3
    order = [0, 1, 2, 1]
    vals, vs = _inputs(server, owners, slots, order, np.random.default_rng(dim), dim)
    got = server.duplicate_many(vs, count)
    for b, v in enumerate(vs):
        ref = server.duplicate(v, count)
        assert _same(server, got[b], ref), b
        ref.dispose()
    shift = 1 << (dim - 1).bit_length()
    d = _client_decrypt(owners[order[1]], server, got[1])
    for i in range(count):
        assert np.array_equal(d[i * shift:i * shift + dim], vals[1])
    server.dispose_many(got + vs)


def test_permute_batch_matches_single_calls(slots3):
    """Three permutations of three selections each, with NULL selections and negative shifts."""
    server, owners, slots = slots3
    rng = np.random.default_rng(4)
    dim = N // 2
    _, vs = _inputs(server, owners, slots, [2, 0, 1], rng, dim)
    masks = [server.plain((rng.random(dim) < 0.3).astype(np.float64)) for _ in range(7)]
    sels = [[masks[0], None, masks[1]], [None, masks[2], masks[3]], [masks[4], masks[5], masks[6]]]
    shifts = [[3, 0, -17], [0, -1, 250], [-1024, 5, 0]]
    got = server.permute_many(vs, list(zip(sels, shifts)), 2000)
    for b, v in enumerate(vs):
        for j in range(3):
            ref = server.permute(v, sels[j], shifts[j], 2000)
            assert _same(server, got[b * 3 + j], ref), (b, j)
            ref.dispose()
    server.dispose_many(got + vs + masks)


@pytest.mark.parametrize("length", [1024, 0x7FFFFFFF])
def test_dot_rows_batch_matches_single_calls(slots3, length):
    """LLPackedDenseLayer's partial sums (length 1024, dense output) and full sums (CNHE_ALL_SLOTS, sparse output of dimension 1)."""
    server, owners, slots = slots3
    rng = np.random.default_rng(length % 97)
    _, vs = _inputs(server, owners, slots, [1, 2, 0], rng, N, high=50)
    rows = [server.plain(rng.integers(-8, 9, N).astype(np.float64)) for _ in range(13)]
    got = server.dot_rows_batch(rows, vs, length)
    for b, v in enumerate(vs):
        for r, row in enumerate(rows):
            ref = server.dot_product(row, v, length)
            assert _same(server, got[b * len(rows) + r], ref), (b, r)
            ref.dispose()
    server.dispose_many(got + vs + rows)


@pytest.mark.parametrize("shift", [1, -1])
def test_interleave_batch_matches_single_calls(slots3, shift):
    server, owners, slots = slots3
    order = [0, 1, 2]
    _, vs = _inputs(server, owners, slots, [o for o in order for _ in range(8)], np.random.default_rng(shift + 5), 1024)
    groups = [vs[8 * b:8 * (b + 1)] for b in range(3)]
    got = server.interleave_many(groups, shift)
    for b, g in enumerate(groups):
        ref = server.interleave(g, shift)
        assert _same(server, got[b], ref), b
        ref.dispose()
    server.dispose_many(got + vs)


@pytest.mark.parametrize("B", [1, 3, 9])
def test_multiply_plain_batch_matches_single_calls(slots3, B):
    """B = 9 crosses the kernel's 8-client register group."""
    server, owners, slots = slots3
    rng = np.random.default_rng(B)
    vals, vs = _inputs(server, owners, slots, [i % 3 for i in range(B)], rng)
    m = rng.integers(0, 2, N // 2).astype(np.float64)
    plain = server.plain(m)
    got = server.multiply_plain_many(vs, plain)
    for b, v in enumerate(vs):
        ref = server.pointwise_multiply(v, plain)
        assert _same(server, got[b], ref), b
        ref.dispose()
    assert np.array_equal(_client_decrypt(owners[(B - 1) % 3], server, got[-1])[: N // 2], vals[-1] * m)
    server.dispose_many(got + vs + [plain])


# ------------------------------------------------------------------------------------------------ the client-by-row plain product
def _outer_against_per_client(eng, orc, t, n, rng):
    """Nine ciphertexts times one plain dense vector: the batched call (the outer product), one call per ciphertext (the broadcast path),
    the single pointwise product, and the CPU oracle on two of them."""
    vals = rng.integers(0, 100, (9, n // 2)).astype(np.float64)
    vs = eng.encrypt_many(vals)
    m = rng.integers(0, t, n // 2)
    plain = eng.plain(m.astype(np.float64))
    got = eng.multiply_plain_many(vs, plain)
    words = eng.export_raw_many(got)
    for b, v in enumerate(vs):
        one = eng.multiply_plain_many([v], plain)[0]
        ref = eng.pointwise_multiply(v, plain)
        assert np.array_equal(words[:, b], eng.export_raw_many([one])[:, 0]), b
        assert np.array_equal(words[:, b], eng.export_raw_many([ref])[:, 0]), b
        eng.dispose_many([one, ref])
    pl = orc.encode(m.astype(np.uint64))
    for b in (0, 8):
        assert np.array_equal(words[0, b, 0], orc.multiply_plain(vs[b].export_raw(), pl)), b
    eng.dispose_many(got + vs + [plain])


@pytest.mark.parametrize("n", [4096, 8192, 16384])
def test_outer_product_equals_broadcast_and_oracle(n):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    t = 65537
    eng = Engine([t], n, 10, 20, -1)
    try:
        eng.keygen(3)
        _outer_against_per_client(eng, Oracle(t, n, -1, 10, 20), t, n, np.random.default_rng(n))
    finally:
        eng.close()


def test_outer_product_integer_transform_fallback(monkeypatch):
    """CNHE_NTT_INT: the broadcast kernel on the shared transforms; the same words."""
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    monkeypatch.setenv("CNHE_NTT_INT", "1")
    t = 65537
    eng = Engine([t], 8192, 10, 20, -1)
    try:
        eng.keygen(3)
        _outer_against_per_client(eng, Oracle(t, 8192, -1, 10, 20), t, 8192, np.random.default_rng(1))
    finally:
        eng.close()


def test_outer_product_wide_moduli_fallback():
    """Coefficient primes above 2^50: off the FP64 path, the same words."""
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    big_q = [576460752303415297, 576460752303210497]
    t = 40961
    eng = Engine([t], 4096, 30, 30, coeff_moduli=big_q)
    try:
        eng.keygen(5)
        _outer_against_per_client(eng, Oracle(t, 4096, -1, 30, 30, custom_q=big_q), t, 4096, np.random.default_rng(2))
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_batch_refusals_leave_the_context_usable(slots3):
    from cryptonets_b200.engine import Engine
    server, owners, slots = slots3
    rng = np.random.default_rng(8)
    _, (a, b, d) = _inputs(server, owners, slots, [0, 1, 1], rng)
    _, (c,) = _inputs(server, owners, slots, [2], rng, 1000)
    plain = server.plain(rng.integers(0, 2, N // 2).astype(np.float64))
    sparse = server.plain(np.ones(3), 1.0, 1)
    other_scale = server.encrypt(np.ones(N // 2), 2.0)

    def usable():
        s = server.multiply_plain_many([a, d], plain)
        assert [v.key_slot for v in s] == [0, slots[1]]
        server.dispose_many(s)

    def refused(fn):
        with pytest.raises(CnheError) as e:
            fn()
        assert e.value.code == ERR_INVALID
        usable()

    refused(lambda: server.duplicate_many([plain, plain], 2))                 # plain inputs
    refused(lambda: server.multiply_plain_many([a, b], sparse))              # a sparse plain operand
    refused(lambda: server.multiply_plain_many([a, c], plain))               # dimensions differ
    refused(lambda: server.duplicate_many([a, other_scale], 2))              # scales differ
    refused(lambda: server.duplicate_many([a, b], 4))                        # count * shift > N
    refused(lambda: server.permute_many([a, b], [([a], [1])], 100))          # an encrypted selection
    refused(lambda: server.duplicate_many([], 2))                            # B < 1
    refused(lambda: check(server.L.cnhe_vecs_interleave_batch(server.h, None, 1, 0, 1, None)))
    other = Engine([T], N, 40, 40, 3)
    other.keygen(9)
    s = server.add_client_compact(other.save_compact_keys(public=False))
    b.set_key_slot(s)
    server.remove_client(s)
    refused(lambda: server.duplicate_many([a, b], 2))                        # a vector bound to a removed slot
    refused(lambda: server.dot_rows_batch([plain], [a, b], 1024))
    other.close()
    server.dispose_many([a, b, c, d, plain, sparse, other_scale])


# ------------------------------------------------------------------------------------------------ networks
def _clients(builder, primes, n, kw, count, images, seeds):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    clients, key_blobs, ct_blobs, scales = [], [], [], []
    for j, seed in enumerate(seeds):
        c = B200BfvFactory(primes, n, SmallModulusCount=count, seed=seed, **kw)
        _, rd = builder(c, images[j:j + 1])
        m = rd.GetNext()
        clients.append(c)
        key_blobs.append(c.SaveCompactKeys())
        ct_blobs.append(c.GetEncryptedMatrixCompact(m.Data, EMatrixFormat.ColumnMajor, 1))
        scales.append(m.Scale)
    return clients, key_blobs, ct_blobs, scales


def _apply_chain(net, m):
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    for layer in reversed(chain):
        m = layer.Apply(m)
    return m


@pytest.mark.parametrize("name", ["lola", "lola_dense"])
def test_lola_networks_served_batched(name, monkeypatch):
    """LoLa (reference parameters) with three clients and LoLa-Dense (one coefficient prime more than the reference's SmallModulusCount = 7,
    so that it decrypts) with two, through serve_batch: no layer falls back to one Apply per client, every client's scores are the
    ciphertexts of a server holding only its keys on the single-image path, and they decrypt to the Raw backend's."""
    from cryptonets_b200 import layers, networks
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.raw import RawFactory
    if name == "lola":
        builder, primes, n, kw, count, B = networks.lola, networks.LOLA_PRIMES, 8192, {}, -1, 3
    else:
        builder, primes, n, kw, count, B = networks.lola_dense, networks.LOLA_DENSE_PRIMES, 16384, dict(
            DecompositionBitCount=60, GaloisDecompositionBitCount=60), 8, 2
    imgs = networks.synthetic_mnist(B, seed=21)
    clients, key_blobs, ct_blobs, scales = _clients(builder, primes, n, kw, count, imgs, range(51, 51 + B))
    fell_back = []
    base = layers.BaseLayer.ApplyBatch

    def spy(self, ms):
        fell_back.append(type(self).__name__)
        return base(self, ms)

    server = B200BfvFactory(key_blobs[0])
    slots = [0] + [server.AddClientKeys(k) for k in key_blobs[1:]]
    try:
        inputs = []
        for j in range(B):
            m = server.LoadCompactMatrix(ct_blobs[j], EMatrixFormat.ColumnMajor, slot=slots[j])
            m.RegisterScale(scales[j])
            inputs.append(m)
        net, _ = builder(server, imgs[:1])
        monkeypatch.setattr(layers.BaseLayer, "ApplyBatch", spy)
        outs = networks.serve_batch(net, inputs)
        monkeypatch.setattr(layers.BaseLayer, "ApplyBatch", base)
        assert fell_back == [], fell_back
        for j in range(B):
            assert all(v.vec.key_slot == slots[j] for v in outs[j].vectors)
            got = server.engine.export_raw_many([v.vec for v in outs[j].vectors])
            alone = B200BfvFactory(key_blobs[j])
            try:
                m = alone.LoadCompactMatrix(ct_blobs[j], EMatrixFormat.ColumnMajor)
                m.RegisterScale(scales[j])
                anet, _ = builder(alone, imgs[:1])
                anet.PrepareNetwork()
                ref = _apply_chain(anet, m)
                assert np.array_equal(got, alone.engine.export_raw_many([v.vec for v in ref.vectors])), j
            finally:
                alone.Dispose()
            scores = np.concatenate([_client_decrypt(clients[j].engine, server.engine, v.vec) for v in outs[j].vectors])
            raw_net, _ = builder(RawFactory(n), imgs[j:j + 1])
            raw_net.PrepareNetwork()
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            got_scores = scores.reshape(-1)[: want.size]
            assert np.allclose(got_scores, want, rtol=1e-9, atol=1e-9) and got_scores.argmax() == want.argmax(), j
    finally:
        server.Dispose()
        for c in clients:
            c.Dispose()
