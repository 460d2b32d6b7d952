"""Several clients in one context: key slots, key switches that take each ciphertext's keys from its slot, and the batched LoLa layers.

Every client has its own secret key and sends a compact evaluation-key blob and compact ciphertexts; one server context holds the keys in
slots and runs the clients' inferences together.  Each client's results must be the ciphertexts a server holding only that client's keys
computes on today's single-image path, bit for bit."""
import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
T, N = 2277377, 8192  # one LoLa plaintext prime: a single stream, so a call's key switch is one wave


def _client_decrypt(client_eng, server_eng, vecs):
    """The client's decryption of server vectors: export the ciphertexts, import them into the client's context, decrypt there."""
    raw = server_eng.export_raw_many(vecs)
    P, n, blocks, _ = raw.shape
    out = []
    for i in range(n):
        v = client_eng.import_raw(np.ascontiguousarray(raw[:, i]), blocks, vecs[i].dim, vecs[i].scale, vecs[i].format)
        out.append(client_eng.decrypt(v))
        v.dispose()
    return out


def test_lola_cifar_two_clients_batched():
    """LoLa-CIFAR with two clients at N = 16384 (the digit-path key switch) and one coefficient modulus more than the reference's
    SmallModulusCount = 8, so that the scores decrypt: each client's scores equal the Raw backend's."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import CIFAR_PRIMES, lola_cifar, serve_batch, synthetic_cifar
    from cryptonets_b200.raw import RawFactory
    kw = dict(DecompositionBitCount=60, GaloisDecompositionBitCount=60)
    imgs = synthetic_cifar(2, seed=12)
    clients, key_blobs, ct_blobs, scales = _clients(lola_cifar, CIFAR_PRIMES, 16384, kw, 9, imgs, (41, 42))
    server = B200BfvFactory(key_blobs[0])
    slots = [0, server.AddClientKeys(key_blobs[1])]
    try:
        inputs = []
        for j in range(2):
            m = server.LoadCompactMatrix(ct_blobs[j], EMatrixFormat.ColumnMajor, slot=slots[j])
            m.RegisterScale(scales[j])
            inputs.append(m)
        net, _ = lola_cifar(server, imgs[:1])
        outs = serve_batch(net, inputs)
        for j in range(2):
            scores = np.concatenate(_client_decrypt(clients[j].engine, server.engine, [v.vec for v in outs[j].vectors]))
            raw_net, _ = lola_cifar(RawFactory(16384), imgs[j:j + 1])
            raw_net.PrepareNetwork()
            want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
            got = scores.reshape(-1)[: want.size]
            # the CRT join to doubles rounds as in the single-client CIFAR test: compared to 1e-9, and the class must agree
            assert np.allclose(got, want, rtol=1e-9, atol=1e-9) and got.argmax() == want.argmax(), j
    finally:
        server.Dispose()
        for c in clients:
            c.Dispose()


# ------------------------------------------------------------------------------------------------ mixed-slot key switches (engine level)
@pytest.fixture(scope="module")
def slots3():
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


def _inputs(server, owners, slots, order, rng):
    """One encrypted vector per entry of `order` (an owner index): encrypted by that owner, uploaded, bound to its slot."""
    vals, vecs = [], []
    for o in order:
        x = rng.integers(0, 1000, N // 2).astype(np.float64)
        v = owners[o].encrypt(x)
        if owners[o] is not server:
            raw = owners[o].export_raw_many([v])
            v.dispose()
            v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N // 2)
            v.set_key_slot(slots[o])
        assert v.key_slot == slots[o]
        vals.append(x)
        vecs.append(v)
    return vals, vecs


def _words(server, vecs):
    return server.export_raw_many(vecs)[:, :, 0]


def _profiled(server, fn):
    server.sync()
    server.prof_enable(True)
    out = fn()
    server.sync()
    prof = server.prof_collect()
    server.prof_enable(False)
    return out, prof


@pytest.mark.parametrize("n,interleaved", [(150, True), (150, False), (40, True)])
def test_mixed_slot_key_switches_match_per_slot_calls(slots3, n, interleaved, monkeypatch):
    """Relinearisation (square) and rotation of n ciphertexts from three slots in one call: the fused kernel reads the per-ciphertext key
    table at 150, the digit path's MAC at 40.  Bit-identical to one call per slot; the first, middle and last outputs decrypt (by their
    owner) to the expected values."""
    monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
    server, owners, slots = slots3
    order = [i % 3 for i in range(n)] if interleaved else sorted(i % 3 for i in range(n))
    vals, vecs = _inputs(server, owners, slots, order, np.random.default_rng(n + interleaved))
    fused = n >= 64
    sq, prof_sq = _profiled(server, lambda: server.layer_square(vecs))
    rot, prof_rot = _profiled(server, lambda: server.rotate_many(vecs, 1))
    for prof in (prof_sq, prof_rot):
        assert prof["keyswitch_mac"]["launches"] > 0
        # the fused key switch runs its inverse transforms itself; the digit path launches them separately
        assert (prof["ntt_inverse"]["launches"] == 0) == fused, prof
    assert (prof_rot["ntt_forward"]["launches"] == 0) == fused, prof_rot
    got_sq, got_rot = _words(server, sq), _words(server, rot)
    for o in range(3):
        idx = [i for i in range(n) if order[i] == o]
        ref_sq = server.layer_square([vecs[i] for i in idx])
        ref_rot = server.rotate_many([vecs[i] for i in idx], 1)
        assert np.array_equal(got_sq[:, idx], _words(server, ref_sq)), o
        assert np.array_equal(got_rot[:, idx], _words(server, ref_rot)), o
        assert all(v.key_slot == slots[o] for v in [sq[i] for i in idx] + [rot[i] for i in idx])
        server.dispose_many(ref_sq + ref_rot)
    for i in (0, n // 2, n - 1):
        owner = owners[order[i]]
        d_sq, d_rot = _client_decrypt(owner, server, [sq[i], rot[i]])
        assert np.array_equal(d_sq[: N // 2], (vals[i] * vals[i]) % T), i
        assert np.array_equal(d_rot[: N // 2], np.roll(vals[i], -1)), i
    server.dispose_many(sq + rot + vecs)


def test_slot_errors_leave_the_context_usable(slots3):
    from cryptonets_b200.engine import Engine
    server, owners, slots = slots3
    rng = np.random.default_rng(3)
    _, (a, b) = _inputs(server, owners, slots, [0, 1], rng)

    def usable():
        s = server.add(a, a)
        assert s.key_slot == 0
        s.dispose()

    with pytest.raises(CnheError) as e:
        server.add(a, b)
    assert e.value.code == ERR_INVALID
    usable()
    other = Engine([T], N, 40, 40, 2)  # another coefficient modulus chain
    other.keygen(7)
    with pytest.raises(CnheError) as e:
        server.add_client_compact(other.save_compact_keys(public=False, galois=[]))
    assert e.value.code == ERR_INVALID
    other.close()
    blob = owners[1].save_compact_keys(public=False, galois=[3])
    with pytest.raises(CnheError) as e:
        server.add_client_compact(blob[:-8])
    assert e.value.code == ERR_INVALID
    usable()
    s = server.add_client_compact(blob)  # holds the element of a one-step rotation only
    b.set_key_slot(s)
    r = server.rotate(b, 1)
    r.dispose()
    with pytest.raises(CnheError) as e:
        server.rotate(b, 2)  # a single NAF hop whose element the slot does not hold
    assert e.value.code == ERR_STATE
    usable()
    server.remove_client(s)
    with pytest.raises(CnheError) as e:
        server.add(b, b)
    assert e.value.code == ERR_INVALID
    with pytest.raises(CnheError) as e:
        b.set_key_slot(s)
    assert e.value.code == ERR_INVALID
    usable()
    server.dispose_many([a, b])


def test_rowmajor_batch_across_waves_matches_single_products(slots3):
    """cnhe_mat_mul_rowmajor_batch with B * n_rows above one 1024-product wave, so that one client's rows straddle two waves: every
    output equals cnhe_mat_mul_rowmajor of its own input bit for bit, dense (one-hot masks) and sparse."""
    server, owners, slots = slots3
    rng = np.random.default_rng(17)
    order = [0, 1, 2, 1]
    _, vs = _inputs(server, owners, slots, order, rng)
    rows = [server.plain(rng.integers(-8, 9, N // 2).astype(np.float64)) for _ in range(300)]  # 4 x 300 products: the last input crosses
    for force_dense in (True, False):
        got = server.mat_mul_rowmajor_batch(rows, vs, force_dense)
        for b, v in enumerate(vs):
            ref = server.mat_mul_rowmajor(rows, v, force_dense)
            assert got[b].key_slot == slots[order[b]]
            assert got[b].blocks == ref.blocks and got[b].dim == ref.dim
            assert np.array_equal(server.export_raw_many([got[b]]), server.export_raw_many([ref])), (force_dense, b)
            ref.dispose()
        server.dispose_many(got)
    server.dispose_many(rows + vs)


# coefficient primes above 2^50: the integer (non-FP64) element-wise kernels and key-switch MAC
BIG_Q = [576460752303415297, 576460752303210497]


def test_mixed_slot_key_switch_on_the_integer_path():
    """The integer key-switch MAC (k_ks_mac, contexts whose coefficient primes are too wide for the FP64 kernels) with a per-ciphertext
    key table: relinearisation and rotation of ciphertexts from two slots, bit-identical to one call per slot, decrypting correctly."""
    from cryptonets_b200.engine import Engine
    t, n_slots = 40961, 2048
    server = Engine([t], 4096, 30, 30, coeff_moduli=BIG_Q)
    client = Engine([t], 4096, 30, 30, coeff_moduli=BIG_Q)
    try:
        server.keygen(300)
        client.keygen(301)
        slot = server.add_client_compact(client.save_compact_keys(public=False))
        owners, slots = [server, client], [0, slot]
        rng = np.random.default_rng(5)
        order = [i % 2 for i in range(12)]
        vals, vecs = [], []
        for o in order:
            x = rng.integers(0, 150, n_slots).astype(np.float64)
            v = owners[o].encrypt(x)
            if o:
                raw = client.export_raw_many([v])
                v.dispose()
                v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, n_slots)
                v.set_key_slot(slot)
            vals.append(x)
            vecs.append(v)
        sq, rot = server.layer_square(vecs), server.rotate_many(vecs, 1)
        got_sq, got_rot = _words(server, sq), _words(server, rot)
        for o in range(2):
            idx = [i for i in range(len(order)) if order[i] == o]
            ref_sq, ref_rot = server.layer_square([vecs[i] for i in idx]), server.rotate_many([vecs[i] for i in idx], 1)
            assert np.array_equal(got_sq[:, idx], _words(server, ref_sq)), o
            assert np.array_equal(got_rot[:, idx], _words(server, ref_rot)), o
            server.dispose_many(ref_sq + ref_rot)
        for i in (0, 1):
            d_sq, d_rot = _client_decrypt(owners[order[i]], server, [sq[i], rot[i]])
            want = (vals[i] * vals[i]) % t
            want[want > t // 2] -= t  # decryption reads residues above t/2 as negative
            assert np.array_equal(d_sq[:n_slots], want), i
            assert np.array_equal(d_rot[:n_slots], np.roll(vals[i], -1)), i
        server.dispose_many(sq + rot + vecs)
    finally:
        client.close()
        server.close()


def test_noise_trace_skips_other_slots(slots3):
    """The noise trace measures budgets with slot 0's secret key: outputs of another slot are recorded as unmeasured (-1)."""
    server, owners, slots = slots3
    _, (a, b) = _inputs(server, owners, slots, [0, 1], np.random.default_rng(9))
    server.trace_noise(True)
    try:
        server.trace_read(clear=True)
        x, y = server.add(a, a), server.add(b, b)
        recs = server.trace_read(clear=True)
        assert len(recs) == 2 and recs[0][3] > 0 and recs[1][3] == -1, recs
        server.dispose_many([x, y])
    finally:
        server.trace_noise(False)
    server.dispose_many([a, b])


# ------------------------------------------------------------------------------------------------ batched LoLa inferences
def _score_words(factory, matrices):
    return [factory.engine.export_raw_many([v.vec for v in m.vectors]) for m in matrices]


def _apply_chain(net, m):
    """Today's single-image path from an imported input matrix: Apply of every layer after the EncryptLayer."""
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    for layer in reversed(chain):
        out = layer.Apply(m)
        m = out
    return m


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


@pytest.mark.parametrize("count", [3, 4])
def test_lola_small_batched_clients_bit_identical_to_single_client_servers(count):
    """Three clients (different seeds) at N = 8192.  At k = 3 the scores are out of noise budget, as on today's path; at k = 4 each client
    also decrypts its scores, which equal the Raw backend's."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, serve_batch, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    kw = dict(DecompositionBitCount=40, GaloisDecompositionBitCount=40)
    imgs = synthetic_mnist(3, seed=11)
    clients, key_blobs, ct_blobs, scales = _clients(lola_small, LOLA_SMALL_PRIMES, 8192, kw, count, imgs, (31, 32, 33))
    server = B200BfvFactory(key_blobs[0])  # slot 0: client 0; slots 1, 2: clients 1, 2
    slots = [0] + [server.AddClientKeys(b) for b in key_blobs[1:]]
    try:
        inputs = []
        for j in range(3):
            m = server.LoadCompactMatrix(ct_blobs[j], EMatrixFormat.ColumnMajor, slot=slots[j])
            m.RegisterScale(scales[j])
            inputs.append(m)
        net, _ = lola_small(server, imgs[:1])
        outs = serve_batch(net, inputs)
        got = _score_words(server, outs)
        for j in range(3):
            assert all(v.vec.key_slot == slots[j] for v in outs[j].vectors)
            alone = B200BfvFactory(key_blobs[j])
            try:
                m = alone.LoadCompactMatrix(ct_blobs[j], EMatrixFormat.ColumnMajor)
                m.RegisterScale(scales[j])
                anet, _ = lola_small(alone, imgs[:1])
                anet.PrepareNetwork()
                ref = _apply_chain(anet, m)
                assert np.array_equal(got[j], _score_words(alone, [ref])[0]), j
            finally:
                alone.Dispose()
            if count == 4:
                scores = np.concatenate(_client_decrypt(clients[j].engine, server.engine, [v.vec for v in outs[j].vectors]))
                raw_net, _ = lola_small(RawFactory(8192), imgs[j:j + 1])
                raw_net.PrepareNetwork()
                want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
                assert np.array_equal(scores.reshape(-1)[: want.size], want), j
    finally:
        server.Dispose()
        for c in clients:
            c.Dispose()
