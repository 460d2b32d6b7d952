"""Levels on the GPU (include/cnhe.h, cnhe_context_derive_level / cnhe_vecs_mod_switch; DESIGN 4.17).

The switch kernel's words equal the Python reference's bit for bit; a derived level's keys equal those of a seeded context created on the
same prefix of primes; every operation at the derived level gives the words the fresh context gives on the same inputs; switched vectors
decrypt to the same values; several clients' key slots follow the vectors down; the refusals leave both contexts usable."""
import numpy as np
import pytest

import mod_switch_ref as R
import worst_case_inputs as W
from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3

# t, N, q: the edge shapes of test_gpu_ring_and_modulus_edges.py with more than one prime, and the N = 16384 default modulus (k = 9)
SHAPES = {
    "n1024-fp": (12289, 1024, W.primes(36, 1024) + W.primes(40, 1024) + W.primes(44, 1024)),
    "n2048-fp49": (40961, 2048, W.primes(49, 2048, 2)),
    "n4096-mixed": (40961, 4096, W.primes(44, 4096) + W.primes(53, 4096) + W.primes(56, 4096)),
    "n1024-narrow": (12289, 1024, W.primes(30, 1024, 2)),
    "n16384-k9": (65537, 16384, None),
}


def _engine(t, N, q, seed=5, dbc=(10, 20)):
    from cryptonets_b200.engine import Engine
    e = Engine([t], N, dbc[0], dbc[1], -1, coeff_moduli=q)
    e.keygen(seed)
    return e


def _raw(eng, vecs):
    """[n][blocks][2][k][N] words of channel 0"""
    a = eng.export_raw_many(vecs)
    return a[0].reshape(len(vecs), -1, 2, eng.k, eng.N)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_kernel_words_every_drop(shape):
    """every k' < k: the switched words of random ciphertexts (and of 0, q - 1 and the half boundaries of the dropped primes planted in
    the coefficients) equal the reference's"""
    t, N, q = SHAPES[shape]
    eng = _engine(t, N, q)
    try:
        rng = np.random.default_rng(1)
        vals = rng.integers(0, t, (2, N)).astype(np.float64)
        src = eng.encrypt_many(vals)
        words = _raw(eng, src)
        # planted words: coefficient 0 = 0, 1 = q - 1, 2 + 2m = the half boundary of prime k-1-m (x = floor(q_j/2) and floor(q_j/2) + 1 mod
        # every prime), overwriting the first ciphertext
        Q = 1
        for p in eng.q:
            Q *= p
        planted = [0, Q - 1]
        for p in eng.q[1:]:
            planted += [p >> 1, (p >> 1) + 1, Q - (p >> 1) - 1]
        for c, x in enumerate(planted):
            for part in range(2):
                words[0, 0, part, :, c] = [x % p for p in eng.q]
        vin = [eng.import_raw(words[i][None], 1, N, 1.0) for i in range(len(src))]
        for k2 in range(1, eng.k):
            lvl = eng.derive_level(k2)
            try:
                out = eng.mod_switch(vin, lvl)
                got = _raw(lvl, out)
                want = R.mod_switch(words, eng.q, k2)
                assert np.array_equal(got, want), (shape, k2)
                assert out[0].key_slot == 0 and out[0].dim == N
            finally:
                lvl.close()
    finally:
        eng.close()


def test_kernel_words_two_channels_several_waves():
    """n spanning several waves (chunk 16), two plaintext channels, vectors of several blocks"""
    from cryptonets_b200.engine import Engine
    t = [40961, 65537]
    eng = Engine(t, 4096, 10, 20, -1)
    eng.keygen(3)
    eng.set_option("chunk", 16)
    try:
        rng = np.random.default_rng(2)
        vecs = [eng.encrypt(rng.integers(-9, 9, 4096 * 3 - 7).astype(np.float64)) for _ in range(13)]  # 39 ciphertexts
        lvl = eng.derive_level(1)
        out = eng.mod_switch(vecs, lvl)
        for ch in range(2):
            a = eng.export_raw_many(vecs)[ch].reshape(13, 3, 2, eng.k, 4096)
            b = lvl.export_raw_many(out)[ch].reshape(13, 3, 2, 1, 4096)
            assert np.array_equal(b, R.mod_switch(a, eng.q, 1)), ch
        assert np.array_equal(lvl.decrypt_many(out), eng.decrypt_many(vecs))
        lvl.close()
    finally:
        eng.close()


@pytest.mark.parametrize("k2", [1, 4, 8])
def test_derived_keys_equal_a_seeded_context(k2):
    from cryptonets_b200.engine import Engine
    t, N = 65537, 16384
    eng = _engine(t, N, None, seed=77, dbc=(60, 60))
    lvl = eng.derive_level(k2)
    fresh = Engine([t], N, 60, 60, -1, coeff_moduli=eng.q[:k2])
    fresh.keygen(77)
    try:
        assert lvl.q == eng.q[:k2] and lvl.bsk == fresh.bsk and lvl.relin_digits == fresh.relin_digits
        for what in (0, 1, 2):
            assert np.array_equal(lvl.export_key(0, what), fresh.export_key(0, what)), what
        for elt in fresh.galois_elts():
            assert np.array_equal(lvl.export_key(0, 3, elt), fresh.export_key(0, 3, elt)), elt
    finally:
        for e in (lvl, fresh, eng):
            e.close()


def _op_pair(centered):
    """(parent, level, fresh) at N = 8192 on q[:3] of the 5-prime default modulus, and a function importing level words into fresh"""
    from cryptonets_b200.engine import Engine
    t, N = 557057, 8192
    eng = Engine([t], N, 10, 20, -1)
    eng.keygen(11)
    eng.set_option("behz_centered_mtilde", centered)
    lvl = eng.derive_level(3)
    fresh = Engine([t], N, 10, 20, -1, coeff_moduli=eng.q[:3])
    fresh.keygen(11)
    fresh.set_option("behz_centered_mtilde", centered)
    return eng, lvl, fresh


def _mirror(lvl, fresh, vecs):
    raw = lvl.export_raw_many(vecs)
    return [fresh.import_raw(np.ascontiguousarray(raw[:, i]), v.blocks, v.dim, v.scale, v.format) for i, v in enumerate(vecs)]


def _same(lvl, fresh, a, b):
    return np.array_equal(lvl.export_raw_many(a), fresh.export_raw_many(b))


@pytest.mark.parametrize("centered", [0, 1])
def test_ops_at_the_derived_level(centered):
    """multiply + relinearise (fused and separate paths: below and above 64 ciphertexts), the square layer, row and column rotations,
    SumAllSlots, conv_dense on the wgmma and FP64 MACs, the diagonal and folded products: the derived level's words equal a fresh seeded
    context's on the same imported inputs"""
    from cryptonets_b200.engine import DENSE, SPARSE
    eng, lvl, fresh = _op_pair(centered)
    try:
        rng = np.random.default_rng(centered)
        top = [eng.encrypt(rng.integers(-40, 40, 8192).astype(np.float64)) for _ in range(70)]
        xs = eng.mod_switch(top, lvl)
        ys = _mirror(lvl, fresh, xs)
        assert _same(lvl, fresh, xs, ys)
        assert _same(lvl, fresh, [lvl.pointwise_multiply(xs[0], xs[1])], [fresh.pointwise_multiply(ys[0], ys[1])])
        for n in (5, 70):
            assert _same(lvl, fresh, lvl.layer_square(xs[:n]), fresh.layer_square(ys[:n])), n
        for amount in (1, -3, 700):
            assert _same(lvl, fresh, [lvl.rotate(xs[2], amount)], [fresh.rotate(ys[2], amount)]), amount
        assert _same(lvl, fresh, [lvl.sum_all_slots(xs[3])], [fresh.sum_all_slots(ys[3])])
        assert _same(lvl, fresh, [lvl.sum_all_slots(xs[3], force_column=1)], [fresh.sum_all_slots(ys[3], force_column=1)])  # column rotation
        # conv_dense: small weights (FP64 MAC) and weights up to 200 (wgmma MAC) over 64 inputs
        K, M = 64, 8
        gather = np.arange(K * M) % K
        for wmax in (3, 200):
            w = rng.integers(-wmax, wmax + 1, (M, K)).astype(np.float64)
            wl = [lvl.plain(r, 1.0, SPARSE) for r in w]
            wf = [fresh.plain(r, 1.0, SPARSE) for r in w]
            a = lvl.layer_conv_dense(xs[:K], gather, wl, None, M, K)
            b = fresh.layer_conv_dense(ys[:K], gather, wf, None, M, K)
            assert _same(lvl, fresh, a, b), wmax
        # diagonal and folded products of a 6 x 300 matrix
        rows = rng.integers(-5, 6, (6, 300)).astype(np.float64)
        xd = eng.mod_switch([eng.encrypt(rng.integers(-5, 6, 300).astype(np.float64)) for _ in range(2)], lvl)
        yd = _mirror(lvl, fresh, xd)
        for fold in (None, 64):
            dl = lvl.diag_prepare([lvl.plain(r, 1.0, DENSE) for r in rows], fold_width=fold)
            df = fresh.diag_prepare([fresh.plain(r, 1.0, DENSE) for r in rows], fold_width=fold)
            assert _same(lvl, fresh, lvl.mat_mul_diagonal(dl, xd), fresh.mat_mul_diagonal(df, yd)), fold
    finally:
        for e in (lvl, fresh, eng):
            e.close()


def test_switched_vectors_decrypt_and_keep_their_budget():
    """after two squares at N = 8192, k = 5: the switched vectors decrypt to the same values, and their budget is at least the smaller of
    the budget before and the level's rounding floor, less one bit"""
    import math
    from cryptonets_b200.engine import Engine
    t, N = 557057, 8192
    eng = Engine([t], N, 10, 20, -1)
    eng.keygen(21)
    try:
        rng = np.random.default_rng(4)
        v = eng.encrypt(rng.integers(-5, 6, N).astype(np.float64))
        v = eng.layer_square(eng.layer_square([v]))[0]
        before = eng.noise_budget(v)
        want = eng.decrypt(v)
        for k2 in (4, 3, 2):
            lvl = eng.derive_level(k2)
            (s,) = eng.mod_switch([v], lvl)
            assert np.array_equal(lvl.decrypt(s), want), k2
            logq = sum(math.log2(p) for p in lvl.q)
            floor = logq - math.log2(t) - math.log2(math.sqrt(2 * math.log(2 * N)) * math.sqrt(N / 18.0)) - 1
            got = lvl.noise_budget(s)
            assert got >= min(before, floor) - 1, (k2, got, before, floor)
            lvl.close()
    finally:
        eng.close()


def test_pending_vector_switches_as_materialised():
    eng, lvl, fresh = _op_pair(0)
    fresh.close()
    try:
        rng = np.random.default_rng(6)
        x = eng.encrypt(rng.integers(-9, 9, 8192).astype(np.float64))
        (a,) = eng.layer_square([x])       # pending: relinearised by the switch
        (b,) = eng.layer_square([x])
        eng.export_raw_many([b])           # materialises b
        sa = eng.mod_switch([a], lvl)
        sb = eng.mod_switch([b], lvl)
        assert _same(lvl, lvl, sa, sb)
    finally:
        lvl.close()
        eng.close()


def test_compact_key_server_with_two_clients():
    """a server without a secret key, two client slots at derivation and a third added afterwards: every client's switched and squared
    vector decrypts at the client's own level to the square of its values"""
    from cryptonets_b200.engine import Engine
    t, N = 557057, 8192
    clients = []
    for j in range(3):
        c = Engine([t], N, 10, 20, -1)
        c.keygen(300 + j)
        clients.append(c)
    server = Engine(None, compact_keys=clients[0].save_compact_keys(galois=[]))
    slots = [0, server.add_client_compact(clients[1].save_compact_keys(public=False, galois=[]))]
    try:
        lvl = server.derive_level(3)
        slots.append(server.add_client_compact(clients[2].save_compact_keys(public=False, galois=[])))
        rng = np.random.default_rng(8)
        vals, ins = [], []
        for j, c in enumerate(clients):
            x = rng.integers(-30, 30, N).astype(np.float64)
            raw = c.export_raw_many([c.encrypt(x)])
            v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N)
            if slots[j]:
                v.set_key_slot(slots[j])
            vals.append(x)
            ins.append(v)
        outs = lvl.layer_square(server.mod_switch(ins, lvl))
        for j, c in enumerate(clients):
            assert outs[j].key_slot == slots[j]
            cl = c.derive_level(3)
            raw = lvl.export_raw_many([outs[j]])
            got = cl.decrypt(cl.import_raw(np.ascontiguousarray(raw[:, 0]), 1, N))
            assert np.array_equal(got, vals[j] ** 2), j
            cl.close()
        lvl.close()
    finally:
        server.close()
        for c in clients:
            c.close()


def test_serve_batch_through_a_mod_switch_layer():
    """LoLa with a switch to 4 primes after act7, where the budget left is far below the level's floors: serving two clients together
    equals serving each alone, and the scores equal the Raw backend's"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import LOLA_PRIMES, lola, serve_batch, synthetic_mnist
    from cryptonets_b200.raw import RawFactory
    primes = LOLA_PRIMES
    imgs = synthetic_mnist(2, seed=3)
    clients = [B200BfvFactory(primes, 8192, seed=500 + j) for j in range(2)]
    blob = lambda f: f.SaveCompactKeys(public=False)
    server = B200BfvFactory(clients[0].SaveCompactKeys())
    slots = [0, server.AddClientKeys(blob(clients[1]))]
    try:
        inputs = []
        for j in range(2):
            _, reader = lola(clients[j], imgs[j:j + 1])
            m = reader.GetNext()
            ct = clients[j].GetEncryptedMatrixCompact(m.Data, EMatrixFormat.ColumnMajor, 1)
            x = server.LoadCompactMatrix(ct, EMatrixFormat.ColumnMajor, slot=slots[j])
            x.RegisterScale(m.Scale)
            inputs.append(x)
        net, _ = lola(server, imgs[:1], levels={"act7": 4})
        together = serve_batch(net, inputs)
        alone = [serve_batch(net, [x])[0] for x in inputs]
        for j in range(2):
            a = [v.vec for v in together[j].vectors]
            b = [v.vec for v in alone[j].vectors]
            eng = together[j].factory.engine
            assert eng.k == 4 and np.array_equal(eng.export_raw_many(a), eng.export_raw_many(b)), j
            cl = clients[j].AtLevel(4).engine
            raw = eng.export_raw_many(a)
            got = np.concatenate([cl.decrypt(cl.import_raw(np.ascontiguousarray(raw[:, i]), a[i].blocks, a[i].dim, a[i].scale, a[i].format))
                                  for i in range(len(a))])
            rn, _ = lola(RawFactory(8192), imgs[j:j + 1], levels={"act7": 4})
            rn.PrepareNetwork()
            want = np.asarray(rn.GetNext().Decrypt()).reshape(-1)
            assert np.allclose(got.reshape(-1)[:want.size], want, rtol=1e-9, atol=1e-6), j
    finally:
        server.Dispose()
        for c in clients:
            c.Dispose()


def test_refusals_leave_both_contexts_usable():
    from cryptonets_b200.engine import Engine
    eng, lvl, fresh = _op_pair(0)
    lvl2 = lvl.derive_level(2)
    try:
        a = eng.encrypt(np.arange(10.0))
        b = lvl.encrypt(np.arange(10.0))
        p = eng.plain(np.arange(10.0))
        for args, why in [(([a, b], lvl2), "mixed levels"), (([a], fresh), "unrelated context"), (([p], lvl), "plain vector"),
                          (([b], eng), "more primes")]:
            with pytest.raises(CnheError) as e:
                eng.mod_switch(*args) if args[0][0] is not b else lvl.mod_switch(*args)
            assert e.value.code == ERR_INVALID, why
        for k2 in (0, eng.k, eng.k + 1):
            with pytest.raises(CnheError) as e:
                eng.derive_level(k2)
            assert e.value.code == ERR_INVALID, k2
        # a grandchild: switched twice or at once, the same words
        once = eng.mod_switch([a], lvl2)
        twice = lvl.mod_switch(eng.mod_switch([a], lvl), lvl2)
        assert _same(lvl2, lvl2, once, twice)
        # recording on either side: CNHE_ERR_STATE, the recording aborted, both contexts usable
        for rec in (eng, lvl):
            rec.capture_begin()
            with pytest.raises(CnheError) as e:
                eng.mod_switch([a], lvl)
            assert e.value.code == ERR_STATE
            with pytest.raises(CnheError):
                rec.capture_end()  # nothing is recording any more
        (s,) = eng.mod_switch([a], lvl)
        assert np.array_equal(lvl.decrypt(s), np.arange(10.0))
        assert np.array_equal(eng.decrypt(eng.rotate(a, 0)), np.arange(10.0))
        # either context may be destroyed first
        lvl.close()
        assert np.array_equal(lvl2.decrypt(once[0]), np.arange(10.0))
    finally:
        for e in (lvl2, lvl, fresh, eng):
            e.close()


def test_capture_of_a_levelled_network_raises_cleanly():
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import LOLA_PRIMES, lola, synthetic_mnist
    f = B200BfvFactory(LOLA_PRIMES[:1], 8192, seed=9)
    try:
        imgs = synthetic_mnist(1, seed=4)
        net, reader = lola(f, imgs, levels={"act7": 4})
        m = reader.GetNext()
        x = f.GetEncryptedMatrix(m.Data, EMatrixFormat.ColumnMajor, 1)
        x.RegisterScale(m.Scale)
        with pytest.raises(CnheError) as e:
            f.CaptureInference(net, x)
        assert e.value.code == ERR_STATE
        f.engine.rotate(x.vectors[0].vec, 1).dispose()  # the factory is usable
    finally:
        f.Dispose()


def test_derived_keys_equal_the_oracles_and_the_packed_copy_is_rebuilt():
    """N = 8192 on 3 of the 5 default primes: the derived sk, pk, rlk and Galois keys equal the CPU oracle's on q[:3]; the packed
    relinearisation keys the fused key switch reads exist in the derived context and equal a fresh q[:3] context's; a switch counts no
    operation"""
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    t, N = 557057, 8192
    eng = Engine([t], N, 10, 20, -1)
    eng.keygen(31)
    lvl = eng.derive_level(3)
    fresh = Engine([t], N, 10, 20, 3)
    fresh.keygen(31)
    orc = Oracle(t, N, 3, 10, 20)
    orc.keygen(31)
    try:
        assert orc.q == lvl.q
        assert np.array_equal(lvl.export_key(0, 0), orc.secret_key())
        assert np.array_equal(lvl.export_key(0, 1), orc.public_key())
        assert np.array_equal(lvl.export_key(0, 2).reshape(-1, 2, 3, N), orc.relin_keys())
        for elt in lvl.galois_elts()[:4]:
            assert np.array_equal(lvl.export_key(0, 3, elt).reshape(-1, 2, 3, N), orc.galois_key(elt)), elt
        packed = lvl.export_key(0, 4)
        assert packed.any() and np.array_equal(packed, fresh.export_key(0, 4))
        a = eng.encrypt(np.arange(5.0))
        eng.op_counts(reset=True)
        lvl.op_counts(reset=True)
        eng.mod_switch([a], lvl)
        assert not any(eng.op_counts().values()) and not any(lvl.op_counts().values())
    finally:
        for e in (lvl, fresh, eng):
            e.close()


def _schedules():
    from cryptonets_b200.networks import LEVEL_SCHEDULES
    return sorted(LEVEL_SCHEDULES)


@pytest.mark.parametrize("name", _schedules())
def test_committed_schedule(name):
    """each committed schedule's network at its test parameters: scores equal the Raw backend's, the operation counts summed over the
    levels equal the unswitched run's, and the final budget is at least the unswitched run's less 2 bits"""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import level_bench as B
    from cryptonets_b200.networks import LEVEL_SCHEDULES
    from cryptonets_b200.raw import RawFactory
    build, _, N, _, _, images = B.NETS[name]
    f = B.factory(name)
    try:
        imgs = images()
        x = B.encrypted_input(f, name, imgs)
        res = {}
        for key, levels in (("full", None), ("levels", LEVEL_SCHEDULES[name])):
            chain = B.chain_of(build(f, imgs, levels=levels)[0])
            for g in B.family(f):
                g.engine.op_counts(reset=True)
            out = B.run(chain, x)
            ops = {}
            for g in B.family(f):
                for op, v in g.engine.op_counts().items():
                    ops[op] = ops.get(op, 0) + v
            res[key] = (np.asarray(out.Decrypt()).reshape(-1), ops, min(B.min_budgets(out, sample=1 << 20)), out.factory.engine.k)
        raw_net, _ = build(RawFactory(N), imgs)
        raw_net.PrepareNetwork()
        want = np.asarray(raw_net.GetNext().Decrypt()).reshape(-1)
        got, ops, budget, k = res["levels"]
        assert k == min(LEVEL_SCHEDULES[name].values())
        assert np.allclose(got[:want.size], want, rtol=1e-9, atol=1e-9) and got[:want.size].argmax() == want.argmax()
        assert ops == res["full"][1]
        assert budget >= res["full"][2] - 2, (budget, res["full"][2])
    finally:
        f.Dispose()
