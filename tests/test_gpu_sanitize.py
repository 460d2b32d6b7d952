"""Sanitisation of results (include/cnhe.h, cnhe_vecs_sanitize; DESIGN 4.18): the words of a seeded call against the Python restatement
(tests/sanitize_ref.py), decryption and noise budget, the flood's range and distribution measured exactly with the secret key, key slots,
derived levels and recorded graphs."""
import os
import sys

import numpy as np
import pytest

import sanitize_ref as sr
from cryptonets_b200._lib import CnheError

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from noise_model import Model  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3
SEED = 321
BIG_Q = [2305843009213317121, 2305843009213120513]  # 61-bit primes = 1 mod 2^15: the integer path

CONFIGS = {
    "n4096": dict(t=[40961], N=4096, count=-1, dbc=(10, 20), q=None),
    "n8192": dict(t=[2277377, 2424833], N=8192, count=3, dbc=(40, 40), q=None),
    "n16384": dict(t=[957181001729], N=16384, count=8, dbc=(60, 60), q=None),
    "q61": dict(t=[40961], N=4096, count=-1, dbc=(30, 30), q=BIG_Q),
}


def _engine(cfg, seed=SEED):
    from cryptonets_b200.engine import Engine
    e = Engine(cfg["t"], cfg["N"], cfg["dbc"][0], cfg["dbc"][1], cfg["count"], coeff_moduli=cfg["q"])
    e.keygen(seed)
    return e


def _oracle(cfg, eng, c, seed=SEED):
    from oracle.oracle_py import Oracle
    o = Oracle(cfg["t"][c], cfg["N"], cfg["count"], cfg["dbc"][0], cfg["dbc"][1], custom_q=cfg["q"])
    o.keygen(seed + c)
    assert [int(x) for x in o.q] == eng.q
    return o


@pytest.fixture(scope="module", params=list(CONFIGS))
def setup(request):
    cfg = CONFIGS[request.param]
    eng = _engine(cfg)
    yield eng, cfg, [_oracle(cfg, eng, c) for c in range(len(cfg["t"]))]
    eng.close()


def _inputs(eng, rng):
    """a dense vector of two blocks and a sparse vector of three elements"""
    from cryptonets_b200.engine import SPARSE
    d = eng.encrypt(rng.integers(-40, 41, eng.N + 7).astype(np.float64))
    s = eng.encrypt(rng.integers(-40, 41, 3).astype(np.float64), 1.0, SPARSE)
    return [d, s]


def _b_values(eng):
    mx = eng.sanitize_max_bits()
    return [b for b in (0, 1, 63, 64, 65, 127, 128) if b <= mx] + [mx]


def test_words_equal_the_reference(setup):
    eng, cfg, orcs = setup
    eng.keygen(SEED)  # the sanitisation nonces restart at 0
    rng = np.random.default_rng(1)
    nonce = 0
    for b in _b_values(eng):
        vin = _inputs(eng, rng)
        out = eng.sanitize(vin, b)
        raw_in, raw_out = eng.export_raw_many(vin[:1]), eng.export_raw_many(out[:1])
        raw_in_s, raw_out_s = eng.export_raw_many(vin[1:]), eng.export_raw_many(out[1:])
        for c, orc in enumerate(orcs):
            cts_in = list(raw_in[c, 0]) + list(raw_in_s[c, 0])
            cts_out = list(raw_out[c, 0]) + list(raw_out_s[c, 0])
            # only the first ciphertext of each vector is composed on the CPU (the slow part); every block shares the layout
            for j in (0, 2):
                want = sr.sanitize(orc, SEED + c, cts_in[j], nonce + j, b)
                assert np.array_equal(np.asarray(cts_out[j]).reshape(want.shape), want), (b, c, j)
        for v, o in zip(vin, out):
            assert o.dim == v.dim and o.format == v.format and o.scale == v.scale and o.key_slot == v.key_slot
        assert np.array_equal(eng.decrypt(out[0]), eng.decrypt(vin[0])) and np.array_equal(eng.decrypt(out[1]), eng.decrypt(vin[1]))
        nonce += 5
        for v in vin + out:
            v.dispose()


def test_decrypts_budget_and_range(setup):
    eng, cfg, orcs = setup
    rng = np.random.default_rng(2)
    mx = eng.sanitize_max_bits()
    x = rng.integers(-40, 41, 100).astype(np.float64)
    v = eng.encrypt(x)
    mdl = Model(dict(N=eng.N, q=eng.q, primes=cfg["t"], mtilde_centered=True, dbc=cfg["dbc"][0], dbc_galois=cfg["dbc"][1]), 0)
    assert mdl.max_flood_bits() == mx
    for b in (20, mx // 2, mx - 1):
        (o,) = eng.sanitize([v], b)
        assert np.array_equal(eng.decrypt(o), x), b
        want = mdl.sanitize(b, eng.noise_budget(v))
        if want is not None:
            assert abs(eng.noise_budget(o) - want) <= 2, (b, eng.noise_budget(o), want)
        o.dispose()
    for bad in (-1, mx + 1):
        with pytest.raises(CnheError) as e:
            eng.sanitize([v], bad)
        assert e.value.code == ERR_INVALID
    p = eng.plain(x)
    with pytest.raises(CnheError) as e:
        eng.sanitize([p], 10)
    assert e.value.code == ERR_INVALID
    v.dispose()
    p.dispose()


@pytest.mark.parametrize("name", ["n4096", "q61"])
def test_flood_noise_is_exact_and_uniform(name):
    from scipy import stats
    cfg = CONFIGS[name]
    eng = _engine(cfg)
    orc = _oracle(cfg, eng, 0)
    try:
        b = 80
        x = np.arange(50, dtype=np.float64)
        v = eng.encrypt(x)
        e_in, _ = sr.noise_poly(orc, eng.export_raw_many([v])[0, 0, 0])
        (o1,) = eng.sanitize([v], b)
        (o2,) = eng.sanitize([v], b)
        w1, w2 = eng.export_raw_many([o1])[0, 0, 0], eng.export_raw_many([o2])[0, 0, 0]
        assert not np.array_equal(w1, w2)  # two calls on one input draw different words
        noise, _ = sr.noise_poly(orc, w1)
        delta = max(abs(e) for e in e_in) + 2 ** 12  # the input's noise and a fresh encryption's (u pk + e, far below 2^12)
        assert all(-(2 ** b) - delta <= e <= 2 ** b + delta for e in noise)
        # the flood dominates: (noise + 2^b) / 2^(b+1) is uniform on [0, 1)
        u = np.array([(e + 2 ** b) / 2 ** (b + 1) for e in noise], dtype=np.float64)
        assert stats.kstest(u, "uniform").pvalue > 1e-4
        assert np.array_equal(eng.decrypt(o1), x) and np.array_equal(eng.decrypt(o2), x)
    finally:
        eng.close()


def test_mixed_key_slots_levels_and_missing_public_key():
    """one call over two clients' slots: each output decrypts under its own client's key; a slot loaded without a public key refuses; a
    derived level sanitises under the restricted keys"""
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS["n8192"]
    server, client = _engine(cfg, 11), _engine(cfg, 12)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=True, galois=[]))
        bare = server.add_client_compact(client.save_compact_keys(public=False, galois=[]))
        rng = np.random.default_rng(3)
        xs = [rng.integers(-30, 31, 64).astype(np.float64) for _ in range(4)]
        vecs = []
        for i, x in enumerate(xs):
            if i % 2:
                cv = client.encrypt(x)
                raw = client.export_raw_many([cv])
                cv.dispose()
                v = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, x.size, 1.0, 0)
                v.set_key_slot(slot)
            else:
                v = server.encrypt(x)
            vecs.append(v)
        out = server.sanitize(vecs, 30)
        for i, (o, x) in enumerate(zip(out, xs)):
            assert o.key_slot == vecs[i].key_slot
            if i % 2:
                raw = server.export_raw_many([o])
                cv = client.import_raw(np.ascontiguousarray(raw[:, 0]), 1, x.size, 1.0, 0)
                assert np.array_equal(client.decrypt(cv), x)
                cv.dispose()
            else:
                assert np.array_equal(server.decrypt(o), x)
        vecs[1].set_key_slot(bare)
        with pytest.raises(CnheError) as e:
            server.sanitize(vecs[1:2], 30)
        assert e.value.code == ERR_STATE and "public key" in str(e.value)
        # a derived level: the restricted public key of slot 0 and of the client's slot
        lvl = server.derive_level(2)
        vecs[1].set_key_slot(slot)
        low = server.mod_switch(vecs[:2], lvl)
        (lo0, lo1) = lvl.sanitize(low, 20)
        assert np.array_equal(lvl.decrypt(lo0), xs[0])
        raw = lvl.export_raw_many([lo1])
        cl = client.derive_level(2)
        cv = cl.import_raw(np.ascontiguousarray(raw[:, 0]), 1, xs[1].size, 1.0, 0)
        assert np.array_equal(cl.decrypt(cv), xs[1])
        for v in vecs + out + low + [lo0, lo1, cv]:
            v.dispose()
        lvl.close()
        cl.close()
    finally:
        server.close()
        client.close()


def _sanitized_net(build, f, imgs, **kw):
    """the network with a SanitizeLayer of flood width log2 N appended (NoiseBits and StatisticalBits 0: fits the final budgets of
    these parameters, whatever the committed bounds)"""
    from cryptonets_b200.layers import SanitizeLayer
    net, reader = build(f, imgs, **kw)
    return SanitizeLayer(Source=net, NoiseBits=0, StatisticalBits=0), reader


def _split(net):
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return layer, chain[::-1]


def _eager(net, m):
    cur = m
    for layer in _split(net)[1]:
        out = layer.Apply(cur)
        if out is not cur and cur is not m:
            cur.Dispose()
        cur = out
    return cur


def _words(m):
    return m.factory.engine.export_raw_many([v.vec for v in m.vectors])


def _lola_small(seed):
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.he import B200BfvFactory
    f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=seed)
    net, reader = _sanitized_net(nw.lola_small, f, nw.synthetic_mnist(2, seed=6))
    net.PrepareNetwork()
    return f, net, _split(net)[0].Apply(reader.GetNext())


def test_recorded_lola_small_ends_in_sanitisation():
    """two replays give different words and equal scores; on a context seeded alike, replay i equals eager call i word for word"""
    f, net, x = _lola_small(41)
    g, net2, y = _lola_small(41)
    try:
        assert np.array_equal(_words(x), _words(y))
        cap = f.CaptureInference(net, x)  # runs the chain once eagerly first: that is sanitisation call 0
        r1 = cap.Run(x)
        s1, w1 = np.asarray(r1.Decrypt()), _words(r1)
        r2 = cap.Run(x)
        s2, w2 = np.asarray(r2.Decrypt()), _words(r2)
        assert np.array_equal(s1, s2) and not np.array_equal(w1, w2)
        eager = [_eager(net2, y) for _ in range(3)]
        assert np.array_equal(_words(eager[1]), w1) and np.array_equal(_words(eager[2]), w2)
        assert np.array_equal(np.asarray(eager[0].Decrypt()), s1)
        for m in eager:
            m.Dispose()
        cap.Dispose()
    finally:
        f.Dispose()
        g.Dispose()


def test_recorded_sanitisation_rebound_to_another_client():
    """a graph recorded on slot 0 and bound to a client's slot sanitises under that client's public key (a new key kind of the binding)"""
    cfg = CONFIGS["n8192"]
    server, client = _engine(cfg, 21), _engine(cfg, 22)
    try:
        slot = server.add_client_compact(client.save_compact_keys(public=True, galois=[]))
        x = np.arange(64, dtype=np.float64) - 20
        v = server.encrypt(x)
        server.capture_begin()
        (o,) = server.sanitize([v], 30)
        g = server.capture_end()
        assert g.slots() == [0]
        g.launch()
        assert np.array_equal(server.decrypt(o), x)
        cv = client.encrypt(2 * x)
        raw = client.export_raw_many([cv])
        w = server.import_raw(np.ascontiguousarray(raw[:, 0]), 1, x.size, 1.0, 0)
        w.set_key_slot(slot)
        g.bind([slot])
        v.set_key_slot(slot)
        server.vecs_assign([v], [w])
        g.launch()
        assert o.key_slot == slot
        back = client.import_raw(np.ascontiguousarray(server.export_raw_many([o])[:, 0]), 1, x.size, 1.0, 0)
        assert np.array_equal(client.decrypt(back), 2 * x)
        # a slot without a public key cannot be bound
        bare = server.add_client_compact(client.save_compact_keys(public=False, galois=[]))
        with pytest.raises(CnheError) as e:
            g.bind([bare])
        assert e.value.code == ERR_STATE and "public key" in str(e.value)
        for t in (back, w, cv, o, v):
            t.dispose()
        g.dispose()
    finally:
        server.close()
        client.close()


def _lola_small_k5(seed=5):
    from cryptonets_b200 import networks as nw
    from cryptonets_b200.he import B200BfvFactory
    return B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=5, seed=seed)


def _raw_scores(build, imgs, **kw):
    from cryptonets_b200.raw import RawFactory
    net, _ = build(RawFactory(8192), imgs, **kw)
    net.PrepareNetwork()
    return np.asarray(net.GetNext().Decrypt()).reshape(-1)


def test_recorded_levelled_inference_with_sanitisation_matches_raw():
    """lola_small on five primes switched to four after act3, recorded across the levels (SpanLevels=True) and ending in a SanitizeLayer:
    replays give the Raw backend's scores and different words"""
    from cryptonets_b200 import networks as nw
    f = _lola_small_k5()
    try:
        imgs = nw.synthetic_mnist(1, seed=6)
        net, reader = _sanitized_net(nw.lola_small, f, imgs, levels={"act3": 4})
        net.PrepareNetwork()
        x = _split(net)[0].Apply(reader.GetNext())
        cap = f.CaptureInference(net, x, SpanLevels=True)
        r1 = cap.Run(x)
        assert r1.factory.engine.k == 4
        s1, w1 = np.asarray(r1.Decrypt()).reshape(-1), _words(r1)
        r2 = cap.Run(x)
        s2, w2 = np.asarray(r2.Decrypt()).reshape(-1), _words(r2)
        assert np.array_equal(s1, s2) and not np.array_equal(w1, w2)
        assert np.array_equal(s1, _raw_scores(nw.lola_small, imgs))
        cap.Dispose()
    finally:
        f.Dispose()


def test_end_to_end_sanitize_true_at_a_budget_that_covers_lambda_40():
    """lola_small on five coefficient primes (one more than its test parameters): its final budget covers the committed output-noise bound
    plus 40 + log2 N flood bits, and sanitize=True scores equal the Raw backend's"""
    from cryptonets_b200 import networks as nw
    f = _lola_small_k5()
    try:
        imgs = nw.synthetic_mnist(1, seed=6)
        net, _ = nw.lola_small(f, imgs, sanitize=True)
        assert net.FloodBits(8192) == nw.OUTPUT_NOISE_BITS["lola_small"] + 40 + 13 <= f.SanitizeMaxBits()
        net.PrepareNetwork()
        got = np.asarray(net.GetNext().Decrypt()).reshape(-1)
        assert np.array_equal(got, _raw_scores(nw.lola_small, imgs, sanitize=True))
    finally:
        f.Dispose()
