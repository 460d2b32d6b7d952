"""One recorded inference serving every client: a graph's key switches bound to other key slots at launch (include/cnhe.h,
cnhe_graph_bind; he.py CapturedInference.Run).

Each replay bound to a client must write, word for word, the ciphertexts the eager calls write for the same input under that client's
keys.  The inputs here are encrypted by the server and tagged with the client's slot: the words are what a key switch under that slot's keys
makes of them, whatever they decrypt to, and they differ from client to client because the keys do."""
import re

import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3


def _split(net):
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return layer, chain[::-1]


def _eager(net, m):
    from cryptonets_b200.layers import TimingLayer
    cur = m
    for layer in _split(net)[1]:
        if isinstance(layer, TimingLayer):
            continue
        out = layer.Apply(cur)
        if out is not cur and cur is not m:
            cur.Dispose()
        cur = out
    return cur


def _in_slot(f, m, slot):
    """a copy of encrypted matrix m whose vectors belong to key slot `slot`"""
    from cryptonets_b200.he import B200BfvMatrix
    c = B200BfvMatrix(f, m.vectors, m.Format)
    for v in c.vectors:
        v.vec.set_key_slot(slot)
    return c


def _words(f, m):
    return f.engine.export_raw_many([v.vec for v in m.vectors])


def _slots(m):
    return {v.vec.key_slot for v in m.vectors}


def _factory(name, ms):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200 import networks as nw
    if name.startswith("lola_small"):
        f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=3, seed=5)
        f.engine.set_option("multi_stream", ms)
        return f, nw.lola_small(f, nw.synthetic_mnist(2, seed=6), dense_method=name.split("_")[-1])
    if name == "lola":
        f = B200BfvFactory(nw.LOLA_PRIMES, 8192, seed=5)
        f.engine.set_option("multi_stream", ms)
        return f, nw.lola(f, nw.synthetic_mnist(2, seed=6))
    if name == "lola_cifar":
        f = B200BfvFactory(nw.CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=8, seed=5)
        f.engine.set_option("multi_stream", ms)
        return f, nw.lola_cifar(f, nw.synthetic_cifar(2), dense_method="diagonal", score_method="folded")
    f = B200BfvFactory(nw.CRYPTONETS_PRIMES, 8192, seed=77)
    f.engine.set_option("multi_stream", ms)
    return f, nw.cryptonets_mnist(f, nw.synthetic_mnist(8192, seed=8), batch_size=8192)


def _clients(f, n, galois=None, relin=True):
    """n new key slots of f, each a fresh key set (under f's secret key, so their results decrypt with it)"""
    return [f.AddClientKeys(f.SaveCompactKeys(public=False, relin=relin, galois=galois)) for _ in range(n)]


def _counted(eng, fn):
    c0, k0 = eng.op_counts(), eng.launch_count()
    out = fn()
    return out, {k: v - c0[k] for k, v in eng.op_counts().items()}, eng.launch_count() - k0


@pytest.mark.parametrize("multi_stream", [1, 0])
@pytest.mark.parametrize("name", ["lola_small_rows", "lola_small_folded", "lola", "lola_cifar"])
def test_rebound_replay_equals_eager_words(name, multi_stream):
    """Recorded on client A's input, run for B, C, A, B: each replay's words equal the eager inference of the same input under the bound
    slot, with the eager operation and kernel counts, and the outputs report that slot.  The clients' words differ from each other."""
    f, (net, rd) = _factory(name, multi_stream)
    try:
        net.PrepareNetwork()
        enc, _ = _split(net)
        x = enc.Apply(rd.GetNext())
        A, B, C = _clients(f, 3)
        ins = {s: _in_slot(f, x, s) for s in (A, B, C)}
        eng = f.engine
        _eager(net, ins[A]).Dispose()  # one-off set-up (scalar-MAC plans, key packing)
        want = {}
        for s in (A, B, C):
            out, ops, kernels = _counted(eng, lambda: _eager(net, ins[s]))
            want[s] = (_words(f, out), ops, kernels)
            out.Dispose()
        assert not np.array_equal(want[A][0], want[B][0])
        cap = f.CaptureInference(net, _in_slot(f, x, A))
        assert cap.graph.slots() == [A]
        for s in (B, C, A, B):
            out, ops, kernels = _counted(eng, lambda: cap.Run(ins[s]))
            assert np.array_equal(_words(f, out), want[s][0]), (name, s)
            assert ops == want[s][1] and kernels == want[s][2]
            assert _slots(out) == {s}
        cap.Dispose()
    finally:
        f.Dispose()


def test_cryptonets_rebound_to_a_relinearisation_only_client():
    """CryptoNets at 8192 images (the deferred-square planes key switch and the packed relinearisation keys): recorded on the server's own
    keys (slot 0), bound to a client holding relinearisation keys only, word for word."""
    f, (net, rd) = _factory("cryptonets", 1)
    try:
        net.PrepareNetwork()
        enc, _ = _split(net)
        x = enc.Apply(rd.GetNext())
        (R,) = _clients(f, 1, galois=[])
        xr = _in_slot(f, x, R)
        out = _eager(net, xr)
        want = _words(f, out)
        out.Dispose()
        cap = f.CaptureInference(net, _in_slot(f, x, 0))
        assert cap.graph.slots() == [0]
        out = cap.Run(xr)
        assert np.array_equal(_words(f, out), want) and _slots(out) == {R}
        cap.Dispose()
    finally:
        f.Dispose()


def test_serve_batch_eight_clients_recorded_once_run_for_eight_others():
    """serve_batch for eight clients recorded once, then run for eight clients added after the recording -- permuted, one client in two
    places -- word for word against the eager serve_batch of the same inputs."""
    from cryptonets_b200.networks import serve_batch
    f, (net, rd) = _factory("lola_small_rows", 1)
    try:
        enc, _ = _split(net)
        x = [enc.Apply(rd.GetNext()) for _ in range(2)]
        first = _clients(f, 8)
        cap = f.CaptureInference(net, [_in_slot(f, x[j % 2], s) for j, s in enumerate(first)])
        assert cap.graph.slots() == sorted(first)
        later = _clients(f, 8)
        order = [later[1], later[0], later[3], later[2], later[5], later[4], later[7], later[1]]
        ins = [_in_slot(f, x[j % 2], s) for j, s in enumerate(order)]
        outs = serve_batch(net, ins)
        want = [_words(f, o) for o in outs]
        for o in outs:
            o.Dispose()
        outs = cap.Run(ins)
        for j in range(8):
            assert np.array_equal(_words(f, outs[j]), want[j]), j
            assert _slots(outs[j]) == {order[j]}
        cap.Dispose()
    finally:
        f.Dispose()


@pytest.mark.parametrize("form", ["fused", "digit", "nolazy", "int"])
def test_every_key_reading_form(form, monkeypatch):
    """The fused key switch (packed relinearisation keys, u64 Galois keys), the digit path on lazy digits (one ciphertext per thread, the
    copy-engine kernel's four per CTA, the per-ciphertext table of a two-client call) and on canonical digits (CNHE_NO_LAZY=1: one and four
    ciphertexts per thread, the table), and the integer MAC (CNHE_NTT_INT=1), each word for word under a rebinding."""
    from cryptonets_b200.networks import serve_batch
    monkeypatch.setenv("CNHE_KS_FUSED", "1" if form in ("fused", "int") else "0")
    if form == "nolazy":
        monkeypatch.setenv("CNHE_NO_LAZY", "1")
    if form == "int":
        monkeypatch.setenv("CNHE_NTT_INT", "1")
    f, (net, rd) = _factory("lola_small_rows", 1)
    try:
        enc, _ = _split(net)
        x = enc.Apply(rd.GetNext())
        A, B, C, D = _clients(f, 4)
        for rec, run in (([A], [B]), ([A, B], [C, D])):  # one slot per call; two slots per call (per-ciphertext key tables)
            ins = [_in_slot(f, x, s) for s in run]
            outs = serve_batch(net, ins)
            want = [_words(f, o) for o in outs]
            for o in outs:
                o.Dispose()
            cap = f.CaptureInference(net, [_in_slot(f, x, s) for s in rec])
            outs = cap.Run(ins)
            for j in range(len(run)):
                assert np.array_equal(_words(f, outs[j]), want[j]), (form, run, j)
            cap.Dispose()
        if form in ("digit", "nolazy"):  # a key switch of at least 64 ciphertexts: four ciphertexts share each key load
            eng = f.engine
            a = eng.encrypt(np.arange(64 * eng.N, dtype=np.float64) % 7)
            a.set_key_slot(A)
            b = eng.encrypt(np.arange(64 * eng.N, dtype=np.float64) % 7)
            b.set_key_slot(B)
            eng.capture_begin()
            g_out = eng.pointwise_multiply(a, a)
            graph = eng.capture_end()
            want = eng.export_raw_many([eng.pointwise_multiply(b, b)])
            graph.bind([B])
            a.set_key_slot(B)
            eng.vecs_assign([a], [b])
            graph.launch()
            assert g_out.key_slot == B
            assert np.array_equal(eng.export_raw_many([g_out]), want)
            graph.dispose()
    finally:
        f.Dispose()


def test_superset_client_decrypts_to_the_eager_scores():
    """Recorded under a client holding only the Galois elements the inference reads, run for a client holding every standard element:
    the bound client follows the recorded hop plan, and its scores decrypt to the eager scores.  (The clients' keys are fresh key sets
    under the server's secret key, so the server decrypts the outputs once they are tagged slot 0.  Four coefficient moduli: at three the
    scores are out of noise budget.)"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200 import networks as nw
    f = B200BfvFactory(nw.LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=4, seed=5)
    net, rd = nw.lola_small(f, nw.synthetic_mnist(2, seed=6))
    try:
        net.PrepareNetwork()
        eng = f.engine
        enc, _ = _split(net)
        x = enc.Apply(rd.GetNext())
        out = _eager(net, x)  # the server's own keys
        want = eng.decrypt_many([v.vec for v in out.vectors])
        out.Dispose()
        # the elements the inference reads: each refused bind of a graph recorded with every element names one the bound client lacks
        probe = f.CaptureInference(net, _in_slot(f, x, _clients(f, 1)[0]))
        needed = []
        while True:
            (A,) = _clients(f, 1, galois=needed)
            try:
                probe.graph.bind([A])
                break
            except CnheError as e:
                m = re.search(r"Galois key of element (\d+)", str(e))
                assert m, str(e)
                needed.append(int(m.group(1)))
        probe.Dispose()
        assert needed and set(needed) < set(eng.galois_elts())
        (S,) = _clients(f, 1)
        cap = f.CaptureInference(net, _in_slot(f, x, A))
        out = cap.Run(_in_slot(f, x, S))
        assert _slots(out) == {S}
        for v in out.vectors:
            v.vec.set_key_slot(0)
        assert np.array_equal(eng.decrypt_many([v.vec for v in out.vectors]), want)
        cap.Dispose()
    finally:
        f.Dispose()


def test_bind_refusals_ordering_and_memory():
    """Refused binds (a missing Galois element names slot and element, a removed slot, a wrong count, while recording) keep the previous
    binding; Run refuses two slots for one recorded slot before touching anything; removing or replacing a bound slot's keys refuses the
    next launch until it is bound again; two launches bound to different clients, enqueued back to back with no host synchronisation,
    each read their own keys; 100 binds allocate nothing."""
    from cryptonets_b200.networks import serve_batch
    f, (net, rd) = _factory("lola_small_rows", 1)
    try:
        net.PrepareNetwork()
        eng = f.engine
        enc, _ = _split(net)
        x = enc.Apply(rd.GetNext())
        A, B, C = _clients(f, 3)
        (R,) = _clients(f, 1, galois=[])
        ins = {s: _in_slot(f, x, s) for s in (A, B, C)}
        want = {}
        for s in (A, B, C):
            out = _eager(net, ins[s])
            want[s] = _words(f, out)
            out.Dispose()
        cap = f.CaptureInference(net, _in_slot(f, x, A))
        g = cap.graph
        g.bind([B])
        with pytest.raises(CnheError) as e:
            g.bind([R])
        assert e.value.code == ERR_STATE and "key slot %d" % R in str(e.value) and "Galois key of element" in str(e.value), str(e.value)
        gone = _clients(f, 1)[0]
        f.RemoveClient(gone)
        for bad in ([gone], [], [A, B]):
            with pytest.raises(CnheError):
                g.bind(bad)
        for v in cap.inputs[0].vectors:  # the previous binding (B) is still in force
            v.vec.set_key_slot(B)
        eng.vecs_assign([v.vec for v in cap.inputs[0].vectors], [v.vec for v in ins[B].vectors])
        g.launch()
        assert np.array_equal(_words(f, cap.outputs[0]), want[B])
        eng.capture_begin()
        with pytest.raises(CnheError) as e:
            g.bind([C])
        assert e.value.code == ERR_STATE
        with pytest.raises(CnheError):
            eng.capture_end()

        # Run with two slots for one recorded slot: refused, the recorded inputs untouched
        cap2 = f.CaptureInference(net, [_in_slot(f, x, A), _in_slot(f, x, A)])
        before = [v.vec.key_slot for m in cap2.inputs for v in m.vectors]
        with pytest.raises(Exception, match="two key slots"):
            cap2.Run([ins[B], ins[C]])
        assert [v.vec.key_slot for m in cap2.inputs for v in m.vectors] == before
        eager = serve_batch(net, [ins[B], ins[B]])
        outs = cap2.Run([ins[B], ins[B]])
        assert all(np.array_equal(_words(f, o), _words(f, w)) for o, w in zip(outs, eager))
        for w in eager:
            w.Dispose()
        cap2.Dispose()

        # back to back, no host synchronisation: launch for B, eager copy of its outputs, launch for C, eager copy
        copies = []
        for s in (B, C):
            out = cap.Run(ins[s])
            copies.append([eng.copy(v.vec) for v in out.vectors])
        for s, cs in zip((B, C), copies):
            assert np.array_equal(eng.export_raw_many(cs), want[s]), s

        # a bound slot whose keys are replaced: the next launch is refused until the graph is bound again
        f.RemoveClient(C)
        with pytest.raises(CnheError) as e:
            g.launch()
        assert e.value.code == ERR_STATE and "key slot %d" % C in str(e.value)
        g.bind([B])
        g.launch()

        nbytes = cap.Info()["device_bytes"]
        for j in range(100):
            g.bind([(A, B)[j % 2]])
        assert cap.Info()["device_bytes"] == nbytes
        cap.Dispose()
    finally:
        f.Dispose()
