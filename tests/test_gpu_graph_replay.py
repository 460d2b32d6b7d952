"""A network's inference recorded once as a CUDA graph and replayed per input (include/cnhe.h, cnhe_capture_begin; he.py CaptureInference).

Every replay must write, word for word, the ciphertexts the eager layer calls write for the same input and keys; what cannot be recorded
is refused with CNHE_ERR_STATE and leaves the context usable; launches count what the eager calls count; and the graph's memory is its
own and goes back when it is destroyed."""
import threading

import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_STATE = -3


def _split(net):
    """(EncryptLayer, the layers after it in order)"""
    from cryptonets_b200.layers import EncryptLayer
    chain, layer = [], net
    while not isinstance(layer, EncryptLayer):
        chain.append(layer)
        layer = layer.Source
    return layer, chain[::-1]


def _encrypted_inputs(net, reader, n):
    enc, _ = _split(net)
    return [enc.Apply(reader.GetNext()) for _ in range(n)]


def _eager(net, m):
    """The network's eager calls on encrypted input m (GetNext's path after the EncryptLayer; m is kept)"""
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


def _copy(f, m):
    """a copy of matrix m: the example a capture records on becomes its input slot, which every Run overwrites"""
    from cryptonets_b200.he import B200BfvMatrix
    return B200BfvMatrix(f, m.vectors, m.Format)


def _words(f, m):
    return f.engine.export_raw_many([v.vec for v in m.vectors])


def _lola_small(ms, method="rows"):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, synthetic_mnist
    f = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=3, seed=5)
    f.engine.set_option("multi_stream", ms)
    net, rd = lola_small(f, synthetic_mnist(3, seed=6), dense_method=method)
    return f, net, rd


def _lola(ms):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import LOLA_PRIMES, lola, synthetic_mnist
    f = B200BfvFactory(LOLA_PRIMES, 8192, seed=5)
    f.engine.set_option("multi_stream", ms)
    net, rd = lola(f, synthetic_mnist(3, seed=6))
    return f, net, rd


def _lola_cifar(ms):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CIFAR_PRIMES, lola_cifar, synthetic_cifar
    f = B200BfvFactory(CIFAR_PRIMES, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=8, seed=5)
    f.engine.set_option("multi_stream", ms)
    net, rd = lola_cifar(f, synthetic_cifar(3), dense_method="diagonal", score_method="folded")
    return f, net, rd


def _cryptonets(ms):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    f.engine.set_option("multi_stream", ms)
    net, rd = cryptonets_mnist(f, synthetic_mnist(3 * 8192, seed=8), batch_size=8192)
    return f, net, rd


NETWORKS = {"lola_small_rows": _lola_small, "lola_small_folded": lambda ms: _lola_small(ms, "folded"), "lola": _lola,
            "lola_cifar": _lola_cifar, "cryptonets_mnist": _cryptonets}


@pytest.mark.parametrize("multi_stream", [1, 0])
@pytest.mark.parametrize("name", list(NETWORKS))
def test_replay_equals_eager_words(name, multi_stream):
    """Recorded on input A, replayed on A, B and C: each replay's output words are the eager calls' words on the same input; the launch
    adds the (warm) eager inference's operation and kernel counts, and the graph holds that many kernel nodes."""
    f, net, rd = NETWORKS[name](multi_stream)
    try:
        net.PrepareNetwork()
        ins = _encrypted_inputs(net, rd, 3)
        eng = f.engine
        _eager(net, ins[0]).Dispose()  # one-off set-up of the first inference (scalar-MAC plans, key packing) is not per-inference work
        want, ops, kernels = [], [], []
        for m in ins:
            c0, k0 = eng.op_counts(), eng.launch_count()
            out = _eager(net, m)
            want.append(_words(f, out))
            ops.append({k: v - c0[k] for k, v in eng.op_counts().items()})
            kernels.append(eng.launch_count() - k0)
            out.Dispose()
        c0, k0 = eng.op_counts(), eng.launch_count()
        example = _copy(f, ins[0])
        cap = f.CaptureInference(net, example)
        # its one eager pass on the example is counted; the recording itself runs and counts nothing
        assert {k: v - c0[k] for k, v in eng.op_counts().items()} == ops[0] and eng.launch_count() - k0 == kernels[0]
        info = cap.Info()
        assert info["kernel_nodes"] == kernels[0] and info["device_bytes"] > 0
        for j in (0, 1, 2, 0):
            c0, k0 = eng.op_counts(), eng.launch_count()
            out = cap.Run(ins[j])
            got = _words(f, out)
            assert np.array_equal(got, want[j]), (name, j)
            assert {k: v - c0[k] for k, v in eng.op_counts().items()} == ops[j]
            assert eng.launch_count() - k0 == kernels[j]
        cap.Dispose()
        for m in ins:
            m.Dispose()
    finally:
        f.Dispose()


def test_serve_batch_eight_clients_replays_client_by_client():
    """lola_small through serve_batch for 8 clients in key slots: the replayed words equal the eager serve_batch's, client by client, on
    two sets of inputs; after one client's slot is removed the graph refuses to launch."""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.interfaces import EMatrixFormat
    from cryptonets_b200.networks import LOLA_SMALL_PRIMES, lola_small, serve_batch, synthetic_mnist
    kw = dict(DecompositionBitCount=40, GaloisDecompositionBitCount=40, SmallModulusCount=3)
    imgs = synthetic_mnist(16, seed=21)
    clients, blobs, cts = [], [], []
    for j in range(8):
        c = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, seed=300 + j, **kw)
        _, rd = lola_small(c, imgs)
        clients.append(c)
        blobs.append(c.SaveCompactKeys(public=False))
        row = []
        for r in range(2):  # two inputs per client: image j and image 8 + j
            rd.pos = j + 8 * r
            m = rd.GetNext()
            row.append((c.GetEncryptedMatrixCompact(m.Data, EMatrixFormat.ColumnMajor, 1), m.Scale))
        cts.append(row)
    server = B200BfvFactory(LOLA_SMALL_PRIMES, 8192, seed=299, **kw)
    try:
        slots = [server.AddClientKeys(b) for b in blobs]
        net, _ = lola_small(server, imgs[:1])

        def inputs(r):
            ms = []
            for j in range(8):
                m = server.LoadCompactMatrix(cts[j][r][0], EMatrixFormat.ColumnMajor, slot=slots[j])
                m.RegisterScale(cts[j][r][1])
                ms.append(m)
            return ms

        sets = [inputs(0), inputs(1)]
        want = []
        for ms in sets:
            outs = serve_batch(net, ms)
            want.append([_words(server, o) for o in outs])
            for o in outs:
                o.Dispose()
        cap = server.CaptureInference(net, inputs(0))  # its own import of set 0: the example becomes the graph's input slot
        for r in (1, 0):
            outs = cap.Run(sets[r])
            for j in range(8):
                assert all(v.vec.key_slot == slots[j] for v in outs[j].vectors)
                assert np.array_equal(_words(server, outs[j]), want[r][j]), (r, j)
        server.RemoveClient(slots[3])
        with pytest.raises(CnheError) as e:
            cap.graph.launch()
        assert e.value.code == ERR_STATE and "key slot %d" % slots[3] in str(e.value)
        with pytest.raises(CnheError):  # and its input vector's slot is gone
            cap.Run(sets[0])
        cap.Dispose()
    finally:
        server.Dispose()
        for c in clients:
            c.Dispose()


@pytest.fixture(scope="module")
def small():
    f, net, rd = _lola_small(1)
    net.PrepareNetwork()
    ins = _encrypted_inputs(net, rd, 2)
    want = []
    for m in ins:
        out = _eager(net, m)
        want.append(_words(f, out))
        out.Dispose()
    yield f, net, ins, want
    f.Dispose()


def _refusals(f, v):
    eng = f.engine
    blob = b"CNHK" + bytes(60)
    other = {}

    def from_thread():
        try:
            eng.add(v, v)
        except CnheError as e:
            other["e"] = e

    def thread_call():
        t = threading.Thread(target=from_thread)
        t.start()
        t.join()
        raise other["e"]

    return [("cnhe_vec_decrypt", lambda: eng.decrypt(v)),
            ("cnhe_vecs_decrypt", lambda: eng.decrypt_many([v])),
            ("cnhe_vec_export_raw", lambda: v.export_raw()),
            ("cnhe_vec_device_ptr", lambda: v.device_ptr()),
            ("cnhe_noise_budget", lambda: eng.noise_budget(v)),
            ("cnhe_context_sync", eng.sync),
            ("cnhe_vec_encrypt", lambda: eng.encrypt(np.ones(8))),
            ("cnhe_vecs_encrypt", lambda: eng.encrypt_many(np.ones((2, 8)))),
            ("cnhe_prof_enable", lambda: eng.prof_enable(True)),
            ("cnhe_trace_read", eng.trace_read),
            ("cnhe_keys_generate", lambda: eng.keygen(5)),
            ("cnhe_context_add_client_compact", lambda: eng.add_client_compact(blob)),
            ("cnhe_context_remove_client", lambda: eng.remove_client(1)),
            ("cnhe_context_set_option", lambda: eng.set_option("chunk", 512)),
            ("cnhe_vec_import_raw", lambda: eng.import_raw(np.zeros(eng.P * eng.ct_words, np.uint64), 1, 8)),
            ("cnhe_capture_begin", eng.capture_begin),
            ("another thread", thread_call)]


def test_refused_calls_abort_the_recording_and_leave_the_context_usable(small):
    """Each call that cannot be part of a graph is refused with CNHE_ERR_STATE naming it; the recording is aborted (capture_end is refused
    too); the same context then runs an eager inference correctly, and records and replays again."""
    f, net, ins, want = small
    eng = f.engine
    v = eng.encrypt(np.arange(8, dtype=np.float64))
    for name, call in _refusals(f, v):
        eng.capture_begin()
        s = eng.add(v, v)  # something recorded before the refusal
        with pytest.raises(CnheError) as e:
            call()
        assert e.value.code == ERR_STATE, name
        assert "records a graph" in str(e.value), (name, str(e.value))
        if name.startswith("cnhe_"):
            assert name in str(e.value), (name, str(e.value))
        with pytest.raises(CnheError) as e:
            eng.capture_end()
        assert e.value.code == ERR_STATE
        s.dispose()
        assert np.array_equal(eng.decrypt(eng.add(v, v)), 2 * np.arange(8)), name
    out = _eager(net, ins[1])
    assert np.array_equal(_words(f, out), want[1])
    out.Dispose()
    example = _copy(f, ins[0])
    cap = f.CaptureInference(net, example)
    assert np.array_equal(_words(f, cap.Run(ins[1])), want[1])
    cap.Dispose()


def test_abort_drops_the_recording():
    """capture_abort drops what was recorded (and is a no-op when nothing is recording); the vectors made while recording can be
    destroyed, and the context computes eagerly afterwards."""
    f, net, rd = _lola_small(1)
    try:
        eng = f.engine
        v = eng.encrypt(np.arange(8, dtype=np.float64))
        eng.capture_abort()
        eng.capture_begin()
        s = eng.add(v, v)
        eng.capture_abort()
        s.dispose()
        with pytest.raises(CnheError):
            eng.capture_end()
        assert np.array_equal(eng.decrypt(eng.add(v, v)), 2 * np.arange(8))
    finally:
        f.Dispose()


def test_eager_calls_and_replays_do_not_disturb_each_other(small):
    """An eager inference between two launches leaves the graph's outputs correct, and a replay leaves an eager output's words as they
    were."""
    f, net, ins, want = small
    example = _copy(f, ins[0])
    cap = f.CaptureInference(net, example)
    eager = _eager(net, ins[1])
    out = cap.Run(ins[0])
    assert np.array_equal(_words(f, out), want[0])
    before = _words(f, eager)
    assert np.array_equal(before, want[1])
    cap.Run(ins[1])
    again = _eager(net, ins[0])  # eager work queued behind a launch
    assert np.array_equal(_words(f, again), want[0])
    assert np.array_equal(_words(f, eager), want[1])
    assert np.array_equal(_words(f, out), want[1])
    for m in (eager, again):
        m.Dispose()
    cap.Dispose()


def test_destroy_returns_the_graph_memory(small):
    """Recording takes about the graph's device bytes from the device; disposing the capture gives them back (cudaMemGetInfo, within
    64 MiB for the driver's allocation rounding)."""
    import torch
    f, net, ins, want = small
    eng = f.engine
    example = _copy(f, ins[0])
    eng.set_option("release_cached_memory", 1)
    free0 = torch.cuda.mem_get_info()[0]
    cap = f.CaptureInference(net, example)
    nbytes = cap.Info()["device_bytes"]
    free1 = torch.cuda.mem_get_info()[0]
    assert free0 - free1 >= 0.9 * nbytes, (free0, free1, nbytes)
    cap.Run(ins[0])
    cap.Dispose()
    eng.set_option("release_cached_memory", 1)
    free2 = torch.cuda.mem_get_info()[0]
    assert free2 >= free0 - (64 << 20), (free0, free2, nbytes)
    example.Dispose()


def _lola16(name):
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200 import networks
    primes = networks.LOLA_DENSE_PRIMES if name == "lola_dense" else networks.LOLA_LARGE_PRIMES
    f = B200BfvFactory(primes, 16384, DecompositionBitCount=60, GaloisDecompositionBitCount=60, SmallModulusCount=7, seed=5)
    net, rd = getattr(networks, name)(f, networks.synthetic_mnist(2, seed=3))
    net.PrepareNetwork()
    return f, net, _encrypted_inputs(net, rd, 2)


def test_lola_dense_replays_word_for_word():
    """LoLa-Dense (LLPreConvLayer's permutations, 16-way packed dense layer) records, and its replays equal the eager words."""
    f, net, ins = _lola16("lola_dense")
    try:
        want = []
        for m in ins:
            out = _eager(net, m)
            want.append(_words(f, out))
            out.Dispose()
        example = _copy(f, ins[0])
        cap = f.CaptureInference(net, example)
        for j in (1, 0):
            assert np.array_equal(_words(f, cap.Run(ins[j])), want[j]), j
        cap.Dispose()
    finally:
        f.Dispose()


def test_lola_large_refuses_to_record():
    """LoLa-Large's row-method dense layer (2608 one-hot-masked rows at N = 16384) needs more scratch than a graph can own: recorded
    blocks are reused only by later allocations of a similar size on the same stream, where the eager pool reuses any freed memory.  The
    recording is refused with CNHE_ERR_STATE naming the call, and the same context then runs the inference eagerly."""
    f, net, ins = _lola16("lola_large")
    try:
        out = _eager(net, ins[1])
        want = _words(f, out)
        out.Dispose()
        with pytest.raises(CnheError) as e:
            f.CaptureInference(net, ins[0])
        assert e.value.code == ERR_STATE and "records a graph" in str(e.value) and "cnhe_" in str(e.value), str(e.value)
        assert "graph can own" in str(e.value)
        out = _eager(net, ins[1])
        assert np.array_equal(_words(f, out), want)
        out.Dispose()
    finally:
        f.Dispose()


def _cryptonets_small():
    """CryptoNets on a 100-image batch: not a multiple of N, so the PoolLayers' bias vectors are real plaintexts (not constants the MAC
    reads from the host); they are built on the layer's first Apply"""
    from cryptonets_b200.he import B200BfvFactory
    from cryptonets_b200.networks import CRYPTONETS_PRIMES, cryptonets_mnist, synthetic_mnist
    f = B200BfvFactory(CRYPTONETS_PRIMES, 8192, seed=77)
    net, rd = cryptonets_mnist(f, synthetic_mnist(100, seed=9), batch_size=100)
    net.PrepareNetwork()
    return f, net, _encrypted_inputs(net, rd, 1)[0]


def test_capture_of_a_cold_network_leaves_its_eager_words_intact():
    """A network whose layers have never run: recorded through CaptureInference, and recorded by hand with the layers' first Apply (bias
    vectors, scalar-MAC plans) inside the recording.  The eager inference afterwards and the replays equal a never-recorded network's
    words (same seed, so the same input ciphertext)."""
    ref, rnet, rx = _cryptonets_small()
    try:
        out = _eager(rnet, rx)
        want = _words(ref, out)
        out.Dispose()
    finally:
        ref.Dispose()
    f, net, x = _cryptonets_small()
    try:
        cap = f.CaptureInference(net, _copy(f, x))
        out = _eager(net, x)
        assert np.array_equal(_words(f, out), want)
        out.Dispose()
        assert np.array_equal(_words(f, cap.Run(x)), want)
        cap.Dispose()
    finally:
        f.Dispose()
    f, net, x = _cryptonets_small()
    try:
        eng = f.engine
        c0, k0 = eng.op_counts(), eng.launch_count()
        eng.capture_begin()
        out = _eager(net, x)
        graph = eng.capture_end()
        assert eng.op_counts() == c0 and eng.launch_count() == k0  # recording runs and counts nothing
        graph.launch()
        assert np.array_equal(_words(f, out), want)
        again = _eager(net, x)  # the layers' state was made by the graph's launch
        assert np.array_equal(_words(f, again), want)
        again.Dispose()
        out.Dispose()
        graph.dispose()
    finally:
        f.Dispose()


def test_buffers_from_before_the_recording():
    """Squares left unrelinearised before the recording cannot be relinearised inside it (refused, the context stays usable); a vector
    made before the recording and released during it stays the graph's until the graph is destroyed, however many eager allocations
    follow."""
    from cryptonets_b200.engine import Engine
    eng = Engine([40961], 4096, 10, 20, -1)
    try:
        eng.keygen(17)
        rng = np.random.default_rng(4)
        q = np.array(eng.q, dtype=np.uint64)[:, None]
        words = (rng.integers(0, 1 << 62, (eng.P, 2, 3, eng.k, eng.N), dtype=np.uint64) % q).astype(np.uint64)
        p = eng.raw_import_products(words, 2)
        eng.capture_begin()
        with pytest.raises(CnheError) as e:
            eng.add(p[0], p[1])
        assert e.value.code == ERR_STATE and "cnhe_vec_add" in str(e.value) and "before the recording" in str(e.value), str(e.value)
        with pytest.raises(CnheError):
            eng.capture_end()
        want = eng.add(p[0], p[1]).export_raw()  # an eager read relinearises them
        eng.capture_begin()
        g_out = eng.add(p[0], p[1])
        graph = eng.capture_end()
        graph.launch()
        assert np.array_equal(g_out.export_raw(), want)

        vals = np.arange(eng.N // 2, dtype=np.float64)
        x = eng.add(eng.encrypt(vals), eng.encrypt(vals))
        want2 = eng.add(x, x).export_raw()
        eng.capture_begin()
        y = eng.add(x, x)
        x.dispose()  # the graph still reads x's ciphertext
        graph2 = eng.capture_end()
        churn = [eng.encrypt(vals + i) for i in range(16)]
        graph2.launch()
        assert np.array_equal(y.export_raw(), want2)
        for v in churn:
            v.dispose()
        graph.dispose()
        graph2.dispose()
    finally:
        eng.close()


def test_assign_refuses_partial_overlap():
    """cnhe_vecs_assign between two vectors of one slab that overlap in part is refused; the same vector is a no-op."""
    from cryptonets_b200.engine import Engine
    eng = Engine([40961], 4096, 10, 20, -1)
    try:
        eng.keygen(17)
        vs = eng.encrypt_many(np.ones((3, eng.N * 2)))  # one slab: two ciphertexts per vector, back to back
        eng.vecs_assign([vs[0]], [vs[0]])
        with pytest.raises(CnheError):
            eng.vecs_assign(vs[0:2], vs[1:3])  # dst run [0, 2) and src run [1, 3) overlap by one vector
    finally:
        eng.close()
