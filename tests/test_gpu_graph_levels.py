"""Recorded inferences that switch levels: one CUDA graph across a context and the levels it switches to (include/cnhe.h,
cnhe_capture_begin_levels; he.py CaptureInference(SpanLevels=True)).

A levelled replay runs the eager levelled calls' kernels with their arguments, so every replay must write, word for word, what an eager
levelled inference writes for the same input, count what it counts in every context, and hold one kernel node per eager launch.  The
inputs differ from replay to replay: a level's stream left outside the capture would run its work once at record time, and the words of
the next input would show it."""
import os
import sys
import threading

import numpy as np
import pytest

from cryptonets_b200._lib import CnheError

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -3

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def _bench():
    import level_bench
    return level_bench


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


def _in_slot(f, m, slot):
    from cryptonets_b200.he import B200BfvMatrix
    c = B200BfvMatrix(f, m.vectors, m.Format)
    for v in c.vectors:
        v.vec.set_key_slot(slot)
    return c


def _counted(f, fn):
    """fn() and, per context of f's family (keyed by prime count), the operation counts and kernel launches it added"""
    fam = _bench().family(f)
    c0 = {g.engine.k: (g.engine.op_counts(), g.engine.launch_count()) for g in fam}
    out = fn()
    d = {}
    for g in _bench().family(f):
        ops0, k0 = c0.get(g.engine.k, ({}, 0))
        d[g.engine.k] = ({k: v - ops0.get(k, 0) for k, v in g.engine.op_counts().items()}, g.engine.launch_count() - k0)
    return out, d


def _raw_scores(build, N, imgs, j):
    from cryptonets_b200.raw import RawFactory
    net, _ = build(RawFactory(N), imgs[j:j + 1])
    net.PrepareNetwork()
    return np.asarray(net.GetNext().Decrypt()).reshape(-1)


def _network(name, multi_stream, n_images):
    """(factory, net, encrypted inputs, images) of a committed schedule's network at its level_bench test parameters"""
    from cryptonets_b200.networks import LEVEL_SCHEDULES
    B = _bench()
    build, _, N, _, _, _ = B.NETS[name]
    f = B.factory(name)
    f.engine.set_option("multi_stream", multi_stream)
    imgs = B.nw.synthetic_mnist(n_images, seed=6)
    net, rd = build(f, imgs, levels=LEVEL_SCHEDULES[name])
    net.PrepareNetwork()
    enc, _ = _split(net)
    xs = [enc.Apply(rd.GetNext()) for _ in range(n_images)]
    return f, net, xs, imgs


def _replays_equal_eager(name, multi_stream, runs):
    """records on input 0, replays inputs `runs`: words, Raw scores, per-context counts and kernel nodes against eager levelled runs"""
    B = _bench()
    build, _, N, _, _, _ = B.NETS[name]
    f, net, xs, imgs = _network(name, multi_stream, max(runs) + 1)
    try:
        _eager(net, xs[0]).Dispose()  # one-off set-up: the levels, scalar-MAC plans, key packing
        want = {}
        for j in set(runs):
            out, counts = _counted(f, lambda: _eager(net, xs[j]))
            want[j] = (_words(out), counts, out.factory.engine.k)
            out.Dispose()
        cap = f.CaptureInference(net, xs[0], SpanLevels=True)
        kernels = sum(c[1] for c in want[runs[0]][1].values())
        assert cap.Info()["kernel_nodes"] == kernels
        assert len(B.family(f)) == len({g.engine.k for g in B.family(f)}) > 1
        seen = []
        for j in runs:
            out, counts = _counted(f, lambda: cap.Run(xs[j]))
            got = _words(out)
            assert out.factory.engine.k == want[j][2]
            assert np.array_equal(got, want[j][0]), (name, multi_stream, j)
            assert counts == want[j][1], (name, j)
            scores = np.asarray(out.Decrypt()).reshape(-1)
            raw = _raw_scores(build, N, imgs, j)
            assert np.allclose(scores[:raw.size], raw, rtol=1e-9, atol=1e-9), (name, j)
            seen.append(got)
        assert not np.array_equal(seen[0], seen[1])  # the inputs differ, and so do the replays' words
        cap.Dispose()
    finally:
        f.Dispose()


@pytest.mark.parametrize("multi_stream", [1, 0])
def test_lola_levelled_replay_equals_eager(multi_stream):
    """LoLa with its committed schedule (5 -> 4 -> 3 primes): three contexts in one graph"""
    _replays_equal_eager("lola", multi_stream, [1, 2, 1])


def test_lola_dense_four_switches():
    """LoLa-Dense with its committed schedule (8 -> 7 -> 6 -> 5 -> 4 primes): five contexts in one graph"""
    _replays_equal_eager("lola_dense", 1, [1, 2])


def _clients(f, n):
    """n new key slots of f, each a fresh compact key set under f's secret key"""
    return [f.AddClientKeys(f.SaveCompactKeys(public=False)) for _ in range(n)]


def test_serve_batch_eight_clients_across_levels():
    """LoLa levelled, recorded through serve_batch for eight clients and run for eight others: each client's words equal its eager
    levelled run, and the outputs report its slot"""
    from cryptonets_b200.networks import serve_batch
    f, net, xs, _ = _network("lola", 1, 4)
    try:
        slots = _clients(f, 16)
        rec = [_in_slot(f, xs[j % 4], s) for j, s in enumerate(slots[:8])]
        run = [_in_slot(f, xs[(j + 1) % 4], s) for j, s in enumerate(slots[8:])]
        for m in serve_batch(net, run):  # one-off set-up, and the restriction of the run clients' keys into the levels
            m.Dispose()
        want = []
        for m in serve_batch(net, run):
            want.append(_words(m))
            m.Dispose()
        cap = f.CaptureInference(net, rec, SpanLevels=True)
        assert cap.graph.slots() == sorted(slots[:8])
        outs = cap.Run(run)
        for j, out in enumerate(outs):
            assert np.array_equal(_words(out), want[j]), j
            assert {v.vec.key_slot for v in out.vectors} == {slots[8 + j]}
        assert not np.array_equal(want[0], want[4])  # same input, different keys
        cap.Dispose()
    finally:
        f.Dispose()


def test_client_added_after_the_recording_and_replaced_keys():
    """A client added to the top context after the recording: its first bind restricts its keys into every level, and its replay equals
    its eager levelled run.  Keys replaced in the top context refuse the next launch until the slot is bound again."""
    from cryptonets_b200.he import B200BfvFactory
    f, net, xs, _ = _network("lola", 1, 3)
    try:
        _eager(net, xs[0]).Dispose()
        cap = f.CaptureInference(net, xs[0], SpanLevels=True)
        assert cap.graph.slots() == [0]
        (late,) = _clients(f, 1)
        xl = _in_slot(f, xs[1], late)
        got = _words(cap.Run(xl))  # restricts the late client's keys into both levels
        out = _eager(net, xl)
        assert np.array_equal(got, _words(out))
        out.Dispose()
        # the same keys imported again in the top context: a new key generation for slot 0
        eng = f.engine
        eng.import_key(0, 2, eng.export_key(0, 2))
        cap.graph.bind([0])
        eng.import_key(0, 2, eng.export_key(0, 2))
        with pytest.raises(CnheError) as e:
            cap.graph.launch()
        assert e.value.code == ERR_STATE
        got = _words(cap.Run(xs[2]))  # Run binds again: the keys are restricted into the levels anew
        out = _eager(net, xs[2])
        assert np.array_equal(got, _words(out))
        out.Dispose()
        assert isinstance(cap.outputs[0].factory, B200BfvFactory) and cap.outputs[0].factory.engine.k == 3
        cap.Dispose()
    finally:
        f.Dispose()


@pytest.fixture
def family():
    """(top k = 5, level k = 3, level k = 2, an unrelated context) at N = 8192, an encrypted vector at the top and one at level 3"""
    from cryptonets_b200.engine import Engine
    t, N = 557057, 8192
    eng = Engine([t], N, 10, 20, -1)
    eng.keygen(11)
    lvl = eng.derive_level(3)
    lvl2 = lvl.derive_level(2)
    other = Engine([t], N, 10, 20, -1)
    other.keygen(12)
    a = eng.encrypt(np.arange(10.0))
    b = lvl.encrypt(np.arange(10.0))
    yield eng, lvl, lvl2, other, a, b
    for e in (lvl2, lvl, other, eng):
        e.close()


def _not_recording(*engines):
    for e in engines:
        with pytest.raises(CnheError) as x:
            e.capture_end()
        assert x.value.code == ERR_STATE


def _usable(eng, lvl, a, b):
    assert np.array_equal(eng.decrypt(eng.rotate(a, 0)), np.arange(10.0))
    assert np.array_equal(lvl.decrypt(lvl.rotate(b, 0)), np.arange(10.0))
    (s,) = eng.mod_switch([a], lvl)
    assert np.array_equal(lvl.decrypt(s), np.arange(10.0))


def test_recorded_switch_on_engines_equals_eager(family):
    """the smallest levelled graph: a rotation at the top, a switch, a rotation and a second switch below; every replay's words equal the
    eager calls', and the level's later eager calls are ordered after the replay"""
    eng, lvl, lvl2, _, a, _ = family
    x = eng.encrypt(np.arange(10.0))

    def chain(v):
        return lvl2.rotate(lvl.mod_switch([lvl.rotate(eng.mod_switch([eng.rotate(v, 1)], lvl)[0], 2)], lvl2)[0], 3)

    ref = chain(a)
    want, values = lvl2.export_raw_many([ref]), lvl2.decrypt(ref)
    eng.capture_begin(levels=[lvl2, lvl])  # any order
    out = chain(x)
    g = eng.capture_end()
    eng.vecs_assign([x], [a])
    g.launch()
    assert np.array_equal(lvl2.export_raw_many([out]), want)
    assert np.array_equal(lvl2.decrypt(out), values)
    g.dispose()


def test_refused_switches_abort_the_whole_recording(family):
    eng, lvl, lvl2, _, a, b = family
    # a switch to a level that is not enlisted
    eng.capture_begin(levels=[lvl])
    with pytest.raises(CnheError) as e:
        eng.mod_switch([a], lvl2)
    assert e.value.code == ERR_STATE
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
    # a switch that would restrict a client's keys into the level (added after the level was derived)
    s = eng.add_client_compact(eng.save_compact_keys(public=False))
    c = eng.encrypt(np.arange(10.0))
    c.set_key_slot(s)
    eng.capture_begin(levels=[lvl])
    with pytest.raises(CnheError) as e:
        eng.mod_switch([c], lvl)
    assert e.value.code == ERR_STATE
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
    (cs,) = eng.mod_switch([c], lvl)  # eagerly, the switch restricts
    assert cs.key_slot == s


def test_refused_calls_abort_the_whole_recording(family):
    eng, lvl, _, _, a, b = family
    # a call on a level from another thread
    eng.capture_begin(levels=[lvl])
    err = []

    def other_thread():
        try:
            lvl.rotate(b, 1)
        except CnheError as x:
            err.append(x.code)

    th = threading.Thread(target=other_thread)
    th.start()
    th.join()
    assert err == [ERR_STATE]
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
    # a call that cannot be recorded, on a level
    eng.capture_begin(levels=[lvl])
    with pytest.raises(CnheError) as e:
        lvl.decrypt(b)
    assert e.value.code == ERR_STATE
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
    # cnhe_capture_end on a level
    eng.capture_begin(levels=[lvl])
    with pytest.raises(CnheError) as e:
        lvl.capture_end()
    assert e.value.code == ERR_STATE
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
    # cnhe_capture_abort on a level ends the whole recording
    eng.capture_begin(levels=[lvl])
    lvl.capture_abort()
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)


def test_destroy_while_an_enlisted_context_records(family):
    """a graph spanning two contexts is not destroyed while either records (the recording is left as it is, as for a single context);
    once it ends, the graph is destroyed"""
    eng, lvl, _, _, a, b = family
    x = eng.encrypt(np.arange(10.0))
    eng.capture_begin(levels=[lvl])
    out = lvl.rotate(eng.mod_switch([x], lvl)[0], 0)
    g = eng.capture_end()
    for rec in (lvl, eng):
        rec.capture_begin()
        with pytest.raises(CnheError) as e:
            g.dispose()
        assert e.value.code == ERR_STATE
        rec.capture_abort()
    g.launch()
    assert np.array_equal(lvl.decrypt(out), np.arange(10.0))
    g.dispose()
    _usable(eng, lvl, a, b)


def test_bad_enlistments(family):
    eng, lvl, lvl2, other, a, b = family
    for owner, levels, why in [(eng, [lvl, lvl], "duplicate"), (eng, [eng], "itself"), (eng, [other], "other family"),
                               (lvl, [eng], "more primes"), (lvl2, [lvl], "more primes"), (lvl, [lvl2, lvl2], "duplicate")]:
        with pytest.raises(CnheError) as e:
            owner.capture_begin(levels=levels)
        assert e.value.code == ERR_INVALID, why
        _not_recording(eng, lvl, lvl2)
    # a level of equal prime count: another derivation at k = 3
    twin = eng.derive_level(3)
    try:
        with pytest.raises(CnheError) as e:
            lvl.capture_begin(levels=[twin])
        assert e.value.code == ERR_INVALID
    finally:
        twin.close()
    # an enlisted context that already records: refused, and its own recording left running
    lvl.capture_begin()
    with pytest.raises(CnheError) as e:
        eng.capture_begin(levels=[lvl])
    assert e.value.code == ERR_STATE
    _not_recording(eng)
    lvl.capture_abort()
    _not_recording(lvl)
    # profiling on an enlisted context: refused as cnhe_capture_begin refuses it
    lvl.prof_enable(True)
    with pytest.raises(CnheError) as e:
        eng.capture_begin(levels=[lvl])
    assert e.value.code == ERR_INVALID
    lvl.prof_enable(False)
    _not_recording(eng, lvl)
    _usable(eng, lvl, a, b)
