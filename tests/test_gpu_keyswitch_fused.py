"""The fused key switch (digit transforms and key product in one kernel, N = 4096 / 8192) against the CPU oracle on sampled
ciphertexts and against the digit path (CNHE_KS_FUSED=0) on all of them, bit for bit: relinearisation, multiply + relinearise and
Galois automorphisms / row rotations, on ragged and full calls.  Calls below the size threshold keep the digit path."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096, count=-1, dbc_r=10, dbc_g=20),
    "cryptonets8192": dict(t=549764251649, N=8192, count=-1, dbc_r=10, dbc_g=20),
    "lola8192": dict(t=2277377, N=8192, count=3, dbc_r=40, dbc_g=40),
}
SAMPLES = (0, 3, 33, 63)


@pytest.fixture(scope="module", params=list(CONFIGS))
def pair(request):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[request.param]
    os.environ.pop("CNHE_KS_FUSED", None)
    eng = Engine([cfg["t"]], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    orc = Oracle(cfg["t"], cfg["N"], cfg["count"], cfg["dbc_r"], cfg["dbc_g"])
    eng.keygen(1234)
    orc.keygen(1234)
    rng = np.random.default_rng(5)
    vals = rng.integers(0, orc.t, (6, orc.N), dtype=np.uint64)
    few = np.stack([orc.encrypt(orc.encode(vals[i]), 4000 + i) for i in range(6)])
    yield eng, orc, request.param, few
    eng.close()


def _batch(few, m):
    cts = np.stack([few[i % len(few)] for i in range(m)])
    cts[1::2] = np.roll(cts[1::2], 1, axis=0)  # neighbouring ciphertexts differ
    return cts


def _run(eng, monkeypatch, fused, fn, out, words):
    """fused: "1" / "0" forces the fused / digit path, None leaves the choice to the library"""
    if fused is None:
        monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
    else:
        monkeypatch.setenv("CNHE_KS_FUSED", fused)
    fn(out)
    return eng.dev_download(out, words).copy()


def _families(eng, fn):
    eng.sync()
    eng.prof_enable(True)
    fn()
    prof = eng.prof_collect()
    eng.prof_enable(False)
    return prof


def _sizes(name):
    return (64, 70, 945) if name == "cryptonets8192" else (64, 70)


def test_relinearize_fused(pair, monkeypatch):
    eng, orc, name, few = pair
    N, k = eng.N, eng.k
    sq = np.stack([orc.multiply(few[i], few[i]) for i in range(len(few))])
    for m in _sizes(name):
        cts3 = _batch(sq, m)
        a, out = eng.dev_from(cts3), eng.dev_alloc(m * 2 * k * N)
        monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
        prof = _families(eng, lambda: eng.raw_relinearize(0, a, m, out))
        assert prof["ntt_forward"]["launches"] == 0 and prof["keyswitch_mac"]["launches"] > 0, "the fused path did not serve %d" % m
        got = eng.dev_download(out, m * 2 * k * N).reshape(m, -1)
        for i in SAMPLES:
            assert np.array_equal(got[i], orc.relinearize(cts3[i])), (m, i)
        ref = _run(eng, monkeypatch, "0", lambda o: eng.raw_relinearize(0, a, m, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(got, ref), m
        eng.dev_free(a)
        eng.dev_free(out)


def test_multiply_relin_fused(pair, monkeypatch):
    eng, orc, name, few = pair
    N, k = eng.N, eng.k
    for m in _sizes(name):
        cts = _batch(few, m)
        a, out = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N)
        fused = _run(eng, monkeypatch, "1", lambda o: eng.raw_multiply_relin(0, a, a, m, o), out, m * 2 * k * N).reshape(m, -1)
        for i in SAMPLES[:3]:
            assert np.array_equal(fused[i], orc.relinearize(orc.multiply(cts[i], cts[i]))), (m, i)
        ref = _run(eng, monkeypatch, "0", lambda o: eng.raw_multiply_relin(0, a, a, m, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(fused, ref), m
        auto = _run(eng, monkeypatch, None, lambda o: eng.raw_multiply_relin(0, a, a, m, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(auto, ref), m
        eng.dev_free(a)
        eng.dev_free(out)


def test_galois_and_rotations_fused(pair, monkeypatch):
    eng, orc, name, few = pair
    N, k = eng.N, eng.k
    m = 70
    cts = _batch(few, m)
    a, out = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N)
    for elt in (2 * N - 1, 3):
        fused = _run(eng, monkeypatch, "1", lambda o: eng.raw_apply_galois(0, a, m, elt, o), out, m * 2 * k * N).reshape(m, -1)
        for i in (0, 69):
            assert np.array_equal(fused[i], orc.apply_galois(cts[i], elt)), (elt, i)
        ref = _run(eng, monkeypatch, "0", lambda o: eng.raw_apply_galois(0, a, m, elt, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(fused, ref), elt
    for steps in (1, -4):
        fused = _run(eng, monkeypatch, "1", lambda o: eng.raw_rotate_rows(0, a, m, steps, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(fused[1], orc.rotate_rows(cts[1], steps)), steps
        ref = _run(eng, monkeypatch, "0", lambda o: eng.raw_rotate_rows(0, a, m, steps, o), out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(fused, ref), steps
    eng.dev_free(a)
    eng.dev_free(out)


def test_small_calls_keep_the_digit_path(pair, monkeypatch):
    """Below the threshold the digit transforms run on their own (family 0 sees them); forcing the fused path there gives the same words."""
    eng, orc, name, few = pair
    N, k = eng.N, eng.k
    m = 8
    sq = np.stack([orc.multiply(few[i % len(few)], few[i % len(few)]) for i in range(m)])
    a, out = eng.dev_from(sq), eng.dev_alloc(m * 2 * k * N)
    monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
    prof = _families(eng, lambda: eng.raw_relinearize(0, a, m, out))
    assert prof["ntt_forward"]["launches"] > 0, "a call of %d ciphertexts took the fused path" % m
    ref = eng.dev_download(out, m * 2 * k * N).reshape(m, -1)
    assert np.array_equal(ref[0], orc.relinearize(sq[0]))
    fused = _run(eng, monkeypatch, "1", lambda o: eng.raw_relinearize(0, a, m, o), out, m * 2 * k * N).reshape(m, -1)
    assert np.array_equal(fused, ref)
    eng.dev_free(a)
    eng.dev_free(out)
