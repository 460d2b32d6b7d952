"""The fused BEHZ square (forward transforms, tensor square and inverse transforms in one CTA-pair kernel, N = 4096 / 8192) against the
separate kernels (CNHE_MUL_FUSED=0) bit for bit on every ciphertext and against the CPU oracle on sampled ones: size-3 products and
multiply + relinearise.  Products of two different ciphertexts, CNHE_NTT_INT and N = 16384 keep the separate kernels."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096, count=-1, dbc_r=10, dbc_g=20),
    "cryptonets8192": dict(t=549764251649, N=8192, count=-1, dbc_r=10, dbc_g=20),
    "lola8192": dict(t=2277377, N=8192, count=3, dbc_r=40, dbc_g=40),
}
SIZES = (1, 3, 64, 945)


def _engine(cfg):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    eng = Engine([cfg["t"]], cfg["N"], cfg["dbc_r"], cfg["dbc_g"], cfg["count"])
    orc = Oracle(cfg["t"], cfg["N"], cfg["count"], cfg["dbc_r"], cfg["dbc_g"])
    eng.keygen(1234)
    orc.keygen(1234)
    rng = np.random.default_rng(9)
    vals = rng.integers(0, orc.t, (6, orc.N), dtype=np.uint64)
    few = np.stack([orc.encrypt(orc.encode(vals[i]), 5000 + i) for i in range(6)])
    return eng, orc, few


@pytest.fixture(scope="module", params=list(CONFIGS))
def pair(request):
    os.environ.pop("CNHE_MUL_FUSED", None)
    eng, orc, few = _engine(CONFIGS[request.param])
    yield eng, orc, few
    eng.close()


def _batch(few, m):
    cts = np.stack([few[i % len(few)] for i in range(m)])
    cts[1::2] = np.roll(cts[1::2], 1, axis=0)  # neighbouring ciphertexts differ
    return cts


def _samples(m):
    return sorted({0, m // 2, m - 1})


def _profiled(eng, monkeypatch, fused, fn):
    """fused: "1" / "0" forces the fused square / the separate kernels, None leaves the choice to the library"""
    if fused is None:
        monkeypatch.delenv("CNHE_MUL_FUSED", raising=False)
    else:
        monkeypatch.setenv("CNHE_MUL_FUSED", fused)
    eng.sync()
    eng.prof_enable(True)
    fn()
    prof = eng.prof_collect()
    eng.prof_enable(False)
    return prof


def _assert_fused(prof):
    # one fused launch (family 0) per wave, no separate inverse transform, lift + floor only (no tensor kernel) in family 2
    assert prof["ntt_forward"]["launches"] > 0 and prof["ntt_inverse"]["launches"] == 0, prof
    assert prof["behz_elementwise"]["launches"] == 2 * prof["ntt_forward"]["launches"], prof


def _assert_separate(prof):
    assert prof["ntt_inverse"]["launches"] > 0, prof


def test_multiply_fused(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    for m in SIZES:
        cts = _batch(few, m)
        a, out = eng.dev_from(cts), eng.dev_alloc(m * 3 * k * N)
        prof = _profiled(eng, monkeypatch, None, lambda: eng.raw_multiply(0, a, a, m, out))
        _assert_fused(prof)
        fused = eng.dev_download(out, m * 3 * k * N).reshape(m, -1).copy()
        for i in _samples(m):
            assert np.array_equal(fused[i], orc.multiply(cts[i], cts[i]).reshape(-1)), (m, i)
        prof = _profiled(eng, monkeypatch, "0", lambda: eng.raw_multiply(0, a, a, m, out))
        _assert_separate(prof)
        ref = eng.dev_download(out, m * 3 * k * N).reshape(m, -1)
        assert np.array_equal(fused, ref), m
        eng.dev_free(a)
        eng.dev_free(out)


def test_multiply_relin_fused(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    for m in SIZES:
        cts = _batch(few, m)
        a, out = eng.dev_from(cts), eng.dev_alloc(m * 2 * k * N)
        _profiled(eng, monkeypatch, "1", lambda: eng.raw_multiply_relin(0, a, a, m, out))
        fused = eng.dev_download(out, m * 2 * k * N).reshape(m, -1).copy()
        for i in _samples(m)[:2]:
            assert np.array_equal(fused[i], orc.relinearize(orc.multiply(cts[i], cts[i])).reshape(-1)), (m, i)
        _profiled(eng, monkeypatch, "0", lambda: eng.raw_multiply_relin(0, a, a, m, out))
        ref = eng.dev_download(out, m * 2 * k * N).reshape(m, -1)
        assert np.array_equal(fused, ref), m
        eng.dev_free(a)
        eng.dev_free(out)


def test_distinct_operands_keep_separate_kernels(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    m = 64
    ca, cb = _batch(few, m), _batch(few[::-1], m)
    a, b, out = eng.dev_from(ca), eng.dev_from(cb), eng.dev_alloc(m * 3 * k * N)
    prof = _profiled(eng, monkeypatch, "1", lambda: eng.raw_multiply(0, a, b, m, out))
    _assert_separate(prof)
    got = eng.dev_download(out, m * 3 * k * N).reshape(m, -1)
    for i in (0, 63):
        assert np.array_equal(got[i], orc.multiply(ca[i], cb[i]).reshape(-1)), i
    for p in (a, b, out):
        eng.dev_free(p)


@pytest.mark.parametrize("name,env", [("cryptonets8192", "CNHE_NTT_INT"), ("default4096", "CNHE_NTT_INT"), ("cifar16384", None)])
def test_fallbacks_keep_separate_kernels(name, env, monkeypatch):
    cfg = dict(CONFIGS, cifar16384=dict(t=957181001729, N=16384, count=8, dbc_r=60, dbc_g=60))[name]
    if env:
        monkeypatch.setenv(env, "1")
    try:
        eng, orc, few = _engine(cfg)
    finally:
        if env:
            monkeypatch.delenv(env)
    N, k = eng.N, eng.k
    m = 3
    cts = _batch(few, m)
    a, out = eng.dev_from(cts), eng.dev_alloc(m * 3 * k * N)
    prof = _profiled(eng, monkeypatch, "1", lambda: eng.raw_multiply(0, a, a, m, out))
    _assert_separate(prof)
    got = eng.dev_download(out, m * 3 * k * N).reshape(m, -1)
    assert np.array_equal(got[0], orc.multiply(cts[0], cts[0]).reshape(-1))
    eng.close()
