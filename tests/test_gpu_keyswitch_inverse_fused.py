"""The fused key switch (N = 4096 / 8192) ends with the inverse transform and the base addition in the same kernel: on its path no
separate inverse transform runs (profiling family ntt_inverse stays empty) and there is one key-switch launch per wave.  Its outputs must
equal the digit path's (CNHE_KS_FUSED=0) bit for bit, with packed relinearisation keys and u64 Galois keys, on ragged waves, and on the
in-place rotate-and-add ladder of a row-major matrix product, whose output span is its input.  A call whose output overlaps its input
(an in-place relinearisation) must take the separate inverse transform instead."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096),
    "cryptonets8192": dict(t=549764251649, N=8192),
}
M = 72  # above the fused threshold


@pytest.fixture(scope="module", params=list(CONFIGS))
def pair(request):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[request.param]
    os.environ.pop("CNHE_KS_FUSED", None)
    eng = Engine([cfg["t"]], cfg["N"], 10, 20)
    orc = Oracle(cfg["t"], cfg["N"], -1, 10, 20)
    eng.keygen(99)
    orc.keygen(99)
    rng = np.random.default_rng(11)
    vals = rng.integers(0, orc.t, (4, orc.N), dtype=np.uint64)
    few = np.stack([orc.encrypt(orc.encode(vals[i]), 700 + i) for i in range(4)])
    yield eng, orc, few
    eng.close()


def _batch(few, m):
    cts = np.stack([few[i % len(few)] for i in range(m)])
    cts[1::2] = np.roll(cts[1::2], 1, axis=0)  # neighbouring ciphertexts differ
    return cts


def _profiled(eng, monkeypatch, fused, fn):
    """fused: "1" / "0" forces the fused / digit path, None leaves the choice to the library"""
    if fused is None:
        monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
    else:
        monkeypatch.setenv("CNHE_KS_FUSED", fused)
    eng.sync()
    eng.prof_enable(True)
    fn()
    prof = eng.prof_collect()
    eng.prof_enable(False)
    return prof


def _fused_against_digits(eng, monkeypatch, fn, out, words, waves=1):
    """runs fn(out) on the library's own choice, which must be the fused path with its inverse inside, then on the digit path"""
    prof = _profiled(eng, monkeypatch, None, lambda: fn(out))
    assert prof["ntt_inverse"]["launches"] == 0, prof
    assert prof["keyswitch_mac"]["launches"] == waves, prof
    got = eng.dev_download(out, words).copy()
    prof = _profiled(eng, monkeypatch, "0", lambda: fn(out))
    assert prof["ntt_inverse"]["launches"] > 0, prof
    assert np.array_equal(got, eng.dev_download(out, words)), "fused and digit paths differ"
    return got


def test_relinearize(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    sq = np.stack([orc.multiply(few[i], few[i]) for i in range(len(few))])
    cts3 = _batch(sq, M)
    a, out = eng.dev_from(cts3), eng.dev_alloc(M * 2 * k * N)
    got = _fused_against_digits(eng, monkeypatch, lambda o: eng.raw_relinearize(0, a, M, o), out, M * 2 * k * N).reshape(M, -1)
    for i in (0, M // 2, M - 1):
        assert np.array_equal(got[i], orc.relinearize(cts3[i])), i
    eng.dev_free(a)
    eng.dev_free(out)


def test_multiply_relin(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    cts = _batch(few, M)
    a, out = eng.dev_from(cts), eng.dev_alloc(M * 2 * k * N)
    got = _fused_against_digits(eng, monkeypatch, lambda o: eng.raw_multiply_relin(0, a, a, M, o), out, M * 2 * k * N).reshape(M, -1)
    for i in (0, M // 2, M - 1):
        assert np.array_equal(got[i], orc.relinearize(orc.multiply(cts[i], cts[i]))), i
    eng.dev_free(a)
    eng.dev_free(out)


def test_apply_galois(pair, monkeypatch):
    eng, orc, few = pair
    N, k = eng.N, eng.k
    cts = _batch(few, M)
    a, out = eng.dev_from(cts), eng.dev_alloc(M * 2 * k * N)
    for elt in (2 * N - 1, 3):
        got = _fused_against_digits(eng, monkeypatch, lambda o: eng.raw_apply_galois(0, a, M, elt, o), out, M * 2 * k * N).reshape(M, -1)
        for i in (0, M // 2, M - 1):
            assert np.array_equal(got[i], orc.apply_galois(cts[i], elt)), (elt, i)
    eng.dev_free(a)
    eng.dev_free(out)


def test_ragged_last_wave(pair, monkeypatch):
    """waves of 64: a relinearisation of 150 ciphertexts runs 64 + 64 + 22, all on the fused kernel"""
    eng, orc, few = pair
    N, k = eng.N, eng.k
    m = 150
    sq = np.stack([orc.multiply(few[i], few[i]) for i in range(len(few))])
    cts3 = _batch(sq, m)
    a, out = eng.dev_from(cts3), eng.dev_alloc(m * 2 * k * N)
    eng.set_option("chunk", 64)
    try:
        got = _fused_against_digits(eng, monkeypatch, lambda o: eng.raw_relinearize(0, a, m, o), out, m * 2 * k * N, waves=3).reshape(m, -1)
    finally:
        eng.set_option("chunk", 1024)
    assert np.array_equal(got[m - 1], orc.relinearize(cts3[m - 1]))
    eng.dev_free(a)
    eng.dev_free(out)


def test_in_place_relinearize_takes_the_separate_inverse(pair, monkeypatch):
    """out2 == in3: the output overlaps the target and the base, so even a forced fused call must leave the inverse to its own kernel"""
    eng, orc, few = pair
    N, k = eng.N, eng.k
    ct3 = orc.multiply(few[0], few[1])
    a = eng.dev_from(ct3)
    prof = _profiled(eng, monkeypatch, "1", lambda: eng.raw_relinearize(0, a, 1, a))
    assert prof["ntt_inverse"]["launches"] > 0, prof
    assert np.array_equal(eng.dev_download(a, 2 * k * N), orc.relinearize(ct3))
    eng.dev_free(a)


def test_row_major_product_rotate_add_in_place(monkeypatch):
    """cnhe_mat_mul_rowmajor sums the slots of all rows' products with x += rotate(x) in place: every step is a fused Galois key switch
    whose output span is the ciphertexts it rotates"""
    from cryptonets_b200.engine import DENSE, Engine
    t, N, rows = 549764251649, 8192, 64
    eng = Engine([t], N, 10, 20)
    try:
        eng.keygen(21)
        rng = np.random.default_rng(3)
        x = rng.integers(-40, 40, N // 2).astype(np.float64)
        w = rng.integers(-40, 40, (rows, N // 2)).astype(np.float64)
        v = eng.encrypt(x, 1.0, DENSE)
        plains = [eng.plain(w[r], 1.0, DENSE) for r in range(rows)]
        results = {}
        for fused in (None, "0"):
            if fused is None:
                monkeypatch.delenv("CNHE_KS_FUSED", raising=False)
            else:
                monkeypatch.setenv("CNHE_KS_FUSED", fused)
            prod = eng.mat_mul_rowmajor(plains, v)
            results[fused] = [prod.export_raw(0, b) for b in range(rows)]
            if fused is None:
                assert np.array_equal(eng.decrypt(prod), w @ x)
        for b in range(rows):
            assert np.array_equal(results[None][b], results["0"][b]), b
    finally:
        eng.close()
