"""The fused key switch and the fused BEHZ square read the twiddles of their unit-stride stages (the last four forward stages of each
half, the first four inverse stages) from the per-thread grouped tables NttTab::wd_split_grp / iwd_split_grp, and hand work from one
pass to the next with warp barriers where producer and consumer are the same half warp.  At N = 4096 and 8192: the fused key switch
against the digit path for relinearisation (packed keys) and Galois automorphisms (u64 keys), the fused square against the separate
kernels (CNHE_MUL_FUSED=0), all bit for bit on every ciphertext, and the CPU oracle on the first, middle and last ciphertext."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

CONFIGS = {
    "default4096": dict(t=40961, N=4096),
    "cryptonets8192": dict(t=549764251649, N=8192),
}
M = 65  # above the fused key switch's threshold, and odd


@pytest.fixture(scope="module", params=list(CONFIGS))
def pair(request):
    from cryptonets_b200.engine import Engine
    from oracle.oracle_py import Oracle
    cfg = CONFIGS[request.param]
    os.environ.pop("CNHE_KS_FUSED", None)
    os.environ.pop("CNHE_MUL_FUSED", None)
    eng = Engine([cfg["t"]], cfg["N"], 10, 20, -1)
    orc = Oracle(cfg["t"], cfg["N"], -1, 10, 20)
    eng.keygen(4321)
    orc.keygen(4321)
    rng = np.random.default_rng(11)
    vals = rng.integers(0, orc.t, (5, orc.N), dtype=np.uint64)
    few = np.stack([orc.encrypt(orc.encode(vals[i]), 7000 + i) for i in range(5)])
    cts = np.stack([few[i % len(few)] for i in range(M)])
    cts[1::2] = np.roll(cts[1::2], 1, axis=0)  # neighbouring ciphertexts differ
    yield eng, orc, cts
    eng.close()


SAMPLES = (0, M // 2, M - 1)


def _run(eng, monkeypatch, var, value, fn, words):
    """fn(out) with var set to value; checks nothing about the path, returns the downloaded output"""
    monkeypatch.setenv(var, value)
    out = eng.dev_alloc(words)
    eng.sync()
    eng.prof_enable(True)
    fn(out)
    prof = eng.prof_collect()
    eng.prof_enable(False)
    got = eng.dev_download(out, words).copy()
    eng.dev_free(out)
    return got, prof


def test_key_switch_relinearize_packed_keys(pair, monkeypatch):
    eng, orc, cts = pair
    N, k = eng.N, eng.k
    cts3 = np.stack([orc.multiply(c, c) for c in cts[:5]])
    cts3 = np.stack([cts3[i % 5] for i in range(M)])
    cts3[1::2] = np.roll(cts3[1::2], 1, axis=0)
    a = eng.dev_from(cts3)
    words = M * 2 * k * N
    fused, prof = _run(eng, monkeypatch, "CNHE_KS_FUSED", "1", lambda o: eng.raw_relinearize(0, a, M, o), words)
    assert prof["ntt_forward"]["launches"] == 0, "the fused key switch did not serve the call"
    want = 8.0 * N * (M * k + M * 2 * k) + 6.0 * N * eng.relin_digits * 2 * k  # 6 bytes per key word: the packed copy
    assert prof["keyswitch_mac"]["bytes"] == pytest.approx(want, rel=1e-9)
    digits, _ = _run(eng, monkeypatch, "CNHE_KS_FUSED", "0", lambda o: eng.raw_relinearize(0, a, M, o), words)
    eng.dev_free(a)
    fused, digits = fused.reshape(M, -1), digits.reshape(M, -1)
    assert np.array_equal(fused, digits)
    for i in SAMPLES:
        assert np.array_equal(fused[i], orc.relinearize(cts3[i])), i


@pytest.mark.parametrize("elt_of_n", [lambda n: 2 * n - 1, lambda n: 3], ids=["conjugate", "elt3"])
def test_key_switch_galois_u64_keys(pair, monkeypatch, elt_of_n):
    eng, orc, cts = pair
    N, k = eng.N, eng.k
    elt = elt_of_n(N)
    a = eng.dev_from(cts)
    words = M * 2 * k * N
    fused, prof = _run(eng, monkeypatch, "CNHE_KS_FUSED", "1", lambda o: eng.raw_apply_galois(0, a, M, elt, o), words)
    assert prof["ntt_forward"]["launches"] == 0, "the fused key switch did not serve the call"
    digits, _ = _run(eng, monkeypatch, "CNHE_KS_FUSED", "0", lambda o: eng.raw_apply_galois(0, a, M, elt, o), words)
    eng.dev_free(a)
    fused, digits = fused.reshape(M, -1), digits.reshape(M, -1)
    assert np.array_equal(fused, digits), elt
    for i in SAMPLES:
        assert np.array_equal(fused[i], orc.apply_galois(cts[i], elt)), (elt, i)


def test_fused_square_every_residue(pair, monkeypatch):
    eng, orc, cts = pair
    N, k = eng.N, eng.k
    a = eng.dev_from(cts)
    words = M * 3 * k * N
    fused, prof = _run(eng, monkeypatch, "CNHE_MUL_FUSED", "1", lambda o: eng.raw_multiply(0, a, a, M, o), words)
    assert prof["ntt_forward"]["launches"] > 0 and prof["ntt_inverse"]["launches"] == 0, "the fused square did not serve the call"
    separate, prof = _run(eng, monkeypatch, "CNHE_MUL_FUSED", "0", lambda o: eng.raw_multiply(0, a, a, M, o), words)
    assert prof["ntt_inverse"]["launches"] > 0
    eng.dev_free(a)
    fused, separate = fused.reshape(M, 3, k, N), separate.reshape(M, 3, k, N)
    # the fused kernel runs one CTA pair per residue of q u Bsk; the floor folds the Bsk residues into every q residue of the output
    for l in range(k):
        assert np.array_equal(fused[:, :, l], separate[:, :, l]), l
    for i in SAMPLES:
        assert np.array_equal(fused[i].reshape(-1), orc.multiply(cts[i], cts[i]).reshape(-1)), i
