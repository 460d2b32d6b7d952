"""The fused key switch reads a 48-bit packed copy of the relinearisation keys, built wherever the keys come into existence.  Every
source of keys -- generated from a test seed, loaded from a saved archive, imported word by word, generated in secure mode -- must give
the same words as the digit path (which reads the u64 keys) on a fused relinearisation, and so must a context with a modulus of 2^48
or more, where no packed copy exists and the fused kernel reads the u64 keys.  Which key form the fused kernel read shows in the bytes
the library books for the key-switch family: 6 per key word packed, 8 as u64."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CT = 65  # above the fused threshold, and odd
CONFIGS = {
    "cryptonets8192": dict(plain_primes=[549764251649], N=8192),
    "default4096": dict(plain_primes=[40961], N=4096),
}


def _relin(eng, monkeypatch, cts3, fused, key_bytes=None):
    """relinearise cts3 on the fused ("1") or digit ("0") path; checks which path served the call and, on the fused path, that the
    kernel read key_bytes (6 or 8) bytes per key word"""
    m, k, N = cts3.shape[0], eng.k, eng.N
    monkeypatch.setenv("CNHE_KS_FUSED", fused)
    a, out = eng.dev_from(cts3), eng.dev_alloc(m * 2 * k * N)
    eng.sync()
    eng.prof_enable(True)
    eng.raw_relinearize(0, a, m, out)
    prof = eng.prof_collect()
    eng.prof_enable(False)
    assert (prof["ntt_forward"]["launches"] == 0) == (fused == "1"), "CNHE_KS_FUSED=%s did not select its path" % fused
    if fused == "1":
        # target residues and accumulators at 8 bytes per word, keys at key_bytes
        want = 8.0 * N * (m * k + m * 2 * k) + key_bytes * N * eng.relin_digits * 2 * k
        assert prof["keyswitch_mac"]["bytes"] == pytest.approx(want, rel=1e-9), "the fused kernel did not read %d-byte key words" % key_bytes
    got = eng.dev_download(out, m * 2 * k * N).reshape(m, -1).copy()
    eng.dev_free(a)
    eng.dev_free(out)
    return got


def _targets(eng, seed):
    """size-3 ciphertexts with canonical uniform residues: a key switch does not care whether they decrypt"""
    q = np.array(eng.q, dtype=np.uint64)
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 1 << 62, (N_CT, 3, eng.k, eng.N), dtype=np.uint64) % q[None, None, :, None]).astype(np.uint64)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_every_key_source_matches_the_digit_path(name, monkeypatch):
    from cryptonets_b200.engine import Engine
    cfg = CONFIGS[name]
    gen = Engine(cfg["plain_primes"], cfg["N"], 10, 20)
    gen.keygen(77)
    cts3 = _targets(gen, 1)
    want = _relin(gen, monkeypatch, cts3, "0")
    assert np.array_equal(_relin(gen, monkeypatch, cts3, "1", 6), want), "generated keys"
    archive, rlk = gen.save_keys(), gen.export_key(0, 2)
    gen.close()

    loaded = Engine(None, archive=archive)
    assert np.array_equal(loaded.export_key(0, 2), rlk)
    assert np.array_equal(_relin(loaded, monkeypatch, cts3, "1", 6), want), "keys loaded from an archive"
    loaded.close()

    imported = Engine(cfg["plain_primes"], cfg["N"], 10, 20)
    imported.keygen(5)  # other keys first: importing must replace the packed copy too
    imported.import_key(0, 2, rlk)
    assert np.array_equal(_relin(imported, monkeypatch, cts3, "1", 6), want), "imported keys"
    imported.close()

    secure = Engine(cfg["plain_primes"], cfg["N"], 10, 20)
    secure.keygen()
    assert np.array_equal(_relin(secure, monkeypatch, cts3, "1", 6), _relin(secure, monkeypatch, cts3, "0")), "secure-mode keys"
    secure.close()


def test_modulus_of_2_48_or_more_reads_u64_keys(monkeypatch):
    from cryptonets_b200.engine import Engine
    # 2^49 - 204799 (49 bits, 1 mod 8192): about half of its key words need more than 48 bits, so a packed copy would lose bits
    q = [562949953216513, 1099511799809]
    eng = Engine([40961], 4096, 10, 20, coeff_moduli=q)
    assert eng.q == q
    eng.keygen(3)
    rlk = eng.export_key(0, 2).reshape(eng.relin_digits, 2, eng.k, eng.N)
    assert (rlk[:, :, 0] >= 1 << 48).mean() > 0.4
    cts3 = _targets(eng, 2)
    assert np.array_equal(_relin(eng, monkeypatch, cts3, "1", 8), _relin(eng, monkeypatch, cts3, "0"))
    eng.close()
