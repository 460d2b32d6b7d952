"""The compact upload format's Python restatement on its own (no GPU): ChaCha20 against RFC 8439 and an independent implementation, the
128-bit draw, bit packing and header parsing."""
import struct

import numpy as np
import pytest

import compact_ref as cr


def test_chacha20_rfc8439_zero_block():
    blk = cr.chacha20_blocks(bytes(32), [0], [0])[0]
    assert blk.astype("<u4").tobytes()[:16].hex() == "76b8e0ada0f13d90405d6ae55386bd28"


def test_chacha20_matches_cryptography():
    ciphers = pytest.importorskip("cryptography.hazmat.primitives.ciphers")
    rng = np.random.default_rng(3)
    for _ in range(8):
        key = rng.bytes(32)
        counter = int(rng.integers(0, 1 << 62)) * 2 + int(rng.integers(0, 2))
        stream = int(rng.integers(0, 1 << 63))
        nonce = counter.to_bytes(8, "little") + stream.to_bytes(8, "little")
        enc = ciphers.Cipher(ciphers.algorithms.ChaCha20(key, nonce), mode=None).encryptor()
        want = enc.update(bytes(64))
        got = cr.chacha20_blocks(key, [counter], [stream])[0].astype("<u4").tobytes()
        assert got == want


def test_keystream_word_indexing():
    key = bytes(range(32))
    w = cr.keystream_words(key, 77, 40)
    for m in (0, 7, 8, 15, 39):
        blk = cr.chacha20_blocks(key, [m >> 3], [77])[0]
        assert int(w[m]) == int(blk[2 * (m & 7)]) | (int(blk[2 * (m & 7) + 1]) << 32)


def test_draw128_is_exact_and_below_q():
    rng = np.random.default_rng(4)
    for q in (1099511480321, (1 << 61) - 1, 40961, (1 << 44) - 63):
        lo = rng.integers(0, 1 << 63, 2000, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
        hi = rng.integers(0, 1 << 63, 2000, dtype=np.uint64) * np.uint64(2)
        got = cr.draw128(q, lo, hi)
        want = [(q * ((int(h) << 64) | int(l))) >> 128 for l, h in zip(lo, hi)]
        assert [int(x) for x in got] == want
        assert all(int(x) < q for x in got)
    assert int(cr.draw128(97, np.uint64(cr.M64), np.uint64(cr.M64))) == 96


@pytest.mark.parametrize("b", [36, 37, 43, 44, 48, 49, 61])
def test_pack_roundtrip(b):
    rng = np.random.default_rng(b)
    for N in (64, 4096):
        v = rng.integers(0, 1 << b, N, dtype=np.uint64)
        v[:3] = [0, (1 << b) - 1, 1]
        words = cr.pack(v, b)
        assert words.size == N * b // 64
        assert np.array_equal(cr.unpack(words, b, N), v)
        # coefficient x occupies bits [x b, (x+1) b) of the little-endian stream
        big = int.from_bytes(words.astype("<u8").tobytes(), "little")
        for x in (0, 1, N // 2, N - 1):
            assert (big >> (x * b)) & ((1 << b) - 1) == int(v[x])


def _blob(N=4096, q=(68719403009, 68719230977), t=(40961, 65537), n=2, B=1, dim=4096):
    k, P = len(q), len(t)
    keys = [bytes([c]) * 32 for c in range(P)]
    W = cr.packed_words_per_ct(q, N)
    payload = np.arange(P * n * B * W, dtype=np.uint64).astype("<u8").tobytes()
    return cr.build_header(N, k, P, n, B, dim, 2.0, q, t, keys) + payload


def test_header_roundtrip():
    blob = _blob()
    h = cr.parse(blob)
    assert (h["N"], h["k"], h["P"], h["n"], h["B"], h["dim"], h["scale"]) == (4096, 2, 2, 2, 1, 4096, 2.0)
    assert h["q"] == [68719403009, 68719230977] and h["t"] == [40961, 65537]
    assert h["keys"][1] == b"\x01" * 32
    assert len(blob) == cr.header_size(2, 2) + 2 * 2 * cr.packed_words_per_ct(h["q"], 4096) * 8
    assert h["payload"].shape == (2, 2, 4096 * 36 * 2 // 64)


def test_header_rejects_malformed():
    blob = _blob()
    with pytest.raises(ValueError, match="truncated"):
        cr.parse(blob[:40])
    with pytest.raises(ValueError, match="truncated"):
        cr.parse(blob[:cr.header_size(2, 2) - 1])
    with pytest.raises(ValueError, match="magic"):
        cr.parse(b"CNHD" + blob[4:])
    with pytest.raises(ValueError, match="version"):
        cr.parse(blob[:4] + struct.pack("<I", 2) + blob[8:])
    with pytest.raises(ValueError, match="length"):
        cr.parse(blob[:-8])
    with pytest.raises(ValueError, match="length"):
        cr.parse(blob + bytes(8))


def test_seeded_key_is_reproducible_and_distinct():
    assert cr.seeded_key(5, 1) == cr.seeded_key(5, 1)
    assert cr.seeded_key(5, 1) != cr.seeded_key(5, 2) != cr.seeded_key(6, 2)
    assert len(cr.seeded_key(5, 1)) == 32
