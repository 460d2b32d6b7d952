"""The compact evaluation-key format's Python restatement on its own (no GPU): header round trip, payload sizes of the three served
parameter sets, and rejection of malformed headers."""
import struct

import numpy as np
import pytest

import compact_keys_ref as kr
import compact_ref as cr

# (N, plaintext moduli, SmallModulusCount, dbc_relin, dbc_galois) -> MB: compact payload with every key, compact payload of what the
# network needs (CryptoNets: pk + relin only; LoLa: up to every element), and the key words of the archive.  "Every element" is the
# distinct standard elements: logN - 2 of them besides 2N-1 come in inverse pairs, and 3^(N/4) is its own inverse (24 at N = 8192).
SETS = {
    "cryptonets_mnist": ((8192, [549764251649, 549764284417], -1, 10, 20), 172.3, 11.6, 505.9),
    "lola_small": ((8192, [2277377, 2424833], 3, 40, 40), 40.2, 40.2, 118.8),
    "lola_cifar": ((16384, [957181001729, 957181034497], 8, 60, 60), 345.8, 345.8, 910.2),
}


def _q(N, count):
    from oracle.oracle_py import Oracle
    return Oracle(65537, N, count).q


def test_standard_elements():
    N = 8192
    e = kr.standard_galois_elts(N)
    assert len(e) == 25 and e[0] == 2 * N - 1
    for i in range(12):
        assert e[1 + 2 * i] == pow(3, 2 ** i, 2 * N) and e[2 + 2 * i] * pow(3, 2 ** i, 2 * N) % (2 * N) == 1
    assert e[-1] == e[-2] == pow(3, N // 4, 2 * N) and pow(e[-1], 2, 2 * N) == 1
    assert kr.distinct_galois_elts(N) == sorted(set(e)) and len(kr.distinct_galois_elts(N)) == 24


@pytest.mark.parametrize("name", list(SETS))
def test_payload_sizes(name):
    (N, t, count, dr, dg), every_mb, needed_mb, archive_mb = SETS[name]
    q = _q(N, count)
    k, P, G = len(q), len(t), len(kr.distinct_galois_elts(N))
    both = kr.SET_PUBLIC | kr.SET_RELIN
    payload = lambda sets, g: kr.blob_size(N, q, P, dr, dg, sets, g) - kr.header_size(k, P, g)
    assert round(payload(both, G) / 1e6, 1) == every_mb
    need = payload(both, 0) if name == "cryptonets_mnist" else payload(both, G)
    assert round(need / 1e6, 1) == needed_mb
    # the archive holds every key word as a u64: pk + relin digits + every Galois element's digits
    D_r, D_g = len(kr.digit_map(q, dr)), len(kr.digit_map(q, dg))
    assert round(P * (1 + D_r + G * D_g) * 2 * k * N * 8 / 1e6, 1) == archive_mb
    assert 2.6 < P * (1 + D_r + G * D_g) * 2 * k * N * 8 / payload(both, G) < 3.0


def _blob(N=4096, q=(68719403009, 68719230977), t=(40961, 65537), sets=3, elts=(3, 8191)):
    P = len(t)
    keys = [bytes([7 + c]) * 32 for c in range(P)]
    pairs = kr.pair_count(list(q), 10, 20, sets, len(elts))
    W = cr.packed_words_per_ct(q, N)
    payload = np.arange(P * pairs * W, dtype=np.uint64).astype("<u8").tobytes()
    return kr.build_header(N, P, 10, 20, sets, q, t, list(elts), keys) + payload


def test_header_roundtrip():
    blob = _blob()
    h = kr.parse(blob)
    assert (h["N"], h["k"], h["P"], h["dbc_r"], h["dbc_g"], h["sets"]) == (4096, 2, 2, 10, 20, 3)
    assert h["q"] == [68719403009, 68719230977] and h["t"] == [40961, 65537] and h["elts"] == [3, 8191]
    assert h["keys"] == [b"\x07" * 32, b"\x08" * 32]
    pairs = 1 + 8 + 2 * 4  # pk, 2 x 4 relin digits of 36-bit moduli at w = 10, 2 elements x 2 x 2 digits at w = 20
    assert h["payload"].shape == (2, pairs, 4096 * 36 * 2 // 64)
    assert len(blob) == kr.header_size(2, 2, 2) + 2 * pairs * 4096 * 36 * 2 // 64 * 8


def test_header_rejects_malformed():
    blob = _blob()
    put = lambda off, fmt, v: blob[:off] + struct.pack(fmt, v) + blob[off + struct.calcsize(fmt):]
    with pytest.raises(ValueError, match="truncated"):
        kr.parse(blob[:30])
    with pytest.raises(ValueError, match="truncated"):
        kr.parse(blob[:kr.header_size(2, 2, 2) - 1])
    with pytest.raises(ValueError, match="magic"):
        kr.parse(b"CNHC" + blob[4:])
    with pytest.raises(ValueError, match="version"):
        kr.parse(put(4, "<I", 2))
    with pytest.raises(ValueError, match="length"):
        kr.parse(blob[:-8])
    with pytest.raises(ValueError, match="length"):
        kr.parse(blob + bytes(8))
    with pytest.raises(ValueError, match="unknown key sets"):
        kr.parse(put(28, "<I", 7))
    elts_off = 36 + 8 * 2 + 8 * 2
    with pytest.raises(ValueError, match="increasing"):
        kr.parse(put(elts_off + 8, "<Q", 3))  # duplicate
    with pytest.raises(ValueError, match="increasing"):
        kr.parse(put(elts_off, "<Q", 8191)[:elts_off + 8] + struct.pack("<Q", 3) + blob[elts_off + 16:])  # unsorted
    with pytest.raises(ValueError, match="standard"):
        kr.parse(put(elts_off, "<Q", 5))
