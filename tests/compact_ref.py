"""Independent Python restatement of the compact upload format (version 1, csrc/compact.cu): ChaCha20, the 128-bit draw of c1, the bit
packing of c0 and the header -- plus the seeded noise sampler and a secret-key encryption composed from the CPU oracle's transforms,
secret key and plain addition.  Test infrastructure: the product never imports this file."""
import struct

import numpy as np

M64 = (1 << 64) - 1
PURPOSE_COMPACT_A, PURPOSE_COMPACT_E, PURPOSE_COMPACT_KEY = 11, 12, 13
MAGIC, VERSION = b"CNHC", 1


def stream_id(purpose, a, b):
    return ((purpose << 48) | (a << 16) | b) & M64


# ---------------------------------------------------------------- ChaCha20 (RFC 8439 block function, 64-bit counter and 64-bit nonce)
def _rotl(v, c):
    return (v << np.uint32(c)) | (v >> np.uint32(32 - c))


def chacha20_blocks(key, counters, streams):
    """key: 32 bytes; counters, streams: equal-length integer sequences -> uint32 [n][16] output blocks"""
    counters = np.asarray(counters, dtype=np.uint64).ravel()
    streams = np.broadcast_to(np.asarray(streams, dtype=np.uint64), counters.shape)
    kw = np.frombuffer(bytes(key), dtype="<u4").astype(np.uint32)
    n = counters.size
    s = np.zeros((16, n), np.uint32)
    s[0:4] = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], np.uint32)[:, None]
    s[4:12] = kw[:, None]
    s[12] = (counters & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    s[13] = (counters >> np.uint64(32)).astype(np.uint32)
    s[14] = (streams & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    s[15] = (streams >> np.uint64(32)).astype(np.uint32)
    x = [s[i].copy() for i in range(16)]

    def qr(a, b, c, d):
        x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 16)
        x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 12)
        x[a] += x[b]; x[d] ^= x[a]; x[d] = _rotl(x[d], 8)
        x[c] += x[d]; x[b] ^= x[c]; x[b] = _rotl(x[b], 7)

    for _ in range(10):
        qr(0, 4, 8, 12); qr(1, 5, 9, 13); qr(2, 6, 10, 14); qr(3, 7, 11, 15)
        qr(0, 5, 10, 15); qr(1, 6, 11, 12); qr(2, 7, 8, 13); qr(3, 4, 9, 14)
    return np.stack([x[i] + s[i] for i in range(16)], axis=1)


def keystream_words(key, stream, n_words):
    """64-bit keystream words w[0..n_words): word m is word m & 7 of block m >> 3"""
    blocks = chacha20_blocks(key, np.arange((n_words + 7) // 8, dtype=np.uint64), stream)
    return blocks.view("<u8").reshape(-1)[:n_words].astype(np.uint64)


# ---------------------------------------------------------------- c1 = floor(q R / 2^128), R = w[2x+1] 2^64 + w[2x]
def _umulhi(a, b):
    a, b = np.asarray(a, np.uint64), np.asarray(b, np.uint64)
    m = np.uint64(0xFFFFFFFF)
    a0, a1, b0, b1 = a & m, a >> np.uint64(32), b & m, b >> np.uint64(32)
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> np.uint64(32)) + (p01 & m) + (p10 & m)
    return p11 + (p01 >> np.uint64(32)) + (p10 >> np.uint64(32)) + (mid >> np.uint64(32))


def draw128(q, r_lo, r_hi):
    q = np.uint64(q)
    with np.errstate(over="ignore"):  # products modulo 2^64 by design
        lo, hi = q * r_hi, _umulhi(q, r_hi)
        s = lo + _umulhi(q, r_lo)
        return hi + (s < lo).astype(np.uint64)


def expand_c1(key, j, l, q, N):
    w = keystream_words(key, stream_id(PURPOSE_COMPACT_A, j, l), 2 * N)
    return draw128(q, w[0::2], w[1::2])


def expand_c1_ct(key, j, q, N):
    """c1 of ciphertext j (all residues) [k][N]"""
    return np.stack([expand_c1(key, j, l, ql, N) for l, ql in enumerate(q)])


# ---------------------------------------------------------------- bit packing
def bitlen(q):
    return int(q).bit_length()


def pack(values, b):
    """values < 2^b (len a multiple of 64) -> little-endian bit stream of len*b/64 words"""
    v = np.asarray(values, dtype=np.uint64)
    n = v.size
    assert (n * b) % 64 == 0
    out = np.zeros(n * b // 64 + 1, np.uint64)
    bit = np.arange(n, dtype=np.uint64) * np.uint64(b)
    w, s = bit >> np.uint64(6), bit & np.uint64(63)
    np.bitwise_or.at(out, w, v << s)
    spill = (s + np.uint64(b)) > np.uint64(64)
    np.bitwise_or.at(out, w[spill] + np.uint64(1), v[spill] >> (np.uint64(64) - s[spill]))
    return out[:-1]


def unpack(words, b, n):
    """inverse of pack: n values of b bits"""
    wd = np.concatenate([np.asarray(words, dtype=np.uint64), np.zeros(1, np.uint64)])
    bit = np.arange(n, dtype=np.uint64) * np.uint64(b)
    w, s = bit >> np.uint64(6), bit & np.uint64(63)
    v = wd[w] >> s
    hi = np.where(s > 0, wd[w + np.uint64(1)] << ((np.uint64(64) - s) & np.uint64(63)), np.uint64(0))
    v = v | np.where((s + np.uint64(b)) > np.uint64(64), hi, np.uint64(0))
    mask = np.uint64(M64 if b == 64 else (1 << b) - 1)
    return v & mask


def packed_words_per_ct(q, N):
    return sum(N * bitlen(x) // 64 for x in q)


def pack_ct_c0(c0, q, N):
    """c0 [k][N] -> packed words of one ciphertext"""
    return np.concatenate([pack(c0[l], bitlen(ql)) for l, ql in enumerate(q)])


def unpack_ct_c0(words, q, N):
    out, off = [], 0
    for ql in q:
        nw = N * bitlen(ql) // 64
        out.append(unpack(words[off:off + nw], bitlen(ql), N))
        off += nw
    return np.stack(out)


# ---------------------------------------------------------------- header
def header_size(k, P):
    return 44 + 8 * k + 40 * P


def build_header(N, k, P, n, B, dim, scale, q, t, keys):
    h = MAGIC + struct.pack("<6I", VERSION, N, k, P, n, B) + struct.pack("<Qd", dim, scale)
    h += struct.pack("<%dQ" % k, *[int(x) for x in q]) + struct.pack("<%dQ" % P, *[int(x) for x in t])
    return h + b"".join(bytes(x) for x in keys)


def parse(blob):
    """-> dict(N, k, P, n, B, dim, scale, q, t, keys, payload [P][n*B][words per ct]); ValueError on a malformed blob"""
    blob = bytes(blob)
    if len(blob) < 44:
        raise ValueError("truncated header")
    if blob[:4] != MAGIC:
        raise ValueError("bad magic")
    version, N, k, P, n, B = struct.unpack_from("<6I", blob, 4)
    if version != VERSION:
        raise ValueError("unsupported version")
    if len(blob) < header_size(k, P):
        raise ValueError("truncated header")
    dim, scale = struct.unpack_from("<Qd", blob, 28)
    q = list(struct.unpack_from("<%dQ" % k, blob, 44))
    t = list(struct.unpack_from("<%dQ" % P, blob, 44 + 8 * k))
    o = 44 + 8 * k + 8 * P
    keys = [blob[o + 32 * c: o + 32 * c + 32] for c in range(P)]
    W = packed_words_per_ct(q, N)
    if len(blob) != header_size(k, P) + P * n * B * W * 8:
        raise ValueError("length does not match the header")
    payload = np.frombuffer(blob, dtype="<u8", offset=header_size(k, P)).astype(np.uint64).reshape(P, n * B, W)
    return dict(N=N, k=k, P=P, n=n, B=B, dim=dim, scale=scale, q=q, t=t, keys=keys, payload=payload)


def expand(hdr, channel):
    """the ordinary ciphertexts [n*B][2][k][N] of one channel of a parsed blob: unpacked (canonicalised) c0 and expanded c1"""
    N, q = hdr["N"], hdr["q"]
    qa = np.array(q, dtype=np.uint64)[:, None]
    out = []
    for j in range(hdr["n"] * hdr["B"]):
        c0 = unpack_ct_c0(hdr["payload"][channel, j], q, N)
        c0 = np.where(c0 >= qa, c0 - qa, c0)
        out.append(np.stack([c0, expand_c1_ct(hdr["keys"][channel], j, q, N)]))
    return np.stack(out)


# ---------------------------------------------------------------- seeded sampler (the deterministic test mode shared with the oracle)
def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def rng64(seed, stream, i):
    return splitmix64((splitmix64(seed ^ ((stream * 0xD1342543DE82EF95) & M64)) + i) & M64)


NOISE_CDF = [0xff141e3023416d2, 0x2e4f850f76b8d9a6, 0x488c5acec8fd6db3, 0x5d1ca569fc3e4ccb, 0x6bbb5699bdd65b9c, 0x75291bf8371e7ecc,
             0x7aad3cf138611a69, 0x7d9aa4d4ab7c76bd, 0x7f0368341f79807c, 0x7fa0f21e3a554470, 0x7fdf5971c6494be2, 0x7ff5c5a33f74a4e1,
             0x7ffd148ddcc40605, 0x7fff3db0052c58c3, 0x7fffd206471c7fcf, 0x7ffff61ba7b56e58, 0x7ffffe11d76ecb8a, 0x7fffffa9c1e61510,
             0x7ffffff3ceaa701f]


def noise(seed, stream, N):
    out = []
    for x in range(N):
        r = rng64(seed, stream, x)
        u = r >> 1
        mag = sum(1 for c in NOISE_CDF if u >= c)
        out.append(-mag if r & 1 else mag)
    return out


def seeded_key(seed, nonce0):
    """K_c of a blob made by a channel seeded with `seed` (cnhe_keys_generate(seed) gives channel c the seed + c)"""
    return b"".join(struct.pack("<Q", rng64(seed, stream_id(PURPOSE_COMPACT_KEY, nonce0, 0), i)) for i in range(4))


def encrypt_symmetric(orc, seed, plain, nonce, a):
    """(-(a s) + e + Delta m, a) with the oracle's secret key (seeded `seed`), e from stream (PURPOSE_COMPACT_E, nonce), a [k][N] given"""
    k, N = orc.k, orc.N
    sk = orc.secret_key().reshape(k, N)
    e = noise(seed, stream_id(PURPOSE_COMPACT_E, nonce, 0), N)
    c0 = []
    for l, ql in enumerate(orc.q):
        an = orc.ntt(l, a[l]).astype(object)
        prod = np.array((an * sk[l].astype(object)) % ql, dtype=np.uint64)
        asl = orc.ntt(l, prod, inverse=True).astype(object)
        c0.append(np.array([(-int(v) + ev) % ql for v, ev in zip(asl, e)], dtype=np.uint64))
    ct = np.concatenate([np.stack(c0).ravel(), np.asarray(a, np.uint64).ravel()])
    return orc.add_plain(ct, plain)
