"""Independent Python restatement of the compact evaluation-key format (version 1, csrc/compact.cu): header, blob order of the key pairs,
the expansion of a, and the expected key set of a seeded client composed from the CPU oracle's secret key and NTTs.  Reuses compact_ref's
ChaCha20, 128-bit draw, packing, noise sampler and seeded expansion key.  Test infrastructure: the product never imports this file."""
import struct

import numpy as np

import compact_ref as cr

PURPOSE_KEYS_A, PURPOSE_KEYS_E = 14, 15
MAGIC, VERSION = b"CNHK", 1
SET_PUBLIC, SET_RELIN = 1, 2


def header_size(k, P, G):
    return 36 + 8 * k + 40 * P + 8 * G


def standard_galois_elts(N):
    """KeyGenerator::galois_keys(dbc)'s elements: 2N-1, then 3^(2^i) and 3^-(2^i) for i < log2(N) - 1.  3 has order N/2 modulo 2N, so
    the last pair is 3^(N/4) twice (an element of order 2); distinct_galois_elts is the set a key blob can list."""
    m2 = 2 * N
    out, p3, n3 = [m2 - 1], 3, pow(3, -1, m2)
    for _ in range(N.bit_length() - 2):
        out += [p3, n3]
        p3, n3 = p3 * p3 % m2, n3 * n3 % m2
    return out


def distinct_galois_elts(N):
    return sorted(set(standard_galois_elts(N)))


def digit_map(q, w):
    """[(residue, shift)] of the base-2^w decomposition: residue-major, low bits first"""
    return [(i, s) for i, ql in enumerate(q) for s in range(0, cr.bitlen(ql), w)]


def pair_count(q, dbc_r, dbc_g, sets, G):
    return (1 if sets & SET_PUBLIC else 0) + (len(digit_map(q, dbc_r)) if sets & SET_RELIN else 0) + G * len(digit_map(q, dbc_g))


def blob_size(N, q, P, dbc_r, dbc_g, sets, G):
    return header_size(len(q), P, G) + P * pair_count(q, dbc_r, dbc_g, sets, G) * cr.packed_words_per_ct(q, N) * 8


def build_header(N, P, dbc_r, dbc_g, sets, q, t, elts, keys):
    h = MAGIC + struct.pack("<8I", VERSION, N, len(q), P, dbc_r, dbc_g, sets, len(elts))
    h += struct.pack("<%dQ" % len(q), *[int(x) for x in q]) + struct.pack("<%dQ" % P, *[int(x) for x in t])
    h += struct.pack("<%dQ" % len(elts), *[int(x) for x in elts])
    return h + b"".join(bytes(x) for x in keys)


def parse(blob):
    """-> dict(N, k, P, dbc_r, dbc_g, sets, q, t, elts, keys, payload [P][pairs][words per pair]); ValueError on a malformed blob"""
    blob = bytes(blob)
    if len(blob) < 36:
        raise ValueError("truncated header")
    if blob[:4] != MAGIC:
        raise ValueError("bad magic")
    version, N, k, P, dbc_r, dbc_g, sets, G = struct.unpack_from("<8I", blob, 4)
    if version != VERSION:
        raise ValueError("unsupported version")
    if sets & ~3:
        raise ValueError("unknown key sets")
    if len(blob) < header_size(k, P, G):
        raise ValueError("truncated header")
    o = 36
    q = list(struct.unpack_from("<%dQ" % k, blob, o))
    o += 8 * k
    t = list(struct.unpack_from("<%dQ" % P, blob, o))
    o += 8 * P
    elts = list(struct.unpack_from("<%dQ" % G, blob, o))
    o += 8 * G
    keys = [blob[o + 32 * c: o + 32 * c + 32] for c in range(P)]
    if any(b <= a for a, b in zip(elts, elts[1:])):
        raise ValueError("Galois elements must be strictly increasing")
    if any(e not in standard_galois_elts(N) for e in elts):
        raise ValueError("not a standard Galois element")
    pairs, W = pair_count(q, dbc_r, dbc_g, sets, G), cr.packed_words_per_ct(q, N)
    if len(blob) != header_size(k, P, G) + P * pairs * W * 8:
        raise ValueError("length does not match the header")
    payload = np.frombuffer(blob, dtype="<u8", offset=header_size(k, P, G)).astype(np.uint64).reshape(P, pairs, W)
    return dict(N=N, k=k, P=P, dbc_r=dbc_r, dbc_g=dbc_g, sets=sets, q=q, t=t, elts=elts, keys=keys, payload=payload)


def expand_a(key, kappa, q, N):
    """a of pair kappa [k][N]: floor(q_l R / 2^128) under stream id (PURPOSE_KEYS_A, kappa, l)"""
    out = []
    for l, ql in enumerate(q):
        w = cr.keystream_words(key, cr.stream_id(PURPOSE_KEYS_A, kappa, l), 2 * N)
        out.append(cr.draw128(ql, w[0::2], w[1::2]))
    return np.stack(out)


def _mulmod(a, b, q):
    return np.array((np.asarray(a).astype(object) * np.asarray(b).astype(object)) % q, dtype=np.uint64)


def galois_secret_ntt(orc, elt):
    """NTT(s(x^elt)) [k][N] from the oracle's secret key"""
    k, N = orc.k, orc.N
    sk = orc.secret_key().reshape(k, N)
    out = []
    idx = (np.arange(N, dtype=np.int64) * elt) % (2 * N)
    for l, ql in enumerate(orc.q):
        s = orc.ntt(l, sk[l], inverse=True).astype(object)
        perm = np.zeros(N, dtype=object)
        lo = idx < N
        perm[idx[lo]] = s[lo]
        perm[idx[~lo] - N] = (-s[~lo]) % ql
        out.append(orc.ntt(l, np.array(perm, dtype=np.uint64)))
    return np.stack(out)


def key_pairs(orc, seed, key, nonce0, kappa0, target, dm):
    """the pairs (b, a) [D][2][k][N] of one key set from pair kappa0 on: b = -(a s + NTT(e)) + 2^shift_d [target]_{src_d} (target None: the
    public key, one pair)"""
    k, N, q = orc.k, orc.N, orc.q
    sk = orc.secret_key().reshape(k, N)
    digits = [None] if target is None else dm
    out = []
    for d, dig in enumerate(digits):
        kappa = kappa0 + d
        a = expand_a(key, kappa, q, N)
        e = np.array(cr.noise(seed, cr.stream_id(PURPOSE_KEYS_E, nonce0 + kappa, 0), N), dtype=object)
        b = []
        for l, ql in enumerate(q):
            en = orc.ntt(l, np.array(e % ql, dtype=np.uint64)).astype(object)
            v = (-(_mulmod(a[l], sk[l], ql).astype(object) + en)) % ql
            if dig is not None and dig[0] == l:
                v = (v + pow(2, dig[1], ql) * target[l].astype(object)) % ql
            b.append(np.array(v, dtype=np.uint64))
        out.append(np.stack([np.stack(b), a]))
    return np.stack(out)


def expected_keys(orcs, seed, sets, elts, nonce0=1):
    """The key blob of a client seeded with `seed` (channel c uses seed + c and the oracle orcs[c]) whose next nonce is nonce0, and the key
    sets per channel: [c] -> dict(pk [2][k][N] or None, rlk [D][2][k][N] or None, glk {elt: [D][2][k][N]})"""
    o0 = orcs[0]
    N, q = o0.N, o0.q
    elts = sorted(elts)
    keys, payload, sets_out = [], [], []
    for c, orc in enumerate(orcs):
        s = seed + c
        key = cr.seeded_key(s, nonce0)
        keys.append(key)
        kappa, got = 0, dict(pk=None, rlk=None, glk={})
        pairs = []
        if sets & SET_PUBLIC:
            got["pk"] = key_pairs(orc, s, key, nonce0, kappa, None, None)[0]
            pairs.append(got["pk"][None])
            kappa += 1
        if sets & SET_RELIN:
            sk = orc.secret_key().reshape(orc.k, N)
            s2 = np.stack([_mulmod(sk[l], sk[l], ql) for l, ql in enumerate(q)])
            got["rlk"] = key_pairs(orc, s, key, nonce0, kappa, s2, digit_map(q, orc.dbc_relin))
            pairs.append(got["rlk"])
            kappa += len(got["rlk"])
        for elt in elts:
            g = key_pairs(orc, s, key, nonce0, kappa, galois_secret_ntt(orc, elt), digit_map(q, orc.dbc_galois))
            got["glk"][elt] = g
            pairs.append(g)
            kappa += len(g)
        for p in pairs:
            for pair in p:
                payload.append(cr.pack_ct_c0(pair[0], q, N))
        sets_out.append(got)
    head = build_header(N, len(orcs), o0.dbc_relin, o0.dbc_galois, sets, q, [orc.t for orc in orcs], elts, keys)
    body = np.concatenate(payload).astype("<u8").tobytes() if payload else b""
    return head + body, sets_out
