"""Independent Python restatement of sanitisation (cnhe_vecs_sanitize, DESIGN 4.18) on a seeded channel: the nonce layout, the draws of
u, e0, e1 and the multi-word flood f, and the output words, composed from compact_ref's seeded sampler and the CPU oracle's transforms and
public key.  Test infrastructure: the product never imports this file."""
import numpy as np

from compact_ref import M64, NOISE_CDF, stream_id

PURPOSE_U, PURPOSE_E0, PURPOSE_E1, PURPOSE_F = 16, 17, 18, 19
NONCES = 1 << 48


def san_stream(purpose, nonce):
    """stream id of ciphertext nonce `nonce` (< 2^48): the low 32 bits in the middle field, the high 16 in the low field"""
    assert 0 <= nonce < NONCES
    return stream_id(purpose, nonce & 0xFFFFFFFF, nonce >> 32)


# ---------------------------------------------------------------- the seeded sampler, vectorised (compact_ref.rng64 on arrays)
def _splitmix64(x):
    x = x + np.uint64(0x9E3779B97F4A7C15)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def rng64_many(seed, stream, idx):
    """compact_ref.rng64(seed, stream, i) for every i of idx (uint64 array)"""
    with np.errstate(over="ignore"):
        h = _splitmix64(np.uint64((seed ^ ((stream * 0xD1342543DE82EF95) & M64)) & M64))
        return _splitmix64(h + np.asarray(idx, np.uint64))


def ternary(r):
    """draw_ternary: floor(3 r / 2^64) - 1"""
    return np.array([((int(v) * 3) >> 64) - 1 for v in r], dtype=np.int64)


def noise(r):
    """draw_noise of every word"""
    u = r >> np.uint64(1)
    mag = np.zeros(r.shape, np.int64)
    for c in NOISE_CDF:
        mag += (u >= np.uint64(c)).astype(np.int64)
    return np.where((r & np.uint64(1)) == 1, -mag, mag)


def flood_words(b):
    """W = ceil((b + 1) / 64) words per coefficient, and the mask of the top one"""
    W = b // 64 + 1
    top = (b + 1) % 64
    return W, (1 << top) - 1 if top else M64


def flood_integers(seed, nonce, N, b):
    """f[x] = F - 2^b as Python integers, F the b + 1 low bits of the little-endian words rng64(stream(F), x W + j), j < W"""
    W, top = flood_words(b)
    w = rng64_many(seed, san_stream(PURPOSE_F, nonce), np.arange(N * W, dtype=np.uint64)).reshape(N, W)
    out = []
    for x in range(N):
        F = 0
        for j in reversed(range(W)):
            v = int(w[x, j]) & (top if j == W - 1 else M64)
            F = (F << 64) | v
        out.append(F - (1 << b))
    return out


def reduce_words(words, b, q):
    """The kernel's reduction of one coefficient's flood into q: Horner over the words (top word masked to the b + 1 bits), less 2^b"""
    W, top = flood_words(b)
    r = 0
    for j in reversed(range(W)):
        v = int(words[j]) & (top if j == W - 1 else M64)
        r = ((r << 64) | v) % q
    return (r - pow(2, b, q)) % q


def draws(seed, nonce, N, b):
    """(u, e0, e1, f) of one ciphertext: u, e0, e1 int64 arrays, f a list of Python integers"""
    x = np.arange(N, dtype=np.uint64)
    u = ternary(rng64_many(seed, san_stream(PURPOSE_U, nonce), x))
    e0 = noise(rng64_many(seed, san_stream(PURPOSE_E0, nonce), x))
    e1 = noise(rng64_many(seed, san_stream(PURPOSE_E1, nonce), x))
    return u, e0, e1, flood_integers(seed, nonce, N, b)


def sanitize(orc, seed, ct, nonce, b, pk=None):
    """Expected words of one sanitised ciphertext ([2][k][N] coefficient form) of a channel seeded with `seed`, under nonce `nonce`, flood
    width b and the public key pk ([2][k][N] NTT form; default: the oracle's)"""
    k, N, q = orc.k, orc.N, orc.q
    pk = (orc.public_key() if pk is None else np.asarray(pk, np.uint64)).reshape(2, k, N)
    ct = np.asarray(ct, np.uint64).reshape(2, k, N)
    u, e0, e1, f = draws(seed, nonce, N, b)
    out = np.zeros((2, k, N), np.uint64)
    for l, ql in enumerate(q):
        un = orc.ntt(l, np.array([int(v) % ql for v in u], np.uint64)).astype(object)
        fl = np.array([v % ql for v in f], dtype=object)
        for p in range(2):
            prod = np.array((un * pk[p, l].astype(object)) % ql, dtype=np.uint64)
            upk = orc.ntt(l, prod, inverse=True).astype(object)
            add = (e0.astype(object) + fl) if p == 0 else e1.astype(object)
            out[p, l] = np.array((ct[p, l].astype(object) + upk + add) % ql, dtype=np.uint64)
    return out


def max_bits(q, t):
    """floor(log2(q / t)) - 2, the widest flood width (q the list of coefficient primes)"""
    Q = 1
    for x in q:
        Q *= int(x)
    return (Q // int(t)).bit_length() - 1 - 2


def noise_poly(orc, ct):
    """The exact noise of a ciphertext ([2][k][N] coefficient form) under the oracle's secret key: v = c0 + c1 s mod Q by CRT, m =
    round(t v / Q) mod t, noise = v - Delta m centred mod Q (Delta = floor(Q / t)).  Returns (noise, m) as lists of Python integers."""
    q, t, N, k = [int(x) for x in orc.q], int(orc.t), orc.N, orc.k
    Q = 1
    for x in q:
        Q *= x
    ct = np.asarray(ct, np.uint64).reshape(2, k, N)
    sk = orc.secret_key().reshape(k, N)
    res = []
    for l, ql in enumerate(q):
        c1n = orc.ntt(l, ct[1, l]).astype(object)
        c1s = orc.ntt(l, np.array((c1n * sk[l].astype(object)) % ql, dtype=np.uint64), inverse=True).astype(object)
        res.append([int(v) % ql for v in (ct[0, l].astype(object) + c1s)])
    crt = [(Q // ql) * pow((Q // ql) % ql, -1, ql) for ql in q]
    delta = Q // t
    noise, msg = [], []
    for x in range(N):
        v = sum(res[l][x] * crt[l] for l in range(k)) % Q
        m = ((t * v + Q // 2) // Q) % t
        e = (v - delta * m) % Q
        if e > Q // 2:
            e -= Q
        noise.append(e)
        msg.append(m)
    return noise, msg
