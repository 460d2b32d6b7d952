/*
 * oracle/bfv_oracle.cpp -- CPU restatement of the SEAL 3.2 BFV hot path used by microsoft/CryptoNets.
 *
 * TEST INFRASTRUCTURE ONLY (see bfv_oracle.h).  PARITY WITH THE REAL SEAL 3.2 BINARY IS UNPINNED:
 * SEAL is an un-vendored NuGet dependency of the reference ("HE Wrapper/packages.config:5",
 * Microsoft.Research.SEALNet 3.2.0, built from microsoft/SEAL tag 3.2.2) and is absent from
 * /root/reference.  Every routine below names the SEAL 3.2 routine it restates and the reference call
 * site (file:line under /root/reference) that makes it part of the hot path.
 *
 * Arithmetic: 64-bit words, unsigned __int128 products, Barrett reduction with floor(2^128/p)
 * (SEAL util/uintarithsmallmod.h barrett_reduce_128), Harvey NTT butterflies with Shoup quotients
 * (SEAL util/smallntt.cpp).  No SIMD intrinsics (SEAL 3.2 has none).
 */
#include "bfv_oracle.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <vector>

typedef uint64_t u64;
typedef unsigned __int128 u128;

static thread_local std::string g_err;
static int fail(const char *msg) { g_err = msg; return -1; }
extern "C" const char *orc_last_error(void) { return g_err.c_str(); }

/* ------------------------------------------------------------------ SmallModulus */
struct Mod {
    u64 p = 0, r0 = 0, r1 = 0; /* floor(2^128/p) = r1:r0  (SEAL SmallModulus::const_ratio) */
    int bits = 0;
};
static Mod make_mod(u64 p) {
    Mod m;
    m.p = p;
    u128 r = (~(u128)0) / p; /* p odd > 1 => floor((2^128-1)/p) == floor(2^128/p) */
    m.r0 = (u64)r;
    m.r1 = (u64)(r >> 64);
    m.bits = 64 - __builtin_clzll(p);
    return m;
}
/* SEAL util::barrett_reduce_128 */
static inline u64 barrett128(u128 x, const Mod &m) {
    u64 lo = (u64)x, hi = (u64)(x >> 64);
    u128 a = ((u128)lo * m.r0) >> 64;
    u128 b = (u128)lo * m.r1;
    u128 c = (u128)hi * m.r0;
    u128 mid = a + (u64)b + (u64)c;
    u64 q = hi * m.r1 + (u64)(b >> 64) + (u64)(c >> 64) + (u64)(mid >> 64);
    u64 r = lo - q * m.p;
    return r >= m.p ? r - m.p : r;
}
static inline u64 mulmod(u64 a, u64 b, const Mod &m) { return barrett128((u128)a * b, m); }
static inline u64 addmod(u64 a, u64 b, const Mod &m) { u64 s = a + b; return s >= m.p ? s - m.p : s; }
static inline u64 submod(u64 a, u64 b, const Mod &m) { return a >= b ? a - b : a + m.p - b; }
static inline u64 negmod(u64 a, const Mod &m) { return a ? m.p - a : 0; }
static u64 powmod(u64 a, u64 e, const Mod &m) {
    u64 r = 1 % m.p;
    a %= m.p;
    while (e) {
        if (e & 1) r = mulmod(r, a, m);
        a = mulmod(a, a, m);
        e >>= 1;
    }
    return r;
}
static u64 invmod(u64 a, const Mod &m) { return powmod(a, m.p - 2, m); } /* p prime */

static bool is_prime(u64 n) {
    if (n < 2) return false;
    for (u64 p : {2ULL, 3ULL, 5ULL, 7ULL, 11ULL, 13ULL, 17ULL, 19ULL, 23ULL, 29ULL, 31ULL, 37ULL}) {
        if (n % p == 0) return n == p;
    }
    Mod m = make_mod(n);
    u64 d = n - 1;
    int s = 0;
    while ((d & 1) == 0) { d >>= 1; s++; }
    for (u64 a : {2ULL, 3ULL, 5ULL, 7ULL, 11ULL, 13ULL, 17ULL, 19ULL, 23ULL, 29ULL, 31ULL, 37ULL}) {
        u64 x = powmod(a, d, m);
        if (x == 1 || x == n - 1) continue;
        bool comp = true;
        for (int i = 1; i < s; i++) {
            x = mulmod(x, x, m);
            if (x == n - 1) { comp = false; break; }
        }
        if (comp) return false;
    }
    return true;
}

static inline u64 bitrev(u64 x, int bits) {
    u64 r = 0;
    for (int i = 0; i < bits; i++) { r = (r << 1) | (x & 1); x >>= 1; }
    return r;
}

/* SEAL util::try_minimal_primitive_root: the smallest primitive `degree`-th root of unity mod p */
extern "C" u64 orc_minimal_primitive_root(u64 degree, u64 p) {
    Mod m = make_mod(p);
    if ((p - 1) % degree) return 0;
    u64 e = (p - 1) / degree, g = 0;
    for (u64 x = 2; x < p; x++) {
        u64 c = powmod(x, e, m);
        if (powmod(c, degree / 2, m) == p - 1) { g = c; break; }
    }
    u64 gsq = mulmod(g, g, m), cur = g, best = g;
    for (u64 i = 0; i < degree / 2; i++) { /* all odd powers */
        if (cur < best) best = cur;
        cur = mulmod(cur, gsq, m);
    }
    return best;
}

/* ------------------------------------------------------------------ SmallNTTTables */
struct NttTables {
    Mod m;
    int logn = 0;
    u64 n = 0, root = 0;
    std::vector<u64> w, ws, iw, iws; /* psi^bitrev(i), floor(w*2^64/p), psi^-bitrev(i), scaled */
    u64 inv_n = 0, inv_n_s = 0;
};
static inline u64 shoup(u64 w, u64 p) { return (u64)(((u128)w << 64) / p); }
static void build_ntt(NttTables &T, u64 p, int logn) {
    T.m = make_mod(p);
    T.logn = logn;
    T.n = 1ULL << logn;
    T.root = orc_minimal_primitive_root(2 * T.n, p);
    u64 iroot = invmod(T.root, T.m);
    T.w.assign(T.n, 0); T.ws.assign(T.n, 0); T.iw.assign(T.n, 0); T.iws.assign(T.n, 0);
    u64 pw = 1, ipw = 1;
    for (u64 i = 0; i < T.n; i++) { /* SEAL ntt_powers_of_primitive_root: dest[reverse_bits(i)] = root^i */
        u64 r = bitrev(i, logn);
        T.w[r] = pw; T.ws[r] = shoup(pw, p);
        T.iw[r] = ipw; T.iws[r] = shoup(ipw, p);
        pw = mulmod(pw, T.root, T.m);
        ipw = mulmod(ipw, iroot, T.m);
    }
    T.inv_n = invmod(T.n % p, T.m);
    T.inv_n_s = shoup(T.inv_n, p);
}
/* SEAL util::ntt_negacyclic_harvey: Cooley-Tukey, natural in, bit-reversed out; lazy [0,4p) inside,
 * canonical [0,p) on exit (the lazy variant's leftovers never reach a ciphertext boundary). */
static void ntt_fwd(u64 *x, const NttTables &T) {
    const u64 p = T.m.p, two_p = 2 * p;
    u64 n = T.n, t = n >> 1;
    for (u64 m = 1; m < n; m <<= 1, t >>= 1) {
        for (u64 i = 0; i < m; i++) {
            const u64 W = T.w[m + i], Ws = T.ws[m + i];
            u64 *X = x + 2 * i * t, *Y = X + t;
            for (u64 j = 0; j < t; j++) {
                u64 a = X[j];
                a -= (a >= two_p) ? two_p : 0;
                u64 Q = (u64)(((u128)Ws * Y[j]) >> 64);
                u64 Tm = W * Y[j] - Q * p;
                X[j] = a + Tm;
                Y[j] = a - Tm + two_p;
            }
        }
    }
    for (u64 i = 0; i < n; i++) {
        u64 v = x[i];
        v -= (v >= two_p) ? two_p : 0;
        v -= (v >= p) ? p : 0;
        x[i] = v;
    }
}
/* SEAL util::inverse_ntt_negacyclic_harvey: Gentleman-Sande, bit-reversed in, natural out, times N^-1 */
static void ntt_inv(u64 *x, const NttTables &T) {
    const u64 p = T.m.p, two_p = 2 * p;
    u64 n = T.n, t = 1;
    for (u64 m = n; m > 1; m >>= 1, t <<= 1) {
        u64 h = m >> 1;
        for (u64 i = 0; i < h; i++) {
            const u64 W = T.iw[h + i], Ws = T.iws[h + i];
            u64 *X = x + 2 * i * t, *Y = X + t;
            for (u64 j = 0; j < t; j++) {
                u64 u = X[j], v = Y[j];
                u64 s = u + v;
                s -= (s >= two_p) ? two_p : 0;
                u64 d = u - v + two_p;
                u64 Q = (u64)(((u128)Ws * d) >> 64);
                X[j] = s;
                Y[j] = W * d - Q * p;
            }
        }
    }
    for (u64 i = 0; i < n; i++) {
        u64 v = x[i];
        u64 Q = (u64)(((u128)T.inv_n_s * v) >> 64);
        v = T.inv_n * v - Q * p;
        v -= (v >= p) ? p : 0;
        x[i] = v;
    }
}

/* ------------------------------------------------------------------ deterministic sampler
 * SEAL draws from std::random_device-seeded generators, which nobody can reproduce; the oracle and the
 * product share this counter-based sampler instead so that keys and fresh ciphertexts are comparable
 * bit for bit (DESIGN.md "sampler").  rng(seed, stream, i) = splitmix64(splitmix64(seed ^ stream*C) + i). */
static inline u64 splitmix(u64 x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
static inline u64 rng64(u64 seed, u64 stream, u64 i) { return splitmix(splitmix(seed ^ (stream * 0xD1342543DE82EF95ULL)) + i); }
static inline u64 stream_id(u64 purpose, u64 a, u64 b) { return (purpose << 48) | (a << 16) | b; }
enum { S_SK = 1, S_PK_A = 2, S_PK_E = 3, S_RLK_A = 4, S_RLK_E = 5, S_GLK_A = 6, S_GLK_E = 7, S_ENC_U = 8, S_ENC_E0 = 9, S_ENC_E1 = 10 };
/* P(|e| <= j) * 2^63 for e = round(N(0, 3.19^2)) conditioned on |e| <= 19 (SEAL: sigma 3.19, max deviation 6 sigma) */
static const u64 NOISE_CDF[19] = {
    0xff141e3023416d2ULL, 0x2e4f850f76b8d9a6ULL, 0x488c5acec8fd6db3ULL, 0x5d1ca569fc3e4ccbULL, 0x6bbb5699bdd65b9cULL,
    0x75291bf8371e7eccULL, 0x7aad3cf138611a69ULL, 0x7d9aa4d4ab7c76bdULL, 0x7f0368341f79807cULL, 0x7fa0f21e3a554470ULL,
    0x7fdf5971c6494be2ULL, 0x7ff5c5a33f74a4e1ULL, 0x7ffd148ddcc40605ULL, 0x7fff3db0052c58c3ULL, 0x7fffd206471c7fcfULL,
    0x7ffff61ba7b56e58ULL, 0x7ffffe11d76ecb8aULL, 0x7fffffa9c1e61510ULL, 0x7ffffff3ceaa701fULL};
static inline int sample_ternary(u64 r) { return (int)(((u128)r * 3) >> 64) - 1; }
static inline int sample_noise(u64 r) {
    u64 u = r >> 1;
    int mag = 0;
    for (int j = 0; j < 19; j++) mag += (u >= NOISE_CDF[j]);
    return (r & 1) ? -mag : mag;
}
static inline u64 sample_uniform(u64 r, u64 p) { return (u64)(((u128)r * p) >> 64); }
static inline u64 lift_small(int v, u64 p) { return v >= 0 ? (u64)v : p - (u64)(-v); }

/* ------------------------------------------------------------------ context */
static const u64 M_SK = 0x1fffffffffe00001ULL, GAMMA = 0x1fffffffffc80001ULL; /* SEAL util/globals.cpp small_mods */
static const u64 M_TILDE = 1ULL << 32;

struct KSKey { std::vector<u64> data; int count = 0; }; /* [count][2][k][N], NTT form */

struct orc_ctx {
    u64 t = 0;
    uint32_t N = 0;
    int logN = 0, k = 0, dbc_relin = 0, dbc_galois = 0;
    int centered_mtilde = 0;
    std::vector<Mod> q;       /* k */
    std::vector<Mod> bsk;     /* k+1 : aux base B then m_sk */
    Mod tmod, gmod;
    std::vector<NttTables> ntt_q, ntt_bsk;
    NttTables ntt_t;
    std::vector<u64> index_map; /* BatchEncoder::matrix_reps_index_map_ */
    /* encryption constants */
    std::vector<u64> delta;      /* floor(q/t) mod q_i     (coeff_div_plain_modulus) */
    std::vector<u64> q_mod_t_q;  /* (q mod t) mod q_i      (upper_half_increment) */
    u64 upper_half_threshold = 0;
    /* BEHZ constants (SEAL util/baseconverter.cpp BaseConverter::generate) */
    std::vector<u64> inv_qhat_mod_q, mtilde_inv_qhat_mod_q, qhat_mod_mtilde;
    std::vector<std::vector<u64>> qhat_mod_bsk; /* [j][i] */
    std::vector<u64> inv_mtilde_mod_bsk, q_mod_bsk, inv_q_mod_bsk;
    u64 inv_q_mod_mtilde = 0; /* q^-1 mod 2^32 */
    std::vector<u64> inv_bhat_mod_b;            /* [j<k] */
    std::vector<std::vector<u64>> bhat_mod_q;   /* [i][j] */
    std::vector<u64> bhat_mod_msk, B_mod_q;
    u64 inv_B_mod_msk = 0;
    /* decrypt */
    std::vector<u64> tgamma_mod_q, qhat_mod_t, qhat_mod_gamma;
    u64 neg_inv_q_mod_t = 0, neg_inv_q_mod_gamma = 0, inv_gamma_mod_t = 0;
    /* keys */
    bool have_keys = false;
    const char *refuse_decrypt = nullptr, *refuse_behz = nullptr; /* q holds gamma / a Bsk prime (build_ctx) */
    std::vector<u64> sk_ntt, sk_coeff, pk; /* sk_coeff: k*N lifted ternary */
    KSKey rlk;
    std::vector<u64> galois_elts;
    std::map<u64, KSKey> glk;
    u64 seed = 0;
};

static std::vector<u64> default_coeff_modulus(uint32_t N) {
    /* SEAL 3.2 DefaultParams.CoeffModulus128(N) (util/globals.cpp default_coeff_modulus_128) */
    switch (N) {
    case 2048: return {0x3fffffff000001ULL};
    case 4096: return {0xffffee001ULL, 0xffffc4001ULL, 0x1ffffe0001ULL};
    case 8192: return {0x7fffffd8001ULL, 0x7fffffc8001ULL, 0xfffffffc001ULL, 0xffffff6c001ULL, 0xfffffebc001ULL};
    case 16384: return {0xfffffffd8001ULL, 0xfffffffa0001ULL, 0xfffffff00001ULL, 0x1fffffff68001ULL, 0x1fffffff50001ULL,
                        0x1ffffffee8001ULL, 0x1ffffffea0001ULL, 0x1ffffffe88001ULL, 0x1ffffffe48001ULL};
    default: return {};
    }
}
/* SEAL small_mods aux_small_mods: 61-bit primes = 1 mod 2^18, descending, after m_sk and gamma */
static std::vector<u64> aux_primes(int count) {
    std::vector<u64> out;
    u64 c = (1ULL << 61) + 1;
    int seen = 0;
    while ((int)out.size() < count) {
        c -= (1ULL << 18);
        if (!is_prime(c)) continue;
        if (seen++ < 2) continue; /* the first two are m_sk and gamma */
        out.push_back(c);
    }
    return out;
}

static u64 prod_mod_except(const std::vector<Mod> &base, int except, const Mod &m) {
    u64 r = 1 % m.p;
    for (int i = 0; i < (int)base.size(); i++)
        if (i != except) r = mulmod(r, base[i].p % m.p, m);
    return r;
}
static u64 inv_mod_pow2_32(u64 a) { /* a odd */
    u64 x = a;                      /* Newton: x <- x(2 - a x) */
    for (int i = 0; i < 6; i++) x *= 2 - a * x;
    return x & 0xffffffffULL;
}

/* multi-precision helpers on little-endian limb vectors (only for floor(q/t), q mod t and noise budget) */
typedef std::vector<u64> Big;
static Big big_mul_small(const Big &a, u64 b) {
    Big r(a.size() + 1, 0);
    u64 carry = 0;
    for (size_t i = 0; i < a.size(); i++) {
        u128 v = (u128)a[i] * b + carry;
        r[i] = (u64)v;
        carry = (u64)(v >> 64);
    }
    r[a.size()] = carry;
    while (r.size() > 1 && r.back() == 0) r.pop_back();
    return r;
}
static Big big_divmod_small(const Big &a, u64 b, u64 &rem) {
    Big q(a.size(), 0);
    u128 r = 0;
    for (size_t i = a.size(); i-- > 0;) {
        u128 cur = (r << 64) | a[i];
        q[i] = (u64)(cur / b);
        r = cur % b;
    }
    rem = (u64)r;
    while (q.size() > 1 && q.back() == 0) q.pop_back();
    return q;
}
static u64 big_mod_small(const Big &a, u64 b) { u64 r; big_divmod_small(a, b, r); return r; }
static int big_cmp(const Big &a, const Big &b) {
    size_t n = std::max(a.size(), b.size());
    for (size_t i = n; i-- > 0;) {
        u64 x = i < a.size() ? a[i] : 0, y = i < b.size() ? b[i] : 0;
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}
static Big big_add(const Big &a, const Big &b) {
    Big r(std::max(a.size(), b.size()) + 1, 0);
    u64 carry = 0;
    for (size_t i = 0; i < r.size(); i++) {
        u128 v = (u128)(i < a.size() ? a[i] : 0) + (i < b.size() ? b[i] : 0) + carry;
        r[i] = (u64)v;
        carry = (u64)(v >> 64);
    }
    while (r.size() > 1 && r.back() == 0) r.pop_back();
    return r;
}
static Big big_sub(const Big &a, const Big &b) { /* a >= b */
    Big r(a.size(), 0);
    u64 borrow = 0;
    for (size_t i = 0; i < a.size(); i++) {
        u64 y = i < b.size() ? b[i] : 0;
        u128 v = (u128)a[i] - y - borrow;
        r[i] = (u64)v;
        borrow = (u64)(v >> 64) ? 1 : 0;
    }
    while (r.size() > 1 && r.back() == 0) r.pop_back();
    return r;
}
static int big_bits(const Big &a) {
    for (size_t i = a.size(); i-- > 0;)
        if (a[i]) return (int)(i * 64 + 64 - __builtin_clzll(a[i]));
    return 0;
}

static orc_ctx *build_ctx(u64 t, uint32_t N, const std::vector<u64> &qv, int dbc_relin, int dbc_galois) {
    if (N < 2 || (N & (N - 1))) { fail("N must be a power of two"); return nullptr; }
    int logN = 0;
    while ((1u << logN) < N) logN++;
    for (u64 p : qv)
        if (!is_prime(p) || (p - 1) % (2ULL * N)) { fail("coefficient modulus must be prime and = 1 mod 2N"); return nullptr; }
    if (!is_prime(t) || (t - 1) % (2ULL * N)) { fail("plain modulus must be prime and = 1 mod 2N (batching)"); return nullptr; }
    orc_ctx *c = new orc_ctx();
    /* gamma, m_sk and the auxiliary primes are 61-bit primes = 1 mod 2^18: a q holding one makes the inverse of q modulo it 0, so the
     * decryption (gamma) or the BEHZ multiply (Bsk) built on it would be silently wrong.  The context stays usable for what does not
     * divide by q there (tables, transforms, keys, encryption, key switches); those operations refuse. */
    std::vector<u64> aux = aux_primes((int)qv.size());
    for (u64 p : qv) {
        if (p == GAMMA) c->refuse_decrypt = "coefficient moduli must not contain gamma = 0x1fffffffffc80001";
        if (p == M_SK || std::find(aux.begin(), aux.end(), p) != aux.end())
            c->refuse_behz = "coefficient moduli must not contain a prime of the BEHZ base Bsk";
    }
    c->t = t; c->N = N; c->logN = logN; c->k = (int)qv.size();
    c->dbc_relin = dbc_relin; c->dbc_galois = dbc_galois;
    int k = c->k;
    for (u64 p : qv) c->q.push_back(make_mod(p));
    for (u64 p : aux) c->bsk.push_back(make_mod(p));
    c->bsk.push_back(make_mod(M_SK));
    c->tmod = make_mod(t);
    c->gmod = make_mod(GAMMA);
    c->ntt_q.resize(k);
    for (int i = 0; i < k; i++) build_ntt(c->ntt_q[i], qv[i], logN);
    c->ntt_bsk.resize(k + 1);
    for (int j = 0; j <= k; j++) build_ntt(c->ntt_bsk[j], c->bsk[j].p, logN);
    build_ntt(c->ntt_t, t, logN);
    /* BatchEncoder::populate_matrix_reps_index_map */
    c->index_map.assign(N, 0);
    {
        u64 row = N >> 1, m = 2ULL * N, gen = 3, pos = 1;
        for (u64 i = 0; i < row; i++) {
            u64 i1 = (pos - 1) >> 1, i2 = (m - pos - 1) >> 1;
            c->index_map[i] = bitrev(i1, logN);
            c->index_map[row | i] = bitrev(i2, logN);
            pos = (pos * gen) & (m - 1);
        }
    }
    /* q as big integer; floor(q/t), q mod t (SEALContext::validate: coeff_div_plain_modulus, upper_half_increment) */
    Big Q{1};
    for (u64 p : qv) Q = big_mul_small(Q, p);
    u64 q_mod_t;
    Big Qdiv = big_divmod_small(Q, t, q_mod_t);
    c->upper_half_threshold = (t + 1) >> 1;
    for (int i = 0; i < k; i++) {
        c->delta.push_back(big_mod_small(Qdiv, qv[i]));
        c->q_mod_t_q.push_back(q_mod_t % qv[i]);
    }
    /* BaseConverter::generate */
    std::vector<Mod> B(c->bsk.begin(), c->bsk.begin() + k);
    for (int i = 0; i < k; i++) {
        u64 qhat = prod_mod_except(c->q, i, c->q[i]);
        u64 inv = invmod(qhat, c->q[i]);
        c->inv_qhat_mod_q.push_back(inv);
        c->mtilde_inv_qhat_mod_q.push_back(mulmod(inv, M_TILDE % qv[i], c->q[i]));
        u64 pm = 1;
        for (int l = 0; l < k; l++)
            if (l != i) pm = (pm * (qv[l] & 0xffffffffULL)) & 0xffffffffULL;
        c->qhat_mod_mtilde.push_back(pm);
    }
    c->qhat_mod_bsk.assign(k + 1, std::vector<u64>(k));
    for (int j = 0; j <= k; j++) {
        for (int i = 0; i < k; i++) c->qhat_mod_bsk[j][i] = prod_mod_except(c->q, i, c->bsk[j]);
        u64 qm = prod_mod_except(c->q, -1, c->bsk[j]);
        c->q_mod_bsk.push_back(qm);
        c->inv_q_mod_bsk.push_back(invmod(qm, c->bsk[j]));
        c->inv_mtilde_mod_bsk.push_back(invmod(M_TILDE % c->bsk[j].p, c->bsk[j]));
    }
    {
        u64 qm = 1;
        for (int l = 0; l < k; l++) qm = (qm * (qv[l] & 0xffffffffULL)) & 0xffffffffULL;
        c->inv_q_mod_mtilde = inv_mod_pow2_32(qm);
    }
    Mod msk = c->bsk[k];
    c->bhat_mod_q.assign(k, std::vector<u64>(k));
    for (int j = 0; j < k; j++) {
        c->inv_bhat_mod_b.push_back(invmod(prod_mod_except(B, j, B[j]), B[j]));
        c->bhat_mod_msk.push_back(prod_mod_except(B, j, msk));
        for (int i = 0; i < k; i++) c->bhat_mod_q[i][j] = prod_mod_except(B, j, c->q[i]);
    }
    c->inv_B_mod_msk = invmod(prod_mod_except(B, -1, msk), msk);
    for (int i = 0; i < k; i++) c->B_mod_q.push_back(prod_mod_except(B, -1, c->q[i]));
    /* decryption constants */
    for (int i = 0; i < k; i++) {
        c->tgamma_mod_q.push_back(mulmod(t % qv[i], GAMMA % qv[i], c->q[i]));
        c->qhat_mod_t.push_back(prod_mod_except(c->q, i, c->tmod));
        c->qhat_mod_gamma.push_back(prod_mod_except(c->q, i, c->gmod));
    }
    c->neg_inv_q_mod_t = negmod(invmod(prod_mod_except(c->q, -1, c->tmod), c->tmod), c->tmod);
    c->neg_inv_q_mod_gamma = negmod(invmod(prod_mod_except(c->q, -1, c->gmod), c->gmod), c->gmod);
    c->inv_gamma_mod_t = invmod(GAMMA % t, c->tmod);
    return c;
}

extern "C" orc_ctx *orc_create(u64 t, uint32_t N, int coeff_count, int dbc_relin, int dbc_galois) {
    std::vector<u64> qv = default_coeff_modulus(N);
    if (qv.empty()) { fail("no default coefficient modulus for this N"); return nullptr; }
    if (coeff_count > 0 && coeff_count < (int)qv.size()) qv.resize(coeff_count); /* AtomicSealBfvVector.cs:148-149 */
    return build_ctx(t, N, qv, dbc_relin, dbc_galois);
}
extern "C" orc_ctx *orc_create_custom(u64 t, uint32_t N, const u64 *q, int k, int dbc_relin, int dbc_galois) {
    return build_ctx(t, N, std::vector<u64>(q, q + k), dbc_relin, dbc_galois);
}
extern "C" void orc_destroy(orc_ctx *c) { delete c; }
extern "C" void orc_set_centered_mtilde(orc_ctx *c, int on) { c->centered_mtilde = on; }
extern "C" uint32_t orc_N(const orc_ctx *c) { return c->N; }
extern "C" int orc_k(const orc_ctx *c) { return c->k; }
extern "C" u64 orc_t(const orc_ctx *c) { return c->t; }
extern "C" u64 orc_gamma(const orc_ctx *) { return GAMMA; }
extern "C" void orc_get_coeff_moduli(const orc_ctx *c, u64 *out) { for (int i = 0; i < c->k; i++) out[i] = c->q[i].p; }
extern "C" void orc_get_bsk_moduli(const orc_ctx *c, u64 *out) { for (int i = 0; i <= c->k; i++) out[i] = c->bsk[i].p; }
static const NttTables &tables(const orc_ctx *c, int which) {
    if (which < c->k) return c->ntt_q[which];
    if (which <= 2 * c->k) return c->ntt_bsk[which - c->k];
    return c->ntt_t;
}
extern "C" void orc_get_ntt_tables(const orc_ctx *c, int which, u64 *w, u64 *ws, u64 *iw, u64 *iws, u64 *inv_n) {
    const NttTables &T = tables(c, which);
    size_t b = c->N * sizeof(u64);
    if (w) memcpy(w, T.w.data(), b);
    if (ws) memcpy(ws, T.ws.data(), b);
    if (iw) memcpy(iw, T.iw.data(), b);
    if (iws) memcpy(iws, T.iws.data(), b);
    if (inv_n) *inv_n = T.inv_n;
}
extern "C" void orc_ntt_forward(const orc_ctx *c, int which, u64 *poly) { ntt_fwd(poly, tables(c, which)); }
extern "C" void orc_ntt_inverse(const orc_ctx *c, int which, u64 *poly) { ntt_inv(poly, tables(c, which)); }

/* ------------------------------------------------------------------ KeyGenerator (SEAL keygenerator.cpp) */
static void dyadic(const u64 *a, const u64 *b, u64 *out, size_t n, const Mod &m) {
    for (size_t i = 0; i < n; i++) out[i] = mulmod(a[i], b[i], m);
}
/* util::apply_galois on one residue polynomial (coefficient form) */
static void galois_poly(const u64 *in, int logN, u64 elt, const Mod &m, u64 *out) {
    u64 n = 1ULL << logN;
    for (u64 i = 0; i < n; i++) {
        u64 raw = i * elt, idx = raw & (n - 1);
        u64 v = in[i];
        if ((raw >> logN) & 1) v = negmod(v, m);
        out[idx] = v;
    }
}
static int digit_count(const orc_ctx *c, int w) { /* KeyGenerator::populate_decomposition_factors */
    int d = 0;
    for (int i = 0; i < c->k; i++) d += (c->q[i].bits + w - 1) / w;
    return d;
}
/* one key-switching key set for target polynomial `target_ntt` (k*N, NTT form): for residue i and digit j the
 * key is (-(a s + e) + [residue i only] 2^{jw} target, a), all in NTT form (KeyGenerator::relin_keys / galois_keys) */
static void make_kskey(const orc_ctx *c, const u64 *target_ntt, int w, u64 purpose_a, u64 purpose_e, u64 key_tag, KSKey &out) {
    const int k = c->k;
    const size_t N = c->N;
    out.count = digit_count(c, w);
    out.data.assign((size_t)out.count * 2 * k * N, 0);
    std::vector<u64> e(N), tmp(N);
    int idx = 0;
    for (int i = 0; i < k; i++) {
        int nd = (c->q[i].bits + w - 1) / w;
        u64 factor = 1;
        for (int j = 0; j < nd; j++, idx++) {
            u64 *c0 = &out.data[(size_t)idx * 2 * k * N], *c1 = c0 + (size_t)k * N;
            u64 tag = key_tag * 256 + idx;
            for (int l = 0; l < k; l++) {
                const Mod &m = c->q[l];
                u64 *a = c1 + l * N;
                for (size_t x = 0; x < N; x++) a[x] = sample_uniform(rng64(c->seed, stream_id(purpose_a, tag, l), x), m.p);
                for (size_t x = 0; x < N; x++) e[x] = lift_small(sample_noise(rng64(c->seed, stream_id(purpose_e, tag, 0), x)), m.p);
                ntt_fwd(e.data(), c->ntt_q[l]);
                dyadic(a, &c->sk_ntt[l * N], tmp.data(), N, m);
                for (size_t x = 0; x < N; x++) c0[l * N + x] = negmod(addmod(tmp[x], e[x], m), m);
            }
            const Mod &mi = c->q[i];
            for (size_t x = 0; x < N; x++) c0[i * N + x] = addmod(c0[i * N + x], mulmod(target_ntt[i * N + x], factor, mi), mi);
            factor = mulmod(factor, (1ULL << w) % mi.p, mi);
        }
    }
}
extern "C" void orc_keygen(orc_ctx *c, u64 seed) {
    const int k = c->k;
    const size_t N = c->N;
    c->seed = seed;
    c->sk_coeff.assign(k * N, 0);
    c->sk_ntt.assign(k * N, 0);
    for (size_t x = 0; x < N; x++) {
        int s = sample_ternary(rng64(seed, stream_id(S_SK, 0, 0), x));
        for (int l = 0; l < k; l++) c->sk_coeff[l * N + x] = lift_small(s, c->q[l].p);
    }
    c->sk_ntt = c->sk_coeff;
    for (int l = 0; l < k; l++) ntt_fwd(&c->sk_ntt[l * N], c->ntt_q[l]);
    /* public key (-(a s + e), a), NTT form */
    c->pk.assign(2 * k * N, 0);
    std::vector<u64> e(N), tmp(N);
    for (int l = 0; l < k; l++) {
        const Mod &m = c->q[l];
        u64 *a = &c->pk[(k + l) * N];
        for (size_t x = 0; x < N; x++) a[x] = sample_uniform(rng64(seed, stream_id(S_PK_A, 0, l), x), m.p);
        for (size_t x = 0; x < N; x++) e[x] = lift_small(sample_noise(rng64(seed, stream_id(S_PK_E, 0, 0), x)), m.p);
        ntt_fwd(e.data(), c->ntt_q[l]);
        dyadic(a, &c->sk_ntt[l * N], tmp.data(), N, m);
        for (size_t x = 0; x < N; x++) c->pk[l * N + x] = negmod(addmod(tmp[x], e[x], m), m);
    }
    /* relinearization keys for s^2 (AtomicSealBfvVector.cs:68 keys.RelinKeys(dbc)) */
    std::vector<u64> s2(k * N);
    for (int l = 0; l < k; l++) dyadic(&c->sk_ntt[l * N], &c->sk_ntt[l * N], &s2[l * N], N, c->q[l]);
    make_kskey(c, s2.data(), c->dbc_relin, S_RLK_A, S_RLK_E, 0, c->rlk);
    /* Galois keys (AtomicSealBfvVector.cs:69 keys.GaloisKeys(dbc)): 2N-1, 3^(2^i), 3^-(2^i) for i < logN-1 */
    c->galois_elts.clear();
    c->glk.clear();
    u64 m2 = 2ULL * N;
    c->galois_elts.push_back(m2 - 1);
    u64 p3 = 3, n3 = 0;
    for (u64 x = 1; x < m2; x += 2)
        if (((x * 3) & (m2 - 1)) == 1) { n3 = x; break; }
    for (int i = 0; i < c->logN - 1; i++) {
        c->galois_elts.push_back(p3);
        p3 = (p3 * p3) & (m2 - 1);
        c->galois_elts.push_back(n3);
        n3 = (n3 * n3) & (m2 - 1);
    }
    std::vector<u64> rs(k * N);
    for (size_t gi = 0; gi < c->galois_elts.size(); gi++) {
        u64 elt = c->galois_elts[gi];
        for (int l = 0; l < k; l++) {
            galois_poly(&c->sk_coeff[l * N], c->logN, elt, c->q[l], &rs[l * N]);
            ntt_fwd(&rs[l * N], c->ntt_q[l]);
        }
        make_kskey(c, rs.data(), c->dbc_galois, S_GLK_A, S_GLK_E, gi + 1, c->glk[elt]);
    }
    c->have_keys = true;
}
extern "C" void orc_get_secret_key(const orc_ctx *c, u64 *out) { memcpy(out, c->sk_ntt.data(), c->sk_ntt.size() * 8); }
extern "C" void orc_get_public_key(const orc_ctx *c, u64 *out) { memcpy(out, c->pk.data(), c->pk.size() * 8); }
extern "C" int orc_relin_key_count(const orc_ctx *c) { return c->rlk.count; }
extern "C" void orc_get_relin_keys(const orc_ctx *c, u64 *out) { memcpy(out, c->rlk.data.data(), c->rlk.data.size() * 8); }
extern "C" int orc_galois_elt_count(const orc_ctx *c) { return (int)c->galois_elts.size(); }
extern "C" void orc_get_galois_elts(const orc_ctx *c, u64 *out) { memcpy(out, c->galois_elts.data(), c->galois_elts.size() * 8); }
extern "C" int orc_galois_key_count(const orc_ctx *c) { return digit_count(c, c->dbc_galois); }
extern "C" int orc_get_galois_key(const orc_ctx *c, u64 elt, u64 *out) {
    auto it = c->glk.find(elt);
    if (it == c->glk.end()) return fail("Galois key not present");
    memcpy(out, it->second.data.data(), it->second.data.size() * 8);
    return 0;
}
extern "C" int orc_set_galois_key(orc_ctx *c, u64 elt, const u64 *in) {
    auto it = c->glk.find(elt);
    if (it == c->glk.end()) return fail("Galois key not present");
    memcpy(it->second.data.data(), in, it->second.data.size() * 8);
    return 0;
}

/* ------------------------------------------------------------------ BatchEncoder (SEAL batchencoder.cpp) */
extern "C" void orc_encode(const orc_ctx *c, const u64 *values, size_t n, u64 *plain) {
    memset(plain, 0, c->N * 8);
    for (size_t i = 0; i < n && i < c->N; i++) plain[c->index_map[i]] = values[i] % c->t;
    ntt_inv(plain, c->ntt_t);
}
extern "C" void orc_decode(const orc_ctx *c, const u64 *plain, u64 *values) {
    std::vector<u64> tmp(plain, plain + c->N);
    ntt_fwd(tmp.data(), c->ntt_t);
    for (size_t i = 0; i < c->N; i++) values[i] = tmp[c->index_map[i]];
}

/* ------------------------------------------------------------------ Encryptor / Decryptor */
/* Encryptor::preencrypt: Delta*m with the upper-half increment, per residue */
static inline u64 scale_plain_coeff(const orc_ctx *c, u64 m, int j) {
    const Mod &qj = c->q[j];
    if (m >= c->upper_half_threshold) return barrett128((u128)c->delta[j] * m + c->q_mod_t_q[j], qj);
    return mulmod(c->delta[j], m, qj);
}
/* Encryptor::encrypt (AtomicSealBfvVector.cs:566,587,1211,1227) */
extern "C" void orc_encrypt(const orc_ctx *c, const u64 *plain, size_t coeff_count, u64 nonce, u64 *ct) {
    const int k = c->k;
    const size_t N = c->N;
    std::vector<u64> u(N), tmp(N);
    for (int l = 0; l < k; l++) {
        const Mod &m = c->q[l];
        for (size_t x = 0; x < N; x++) u[x] = lift_small(sample_ternary(rng64(c->seed, stream_id(S_ENC_U, nonce, 0), x)), m.p);
        ntt_fwd(u.data(), c->ntt_q[l]);
        for (int part = 0; part < 2; part++) {
            u64 *dst = ct + (part * k + l) * N;
            dyadic(u.data(), &c->pk[(part * k + l) * N], tmp.data(), N, m);
            ntt_inv(tmp.data(), c->ntt_q[l]);
            u64 sid = stream_id(part == 0 ? S_ENC_E0 : S_ENC_E1, nonce, 0);
            for (size_t x = 0; x < N; x++) {
                u64 v = addmod(tmp[x], lift_small(sample_noise(rng64(c->seed, sid, x)), m.p), m);
                if (part == 0 && x < coeff_count) v = addmod(v, scale_plain_coeff(c, plain[x], l), m);
                dst[x] = v;
            }
        }
    }
}
/* c0 + c1 s (+ c2 s^2) mod q, coefficient form */
static void dot_with_secret(const orc_ctx *c, const u64 *ct, int size, u64 *out) {
    const int k = c->k;
    const size_t N = c->N;
    std::vector<u64> tmp(N), acc(N), spow(N);
    for (int l = 0; l < k; l++) {
        const Mod &m = c->q[l];
        std::fill(acc.begin(), acc.end(), 0);
        memcpy(spow.data(), &c->sk_ntt[l * N], N * 8);
        for (int part = 1; part < size; part++) {
            memcpy(tmp.data(), ct + ((size_t)part * k + l) * N, N * 8);
            ntt_fwd(tmp.data(), c->ntt_q[l]);
            for (size_t x = 0; x < N; x++) acc[x] = addmod(acc[x], mulmod(tmp[x], spow[x], m), m);
            if (part + 1 < size) dyadic(spow.data(), &c->sk_ntt[l * N], spow.data(), N, m);
        }
        ntt_inv(acc.data(), c->ntt_q[l]);
        for (size_t x = 0; x < N; x++) out[l * N + x] = addmod(acc[x], ct[l * N + x], m);
    }
}
/* Decryptor::decrypt (BFV): scale-and-round through {t, gamma} (AtomicSealBfvVector.cs:1042,1085) */
extern "C" int orc_decrypt(const orc_ctx *c, const u64 *ct, int size, u64 *plain) {
    if (c->refuse_decrypt) return fail(c->refuse_decrypt);
    if (!c->have_keys) return fail("no keys");
    if (size < 2 || size > 3) return fail("ciphertext size must be 2 or 3");
    const int k = c->k;
    const size_t N = c->N;
    std::vector<u64> x(k * N);
    dot_with_secret(c, ct, size, x.data());
    const u64 gamma_div_2 = GAMMA >> 1;
    for (size_t n = 0; n < N; n++) {
        u128 st = 0, sg = 0;
        for (int i = 0; i < k; i++) {
            u64 v = mulmod(x[i * N + n], c->tgamma_mod_q[i], c->q[i]);
            v = mulmod(v, c->inv_qhat_mod_q[i], c->q[i]); /* BaseConverter::fastbconv_plain_gamma */
            st += (u128)v * c->qhat_mod_t[i];
            sg += (u128)v * c->qhat_mod_gamma[i];
        }
        u64 vt = mulmod(barrett128(st, c->tmod), c->neg_inv_q_mod_t, c->tmod);
        u64 vg = mulmod(barrett128(sg, c->gmod), c->neg_inv_q_mod_gamma, c->gmod);
        u64 r;
        if (vg > gamma_div_2) r = addmod(vt, (GAMMA - vg) % c->t, c->tmod);
        else r = submod(vt, vg % c->t, c->tmod);
        plain[n] = r ? mulmod(r, c->inv_gamma_mod_t, c->tmod) : 0;
    }
    return 0;
}
/* Decryptor::invariant_noise_budget (CryptoTracker.cs:45) */
extern "C" int orc_noise_budget(const orc_ctx *c, const u64 *ct, int size) {
    const int k = c->k;
    const size_t N = c->N;
    std::vector<u64> x(k * N);
    dot_with_secret(c, ct, size, x.data());
    Big Q{1};
    for (int i = 0; i < k; i++) Q = big_mul_small(Q, c->q[i].p);
    std::vector<Big> qhat(k);
    for (int i = 0; i < k; i++) {
        qhat[i] = Big{1};
        for (int l = 0; l < k; l++)
            if (l != i) qhat[i] = big_mul_small(qhat[i], c->q[l].p);
    }
    Big half = Q;
    { u64 r; half = big_divmod_small(Q, 2, r); }
    int maxbits = 0;
    for (size_t n = 0; n < N; n++) {
        /* v = t * x mod q, centred */
        Big acc{0};
        for (int i = 0; i < k; i++) {
            u64 v = mulmod(mulmod(x[i * N + n], c->t % c->q[i].p, c->q[i]), c->inv_qhat_mod_q[i], c->q[i]);
            acc = big_add(acc, big_mul_small(qhat[i], v));
        }
        while (big_cmp(acc, Q) >= 0) acc = big_sub(acc, Q);
        if (big_cmp(acc, half) > 0) acc = big_sub(Q, acc);
        maxbits = std::max(maxbits, big_bits(acc));
    }
    int b = big_bits(Q) - maxbits - 1;
    return b < 0 ? 0 : b;
}

/* ------------------------------------------------------------------ Evaluator: linear ops */
extern "C" void orc_add(const orc_ctx *c, const u64 *a, const u64 *b, int size, u64 *out) {
    const size_t N = c->N;
    for (int s = 0; s < size; s++)
        for (int l = 0; l < c->k; l++) {
            size_t o = ((size_t)s * c->k + l) * N;
            for (size_t x = 0; x < N; x++) out[o + x] = addmod(a[o + x], b[o + x], c->q[l]);
        }
}
extern "C" void orc_sub(const orc_ctx *c, const u64 *a, const u64 *b, int size, u64 *out) {
    const size_t N = c->N;
    for (int s = 0; s < size; s++)
        for (int l = 0; l < c->k; l++) {
            size_t o = ((size_t)s * c->k + l) * N;
            for (size_t x = 0; x < N; x++) out[o + x] = submod(a[o + x], b[o + x], c->q[l]);
        }
}
extern "C" void orc_negate(const orc_ctx *c, const u64 *a, int size, u64 *out) {
    const size_t N = c->N;
    for (int s = 0; s < size; s++)
        for (int l = 0; l < c->k; l++) {
            size_t o = ((size_t)s * c->k + l) * N;
            for (size_t x = 0; x < N; x++) out[o + x] = negmod(a[o + x], c->q[l]);
        }
}
/* Evaluator::add_plain / sub_plain (AtomicSealBfvVector.cs:1019,1267): Delta*m into c0 */
static void addsub_plain(const orc_ctx *c, const u64 *ct, int size, const u64 *plain, size_t cc, u64 *out, bool sub) {
    const size_t N = c->N;
    if (out != ct) memcpy(out, ct, (size_t)size * c->k * N * 8);
    for (int l = 0; l < c->k; l++)
        for (size_t x = 0; x < cc; x++) {
            u64 v = scale_plain_coeff(c, plain[x], l);
            out[l * N + x] = sub ? submod(out[l * N + x], v, c->q[l]) : addmod(out[l * N + x], v, c->q[l]);
        }
}
extern "C" void orc_add_plain(const orc_ctx *c, const u64 *ct, int size, const u64 *plain, size_t cc, u64 *out) { addsub_plain(c, ct, size, plain, cc, out, false); }
extern "C" void orc_sub_plain(const orc_ctx *c, const u64 *ct, int size, const u64 *plain, size_t cc, u64 *out) { addsub_plain(c, ct, size, plain, cc, out, true); }

/* Evaluator::multiply_plain (AtomicSealBfvVector.cs:472,482,571,592,803,855,942,1455):
 * monomial fast path (negacyclic_multiply_poly_mono_coeffmod) or lift + NTT + dyadic + INTT */
static inline u64 lift_plain_coeff(const orc_ctx *c, u64 m, int j) { /* plain_upper_half_increment = q_j - t (fast plain lift) */
    return m >= c->upper_half_threshold ? m + (c->q[j].p - c->t) : m;
}
extern "C" int orc_multiply_plain(const orc_ctx *c, const u64 *ct, int size, const u64 *plain, size_t cc, u64 *out) {
    const int k = c->k;
    const size_t N = c->N;
    size_t nz = 0, last = 0;
    for (size_t x = 0; x < cc; x++)
        if (plain[x]) { nz++; last = x; }
    if (nz == 0) return fail("plain cannot be zero (result would be transparent)");
    if (nz == 1) {
        std::vector<u64> tmp(N);
        for (int s = 0; s < size; s++)
            for (int l = 0; l < k; l++) {
                const Mod &m = c->q[l];
                const u64 *src = ct + ((size_t)s * k + l) * N;
                u64 *dst = out + ((size_t)s * k + l) * N;
                u64 w = lift_plain_coeff(c, plain[last], l);
                for (size_t x = 0; x < N; x++) { /* x^e * src, negacyclic */
                    size_t idx = x + last;
                    u64 v = mulmod(src[x], w, m);
                    if (idx >= N) { idx -= N; v = negmod(v, m); }
                    tmp[idx] = v;
                }
                memcpy(dst, tmp.data(), N * 8);
            }
        return 0;
    }
    std::vector<u64> pl(N), tmp(N);
    for (int l = 0; l < k; l++) {
        const Mod &m = c->q[l];
        std::fill(pl.begin(), pl.end(), 0);
        for (size_t x = 0; x < cc; x++) pl[x] = lift_plain_coeff(c, plain[x], l);
        ntt_fwd(pl.data(), c->ntt_q[l]);
        for (int s = 0; s < size; s++) {
            memcpy(tmp.data(), ct + ((size_t)s * k + l) * N, N * 8);
            ntt_fwd(tmp.data(), c->ntt_q[l]);
            dyadic(tmp.data(), pl.data(), tmp.data(), N, m);
            ntt_inv(tmp.data(), c->ntt_q[l]);
            memcpy(out + ((size_t)s * k + l) * N, tmp.data(), N * 8);
        }
    }
    return 0;
}

/* ------------------------------------------------------------------ BEHZ multiply (SEAL evaluator.cpp bfv_multiply,
 * util/baseconverter.cpp fastbconv_mtilde / mont_rq / fast_floor / fastbconv_sk)
 * reached from AtomicSealBfvVector.cs:461,546,786,839,1457 */
extern "C" int orc_behz_lift(const orc_ctx *c, const u64 *in, u64 *out) {
    if (c->refuse_behz) return fail(c->refuse_behz);
    const int k = c->k;
    const size_t N = c->N;
    u64 tmp[16];
    for (size_t n = 0; n < N; n++) {
        /* fastbconv_mtilde: |x * m~ * qhat_i^-1|_qi, then sum against qhat_i mod target */
        u64 sm = 0;
        for (int i = 0; i < k; i++) {
            tmp[i] = mulmod(in[i * N + n], c->mtilde_inv_qhat_mod_q[i], c->q[i]);
            sm += tmp[i] * c->qhat_mod_mtilde[i]; /* only the low 32 bits matter */
        }
        sm &= 0xffffffffULL;
        /* mont_rq: r = -x_mtilde * q^-1 mod m~ */
        u64 r = (M_TILDE - ((sm * c->inv_q_mod_mtilde) & 0xffffffffULL)) & 0xffffffffULL;
        for (int j = 0; j <= k; j++) {
            const Mod &bj = c->bsk[j];
            u128 acc = 0;
            for (int i = 0; i < k; i++) acc += (u128)tmp[i] * c->qhat_mod_bsk[j][i];
            u64 xb = barrett128(acc, bj);
            u64 rr = r;
            if (c->centered_mtilde && r >= (M_TILDE >> 1)) rr = r + (bj.p - M_TILDE);
            u64 v = barrett128((u128)c->q_mod_bsk[j] * rr + xb, bj);
            out[j * N + n] = mulmod(v, c->inv_mtilde_mod_bsk[j], bj);
        }
    }
    return 0;
}
/* in: [k q-residues | k+1 Bsk residues] of t*d ; out: k q-residues of floor-ish(t*d/q) */
extern "C" int orc_behz_floor(const orc_ctx *c, const u64 *in, u64 *out) {
    if (c->refuse_behz) return fail(c->refuse_behz);
    const int k = c->k;
    const size_t N = c->N;
    const Mod &msk = c->bsk[k];
    const u64 msk_div_2 = msk.p >> 1;
    u64 tmp[16], fl[17];
    for (size_t n = 0; n < N; n++) {
        /* fast_floor: (x_bsk - fastbconv_q->bsk(x_q)) * q^-1 mod bsk_j */
        for (int i = 0; i < k; i++) tmp[i] = mulmod(in[i * N + n], c->inv_qhat_mod_q[i], c->q[i]);
        for (int j = 0; j <= k; j++) {
            const Mod &bj = c->bsk[j];
            u128 acc = 0;
            for (int i = 0; i < k; i++) acc += (u128)tmp[i] * c->qhat_mod_bsk[j][i];
            u64 conv = barrett128(acc, bj);
            fl[j] = mulmod(in[(k + j) * N + n] + (bj.p - conv), c->inv_q_mod_bsk[j], bj);
        }
        /* fastbconv_sk: B -> q with Shenoy-Kumaresan correction through m_sk */
        for (int j = 0; j < k; j++) tmp[j] = mulmod(fl[j], c->inv_bhat_mod_b[j], c->bsk[j]);
        u128 am = 0;
        for (int j = 0; j < k; j++) am += (u128)tmp[j] * c->bhat_mod_msk[j];
        u64 alpha = mulmod(barrett128(am, msk) + (msk.p - fl[k]), c->inv_B_mod_msk, msk);
        for (int i = 0; i < k; i++) {
            const Mod &qi = c->q[i];
            u128 acc = 0;
            for (int j = 0; j < k; j++) acc += (u128)tmp[j] * c->bhat_mod_q[i][j];
            u64 v = barrett128(acc, qi);
            if (alpha > msk_div_2) v = barrett128((u128)c->B_mod_q[i] * (msk.p - alpha) + v, qi);
            else v = barrett128((u128)(qi.p - c->B_mod_q[i]) * alpha + v, qi);
            out[i * N + n] = v;
        }
    }
    return 0;
}
extern "C" int orc_multiply(const orc_ctx *c, const u64 *a, const u64 *b, u64 *out) {
    if (c->refuse_behz) return fail(c->refuse_behz);
    const int k = c->k, kb = k + 1;
    const size_t N = c->N;
    /* steps 0-1: both operands into Bsk, then NTT everything */
    static thread_local std::vector<u64> aq, bq, ab, bb, tog, d;
    aq.assign(a, a + 2 * k * N);
    bq.assign(b, b + 2 * k * N);
    ab.resize(2 * kb * N);
    bb.resize(2 * kb * N);
    tog.resize((size_t)(k + kb) * N);
    d.resize(N);
    for (int s = 0; s < 2; s++) {
        orc_behz_lift(c, a + (size_t)s * k * N, &ab[(size_t)s * kb * N]);
        orc_behz_lift(c, b + (size_t)s * k * N, &bb[(size_t)s * kb * N]);
    }
    for (int s = 0; s < 2; s++) {
        for (int l = 0; l < k; l++) { ntt_fwd(&aq[((size_t)s * k + l) * N], c->ntt_q[l]); ntt_fwd(&bq[((size_t)s * k + l) * N], c->ntt_q[l]); }
        for (int j = 0; j < kb; j++) { ntt_fwd(&ab[((size_t)s * kb + j) * N], c->ntt_bsk[j]); ntt_fwd(&bb[((size_t)s * kb + j) * N], c->ntt_bsk[j]); }
    }
    /* step 2: tensor, INTT, times t, gathered as [q | Bsk] per destination polynomial */
    for (int dst = 0; dst < 3; dst++) {
        for (int l = 0; l < k + kb; l++) {
            const bool inq = l < k;
            const Mod &m = inq ? c->q[l] : c->bsk[l - k];
            const NttTables &T = inq ? c->ntt_q[l] : c->ntt_bsk[l - k];
            auto A = [&](int s) { return inq ? &aq[((size_t)s * k + l) * N] : &ab[((size_t)s * kb + (l - k)) * N]; };
            auto Bp = [&](int s) { return inq ? &bq[((size_t)s * k + l) * N] : &bb[((size_t)s * kb + (l - k)) * N]; };
            for (size_t x = 0; x < N; x++) {
                u64 v;
                if (dst == 0) v = mulmod(A(0)[x], Bp(0)[x], m);
                else if (dst == 2) v = mulmod(A(1)[x], Bp(1)[x], m);
                else v = addmod(mulmod(A(0)[x], Bp(1)[x], m), mulmod(A(1)[x], Bp(0)[x], m), m);
                d[x] = v;
            }
            ntt_inv(d.data(), T);
            u64 tm = c->t % m.p;
            for (size_t x = 0; x < N; x++) tog[(size_t)l * N + x] = mulmod(d[x], tm, m);
        }
        /* steps 3-4 */
        orc_behz_floor(c, tog.data(), out + (size_t)dst * k * N);
    }
    return 0;
}

/* ------------------------------------------------------------------ key switching
 * Evaluator::relinearize_one_step / the key-switch half of apply_galois (SEAL 3.2, decomposition bit count w):
 * for source residue i, digit j: d = (c mod q_i >> jw) & (2^w-1); for every target residue l:
 * acc{0,1}[l] += NTT_l(d) * key[(i,j)][{0,1}][l]; then INTT and add. */
static void key_switch(const orc_ctx *c, const u64 *target /*k*N coeff form*/, const KSKey &key, int w, u64 *acc0, u64 *acc1) {
    const int k = c->k;
    const size_t N = c->N;
    /* per-thread scratch (SEAL uses a per-thread MemoryPoolHandle the same way, AtomicSealBfvVector.cs:27) */
    static thread_local std::vector<u128> w0, w1;
    static thread_local std::vector<u64> dig, tmp;
    w0.assign((size_t)k * N, 0);
    w1.assign((size_t)k * N, 0);
    dig.resize(N);
    tmp.resize(N);
    int idx = 0;
    const u64 mask = (w >= 64) ? ~0ULL : ((1ULL << w) - 1);
    for (int i = 0; i < k; i++) {
        int nd = (c->q[i].bits + w - 1) / w;
        for (int j = 0; j < nd; j++, idx++) {
            int shift = j * w;
            for (size_t x = 0; x < N; x++) dig[x] = (target[i * N + x] >> shift) & mask;
            const u64 *k0 = &key.data[(size_t)idx * 2 * k * N], *k1 = k0 + (size_t)k * N;
            for (int l = 0; l < k; l++) {
                const Mod &m = c->q[l];
                for (size_t x = 0; x < N; x++) tmp[x] = dig[x] >= m.p ? dig[x] % m.p : dig[x];
                ntt_fwd(tmp.data(), c->ntt_q[l]);
                u128 *a0 = &w0[(size_t)l * N], *a1 = &w1[(size_t)l * N];
                const u64 *p0 = k0 + l * N, *p1 = k1 + l * N;
                for (size_t x = 0; x < N; x++) {
                    a0[x] += (u128)tmp[x] * p0[x];
                    a1[x] += (u128)tmp[x] * p1[x];
                }
            }
            if ((idx & 7) == 7) { /* keep the 128-bit accumulators from overflowing for 61-bit moduli */
                for (int l = 0; l < k; l++)
                    for (size_t x = 0; x < N; x++) {
                        w0[(size_t)l * N + x] = barrett128(w0[(size_t)l * N + x], c->q[l]);
                        w1[(size_t)l * N + x] = barrett128(w1[(size_t)l * N + x], c->q[l]);
                    }
            }
        }
    }
    for (int l = 0; l < k; l++) {
        for (size_t x = 0; x < N; x++) {
            acc0[l * N + x] = barrett128(w0[(size_t)l * N + x], c->q[l]);
            acc1[l * N + x] = barrett128(w1[(size_t)l * N + x], c->q[l]);
        }
        ntt_inv(acc0 + l * N, c->ntt_q[l]);
        ntt_inv(acc1 + l * N, c->ntt_q[l]);
    }
}
/* Evaluator::relinearize (AtomicSealBfvVector.cs:462,547,787,840) */
extern "C" int orc_relinearize(const orc_ctx *c, const u64 *ct3, u64 *out) {
    if (!c->have_keys) return fail("no keys");
    const int k = c->k;
    const size_t N = c->N;
    static thread_local std::vector<u64> a0, a1;
    a0.resize(k * N);
    a1.resize(k * N);
    key_switch(c, ct3 + (size_t)2 * k * N, c->rlk, c->dbc_relin, a0.data(), a1.data());
    for (int l = 0; l < k; l++)
        for (size_t x = 0; x < N; x++) {
            out[l * N + x] = addmod(ct3[l * N + x], a0[l * N + x], c->q[l]);
            out[(k + l) * N + x] = addmod(ct3[(k + l) * N + x], a1[l * N + x], c->q[l]);
        }
    return 0;
}
/* Evaluator::apply_galois_inplace */
extern "C" int orc_apply_galois(const orc_ctx *c, const u64 *ct, u64 elt, u64 *out) {
    if (!c->have_keys) return fail("no keys");
    auto it = c->glk.find(elt);
    if (it == c->glk.end()) return fail("Galois key not present");
    const int k = c->k;
    const size_t N = c->N;
    std::vector<u64> t0(k * N), t1(k * N), a0(k * N), a1(k * N);
    for (int l = 0; l < k; l++) {
        galois_poly(ct + l * N, c->logN, elt, c->q[l], &t0[l * N]);
        galois_poly(ct + (k + l) * N, c->logN, elt, c->q[l], &t1[l * N]);
    }
    key_switch(c, t1.data(), it->second, c->dbc_galois, a0.data(), a1.data());
    for (int l = 0; l < k; l++)
        for (size_t x = 0; x < N; x++) {
            out[l * N + x] = addmod(t0[l * N + x], a0[l * N + x], c->q[l]);
            out[(k + l) * N + x] = a1[l * N + x];
        }
    return 0;
}
/* Evaluator::galois_elt_from_step: positive = rotate left */
extern "C" u64 orc_galois_elt_from_step(const orc_ctx *c, int steps) {
    u64 n = c->N, m = 2 * n;
    if (steps == 0) return m - 1;
    bool neg = steps < 0;
    u64 pos = neg ? (u64)(-(int64_t)steps) : (u64)steps;
    if (pos >= (n >> 1)) return 0;
    u64 s = neg ? (n >> 1) - pos : pos;
    u64 elt = 1;
    for (u64 i = 0; i < s; i++) elt = (elt * 3) & (m - 1);
    return elt;
}
static std::vector<int> naf(int value) { /* SEAL util::naf */
    std::vector<int> res;
    bool sign = value < 0;
    int v = sign ? -value : value;
    for (int i = 0; v; i++) {
        int zi = (v & 1) ? 2 - (v & 3) : 0;
        v = (v - zi) >> 1;
        if (zi) res.push_back((sign ? -zi : zi) * (1 << i));
    }
    return res;
}
/* Evaluator::rotate_internal (RotateRows call sites AtomicSealBfvVector.cs:625-660,864,1420,1458) */
extern "C" int orc_rotate_rows(const orc_ctx *c, const u64 *ct, int steps, u64 *out) {
    const size_t words = (size_t)2 * c->k * c->N;
    if (steps == 0) { if (out != ct) memcpy(out, ct, words * 8); return 0; }
    u64 elt = orc_galois_elt_from_step(c, steps);
    if (!elt) return fail("step count too large");
    if (c->glk.count(elt)) return orc_apply_galois(c, ct, elt, out);
    std::vector<int> steps_naf = naf(steps);
    if (steps_naf.size() == 1) return fail("Galois key not present");
    std::vector<u64> cur(ct, ct + words), nxt(words);
    for (int s : steps_naf) {
        if ((size_t)(s < 0 ? -s : s) == (c->N >> 1)) continue;
        int rc = orc_rotate_rows(c, cur.data(), s, nxt.data());
        if (rc) return rc;
        cur.swap(nxt);
    }
    memcpy(out, cur.data(), words * 8);
    return 0;
}
extern "C" int orc_rotate_columns(const orc_ctx *c, const u64 *ct, u64 *out) { return orc_apply_galois(c, ct, 2ULL * c->N - 1, out); }

/* ------------------------------------------------------------------ threaded layer drivers (CPU baseline) */
template <class F> static void parallel_for(int count, int threads, F f) { /* Utils.cs:46-88 */
    if (threads < 1) threads = 1;
    if (count < 2 || threads == 1) { for (int i = 0; i < count; i++) f(i); return; }
    std::atomic<int> next(0);
    std::vector<std::thread> pool;
    int nt = std::min(threads, count);
    for (int w = 0; w < nt; w++)
        pool.emplace_back([&]() { for (;;) { int i = next.fetch_add(1); if (i >= count) break; f(i); } });
    for (auto &th : pool) th.join();
}
extern "C" int orc_mac_layer(const orc_ctx *c, const u64 *in, int n_in, const int32_t *gather, const u64 *weights, const u64 *bias,
                             int M, int K, u64 *out, int threads, int m_begin, int m_step) {
    const int k = c->k;
    const size_t N = c->N, ctw = (size_t)2 * k * N;
    if (m_step < 1) m_step = 1;
    std::vector<int> ms;
    for (int m = m_begin; m < M; m += m_step) ms.push_back(m);
    std::atomic<int> bad(0);
    parallel_for((int)ms.size(), threads, [&](int mi) {
        int m = ms[mi];
        u64 *dst = out + (size_t)m * ctw;
        bool first = true;
        for (int kk = 0; kk < K; kk++) {
            int g = gather ? gather[(size_t)m * K + kk] : kk;
            u64 w = weights[(size_t)m * K + kk];
            if (g < 0 || w == 0) continue; /* AtomicSealBfvVector.cs:468 zero plaintexts are skipped */
            if (g >= n_in) { bad = 1; continue; }
            const u64 *src = in + (size_t)g * ctw;
            /* MultiplyPlain (monomial path) then Add, as the reference issues them */
            for (int s = 0; s < 2; s++)
                for (int l = 0; l < k; l++) {
                    const Mod &mod = c->q[l];
                    u64 wl = lift_plain_coeff(c, w, l);
                    size_t o = ((size_t)s * k + l) * N;
                    if (first) for (size_t x = 0; x < N; x++) dst[o + x] = mulmod(src[o + x], wl, mod);
                    else for (size_t x = 0; x < N; x++) dst[o + x] = addmod(dst[o + x], mulmod(src[o + x], wl, mod), mod);
                }
            first = false;
        }
        if (first) { bad = 2; memset(dst, 0, ctw * 8); }
        if (bias) /* AddPlain of the constant polynomial b (PoolLayer.cs:219; dense plain vector of equal slots) */
            for (int l = 0; l < k; l++) dst[l * N] = addmod(dst[l * N], scale_plain_coeff(c, bias[m], l), c->q[l]);
    });
    if (bad == 1) return fail("gather index out of range");
    if (bad == 2) return fail("an output has no non-zero tap (transparent ciphertext)");
    return 0;
}
extern "C" int orc_square_layer(const orc_ctx *c, const u64 *in, int n, u64 *out, int threads, int begin, int step) {
    if (c->refuse_behz) return fail(c->refuse_behz);
    const size_t ctw = (size_t)2 * c->k * c->N;
    if (step < 1) step = 1;
    std::vector<int> is;
    for (int i = begin; i < n; i += step) is.push_back(i);
    parallel_for((int)is.size(), threads, [&](int ii) {
        int i = is[ii];
        static thread_local std::vector<u64> t3;
        t3.resize(ctw / 2 * 3);
        orc_multiply(c, in + (size_t)i * ctw, in + (size_t)i * ctw, t3.data());
        orc_relinearize(c, t3.data(), out + (size_t)i * ctw);
    });
    return 0;
}
extern "C" int orc_ntt_batch(const orc_ctx *c, int which, u64 *polys, int n, int inverse, int threads) {
    const NttTables &T = tables(c, which);
    parallel_for(n, threads, [&](int i) {
        if (inverse) ntt_inv(polys + (size_t)i * c->N, T);
        else ntt_fwd(polys + (size_t)i * c->N, T);
    });
    return 0;
}
