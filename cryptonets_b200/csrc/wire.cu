// Wire / on-disk formats of the reference (SURVEY.md section 8f-3): the key archive and the text serialisation of vectors.
//
// Containers -- fully specified by the reference's C#:
//   key archive   EncryptedSealBfvEnvironment.Save ("HE Wrapper/EncryptedSealBfvVector.cs:104-134"): ZIP archive, one entry
//                 `environmentNNN` per plaintext modulus holding AtomicSealBfvEncryptedEnvironment.SaveToStream
//                 ("HE Wrapper/AtomicSealBfvVector.cs:93-104"): EncryptionParameters, PublicKey, RelinKeys, GaloisKeys, SecretKey (an empty
//                 SecretKey when saved without private keys); read back by LoadFromStream (":106-131") / the factory's file constructor.
//   vector text   EncryptedSealBfvVector.Write / Read (":414-439") around AtomicSealBfvEncryptedVector.Write / Read
//                 ("AtomicSealBfvVector.cs:1273-1345"): text lines; the SEAL objects of one channel concatenated, base64 on one line.
//
// SEAL 3.2 binary streams inside them -- PARITY WITH THE REAL SEAL 3.2 BINARY IS UNPINNED: SEAL is not in the reference tree and cannot
// be built here; the layouts are restated from knowledge of SEAL 3.2.x (little endian):
//   EncryptionParameters::Save   u8 scheme (1 = BFV) | u64 poly_modulus_degree | u64 coeff_mod_count | u64 per coefficient modulus |
//                                u64 plain modulus | f64 noise_standard_deviation (3.20)
//   parms_id                     SHA3-256 of the u64 array [scheme, N, q_0.., t, bits(noise_standard_deviation)]
//   Ciphertext::save             parms_id | u8 is_ntt_form | u64 size | u64 N | u64 coeff_mod_count | f64 scale | u64 word count | words
//   Plaintext::save              parms_id (zero for a message) | f64 scale | u64 coefficient count | words
//   PublicKey = its ciphertext (NTT form); SecretKey = its plaintext (NTT form, k*N words)
//   RelinKeys / GaloisKeys       parms_id | i32 decomposition_bit_count | u64 dim1 | per entry: u64 dim2, ciphertexts (NTT form)
//                                (RelinKeys: one entry, s^2; GaloisKeys: N entries indexed (galois_elt - 1) / 2, absent ones empty)
// tests/test_wire_formats.py checks every byte against an independent Python restatement (oracle/wire_py.py) and restates the
// reference's SaveLoadKeys / SaveAndLoadMatrix tests ("HE Wrapper Tests/BasicOperations.cs:291-331").
#include <cinttypes>
#include <cstdio>
#include <cstring>

#include "hostmath.h"
#include "vec.h"

namespace {

const double NOISE_STANDARD_DEVIATION = 3.20;

// ---------------------------------------------------------------- SHA3-256 (FIPS 202)
void keccak_f(uint64_t st[25]) {
    static const uint64_t RC[24] = {0x0000000000000001ULL, 0x0000000000008082ULL, 0x800000000000808aULL, 0x8000000080008000ULL, 0x000000000000808bULL,
                                    0x0000000080000001ULL, 0x8000000080008081ULL, 0x8000000000008009ULL, 0x000000000000008aULL, 0x0000000000000088ULL,
                                    0x0000000080008009ULL, 0x000000008000000aULL, 0x000000008000808bULL, 0x800000000000008bULL, 0x8000000000008089ULL,
                                    0x8000000000008003ULL, 0x8000000000008002ULL, 0x8000000000000080ULL, 0x000000000000800aULL, 0x800000008000000aULL,
                                    0x8000000080008081ULL, 0x8000000000008080ULL, 0x0000000080000001ULL, 0x8000000080008008ULL};
    static const int ROT[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
    static const int PIL[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
    for (int r = 0; r < 24; r++) {
        uint64_t bc[5];
        for (int i = 0; i < 5; i++) bc[i] = st[i] ^ st[i + 5] ^ st[i + 10] ^ st[i + 15] ^ st[i + 20];
        for (int i = 0; i < 5; i++) {
            const uint64_t t = bc[(i + 4) % 5] ^ ((bc[(i + 1) % 5] << 1) | (bc[(i + 1) % 5] >> 63));
            for (int j = 0; j < 25; j += 5) st[j + i] ^= t;
        }
        uint64_t t = st[1];
        for (int i = 0; i < 24; i++) {
            const int j = PIL[i];
            const uint64_t b = st[j];
            st[j] = (t << ROT[i]) | (t >> (64 - ROT[i]));
            t = b;
        }
        for (int j = 0; j < 25; j += 5) {
            for (int i = 0; i < 5; i++) bc[i] = st[j + i];
            for (int i = 0; i < 5; i++) st[j + i] ^= (~bc[(i + 1) % 5]) & bc[(i + 2) % 5];
        }
        st[0] ^= RC[r];
    }
}
void sha3_256(const uint8_t *in, size_t len, uint8_t out[32]) {
    uint64_t st[25];
    memset(st, 0, sizeof(st));
    const size_t rate = 136;
    uint8_t block[136];
    while (len >= rate) {
        for (size_t i = 0; i < rate / 8; i++) { uint64_t w; memcpy(&w, in + 8 * i, 8); st[i] ^= w; }
        keccak_f(st);
        in += rate;
        len -= rate;
    }
    memset(block, 0, rate);
    memcpy(block, in, len);
    block[len] ^= 0x06;
    block[rate - 1] ^= 0x80;
    for (size_t i = 0; i < rate / 8; i++) { uint64_t w; memcpy(&w, block + 8 * i, 8); st[i] ^= w; }
    keccak_f(st);
    memcpy(out, st, 32);
}

// ---------------------------------------------------------------- byte streams
struct Writer {
    std::vector<uint8_t> b;
    void raw(const void *p, size_t n) { const uint8_t *q = (const uint8_t *)p; b.insert(b.end(), q, q + n); }
    void u8(uint8_t v) { b.push_back(v); }
    void u16(uint16_t v) { raw(&v, 2); }
    void u32(uint32_t v) { raw(&v, 4); }
    void i32(int32_t v) { raw(&v, 4); }
    void u64_(uint64_t v) { raw(&v, 8); }
    void f64(double v) { raw(&v, 8); }
};
struct Reader {
    const uint8_t *p, *end;
    Reader(const uint8_t *b, size_t n) : p(b), end(b + n) {}
    void need(size_t n) const { if ((size_t)(end - p) < n) throw Error(CNHE_ERR_INVALID, "truncated stream"); }
    void raw(void *d, size_t n) { need(n); memcpy(d, p, n); p += n; }
    uint8_t u8() { uint8_t v; raw(&v, 1); return v; }
    uint16_t u16() { uint16_t v; raw(&v, 2); return v; }
    uint32_t u32() { uint32_t v; raw(&v, 4); return v; }
    int32_t i32() { int32_t v; raw(&v, 4); return v; }
    uint64_t u64_() { uint64_t v; raw(&v, 8); return v; }
    double f64() { double v; raw(&v, 8); return v; }
    size_t left() const { return (size_t)(end - p); }
};

typedef uint8_t ParmsId[32];
void compute_parms_id(uint64_t N, const std::vector<u64> &q, u64 t, ParmsId out) {
    std::vector<uint64_t> d;
    d.push_back(1);
    d.push_back(N);
    for (u64 x : q) d.push_back(x);
    d.push_back(t);
    uint64_t bits;
    memcpy(&bits, &NOISE_STANDARD_DEVIATION, 8);
    d.push_back(bits);
    sha3_256(reinterpret_cast<const uint8_t *>(d.data()), d.size() * 8, out);
}
void write_ciphertext(Writer &w, const ParmsId pid, const u64 *words, uint64_t N, uint64_t k, uint64_t size, bool ntt) {
    w.raw(pid, 32);
    w.u8(ntt ? 1 : 0);
    w.u64_(size); w.u64_(N); w.u64_(k);
    w.f64(1.0);
    w.u64_(size * k * N);
    w.raw(words, size * k * N * 8);
}
// reads one ciphertext into dst (size*k*N words expected)
void read_ciphertext(Reader &r, const ParmsId pid, u64 *dst, uint64_t N, uint64_t k, uint64_t size, bool ntt) {
    ParmsId got;
    r.raw(got, 32);
    if (memcmp(got, pid, 32)) throw Error(CNHE_ERR_INVALID, "ciphertext parms_id does not match the context's encryption parameters");
    const bool is_ntt = r.u8() != 0;
    const uint64_t s = r.u64_(), n = r.u64_(), kk = r.u64_();
    r.f64();
    const uint64_t cnt = r.u64_();
    if (s != size || n != N || kk != k || cnt != size * k * N || is_ntt != ntt) throw Error(CNHE_ERR_INVALID, "ciphertext shape does not match the context");
    r.raw(dst, cnt * 8);
}

// ---------------------------------------------------------------- ZIP (stored entries; also reads deflate streams made of stored blocks)
uint32_t crc32_of(const uint8_t *p, size_t n) {
    static uint32_t table[256];
    static bool init = false;
    if (!init) {
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int j = 0; j < 8; j++) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            table[i] = c;
        }
        init = true;
    }
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) c = table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}
struct ZipEntry { std::string name; std::vector<uint8_t> data; };
void zip_write(Writer &w, const std::vector<ZipEntry> &entries) {
    struct Cd { uint32_t crc, size, offset; };
    std::vector<Cd> cds;
    for (const ZipEntry &e : entries) {
        if (e.data.size() >= 0xFFFFFFFFull || w.b.size() >= 0xFFFFFFFFull) throw Error(CNHE_ERR_INVALID, "key archive entry exceeds the 4 GiB ZIP limit");
        Cd cd{crc32_of(e.data.data(), e.data.size()), (uint32_t)e.data.size(), (uint32_t)w.b.size()};
        cds.push_back(cd);
        w.u32(0x04034b50); w.u16(20); w.u16(0); w.u16(0); w.u16(0); w.u16(0x21); // version, flags, method 0 (stored), time, date 1980-01-01
        w.u32(cd.crc); w.u32(cd.size); w.u32(cd.size);
        w.u16((uint16_t)e.name.size()); w.u16(0);
        w.raw(e.name.data(), e.name.size());
        w.raw(e.data.data(), e.data.size());
    }
    const size_t cd_start = w.b.size();
    for (size_t i = 0; i < entries.size(); i++) {
        w.u32(0x02014b50); w.u16(20); w.u16(20); w.u16(0); w.u16(0); w.u16(0); w.u16(0x21);
        w.u32(cds[i].crc); w.u32(cds[i].size); w.u32(cds[i].size);
        w.u16((uint16_t)entries[i].name.size()); w.u16(0); w.u16(0); w.u16(0); w.u16(0); w.u32(0);
        w.u32(cds[i].offset);
        w.raw(entries[i].name.data(), entries[i].name.size());
    }
    const size_t cd_size = w.b.size() - cd_start;
    w.u32(0x06054b50); w.u16(0); w.u16(0); w.u16((uint16_t)entries.size()); w.u16((uint16_t)entries.size());
    w.u32((uint32_t)cd_size); w.u32((uint32_t)cd_start); w.u16(0);
}
// .NET's ZipArchive with CompressionLevel.NoCompression emits a DEFLATE stream consisting of stored blocks: undo that framing
std::vector<uint8_t> inflate_stored_only(const uint8_t *p, size_t n, size_t expect) {
    std::vector<uint8_t> out;
    out.reserve(expect);
    size_t i = 0;
    for (;;) {
        if (i >= n) throw Error(CNHE_ERR_INVALID, "truncated deflate stream");
        const uint8_t hdr = p[i++];
        if ((hdr >> 1) & 3) throw Error(CNHE_ERR_INVALID, "compressed key archives are not supported (expecting stored / no-compression entries)");
        if (i + 4 > n) throw Error(CNHE_ERR_INVALID, "truncated deflate stream");
        const uint16_t len = (uint16_t)(p[i] | (p[i + 1] << 8)), nlen = (uint16_t)(p[i + 2] | (p[i + 3] << 8));
        i += 4;
        if ((uint16_t)~len != nlen || i + len > n) throw Error(CNHE_ERR_INVALID, "corrupt deflate stored block");
        out.insert(out.end(), p + i, p + i + len);
        i += len;
        if (hdr & 1) break;
    }
    return out;
}
std::vector<ZipEntry> zip_read(const uint8_t *b, size_t n) {
    if (n < 22) throw Error(CNHE_ERR_INVALID, "not a ZIP archive");
    size_t eocd = n - 22;
    while (true) {
        if (b[eocd] == 0x50 && b[eocd + 1] == 0x4b && b[eocd + 2] == 0x05 && b[eocd + 3] == 0x06) break;
        if (eocd == 0 || n - eocd > 22 + 65535) throw Error(CNHE_ERR_INVALID, "not a ZIP archive (no end-of-central-directory record)");
        eocd--;
    }
    Reader e(b + eocd + 4, n - eocd - 4);
    e.u16(); e.u16(); e.u16();
    const uint16_t count = e.u16();
    e.u32();
    const uint32_t cd_off = e.u32();
    if (cd_off > n) throw Error(CNHE_ERR_INVALID, "corrupt ZIP archive");
    Reader cd(b + cd_off, n - cd_off);
    std::vector<ZipEntry> out;
    for (int i = 0; i < count; i++) {
        if (cd.u32() != 0x02014b50) throw Error(CNHE_ERR_INVALID, "corrupt ZIP central directory");
        cd.u16(); cd.u16(); cd.u16();
        const uint16_t method = cd.u16();
        cd.u16(); cd.u16();
        const uint32_t crc = cd.u32(), csize = cd.u32(), usize = cd.u32();
        const uint16_t nlen = cd.u16(), xlen = cd.u16(), clen = cd.u16();
        cd.u16(); cd.u16(); cd.u32();
        const uint32_t lho = cd.u32();
        ZipEntry ze;
        ze.name.resize(nlen);
        cd.raw(&ze.name[0], nlen);
        cd.need((size_t)xlen + clen);
        cd.p += xlen + clen;
        if (csize == 0xFFFFFFFFu || usize == 0xFFFFFFFFu) throw Error(CNHE_ERR_INVALID, "ZIP64 archives are not supported");
        if ((size_t)lho + 30 > n) throw Error(CNHE_ERR_INVALID, "corrupt ZIP archive");
        Reader lh(b + lho, n - lho);
        if (lh.u32() != 0x04034b50) throw Error(CNHE_ERR_INVALID, "corrupt ZIP local header");
        lh.p += 22;
        const uint16_t ln = lh.u16(), lx = lh.u16();
        lh.need((size_t)ln + lx + csize);
        const uint8_t *data = lh.p + ln + lx;
        if (method == 0) ze.data.assign(data, data + csize);
        else if (method == 8) ze.data = inflate_stored_only(data, csize, usize);
        else throw Error(CNHE_ERR_INVALID, "unsupported ZIP compression method");
        if (ze.data.size() != usize || crc32_of(ze.data.data(), ze.data.size()) != crc) throw Error(CNHE_ERR_INVALID, "ZIP entry fails its CRC");
        out.push_back(std::move(ze));
    }
    return out;
}

// ---------------------------------------------------------------- base64
const char B64[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
void b64_encode(const std::vector<uint8_t> &in, std::string &out) {
    size_t i = 0;
    out.reserve(out.size() + (in.size() + 2) / 3 * 4);
    for (; i + 2 < in.size(); i += 3) {
        const uint32_t v = (in[i] << 16) | (in[i + 1] << 8) | in[i + 2];
        out += B64[v >> 18]; out += B64[(v >> 12) & 63]; out += B64[(v >> 6) & 63]; out += B64[v & 63];
    }
    if (i + 1 == in.size()) {
        const uint32_t v = in[i] << 16;
        out += B64[v >> 18]; out += B64[(v >> 12) & 63]; out += "==";
    } else if (i + 2 == in.size()) {
        const uint32_t v = (in[i] << 16) | (in[i + 1] << 8);
        out += B64[v >> 18]; out += B64[(v >> 12) & 63]; out += B64[(v >> 6) & 63]; out += '=';
    }
}
std::vector<uint8_t> b64_decode(const char *s, size_t n) {
    static int8_t dec[256];
    static bool init = false;
    if (!init) {
        memset(dec, -1, sizeof(dec));
        for (int i = 0; i < 64; i++) dec[(uint8_t)B64[i]] = (int8_t)i;
        init = true;
    }
    std::vector<uint8_t> out;
    out.reserve(n / 4 * 3);
    uint32_t acc = 0;
    int bits = 0;
    for (size_t i = 0; i < n; i++) {
        if (s[i] == '=') break;
        const int8_t d = dec[(uint8_t)s[i]];
        if (d < 0) throw Error(CNHE_ERR_INVALID, "bad base64 data");
        acc = (acc << 6) | (uint32_t)d;
        bits += 6;
        if (bits >= 8) { bits -= 8; out.push_back((uint8_t)(acc >> bits)); }
    }
    return out;
}

// ---------------------------------------------------------------- text lines
struct Lines {
    const char *p, *end;
    Lines(const char *s, size_t n) : p(s), end(s + n) {}
    // next line without its terminator (accepts \n and \r\n)
    bool next(const char *&s, size_t &n) {
        if (p >= end) return false;
        const char *e = (const char *)memchr(p, '\n', (size_t)(end - p));
        const char *stop = e ? e : end;
        s = p;
        n = (size_t)(stop - p);
        if (n && s[n - 1] == '\r') n--;
        p = e ? e + 1 : end;
        return true;
    }
    std::string str() {
        const char *s; size_t n;
        if (!next(s, n)) throw Error(CNHE_ERR_INVALID, "Bad stream format.");
        return std::string(s, n);
    }
    void expect(const char *what) { if (str() != what) throw Error(CNHE_ERR_INVALID, "Bad stream format."); }
};
std::string fmt_double(double v) { // .NET Framework Double.ToString(): 15 significant digits, shortest form
    char buf[64];
    snprintf(buf, sizeof(buf), "%.15g", v);
    return buf;
}
const char *NL = "\r\n"; // StreamWriter.WriteLine on the reference's platform

} // namespace

// ==================================================================================================== key archive
extern "C" int cnhe_keys_save(cnhe_ctx *h, int with_private_keys, uint8_t *dst, size_t cap, size_t *needed) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (!needed) fail("null argument");
    const uint64_t N = c.N, k = (uint64_t)c.k, kN = k * N;
    std::vector<ZipEntry> entries;
    for (int ci = 0; ci < c.P; ci++) {
        Channel &ch = c.ch[ci];
        if (!ch.have_pk || !ch.have_rlk) fail("keys have not been generated");
        if (with_private_keys && !ch.have_sk) fail("no secret key to save");
        c.set_channel(ci);
        ParmsId pid;
        compute_parms_id(N, c.q, ch.t, pid);
        Writer w;
        w.u8(1); w.u64_(N); w.u64_(k);
        for (u64 q : c.q) w.u64_(q);
        w.u64_(ch.t);
        w.f64(NOISE_STANDARD_DEVIATION);
        std::vector<u64> host;
        auto fetch = [&](const BufRef &b, size_t words) {
            host.resize(words);
            CNHE_CUDA(cudaMemcpyAsync(host.data(), b->p, words * 8, cudaMemcpyDeviceToHost, c.stream));
            c.sync();
        };
        fetch(ch.pk, 2 * kN);
        write_ciphertext(w, pid, host.data(), N, k, 2, true);
        auto write_kswitch = [&](int dbc, uint64_t dim1, const std::map<uint64_t, BufRef> &at, int D) {
            w.raw(pid, 32);
            w.i32(dbc);
            w.u64_(dim1);
            for (uint64_t i = 0; i < dim1; i++) {
                auto it = at.find(i);
                if (it == at.end()) { w.u64_(0); continue; }
                w.u64_((uint64_t)D);
                fetch(it->second, (size_t)D * 2 * kN);
                for (int d = 0; d < D; d++) write_ciphertext(w, pid, host.data() + (size_t)d * 2 * kN, N, k, 2, true);
            }
        };
        write_kswitch(c.dbc_relin, 1, {{0, ch.rlk}}, c.dm_relin.D);
        std::map<uint64_t, BufRef> gal;
        for (auto &kv : ch.glk) gal[(kv.first - 1) >> 1] = kv.second;
        write_kswitch(c.dbc_galois, N, gal, c.dm_galois.D);
        if (with_private_keys) {
            fetch(ch.sk, kN);
            w.raw(pid, 32); w.f64(1.0); w.u64_(kN); w.raw(host.data(), kN * 8);
        } else { // `new SecretKey().Save(stream)`: an empty plaintext
            const ParmsId zero = {0};
            w.raw(zero, 32); w.f64(1.0); w.u64_(0);
        }
        char name[32];
        snprintf(name, sizeof(name), "environment%03d", ci);
        ZipEntry ze;
        ze.name = name;
        ze.data = std::move(w.b);
        entries.push_back(std::move(ze));
    }
    Writer zw;
    zip_write(zw, entries);
    *needed = zw.b.size();
    if (dst) {
        if (cap < zw.b.size()) fail("destination too small");
        memcpy(dst, zw.b.data(), zw.b.size());
    }
    API_END
}

extern "C" int cnhe_context_load(const uint8_t *archive, size_t len, int device, cnhe_ctx **out) {
    try {
        if (!archive || !out) fail("null argument");
        std::vector<ZipEntry> entries = zip_read(archive, len);
        std::vector<ZipEntry *> envs;
        for (ZipEntry &e : entries)
            if (e.name.compare(0, 11, "environment") == 0) envs.push_back(&e);
        std::sort(envs.begin(), envs.end(), [](ZipEntry *a, ZipEntry *b) { return a->name < b->name; });
        if (envs.empty()) fail("the archive holds no environmentNNN entry");
        struct Parsed { uint64_t N; std::vector<u64> q; u64 t; int dbc_r, dbc_g; const uint8_t *pk, *rlk, *glk, *sk; size_t rest; };
        // first pass: parameters (so the context can be created), then a second pass imports the keys
        uint64_t N = 0;
        std::vector<u64> q, primes;
        std::vector<int> dbc(2, 0);
        for (size_t i = 0; i < envs.size(); i++) {
            Reader r(envs[i]->data.data(), envs[i]->data.size());
            if (r.u8() != 1) fail("not a BFV parameter set");
            const uint64_t n = r.u64_(), kk = r.u64_();
            if (kk < 1 || kk > (uint64_t)KMAX) fail("unsupported coefficient modulus count");
            std::vector<u64> qq(kk);
            for (auto &x : qq) x = r.u64_();
            const u64 t = r.u64_();
            r.f64();
            if (i == 0) { N = n; q = qq; }
            else if (n != N || qq != q) fail("the environments of one archive must share the polynomial degree and coefficient modulus");
            primes.push_back(t);
            // skip the public key to reach the decomposition bit counts
            const size_t ctb = 32 + 1 + 24 + 8 + 8 + 2 * kk * n * 8;
            r.need(ctb);
            r.p += ctb;
            r.need(32 + 4);
            r.p += 32;
            const int dr = r.i32();
            uint64_t dim1 = r.u64_();
            for (uint64_t e = 0; e < dim1; e++) {
                const uint64_t dim2 = r.u64_();
                r.need(dim2 * ctb);
                r.p += dim2 * ctb;
            }
            r.need(32 + 4);
            r.p += 32;
            const int dg = r.i32();
            if (i == 0) { dbc[0] = dr; dbc[1] = dg; }
            else if (dr != dbc[0] || dg != dbc[1]) fail("the environments of one archive must share the decomposition bit counts");
        }
        std::unique_ptr<cnhe_ctx> ctx(new cnhe_ctx{nullptr});
        ctx->c = context_create(primes.data(), (int)primes.size(), (uint32_t)N, q.data(), (int)q.size(), dbc[0], dbc[1], device);
        Context &c = *ctx->c;
        std::unique_ptr<Context> guard(ctx->c);
        {
            std::lock_guard<std::recursive_mutex> lock(c.mu);
            const uint64_t k = (uint64_t)c.k, kN = k * N;
            for (int ci = 0; ci < c.P; ci++) {
                c.set_channel(ci);
                Channel &ch = c.ch[ci];
                Reader r(envs[ci]->data.data(), envs[ci]->data.size());
                r.p += 1 + 16 + 8 * k + 16;
                ParmsId pid;
                compute_parms_id(N, c.q, ch.t, pid);
                std::vector<u64> host;
                auto put = [&](int what, u64 arg, size_t words) {
                    size_t w2;
                    BufRef &b = key_slot(c, ci, what, arg, w2, true);
                    if (w2 != words) throw Error(CNHE_ERR_INVALID, "key size does not match the context");
                    CNHE_CUDA(cudaMemcpyAsync(b->p, host.data(), words * 8, cudaMemcpyHostToDevice, c.stream));
                    c.sync();
                };
                host.resize(2 * kN);
                read_ciphertext(r, pid, host.data(), N, k, 2, true);
                put(1, 0, 2 * kN);
                ch.have_pk = true;
                auto read_kswitch = [&](int what, int D, uint64_t expect_dim1) {
                    ParmsId got;
                    r.raw(got, 32);
                    if (memcmp(got, pid, 32)) throw Error(CNHE_ERR_INVALID, "key parms_id does not match the encryption parameters");
                    r.i32();
                    const uint64_t dim1 = r.u64_();
                    if (dim1 != expect_dim1) throw Error(CNHE_ERR_INVALID, "unexpected key set size");
                    for (uint64_t e = 0; e < dim1; e++) {
                        const uint64_t dim2 = r.u64_();
                        if (dim2 == 0) continue;
                        if (dim2 != (uint64_t)D) throw Error(CNHE_ERR_INVALID, "key digit count does not match the decomposition bit count");
                        host.resize((size_t)D * 2 * kN);
                        for (int d = 0; d < D; d++) read_ciphertext(r, pid, host.data() + (size_t)d * 2 * kN, N, k, 2, true);
                        put(what, what == 3 ? 2 * e + 1 : 0, (size_t)D * 2 * kN);
                    }
                };
                read_kswitch(2, c.dm_relin.D, 1);
                rlk_ready(c, ci);
                read_kswitch(3, c.dm_galois.D, N);
                ParmsId spid;
                r.raw(spid, 32);
                r.f64();
                const uint64_t cnt = r.u64_();
                if (cnt) {
                    if (cnt != kN || memcmp(spid, pid, 32)) throw Error(CNHE_ERR_INVALID, "secret key does not match the encryption parameters");
                    host.resize(kN);
                    r.raw(host.data(), kN * 8);
                    put(0, 0, kN);
                    ch.have_sk = true;
                }
                if (r.left()) throw Error(CNHE_ERR_INVALID, "trailing bytes after the secret key");
            }
        }
        guard.release();
        *out = ctx.release();
    } catch (const Error &e) { return set_err(e.code, e.what()); } catch (const std::exception &e) { return set_err(CNHE_ERR_INVALID, e.what()); }
    return CNHE_OK;
}

// ==================================================================================================== vector text
extern "C" int cnhe_vec_write(cnhe_ctx *h, const cnhe_vec *v, char *dst, size_t cap, size_t *needed) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    same_ctx(c, v);
    if (!needed) fail("null argument");
    const uint64_t N = c.N, k = (uint64_t)c.k;
    std::string s;
    s += "<Start LargeEncryptedVector>"; s += NL;
    s += fmt_double(v->scale); s += NL;
    s += std::to_string(c.P); s += NL;
    for (int ci = 0; ci < c.P; ci++) {
        c.set_channel(ci);
        ParmsId pid;
        compute_parms_id(N, c.q, c.ch[ci].t, pid);
        s += "<Start EncryptedVector>"; s += NL;
        s += "1"; s += NL;      // the wrapper builds its atomic vectors with Scale 1 ...
        s += "False"; s += NL;  // ... and SignedNumbers false ("EncryptedSealBfvVector.cs:183-186")
        s += v->format == CNHE_DENSE ? "dense" : "sparse"; s += NL;
        s += std::to_string(v->dim); s += NL;
        s += v->enc ? "Encrypted" : "Plain"; s += NL;
        s += std::to_string(v->blocks); s += NL;
        Writer w;
        if (v->enc) {
            std::vector<u64> host((size_t)v->blocks * c.ct_words());
            CNHE_CUDA(cudaMemcpyAsync(host.data(), v->ptr(ci), host.size() * 8, cudaMemcpyDeviceToHost, c.stream));
            c.sync();
            for (int b = 0; b < v->blocks; b++) write_ciphertext(w, pid, host.data() + (size_t)b * c.ct_words(), N, k, 2, false);
        } else {
            const ParmsId zero = {0};
            const size_t unit = v->unit();
            std::vector<u64> host((size_t)v->blocks * unit);
            if (v->format == CNHE_SPARSE) host = v->scalars[ci];
            else {
                CNHE_CUDA(cudaMemcpyAsync(host.data(), v->ptr(ci), host.size() * 8, cudaMemcpyDeviceToHost, c.stream));
                c.sync();
            }
            for (int b = 0; b < v->blocks; b++) { w.raw(zero, 32); w.f64(1.0); w.u64_(unit); w.raw(host.data() + (size_t)b * unit, unit * 8); }
        }
        b64_encode(w.b, s);
        s += NL;
        s += "<End EncryptedVector>"; s += NL;
    }
    s += "<End LargeEncryptedVector>"; s += NL;
    *needed = s.size();
    if (dst) {
        if (cap < s.size()) fail("destination too small");
        memcpy(dst, s.data(), s.size());
    }
    API_END
}

extern "C" int cnhe_vec_read(cnhe_ctx *h, const char *text, size_t len, cnhe_vec **out, size_t *consumed) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    if (!text || !out) fail("null argument");
    const uint64_t N = c.N, k = (uint64_t)c.k;
    Lines L(text, len);
    L.expect("<Start LargeEncryptedVector>");
    const double scale = atof(L.str().c_str());
    if (atoi(L.str().c_str()) != c.P) fail("the vector was written with a different number of plaintext moduli");
    std::unique_ptr<cnhe_vec> v;
    for (int ci = 0; ci < c.P; ci++) {
        c.set_channel(ci);
        L.expect("<Start EncryptedVector>");
        L.str(); // atomic scale (1)
        L.str(); // IsSigned
        const std::string fmt = L.str();
        const int format = fmt == "dense" ? CNHE_DENSE : (fmt == "sparse" ? CNHE_SPARSE : -1);
        if (format < 0) fail("unknown format");
        const uint64_t dim = strtoull(L.str().c_str(), nullptr, 10);
        const std::string mode = L.str();
        if (mode != "Encrypted" && mode != "Plain") fail("unknown format");
        const bool enc = mode == "Encrypted";
        const int blocks = atoi(L.str().c_str());
        if (blocks < 1) fail("Bad stream format.");
        const char *b64; size_t b64n;
        if (!L.next(b64, b64n)) fail("Bad stream format.");
        std::vector<uint8_t> blob = b64_decode(b64, b64n);
        L.expect("<End EncryptedVector>");
        if (ci == 0) {
            v.reset(new_vec(c, dim, scale, format, enc, blocks));
            if (!enc && format == CNHE_SPARSE) v->scalars.assign(c.P, std::vector<u64>());
            alloc_channels(v.get());
        } else if (v->dim != dim || v->format != format || v->enc != enc || v->blocks != blocks) fail("the channels of one vector disagree");
        Reader r(blob.data(), blob.size());
        ParmsId pid;
        compute_parms_id(N, c.q, c.ch[ci].t, pid);
        const size_t unit = v->unit();
        std::vector<u64> host((size_t)blocks * unit);
        for (int b = 0; b < blocks; b++) {
            if (enc) read_ciphertext(r, pid, host.data() + (size_t)b * unit, N, k, 2, false);
            else {
                r.need(40);
                r.p += 40; // parms_id, scale
                const uint64_t cnt = r.u64_();
                if (cnt > unit) fail("plaintext larger than the polynomial degree");
                std::fill(host.begin() + (size_t)b * unit, host.begin() + (size_t)(b + 1) * unit, 0);
                r.raw(host.data() + (size_t)b * unit, cnt * 8);
                for (uint64_t i = 0; i < cnt; i++)
                    if (host[(size_t)b * unit + i] >= c.ch[ci].t) fail("plaintext coefficient out of range");
            }
        }
        if (r.left()) fail("trailing bytes in the vector payload");
        if (!enc && format == CNHE_SPARSE) v->scalars[ci] = host;
        CNHE_CUDA(cudaMemcpyAsync(v->ptr(ci), host.data(), host.size() * 8, cudaMemcpyHostToDevice, c.stream));
        c.sync();
    }
    L.expect("<End LargeEncryptedVector>");
    if (consumed) *consumed = (size_t)(L.p - text);
    *out = v.release();
    API_END
}
