// Device-side 64-bit modular arithmetic for the BFV hot path (sm_90a).
// Integer pipes only: 64x64->128 products are IMAD.WIDE chains; there is no tensor-core formulation of a
// modular 64-bit butterfly.  All routines return canonical residues unless the name says "lazy".
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace cnhe {

typedef unsigned long long u64;
typedef unsigned int u32;

// One modulus as the kernels see it: p and floor(2^128/p) (two words), p < 2^62.
struct DMod {
    u64 p, r0, r1;
};

struct U128 {
    u64 lo, hi;
};

__device__ __forceinline__ U128 mul64wide(u64 a, u64 b) {
    U128 r;
    r.lo = a * b;
    r.hi = __umul64hi(a, b);
    return r;
}
// acc += a*b (128-bit)
__device__ __forceinline__ void mac128(U128 &acc, u64 a, u64 b) {
    u64 lo = a * b, hi = __umul64hi(a, b);
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, %3;" : "+l"(acc.lo), "+l"(acc.hi) : "l"(lo), "l"(hi));
}
__device__ __forceinline__ void add128(U128 &acc, u64 v) {
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, 0;" : "+l"(acc.lo), "+l"(acc.hi) : "l"(v));
}
// x mod p for x < 2^128 (Barrett with floor(2^128/p)); one conditional subtraction at the end.
__device__ __forceinline__ u64 barrett128(U128 x, const DMod &m) {
    u64 a = __umul64hi(x.lo, m.r0);
    u64 b_lo = x.lo * m.r1, b_hi = __umul64hi(x.lo, m.r1);
    u64 c_lo = x.hi * m.r0, c_hi = __umul64hi(x.hi, m.r0);
    u64 carry;
    // carry out of a + b_lo + c_lo
    asm("{\n\t.reg .u64 t;\n\tadd.cc.u64 t, %1, %2;\n\taddc.u64 %0, 0, 0;\n\tadd.cc.u64 t, t, %3;\n\taddc.u64 %0, %0, 0;\n\t}"
        : "=l"(carry)
        : "l"(a), "l"(b_lo), "l"(c_lo));
    u64 q = x.hi * m.r1 + b_hi + c_hi + carry;
    u64 r = x.lo - q * m.p;
    return r >= m.p ? r - m.p : r;
}
__device__ __forceinline__ u64 mulmod(u64 a, u64 b, const DMod &m) { return barrett128(mul64wide(a, b), m); }
__device__ __forceinline__ u64 addmod(u64 a, u64 b, u64 p) {
    u64 s = a + b;
    return s >= p ? s - p : s;
}
__device__ __forceinline__ u64 submod(u64 a, u64 b, u64 p) { return a >= b ? a - b : a + p - b; }
__device__ __forceinline__ u64 negmod(u64 a, u64 p) { return a ? p - a : 0; }
// x mod p for a 64-bit x (x may exceed p by any amount)
__device__ __forceinline__ u64 reduce64(u64 x, const DMod &m) {
    u64 q = __umul64hi(x, m.r1); // >= floor(x/p) - 2 (the r0 word of the ratio is dropped)
    u64 r = x - q * m.p;
    r = r >= 2 * m.p ? r - 2 * m.p : r;
    return r >= m.p ? r - m.p : r;
}
// Shoup multiplication: w fixed with ws = floor(w 2^64 / p); result in [0, 2p) for any 64-bit x.
__device__ __forceinline__ u64 mul_shoup_lazy(u64 x, u64 w, u64 ws, u64 p) {
    u64 q = __umul64hi(ws, x);
    return w * x - q * p;
}

// ---- randomness.  Two generators behind one interface (RngKey):
//  * secure (default): ChaCha20 keyed with 256 bits of OS entropy (getrandom) drawn per channel when the context is created and again at
//    every cnhe_keys_generate_secure; block counter = index / 8, nonce = 64-bit stream id.  This is what SEAL's std::random_device-seeded
//    sampler provides the reference: secret key, key-switching masks and the encryption randomness (u, e0, e1) are unpredictable.
//  * deterministic (tests only, explicit seed): the counter-based splitmix64 sampler shared with the CPU oracle, so that keys and fresh
//    ciphertexts are bit-comparable.  splitmix64 is an invertible mixer, NOT a cipher: never use a seeded context for real data.
__host__ __device__ __forceinline__ u64 splitmix64(u64 x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
struct RngKey {
    u32 key[8]; // ChaCha20 key (secure mode)
    u64 seed;   // deterministic mode
    int secure, pad_;
};
__host__ __device__ __forceinline__ u32 rotl32(u32 v, int c) { return (v << c) | (v >> (32 - c)); }
#define CNHE_QR(a, b, c, d)                                                                                            \
    a += b; d ^= a; d = rotl32(d, 16);                                                                                 \
    c += d; b ^= c; b = rotl32(b, 12);                                                                                 \
    a += b; d ^= a; d = rotl32(d, 8);                                                                                  \
    c += d; b ^= c; b = rotl32(b, 7);
// word `i & 7` (64-bit) of ChaCha20 block `i >> 3` under nonce `stream`
__host__ __device__ __forceinline__ u64 chacha20_word(const RngKey &rk, u64 stream, u64 i) {
    const u64 blk = i >> 3;
    u32 s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, rk.key[0], rk.key[1], rk.key[2], rk.key[3], rk.key[4], rk.key[5],
                 rk.key[6],   rk.key[7],   (u32)blk,    (u32)(blk >> 32), (u32)stream, (u32)(stream >> 32)};
    u32 x[16];
#pragma unroll
    for (int j = 0; j < 16; j++) x[j] = s[j];
#pragma unroll 1
    for (int r = 0; r < 10; r++) {
        CNHE_QR(x[0], x[4], x[8], x[12]) CNHE_QR(x[1], x[5], x[9], x[13]) CNHE_QR(x[2], x[6], x[10], x[14]) CNHE_QR(x[3], x[7], x[11], x[15])
        CNHE_QR(x[0], x[5], x[10], x[15]) CNHE_QR(x[1], x[6], x[11], x[12]) CNHE_QR(x[2], x[7], x[8], x[13]) CNHE_QR(x[3], x[4], x[9], x[14])
    }
    const int w = (int)(i & 7) * 2;
    u32 lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 16; j += 2)
        if (j == w) { lo = x[j] + s[j]; hi = x[j + 1] + s[j + 1]; }
    return ((u64)hi << 32) | lo;
}
__host__ __device__ __forceinline__ u64 rng64(u64 seed, u64 stream, u64 i) {
    return splitmix64(splitmix64(seed ^ (stream * 0xD1342543DE82EF95ULL)) + i);
}
__host__ __device__ __forceinline__ u64 rng64(const RngKey &rk, u64 stream, u64 i) {
    return rk.secure ? chacha20_word(rk, stream, i) : rng64(rk.seed, stream, i);
}
__host__ __device__ __forceinline__ u64 stream_id(u64 purpose, u64 a, u64 b) { return (purpose << 48) | (a << 16) | b; }

} // namespace cnhe
