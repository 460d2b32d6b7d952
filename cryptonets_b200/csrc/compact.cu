// Compact ciphertext upload: seeded secret-key encryption with bit-packed residues, expanded on the GPU at import.
//
// Format version 1 (this library's own, little endian) -- one blob for n dense vectors of `dim` values, B = ceil(dim / N)
// ciphertext blocks per vector (as cnhe_vecs_encrypt):
//   header   "CNHC" | u32 version = 1 | u32 N | u32 k | u32 P | u32 n | u32 B | u64 dim | f64 scale | k x u64 coefficient moduli q_l |
//            P x u64 plaintext moduli t_c | P x 32-byte expansion keys K_c
//   payload  for channel c, vector i, block b, residue l: the N coefficients of c0 as a little-endian bit stream, coefficient x at bits
//            [x b_l, (x+1) b_l) with b_l = bitlen(q_l); each residue fills exactly N b_l / 64 words
//   c1       of ciphertext j = i B + b of channel c, residue l, coefficient x: floor(q_l R / 2^128), R = w[2x+1] 2^64 + w[2x], where w[m] is
//            64-bit word m of the ChaCha20 keystream under key K_c and stream id stream_id(PURPOSE_COMPACT_A, j, l): word m & 7 of block
//            m >> 3, 64-bit block counter in state words 12-13, 64-bit stream id in words 14-15 (the indexing of chacha20_word).
//            The 128-bit draw is within q_l / 2^129 of uniform per coefficient.
// A secret-key encryption is (c0, c1) = (-(a s) + e + Delta m, a) with a uniform: the client derives a from K_c and sends only c0 and K_c,
// 2.6-2.9x fewer bytes than the ciphertexts.  The server regenerates a here (k_compact_expand); every later operation sees ordinary
// ciphertexts in SEAL's layout [poly][residue][coeff].
//
// Compact evaluation keys, format version 1 (the same expansion; one blob per key set, made with cnhe_keys_save_compact):
//   header   "CNHK" | u32 version = 1 | u32 N | u32 k | u32 P | u32 dbc_relin | u32 dbc_galois | u32 sets (bit 0 public key, bit 1
//            relinearisation keys) | u32 G | k x u64 q_l | P x u64 t_c | G x u64 Galois elements (strictly increasing, each one of the
//            context's standard elements) | P x 32-byte expansion keys K_c
//   payload  for channel c, key pair kappa, residue l: the N words of part 0 (b) as the same bit stream as c0 above
//   pairs    kappa in blob order: the public key (if present), the D_r relinearisation digits, then for each listed element the D_g digits
//            of its Galois key (digit order of the decomposition map: residue-major, low bits first)
//   part 1   (a) of pair kappa, residue l, word x: floor(q_l R / 2^128) as above under stream id stream_id(PURPOSE_KEYS_A, kappa, l); a is
//            uniform in the NTT domain as well, so it is the key's NTT-form a directly
// A key pair is (b, a) = (-(a s + e) + 2^{shift_d} [target]_{src_d}, a) in NTT form -- target s^2 for relinearisation, s(x^g) for Galois
// element g, none for the public key -- with e the channel's noise sampler under stream_id(PURPOSE_KEYS_E, nonce0 + kappa, 0).  The
// server writes (b, a) straight into its key slots with k_compact_expand.
#include "kernels.h"

namespace cnhe {

#define CNHE_QRF(a, b, c, d)                                                                                           \
    a += b; d ^= a; d = __funnelshift_l(d, d, 16);                                                                     \
    c += d; b ^= c; b = __funnelshift_l(b, b, 12);                                                                     \
    a += b; d ^= a; d = __funnelshift_l(d, d, 8);                                                                      \
    c += d; b ^= c; b = __funnelshift_l(b, b, 7);

// one ChaCha20 block (the 16 output words, key and state added back) in registers
__device__ __forceinline__ void chacha20_block(const CompactKey &key, u64 blk, u64 stream, u32 x[16]) {
    const u32 s[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, key.w[0], key.w[1], key.w[2], key.w[3], key.w[4], key.w[5],
                       key.w[6],    key.w[7],    (u32)blk,    (u32)(blk >> 32), (u32)stream, (u32)(stream >> 32)};
#pragma unroll
    for (int j = 0; j < 16; j++) x[j] = s[j];
#pragma unroll
    for (int r = 0; r < 10; r++) {
        CNHE_QRF(x[0], x[4], x[8], x[12]) CNHE_QRF(x[1], x[5], x[9], x[13]) CNHE_QRF(x[2], x[6], x[10], x[14]) CNHE_QRF(x[3], x[7], x[11], x[15])
        CNHE_QRF(x[0], x[5], x[10], x[15]) CNHE_QRF(x[1], x[6], x[11], x[12]) CNHE_QRF(x[2], x[7], x[8], x[13]) CNHE_QRF(x[3], x[4], x[9], x[14])
    }
#pragma unroll
    for (int j = 0; j < 16; j++) x[j] += s[j];
}
// floor(q (r_hi 2^64 + r_lo) / 2^128) = high word of q r_hi + umulhi(q, r_lo)
__device__ __forceinline__ u64 draw128(u64 q, u64 r_lo, u64 r_hi) {
    u64 lo = q * r_hi, hi = __umul64hi(q, r_hi);
    const u64 t = __umul64hi(q, r_lo);
    asm("add.cc.u64 %0, %0, %2;\n\taddc.u64 %1, %1, 0;" : "+l"(lo), "+l"(hi) : "l"(t));
    return hi;
}

// sh.bits[l] / sh.off[l] by unrolled selection: a dynamic index into the parameter struct would copy it to the stack
__device__ __forceinline__ int shape_bits(const CompactShape &sh, int l) {
    int b = 0;
#pragma unroll
    for (int t = 0; t < KMAX; t++) b = t == l ? sh.bits[t] : b;
    return b;
}
__device__ __forceinline__ u64 shape_off(const CompactShape &sh, int l) {
    u64 o = 0;
#pragma unroll
    for (int t = 0; t <= KMAX; t++) o = t == l ? sh.off[t] : o;
    return o;
}

// One thread per (ciphertext j, residue l, ChaCha20 block g): coefficients 4g..4g+3 of c1 from the block, and the same coefficients of c0
// unpacked from the payload (packed == null: c0 is left alone -- the client's draw of a).  ct [n][2][k][N]; packed [n][sum_l N b_l / 64].
__global__ void __launch_bounds__(256) k_compact_expand(u64 *__restrict__ ct, const u64 *__restrict__ packed, CompactKey key, u64 purpose, u64 j0,
                                                       int n, CompactShape sh, const BehzConst *__restrict__ bc) {
    const int k = sh.k, logn = sh.logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)n * k) << (logn - 2)) return;
    const u32 g = (u32)(i & ((1u << (logn - 2)) - 1));
    const size_t jl = i >> (logn - 2);
    const int l = (int)(jl % k);
    const size_t j = jl / k;
    const u64 q = bc->q[l].p;
    u32 x[16];
    chacha20_block(key, g, stream_id(purpose, j0 + j, (u64)l), x);
    const size_t kN = (size_t)k << logn;
    u64 *c1 = ct + (2 * j + 1) * kN + ((size_t)l << logn) + 4 * (size_t)g;
    u64 v[4];
#pragma unroll
    for (int t = 0; t < 4; t++)
        v[t] = draw128(q, ((u64)x[4 * t + 1] << 32) | x[4 * t], ((u64)x[4 * t + 3] << 32) | x[4 * t + 2]);
    reinterpret_cast<ulonglong2 *>(c1)[0] = make_ulonglong2(v[0], v[1]);
    reinterpret_cast<ulonglong2 *>(c1)[1] = make_ulonglong2(v[2], v[3]);
    if (!packed) return;
    const int b = shape_bits(sh, l);
    const u64 mask = b == 64 ? ~0ULL : (1ULL << b) - 1;
    const u64 *src = packed + j * shape_off(sh, k) + shape_off(sh, l);
#pragma unroll
    for (int t = 0; t < 4; t++) {
        const u64 bit = (u64)(4 * g + t) * b;
        const u64 w = bit >> 6;
        const int s = (int)(bit & 63);
        u64 r = __ldg(src + w) >> s;
        if (s + b > 64) r |= __ldg(src + w + 1) << (64 - s);
        r &= mask;
        v[t] = r >= q ? r - q : r; // r < 2^b < 2q: one subtraction makes any payload word canonical
    }
    u64 *c0 = c1 - kN;
    reinterpret_cast<ulonglong2 *>(c0)[0] = make_ulonglong2(v[0], v[1]);
    reinterpret_cast<ulonglong2 *>(c0)[1] = make_ulonglong2(v[2], v[3]);
}

// One thread per output word: the (at most 3 for b >= 33) coefficients of c0 that overlap it are gathered, so the writes are coalesced.
__global__ void __launch_bounds__(256) k_pack_residues(const u64 *__restrict__ ct, u64 *__restrict__ packed, int n, CompactShape sh) {
    const int k = sh.k, logn = sh.logn;
    const size_t W = shape_off(sh, k);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * W) return;
    const size_t j = i / W, r = i % W;
    int l = 0;
#pragma unroll
    for (int t = 1; t < KMAX; t++) l = t < k && sh.off[t] <= r ? t : l;
    const int b = shape_bits(sh, l);
    const u64 bit0 = (u64)(r - shape_off(sh, l)) << 6;
    const u64 *c0 = ct + j * ((size_t)2 * k << logn) + ((size_t)l << logn);
    u64 out = 0;
    for (u64 x = bit0 / b; x < (1ULL << logn) && x * b < bit0 + 64; x++) {
        const u64 v = __ldg(c0 + x);
        const long long d = (long long)(x * b) - (long long)bit0;
        out |= d >= 0 ? v << d : v >> -d;
    }
    packed[i] = out;
}

cudaError_t launch_compact_expand(u64 *ct, const u64 *packed, const CompactKey &key, u64 purpose, u64 j0, int n, const CompactShape &sh,
                                  const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const size_t threads = ((size_t)n * sh.k) << (sh.logn - 2);
    k_compact_expand<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(ct, packed, key, purpose, j0, n, sh, bc);
    return cudaGetLastError();
}
cudaError_t launch_pack_residues(const u64 *ct, u64 *packed, int n, const CompactShape &sh, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const size_t threads = (size_t)n * sh.off[sh.k];
    k_pack_residues<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(ct, packed, n, sh);
    return cudaGetLastError();
}

} // namespace cnhe
