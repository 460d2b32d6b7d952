// Values in and out of the plaintext channels on the GPU: the split of doubles into residues (the wrapper's SplitBigNumbers) fused into
// the encode scatter, and the CRT join of decrypted residues back into doubles (JoinSplitNumbers).  Both restate the host arithmetic bit
// for bit; DESIGN 4.19 gives the rules and tests/values_ref.py restates them with Python integers.
#include "kernels.h"

namespace cnhe {

typedef unsigned __int128 u128;

static inline unsigned blocks_for(size_t threads, int per = 256) { return (unsigned)((threads + per - 1) / per); }

// |w| of an integral double below 2^127, exactly
__device__ __forceinline__ u128 integral_magnitude(double w) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(w) & 0x7fffffffffffffffULL;
    if (bits == 0) return 0;
    const int e = (int)(bits >> 52) - 1075;
    const u128 mant = (u128)((bits & 0xfffffffffffffULL) | (1ULL << 52));
    return e >= 0 ? mant << e : mant >> -e; // w integral: the bits shifted out are zero
}

// the residue mod t of one value: w = rint(v scale) (one IEEE product, ties to even), |w| < 1.5e38, mag = |w| mod B, z = B - mag for
// negative non-zero w; out of range sets *bad
__device__ __forceinline__ u64 split_residue(double v, double scale, u128 big, u64 t, int *bad) {
    const double w = rint(__dmul_rn(v, scale));
    if (!(fabs(w) < 1.5e38)) {
        *bad = 1;
        return 0;
    }
    u128 mag = integral_magnitude(w);
    if (mag >= big) mag %= big;
    const u128 z = (w < 0 && mag) ? big - mag : mag;
    return (u64)(z % t);
}

// dense: plain[c][index_map[j]] = residue of value b N + j of vector i = c / bl, block b = c % bl (zero past dim); sparse (index_map
// null): plain[j] = residue of value j, j < count
__global__ void __launch_bounds__(256) k_split_scatter(const double *__restrict__ values, u64 *__restrict__ plain, u64 count, u64 dim, int bl,
                                                      double scale, u128 big, u64 t, const u32 *__restrict__ index_map, int logn, int *bad) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    if (!index_map) {
        plain[i] = split_residue(values[i], scale, big, t, bad);
        return;
    }
    const int N = 1 << logn, j = (int)(i & (N - 1));
    const size_t c = i >> logn, vec = c / bl, e = (c % bl) * N + j;
    plain[c * N + index_map[j]] = e < dim ? split_residue(values[vec * dim + e], scale, big, t, bad) : 0;
}

cudaError_t launch_split_scatter(const double *values, u64 *plain, int n_ct, int bl, u64 dim, double scale, u128 big, u64 t, const u32 *index_map,
                                 int logn, int *bad, cudaStream_t s) {
    const u64 count = index_map ? (u64)n_ct << logn : dim;
    if (!count) return cudaSuccess;
    k_split_scatter<<<blocks_for(count), 256, 0, s>>>(values, plain, count, dim, bl, scale, big, t, index_map, logn, bad);
    return cudaGetLastError();
}

// ct_tab[i] = (c0, c1) [2][kN] -> c0[i], c1[i] [kN] each
__global__ void __launch_bounds__(256) k_split_parts(const u64 *const *__restrict__ ct_tab, u64 *__restrict__ c0, u64 *__restrict__ c1, size_t kN,
                                                    size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t c = i / kN, x = i % kN;
    const u64 *src = ct_tab[c];
    c0[i] = src[x];
    c1[i] = src[kN + x];
}
cudaError_t launch_split_parts(const u64 *const *ct_tab, u64 *c0, u64 *c1, int n, size_t kN, cudaStream_t s) {
    const size_t total = (size_t)n * kN;
    if (!total) return cudaSuccess;
    k_split_parts<<<blocks_for(total), 256, 0, s>>>(ct_tab, c0, c1, kN, total);
    return cudaGetLastError();
}

// a b mod m for a < m < 2^126, b < 2^64: shift and add, each partial sum below 2^127
__device__ __forceinline__ u128 mulmod_u128(u128 a, u64 b, u128 m) {
    u128 r = 0;
    while (b) {
        if (b & 1) {
            r += a;
            if (r >= m) r -= m;
        }
        a += a;
        if (a >= m) a -= m;
        b >>= 1;
    }
    return r;
}
// x as a double, rounded to nearest with ties to even (as GCC's __floatuntidf): the top 64 bits with every lower bit folded into a sticky
// bit 0, which lies below the rounding position of a 64-bit integer, then one correctly rounded conversion and an exact power-of-two scale
__device__ __forceinline__ double u128_to_double_rn(u128 x) {
    const u64 hi = (u64)(x >> 64);
    if (!hi) return __ull2double_rn((u64)x);
    const int shift = 64 - __clzll((long long)hi); // bits above the low 64
    const u64 top = (u64)(x >> shift) | (((x & (((u128)1 << shift) - 1)) != 0) ? 1 : 0);
    return ldexp(__ull2double_rn(top), shift);
}

// out[i][j] = centred CRT join of the P residues of value j of vector i, over scale[i]
__global__ void __launch_bounds__(256) k_crt_join(const JoinSrc *__restrict__ src, double *__restrict__ out, int n, u64 dim, JoinConst jc) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * dim) return;
    const size_t v = i / dim, j = i % dim;
    u128 acc = 0;
    const u128 big = ((u128)jc.big_hi << 64) | jc.big_lo;
    for (int ch = 0; ch < jc.P; ch++) {
        const JoinSrc s = src[(size_t)ch * n + v];
        const u64 r = j < s.count ? s.p[j * s.stride] : 0;
        acc += mulmod_u128(((u128)jc.coeff_hi[ch] << 64) | jc.coeff_lo[ch], r, big);
        if (acc >= big) acc -= big;
    }
    const double val = acc * 2 > big ? -u128_to_double_rn(big - acc) : u128_to_double_rn(acc);
    out[i] = __ddiv_rn(val, src[v].scale);
}
cudaError_t launch_crt_join(const JoinSrc *src, double *out, int n, u64 dim, const JoinConst &jc, cudaStream_t s) {
    const size_t total = (size_t)n * dim;
    if (!total) return cudaSuccess;
    k_crt_join<<<blocks_for(total), 256, 0, s>>>(src, out, n, dim, jc);
    return cudaGetLastError();
}

} // namespace cnhe
