// K3/K4/K7/K8/K9/K10 element-wise kernels of the BFV hot path (sm_90a): ciphertext add/sub/negate/add-many, plain add,
// constant-plaintext scaling, dyadic products, the Galois coefficient permutation, the scalar multiply-accumulate layer
// (CryptoNets conv/dense), sampling, BatchEncoder scatter/gather.
//
// Reference call sites (/root/reference "HE Wrapper/AtomicSealBfvVector.cs"): Add/AddMany :491,:502,:917,:1005;
// AddPlain/SubPlain :1019,:1267; MultiplyPlain (constant plaintext) :472; RotateRows/Columns :625-660,:864,:914;
// BatchEncoder :1130,:1050; Encryptor :1211.  SEAL 3.2 routines replaced: add_poly_poly_coeffmod,
// Encryptor::preencrypt, negacyclic_multiply_poly_mono_coeffmod (exponent 0), dyadic_product_coeffmod,
// util::apply_galois, BatchEncoder::encode/decode index map.
// All are HBM-bound streaming kernels except the MAC layer, which is integer-ALU bound (DESIGN.md section 5).
#include "fparith.cuh"
#include "kernels.h"
#include "plainops.cuh"

namespace cnhe {

static inline unsigned blocks_for(size_t threads, int per = 256) { return (unsigned)((threads + per - 1) / per); }

__device__ __forceinline__ u64 q_of(const BehzConst *bc, int l) { return bc->q[l].p; }

// ---------------------------------------------------------------- ct +/- ct, negate, add-many
__global__ void __launch_bounds__(256) k_ct_addsub(const u64 *a, const u64 *b, u64 *out, size_t words, int k, int logn,
                                                  const BehzConst *__restrict__ bc, int sub) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    const u64 p = q_of(bc, (int)((i >> logn) % k));
    out[i] = sub ? submod(a[i], b[i], p) : addmod(a[i], b[i], p);
}
// out[c] = a[c] + E.x[c] on both polynomials, + Delta C on c0 as the floor epilogue adds it (E.c at coefficient 0, or the ciphertext's
// E.c_poly plaintext): n size-2 ciphertexts, the cubic activation's q1 = u + x + gamma (cnhe_layer_poly).  E.a and E.b are not used
__global__ void __launch_bounds__(256) k_ct_add_epi(const u64 *a, u64 *out, int n, int k, int logn, const BehzConst *__restrict__ bc,
                                                   const __grid_constant__ FloorEpi E) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t N = (size_t)1 << logn, per = 2 * (size_t)k * N;
    if (i >= (size_t)n * per) return;
    const size_t c = i / per, w = i % per;
    const int l = (int)((w >> logn) % k), x = (int)(w & (N - 1));
    const u64 p = q_of(bc, l);
    u64 v = addmod(a[i], E.x[c][w], p);
    if (w < (size_t)k * N) { // c0
        const u64 *cs = E.c_poly ? E.c_poly[c] : nullptr;
        if (cs) v = addmod(v, cs[w], p);
        else if (x == 0) v = addmod(v, E.c[l], p);
    }
    out[i] = v;
}
__global__ void __launch_bounds__(256) k_ct_negate(const u64 *a, u64 *out, size_t words, int k, int logn, const BehzConst *__restrict__ bc) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    out[i] = negmod(a[i], q_of(bc, (int)((i >> logn) % k)));
}
__global__ void __launch_bounds__(256) k_ct_add_many(const u64 *const *__restrict__ in, int n_in, u64 *out, size_t words, int k, int logn,
                                                    const BehzConst *__restrict__ bc) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= words) return;
    const u64 p = q_of(bc, (int)((i >> logn) % k));
    u64 acc = in[0][i];
    for (int j = 1; j < n_in; j++) acc = addmod(acc, in[j][i], p);
    out[i] = acc;
}

// ---------------------------------------------------------------- Delta*m helpers (scale_plain: plainops.cuh)
__device__ __forceinline__ u64 lift_plain(u64 m, u64 q, const PlainConst &pc) { return m >= pc.threshold ? m + (q - pc.t) : m; }

__global__ void __launch_bounds__(256) k_ct_add_plain(const u64 *ct, u64 *out, int n, int size, const u64 *__restrict__ plain,
                                                     size_t plain_stride, int coeffs, int k, int logn, const BehzConst *__restrict__ bc,
                                                     PlainConst pc, int sub) {
    const int N = 1 << logn;
    const size_t per_ct = (size_t)size * k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= per_ct * n) return;
    const size_t c = i / per_ct, r = i % per_ct;
    u64 v = ct[i];
    if (r < (size_t)k * N) { // c0 only
        const int l = (int)(r >> logn), x = (int)(r & (N - 1));
        if (x < coeffs) {
            const u64 m = plain[c * plain_stride + x];
            if (m) {
                const DMod q = bc->q[l];
                const u64 sc = scale_plain(m, l, q, pc);
                v = sub ? submod(v, sc, q.p) : addmod(v, sc, q.p);
            }
        }
    }
    out[i] = v;
}
__global__ void __launch_bounds__(256) k_ct_scale(const u64 *in, u64 *out, int n, int size, const u64 *__restrict__ scalars, int k, int logn,
                                                 const BehzConst *__restrict__ bc, PlainConst pc) {
    const int N = 1 << logn;
    const size_t per_ct = (size_t)size * k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= per_ct * n) return;
    const size_t c = i / per_ct;
    const int l = (int)((i >> logn) % k);
    const DMod q = bc->q[l];
    out[i] = mulmod(in[i], lift_plain(scalars[c], q.p, pc), q);
}
__global__ void __launch_bounds__(256) k_plain_lift(const u64 *__restrict__ plain, u64 *__restrict__ lifted, int n, int coeffs, int k, int logn,
                                                   const BehzConst *__restrict__ bc, PlainConst pc) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)n * k) << logn) return;
    const int x = (int)(i & (N - 1)), l = (int)((i >> logn) % k);
    const size_t c = (i >> logn) / k;
    const u64 m = x < coeffs ? plain[c * N + x] : 0;
    lifted[i] = lift_plain(m, bc->q[l].p, pc);
}
__global__ void __launch_bounds__(256) k_dyadic_bcast(const u64 *a, const u64 *b, u64 *out, int n, int size, int a_per_ct, int b_per_ct, int k,
                                                     int logn, const BehzConst *__restrict__ bc) {
    const int N = 1 << logn;
    const size_t kN = (size_t)k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * size * kN) return;
    const size_t c = i / (size * kN), r = i % kN;
    const int l = (int)(r >> logn);
    out[i] = mulmod(a[a_per_ct ? i : i % (size * kN)], b[(b_per_ct ? c : 0) * kN + r], bc->q[l]);
}
// out[b * out_rows + r][p][l][i] = ct[b][p][l][i] * pl[r][l][i]  (NTT form, canonical in and out; every q_l < 2^50).  One thread per
// (r, l, i) loads the plaintext word once and multiplies it into CB clients' two polynomials (B > CB: once per CB clients).  The CTAs of one (l, coefficient
// tile) are consecutive over r, so the R rows read the same ciphertext words at about the same time, from L2.  fmodmul of canonical
// operands is congruent to the product and within (-q, q); re-centred and made canonical it is the unique residue mulmod gives.
template <int CB>
__global__ void __launch_bounds__(256) k_dyadic_outer(const u64 *__restrict__ ct, const u64 *__restrict__ pl, u64 *__restrict__ out, int B, int R,
                                                     int out_rows, int logn, const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k, tiles = N >> 8;
    const int r = blockIdx.x % R, tile = (blockIdx.x / R) % tiles, l = blockIdx.x / (R * tiles);
    const int i = (tile << 8) + threadIdx.x;
    const double p = F.qd[l], pinv = F.qinv[l];
    const size_t kN = (size_t)k * N, ctw = 2 * kN, at = (size_t)l * N + i;
    const double d = u2d(pl[(size_t)r * kN + at]);
    for (int b0 = 0; b0 < B; b0 += CB) {
        double x[CB][2];
#pragma unroll
        for (int cb = 0; cb < CB; cb++)
            if (b0 + cb < B) {
                x[cb][0] = u2d(ct[(size_t)(b0 + cb) * ctw + at]);
                x[cb][1] = u2d(ct[(size_t)(b0 + cb) * ctw + kN + at]);
            }
#pragma unroll
        for (int cb = 0; cb < CB; cb++) {
            if (b0 + cb >= B) break;
            u64 *o = out + ((size_t)(b0 + cb) * out_rows + r) * ctw + at;
            o[0] = fsmall_u(frecenter(fmodmul(x[cb][0], d, p, pinv), p, pinv), F.q_u[l]);
            o[kN] = fsmall_u(frecenter(fmodmul(x[cb][1], d, p, pinv), p, pinv), F.q_u[l]);
        }
    }
}

// ---------------------------------------------------------------- Galois permutation (gather form)
// add_back: the base of the key switch also carries the UNROTATED ciphertext (c0 + perm(c0), c1), so that key switch + base == x + rotate(x):
// one step of the rotate-and-sum ladder (SumAllSlots) without a separate addition pass
__global__ void __launch_bounds__(256) k_galois(const u64 *__restrict__ in, const u64 *const *__restrict__ in_ptrs, u64 *__restrict__ out_base,
                                               u64 *__restrict__ perm_c1, int n, u64 elt_inv, int k, int logn, const BehzConst *__restrict__ bc,
                                               int add_back) {
    const int N = 1 << logn;
    const size_t kN = (size_t)k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * 2 * kN) return;
    const size_t c = i / (2 * kN), r = i % (2 * kN);
    const int part = (int)(r / kN), l = (int)((r % kN) >> logn), j = (int)(r & (N - 1));
    const u64 raw = ((u64)j * elt_inv) & (2 * (u64)N - 1);
    const int src = (int)(raw & (N - 1));
    const u64 *ct = in_ptrs ? in_ptrs[c] : in + c * 2 * kN; // gathered inputs (batched rotations of scattered ciphertexts) or a packed array
    u64 v = ct[(size_t)part * kN + (size_t)l * N + src];
    if (raw >> logn) v = negmod(v, bc->q[l].p);
    if (part == 0) {
        if (add_back) {
            out_base[c * 2 * kN + (size_t)l * N + j] = addmod(v, ct[(size_t)l * N + j], bc->q[l].p);
            out_base[c * 2 * kN + kN + (size_t)l * N + j] = ct[kN + (size_t)l * N + j];
        } else {
            out_base[c * 2 * kN + (size_t)l * N + j] = v;
            out_base[c * 2 * kN + kN + (size_t)l * N + j] = 0;
        }
    } else {
        perm_c1[c * kN + (size_t)l * N + j] = v;
    }
}

// ---------------------------------------------------------------- K4: scalar multiply-accumulate layer
// One CTA column handles 2 consecutive words of the 2kN-word ciphertext per thread; blockIdx.y walks tiles of up to
// 8 outputs that share one gather row, so every input word is loaded once per tile and reused 8 times from registers.
// Accumulation is exact 128-bit (weights are lifted residues < q_l < 2^62, K*q^2 < 2^128 is checked on the host),
// with one Barrett reduction per output word.
constexpr int MAC_TM = 8;
__global__ void __launch_bounds__(128) k_mac_layer(const u64 *const *__restrict__ in_ptrs, const int *__restrict__ gather,
                                                  const MacTile *__restrict__ tiles, const u64 *const *__restrict__ w_ptrs,
                                                  const u64 *__restrict__ bias, int K, u64 *const *__restrict__ out_ptrs, int polys, int k,
                                                  int logn, const BehzConst *__restrict__ bc, PlainConst pc) {
    const int N = 1 << logn;
    const size_t word = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; // two words per thread (16-byte accesses)
    const size_t ct_words = (size_t)polys * k * N;
    if (word >= ct_words) return;
    const MacTile tile = tiles[blockIdx.y];
    const int l = (int)((word >> logn) % k);
    const int *grow = gather + (size_t)tile.gather_row * K;
    const DMod q = bc->q[l];
    const u64 lift = q.p - pc.t;
    const u64 *wrow[MAC_TM];
#pragma unroll
    for (int m = 0; m < MAC_TM; m++) wrow[m] = m < tile.n_out ? w_ptrs[tile.out_index[m]] : nullptr;
    U128 acc[MAC_TM][2];
#pragma unroll
    for (int m = 0; m < MAC_TM; m++) acc[m][0] = acc[m][1] = U128{0, 0};
    for (int kk = 0; kk < K; kk++) {
        const int g = grow[kk];
        if (g < 0) continue;
        const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(in_ptrs[g] + word);
#pragma unroll
        for (int m = 0; m < MAC_TM; m++) {
            if (m < tile.n_out) {
                u64 w = __ldg(wrow[m] + kk);
                w += w >= pc.threshold ? lift : 0; // plain_upper_half_increment: negative weights become q_l - |w|
                mac128(acc[m][0], v.x, w);
                mac128(acc[m][1], v.y, w);
            }
        }
    }
    const bool c0_first = bias && word < (size_t)k * N && (word & (N - 1)) == 0; // constant coefficient of c0
#pragma unroll
    for (int m = 0; m < MAC_TM; m++) {
        if (m < tile.n_out) {
            const int o = tile.out_index[m];
            u64 r0 = barrett128(acc[m][0], q), r1 = barrett128(acc[m][1], q);
            if (c0_first) {
                const u64 b = bias[o];
                if (b) r0 = addmod(r0, scale_plain(b, l, q, pc), q.p);
            }
            *reinterpret_cast<ulonglong2 *>(out_ptrs[o] + word) = make_ulonglong2(r0, r1);
        }
    }
}

// FP64 variant for small weights (|w| < 2^17, K*|w|*2^26 < 2^52 checked on the host): every ciphertext word is split into two
// 26-bit halves and w*x is accumulated exactly in doubles -- 2 DFMA per multiply-accumulate instead of a 64x64->128 integer
// product (mul.hi.u64 issues at a fraction of the DFMA rate: tools/pipe_bench.cu).
// The result sum_k w_k x_k is then reduced once, so the output is the same canonical residue as the integer path.
__device__ __forceinline__ double mac_u2d(u64 x) { return __dsub_rn(__longlong_as_double((long long)(x | 0x4330000000000000ULL)), 4503599627370496.0); }
__device__ __forceinline__ u64 mac_signed_reduce(double lo, double hi, const DMod &q) { // value = lo + hi * 2^26, both exact integers
    const long long a = __double2ll_rn(lo), b = __double2ll_rn(hi);
    __int128 s = (__int128)a + ((__int128)b << 26);
    const bool neg = s < 0;
    unsigned __int128 mag = neg ? (unsigned __int128)(-s) : (unsigned __int128)s;
    U128 m;
    m.lo = (u64)mag;
    m.hi = (u64)(mag >> 64);
    const u64 r = barrett128(m, q);
    return neg ? negmod(r, q.p) : r;
}
constexpr int MAC_KC = 64; // taps staged per chunk (pointers + weights in shared memory)
constexpr int MAC_U = 8;   // loads in flight per thread
__global__ void __launch_bounds__(128) k_mac_layer_fp(const u64 *const *__restrict__ in_ptrs, const int *__restrict__ gather,
                                                     const MacTile *__restrict__ tiles, const double *__restrict__ wd, const u64 *__restrict__ bias,
                                                     int K, u64 *const *__restrict__ out_ptrs, int polys, int k, int logn,
                                                     const BehzConst *__restrict__ bc, PlainConst pc) {
    __shared__ const u64 *sptr[MAC_KC];
    __shared__ double sw[MAC_KC][MAC_TM];
    const int N = 1 << logn;
    const size_t word = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    const size_t ct_words = (size_t)polys * k * N;
    const bool active = word < ct_words;
    const size_t w_off = active ? word : 0;
    const MacTile tile = tiles[blockIdx.y];
    const int l = (int)((w_off >> logn) % k);
    const int *grow = gather + (size_t)tile.gather_row * K;
    double a0[MAC_TM][2], a1[MAC_TM][2];
#pragma unroll
    for (int m = 0; m < MAC_TM; m++) a0[m][0] = a0[m][1] = a1[m][0] = a1[m][1] = 0.0;
    for (int k0 = 0; k0 < K; k0 += MAC_KC) {
        const int kc = min(MAC_KC, K - k0);
        __syncthreads();
        // stage this chunk: padded taps (gather < 0) become a valid pointer with zero weights, so the inner loop is branch free
        for (int i = threadIdx.x; i < MAC_KC; i += blockDim.x) {
            const int g = i < kc ? grow[k0 + i] : -1;
            sptr[i] = in_ptrs[g < 0 ? 0 : g];
        }
        for (int i = threadIdx.x; i < MAC_KC * MAC_TM; i += blockDim.x) {
            const int kk = i / MAC_TM, m = i % MAC_TM;
            const bool live = kk < kc && m < tile.n_out && grow[k0 + kk] >= 0;
            sw[kk][m] = live ? wd[(size_t)tile.out_index[m] * K + k0 + kk] : 0.0;
        }
        __syncthreads();
        for (int kk = 0; kk < MAC_KC; kk += MAC_U) {
            if (kk >= kc) break;
            ulonglong2 v[MAC_U];
#pragma unroll
            for (int u = 0; u < MAC_U; u++) v[u] = *reinterpret_cast<const ulonglong2 *>(sptr[kk + u] + w_off);
#pragma unroll
            for (int u = 0; u < MAC_U; u++) {
                const double x0 = mac_u2d(v[u].x & 0x3ffffffULL), x1 = mac_u2d(v[u].x >> 26);
                const double y0 = mac_u2d(v[u].y & 0x3ffffffULL), y1 = mac_u2d(v[u].y >> 26);
#pragma unroll
                for (int m = 0; m < MAC_TM; m++) {
                    const double w = sw[kk + u][m];
                    a0[m][0] = __fma_rn(w, x0, a0[m][0]);
                    a1[m][0] = __fma_rn(w, x1, a1[m][0]);
                    a0[m][1] = __fma_rn(w, y0, a0[m][1]);
                    a1[m][1] = __fma_rn(w, y1, a1[m][1]);
                }
            }
        }
    }
    if (!active) return;
    const DMod q = bc->q[l];
    const bool c0_first = bias && word < (size_t)k * N && (word & (N - 1)) == 0;
#pragma unroll
    for (int m = 0; m < MAC_TM; m++) {
        if (m < tile.n_out) {
            const int o = tile.out_index[m];
            u64 r0 = mac_signed_reduce(a0[m][0], a1[m][0], q), r1 = mac_signed_reduce(a0[m][1], a1[m][1], q);
            if (c0_first) {
                const u64 b = bias[o];
                if (b) r0 = addmod(r0, scale_plain(b, l, q, pc), q.p);
            }
            *reinterpret_cast<ulonglong2 *>(out_ptrs[o] + word) = make_ulonglong2(r0, r1);
        }
    }
}

// ---------------------------------------------------------------- sampling (counter-based, shared with the oracle)
__constant__ u64 NOISE_CDF[19] = {0xff141e3023416d2ULL,  0x2e4f850f76b8d9a6ULL, 0x488c5acec8fd6db3ULL, 0x5d1ca569fc3e4ccbULL, 0x6bbb5699bdd65b9cULL,
                                  0x75291bf8371e7eccULL, 0x7aad3cf138611a69ULL, 0x7d9aa4d4ab7c76bdULL, 0x7f0368341f79807cULL, 0x7fa0f21e3a554470ULL,
                                  0x7fdf5971c6494be2ULL, 0x7ff5c5a33f74a4e1ULL, 0x7ffd148ddcc40605ULL, 0x7fff3db0052c58c3ULL, 0x7fffd206471c7fcfULL,
                                  0x7ffff61ba7b56e58ULL, 0x7ffffe11d76ecb8aULL, 0x7fffffa9c1e61510ULL, 0x7ffffff3ceaa701fULL};
__device__ __forceinline__ int draw_ternary(u64 r) { return (int)__umul64hi(r, 3) - 1; }
__device__ __forceinline__ int draw_noise(u64 r) {
    const u64 u = r >> 1;
    int mag = 0;
#pragma unroll
    for (int j = 0; j < 19; j++) mag += (u >= NOISE_CDF[j]);
    return (r & 1) ? -mag : mag;
}
__device__ __forceinline__ u64 lift_small(int v, u64 p) { return v >= 0 ? (u64)v : p - (u64)(-v); }

__global__ void __launch_bounds__(256) k_sample(u64 *__restrict__ out, int n, int kind, RngKey seed, u64 stream0, u64 stream_step, int k, int logn,
                                               const BehzConst *__restrict__ bc) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)n * k) << logn) return;
    const int x = (int)(i & (N - 1)), l = (int)((i >> logn) % k);
    const size_t item = (i >> logn) / k;
    const u64 p = bc->q[l].p;
    u64 stream = stream0 + item * stream_step;
    u64 v;
    if (kind == SAMPLE_UNIFORM) v = __umul64hi(rng64(seed, stream + l, x), p);
    else if (kind == SAMPLE_TERNARY) v = lift_small(draw_ternary(rng64(seed, stream, x)), p);
    else v = lift_small(draw_noise(rng64(seed, stream, x)), p);
    out[i] = v;
}

__global__ void __launch_bounds__(256) k_encode_scatter(const u64 *__restrict__ values, u64 *__restrict__ plain, int n, int count,
                                                       const u32 *__restrict__ index_map, int logn) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n << logn) return;
    const int j = (int)(i & (N - 1));
    const size_t c = i >> logn;
    plain[c * N + index_map[j]] = j < count ? values[c * count + j] : 0;
}
// plain[i] = BatchEncoder scatter of the one-hot slot vector e_(first_col + i): a single 1 at index_map[first_col + i]
__global__ void __launch_bounds__(256) k_onehot_scatter(u64 *__restrict__ plain, int n, int first_col, const u32 *__restrict__ index_map, int logn) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n << logn) return;
    const int x = (int)(i & (N - 1));
    const size_t row = i >> logn;
    plain[i] = (u32)x == index_map[first_col + row] ? 1 : 0;
}
__global__ void __launch_bounds__(256) k_decode_gather(const u64 *__restrict__ plain_ntt, u64 *__restrict__ values, int n,
                                                      const u32 *__restrict__ index_map, int logn) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n << logn) return;
    const int j = (int)(i & (N - 1));
    const size_t c = i >> logn;
    values[i] = plain_ntt[c * N + index_map[j]];
}
// ct[c] holds u*pk (both parts, coefficient form); add e0 + Delta*m to part 0 and e1 to part 1
__global__ void __launch_bounds__(256) k_encrypt_finish(u64 *ct, const u64 *__restrict__ plain, size_t plain_stride, int n, int coeffs, RngKey seed,
                                                       u64 nonce0, int k, int logn, const BehzConst *__restrict__ bc, PlainConst pc) {
    const int N = 1 << logn;
    const size_t kN = (size_t)k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * 2 * kN) return;
    const size_t c = i / (2 * kN), r = i % (2 * kN);
    const int part = (int)(r / kN), l = (int)((r % kN) >> logn), x = (int)(r & (N - 1));
    const DMod q = bc->q[l];
    const u64 nonce = nonce0 + c;
    const u64 sid = stream_id(part == 0 ? 9 : 10, nonce, 0);
    u64 v = addmod(ct[i], lift_small(draw_noise(rng64(seed, sid, x)), q.p), q.p);
    if (part == 0 && x < coeffs) {
        const u64 m = plain[c * plain_stride + x];
        if (m) v = addmod(v, scale_plain(m, l, q, pc), q.p);
    }
    ct[i] = v;
}
// secret-key encryption: part 0 = -(a s) + e + Delta*m (the same Delta and upper-half handling as above), part 1 = a stays as written
__global__ void __launch_bounds__(256) k_encrypt_finish_sk(u64 *ct, const u64 *__restrict__ as, const u64 *__restrict__ plain, size_t plain_stride,
                                                          int n, int coeffs, RngKey seed, u64 nonce0, int k, int logn, const BehzConst *__restrict__ bc,
                                                          PlainConst pc) {
    const int N = 1 << logn;
    const size_t kN = (size_t)k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * kN) return;
    const size_t c = i / kN, r = i % kN;
    const int l = (int)(r >> logn), x = (int)(r & (N - 1));
    const DMod q = bc->q[l];
    const u64 sid = stream_id(PURPOSE_COMPACT_E, nonce0 + c, 0);
    u64 v = addmod(negmod(as[i], q.p), lift_small(draw_noise(rng64(seed, sid, x)), q.p), q.p);
    if (x < coeffs) {
        const u64 m = plain[c * plain_stride + x];
        if (m) v = addmod(v, scale_plain(m, l, q, pc), q.p);
    }
    ct[c * 2 * kN + r] = v;
}
// ---------------------------------------------------------------- sanitisation (DESIGN 4.18)
__global__ void k_sanitize_take(u64 *counter, u64 n, u64 *base) {
    const u64 v = *counter;
    *base = v;
    *counter = v + n;
}
// one thread per coefficient: the ternary draw once, written into every residue
__global__ void __launch_bounds__(256) k_sanitize_u(u64 *__restrict__ u, int n, const u64 *__restrict__ base, RngKey rk, int k, int logn,
                                                   const BehzConst *__restrict__ bc) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n << logn) return;
    const size_t c = i >> logn;
    const int x = (int)(i & (N - 1));
    const int v = draw_ternary(rng64(rk, sanitize_stream(PURPOSE_SAN_U, *base + c), (u64)x));
    u64 *dst = u + c * k * N + x;
    for (int l = 0; l < k; l++) dst[(size_t)l * N] = lift_small(v, bc->q[l].p);
}
template <bool REF>
__global__ void __launch_bounds__(256) k_sanitize_upk(const u64 *const *__restrict__ pk_tab, const u64 *__restrict__ u, u64 *__restrict__ out, int n,
                                                     int k, int logn, const BehzConst *__restrict__ bc) {
    const size_t kN = (size_t)k << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * 2 * kN) return;
    const size_t c = i / (2 * kN), r = i % (2 * kN), w = r % kN;
    const u64 *pk = key_base<REF>(pk_tab[c]);
    out[i] = mulmod(pk[r], u[c * kN + w], bc->q[w >> logn]);
}
// One thread per coefficient x of ciphertext c: e0, e1 and the W flood words are drawn once, F is reduced into each q_l by Horner over the
// words (barrett128 of r 2^64 + w_j), and the 2k words of the coefficient are read from in and out and written to out once
__global__ void __launch_bounds__(256) k_sanitize_finish(const u64 *const *__restrict__ in, u64 *__restrict__ out, int n, const u64 *__restrict__ base,
                                                        RngKey rk, const __grid_constant__ SanitizeConst S, int logn) {
    const int N = 1 << logn, k = S.k, W = S.words;
    const size_t kN = (size_t)k * N;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n << logn) return;
    const size_t c = i >> logn;
    const int x = (int)(i & (N - 1));
    const u64 nonce = *base + c;
    const int e0 = draw_noise(rng64(rk, sanitize_stream(PURPOSE_SAN_E0, nonce), (u64)x));
    const int e1 = draw_noise(rng64(rk, sanitize_stream(PURPOSE_SAN_E1, nonce), (u64)x));
    const u64 sf = sanitize_stream(PURPOSE_SAN_F, nonce);
    u64 w[KMAX];
#pragma unroll
    for (int j = 0; j < KMAX; j++)
        if (j < W) w[j] = rng64(rk, sf, (u64)x * W + j) & (j == W - 1 ? S.top_mask : ~0ULL); // constant indices: w stays in registers
    const u64 *src = in[c] + x;
    u64 *dst = out + c * 2 * kN + x;
    for (int l = 0; l < k; l++) {
        const DMod q = S.q[l];
        u64 F = 0;
#pragma unroll
        for (int j = KMAX - 1; j >= 0; j--)
            if (j < W) F = barrett128(U128{w[j], F}, q);
        const u64 f = submod(F, S.pow2b[l], q.p);
        const size_t o0 = (size_t)l * N, o1 = kN + o0;
        const u64 v0 = addmod(addmod(src[o0], dst[o0], q.p), addmod(lift_small(e0, q.p), f, q.p), q.p);
        const u64 v1 = addmod(addmod(src[o1], dst[o1], q.p), lift_small(e1, q.p), q.p);
        dst[o0] = v0;
        dst[o1] = v1;
    }
}
cudaError_t launch_sanitize_take(u64 *counter, u64 n, u64 *base, cudaStream_t s) {
    k_sanitize_take<<<1, 1, 0, s>>>(counter, n, base);
    return cudaGetLastError();
}
cudaError_t launch_sanitize_u(u64 *u, int n, const u64 *base, const RngKey &rk, int k, int logn, const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_sanitize_u<<<blocks_for((size_t)n << logn), 256, 0, s>>>(u, n, base, rk, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_sanitize_upk(const u64 *const *pk_tab, const u64 *u, u64 *out, int n, int k, int logn, const BehzConst *bc, bool ref,
                                cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const unsigned g = blocks_for(((size_t)n * 2 * k) << logn);
    if (ref) k_sanitize_upk<true><<<g, 256, 0, s>>>(pk_tab, u, out, n, k, logn, bc);
    else k_sanitize_upk<false><<<g, 256, 0, s>>>(pk_tab, u, out, n, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_sanitize_finish(const u64 *const *in, u64 *out, int n, const u64 *base, const RngKey &rk, const SanitizeConst &S, int logn,
                                   cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_sanitize_finish<<<blocks_for((size_t)n << logn), 256, 0, s>>>(in, out, n, base, rk, S, logn);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) k_fill_zero(u64 *p, size_t words) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < words) p[i] = 0;
}

__global__ void __launch_bounds__(256) k_key_add_scaled(u64 *keys, const u64 *__restrict__ target, const u64 *__restrict__ factors, DigitMap dm, int k,
                                                       int logn, const BehzConst *__restrict__ bc) {
    const int N = 1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)dm.D << logn) return;
    const int x = (int)(i & (N - 1)), d = (int)(i >> logn), r = dm.src[d];
    const DMod q = bc->q[r];
    u64 *dst = keys + ((size_t)d * 2 * k + r) * N + x;
    *dst = addmod(*dst, mulmod(target[(size_t)r * N + x], factors[d], q), q.p);
}

// ---------------------------------------------------------------- launchers
cudaError_t launch_key_add_scaled(u64 *keys, const u64 *target, const u64 *factors, const DigitMap &dm, int k, int logn, const BehzConst *bc,
                                  cudaStream_t s) {
    k_key_add_scaled<<<blocks_for((size_t)dm.D << logn), 256, 0, s>>>(keys, target, factors, dm, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_ct_add(const u64 *a, const u64 *b, u64 *out, size_t words, int k, int logn, const BehzConst *bc, int sub, cudaStream_t s) {
    if (!words) return cudaSuccess;
    k_ct_addsub<<<blocks_for(words), 256, 0, s>>>(a, b, out, words, k, logn, bc, sub);
    return cudaGetLastError();
}
cudaError_t launch_ct_add_epi(const u64 *a, u64 *out, int n, int k, int logn, const BehzConst *bc, const FloorEpi &epi, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_ct_add_epi<<<blocks_for(((size_t)n * 2 * k) << logn), 256, 0, s>>>(a, out, n, k, logn, bc, epi);
    return cudaGetLastError();
}
cudaError_t launch_ct_negate(const u64 *a, u64 *out, size_t words, int k, int logn, const BehzConst *bc, cudaStream_t s) {
    if (!words) return cudaSuccess;
    k_ct_negate<<<blocks_for(words), 256, 0, s>>>(a, out, words, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_ct_add_many(const u64 *const *in_ptrs, int n_in, u64 *out, size_t words, int k, int logn, const BehzConst *bc, cudaStream_t s) {
    if (!words || n_in <= 0) return cudaSuccess;
    k_ct_add_many<<<blocks_for(words), 256, 0, s>>>(in_ptrs, n_in, out, words, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_ct_add_plain(const u64 *ct, u64 *out, int n, int size, const u64 *plain, size_t plain_stride, int coeffs, int k, int logn,
                                const BehzConst *bc, PlainConst pc, int sub, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_ct_add_plain<<<blocks_for(((size_t)n * size * k) << logn), 256, 0, s>>>(ct, out, n, size, plain, plain_stride, coeffs, k, logn, bc, pc, sub);
    return cudaGetLastError();
}
cudaError_t launch_ct_scale(const u64 *in, u64 *out, int n, int size, const u64 *scalars, int k, int logn, const BehzConst *bc, PlainConst pc,
                            cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_ct_scale<<<blocks_for(((size_t)n * size * k) << logn), 256, 0, s>>>(in, out, n, size, scalars, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_plain_lift(const u64 *plain, u64 *lifted, int n, int coeffs, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_plain_lift<<<blocks_for(((size_t)n * k) << logn), 256, 0, s>>>(plain, lifted, n, coeffs, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_dyadic_bcast(const u64 *a, const u64 *b, u64 *out, int n, int size, int a_per_ct, int b_per_ct, int k, int logn,
                                const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_dyadic_bcast<<<blocks_for(((size_t)n * size * k) << logn), 256, 0, s>>>(a, b, out, n, size, a_per_ct, b_per_ct, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_dyadic_outer(const u64 *ct, const u64 *pl, u64 *out, int B, int R, int out_rows, int k, int logn, const BehzConstF *f,
                                cudaStream_t s) {
    if (B <= 0 || R <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)R * (unsigned)((1 << logn) >> 8) * (unsigned)k;
    if (B == 1) k_dyadic_outer<1><<<grid, 256, 0, s>>>(ct, pl, out, B, R, out_rows, logn, *f);
    else if (B == 2) k_dyadic_outer<2><<<grid, 256, 0, s>>>(ct, pl, out, B, R, out_rows, logn, *f);
    else if (B <= 4) k_dyadic_outer<4><<<grid, 256, 0, s>>>(ct, pl, out, B, R, out_rows, logn, *f);
    else k_dyadic_outer<8><<<grid, 256, 0, s>>>(ct, pl, out, B, R, out_rows, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_galois(const u64 *in, u64 *out_base, u64 *perm_c1, int n, u64 elt_inv, int k, int logn, const BehzConst *bc, cudaStream_t s,
                          int add_back) {
    if (n <= 0) return cudaSuccess;
    k_galois<<<blocks_for(((size_t)n * 2 * k) << logn), 256, 0, s>>>(in, nullptr, out_base, perm_c1, n, elt_inv, k, logn, bc, add_back);
    return cudaGetLastError();
}
cudaError_t launch_galois_gather(const u64 *const *in_ptrs, u64 *out_base, u64 *perm_c1, int n, u64 elt_inv, int k, int logn, const BehzConst *bc,
                                 cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_galois<<<blocks_for(((size_t)n * 2 * k) << logn), 256, 0, s>>>(nullptr, in_ptrs, out_base, perm_c1, n, elt_inv, k, logn, bc, 0);
    return cudaGetLastError();
}
cudaError_t launch_mac_layer(const u64 *const *in_ptrs, const int *gather, const MacTile *tiles, int n_tiles, const u64 *const *w_ptrs,
                             const u64 *bias, int K, u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc,
                             cudaStream_t s) {
    if (n_tiles <= 0) return cudaSuccess;
    const size_t pairs = ((size_t)polys * k << logn) / 2;
    dim3 grid(blocks_for(pairs, 128), n_tiles);
    k_mac_layer<<<grid, 128, 0, s>>>(in_ptrs, gather, tiles, w_ptrs, bias, K, out_ptrs, polys, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_mac_layer_fp(const u64 *const *in_ptrs, const int *gather, const MacTile *tiles, int n_tiles, const double *wd, const u64 *bias,
                                int K, u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    if (n_tiles <= 0) return cudaSuccess;
    const size_t pairs = ((size_t)polys * k << logn) / 2;
    dim3 grid(blocks_for(pairs, 128), n_tiles);
    k_mac_layer_fp<<<grid, 128, 0, s>>>(in_ptrs, gather, tiles, wd, bias, K, out_ptrs, polys, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_sample(u64 *out, int n, int kind, const RngKey &seed, u64 stream0, u64 stream_step, int k, int logn, const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_sample<<<blocks_for(((size_t)n * k) << logn), 256, 0, s>>>(out, n, kind, seed, stream0, stream_step, k, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_encode_scatter(const u64 *values, u64 *plain, int n, int count, const u32 *index_map, int logn, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_encode_scatter<<<blocks_for((size_t)n << logn), 256, 0, s>>>(values, plain, n, count, index_map, logn);
    return cudaGetLastError();
}
cudaError_t launch_onehot_scatter(u64 *plain, int n, int first_col, const u32 *index_map, int logn, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_onehot_scatter<<<blocks_for((size_t)n << logn), 256, 0, s>>>(plain, n, first_col, index_map, logn);
    return cudaGetLastError();
}
cudaError_t launch_decode_gather(const u64 *plain_ntt, u64 *values, int n, const u32 *index_map, int logn, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_decode_gather<<<blocks_for((size_t)n << logn), 256, 0, s>>>(plain_ntt, values, n, index_map, logn);
    return cudaGetLastError();
}
cudaError_t launch_encrypt_finish(u64 *ct, const u64 *plain, size_t plain_stride, int n, int coeffs, const RngKey &seed, u64 nonce0, int k, int logn,
                                  const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_encrypt_finish<<<blocks_for(((size_t)n * 2 * k) << logn), 256, 0, s>>>(ct, plain, plain_stride, n, coeffs, seed, nonce0, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_encrypt_finish_sk(u64 *ct, const u64 *as, const u64 *plain, size_t plain_stride, int n, int coeffs, const RngKey &seed, u64 nonce0,
                                     int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_encrypt_finish_sk<<<blocks_for(((size_t)n * k) << logn), 256, 0, s>>>(ct, as, plain, plain_stride, n, coeffs, seed, nonce0, k, logn, bc, pc);
    return cudaGetLastError();
}
cudaError_t launch_fill_zero(u64 *p, size_t words, cudaStream_t s) {
    if (!words) return cudaSuccess;
    k_fill_zero<<<blocks_for(words), 256, 0, s>>>(p, words);
    return cudaGetLastError();
}

// ---------------------------------------------------------------- modulus switch (Evaluator::mod_switch_scale_to_next, BFV)
// One thread per coefficient of one polynomial: its k words are read once, the primes k-1 .. k_out are dropped in registers, and its
// k_out words are written once.  Every index into x is a compile-time constant after unrolling, so x stays in registers.
__global__ void __launch_bounds__(256) k_mod_switch(const u64 *const *__restrict__ in, u64 *out, int n, int logn,
                                                   const __grid_constant__ ModSwitchConst M) {
    const size_t N = (size_t)1 << logn;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * 2 * N) return;
    const size_t poly = i >> logn, x = i & (N - 1), c = poly >> 1, part = poly & 1;
    const u64 *src = in[c] + part * M.k * N + x;
    u64 v[KMAX];
#pragma unroll
    for (int l = 0; l < KMAX; l++) v[l] = l < M.k ? src[(size_t)l * N] : 0;
#pragma unroll
    for (int j = KMAX - 1; j >= 1; j--) {
        if (j >= M.k || j < M.k_out) continue;
        u64 r = v[j] + M.half[j]; // (x_j + floor(q_j / 2)) mod q_j: both terms below q_j < 2^61
        if (r >= M.q[j].p) r -= M.q[j].p;
#pragma unroll
        for (int l = 0; l < KMAX - 1; l++) {
            if (l >= j) continue;
            const u64 p = M.q[l].p;
            const u64 d = addmod(submod(v[l], reduce64(r, M.q[l]), p), M.half_mod[j][l], p);
            const u64 y = mul_shoup_lazy(d, M.inv[j][l], M.inv_s[j][l], p);
            v[l] = y >= p ? y - p : y;
        }
    }
    u64 *dst = out + (c * 2 + part) * M.k_out * N + x;
#pragma unroll
    for (int l = 0; l < KMAX; l++)
        if (l < M.k_out) dst[(size_t)l * N] = v[l];
}
cudaError_t launch_mod_switch(const u64 *const *in, u64 *out, int n, int logn, const ModSwitchConst &M, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_mod_switch<<<blocks_for(((size_t)n * 2) << logn), 256, 0, s>>>(in, out, n, logn, M);
    return cudaGetLastError();
}

} // namespace cnhe
