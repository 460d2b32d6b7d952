// K5/K6 element-wise stages of the BFV ciphertext x ciphertext multiply and of key switching (sm_90a).
//
// Replaces, stage by stage, SEAL 3.2 Evaluator::bfv_multiply and util::BaseConverter::{fastbconv_mtilde, mont_rq,
// fast_floor, fastbconv_sk}, the 128-bit lazy inner product of Evaluator::relinearize_one_step / apply_galois, and the
// scale-and-round of Decryptor::decrypt -- reached from /root/reference "HE Wrapper/AtomicSealBfvVector.cs"
// :461-462,:546-547,:786-787,:839-840 (Multiply+Relinearize), every Rotate* call site, and :1042,:1085 (Decrypt).
// These kernels are per-coefficient (one thread owns one coefficient index across all RNS residues), fully
// coalesced along the coefficient axis, HBM-bound, and keep the per-context constants in shared memory.
#include "kernels.h"

namespace cnhe {

__device__ __forceinline__ void load_consts(BehzConst *dst, const BehzConst *src) {
    const int words = sizeof(BehzConst) / 8;
    const u64 *s = reinterpret_cast<const u64 *>(src);
    u64 *d = reinterpret_cast<u64 *>(dst);
    for (int i = threadIdx.x; i < words; i += blockDim.x) d[i] = s[i];
    __syncthreads();
}
static_assert(sizeof(BehzConst) % 8 == 0, "BehzConst must be a whole number of words");

constexpr u64 MT_MASK = 0xffffffffULL;
constexpr u64 M_TILDE = 1ULL << 32;

// ---- fastbconv_mtilde + mont_rq: q -> Bsk, with the q residues copied in front ("together" layout)
__global__ void __launch_bounds__(256) k_behz_lift(const u64 *const *__restrict__ ct_ptrs, u64 *__restrict__ out, int n_polys, int logn,
                                                  const BehzConst *__restrict__ gbc) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k, kb = bc.kb, kt = k + kb;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)n_polys << logn) return;
    const int x = (int)(gid & (N - 1)), poly = (int)(gid >> logn);
    const u64 *src = ct_ptrs[poly >> 1] + (size_t)(poly & 1) * k * N + x;
    u64 *dst = out + (size_t)poly * kt * N + x;
    u64 tmp[KMAX];
    u64 sm = 0;
#pragma unroll
    for (int i = 0; i < KMAX; i++) {
        if (i < k) {
            u64 v = src[(size_t)i * N];
            dst[(size_t)i * N] = v;
            tmp[i] = mulmod(v, bc.mtilde_inv_qhat_mod_q[i], bc.q[i]);
            sm += tmp[i] * bc.qhat_mod_mtilde[i];
        }
    }
    sm &= MT_MASK;
    const u64 r = (M_TILDE - ((sm * bc.inv_q_mod_mtilde) & MT_MASK)) & MT_MASK;
    for (int j = 0; j < kb; j++) {
        const DMod bj = bc.bsk[j];
        U128 acc = {0, 0};
#pragma unroll
        for (int i = 0; i < KMAX; i++)
            if (i < k) mac128(acc, tmp[i], bc.qhat_mod_bsk[j][i]);
        u64 xb = barrett128(acc, bj);
        u64 rr = r;
        if (bc.centered_mtilde && r >= (M_TILDE >> 1)) rr = r + (bj.p - M_TILDE);
        U128 t = mul64wide(bc.q_mod_bsk[j], rr);
        add128(t, xb);
        u64 v = barrett128(t, bj);
        dst[(size_t)(k + j) * N] = mulmod(v, bc.inv_mtilde_mod_bsk[j], bj);
    }
}

// ---- tensor product in the NTT domain, all 2k+1 residues
__global__ void __launch_bounds__(256) k_behz_tensor(const u64 *a, const u64 *b, u64 *__restrict__ d, int n, int logn,
                                                    const BehzConst *__restrict__ gbc) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k, kb = bc.kb, kt = k + kb;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= ((size_t)n * kt) << logn) return;
    const int x = (int)(gid & (N - 1));
    const int l = (int)((gid >> logn) % kt), c = (int)((gid >> logn) / kt);
    const DMod m = l < k ? bc.q[l] : bc.bsk[l - k];
    const size_t in0 = ((size_t)(c * 2 + 0) * kt + l) * N + x, in1 = ((size_t)(c * 2 + 1) * kt + l) * N + x;
    const u64 a0 = a[in0], a1 = a[in1];
    u64 d0, d1, d2;
    if (a == b) {
        d0 = mulmod(a0, a0, m);
        d2 = mulmod(a1, a1, m);
        u64 cross = mulmod(a0, a1, m);
        d1 = addmod(cross, cross, m.p);
    } else {
        const u64 b0 = b[in0], b1 = b[in1];
        d0 = mulmod(a0, b0, m);
        d2 = mulmod(a1, b1, m);
        d1 = addmod(mulmod(a0, b1, m), mulmod(a1, b0, m), m.p);
    }
    const size_t o = ((size_t)(c * 3) * kt + l) * N + x;
    d[o] = d0;
    d[o + (size_t)kt * N] = d1;
    d[o + (size_t)2 * kt * N] = d2;
}

// ---- sum of T tensor products per output (op_multiply_sum; the FP64 twin is k_behz_tensor_mac_fp): d[o] = sum_j a[o T + j] (x) b[j],
// a [n_out T][2][kt][N], b [T][2][kt][N], d [n_out][3][kt][N], canonical words.  One thread per (output, residue, coefficient), CTAs ordered
// output fastest as in the FP64 kernel.  128-bit sums of at most 8 products of 62-bit words (4 terms: d1 takes two per term) between
// Barrett reductions, as in k_ks_mac.
__global__ void __launch_bounds__(256) k_behz_tensor_mac(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 *__restrict__ d, int n_out, int T,
                                                        int logn, const BehzConst *__restrict__ gbc) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k, kt = k + bc.kb, tiles = N >> 8;
    const int o = blockIdx.x % n_out, tile = (blockIdx.x / n_out) % tiles, l = blockIdx.x / (n_out * tiles);
    const int x = (tile << 8) + threadIdx.x;
    const DMod m = l < k ? bc.q[l] : bc.bsk[l - k];
    const size_t ktN = (size_t)kt * N, ct = 2 * ktN;
    const u64 *ap = a + (size_t)o * T * ct + (size_t)l * N + x, *bp = b + (size_t)l * N + x;
    U128 r0 = {0, 0}, r1 = {0, 0}, r2 = {0, 0};
    for (int j0 = 0; j0 < T; j0 += 4) {
        U128 s0 = {0, 0}, s1 = {0, 0}, s2 = {0, 0};
        const int j1 = min(T, j0 + 4);
        for (int j = j0; j < j1; j++) {
            const u64 a0 = __ldcs(ap + (size_t)j * ct), a1 = __ldcs(ap + (size_t)j * ct + ktN);
            const u64 b0 = __ldg(bp + (size_t)j * ct), b1 = __ldg(bp + (size_t)j * ct + ktN);
            mac128(s0, a0, b0);
            mac128(s1, a0, b1);
            mac128(s1, a1, b0);
            mac128(s2, a1, b1);
        }
        add128(r0, barrett128(s0, m));
        add128(r1, barrett128(s1, m));
        add128(r2, barrett128(s2, m));
    }
    u64 *dp = d + (size_t)o * 3 * ktN + (size_t)l * N + x;
    dp[0] = barrett128(r0, m);
    dp[ktN] = barrett128(r1, m);
    dp[2 * ktN] = barrett128(r2, m);
}

// ---- times t, fast_floor (q u Bsk -> Bsk), fastbconv_sk (Bsk -> q)
// EPI: the FloorEpi epilogue on every output word (A v, + B x on c0 and c1, + Delta C on c0)
// PAIR (with EPI): output ciphertext c is the floor of product 2c minus the floor of product 2c + 1, then the epilogue.  The thread
// floors product 2c + 1 first and parks its words in its own output words, which it reads back after flooring product 2c
template <bool EPI, bool PAIR = false>
__global__ void __launch_bounds__(256) k_behz_floor(const u64 *__restrict__ d, u64 *__restrict__ out, int n_polys, u64 t, int logn,
                                                   const BehzConst *__restrict__ gbc, const __grid_constant__ FloorEpi E) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k, kb = bc.kb, kt = k + kb;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)n_polys << logn) return;
    const int x = (int)(gid & (N - 1)), poly = (int)(gid >> logn);
    u64 *dst = out + (size_t)poly * k * N + x;
    const int na = kb - 1; // auxiliary primes (the base B); bsk[na] is m_sk
#pragma unroll 1
    for (int h = 0; h < (PAIR ? 2 : 1); h++) {
        // the product polynomial read: the output's own, or (PAIR) polynomial poly % 3 of product 2 (poly / 3) + 1 - h
        const u64 *src = d + (size_t)(PAIR ? (poly / 3 * 2 + 1 - h) * 3 + poly % 3 : poly) * kt * N + x;
        u64 tmp[KBMAX], fl[KBMAX];
#pragma unroll
        for (int i = 0; i < KMAX; i++)
            if (i < k) {
                u64 v = mulmod(src[(size_t)i * N], t, bc.q[i]); // t < q_i is enforced at context creation
                tmp[i] = mulmod(v, bc.inv_qhat_mod_q[i], bc.q[i]);
            }
#pragma unroll
        for (int j = 0; j < KBMAX; j++)
            if (j < kb) {
                const DMod bj = bc.bsk[j];
                U128 acc = {0, 0};
#pragma unroll
                for (int i = 0; i < KMAX; i++)
                    if (i < k) mac128(acc, tmp[i], bc.qhat_mod_bsk[j][i]);
                u64 conv = barrett128(acc, bj);
                u64 xb = mulmod(src[(size_t)(k + j) * N], t, bj);
                fl[j] = mulmod(xb + (bj.p - conv), bc.inv_q_mod_bsk[j], bj);
            }
        const DMod msk = bc.bsk[na];
#pragma unroll
        for (int j = 0; j < KBMAX; j++)
            if (j < na) tmp[j] = mulmod(fl[j], bc.inv_bhat_mod_b[j], bc.bsk[j]);
        U128 am = {0, 0};
#pragma unroll
        for (int j = 0; j < KBMAX; j++)
            if (j < na) mac128(am, tmp[j], bc.bhat_mod_msk[j]);
        const u64 alpha = mulmod(barrett128(am, msk) + (msk.p - fl[na]), bc.inv_B_mod_msk, msk);
        const bool neg = alpha > (msk.p >> 1);
        const int part = poly % 3;
        const u64 *xs = EPI && part < 2 ? E.x[poly / 3] + (size_t)part * k * N + x : nullptr;
        const u64 *cs = EPI && part == 0 && E.c_poly ? E.c_poly[poly / 3] : nullptr; // Delta-scaled constant plaintext (nullptr: C at x = 0)
        if (cs) cs += x;
        for (int i = 0; i < k; i++) {
            const DMod qi = bc.q[i];
            U128 acc = {0, 0};
#pragma unroll
            for (int j = 0; j < KBMAX; j++)
                if (j < na) mac128(acc, tmp[j], bc.bhat_mod_q[i][j]);
            u64 v = barrett128(acc, qi);
            U128 c = neg ? mul64wide(bc.B_mod_q[i], msk.p - alpha) : mul64wide(qi.p - bc.B_mod_q[i], alpha);
            add128(c, v);
            v = barrett128(c, qi);
            if (PAIR && h == 0) {
                dst[(size_t)i * N] = v;
                continue;
            }
            if (PAIR) {
                const u64 w = dst[(size_t)i * N];
                v = v >= w ? v - w : v + (qi.p - w);
            }
            if (EPI) {
                v = mulmod(v, E.a[i], qi);
                if (part < 2) {
                    v = addmod(v, mulmod(xs[(size_t)i * N], E.b[i], qi), qi.p);
                    if (cs) v = addmod(v, cs[(size_t)i * N], qi.p);
                    else if (part == 0 && x == 0) v = addmod(v, E.c[i], qi.p);
                }
            }
            dst[(size_t)i * N] = v;
        }
    }
}

// ---- key-switch inner product: acc{0,1}[c][l][x] = sum_d digits[c][l][d][x] * key[d][{0,1}][l][x]
// key_tab: nullptr, or one key base per ciphertext (calls whose ciphertexts belong to different key slots); REF: key and the key_tab
// entries are key references (kernels.h key_base), the form a recorded graph's key switches take
template <bool REF = false>
__global__ void __launch_bounds__(256) k_ks_mac(const u64 *__restrict__ digits, const u64 *__restrict__ key, const u64 *const *__restrict__ key_tab,
                                               u64 *__restrict__ acc, int n, int D, int logn, const BehzConst *__restrict__ gbc) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= ((size_t)n * k) << logn) return;
    const int x = (int)(gid & (N - 1));
    const int l = (int)((gid >> logn) % k), c = (int)((gid >> logn) / k);
    const DMod m = bc.q[l];
    const u64 *dg = digits + ((size_t)c * k + l) * D * N + x;
    const u64 *k0 = key_base<REF>(key_tab ? key_tab[c] : key) + (size_t)l * N + x;
    const size_t dstride = (size_t)N, kpoly = (size_t)k * N, kstride = (size_t)2 * k * N;
    U128 a0 = {0, 0}, a1 = {0, 0};
    for (int d0 = 0; d0 < D; d0 += 8) { // at most 8 products of 62x62 bits between reductions
        U128 s0 = {0, 0}, s1 = {0, 0};
        const int dend = min(D, d0 + 8);
        for (int dd = d0; dd < dend; dd++) {
            const u64 v = dg[(size_t)dd * dstride];
            mac128(s0, v, __ldg(k0 + (size_t)dd * kstride));
            mac128(s1, v, __ldg(k0 + (size_t)dd * kstride + kpoly));
        }
        add128(a0, barrett128(s0, m));
        add128(a1, barrett128(s1, m));
    }
    const size_t o = ((size_t)(c * 2) * k + l) * N + x;
    acc[o] = barrett128(a0, m);
    acc[o + (size_t)k * N] = barrett128(a1, m);
}

// ---- Decryptor::decrypt scale-and-round through {t, gamma}
__global__ void __launch_bounds__(256) k_decrypt_round(const u64 *__restrict__ xs, u64 *__restrict__ plain, int n, int logn,
                                                      const BehzConst *__restrict__ gbc, PlainConst pc) {
    __shared__ BehzConst bc;
    load_consts(&bc, gbc);
    const int N = 1 << logn, k = bc.k;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)n << logn) return;
    const int x = (int)(gid & (N - 1)), c = (int)(gid >> logn);
    const u64 *src = xs + (size_t)c * k * N + x;
    U128 st = {0, 0}, sg = {0, 0};
    for (int i = 0; i < k; i++) {
        u64 v = mulmod(src[(size_t)i * N], pc.tgamma_mod_q[i], bc.q[i]);
        v = mulmod(v, bc.inv_qhat_mod_q[i], bc.q[i]);
        mac128(st, v, pc.qhat_mod_t[i]);
        mac128(sg, v, pc.qhat_mod_gamma[i]);
    }
    const u64 vt = mulmod(barrett128(st, pc.tmod), pc.neg_inv_q_mod_t, pc.tmod);
    const u64 vg = mulmod(barrett128(sg, pc.gmod), pc.neg_inv_q_mod_gamma, pc.gmod);
    u64 r;
    if (vg > (pc.gamma >> 1)) r = addmod(vt, reduce64(pc.gamma - vg, pc.tmod), pc.t);
    else r = submod(vt, reduce64(vg, pc.tmod), pc.t);
    plain[gid] = r ? mulmod(r, pc.inv_gamma_mod_t, pc.tmod) : 0;
}

static inline unsigned blocks_for(size_t threads) { return (unsigned)((threads + 255) / 256); }

cudaError_t launch_behz_lift(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_behz_lift<<<blocks_for((size_t)n * 2 << logn), 256, 0, s>>>(ct_ptrs, out, n * 2, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_behz_floor(const u64 *d, u64 *out3, int n, u64 t, int logn, const BehzConst *bc, cudaStream_t s, const FloorEpi *epi,
                              bool pair) {
    if (n <= 0) return cudaSuccess;
    if (pair && !epi) return cudaErrorInvalidValue;
    const FloorEpi none{};
    if (pair) k_behz_floor<true, true><<<blocks_for((size_t)n * 3 << logn), 256, 0, s>>>(d, out3, n * 3, t, logn, bc, *epi);
    else if (epi) k_behz_floor<true><<<blocks_for((size_t)n * 3 << logn), 256, 0, s>>>(d, out3, n * 3, t, logn, bc, *epi);
    else k_behz_floor<false><<<blocks_for((size_t)n * 3 << logn), 256, 0, s>>>(d, out3, n * 3, t, logn, bc, none);
    return cudaGetLastError();
}
cudaError_t launch_behz_tensor(const u64 *a, const u64 *b, u64 *d, int n, int kt, int logn, const BehzConst *bc, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_behz_tensor<<<blocks_for(((size_t)n * kt) << logn), 256, 0, s>>>(a, b, d, n, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_behz_tensor_mac(const u64 *a, const u64 *b, u64 *d, int n_out, int T, int kt, int logn, const BehzConst *bc, cudaStream_t s) {
    if (n_out <= 0) return cudaSuccess;
    if (logn < 8) return cudaErrorInvalidValue;
    k_behz_tensor_mac<<<(unsigned)((size_t)n_out * ((size_t)1 << (logn - 8)) * kt), 256, 0, s>>>(a, b, d, n_out, T, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_ks_mac(const u64 *digits, const u64 *key, const u64 *const *key_tab, u64 *acc, int n, int D, int k, int logn, const BehzConst *bc,
                          cudaStream_t s, bool ref) {
    if (n <= 0) return cudaSuccess;
    if (ref) k_ks_mac<true><<<blocks_for(((size_t)n * k) << logn), 256, 0, s>>>(digits, key, key_tab, acc, n, D, logn, bc);
    else k_ks_mac<<<blocks_for(((size_t)n * k) << logn), 256, 0, s>>>(digits, key, key_tab, acc, n, D, logn, bc);
    return cudaGetLastError();
}
cudaError_t launch_decrypt_round(const u64 *x, u64 *plain, int n, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    (void)k;
    if (n <= 0) return cudaSuccess;
    k_decrypt_round<<<blocks_for((size_t)n << logn), 256, 0, s>>>(x, plain, n, logn, bc, pc);
    return cudaGetLastError();
}

} // namespace cnhe
