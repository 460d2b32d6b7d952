// FP64 variants of the BEHZ / key-switch element-wise kernels (behz.cu) for moduli below 2^50.
//
// Same functions, same residues, different pipe: every modular product here is by a constant or of two residues
// below 2^50, so it runs as the 6-instruction error-free FP64 product of fparith.cuh instead of a Barrett reduction of a
// 128-bit integer product (4 mul.hi.u64 + 6 mul.lo.u64, the slowest instructions on the integer pipe).  Wherever SEAL's
// algorithm depends on the *representative* of a residue (the fast base conversions sum [x c]_p * c' over the integers),
// the canonical representative in [0,p) is formed first, exactly as in behz.cu.
// The buffers these kernels exchange with the NTT kernels (lift output, tensor input and output, digit input, accumulator output) hold
// lazy doubles (fparith.cuh) instead of canonical words; the floor's output is canonical.
#include "fparith.cuh"
#include "kernels.h"

namespace cnhe {

// The conversion constants travel as a __grid_constant__ kernel parameter (3 KB, constant bank): with the loops over residues fully
// unrolled every constant is an immediate c[bank][offset] operand of its DFMA -- no shared-memory copy, no LDS per product.
static_assert(sizeof(BehzConstF) % 8 == 0 && sizeof(BehzConstF) <= 3584, "BehzConstF must fit the kernel parameter space");

// BSK_ONLY: only the Bsk residues are written, out [n_polys][kb][N] (the fused square reads the q residues from the ciphertext itself)
template <bool BSK_ONLY>
__global__ void __launch_bounds__(256) k_behz_lift_fp(const u64 *const *__restrict__ ct_ptrs, u64 *__restrict__ out, int n_polys, int logn,
                                                     const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k, kb = F.kb, kt = k + kb;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)n_polys << logn) return;
    const int x = (int)(gid & (N - 1)), poly = (int)(gid >> logn);
    const u64 *src = ct_ptrs[poly >> 1] + (size_t)(poly & 1) * k * N + x;
    u64 *dst = out + (size_t)poly * kt * N + x, *dst_b = BSK_ONLY ? out + (size_t)poly * kb * N + x : dst + (size_t)k * N;
    double tmp[KMAX];
    u64 sm = 0;
#pragma unroll
    for (int i = 0; i < KMAX; i++)
        if (i < k) {
            const u64 v = src[(size_t)i * N];
            const double vd = u2d(v);
            if (!BSK_ONLY) dst[(size_t)i * N] = lazy_bits(vd);
            tmp[i] = fcanon(fmodmul(vd, F.mtilde_inv_qhat_mod_q[i], F.qd[i], F.qinv[i]), F.qd[i], F.qinv[i]);
            sm += d2u(tmp[i]) * F.qhat_mod_mtilde[i];
        }
    sm &= 0xffffffffULL;
    const u64 r = ((1ULL << 32) - ((sm * F.inv_q_mod_mtilde) & 0xffffffffULL)) & 0xffffffffULL;
    double rr = u2d(r);
    if (F.centered_mtilde && r >= (1ULL << 31)) rr -= 4294967296.0;
#pragma unroll
    for (int j = 0; j < KBMAX; j++) {
        if (j >= kb) break;
        const double p = F.bd[j], pinv = F.binv[j];
        double acc = fmodmul(rr, F.q_mod_bsk[j], p, pinv);
#pragma unroll
        for (int i = 0; i < KMAX; i++)
            if (i < k) acc = __dadd_rn(acc, fmodmul(tmp[i], F.qhat_mod_bsk[j][i], p, pinv));
        const double r = fmodmul(acc, F.inv_mtilde_mod_bsk[j], p, pinv); // fresh product: |r| <= 0.51 p
        dst_b[(size_t)j * N] = lazy_bits(r);
    }
}

__global__ void __launch_bounds__(256) k_behz_tensor_fp(const u64 *a, const u64 *b, u64 *__restrict__ d, int n, int logn,
                                                       const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k, kt = k + F.kb;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= ((size_t)n * kt) << logn) return;
    const int x = (int)(gid & (N - 1));
    const int l = (int)((gid >> logn) % kt), c = (int)((gid >> logn) / kt);
    const double p = l < k ? F.qd[l] : F.bd[l - k], pinv = l < k ? F.qinv[l] : F.binv[l - k];
    const size_t in0 = ((size_t)(c * 2 + 0) * kt + l) * N + x, in1 = ((size_t)(c * 2 + 1) * kt + l) * N + x;
    const double a0 = ld_lazy(a + in0), a1 = ld_lazy(a + in1);
    double d0, d1, d2;
    if (a == b) {
        d0 = fmodmul(a0, a0, p, pinv);
        d2 = fmodmul(a1, a1, p, pinv);
        const double cross = fmodmul(a0, a1, p, pinv);
        d1 = __dadd_rn(cross, cross);
    } else {
        const double b0 = ld_lazy(b + in0), b1 = ld_lazy(b + in1);
        d0 = fmodmul(a0, b0, p, pinv);
        d2 = fmodmul(a1, b1, p, pinv);
        d1 = __dadd_rn(fmodmul(a0, b1, p, pinv), fmodmul(a1, b0, p, pinv));
    }
    const size_t o = ((size_t)(c * 3) * kt + l) * N + x;
    // |d0|, |d2| <= 0.51 p, |d1| <= 1.02 p: within the inverse transform's input bound (1.25 p)
    d[o] = lazy_bits(d0);
    d[o + (size_t)kt * N] = lazy_bits(d1);
    d[o + (size_t)2 * kt * N] = lazy_bits(d2);
}

// Sum of T tensor products per output in the NTT domain (op_multiply_sum): d[o] = sum_j a[o T + j] (x) b[j], i.e. per residue l of q u Bsk
//   d0 = sum a0 b0,   d1 = sum (a0 b1 + a1 b0),   d2 = sum a1 b1
// a [n_out T][2][kt][N] (the column operands, streamed once), b [T][2][kt][N] (shared by every output), d [n_out][3][kt][N] in
// k_behz_tensor_fp's layout.  One thread per (output, residue, coefficient pair) keeps the six sums in registers.  CTA order: output
// fastest, then the 512-coefficient tile, then the residue -- the CTAs of one (l, tile) run together and read the shared b words through
// L2, as k_diag_mac orders its giant steps.  Arithmetic: fmodmul of lazy operands, |r| <= p/2 + |a b| 2^-52 (the rounding of h pinv):
// below 0.95 p for the forward output (A^2 p < 0.9 * 2^51, fp_schedule re-centres the output otherwise).  dadd, re-centred after every
// 8th term and at the end: d1 gains two products per term, so a carry (<= p/2 + 1) and 8 terms stay below 15.7 p < 2^53; without the
// in-loop re-centre 17 coherent terms of about p pass 2^53 (tests/fp64_accumulators.py).  The outputs are re-centred, within the inverse
// transform's input bound (1.25 p).
__global__ void __launch_bounds__(256) k_behz_tensor_mac_fp(const u64 *__restrict__ a, const u64 *__restrict__ b, u64 *__restrict__ d, int n_out,
                                                           int T, int logn, const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k, kt = k + F.kb, tiles = N >> 9;
    const int o = blockIdx.x % n_out, tile = (blockIdx.x / n_out) % tiles, l = blockIdx.x / (n_out * tiles);
    const int x = (tile << 9) + 2 * threadIdx.x;
    const double p = l < k ? F.qd[l] : F.bd[l - k], pinv = l < k ? F.qinv[l] : F.binv[l - k];
    const size_t ktN = (size_t)kt * N, ct = 2 * ktN;
    const u64 *ap = a + (size_t)o * T * ct + (size_t)l * N + x, *bp = b + (size_t)l * N + x;
    auto ld = [](const u64 *q, bool stream) {
        const ulonglong2 v = stream ? __ldcs(reinterpret_cast<const ulonglong2 *>(q)) : __ldg(reinterpret_cast<const ulonglong2 *>(q));
        return make_double2(__longlong_as_double((long long)v.x), __longlong_as_double((long long)v.y));
    };
    double s[3][2] = {{0.0, 0.0}, {0.0, 0.0}, {0.0, 0.0}}; // [polynomial][coefficient of the pair]
    for (int j = 0; j < T; j++) {
        const double2 a0 = ld(ap + (size_t)j * ct, true), a1 = ld(ap + (size_t)j * ct + ktN, true); // each column word is read once
        const double2 b0 = ld(bp + (size_t)j * ct, false), b1 = ld(bp + (size_t)j * ct + ktN, false);
        s[0][0] = __dadd_rn(s[0][0], fmodmul(a0.x, b0.x, p, pinv));
        s[0][1] = __dadd_rn(s[0][1], fmodmul(a0.y, b0.y, p, pinv));
        s[1][0] = __dadd_rn(s[1][0], __dadd_rn(fmodmul(a0.x, b1.x, p, pinv), fmodmul(a1.x, b0.x, p, pinv)));
        s[1][1] = __dadd_rn(s[1][1], __dadd_rn(fmodmul(a0.y, b1.y, p, pinv), fmodmul(a1.y, b0.y, p, pinv)));
        s[2][0] = __dadd_rn(s[2][0], fmodmul(a1.x, b1.x, p, pinv));
        s[2][1] = __dadd_rn(s[2][1], fmodmul(a1.y, b1.y, p, pinv));
        if ((j & 7) == 7) {
#pragma unroll
            for (int u = 0; u < 3; u++) { s[u][0] = frecenter(s[u][0], p, pinv); s[u][1] = frecenter(s[u][1], p, pinv); }
        }
    }
    u64 *dp = d + (size_t)o * 3 * ktN + (size_t)l * N + x;
#pragma unroll
    for (int u = 0; u < 3; u++) {
        const double v0 = frecenter(s[u][0], p, pinv), v1 = frecenter(s[u][1], p, pinv);
        *reinterpret_cast<ulonglong2 *>(dp + (size_t)u * ktN) = make_ulonglong2(lazy_bits(v0), lazy_bits(v1));
    }
}

// The floor's epilogue (FloorEpi; EPI = true instantiations only): v is residue i (any integer |v| < 2^52) of output polynomial
// `part` of ciphertext ct at coefficient x, xs the same coefficient of the input's polynomial `part` (part < 2), cs the same coefficient
// of ct's Delta-scaled constant plaintext (c0 only; nullptr: the constant polynomial C).  Returns A v + B x + Delta C, |r| < 2.1 p: the
// caller's fcanon_u makes it canonical.
__device__ __forceinline__ double floor_epi_fp(double v, const FloorEpi &E, const u64 *xs, const u64 *cs, int part, int x, int i, int N, double p,
                                               double pinv) {
    double r = fmodmul(frecenter(v, p, pinv), E.a_d[i], p, pinv);
    if (part < 2) {
        r = __dadd_rn(r, fmodmul(u2d(xs[(size_t)i * N]), E.b_d[i], p, pinv));
        if (cs) r = __dadd_rn(r, u2d(cs[(size_t)i * N]));
        else if (part == 0 && x == 0) r = __dadd_rn(r, E.c_d[i]);
    }
    return r;
}
// the input words the epilogue adds to output polynomial `poly` of the launch (c0, c1 of ciphertext poly / 3), or nullptr for c2
__device__ __forceinline__ const u64 *floor_epi_src(const FloorEpi &E, size_t poly, int x, int k, int N) {
    const int part = (int)(poly % 3);
    return part < 2 ? E.x[poly / 3] + (size_t)part * k * N + x : nullptr;
}
// the Delta-scaled constant plaintext's words at coefficient x for output polynomial `poly` (c0 of a ciphertext that has one), or nullptr
__device__ __forceinline__ const u64 *floor_epi_cpoly(const FloorEpi &E, size_t poly, int x) {
    if (!E.c_poly || poly % 3 != 0) return nullptr;
    const u64 *cs = E.c_poly[poly / 3];
    return cs ? cs + x : nullptr;
}

// the product polynomial a floor thread reads for output polynomial `poly`: itself, or (PAIR) polynomial poly % 3 of product 2 (poly / 3) + sel
__device__ __forceinline__ size_t floor_src_poly(size_t poly, bool pair, int sel) { return pair ? (poly / 3 * 2 + sel) * 3 + poly % 3 : poly; }

// fast_floor + fastbconv_sk on lazy input, with the constant factors folded into the conversion matrices (FloorConstF): -19 % FP64
// instructions, -12 % time for the element-wise family against the unfolded sequence.  Same outputs as k_behz_floor (behz.cu): every
// folded product is the same residue class and the canonical representatives are formed at the same points.  ITERS > 1 walks several
// coefficients per thread with the next one's loads issued early -- measured 60 % slower (170 registers, one CTA per SM), so only
// ITERS = 1 is built.
// PAIR (ITERS = 1, with EPI): output ciphertext c is the floor of product 2c minus the floor of product 2c + 1, then the epilogue
// (FloorEpi).  The thread floors product 2c + 1 first and parks its canonical words in its own output words, which it reads back after
// flooring product 2c
template <int ITERS, bool EPI, bool PAIR = false>
__global__ void __launch_bounds__(256) k_behz_floor_fold_fp(const u64 *__restrict__ d, u64 *__restrict__ out, size_t total, int logn,
                                                           const __grid_constant__ FloorConstF F, const __grid_constant__ FloorEpi E) {
    const int N = 1 << logn, k = F.k, kb = F.kb, kt = k + kb, na = kb - 1;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    static_assert(!PAIR || ITERS == 1, "the pair floor walks one coefficient per thread");
    double cq[KMAX], cb[KBMAX], nq[KMAX], nb[KBMAX]; // current / next coefficient: residues mod q_i and mod the Bsk primes
    auto load = [&](double (&vq)[KMAX], double (&vb)[KBMAX], size_t g, int sel) {
        const u64 *src = d + floor_src_poly(g >> logn, PAIR, sel) * (size_t)kt * N + (g & (size_t)(N - 1));
#pragma unroll
        for (int i = 0; i < KMAX; i++)
            if (i < k) vq[i] = ld_lazy(src + (size_t)i * N);
        src += (size_t)k * N;
#pragma unroll
        for (int j = 0; j < KBMAX; j++)
            if (j < kb) vb[j] = ld_lazy(src + (size_t)j * N);
    };
    if (gid < total) load(cq, cb, gid, PAIR ? 1 : 0);
#pragma unroll 1
    for (int it = 0; it < ITERS; it++, gid += stride) {
        if (gid >= total) return;
        const bool more = ITERS > 1 && it + 1 < ITERS && gid + stride < total;
        if (more) load(nq, nb, gid + stride, 0);
#pragma unroll 1
        for (int h = 0; h < (PAIR ? 2 : 1); h++) {
            if (PAIR && h == 1) load(cq, cb, gid, 0);
            double tmp[KBMAX];
            // [x t q-hat_i^-1]_{q_i}, canonical representative (the base conversion sums these integers)
#pragma unroll
            for (int i = 0; i < KMAX; i++)
                if (i < k) tmp[i] = fcanon(fmodmul(cq[i], F.xq[i], F.qd[i], F.qinv[i]), F.qd[i], F.qinv[i]);
            double fl[KBMAX];
#pragma unroll
            for (int j = 0; j < KBMAX; j++)
                if (j < kb) {
                    const double p = F.bd[j], pinv = F.binv[j];
                    double acc = fmodmul(cb[j], F.xb[j], p, pinv);
#pragma unroll
                    for (int i = 0; i < KMAX; i++)
                        if (i < k) acc = __dsub_rn(acc, fmodmul(tmp[i], F.conv[j][i], p, pinv));
                    fl[j] = acc; // j < na: floor_j * B-hat_j^-1 mod p_j;  j = na: floor mod m_sk   (|acc| <= (k+1) * 0.51 p)
                }
            double pm = 0.0, pminv = 0.0, am = 0.0, fl_sk = 0.0;
#pragma unroll
            for (int j = 0; j < KBMAX; j++)
                if (j == na) { pm = F.bd[j]; pminv = F.binv[j]; fl_sk = fl[j]; }
#pragma unroll
            for (int j = 0; j < KBMAX; j++)
                if (j < na) {
                    tmp[j] = fcanon(fl[j], F.bd[j], F.binv[j]);
                    am = __dadd_rn(am, fmodmul(tmp[j], F.bhat_mod_msk[j], pm, pminv));
                }
            const double alpha = fcanon(fmodmul(frecenter(__dsub_rn(am, fl_sk), pm, pminv), F.inv_B_mod_msk, pm, pminv), pm, pminv);
            const double alpha_c = alpha > F.msk_half ? __dsub_rn(alpha, pm) : alpha;
            u64 *dst = out + (gid >> logn) * (size_t)k * N + (gid & (size_t)(N - 1));
            const int x = (int)(gid & (size_t)(N - 1));
            const u64 *xs = EPI ? floor_epi_src(E, gid >> logn, x, k, N) : nullptr, *cs = EPI ? floor_epi_cpoly(E, gid >> logn, x) : nullptr;
#pragma unroll
            for (int i = 0; i < KMAX; i++) {
                if (i >= k) break;
                const double p = F.qd[i], pinv = F.qinv[i];
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < KBMAX; j++)
                    if (j < na) v = __dadd_rn(v, fmodmul(tmp[j], F.bhat_mod_q[i][j], p, pinv));
                v = __dsub_rn(v, fmodmul(alpha_c, F.B_mod_q[i], p, pinv));
                if (PAIR && h == 0) {
                    dst[(size_t)i * N] = fcanon_u(v, p, pinv);
                    continue;
                }
                if (PAIR) v = __dsub_rn(fcanon(v, p, pinv), u2d(dst[(size_t)i * N])); // |v| < p
                if (EPI) v = floor_epi_fp(v, E, xs, cs, (int)((gid >> logn) % 3), x, i, N, p, pinv);
                dst[(size_t)i * N] = fcanon_u(v, p, pinv);
            }
        }
        if (more) {
#pragma unroll
            for (int i = 0; i < KMAX; i++) cq[i] = nq[i];
#pragma unroll
            for (int j = 0; j < KBMAX; j++) cb[j] = nb[j];
        }
    }
}

// One thread: two adjacent coefficients of residue l of one ciphertext, walking the D digit transforms (adjacent polynomials in the
// [c][l][d][N] layout) with 16-byte loads, UNR digits in flight: the kernel is bound by the digit stream out of HBM (8 MB per
// ciphertext at N=8192, D=25), the key (16 MB per channel) is re-read out of L2 by every ciphertext.
__device__ __forceinline__ ulonglong2 ldcs2(const u64 *p) { // streaming (evict-first): each digit word is read exactly once
    ulonglong2 v;
    asm volatile("ld.global.cs.v2.u64 {%0,%1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
    return v;
}
// CT ciphertexts per thread: the two key words of a (digit, residue, coefficient pair) are fetched from L2 once and used for all of
// them.  With one ciphertext per thread the kernel moved 48 bytes through L2 for every 16 bytes of the digit stream and sat on the L2
// bandwidth (3.9 TB/s of HBM reads = 11.7 TB/s out of L2); with four it is 24 bytes.
// TAB (CT == 1 only): ciphertext c0 reads its keys at key_tab[c0] instead of key (calls whose ciphertexts belong to different key slots);
// a template argument so that the single-key instantiations stay exactly as they were (the table read costs 12 registers).
// REF: key and the key_tab entries are key references (kernels.h key_base), the form a recorded graph's key switches take
template <int UNR, int CT, bool TAB = false, bool REF = false>
__global__ void __launch_bounds__(256) k_ks_mac_fp(const u64 *__restrict__ digits, const u64 *__restrict__ key, const u64 *const *__restrict__ key_tab,
                                                  u64 *__restrict__ acc, int n, int D, int logn, const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int n_groups = (n + CT - 1) / CT;
    if (gid >= ((size_t)n_groups * k) << (logn - 1)) return;
    const int x = (int)(gid & (N / 2 - 1)) * 2;
    const int l = (int)((gid >> (logn - 1)) % k), c0 = (int)((gid >> (logn - 1)) / k) * CT;
    const double p = F.qd[l], pinv = F.qinv[l];
    const size_t kpoly = (size_t)k * N, kstride = (size_t)2 * k * N, cstride = (size_t)k * D * N;
    const u64 *dg = digits + ((size_t)c0 * k + l) * D * N + x;
    const u64 *k0 = key_base<REF>(TAB ? key_tab[c0] : key) + (size_t)l * N + x;
    double a[CT][4]; // [ciphertext][key poly * 2 + coefficient]
#pragma unroll
    for (int ci = 0; ci < CT; ci++) a[ci][0] = a[ci][1] = a[ci][2] = a[ci][3] = 0.0;
#pragma unroll UNR
    for (int dd = 0; dd < D; dd++) {
        ulonglong2 vu[CT];
#pragma unroll
        for (int ci = 0; ci < CT; ci++)
            vu[ci] = c0 + ci < n ? ldcs2(dg + (size_t)ci * cstride + (size_t)dd * N) : make_ulonglong2(0, 0);
        const ulonglong2 w0u = __ldg(reinterpret_cast<const ulonglong2 *>(k0 + (size_t)dd * kstride));
        const ulonglong2 w1u = __ldg(reinterpret_cast<const ulonglong2 *>(k0 + (size_t)dd * kstride + kpoly));
        const double w00 = u2d(w0u.x), w01 = u2d(w0u.y), w10 = u2d(w1u.x), w11 = u2d(w1u.y);
#pragma unroll
        for (int ci = 0; ci < CT; ci++) {
            const double v0 = __longlong_as_double((long long)vu[ci].x), v1 = __longlong_as_double((long long)vu[ci].y);
            a[ci][0] = __dadd_rn(a[ci][0], fmodmul(v0, w00, p, pinv));
            a[ci][1] = __dadd_rn(a[ci][1], fmodmul(v1, w01, p, pinv));
            a[ci][2] = __dadd_rn(a[ci][2], fmodmul(v0, w10, p, pinv));
            a[ci][3] = __dadd_rn(a[ci][3], fmodmul(v1, w11, p, pinv));
        }
        if ((dd & 7) == 7) { // sums of 8 fresh products stay below 4.1 p; re-centre before they could leave the exact range
#pragma unroll
            for (int ci = 0; ci < CT; ci++)
#pragma unroll
                for (int j = 0; j < 4; j++) a[ci][j] = frecenter(a[ci][j], p, pinv);
        }
    }
#pragma unroll
    for (int ci = 0; ci < CT; ci++) {
        if (c0 + ci >= n) break;
#pragma unroll
        for (int j = 0; j < 4; j++) a[ci][j] = frecenter(a[ci][j], p, pinv);
        const size_t o = ((size_t)((c0 + ci) * 2) * k + l) * N + x;
        *reinterpret_cast<ulonglong2 *>(acc + o) = make_ulonglong2(lazy_bits(a[ci][0]), lazy_bits(a[ci][1]));
        *reinterpret_cast<ulonglong2 *>(acc + o + kpoly) = make_ulonglong2(lazy_bits(a[ci][2]), lazy_bits(a[ci][3]));
    }
}

// ---- the same inner product with the operands staged by the copy engine (cp.async.bulk -> shared memory ring, mbarriers): the register
// version above is bound by load latency (ncu: long_scoreboard 10 stall cycles per issue, 49 % of DRAM bandwidth) -- it can keep only as
// many bytes in flight as it has registers for.  Here one producer thread streams, per digit, the tile's slice of CT digit polynomials
// (HBM) and of the two key polynomials (L2) into a four-stage ring; 256 consumer threads (2 coefficients each) run the identical
// arithmetic in the identical order out of shared memory.  CTA = (group of CT ciphertexts, residue l, 512 coefficients).
constexpr int KT_X = 512, KT_STAGES = 4, KT_CONSUMERS = 256, KT_THREADS = KT_CONSUMERS + 32;
__device__ __forceinline__ unsigned kt_sptr(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void kt_wait(unsigned long long *bar, unsigned parity) {
    const unsigned a = kt_sptr(bar);
    unsigned done = 0;
    for (unsigned spin = 0; !done; spin++) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(a), "r"(parity) : "memory");
        if (!done && spin > (1u << 28)) __trap(); // a protocol error fails the launch instead of hanging the GPU
    }
}
template <int CT, bool REF = false>
__global__ void __launch_bounds__(KT_THREADS, 2) k_ks_mac_tma(const u64 *__restrict__ digits, const u64 *__restrict__ key, u64 *__restrict__ acc, int n, int D,
                                                             int logn, const __grid_constant__ BehzConstF F) {
    extern __shared__ __align__(128) unsigned char kt_smem[];
    constexpr int STAGE_BYTES = (CT + 2) * KT_X * 8;
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(kt_smem + KT_STAGES * STAGE_BYTES);
    unsigned long long *full = bars, *empty = bars + KT_STAGES;
    const int N = 1 << logn, k = F.k, tid = threadIdx.x;
    const int tiles = N / KT_X;
    const int tile = blockIdx.x % tiles, l = (blockIdx.x / tiles) % k, c0 = (blockIdx.x / (tiles * k)) * CT;
    const int x0 = tile * KT_X;
    const size_t kpoly = (size_t)k * N, kstride = (size_t)2 * k * N, cstride = (size_t)k * D * N;
    const int n_here = min(CT, n - c0);
    if (tid == 0) {
        for (int i = 0; i < KT_STAGES; i++) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(kt_sptr(full + i)), "r"(1u));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(kt_sptr(empty + i)), "r"((unsigned)KT_CONSUMERS));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid >= KT_CONSUMERS) {
        if (tid == KT_CONSUMERS) { // producer
            const u64 *dg = digits + ((size_t)c0 * k + l) * D * N + x0;
            const u64 *k0 = key_base<REF>(key) + (size_t)l * N + x0;
            for (int dd = 0; dd < D; dd++) {
                const int s = dd % KT_STAGES;
                kt_wait(empty + s, (((unsigned)dd / KT_STAGES) & 1) ^ 1);
                unsigned char *st = kt_smem + s * STAGE_BYTES;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(kt_sptr(full + s)), "r"((unsigned)((n_here + 2) * KT_X * 8)) : "memory");
                for (int ci = 0; ci < n_here; ci++)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(kt_sptr(st + ci * KT_X * 8)),
                                 "l"(dg + (size_t)ci * cstride + (size_t)dd * N), "r"((unsigned)(KT_X * 8)), "r"(kt_sptr(full + s))
                                 : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(kt_sptr(st + CT * KT_X * 8)),
                             "l"(k0 + (size_t)dd * kstride), "r"((unsigned)(KT_X * 8)), "r"(kt_sptr(full + s))
                             : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(kt_sptr(st + (CT + 1) * KT_X * 8)),
                             "l"(k0 + (size_t)dd * kstride + kpoly), "r"((unsigned)(KT_X * 8)), "r"(kt_sptr(full + s))
                             : "memory");
            }
        }
        return;
    }
    const double p = F.qd[l], pinv = F.qinv[l];
    double a[CT][4]; // [ciphertext][key poly * 2 + coefficient]
#pragma unroll
    for (int ci = 0; ci < CT; ci++) a[ci][0] = a[ci][1] = a[ci][2] = a[ci][3] = 0.0;
    for (int dd = 0; dd < D; dd++) {
        const int s = dd % KT_STAGES;
        kt_wait(full + s, ((unsigned)dd / KT_STAGES) & 1);
        const ulonglong2 *st = reinterpret_cast<const ulonglong2 *>(kt_smem + s * STAGE_BYTES);
        const ulonglong2 w0u = st[CT * (KT_X / 2) + tid], w1u = st[(CT + 1) * (KT_X / 2) + tid];
        const double w00 = u2d(w0u.x), w01 = u2d(w0u.y), w10 = u2d(w1u.x), w11 = u2d(w1u.y);
#pragma unroll
        for (int ci = 0; ci < CT; ci++) {
            if (ci < n_here) {
                const ulonglong2 vu = st[ci * (KT_X / 2) + tid];
                const double v0 = __longlong_as_double((long long)vu.x), v1 = __longlong_as_double((long long)vu.y);
                a[ci][0] = __dadd_rn(a[ci][0], fmodmul(v0, w00, p, pinv));
                a[ci][1] = __dadd_rn(a[ci][1], fmodmul(v1, w01, p, pinv));
                a[ci][2] = __dadd_rn(a[ci][2], fmodmul(v0, w10, p, pinv));
                a[ci][3] = __dadd_rn(a[ci][3], fmodmul(v1, w11, p, pinv));
            }
        }
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(kt_sptr(empty + s)) : "memory"); // this thread is done with the stage
        if ((dd & 7) == 7) { // sums of 8 fresh products stay below 4.1 p; re-centre before they could leave the exact range
#pragma unroll
            for (int ci = 0; ci < CT; ci++)
#pragma unroll
                for (int j = 0; j < 4; j++) a[ci][j] = frecenter(a[ci][j], p, pinv);
        }
    }
    const int x = x0 + 2 * tid;
#pragma unroll
    for (int ci = 0; ci < CT; ci++) {
        if (ci >= n_here) break;
#pragma unroll
        for (int j = 0; j < 4; j++) a[ci][j] = frecenter(a[ci][j], p, pinv);
        const size_t o = ((size_t)((c0 + ci) * 2) * k + l) * N + x;
        *reinterpret_cast<ulonglong2 *>(acc + o) = make_ulonglong2(lazy_bits(a[ci][0]), lazy_bits(a[ci][1]));
        *reinterpret_cast<ulonglong2 *>(acc + o + kpoly) = make_ulonglong2(lazy_bits(a[ci][2]), lazy_bits(a[ci][3]));
    }
}

static inline unsigned blocks_for(size_t threads) { return (unsigned)((threads + 255) / 256); }

// `f` is the HOST copy of the constants (passed by value into the kernel's parameter space)
cudaError_t launch_behz_lift_fp(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConstF *f, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_behz_lift_fp<false><<<blocks_for((size_t)n * 2 << logn), 256, 0, s>>>(ct_ptrs, out, n * 2, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_behz_lift_bsk_fp(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConstF *f, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_behz_lift_fp<true><<<blocks_for((size_t)n * 2 << logn), 256, 0, s>>>(ct_ptrs, out, n * 2, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_behz_tensor_fp(const u64 *a, const u64 *b, u64 *d, int n, int kt, int logn, const BehzConstF *f, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_behz_tensor_fp<<<blocks_for(((size_t)n * kt) << logn), 256, 0, s>>>(a, b, d, n, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_behz_tensor_mac_fp(const u64 *a, const u64 *b, u64 *d, int n_out, int T, int kt, int logn, const BehzConstF *f, cudaStream_t s) {
    if (n_out <= 0) return cudaSuccess;
    if (logn < 9) return cudaErrorInvalidValue; // whole 512-coefficient tiles
    const unsigned grid = (unsigned)((size_t)n_out * ((size_t)1 << (logn - 9)) * kt);
    k_behz_tensor_mac_fp<<<grid, 256, 0, s>>>(a, b, d, n_out, T, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_behz_floor_fold_fp(const u64 *d, u64 *out3, int n, int logn, const FloorConstF *f, cudaStream_t s, const FloorEpi *epi,
                                     bool pair) {
    if (n <= 0) return cudaSuccess;
    if (pair && !epi) return cudaErrorInvalidValue;
    const size_t total = (size_t)n * 3 << logn;
    const FloorEpi none{};
    if (pair) k_behz_floor_fold_fp<1, true, true><<<blocks_for(total), 256, 0, s>>>(d, out3, total, logn, *f, *epi);
    else if (epi) k_behz_floor_fold_fp<1, true><<<blocks_for(total), 256, 0, s>>>(d, out3, total, logn, *f, *epi);
    else k_behz_floor_fold_fp<1, false><<<blocks_for(total), 256, 0, s>>>(d, out3, total, logn, *f, none);
    return cudaGetLastError();
}
// REF: the recorded form (key references); the same kernel, grid and arithmetic as the pointer form for every n
template <bool REF>
static cudaError_t ks_mac_fp(const u64 *digits, const u64 *key, const u64 *const *key_tab, u64 *acc, int n, int D, int k, int logn,
                             const BehzConstF *f, cudaStream_t s) {
    // key reuse pays once the launch fills the GPU anyway: with few ciphertexts (LoLa: 1-32 per call) four per CTA leaves SMs idle.
    // Per-ciphertext keys share nothing: one ciphertext per thread, and the copy-engine kernel (one key stream per CTA) is not used
    static_assert(1024 % KT_X == 0, "every ring (N >= 1024) is a whole number of tiles");
    if (n >= 64 && !key_tab) { // full waves: the copy-engine-staged kernel
        constexpr int smem = KT_STAGES * (4 + 2) * KT_X * 8 + 2 * KT_STAGES * 8;
        cudaError_t e = cudaFuncSetAttribute(k_ks_mac_tma<4, REF>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)(((1 << logn) / KT_X) * k * ((n + 3) / 4));
        k_ks_mac_tma<4, REF><<<grid, KT_THREADS, smem, s>>>(digits, key, acc, n, D, logn, *f);
        return cudaGetLastError();
    }
    const unsigned blocks = blocks_for(((size_t)n * k) << (logn - 1));
    if (key_tab) k_ks_mac_fp<1, 1, true, REF><<<blocks, 256, 0, s>>>(digits, key, key_tab, acc, n, D, logn, *f);
    else k_ks_mac_fp<1, 1, false, REF><<<blocks, 256, 0, s>>>(digits, key, nullptr, acc, n, D, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_ks_mac_fp(const u64 *digits, const u64 *key, const u64 *const *key_tab, u64 *acc, int n, int D, int k, int logn,
                             const BehzConstF *f, cudaStream_t s, bool ref) {
    if (n <= 0) return cudaSuccess;
    return ref ? ks_mac_fp<true>(digits, key, key_tab, acc, n, D, k, logn, f, s) : ks_mac_fp<false>(digits, key, key_tab, acc, n, D, k, logn, f, s);
}

} // namespace cnhe
