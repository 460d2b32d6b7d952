// K1/K2: batched negacyclic NTT / inverse NTT over one residue polynomial per CTA  (sm_90a).
//
// Replaces SEAL 3.2 util::ntt_negacyclic_harvey(_lazy) / inverse_ntt_negacyclic_harvey(_lazy), reached from every
// Evaluator.Multiply / Relinearize / Rotate* / dense MultiplyPlain call site of
// /root/reference "HE Wrapper/AtomicSealBfvVector.cs" (map in SURVEY.md section 8a).
//
// Design: the whole residue polynomial (8N bytes: 32..128 KiB) lives in shared memory for the duration of the
// transform, so HBM sees exactly one read and one write of it (16N algorithmic bytes).  Each thread owns 16
// coefficients in registers and runs 2..4 radix-2 stages per pass (3..4 passes for log2 N = 10..14); twiddles and
// their Shoup quotients come through the read-only path (L1/L2-resident: 16N bytes per modulus shared by the batch).
// Butterflies are Harvey lazy butterflies on the integer pipe (values in [0,4p) forward, [0,2p) inverse); the result
// written back is canonical, which is what makes the kernel bit-comparable with the CPU oracle.
// Shared-memory layout: word i is stored at i ^ (((i>>4)&7)<<1) so that the unit-stride last pass (16 consecutive
// words per thread, 16-byte accesses) and the strided passes (gap >= 16 words) are both bank-conflict free.
#include <cuda.h> // CUtensorMap (the encoder is fetched through cudaGetDriverEntryPoint: no libcuda link dependency)

#include "kernels.h"
#include "fparith.cuh"

namespace cnhe {

__device__ __forceinline__ int swz(int i) { return i ^ (((i >> 4) & 7) << 1); }

__device__ __forceinline__ void ct_butterfly(u64 &X, u64 &Y, u64 W, u64 Ws, u64 p, u64 two_p) {
    u64 a = X;
    a = a >= two_p ? a - two_p : a;
    u64 t = mul_shoup_lazy(Y, W, Ws, p);
    X = a + t;
    Y = a - t + two_p;
}
__device__ __forceinline__ void gs_butterfly(u64 &X, u64 &Y, u64 W, u64 Ws, u64 p, u64 two_p) {
    u64 u = X, v = Y;
    u64 s = u + v;
    X = s >= two_p ? s - two_p : s;
    Y = mul_shoup_lazy(u - v + two_p, W, Ws, p);
}

struct FwdSrc {
    const u64 *src; // polynomial base (plain) or digit source polynomial
    int shift;      // digit mode
    u64 mask;
    bool digit, need_reduce;
};
__device__ __forceinline__ u64 fwd_load(const FwdSrc &s, int idx, const DMod &m) {
    u64 v = s.src[idx];
    if (s.digit) {
        v = (v >> s.shift) & s.mask;
        if (s.need_reduce) v = reduce64(v, m);
    }
    return v;
}

// Forward pass covering stages [S0, S0+R), gap of its last stage g = N >> (S0+R) >= 16.
template <int LOGN, int S0, int R, bool FROM_G>
__device__ __forceinline__ void fwd_pass(u64 *sm, const FwdSrc &src, const NttTab &tb, int tid) {
    constexpr int T = (1 << LOGN) / 16, G = 16 >> R, E = 1 << R, LG = LOGN - S0 - R;
    const u64 p = tb.mod.p, two_p = 2 * p;
#pragma unroll
    for (int gg = 0; gg < G; gg++) {
        const int gid = tid + gg * T;
        const int c = gid & ((1 << LG) - 1), j = gid >> LG;
        const int base = (j << (LG + R)) + c;
        u64 x[E];
#pragma unroll
        for (int e = 0; e < E; e++) x[e] = FROM_G ? fwd_load(src, base + (e << LG), tb.mod) : sm[swz(base + (e << LG))];
#pragma unroll
        for (int u = 0; u < R; u++) {
            const int h = E >> (u + 1);
#pragma unroll
            for (int e = 0; e < E; e++) {
                if (e & h) continue;
                const int tw = (1 << (S0 + u)) + (j << u) + (e >> (R - u));
                ct_butterfly(x[e], x[e + h], __ldg(tb.w + tw), __ldg(tb.ws + tw), p, two_p);
            }
        }
#pragma unroll
        for (int e = 0; e < E; e++) sm[swz(base + (e << LG))] = x[e];
    }
}
// Last forward pass: stages [LOGN-4, LOGN), 16 consecutive words per thread; canonical output left in smem.
template <int LOGN>
__device__ __forceinline__ void fwd_last(u64 *sm, const NttTab &tb, int tid) {
    constexpr int S0 = LOGN - 4;
    const u64 p = tb.mod.p, two_p = 2 * p;
    ulonglong2 *smv = reinterpret_cast<ulonglong2 *>(sm);
    const int j = tid, xr = j & 7;
    u64 x[16];
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        ulonglong2 v = smv[j * 8 + (ch ^ xr)];
        x[2 * ch] = v.x;
        x[2 * ch + 1] = v.y;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int h = 8 >> u;
#pragma unroll
        for (int e = 0; e < 16; e++) {
            if (e & h) continue;
            const int tw = (1 << (S0 + u)) + (j << u) + (e >> (4 - u));
            ct_butterfly(x[e], x[e + h], __ldg(tb.w + tw), __ldg(tb.ws + tw), p, two_p);
        }
    }
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        u64 a = x[2 * ch], b = x[2 * ch + 1];
        a = a >= two_p ? a - two_p : a;
        a = a >= p ? a - p : a;
        b = b >= two_p ? b - two_p : b;
        b = b >= p ? b - p : b;
        smv[j * 8 + (ch ^ xr)] = make_ulonglong2(a, b);
    }
}
template <int LOGN>
__device__ __forceinline__ void smem_to_global(const u64 *sm, u64 *dst, int tid) {
    constexpr int T = (1 << LOGN) / 16;
    const ulonglong2 *smv = reinterpret_cast<const ulonglong2 *>(sm);
    ulonglong2 *dv = reinterpret_cast<ulonglong2 *>(dst);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int ch = tid + i * T;
        dv[ch] = smv[ch ^ ((ch >> 3) & 7)];
    }
}
template <int LOGN>
__device__ __forceinline__ void global_to_smem(u64 *sm, const u64 *src, int tid) {
    constexpr int T = (1 << LOGN) / 16;
    ulonglong2 *smv = reinterpret_cast<ulonglong2 *>(sm);
    const ulonglong2 *sv = reinterpret_cast<const ulonglong2 *>(src);
    ulonglong2 v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = sv[tid + i * T];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int ch = tid + i * T;
        smv[ch ^ ((ch >> 3) & 7)] = v[i];
    }
}

template <int LOGN>
__device__ __forceinline__ void fwd_body(u64 *sm, const FwdSrc &src, const NttTab &tb, int tid) {
    if constexpr (LOGN == 10) {
        fwd_pass<10, 0, 2, true>(sm, src, tb, tid); __syncthreads();
        fwd_pass<10, 2, 4, false>(sm, src, tb, tid); __syncthreads();
    } else if constexpr (LOGN == 11) {
        fwd_pass<11, 0, 3, true>(sm, src, tb, tid); __syncthreads();
        fwd_pass<11, 3, 4, false>(sm, src, tb, tid); __syncthreads();
    } else if constexpr (LOGN == 12) {
        fwd_pass<12, 0, 4, true>(sm, src, tb, tid); __syncthreads();
        fwd_pass<12, 4, 4, false>(sm, src, tb, tid); __syncthreads();
    } else if constexpr (LOGN == 13) {
        fwd_pass<13, 0, 3, true>(sm, src, tb, tid); __syncthreads();
        fwd_pass<13, 3, 3, false>(sm, src, tb, tid); __syncthreads();
        fwd_pass<13, 6, 3, false>(sm, src, tb, tid); __syncthreads();
    } else {
        fwd_pass<14, 0, 3, true>(sm, src, tb, tid); __syncthreads();
        fwd_pass<14, 3, 3, false>(sm, src, tb, tid); __syncthreads();
        fwd_pass<14, 6, 4, false>(sm, src, tb, tid); __syncthreads();
    }
    fwd_last<LOGN>(sm, tb, tid);
    __syncthreads();
}

constexpr int min_blocks(int logn) { return logn >= 14 ? 1 : (logn == 13 ? 2 : (logn == 12 ? 3 : 2)); }

template <int LOGN>
__global__ void __launch_bounds__((1 << LOGN) / 16, min_blocks(LOGN))
k_ntt_forward(const u64 *src, u64 *dst, const NttTab *__restrict__ tabs, int mod_base, int mod_count) {
    extern __shared__ __align__(16) u64 sm[];
    constexpr int N = 1 << LOGN;
    const int b = blockIdx.x, tid = threadIdx.x;
    const NttTab tb = tabs[mod_base + b % mod_count];
    FwdSrc fs;
    fs.src = src + (size_t)b * N;
    fs.digit = false; fs.need_reduce = false; fs.shift = 0; fs.mask = 0;
    fwd_body<LOGN>(sm, fs, tb, tid);
    smem_to_global<LOGN>(sm, dst + (size_t)b * N, tid);
}

template <int LOGN>
__global__ void __launch_bounds__((1 << LOGN) / 16, min_blocks(LOGN))
k_ntt_forward_digits(const u64 *target, size_t ct_stride, u64 *dst, const NttTab *__restrict__ tabs, int k, DigitMap dm) {
    extern __shared__ __align__(16) u64 sm[];
    constexpr int N = 1 << LOGN;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int l = b % k, d = (b / k) % dm.D, c = b / (k * dm.D);
    const NttTab tb = tabs[l];
    FwdSrc fs;
    fs.src = target + (size_t)c * ct_stride + (size_t)dm.src[d] * N;
    fs.digit = true;
    fs.shift = dm.shift[d];
    fs.mask = dm.mask;
    fs.need_reduce = dm.mask >= tb.mod.p;
    fwd_body<LOGN>(sm, fs, tb, tid);
    smem_to_global<LOGN>(sm, dst + (((size_t)c * k + l) * dm.D + d) * N, tid); // [c][l][d]: the layout the key MAC streams
}

// ---------------------------------------------------------------- inverse
template <int LOGN>
__device__ __forceinline__ void inv_first(u64 *sm, const NttTab &tb, int tid) {
    constexpr int N = 1 << LOGN;
    const u64 p = tb.mod.p, two_p = 2 * p;
    ulonglong2 *smv = reinterpret_cast<ulonglong2 *>(sm);
    const int j = tid, xr = j & 7;
    u64 x[16];
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        ulonglong2 v = smv[j * 8 + (ch ^ xr)];
        x[2 * ch] = v.x;
        x[2 * ch + 1] = v.y;
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int h = 1 << u;
#pragma unroll
        for (int e = 0; e < 16; e++) {
            if (e & h) continue;
            const int tw = (N >> (u + 1)) + (j << (3 - u)) + (e >> (u + 1));
            gs_butterfly(x[e], x[e + h], __ldg(tb.iw + tw), __ldg(tb.iws + tw), p, two_p);
        }
    }
#pragma unroll
    for (int ch = 0; ch < 8; ch++) smv[j * 8 + (ch ^ xr)] = make_ulonglong2(x[2 * ch], x[2 * ch + 1]);
}
// Inverse pass covering stages [V0, V0+R) (gap of its first stage g = 1<<V0 >= 16).  LAST: scale by N^-1,
// canonicalise and write straight to global (optionally adding `base`).
template <int LOGN, int V0, int R, bool LAST>
__device__ __forceinline__ void inv_pass(u64 *sm, u64 *dst, const u64 *base_add, const NttTab &tb, int tid) {
    constexpr int N = 1 << LOGN, T = N / 16, G = 16 >> R, E = 1 << R;
    const u64 p = tb.mod.p, two_p = 2 * p;
#pragma unroll
    for (int gg = 0; gg < G; gg++) {
        const int gid = tid + gg * T;
        const int c = gid & ((1 << V0) - 1), j = gid >> V0;
        const int base = (j << (V0 + R)) + c;
        u64 x[E];
#pragma unroll
        for (int e = 0; e < E; e++) x[e] = sm[swz(base + (e << V0))];
#pragma unroll
        for (int u = 0; u < R; u++) {
            const int h = 1 << u;
#pragma unroll
            for (int e = 0; e < E; e++) {
                if (e & h) continue;
                const int tw = (N >> (V0 + u + 1)) + (j << (R - 1 - u)) + (e >> (u + 1));
                gs_butterfly(x[e], x[e + h], __ldg(tb.iw + tw), __ldg(tb.iws + tw), p, two_p);
            }
        }
        if constexpr (LAST) {
#pragma unroll
            for (int e = 0; e < E; e++) {
                u64 v = mul_shoup_lazy(x[e], tb.inv_n, tb.inv_n_s, p);
                v = v >= p ? v - p : v;
                const int idx = base + (e << V0);
                if (base_add) v = addmod(v, base_add[idx], p);
                dst[idx] = v;
            }
        } else {
#pragma unroll
            for (int e = 0; e < E; e++) sm[swz(base + (e << V0))] = x[e];
        }
    }
}

template <int LOGN>
__global__ void __launch_bounds__((1 << LOGN) / 16, min_blocks(LOGN))
k_ntt_inverse(const u64 *src, const u64 *base_add, int base_group, size_t base_stride, u64 *dst, const NttTab *__restrict__ tabs, int mod_base,
              int mod_count) {
    extern __shared__ __align__(16) u64 sm[];
    constexpr int N = 1 << LOGN;
    const int b = blockIdx.x, tid = threadIdx.x;
    const NttTab tb = tabs[mod_base + b % mod_count];
    global_to_smem<LOGN>(sm, src + (size_t)b * N, tid);
    __syncthreads();
    inv_first<LOGN>(sm, tb, tid);
    __syncthreads();
    u64 *d = dst + (size_t)b * N;
    const u64 *ba = base_add ? base_add + (size_t)(b / base_group) * base_stride + (size_t)(b % base_group) * N : nullptr;
    if constexpr (LOGN == 10) {
        inv_pass<10, 4, 4, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<10, 8, 2, true>(sm, d, ba, tb, tid);
    } else if constexpr (LOGN == 11) {
        inv_pass<11, 4, 4, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<11, 8, 3, true>(sm, d, ba, tb, tid);
    } else if constexpr (LOGN == 12) {
        inv_pass<12, 4, 4, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<12, 8, 4, true>(sm, d, ba, tb, tid);
    } else if constexpr (LOGN == 13) {
        inv_pass<13, 4, 3, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<13, 7, 3, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<13, 10, 3, true>(sm, d, ba, tb, tid);
    } else {
        inv_pass<14, 4, 4, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<14, 8, 3, false>(sm, d, ba, tb, tid); __syncthreads();
        inv_pass<14, 11, 3, true>(sm, d, ba, tb, tid);
    }
}

// ================================================================ FP64 butterfly path (p < 2^50)
// A 64x64->128-bit integer product costs ~9 IMAD-pipe slots (IMAD.WIDE and above all mul.hi.u64 issue well below the DFMA/DADD
// rate: tools/pipe_bench.cu) while DFMA/DADD overlap with the integer ALU.  For moduli below 2^50 -- all of SEAL's default coefficient primes and the 48-bit auxiliary base -- the butterfly
// is therefore done in double precision with error-free transformations:
//     h = a*w, l = fma(a,w,-h) (exact product h+l),  q = rint(h/p),  r = fma(-q,p,h) + l  ==  a*w - q*p  exactly,
// 6 DP ops for the modular product + 2 for the butterfly, no integer corrections at all: values stay centred and small
// (|r| <= (0.5 + 1.5|a|/2^53) p) and the host schedules a re-centring pass only where the bound could reach 2^52.
// The transform computed is the same function as the integer path (canonical output), so results are bit-identical.
// twiddles with table index < TWC are served from a per-CTA shared-memory copy (loaded once, under the first data loads)
constexpr int TWC = 512;
__device__ __forceinline__ void load_twiddle_cache(double *twc, const double *tw, int tid, int nthreads) {
    for (int i = tid; i < TWC; i += nthreads) twc[i] = __ldg(tw + i);
}
// a thread moves 4 consecutive words (one full 32-byte sector) as two adjacent 128-bit accesses, the widest global access sm_90 has
__device__ __forceinline__ void ldg256(const u64 *p, u64 &a, u64 &b, u64 &c, u64 &d) {
    asm volatile("ld.global.v2.b64 {%0,%1}, [%4];\n\tld.global.v2.b64 {%2,%3}, [%4+16];" : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
}
__device__ __forceinline__ void stg256(u64 *p, u64 a, u64 b, u64 c, u64 d) {
    asm volatile("st.global.v2.b64 [%0], {%1,%2};\n\tst.global.v2.b64 [%0+16], {%3,%4};" ::"l"(p), "l"(a), "l"(b), "l"(c), "l"(d) : "memory");
}

// Shared-memory round trips are what keeps the FP64 pipe idle (tools/dp_pass_bench.cu: 96 % utilisation on registers, ~62 %
// with an LDS/STS round trip every 3 stages), so the FP64 transform uses as few, as fat passes as the register file allows:
// N=8192 is 5+4+4 stages (was 3+3+3+4), the first pass reads HBM directly, the last one writes HBM directly.
// A pass over stages [S0, S0+R) is executed by "virtual threads": N/32 of them for R=5 (32 coefficients each), N/16 otherwise
// (16 coefficients: one radix-16 group, or two adjacent columns of radix-8 / four of radix-4 with 16-byte accesses).
// first-pass load: canonical u64 word, a digit of it, or (IN_F) a lazy double written by the producing kernel
template <bool IN_F>
__device__ __forceinline__ double fwd_load_fp(const FwdSrc &s, int idx, double p, double pinv) {
    if constexpr (IN_F) return ld_lazy(s.src + idx);
    u64 v = s.src[idx];
    if (s.digit) {
        v = (v >> s.shift) & s.mask; // source residue < 2^50, so every digit converts exactly
        const double x = u2d(v);
        return s.need_reduce ? frecenter(x, p, pinv) : x;
    }
    return u2d(v);
}
template <int LOGN, int S0, int R, bool FROM_G, int PASS, bool IN_F, int NV = 1>
__device__ __forceinline__ void fwd_pass_fp(double *sm, const double *twc, const FwdSrc &src, const NttTab &tb, int vt, int vstride = 0) {
    constexpr int E = 1 << R, LG = LOGN - S0 - R;
    constexpr bool CACHED = (S0 + R) <= 9; // every twiddle index of this pass is below TWC
    const double p = tb.pd, pinv = tb.pinv;
    const bool rc = (tb.fwd_recenter >> PASS) & 1;
    if constexpr (R <= 3) {
        constexpr int T = (1 << LOGN) / 16, G = 16 >> R;
#pragma unroll
        for (int gg = 0; gg < G / 2; gg++) {
            const int gid = vt + gg * T;
            const int c2 = gid & ((1 << (LG - 1)) - 1), j = gid >> (LG - 1);
            const int base = (j << (LG + R)) + 2 * c2;
            double x[E], y[E];
#pragma unroll
            for (int e = 0; e < E; e++) {
                const int idx = base + (e << LG);
                if constexpr (FROM_G) {
                    x[e] = fwd_load_fp<IN_F>(src, idx, p, pinv);
                    y[e] = fwd_load_fp<IN_F>(src, idx + 1, p, pinv);
                } else {
                    const double2 v = *reinterpret_cast<const double2 *>(sm + swz(idx));
                    x[e] = v.x;
                    y[e] = v.y;
                }
            }
            if (rc) {
#pragma unroll
                for (int e = 0; e < E; e++) { x[e] = frecenter(x[e], p, pinv); y[e] = frecenter(y[e], p, pinv); }
            }
#pragma unroll
            for (int u = 0; u < R; u++) {
                const int h = E >> (u + 1);
#pragma unroll
                for (int e = 0; e < E; e++) {
                    if (e & h) continue;
                    const int ti = (1 << (S0 + u)) + (j << u) + (e >> (R - u));
                    const double w = CACHED ? twc[ti] : __ldg(tb.wd + ti);
                    const double t0 = fmodmul(x[e + h], w, p, pinv), t1 = fmodmul(y[e + h], w, p, pinv);
                    const double a0 = x[e], a1 = y[e];
                    x[e] = __dadd_rn(a0, t0);
                    x[e + h] = __dsub_rn(a0, t0);
                    y[e] = __dadd_rn(a1, t1);
                    y[e + h] = __dsub_rn(a1, t1);
                }
            }
#pragma unroll
            for (int e = 0; e < E; e++) *reinterpret_cast<double2 *>(sm + swz(base + (e << LG))) = make_double2(x[e], y[e]);
        }
    } else {
        // NV independent groups per call (virtual threads vt, vt + vstride, ...): all their shared-memory loads are issued before
        // the first butterfly, so one group's LDS latency hides under the other's arithmetic (the compiler cannot hoist them itself
        // across the stores of the previous group)
        double x[NV][E];
        int jj[NV], bb[NV];
#pragma unroll
        for (int i = 0; i < NV; i++) {
            const int v = vt + i * vstride;
            const int c = v & ((1 << LG) - 1);
            jj[i] = v >> LG;
            bb[i] = (jj[i] << (LG + R)) + c;
#pragma unroll
            for (int e = 0; e < E; e++) {
                if constexpr (FROM_G) x[i][e] = fwd_load_fp<IN_F>(src, bb[i] + (e << LG), p, pinv);
                else x[i][e] = sm[swz(bb[i] + (e << LG))];
            }
        }
        if (rc) {
#pragma unroll
            for (int i = 0; i < NV; i++)
#pragma unroll
                for (int e = 0; e < E; e++) x[i][e] = frecenter(x[i][e], p, pinv);
        }
#pragma unroll
        for (int i = 0; i < NV; i++) {
#pragma unroll
            for (int u = 0; u < R; u++) {
                const int h = E >> (u + 1);
#pragma unroll
                for (int e = 0; e < E; e++) {
                    if (e & h) continue;
                    const int ti = (1 << (S0 + u)) + (jj[i] << u) + (e >> (R - u));
                    const double w = CACHED ? twc[ti] : __ldg(tb.wd + ti);
                    const double t = fmodmul(x[i][e + h], w, p, pinv);
                    const double a = x[i][e];
                    x[i][e] = __dadd_rn(a, t);
                    x[i][e + h] = __dsub_rn(a, t);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < NV; i++)
#pragma unroll
            for (int e = 0; e < E; e++) sm[swz(bb[i] + (e << LG))] = x[i][e];
    }
}
// First forward pass split in two so that its HBM loads are in flight while the CTA fills its twiddle cache and waits at the
// barrier (ncu source view: 11 % of a transform's warp time sat in that fill with no data load outstanding).
// fwd_first_load: E = 2^R raw words of virtual thread vt (stride N/E); fwd_first_compute: convert, R stages, store to smem.
template <int LOGN, int R, bool IN_F>
__device__ __forceinline__ void fwd_first_load(u64 (&raw)[1 << R], const FwdSrc &src, int vt) {
    constexpr int E = 1 << R, LG = LOGN - R;
#pragma unroll
    for (int e = 0; e < E; e++) raw[e] = src.src[vt + (e << LG)];
}
template <int LOGN, int R, bool IN_F>
__device__ __forceinline__ void fwd_first_compute(double *sm, const double *twc, const u64 (&raw)[1 << R], const FwdSrc &src, const NttTab &tb, int vt) {
    constexpr int E = 1 << R, LG = LOGN - R;
    const double p = tb.pd, pinv = tb.pinv;
    double x[E];
#pragma unroll
    for (int e = 0; e < E; e++) {
        if constexpr (IN_F) x[e] = __longlong_as_double((long long)raw[e]);
        else {
            u64 v = raw[e];
            if (src.digit) v = (v >> src.shift) & src.mask; // source residue < 2^50, so every digit converts exactly
            x[e] = u2d(v);
            if (src.digit && src.need_reduce) x[e] = frecenter(x[e], p, pinv);
        }
    }
#pragma unroll
    for (int u = 0; u < R; u++) { // j = 0: the whole CTA uses twiddles [2^u, 2^(u+1)) in stage u
        const int h = E >> (u + 1);
#pragma unroll
        for (int e = 0; e < E; e++) {
            if (e & h) continue;
            const double w = twc[(1 << u) + (e >> (R - u))];
            const double t = fmodmul(x[e + h], w, p, pinv);
            const double a = x[e];
            x[e] = __dadd_rn(a, t);
            x[e + h] = __dsub_rn(a, t);
        }
    }
#pragma unroll
    for (int e = 0; e < E; e++) sm[swz(vt + (e << LG))] = x[e];
}

// words 16j .. 16j+15 of a swizzled shared-memory polynomial (16-byte accesses, conflict free)
__device__ __forceinline__ void ld_group16(const double *sm, int j, double (&x)[16]) {
    const double2 *smv = reinterpret_cast<const double2 *>(sm);
    const int xr = j & 7;
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        const double2 v = smv[j * 8 + (ch ^ xr)];
        x[2 * ch] = v.x;
        x[2 * ch + 1] = v.y;
    }
}
__device__ __forceinline__ void st_group16(double *sm, int j, const double (&x)[16]) {
    double2 *smv = reinterpret_cast<double2 *>(sm);
    const int xr = j & 7;
#pragma unroll
    for (int ch = 0; ch < 8; ch++) smv[j * 8 + (ch ^ xr)] = make_double2(x[2 * ch], x[2 * ch + 1]);
}
// stage LOGN-4+u of the forward transform on 16 consecutive coefficients; tw[i] is the twiddle of their i-th butterfly block (2^u of them)
template <int U>
__device__ __forceinline__ void fwd_last_stage(double (&x)[16], const double *tw, double p, double pinv) {
    constexpr int h = 8 >> U;
#pragma unroll
    for (int e = 0; e < 16; e++) {
        if (e & h) continue;
        const double t = fmodmul(x[e + h], tw[e >> (4 - U)], p, pinv);
        const double a = x[e];
        x[e] = __dadd_rn(a, t);
        x[e + h] = __dsub_rn(a, t);
    }
}
// stages [LOGN-4, LOGN) of the forward transform on the 16 consecutive coefficients of group j (pass PASS of the schedule)
template <int LOGN, int PASS>
__device__ __forceinline__ void fwd_last_stages(double (&x)[16], const NttTab &tb, int j) {
    constexpr int S0 = LOGN - 4;
    const double p = tb.pd, pinv = tb.pinv;
    const bool rc = (tb.fwd_recenter >> PASS) & 1;
    if (rc) {
#pragma unroll
        for (int e = 0; e < 16; e++) x[e] = frecenter(x[e], p, pinv);
    }
    // twiddles of this pass: 1 + 2 + 4 + 8 consecutive doubles per thread, fetched as 16-byte loads up front
    double tw[15];
    tw[0] = __ldg(tb.wd + ((1 << S0) + j));
    {
        const double2 a = __ldg(reinterpret_cast<const double2 *>(tb.wd + ((1 << (S0 + 1)) + (j << 1))));
        tw[1] = a.x; tw[2] = a.y;
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const double2 b = __ldg(reinterpret_cast<const double2 *>(tb.wd + ((1 << (S0 + 2)) + (j << 2) + 2 * i)));
            tw[3 + 2 * i] = b.x; tw[4 + 2 * i] = b.y;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const double2 c = __ldg(reinterpret_cast<const double2 *>(tb.wd + ((1 << (S0 + 3)) + (j << 3) + 2 * i)));
            tw[7 + 2 * i] = c.x; tw[8 + 2 * i] = c.y;
        }
    }
    fwd_last_stage<0>(x, tw, p, pinv);
    fwd_last_stage<1>(x, tw + 1, p, pinv);
    fwd_last_stage<2>(x, tw + 3, p, pinv);
    fwd_last_stage<3>(x, tw + 7, p, pinv);
}
// NG twiddle groups of one thread (grouped tables, NttTab::wd_split_grp): g points at its first group, groups are `stride` apart
template <int NG>
__device__ __forceinline__ void ld_tw_groups(double *tw, const double2 *g, int stride) {
#pragma unroll
    for (int i = 0; i < NG; i++) {
        const double2 v = __ldg(g + i * stride);
        tw[2 * i] = v.x;
        tw[2 * i + 1] = v.y;
    }
}
// The same on the half transforms of the fused kernels, twiddles from the grouped table (NttTab::wd_split_grp): g = this half's groups,
// [group][LOGN-point transform's N/16 threads].  Each stage loads its own groups just before its butterflies: every warp load is 512
// contiguous bytes, where the strided table puts the 32 lanes of the last stage's loads on 16 cache lines
template <int LOGN, int PASS>
__device__ __forceinline__ void fwd_last_stages_grp(double (&x)[16], const NttTab &tb, const double2 *g, int j) {
    constexpr int T = (1 << LOGN) / 16;
    const double p = tb.pd, pinv = tb.pinv;
    if ((tb.fwd_recenter >> PASS) & 1) {
#pragma unroll
        for (int e = 0; e < 16; e++) x[e] = frecenter(x[e], p, pinv);
    }
    double tw[8];
    tw[0] = __ldg(reinterpret_cast<const double *>(g + j)); // group 0: the twiddle and a pad word
    fwd_last_stage<0>(x, tw, p, pinv);
    ld_tw_groups<1>(tw, g + T + j, T);
    fwd_last_stage<1>(x, tw, p, pinv);
    ld_tw_groups<2>(tw, g + 2 * T + j, T);
    fwd_last_stage<2>(x, tw, p, pinv);
    ld_tw_groups<4>(tw, g + 4 * T + j, T);
    fwd_last_stage<3>(x, tw, p, pinv);
}
// Last forward pass: stages [LOGN-4, LOGN) on 16 consecutive words; canonical result goes straight to HBM.
template <int LOGN, int PASS, bool OUT_F>
__device__ __forceinline__ void fwd_last_fp(const double *sm, u64 *dst, const NttTab &tb, int j) {
    const double p = tb.pd, pinv = tb.pinv;
    double x[16];
    ld_group16(sm, j, x);
    fwd_last_stages<LOGN, PASS>(x, tb, j);
    u64 *o = dst + 16 * j;
    if constexpr (OUT_F) { // lazy doubles: |x| <= fwd bound * p; re-centred only where the consumer's product could overflow (host flag)
        if (tb.fwd_out_rc) {
#pragma unroll
            for (int e = 0; e < 16; e++) x[e] = frecenter(x[e], p, pinv);
        }
#pragma unroll
        for (int g = 0; g < 4; g++) stg256(o + 4 * g, lazy_bits(x[4 * g]), lazy_bits(x[4 * g + 1]), lazy_bits(x[4 * g + 2]), lazy_bits(x[4 * g + 3]));
    } else {
#pragma unroll
        for (int g = 0; g < 4; g++)
            stg256(o + 4 * g, fcanon_u(x[4 * g], p, pinv), fcanon_u(x[4 * g + 1], p, pinv), fcanon_u(x[4 * g + 2], p, pinv), fcanon_u(x[4 * g + 3], p, pinv));
    }
}

#define CNHE_VTN(COUNT, stmt) _Pragma("unroll") for (int vt = tid; vt < (COUNT); vt += TR) { stmt; }
__host__ __device__ constexpr int fp_threads(int logn) { return logn >= 13 ? (1 << logn) / 32 : (1 << logn) / 16; }
__host__ __device__ constexpr int fp_min_blocks(int logn) { return logn == 13 ? 2 : 3; }

// Ask L2 for the polynomial that the CTA taking this one's place will read (CTAs are dispatched in blockIdx order, so that
// is about `resident` blocks ahead): its first-pass loads then hit L2 instead of waiting on HBM with the FP64 pipe idle.
template <int LOGN>
__device__ __forceinline__ void prefetch_next_poly(const u64 *src_base, int b, int n_polys, int tid) {
    constexpr int N = 1 << LOGN, TR = fp_threads(LOGN);
    const int ahead = b + 132 * fp_min_blocks(LOGN); // 132 SMs on an H100 SXM
    if (ahead < n_polys) {
        const char *p = reinterpret_cast<const char *>(src_base + (size_t)ahead * N);
        for (int i = tid * 128; i < N * 8; i += TR * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + i));
    }
}
template <int LOGN, bool IN_F, bool OUT_F>
__device__ __forceinline__ void fwd_body_fp(double *sm, const FwdSrc &src, u64 *dst, const NttTab &tb, int tid) {
    constexpr int N = 1 << LOGN, TR = fp_threads(LOGN);
    double *twc = sm + N;
    static_assert(LOGN <= 13, "N = 16384 runs on CTA pairs (k_ntt_forward_split)");
    if constexpr (LOGN == 12) { // loads first, then the twiddle cache fill (+2..3 %; -3 % at N=8192, which keeps the plain order)
        constexpr int R1 = 4;
        static_assert((N >> R1) == TR, "first pass: one virtual thread per thread");
        u64 raw[1 << R1];
        fwd_first_load<LOGN, R1, IN_F>(raw, src, tid);
        load_twiddle_cache(twc, tb.wd, tid, TR);
        __syncthreads();
        fwd_first_compute<LOGN, R1, IN_F>(sm, twc, raw, src, tb, tid);
        __syncthreads();
        CNHE_VTN(N / 16, (fwd_pass_fp<12, 4, 4, false, 1, false>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_last_fp<12, 2, OUT_F>(sm, dst, tb, vt)));
        return;
    }
    load_twiddle_cache(twc, tb.wd, tid, TR);
    __syncthreads();
    if constexpr (LOGN == 10) {
        CNHE_VTN(N / 16, (fwd_pass_fp<10, 0, 2, true, 0, IN_F>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_pass_fp<10, 2, 4, false, 1, false>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_last_fp<10, 2, OUT_F>(sm, dst, tb, vt)));
    } else if constexpr (LOGN == 11) {
        CNHE_VTN(N / 16, (fwd_pass_fp<11, 0, 3, true, 0, IN_F>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_pass_fp<11, 3, 4, false, 1, false>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_last_fp<11, 2, OUT_F>(sm, dst, tb, vt)));
    } else if constexpr (LOGN == 13) {
        CNHE_VTN(N / 32, (fwd_pass_fp<13, 0, 5, true, 0, IN_F>(sm, twc, src, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (fwd_pass_fp<13, 5, 4, false, 1, false>(sm, twc, src, tb, vt))); __syncthreads(); // NV=2 (both groups' loads first) measured 5% slower
        CNHE_VTN(N / 16, (fwd_last_fp<13, 2, OUT_F>(sm, dst, tb, vt)));
    }
}
template <int LOGN, bool IN_F, bool OUT_F>
__global__ void __launch_bounds__(fp_threads(LOGN), fp_min_blocks(LOGN))
k_ntt_forward_fp(const u64 *src, u64 *dst, const NttTab *__restrict__ tabs, int mod_base, int mod_count) {
    extern __shared__ __align__(16) u64 sm[];
    constexpr int N = 1 << LOGN;
    const int b = blockIdx.x, tid = threadIdx.x;
    const NttTab tb = tabs[mod_base + b % mod_count];
    FwdSrc fs;
    fs.src = src + (size_t)b * N;
    fs.digit = false; fs.need_reduce = false; fs.shift = 0; fs.mask = 0;
    prefetch_next_poly<LOGN>(src, b, gridDim.x, tid);
    fwd_body_fp<LOGN, IN_F, OUT_F>(reinterpret_cast<double *>(sm), fs, dst + (size_t)b * N, tb, tid);
}
// target: ciphertext c's polynomial with `k` residues starts at target + c * ct_stride (words)
template <int LOGN, bool OUT_F>
__global__ void __launch_bounds__(fp_threads(LOGN), fp_min_blocks(LOGN))
k_ntt_forward_digits_fp(const u64 *target, size_t ct_stride, u64 *dst, const NttTab *__restrict__ tabs, int k, DigitMap dm) {
    extern __shared__ __align__(16) u64 sm[];
    constexpr int N = 1 << LOGN;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int l = b % k, d = (b / k) % dm.D, c = b / (k * dm.D);
    const NttTab tb = tabs[l];
    FwdSrc fs;
    fs.src = target + (size_t)c * ct_stride + (size_t)dm.src[d] * N;
    fs.digit = true;
    fs.shift = dm.shift[d];
    fs.mask = dm.mask;
    fs.need_reduce = dm.mask >= tb.mod.p;
    fwd_body_fp<LOGN, false, OUT_F>(reinterpret_cast<double *>(sm), fs, dst + (((size_t)c * k + l) * dm.D + d) * N, tb, tid); // [c][l][d]
}

// ---- inverse, FP64: stage U (0..3) on 16 consecutive coefficients; tw[i] is the twiddle of their i-th butterfly block (8 >> U of them)
template <int U>
__device__ __forceinline__ void inv_first_stage(double (&x)[16], const double *tw, const NttTab &tb) {
    constexpr int h = 1 << U;
    const double p = tb.pd, pinv = tb.pinv;
#pragma unroll
    for (int e = 0; e < 16; e++) {
        if (e & h) continue;
        const double a = x[e], bq = x[e + h];
        x[e] = __dadd_rn(a, bq);
        x[e + h] = fmodmul(__dsub_rn(a, bq), tw[e >> (U + 1)], p, pinv);
    }
    if ((tb.inv_recenter >> U) & 1) { // uniform branch: the host schedules a re-centring of the sums on very few stages
#pragma unroll
        for (int e = 0; e < 16; e++)
            if (!(e & h)) x[e] = frecenter(x[e], p, pinv);
    }
}
// stages 0..3 on the 16 consecutive coefficients of group j
template <int LOGN>
__device__ __forceinline__ void inv_first_stages(double (&x)[16], const NttTab &tb, int j) {
    constexpr int N = 1 << LOGN;
    // stage u uses 8 >> u consecutive inverse twiddles: 8 + 4 + 2 + 1 doubles per thread, 16-byte loads
    double tw[15];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const double2 a = __ldg(reinterpret_cast<const double2 *>(tb.iwd + ((N >> 1) + (j << 3) + 2 * i)));
        tw[2 * i] = a.x; tw[2 * i + 1] = a.y;
    }
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const double2 a = __ldg(reinterpret_cast<const double2 *>(tb.iwd + ((N >> 2) + (j << 2) + 2 * i)));
        tw[8 + 2 * i] = a.x; tw[9 + 2 * i] = a.y;
    }
    {
        const double2 a = __ldg(reinterpret_cast<const double2 *>(tb.iwd + ((N >> 3) + (j << 1))));
        tw[12] = a.x; tw[13] = a.y;
        tw[14] = __ldg(tb.iwd + ((N >> 4) + j));
    }
    inv_first_stage<0>(x, tw, tb);
    inv_first_stage<1>(x, tw + 8, tb);
    inv_first_stage<2>(x, tw + 12, tb);
    inv_first_stage<3>(x, tw + 14, tb);
}
// The same on the half transforms of the fused kernels, twiddles from the grouped table (NttTab::iwd_split_grp): g = this half's groups,
// [group][LOGN-point transform's N/16 threads].  Each stage loads its own groups just before its butterflies (all 15 twiddles at once
// spill in k_behz_square_fused)
template <int LOGN>
__device__ __forceinline__ void inv_first_stages_grp(double (&x)[16], const NttTab &tb, const double2 *g, int j) {
    constexpr int T = (1 << LOGN) / 16;
    double tw[8];
    ld_tw_groups<4>(tw, g + j, T);
    inv_first_stage<0>(x, tw, tb);
    ld_tw_groups<2>(tw, g + 4 * T + j, T);
    inv_first_stage<1>(x, tw, tb);
    ld_tw_groups<1>(tw, g + 6 * T + j, T);
    inv_first_stage<2>(x, tw, tb);
    tw[0] = __ldg(reinterpret_cast<const double *>(g + 7 * T + j)); // group 7: the twiddle and a pad word
    inv_first_stage<3>(x, tw, tb);
}
// first pass reads 16 consecutive words per virtual thread straight from HBM (256-bit loads)
template <int LOGN, bool IN_F>
__device__ __forceinline__ void inv_first_fp(double *sm, const u64 *src, const NttTab &tb, int j) {
    double x[16];
#pragma unroll
    for (int g = 0; g < 4; g++) {
        u64 v0, v1, v2, v3;
        ldg256(src + 16 * j + 4 * g, v0, v1, v2, v3);
        if constexpr (IN_F) {
            x[4 * g] = __longlong_as_double((long long)v0);
            x[4 * g + 1] = __longlong_as_double((long long)v1);
            x[4 * g + 2] = __longlong_as_double((long long)v2);
            x[4 * g + 3] = __longlong_as_double((long long)v3);
        } else {
            x[4 * g] = u2d(v0);
            x[4 * g + 1] = u2d(v1);
            x[4 * g + 2] = u2d(v2);
            x[4 * g + 3] = u2d(v3);
        }
    }
    inv_first_stages<LOGN>(x, tb, j);
    st_group16(sm, j, x);
}
// The last stage (one twiddle, iw[1]) carries N^-1: sums are multiplied by N^-1, differences by iw[1]*N^-1, so every output is a
// fresh modular product in (-0.51p, 0.51p): written as is (OUT_F, lazy double) or sign-fixed on the integer pipe (canonical).
struct NoHook {
    __device__ __forceinline__ void operator()() const {}
};
// `after_load` runs once every input of the call sits in registers (the persistent kernels release / refill the shared-memory slot there)
template <int LOGN, int V0, int R, bool LAST, bool OUT_F, int NV = 1, class Hook = NoHook>
__device__ __forceinline__ void inv_pass_fp(double *sm, const double *twc, u64 *dst, const u64 *base_add, const NttTab &tb, int vt, int vstride = 0,
                                            Hook after_load = Hook()) {
    constexpr int N = 1 << LOGN, E = 1 << R;
    constexpr bool CACHED = (N >> V0) <= TWC; // stage v reads indices [N>>(v+1), N>>v)
    const double p = tb.pd, pinv = tb.pinv;
    auto finish = [&](double v, int idx) {
        if constexpr (OUT_F) return lazy_bits(v);
        u64 o = fsmall_u(v, tb.mod.p);
        if (base_add) o = addmod(o, base_add[idx], tb.mod.p);
        return o;
    };
    if constexpr (R <= 3) {
        constexpr int T = N / 16, G = 16 >> R;
#pragma unroll
        for (int gg = 0; gg < G / 2; gg++) {
            const int gid = vt + gg * T;
            const int c2 = gid & ((1 << (V0 - 1)) - 1), j = gid >> (V0 - 1);
            const int base = (j << (V0 + R)) + 2 * c2;
            double x[E], y[E];
#pragma unroll
            for (int e = 0; e < E; e++) {
                const double2 v = *reinterpret_cast<const double2 *>(sm + swz(base + (e << V0)));
                x[e] = v.x;
                y[e] = v.y;
            }
#pragma unroll
            for (int u = 0; u < R; u++) {
                const int h = 1 << u;
                const bool rc = (tb.inv_recenter >> (V0 + u)) & 1;
#pragma unroll
                for (int e = 0; e < E; e++) {
                    if (e & h) continue;
                    const int ti = (N >> (V0 + u + 1)) + (j << (R - 1 - u)) + (e >> (u + 1));
                    const double w = CACHED ? twc[ti] : __ldg(tb.iwd + ti);
                    const double a0 = x[e], b0 = x[e + h], a1 = y[e], b1 = y[e + h];
                    if (LAST && u == R - 1) {
                        x[e] = fmodmul(__dadd_rn(a0, b0), tb.inv_n_d, p, pinv);
                        y[e] = fmodmul(__dadd_rn(a1, b1), tb.inv_n_d, p, pinv);
                        x[e + h] = fmodmul(__dsub_rn(a0, b0), tb.inv_n_w_d, p, pinv);
                        y[e + h] = fmodmul(__dsub_rn(a1, b1), tb.inv_n_w_d, p, pinv);
                    } else {
                        x[e] = __dadd_rn(a0, b0);
                        y[e] = __dadd_rn(a1, b1);
                        x[e + h] = fmodmul(__dsub_rn(a0, b0), w, p, pinv);
                        y[e + h] = fmodmul(__dsub_rn(a1, b1), w, p, pinv);
                    }
                }
                if (rc && !(LAST && u == R - 1)) {
#pragma unroll
                    for (int e = 0; e < E; e++)
                        if (!(e & h)) { x[e] = frecenter(x[e], p, pinv); y[e] = frecenter(y[e], p, pinv); }
                }
            }
            if constexpr (LAST) {
#pragma unroll
                for (int e = 0; e < E; e++) {
                    const int idx = base + (e << V0);
                    *reinterpret_cast<ulonglong2 *>(dst + idx) = make_ulonglong2(finish(x[e], idx), finish(y[e], idx + 1));
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; e++) *reinterpret_cast<double2 *>(sm + swz(base + (e << V0))) = make_double2(x[e], y[e]);
            }
        }
    } else {
        double x[NV][E];
        int jj[NV], bb[NV];
#pragma unroll
        for (int i = 0; i < NV; i++) { // NV independent groups: loads first (see fwd_pass_fp)
            const int v = vt + i * vstride;
            const int c = v & ((1 << V0) - 1);
            jj[i] = v >> V0;
            bb[i] = (jj[i] << (V0 + R)) + c;
#pragma unroll
            for (int e = 0; e < E; e++) x[i][e] = sm[swz(bb[i] + (e << V0))];
        }
        after_load();
#pragma unroll
        for (int i = 0; i < NV; i++) {
#pragma unroll
            for (int u = 0; u < R; u++) {
                const int h = 1 << u;
                const bool rc = (tb.inv_recenter >> (V0 + u)) & 1;
#pragma unroll
                for (int e = 0; e < E; e++) {
                    if (e & h) continue;
                    const int ti = (N >> (V0 + u + 1)) + (jj[i] << (R - 1 - u)) + (e >> (u + 1));
                    const double w = CACHED ? twc[ti] : __ldg(tb.iwd + ti);
                    const double a = x[i][e], bq = x[i][e + h];
                    if (LAST && u == R - 1) {
                        x[i][e] = fmodmul(__dadd_rn(a, bq), tb.inv_n_d, p, pinv);
                        x[i][e + h] = fmodmul(__dsub_rn(a, bq), tb.inv_n_w_d, p, pinv);
                    } else {
                        x[i][e] = __dadd_rn(a, bq);
                        x[i][e + h] = fmodmul(__dsub_rn(a, bq), w, p, pinv);
                    }
                }
                if (rc && !(LAST && u == R - 1)) {
#pragma unroll
                    for (int e = 0; e < E; e++)
                        if (!(e & h)) x[i][e] = frecenter(x[i][e], p, pinv);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < NV; i++) {
            if constexpr (LAST) {
#pragma unroll
                for (int e = 0; e < E; e++) {
                    const int idx = bb[i] + (e << V0);
                    dst[idx] = finish(x[i][e], idx);
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; e++) sm[swz(bb[i] + (e << V0))] = x[i][e];
            }
        }
    }
}
// base_add (optional): polynomial b is added to base_add[(b / base_group) * base_stride + (b % base_group) * N] (canonical output only)
template <int LOGN, bool IN_F, bool OUT_F>
__global__ void __launch_bounds__(fp_threads(LOGN), fp_min_blocks(LOGN))
k_ntt_inverse_fp(const u64 *src, const u64 *base_add, int base_group, size_t base_stride, u64 *dst, const NttTab *__restrict__ tabs, int mod_base,
                 int mod_count) {
    static_assert(LOGN <= 11, "N = 4096 / 8192 run on the persistent k_ntt_inverse_ws, N = 16384 on CTA pairs (k_ntt_inverse_split)");
    extern __shared__ __align__(16) u64 smraw[];
    constexpr int N = 1 << LOGN, TR = fp_threads(LOGN);
    const int b = blockIdx.x, tid = threadIdx.x;
    const NttTab tb = tabs[mod_base + b % mod_count];
    double *sm = reinterpret_cast<double *>(smraw);
    double *twc = sm + N;
    load_twiddle_cache(twc, tb.iwd, tid, TR);
    prefetch_next_poly<LOGN>(src, b, gridDim.x, tid);
    const u64 *s = src + (size_t)b * N;
    u64 *d = dst + (size_t)b * N;
    const u64 *ba = base_add ? base_add + (size_t)(b / base_group) * base_stride + (size_t)(b % base_group) * N : nullptr;
    if (ba) { // the base polynomial is consumed by the epilogue, ~20k cycles from now: have it waiting in L2
        const char *pb = reinterpret_cast<const char *>(ba);
        for (int i = tid * 128; i < N * 8; i += TR * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb + i));
    }
    CNHE_VTN(N / 16, (inv_first_fp<LOGN, IN_F>(sm, s, tb, vt)));
    __syncthreads();
    if constexpr (LOGN == 10) {
        CNHE_VTN(N / 16, (inv_pass_fp<10, 4, 4, false, false>(sm, twc, d, ba, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (inv_pass_fp<10, 8, 2, true, OUT_F>(sm, twc, d, ba, tb, vt)));
    } else {
        CNHE_VTN(N / 16, (inv_pass_fp<11, 4, 4, false, false>(sm, twc, d, ba, tb, vt))); __syncthreads();
        CNHE_VTN(N / 16, (inv_pass_fp<11, 8, 3, true, OUT_F>(sm, twc, d, ba, tb, vt)));
    }
}

// ================================================================ N = 16384 on CTA pairs ("split")
// A 16384-point polynomial is 128 KB of doubles: one CTA per SM, every warp of the SM at the same barrier, loads never overlapping
// butterflies (0.36 of the HBM roofline against 0.50 at N = 8192).  After the first Cooley-Tukey stage the two halves of the polynomial
// are independent 8192-point transforms with their own twiddle tables (NttTab::wd_split holds them), so a cluster of two CTAs takes one
// polynomial: CTA h computes half h -- x[i] +- w x[i + N/2] on the way in from global memory (the pair reads the same lines at the same
// time: one trip to HBM, the second read is an L2 hit), then the 5+4+4 passes of the 8192-point kernel in 64 KB of shared memory, 2-3 CTAs
// per SM.  The inverse runs the 13 in-half stages first and the pair exchanges the halves through distributed shared memory for the last
// butterfly, which carries N^-1.  src == dst is allowed: the pair meets at a cluster barrier between its loads and its stores.
constexpr int SPLIT_LOGN = 13, SPLIT_H = 1 << SPLIT_LOGN, SPLIT_THREADS = SPLIT_H / 32;
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned dsmem_base(const void *p, unsigned rank) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"((unsigned)__cvta_generic_to_shared(p)), "r"(rank));
    return r;
}
__device__ __forceinline__ double ld_dsmem(unsigned addr) {
    double v;
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
    return v;
}
// first pass of half `upper` of a 2^(HLOGN+1)-point transform: its stage 0 folded into the loads, then HLOGN - 8 stages (j = 0: low
// twiddles only), so that two 4-stage passes finish the half
template <int HLOGN, bool IN_F>
__device__ __forceinline__ void fwd_split_first(double *sm, const double *twc, const FwdSrc &src, const NttTab &tb, int vt, double w0, bool upper) {
    constexpr int R = HLOGN - 8, E = 1 << R, LG = HLOGN - R;
    const double p = tb.pd, pinv = tb.pinv;
    double x[E];
#pragma unroll
    for (int e = 0; e < E; e++) {
        const int idx = vt + (e << LG);
        const double a = fwd_load_fp<IN_F>(src, idx, p, pinv), c = fwd_load_fp<IN_F>(src, idx + (1 << HLOGN), p, pinv);
        const double t = fmodmul(c, w0, p, pinv);
        x[e] = upper ? __dsub_rn(a, t) : __dadd_rn(a, t);
    }
#pragma unroll
    for (int u = 0; u < R; u++) {
        const int h = E >> (u + 1);
#pragma unroll
        for (int e = 0; e < E; e++) {
            if (e & h) continue;
            const double w = twc[(1 << u) + (e >> (R - u))];
            const double t = fmodmul(x[e + h], w, p, pinv);
            const double a = x[e];
            x[e] = __dadd_rn(a, t);
            x[e + h] = __dsub_rn(a, t);
        }
    }
#pragma unroll
    for (int e = 0; e < E; e++) sm[swz(vt + (e << LG))] = x[e];
}
template <bool IN_F, bool OUT_F>
__device__ __forceinline__ void fwd_split_body(double *sm, const FwdSrc &src, u64 *dst, NttTab &tb, int half, int tid) {
    constexpr int TR = SPLIT_THREADS;
    double *twc = sm + SPLIT_H;
    const double w0 = __ldg(tb.wd + 1);
    tb.wd = tb.wd_split + half * SPLIT_H;
    tb.fwd_recenter = tb.fwd_recenter_split;
    load_twiddle_cache(twc, tb.wd, tid, TR);
    __syncthreads();
    fwd_split_first<SPLIT_LOGN, IN_F>(sm, twc, src, tb, tid, w0, half != 0);
    cluster_arrive(); // this CTA has read everything it needs from the source polynomial
    __syncthreads();
    CNHE_VTN(SPLIT_H / 16, (fwd_pass_fp<SPLIT_LOGN, 5, 4, false, 1, false>(sm, twc, src, tb, vt))); __syncthreads();
    cluster_wait(); // ... and so has its partner: the halves may be written in place
    CNHE_VTN(SPLIT_H / 16, (fwd_last_fp<SPLIT_LOGN, 2, OUT_F>(sm, dst, tb, vt)));
}
template <bool IN_F, bool OUT_F>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(SPLIT_THREADS, 2)
k_ntt_forward_split(const u64 *src, u64 *dst, const NttTab *__restrict__ tabs, int mod_base, int mod_count) {
    extern __shared__ __align__(16) u64 sm[];
    const int b = blockIdx.x >> 1, half = blockIdx.x & 1, tid = threadIdx.x;
    NttTab tb = tabs[mod_base + b % mod_count];
    FwdSrc fs;
    fs.src = src + (size_t)b * (2 * SPLIT_H);
    fs.digit = false; fs.need_reduce = false; fs.shift = 0; fs.mask = 0;
    fwd_split_body<IN_F, OUT_F>(reinterpret_cast<double *>(sm), fs, dst + (size_t)b * (2 * SPLIT_H) + half * SPLIT_H, tb, half, tid);
}
template <bool OUT_F>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(SPLIT_THREADS, 2)
k_ntt_forward_digits_split(const u64 *target, size_t ct_stride, u64 *dst, const NttTab *__restrict__ tabs, int k, DigitMap dm) {
    extern __shared__ __align__(16) u64 sm[];
    const int b = blockIdx.x >> 1, half = blockIdx.x & 1, tid = threadIdx.x;
    const int l = b % k, d = (b / k) % dm.D, c = b / (k * dm.D);
    NttTab tb = tabs[l];
    FwdSrc fs;
    fs.src = target + (size_t)c * ct_stride + (size_t)dm.src[d] * (2 * SPLIT_H);
    fs.digit = true;
    fs.shift = dm.shift[d];
    fs.mask = dm.mask;
    fs.need_reduce = dm.mask >= tb.mod.p;
    fwd_split_body<false, OUT_F>(reinterpret_cast<double *>(sm), fs, dst + (((size_t)c * k + l) * dm.D + d) * (2 * SPLIT_H) + half * SPLIT_H, tb, half, tid);
}
// last in-half pass (stages 8 .. HLOGN-1) and the cross-half butterfly of NB polynomials (consecutive half buffers of sm; polynomial b goes to
// dst + b * dst_stride and, with a base, adds base_add + b * dst_stride): own results go to shared memory for the partner, the partner's
// come back through DSMEM; half 0 keeps the sums
// (times N^-1), half 1 the differences (times iw[1] N^-1).  One pair of cluster barriers serves all NB polynomials.
template <int HLOGN, int TR, bool OUT_F, int NB = 1>
__device__ __forceinline__ void inv_split_last(double *sm, const double *twc, u64 *dst, size_t dst_stride, const u64 *base_add, const NttTab &tb,
                                               int tid, int half) {
    constexpr int V0 = 8, R = HLOGN - V0, E = 1 << R, H = 1 << HLOGN;
    static_assert(E >= 8, "the cross-half stage reads the partner in batches of 8");
    const double p = tb.pd, pinv = tb.pinv;
#pragma unroll 1
    for (int b = 0; b < NB; b++) {
        double *s = sm + b * H;
        for (int vt = tid; vt < (H >> R); vt += TR) {
            double x[E];
#pragma unroll
            for (int e = 0; e < E; e++) x[e] = s[swz(vt + (e << V0))];
#pragma unroll
            for (int u = 0; u < R; u++) {
                const int h = 1 << u;
                const bool rc = (tb.inv_recenter >> (V0 + u)) & 1;
#pragma unroll
                for (int e = 0; e < E; e++) {
                    if (e & h) continue;
                    const double w = twc[(H >> (V0 + u + 1)) + (e >> (u + 1))];
                    const double a = x[e], bq = x[e + h];
                    x[e] = __dadd_rn(a, bq);
                    x[e + h] = fmodmul(__dsub_rn(a, bq), w, p, pinv);
                }
                if (rc) {
#pragma unroll
                    for (int e = 0; e < E; e++)
                        if (!(e & h)) x[e] = frecenter(x[e], p, pinv);
                }
            }
#pragma unroll
            for (int e = 0; e < E; e++) s[swz(vt + (e << V0))] = x[e];
        }
    }
    cluster_arrive();
    cluster_wait(); // both halves are complete and visible across the pair
    const unsigned peer = dsmem_base(sm, (unsigned)(half ^ 1));
    const double scale = half ? tb.inv_n_w_d : tb.inv_n_d;
#pragma unroll 1
    for (int b = 0; b < NB; b++) {
        const double *s = sm + b * H;
        u64 *d = dst + b * dst_stride;
        const u64 *ba = base_add ? base_add + b * dst_stride : nullptr;
        for (int vt = tid; vt < (H >> R); vt += TR) {
#pragma unroll
            for (int e0 = 0; e0 < E; e0 += 8) { // own values back from shared memory, the partner's in batches of 8 (all at once would spill)
                double r[8];
#pragma unroll
                for (int i = 0; i < 8; i++) r[i] = ld_dsmem(peer + 8u * (unsigned)(b * H + swz(vt + ((e0 + i) << V0))));
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const int idx = vt + ((e0 + i) << V0);
                    const double x = s[swz(idx)];
                    const double v = fmodmul(half ? __dsub_rn(r[i], x) : __dadd_rn(x, r[i]), scale, p, pinv);
                    if constexpr (OUT_F) d[idx] = lazy_bits(v);
                    else {
                        u64 o = fsmall_u(v, tb.mod.p);
                        if (ba) o = addmod(o, ba[idx], tb.mod.p);
                        d[idx] = o;
                    }
                }
            }
        }
    }
    cluster_arrive(); // done with the partner's memory: either CTA may exit once both have said so
    cluster_wait();
}
template <bool IN_F, bool OUT_F>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(SPLIT_THREADS, 2)
k_ntt_inverse_split(const u64 *src, const u64 *base_add, int base_group, size_t base_stride, u64 *dst, const NttTab *__restrict__ tabs, int mod_base,
                    int mod_count) {
    extern __shared__ __align__(16) u64 smraw[];
    constexpr int TR = SPLIT_THREADS, H = SPLIT_H;
    const int b = blockIdx.x >> 1, half = blockIdx.x & 1, tid = threadIdx.x;
    NttTab tb = tabs[mod_base + b % mod_count];
    tb.iwd = tb.iwd_split + half * H;
    double *sm = reinterpret_cast<double *>(smraw);
    double *twc = sm + H;
    load_twiddle_cache(twc, tb.iwd, tid, TR);
    const u64 *s = src + (size_t)b * (2 * H) + half * H;
    u64 *d = dst + (size_t)b * (2 * H) + half * H;
    const u64 *ba = base_add ? base_add + (size_t)(b / base_group) * base_stride + (size_t)(b % base_group) * (2 * H) + half * H : nullptr;
    if (ba) {
        const char *pb = reinterpret_cast<const char *>(ba);
        for (int i = tid * 128; i < H * 8; i += TR * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb + i));
    }
    CNHE_VTN(H / 16, (inv_first_fp<SPLIT_LOGN, IN_F>(sm, s, tb, vt)));
    __syncthreads();
    CNHE_VTN(H / 16, (inv_pass_fp<SPLIT_LOGN, 4, 4, false, false>(sm, twc, d, ba, tb, vt))); __syncthreads();
    inv_split_last<SPLIT_LOGN, TR, OUT_F>(sm, twc, d, 0, ba, tb, tid, half);
}

// ================================================================ fused key switch, N = 4096 / 8192
// out[c][p][l] = base_c[p][l] + INTT_l(sum_d NTT_l(digit_d(target_c)) * key[d][p][l])  without the digit transforms or the NTT-domain
// accumulator ever reaching HBM.  The digit path
// (k_ntt_forward_digits_fp + k_ks_mac_tma) writes every digit transform as lazy doubles and reads it back once: 2 x 64 KiB per transform at
// N = 8192, 31 GB per CryptoNets step, more than the FP64 work of the transforms costs on an H100.  Here a CTA owns one half of the
// transform of one (ciphertext c, residue l) and walks all D digits: after the first stage the two halves of an N-point transform are
// independent N/2-point transforms (the split form of the N = 16384 kernels), so CTA h folds stage 0 into its loads (it reads both halves
// of the source residue, an L2 hit: the partner and the other residues' CTAs read the same lines at about the same time), runs the
// N/2-point passes in shared memory and, in the last pass, multiplies its 16 coefficients per thread by the matching key words and
// accumulates them: thread j owns coefficients 16j..16j+15 of both accumulators, polynomial 0 in registers and polynomial 1 in shared
// memory in the group layout of st_group16 (every thread touches only its own group, no extra barrier).
// Shared memory is [work 0][work 1][acc 1][twiddle caches]: digit d's passes run in work buffer d & 1, so one block barrier per digit
// (the all-to-all hand-off after the first pass) is all the loop needs, and warps may drift up to a digit apart.
// The twiddle cache is filled once per CTA instead of once per transform, and a warp's next digit's source words are in flight while
// other warps finish the current digit.  Same arithmetic as the MAC kernels (fmodmul + dadd, re-centred every 8 digits and
// at the end), so the accumulators end at |x| <= 0.51 p, within the inverse transform's 1.25 p input bound.
// Epilogue: the pair of CTAs is a cluster and finishes the key switch as k_behz_square_fused does: thread j's group of each accumulator is
// exactly the group the split inverse's first four stages work on, so it runs them in registers and stores the two results as
// consecutive half buffers (polynomial 0 into work buffer 1, polynomial 1 in place over its accumulator), then the
// remaining in-half pass of both and the cross-half stage (N^-1, canonical output, plus the base word) through DSMEM.  The base half is
// prefetched to L2 during the last digit.  Compared with writing the accumulator and running k_ntt_inverse_ws, every (ciphertext,
// polynomial, residue) saves an 8N-byte HBM write and read and a second kernel.  Other CTAs may still read target and base words while a
// cluster writes its output: `out` must overlap neither (the host takes the digit path otherwise).
// Keys: with PK the kernel reads the 48-bit packed copy of launch_pack_keys48 instead of the canonical u64 keys.  The key loads are the
// kernel's costliest memory traffic (keys replaced by register values: -35 % kernel time at N = 8192, source words: -3.5 %, DESIGN
// §4.4): a thread's 16 u64 words are 128 contiguous bytes, so each 16-byte load of a warp touches 32 cache lines and the lines are
// fetched from L2 again before the thread's next load uses their second half.  The packed copy holds the same words in 6 bytes each,
// laid out [D][2][k][half][6][TR] in 16-byte groups: group g of thread j is its bytes 16g..16g+15, so a warp's load is 512 contiguous
// bytes and a thread reads 96 B instead of 128.
// key_tab: nullptr (every ciphertext uses key / keyp), or a device table of one key base per ciphertext -- packed copies with PK, u64
// keys without -- for calls whose ciphertexts belong to different key slots.  Same grid, same arithmetic either way.
// REF: key, keyp and the key_tab entries are key references (kernels.h key_base), the form a recorded graph's key switches take; the
// base a CTA reads is loaded once, before the digit loop.
template <int HLOGN>
__host__ __device__ constexpr int ks_fused_threads() { return (1 << HLOGN) / 16; }
template <int HLOGN>
__host__ __device__ constexpr int ks_fused_smem() { return (1 << HLOGN) * 8 * 3 + 2 * TWC * 8; } // two work buffers, polynomial-1 accumulator, two twiddle caches
// a word below 2^48 given as its low 32 bits and bits 32..47, as an exact double (u2d of the same word)
__device__ __forceinline__ double u48d(unsigned lo, unsigned hi16) { return __dsub_rn(__hiloint2double((int)(hi16 | 0x43300000u), (int)lo), FP_TWO52); }
// packed copy: the 16 key words of (polynomial b, half, thread j), 48 bits each, little-endian in 24 u32: word 2m in u32 3m and the low
// half of 3m+1, word 2m+1 in the high half of 3m+1 and in 3m+2
template <int HLOGN>
__global__ void __launch_bounds__(256) k_pack_keys48(const u64 *__restrict__ key, uint4 *__restrict__ out, int n_polys) {
    constexpr int H = 1 << HLOGN, TR = ks_fused_threads<HLOGN>();
    const int gt = blockIdx.x * blockDim.x + threadIdx.x;
    if (gt >= n_polys * 2 * TR) return;
    const int j = gt % TR, bh = gt / TR; // bh = polynomial * 2 + half
    const u64 *w = key + (size_t)bh * H + 16 * j;
    unsigned u[24];
#pragma unroll
    for (int m = 0; m < 8; m++) {
        const u64 a = w[2 * m], b = w[2 * m + 1];
        u[3 * m] = (unsigned)a;
        u[3 * m + 1] = (unsigned)(a >> 32 & 0xffff) | (unsigned)b << 16;
        u[3 * m + 2] = (unsigned)(b >> 16);
    }
    uint4 *o = out + (size_t)bh * 6 * TR + j;
#pragma unroll
    for (int g = 0; g < 6; g++) o[g * TR] = make_uint4(u[4 * g], u[4 * g + 1], u[4 * g + 2], u[4 * g + 3]);
}
// Plane source (PL): digit d of ciphertext c is int32 plane d of planes + c * D * N instead of a cut of the target words -- the digit
// sums S = sum_j W_j digit_d(c2_j) of a scalar-MAC layer over unrelinearised squares (DESIGN 4.15).  |S| < min q_l (host-checked),
// the same input bound as a canonical digit, so nothing after the loads changes; `target` and `ct_stride` are unused.
template <int HLOGN, bool PK, bool PL, bool REF = false>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(ks_fused_threads<HLOGN>(), HLOGN == 12 ? 2 : 4)
k_key_switch_fused(const u64 *__restrict__ target, size_t ct_stride, const int *__restrict__ planes, const u64 *__restrict__ key,
                   const uint4 *__restrict__ keyp, const u64 *const *__restrict__ key_tab, const u64 *__restrict__ base, size_t base_stride,
                   u64 *__restrict__ out, const NttTab *__restrict__ tabs, int k, DigitMap dm) {
    constexpr int H = 1 << HLOGN, TR = ks_fused_threads<HLOGN>(), N = 2 * H;
    constexpr int R1 = HLOGN - 8, E1 = 1 << R1, LG1 = HLOGN - R1; // first pass: stage 0 on the loads, then R1 stages; then 4 + 4
    extern __shared__ __align__(16) u64 ks_raw[];
    double *sm = reinterpret_cast<double *>(ks_raw);           // [3][H]: work buffers 0 and 1, polynomial-1 accumulator
    double *acc1 = sm + 2 * H;                                 // group layout (st_group16); work 1 and acc 1 are the inverse's half buffers
    double *twc = sm + 3 * H, *twci = twc + TWC;               // forward / inverse twiddles of this half
    const int half = blockIdx.x & 1, l = (blockIdx.x >> 1) % k, c = (blockIdx.x >> 1) / k, tid = threadIdx.x;
    NttTab tb = tabs[l];
    const double w0 = __ldg(tb.wd + 1);
    tb.wd = tb.wd_split + half * H;
    tb.iwd = tb.iwd_split + half * H;
    tb.fwd_recenter = tb.fwd_recenter_split;
    const double2 *twg = reinterpret_cast<const double2 *>(tb.wd_split_grp + half * H); // last forward pass, grouped
    const double p = tb.pd, pinv = tb.pinv;
    const bool need_reduce = dm.mask >= tb.mod.p;
    const u64 *src_c = target + (size_t)c * ct_stride;
    const size_t kpoly = (size_t)k * N, kstride = 2 * kpoly;
    if (key_tab) { // per-ciphertext keys (several clients' key slots in one call): the table holds the form this instantiation reads
        if constexpr (PK) keyp = key_base<REF>(reinterpret_cast<const uint4 *>(key_tab[c]));
        else key = key_base<REF>(key_tab[c]);
    } else if constexpr (REF) {
        if constexpr (PK) keyp = key_base<REF>(keyp);
        else key = key_base<REF>(key);
    }
    const u64 *key_l = key + (size_t)l * N + half * H + 16 * tid;
    load_twiddle_cache(twc, tb.wd, tid, TR);
    load_twiddle_cache(twci, tb.iwd, tid, TR);
    double acc0[16]; // polynomial 0's accumulator: coefficients 16 tid .. 16 tid + 15
#pragma unroll
    for (int e = 0; e < 16; e++) acc0[e] = 0.0;
    st_group16(acc1, tid, acc0);
    auto cut = [&](u64 v, int shift) { // digit of a canonical word: exact below 2^50
        const double x = u2d((v >> shift) & dm.mask);
        return need_reduce ? frecenter(x, p, pinv) : x;
    };
    __syncthreads(); // the twiddle caches are filled
#pragma unroll 1
    for (int d = 0; d < dm.D; d++) {
        // Digit d runs in work buffer d & 1, whose last user was digit d - 2: every thread passed the barrier after digit d - 1's first
        // pass only once it had finished digit d - 2 (its middle- and last-pass reads included), and this thread has passed that barrier
        // too, so the first-pass stores below need no barrier of their own.
        double *wb = sm + (d & 1) * H;
        const u64 *src = src_c + (size_t)dm.src[d] * N;
        const int shift = dm.shift[d];
        if (d == dm.D - 1) { // the epilogue adds this half of both base polynomials: have them waiting in L2
#pragma unroll
            for (int kp = 0; kp < 2; kp++) {
                const char *pb = reinterpret_cast<const char *>(base + (size_t)c * base_stride + kp * kpoly + (size_t)l * N + half * H);
                for (int i = tid * 128; i < H * 8; i += TR * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb + i));
            }
        }
        constexpr int VT1 = (H >> R1) / TR; // first-pass virtual threads per thread
        double xs[VT1][E1]; // stage 0 of the N-point transform
#pragma unroll
        for (int v = 0; v < VT1; v++)
#pragma unroll
            for (int e = 0; e < E1; e++) {
                const int idx = tid + v * TR + (e << LG1);
                double a, t;
                if constexpr (PL) {
                    const int *pl = planes + ((size_t)c * dm.D + d) * N;
                    a = (double)pl[idx];
                    t = fmodmul((double)pl[idx + H], w0, p, pinv);
                } else {
                    a = cut(src[idx], shift);
                    t = fmodmul(cut(src[idx + H], shift), w0, p, pinv);
                }
                xs[v][e] = half ? __dsub_rn(a, t) : __dadd_rn(a, t);
            }
#pragma unroll
        for (int v = 0; v < VT1; v++) {
            const int vt = tid + v * TR;
            double (&x)[E1] = xs[v];
#pragma unroll
            for (int u = 0; u < R1; u++) {
                const int h = E1 >> (u + 1);
#pragma unroll
                for (int e = 0; e < E1; e++) {
                    if (e & h) continue;
                    const double w = twc[(1 << u) + (e >> (R1 - u))];
                    const double t = fmodmul(x[e + h], w, p, pinv);
                    const double a = x[e];
                    x[e] = __dadd_rn(a, t);
                    x[e + h] = __dsub_rn(a, t);
                }
            }
            // swz only moves bits 1..3 by bits 4..6, so with LG1 >= 7 this is wb[swz(vt + (e << LG1))]: one address register and
            // immediate offsets instead of 2^R1 swizzled offsets the compiler would keep live through the digit loop
            static_assert(LG1 >= 7, "first-pass store offsets must not touch the swizzle's bits");
            double *o = wb + swz(vt);
#pragma unroll
            for (int e = 0; e < E1; e++) o[e << LG1] = x[e];
        }
        __syncthreads(); // the first pass is all-to-all
        {
            FwdSrc unused;
            unused.src = nullptr; unused.digit = false; unused.need_reduce = false; unused.shift = 0; unused.mask = 0;
            fwd_pass_fp<HLOGN, R1, 4, false, 1, false>(wb, twc, unused, tb, tid);
        }
        __syncwarp(); // the middle pass wrote 256-coefficient block tid >> 4, whose groups 16j..16j+15 this half warp reads next
        // last pass (stages HLOGN-4 .. HLOGN-1 on 16 consecutive coefficients), then the key product
        double x[16];
        // j is tid, opaque to the compiler: the 8 chunk offsets of the thread's group (work buffer and acc 1) are recomputed each digit,
        // a few integer instructions, instead of being held in registers through the loop beside acc0, where they would spill
        int j = tid;
        asm volatile("" : "+r"(j));
        double2 *acc1v = reinterpret_cast<double2 *>(acc1) + 8 * j; // pair i of the group sits at acc1v[i ^ (j & 7)] (st_group16)
        const int xr = j & 7;
        ld_group16(wb, j, x);
        fwd_last_stages_grp<HLOGN, 2>(x, tb, twg, tid);
        if (tb.split_out_rc) {
#pragma unroll
            for (int e = 0; e < 16; e++) x[e] = frecenter(x[e], p, pinv);
        }
        const bool rc = (d & 7) == 7 || d == dm.D - 1;
        // coefficient pair i (words 2i, 2i+1) of key polynomial kp into its accumulator; sums of 8 fresh products stay below 4.1 p, so
        // they are re-centred before they could leave the exact range (and at the end)
        auto mac = [&](int kp, int i, double k0, double k1) {
            if (kp == 0) {
                acc0[2 * i] = __dadd_rn(acc0[2 * i], fmodmul(x[2 * i], k0, p, pinv));
                acc0[2 * i + 1] = __dadd_rn(acc0[2 * i + 1], fmodmul(x[2 * i + 1], k1, p, pinv));
                if (rc) {
                    acc0[2 * i] = frecenter(acc0[2 * i], p, pinv);
                    acc0[2 * i + 1] = frecenter(acc0[2 * i + 1], p, pinv);
                }
            } else {
                double2 a = acc1v[i ^ xr];
                a.x = __dadd_rn(a.x, fmodmul(x[2 * i], k0, p, pinv));
                a.y = __dadd_rn(a.y, fmodmul(x[2 * i + 1], k1, p, pinv));
                if (rc) {
                    a.x = frecenter(a.x, p, pinv);
                    a.y = frecenter(a.y, p, pinv);
                }
                acc1v[i ^ xr] = a;
            }
        };
#pragma unroll
        for (int kp = 0; kp < 2; kp++) {
            if constexpr (PK) {
                const uint4 *kw = keyp + ((((size_t)d * 2 + kp) * k + l) * 2 + half) * 6 * TR + tid;
#pragma unroll
                for (int hb = 0; hb < 2; hb++) { // 8 words from 3 groups at a time: all 24 u32 beside acc0 would not fit in 128 registers
                    unsigned u[12];
#pragma unroll
                    for (int g = 0; g < 3; g++) {
                        const uint4 v = __ldg(kw + (3 * hb + g) * TR);
                        u[4 * g] = v.x; u[4 * g + 1] = v.y; u[4 * g + 2] = v.z; u[4 * g + 3] = v.w;
                    }
#pragma unroll
                    for (int m = 0; m < 4; m++)
                        mac(kp, 4 * hb + m, u48d(u[3 * m], u[3 * m + 1] & 0xffff),
                            u48d(__funnelshift_r(u[3 * m + 1], u[3 * m + 2], 16), u[3 * m + 2] >> 16));
                }
            } else {
                const u64 *kw = key_l + (size_t)d * kstride + kp * kpoly;
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    const ulonglong2 w = __ldg(reinterpret_cast<const ulonglong2 *>(kw) + i);
                    mac(kp, i, u2d(w.x), u2d(w.y));
                }
            }
        }
    }
    // The inverse's table fields are read again here: held in registers through the digit loop beside acc0, they would spill.  The
    // empty asm hides that the pointer is tabs + l, so the compiler cannot reuse the loads made before the loop.
    const NttTab *tabl = tabs + l;
    asm("" : "+l"(tabl));
    NttTab ti = *tabl;
    ti.iwd = ti.iwd_split + half * H;
    const double2 *twgi = reinterpret_cast<const double2 *>(ti.iwd_split_grp + half * H); // first inverse stages, grouped
    // Inverse stages 0..3 of both accumulators in registers, each on the thread's own group: polynomial 0 into work buffer 1 (whichever
    // buffer the last digit used, group tid of it is read by no other thread now), polynomial 1 in place.
    inv_first_stages_grp<HLOGN>(acc0, ti, twgi, tid);
    st_group16(sm + H, tid, acc0);
    {
        double x[16];
        ld_group16(acc1, tid, x);
        inv_first_stages_grp<HLOGN>(x, ti, twgi, tid);
        st_group16(acc1, tid, x);
    }
    __syncwarp(); // inv_pass_fp<.., 4, 4> works on 256-coefficient block tid >> 4 of each buffer: the groups this half warp just stored
#pragma unroll 1
    for (int r = 1; r < 3; r++) CNHE_VTN(H / 16, (inv_pass_fp<HLOGN, 4, 4, false, false>(sm + r * H, twci, nullptr, nullptr, ti, vt)));
    __syncthreads();
    const size_t ol = (size_t)l * N + half * H;
    inv_split_last<HLOGN, TR, false, 2>(sm + H, twci, out + (size_t)c * kstride + ol, kpoly, base + (size_t)c * base_stride + ol, ti, tid, half);
}

// ================================================================ fused BEHZ square, N = 4096 / 8192
// The square of a ciphertext in the extended base q u Bsk: d0 = c0^2, d1 = 2 c0 c1, d2 = c1^2 pointwise in the NTT domain, back in the
// coefficient domain.  Within one residue l the forward transforms, the products and the inverse transforms never leave that residue,
// so a cluster of two CTAs takes (ciphertext c, residue l) and only the lift before and the floor after cross residues.  As separate
// kernels (lift -> forward -> tensor -> inverse -> floor) every step is an HBM round trip of the whole extended ciphertext: 245
// polynomial passes per ciphertext at k = 5, kb = 6, against 125 here.  CTA h owns half h of the N-point transforms (the split form of
// the N = 16384 kernels and of the fused key switch): it folds stage 0 into its loads of both halves of c0_l and c1_l (the partner's
// reads of the same lines are L2 hits), runs the N/2-point forward passes of both, squares in registers right after the last forward
// pass and runs the first inverse pass on the same 16 coefficients per thread, then the remaining inverse passes of the three products
// together and the cross-half last stage (which carries N^-1) through DSMEM.  Lazy bounds: the forward output is re-centred where
// split_out_rc says so (|c|^2 p < 2^51); |d1| <= 1.02 p is within the inverse's 1.25 p input bound; inv_recenter is the full transform's.
// Sources: residue l < k is the canonical input residue itself, l >= k the lift's lazy Bsk residue ([c][2][kb][N]).  Output: lazy
// doubles in the [c][3][kt][N] layout of the separate inverse transforms, which the floor reads.
template <int HLOGN>
__host__ __device__ constexpr int sq_fused_threads() { return (1 << HLOGN) / 16; }
template <int HLOGN>
__host__ __device__ constexpr int sq_fused_smem() { return (1 << HLOGN) * 8 * 3 + 2 * TWC * 8; } // three half buffers, two twiddle caches
template <int HLOGN>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(sq_fused_threads<HLOGN>(), HLOGN == 12 ? 2 : 4)
k_behz_square_fused(const u64 *const *__restrict__ ct_ptrs, const u64 *__restrict__ lift, u64 *__restrict__ d, const NttTab *__restrict__ tabs,
                    int k, int kt) {
    constexpr int H = 1 << HLOGN, TR = sq_fused_threads<HLOGN>(), N = 2 * H, R1 = HLOGN - 8;
    extern __shared__ __align__(16) u64 sq_raw[];
    double *sm = reinterpret_cast<double *>(sq_raw); // [3][H]: c0 then d0, c1 then d1, d2
    double *twc = sm + 3 * H, *twci = twc + TWC;    // forward / inverse twiddles of this half
    const int half = blockIdx.x & 1, l = (blockIdx.x >> 1) % kt, c = (blockIdx.x >> 1) / kt, tid = threadIdx.x;
    NttTab tb = tabs[l];
    const double w0 = __ldg(tb.wd + 1);
    tb.wd = tb.wd_split + half * H;
    tb.iwd = tb.iwd_split + half * H;
    tb.fwd_recenter = tb.fwd_recenter_split;
    const double p = tb.pd, pinv = tb.pinv;
    FwdSrc fs;
    fs.digit = false; fs.need_reduce = false; fs.shift = 0; fs.mask = 0;
    load_twiddle_cache(twc, tb.wd, tid, TR);
    load_twiddle_cache(twci, tb.iwd, tid, TR);
    __syncthreads();
#pragma unroll 1
    for (int r = 0; r < 2; r++) {
        if (l < k) {
            fs.src = ct_ptrs[c] + ((size_t)r * k + l) * N;
            CNHE_VTN(H >> R1, (fwd_split_first<HLOGN, false>(sm + r * H, twc, fs, tb, vt, w0, half != 0)));
        } else {
            fs.src = lift + ((size_t)(c * 2 + r) * (kt - k) + (l - k)) * N;
            CNHE_VTN(H >> R1, (fwd_split_first<HLOGN, true>(sm + r * H, twc, fs, tb, vt, w0, half != 0)));
        }
    }
    __syncthreads();
#pragma unroll 1
    for (int r = 0; r < 2; r++) CNHE_VTN(H / 16, (fwd_pass_fp<HLOGN, R1, 4, false, 1, false>(sm + r * H, twc, fs, tb, vt)));
    __syncwarp(); // the pass above wrote 256-coefficient block tid >> 4 of each buffer, whose groups 16j..16j+15 this half warp reads next
    {
        // thread j owns coefficients 16j .. 16j+15 of every buffer from the last forward pass to the first inverse pass: no barrier.
        // One group of 16 in registers per transform step (two plus the twiddles spill): c0 and c1 wait in their own slots
        const int j = tid;
        const double2 *twg = reinterpret_cast<const double2 *>(tb.wd_split_grp + half * H);
        const double2 *twgi = reinterpret_cast<const double2 *>(tb.iwd_split_grp + half * H);
        double x[16], y[16];
#pragma unroll 1
        for (int r = 0; r < 2; r++) {
            ld_group16(sm + r * H, j, x);
            if constexpr (HLOGN == 12) fwd_last_stages_grp<HLOGN, 2>(x, tb, twg, j);
            else fwd_last_stages<HLOGN, 2>(x, tb, j); // N = 4096: with the grouped loads ptxas spills 8 bytes here
            if (tb.split_out_rc) {
#pragma unroll
                for (int e = 0; e < 16; e++) x[e] = frecenter(x[e], p, pinv);
            }
            st_group16(sm + r * H, j, x);
        }
        // the products of k_behz_tensor_fp (square): d2 = c1^2, d1 = 2 c0 c1, d0 = c0^2, each overwriting a slot no longer read
        ld_group16(sm + H, j, x);
#pragma unroll
        for (int e = 0; e < 16; e++) x[e] = fmodmul(x[e], x[e], p, pinv);
        inv_first_stages_grp<HLOGN>(x, tb, twgi, j);
        st_group16(sm + 2 * H, j, x);
        ld_group16(sm, j, x);
        ld_group16(sm + H, j, y);
#pragma unroll
        for (int e = 0; e < 16; e++) {
            const double cross = fmodmul(x[e], y[e], p, pinv);
            y[e] = __dadd_rn(cross, cross);
        }
        inv_first_stages_grp<HLOGN>(y, tb, twgi, j);
        st_group16(sm + H, j, y);
#pragma unroll
        for (int e = 0; e < 16; e++) x[e] = fmodmul(x[e], x[e], p, pinv);
        inv_first_stages_grp<HLOGN>(x, tb, twgi, j);
        st_group16(sm, j, x);
    }
    __syncwarp(); // inv_pass_fp<.., 4, 4> works on 256-coefficient block tid >> 4 of each buffer: the groups this half warp just stored
#pragma unroll 1
    for (int r = 0; r < 3; r++) CNHE_VTN(H / 16, (inv_pass_fp<HLOGN, 4, 4, false, false>(sm + r * H, twci, nullptr, nullptr, tb, vt)));
    __syncthreads();
    inv_split_last<HLOGN, TR, true, 3>(sm, twci, d + ((size_t)c * 3 * kt + l) * N + half * H, (size_t)kt * N, nullptr, tb, tid, half);
}

// ================================================================ persistent TMA-staged inverse transform, N = 4096 / 8192
// One persistent CTA per SM.  Each CTA is pinned to ONE modulus (CTA c serves the polynomials whose table index is c mod #moduli), so
// the twiddles it needs never change: the 15N/16 twiddles of the four unit-stride stages -- the ones that used to be fetched from L2 by
// every polynomial (as many bytes as the polynomial itself, and the top stall of the one-CTA-per-polynomial kernel) -- are staged into
// shared memory ONCE per CTA with cp.async.bulk, transposed so that lane j reads word m*T + j (conflict-free), next to the 512 low
// twiddles of the strided stages.  Polynomials arrive by cp.async.bulk.tensor (a 2-D tensor map over the source array, 128-byte rows,
// SWIZZLE_128B -- exactly the XOR layout swz() the butterfly passes use, so the hardware produces the bank-conflict-free layout on the
// way in), completing on an mbarrier.  Two groups of 8 warps each own one polynomial slot: three fat passes in place between named
// barriers of the group, results written straight from registers, then one elected thread refills the slot with the group's next
// polynomial.  No compute warp ever waits on HBM or L2 for data or twiddles, there is no CTA launch/exit (store drain) per polynomial,
// and the groups run out of phase so that one group's shared-memory round trips and slot refill hide under the other's FP64 work.
// The forward transform stays one CTA per polynomial (k_ntt_forward_fp): staged the same way it gained nothing, and its digit-cutting
// form was slower (DESIGN.md §4.2).
constexpr int WS_GROUPS = 2, WS_GROUP_THREADS = 256, WS_THREADS = WS_GROUPS * WS_GROUP_THREADS;
constexpr unsigned WS_STAGGER_NS = 5000; // group 1 starts this much later than group 0 (the groups should not walk through the passes in lockstep)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// (a suspend-time hint on the try_wait -- the waiting warps sleep instead of spinning -- measured 3 % slower here: the wake-up latency
// costs more than the issue slots the spinning takes from the other group; mac_umma.cu, with ten mostly-waiting warps, keeps the hint)
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(
                     smem_u32(bar)),
                 "r"(parity)
                 : "memory");
}
__device__ __forceinline__ void tma_load_rows(void *dst, const void *tmap, int row, unsigned long long *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
                 "l"(tmap), "r"(0), "r"(row), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_load(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void ws_delay(unsigned ns) {
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do {
        __nanosleep(200);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    } while (t1 - t0 < ns);
}
__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, %1;" ::"r"(g + 1), "n"(WS_GROUP_THREADS) : "memory"); }

// a __grid_constant__ kernel parameter: read from the parameter bank where used (passed as a plain value, the small record is copied
// into registers and the kernel, already at 128 registers, spills more)
struct WsArgs {
    int n_polys, mod_base, mod_count; // polynomial b uses table mod_base + b % mod_count, source row b * N/16, destination b * N
    // optional base added to the canonical result
    const u64 *base_add;
    int base_group;
    size_t base_stride;
};
// stage polynomial `b` into a slot; called by one thread
template <int LOGN>
__device__ __forceinline__ void ws_issue(const CUtensorMap *tmap, double *slot, unsigned long long *full, int b) {
    constexpr int N = 1 << LOGN;
    constexpr int BOX_ROWS = 256, BOXES = (N / 16) / BOX_ROWS;
    const long long row = (long long)b * (N / 16); // first 128-byte row of the polynomial in the tensor map
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // the slot's previous contents were read through the generic proxy
    mbar_expect_tx(full, (unsigned)(N * 8));
#pragma unroll
    for (int x = 0; x < BOXES; x++) tma_load_rows(slot + x * BOX_ROWS * 16, tmap, (int)(row + x * BOX_ROWS), full);
}
// first inverse pass on the staged words: stages 0..3 on 16 consecutive coefficients, in place; twiddles from the resident table
template <int LOGN, bool IN_F>
__device__ __forceinline__ void inv_first_staged(double *sm, const NttTab &tb, const double *hi, int j) {
    constexpr int T = (1 << LOGN) / 16;
    const double p = tb.pd, pinv = tb.pinv;
    double2 *smv = reinterpret_cast<double2 *>(sm);
    const int xr = j & 7;
    double x[16];
#pragma unroll
    for (int ch = 0; ch < 8; ch++) {
        const double2 v = smv[j * 8 + (ch ^ xr)];
        if constexpr (IN_F) { x[2 * ch] = v.x; x[2 * ch + 1] = v.y; }
        else { x[2 * ch] = u2d((u64)__double_as_longlong(v.x)); x[2 * ch + 1] = u2d((u64)__double_as_longlong(v.y)); }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int h = 1 << u;
        const bool rc = (tb.inv_recenter >> u) & 1;
#pragma unroll
        for (int e = 0; e < 16; e++) {
            if (e & h) continue;
            const double w = hi[((16 - (16 >> u)) + (e >> (u + 1))) * T + j];
            const double a = x[e], bq = x[e + h];
            x[e] = __dadd_rn(a, bq);
            x[e + h] = fmodmul(__dsub_rn(a, bq), w, p, pinv);
        }
        if (rc) {
#pragma unroll
            for (int e = 0; e < 16; e++)
                if (!(e & h)) x[e] = frecenter(x[e], p, pinv);
        }
    }
#pragma unroll
    for (int ch = 0; ch < 8; ch++) smv[j * 8 + (ch ^ xr)] = make_double2(x[2 * ch], x[2 * ch + 1]);
}

#define CNHE_WS_VT(COUNT, stmt) _Pragma("unroll") for (int vt = gt; vt < (COUNT); vt += WS_GROUP_THREADS) { stmt; }
template <int LOGN>
__host__ __device__ constexpr int ws_hi_words() { return 15 * (1 << LOGN) / 16; }
template <int LOGN>
__host__ __device__ constexpr int ws_smem_bytes() { return (WS_GROUPS * (1 << LOGN) + ws_hi_words<LOGN>() + TWC) * 8 + 64 + (int)sizeof(NttTab) + 1024; }

// shared prologue: carve shared memory, stage the CTA's twiddle tables and the first polynomial of each group
struct WsSmem {
    double *slots, *hi, *lo; // slot g = slots + g * N (plain pointer arithmetic on the __shared__ symbol keeps the address space)
    unsigned long long *full, *tbar, *empty;
    NttTab *tab; // the CTA's modulus record, copied once: per-polynomial reads are LDS instead of (L1-missing) global loads
};
template <int LOGN>
__device__ __forceinline__ WsSmem ws_carve(unsigned char *raw) {
    constexpr int N = 1 << LOGN;
    WsSmem w;
    // SWIZZLE_128B wants 1024-byte aligned slots.  The padding is added to the __shared__ symbol itself (no integer round trip), so the
    // compiler still knows every derived pointer is shared memory and emits LDS/STS instead of generic loads
    const unsigned pad = (1024u - (smem_u32(raw) & 1023u)) & 1023u;
    double *base = reinterpret_cast<double *>(raw + pad);
    w.slots = base;
    w.hi = base + (size_t)WS_GROUPS * N;
    w.lo = w.hi + ws_hi_words<LOGN>();
    w.full = reinterpret_cast<unsigned long long *>(w.lo + TWC);
    w.tbar = w.full + WS_GROUPS;
    w.empty = w.tbar + 1;
    w.tab = reinterpret_cast<NttTab *>(w.empty + WS_GROUPS);
    return w;
}
// which polynomials this CTA serves: class m = blockIdx % mc (its modulus), the r-th CTA of the S CTAs of that class takes j = r, r + S, ...
struct WsWalk {
    int m, mc, r, S;
    __device__ __forceinline__ int poly(int s) const { return m + mc * (r + s * S); } // sequence number -> polynomial index (may run past n_polys)
};
__device__ __forceinline__ WsWalk ws_walk(int mc) {
    WsWalk w;
    w.mc = mc;
    w.m = blockIdx.x % mc;
    w.r = blockIdx.x / mc;
    w.S = ((int)gridDim.x - w.m + mc - 1) / mc;
    return w;
}

template <int LOGN, bool IN_F, bool OUT_F>
__global__ void __launch_bounds__(WS_THREADS, 1)
k_ntt_inverse_ws(const __grid_constant__ CUtensorMap tmap, u64 *dst, const NttTab *__restrict__ tabs, const __grid_constant__ WsArgs a) {
    static_assert(LOGN == 12 || LOGN == 13, "the staged transform covers N = 4096 and 8192");
    constexpr int N = 1 << LOGN;
    extern __shared__ unsigned char ws_raw[];
    const int tid = threadIdx.x;
    {
        const WsSmem sm_ = ws_carve<LOGN>(ws_raw);
        const WsWalk walk = ws_walk(a.mod_count);
        if (tid == 0) {
            const NttTab &tb0 = tabs[a.mod_base + walk.m];
            *sm_.tab = tb0;
            for (int g = 0; g < WS_GROUPS; g++) { mbar_init(&sm_.full[g], 1); mbar_init(&sm_.empty[g], WS_GROUP_THREADS); }
            mbar_init(sm_.tbar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            mbar_expect_tx(sm_.tbar, (unsigned)((ws_hi_words<LOGN>() + TWC) * 8));
            bulk_load(sm_.hi, tb0.iwd_hi, ws_hi_words<LOGN>() * 8, sm_.tbar);
            bulk_load(sm_.lo, tb0.iwd, TWC * 8, sm_.tbar);
            for (int g = 0; g < WS_GROUPS; g++)
                if (walk.poly(g) < a.n_polys) ws_issue<LOGN>(&tmap, sm_.slots + (size_t)g * N, &sm_.full[g], walk.poly(g));
        }
        __syncthreads();
        mbar_wait(sm_.tbar, 0);
    }
    const int g = tid / WS_GROUP_THREADS, gt = tid % WS_GROUP_THREADS;
    if (g == 1) ws_delay(WS_STAGGER_NS);
#pragma unroll 1
    for (int t = 0;; t++) {
        const WsWalk walk = ws_walk(a.mod_count);
        const int b = walk.poly(g + WS_GROUPS * t);
        if (b >= a.n_polys) break;
        const WsSmem sm_ = ws_carve<LOGN>(ws_raw);
        const NttTab &tb = *sm_.tab;
        double *sm = sm_.slots + (size_t)g * N;
        const double *twc = sm_.lo, *hi = sm_.hi;
        u64 *d = dst + (size_t)b * N;
        const u64 *ba = a.base_add ? a.base_add + (size_t)(b / a.base_group) * a.base_stride + (size_t)(b % a.base_group) * N : nullptr;
        if (ba) { // consumed by the epilogue most of a transform from now: have it waiting in L2
            const char *pb = reinterpret_cast<const char *>(ba);
            for (int i = gt * 128; i < N * 8; i += WS_GROUP_THREADS * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(pb + i));
        }
        auto refill = [&]() {
            mbar_arrive(&sm_.empty[g]);
            const int nb = walk.poly(g + WS_GROUPS * (t + 1));
            if (gt == 0 && nb < a.n_polys) {
                mbar_wait(&sm_.empty[g], t & 1);
                ws_issue<LOGN>(&tmap, sm, &sm_.full[g], nb);
            }
        };
        mbar_wait(&sm_.full[g], t & 1);
        CNHE_WS_VT(N / 16, (inv_first_staged<LOGN, IN_F>(sm, tb, hi, vt))); group_sync(g);
        if constexpr (LOGN == 13) {
            CNHE_WS_VT(N / 16, (inv_pass_fp<13, 4, 4, false, false>(sm, twc, d, ba, tb, vt))); group_sync(g);
            inv_pass_fp<13, 8, 5, true, OUT_F, 1>(sm, twc, d, ba, tb, gt, 0, refill); // one radix-32 group per thread
        } else {
            CNHE_WS_VT(N / 16, (inv_pass_fp<12, 4, 4, false, false>(sm, twc, d, ba, tb, vt))); group_sync(g);
            inv_pass_fp<12, 8, 4, true, OUT_F, 1>(sm, twc, d, ba, tb, gt, 0, refill);
        }
    }
}

int ntt_pass_radices(int logn, int inverse, int *r) {
    static const int F[5][4] = {{2, 4, 4, 0}, {3, 4, 4, 0}, {4, 4, 4, 0}, {5, 4, 4, 0}, {5, 5, 4, 0}};
    static const int I[5][4] = {{4, 4, 2, 0}, {4, 4, 3, 0}, {4, 4, 4, 0}, {4, 4, 5, 0}, {4, 5, 5, 0}};
    if (logn < 10 || logn > 14) return 0;
    int n = 0;
    for (int i = 0; i < 4; i++) {
        r[i] = inverse ? I[logn - 10][i] : F[logn - 10][i];
        if (r[i]) n++;
    }
    return n;
}

// ---------------------------------------------------------------- launchers
int ntt_kernel_smem_bytes(int logn) { return (1 << logn) * 8 + TWC * 8; } // polynomial + twiddle cache (FP64 path)

template <class K>
static cudaError_t prep(K kern, int logn) {
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, ntt_kernel_smem_bytes(logn));
}

// ---- tensor maps (the persistent inverse transform, mac_umma.cu): the encoder is a driver entry point
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) p = nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}
constexpr int SPLIT_SMEM = SPLIT_H * 8 + TWC * 8;
template <class K>
static cudaError_t split_prep(K kern) {
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SPLIT_SMEM);
}
static int sm_count() {
    static int n = [] {
        int dev = 0, v = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        return v;
    }();
    return n;
}
// rows of 16 words (128 bytes) starting at `base`; boxes of 256 rows, hardware swizzle = swz()
static cudaError_t make_row_map(CUtensorMap *m, const u64 *base, size_t words) {
    if (encode_tiled() == nullptr) return cudaErrorNotSupported; // every CUDA 12 driver (the least an sm_90a binary loads on) exports it
    const cuuint64_t dims[2] = {16, (cuuint64_t)(words / 16)};
    const cuuint64_t strides[1] = {128};
    const cuuint32_t box[2] = {16, 256}, estr[2] = {1, 1};
    if (words % 16 || dims[1] < 256 || (reinterpret_cast<uintptr_t>(base) & 15)) return cudaErrorInvalidValue;
    const CUresult r = encode_tiled()(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<u64 *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}
// General 2-D map over 64-bit words for other kernels (mac_umma.cu): `rows` rows of `inner_words` words, `row_stride` bytes apart, box of
// box_words x box_rows, optionally SWIZZLE_128B (box rows of 128 bytes), out-of-bounds rows read as zero.  `map` points at a CUtensorMap (128 bytes, 64-byte aligned).
cudaError_t make_word_map_2d(void *map, const u64 *base, size_t inner_words, size_t rows, size_t row_stride, unsigned box_words, unsigned box_rows,
                             int swizzle128) {
    if (encode_tiled() == nullptr) return cudaErrorNotSupported;
    const cuuint64_t dims[2] = {(cuuint64_t)inner_words, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)row_stride};
    const cuuint32_t box[2] = {box_words, box_rows}, estr[2] = {1, 1};
    if ((row_stride & 15) || (reinterpret_cast<uintptr_t>(base) & 15) || box_words > 256 || box_rows > 256 || (swizzle128 && box_words != 16))
        return cudaErrorInvalidValue;
    const CUresult r = encode_tiled()(reinterpret_cast<CUtensorMap *>(map), CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<u64 *>(base), dims, strides, box, estr,
                                      CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

#define CNHE_DISPATCH_LOGN(logn, ...)                                                                                 \
    switch (logn) {                                                                                                     \
    case 10: { constexpr int L = 10; __VA_ARGS__; } break;                                                                     \
    case 11: { constexpr int L = 11; __VA_ARGS__; } break;                                                                     \
    case 12: { constexpr int L = 12; __VA_ARGS__; } break;                                                                     \
    case 13: { constexpr int L = 13; __VA_ARGS__; } break;                                                                     \
    case 14: { constexpr int L = 14; __VA_ARGS__; } break;                                                                     \
    default: return cudaErrorInvalidValue;                                                                              \
    }

// FP64 transforms by ring degree.  Forward: one CTA per polynomial up to N = 8192, CTA pairs at N = 16384.  Inverse: one CTA per
// polynomial at N = 1024 / 2048, the persistent kernel at N = 4096 / 8192, CTA pairs at N = 16384.
template <int L, bool LAZY>
static cudaError_t launch_fwd_fp(const u64 *src, u64 *dst, int n_polys, const NttTab *tabs, int mod_base, int mod_count, cudaStream_t s) {
    if constexpr (L == 14) {
        cudaError_t e = split_prep(k_ntt_forward_split<LAZY, LAZY>);
        if (e != cudaSuccess) return e;
        k_ntt_forward_split<LAZY, LAZY><<<2 * n_polys, SPLIT_THREADS, SPLIT_SMEM, s>>>(src, dst, tabs, mod_base, mod_count);
    } else {
        cudaError_t e = prep(k_ntt_forward_fp<L, LAZY, LAZY>, L);
        if (e != cudaSuccess) return e;
        k_ntt_forward_fp<L, LAZY, LAZY><<<n_polys, fp_threads(L), ntt_kernel_smem_bytes(L), s>>>(src, dst, tabs, mod_base, mod_count);
    }
    return cudaGetLastError();
}
template <int L, bool OUT_F>
static cudaError_t launch_fwd_digits_fp(const u64 *target, size_t ct_stride, u64 *dst, int n_polys, int k, const DigitMap &dm, const NttTab *tabs,
                                        cudaStream_t s) {
    if constexpr (L == 14) {
        cudaError_t e = split_prep(k_ntt_forward_digits_split<OUT_F>);
        if (e != cudaSuccess) return e;
        k_ntt_forward_digits_split<OUT_F><<<2 * n_polys, SPLIT_THREADS, SPLIT_SMEM, s>>>(target, ct_stride, dst, tabs, k, dm);
    } else {
        cudaError_t e = prep(k_ntt_forward_digits_fp<L, OUT_F>, L);
        if (e != cudaSuccess) return e;
        k_ntt_forward_digits_fp<L, OUT_F><<<n_polys, fp_threads(L), ntt_kernel_smem_bytes(L), s>>>(target, ct_stride, dst, tabs, k, dm);
    }
    return cudaGetLastError();
}
template <int L, bool IN_F, bool OUT_F>
static cudaError_t launch_inv_fp(const u64 *src, const u64 *base, int base_group, size_t base_stride, u64 *dst, int n_polys, const NttTab *tabs,
                                 int mod_base, int mod_count, cudaStream_t s) {
    if constexpr (L == 14) {
        cudaError_t e = split_prep(k_ntt_inverse_split<IN_F, OUT_F>);
        if (e != cudaSuccess) return e;
        k_ntt_inverse_split<IN_F, OUT_F><<<2 * n_polys, SPLIT_THREADS, SPLIT_SMEM, s>>>(src, base, base_group, base_stride, dst, tabs, mod_base, mod_count);
    } else if constexpr (L >= 12) { // tensor map over the source array, persistent grid of one CTA per SM
        CUtensorMap map;
        cudaError_t e = make_row_map(&map, src, (size_t)n_polys << L);
        if (e != cudaSuccess) return e;
        const WsArgs a = {n_polys, mod_base, mod_count, base, base_group, base_stride};
        constexpr int smem = ws_smem_bytes<L>();
        e = cudaFuncSetAttribute(k_ntt_inverse_ws<L, IN_F, OUT_F>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return e;
        int grid = sm_count();
        if (mod_count <= grid) grid -= grid % mod_count; // equally many CTAs per modulus: every CTA is pinned to one
        if (n_polys < grid) grid = n_polys;
        k_ntt_inverse_ws<L, IN_F, OUT_F><<<grid, WS_THREADS, smem, s>>>(map, dst, tabs, a);
    } else {
        cudaError_t e = prep(k_ntt_inverse_fp<L, IN_F, OUT_F>, L);
        if (e != cudaSuccess) return e;
        k_ntt_inverse_fp<L, IN_F, OUT_F><<<n_polys, fp_threads(L), ntt_kernel_smem_bytes(L), s>>>(src, base, base_group, base_stride, dst, tabs, mod_base,
                                                                                                mod_count);
    }
    return cudaGetLastError();
}

// `fp`: 0 = integer Harvey butterflies; NTT_FP = FP64 butterflies, optionally | NTT_IN_F (source holds lazy doubles) | NTT_OUT_F
// (destination receives lazy doubles instead of canonical words)
cudaError_t launch_ntt_forward(const u64 *src, u64 *dst, int n_polys, int logn, const NttTab *tabs, int mod_base, int mod_count, int fp,
                               cudaStream_t s) {
    if (n_polys <= 0) return cudaSuccess;
    if (fp & NTT_FP) {
        const bool lazy = (fp & (NTT_IN_F | NTT_OUT_F)) == (NTT_IN_F | NTT_OUT_F);
        if (!lazy && (fp & (NTT_IN_F | NTT_OUT_F))) return cudaErrorInvalidValue; // only canonical->canonical and lazy->lazy are built
        CNHE_DISPATCH_LOGN(logn, return lazy ? launch_fwd_fp<L, true>(src, dst, n_polys, tabs, mod_base, mod_count, s)
                                             : launch_fwd_fp<L, false>(src, dst, n_polys, tabs, mod_base, mod_count, s));
    }
    CNHE_DISPATCH_LOGN(logn, {
        cudaError_t e = prep(k_ntt_forward<L>, L);
        if (e != cudaSuccess) return e;
        k_ntt_forward<L><<<n_polys, (1 << L) / 16, ntt_kernel_smem_bytes(L), s>>>(src, dst, tabs, mod_base, mod_count);
    });
    return cudaGetLastError();
}
cudaError_t launch_ntt_forward_digits(const u64 *target, size_t ct_stride, u64 *dst, int n_ct, int k, const DigitMap &dm, int logn,
                                      const NttTab *tabs, int fp, cudaStream_t s) {
    if (n_ct <= 0) return cudaSuccess;
    if (fp & NTT_FP) {
        if (fp & NTT_IN_F) return cudaErrorInvalidValue; // digits are cut from canonical words
        const int n_polys = n_ct * dm.D * k;
        CNHE_DISPATCH_LOGN(logn, return (fp & NTT_OUT_F) ? launch_fwd_digits_fp<L, true>(target, ct_stride, dst, n_polys, k, dm, tabs, s)
                                                         : launch_fwd_digits_fp<L, false>(target, ct_stride, dst, n_polys, k, dm, tabs, s));
    }
    CNHE_DISPATCH_LOGN(logn, {
        cudaError_t e = prep(k_ntt_forward_digits<L>, L);
        if (e != cudaSuccess) return e;
        k_ntt_forward_digits<L><<<n_ct * dm.D * k, (1 << L) / 16, ntt_kernel_smem_bytes(L), s>>>(target, ct_stride, dst, tabs, k, dm);
    });
    return cudaGetLastError();
}
template <int HL, bool PK, bool PL, bool REF>
static cudaError_t launch_ks_fused(const u64 *target, size_t ct_stride, const int *planes, const u64 *key, const uint4 *keyp,
                                   const u64 *const *key_tab, const u64 *base, size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm,
                                   const NttTab *tabs, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(k_key_switch_fused<HL, PK, PL, REF>, cudaFuncAttributeMaxDynamicSharedMemorySize, ks_fused_smem<HL>());
    if (e != cudaSuccess) return e;
    k_key_switch_fused<HL, PK, PL, REF><<<2 * n_ct * k, ks_fused_threads<HL>(), ks_fused_smem<HL>(), s>>>(target, ct_stride, planes, key, keyp,
                                                                                                        key_tab, base, base_stride, out, tabs, k, dm);
    return cudaGetLastError();
}
template <int HL, bool PL>
static cudaError_t launch_ks_fused(const u64 *target, size_t ct_stride, const int *planes, const u64 *key, const uint4 *keyp,
                                   const u64 *const *key_tab, const u64 *base, size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm,
                                   const NttTab *tabs, cudaStream_t s, bool ref) {
    if (ref)
        return keyp ? launch_ks_fused<HL, true, PL, true>(target, ct_stride, planes, key, keyp, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s)
                    : launch_ks_fused<HL, false, PL, true>(target, ct_stride, planes, key, keyp, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s);
    return keyp ? launch_ks_fused<HL, true, PL, false>(target, ct_stride, planes, key, keyp, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s)
                : launch_ks_fused<HL, false, PL, false>(target, ct_stride, planes, key, keyp, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s);
}
cudaError_t launch_key_switch_fused(const u64 *target, size_t ct_stride, const u64 *key, const uint4 *key_packed, const u64 *const *key_tab,
                                    const u64 *base, size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm, int logn,
                                    const NttTab *tabs, cudaStream_t s, bool ref) {
    if (n_ct <= 0) return cudaSuccess;
    if (logn == 13) return launch_ks_fused<12, false>(target, ct_stride, nullptr, key, key_packed, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s, ref);
    if (logn == 12) return launch_ks_fused<11, false>(target, ct_stride, nullptr, key, key_packed, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s, ref);
    return cudaErrorInvalidValue;
}
cudaError_t launch_key_switch_planes(const int *planes, const u64 *key, const uint4 *key_packed, const u64 *const *key_tab, const u64 *base,
                                     size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm, int logn, const NttTab *tabs, cudaStream_t s,
                                     bool ref) {
    if (n_ct <= 0) return cudaSuccess;
    if (logn == 13) return launch_ks_fused<12, true>(nullptr, 0, planes, key, key_packed, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s, ref);
    if (logn == 12) return launch_ks_fused<11, true>(nullptr, 0, planes, key, key_packed, key_tab, base, base_stride, out, n_ct, k, dm, tabs, s, ref);
    return cudaErrorInvalidValue;
}
template <int HL>
static cudaError_t launch_sq_fused(const u64 *const *ct_ptrs, const u64 *lift, u64 *d, int n_ct, int k, int kt, const NttTab *tabs, cudaStream_t s) {
    cudaError_t e = cudaFuncSetAttribute(k_behz_square_fused<HL>, cudaFuncAttributeMaxDynamicSharedMemorySize, sq_fused_smem<HL>());
    if (e != cudaSuccess) return e;
    k_behz_square_fused<HL><<<2 * n_ct * kt, sq_fused_threads<HL>(), sq_fused_smem<HL>(), s>>>(ct_ptrs, lift, d, tabs, k, kt);
    return cudaGetLastError();
}
cudaError_t launch_behz_square_fused(const u64 *const *ct_ptrs, const u64 *lift_bsk, u64 *d, int n_ct, int k, int kt, int logn, const NttTab *tabs,
                                     cudaStream_t s) {
    if (n_ct <= 0) return cudaSuccess;
    if (logn == 13) return launch_sq_fused<12>(ct_ptrs, lift_bsk, d, n_ct, k, kt, tabs, s);
    if (logn == 12) return launch_sq_fused<11>(ct_ptrs, lift_bsk, d, n_ct, k, kt, tabs, s);
    return cudaErrorInvalidValue;
}
template <int HL>
static cudaError_t launch_pk48(const u64 *key, uint4 *out, int n_polys, cudaStream_t s) {
    const int threads = n_polys * 2 * ks_fused_threads<HL>();
    k_pack_keys48<HL><<<(threads + 255) / 256, 256, 0, s>>>(key, out, n_polys);
    return cudaGetLastError();
}
cudaError_t launch_pack_keys48(const u64 *key, uint4 *out, int n_polys, int logn, cudaStream_t s) {
    if (n_polys <= 0) return cudaSuccess;
    if (logn == 13) return launch_pk48<12>(key, out, n_polys, s);
    if (logn == 12) return launch_pk48<11>(key, out, n_polys, s);
    return cudaErrorInvalidValue;
}
static cudaError_t launch_inv(const u64 *src, const u64 *base, int base_group, size_t base_stride, u64 *dst, int n_polys, int logn,
                              const NttTab *tabs, int mod_base, int mod_count, int fp, cudaStream_t s) {
    if (n_polys <= 0) return cudaSuccess;
    if (base_group < 1) base_group = 1;
    if (fp & NTT_FP) {
        const bool in_f = fp & NTT_IN_F, out_f = fp & NTT_OUT_F;
        if (out_f && (!in_f || base)) return cudaErrorInvalidValue; // built: canonical->canonical, lazy->lazy, lazy->canonical(+base)
        CNHE_DISPATCH_LOGN(logn, return out_f  ? launch_inv_fp<L, true, true>(src, base, base_group, base_stride, dst, n_polys, tabs, mod_base, mod_count, s)
                                        : in_f ? launch_inv_fp<L, true, false>(src, base, base_group, base_stride, dst, n_polys, tabs, mod_base, mod_count, s)
                                               : launch_inv_fp<L, false, false>(src, base, base_group, base_stride, dst, n_polys, tabs, mod_base, mod_count, s));
    }
    CNHE_DISPATCH_LOGN(logn, {
        cudaError_t e = prep(k_ntt_inverse<L>, L);
        if (e != cudaSuccess) return e;
        k_ntt_inverse<L><<<n_polys, (1 << L) / 16, ntt_kernel_smem_bytes(L), s>>>(src, base, base_group, base_stride, dst, tabs, mod_base, mod_count);
    });
    return cudaGetLastError();
}
cudaError_t launch_ntt_inverse(const u64 *src, u64 *dst, int n_polys, int logn, const NttTab *tabs, int mod_base, int mod_count, int fp,
                               cudaStream_t s) {
    return launch_inv(src, nullptr, 1, 0, dst, n_polys, logn, tabs, mod_base, mod_count, fp, s);
}
cudaError_t launch_ntt_inverse_add(const u64 *src, const u64 *base, int base_group, size_t base_stride, u64 *dst, int n_polys, int logn,
                                   const NttTab *tabs, int mod_base, int mod_count, int fp, cudaStream_t s) {
    return launch_inv(src, base, base_group, base_stride, dst, n_polys, logn, tabs, mod_base, mod_count, fp, s);
}

} // namespace cnhe
