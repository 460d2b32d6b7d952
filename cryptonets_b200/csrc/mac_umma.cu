// Scalar-MAC layers (dense and convolution) on the Hopper tensor cores: wgmma.mma_async s8 x u8 -> s32, operands in shared memory,
// accumulators in registers.
//
// Same arithmetic as mac_imma.cu (the layer IS a matrix product over 8-bit limbs of the ciphertext words:
//     x = sum_a 2^(8a) x_a,  P_a[m][c] = sum_k W[m][k] x_a[k][c],  out = sum_a 2^(8a) P_a mod q_l,
// NeuralNetworks/PoolLayer.cs:196-227), generalised from "one window covers the whole input" to BUNDLES: a bundle is a set of at most
// 128 outputs whose taps lie in a window of consecutive inputs (a dense layer is one bundle; a strided convolution is one bundle per
// output row, and all interior rows share one weight matrix because the window slides with them).  What the mma.sync kernel is limited
// by -- every warp loads and shuffles its own operands, so loads, address arithmetic and accumulators all compete for registers -- is
// moved off the consumers:
//   * the ciphertext words arrive by TMA into a six-stage ring, two cp.async.bulk.tensor requests per stage (a 2-D map over the
//     slab the layer's inputs sit in: 32 taps x 16 words each, SWIZZLE_128B), issued by one producer warp that only waits on
//     mbarriers.  The few taps whose weights exceed a signed byte (W = W1 + W2) are gathered into a scratch slab by the host call and
//     appear a second time, as extra chunks with W2 as their weights, through a second map;
//   * the weights of the whole layer stay resident in shared memory from the start of the CTA (A operand, packed by the host in
//     core-matrix order: 8-row x 16-byte core matrices, K-major, no swizzle);
//   * the 256 consumer threads (two warpgroups) turn a raw stage into the B operand -- limb a of word n is row a*32 + n of a K-major
//     unswizzled tile -- with three byte permutes per limb and conflict-free 32-bit stores, then each warpgroup issues one
//     m64n32k32 wgmma per limb for its 64 output rows.  The wgmma runs asynchronously under the cutting of the next stage;
//   * the epilogue reads the accumulators straight from registers: a thread holds 8 words of 2 output rows for every limb, so the
//     limbs combine without any exchange;
//   * persistent CTAs (one per SM) walk the 32-word tiles of the ciphertext, and inside a tile the bundles of the layer.
// Warp roles: 0-7 consumers (warpgroup 0 = output rows 0-63 of a bundle, warpgroup 1 = rows 64-127), 8 TMA producer.
// Output words are bit-identical to k_mac_dense_imma / k_mac_layer_fp and to the oracle (tests/test_gpu_kernels.py:
// test_dense_layer_on_tensor_cores, test_convolution_on_tensor_cores, test_tensor_core_layers_randomised).
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cuda.h> // CUtensorMap
#include "fparith.cuh"
#include "kernels.h"
#include "plainops.cuh"

namespace cnhe {
namespace {

constexpr int UM_TN = 32;                            // ciphertext words per tile
constexpr int UM_M = 128;                            // MMA rows (outputs, zero padded): two warpgroups of 64
constexpr int UM_CHUNK = 32;                         // taps per MMA (K of the 8-bit wgmma)
constexpr int UM_RAW_STAGES = 6, UM_B_STAGES = 4;
constexpr int UM_RAW_BYTES = UM_CHUNK * UM_TN * 8;   // 8192: two halves of 32 taps x 16 words (128-byte rows, hardware swizzle)
constexpr int UM_A_CHUNK = UM_M * UM_CHUNK;          // 4096 bytes of weights per chunk
constexpr int UM_CONSUMERS = 256;                    // warps 0-7
constexpr int UM_THREADS = UM_CONSUMERS + 32;        // + warp 8, the producer

__device__ __forceinline__ unsigned sptr(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sptr(bar)), "r"(count));
}
__device__ __forceinline__ void mb_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sptr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(sptr(bar)) : "memory");
}
// bounded wait: a protocol error traps (the launch fails with an error) instead of hanging the GPU.  The try_wait carries a suspend-time
// hint, so a waiting warp sleeps in hardware instead of spinning and taking issue slots from the working warps of its scheduler
__device__ __forceinline__ void mb_wait(unsigned long long *bar, unsigned parity) {
    const unsigned a = sptr(bar);
    unsigned done = 0;
    for (unsigned spin = 0; !done; spin++) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(a), "r"(parity), "r"(20000u)
                     : "memory");
        if (!done && spin > (1u << 22)) __trap();
    }
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(sptr(dst)), "l"(src), "r"(bytes),
                 "r"(sptr(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_g2s_2d(void *dst, const void *tmap, int c0, int c1, unsigned long long *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(sptr(dst)), "l"(tmap),
                 "r"(c0), "r"(c1), "r"(sptr(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(UM_CONSUMERS) : "memory"); }
// K-major operand without swizzle: 8-row x 16-byte core matrices; lbo = distance between the two 16-byte K halves, sbo = distance
// between 8-row groups (bytes); layout type 0 (no swizzle) in bits 62-63
__device__ __forceinline__ u64 wgmma_desc(unsigned saddr, unsigned lbo, unsigned sbo) {
    return (u64)((saddr & 0x3FFFFu) >> 4) | ((u64)(lbo >> 4) << 16) | ((u64)(sbo >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads or writes across an asynchronous wgmma
__device__ __forceinline__ void acc_fence(int (&d)[16]) {
#pragma unroll
    for (int i = 0; i < 16; i++) asm volatile("" : "+r"(d[i])::"memory");
}
// D[64 x 32] (+)= A[64 x 32 signed bytes] * B[32 x 32 unsigned bytes]^T; fragment: d[i] is row 16 * warp + lane / 4 + 8 * ((i >> 1) & 1),
// column 8 * (i >> 2) + 2 * (lane & 3) + (i & 1)
__device__ __forceinline__ void wgmma_i8(int (&d)[16], u64 adesc, u64 bdesc, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.u8 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
                   "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate)
                 : "memory");
}
// exact double of a signed integer |x| < 2^51: one integer add, one FP64 add (inverse of d2i)
__device__ __forceinline__ double i2d(long long x) { return __dsub_rn(__longlong_as_double(x + 0x4338000000000000LL), FP_MAGIC); }
__device__ __forceinline__ void stg128(u64 *p, u64 a, u64 b) { asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory"); }

struct UmSmem { // offsets into the dynamic shared memory block (bytes), after the 1024-byte alignment pad
    int w, raw, b, dst, bun, rows, mod, bars, total;
};
constexpr int UM_MAX_RES = 9; // coefficient moduli (KMAX)
__host__ __device__ inline UmSmem um_layout(int a_bytes, int total_chunks, int n_out_total, int n_bundles, int limbs) {
    UmSmem s;
    s.w = 0;                                                // weight matrices (A operands), 4096 bytes per chunk
    s.raw = s.w + a_bytes;                                  // raw ring (1024-byte aligned: swizzle atoms)
    s.b = s.raw + UM_RAW_STAGES * UM_RAW_BYTES;             // B-operand ring
    s.dst = s.b + UM_B_STAGES * limbs * UM_TN * UM_CHUNK;   // destination pointer of every output, in bundle order
    s.bun = s.dst + ((n_out_total * 8 + 15) & ~15);         // bundle records
    s.rows = s.bun + ((n_bundles * (int)sizeof(UmBundle) + 15) & ~15); // first tap row of every chunk (bit 30: scratch slab)
    s.mod = s.rows + ((total_chunks * 4 + 15) & ~15);       // per residue: p, 1/p, 2^(8a) mod p as doubles
    s.bars = s.mod + UM_MAX_RES * 8 * 8;
    s.total = s.bars + 256 + 1024;                          // + alignment slack
    return s;
}

// wpack: per chunk 4096 bytes, weight (row r, tap kb of the chunk) at (r >> 3) * 256 + (kb >> 4) * 128 + (r & 7) * 16 + (kb & 15)
// DIG (digit mode, size-3 inputs, DESIGN 4.15): the tiles of c0 and c1 as above into 2kN-word outputs, then every tile of c2 once per
// group of LIMBS / 2 key-switch digits.  A digit tile cuts each word at the digit boundaries instead of the byte boundaries, two limbs
// per digit (bits [i w, i w + 8) and [i w + 8, (i + 1) w)), and its epilogue writes S = P_lo + 256 P_hi, the exact integer digit sum,
// into the output's int32 plane of that digit (|S| < 2^31 is host-checked).  Same ring, same MMAs, same weights.
template <int LIMBS, bool DIG>
__global__ void __launch_bounds__(UM_THREADS, 1)
k_mac_umma(const __grid_constant__ CUtensorMap tmap0, const __grid_constant__ CUtensorMap tmap1, const UmBundle *__restrict__ bundles, int n_bundles,
           const int *__restrict__ chunk_rows, int total_chunks, const unsigned char *__restrict__ wpack, int a_bytes,
           u64 *const *__restrict__ out_ptrs, const u64 *__restrict__ bias, int n_out_total, int polys, int k, int logn,
           const BehzConst *__restrict__ bc, PlainConst pc, const __grid_constant__ UmDigits dg, unsigned long long *prof) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((1024u - (sptr(smem_raw) & 1023u)) & 1023u);
    // CNHE_UMMA_PROF=1: CTA 0 reports, per role, the cycles spent in each of its waits and in its work (prof[role * 4 + i])
    const bool profiling = prof != nullptr && blockIdx.x == 0;
    long long t_a = 0, t_b = 0, t_c = 0, t0 = 0;
#define UM_T0() if (profiling) t0 = clock64()
#define UM_ACC(x) if (profiling) { const long long t1_ = clock64(); x += t1_ - t0; t0 = t1_; }
    constexpr int B_BYTES = LIMBS * UM_TN * UM_CHUNK;
    const UmSmem L = um_layout(a_bytes, total_chunks, n_out_total, n_bundles, LIMBS);
    unsigned char *sw = smem + L.w, *sraw = smem + L.raw, *sb = smem + L.b;
    u64 **sdst = reinterpret_cast<u64 **>(smem + L.dst);
    UmBundle *sbun = reinterpret_cast<UmBundle *>(smem + L.bun);
    int *srows = reinterpret_cast<int *>(smem + L.rows);
    double *smod = reinterpret_cast<double *>(smem + L.mod);
    unsigned long long *bars = reinterpret_cast<unsigned long long *>(smem + L.bars);
    unsigned long long *raw_full = bars, *raw_empty = raw_full + UM_RAW_STAGES, *w_full = raw_empty + UM_RAW_STAGES;
    static_assert((2 * UM_RAW_STAGES + 1) * 8 <= 256, "barrier block");
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int N = 1 << logn;
    // DIG: main tiles over c0 and c1, then dg.groups passes over the kN / 32 tiles of c2
    const int n_main = (int)(((size_t)(DIG ? 2 : polys) * k << logn) / UM_TN), c2_tiles = (int)(((size_t)k << logn) / UM_TN);
    const int n_tiles = DIG ? n_main + dg.groups * c2_tiles : n_main;

    if (tid == 0) {
        for (int i = 0; i < UM_RAW_STAGES; i++) { mb_init(raw_full + i, 1); mb_init(raw_empty + i, UM_CONSUMERS); }
        mb_init(w_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // tables and modulus constants: fetched once, so that no role touches global memory for them again
    for (int i = tid; i < n_out_total; i += UM_THREADS) sdst[i] = out_ptrs[i];
    for (int i = tid; i < n_bundles; i += UM_THREADS) sbun[i] = bundles[i];
    for (int i = tid; i < total_chunks; i += UM_THREADS) srows[i] = chunk_rows[i];
    if (tid < k) {
        const double p = (double)bc->q[tid].p, pinv = 1.0 / p;
        smod[tid * 8] = p;
        smod[tid * 8 + 1] = pinv;
        for (int a = 3; a < 8; a++) smod[tid * 8 + a - 1] = frecenter((double)(1ULL << (8 * a)), p, pinv); // slots 2..6 = a 3..7
    }
    __syncthreads();

    if (warp == UM_CONSUMERS / 32) {
        // ---- producer (one thread): the weight matrices once, then two tensor-map requests per stage
        if (lane == 0) {
            mb_expect_tx(w_full, (unsigned)a_bytes);
            for (int o = 0; o < a_bytes; o += UM_A_CHUNK) bulk_g2s(sw + o, wpack + o, UM_A_CHUNK, w_full);
            unsigned it = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int col0 = (!DIG || tile < n_main) ? tile * UM_TN : (2 * c2_tiles + (tile - n_main) % c2_tiles) * UM_TN;
                for (int b = 0; b < n_bundles; b++) {
                    const UmBundle bn = sbun[b];
                    for (int c = 0; c < bn.n_chunks; c++, it++) {
                        const unsigned s = it % UM_RAW_STAGES, ph = (it / UM_RAW_STAGES) & 1;
                        UM_T0();
                        mb_wait(raw_empty + s, ph ^ 1); // a fresh barrier passes the wait for the "previous" phase
                        UM_ACC(t_a);
                        mb_expect_tx(raw_full + s, UM_RAW_BYTES);
                        const int e = srows[bn.chunk0 + c];
                        const void *map = (e >> 30) ? (const void *)&tmap1 : (const void *)&tmap0;
                        const int row = e & 0x3fffffff;
                        tma_g2s_2d(sraw + s * UM_RAW_BYTES, map, col0, row, raw_full + s);
                        tma_g2s_2d(sraw + s * UM_RAW_BYTES + UM_RAW_BYTES / 2, map, col0 + 16, row, raw_full + s);
                        UM_ACC(t_b);
                    }
                }
            }
            if (profiling) { prof[0] = t_a; prof[1] = t_b; }
        }
        return;
    }

    // ---- consumers.  Cutting: thread (q = tap quad 0..7, n = word 0..31) packs limb a of taps 4q..4q+3 into one 32-bit store at B row
    // a*32+n, bytes 4q..4q+3.  Lane = (q & 3) + 4 * (n & 7): the 32 stores of a warp fill one 8-row core matrix half (512 contiguous
    // bytes, conflict free); the 64-bit loads touch 8 consecutive words of 4 tap rows 4 apart, which the hardware swizzle (16-byte chunk
    // index XOR row & 7) spreads over both halves of the banks.
    const int wg = warp >> 2;
    const int n = (warp & 3) * 8 + (lane >> 2), qh = warp >> 2, q = qh * 4 + (lane & 3);
    const int half_off = (n >> 4) * (UM_RAW_BYTES / 2), j16 = (n & 15) >> 1, sub = (n & 1) * 8;
    // accumulator fragment of this thread: output rows r0 and r0 + 8 of the bundle, words 8j + 2 (lane & 3) + {0, 1} of the tile
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
    int acc[LIMBS][16];
    mb_wait(w_full, 0);
    unsigned it = 0;
    long long t_d = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const bool dig = DIG && tile >= n_main;
        const int dgrp = dig ? (tile - n_main) / c2_tiles : 0; // digit tile: its group, and the coefficients it covers in its residue
        const size_t col0 = dig ? (size_t)(2 * c2_tiles + (tile - n_main) % c2_tiles) * UM_TN : (size_t)tile * UM_TN;
        const int l = (int)((col0 >> logn) % k);
        const double p = smod[l * 8], pinv = smod[l * 8 + 1];
        const double c24 = smod[l * 8 + 2], c48 = smod[l * 8 + 5]; // 2^24, 2^48 mod p
        const bool bias_tile = bias && col0 < (size_t)k * N && (col0 & (size_t)(N - 1)) == 0; // coefficient 0 of a c0 polynomial
        for (int b = 0; b < n_bundles; b++) {
            const UmBundle bn = sbun[b];
            const bool active = wg * 64 < bn.n_out; // a warpgroup whose 64 rows are all padding issues no MMA (uniform per warpgroup)
            for (int c = 0; c < bn.n_chunks; c++, it++) {
                const unsigned rs = it % UM_RAW_STAGES, rph = (it / UM_RAW_STAGES) & 1;
                // B stage it % 4 was last read by the MMAs of chunk it - 4: every consumer has waited for those of chunk it - 3 (the
                // wait_group below, at chunk it - 2) before the barrier of chunk it - 1, which this thread has passed
                unsigned char *bst = sb + (it % UM_B_STAGES) * B_BYTES;
                UM_T0();
                mb_wait(raw_full + rs, rph);
                UM_ACC(t_a);
                const unsigned char *raw = sraw + rs * UM_RAW_BYTES + half_off + sub;
                unsigned lo[4], hi[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int r = 4 * q + j;
                    const uint2 t = *reinterpret_cast<const uint2 *>(raw + r * 128 + ((j16 ^ (r & 7)) << 4));
                    lo[j] = t.x;
                    hi[j] = t.y;
                }
                mb_arrive(raw_empty + rs);
                if (DIG && dig) { // limb a: half a & 1 of digit dgrp * LIMBS / 2 + a / 2 of the four words (0 past the residue's digits)
                    const int nd = dg.count[l];
#pragma unroll
                    for (int a = 0; a < LIMBS; a++) {
                        const int i = dgrp * (LIMBS / 2) + (a >> 1);
                        unsigned w = 0;
                        if (a < 2 * (LIMBS / 2) && i < nd) {
                            const int sh = i * dg.w + 8 * (a & 1);
                            const unsigned m = (a & 1) ? (dg.mask >> 8) : (dg.mask & 0xFFu);
#pragma unroll
                            for (int j = 0; j < 4; j++) w |= ((unsigned)((((u64)hi[j] << 32) | lo[j]) >> sh) & m) << (8 * j);
                        }
                        const int row = a * UM_TN + n;
                        *reinterpret_cast<unsigned *>(bst + (row >> 3) * 256 + qh * 128 + (row & 7) * 16 + (lane & 3) * 4) = w;
                    }
                } else {
#pragma unroll
                for (int a = 0; a < LIMBS; a++) { // byte a of the four words -> one 32-bit word, three byte permutes
                    const unsigned sel = (a & 3) | (((a & 3) + 4) << 4);
                    const unsigned t01 = __byte_perm(a < 4 ? lo[0] : hi[0], a < 4 ? lo[1] : hi[1], sel);
                    const unsigned t23 = __byte_perm(a < 4 ? lo[2] : hi[2], a < 4 ? lo[3] : hi[3], sel);
                    const unsigned w = __byte_perm(t01, t23, 0x5410);
                    const int row = a * UM_TN + n;
                    *reinterpret_cast<unsigned *>(bst + (row >> 3) * 256 + qh * 128 + (row & 7) * 16 + (lane & 3) * 4) = w;
                }
                }
                fence_async_smem(); // generic-proxy stores -> visible to the tensor core's (async proxy) reads
                consumers_sync();
                UM_ACC(t_b);
                if (active) {
#pragma unroll
                    for (int a = 0; a < LIMBS; a++) acc_fence(acc[a]);
                    wgmma_fence();
                    const u64 adesc = wgmma_desc(sptr(sw + bn.a_off + c * UM_A_CHUNK + wg * (UM_A_CHUNK / 2)), 128, 256);
#pragma unroll
                    for (int a = 0; a < LIMBS; a++) wgmma_i8(acc[a], adesc, wgmma_desc(sptr(bst + a * (UM_TN * UM_CHUNK)), 128, 256), c > 0);
                    wgmma_commit();
#pragma unroll
                    for (int a = 0; a < LIMBS; a++) acc_fence(acc[a]);
                }
                wgmma_wait<1>();
                UM_ACC(t_c);
            }
            // ---- epilogue: out = sum_a 2^(8a) P_a mod q_l, exact in FP64 for p < 2^50: the three low limbs combine below 2^48 without
            // reduction, every higher limb is a modular product with 2^(8a) mod p
            wgmma_wait<0>();
#pragma unroll
            for (int a = 0; a < LIMBS; a++) acc_fence(acc[a]);
            if (DIG && dig) {
                if (active && (warp & 3) * 16 + wg * 64 < bn.n_out) {
                    const int nd = dg.count[l], nc = (int)(col0 & (size_t)(N - 1)) + c0;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        const int m = r0 + 8 * h;
                        if (m >= bn.n_out) continue;
                        int *prow = dg.planes[bn.out0 + m] + nc;
#pragma unroll
                        for (int ii = 0; ii < LIMBS / 2; ii++) {
                            const int i = dgrp * (LIMBS / 2) + ii;
                            if (i >= nd) continue;
                            int *o = prow + (size_t)(dg.first[l] + i) * N;
#pragma unroll
                            for (int j = 0; j < 4; j++) {
                                const int e0 = 4 * j + 2 * h;
                                const int v0 = acc[2 * ii][e0] + (int)((unsigned)acc[2 * ii + 1][e0] << 8);
                                const int v1 = acc[2 * ii][e0 + 1] + (int)((unsigned)acc[2 * ii + 1][e0 + 1] << 8);
                                asm volatile("st.global.v2.b32 [%0], {%1,%2};" ::"l"(o + 8 * j), "r"(v0), "r"(v1) : "memory");
                            }
                        }
                    }
                }
                UM_ACC(t_d);
                continue;
            }
            if (active && (warp & 3) * 16 + wg * 64 < bn.n_out) { // warps whose 16 rows are all padding skip the arithmetic (uniform per warp)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const int m = r0 + 8 * h;
                    if (m >= bn.n_out) continue;
                    u64 *orow = sdst[bn.out0 + m] + col0;
                    u64 res[8];
#pragma unroll
                    for (int j = 0; j < 4; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const int i = 4 * j + 2 * h + e;
                            // limbs 0..2 and 3..5 combine exactly on the integer pipe (each sum below 2^48); one modular product joins them
                            const long long lo = (long long)acc[0][i] + ((long long)acc[1][i] << 8) + ((long long)acc[2][i] << 16);
                            long long hi = (long long)acc[3][i] + ((long long)acc[4][i] << 8);
                            if constexpr (LIMBS >= 6) hi += (long long)acc[5][i] << 16;
                            double rr = __dadd_rn(i2d(lo), fmodmul(i2d(hi), c24, p, pinv));
                            if constexpr (LIMBS == 7) rr = __dadd_rn(rr, fmodmul((double)acc[6][i], c48, p, pinv));
                            res[2 * j + e] = fcanon_u(rr, p, pinv);
                        }
                    if (bias_tile && c0 == 0) { // constant-plaintext bias: Delta*b on coefficient 0 of c0 (add_plain)
                        const u64 bv = bias[bn.out0 + m];
                        const DMod qm = bc->q[l];
                        if (bv) res[0] = addmod(res[0], scale_plain(bv, l, qm, pc), qm.p);
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) stg128(orow + 8 * j + c0, res[2 * j], res[2 * j + 1]);
                }
            }
            UM_ACC(t_d);
        }
    }
    if (profiling && tid == 0) { prof[8] = t_a; prof[9] = t_b; prof[10] = t_c; prof[12] = t_d; }
#undef UM_T0
#undef UM_ACC
}

int sm_count_cached() {
    static int n = [] {
        int dev = 0, v = 132;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
        return v;
    }();
    return n;
}

template <int LIMBS, bool DIG>
cudaError_t umma_go(const CUtensorMap &map0, const CUtensorMap &map1, const UmmaLaunch &a, cudaStream_t s) {
    const UmSmem L = um_layout(a.a_bytes, a.total_chunks, a.n_out_total, a.n_bundles, LIMBS);
    cudaError_t e = cudaFuncSetAttribute(k_mac_umma<LIMBS, DIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total);
    if (e != cudaSuccess) return e;
    const int n_tiles = (int)((((size_t)(DIG ? 2 + a.dig.groups : a.polys)) * a.k << a.logn) / UM_TN);
    const int grid = std::min(sm_count_cached(), n_tiles);
    const bool want_prof = getenv("CNHE_UMMA_PROF") != nullptr; // read per launch: tests switch it on to see which kernel served a layer
    unsigned long long *prof = nullptr;
    if (want_prof) {
        static unsigned long long *buf = nullptr;
        if (!buf) cudaMalloc((void **)&buf, 16 * sizeof(unsigned long long));
        cudaMemsetAsync(buf, 0, 16 * sizeof(unsigned long long), s);
        prof = buf;
    }
    k_mac_umma<LIMBS, DIG><<<grid, UM_THREADS, L.total, s>>>(map0, map1, a.bundles, a.n_bundles, a.chunk_rows, a.total_chunks, a.wpack, a.a_bytes,
                                                             a.out_ptrs, a.bias, a.n_out_total, a.polys, a.k, a.logn, a.bc, a.pc, a.dig, prof);
    if (want_prof) {
        unsigned long long h[16];
        cudaMemcpyAsync(h, prof, sizeof(h), cudaMemcpyDeviceToHost, s);
        cudaStreamSynchronize(s);
        fprintf(stderr, "[umma%s bundles=%d chunks/tile=%d outputs=%d weights=%d KB tiles/cta=%.1f] producer: wait_empty %llu issue %llu | "
                        "consumers: wait_raw %llu cut %llu mma %llu epilogue %llu (cycles, CTA 0)\n",
                DIG ? " digits" : "", a.n_bundles, a.total_chunks, a.n_out_total, a.a_bytes / 1024, (double)n_tiles / grid, h[0], h[1], h[8], h[9], h[10], h[12]);
    }
    return cudaGetLastError();
}

} // namespace

// shared memory the plan needs against what an SM has
bool mac_umma_fits(int a_bytes, int total_chunks, int n_out_total, int n_bundles, int limbs) {
    if (limbs < 5 || limbs > 7 || n_bundles < 1 || a_bytes < UM_A_CHUNK) return false;
    return um_layout(a_bytes, total_chunks, n_out_total, n_bundles, limbs).total <= 227 * 1024;
}
// host-side packing of one bundle's signed 8-bit weight matrix (w[r * cols + c], cols a multiple of 32) into the A-operand order
void mac_umma_pack(const signed char *w, int rows, int cols, unsigned char *out) {
    const int chunks = cols / UM_CHUNK;
    memset(out, 0, (size_t)chunks * UM_A_CHUNK);
    for (int r = 0; r < rows; r++)
        for (int kk = 0; kk < cols; kk++) {
            const int c = kk / UM_CHUNK, kb = kk % UM_CHUNK;
            out[(size_t)c * UM_A_CHUNK + (r >> 3) * 256 + (kb >> 4) * 128 + (r & 7) * 16 + (kb & 15)] = (unsigned char)w[(size_t)r * cols + kk];
        }
}
cudaError_t launch_mac_umma(const UmmaLaunch &a, cudaStream_t s) {
    alignas(64) CUtensorMap map0, map1;
    const size_t ctw = (size_t)a.polys * a.k << a.logn; // words per input: the maps' width and the scratch slab's row stride
    cudaError_t e = make_word_map_2d(&map0, a.slab, ctw, a.slab_rows, a.slab_stride_words * 8, UM_TN / 2, UM_CHUNK, 1);
    if (e != cudaSuccess) return e;
    if (a.scratch_rows > 0) {
        e = make_word_map_2d(&map1, a.scratch, ctw, a.scratch_rows, ctw * 8, UM_TN / 2, UM_CHUNK, 1);
        if (e != cudaSuccess) return e;
    } else
        map1 = map0;
    if (a.dig.planes) {
        if (a.polys != 3) return cudaErrorInvalidValue;
        switch (a.limbs) {
        case 5: return umma_go<5, true>(map0, map1, a, s);
        case 6: return umma_go<6, true>(map0, map1, a, s);
        case 7: return umma_go<7, true>(map0, map1, a, s);
        default: return cudaErrorInvalidValue;
        }
    }
    switch (a.limbs) {
    case 5: return umma_go<5, false>(map0, map1, a, s);
    case 6: return umma_go<6, false>(map0, map1, a, s);
    case 7: return umma_go<7, false>(map0, map1, a, s);
    default: return cudaErrorInvalidValue;
    }
}

} // namespace cnhe
