// Dense scalar-MAC layer on the integer tensor cores (sm_90a, mma.sync m16n8k32 s8 x u8 -> s32).
//
// A dense layer over per-pixel ciphertexts (PoolLayer with one window covering the whole input: CryptoNets' 845 -> 100 and
// 100 -> 10 layers, NeuralNetworks/PoolLayer.cs:196-227) IS a matrix product: out[m][c] = sum_k W[m][k] * x[k][c] mod q_l, with c
// running over the 2*k*N words of a ciphertext, x the 44..50-bit residues and W the small signed integer weights.  The modular
// structure only matters at the end, so the product is done exactly over the integers on 8-bit limbs:
//     x = sum_a 2^(8a) x_a (x_a in [0,256)),  P_a[m][c] = sum_k W[m][k] x_a[k][c]  (|P_a| < 2^31 for K*127*255 < 2^31),
//     out = sum_a 2^(8a) P_a mod q_l  (Horner in FP64 with a re-centring per limb), canonical residue in [0, q_l).
// Same residues as k_mac_layer / k_mac_layer_fp (tests/test_gpu_kernels.py::test_mac_layer_*), 6 limb products instead of
// K*M 64-bit modular multiply-adds per word: the layer becomes bound by reading its inputs once.
//
// CTA: 256 threads, a tile of TN = 16 ciphertext words x up to 128 outputs (two CTAs per SM); warp w owns outputs [16w, 16w+16).  Per 32-tap chunk
// the CTA loads 32 x TN words (each loader thread 4 taps of one word), cuts them into limbs and stores them tap-major per word
// (32-byte rows with a half-row swizzle: conflict-free stores and ldmatrix); every warp then issues limbs x TN/8 MMAs against its A
// fragment (weights pre-packed in fragment order on the host, L2 resident).
#include "fparith.cuh"
#include "kernels.h"
#include "plainops.cuh"

namespace cnhe {

constexpr int IM_TN = 16;     // ciphertext words per CTA
constexpr int IM_ROW = 32;     // bytes per (word, limb) row of 32 taps; the two 16-byte halves are swapped on rows with bit 2 set, which
                               // makes both the loaders' 32-bit stores and the 8-row ldmatrix reads bank-conflict free

__device__ __forceinline__ void ldmatrix_x4(unsigned &r0, unsigned &r1, unsigned &r2, unsigned &r3, const void *smem_row) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(smem_row);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void imma_s8u8(int (&c)[4], const uint4 &a, unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}

// wfrag: [m-tile][tap chunk][lane] uint4, the m16n8k32 A fragment of the (zero padded) signed 8-bit weight matrix
template <int LIMBS>
__global__ void __launch_bounds__(256, 2) k_mac_dense_imma(const u64 *const *__restrict__ in_ptrs, const uint4 *__restrict__ wfrag,
                                                      const uint4 *__restrict__ wfrag2, const u64 *__restrict__ bias,
                                                      int K, int M, u64 *const *__restrict__ out_ptrs, int k, int logn,
                                                      const BehzConst *__restrict__ bc, PlainConst pc) {
    constexpr int TN = IM_TN, NT8 = TN / 8; // n8 tiles per warp
    __shared__ __align__(16) unsigned char sb[2][LIMBS][TN][IM_ROW];
    const int N = 1 << logn;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t col0 = (size_t)blockIdx.x * TN;            // first ciphertext word of the tile
    const int l = (int)((col0 >> logn) % k);                // its residue
    const int chunks = (K + 31) / 32;
    const int mt = blockIdx.y * 8 + warp;                   // this warp's m16 tile
    const bool have_m = mt * 16 < M;
    // loader role (threads 0 .. 8*TN-1): word n of the tile, taps 4*kq .. 4*kq+3 of the chunk
    const int ln = tid >> 3, kq = tid & 7;
    const bool loader = ln < TN;
    const int sw_off = (((kq >> 2) ^ ((ln >> 2) & 1)) << 4) + ((kq & 3) << 2); // byte offset of this thread's word inside its row
    int acc[LIMBS][NT8][4];
#pragma unroll
    for (int a = 0; a < LIMBS; a++)
#pragma unroll
        for (int j = 0; j < NT8; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) acc[a][j][e] = 0;

    u64 v[4];
    auto fetch = [&](int chunk) {
        if (!loader) return;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int kk = chunk * 32 + kq * 4 + j;
            v[j] = kk < K ? in_ptrs[kk][col0 + ln] : 0ULL;
        }
    };
    auto stage = [&](int buf) { // limb a of the four taps -> one 32-bit word (tap j in byte j)
        if (!loader) return;
#pragma unroll
        for (int a = 0; a < LIMBS; a++) {
            const unsigned b0 = (unsigned)(v[0] >> (8 * a)) & 0xffu, b1 = (unsigned)(v[1] >> (8 * a)) & 0xffu;
            const unsigned b2 = (unsigned)(v[2] >> (8 * a)) & 0xffu, b3 = (unsigned)(v[3] >> (8 * a)) & 0xffu;
            *reinterpret_cast<unsigned *>(&sb[buf][a][ln][sw_off]) = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
        }
    };

    fetch(0);
    for (int c = 0; c < chunks; c++) {
        const int buf = c & 1;
        stage(buf);
        if (c + 1 < chunks) fetch(c + 1); // in flight during this chunk's MMAs
        __syncthreads();                  // stage(buf) visible; the buffer written two chunks ago is free again after this barrier
        if (have_m) {
            const uint4 afrag = __ldg(wfrag + ((size_t)mt * chunks + c) * 32 + lane);
            // weights beyond +-127 (up to +-254) are split W = W1 + W2 on the host; W2 is almost always zero for a whole fragment
            uint4 afrag2 = make_uint4(0, 0, 0, 0);
            if (wfrag2) afrag2 = __ldg(wfrag2 + ((size_t)mt * chunks + c) * 32 + lane);
            const bool second = __any_sync(0xffffffffu, (afrag2.x | afrag2.y | afrag2.z | afrag2.w) != 0);
            const int mat = lane >> 3, r = lane & 7;
#pragma unroll
            for (int a = 0; a < LIMBS; a++) {
#pragma unroll
                for (int jp = 0; jp < NT8 / 2; jp++) { // two n8 tiles per ldmatrix.x4
                    unsigned b0, b1, b2, b3;
                    const int row = jp * 16 + (mat >> 1) * 8 + r;
                    ldmatrix_x4(b0, b1, b2, b3, &sb[buf][a][row][((mat & 1) ^ ((row >> 2) & 1)) << 4]);
                    imma_s8u8(acc[a][jp * 2], afrag, b0, b1);
                    imma_s8u8(acc[a][jp * 2 + 1], afrag, b2, b3);
                    if (second) {
                        imma_s8u8(acc[a][jp * 2], afrag2, b0, b1);
                        imma_s8u8(acc[a][jp * 2 + 1], afrag2, b2, b3);
                    }
                }
            }
        }
    }
    if (!have_m) return;
    // ---- epilogue: out = sum_a 2^(8a) P_a mod q_l, exact in FP64 for any p < 2^50: the three low limbs combine below 2^48 without
    // reduction, every higher limb is a modular product with the constant 2^(8a) mod p
    const DMod q = bc->q[l];
    const double p = (double)q.p, pinv = 1.0 / p;
    double cpow[LIMBS];
#pragma unroll
    for (int a = 3; a < LIMBS; a++) cpow[a] = frecenter((double)(1ULL << (8 * a)), p, pinv);
    const bool in_c0 = bias && col0 < (size_t)k * N;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const int m = mt * 16 + (lane >> 2) + half * 8;
        if (m >= M) continue;
        u64 *orow = out_ptrs[m];
#pragma unroll
        for (int j = 0; j < NT8; j++) {
            u64 res[2];
#pragma unroll
            for (int e = 0; e < 2; e++) {
                double rr = __fma_rn((double)acc[2][j][half * 2 + e], 65536.0, __fma_rn((double)acc[1][j][half * 2 + e], 256.0, (double)acc[0][j][half * 2 + e]));
#pragma unroll
                for (int a = 3; a < LIMBS; a++) rr = __dadd_rn(rr, fmodmul((double)acc[a][j][half * 2 + e], cpow[a], p, pinv));
                res[e] = fcanon_u(rr, p, pinv);
            }
            const size_t word = col0 + j * 8 + (lane & 3) * 2;
            if (in_c0 && (word & (size_t)(N - 1)) == 0) { // constant-plaintext bias: Delta*b on coefficient 0 of c0 (add_plain)
                const u64 b = bias[m];
                if (b) res[0] = addmod(res[0], scale_plain(b, l, q, pc), q.p);
            }
            *reinterpret_cast<ulonglong2 *>(orow + word) = make_ulonglong2(res[0], res[1]);
        }
    }
}

template <int LIMBS>
static void imma_go(const u64 *const *in_ptrs, const uint4 *wf, const uint4 *wf2, const u64 *bias, int K, int M, u64 *const *out_ptrs, int polys, int k,
                    int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    const size_t ct_words = (size_t)polys * k << logn;
    dim3 grid((unsigned)(ct_words / IM_TN), (unsigned)((M + 127) / 128));
    k_mac_dense_imma<LIMBS><<<grid, 256, 0, s>>>(in_ptrs, wf, wf2, bias, K, M, out_ptrs, k, logn, bc, pc);
}
cudaError_t launch_mac_dense_imma(const u64 *const *in_ptrs, const void *wfrag, const void *wfrag2, const u64 *bias, int K, int M, int limbs,
                                  u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s) {
    const uint4 *wf = reinterpret_cast<const uint4 *>(wfrag), *wf2 = reinterpret_cast<const uint4 *>(wfrag2);
    switch (limbs) {
    case 5: imma_go<5>(in_ptrs, wf, wf2, bias, K, M, out_ptrs, polys, k, logn, bc, pc, s); break;
    case 6: imma_go<6>(in_ptrs, wf, wf2, bias, K, M, out_ptrs, polys, k, logn, bc, pc, s); break;
    case 7: imma_go<7>(in_ptrs, wf, wf2, bias, K, M, out_ptrs, polys, k, logn, bc, pc, s); break;
    default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

} // namespace cnhe
