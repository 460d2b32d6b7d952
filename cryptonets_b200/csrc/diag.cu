// Kernels of the diagonal (Halevi-Shoup) matrix-vector product with baby-step / giant-step (DESIGN.md section 4.10).
//
// Slot layout: slot i of a plaintext sits at row a = i / (N/2), column x = i % (N/2) (the BatchEncoder's matrix); rotate_rows(s) moves
// column x + s of both rows to column x, rotate_columns swaps the rows.  Diagonal (b, s) of a matrix M holds, at slot (a, x), the weight
// M[(a, x), (a ^ b, x + s mod N/2)].  With s = n1 g + h the stored plaintext is that diagonal rotated right by n1 g, so that
//   y = sum_g rotate_rows(n1 g)( sum_{b,h} D'[g][b,h] (.) rotate_columns^b rotate_rows(h)(v) ).
#include "fparith.cuh"
#include "kernels.h"

namespace cnhe {

static inline unsigned diag_blocks(size_t threads) { return (unsigned)((threads + 255) / 256); }

// flags[b * N/2 + s] = 1 when diagonal (b, s) of the R x dim matrix has a nonzero weight.  vals [R][N]: the rows' slot values mod t.
__global__ void __launch_bounds__(256) k_diag_flags(const u64 *__restrict__ vals, int R, int dim, int logn, unsigned *__restrict__ flags) {
    const int N = 1 << logn, half = N >> 1;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)R << logn) return;
    const int r = (int)(gid >> logn), bs = (int)(gid & (N - 1)); // bs = b * N/2 + s
    const int b = bs >> (logn - 1), s = bs & (half - 1);
    const int a = r >> (logn - 1), x = r & (half - 1);
    const int col = ((a ^ b) << (logn - 1)) | ((x + s) & (half - 1));
    if (col < dim && vals[(size_t)r * N + col] != 0) flags[bs] = 1;
}

// The folded product's flags (R <= N/2): flags[d] = 1, 0 <= d < N/2, when some nonzero weight M[r, col] has col - r = d mod N/2.  Wrapped
// diagonal j of fold width W (a power of two dividing N/2), E_j[(a, x)] = M[x mod W, a N/2 + (x + j mod N/2)], is nonzero exactly when
// flags[d] is set for some d = j mod W, so this one pass serves every width the planner weighs.
__global__ void __launch_bounds__(256) k_diag_flags_folded(const u64 *__restrict__ vals, int R, int dim, int logn, unsigned *__restrict__ flags) {
    const int N = 1 << logn, half = N >> 1;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)R << logn) return;
    const int r = (int)(gid >> logn), col = (int)(gid & (N - 1));
    if (col < dim && vals[gid] != 0) flags[(col - r) & (half - 1)] = 1;
}

// out[j][(a, x)] = M[(a, x - n1 g_j mod N/2), (a ^ b_j, x + h_j mod N/2)] (0 outside R x dim): the pre-rotated diagonal j, in slot order.
// desc[j] = (b_j, n1 g_j, h_j).  fold = W > 0 (the folded product, b_j = 0): the row is (x - n1 g_j) mod W instead, so that out[j] is
// wrapped diagonal n1 g_j + h_j rotated right by n1 g_j.
__global__ void __launch_bounds__(256) k_diag_gather(const u64 *__restrict__ vals, int R, int dim, const int3 *__restrict__ desc, int nd, int logn,
                                                     int fold, u64 *__restrict__ out) {
    const int N = 1 << logn, half = N >> 1;
    const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (size_t)nd << logn) return;
    const int j = (int)(gid >> logn), i = (int)(gid & (N - 1));
    const int3 d = desc[j];
    const int a = i >> (logn - 1), x = i & (half - 1);
    const int r = fold ? (x - d.y) & (fold - 1) : (a << (logn - 1)) | ((x - d.y) & (half - 1));
    const int col = ((a ^ d.x) << (logn - 1)) | ((x + d.z) & (half - 1));
    out[gid] = r < R && col < dim ? vals[(size_t)r * N + col] : 0;
}

// acc[g][b][p][l][i] = sum_{j in [g_start[g], g_start[g+1])} dhat[j][l][i] * xhat[xsel[j]][b][p][l][i]  (mod q_l, canonical out)
// dhat: the wave's lifted diagonals in NTT form [nd][k][N]; xhat: the baby-step ciphertexts in NTT form [2 n1][B][2][k][N], canonical.
// One thread per (g, l, i) keeps CB clients' two accumulators in registers, so a diagonal word is loaded once for CB clients and both
// polynomials (B > CB: once per CB clients).  The CTAs of one (l, coefficient tile) are consecutive over g: the giant steps of a wave read
// the same baby-step words at about the same time, and those reads are served by L2.  Arithmetic: fmodmul products of canonical operands
// a, w < q < 2^49, |r| <= q/2 + a w 2^-52 < 0.625 q (the rounding of h pinv moves r past q/2), summed with dadd and re-centred after
// every 8th term and at the end.  A re-centred carry (<= q/2 + 1) and 8 products stay below 5.5 q < 2^52, inside the 2^53 range of exact
// double sums; without the in-loop re-centre 33 coherent products of about q/2 pass 2^53 (tests/fp64_accumulators.py models the sum).
template <int CB>
__global__ void __launch_bounds__(256) k_diag_mac(const u64 *__restrict__ dhat, const u64 *__restrict__ xhat, const int *__restrict__ g_start,
                                                  const int *__restrict__ xsel, u64 *__restrict__ acc, int ng, int B, int logn,
                                                  const __grid_constant__ BehzConstF F) {
    const int N = 1 << logn, k = F.k, tiles = N >> 8;
    const int g = blockIdx.x % ng, tile = (blockIdx.x / ng) % tiles, l = blockIdx.x / (ng * tiles);
    const int i = (tile << 8) + threadIdx.x;
    const double p = F.qd[l], pinv = F.qinv[l];
    const size_t kN = (size_t)k * N, ct = 2 * kN;
    const int j0 = g_start[g], j1 = g_start[g + 1];
    for (int b0 = 0; b0 < B; b0 += CB) {
        double a[CB][2];
#pragma unroll
        for (int cb = 0; cb < CB; cb++) a[cb][0] = a[cb][1] = 0.0;
        for (int j = j0; j < j1; j++) {
            const double d = u2d(dhat[(size_t)j * kN + (size_t)l * N + i]);
            const u64 *xs = xhat + ((size_t)xsel[j] * B + b0) * ct + (size_t)l * N + i;
#pragma unroll
            for (int cb = 0; cb < CB; cb++) {
                if (b0 + cb < B) {
                    a[cb][0] = __dadd_rn(a[cb][0], fmodmul(u2d(xs[cb * ct]), d, p, pinv));
                    a[cb][1] = __dadd_rn(a[cb][1], fmodmul(u2d(xs[cb * ct + kN]), d, p, pinv));
                }
            }
            if (((j - j0) & 7) == 7) { // a carry and 8 fresh products stay below 5.5 q; re-centre before they could leave the exact range
#pragma unroll
                for (int cb = 0; cb < CB; cb++) {
                    a[cb][0] = frecenter(a[cb][0], p, pinv);
                    a[cb][1] = frecenter(a[cb][1], p, pinv);
                }
            }
        }
#pragma unroll
        for (int cb = 0; cb < CB; cb++) {
            if (b0 + cb >= B) break;
            u64 *o = acc + ((size_t)g * B + b0 + cb) * ct + (size_t)l * N + i;
            o[0] = fsmall_u(frecenter(a[cb][0], p, pinv), F.q_u[l]);
            o[kN] = fsmall_u(frecenter(a[cb][1], p, pinv), F.q_u[l]);
        }
    }
}

// One term of k_diag_mac_resident: CB clients' two polynomials at a coefficient pair, x loaded as 16-byte words.
template <int CB>
__device__ __forceinline__ void diag_mac_pair(double (&a)[CB][2][2], const u64 *xs, size_t ct, size_t kN, int nb, double d0, double d1, double p,
                                              double pinv) {
#pragma unroll
    for (int cb = 0; cb < CB; cb++) {
        if (cb < nb) {
            const ulonglong2 x0 = __ldg(reinterpret_cast<const ulonglong2 *>(xs + cb * ct));
            const ulonglong2 x1 = __ldg(reinterpret_cast<const ulonglong2 *>(xs + cb * ct + kN));
            a[cb][0][0] = __dadd_rn(a[cb][0][0], fmodmul(u2d(x0.x), d0, p, pinv));
            a[cb][0][1] = __dadd_rn(a[cb][0][1], fmodmul(u2d(x0.y), d1, p, pinv));
            a[cb][1][0] = __dadd_rn(a[cb][1][0], fmodmul(u2d(x1.x), d0, p, pinv));
            a[cb][1][1] = __dadd_rn(a[cb][1][1], fmodmul(u2d(x1.y), d1, p, pinv));
        }
    }
}

// k_diag_mac over diagonals held resident in NTT form (cnhe_diag_prepare_ntt): nothing produced them just before, so every diagonal word
// streams from HBM, and the kernel is built for that.  One thread per (g, l, coefficient pair): 16-byte loads of the diagonal and of the
// baby-step words.  A full re-centring period (8 diagonals) is straight-line code in chunks of D = 2 diagonals: a chunk's two diagonal
// loads (evict-first, so that they do not push the baby-step words the giant steps share out of L2) and baby-step indices are issued
// before its first product, so they are in flight together with the baby-step loads the compiler hoists (4 and 8 took more registers
// and were no faster, DESIGN.md 4.10).  CTA order as in k_diag_mac (g fastest, then the 512-coefficient tile, then l).  Per
// (g, client, l, i) the arithmetic is k_diag_mac's in the same order: fmodmul of canonical operands, dadd, re-centred after every 8th term
// and at the end (below 5.5 q < 2^52 in between, as there), fsmall_u -- so the outputs are bit-identical.
template <int CB>
__global__ void __launch_bounds__(256) k_diag_mac_resident(const u64 *__restrict__ dhat, const u64 *__restrict__ xhat, const int *__restrict__ g_start,
                                                           const int *__restrict__ xsel, u64 *__restrict__ acc, int ng, int B, int logn,
                                                           const __grid_constant__ BehzConstF F) {
    constexpr int D = 2;
    const int N = 1 << logn, k = F.k, tiles = N >> 9;
    const int g = blockIdx.x % ng, tile = (blockIdx.x / ng) % tiles, l = blockIdx.x / (ng * tiles);
    const int i = (tile << 9) + 2 * threadIdx.x;
    const double p = F.qd[l], pinv = F.qinv[l];
    const size_t kN = (size_t)k * N, ct = 2 * kN;
    const int j0 = g_start[g], j1 = g_start[g + 1];
    const u64 *dl = dhat + (size_t)l * N + i;
    for (int b0 = 0; b0 < B; b0 += CB) {
        const int nb = B - b0;
        const u64 *xl = xhat + (size_t)b0 * ct + (size_t)l * N + i;
        double a[CB][2][2]; // [client][polynomial][coefficient of the pair]
#pragma unroll
        for (int cb = 0; cb < CB; cb++) a[cb][0][0] = a[cb][0][1] = a[cb][1][0] = a[cb][1][1] = 0.0;
        int jb = j0;
        for (; jb + 8 <= j1; jb += 8) {
#pragma unroll
            for (int c0 = 0; c0 < 8; c0 += D) {
                ulonglong2 dv[D];
                int xv[D];
#pragma unroll
                for (int u = 0; u < D; u++) {
                    dv[u] = __ldcs(reinterpret_cast<const ulonglong2 *>(dl + (size_t)(jb + c0 + u) * kN));
                    xv[u] = __ldg(xsel + jb + c0 + u);
                }
#pragma unroll
                for (int u = 0; u < D; u++)
                    diag_mac_pair<CB>(a, xl + (size_t)xv[u] * B * ct, ct, kN, nb, u2d(dv[u].x), u2d(dv[u].y), p, pinv);
            }
#pragma unroll
            for (int cb = 0; cb < CB; cb++) // k_diag_mac's re-centring after every 8th term
#pragma unroll
                for (int e = 0; e < 4; e++) a[cb][e >> 1][e & 1] = frecenter(a[cb][e >> 1][e & 1], p, pinv);
        }
        for (int j = jb; j < j1; j++) { // the group's last, partial period
            const ulonglong2 d = __ldcs(reinterpret_cast<const ulonglong2 *>(dl + (size_t)j * kN));
            diag_mac_pair<CB>(a, xl + (size_t)xsel[j] * B * ct, ct, kN, nb, u2d(d.x), u2d(d.y), p, pinv);
        }
#pragma unroll
        for (int cb = 0; cb < CB; cb++) {
            if (cb >= nb) break;
            u64 *o = acc + ((size_t)g * B + b0 + cb) * ct + (size_t)l * N + i;
            const u64 q = F.q_u[l];
            *reinterpret_cast<ulonglong2 *>(o) =
                make_ulonglong2(fsmall_u(frecenter(a[cb][0][0], p, pinv), q), fsmall_u(frecenter(a[cb][0][1], p, pinv), q));
            *reinterpret_cast<ulonglong2 *>(o + kN) =
                make_ulonglong2(fsmall_u(frecenter(a[cb][1][0], p, pinv), q), fsmall_u(frecenter(a[cb][1][1], p, pinv), q));
        }
    }
}

cudaError_t launch_diag_flags(const u64 *vals, int R, int dim, int logn, unsigned *flags, cudaStream_t s) {
    if (R <= 0) return cudaSuccess;
    k_diag_flags<<<diag_blocks((size_t)R << logn), 256, 0, s>>>(vals, R, dim, logn, flags);
    return cudaGetLastError();
}
cudaError_t launch_diag_flags_folded(const u64 *vals, int R, int dim, int logn, unsigned *flags, cudaStream_t s) {
    if (R <= 0) return cudaSuccess;
    k_diag_flags_folded<<<diag_blocks((size_t)R << logn), 256, 0, s>>>(vals, R, dim, logn, flags);
    return cudaGetLastError();
}
cudaError_t launch_diag_gather(const u64 *vals, int R, int dim, const int *desc, int nd, int logn, int fold, u64 *out, cudaStream_t s) {
    if (nd <= 0) return cudaSuccess;
    k_diag_gather<<<diag_blocks((size_t)nd << logn), 256, 0, s>>>(vals, R, dim, reinterpret_cast<const int3 *>(desc), nd, logn, fold, out);
    return cudaGetLastError();
}
cudaError_t launch_diag_mac(const u64 *dhat, const u64 *xhat, const int *g_start, const int *xsel, u64 *acc, int ng, int B, int k, int logn,
                            const BehzConstF *f, cudaStream_t s) {
    if (ng <= 0 || B <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)ng * (unsigned)((1 << logn) >> 8) * (unsigned)k;
    if (B == 1) k_diag_mac<1><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else if (B == 2) k_diag_mac<2><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else if (B <= 4) k_diag_mac<4><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else k_diag_mac<8><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    return cudaGetLastError();
}
cudaError_t launch_diag_mac_resident(const u64 *dhat, const u64 *xhat, const int *g_start, const int *xsel, u64 *acc, int ng, int B, int k,
                                     int logn, const BehzConstF *f, cudaStream_t s) {
    if (ng <= 0 || B <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)ng * (unsigned)((1 << logn) >> 9) * (unsigned)k;
    if (B == 1) k_diag_mac_resident<1><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else if (B == 2) k_diag_mac_resident<2><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else if (B <= 4) k_diag_mac_resident<4><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    else k_diag_mac_resident<8><<<grid, 256, 0, s>>>(dhat, xhat, g_start, xsel, acc, ng, B, logn, *f);
    return cudaGetLastError();
}

} // namespace cnhe
