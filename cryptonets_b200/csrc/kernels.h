// Kernel launch interface between the host runtime (context.cu / vec.cu / api.cu) and the CUDA kernels.
// Every launcher is asynchronous on the given stream and returns the cudaError_t of the launch.
#pragma once
#include "modarith.cuh"

namespace cnhe {

// NTT tables of one modulus in HBM (N words each); the kernels index an array of these by modulus id:
//   0..k-1 coefficient primes q_i, k..k+kb-1 the BEHZ base Bsk (aux primes then m_sk), k+kb.. plain moduli.
struct NttTab {
    const u64 *w, *ws;   // psi^bitrev(i) and floor(w 2^64 / p)        (forward, Cooley-Tukey order)
    const u64 *iw, *iws; // psi^-bitrev(i) and its Shoup quotient       (inverse, Gentleman-Sande order)
    u64 inv_n, inv_n_s;  // N^-1 mod p and its Shoup quotient
    DMod mod;
    // FP64 butterfly path (p < 2^50): the same twiddles as exact doubles, centred in (-p/2, p/2]
    const double *wd, *iwd;
    // N = 4096 / 8192: the 15N/16 inverse twiddles of the four unit-stride stages, transposed for the persistent inverse transform:
    // iwd_hi[m * N/16 + j] is the m-th twiddle (m = 0..14: 8 + 4 + 2 + 1 per stage) of the 16-coefficient group j in the first pass
    const double *iwd_hi;
    double pd, pinv, inv_n_d;
    double inv_n_w_d;                   // iw[1] * N^-1 mod p, centred: the last inverse stage carries the N^-1 scaling
    int fp_ok;                          // 1 when the FP64 path is exact for this modulus and N
    unsigned fwd_recenter, inv_recenter; // forward: bit i = re-centre at the start of pass i; inverse: bit v = re-centre the sums of stage v
    // Split form (ntt.cu, N = 4096 / 8192 / 16384): after the first stage the two halves of an N-point transform are independent
    // N/2-point transforms -- the CTA-pair transforms of N = 16384, the fused key switch and the fused square run them.  wd_split /
    // iwd_split hold the two halves' twiddle tables ([half][N/2], indexed like wd / iwd of an N/2-point transform), fwd_recenter_split
    // is the forward schedule of the passes 1+(logN-9) | 4 | 4, split_ok = 1 when that schedule is exact, split_out_rc is fwd_out_rc
    // for the fused kernels' output (N = 16384 has no other schedule: fwd_out_rc there covers the split one)
    unsigned fwd_recenter_split;
    const double *wd_split;
    int split_ok, split_out_rc;
    const double *iwd_split;
    // N = 4096 / 8192: the same halves' twiddles of the four unit-stride stages regrouped per thread for the fused kernels (ntt.cu,
    // fwd_last_stages_grp / inv_first_stages_grp): thread j's 15 twiddles, padded to 16, as double2 groups [half][group 0..7][thread j
    // of N/32], so a warp's load of one group is 512 contiguous bytes.  Forward (the last four stages of a half): group 0 = the first of
    // them's twiddle and a pad word, 1 = the second's two, 2..3 the third's four, 4..7 the fourth's eight.  Inverse (stages 0..3):
    // groups 0..3 stage 0, 4..5 stage 1, 6 stage 2, 7 = stage 3's twiddle and a pad word.  Built for the q and Bsk moduli only
    const double *wd_split_grp, *iwd_split_grp;
    int fwd_out_rc;                    // lazy forward output must be re-centred (its bound squared would overflow the consumer's product)
    double fwd_out_bound;               // |forward lazy output| <= fwd_out_bound * p
};

// Base-2^w digit decomposition used by relinearisation / Galois key switching: digit d comes from residue
// src[d] of the target polynomial, bits [shift[d], shift[d]+w).
struct DigitMap {
    unsigned char src[64];
    unsigned char shift[64];
    int D;
    u64 mask;
};

// Key references (DESIGN 4.16).  A key switch recorded into a graph is given, in place of each key base, the address of a device word
// that holds the base: the graph's key binding, which the host rewrites between launches so that one recording reads any client's keys.
// With REF, a launcher's key, key_packed and key_tab entries are such addresses; the kernel loads the base through them once.
template <bool REF, class T>
__device__ __forceinline__ const T *key_base(const T *p) {
    if constexpr (REF) return *reinterpret_cast<const T *const *>(p);
    else return p;
}

// `fp` argument of the NTT launchers
enum NttFormat { NTT_FP = 1, NTT_IN_F = 2, NTT_OUT_F = 4 };
enum NttLoad { NTT_LOAD_PLAIN = 0, NTT_LOAD_DIGIT = 1 };
enum NttStore { NTT_STORE_PLAIN = 0, NTT_STORE_ADD = 1 };

// In-place / out-of-place batched negacyclic NTT.  Polynomial b (0 <= b < n_polys) uses modulus
// mod_base + (b % mod_count).  src == dst allowed.
// fp: 1 = every modulus of the range has fp_ok (FP64 butterflies), 0 = integer Harvey butterflies (any p < 2^62)
cudaError_t launch_ntt_forward(const u64 *src, u64 *dst, int n_polys, int logn, const NttTab *tabs, int mod_base, int mod_count, int fp,
                               cudaStream_t s);
cudaError_t launch_ntt_inverse(const u64 *src, u64 *dst, int n_polys, int logn, const NttTab *tabs, int mod_base, int mod_count, int fp,
                               cudaStream_t s);
// dst[((c*k + l)*D + d)] = NTT_l( digit d of target[c] )   target: [n_ct][k][N] coefficient form
// ciphertext c's k-residue target polynomial starts at target + c * ct_stride (words); fp: 0, or NTT_FP | NTT_OUT_F (lazy doubles out)
cudaError_t launch_ntt_forward_digits(const u64 *target, size_t ct_stride, u64 *dst, int n_ct, int k, const DigitMap &dm, int logn,
                                      const NttTab *tabs, int fp, cudaStream_t s);
// Fused key switch (N = 4096 / 8192, FP64 path): out[c][p][l] = base_c[p][l] + INTT_l(sum_d NTT_l(digit d of target[c]) * key[d][p][l])
// (mod q_l, canonical), key [D][2][k][N] canonical NTT form, base polynomial p of ciphertext c at base + c * base_stride + p * k * N, out
// packed [n_ct][2][k][N] -- what launch_ntt_forward_digits, launch_ks_mac_fp and launch_ntt_inverse_add compute, with no digit
// buffer and no accumulator.  out must overlap neither the target nor the base words: other CTAs still read them while one writes.
// key_packed: nullptr, or the copy of `key` made by launch_pack_keys48 (every q_l < 2^48), which the kernel then reads instead.
// key_tab: nullptr, or a device table of n_ct key bases (ciphertext c reads key_tab[c] in place of key, or of key_packed when that is set)
// ref: key, key_packed and the key_tab entries are key references (key_base above), not bases
cudaError_t launch_key_switch_fused(const u64 *target, size_t ct_stride, const u64 *key, const uint4 *key_packed, const u64 *const *key_tab,
                                    const u64 *base, size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm, int logn,
                                    const NttTab *tabs, cudaStream_t s, bool ref = false);
// The fused key switch with its digits read from int32 planes: digit d of ciphertext c is planes[(c * D + d) * N + i], |value| < min q_l
// (the digit sums of a scalar-MAC layer over unrelinearised products, DESIGN 4.15); keys, base, out, key_tab and ref as above
cudaError_t launch_key_switch_planes(const int *planes, const u64 *key, const uint4 *key_packed, const u64 *const *key_tab, const u64 *base,
                                     size_t base_stride, u64 *out, int n_ct, int k, const DigitMap &dm, int logn, const NttTab *tabs, cudaStream_t s,
                                     bool ref = false);
// the fused key switch's packed key copy: n_polys canonical N-word polynomials (words < 2^48) -> 6N bytes each, thread-interleaved (ntt.cu)
cudaError_t launch_pack_keys48(const u64 *key, uint4 *out, int n_polys, int logn, cudaStream_t s);
// dst[b] = INTT(src[b]) + base[(b / base_group) * base_stride + (b % base_group) * N]  (mod p)
cudaError_t launch_ntt_inverse_add(const u64 *src, const u64 *base, int base_group, size_t base_stride, u64 *dst, int n_polys, int logn,
                                   const NttTab *tabs, int mod_base, int mod_count, int fp, cudaStream_t s);
// pass structure shared by host (re-centring masks) and device: radix (log2) of each pass, forward and inverse
int ntt_pass_radices(int logn, int inverse, int *radices /*4*/);
int ntt_kernel_smem_bytes(int logn);

} // namespace cnhe

// ---------------------------------------------------------------------------------------------------------------
namespace cnhe {

constexpr int KMAX = 9;   // up to 9 coefficient primes (N = 16384 default table)
constexpr int KBMAX = 12; // up to 12 primes in the BEHZ base Bsk (auxiliary primes + m_sk)

// Everything the BEHZ kernels need that depends only on (q, Bsk, m~): SEAL 3.2 util::BaseConverter::generate.
struct BehzConst {
    int k, kb, centered_mtilde, pad_; // k coefficient primes; kb primes in Bsk = (kb-1) auxiliary primes then m_sk
    DMod q[KMAX], bsk[KBMAX];
    u64 inv_qhat_mod_q[KMAX];        // (q/q_i)^-1 mod q_i
    u64 mtilde_inv_qhat_mod_q[KMAX]; // m~ (q/q_i)^-1 mod q_i
    u64 qhat_mod_mtilde[KMAX];       // (q/q_i) mod 2^32
    u64 inv_q_mod_mtilde;            // q^-1 mod 2^32
    u64 qhat_mod_bsk[KBMAX][KMAX];
    u64 q_mod_bsk[KBMAX], inv_q_mod_bsk[KBMAX], inv_mtilde_mod_bsk[KBMAX];
    u64 inv_bhat_mod_b[KBMAX];       // (B/b_j)^-1 mod b_j
    u64 bhat_mod_q[KMAX][KBMAX];     // (B/b_j) mod q_i
    u64 bhat_mod_msk[KBMAX];
    u64 inv_B_mod_msk, B_mod_q[KMAX];
};
// The same constants as exact doubles, centred in (-p/2, p/2], for the FP64 kernels (behz_fp.cu); valid when every
// coefficient and Bsk prime is below 2^50.
struct BehzConstF {
    int k, kb, centered_mtilde, pad_;
    double qd[KMAX], qinv[KMAX], bd[KBMAX], binv[KBMAX];
    double inv_qhat_mod_q[KMAX], mtilde_inv_qhat_mod_q[KMAX];
    u64 qhat_mod_mtilde[KMAX], inv_q_mod_mtilde;
    double qhat_mod_bsk[KBMAX][KMAX];
    double q_mod_bsk[KBMAX], inv_q_mod_bsk[KBMAX], inv_mtilde_mod_bsk[KBMAX];
    double inv_bhat_mod_b[KBMAX], bhat_mod_q[KMAX][KBMAX], bhat_mod_msk[KBMAX];
    double inv_B_mod_msk, msk_half, B_mod_q[KMAX];
    u64 q_u[KMAX]; // the coefficient moduli as integers (sign fix-up of canonical outputs on the integer pipe)
};
// Constants of the folded fast_floor / fastbconv_sk kernel (k_behz_floor_fold_fp), per plaintext modulus: every product by a constant
// that SEAL applies in sequence (x t, x q-hat_i^-1, x q^-1, x B-hat_j^-1) is merged into the next conversion matrix on the host --
// the same residues (modular arithmetic is exact), 19 % fewer FP64 instructions.
struct FloorConstF {
    int k, kb, pad0_, pad1_;
    double qd[KMAX], qinv[KMAX], bd[KBMAX], binv[KBMAX];
    double xq[KMAX];              // t * (q/q_i)^-1 mod q_i
    double xb[KBMAX];             // j < kb-1: t * q^-1 * B-hat_j^-1 mod p_j;  j = kb-1 (m_sk): t * q^-1 mod m_sk
    double conv[KBMAX][KMAX];     // (q/q_i) * q^-1 (* B-hat_j^-1 for j < kb-1) mod p_j
    double bhat_mod_q[KMAX][KBMAX], bhat_mod_msk[KBMAX];
    double inv_B_mod_msk, msk_half, B_mod_q[KMAX];
};
// Epilogue of the BEHZ floor kernels (the quadratic activation A ct^2 + B x + C, cnhe_layer_poly2): every output polynomial times A,
// B x added to c0 and c1, Delta C added to c0, mod q_l and canonical -- the words of multiply_plain(A) on the size-3 product, then (after
// the key switch, which is linear) multiply_plain(x, B) and add_plain(C).  x[c]: the ciphertext whose B multiple output c of the launch
// gets ([2][k][N], canonical coefficient form; a device pointer table) -- the squared operand itself, or (the second level of
// cnhe_layer_poly's quartic and cubic) the activation's original input.  Per residue: A and B lifted into q_l with the upper-half increment, Delta C
// scaled as add_plain scales it; the *_d copies centred as exact doubles for the FP64 kernels.  C is the constant polynomial (every slot)
// unless c_poly (nullptr, or a device table of one entry per ciphertext of the launch) gives the ciphertext a plaintext of its own:
// c_poly[c] = nullptr, or [k][N] canonical words Delta m (+ q mod t where m is in the upper half) of a plaintext m, added to c0 in
// place of Delta C at coefficient 0 (a dense vector's last, partly filled block: C in its data slots only)
struct FloorEpi {
    const u64 *const *x;
    const u64 *const *c_poly;
    u64 a[KMAX], b[KMAX], c[KMAX];
    double a_d[KMAX], b_d[KMAX], c_d[KMAX];
};
// Per plaintext modulus t.
struct PlainConst {
    u64 t, threshold;                 // (t+1)/2
    u64 delta[KMAX], q_mod_t[KMAX];   // floor(q/t) mod q_i, (q mod t) mod q_i
    // decryption (Decryptor::decrypt, gamma base)
    DMod tmod, gmod;
    u64 tgamma_mod_q[KMAX], qhat_mod_t[KMAX], qhat_mod_gamma[KMAX];
    u64 neg_inv_q_mod_t, neg_inv_q_mod_gamma, inv_gamma_mod_t, gamma;
};

// ---- elementwise over ciphertext words (words = n * size * k * N; residue of word w is (w / N) % k)
cudaError_t launch_ct_add(const u64 *a, const u64 *b, u64 *out, size_t words, int k, int logn, const BehzConst *bc, int sub, cudaStream_t s);
cudaError_t launch_ct_negate(const u64 *a, u64 *out, size_t words, int k, int logn, const BehzConst *bc, cudaStream_t s);
// out[c] = a[c] + epi.x[c] + Delta C on c0 (FloorEpi's constant term; A and B unused): n size-2 ciphertexts
cudaError_t launch_ct_add_epi(const u64 *a, u64 *out, int n, int k, int logn, const BehzConst *bc, const FloorEpi &epi, cudaStream_t s);
// out = sum_j in_ptrs[j]  (AddMany)
cudaError_t launch_ct_add_many(const u64 *const *in_ptrs, int n_in, u64 *out, size_t words, int k, int logn, const BehzConst *bc, cudaStream_t s);
// ct (size polys) (+/-)= Delta*plain on c0; plain has `coeffs` coefficients mod t.  n cts, plain shared (plain_stride 0) or per ct.
cudaError_t launch_ct_add_plain(const u64 *ct, u64 *out, int n, int size, const u64 *plain, size_t plain_stride, int coeffs, int k,
                                int logn, const BehzConst *bc, PlainConst pc, int sub, cudaStream_t s);
// out[n] = in[n] * scalar (constant plaintext, lifted per residue)      (multiply_plain monomial path, exponent 0)
cudaError_t launch_ct_scale(const u64 *in, u64 *out, int n, int size, const u64 *scalars /*n values mod t, device*/, int k, int logn,
                            const BehzConst *bc, PlainConst pc, cudaStream_t s);
// lifted[l][x] = plain[x] (+ q_l - t if in the upper half)   (multiply_plain generic path)
cudaError_t launch_plain_lift(const u64 *plain, u64 *lifted, int n, int coeffs, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s);
// out[c][part][l][x] = a[c or 0][part][l][x] * b[c or 0][l][x]
cudaError_t launch_dyadic_bcast(const u64 *a, const u64 *b, u64 *out, int n, int size, int a_per_ct, int b_per_ct, int k, int logn,
                                const BehzConst *bc, cudaStream_t s);
// out[b * out_rows + r][p][l][x] = ct[b][p][l][x] * pl[r][l][x]: B ciphertexts [B][2][k][N] times R lifted plaintexts [R][k][N], NTT form,
// canonical in and out (FP64 path: every q_l < 2^50; the same words as launch_dyadic_bcast)
cudaError_t launch_dyadic_outer(const u64 *ct, const u64 *pl, u64 *out, int B, int R, int out_rows, int k, int logn, const BehzConstF *f,
                                cudaStream_t s);
// Galois: out[c] = (perm(c0), 0), perm1[c] = perm(c1)   (util::apply_galois)
cudaError_t launch_galois(const u64 *in, u64 *out_base, u64 *perm_c1, int n, u64 elt_inv, int k, int logn, const BehzConst *bc, cudaStream_t s,
                          int add_back = 0); // add_back: base = (c0 + perm(c0), c1) -> key switch + base = x + rotate(x)
// the same with the n input ciphertexts given by a device pointer table
cudaError_t launch_galois_gather(const u64 *const *in_ptrs, u64 *out_base, u64 *perm_c1, int n, u64 elt_inv, int k, int logn, const BehzConst *bc,
                                 cudaStream_t s);

// ---- modulus switch (BFV mod_switch_to_next, applied k - k_out times): out [n][2][k_out][N] from in[c] [2][k][N], coefficient form,
// canonical words.  Dropping prime j maps every residue i < j to (x_i - (r mod q_i) + (floor(q_j / 2) mod q_i)) q_j^-1 mod q_i with
// r = (x_j + floor(q_j / 2)) mod q_j: round(x / q_j) on the representative x of [0, q).  Any order of widths, q_l < 2^61.
struct ModSwitchConst {
    int k, k_out;
    DMod q[KMAX];
    u64 half[KMAX];               // floor(q_j / 2)
    u64 half_mod[KMAX][KMAX];     // [j][i]: floor(q_j / 2) mod q_i
    u64 inv[KMAX][KMAX], inv_s[KMAX][KMAX]; // [j][i]: q_j^-1 mod q_i and its Shoup quotient
};
cudaError_t launch_mod_switch(const u64 *const *in, u64 *out, int n, int logn, const ModSwitchConst &M, cudaStream_t s);

// ---- K4: out[m] = sum_k w[m][k] * in[gather[m][k]] (+ Delta*bias[m] on coefficient 0 of c0)
// polys: polynomials per ciphertext, 2, or 3 for size-3 products (the sum is linear in each polynomial); every MAC launcher takes it
struct MacTile {
    int n_out;       // outputs in this tile (<= 8) sharing one gather row
    int gather_row;  // row index into gather[] (K entries)
    int out_index[8];
};
// w_ptrs[m]: K weights mod t (device); bias[m] mod t or null
cudaError_t launch_mac_layer(const u64 *const *in_ptrs, const int *gather, const MacTile *tiles, int n_tiles, const u64 *const *w_ptrs,
                             const u64 *bias, int K, u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc,
                             cudaStream_t s);

// small-weight variant: wd[m*K + kk] = signed weight as an exact double (|w| < 2^17 and K*|w|*2^26 < 2^52, host-checked)
cudaError_t launch_mac_layer_fp(const u64 *const *in_ptrs, const int *gather, const MacTile *tiles, int n_tiles, const double *wd, const u64 *bias,
                                int K, u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s);

// ---- K5: BEHZ multiply pieces
// in: ct pointers (each [2][k][N]); out together layout [n][2][k+kb][N] (q residues copied, then Bsk residues)
cudaError_t launch_behz_lift(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConst *bc, cudaStream_t s);
// d[n][3][2k+1][N] from NTT-form a,b [n][2][2k+1][N]
cudaError_t launch_behz_tensor(const u64 *a, const u64 *b, u64 *d, int n, int kt, int logn, const BehzConst *bc, cudaStream_t s);
// d (coefficient form) -> times t, fast_floor, fastbconv_sk -> out3[n][3][k][N]
// epi (host copy, every floor launcher): nullptr, or the FloorEpi applied to the outputs (its x table lists the launch's n ciphertexts)
// pair (every floor launcher; needs epi): d holds 2n products [2n][3][kt][N], and output c is floor(product 2c) - floor(product 2c + 1)
// mod q_l before the epilogue (the cubic activation's level 2, cnhe_layer_poly)
cudaError_t launch_behz_floor(const u64 *d, u64 *out3, int n, u64 t, int logn, const BehzConst *bc, cudaStream_t s, const FloorEpi *epi = nullptr,
                              bool pair = false);
// FP64 (behz_fp.cu): the buffers exchanged with the NTT kernels (lift output, tensor input/output, digit input, accumulator output) hold
// lazy doubles (fparith.cuh) -- pair with NTT_IN_F / NTT_OUT_F on the transforms in between
cudaError_t launch_behz_lift_fp(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConstF *f, cudaStream_t s);
// lazy Bsk residues only, out [n][2][kb][N]: the source of the fused square's residues l >= k
cudaError_t launch_behz_lift_bsk_fp(const u64 *const *ct_ptrs, u64 *out, int n, int logn, const BehzConstF *f, cudaStream_t s);
// Fused square (N = 4096 / 8192, ntt.cu): d [n][3][kt][N] lazy doubles, coefficient form, from ciphertexts ct_ptrs[c] ([2][k][N]) and
// their lifted Bsk residues lift_bsk ([n][2][kb][N], launch_behz_lift_bsk_fp) -- what forward transforms, the square tensor and inverse
// transforms compute on the output of launch_behz_lift_fp; needs split_ok on all kt moduli
cudaError_t launch_behz_square_fused(const u64 *const *ct_ptrs, const u64 *lift_bsk, u64 *d, int n_ct, int k, int kt, int logn, const NttTab *tabs,
                                     cudaStream_t s);
cudaError_t launch_behz_tensor_fp(const u64 *a, const u64 *b, u64 *d, int n, int kt, int logn, const BehzConstF *f, cudaStream_t s);
// sums of T tensor products per output: d[o] = sum_j a[o T + j] (x) b[j], a [n_out T][2][kt][N] and b [T][2][kt][N] in NTT form, d
// [n_out][3][kt][N] as launch_behz_tensor writes one product (integer: canonical words; FP64: lazy doubles in and out)
cudaError_t launch_behz_tensor_mac_fp(const u64 *a, const u64 *b, u64 *d, int n_out, int T, int kt, int logn, const BehzConstF *f, cudaStream_t s);
cudaError_t launch_behz_tensor_mac(const u64 *a, const u64 *b, u64 *d, int n_out, int T, int kt, int logn, const BehzConst *bc, cudaStream_t s);
// the floor of launch_behz_floor on lazy input, with folded constants
cudaError_t launch_behz_floor_fold_fp(const u64 *d, u64 *out3, int n, int logn, const FloorConstF *f, cudaStream_t s, const FloorEpi *epi = nullptr,
                                     bool pair = false);
cudaError_t launch_ks_mac_fp(const u64 *digits, const u64 *key, const u64 *const *key_tab, u64 *acc, int n, int D, int k, int logn,
                             const BehzConstF *f, cudaStream_t s, bool ref = false);
// ---- K6: key-switch inner product. digits [n][D][k][N] (NTT), key [D][2][k][N] (NTT) -> acc [n][2][k][N] (NTT)
// key_tab: nullptr, or a device table of n key bases (ciphertext c reads key_tab[c] in place of key); ref: key and the key_tab entries
// are key references (key_base), as for the fused key switch
cudaError_t launch_ks_mac(const u64 *digits, const u64 *key, const u64 *const *key_tab, u64 *acc, int n, int D, int k, int logn, const BehzConst *bc,
                          cudaStream_t s, bool ref = false);
// split a size-3 array [n][3][k][N] view: base[n][2][k][N] = (c0,c1), c2[n][k][N]

// ---- diagonal matrix-vector product (diag.cu; slot layout and indices there)
// flags[b * N/2 + s] = 1 where diagonal (b, s) of the R x dim matrix whose rows' slot values are vals [R][N] has a nonzero weight
// (flags is not cleared)
cudaError_t launch_diag_flags(const u64 *vals, int R, int dim, int logn, unsigned *flags, cudaStream_t s);
// folded product (R <= N/2): flags[d] = 1, d < N/2, where a nonzero weight M[r, col] has col - r = d mod N/2 (flags is not cleared)
cudaError_t launch_diag_flags_folded(const u64 *vals, int R, int dim, int logn, unsigned *flags, cudaStream_t s);
// out[j] (slot values [nd][N]) = diagonal (b, n1 g + h) rotated right by n1 g, desc[j] = (b, n1 g, h) as three ints (device); fold = W > 0:
// wrapped diagonal n1 g + h of fold width W (b = 0) rotated right by n1 g
cudaError_t launch_diag_gather(const u64 *vals, int R, int dim, const int *desc, int nd, int logn, int fold, u64 *out, cudaStream_t s);
// acc[g][b][p][l] = sum_{j = g_start[g]}^{g_start[g+1]-1} dhat[j][l] * xhat[xsel[j]][b][p][l]  (NTT form, canonical in and out; FP64 path)
cudaError_t launch_diag_mac(const u64 *dhat, const u64 *xhat, const int *g_start, const int *xsel, u64 *acc, int ng, int B, int k, int logn,
                            const BehzConstF *f, cudaStream_t s);
// the same sums, bit-identical, over diagonals held resident in NTT form (streamed from HBM: 16-byte loads, two diagonals' loads issued
// together)
cudaError_t launch_diag_mac_resident(const u64 *dhat, const u64 *xhat, const int *g_start, const int *xsel, u64 *acc, int ng, int B, int k,
                                     int logn, const BehzConstF *f, cudaStream_t s);

// ---- sampling / encode / encrypt / decrypt
enum SampleKind { SAMPLE_TERNARY = 0, SAMPLE_NOISE = 1, SAMPLE_UNIFORM = 2 };
// out[i][l][x] for i<n: stream ids stream0 + i*stream_step (+ l for UNIFORM); lifted into each residue
// Dense layer (every output reads the same K inputs) on the integer tensor cores: wfrag = signed 8-bit weights packed as m16n8k32
// A fragments [ceil(M/16)][ceil(K/32)][32 lanes][16 bytes]; weights in [-254, 254] are split W = W1 + W2 (wfrag2, may be null);
// limbs = ceil(bits(q)/8); needs K*254*255 < 2^31 and every coefficient prime below 2^50 (the limb sums are joined modulo q_l in FP64:
// (double)p must be exact and fcanon_u's input below 2^51; wider moduli belong to the 128-bit launch_mac_layer)
cudaError_t launch_mac_dense_imma(const u64 *const *in_ptrs, const void *wfrag, const void *wfrag2, const u64 *bias, int K, int M, int limbs,
                                  u64 *const *out_ptrs, int polys, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s);
// Scalar-MAC layers on wgmma (mac_umma.cu).  The layer's inputs are rows of one slab (input i at slab + i * slab_stride_words); a
// BUNDLE is up to 128 outputs whose taps lie in a window of consecutive inputs: chunk j of the bundle multiplies the 32 inputs that start
// at row chunk_rows[chunk0 + j] (bit 30 set: a row of the scratch slab that holds the W2 taps) with the 128 x 32 weight block at
// wpack + a_off + j * 4096.  Outputs and constant biases are listed in bundle order (out0 = first entry of the bundle).  The epilogue
// joins the limb sums in FP64, exact only when every coefficient prime is below 2^50, as for launch_mac_dense_imma.
struct UmBundle {
    int chunk0, n_chunks, a_off, n_out, out0;
};
// Digit mode of the wgmma MAC (size-3 inputs): the c2 digit sums of every output into int32 planes [D][N] instead of a reduced c2
struct UmDigits {
    int *const *planes;          // device, bundle order: each output's planes; null = no digit mode
    int w, groups;               // digit width; digit groups of limbs / 2 digits per residue
    unsigned mask;               // 2^w - 1
    unsigned char first[KMAX], count[KMAX]; // per residue: its first digit and its number of digits (DigitMap order)
};
struct UmmaLaunch {
    const u64 *slab;            // input 0
    size_t slab_stride_words;   // distance between consecutive inputs
    size_t slab_rows;           // number of inputs
    const u64 *scratch;         // W2 taps gathered side by side (polys * k * N words apart), or null
    size_t scratch_rows;
    const UmBundle *bundles;    // device
    int n_bundles;
    const int *chunk_rows;      // device
    int total_chunks;           // chunks per tile (sum over the bundles)
    const unsigned char *wpack; // device: a_bytes of weight blocks (identical matrices stored once)
    int a_bytes;
    u64 *const *out_ptrs;       // device, bundle order
    const u64 *bias;            // device, bundle order; null = no constant bias
    int n_out_total;
    int limbs, polys, k, logn;  // polys: 2, or 3 for size-3 inputs (slab_stride_words >= 3kN)
    const BehzConst *bc;
    PlainConst pc;
    UmDigits dig;               // digit mode (polys == 3): outputs get c0 and c1 only (2kN words), c2 goes to the digit planes
};
bool mac_umma_fits(int a_bytes, int total_chunks, int n_out_total, int n_bundles, int limbs);
void mac_umma_pack(const signed char *w, int rows, int cols, unsigned char *out); // cols a multiple of 32; out: cols / 32 * 4096 bytes
cudaError_t launch_mac_umma(const UmmaLaunch &a, cudaStream_t s);
// 2-D tensor map over 64-bit words (ntt.cu): rows of inner_words words, row_stride bytes apart; swizzle128: rows of the box are 128 bytes
cudaError_t make_word_map_2d(void *map, const u64 *base, size_t inner_words, size_t rows, size_t row_stride, unsigned box_words, unsigned box_rows,
                             int swizzle128);
cudaError_t launch_sample(u64 *out, int n, int kind, const RngKey &seed, u64 stream0, u64 stream_step, int k, int logn, const BehzConst *bc, cudaStream_t s);
// plain[i][index_map[j]] = values[i][j]  (j < count), zero elsewhere
cudaError_t launch_encode_scatter(const u64 *values, u64 *plain, int n, int count, const u32 *index_map, int logn, cudaStream_t s);
// plain[i][index_map[first_col + i]] = 1, zero elsewhere (one-hot slot masks, encoded form before the inverse transform)
cudaError_t launch_onehot_scatter(u64 *plain, int n, int first_col, const u32 *index_map, int logn, cudaStream_t s);
cudaError_t launch_decode_gather(const u64 *plain_ntt, u64 *values, int n, const u32 *index_map, int logn, cudaStream_t s);
// ---- values in and out of the channels (values.cu, DESIGN 4.19)
// dense (index_map set): plain[c][index_map[j]] = the residue mod t of value (c % bl) N + j of vector c / bl of values [n][dim] (zero past
// dim), c < n_ct; sparse (index_map null): plain[j] = the residue of values[j], j < dim.  Residue: w = rint(v scale), |w| mod big, made
// big - |w| mod big when w < 0.  A value with !(|w| < 1.5e38) sets *bad and writes 0.
cudaError_t launch_split_scatter(const double *values, u64 *plain, int n_ct, int bl, u64 dim, double scale, unsigned __int128 big, u64 t,
                                 const u32 *index_map, int logn, int *bad, cudaStream_t s);
// c0[i], c1[i] ([kN] each) = the two parts of ciphertext ct_tab[i] ([2][kN])
cudaError_t launch_split_parts(const u64 *const *ct_tab, u64 *c0, u64 *c1, int n, size_t kN, cudaStream_t s);
// where the join finds one vector's residues of one channel: value j at p[j stride] for j < count, zero past it; scale: the vector's
// (read from the channel-0 entries)
struct JoinSrc {
    const u64 *p;
    u64 stride, count;
    double scale;
};
struct JoinConst {
    int P;
    u64 big_lo, big_hi;                 // B, the product of the plaintext moduli (< 2^126)
    u64 coeff_lo[16], coeff_hi[16];     // the CRT coefficients mod B
};
// out[i][j] = centred sum over the channels of coeff_ch r_ch mod B, as a double rounded to nearest even, over the vector's scale;
// src [P][n]
cudaError_t launch_crt_join(const JoinSrc *src, double *out, int n, u64 dim, const JoinConst &jc, cudaStream_t s);
// ct[i] (already u*pk, coefficient form) += (e0 + Delta*m_i, e1)
cudaError_t launch_encrypt_finish(u64 *ct, const u64 *plain, size_t plain_stride, int n, int coeffs, const RngKey &seed, u64 nonce0, int k, int logn,
                                  const BehzConst *bc, PlainConst pc, cudaStream_t s);
// secret-key variant: ct[i] part 0 = -as[i] + e + Delta*m_i, part 1 (a) untouched; as [n][k][N] = a*s in coefficient form
cudaError_t launch_encrypt_finish_sk(u64 *ct, const u64 *as, const u64 *plain, size_t plain_stride, int n, int coeffs, const RngKey &seed, u64 nonce0,
                                     int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s);

// ---- sanitisation (circuit privacy, DESIGN 4.18).  Ciphertext i of a call draws under nonce v = *base + i (base: the word the
// one-thread take kernel wrote) on the streams stream_id(purpose, v mod 2^32, v >> 32) of these purposes: u, e0, e1 and the flood f
constexpr u64 PURPOSE_SAN_U = 16, PURPOSE_SAN_E0 = 17, PURPOSE_SAN_E1 = 18, PURPOSE_SAN_F = 19;
constexpr u64 SANITIZE_NONCES = 1ULL << 48; // nonces per channel key: 32 bits in the stream id's middle field, 16 in its low field
__host__ __device__ __forceinline__ u64 sanitize_stream(u64 purpose, u64 nonce) { return stream_id(purpose, nonce & 0xffffffffULL, nonce >> 32); }
// the flood f of one coefficient: words w_j = rng64(stream(PURPOSE_SAN_F), x W + j), j < W = ceil((b + 1) / 64), read as one
// little-endian integer F of b + 1 bits (the top word masked); f = F - 2^b
struct SanitizeConst {
    int k, words;        // W
    u64 top_mask;        // mask of word W - 1
    DMod q[KMAX];
    u64 pow2b[KMAX];     // 2^b mod q_l
};
// *base = *counter, *counter += n (one thread)
cudaError_t launch_sanitize_take(u64 *counter, u64 n, u64 *base, cudaStream_t s);
// u[i][l][x] = ternary of ciphertext i, lifted into every q_l, i < n
cudaError_t launch_sanitize_u(u64 *u, int n, const u64 *base, const RngKey &rk, int k, int logn, const BehzConst *bc, cudaStream_t s);
// out[i][p][l] = pk_tab[i][p][l] * u[i][l] (NTT form); ref: the pk_tab entries are key references (key_base)
cudaError_t launch_sanitize_upk(const u64 *const *pk_tab, const u64 *u, u64 *out, int n, int k, int logn, const BehzConst *bc, bool ref,
                                cudaStream_t s);
// out[i] = in[i] + out[i] + (e0 + f, e1) (coefficient form; out holds u pk): one thread per coefficient of a ciphertext
cudaError_t launch_sanitize_finish(const u64 *const *in, u64 *out, int n, const u64 *base, const RngKey &rk, const SanitizeConst &S, int logn,
                                   cudaStream_t s);

// ---- compact ciphertext upload (compact.cu; format in its header comment)
// stream-id purposes no other sampler call uses: the expanded c1, the noise e of a secret-key encryption, a test-seeded expansion key;
// the expanded a and the noise e of a compact key set's pairs
constexpr u64 PURPOSE_COMPACT_A = 11, PURPOSE_COMPACT_E = 12, PURPOSE_COMPACT_KEY = 13, PURPOSE_KEYS_A = 14, PURPOSE_KEYS_E = 15;
struct CompactKey {
    u32 w[8]; // ChaCha20 key K_c (the 32 header bytes as little-endian words)
};
struct CompactShape {
    int k, logn;
    int bits[KMAX];      // b_l = bitlen(q_l)
    u64 off[KMAX + 1];   // word offset of residue l inside one packed ciphertext; off[k] = words per ciphertext
};
// ct[j] = (c0 unpacked from packed[j] and made canonical, c1 expanded from key under stream_id(purpose, j0 + j, l)), j < n; packed == null:
// only c1 is written.  purpose: PURPOSE_COMPACT_A for ciphertexts, PURPOSE_KEYS_A for key pairs (ct is then [D][2][k][N] keys)
cudaError_t launch_compact_expand(u64 *ct, const u64 *packed, const CompactKey &key, u64 purpose, u64 j0, int n, const CompactShape &sh,
                                  const BehzConst *bc, cudaStream_t s);
// packed[j] = bit-packed c0 of ct[j] (canonical residues), j < n
cudaError_t launch_pack_residues(const u64 *ct, u64 *packed, int n, const CompactShape &sh, cudaStream_t s);
// x[n][k][N] = c0 + c1*s (coefficient form) -> plain[n][N]
cudaError_t launch_decrypt_round(const u64 *x, u64 *plain, int n, int k, int logn, const BehzConst *bc, PlainConst pc, cudaStream_t s);
cudaError_t launch_fill_zero(u64 *p, size_t words, cudaStream_t s);
// keys[d][0][src[d]][x] += factors[d] * target[src[d]][x]   (KeyGenerator: the 2^{jw} s' term of key-switching key d)
cudaError_t launch_key_add_scaled(u64 *keys, const u64 *target, const u64 *factors, const DigitMap &dm, int k, int logn, const BehzConst *bc,
                                  cudaStream_t s);

} // namespace cnhe
