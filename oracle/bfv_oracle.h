/*
 * oracle/bfv_oracle.h -- C interface of the CPU oracle.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (cryptonets_b200/, libcnhe.so)
 * may include, link or call this.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg use it, and only as the checker / timed CPU baseline.
 *
 * It restates, step by step, the BFV algorithms of Microsoft SEAL 3.2 that the reference
 * (microsoft/CryptoNets, "HE Wrapper/AtomicSealBfvVector.cs") reaches through SEALNet 3.2.0
 * ("HE Wrapper/packages.config:5").  SEAL itself is NOT in /root/reference and cannot be built
 * here, so PARITY WITH THE REAL SEAL BINARY IS UNPINNED; what is pinned is
 *   (i)  decrypted results == the reference's own known-answer tests (HE Wrapper Tests/BasicOperations.cs),
 *   (ii) an independent big-integer textbook BFV (oracle/textbook_bfv.py) on small N.
 *
 * Layout of every ciphertext buffer: [size][k][N] uint64, coefficient (non-NTT) form, canonical
 * residues in [0,q_i) -- SEAL's in-memory layout.
 */
#ifndef BFV_ORACLE_H
#define BFV_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_ctx orc_ctx;

/* coeff_count: number of default coefficient primes to keep (prefix of DefaultParams.CoeffModulus128(N)),
 * <=0 = all  (AtomicSealBfvVector.cs:140-151).  dbc_*: decomposition bit counts (IFactory.cs:244-245). */
orc_ctx *orc_create(uint64_t plain_modulus, uint32_t N, int coeff_count, int dbc_relin, int dbc_galois);
/* explicit coefficient moduli (used by small-N cross checks, and as transform tables of any NTT primes).  A q holding gamma makes
 * orc_decrypt fail; a q holding a prime of the Bsk base (m_sk or the first k auxiliary primes) makes orc_multiply, orc_square_layer
 * and the BEHZ stages fail: their constants divide by q modulo that prime, which is 0. */
orc_ctx *orc_create_custom(uint64_t plain_modulus, uint32_t N, const uint64_t *q, int k, int dbc_relin, int dbc_galois);
void orc_destroy(orc_ctx *);
const char *orc_last_error(void);
/* 0 (default, our reading of SEAL 3.2 mont_rq) = r_mtilde in [0,m~); 1 = centred (SEAL >= 3.3 style) */
void orc_set_centered_mtilde(orc_ctx *, int on);

uint32_t orc_N(const orc_ctx *);
int orc_k(const orc_ctx *);
uint64_t orc_t(const orc_ctx *);
void orc_get_coeff_moduli(const orc_ctx *, uint64_t *out /*k*/);
void orc_get_bsk_moduli(const orc_ctx *, uint64_t *out /*k+1, m_sk last*/);
uint64_t orc_gamma(const orc_ctx *);
/* which: 0..k-1 coefficient primes, k..2k Bsk primes, 2k+1 plain modulus.  Each out array has N words. */
void orc_get_ntt_tables(const orc_ctx *, int which, uint64_t *root_powers, uint64_t *scaled_root_powers,
                        uint64_t *inv_root_powers, uint64_t *scaled_inv_root_powers, uint64_t *inv_n);
uint64_t orc_minimal_primitive_root(uint64_t degree, uint64_t p);

/* raw NTT on one residue polynomial, canonical in / canonical out (bit-reversed NTT order) */
void orc_ntt_forward(const orc_ctx *, int which, uint64_t *poly);
void orc_ntt_inverse(const orc_ctx *, int which, uint64_t *poly);

/* keys.  deterministic in seed (counter-based sampler shared with the product, see DESIGN.md) */
void orc_keygen(orc_ctx *, uint64_t seed);
void orc_get_secret_key(const orc_ctx *, uint64_t *out /*k*N, NTT form*/);
void orc_get_public_key(const orc_ctx *, uint64_t *out /*2*k*N, NTT form*/);
int orc_relin_key_count(const orc_ctx *);
void orc_get_relin_keys(const orc_ctx *, uint64_t *out /*count*2*k*N, NTT form*/);
int orc_galois_elt_count(const orc_ctx *);
void orc_get_galois_elts(const orc_ctx *, uint64_t *out);
int orc_galois_key_count(const orc_ctx *); /* digits per element */
int orc_get_galois_key(const orc_ctx *, uint64_t elt, uint64_t *out /*count*2*k*N*/);
/* replaces the key of an element the context holds: the rotations of a server's client key slot, whose keys are not keygen's */
int orc_set_galois_key(orc_ctx *, uint64_t elt, const uint64_t *in /*count*2*k*N*/);

/* BatchEncoder */
void orc_encode(const orc_ctx *, const uint64_t *values, size_t n, uint64_t *plain /*N*/);
void orc_decode(const orc_ctx *, const uint64_t *plain, uint64_t *values /*N*/);

/* Encryptor / Decryptor.  plain has coeff_count (<=N) coefficients in [0,t) */
void orc_encrypt(const orc_ctx *, const uint64_t *plain, size_t coeff_count, uint64_t nonce, uint64_t *ct /*2kN*/);
int orc_decrypt(const orc_ctx *, const uint64_t *ct, int size, uint64_t *plain /*N*/);
int orc_noise_budget(const orc_ctx *, const uint64_t *ct, int size);

/* Evaluator */
void orc_add(const orc_ctx *, const uint64_t *a, const uint64_t *b, int size, uint64_t *out);
void orc_sub(const orc_ctx *, const uint64_t *a, const uint64_t *b, int size, uint64_t *out);
void orc_negate(const orc_ctx *, const uint64_t *a, int size, uint64_t *out);
void orc_add_plain(const orc_ctx *, const uint64_t *ct, int size, const uint64_t *plain, size_t coeff_count, uint64_t *out);
void orc_sub_plain(const orc_ctx *, const uint64_t *ct, int size, const uint64_t *plain, size_t coeff_count, uint64_t *out);
int orc_multiply_plain(const orc_ctx *, const uint64_t *ct, int size, const uint64_t *plain, size_t coeff_count, uint64_t *out);
int orc_multiply(const orc_ctx *, const uint64_t *a, const uint64_t *b, uint64_t *out /*3kN*/);
int orc_relinearize(const orc_ctx *, const uint64_t *ct3, uint64_t *out /*2kN*/);
int orc_apply_galois(const orc_ctx *, const uint64_t *ct, uint64_t elt, uint64_t *out);
int orc_rotate_rows(const orc_ctx *, const uint64_t *ct, int steps, uint64_t *out);
int orc_rotate_columns(const orc_ctx *, const uint64_t *ct, uint64_t *out);
uint64_t orc_galois_elt_from_step(const orc_ctx *, int steps);

/* individual BEHZ stages (exposed so each GPU kernel can be checked on its own) */
int orc_behz_lift(const orc_ctx *, const uint64_t *poly_q /*kN*/, uint64_t *poly_bsk /*(k+1)N*/); /* fastbconv_mtilde + mont_rq */
int orc_behz_floor(const orc_ctx *, const uint64_t *poly_q_bsk /*(2k+1)N, already *t */, uint64_t *poly_q /*kN*/); /* fast_floor + fastbconv_sk */

/* Multi-threaded layer-level drivers = the timed CPU baseline (mirrors Utils.ParallelProcessInEnv,
 * "HE Wrapper/Utils.cs:46-88": `threads` workers pulling output indices from an atomic counter). */
/* out[m] = sum_k weights[m*K+k] * in[gather[m*K+k]] (+ Delta*bias[m] on the constant coefficient);
 * weights/bias are residues in [0,t); gather <0 => tap skipped; zero weights skipped
 * (AtomicSealBfvVector.cs:434-521, PoolLayer.cs:196-227). */
int orc_mac_layer(const orc_ctx *, const uint64_t *in_cts, int n_in, const int32_t *gather, const uint64_t *weights,
                  const uint64_t *bias /*may be NULL*/, int M, int K, uint64_t *out_cts, int threads,
                  int m_begin, int m_step);
/* out[i] = relinearize(multiply(in[i], in[i]))   (SquareActivation.cs:10-13 -> AtomicSealBfvVector.cs:830-846) */
int orc_square_layer(const orc_ctx *, const uint64_t *in_cts, int n, uint64_t *out_cts, int threads, int begin, int step);
int orc_ntt_batch(const orc_ctx *, int which, uint64_t *polys, int n, int inverse, int threads);

#ifdef __cplusplus
}
#endif
#endif
