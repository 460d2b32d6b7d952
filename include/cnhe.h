/*
 * cnhe.h -- C ABI of libcnhe.so, the H100-native BFV engine behind the CryptoNets plugin API.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  A C# `B200BfvFactory : IFactory` binds these 121 entry points
 * with [DllImport("cnhe")] (stub in INTEGRATION.md); the Python mirror in cryptonets_b200/ binds them with ctypes.
 * One cnhe_vec is one reference `EncryptedSealBfvVector` ("HE Wrapper/EncryptedSealBfvVector.cs:150-573"): P
 * plaintext-modulus channels, each an `AtomicSealBfvEncryptedVector` ("HE Wrapper/AtomicSealBfvVector.cs:303-1476")
 * whose SEAL Ciphertext[] / Plaintext[] live in GPU HBM.  Every call is batched over blocks and channels;
 * nothing here computes on the CPU and the library fails at load/first call when no CUDA device is present.
 *
 * Conventions: every function returns 0 (CNHE_OK) or a negative error code; cnhe_last_error() gives the message of
 * the last failure on the calling thread (the reference throws System.Exception with the same wording where it has
 * one).  Nothing throws across the ABI.  Handles are opaque; vectors are immutable after creation except for the
 * metadata setters; destroying a vector that another vector/matrix aliases is safe (buffers are reference counted,
 * mirroring `CopyVectors:false` / `DataDisposedExternaly` in "HE Wrapper/EncryptedSealBfvMatrix.cs:32-58").
 * Calls may come from several host threads (reference: one IComputationEnvironment per thread,
 * "HE Wrapper/Utils.cs:46-88"); work is serialised onto the context's CUDA stream.
 *
 * Raw ciphertext layout (import/export): SEAL's in-memory layout, [poly][residue][coefficient] uint64, coefficient
 * (non-NTT) form, canonical residues.
 */
#ifndef CNHE_H
#define CNHE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define CNHE_OK 0
#define CNHE_ERR_INVALID (-1)   /* bad argument / dimension / format / scale mismatch (reference: System.Exception) */
#define CNHE_ERR_CUDA (-2)      /* CUDA runtime failure, including "no device" */
#define CNHE_ERR_STATE (-3)     /* keys missing, etc. */
#define CNHE_ERR_UNSUPPORTED (-4)

#define CNHE_DENSE 0  /* EVectorFormat.dense  ("HE Wrapper/IVector.cs:15-18") */
#define CNHE_SPARSE 1 /* EVectorFormat.sparse */
#define CNHE_ALL_SLOTS 0x7fffffffu /* Int32.MaxValue length of SumAllSlots ("AtomicSealBfvVector.cs:873,880") */

typedef struct cnhe_ctx cnhe_ctx; /* == EncryptedSealBfvFactory + its reference EncryptedSealBfvEnvironment */
typedef struct cnhe_vec cnhe_vec; /* == EncryptedSealBfvVector */

const char *cnhe_last_error(void);
const char *cnhe_version(void);

/* ---- context & keys ------------------------------------------------------------------------------------------ */
/* new EncryptedSealBfvFactory(primes, n, DecompositionBitCount, GaloisDecompositionBitCount, SmallModulusCount)
 * ("HE Wrapper/IFactory.cs:255-260"); coefficient modulus = first small_modulus_count entries (<=0: all) of
 * DefaultParams.CoeffModulus128(N) ("AtomicSealBfvVector.cs:140-151").  Builds every device table; no keys yet. */
int cnhe_context_create(const uint64_t *plain_primes, int P, uint32_t N, int dbc_relin, int dbc_galois,
                        int small_modulus_count, int device, cnhe_ctx **out);
/* same with explicit coefficient moduli (AtomicSealBfvVector.cs:152-161 Parms(t, n, coefModulus)): 1..9 primes = 1 mod 2N below
 * 2^61, each larger than every plaintext prime.  CNHE_ERR_INVALID for a q holding gamma = 0x1fffffffffc80001 (decryption's auxiliary
 * prime) or a prime of the BEHZ base (under CNHE_AUX_BASE=seal: m_sk = 0x1fffffffffe00001 and SEAL's first k auxiliary primes), which
 * would make decryption or the multiply silently wrong, and for a q whose auxiliary base would need more than 12 primes. */
int cnhe_context_create_custom(const uint64_t *plain_primes, int P, uint32_t N, const uint64_t *coeff_moduli, int k,
                               int dbc_relin, int dbc_galois, int device, cnhe_ctx **out);
int cnhe_context_destroy(cnhe_ctx *);
int cnhe_context_info(const cnhe_ctx *, uint32_t *N, int *k, int *P, int *relin_digits, int *galois_digits, int *galois_elts);
int cnhe_context_coeff_moduli(const cnhe_ctx *, uint64_t *out_k);
int cnhe_context_plain_moduli(const cnhe_ctx *, uint64_t *out_P);
/* the BEHZ auxiliary base Bsk (auxiliary primes, m_sk last); out may be NULL to query the count.  NTT modulus ids:
 * 0..k-1 coefficient primes, k..k+count-1 Bsk, k+count+c plaintext modulus c */
int cnhe_context_bsk_moduli(const cnhe_ctx *, uint64_t *out, int *count);
/* K_c of cnhe_mat_mul_colmajor_sparse_deferred: the most ciphertext products whose sum one BEHZ floor rounds exactly in this context's
 * Bsk, derived at context creation (DESIGN.md 4.14); at least 1, at most INT32_MAX */
int cnhe_context_product_sum_terms(const cnhe_ctx *, int *terms);
int cnhe_context_galois_elts(const cnhe_ctx *, uint64_t *out);
/* options: "behz_centered_mtilde" (0/1), "chunk" (ciphertexts per multiply/key-switch wave), "multi_stream" (1: one CUDA
 * stream per plaintext modulus, default; 0: everything on one stream; refused while imported batches are alive),
 * "trace_noise" (1: record the invariant noise budget after every evaluator-level operation, see cnhe_trace_read),
 * "release_cached_memory" (any value: hand the scratch blocks the context keeps for reuse back to the driver, e.g. before preparing a
 * large resident matrix) */
int cnhe_context_set_option(cnhe_ctx *, const char *name, int64_t value);
int cnhe_context_sync(cnhe_ctx *);
/* interop with the caller's own GPU work (the NCCL all-gather of the score ciphertexts): the CUDA stream (cudaStream_t as an integer) of a
 * channel, and the fences of the per-channel streams -- join: stream 0 waits for every channel's tail; fork: every channel waits for
 * stream 0.  Work the caller enqueues on stream 0 between a join and a fork is ordered after everything queued before the join and
 * before everything queued after the fork. */
int cnhe_context_stream(cnhe_ctx *, int channel, uint64_t *stream);
int cnhe_context_join_streams(cnhe_ctx *);
int cnhe_context_fork_streams(cnhe_ctx *);
/* EncryptedSealBfvEnvironment.GenerateEncryptionKeys ("EncryptedSealBfvVector.cs:92-102") -> KeyGenerator, RelinKeys(dbc),
 * GaloisKeys(dbc) ("AtomicSealBfvVector.cs:62-74"), sampled on the device.
 * cnhe_keys_generate_secure: every channel draws a fresh 256-bit ChaCha20 key from the OS (getrandom) -- secret key, key masks and all
 * later encryption randomness come from it (what SEAL's std::random_device gives the reference).  This is the production call.
 * A context is born with such a key per channel, so encrypting under an imported public key is safe without any seeding call.
 * cnhe_keys_generate(seed): DETERMINISTIC, TESTS ONLY -- the counter-based splitmix64 sampler shared with the CPU oracle (channel c uses
 * seed + c), so keys and fresh ciphertexts are bit-comparable; its outputs are predictable from the public key. */
int cnhe_keys_generate_secure(cnhe_ctx *);
int cnhe_keys_generate(cnhe_ctx *, uint64_t seed);
/* what: 0 secret key [k][N] (NTT form), 1 public key [2][k][N], 2 relin keys [D][2][k][N], 3 Galois key of element
 * `arg` [D][2][k][N]; export only: 4 the relin keys' packed copy the fused key switch reads (48-bit words, D 2 k N 6 / 8 words;
 * CNHE_ERR_STATE where the context keeps none: the fused key switch does not run or some q_l >= 2^48).  Stand-in for the SEAL key
 * streams of SaveToStream/LoadFromStream ("AtomicSealBfvVector.cs:93-130"). */
int cnhe_keys_export(cnhe_ctx *, int channel, int what, uint64_t arg, uint64_t *dst, size_t cap_words);
int cnhe_keys_import(cnhe_ctx *, int channel, int what, uint64_t arg, const uint64_t *src, size_t words);
int cnhe_keys_set_seed(cnhe_ctx *, int channel, uint64_t seed); /* TESTS ONLY: later encryptions of that channel use the deterministic sampler */
/* OperationsCount ("HE Wrapper/AtomicSealBfvVector.cs:211-294"): evaluator-level operations issued since creation / the last reset, in
 * the order Encryption, Decryption, Multiplication, Relinarization, PlainMultiplication (dense plaintext), ScalarMultiplication (constant
 * plaintext: SEAL's monomial multiply_plain), Addition, PlainAddition, Subtraction, PlainSubtraction, Rotation (row-rotation hops),
 * ColumnRotation, AddMany, AddManyItemCount.  cnhe_op_name(i) names counter i. */
#define CNHE_OP_COUNT 14
int cnhe_op_counts(cnhe_ctx *, uint64_t *out, int cap, int reset);
const char *cnhe_op_name(int kind);
/* CryptoTracker.TestBudget ("HE Wrapper/CryptoTracker.cs:41-52") as a trace: with option "trace_noise" on, every evaluator-level
 * operation appends a record of eight int32: kind, channel, count, invariant noise budget of its first output ciphertext (-1 when not
 * measured), the budgets its first and second input ciphertexts had when they were last measured (-1 unknown), an operation-specific
 * auxiliary value in thousandths (log2 |scalar| of a constant multiply, log2 of the root-sum-square weight of a MAC output, log2 of the
 * root-sum-square input noise of an AddMany) and a reserved word.  out may be NULL to query the record count.  Switching the option off
 * forgets the per-ciphertext budgets. */
int cnhe_trace_read(cnhe_ctx *, int32_t *out, size_t cap_records, size_t *n_records, int clear);

/* ---- wire / on-disk formats (SURVEY.md 8f-3).  The containers are the reference's; the SEAL 3.2 binary streams inside them are
 * restated from knowledge of SEAL 3.2.x and are UNPINNED against the real binary (see csrc/wire.cu for every layout).
 * cnhe_keys_save: EncryptedSealBfvEnvironment.Save ("HE Wrapper/EncryptedSealBfvVector.cs:104-134", IFactory.Save "IFactory.cs:484-495"):
 *   ZIP archive with one `environmentNNN` entry per plaintext modulus = AtomicSealBfvEncryptedEnvironment.SaveToStream
 *   ("AtomicSealBfvVector.cs:93-104").  dst may be NULL to query the size.
 * cnhe_context_load: the factory's file constructor (EncryptedSealBfvFactory(fileName), LoadFromStream "AtomicSealBfvVector.cs:106-131"):
 *   parameters (N, coefficient moduli, plaintext moduli, decomposition bit counts) and keys come from the archive; a context loaded
 *   from an archive without secret keys can encrypt and evaluate but not decrypt.
 * cnhe_vec_write / cnhe_vec_read: EncryptedSealBfvVector.Write / Read (":414-439", "AtomicSealBfvVector.cs:1273-1345"), the text form
 *   IFactory.LoadVector / LoadMatrix parse ("IFactory.cs:474-483"; a matrix is the reference's three header lines around its vectors). */
int cnhe_keys_save(cnhe_ctx *, int with_private_keys, uint8_t *dst, size_t cap, size_t *needed);
int cnhe_context_load(const uint8_t *archive, size_t len, int device, cnhe_ctx **out);
/* Compact evaluation keys (format version 1, this library's own; csrc/compact.cu has every field).  Half of every key pair is the uniform
 * polynomial a, which the server regenerates on the GPU from one 32-byte ChaCha20 key K_c per plaintext modulus (the ciphertext blob's
 * expansion); the other half, b, travels bit-packed at bitlen(q_l) bits per word: 2.6-2.9x smaller than the archive's key words, and
 * Galois elements the network never rotates by can be left out.  Blob: "CNHK" | u32 version = 1 | u32 N, k, P, dbc_relin, dbc_galois |
 * u32 sets (bit 0 public key, bit 1 relinearisation keys) | u32 G | k x u64 q_l | P x u64 t_c | G x u64 Galois elements (strictly
 * increasing) | P x 32-byte K_c | payload [P][pairs][k] packed b residues.  Pairs: public key, the relinearisation digits, then the Galois
 * digits of each listed element; a of pair kappa, residue l, word x is floor(q_l R / 2^128) with R = w[2x+1] 2^64 + w[2x], w the ChaCha20
 * keystream under K_c and stream id (14 << 48) | (kappa << 16) | l.
 * cnhe_keys_save_compact: the client side; needs the secret key (CNHE_ERR_STATE otherwise).  sets as above (other bits: CNHE_ERR_INVALID);
 * n_galois = -1 selects every element of cnhe_context_galois_elts, 0 none, otherwise galois_elts lists n_galois of them (any order;
 * duplicates and other elements: CNHE_ERR_INVALID).  The blob carries a FRESHLY generated key set under the context's secret key -- the
 * context's own keys are left untouched -- with one encryption nonce per pair for its noise.  K_c is a fresh OS draw per call and channel,
 * or seed-derived on a context seeded by cnhe_keys_generate(seed) (tests only).  dst == NULL queries the size in *needed, which depends on
 * the parameters and the selection only.  Counts no evaluator operation.
 * cnhe_context_load_compact: the server side, like cnhe_context_load: parameters come from the header, the keys are expanded on the GPU
 * straight into the key slots.  The context has no secret key and exactly the key sets the blob lists (missing ones refuse with
 * CNHE_ERR_STATE as usual).  Every header field, the element list and the exact length are checked on the host before anything is
 * allocated (CNHE_ERR_INVALID, no context).  Returns once the keys are complete. */
int cnhe_keys_save_compact(cnhe_ctx *, int sets, const uint64_t *galois_elts, int n_galois, uint8_t *dst, size_t cap, size_t *needed);
int cnhe_context_load_compact(const uint8_t *blob, size_t len, int device, cnhe_ctx **out);
/* Key slots: one context serves several clients, each with its own secret key.  Slot 0 is the context's own keys; every other slot holds
 * one client's evaluation keys.  cnhe_context_add_client_compact loads a compact key blob (format above; its public key, if any, is not
 * kept) into a new slot and returns its number in *slot: the relinearisation keys (with the fused key switch's packed copy) and the
 * listed Galois elements.  The blob is checked on the host before anything is allocated -- every header field, the exact length, and N,
 * k, every q_l, P, every t_c and both decomposition bit counts against the context's -- a defect or mismatch is CNHE_ERR_INVALID.
 * Returns once the keys are complete.  cnhe_context_remove_client frees a slot; its number is not handed out again, and operations on
 * vectors still bound to it fail with CNHE_ERR_INVALID.
 * Every encrypted vector is bound to a slot (0 when created, imported or read); cnhe_vec_set_key_slot binds it to another one (a
 * ciphertext a client encrypted and uploaded), cnhe_vec_key_slot reports it (-1 for a plain vector, which has none).  Results inherit
 * their operands' slot; two encrypted operands of different slots are CNHE_ERR_INVALID; a key switch that needs a key the slot does not
 * hold is CNHE_ERR_STATE, as a missing key is on a single-client context (a multi-hop rotation is planned from the Galois elements every
 * slot of the call holds).  Decryption and noise budgets need the secret key: slot 0 only (CNHE_ERR_STATE otherwise). */
int cnhe_context_add_client_compact(cnhe_ctx *, const uint8_t *blob, size_t len, int *slot);
int cnhe_context_remove_client(cnhe_ctx *, int slot);
int cnhe_vec_set_key_slot(cnhe_vec *, int slot);
int cnhe_vec_key_slot(const cnhe_vec *, int *slot);
/* Levels (modulus switching, SEAL's mod_switch_to_next for BFV; DESIGN 4.17).  cnhe_context_derive_level creates in *out a context on
 * the first k coefficient primes of this one (1 <= k < its k, else CNHE_ERR_INVALID): the same plaintext primes, N, decomposition bit
 * counts, device and Galois element list, with the tables, BEHZ base and options a context created on q_0..q_{k-1} would have, and the
 * options behz_centered_mtilde, chunk and multi_stream copied.  Its keys are the restriction of this context's: the secret and public
 * keys' rows l < k, and of every key-switching key the digits of residues l < k with their rows l < k -- word for word the keys a seeded
 * context on q_0..q_{k-1} generates.  Every live key slot is restricted too; a context without a secret key (cnhe_context_load_compact)
 * derives as well.  A seeded channel sampler is inherited.  The two contexts are independent afterwards: either may be destroyed first.
 * cnhe_vecs_mod_switch writes in out[i] vector in[i] of context `from` switched to context `to`, which must be a level of the same
 * family (derived from the same created context, directly or through other levels) with fewer primes: every ciphertext drops the primes
 * q_{k-1} .. q_{k'} one at a time, x -> round(x / q_j) mod q_0..q_{j-1}, in one pass over its words.  Encrypted vectors only; a
 * pending (deferred-relinearisation) vector is relinearised first.  Outputs keep dimension, scale, format and key slot, one slab per
 * channel; a slot whose keys in `from` were added or replaced since `to` was derived is restricted into `to` first, under the same
 * number.  Counts no operation.  `to`'s streams wait for the inputs and `from`'s streams for the switch.  CNHE_ERR_INVALID for vectors
 * of another context, plain vectors or an unrelated / not smaller `to`.  The switch is recorded when both contexts are enlisted in one
 * recording (cnhe_capture_begin_levels): its pointer table goes to the graph's memory and the event hand-off between the two contexts'
 * streams becomes an edge of the graph.  CNHE_ERR_STATE, the recording aborted, while one context records alone or the two record
 * different graphs, and while recording a switch that would have to restrict a slot's keys into `to` (the restriction synchronises: run
 * the chain once eagerly first, as CaptureInference does, or bind the graph to the slot, cnhe_graph_bind). */
int cnhe_context_derive_level(cnhe_ctx *, int k, cnhe_ctx **out);
int cnhe_vecs_mod_switch(cnhe_ctx *from, const cnhe_vec *const *in, int n, cnhe_ctx *to, cnhe_vec **out /*n*/);
int cnhe_vec_write(cnhe_ctx *, const cnhe_vec *, char *dst, size_t cap, size_t *needed);
int cnhe_vec_read(cnhe_ctx *, const char *text, size_t len, cnhe_vec **out, size_t *consumed);

/* ---- vectors: creation, metadata, disposal ---------------------------------------------------------------------- */
/* IFactory.GetEncryptedVector / GetPlainVector ("HE Wrapper/IFactory.cs:311-328"): round(v*scale), CRT split over the
 * plain primes ("EncryptedSealBfvVector.cs:352-365"), BatchEncoder.Encode per N-slot block (dense) or one constant
 * polynomial per element (sparse) ("AtomicSealBfvVector.cs:1114-1142"), Encryptor.Encrypt (":1202-1216"). */
int cnhe_vec_encrypt(cnhe_ctx *, const double *v, uint64_t dim, double scale, int format, cnhe_vec **out);
int cnhe_vec_plain(cnhe_ctx *, const double *v, uint64_t dim, double scale, int format, cnhe_vec **out);
/* the BigInteger overloads IFactory.GetPlainVector / GetEncryptedVector(IEnumerable<BigInteger>, format) ("IFactory.cs:29,43";
 * "EncryptedSealBfvVector.cs:188-199"): residues [P][dim], already reduced modulo each plaintext prime by the caller (SplitBigNumbers) */
int cnhe_vec_from_residues(cnhe_ctx *, const uint64_t *residues, uint64_t dim, double scale, int format, int encrypt, cnhe_vec **out);
/* batched form of IFactory.GetEncryptedMatrix ("IFactory.cs:353-380"): n dense vectors of `dim` values, v row-major [n][dim] */
int cnhe_vecs_encrypt(cnhe_ctx *, const double *v, int n, uint64_t dim, double scale, cnhe_vec **out);
/* IVector.Decrypt ("EncryptedSealBfvVector.cs:332-337,381-395"; "AtomicSealBfvVector.cs:1030-1067") */
int cnhe_vec_decrypt(cnhe_ctx *, const cnhe_vec *, double *out, uint64_t cap);
int cnhe_vecs_decrypt(cnhe_ctx *, const cnhe_vec *const *vecs, int n, double *out /*[n][dim]*/, uint64_t dim);
/* IVector.DecryptFullPrecision ("EncryptedSealBfvVector.cs:343-348"): per-channel residues [P][dim]; the caller joins them with big
 * integers (JoinSplitNumbers ":397-411") */
int cnhe_vec_decrypt_residues(cnhe_ctx *, const cnhe_vec *, uint64_t *out, uint64_t cap_words);
int cnhe_vec_copy(cnhe_ctx *, const cnhe_vec *, cnhe_vec **out); /* IFactory.CopyVector */
int cnhe_vec_destroy(cnhe_vec *);
/* Dispose of n vectors in one call (the Dispose loop of EncryptedSealBfvMatrix, EncryptedSealBfvMatrix.cs Dispose); null entries are skipped. */
int cnhe_vecs_destroy(cnhe_vec *const *vecs, int n);
int cnhe_vec_meta(const cnhe_vec *, uint64_t *dim, double *scale, int *format, int *is_encrypted, int *blocks, uint64_t *block_size);
int cnhe_vec_register_scale(cnhe_vec *, double scale); /* IVector.RegisterScale */
int cnhe_vec_register_dim(cnhe_vec *, uint64_t dim);   /* AtomicSealBfvVector.cs:316-319 */
/* raw ciphertext access for parity tests: block `block` of channel `channel`, 2*k*N words */
int cnhe_vec_export_raw(cnhe_ctx *, const cnhe_vec *, int channel, int block, uint64_t *dst, size_t cap_words);
int cnhe_vec_import_raw(cnhe_ctx *, const uint64_t *src /*[P][blocks][2kN]*/, int blocks, uint64_t dim, double scale, int format,
                        cnhe_vec **out);
/* batched forms: n vectors of `blocks` ciphertexts each; host layout [P][n][blocks][2kN].  One copy per channel; the
 * host buffer may be pinned (cudaHostAlloc / torch pin_memory) for full PCIe rate. */
int cnhe_vecs_import_raw(cnhe_ctx *, const uint64_t *src, int n, int blocks, uint64_t dim, double scale, int format, cnhe_vec **out);
int cnhe_vecs_export_raw(cnhe_ctx *, const cnhe_vec *const *vecs, int n, uint64_t *dst, size_t cap_words);
/* Asynchronous form for a pipelined serving loop: the device-to-host copies are queued behind the kernels that produce the vectors
 * and the call returns at once with a ticket; cnhe_export_wait(ticket) blocks until exactly those copies have landed in `dst`
 * (pinned host memory), without waiting for work queued afterwards.  Up to 8 tickets may be outstanding. */
int cnhe_vecs_export_raw_async(cnhe_ctx *, const cnhe_vec *const *vecs, int n, uint64_t *dst, size_t cap_words, int *ticket);
int cnhe_export_wait(cnhe_ctx *, int ticket);
/* Compact upload (format version 1, this library's own; csrc/compact.cu has every field).  A secret-key encryption is
 * (c0, c1) = (-(a s) + e + Delta m, a) with a uniform, so the data owner (who holds the secret key) sends c0 bit-packed at bitlen(q_l)
 * bits per residue plus one 32-byte ChaCha20 key K_c per plaintext modulus from which the server regenerates a on the GPU: 2.6-2.9x
 * fewer bytes than cnhe_vecs_import_raw's ciphertexts.  Blob: "CNHC" | u32 version = 1 | u32 N, k, P, n, B | u64 dim | f64 scale |
 * k x u64 q_l | P x u64 t_c | P x 32-byte K_c | payload [P][n][B][k] packed c0 residues (N bitlen(q_l) / 64 words each); c1 of
 * ciphertext j = i B + b, residue l, coefficient x is floor(q_l R / 2^128) with R = w[2x+1] 2^64 + w[2x], w[m] = 64-bit word m of the
 * ChaCha20 keystream under K_c and stream id (11 << 48) | (j << 16) | l (block counter m >> 3, word m & 7).
 * cnhe_vecs_encrypt_compact: seeded secret-key encryption of n dense vectors v[n][dim] (scale, CRT split and encoding as
 * cnhe_vecs_encrypt) into one blob; dst == NULL queries the size in *needed.  Needs the secret key (CNHE_ERR_STATE otherwise).  A secure
 * context draws a fresh K_c from the OS per call and channel; a context seeded by cnhe_keys_generate(seed) derives it from the seed.
 * Counted as Encryption.
 * cnhe_vecs_import_compact: the blob's vectors as ordinary encrypted dense vectors, asynchronous like cnhe_vecs_import_raw; out has room
 * for cap vectors, *n receives the count.  Every header field is checked against the context (CNHE_ERR_INVALID, no vector created).
 * Lifetime of src: pageable memory may be reused when the call returns; pinned memory (cudaHostAlloc / torch pin_memory) is read by an
 * asynchronous copy and must stay unchanged until the imported vectors have been consumed (e.g. their outputs exported). */
int cnhe_vecs_encrypt_compact(cnhe_ctx *, const double *v, int n, uint64_t dim, double scale, uint8_t *dst, size_t cap, size_t *needed);
int cnhe_vecs_import_compact(cnhe_ctx *, const uint8_t *src, size_t len, cnhe_vec **out, int cap, int *n);
/* device pointer of a channel's ciphertext blocks (for NCCL gathers through torch; plumbing only) */
int cnhe_vec_device_ptr(const cnhe_vec *, int channel, uint64_t *dptr, size_t *words);
int cnhe_noise_budget(cnhe_ctx *, const cnhe_vec *, int channel, int block, int *bits); /* CryptoTracker.cs:41-52 */

/* ---- IVector operations ------------------------------------------------------------------------------------------ */
int cnhe_vec_add(cnhe_ctx *, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out);          /* AtomicSealBfvVector.cs:983-1024 */
int cnhe_vec_sub(cnhe_ctx *, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out);          /* :1238-1271 */
int cnhe_vec_pointwise_multiply(cnhe_ctx *, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out); /* :813-860, :774-810 */
/* length == CNHE_ALL_SLOTS: full sum; force_column < 0: none */
int cnhe_vec_sum_all_slots(cnhe_ctx *, const cnhe_vec *a, uint64_t length, int force_column, cnhe_vec **out); /* :888-955 */
int cnhe_vec_dot_product(cnhe_ctx *, const cnhe_vec *a, const cnhe_vec *b, uint64_t length, int force_column, cnhe_vec **out); /* :964-977 */
int cnhe_vec_rotate(cnhe_ctx *, const cnhe_vec *a, int amount, cnhe_vec **out);              /* :1414-1430 */
int cnhe_vec_duplicate(cnhe_ctx *, const cnhe_vec *a, uint64_t count, cnhe_vec **out);       /* :1370-1408 */
int cnhe_vec_permute(cnhe_ctx *, const cnhe_vec *a, const cnhe_vec *const *selections, const int *shifts, int n,
                     uint64_t output_dim, cnhe_vec **out);                                   /* :1436-1475 */
int cnhe_vecs_interleave(cnhe_ctx *, const cnhe_vec *const *vecs, int n, int shift, cnhe_vec **out); /* :600-750 */
int cnhe_vecs_stack(cnhe_ctx *, const cnhe_vec *const *vecs, int n, cnhe_vec **out);         /* :756-761 */
/* cnhe_vecs_stack of B groups of n vectors, vecs [B][n] (one LoLa vectorize layer per client; the groups' key slots may differ, a group's
 * must not): out[b] is bit-identical to cnhe_vecs_stack(vecs + b * n, n), the rotations of all groups share key-switch waves. */
int cnhe_vecs_stack_batch(cnhe_ctx *, const cnhe_vec *const *vecs, int n, int B, cnhe_vec **out /*B*/);
int cnhe_vecs_generate_sparse_of_array(cnhe_ctx *, const cnhe_vec *const *vecs, int n, cnhe_vec **out); /* :1347-1359 */
/* One vector operation for B vectors at once (one per client, as many LoLa layers serve several clients in one pass; their key slots may
 * differ).  Each output is bit-identical to the single call named; every key-switching stage runs as one wave over all clients, and the
 * plain products of several clients with the same plaintexts transform each plaintext once.  The inputs must share dimension, scale,
 * format, block count and encryption (CNHE_ERR_INVALID otherwise, as for B < 1); other refusals are the single call's.
 * cnhe_vecs_duplicate_batch: out[b] = cnhe_vec_duplicate(vecs[b], count); cnhe_vec_duplicate is the case B = 1.
 * cnhe_vecs_permute_batch: out[b * n_perm + j] = cnhe_vec_permute(vecs[b], selections + j * n_sel, shifts + j * n_sel, n_sel, output_dim)
 *   (selections [n_perm][n_sel], NULL entries skipped; LLPreConvLayer's permutations of one image); cnhe_vec_permute is the case B = 1,
 *   n_perm = 1.  Both count one PlainMultiplication per non-NULL selection of every output, a selection listed twice included.
 * cnhe_vecs_interleave_batch: out[b] = cnhe_vecs_interleave(vecs + b * n, n, shift), vecs [B][n].
 * cnhe_vecs_multiply_plain: out[i] = cnhe_vec_pointwise_multiply(vecs[i], plain) for n encrypted vectors and one plain dense vector. */
int cnhe_vecs_duplicate_batch(cnhe_ctx *, const cnhe_vec *const *vecs, int B, uint64_t count, cnhe_vec **out /*B*/);
int cnhe_vecs_permute_batch(cnhe_ctx *, const cnhe_vec *const *vecs, int B, const cnhe_vec *const *selections, const int *shifts, int n_perm,
                            int n_sel, uint64_t output_dim, cnhe_vec **out /*B*n_perm*/);
int cnhe_vecs_interleave_batch(cnhe_ctx *, const cnhe_vec *const *vecs, int n, int B, int shift, cnhe_vec **out /*B*/);
int cnhe_vecs_multiply_plain(cnhe_ctx *, const cnhe_vec *const *vecs, int n, const cnhe_vec *plain, cnhe_vec **out /*n*/);
/* cnhe_vec_rotate of n vectors by the same amount in one pass (out[i] = rotation of vecs[i]); the vectors may belong to different key
 * slots.  Bit-identical to n cnhe_vec_rotate calls; cnhe_vec_rotate is the case n = 1. */
int cnhe_vecs_rotate(cnhe_ctx *, const cnhe_vec *const *vecs, int n, int amount, cnhe_vec **out /*n*/);

/* ---- IMatrix.Mul and the fused layer entry points ------------------------------------------------------------------ */
/* ColumnMajor matrix x sparse vector ("EncryptedSealBfvMatrix.cs:70-78" -> "AtomicSealBfvVector.cs:434-521") */
int cnhe_mat_mul_colmajor_sparse(cnhe_ctx *, const cnhe_vec *const *cols, int K, const cnhe_vec *sparse, cnhe_vec **out);
/* The same product with encrypted columns and an encrypted sparse vector, relinearised once per output block instead of once per product
 * (DESIGN.md 4.14).  Per plaintext prime and output block i:
 *   X_i = sum_k lift(cols[k]_i) (x) lift(sparse_k)   (size 3, base q u Bsk, summed in NTT form)
 *   Y_i = sum over chunks of floor_BEHZ(INTT(X_i restricted to the chunk's terms))   (mod q)
 *   out_i = relinearize(Y_i)
 * The K terms are cut into chunks of at most K_c (cnhe_context_product_sum_terms) in index order; each chunk is floored once.  The output
 * decrypts to cnhe_mat_mul_colmajor_sparse's values, dense, at scale(cols) scale(sparse), with the columns' dimension and blocks, but its
 * words differ: one floor-rounding term per chunk and one key-switch term per output instead of K of each.  Argument checks and messages are
 * cnhe_mat_mul_colmajor_sparse's; the columns must share dimension and blocks, every operand must be encrypted and in one key slot
 * (CNHE_ERR_INVALID otherwise, naming the existing call), and a chunk whose lifted operands and one output's sums need more than 8 GiB of
 * scratch is refused.  Counted as K bl Multiply, bl (K - 1) Addition, bl Relinearize and K bl AddMany items. */
int cnhe_mat_mul_colmajor_sparse_deferred(cnhe_ctx *, const cnhe_vec *const *cols, int K, const cnhe_vec *sparse, cnhe_vec **out);
/* RowMajor plain matrix x encrypted dense vector ("EncryptedSealBfvMatrix.cs:79-120" -> DotProduct per row = MultiplyPlain +
 * SumAllSlots, "AtomicSealBfvVector.cs:964-977,888-955"); force_dense: one-hot mask per row, rows summed into one dense vector */
int cnhe_mat_mul_rowmajor(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *v, int force_dense, cnhe_vec **out);
/* the same product for a contiguous slice of the rows (rows[i] = global row first_row + i of total_rows): the unit of the
 * intra-inference multi-GPU split of SURVEY.md 8e.  force_dense: one-hot masks at the global columns, so the ranks' partial results add up
 * to the full product ("EncryptedSealBfvMatrix.cs:92-116" sums the masked rows the same way); otherwise this slice's sparse elements. */
int cnhe_mat_mul_rowmajor_shard(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *v, int force_dense, int first_row,
                                int total_rows, cnhe_vec **out);
/* cnhe_mat_mul_rowmajor of one plain matrix with B vectors at once (one inference per client; their key slots may differ): out[b] is
 * bit-identical to cnhe_mat_mul_rowmajor(rows, n_rows, vs[b], force_dense), the key switches of all B x n_rows products share waves. */
int cnhe_mat_mul_rowmajor_batch(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *const *vs, int B, int force_dense,
                                cnhe_vec **out /*B*/);
/* DotProduct of every plain row with every encrypted vector (LLPackedDenseLayer's partial sums for B clients): out[b * n_rows + r] is
 * bit-identical to cnhe_vec_dot_product(rows[r], vs[b], length, -1), dimension and format included.  Rows and vectors as
 * cnhe_mat_mul_rowmajor_batch takes them. */
int cnhe_mat_dot_rows_batch(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *const *vs, int B, uint64_t length,
                            cnhe_vec **out /*B*n_rows*/);
/* Diagonal (Halevi-Shoup) product with baby-step / giant-step, the opt-in alternative to the ForceDenseFormat row-major product above for
 * large dense layers: about sqrt(N) rotations per input instead of 14 per row, and no one-hot mask multiply (DESIGN.md section 4.10).
 * Slot i sits at row i / (N/2), column i % (N/2) of the BatchEncoder's matrix.  Diagonal (b, s) of a matrix M (b in {0, 1}, s < N/2)
 * holds M[(a, x), (a ^ b, x + s mod N/2)] at slot (a, x); with s = n1 g + h it is stored rotated right by n1 g, and
 *   y = sum_g rotate_rows(n1 g)( sum_{b,h} diag'(b, n1 g + h) (.) rotate_columns^b rotate_rows(h)(v) ).
 * cnhe_diag_prepare: rows are n_rows <= N plain, dense, single-block vectors of one dim and one scale (what cnhe_mat_mul_rowmajor takes);
 *   the diagonals are formed, pre-rotated and encoded on the GPU, all-zero ones dropped (an all-zero matrix keeps one zero diagonal).
 *   baby_steps: n1, a power of two dividing N/2, or 0 to take the n1 with the fewest key switches per input, counted from the rotation hops
 *   over the context's Galois elements.  Anything else is CNHE_ERR_INVALID.  The rows may be destroyed afterwards.
 * cnhe_diag_info: rows, dim, n1, n2 = N/2 / n1, stored diagonals and the device bytes they hold (any pointer may be NULL).
 * cnhe_diag_export: stored diagonal `index` of a channel (N coefficients, mod t) and its (b, g, h) in bgh[3] (either may be NULL);
 *   diagonals are stored by g, then b, then h.
 * cnhe_mat_mul_diagonal: out[b] = M vs[b] for B encrypted, dense, single-block vectors of dim M's dim and one scale; their key slots may
 *   differ, out[b] keeps vs[b]'s.  out[b] is dense of dim n_rows and scale vs.scale * row scale, and decrypts to what
 *   cnhe_mat_mul_rowmajor(rows, vs[b], force_dense = 1) decrypts to (it is a different ciphertext).  A missing Galois key is CNHE_ERR_STATE.
 *   Counted as row-rotation hops, column rotations, plain multiplications, additions and one AddMany per output.
 * cnhe_diag_prepare_ntt: cnhe_diag_prepare (same checks, n1 and stored diagonals), and the diagonals of the longest prefix of whole
 *   giant-step groups whose NTT forms, summed over all channels (k N 8 bytes per diagonal and channel), fit in max_ntt_bytes are also held
 *   resident: lifted into every q_l and forward transformed, canonical, [diag][k][N] per channel -- the words cnhe_mat_mul_diagonal
 *   otherwise computes on every call.  UINT64_MAX holds the whole matrix, 0 none (the object then behaves as cnhe_diag_prepare's).
 *   cnhe_mat_mul_diagonal skips the lift and the transforms of the resident groups and runs a MAC kernel built to stream them from HBM;
 *   its outputs and counts are word for word the same.
 *   The coefficient-form diagonals stay (cnhe_diag_export is unchanged); device_bytes of cnhe_diag_info counts both forms.
 * cnhe_diag_ntt_info: resident giant-step groups, resident diagonals and the device bytes of their NTT forms (any pointer may be NULL).
 * cnhe_diag_export_ntt: the k N resident words of stored diagonal `index` of a channel ([k][N]); an index outside the resident prefix,
 *   a bad channel, cap_words < k N or another context's matrix is CNHE_ERR_INVALID.
 * cnhe_diag_prepare_folded: the folded (hybrid) diagonal product for matrices with few rows, R = n_rows <= N/2 and dim <= N; with
 *   n = N/2 and fold width W (a power of two, R <= W <= n) it keeps the W wrapped diagonals
 *     E_j[(a, x)] = M[x mod W, a n + (x + j mod n)]   (0 where the row is >= R or the column >= dim), j = n1 g + h < W,
 *   each rotated right by n1 g and stored as (b, g, h) = (0, g, h), all-zero ones dropped.  cnhe_mat_mul_diagonal then computes
 *     y' = sum_g rotate_rows(n1 g)( sum_h E'_{n1 g + h} (.) rotate_rows(h)(v) ),  y' += rotate_columns(y') when dim > n,
 *     y' += rotate_rows(s)(y') for s = W, 2W, ..., n/2,  y = mask_R (.) y'   (mask_R: 1 in slots 0 .. R-1, 0 elsewhere),
 *   so out[b] is dense of dim R (slot i = row i's sum, every other slot 0): one ciphertext per plaintext prime.  fold_width = 0 and / or
 *   baby_steps = 0 let the library choose W and / or n1 with the fewest key switches per input (BSGS rotations counted as for
 *   cnhe_diag_prepare, plus one when dim > n, plus log2(n / W)); on a tie the smaller W, then the smaller n1.  max_ntt_bytes as for
 *   cnhe_diag_prepare_ntt.  R > n, dim > N, a W that is not 0 or a power of two in [R, n], an n1 that does not divide W and whatever
 *   cnhe_diag_prepare refuses are CNHE_ERR_INVALID.  cnhe_diag_info reports n2 = W / n1; the export calls work unchanged (b = 0).
 *   Counted as the unfolded product, plus the fold's hops, column rotations and additions and one plain multiplication per output.
 * cnhe_diag_fold_width: W of a folded matrix, 0 for one from cnhe_diag_prepare or cnhe_diag_prepare_ntt. */
typedef struct cnhe_diag cnhe_diag;
int cnhe_diag_prepare(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, int baby_steps, cnhe_diag **out);
int cnhe_diag_prepare_ntt(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, int baby_steps, uint64_t max_ntt_bytes, cnhe_diag **out);
int cnhe_diag_info(const cnhe_diag *, int *n_rows, uint64_t *dim, int *n1, int *n2, int *n_diags, uint64_t *device_bytes);
int cnhe_diag_ntt_info(const cnhe_diag *, int *resident_giant_steps, int *resident_diags, uint64_t *ntt_bytes);
int cnhe_diag_export(cnhe_ctx *, const cnhe_diag *, int channel, int index, uint64_t *dst, size_t cap_words, int *bgh);
int cnhe_diag_export_ntt(cnhe_ctx *, const cnhe_diag *, int channel, int index, uint64_t *dst /* k*N */, size_t cap_words);
int cnhe_diag_destroy(cnhe_diag *);
int cnhe_mat_mul_diagonal(cnhe_ctx *, const cnhe_diag *, const cnhe_vec *const *vs, int B, cnhe_vec **out /*B*/);
int cnhe_diag_prepare_folded(cnhe_ctx *, const cnhe_vec *const *rows, int n_rows, int fold_width, int baby_steps, uint64_t max_ntt_bytes,
                             cnhe_diag **out);
int cnhe_diag_fold_width(const cnhe_diag *, int *width);
/* Whole PoolLayer.Apply with weights ("NeuralNetworks/PoolLayer.cs:149-229"): out[m] = sum_k weights[m][k] * in[gather[m*K+k]]
 * + bias[m].  The inputs may belong to different key slots (several clients' images side by side) as long as each output's taps share
 * one; the output takes it.  weights[m] is a plain SPARSE vector of dim K, bias[m] a plain DENSE vector (or NULL); gather < 0 is a
 * padded tap (the reference multiplies a fresh encryption of zero there; we add nothing -- same decryption). */
int cnhe_layer_conv_dense(cnhe_ctx *, const cnhe_vec *const *in, int n_in, const int32_t *gather, const cnhe_vec *const *weights,
                          const cnhe_vec *const *bias, int M, int K, cnhe_vec **out /*M*/);
/* SquareActivation.Apply over a whole matrix ("NeuralNetworks/SquareActivation.cs:10-13"): out[i] = in[i] (.) in[i].  The vectors may
 * belong to different key slots (several clients' layers in one call): each is relinearised under its own slot's keys. */
int cnhe_layer_square(cnhe_ctx *, const cnhe_vec *const *in, int n, cnhe_vec **out /*n*/);
/* Quadratic activation a x^2 + b x + c over a whole matrix, in the passes of cnhe_layer_square: out[i] is, word for word,
 *   relinearize(multiply_plain(in[i] (.) in[i], a)) + multiply_plain(in[i], b) + c      (scale scale(a) s^2, s = scale of the inputs)
 * with the terms applied inside the product's BEHZ floor kernel.  a, b, c are plain SPARSE vectors of dimension 1 (cnhe_vec_plain);
 * b and c may be NULL.  A term that is 0 mod a plaintext prime contributes nothing in that channel.  Slots: C is added to the data slots of
 * a dense vector only -- the last block of a vector whose dimension is not a multiple of N gets add_plain of the plaintext with C in its
 * data slots and 0 in its padding slots, so padding stays zero as it does for cnhe_layer_square (rotations and cnhe_vec_duplicate add
 * whole ciphertexts); every other ciphertext, and every ciphertext of a sparse vector, gets the constant plaintext C (all N slots).  (a, b, c) = (1, NULL, NULL) gives
 * cnhe_layer_square's words.  The inputs must share one scale, and scale(b) s and scale(c) must equal scale(a) s^2 exactly; the vectors
 * may belong to different key slots, as for cnhe_layer_square.  Operation counts are those of the composition. */
int cnhe_layer_poly2(cnhe_ctx *, const cnhe_vec *const *in, int n, const cnhe_vec *a, const cnhe_vec *b, const cnhe_vec *c, cnhe_vec **out /*n*/);
/* Polynomial activation P(x) = sum_j coeffs[j] x^j of degree 3 or 4 over a whole matrix, in two multiplicative levels built from squares
 * only (DESIGN.md section 4.12).  coeffs has degree + 1 entries, coeffs[j] the coefficient of x^j: plain SPARSE vectors of dimension 1
 * at scale W s^(degree - j), W = scale(coeffs[degree]), s = scale of the inputs; NULL means 0, except coeffs[degree], which is required
 * and must be nonzero mod every plaintext prime.  The output scale is W s^degree.  Per plaintext prime, with the constants of DESIGN 4.12
 * and "+ K" a constant added as cnhe_layer_poly2 adds c (data slots only on a dense vector), out[i] is, word for word,
 *   quartic:  q = cnhe_layer_poly2(x; 1, beta, gamma);  relinearize(A (.) multiply(q, q)) + multiply_plain(x, D') + E'
 *   cubic:    u = relinearize(multiply(x, x));  q1 = add(u, x) + gamma;
 *             relinearize(lambda (.) (multiply(q1, q1) - multiply(u, u))) + multiply_plain(x, C') + D'
 * where K (.) multiplies all three polynomials of a size-3 ciphertext by the constant K.  The inputs must share one scale, and the
 * vectors may belong to different key slots, as for cnhe_layer_square.  Operation counts are those of the composition. */
int cnhe_layer_poly(cnhe_ctx *, const cnhe_vec *const *in, int n, const cnhe_vec *const *coeffs /*degree + 1*/, int degree,
                    cnhe_vec **out /*n*/);
/* The square (a, b, c all NULL) or the quadratic activation of cnhe_layer_poly2, followed by the layer of cnhe_layer_conv_dense, with the
 * relinearisation deferred to the layer's outputs: M key switches per block instead of n_in.  Per plaintext prime, out[m] is, word for word,
 *   P3(x)  = A (.) multiply(x, x) + (B x0 + Delta C, B x1, 0)      (size 3; (A, B, C) = (1, 0, 0) when a is NULL)
 *   out[m] = relinearize(sum_k w[m][k] (.) P3(in[gather[m*K+k]]) + add_plain(bias[m]))
 * where w (.) multiplies all three polynomials by the weight, lifted as the scalar MAC lifts it, and the bias goes to c0.  The same
 * decryption as cnhe_layer_conv_dense over cnhe_layer_poly2's (or cnhe_layer_square's) outputs, with one key-switch noise term per output
 * instead of a weighted sum of them.  a, b, c follow cnhe_layer_poly2 (C in the data slots of a dense vector only); in, gather, weights,
 * bias and the key slots follow cnhe_layer_conv_dense.  The output scale is scale(a) s^2 scale(w) (s^2 scale(w) for the square), which the
 * bias must share.  Operation counts are those of the composition: n_in * blocks multiplications, the activation's terms, the scalar MAC's
 * counts and M * blocks relinearisations.  All n_in * blocks size-3 products of a plaintext prime are held at once: a call that needs
 * more than 8 GiB for them is refused (CNHE_ERR_INVALID). */
int cnhe_layer_activation_conv_dense(cnhe_ctx *, const cnhe_vec *const *in, int n_in, const cnhe_vec *a, const cnhe_vec *b, const cnhe_vec *c,
                                     const int32_t *gather, const cnhe_vec *const *weights, const cnhe_vec *const *bias, int M, int K,
                                     cnhe_vec **out /*M*/);

/* ---- recording and replaying a chain of calls as one CUDA graph -------------------------------------------------- */
/* A latency-bound inference (one LoLa image) spends its time launching hundreds of small kernels and preparing their arguments on the
 * host.  Recorded once, for fixed shapes and prepared weights, the same chain replays as one graph launch per input: the same sm_90a
 * kernels in the same order with the same arguments, and no host work between them.  Its key switches read their keys through the
 * graph's key binding, so one recording serves every client of the context (cnhe_graph_bind).
 * cnhe_capture_begin: from now on the context records its calls instead of running them (CNHE_ERR_STATE while already recording, and
 *   CNHE_ERR_INVALID while profiling or the noise trace is on).  Works with "multi_stream" 0 and 1: the channel streams fork from the
 *   capturing stream and join it through events, as cnhe_context_fork_streams / cnhe_context_join_streams order them.
 * cnhe_capture_end: instantiates what was recorded into *out.  cnhe_capture_abort: drops the recording (a no-op when not recording); the
 *   context stays usable.
 * cnhe_graph_launch: enqueues one replay on the context's streams -- asynchronous and ordered with the calls before and after it, like any
 *   other call.  CNHE_ERR_STATE when a key slot the graph is bound to has since been removed or had its keys replaced (key generation
 *   or import) -- binding it again reads the new keys -- and while the context records.  Each launch adds the recorded operation counts to cnhe_op_counts and the recorded kernel
 *   count to cnhe_kernel_launch_count: per-inference figures match the eager calls'.  Recording itself counts nothing.
 * cnhe_graph_slots: the graph's key positions -- the distinct key slots its recorded key switches read, in ascending slot number -- into
 *   slots[0 .. min(cap, *n)), their number into *n (slots may be NULL).
 * cnhe_graph_bind: binds key position i to key slot slots[i] (n = the number of positions, CNHE_ERR_INVALID otherwise): from the next
 *   launch on, every recorded key switch that read position i's keys -- relinearisation keys (u64 or 48-bit packed) and Galois keys -- reads
 *   slot slots[i]'s keys of the same kind instead.  Several positions may be bound to one slot.  The recording is the first binding (every
 *   position bound to itself), so a graph never bound behaves as recorded.  Before changing anything the call checks that each slot is live
 *   (CNHE_ERR_INVALID) and holds every key its position's key switches read, per plaintext channel: the relinearisation keys in the form
 *   recorded and each recorded Galois element (CNHE_ERR_STATE naming the slot and the element otherwise).  A refused bind leaves the
 *   previous binding in force; refused while the context records.  A launch reads the bound slots' keys as they were when bound.  Binds and
 *   launches are ordered like any call: launches bound to different clients may be enqueued back to back without a host synchronisation,
 *   and each reads its own binding.  A bind allocates no device memory, with one exception for a graph that spans levels: a bound slot
 *   whose keys in an enlisted level are not those of the graph's context (a client added to, replaced in or removed from the context since
 *   the level was derived or last switched to) is first restricted into that level, as the eager switch would (that allocates the level's
 *   copy of the keys and synchronises).  Slots are numbered alike in every context of a family, so positions are slot numbers there too.
 *   Vectors created while recording report, and are key-switched and decrypted under, the slot their slot's position is bound to
 *   (cnhe_vec_key_slot).  The recorded input vectors predate the recording: retag them (cnhe_vec_set_key_slot) before cnhe_vecs_assign.
 *   Rotation hop plans and the choice of key-switch path stay as recorded: a client holding the recording client's Galois elements gets,
 *   word for word, its eager inference's ciphertexts; a client holding more elements follows the recorded (possibly longer) hop plan, whose
 *   results decrypt to the same values but whose words can differ from an eager run, which plans from that client's own elements.
 * cnhe_graph_info: the graph's kernel nodes and the device bytes it owns (either pointer may be NULL).
 * cnhe_graph_destroy: waits for the context's queued work and releases the graph (CNHE_ERR_STATE while the context records).  Destroy every
 *   graph before any context it spans.
 * cnhe_capture_begin_levels: a recording on `ctx` that also enlists the n contexts levels[0..n) -- levels of ctx's family with fewer
 *   primes (cnhe_context_derive_level), typically the ones a levelled network switches to.  Calls on any enlisted context, and the
 *   cnhe_vecs_mod_switch calls between them, are captured into the one graph cnhe_capture_end(ctx) returns; it is launched, bound and
 *   destroyed like any other.  CNHE_ERR_INVALID for a null argument, a level listed twice, ctx itself, a context of another family or one
 *   with no fewer primes than ctx, and, as for cnhe_capture_begin, while any of the contexts profiles or traces noise; CNHE_ERR_STATE while
 *   any of them records (ctx's own recording is then aborted, an enlisted level's is left running).
 *   Streams: the capture runs on ctx's channel stream 0, and at begin every channel stream of every enlisted context forks from it (an
 *     event on that stream, a wait on each of theirs), before any call: a stream left out would run its work (a bias upload, a plain
 *     vector) once, at record time, and never in a replay.  cnhe_capture_end joins every enlisted stream back into ctx's stream 0 first.
 *     A launch joins every stream of every enlisted context into ctx's stream 0, launches there, then forks them all again, so a later
 *     eager call on a level (decrypting the scores) is ordered after the replay.
 *   One recording: the enlisted contexts share the graph's memory, its key binding and its fate.  A call refused or failing on any of
 *     them -- another thread's call included -- aborts the recording of every one, after which each computes eagerly;
 *     cnhe_capture_abort on any of them does the same.  cnhe_capture_end must be called on ctx (on a level it is refused, and aborts).
 *     Buffers from before the recording that a level releases during it stay allocated until the graph is destroyed.
 *   Counts: each context's operation counters and kernel count are restored when the recording ends, and each launch adds to every
 *     context what was recorded on it: after a launch every context's counts equal those of one eager levelled inference.
 *   Key binding: a recorded key switch on a level reads that level's keys of the bound slot (see the restriction under cnhe_graph_bind).
 *     A launch is refused (CNHE_ERR_STATE) when a bound slot's keys changed since the bind in any enlisted context.
 *   cnhe_graph_destroy synchronises every enlisted context, and is refused while any of them records.
 * cnhe_vecs_assign: copies each src[i]'s ciphertext words into dst[i], device to device, ordered like any call: how a new input enters a
 *   graph's recorded input vectors.  Both must be encrypted and match in dimension, blocks, format, scale and key slot (the recording acted
 *   on those); the slots must be live, as for the calls that take several vectors, and a destination may not partly overlap its source
 *   (CNHE_ERR_INVALID otherwise).  May be recorded.
 * What a recording means:
 *   Outputs: vectors created while recording belong to the graph.  Their words are defined once a launch completes and are overwritten by
 *     the next launch.  Destroying an intermediate while recording lets later recorded allocations reuse its memory inside the graph; it
 *     frees nothing outside the graph.  Vectors made by an aborted recording hold no defined words.
 *   Memory: recorded allocations come from device memory the graph owns, never from the context's scratch recycling or upload slots, so
 *     no eager call is handed a block a replay writes.  It returns to the driver once the graph and every vector made while recording are
 *     destroyed.  Vectors, keys and prepared matrices created before the recording are read in place by every launch and must outlive the
 *     graph; a buffer of theirs that is released while recording stays allocated until the graph is destroyed.
 *   Constants: pointer tables, masks, scalar tables and every other host-built argument are copied once, at record time, into the graph's
 *     memory; a launch reads nothing from the host.
 *   Host decisions (which key-switch path, whether a square stays unrelinearised for the next layer, wave sizes) are taken at record time
 *     and replay as recorded.
 *   Refused while recording, with CNHE_ERR_STATE naming the call: every call that returns words or decisions to the host (decryption,
 *     exports, cnhe_vec_device_ptr, noise budgets, cnhe_context_sync, preparing a diagonal matrix), every call that samples randomness
 *     (encryption, including the fresh encryptions of zero an unfused layer makes: a replay would reuse it for every input), uploads,
 *     profiling, the noise trace, key generation, import and export, adding or removing clients, cnhe_context_set_option, resetting the
 *     operation counters, reading squares a cnhe_layer_square made before the recording and left unrelinearised (read them once
 *     first: relinearised inside the graph they would hold no words until a launch), and any call on the context from another thread
 *     than the recording one.  Any call that fails while recording
 *     aborts the recording, as cnhe_capture_abort does; cnhe_capture_end then reports CNHE_ERR_STATE. */
typedef struct cnhe_graph cnhe_graph;
int cnhe_capture_begin(cnhe_ctx *);
int cnhe_capture_begin_levels(cnhe_ctx *ctx, cnhe_ctx *const *levels, int n);
int cnhe_capture_end(cnhe_ctx *, cnhe_graph **out);
int cnhe_capture_abort(cnhe_ctx *);
int cnhe_graph_launch(cnhe_graph *);
int cnhe_graph_slots(const cnhe_graph *, int *slots, int cap, int *n);
int cnhe_graph_bind(cnhe_graph *, const int *slots, int n);
int cnhe_graph_info(const cnhe_graph *, uint64_t *kernel_nodes, uint64_t *device_bytes);
int cnhe_graph_destroy(cnhe_graph *);
int cnhe_vecs_assign(cnhe_ctx *, cnhe_vec *const *dst, const cnhe_vec *const *src, int n);

/* ---- micro-benchmark / kernel-level entry points on caller-owned device memory ("raw") --------------------------- */
int cnhe_dev_alloc(cnhe_ctx *, size_t words, uint64_t *dptr);
int cnhe_dev_free(cnhe_ctx *, uint64_t dptr);
int cnhe_dev_upload(cnhe_ctx *, uint64_t dptr, const uint64_t *src, size_t words);
int cnhe_dev_download(cnhe_ctx *, uint64_t *dst, uint64_t dptr, size_t words);
/* n_polys residue polynomials at src; polynomial b uses modulus id mod_base + b % mod_count
 * (ids: see cnhe_context_bsk_moduli) */
int cnhe_raw_ntt(cnhe_ctx *, uint64_t src, uint64_t dst, int n_polys, int mod_base, int mod_count, int inverse);
int cnhe_raw_multiply(cnhe_ctx *, int channel, uint64_t a, uint64_t b, int n, uint64_t out3);     /* Evaluator.Multiply, size 3 out */
int cnhe_raw_relinearize(cnhe_ctx *, int channel, uint64_t in3, int n, uint64_t out2);
int cnhe_raw_multiply_relin(cnhe_ctx *, int channel, uint64_t a, uint64_t b, int n, uint64_t out2);
int cnhe_raw_apply_galois(cnhe_ctx *, int channel, uint64_t in, int n, uint64_t galois_elt, uint64_t out);
int cnhe_raw_rotate_rows(cnhe_ctx *, int channel, uint64_t in, int n, int steps, uint64_t out);
int cnhe_raw_behz_lift(cnhe_ctx *, uint64_t in_cts, int n, uint64_t out_together);
int cnhe_raw_behz_floor(cnhe_ctx *, int channel, uint64_t d_together, int n, uint64_t out3);
int cnhe_dev_copy(cnhe_ctx *, uint64_t dst, uint64_t src, size_t words); /* device to device, on the context stream */
/* n size-3 products from host words [P][n][3][k][N] as n one-block dense vectors of dimension dim (<= N) in key slot `slot`, left
 * unrelinearised in one group exactly as cnhe_layer_square leaves its squares: a scalar-MAC layer over all of them takes the exact
 * path (DESIGN 4.15), any other read relinearises the group.  For parity tests of that path with chosen digits.  CNHE_ERR_INVALID where
 * cnhe_layer_square would relinearise at once (noise trace, no plane-source key switch, digits wider than 16 bits, more than 8 GiB of
 * products) and for words that are not canonical residues. */
int cnhe_raw_import_products(cnhe_ctx *, const uint64_t *words, int n, uint64_t dim, double scale, int slot, cnhe_vec **out);
/* per-kernel-family device timing (CUDA events around the launches on the context stream): enable, run, collect.
 * family: 0 ntt forward (incl. digit variant), 1 ntt inverse, 2 behz element-wise, 3 key-switch mac, 4 scalar mac layer, 5 other */
int cnhe_prof_enable(cnhe_ctx *, int on);
int cnhe_prof_collect(cnhe_ctx *, int family, double *total_ms, uint64_t *launches, double *algorithmic_bytes);
int cnhe_raw_event_timing(cnhe_ctx *, int start); /* start=1: record start event; start=0: record stop, return via cnhe_raw_elapsed_ms */
int cnhe_raw_elapsed_ms(cnhe_ctx *, float *ms);
uint64_t cnhe_kernel_launch_count(const cnhe_ctx *); /* kernels launched by this library since context creation */

#ifdef __cplusplus
}
#endif
#endif
