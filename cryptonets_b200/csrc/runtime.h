// Host runtime of libcnhe: context (device tables, keys, workspace) and the ciphertext-array operations the vector
// layer (vec.cu) is built from.  Mirrors AtomicSealBfvEncryptedEnvironment ("HE Wrapper/AtomicSealBfvVector.cs:19-206")
// plus the SEAL objects it owns (SEALContext, KeyGenerator, Evaluator, Encryptor, Decryptor, BatchEncoder).
#pragma once
#include <cstdint>
#include <algorithm>
#include <atomic>
#include <map>
#include <unordered_map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "kernels.h"

namespace cnhe {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};
void cuda_check(cudaError_t e, const char *what);
#define CNHE_CUDA(x) ::cnhe::cuda_check((x), #x)

// Device memory of one recorded graph (cnhe_capture_begin .. cnhe_capture_end): every allocation made while recording comes from here, never
// from the stream-ordered pool or the context's recycle list, so no eager call can be handed a block a replay writes.  A block released
// while recording goes to a per-stream free list that later recorded allocations on the same stream take from (stream order inside the
// graph makes that safe, as it does for the recycle list); once the recording ends nothing is reused.  Host-built constants get blocks of
// their own that are never released.  The memory goes back to the driver when the graph and every buffer cut from it are gone.
struct GraphArena {
    std::vector<void *> blocks;
    size_t bytes = 0;
    bool recording = true;
    struct Free { u64 *p; size_t words; cudaStream_t stream; };
    std::vector<Free> free;
    unsigned char *const_block = nullptr;
    size_t const_off = 0, const_cap = 0;
    u64 *take(size_t words, cudaStream_t s, size_t &got_words);
    void give(u64 *p, size_t words, cudaStream_t s) { if (recording) free.push_back({p, words, s}); }
    void *fresh(size_t bytes); // nullptr when the device is out of memory
    // a device copy of `bytes` host bytes, complete on return (copied on `s`, a stream outside the recording)
    const void *constant(const void *src, size_t bytes, cudaStream_t s);
    ~GraphArena();
};

// Reference-counted device allocation (stream-ordered pool).
struct DevBuf {
    u64 *p = nullptr;
    size_t words = 0;
    cudaStream_t stream = nullptr; // release stream: the channel the buffer belongs to (also the allocation stream unless given)
    struct Context *owner = nullptr; // set: a large block goes back to the context's per-stream recycle list instead of the driver pool
    DevBuf(size_t w, cudaStream_t s);
    DevBuf(size_t w, cudaStream_t s, struct Context *owner);
    int upload_slot = -1; // >= 0: the block is one of the context's persistent upload slots (returned, not freed)
    std::shared_ptr<GraphArena> arena; // set: allocated while recording a graph, from that graph's memory
    ~DevBuf();
    DevBuf(const DevBuf &) = delete;
};
typedef std::shared_ptr<DevBuf> BufRef;

// The key binding of a recorded graph (DESIGN 4.16).  While recording, every key base a key switch hands a kernel is replaced by a key
// reference: the address of one word of `table`, a small device array the graph owns, that stands for one key of one key slot and
// channel -- the relinearisation keys, their packed copy, the keys of one Galois element, or the public key (sanitisation).  The graph's key positions are the distinct
// slots its references name, in ascending order.  Binding (cnhe_graph_bind) points every word of a position at another slot's key of
// the same kind, and the next launch copies the words into the table before the recorded kernels read them.
struct KeyBinding {
    enum Kind { RLK, RLK_PACKED, GALOIS, PK };
    struct Key { int slot, channel, kind; u64 elt; int member; }; // member: the enlisted context whose key pick took it (RecGroup)
    std::map<const u64 *, Key> seen;      // while recording: every key base picked for a key switch, and which key it is
    std::map<const u64 *, size_t> word;   // key base -> its table word
    std::vector<Key> words;               // the key each table word stands for, in the order they were handed out
    const u64 **table = nullptr;          // device, `cap` words (graph memory)
    size_t cap = 0;
    std::map<int, int> to;                // recorded slot -> the slot it is bound to (identity until the first bind)
    int slot(int s) const { const auto it = to.find(s); return it == to.end() ? s : it->second; }
    const u64 *ref(const u64 *base);      // the key reference of a key base picked while recording
};

// The contexts one recording spans (cnhe_capture_begin_levels; one context for cnhe_capture_begin): the capture runs on members[0]'s
// stream 0, and every channel stream of every member forks from it.  Members are ordered by descending prime count, the order their
// locks are taken in.  abort_requested: a refused call found another member's lock taken (a call in flight on another thread), so the
// recording could not end at once; the recording thread's next call on any member ends it.
struct RecGroup {
    std::vector<struct Context *> members;
    std::atomic<bool> abort_requested{false};
};

// State of a context while it records its calls into a CUDA graph (stream capture of the channel streams, vec.cu cnhe_capture_*)
struct Recording {
    std::thread::id thread;             // the recording thread: calls from any other thread are refused
    std::shared_ptr<RecGroup> group;    // the contexts of the recording, shared by every member's Recording
    int member = 0;                     // this context's index in group->members
    std::shared_ptr<GraphArena> arena;  // shared by every member
    std::vector<uint64_t> op0;          // operation counters and kernel count when the recording began: restored when it ends, the
    uint64_t launches0 = 0;             // difference is what every launch of the graph adds
    std::vector<uint64_t> sanitized0;   // the same for the channels' sanitisation nonces (Channel::sanitized)
    std::shared_ptr<KeyBinding> keys;   // the references the recorded key switches read their keys through (shared by every member)
    std::vector<std::shared_ptr<void>> keep; // cached host-built device tables (scalar-MAC plans) the recorded kernels read
    // buffers allocated before the recording and released during it: the graph may read them, so they are freed (or recycled) outside
    // it, when the graph is destroyed (at once when the recording is aborted)
    struct Deferred { u64 *p; size_t words; cudaStream_t stream; int upload_slot; };
    std::vector<Deferred> deferred;
};

// the keys of one client under one plaintext modulus: evaluation keys, and the public key that sanitisation encrypts zero under
struct KeySet {
    bool have_rlk = false, have_pk = false;
    BufRef rlk, pk;   // pk: [2][k][N] NTT form
    BufRef rlk_packed; // rlk with 48-bit words for the fused key switch (set by rlk_ready when that kernel can run and every q_l < 2^48)
    std::map<u64, BufRef> glk;
};
struct Channel : KeySet { // one plaintext modulus (one AtomicSealBfvEncryptedEnvironment); its own keys are key slot 0
    u64 t = 0;
    PlainConst pc;
    int mod_id = 0; // NTT table id of t
    bool have_sk = false;
    BufRef sk;
    RngKey rng;    // secure (ChaCha20 keyed from the OS) unless a deterministic test seed was requested explicitly
    u64 nonce = 1; // running encryption counter (32 bits enter the stream id; a secure channel re-keys before it wraps)
    // Sanitisation nonces (DESIGN 4.18) come from a device counter, d_sanitize_nonce[channel], that the call's first kernel reads and
    // advances, so that every replay of a recorded graph draws fresh randomness; `sanitized` is the host's count of the nonces handed out
    // (eager calls and graph launches), which keeps the counter below SANITIZE_NONCES
    u64 sanitized = 0;
    FloorConstF floor_f; // folded fast_floor constants for this t (valid when the context's fp_elementwise is set)
};

struct Context {
    int device = 0;
    uint32_t N = 0;
    int logN = 0, k = 0, kb = 0, P = 0, dbc_relin = 0, dbc_galois = 0; // kb: primes in the BEHZ base Bsk
    std::vector<u64> q, bsk, t;
    BehzConst h_bc;
    BehzConst *d_bc = nullptr;
    BehzConstF h_bf;
    BehzConstF *d_bf = nullptr;
    // the FP64 element-wise path: every q_i and Bsk prime small enough for the FP64 element-wise kernels, and every one of their transforms
    // exact on FP64 butterflies (fp_ok), so that lazy doubles pass between the kernels of a multiply / key switch
    bool fp_elementwise = false;
    std::vector<NttTab> h_tabs;
    NttTab *d_tabs = nullptr;
    u64 *d_table_mem = nullptr;
    std::vector<u32> h_index_map;
    u32 *d_index_map = nullptr;
    DigitMap dm_relin, dm_galois;
    std::vector<u64> galois_elts;
    std::vector<Channel> ch;
    // Key slots: slot 0 is the channels' own keys, slot s >= 1 another client's evaluation keys, clients[s - 1][channel] (an empty entry
    // is a removed slot).  Every ciphertext is bound to one slot; a key switch takes each ciphertext's keys from its slot.
    std::vector<std::vector<KeySet>> clients;
    int slot = 0; // key slot of the ciphertexts the current public call works on (reset to 0 by every call; vec.cu sets it from the operands)
    bool foreign = false; // the current call touches ciphertexts of a slot other than 0: the noise trace cannot measure them (no secret key)
    bool slot_live(int s) const { return s == 0 || (s > 0 && (size_t)s <= clients.size() && !clients[s - 1].empty()); }
    u64 *d_sanitize_nonce = nullptr; // [P] device counters of the channels' sanitisation nonces (Channel::sanitized)
    const KeySet &keys(int channel, int s) const;
    // key generation of a slot: bumped whenever its keys are replaced or removed, so that a graph recorded against them refuses to launch
    std::map<int, uint64_t> key_gen;
    void keys_changed(int s) { key_gen[s]++; origin.erase(s); }

    // ---- levels (DESIGN 4.17).  A context made by context_derive holds the first k' of its parent's coefficient primes; every context
    // of one family shares `root`, the serial of the context created from parameters.  The keys of a slot are named by their origin:
    // (serial, key generation) of the context whose own keys they are, carried along when they are restricted into a derived context
    uint64_t serial = 0, root = 0;
    std::map<int, std::pair<uint64_t, uint64_t>> origin; // slots whose keys were restricted from another context of the family
    std::pair<uint64_t, uint64_t> key_origin(int s) const {
        const auto it = origin.find(s);
        if (it != origin.end()) return it->second;
        const auto g = key_gen.find(s);
        return {serial, g == key_gen.end() ? 0 : g->second};
    }

    // ---- graph recording (vec.cu, cnhe_capture_*).  `api`: the public call in progress, named in refusals
    std::unique_ptr<Recording> rec;
    const char *api = "";
    [[noreturn]] void refuse(const char *why) const; // CNHE_ERR_STATE: the call cannot be recorded
    // host -> device copy of `bytes` on `stream`.  While recording, the bytes are copied once into a constant block of the graph's memory
    // and the graph copies them from there on every launch (a host buffer may be gone by then, and pageable copies cannot be recorded)
    void upload(void *dst, const void *src, size_t bytes);
    // waits until the host buffers handed to upload / h2d have been read; while recording they were read at once, so nothing waits
    void host_fence() { if (!rec) sync(); }
    // one CUDA stream per plaintext-modulus channel (the reference runs one Task per prime, EncryptedSealBfvVector.cs:225-236):
    // channels are independent until decryption, so their kernels and host<->device copies overlap.  `stream` is the stream of the
    // channel currently being issued (set_channel).
    std::vector<cudaStream_t> streams;
    cudaStream_t stream = nullptr;
    bool multi_stream = true;
    void set_channel(int ch) { stream = streams[multi_stream ? ch : 0]; }
    void join_streams(); // stream 0 waits for the tail of every other stream
    void fork_streams(); // every other stream waits for the tail of stream 0
    // bulk ciphertext uploads (cnhe_vecs_import_raw) run on their own stream, fenced by events against the owning channel's stream:
    // the upload of the next batch overlaps the kernels of the current one (double buffering across API calls)
    cudaStream_t copy_stream = nullptr;
    // persistent device blocks for uploaded ciphertext batches: a slot is handed out again once the event recorded at its release (on
    // the consuming channel's stream) allows it -- no driver allocation in the steady state, and with three slots in rotation the
    // upload of batch i+1 never waits for batch i's kernels
    struct UploadSlot { u64 *p; size_t words; cudaEvent_t released; bool busy; uint64_t stamp; };
    std::vector<UploadSlot> upload_slots;
    uint64_t upload_stamp = 0;
    BufRef alloc_upload(size_t words, cudaStream_t release_stream); // the copy stream is made to wait for the slot's last release
    void release_upload(int slot, cudaStream_t s);
    cudaEvent_t ev_copy = nullptr;
    std::vector<cudaEvent_t> ev_export; // ring of 8 tickets x P channel events (cnhe_vecs_export_raw_async)
    int export_next = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_join = nullptr;
    std::recursive_mutex mu;
    std::vector<BufRef> temps; // workspace temporaries of the operation in flight (guarded by mu)
    // ---- operation counters (the reference's OperationsCount, "HE Wrapper/AtomicSealBfvVector.cs:211-294") and the optional
    // per-operation noise-budget trace (CryptoTracker.TestBudget, "HE Wrapper/CryptoTracker.cs:41-52")
    enum OpKind { OP_ENCRYPT, OP_DECRYPT, OP_MULTIPLY, OP_RELINEARIZE, OP_MULTIPLY_PLAIN, OP_MULTIPLY_SCALAR, OP_ADD, OP_ADD_PLAIN, OP_SUB,
                  OP_SUB_PLAIN, OP_ROTATE_ROWS_HOP, OP_ROTATE_COLUMNS, OP_ADD_MANY, OP_ADD_MANY_ITEMS, OP_COUNT };
    uint64_t op_count[OP_COUNT] = {0};
    bool trace_noise = false;
    struct TraceRec { int kind, channel, n, budget, in0, in1, aux_milli, reserved; };
    std::vector<TraceRec> trace;
    std::map<const u64 *, int> budget_of; // tracing only: last measured budget of the ciphertext at a device address
    // count `n` operations of `kind`; with tracing on, also record the invariant noise budget of the first output ciphertext next to the
    // budgets its first input ciphertexts had (so that every operation can be checked against the analytic noise model on its own) and
    // an operation-specific `aux` value (log2 of the scalar / of the root-sum-square weight of a MAC output)
    void note(OpKind kind, int channel, int n, const u64 *first_out = nullptr, const u64 *in0 = nullptr, const u64 *in1 = nullptr, double aux = 0);
    void note_copy(const u64 *dst, const u64 *src) { // a device-to-device copy of a ciphertext keeps its budget
        if (!trace_noise) return;
        auto it = budget_of.find(src);
        if (it != budget_of.end()) budget_of[dst] = it->second; else budget_of.erase(dst);
    }
    int known_budget(const u64 *p) const { auto it = budget_of.find(p); return it == budget_of.end() ? -1 : it->second; }
    // K_c of op_multiply_sum: the most tensor products whose sum the BEHZ floor still rounds exactly in this context's base Bsk (DESIGN 4.14)
    int sum_terms = 1;
    int chunk = 1024; // ciphertexts per kernel wave (upper bound: wave() also keeps a wave's scratch under ~8 GiB)
    int wave(size_t words_per_ct) const { // ciphertexts per wave for an operation needing `words_per_ct` scratch words per ciphertext
        const size_t fit = ((size_t)1 << 30) / (words_per_ct ? words_per_ct : 1); // 2^30 words = 8 GiB
        // with one stream per plaintext modulus the channels' kernels interleave on the GPU: 128-ciphertext waves keep that interleaving
        // fine grained (measured: 28.8 ms per pipelined batch against 35.2 ms with whole-layer waves); a single stream prefers one wave
        const size_t cap = multi_stream && streams.size() > 1 ? std::min(chunk, 128) : chunk;
        return (int)std::max<size_t>(16, std::min<size_t>(cap, fit));
    }
    uint64_t launches = 0;
    // optional per-kernel-family timing
    bool prof = false;
    struct ProfRec { int family; double bytes; cudaEvent_t e0, e1; };
    std::vector<ProfRec> prof_recs;
    std::vector<cudaEvent_t> prof_pool;
    static constexpr int PROF_FAMILIES = 7; // cnhe_prof_collect's families; 6: the sanitisation finish kernel
    double prof_ms[PROF_FAMILIES] = {0}, prof_bytes[PROF_FAMILIES] = {0};
    uint64_t prof_n[PROF_FAMILIES] = {0};
    void prof_begin(int family, double bytes);
    void prof_end();
    void prof_flush();
    size_t ws_used = 0; // words handed out as temporaries since the last release (diagnostic)
    // host CRT data of the wrapper ("HE Wrapper/EncryptedSealBfvVector.cs:79-90")
    unsigned __int128 big_factor = 0;
    std::vector<unsigned __int128> crt_coeff;

    // pinned staging ring for small host->device uploads (pointer tables, weights, tiles): truly asynchronous copies
    unsigned char *stage_buf = nullptr;
    size_t stage_size = 0, stage_off = 0;
    // the ring is cut into STAGE_PARTS parts; leaving a part records one event per channel stream, entering it waits for the events of
    // its previous use (several parts ago: already complete in the steady state) -- no device-wide sync when the ring wraps
    static constexpr int STAGE_PARTS = 8;
    std::vector<cudaEvent_t> stage_ev; // [part][stream]
    std::vector<char> stage_ev_set;
    void h2d(void *dst, const void *src, size_t bytes); // async on `stream`; `src` may be freed on return

    ~Context();
    size_t ct_words() const { return (size_t)2 * k * N; }
    u64 *ws_alloc(size_t words); // temporary of the current operation: released (stream ordered / recycled) by WsScope or the next API call
    BufRef alloc(size_t words) { return std::make_shared<DevBuf>(words, stream, this); }
    // Large blocks (layer slabs, the 1 GB digit waves) are recycled per stream: a block released on stream S is handed to the next
    // request of a similar size on S without a driver call -- stream order makes that safe, and it removes cudaMallocAsync's slow path
    // (measured: 120 ms for 1 GB when the pool has no fitting free block) from the steady state.
    struct Recycled { u64 *p; size_t words; cudaStream_t stream; };
    std::vector<Recycled> recycle;
    size_t recycle_words = 0;
    bool recycle_on = true;
    u64 *take_recycled(size_t words, cudaStream_t s, size_t &got_words);
    bool give_recycled(u64 *p, size_t words, cudaStream_t s);
    void drop_recycled();
    void launched(int n = 1) { launches += n; }
    void check(cudaError_t e, const char *what) { cuda_check(e, what); launched(); if (trace_ms > 0) trace_gap(what); }
    std::unordered_map<u64, std::shared_ptr<void>> umma_plans; // wgmma layer plans (vec.cu), keyed by a hash of the layer's weights and gather table
    double trace_ms = 0; // CNHE_TRACE_SLOW: report host-side gaps between consecutive launches longer than this
    void trace_gap(const char *what);
    void sync(); // waits for every channel stream; refused while recording
};
// ends the capture of a recording group (every member's lock held): every member's capturing streams join members[0]'s stream 0, whose
// capture ends; returns the captured graph (nullptr when the capture failed; keep: false destroys it)
cudaGraph_t end_capture(RecGroup &g, bool keep);
// ends c's part of its recording once the capture has ended, and restores its operation counters.  The buffers from before the recording
// that were released during it may still be read by the graph: they move to *hold (the graph releases them when it is destroyed), or are
// released at once when hold is nullptr (an aborted recording)
void end_part(Context &c, std::vector<Recording::Deferred> *hold = nullptr);
// aborts the recording c takes part in (c's lock held), for every member: at once when every member's lock can be taken without waiting,
// else by setting abort_requested (another thread is inside a call on a member; a capture must not end under a call that issues into it)
void abort_recording(Context &c);
void release_deferred(Context &c, const std::vector<Recording::Deferred> &d); // as their DevBufs would have released them

void ws_release_all(Context &c); // drop every workspace temporary (call at the start of a public operation)
struct WsScope {                  // temporaries allocated inside the scope are released when it ends
    Context &c;
    size_t mark;
    explicit WsScope(Context &ctx);
    ~WsScope();
};

Context *context_create(const u64 *plain_primes, int P, uint32_t N, const u64 *coeff, int k, int dbc_relin, int dbc_galois, int device);
// A context on the first k of parent's coefficient primes (1 <= k < parent.k), created as context_create creates one on them, that starts
// with the parent's options and the restriction of every key slot's keys (restrict_keys)
Context *context_derive(Context &parent, int k);
// Makes slot s of dst (fewer primes, same family) hold the restriction of src's slot s keys: the secret key and each key-switching key
// cut to its rows and digits of residues < dst.k, the public key to its rows; a slot src does not hold is emptied.  Returns once the copies
// and the packed relinearisation keys are complete.
void restrict_keys(Context &dst, const Context &src, int s);
// out [n][2][dst.k][N] (dst's memory) = the n ciphertexts in[c] of src ([2][src.k][N], coefficient form) with primes src.k-1 .. dst.k
// dropped (launch_mod_switch), on dst's stream `ch`: that stream first waits for src's stream `ch`, and src's stream waits for the kernel
void op_mod_switch(Context &src, Context &dst, int ch, const std::vector<const u64 *> &in, u64 *out);
std::vector<u64> default_coeff_modulus(uint32_t N);

// ---- keys
void keys_generate(Context &c, u64 seed); // deterministic sampler: tests only
void keys_generate_secure(Context &c);    // fresh OS entropy per channel
void rng_from_os(RngKey &rk);
const char *op_kind_name(int kind);
BufRef &key_slot(Context &c, int channel, int what, u64 arg, size_t &words, bool create);
// marks a channel's relinearisation keys present once they are written to its rlk slot (generated or loaded), and rebuilds the packed
// copy the fused key switch reads; returns once that copy is complete
void rlk_ready(Context &c, int channel);
void rlk_ready(Context &c, KeySet &ks); // the same for a key slot's key set

// ---- ciphertext-array operations (all asynchronous on c.stream; device pointers)
// upload a host array of device pointers into workspace memory
const u64 *const *upload_ptrs(Context &c, const std::vector<const u64 *> &ptrs);
u64 *const *upload_ptrs_mut(Context &c, const std::vector<u64 *> &ptrs);

void op_ntt(Context &c, const u64 *src, u64 *dst, int n_polys, int mod_base, int mod_count, bool inverse);
// out3[n][3][k][N] = a[i] * b[i]  (BEHZ).  a_ptrs/b_ptrs: host vectors of device ciphertext pointers.
// epi (squares only): nullptr, or op_multiply_relin's floor epilogue applied to the size-3 products, A (.) a^2 + (B x0 + Delta C, B x1, 0)
void op_multiply(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, u64 *out3, const FloorEpi *epi = nullptr);
// Key-switching operations take the keys of ciphertext i from key slot slots[i] when a per-ciphertext slot table is given (n entries,
// host), otherwise every ciphertext uses the call's slot c.slot.  A missing key is CNHE_ERR_STATE.
// book: count the relinearisations (false: the caller booked them, as a deferred square does when it is made)
void op_relinearize(Context &c, int ch, const u64 *in3, int n, u64 *out2, const int *slots = nullptr, bool book = true);
// epi (squares only, a[i] == b[i]): nullptr, or the quadratic activation out2 = relin(A a^2) + B x + Delta C (floor_epi) applied in the
// BEHZ floor kernel.  x: epi->x, a device table of one input per output of the call (cnhe_layer_poly's second level: the activation's
// original input), or nullptr for the squared operand itself; c_poly, when set, has one entry per output of the call.
// pair (with epi): a holds 2n operands and output i is relin(A (a[2i]^2 - a[2i+1]^2)) + B x[i] + Delta C -- 2n squares, one floor and one
// key switch per output (the cubic activation's second level); slots then has n entries
// Relinearisation whose key-switch digits arrive as int32 planes (DESIGN 4.15): out2[i] = base_i + sum_d planes_i[d] * rlk_d, base and
// out2 packed [n][2][k][N], planes [n][D][N] with |value| < min q_l; slots as in op_relinearize.  Counts nothing (the caller booked the
// relinearisations).  relin_planes_built: whether the context has the fused key switch this needs.
bool relin_planes_built(const Context &c);
void op_relinearize_planes(Context &c, int ch, const int *planes, int n, const u64 *base, u64 *out2, const int *slots);
void op_multiply_relin(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, u64 *out2,
                       const int *slots = nullptr, const FloorEpi *epi = nullptr, bool pair = false);
// Sums of products with one floor per chunk and one relinearisation per output (DESIGN 4.14): out2[o] = relinearize(sum over the chunks of
// floor(sum_{j in chunk} a[o T + j] (x) b[j])), the chunks T terms split into runs of at most c.sum_terms in index order, their floors added
// mod q.  a: n_out * T ciphertexts (output o's terms at o T + j), b: T ciphertexts shared by every output.  Each ciphertext is lifted and
// transformed once.  Counted as n_out T multiplications, n_out (T - 1) additions and n_out relinearisations.  CNHE_ERR_INVALID when a
// chunk and one output's operands need more than 8 GiB of scratch (multiply_sum_wave == 0); slots as in op_relinearize (n_out entries)
void op_multiply_sum(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, int T, int n_out, u64 *out2,
                     const int *slots = nullptr);
// outputs per wave of op_multiply_sum next to a chunk of T terms, or 0 when not even one fits under the 8 GiB scratch cap
int multiply_sum_wave(const Context &c, int T);
// the FloorEpi constants of A, B, C (residues mod the channel's t): A and B lifted into every q_l as multiply_plain lifts a constant
// plaintext, C scaled as add_plain scales it
FloorEpi floor_epi(const Context &c, int ch, u64 A, u64 B, u64 C);
// the keys of a key switch: one set for every ciphertext, or one per ciphertext (several key slots in one call)
struct KsKeys {
    const u64 *key = nullptr, *packed = nullptr; // uniform call; packed: the 48-bit copy for the fused kernel (nullptr: u64 keys)
    std::vector<const u64 *> keys, packs;        // per ciphertext (empty: uniform); packs empty when some key has no packed copy
    // Key bases, also while recording: op_key_switch and op_relinearize_planes turn the ones they pass into key references (KeyBinding)
    bool per_ct() const { return !keys.empty(); }
    KsKeys slice(int c0, int m) const;
};
KsKeys relin_keys(Context &c, int ch, int n, const int *slots);
KsKeys galois_keys(Context &c, int ch, int n, const int *slots, u64 elt);
void op_key_switch(Context &c, const u64 *target, size_t target_stride, int n, const KsKeys &keys, const DigitMap &dm, const u64 *base,
                   size_t base_stride, u64 *out);
void op_apply_galois(Context &c, int ch, const u64 *in, int n, u64 elt, u64 *out, bool add_back = false, const int *slots = nullptr);
// out = in + rotate(in) in one pass, if possible
bool op_rotate_add(Context &c, int ch, const u64 *in, int n, int steps, bool columns, u64 *out, const int *slots = nullptr);
void op_rotate_rows(Context &c, int ch, const u64 *in, int n, int steps, u64 *out, const int *slots = nullptr); // steps == 0 copies
void op_rotate_columns(Context &c, int ch, const u64 *in, int n, u64 *out, const int *slots = nullptr);
// Many independent single-ciphertext row rotations with DIFFERENT step counts (Interleave / Stack / Duplicate rotate every vector by its
// own offset): each job walks the hop sequence rotate_rows would take for it (exact key or NAF hops), and hops with the same Galois
// element are batched across jobs into one key-switch wave.  Per ciphertext the operations and their order are exactly those of
// op_rotate_rows, so the outputs are bit-identical.  slot < 0: the call's slot.  A step takes its exact key only when every job's slot
// holds it (the hops are planned from the elements the call's slots have in common).
struct RotateJob { const u64 *src; int steps; u64 *dst; int slot = -1; };
void op_rotate_rows_multi(Context &c, int ch, const std::vector<RotateJob> &jobs);
u64 galois_elt_from_step(const Context &c, int steps);
// the hops of a row rotation by `steps` whose Galois key is missing (Evaluator::rotate_internal): the NAF terms of steps, least significant
// first, without a term of +-N/2, which maps each row of N/2 slots onto itself
std::vector<int> naf_hops(uint32_t N, int steps);
// dense plaintext (coefficient form mod t, [n or 1][N]) times ciphertexts [n][2kN]
void op_multiply_plain_dense(Context &c, int ch, const u64 *ct, int n, const u64 *plain, bool plain_per_ct, u64 *out);
void op_multiply_plain_dense_bcast(Context &c, int ch, const u64 *ct, const u64 *plains, int n, u64 *out);
// B ciphertexts times R dense plaintexts (contiguous [R][N]): out [B][R][2kN], out[b * R + r] = cts[b] * plains[r], word for word what
// op_multiply_plain_dense_bcast(cts[b], plains, R) writes; counted as B * R plain multiplications
void op_multiply_plain_dense_outer(Context &c, int ch, const std::vector<const u64 *> &cts, const u64 *plains, int R, u64 *out);
// values [n][count] (mod t, device) -> plain [n][N] coefficient form
void op_encode(Context &c, int ch, const u64 *values, int n, int count, u64 *plain);
void op_decode(Context &c, int ch, const u64 *plain, int n, u64 *values);
// plain[i] = BatchEncoder.Encode(e_(first_col + i)) for i < n, built on the device (the one-hot masks of ForceOutputInColumn)
void op_encode_onehot(Context &c, int ch, int n, int first_col, u64 *plain);
// plain [n][plain_stride] (first `coeffs` coefficients used) -> ct [n][2kN]; nonces nonce0..nonce0+n-1
// reserve n consecutive encryption nonces of a channel (a secure channel re-keys from the OS before the 32-bit counter wraps)
u64 take_nonces(Context &c, int ch, u64 n);
void op_encrypt(Context &c, int ch, const u64 *plain, size_t plain_stride, int n, int coeffs, u64 nonce0, u64 *ct);
void op_decrypt(Context &c, int ch, const u64 *ct, int n, u64 *plain);
// plain [n][N] = decryptions of the ciphertexts at cts[i] (any addresses), one wave of kernels per c.wave(3kN) ciphertexts
void op_decrypt_many(Context &c, int ch, const std::vector<const u64 *> &cts, u64 *plain);
// values [n][dim] doubles (device) -> plain: dense [n][bl][N] coefficient form (bl = ceil(dim / N), the split fused into the encode scatter,
// a short last block zero padded); sparse (n = 1) [dim] residues.  Out-of-range values set *bad (DESIGN 4.19)
void op_encode_values(Context &c, int ch, const double *values, int n, uint64_t dim, double scale, bool dense, u64 *plain, int *bad);
// ---- compact ciphertext upload (format: compact.cu)
CompactShape compact_shape(const Context &c); // bit lengths of the q_l and the packed word offsets of one ciphertext
// expansion key K_c of one blob: a fresh OS draw on a secure channel; four words of the seeded sampler on a test channel (reproducible)
CompactKey compact_key(Context &c, int ch, u64 nonce0);
// seeded secret-key encryption of plain [n][N] (coefficient form) under nonces nonce0.. and key K_c -> packed c0 [n][off[k]] (device)
void op_encrypt_compact(Context &c, int ch, const u64 *plain, int n, u64 nonce0, const CompactKey &key, u64 *packed);
// packed [n][off[k]] + K_c -> ct [n][2kN] on stream s (timed as family 5 when profiling)
void op_compact_expand(Context &c, const u64 *packed, const CompactKey &key, int n, u64 *ct, cudaStream_t s);
// ---- compact key sets (format: compact.cu).  sets: bit 0 public key, bit 1 relinearisation keys; elts: Galois elements in blob order
std::vector<u64> standard_galois_elts(uint32_t N); // KeyGenerator::galois_keys(dbc)'s elements, in the context's order
size_t compact_key_pairs(const Context &c, int sets, size_t n_galois);
// a fresh key set under the channel's secret key (its own keys are untouched): pair kappa's a expanded from K_c, e under nonce0 + kappa
// -> packed b [pairs][off[k]] (device)
void op_keys_save_compact(Context &c, int ch, int sets, const std::vector<u64> &elts, u64 nonce0, const CompactKey &key, u64 *packed);
// packed b [pairs][off[k]] (device) + K_c -> the channel's key slots; returns once the keys are complete
void op_keys_load_compact(Context &c, int ch, int sets, const std::vector<u64> &elts, const u64 *packed, const CompactKey &key);
// the same into a key slot's key set (relinearisation and Galois keys; a public key pair in the blob is skipped)
void op_keys_load_compact(Context &c, KeySet &dst, int sets, const std::vector<u64> &elts, const u64 *packed, const CompactKey &key);
int op_noise_budget(Context &c, int ch, const u64 *ct);
// ---- sanitisation (circuit privacy, DESIGN 4.18; kernels in sanitize.cu)
// the widest flood the context allows: floor(log2(q / t)) - 2 for the smallest such value over its plaintext moduli
int sanitize_max_bits(const Context &c);
// takes n sanitisation nonces of a channel on the host's count: CNHE_ERR_STATE when the count would pass SANITIZE_NONCES
void sanitize_reserve(Context &c, int ch, u64 n);
// out[i] = in[i] + (pk0 u + e0 + f, pk1 u + e1) under the public key of key slot slots[i] (n entries); u ternary, e0, e1 clipped normal,
// f uniform in [-2^b, 2^b), drawn under the nonces the device counter hands out; out packed [n][2][k][N], coefficient form.  Counted as n
// encryptions and n additions.  A slot without a public key is CNHE_ERR_STATE (-3)
void op_sanitize(Context &c, int ch, const std::vector<const u64 *> &in, const int *slots, int flood_bits, u64 *out);

} // namespace cnhe
