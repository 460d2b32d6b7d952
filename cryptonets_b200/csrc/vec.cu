// C ABI of libcnhe (include/cnhe.h) and the vector layer behind it.
//
// One cnhe_vec is the reference's EncryptedSealBfvVector ("HE Wrapper/EncryptedSealBfvVector.cs:150-573"): P channels,
// one per plaintext modulus, each carrying what AtomicSealBfvEncryptedVector ("HE Wrapper/AtomicSealBfvVector.cs:303-326")
// keeps in `Ciphertext[] encData` / `Plaintext[] plainData` -- here blocks of HBM.  The functions below restate that
// class method by method (cited inline); the arithmetic itself is in the CUDA kernels.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdlib>
#include <climits>
#include <cstring>
#include <optional>
#include <set>
#include <unordered_map>

#include "hostmath.h"
#include "vec.h"

typedef unsigned __int128 u128;

static thread_local std::string g_err;
int set_err(int code, const std::string &m) {
    g_err = m;
    return code;
}
extern "C" const char *cnhe_last_error(void) { return g_err.c_str(); }
void api_enter(Context &c, const char *name) {
    c.api = name;
    if (!c.rec) return;
    if (c.rec->thread != std::this_thread::get_id()) c.refuse("was called from another thread than the recording one");
    if (c.rec->group->abort_requested) abort_recording(c); // a call refused on another thread while this one was inside a call
}
int api_fail(Context &c, int code, const std::string &m) {
    std::lock_guard<std::recursive_mutex> lock(c.mu);
    if (c.rec) abort_recording(c);
    return set_err(code, m);
}
extern "C" const char *cnhe_version(void) { return "cnhe-b200 0.3 (sm_90a)"; }

// ---------------------------------------------------------------------------------------------------- context & keys
extern "C" int cnhe_context_create_custom(const uint64_t *plain_primes, int P, uint32_t N, const uint64_t *coeff, int k, int dbc_relin,
                                          int dbc_galois, int device, cnhe_ctx **out) {
    try {
        if (!plain_primes || !coeff || !out) fail("null argument");
        std::vector<u64> pp(plain_primes, plain_primes + P), cc(coeff, coeff + k);
        Context *c = context_create(pp.data(), P, N, cc.data(), k, dbc_relin, dbc_galois, device);
        *out = new cnhe_ctx{c};
    } catch (const Error &e) { return set_err(e.code, e.what()); } catch (const std::exception &e) { return set_err(CNHE_ERR_INVALID, e.what()); }
    return CNHE_OK;
}
extern "C" int cnhe_context_create(const uint64_t *plain_primes, int P, uint32_t N, int dbc_relin, int dbc_galois, int small_modulus_count,
                                   int device, cnhe_ctx **out) {
    std::vector<u64> q = default_coeff_modulus(N);
    if (q.empty()) return set_err(CNHE_ERR_INVALID, "no default coefficient modulus for this PolyModulusDegree");
    if (small_modulus_count > 0 && small_modulus_count < (int)q.size()) q.resize(small_modulus_count); // AtomicSealBfvVector.cs:148-149
    std::vector<uint64_t> qq(q.begin(), q.end());
    return cnhe_context_create_custom(plain_primes, P, N, qq.data(), (int)qq.size(), dbc_relin, dbc_galois, device, out);
}
extern "C" int cnhe_context_destroy(cnhe_ctx *h) {
    if (!h) return CNHE_OK;
    delete h->c;
    delete h;
    return CNHE_OK;
}
extern "C" int cnhe_context_info(const cnhe_ctx *h, uint32_t *N, int *k, int *P, int *relin_digits, int *galois_digits, int *galois_elts) {
    if (!h) return set_err(CNHE_ERR_INVALID, "null context");
    const Context &c = *h->c;
    if (N) *N = c.N;
    if (k) *k = c.k;
    if (P) *P = c.P;
    if (relin_digits) *relin_digits = c.dm_relin.D;
    if (galois_digits) *galois_digits = c.dm_galois.D;
    if (galois_elts) *galois_elts = (int)c.galois_elts.size();
    return CNHE_OK;
}
extern "C" int cnhe_context_coeff_moduli(const cnhe_ctx *h, uint64_t *out) {
    if (!h || !out) return set_err(CNHE_ERR_INVALID, "null argument");
    for (int i = 0; i < h->c->k; i++) out[i] = h->c->q[i];
    return CNHE_OK;
}
extern "C" int cnhe_context_bsk_moduli(const cnhe_ctx *h, uint64_t *out, int *count) {
    if (!h || !count) return set_err(CNHE_ERR_INVALID, "null argument");
    *count = h->c->kb;
    if (out)
        for (int i = 0; i < h->c->kb; i++) out[i] = h->c->bsk[i];
    return CNHE_OK;
}
extern "C" int cnhe_context_plain_moduli(const cnhe_ctx *h, uint64_t *out) {
    if (!h || !out) return set_err(CNHE_ERR_INVALID, "null argument");
    for (int i = 0; i < h->c->P; i++) out[i] = h->c->t[i];
    return CNHE_OK;
}
extern "C" int cnhe_context_galois_elts(const cnhe_ctx *h, uint64_t *out) {
    if (!h || !out) return set_err(CNHE_ERR_INVALID, "null argument");
    for (size_t i = 0; i < h->c->galois_elts.size(); i++) out[i] = h->c->galois_elts[i];
    return CNHE_OK;
}
extern "C" int cnhe_context_set_option(cnhe_ctx *h, const char *name, int64_t value) {
    API_BEGIN(h)
    not_recorded(c, "changes the context's options");
    std::string n(name ? name : "");
    if (n == "behz_centered_mtilde") {
        c.h_bc.centered_mtilde = value ? 1 : 0;
        c.h_bf.centered_mtilde = value ? 1 : 0;
        CNHE_CUDA(cudaMemcpyAsync(c.d_bc, &c.h_bc, sizeof(BehzConst), cudaMemcpyHostToDevice, c.stream));
        CNHE_CUDA(cudaMemcpyAsync(c.d_bf, &c.h_bf, sizeof(BehzConstF), cudaMemcpyHostToDevice, c.stream));
        c.sync();
    } else if (n == "multi_stream") {
        // buffers remember the stream they are released on: switching the stream mode with work or uploads in flight would let the
        // recycler hand a block out while another stream still reads it.  Quiesce, drop the per-stream free lists, then switch.
        for (const Context::UploadSlot &u : c.upload_slots)
            if (u.busy) fail("multi_stream cannot change while imported batches are alive (dispose them first)");
        c.sync();
        CNHE_CUDA(cudaStreamSynchronize(c.copy_stream));
        c.drop_recycled();
        c.multi_stream = value != 0;
    } else if (n == "trace_noise") {
        c.trace_noise = value != 0;
        c.trace.clear();
        if (!c.trace_noise) c.budget_of.clear();
    } else if (n == "release_cached_memory") {
        // give the device memory this context keeps for reuse (parked scratch blocks, the stream-ordered pool's freed blocks) back to the
        // driver, e.g. before preparing a large resident matrix; buffers in use are untouched
        c.sync();
        CNHE_CUDA(cudaStreamSynchronize(c.copy_stream));
        c.drop_recycled();
        CNHE_CUDA(cudaDeviceSynchronize());
        cudaMemPool_t pool;
        CNHE_CUDA(cudaDeviceGetDefaultMemPool(&pool, c.device));
        CNHE_CUDA(cudaMemPoolTrimTo(pool, 0));
    } else if (n == "chunk") {
        if (value < 1 || value > 4096) fail("chunk must be in [1,4096]");
        c.chunk = (int)value;
    } else fail("unknown option");
    API_END
}
// Interop with the caller's own GPU work (NCCL collectives, torch copies): the CUDA stream of a plaintext-modulus channel, and the two
// fences of the per-channel streams -- join: stream 0 waits for the tail of every channel; fork: every channel waits for stream 0.
// A caller that enqueues on stream 0 between a join and a fork is ordered after everything queued so far and before everything queued later.
extern "C" int cnhe_context_stream(cnhe_ctx *h, int channel, uint64_t *stream) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P || !stream) fail("bad arguments");
    *stream = (uint64_t)c.streams[c.multi_stream ? channel : 0];
    API_END
}
extern "C" int cnhe_context_join_streams(cnhe_ctx *h) {
    API_BEGIN(h)
    c.join_streams();
    API_END
}
extern "C" int cnhe_context_fork_streams(cnhe_ctx *h) {
    API_BEGIN(h)
    c.fork_streams();
    API_END
}
extern "C" int cnhe_context_sync(cnhe_ctx *h) {
    API_BEGIN(h)
    c.sync();
    API_END
}
extern "C" uint64_t cnhe_kernel_launch_count(const cnhe_ctx *h) { return h ? h->c->launches : 0; }

// ---------------------------------------------------------------------------------------------------- graph recording and replay
// The context's calls are captured from its channel streams into one CUDA graph (stream capture, relaxed mode: the record-time copies of
// host constants and the allocations of the graph's memory happen outside the captured streams).  Channel streams fork from stream 0 when
// the recording begins and join it before it ends, as fork_streams / join_streams order them for eager calls.  A recording that enlists
// levels (cnhe_capture_begin_levels) forks every channel stream of every level from the same stream 0, so the mod switches' event
// hand-offs between the contexts' streams are captured like any other cross-stream order.
struct cnhe_graph {
    cnhe_ctx *h = nullptr;
    std::vector<Context *> members; // the contexts the recording spanned: members[0] is h's, the rest its enlisted levels (lock order)
    cudaGraphExec_t exec = nullptr;
    std::shared_ptr<GraphArena> arena;
    std::vector<std::vector<uint64_t>> ops; // per member: the operation counts one launch adds
    std::vector<uint64_t> launches;         // per member: the kernel launches one launch adds (what the recorded calls counted)
    uint64_t kernel_nodes = 0;
    // key binding (cnhe_graph_bind): the key positions (recorded slots, ascending), the slot each is bound to and, per member, that slot's
    // key generation when it was bound, and the words of the device table under that binding
    std::shared_ptr<KeyBinding> keys;
    std::vector<int> positions, bound;
    std::vector<std::vector<uint64_t>> bound_gen;
    std::vector<const u64 *> words;
    bool words_sent = false; // the device table holds `words` (or will, once the copy queued by the last launch has run)
    std::vector<std::shared_ptr<void>> keep;
    std::vector<std::vector<Recording::Deferred>> held; // per member: buffers from before the recording, released during it (the graph may read them)
};
static uint64_t key_gen(const Context &c, int s) {
    const auto it = c.key_gen.find(s);
    return it == c.key_gen.end() ? 0 : it->second;
}
typedef std::vector<std::unique_lock<std::recursive_mutex>> Locks;
// the locks of members[1..] (the caller holds members[0]'s), taken in member order
static Locks lock_members(const std::vector<Context *> &members) {
    Locks l;
    for (size_t i = 1; i < members.size(); i++) l.emplace_back(members[i]->mu);
    return l;
}
// a graph call on the levels a graph spans: each is locked and entered like a public call; while one records, the call is refused and
// that recording aborted, as a refused call on the graph's own context aborts its recording
static Locks enter_levels(cnhe_graph &g, const char *name, const char *why) {
    Locks l = lock_members(g.members);
    for (size_t i = 1; i < g.members.size(); i++) {
        Context &m = *g.members[i];
        m.api = name;
        if (m.rec) {
            abort_recording(m);
            throw Error(CNHE_ERR_STATE, std::string(name) + " " + why + ": refused while a level the graph spans records a graph (the recording was aborted)");
        }
        m.set_channel(0);
        m.slot = 0;
        ws_release_all(m);
    }
    return l;
}
// Binds key position i of g to slots[i]: checks that every slot is live, restricts into each level a slot whose keys there are not the
// graph's context's (as the eager switch would), checks that every slot holds every key its position's references stand for in the
// recorded form, in the context that read it, then (and only then) takes the binding.  The device table is rewritten by the next launch.
static void bind_graph(cnhe_graph &g, const int *slots) {
    Context &top = *g.members[0];
    const size_t np = g.positions.size();
    for (size_t i = 0; i < np; i++)
        if (!top.slot_live(slots[i])) fail(("cnhe_graph_bind: no such key slot " + std::to_string(slots[i])).c_str());
    for (size_t mi = 1; mi < g.members.size(); mi++)
        for (size_t i = 0; i < np; i++)
            if (g.members[mi]->key_origin(slots[i]) != top.key_origin(slots[i])) restrict_keys(*g.members[mi], top, slots[i]);
    std::vector<const u64 *> words;
    for (const KeyBinding::Key &k : g.keys->words) {
        const int s = slots[std::lower_bound(g.positions.begin(), g.positions.end(), k.slot) - g.positions.begin()];
        const Context &m = *g.members[k.member];
        const KeySet &ks = m.keys(k.channel, s);
        auto missing = [&](const std::string &what) {
            throw Error(CNHE_ERR_STATE, "cnhe_graph_bind: key slot " + std::to_string(s) + " (plaintext channel " + std::to_string(k.channel) +
                                            (k.member ? ", level of " + std::to_string(m.k) + " primes" : std::string()) + ") holds no " + what +
                                            ", which the graph reads");
        };
        if (k.kind == KeyBinding::GALOIS) {
            const auto it = ks.glk.find(k.elt);
            if (it == ks.glk.end()) missing("Galois key of element " + std::to_string(k.elt));
            words.push_back(it->second->p);
        } else if (!ks.have_rlk || (k.kind == KeyBinding::RLK_PACKED && !ks.rlk_packed)) {
            missing(k.kind == KeyBinding::RLK ? "relinearization keys" : "packed relinearization keys");
        } else words.push_back(k.kind == KeyBinding::RLK ? ks.rlk->p : ks.rlk_packed->p);
    }
    g.bound.assign(slots, slots + np);
    g.bound_gen.assign(g.members.size(), {});
    for (size_t mi = 0; mi < g.members.size(); mi++)
        for (size_t i = 0; i < np; i++) g.bound_gen[mi].push_back(key_gen(*g.members[mi], slots[i]));
    for (size_t i = 0; i < np; i++) g.keys->to[g.positions[i]] = slots[i];
    if (words != g.words) {
        g.words = std::move(words);
        g.words_sent = false;
    }
}
// starts a recording on members[0] that enlists the rest (every member locked, none recording)
static void start_recording(const std::vector<Context *> &members) {
    Context &c = *members[0];
    for (Context *m : members) {
        if (m->prof) fail("cnhe_capture_begin: profiling is on (cnhe_prof_enable)");
        if (m->trace_noise) fail("cnhe_capture_begin: the noise trace is on (option trace_noise)");
    }
    auto grp = std::make_shared<RecGroup>();
    grp->members = members;
    auto arena = std::make_shared<GraphArena>();
    // the key binding's device table: one word for every key the members' slots hold (a recording reads each at most once)
    auto keys = std::make_shared<KeyBinding>();
    for (Context *m : members)
        for (int s = 0; s <= (int)m->clients.size(); s++)
            if (m->slot_live(s))
                for (int ch = 0; ch < m->P; ch++) keys->cap += 2 + m->keys(ch, s).glk.size();
    const std::vector<const u64 *> zeros(keys->cap);
    keys->table = static_cast<const u64 **>(const_cast<void *>(arena->constant(zeros.data(), zeros.size() * sizeof(u64 *), c.copy_stream)));
    CNHE_CUDA(cudaStreamBeginCapture(c.streams[0], cudaStreamCaptureModeRelaxed));
    for (size_t i = 0; i < members.size(); i++) {
        Context &m = *members[i];
        auto r = std::make_unique<Recording>();
        r->thread = std::this_thread::get_id();
        r->group = grp;
        r->member = (int)i;
        r->arena = arena;
        r->op0.assign(m.op_count, m.op_count + Context::OP_COUNT);
        r->launches0 = m.launches;
        r->keys = keys;
        m.rec = std::move(r);
    }
    // every channel stream of every member joins the capture before any call: a stream left out would run its work once, now
    CNHE_CUDA(cudaEventRecord(c.ev_join, c.streams[0]));
    for (Context *m : members)
        for (cudaStream_t s : m->streams)
            if (s != c.streams[0]) CNHE_CUDA(cudaStreamWaitEvent(s, c.ev_join, 0));
}
extern "C" int cnhe_capture_begin(cnhe_ctx *h) {
    API_BEGIN(h)
    if (c.rec) c.refuse("cannot start a second recording");
    start_recording({&c});
    API_END
}
extern "C" int cnhe_capture_begin_levels(cnhe_ctx *h, cnhe_ctx *const *levels, int n) {
    API_BEGIN(h)
    if (n < 0 || (n > 0 && !levels)) fail("cnhe_capture_begin_levels: null argument");
    std::vector<Context *> members{&c};
    for (int i = 0; i < n; i++) {
        if (!levels[i]) fail("cnhe_capture_begin_levels: null level");
        Context *m = levels[i]->c;
        if (m == &c) fail("cnhe_capture_begin_levels: the recording context cannot enlist itself");
        if (std::find(members.begin(), members.end(), m) != members.end()) fail("cnhe_capture_begin_levels: a level is listed twice");
        if (m->root != c.root) fail("cnhe_capture_begin_levels: a level of another context family");
        if (m->k >= c.k) fail("cnhe_capture_begin_levels: a level needs fewer coefficient primes than the recording context");
        members.push_back(m);
    }
    // lock order: more primes first, as cnhe_vecs_mod_switch takes them (ties by address)
    std::sort(members.begin() + 1, members.end(), [](const Context *a, const Context *b) { return a->k != b->k ? a->k > b->k : a < b; });
    const Locks locks = lock_members(members);
    if (c.rec) c.refuse("cannot start a second recording");
    for (size_t i = 1; i < members.size(); i++)
        if (members[i]->rec) throw Error(CNHE_ERR_STATE, "cnhe_capture_begin_levels: an enlisted level already records a graph");
    start_recording(members);
    API_END
}
extern "C" int cnhe_capture_abort(cnhe_ctx *h) {
    API_BEGIN(h)
    if (c.rec) abort_recording(c);
    API_END
}
extern "C" int cnhe_capture_end(cnhe_ctx *h, cnhe_graph **out) {
    API_BEGIN(h)
    if (!c.rec) throw Error(CNHE_ERR_STATE, "cnhe_capture_end: the context is not recording (was the recording aborted by a refused call?)");
    if (c.rec->member != 0) c.refuse("ends a recording that began on another context (end it there)");
    if (!out) fail("null argument");
    const std::shared_ptr<RecGroup> grp = c.rec->group;
    const Locks locks = lock_members(grp->members);
    if (grp->abort_requested) {
        abort_recording(c);
        throw Error(CNHE_ERR_STATE, "cnhe_capture_end: the recording was aborted by a call refused on another thread");
    }
    std::unique_ptr<cnhe_graph> g(new cnhe_graph);
    g->h = h;
    g->members = grp->members;
    g->arena = c.rec->arena;
    g->keys = c.rec->keys;
    for (Context *m : g->members) {
        g->keep.insert(g->keep.end(), m->rec->keep.begin(), m->rec->keep.end());
        std::vector<uint64_t> ops;
        for (int i = 0; i < Context::OP_COUNT; i++) ops.push_back(m->op_count[i] - m->rec->op0[i]);
        g->ops.push_back(std::move(ops));
        g->launches.push_back(m->launches - m->rec->launches0);
    }
    cudaGraph_t graph = end_capture(*grp, true);
    g->held.resize(g->members.size());
    for (size_t i = 0; i < g->members.size(); i++) end_part(*g->members[i], &g->held[i]);
    auto release_held = [&] {
        for (size_t i = 0; i < g->members.size(); i++) release_deferred(*g->members[i], g->held[i]);
    };
    if (!graph) {
        release_held();
        throw Error(CNHE_ERR_CUDA, "cnhe_capture_end: the CUDA stream capture failed");
    }
    size_t n = 0;
    cudaError_t e = cudaGraphGetNodes(graph, nullptr, &n);
    std::vector<cudaGraphNode_t> nodes(n);
    if (e == cudaSuccess && n) e = cudaGraphGetNodes(graph, nodes.data(), &n);
    for (size_t i = 0; i < n && e == cudaSuccess; i++) {
        cudaGraphNodeType t;
        e = cudaGraphNodeGetType(nodes[i], &t);
        g->kernel_nodes += e == cudaSuccess && t == cudaGraphNodeTypeKernel;
    }
    if (e == cudaSuccess) e = cudaGraphInstantiate(&g->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) release_held();
    CNHE_CUDA(e);
    // the recording is the first binding: every position bound to itself
    g->keys->seen.clear();
    g->keys->word.clear();
    std::set<int> pos;
    for (const KeyBinding::Key &k : g->keys->words) pos.insert(k.slot);
    g->positions.assign(pos.begin(), pos.end());
    bind_graph(*g, g->positions.data());
    *out = g.release();
    API_END
}
extern "C" int cnhe_graph_slots(const cnhe_graph *g, int *slots, int cap, int *n) {
    if (!g || !n) return set_err(CNHE_ERR_INVALID, "null argument");
    *n = (int)g->positions.size();
    if (slots)
        for (int i = 0; i < *n && i < cap; i++) slots[i] = g->positions[i];
    return CNHE_OK;
}
extern "C" int cnhe_graph_bind(cnhe_graph *g, const int *slots, int n) {
    if (!g) return set_err(CNHE_ERR_INVALID, "null graph");
    API_BEGIN(g->h)
    not_recorded(c, "binds a recorded graph to key slots");
    const Locks locks = enter_levels(*g, "cnhe_graph_bind", "binds a recorded graph to key slots");
    if (n != (int)g->positions.size() || (n > 0 && !slots))
        fail(("cnhe_graph_bind: the graph has " + std::to_string(g->positions.size()) + " key positions (cnhe_graph_slots), " +
              std::to_string(n) + " slots were given").c_str());
    bind_graph(*g, slots);
    API_END
}
extern "C" int cnhe_graph_launch(cnhe_graph *g) {
    if (!g) return set_err(CNHE_ERR_INVALID, "null graph");
    API_BEGIN(g->h)
    not_recorded(c, "launches a recorded graph");
    const Locks locks = enter_levels(*g, "cnhe_graph_launch", "launches a recorded graph");
    for (size_t mi = 0; mi < g->members.size(); mi++) {
        const Context &m = *g->members[mi];
        for (size_t i = 0; i < g->bound.size(); i++) {
            const int s = g->bound[i];
            if (!m.slot_live(s) || key_gen(m, s) != g->bound_gen[mi][i])
                throw Error(CNHE_ERR_STATE, "cnhe_graph_launch: the keys of key slot " + std::to_string(s) +
                                                (mi ? " in the level of " + std::to_string(m.k) + " primes" : std::string()) +
                                                " were removed or replaced after the graph was recorded or bound to it (cnhe_graph_bind)");
        }
    }
    // after every call queued before, on any channel of any context the graph spans
    c.join_streams();
    for (size_t mi = 1; mi < g->members.size(); mi++) {
        Context &m = *g->members[mi];
        for (cudaStream_t s : m.streams) {
            CNHE_CUDA(cudaEventRecord(m.ev_join, s));
            CNHE_CUDA(cudaStreamWaitEvent(c.streams[0], m.ev_join, 0));
        }
    }
    if (!g->words_sent) { // a new binding: stream 0 orders the copy after the previous launch's kernels and before this one's
        c.h2d(g->keys->table, g->words.data(), g->words.size() * sizeof(u64 *));
        g->words_sent = true;
    }
    CNHE_CUDA(cudaGraphLaunch(g->exec, c.streams[0]));
    // before every call queued after (a level's decryption of the scores, say)
    c.fork_streams();
    if (g->members.size() > 1) {
        CNHE_CUDA(cudaEventRecord(c.ev_join, c.streams[0]));
        for (size_t mi = 1; mi < g->members.size(); mi++)
            for (cudaStream_t s : g->members[mi]->streams) CNHE_CUDA(cudaStreamWaitEvent(s, c.ev_join, 0));
    }
    for (size_t mi = 0; mi < g->members.size(); mi++) {
        Context &m = *g->members[mi];
        for (int i = 0; i < Context::OP_COUNT; i++) m.op_count[i] += g->ops[mi][i];
        m.launches += g->launches[mi];
    }
    API_END
}
extern "C" int cnhe_graph_info(const cnhe_graph *g, uint64_t *kernel_nodes, uint64_t *device_bytes) {
    if (!g) return set_err(CNHE_ERR_INVALID, "null graph");
    if (kernel_nodes) *kernel_nodes = g->kernel_nodes;
    if (device_bytes) *device_bytes = g->arena->bytes;
    return CNHE_OK;
}
extern "C" int cnhe_graph_destroy(cnhe_graph *g) {
    if (!g) return CNHE_OK;
    Context &c = *g->h->c;
    try {
        std::lock_guard<std::recursive_mutex> lock(c.mu);
        const Locks locks = lock_members(g->members);
        for (Context *m : g->members)
            if (m->rec) return set_err(CNHE_ERR_STATE, "cnhe_graph_destroy: refused while a context the graph spans records a graph");
        CNHE_CUDA(cudaSetDevice(c.device));
        for (Context *m : g->members) m->sync(); // no launch still runs in the memory about to be freed
        CNHE_CUDA(cudaGraphExecDestroy(g->exec));
        for (size_t i = 0; i < g->members.size(); i++) release_deferred(*g->members[i], g->held[i]);
        delete g;
    } catch (const Error &e) { return set_err(e.code, e.what()); }
    return CNHE_OK;
}
extern "C" int cnhe_keys_generate(cnhe_ctx *h, uint64_t seed) {
    API_BEGIN(h)
    not_recorded(c, "replaces keys");
    c.keys_changed(0);
    keys_generate(c, seed);
    API_END
}
extern "C" int cnhe_keys_generate_secure(cnhe_ctx *h) {
    API_BEGIN(h)
    not_recorded(c, "replaces keys");
    c.keys_changed(0);
    keys_generate_secure(c);
    API_END
}
// OperationsCount / CryptoTracker mirrors
extern "C" int cnhe_op_counts(cnhe_ctx *h, uint64_t *out, int cap, int reset) {
    API_BEGIN(h)
    if (!out || cap < Context::OP_COUNT) fail("need room for CNHE_OP_COUNT counters");
    if (reset) not_recorded(c, "resets the operation counters");
    for (int i = 0; i < Context::OP_COUNT; i++) out[i] = c.op_count[i];
    if (reset) for (int i = 0; i < Context::OP_COUNT; i++) c.op_count[i] = 0;
    API_END
}
extern "C" const char *cnhe_op_name(int kind) { return op_kind_name(kind); }
extern "C" int cnhe_trace_read(cnhe_ctx *h, int32_t *out, size_t cap_records, size_t *n_records, int clear) {
    API_BEGIN(h)
    not_recorded(c, "reads the noise trace");
    if (n_records) *n_records = c.trace.size();
    if (out) {
        const size_t n = std::min(cap_records, c.trace.size());
        static_assert(sizeof(Context::TraceRec) == 8 * sizeof(int32_t), "trace record layout");
        memcpy(out, c.trace.data(), n * sizeof(Context::TraceRec));
    }
    if (clear) { c.trace.clear(); }
    API_END
}
extern "C" int cnhe_keys_set_seed(cnhe_ctx *h, int channel, uint64_t seed) {
    API_BEGIN(h)
    not_recorded(c, "changes a channel's sampler");
    if (channel < 0 || channel >= c.P) fail("bad channel");
    memset(&c.ch[channel].rng, 0, sizeof(RngKey)); // deterministic sampler (tests): see cnhe.h
    c.ch[channel].rng.seed = seed;
    API_END
}
extern "C" int cnhe_keys_export(cnhe_ctx *h, int channel, int what, uint64_t arg, uint64_t *dst, size_t cap) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (what == 4) { // the packed relinearisation keys the fused key switch reads
        if (channel < 0 || channel >= c.P) fail("bad channel");
        const BufRef &pk = c.ch[channel].rlk_packed;
        if (!pk) throw Error(CNHE_ERR_STATE, "the channel holds no packed relinearization keys");
        const size_t words = (size_t)c.dm_relin.D * 2 * c.k * c.N * 6 / 8;
        if (cap < words) fail("destination too small");
        CNHE_CUDA(cudaMemcpyAsync(dst, pk->p, words * 8, cudaMemcpyDeviceToHost, c.stream));
        c.sync();
        return CNHE_OK;
    }
    size_t words;
    BufRef &b = key_slot(c, channel, what, arg, words, false);
    if (cap < words) fail("destination too small");
    CNHE_CUDA(cudaMemcpyAsync(dst, b->p, words * 8, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    API_END
}
extern "C" int cnhe_keys_import(cnhe_ctx *h, int channel, int what, uint64_t arg, const uint64_t *src, size_t nwords) {
    API_BEGIN(h)
    not_recorded(c, "replaces keys");
    c.keys_changed(0);
    size_t words;
    BufRef &b = key_slot(c, channel, what, arg, words, true);
    if (nwords != words) fail("wrong key size");
    CNHE_CUDA(cudaMemcpyAsync(b->p, src, words * 8, cudaMemcpyHostToDevice, c.stream));
    c.sync();
    Channel &ch = c.ch[channel];
    if (what == 0) ch.have_sk = true;
    if (what == 1) ch.have_pk = true;
    if (what == 2) rlk_ready(c, channel);
    API_END
}

// ---------------------------------------------------------------------------------------------------- raw / microbench
extern "C" int cnhe_dev_alloc(cnhe_ctx *h, size_t words, uint64_t *dptr) {
    API_BEGIN(h)
    void *p = nullptr;
    CNHE_CUDA(cudaMalloc(&p, words * 8));
    *dptr = (uint64_t)p;
    API_END
}
extern "C" int cnhe_dev_free(cnhe_ctx *h, uint64_t dptr) {
    API_BEGIN(h)
    c.sync();
    CNHE_CUDA(cudaFree((void *)dptr));
    API_END
}
extern "C" int cnhe_dev_upload(cnhe_ctx *h, uint64_t dptr, const uint64_t *src, size_t words) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    CNHE_CUDA(cudaMemcpyAsync((void *)dptr, src, words * 8, cudaMemcpyHostToDevice, c.stream));
    c.sync();
    API_END
}
extern "C" int cnhe_dev_download(cnhe_ctx *h, uint64_t *dst, uint64_t dptr, size_t words) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    CNHE_CUDA(cudaMemcpyAsync(dst, (void *)dptr, words * 8, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    API_END
}
extern "C" int cnhe_raw_ntt(cnhe_ctx *h, uint64_t src, uint64_t dst, int n_polys, int mod_base, int mod_count, int inverse) {
    API_BEGIN(h)
    if (mod_base < 0 || mod_count < 1 || mod_base + mod_count > c.k + c.kb + c.P) fail("bad modulus range");
    op_ntt(c, (const u64 *)src, (u64 *)dst, n_polys, mod_base, mod_count, inverse != 0);
    API_END
}
static std::vector<const u64 *> strided(uint64_t base, int n, size_t words) {
    std::vector<const u64 *> v(n);
    for (int i = 0; i < n; i++) v[i] = (const u64 *)base + (size_t)i * words;
    return v;
}
extern "C" int cnhe_raw_multiply(cnhe_ctx *h, int channel, uint64_t a, uint64_t b, int n, uint64_t out3) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    op_multiply(c, channel, strided(a, n, c.ct_words()), strided(b, n, c.ct_words()), (u64 *)out3);
    API_END
}
extern "C" int cnhe_raw_relinearize(cnhe_ctx *h, int channel, uint64_t in3, int n, uint64_t out2) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    op_relinearize(c, channel, (const u64 *)in3, n, (u64 *)out2);
    API_END
}
extern "C" int cnhe_raw_multiply_relin(cnhe_ctx *h, int channel, uint64_t a, uint64_t b, int n, uint64_t out2) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    op_multiply_relin(c, channel, strided(a, n, c.ct_words()), strided(b, n, c.ct_words()), (u64 *)out2);
    API_END
}
extern "C" int cnhe_raw_apply_galois(cnhe_ctx *h, int channel, uint64_t in, int n, uint64_t elt, uint64_t out) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    op_apply_galois(c, channel, (const u64 *)in, n, elt, (u64 *)out);
    API_END
}
extern "C" int cnhe_raw_rotate_rows(cnhe_ctx *h, int channel, uint64_t in, int n, int steps, uint64_t out) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    op_rotate_rows(c, channel, (const u64 *)in, n, steps, (u64 *)out);
    API_END
}
extern "C" int cnhe_raw_behz_lift(cnhe_ctx *h, uint64_t in_cts, int n, uint64_t out) {
    API_BEGIN(h)
    if (c.fp_elementwise)
        c.check(launch_behz_lift_fp(upload_ptrs(c, strided(in_cts, n, c.ct_words())), (u64 *)out, n, c.logN, &c.h_bf, 0, c.stream), "behz_lift_fp");
    else c.check(launch_behz_lift(upload_ptrs(c, strided(in_cts, n, c.ct_words())), (u64 *)out, n, c.logN, c.d_bc, c.stream), "behz_lift");
    API_END
}
extern "C" int cnhe_raw_behz_floor(cnhe_ctx *h, int channel, uint64_t d, int n, uint64_t out3) {
    API_BEGIN(h)
    if (channel < 0 || channel >= c.P) fail("bad channel");
    c.set_channel(channel);
    if (c.fp_elementwise) c.check(launch_behz_floor_fp((const u64 *)d, (u64 *)out3, n, c.ch[channel].t, c.logN, &c.h_bf, c.stream), "behz_floor_fp");
    else c.check(launch_behz_floor((const u64 *)d, (u64 *)out3, n, c.ch[channel].t, c.logN, c.d_bc, c.stream), "behz_floor");
    API_END
}
extern "C" int cnhe_dev_copy(cnhe_ctx *h, uint64_t dst, uint64_t src, size_t words) {
    API_BEGIN(h)
    // the pointers may belong to any channel: order the copy after every channel's queued work and before anything queued later
    c.join_streams();
    CNHE_CUDA(cudaMemcpyAsync((void *)dst, (const void *)src, words * 8, cudaMemcpyDeviceToDevice, c.streams[0]));
    c.fork_streams();
    API_END
}
extern "C" int cnhe_prof_enable(cnhe_ctx *h, int on) {
    API_BEGIN(h)
    not_recorded(c, "profiles");
    c.prof_flush();
    c.prof = on != 0;
    if (on) for (int i = 0; i < 6; i++) { c.prof_ms[i] = 0; c.prof_bytes[i] = 0; c.prof_n[i] = 0; }
    API_END
}
extern "C" int cnhe_prof_collect(cnhe_ctx *h, int family, double *total_ms, uint64_t *launches, double *bytes) {
    API_BEGIN(h)
    not_recorded(c, "profiles");
    if (family < 0 || family > 5) fail("bad family");
    c.prof_flush();
    if (total_ms) *total_ms = c.prof_ms[family];
    if (launches) *launches = c.prof_n[family];
    if (bytes) *bytes = c.prof_bytes[family];
    API_END
}
extern "C" int cnhe_raw_event_timing(cnhe_ctx *h, int start) {
    API_BEGIN(h)
    not_recorded(c, "profiles");
    if (start) {
        c.join_streams();
        CNHE_CUDA(cudaEventRecord(c.ev0, c.streams[0]));
        c.fork_streams();
    } else {
        c.join_streams();
        CNHE_CUDA(cudaEventRecord(c.ev1, c.streams[0]));
    }
    API_END
}
extern "C" int cnhe_raw_elapsed_ms(cnhe_ctx *h, float *ms) {
    API_BEGIN(h)
    not_recorded(c, "profiles");
    CNHE_CUDA(cudaEventSynchronize(c.ev1));
    CNHE_CUDA(cudaEventElapsedTime(ms, c.ev0, c.ev1));
    API_END
}

// ---------------------------------------------------------------------------------------------------- vector helpers
cnhe_vec *new_vec(Context &c, uint64_t dim, double scale, int format, bool enc, int blocks) {
    cnhe_vec *v = new cnhe_vec();
    v->ctx = &c;
    v->dim = dim;
    v->scale = scale;
    v->format = format;
    v->enc = enc;
    v->slot = c.slot;
    if (c.rec) v->binding = c.rec->keys;
    v->blocks = blocks;
    v->buf.resize(c.P);
    v->off.assign(c.P, 0);
    return v;
}
void alloc_channels(cnhe_vec *v) {
    for (int ch = 0; ch < v->ctx->P; ch++) {
        v->ctx->set_channel(ch);
        v->buf[ch] = v->ctx->alloc((size_t)v->blocks * v->unit());
    }
}
// v's blocks as a view of one slab per channel, starting `ct` ciphertexts in: the outputs of a batched call share one allocation
static cnhe_vec *slab_view(cnhe_vec *v, const std::vector<BufRef> &slab, size_t ct) {
    for (int ch = 0; ch < v->ctx->P; ch++) {
        v->buf[ch] = slab[ch];
        v->off[ch] = ct * v->ctx->ct_words();
    }
    return v;
}
// An output of a batched call: an encrypted vector shaped like `like` (dimension, format, blocks) at `scale` and in key slot `slot`,
// viewing the call's slab from ciphertext `ct` on
static cnhe_vec *slab_output(Context &c, const std::vector<BufRef> &slab, size_t ct, const cnhe_vec *like, double scale, int slot) {
    cnhe_vec *v = slab_view(new_vec(c, like->dim, scale, like->format, true, like->blocks), slab, ct);
    v->slot = slot;
    return v;
}
static cnhe_vec *alias_of(const cnhe_vec *a) { return new cnhe_vec(*a); } // shares the reference-counted buffers
cnhe_vec::cnhe_vec(const cnhe_vec &o)
    : ctx(o.ctx), dim(o.dim), scale(o.scale), format(o.format), enc(o.enc), slot(o.slot), binding(o.binding), blocks(o.blocks), buf(o.buf), off(o.off),
      scalars(o.scalars), is_const(o.is_const), const_val(o.const_val), pend(o.pend), pend_ct(o.pend_ct) {
    if (pend) pend->members.push_back(this);
}
cnhe_vec::~cnhe_vec() {
    if (!pend) return;
    auto &m = pend->members;
    m.erase(std::remove(m.begin(), m.end(), this), m.end());
}
// Relinearises v's pending group, if it has one: one op_relinearize per channel over all the group's products (the eager square's call,
// run later), then every member points at its ciphertexts in the result
void materialise(Context &c, const cnhe_vec *v) {
    if (!v || !v->pend) return;
    const std::shared_ptr<PendingGroup> g = v->pend;
    // a group made before the recording would be re-pointed at graph memory that holds no words until a launch: read it first
    if (c.rec && g->slab3[0]->arena != c.rec->arena) c.refuse("relinearises squares made before the recording (read them once first)");
    const cudaStream_t s0 = c.stream;
    const size_t ctw = c.ct_words();
    std::vector<int> slots = g->ct_slot; // squares recorded into a graph: under the slots the graph is bound to
    if (v->binding)
        for (int &s : slots) s = v->binding->slot(s);
    std::vector<BufRef> slab2(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        slab2[ch] = c.alloc((size_t)g->total * ctw);
        op_relinearize(c, ch, g->slab3[ch]->p, g->total, slab2[ch]->p, slots.data(), false); // booked by the square
    }
    c.stream = s0;
    for (cnhe_vec *m : g->members) {
        m->buf = slab2;
        for (int ch = 0; ch < c.P; ch++) m->off[ch] = m->pend_ct * ctw;
        m->pend.reset();
    }
    g->members.clear();
    g->slab3.clear();
}
void same_ctx(Context &c, const cnhe_vec *v) {
    if (!v) fail("null vector");
    if (v->ctx != &c) fail("vector belongs to another context");
    materialise(c, v);
}
int use_slot(Context &c, const cnhe_vec *const *vs, int n) {
    int s = -1;
    for (int i = 0; i < n; i++) {
        if (vs[i] && vs[i]->ctx == &c) materialise(c, vs[i]);
        if (!vs[i] || !vs[i]->enc) continue;
        if (s >= 0 && vs[i]->key_slot() != s) fail("encrypted operands belong to different key slots");
        s = vs[i]->key_slot();
    }
    if (s < 0) s = 0;
    if (!c.slot_live(s)) fail("the vector's key slot was removed");
    c.slot = s;
    c.foreign = s != 0;
    return s;
}
// key slot of each encrypted vector, checked against the context (layer entry points that serve several clients in one call); keep_pending:
// leave pending vectors as they are (the scalar-MAC layer's exact path reads them unrelinearised)
static std::vector<int> vec_slots(Context &c, const cnhe_vec *const *vs, int n, bool keep_pending = false) {
    std::vector<int> s(n);
    for (int i = 0; i < n; i++) {
        if (!keep_pending && vs[i]->ctx == &c) materialise(c, vs[i]);
        s[i] = vs[i]->key_slot();
        if (!c.slot_live(s[i])) fail("the vector's key slot was removed");
        if (s[i] != 0) c.foreign = true;
    }
    return s;
}
// SplitBigNumbers ("EncryptedSealBfvVector.cs:352-365"): round(v*scale) -> +bigFactor if negative -> residues
static void split_values(Context &c, const double *v, uint64_t n, double scale, std::vector<std::vector<u64>> &res) {
    res.assign(c.P, std::vector<u64>(n));
    for (uint64_t j = 0; j < n; j++) {
        const double w = std::nearbyint(v[j] * scale); // Math.Round: to nearest, ties to even
        if (!(std::fabs(w) < 1.5e38)) fail("value out of range");
        const bool neg = w < 0;
        u128 mag = (u128)(neg ? -w : w);
        if (mag >= c.big_factor) mag %= c.big_factor;
        const u128 z = (neg && mag) ? c.big_factor - mag : mag;
        for (int i = 0; i < c.P; i++) res[i][j] = (u64)(z % c.t[i]);
    }
}
static u128 mulmod_u128(u128 a, u64 b, u128 m) { // a < m < 2^126
    u128 r = 0;
    while (b) {
        if (b & 1) { r += a; if (r >= m) r -= m; }
        a += a; if (a >= m) a -= m;
        b >>= 1;
    }
    return r;
}
// JoinSplitNumbers ("EncryptedSealBfvVector.cs:381-395")
static void join_values(Context &c, const std::vector<std::vector<u64>> &split, uint64_t n, double scale, double *out) {
    for (uint64_t j = 0; j < n; j++) {
        u128 acc = 0;
        for (int i = 0; i < c.P; i++) {
            acc += mulmod_u128(c.crt_coeff[i] % c.big_factor, split[i][j], c.big_factor);
            if (acc >= c.big_factor) acc -= c.big_factor;
        }
        double val;
        if (acc * 2 > c.big_factor) val = -(double)(c.big_factor - acc);
        else val = (double)acc;
        out[j] = val / scale;
    }
}

static cnhe_vec *make_vector_split(Context &c, const std::vector<std::vector<u64>> &split, const double *v, uint64_t dim, double scale, int format,
                                   bool encrypt);
static cnhe_vec *make_vector(Context &c, const double *v, uint64_t dim, double scale, int format, bool encrypt) {
    if (!v && dim) fail("null values");
    if (format != CNHE_DENSE && format != CNHE_SPARSE) fail("bad format");
    if (scale == 0) scale = 1; // AtomicSealBfvVector.cs:1120
    std::vector<std::vector<u64>> split;
    split_values(c, v, dim, scale, split);
    return make_vector_split(c, split, v, dim, scale, format, encrypt);
}
// `split`: per plaintext modulus the residues of the (already scaled and rounded) values; `v` (may be null) only feeds the
// all-slots-equal shortcut of plain dense vectors
static cnhe_vec *make_vector_split(Context &c, const std::vector<std::vector<u64>> &split, const double *v, uint64_t dim, double scale, int format,
                                   bool encrypt) {
    const size_t N = c.N;
    const int blocks = format == CNHE_DENSE ? (int)((dim + N - 1) / N) : (int)dim;
    if (blocks < 1) fail("empty vector");
    cnhe_vec *out = new_vec(c, dim, scale, format, encrypt, blocks);
    std::unique_ptr<cnhe_vec> guard(out);
    if (format == CNHE_SPARSE && !encrypt) {
        out->scalars = split;
        for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
            out->buf[ch] = c.alloc(dim);
            c.upload(out->buf[ch]->p, split[ch].data(), dim * 8);
        }
        c.host_fence();
        return guard.release();
    }
    alloc_channels(out);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        if (format == CNHE_DENSE) {
            // BatchEncoder.Encode per N-slot chunk (AtomicSealBfvVector.cs:1123-1133); a short last chunk is zero padded
            std::vector<u64> padded((size_t)blocks * N, 0);
            memcpy(padded.data(), split[ch].data(), dim * 8);
            u64 *dvals = c.ws_alloc((size_t)blocks * N);
            c.upload(dvals, padded.data(), padded.size() * 8);
            u64 *plain = encrypt ? c.ws_alloc((size_t)blocks * N) : out->ptr(ch);
            op_encode(c, ch, dvals, blocks, (int)N, plain);
            if (encrypt) {
                op_encrypt(c, ch, plain, N, blocks, (int)N, take_nonces(c, ch, blocks), out->ptr(ch));
            }
        } else { // sparse encrypted: one constant-polynomial plaintext per element (AtomicSealBfvVector.cs:1135-1138)
            u64 *dvals = c.ws_alloc(dim);
            c.upload(dvals, split[ch].data(), dim * 8);
            op_encrypt(c, ch, dvals, 1, blocks, 1, take_nonces(c, ch, blocks), out->ptr(ch));
        }
        c.host_fence(); // host staging buffers go out of scope
    }
    if (v && !encrypt && format == CNHE_DENSE && dim % N == 0) { // every slot equal => every plaintext is the constant polynomial
        bool all_eq = true;
        for (uint64_t j = 1; j < dim && all_eq; j++) all_eq = v[j] == v[0];
        if (all_eq) {
            out->is_const = true;
            for (int ch = 0; ch < c.P; ch++) out->const_val.push_back(split[ch][0]);
        }
    }
    return guard.release();
}

extern "C" int cnhe_vec_encrypt(cnhe_ctx *h, const double *v, uint64_t dim, double scale, int format, cnhe_vec **out) {
    API_BEGIN(h)
    not_recorded(c, "samples encryption randomness (a replay would reuse it for every input)");
    *out = make_vector(c, v, dim, scale, format, true);
    API_END
}
// BigInteger entry points of the factory ("HE Wrapper/IFactory.cs:29,43" -> EncryptedSealBfvVector(IEnumerable<BigInteger>, ...),
// "EncryptedSealBfvVector.cs:188-199"): the host reduces each big integer modulo every plaintext prime (SplitBigNumbers, ":367-379")
extern "C" int cnhe_vec_from_residues(cnhe_ctx *h, const uint64_t *residues, uint64_t dim, double scale, int format, int encrypt, cnhe_vec **out) {
    API_BEGIN(h)
    if (!residues || !out || dim < 1) fail("bad arguments");
    if (format != CNHE_DENSE && format != CNHE_SPARSE) fail("bad format");
    if (encrypt) not_recorded(c, "samples encryption randomness (a replay would reuse it for every input)");
    std::vector<std::vector<u64>> split(c.P, std::vector<u64>(dim));
    for (int ch = 0; ch < c.P; ch++)
        for (uint64_t j = 0; j < dim; j++) {
            split[ch][j] = residues[(size_t)ch * dim + j];
            if (split[ch][j] >= c.t[ch]) fail("residue not reduced modulo its plaintext prime");
        }
    *out = make_vector_split(c, split, nullptr, dim, scale == 0 ? 1 : scale, format, encrypt != 0);
    API_END
}
extern "C" int cnhe_vec_plain(cnhe_ctx *h, const double *v, uint64_t dim, double scale, int format, cnhe_vec **out) {
    API_BEGIN(h)
    *out = make_vector(c, v, dim, scale, format, false);
    API_END
}
// n dense single-block-or-more vectors encrypted in one wave per channel (GetEncryptedMatrix, IFactory.cs:353-380)
extern "C" int cnhe_vecs_encrypt(cnhe_ctx *h, const double *v, int n, uint64_t dim, double scale, cnhe_vec **out) {
    API_BEGIN(h)
    not_recorded(c, "samples encryption randomness (a replay would reuse it for every input)");
    if (n < 1 || !v || !out) fail("bad arguments");
    if (scale == 0) scale = 1;
    const size_t N = c.N;
    const int bl = (int)((dim + N - 1) / N);
    std::vector<std::vector<u64>> split;
    split_values(c, v, (uint64_t)n * dim, scale, split);
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<u64> padded((size_t)n * bl * N, 0);
        for (int i = 0; i < n; i++) memcpy(&padded[(size_t)i * bl * N], &split[ch][(size_t)i * dim], dim * 8);
        u64 *dvals = c.ws_alloc(padded.size()), *plain = c.ws_alloc(padded.size());
        CNHE_CUDA(cudaMemcpyAsync(dvals, padded.data(), padded.size() * 8, cudaMemcpyHostToDevice, c.stream));
        op_encode(c, ch, dvals, n * bl, (int)N, plain);
        big[ch] = c.alloc((size_t)n * bl * c.ct_words());
        op_encrypt(c, ch, plain, N, n * bl, (int)N, take_nonces(c, ch, (u64)n * bl), big[ch]->p);
        c.sync();
    }
    for (int i = 0; i < n; i++) out[i] = slab_view(new_vec(c, dim, scale, CNHE_DENSE, true, bl), big, (size_t)i * bl);
    API_END
}

// Decrypt of the blocks of one channel into residues (dense: first `dim` slots; sparse: constant coefficients)
static void decrypt_channel(Context &c, const cnhe_vec *v, int ch, std::vector<u64> &res) {
    const size_t N = c.N;
    res.assign(v->dim, 0);
    if (!v->enc && v->format == CNHE_SPARSE) { res = v->scalars[ch]; return; }
    u64 *plain;
    if (v->enc) {
        if (v->key_slot() != 0) throw Error(CNHE_ERR_STATE, "the context holds no secret key of the vector's key slot");
        plain = c.ws_alloc((size_t)v->blocks * N);
        op_decrypt(c, ch, v->ptr(ch), v->blocks, plain);
    } else plain = v->ptr(ch);
    if (v->format == CNHE_DENSE) {
        u64 *vals = c.ws_alloc((size_t)v->blocks * N);
        op_decode(c, ch, plain, v->blocks, vals);
        std::vector<u64> hostv((size_t)v->blocks * N);
        CNHE_CUDA(cudaMemcpyAsync(hostv.data(), vals, hostv.size() * 8, cudaMemcpyDeviceToHost, c.stream));
        c.sync();
        const uint64_t take = std::min<uint64_t>(v->dim, hostv.size());
        memcpy(res.data(), hostv.data(), take * 8);
    } else {
        std::vector<u64> hostv(v->blocks);
        CNHE_CUDA(cudaMemcpy2DAsync(hostv.data(), 8, plain, N * 8, 8, v->blocks, cudaMemcpyDeviceToHost, c.stream));
        c.sync();
        const uint64_t take = std::min<uint64_t>(v->dim, hostv.size());
        memcpy(res.data(), hostv.data(), take * 8);
    }
}
// Decrypt of v's `dim` values: every channel's residues, joined
static void decrypt_values(Context &c, const cnhe_vec *v, double *out) {
    std::vector<std::vector<u64>> split(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        decrypt_channel(c, v, ch, split[ch]);
    }
    join_values(c, split, v->dim, v->scale, out);
}
extern "C" int cnhe_vec_decrypt(cnhe_ctx *h, const cnhe_vec *v, double *out, uint64_t cap) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    same_ctx(c, v);
    if (cap < v->dim) fail("destination too small");
    decrypt_values(c, v, out);
    API_END
}
// DecryptFullPrecision ("EncryptedSealBfvVector.cs:343-348"): the residues of every channel, for the caller's BigInteger CRT join
// (JoinSplitNumbers, ":397-411"); out is [P][dim]
extern "C" int cnhe_vec_decrypt_residues(cnhe_ctx *h, const cnhe_vec *v, uint64_t *out, uint64_t cap) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    same_ctx(c, v);
    if (!out || cap < v->dim * (uint64_t)c.P) fail("destination too small");
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<u64> r;
        decrypt_channel(c, v, ch, r);
        memcpy(out + (size_t)ch * v->dim, r.data(), v->dim * 8);
    }
    API_END
}
extern "C" int cnhe_vecs_decrypt(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, double *out, uint64_t dim) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    for (int i = 0; i < n; i++) {
        same_ctx(c, vecs[i]);
        if (vecs[i]->dim != dim) fail("all vectors must have the same dimension");
        decrypt_values(c, vecs[i], out + (size_t)i * dim);
    }
    API_END
}
// New words for existing encrypted vectors (a graph's recorded inputs): dst[i] takes src[i]'s ciphertexts, device to device on each
// channel's stream.  Host-side attributes a recording may have acted on (dimension, blocks, format, scale, key slot) must match.
extern "C" int cnhe_vecs_assign(cnhe_ctx *h, cnhe_vec *const *dst, const cnhe_vec *const *src, int n) {
    API_BEGIN(h)
    if (!dst || !src || n < 1) fail("bad arguments");
    for (int i = 0; i < n; i++) {
        if (!dst[i] || !src[i]) fail("null vector");
        if (dst[i]->ctx != &c || src[i]->ctx != &c) fail("vector belongs to another context");
    }
    vec_slots(c, src, n); // the sources' key slots are live; pending sources are relinearised
    vec_slots(c, dst, n, true);
    for (int i = 0; i < n; i++) {
        const cnhe_vec *d = dst[i], *s = src[i];
        if (!d->enc || !s->enc) fail("cnhe_vecs_assign copies encrypted vectors only");
        if (d->pend) fail("the destination's squares are not relinearised (it was made by a square layer and never read)");
        if (d->dim != s->dim || d->blocks != s->blocks || d->format != s->format) fail("source and destination differ in shape");
        if (d->scale != s->scale) fail("source and destination differ in scale");
        if (d->key_slot() != s->key_slot()) fail("source and destination belong to different key slots");
    }
    // a destination may be its own source (nothing to copy) but may not overlap any other source: the copies (coalesced below) would
    // read words they, or an earlier copy, overwrite
    const size_t ctw = c.ct_words();
    for (int ch = 0; ch < c.P; ch++) {
        std::vector<std::pair<const u64 *, int>> by_start(n);
        for (int i = 0; i < n; i++) by_start[i] = {src[i]->ptr(ch), i};
        std::sort(by_start.begin(), by_start.end());
        std::vector<const u64 *> reach(n); // reach[k]: the furthest end of the sources sorted up to k
        for (int k = 0; k < n; k++) {
            const u64 *e = by_start[k].first + src[by_start[k].second]->blocks * ctw;
            reach[k] = k && reach[k - 1] > e ? reach[k - 1] : e;
        }
        for (int i = 0; i < n; i++) {
            const u64 *a = dst[i]->ptr(ch), *a_end = a + dst[i]->blocks * ctw;
            for (int k = (int)(std::lower_bound(by_start.begin(), by_start.end(), std::make_pair(a_end, -1)) - by_start.begin()) - 1;
                 k >= 0 && reach[k] > a; k--) {
                const int j = by_start[k].second;
                if (by_start[k].first + src[j]->blocks * ctw > a && !(j == i && by_start[k].first == a))
                    fail("a destination overlaps a source other than its own");
            }
        }
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        for (int i = 0, j; i < n; i = j) { // one copy per run of vectors that lie back to back in one slab on both sides
            size_t words = dst[i]->blocks * ctw;
            for (j = i + 1; j < n && dst[j]->buf[ch] == dst[i]->buf[ch] && src[j]->buf[ch] == src[i]->buf[ch] &&
                            dst[j]->ptr(ch) == dst[i]->ptr(ch) + words && src[j]->ptr(ch) == src[i]->ptr(ch) + words;
                 j++)
                words += dst[j]->blocks * ctw;
            if (dst[i]->ptr(ch) != src[i]->ptr(ch))
                CNHE_CUDA(cudaMemcpyAsync(dst[i]->ptr(ch), src[i]->ptr(ch), words * 8, cudaMemcpyDeviceToDevice, c.stream));
        }
    }
    API_END
}
extern "C" int cnhe_vec_copy(cnhe_ctx *h, const cnhe_vec *v, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, v);
    cnhe_vec *o = new cnhe_vec(*v);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        const size_t words = (size_t)v->blocks * v->unit();
        o->buf[ch] = c.alloc(words);
        o->off[ch] = 0;
        CNHE_CUDA(cudaMemcpyAsync(o->buf[ch]->p, v->ptr(ch), words * 8, cudaMemcpyDeviceToDevice, c.stream));
    }
    *out = o;
    API_END
}
extern "C" int cnhe_vec_destroy(cnhe_vec *v) {
    if (!v) return CNHE_OK;
    try {
        std::lock_guard<std::recursive_mutex> lock(v->ctx->mu);
        cudaSetDevice(v->ctx->device);
        delete v;
    } catch (...) { return set_err(CNHE_ERR_INVALID, "destroy failed"); }
    return CNHE_OK;
}
extern "C" int cnhe_vecs_destroy(cnhe_vec *const *vecs, int n) {
    if (!vecs || n < 1) return CNHE_OK;
    try {
        Context *ctx = nullptr;
        for (int i = 0; i < n && !ctx; i++)
            if (vecs[i]) ctx = vecs[i]->ctx;
        if (!ctx) return CNHE_OK;
        std::lock_guard<std::recursive_mutex> lock(ctx->mu);
        cudaSetDevice(ctx->device);
        for (int i = 0; i < n; i++)
            if (vecs[i]) {
                if (vecs[i]->ctx != ctx) return set_err(CNHE_ERR_INVALID, "vectors of different contexts");
                delete vecs[i];
            }
    } catch (...) { return set_err(CNHE_ERR_INVALID, "destroy failed"); }
    return CNHE_OK;
}
extern "C" int cnhe_vec_meta(const cnhe_vec *v, uint64_t *dim, double *scale, int *format, int *is_encrypted, int *blocks, uint64_t *block_size) {
    if (!v) return set_err(CNHE_ERR_INVALID, "null vector");
    if (dim) *dim = v->dim;
    if (scale) *scale = v->scale;
    if (format) *format = v->format;
    if (is_encrypted) *is_encrypted = v->enc ? 1 : 0;
    if (blocks) *blocks = v->blocks;
    if (block_size) *block_size = v->ctx->N;
    return CNHE_OK;
}
extern "C" int cnhe_vec_register_scale(cnhe_vec *v, double scale) {
    if (!v) return set_err(CNHE_ERR_INVALID, "null vector");
    v->scale = scale;
    return CNHE_OK;
}
extern "C" int cnhe_vec_register_dim(cnhe_vec *v, uint64_t dim) {
    if (!v) return set_err(CNHE_ERR_INVALID, "null vector");
    v->dim = dim;
    return CNHE_OK;
}
extern "C" int cnhe_vec_export_raw(cnhe_ctx *h, const cnhe_vec *v, int channel, int block, uint64_t *dst, size_t cap) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    same_ctx(c, v);
    if (!v->enc) fail("vector is not encrypted");
    if (channel < 0 || channel >= c.P || block < 0 || block >= v->blocks) fail("bad channel/block");
    if (cap < c.ct_words()) fail("destination too small");
    CNHE_CUDA(cudaMemcpyAsync(dst, v->block(channel, block), c.ct_words() * 8, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    API_END
}
extern "C" int cnhe_vec_import_raw(cnhe_ctx *h, const uint64_t *src, int blocks, uint64_t dim, double scale, int format, cnhe_vec **out) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    if (!src || blocks < 1) fail("bad arguments");
    cnhe_vec *o = new_vec(c, dim, scale, format, true, blocks);
    alloc_channels(o);
    const size_t words = (size_t)blocks * c.ct_words();
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        CNHE_CUDA(cudaMemcpyAsync(o->ptr(ch), src + (size_t)ch * words, words * 8, cudaMemcpyDefault, c.stream)); // host or device source
    }
    c.sync();
    *out = o;
    API_END
}
extern "C" int cnhe_vecs_import_raw(cnhe_ctx *h, const uint64_t *src, int n, int blocks, uint64_t dim, double scale, int format, cnhe_vec **out) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    if (!src || n < 1 || blocks < 1 || !out) fail("bad arguments");
    const size_t per = (size_t)blocks * c.ct_words(), words = (size_t)n * per;
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        // the block comes from the context's rotating upload slots and the copy is ordered on the upload stream only (not behind the
        // kernels already queued on the channel's stream): channels follow each other over PCIe, channel 0 computes while channel 1 is
        // still uploading, and an import issued before the previous batch is exported overlaps that batch's kernels
        big[ch] = c.alloc_upload(words, c.stream);
        CNHE_CUDA(cudaMemcpyAsync(big[ch]->p, src + (size_t)ch * words, words * 8, cudaMemcpyHostToDevice, c.copy_stream));
        CNHE_CUDA(cudaEventRecord(c.ev_copy, c.copy_stream));
        CNHE_CUDA(cudaStreamWaitEvent(c.stream, c.ev_copy, 0));
    }
    for (int i = 0; i < n; i++) out[i] = slab_view(new_vec(c, dim, scale, format, true, blocks), big, (size_t)i * blocks);
    API_END
}
// ---------------------------------------------------------------------------------------- compact upload (format: csrc/compact.cu)
static size_t compact_header_bytes(int k, int P) { return 44 + 8 * (size_t)k + 40 * (size_t)P; }
struct CompactHeader {
    uint32_t n = 0, B = 0;
    uint64_t dim = 0;
    double scale = 1;
    std::vector<CompactKey> keys;
    size_t header_bytes = 0, channel_words = 0; // packed words per channel
};
// the blob's header checked against the context; any mismatch is CNHE_ERR_INVALID
static CompactHeader parse_compact(const Context &c, const uint8_t *src, size_t len) {
    auto rd32 = [&](size_t off) { uint32_t v; memcpy(&v, src + off, 4); return v; };
    auto rd64 = [&](size_t off) { uint64_t v; memcpy(&v, src + off, 8); return v; };
    if (len < 44) fail("compact blob: truncated header");
    if (memcmp(src, "CNHC", 4) != 0) fail("compact blob: bad magic");
    if (rd32(4) != 1) fail("compact blob: unsupported version");
    const uint32_t N = rd32(8), k = rd32(12), P = rd32(16);
    if (N != c.N) fail("compact blob: ring dimension differs from the context's");
    if ((int)k != c.k) fail("compact blob: coefficient modulus count differs from the context's");
    if ((int)P != c.P) fail("compact blob: plaintext modulus count differs from the context's");
    CompactHeader hd;
    hd.header_bytes = compact_header_bytes(c.k, c.P);
    if (len < hd.header_bytes) fail("compact blob: truncated header");
    hd.n = rd32(20);
    hd.B = rd32(24);
    hd.dim = rd64(28);
    memcpy(&hd.scale, src + 36, 8);
    for (int l = 0; l < c.k; l++)
        if (rd64(44 + 8 * (size_t)l) != c.q[l]) fail("compact blob: coefficient modulus differs from the context's");
    for (int ch = 0; ch < c.P; ch++)
        if (rd64(44 + 8 * (size_t)c.k + 8 * (size_t)ch) != c.t[ch]) fail("compact blob: plaintext modulus differs from the context's");
    if (hd.n < 1 || hd.B < 1) fail("compact blob: empty");
    if ((uint64_t)hd.n * hd.B >= (1ULL << 32) || hd.n > (uint32_t)INT_MAX) fail("compact blob: too many ciphertexts");
    if (hd.dim < 1 || (hd.dim + c.N - 1) / c.N != hd.B) fail("compact blob: dimension does not match the block count");
    if (!std::isfinite(hd.scale) || hd.scale == 0) fail("compact blob: bad scale");
    hd.keys.resize(c.P);
    for (int ch = 0; ch < c.P; ch++) memcpy(hd.keys[ch].w, src + 44 + 8 * (size_t)(c.k + c.P) + 32 * (size_t)ch, 32);
    hd.channel_words = (size_t)hd.n * hd.B * compact_shape(c).off[c.k];
    if (len != hd.header_bytes + (size_t)c.P * hd.channel_words * 8) fail("compact blob: length does not match the header");
    return hd;
}
extern "C" int cnhe_vecs_encrypt_compact(cnhe_ctx *h, const double *v, int n, uint64_t dim, double scale, uint8_t *dst, size_t cap, size_t *needed) {
    API_BEGIN(h)
    not_recorded(c, "samples encryption randomness (a replay would reuse it for every input)");
    if (n < 1 || dim < 1 || !v || (!dst && !needed)) fail("bad arguments");
    if (scale == 0) scale = 1;
    const size_t N = c.N;
    const uint64_t bl = (dim + N - 1) / N, nct = (uint64_t)n * bl;
    if (nct >= (1ULL << 32)) fail("too many ciphertexts in one blob");
    const CompactShape sh = compact_shape(c);
    const size_t hdr = compact_header_bytes(c.k, c.P), per_ch = (size_t)nct * sh.off[c.k] * 8, total = hdr + (size_t)c.P * per_ch;
    if (needed) *needed = total;
    if (!dst) return CNHE_OK;
    if (cap < total) fail("destination too small");
    for (int ch = 0; ch < c.P; ch++)
        if (!c.ch[ch].have_sk) throw Error(CNHE_ERR_STATE, "secret key is missing");
    std::vector<std::vector<u64>> split;
    split_values(c, v, (uint64_t)n * dim, scale, split);
    std::vector<CompactKey> keys(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<u64> padded((size_t)nct * N, 0);
        for (int i = 0; i < n; i++) memcpy(&padded[(size_t)i * bl * N], &split[ch][(size_t)i * dim], dim * 8);
        u64 *dvals = c.ws_alloc(padded.size()), *plain = c.ws_alloc(padded.size()), *packed = c.ws_alloc((size_t)nct * sh.off[c.k]);
        CNHE_CUDA(cudaMemcpyAsync(dvals, padded.data(), padded.size() * 8, cudaMemcpyHostToDevice, c.stream));
        op_encode(c, ch, dvals, (int)nct, (int)N, plain);
        const u64 nonce0 = take_nonces(c, ch, nct);
        keys[ch] = compact_key(c, ch, nonce0);
        op_encrypt_compact(c, ch, plain, (int)nct, nonce0, keys[ch], packed);
        CNHE_CUDA(cudaMemcpyAsync(dst + hdr + ch * per_ch, packed, per_ch, cudaMemcpyDeviceToHost, c.stream));
        c.sync();
    }
    auto wr32 = [&](size_t off, uint32_t x) { memcpy(dst + off, &x, 4); };
    auto wr64 = [&](size_t off, uint64_t x) { memcpy(dst + off, &x, 8); };
    memcpy(dst, "CNHC", 4);
    wr32(4, 1);
    wr32(8, c.N);
    wr32(12, (uint32_t)c.k);
    wr32(16, (uint32_t)c.P);
    wr32(20, (uint32_t)n);
    wr32(24, (uint32_t)bl);
    wr64(28, dim);
    memcpy(dst + 36, &scale, 8);
    for (int l = 0; l < c.k; l++) wr64(44 + 8 * (size_t)l, c.q[l]);
    for (int ch = 0; ch < c.P; ch++) wr64(44 + 8 * (size_t)c.k + 8 * (size_t)ch, c.t[ch]);
    for (int ch = 0; ch < c.P; ch++) memcpy(dst + 44 + 8 * (size_t)(c.k + c.P) + 32 * (size_t)ch, keys[ch].w, 32);
    API_END
}
// Like cnhe_vecs_import_raw: the packed bytes go to a staging upload slot on the upload stream, k_compact_expand writes the ciphertexts
// into a persistent upload slot on the same stream, and the channel's stream waits for it -- the call returns at once.
extern "C" int cnhe_vecs_import_compact(cnhe_ctx *h, const uint8_t *src, size_t len, cnhe_vec **out, int cap, int *n) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    if (!src || !out || !n) fail("bad arguments");
    const CompactHeader hd = parse_compact(c, src, len);
    *n = (int)hd.n;
    if (cap < (int)hd.n) fail("output array too small for the blob's vectors");
    const int nct = (int)(hd.n * hd.B);
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        BufRef stage = c.alloc_upload(hd.channel_words, c.copy_stream); // released behind the expansion on the upload stream
        CNHE_CUDA(cudaMemcpyAsync(stage->p, src + hd.header_bytes + (size_t)ch * hd.channel_words * 8, hd.channel_words * 8, cudaMemcpyHostToDevice,
                                  c.copy_stream));
        big[ch] = c.alloc_upload((size_t)nct * c.ct_words(), c.stream);
        op_compact_expand(c, stage->p, hd.keys[ch], nct, big[ch]->p, c.copy_stream);
        CNHE_CUDA(cudaEventRecord(c.ev_copy, c.copy_stream));
        CNHE_CUDA(cudaStreamWaitEvent(c.stream, c.ev_copy, 0));
    }
    for (uint32_t i = 0; i < hd.n; i++) out[i] = slab_view(new_vec(c, hd.dim, hd.scale, CNHE_DENSE, true, (int)hd.B), big, (size_t)i * hd.B);
    API_END
}
// ---------------------------------------------------------------------------------------- compact key sets (format: csrc/compact.cu)
static size_t key_header_bytes(int k, int P, size_t G) { return 36 + 8 * (size_t)k + 40 * (size_t)P + 8 * G; }
// the caller's element selection in blob order (increasing); -1: every standard element.  The standard list names 3^(N/4) twice (it is
// its own inverse), so "every element" is the distinct ones.
static std::vector<u64> select_galois(const Context &c, const uint64_t *elts, int n) {
    std::vector<u64> std_elts = c.galois_elts;
    std::sort(std_elts.begin(), std_elts.end());
    std_elts.erase(std::unique(std_elts.begin(), std_elts.end()), std_elts.end());
    if (n == -1) return std_elts;
    if (n < 0 || (n > 0 && !elts)) fail("bad Galois element list");
    std::vector<u64> out(elts, elts + n);
    std::sort(out.begin(), out.end());
    for (size_t i = 0; i < out.size(); i++) {
        if (i && out[i] == out[i - 1]) fail("duplicate Galois element");
        if (!std::binary_search(std_elts.begin(), std_elts.end(), out[i])) fail("not one of the context's Galois elements");
    }
    return out;
}
extern "C" int cnhe_keys_save_compact(cnhe_ctx *h, int sets, const uint64_t *galois_elts, int n_galois, uint8_t *dst, size_t cap, size_t *needed) {
    API_BEGIN(h)
    not_recorded(c, "generates keys");
    if (!dst && !needed) fail("bad arguments");
    if (sets & ~3) fail("unknown key sets (bit 0 public key, bit 1 relinearization keys)");
    const std::vector<u64> elts = select_galois(c, galois_elts, n_galois);
    const CompactShape sh = compact_shape(c);
    const size_t pairs = compact_key_pairs(c, sets, elts.size()), hdr = key_header_bytes(c.k, c.P, elts.size());
    const size_t per_ch = pairs * sh.off[c.k] * 8, total = hdr + (size_t)c.P * per_ch;
    if (needed) *needed = total;
    if (!dst) return CNHE_OK;
    if (cap < total) fail("destination too small");
    for (int ch = 0; ch < c.P; ch++)
        if (!c.ch[ch].have_sk) throw Error(CNHE_ERR_STATE, "secret key is missing");
    std::vector<CompactKey> keys(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        const u64 nonce0 = take_nonces(c, ch, std::max<size_t>(pairs, 1)); // one noise nonce per pair; K_c stays unique even for no pairs
        keys[ch] = compact_key(c, ch, nonce0);
        if (pairs) {
            u64 *packed = c.ws_alloc(pairs * sh.off[c.k]);
            op_keys_save_compact(c, ch, sets, elts, nonce0, keys[ch], packed);
            CNHE_CUDA(cudaMemcpyAsync(dst + hdr + ch * per_ch, packed, per_ch, cudaMemcpyDeviceToHost, c.stream));
        }
        c.sync();
        ws_release_all(c);
    }
    auto wr32 = [&](size_t off, uint32_t x) { memcpy(dst + off, &x, 4); };
    auto wr64 = [&](size_t off, uint64_t x) { memcpy(dst + off, &x, 8); };
    memcpy(dst, "CNHK", 4);
    wr32(4, 1);
    wr32(8, c.N);
    wr32(12, (uint32_t)c.k);
    wr32(16, (uint32_t)c.P);
    wr32(20, (uint32_t)c.dbc_relin);
    wr32(24, (uint32_t)c.dbc_galois);
    wr32(28, (uint32_t)sets);
    wr32(32, (uint32_t)elts.size());
    size_t o = 36;
    for (int l = 0; l < c.k; l++, o += 8) wr64(o, c.q[l]);
    for (int ch = 0; ch < c.P; ch++, o += 8) wr64(o, c.t[ch]);
    for (u64 e : elts) { wr64(o, e); o += 8; }
    for (int ch = 0; ch < c.P; ch++, o += 32) memcpy(dst + o, keys[ch].w, 32);
    API_END
}
struct KeyBlob {
    uint32_t N = 0, k = 0, P = 0, dbc_relin = 0, dbc_galois = 0, sets = 0;
    std::vector<u64> q, t, elts;
    std::vector<CompactKey> keys;
    size_t header_bytes = 0, channel_words = 0; // packed words per channel
};
// every header field and the exact length, on the host; any defect is CNHE_ERR_INVALID
static KeyBlob parse_compact_keys(const uint8_t *src, size_t len) {
    auto rd32 = [&](size_t off) { uint32_t v; memcpy(&v, src + off, 4); return v; };
    auto rd64 = [&](size_t off) { uint64_t v; memcpy(&v, src + off, 8); return v; };
    if (len < 36) fail("compact key blob: truncated header");
    if (memcmp(src, "CNHK", 4) != 0) fail("compact key blob: bad magic");
    if (rd32(4) != 1) fail("compact key blob: unsupported version");
    KeyBlob kb;
    kb.N = rd32(8);
    kb.k = rd32(12);
    kb.P = rd32(16);
    kb.dbc_relin = rd32(20);
    kb.dbc_galois = rd32(24);
    kb.sets = rd32(28);
    const uint32_t G = rd32(32);
    if (kb.sets & ~3u) fail("compact key blob: unknown key sets");
    if (kb.N < 1024 || kb.N > 16384 || (kb.N & (kb.N - 1))) fail("compact key blob: PolyModulusDegree must be a power of two in [1024, 16384]");
    if (kb.k < 1 || kb.k > (uint32_t)KMAX) fail("compact key blob: need 1..9 coefficient primes");
    if (kb.P < 1 || kb.P > 16) fail("compact key blob: need 1..16 plaintext primes");
    if (kb.dbc_relin < 1 || kb.dbc_relin > 60 || kb.dbc_galois < 1 || kb.dbc_galois > 60) fail("compact key blob: bad decomposition bit count");
    const std::vector<u64> std_elts = standard_galois_elts(kb.N);
    if (G >= std_elts.size()) fail("compact key blob: more Galois elements than the context has"); // one standard element is listed twice
    kb.header_bytes = key_header_bytes((int)kb.k, (int)kb.P, G);
    if (len < kb.header_bytes) fail("compact key blob: truncated header");
    size_t o = 36;
    for (uint32_t l = 0; l < kb.k; l++, o += 8) kb.q.push_back(rd64(o));
    for (uint32_t ch = 0; ch < kb.P; ch++, o += 8) kb.t.push_back(rd64(o));
    for (uint32_t g = 0; g < G; g++, o += 8) kb.elts.push_back(rd64(o));
    kb.keys.resize(kb.P);
    for (uint32_t ch = 0; ch < kb.P; ch++, o += 32) memcpy(kb.keys[ch].w, src + o, 32);
    for (uint32_t g = 0; g < G; g++) {
        if (g && kb.elts[g] <= kb.elts[g - 1]) fail("compact key blob: Galois elements must be strictly increasing");
        if (std::find(std_elts.begin(), std_elts.end(), kb.elts[g]) == std_elts.end()) fail("compact key blob: not a standard Galois element");
    }
    size_t words = 0, d_relin = 0, d_galois = 0; // packed words per pair; digits per key (make_digit_map: ceil(bitlen(q_l) / w) each)
    for (u64 q : kb.q) {
        if (q < 2) fail("compact key blob: bad coefficient modulus");
        const size_t b = 64 - __builtin_clzll(q);
        words += kb.N * b / 64;
        d_relin += (b + kb.dbc_relin - 1) / kb.dbc_relin;
        d_galois += (b + kb.dbc_galois - 1) / kb.dbc_galois;
    }
    const size_t pairs = ((kb.sets & 1) ? 1 : 0) + ((kb.sets & 2) ? d_relin : 0) + (size_t)G * d_galois;
    kb.channel_words = pairs * words;
    if (len != kb.header_bytes + (size_t)kb.P * kb.channel_words * 8) fail("compact key blob: length does not match the header");
    return kb;
}
extern "C" int cnhe_context_load_compact(const uint8_t *blob, size_t len, int device, cnhe_ctx **out) {
    try {
        if (!blob || !out) fail("null argument");
        const KeyBlob kb = parse_compact_keys(blob, len);
        std::unique_ptr<cnhe_ctx> ctx(new cnhe_ctx{nullptr});
        ctx->c = context_create(kb.t.data(), (int)kb.P, kb.N, kb.q.data(), (int)kb.k, (int)kb.dbc_relin, (int)kb.dbc_galois, device);
        Context &c = *ctx->c;
        std::unique_ptr<Context> guard(ctx->c);
        {
            std::lock_guard<std::recursive_mutex> lock(c.mu);
            if (compact_key_pairs(c, (int)kb.sets, kb.elts.size()) * compact_shape(c).off[c.k] != kb.channel_words)
                fail("compact key blob: key sizes do not match the context");
            for (int ci = 0; ci < c.P && kb.channel_words; ci++) {
                c.set_channel(ci);
                u64 *stage = c.ws_alloc(kb.channel_words); // the channel's packed payload in one copy
                CNHE_CUDA(cudaMemcpyAsync(stage, blob + kb.header_bytes + (size_t)ci * kb.channel_words * 8, kb.channel_words * 8,
                                          cudaMemcpyHostToDevice, c.stream));
                op_keys_load_compact(c, ci, (int)kb.sets, kb.elts, stage, kb.keys[ci]);
                c.sync();
                ws_release_all(c);
            }
        }
        guard.release();
        *out = ctx.release();
    } catch (const Error &e) { return set_err(e.code, e.what()); } catch (const std::exception &e) { return set_err(CNHE_ERR_INVALID, e.what()); }
    return CNHE_OK;
}
// ---------------------------------------------------------------------------------------------------- key slots (several clients)
extern "C" int cnhe_context_add_client_compact(cnhe_ctx *h, const uint8_t *blob, size_t len, int *slot) {
    API_BEGIN(h)
    not_recorded(c, "adds a client's keys");
    if (!blob || !slot) fail("null argument");
    const KeyBlob kb = parse_compact_keys(blob, len); // every header field and the exact length, before anything is allocated
    bool same = kb.N == c.N && (int)kb.k == c.k && (int)kb.P == c.P && (int)kb.dbc_relin == c.dbc_relin && (int)kb.dbc_galois == c.dbc_galois;
    for (int l = 0; same && l < c.k; l++) same = kb.q[l] == c.q[l];
    for (int ch = 0; same && ch < c.P; ch++) same = kb.t[ch] == c.t[ch];
    if (!same) fail("compact key blob: parameters differ from the context's");
    if (compact_key_pairs(c, (int)kb.sets, kb.elts.size()) * compact_shape(c).off[c.k] != kb.channel_words)
        fail("compact key blob: key sizes do not match the context");
    // slot numbers are never reused: a vector still bound to a removed slot is refused instead of meeting another client's keys
    std::vector<KeySet> keys(c.P);
    for (int ci = 0; ci < c.P && kb.channel_words; ci++) {
        c.set_channel(ci);
        u64 *stage = c.ws_alloc(kb.channel_words);
        CNHE_CUDA(cudaMemcpyAsync(stage, blob + kb.header_bytes + (size_t)ci * kb.channel_words * 8, kb.channel_words * 8, cudaMemcpyHostToDevice,
                                  c.stream));
        op_keys_load_compact(c, keys[ci], (int)kb.sets, kb.elts, stage, kb.keys[ci]);
        c.sync();
        ws_release_all(c);
    }
    c.clients.push_back(std::move(keys));
    *slot = (int)c.clients.size();
    API_END
}
extern "C" int cnhe_context_remove_client(cnhe_ctx *h, int slot) {
    API_BEGIN(h)
    not_recorded(c, "removes a client's keys");
    if (slot < 1 || !c.slot_live(slot)) fail("no such key slot");
    c.sync(); // no queued key switch still reads the keys
    c.clients[slot - 1].clear();
    c.keys_changed(slot);
    API_END
}
// ---------------------------------------------------------------------------------------------------- levels (DESIGN 4.17)
extern "C" int cnhe_context_derive_level(cnhe_ctx *h, int k, cnhe_ctx **out) {
    API_BEGIN(h)
    not_recorded(c, "creates a context");
    if (!out) fail("null argument");
    if (k < 1 || k >= c.k) fail("cnhe_context_derive_level: need 1 <= k < the context's coefficient prime count");
    c.sync(); // the parent's keys are complete
    std::unique_ptr<Context> child(context_derive(c, k));
    *out = new cnhe_ctx{child.release()};
    API_END
}
extern "C" int cnhe_vecs_mod_switch(cnhe_ctx *h, const cnhe_vec *const *in, int n, cnhe_ctx *to, cnhe_vec **out) {
    API_BEGIN(h)
    if (!to || to == h || !in || !out || n < 1) fail("bad arguments");
    Context &d = *to->c;
    // root and k never change after creation: checked before the second lock, so every call that takes it locks the context with more
    // primes first, and two switches of one family cannot wait on each other's locks
    if (d.root != c.root || d.k >= c.k) fail("cnhe_vecs_mod_switch: the destination must be a level of the same context family with fewer primes");
    std::lock_guard<std::recursive_mutex> lock_to(d.mu);
    // the switch spans two contexts' streams and key slots: it is part of a graph only when both contexts are enlisted in one recording
    // (cnhe_capture_begin_levels), whose capture holds both contexts' streams
    if (d.rec) api_enter(d, __func__); // a call on another thread than the recording one is refused
    const bool recorded = c.rec && d.rec && c.rec->group == d.rec->group;
    if (!recorded) {
        not_recorded(c, "switches vectors to a level that is not enlisted in the same recording (cnhe_capture_begin_levels)");
        if (d.rec) {
            abort_recording(d);
            throw Error(CNHE_ERR_STATE, "cnhe_vecs_mod_switch: the destination context records a graph that does not enlist the source; the "
                                        "switch cannot be recorded (the recording was aborted)");
        }
    }
    for (int i = 0; i < n; i++) {
        same_ctx(c, in[i]); // a pending vector is relinearised here
        if (!in[i]->enc) fail("cnhe_vecs_mod_switch: only encrypted vectors switch levels");
    }
    const std::vector<int> slots = vec_slots(c, in, n);
    CNHE_CUDA(cudaSetDevice(d.device));
    d.set_channel(0);
    d.slot = 0;
    ws_release_all(d);
    for (int s : std::set<int>(slots.begin(), slots.end()))
        if (d.key_origin(s) != c.key_origin(s)) {
            // restrict_keys synchronises; an eager run of the same chain restricts first, and a graph's bind restricts for later clients
            if (recorded) c.refuse("would restrict a key slot's keys into the level (run the switch once eagerly first)");
            restrict_keys(d, c, s);
        }
    size_t total = 0;
    for (int i = 0; i < n; i++) total += in[i]->blocks;
    std::vector<BufRef> slab(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        d.set_channel(ch);
        slab[ch] = d.alloc(total * d.ct_words());
        std::vector<const u64 *> ptrs;
        for (int i = 0; i < n; i++)
            for (int b = 0; b < in[i]->blocks; b++) ptrs.push_back(in[i]->block(ch, b));
        op_mod_switch(c, d, ch, ptrs, slab[ch]->p);
    }
    d.set_channel(0);
    size_t ct = 0;
    for (int i = 0; i < n; i++) {
        out[i] = slab_output(d, slab, ct, in[i], in[i]->scale, slots[i]);
        ct += in[i]->blocks;
    }
    API_END
}
extern "C" int cnhe_vec_set_key_slot(cnhe_vec *v, int slot) {
    if (!v) return set_err(CNHE_ERR_INVALID, "null vector");
    std::lock_guard<std::recursive_mutex> lock(v->ctx->mu);
    if (!v->enc) return set_err(CNHE_ERR_INVALID, "plain vectors have no key slot");
    if (!v->ctx->slot_live(slot)) return set_err(CNHE_ERR_INVALID, "no such key slot");
    v->slot = slot;
    v->binding.reset();
    return CNHE_OK;
}
extern "C" int cnhe_vec_key_slot(const cnhe_vec *v, int *slot) {
    if (!v || !slot) return set_err(CNHE_ERR_INVALID, "null argument");
    *slot = v->enc ? v->key_slot() : -1;
    return CNHE_OK;
}
// Rotate (AtomicSealBfvVector.cs:1414-1430, first block only) of n vectors by the same amount, their key slots may differ: the hops of
// all vectors share each key-switch wave
static void rotate_vecs(Context &c, const cnhe_vec *const *vecs, int n, int amount, cnhe_vec **out) {
    if (n < 1 || !vecs || !out) fail("bad arguments");
    for (int i = 0; i < n; i++) {
        same_ctx(c, vecs[i]);
        if (!vecs[i]->enc) fail("Rotate operates only on encrypted data");
        if (vecs[i]->format == CNHE_SPARSE) fail("Rotate operates only on dense vectors");
    }
    const std::vector<int> slots = vec_slots(c, vecs, n);
    std::vector<std::unique_ptr<cnhe_vec>> outs(n);
    for (int i = 0; i < n; i++) {
        outs[i].reset(new_vec(c, vecs[i]->dim, vecs[i]->scale, CNHE_DENSE, true, 1));
        outs[i]->slot = slots[i];
        alloc_channels(outs[i].get());
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<RotateJob> jobs;
        for (int i = 0; i < n; i++) jobs.push_back({vecs[i]->ptr(ch), amount, outs[i]->ptr(ch), slots[i]});
        op_rotate_rows_multi(c, ch, jobs);
    }
    for (int i = 0; i < n; i++) out[i] = outs[i].release();
}
extern "C" int cnhe_vec_rotate(cnhe_ctx *h, const cnhe_vec *a, int amount, cnhe_vec **out) {
    API_BEGIN(h)
    rotate_vecs(c, &a, 1, amount, out);
    API_END
}
extern "C" int cnhe_vecs_rotate(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, int amount, cnhe_vec **out) {
    API_BEGIN(h)
    rotate_vecs(c, vecs, n, amount, out);
    API_END
}
extern "C" int cnhe_vecs_export_raw(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, uint64_t *dst, size_t cap) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (n < 1 || !dst) fail("bad arguments");
    const int blocks = vecs[0]->blocks;
    const size_t per = (size_t)blocks * c.ct_words();
    if (cap < (size_t)c.P * n * per) fail("destination too small");
    for (int i = 0; i < n; i++) {
        same_ctx(c, vecs[i]);
        if (!vecs[i]->enc || vecs[i]->blocks != blocks) fail("expecting encrypted vectors with equal block counts");
        for (int ch = 0; ch < c.P; ch++) {
            c.set_channel(ch);
            CNHE_CUDA(cudaMemcpyAsync(dst + ((size_t)ch * n + i) * per, vecs[i]->ptr(ch), per * 8, cudaMemcpyDeviceToHost, c.stream));
        }
    }
    c.sync();
    API_END
}
extern "C" int cnhe_vecs_export_raw_async(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, uint64_t *dst, size_t cap, int *ticket) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (n < 1 || !dst || !ticket) fail("bad arguments");
    const int blocks = vecs[0]->blocks;
    const size_t per = (size_t)blocks * c.ct_words();
    if (cap < (size_t)c.P * n * per) fail("destination too small");
    for (int i = 0; i < n; i++) {
        same_ctx(c, vecs[i]);
        if (!vecs[i]->enc || vecs[i]->blocks != blocks) fail("expecting encrypted vectors with equal block counts");
    }
    if (c.ev_export.empty()) {
        c.ev_export.resize((size_t)8 * c.P);
        for (cudaEvent_t &e : c.ev_export) CNHE_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    const int t = c.export_next;
    c.export_next = (c.export_next + 1) & 7;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        for (int i = 0; i < n; i++)
            CNHE_CUDA(cudaMemcpyAsync(dst + ((size_t)ch * n + i) * per, vecs[i]->ptr(ch), per * 8, cudaMemcpyDeviceToHost, c.stream));
        CNHE_CUDA(cudaEventRecord(c.ev_export[(size_t)t * c.P + ch], c.stream));
    }
    *ticket = t;
    API_END
}
extern "C" int cnhe_export_wait(cnhe_ctx *h, int ticket) {
    if (!h) return set_err(CNHE_ERR_INVALID, "null context");
    Context &c = *h->c;
    try {
        if (ticket < 0 || ticket > 7 || c.ev_export.empty()) fail("bad ticket");
        // no context lock: waiting must not block another thread that is queueing the next batch
        CNHE_CUDA(cudaSetDevice(c.device));
        for (int ch = 0; ch < c.P; ch++) CNHE_CUDA(cudaEventSynchronize(c.ev_export[(size_t)ticket * c.P + ch]));
    }
    catch (const Error &e) { return set_err(e.code, e.what()); }
    catch (const std::exception &e) { return set_err(CNHE_ERR_INVALID, e.what()); }
    return CNHE_OK;
}
extern "C" int cnhe_vec_device_ptr(const cnhe_vec *v, int channel, uint64_t *dptr, size_t *words) {
    if (!v || channel < 0 || channel >= v->ctx->P) return set_err(CNHE_ERR_INVALID, "bad arguments");
    cnhe_ctx h{v->ctx};
    API_BEGIN(&h)
    not_recorded(c, "hands device words to the caller");
    if (v->pend) { // the caller reads the words: relinearise them first
        materialise(c, v);
        c.sync();
    }
    *dptr = (uint64_t)v->ptr(channel);
    if (words) *words = (size_t)v->blocks * v->unit();
    API_END
}
extern "C" int cnhe_noise_budget(cnhe_ctx *h, const cnhe_vec *v, int channel, int block, int *bits) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    same_ctx(c, v);
    if (!v->enc || channel < 0 || channel >= c.P || block < 0 || block >= v->blocks) fail("bad arguments");
    if (v->key_slot() != 0) throw Error(CNHE_ERR_STATE, "the context holds no secret key of the vector's key slot");
    *bits = op_noise_budget(c, channel, v->block(channel, block));
    API_END
}

static double log2_centred(u64 v, u64 t) { // log2 |v| of a residue mod t read as a centred integer
    const double d = v > t / 2 ? (double)(t - v) : (double)v;
    return d > 0 ? std::log2(d) : 0;
}
// evaluator.Add/Sub/AddMany launches that also feed the operation counters / noise trace (OperationsCount, CryptoTracker)
static void do_add(Context &c, int ch, const u64 *a, const u64 *b, u64 *out, size_t words, int sub) {
    c.check(launch_ct_add(a, b, out, words, c.k, c.logN, c.d_bc, sub, c.stream), sub ? "ct_sub" : "ct_add");
    c.note(sub ? Context::OP_SUB : Context::OP_ADD, ch, (int)(words / c.ct_words()), out, a, b);
}
static void do_add_many(Context &c, int ch, const std::vector<const u64 *> &terms, u64 *out) {
    const int n_in = (int)terms.size();
    c.check(launch_ct_add_many(upload_ptrs(c, terms), n_in, out, c.ct_words(), c.k, c.logN, c.d_bc, c.stream), "ct_add_many");
    c.op_count[Context::OP_ADD_MANY_ITEMS] += (uint64_t)n_in;
    double aux = 0; // tracing: log2 of the root-sum-square of the items' noise peaks 2^-(budget+1), i.e. the model's prediction input
    if (c.trace_noise) {
        double ss = 0;
        bool all = true;
        for (const u64 *t : terms) { const int b = c.known_budget(t); if (b < 0) { all = false; break; } ss += std::exp2(-2.0 * (b + 1)); }
        aux = all && ss > 0 ? 0.5 * std::log2(ss) : 0;
    }
    c.note(Context::OP_ADD_MANY, ch, 1, out, terms.empty() ? nullptr : terms[0], nullptr, aux);
    if (c.trace_noise && !c.trace.empty()) c.trace.back().n = n_in;
}

// ---------------------------------------------------------------------------------------------------- IVector operations
static void check_pair(const cnhe_vec *a, const cnhe_vec *b) {
    if (a->dim != b->dim) fail("Dimensions do not match");
    if (a->format != b->format) fail("Format mismatch");
}
// Add / Subtract (AtomicSealBfvVector.cs:983-1024, 1238-1271; wrapper EncryptedSealBfvVector.cs:271-282, 457-471)
static cnhe_vec *addsub(Context &c, const cnhe_vec *a, const cnhe_vec *b, bool sub) {
    if (!sub && a->scale == 0) return alias_of(b);
    if (b->scale == 0) return alias_of(a);
    if (a->scale != b->scale) fail("Scales do not match.");
    check_pair(a, b);
    if (!a->enc && !b->enc) fail("adding two plaintexts is not supported");
    if (sub && !a->enc) fail("the first argument for subtraction must be encrypted");
    const cnhe_vec *e = a->enc ? a : b, *p = a->enc ? b : a;
    if (e->blocks != p->blocks) fail("Dimensions do not match");
    cnhe_vec *o = new_vec(c, a->dim, a->scale, a->format, true, e->blocks);
    alloc_channels(o);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        if (p->enc) {
            do_add(c, ch, a->ptr(ch), b->ptr(ch), o->ptr(ch), (size_t)e->blocks * c.ct_words(), sub);
        } else {
            const bool dense = p->format == CNHE_DENSE;
            c.check(launch_ct_add_plain(e->ptr(ch), o->ptr(ch), e->blocks, 2, p->ptr(ch), dense ? c.N : 1, dense ? (int)c.N : 1, c.k, c.logN, c.d_bc,
                                        c.ch[ch].pc, sub, c.stream),
                    "ct_add_plain");
            c.note(sub ? Context::OP_SUB_PLAIN : Context::OP_ADD_PLAIN, ch, e->blocks, o->ptr(ch), e->ptr(ch));
        }
    }
    return o;
}
extern "C" int cnhe_vec_add(cnhe_ctx *h, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, a); same_ctx(c, b);
    use_slot(c, {a, b});
    *out = addsub(c, a, b, false);
    API_END
}
extern "C" int cnhe_vec_sub(cnhe_ctx *h, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, a); same_ctx(c, b);
    use_slot(c, {a, b});
    *out = addsub(c, a, b, true);
    API_END
}

static std::vector<const u64 *> block_ptrs(const cnhe_vec *v, int ch, int repeat_first = 0) {
    std::vector<const u64 *> p;
    if (repeat_first) p.assign(repeat_first, v->block(ch, 0));
    else for (int b = 0; b < v->blocks; b++) p.push_back(v->block(ch, b));
    return p;
}
// PointwiseMultiplySparseDimOne (AtomicSealBfvVector.cs:774-810): `s` is the sparse dimension-one operand
static cnhe_vec *mul_sparse_dim_one(Context &c, const cnhe_vec *self, const cnhe_vec *s) {
    cnhe_vec *o = new_vec(c, self->dim, self->scale * s->scale, self->format, true, self->blocks);
    std::unique_ptr<cnhe_vec> guard(o);
    alloc_channels(o);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        if (self->enc && s->enc) {
            op_multiply_relin(c, ch, block_ptrs(s, ch, self->blocks), block_ptrs(self, ch), o->ptr(ch));
        } else if (self->enc) { // constant plaintext times every block
            std::vector<u64> sc(self->blocks, s->scalars[ch][0]);
            if (sc[0] == 0) fail("plain cannot be zero (the result would be a transparent ciphertext)");
            u64 *d = c.ws_alloc(sc.size());
            c.upload(d, sc.data(), sc.size() * 8);
            c.check(launch_ct_scale(self->ptr(ch), o->ptr(ch), self->blocks, 2, d, c.k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "ct_scale");
            c.note(Context::OP_MULTIPLY_SCALAR, ch, self->blocks, o->ptr(ch), self->ptr(ch), nullptr, log2_centred(sc[0], c.t[ch]));
            c.host_fence();
        } else { // plain blocks times the single ciphertext of s
            if (self->format != CNHE_DENSE) fail("unsupported plain format");
            u64 *rep = c.ws_alloc((size_t)self->blocks * c.ct_words());
            for (int b = 0; b < self->blocks; b++)
                { CNHE_CUDA(cudaMemcpyAsync(rep + (size_t)b * c.ct_words(), s->block(ch, 0), c.ct_words() * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(rep + (size_t)b * c.ct_words(), s->block(ch, 0)); }
            op_multiply_plain_dense(c, ch, rep, self->blocks, self->ptr(ch), true, o->ptr(ch));
        }
    }
    return guard.release();
}
// PointwiseMultiply (AtomicSealBfvVector.cs:813-860)
static cnhe_vec *pointwise_multiply(Context &c, const cnhe_vec *a, const cnhe_vec *b) {
    if (!a->enc && !b->enc) fail("multiplying two plaintexts is not implemented");
    if (a->dim == 1 && a->format == CNHE_SPARSE) return mul_sparse_dim_one(c, b, a);
    if (b->dim == 1 && b->format == CNHE_SPARSE) return mul_sparse_dim_one(c, a, b);
    check_pair(a, b);
    if (a->blocks != b->blocks) fail("Dimensions do not match");
    cnhe_vec *o = new_vec(c, a->dim, a->scale * b->scale, a->format, true, a->blocks);
    std::unique_ptr<cnhe_vec> guard(o);
    alloc_channels(o);
    const cnhe_vec *e = a->enc ? a : b, *p = a->enc ? b : a;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        if (a->enc && b->enc) {
            op_multiply_relin(c, ch, block_ptrs(b, ch), block_ptrs(a, ch), o->ptr(ch)); // evaluator.Multiply(ev.encData[i], encData[i])
        } else if (p->format == CNHE_DENSE) {
            op_multiply_plain_dense(c, ch, e->ptr(ch), e->blocks, p->ptr(ch), true, o->ptr(ch));
        } else {
            for (u64 s : p->scalars[ch])
                if (s == 0) fail("plain cannot be zero (the result would be a transparent ciphertext)");
            c.check(launch_ct_scale(e->ptr(ch), o->ptr(ch), e->blocks, 2, p->ptr(ch), c.k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "ct_scale");
            c.note(Context::OP_MULTIPLY_SCALAR, ch, e->blocks, o->ptr(ch), e->ptr(ch), nullptr, log2_centred(p->scalars[ch][0], c.t[ch]));
        }
    }
    return guard.release();
}
extern "C" int cnhe_vec_pointwise_multiply(cnhe_ctx *h, const cnhe_vec *a, const cnhe_vec *b, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, a); same_ctx(c, b);
    use_slot(c, {a, b});
    *out = pointwise_multiply(c, a, b);
    API_END
}

// The rotate-and-add ladder of SumAllSlots (AtomicSealBfvVector.cs:888-955) on n single-block ciphertexts in place, one key-switch wave per
// step for all n; returns the summed length.  slots: per-ciphertext key slots (nullptr: the call's slot).  The folded diagonal product
// starts the row steps at `first` (its fold width) and skips the column step when `columns` is false.
static uint64_t sum_slots_batched(Context &c, int ch, u64 *cts, int n, uint64_t length, const int *slots = nullptr, uint64_t first = 1,
                                  bool columns = true) {
    const size_t N = c.N, words = (size_t)n * c.ct_words();
    uint64_t len = length;
    u64 *tmp = c.ws_alloc(words);
    // every step is x += rotate(x): fused into the rotation (the permutation kernel folds x into the key switch's base) when the step
    // has its own Galois key -- it does for the powers of two the ladder walks -- else rotate, then add
    if (len >= N / 2) {
        if (columns && !op_rotate_add(c, ch, cts, n, 0, true, cts, slots)) {
            op_rotate_columns(c, ch, cts, n, tmp, slots);
            do_add(c, ch, cts, tmp, cts, words, 0);
        }
        len = N / 2;
    }
    for (uint64_t steps = first; steps < len; steps *= 2) { // RotateRowsAndAdd(sum, steps): RotateRows(c, -steps)
        if (op_rotate_add(c, ch, cts, n, -(int)steps, false, cts, slots)) continue;
        op_rotate_rows(c, ch, cts, n, -(int)steps, tmp, slots);
        do_add(c, ch, cts, tmp, cts, words, 0);
    }
    return len;
}
// SumAllSlots (AtomicSealBfvVector.cs:888-955)
static cnhe_vec *sum_all_slots(Context &c, const cnhe_vec *a, uint64_t length, int force_column) {
    if (a->format != CNHE_DENSE) fail("Expecting dense vector format");
    if (length != CNHE_ALL_SLOTS && force_column >= 0) fail("forcing output in a column works only when doing complete sum");
    if (!a->enc) fail("SumAllSlots can be applied to encrypted data only");
    if (length == 0) fail("Can't sum over less then one element");
    if (length == 1) return alias_of(a);
    const size_t N = c.N, ctw = c.ct_words();
    uint64_t len = length;
    cnhe_vec *o = new_vec(c, a->dim, a->scale, CNHE_DENSE, true, 1);
    std::unique_ptr<cnhe_vec> guard(o);
    alloc_channels(o);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        u64 *sum = o->ptr(ch);
        if (a->blocks > 1) { // AddMany over the blocks
            std::vector<const u64 *> ptrs = block_ptrs(a, ch);
            do_add_many(c, ch, ptrs, sum);
        } else {
            CNHE_CUDA(cudaMemcpyAsync(sum, a->ptr(ch), ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(sum, a->ptr(ch));
        }
        len = sum_slots_batched(c, ch, sum, 1, length);
        if (force_column >= 0) { // one-hot mask (":936-945")
            if ((size_t)force_column >= N) fail("column out of range");
            std::vector<u64> onehot(N, 0);
            onehot[force_column] = 1;
            u64 *dv = c.ws_alloc(N), *pl = c.ws_alloc(N);
            c.upload(dv, onehot.data(), N * 8);
            op_encode(c, ch, dv, 1, (int)N, pl);
            op_multiply_plain_dense(c, ch, sum, 1, pl, false, sum);
            c.host_fence();
            len = 1;
        }
    }
    o->dim = (len >= N / 2) ? 1 : a->dim;
    o->format = (len >= N) ? CNHE_SPARSE : CNHE_DENSE;
    return guard.release();
}
extern "C" int cnhe_vec_sum_all_slots(cnhe_ctx *h, const cnhe_vec *a, uint64_t length, int force_column, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, a);
    use_slot(c, {a});
    *out = sum_all_slots(c, a, length, force_column);
    API_END
}
extern "C" int cnhe_vec_dot_product(cnhe_ctx *h, const cnhe_vec *a, const cnhe_vec *b, uint64_t length, int force_column, cnhe_vec **out) {
    API_BEGIN(h)
    same_ctx(c, a); same_ctx(c, b);
    use_slot(c, {a, b});
    std::unique_ptr<cnhe_vec> mul(pointwise_multiply(c, a, b)); // AtomicSealBfvVector.cs:964-977
    *out = sum_all_slots(c, mul.get(), length, force_column);
    API_END
}
// GenerateSparseOfArray (AtomicSealBfvVector.cs:1347-1359)
extern "C" int cnhe_vecs_generate_sparse_of_array(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, cnhe_vec **out) {
    API_BEGIN(h)
    if (n < 1) fail("empty array");
    for (int i = 0; i < n; i++) { same_ctx(c, vecs[i]); if (!vecs[i]->enc) fail("expecting encrypted vectors"); }
    use_slot(c, vecs, n);
    cnhe_vec *o = new_vec(c, (uint64_t)n, vecs[0]->scale, CNHE_SPARSE, true, n);
    alloc_channels(o);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        for (int i = 0; i < n; i++)
            { CNHE_CUDA(cudaMemcpyAsync(o->block(ch, i), vecs[i]->block(ch, 0), c.ct_words() * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(o->block(ch, i), vecs[i]->block(ch, 0)); }
    }
    *out = o;
    API_END
}

// Inteleave (AtomicSealBfvVector.cs:600-722): place vector k at slot offset shift*k
// Phase 1 of one interleave: where every vector goes, and the rotation jobs that put it there (under key slot `slot`)
struct Placed { int kind, start_block, end_block, in_block; u64 *v; }; // kind 0 lower, 1 upper, 2 straddles into the next block, 3 straddles lower/upper
static void interleave_place(Context &c, int ch, const std::vector<const cnhe_vec *> &vecs, int shift, int out_blocks, int slot,
                             std::vector<Placed> &placed, std::vector<RotateJob> &jobs) {
    const int block_size = (int)c.N, half = block_size / 2;
    const size_t ctw = c.ct_words();
    const int abs_shift = shift < 0 ? -shift : shift;
    if (shift < 0 && out_blocks > 1) fail("Negative shifts with multiple output blocks are not implemented yet");
    if (abs_shift > half && out_blocks > 1) fail("Shifts of more than half block size with multiple output blocks are not implemented yet");
    if ((long long)abs_shift * (long long)vecs.size() > (long long)block_size * out_blocks) fail("not enough room for interleaving");
    // every vector's rotation (RotateRowsInplace of its own offset, ":625-660") -- independent of each other, so they are queued and
    // executed together: hops with the same Galois element share one key-switch wave (same per-ciphertext operations and order as one
    // rotate_rows call per vector, hence the same ciphertexts)
    placed.assign(vecs.size(), Placed{});
    for (size_t kk = 0; kk < vecs.size(); kk++) {
        long long this_shift = (long long)shift * (long long)kk;
        if (this_shift < 0) this_shift = half + this_shift;
        const int in_block = (int)(this_shift % block_size);
        const int start_block = (int)(this_shift / block_size), end_block = (int)((this_shift + abs_shift) / block_size);
        u64 *v = c.ws_alloc(ctw);
        const u64 *src = vecs[kk]->block(ch, 0);
        Placed &pl = placed[kk];
        pl.start_block = start_block; pl.end_block = end_block; pl.in_block = in_block; pl.v = v;
        if (in_block == 0) {
            CNHE_CUDA(cudaMemcpyAsync(v, src, ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(v, src);
            pl.kind = 0;
        } else if (in_block + abs_shift < half) {
            jobs.push_back({src, -(int)this_shift, v, slot});
            pl.kind = 0;
        } else if (in_block >= half) {
            jobs.push_back({src, -(in_block - half), v, slot});
            pl.kind = start_block == end_block ? 1 : 2;
        } else {
            jobs.push_back({src, -in_block, v, slot});
            pl.kind = 3;
        }
    }
}
// Phase 2 (after the rotation jobs ran): split the vectors that straddle a half / block boundary and sum every output block; key
// switches use the call's slot c.slot
static void interleave_finish(Context &c, int ch, const std::vector<const cnhe_vec *> &vecs, int shift, int out_blocks,
                              const std::vector<Placed> &placed, u64 *out) {
    const int block_size = (int)c.N, half = block_size / 2;
    const size_t ctw = c.ct_words();
    const int abs_shift = shift < 0 ? -shift : shift;
    std::vector<std::vector<const u64 *>> lower(out_blocks), upper(out_blocks);
    auto ones_plain = [&](int count) { // BatchEncoder.Encode of `count` ones
        std::vector<u64> v(block_size, 0);
        for (int i = 0; i < count; i++) v[i] = 1;
        u64 *dv = c.ws_alloc(block_size), *pl = c.ws_alloc(block_size);
        c.upload(dv, v.data(), (size_t)block_size * 8);
        op_encode(c, ch, dv, 1, block_size, pl);
        c.host_fence();
        return pl;
    };
    // split the vectors that straddle a half / block boundary with a one-hot-prefix mask (":640-672") and file every piece
    for (size_t kk = 0; kk < vecs.size(); kk++) {
        const Placed &pl = placed[kk];
        u64 *v = pl.v;
        const int start_block = pl.start_block, end_block = pl.end_block, in_block = pl.in_block;
        if (pl.kind == 0) {
            lower[start_block].push_back(v);
        } else if (pl.kind == 1) {
            upper[start_block].push_back(v);
        } else if (pl.kind == 2) { // straddles the upper half of this block and the lower half of the next
            const int upper_part = (in_block + abs_shift) - block_size;
            u64 *v2 = c.ws_alloc(ctw);
            CNHE_CUDA(cudaMemcpyAsync(v2, v, ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(v2, v);
            op_multiply_plain_dense(c, ch, v, 1, ones_plain(upper_part), false, v);
            do_add(c, ch, v2, v, v2, ctw, 1);
            upper[start_block].push_back(v2);
            if (end_block >= out_blocks) fail("not enough room for interleaving");
            lower[end_block].push_back(v);
        } else { // straddles lower and upper half of the same block
            const int upper_part = (in_block + abs_shift) - half;
            if (upper_part > 0) {
                u64 *v2 = c.ws_alloc(ctw);
                CNHE_CUDA(cudaMemcpyAsync(v2, v, ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(v2, v);
                op_multiply_plain_dense(c, ch, v, 1, ones_plain(upper_part), false, v);
                do_add(c, ch, v2, v, v2, ctw, 1);
                upper[start_block].push_back(v);
                lower[start_block].push_back(v2);
            } else {
                lower[start_block].push_back(v);
            }
        }
    }
    for (int i = 0; i < out_blocks; i++) {
        u64 *res = out + (size_t)i * ctw;
        if (lower[i].empty()) fail("an output block received no vector");
        do_add_many(c, ch, lower[i], res);
        if (!upper[i].empty()) {
            u64 *t = c.ws_alloc(ctw);
            do_add_many(c, ch, upper[i], t);
            op_rotate_columns(c, ch, t, 1, t);
            do_add(c, ch, res, t, res, ctw, 0);
        }
    }
}
// Interleave (AtomicSealBfvVector.cs:729-750) of B groups of n vectors each, one output per group; the groups' key slots may differ (one
// LoLa vectorize layer per client).  The rotations of all groups run as one set of jobs (one key-switch wave per hop for all groups), then
// each group's masks and sums under its own slot: out[b] is bit-identical to the interleave of group b alone.  stack: Stack
// (":756-761"), the interleave with shift = dim whose output has dimension dim * n; otherwise every group takes `shift`.
static void interleave_groups(Context &c, const cnhe_vec *const *vecs, int n, int B, int shift, bool stack, cnhe_vec **out) {
    if (n < 1 || B < 1 || !vecs || !out) fail("bad arguments");
    struct Group { std::vector<const cnhe_vec *> vecs; int shift, out_blocks, slot; std::vector<Placed> placed; };
    std::vector<Group> gs(B);
    bool foreign = false;
    for (int b = 0; b < B; b++) {
        Group &g = gs[b];
        g.vecs.assign(vecs + (size_t)b * n, vecs + (size_t)(b + 1) * n);
        for (auto v : g.vecs) { same_ctx(c, v); if (!v->enc) fail("expecting encrypted vectors"); }
        if (g.vecs[0]->format != CNHE_DENSE) fail("Expecting dense vector");
        g.slot = use_slot(c, g.vecs.data(), n);
        foreign = foreign || g.slot != 0;
        g.shift = stack ? (int)g.vecs[0]->dim : shift;
        g.out_blocks = g.shift > 0 ? (int)std::ceil((double)(g.vecs[0]->dim * (uint64_t)n) / (double)c.N) : 1;
    }
    c.foreign = foreign;
    std::vector<std::unique_ptr<cnhe_vec>> outs(B);
    for (int b = 0; b < B; b++) {
        c.slot = gs[b].slot;
        outs[b].reset(new_vec(c, gs[b].vecs[0]->dim, gs[b].vecs[0]->scale, CNHE_DENSE, true, gs[b].out_blocks));
        alloc_channels(outs[b].get());
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<RotateJob> jobs;
        for (Group &g : gs) interleave_place(c, ch, g.vecs, g.shift, g.out_blocks, g.slot, g.placed, jobs);
        op_rotate_rows_multi(c, ch, jobs);
        for (int b = 0; b < B; b++) {
            c.slot = gs[b].slot;
            interleave_finish(c, ch, gs[b].vecs, gs[b].shift, gs[b].out_blocks, gs[b].placed, outs[b]->ptr(ch));
        }
    }
    for (int b = 0; b < B; b++) {
        if (stack) outs[b]->dim *= (uint64_t)n;
        out[b] = outs[b].release();
    }
}
extern "C" int cnhe_vecs_interleave(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, int shift, cnhe_vec **out) {
    API_BEGIN(h)
    interleave_groups(c, vecs, n, 1, shift, false, out);
    API_END
}
extern "C" int cnhe_vecs_stack(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, cnhe_vec **out) {
    API_BEGIN(h)
    interleave_groups(c, vecs, n, 1, 0, true, out);
    API_END
}
// cnhe_vecs_stack of B groups of n vectors each: out[b] is bit-identical to cnhe_vecs_stack(vecs + b * n, n)
extern "C" int cnhe_vecs_stack_batch(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, int B, cnhe_vec **out) {
    API_BEGIN(h)
    interleave_groups(c, vecs, n, B, 0, true, out);
    API_END
}
// cnhe_vecs_interleave of B groups of n vectors each: out[b] is bit-identical to cnhe_vecs_interleave(vecs + b * n, n, shift)
extern "C" int cnhe_vecs_interleave_batch(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, int B, int shift, cnhe_vec **out) {
    API_BEGIN(h)
    interleave_groups(c, vecs, n, B, shift, false, out);
    API_END
}

// ---------------------------------------------------------------------------------------------------- one operation, B clients
// The B inputs of a batched vector operation: the same context, live key slots, and one dim, scale, format and block count
static std::vector<int> batch_inputs(Context &c, const cnhe_vec *const *vecs, int B, cnhe_vec **out) {
    if (!vecs || B < 1 || !out) fail("bad arguments");
    for (int b = 0; b < B; b++) {
        same_ctx(c, vecs[b]);
        if (vecs[b]->dim != vecs[0]->dim || vecs[b]->scale != vecs[0]->scale || vecs[b]->format != vecs[0]->format ||
            vecs[b]->blocks != vecs[0]->blocks || vecs[b]->enc != vecs[0]->enc)
            fail("the input vectors must share dimension, scale, format and block count");
    }
    return vec_slots(c, vecs, B);
}
// B single-ciphertext outputs in one slab per channel, bound to their inputs' slots
static std::vector<std::unique_ptr<cnhe_vec>> batch_outputs(Context &c, int n, const std::vector<int> &slot_of, uint64_t dim, double scale) {
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        big[ch] = c.alloc((size_t)n * c.ct_words());
    }
    std::vector<std::unique_ptr<cnhe_vec>> outs(n);
    for (int i = 0; i < n; i++) {
        outs[i].reset(slab_view(new_vec(c, dim, scale, CNHE_DENSE, true, 1), big, (size_t)i));
        outs[i]->slot = slot_of[i];
    }
    return outs;
}
// Duplicate (AtomicSealBfvVector.cs:1370-1408) of B vectors (one per client; key slots may differ): the column rotations in one call,
// every client's count - 1 row rotations in one op_rotate_rows_multi, then each client's additions in the reference's order
static void duplicate_vecs(Context &c, const cnhe_vec *const *vecs, int B, uint64_t count, cnhe_vec **out) {
    const std::vector<int> slots = batch_inputs(c, vecs, B, out);
    const cnhe_vec *a = vecs[0];
    uint64_t shift = 1;
    while (shift < a->dim) shift *= 2;
    if (!a->enc) fail("Duplicate operates only on encrypted data");
    if (a->format == CNHE_SPARSE) fail("Duplicate operates only on dense vectors");
    const size_t N = c.N, ctw = c.ct_words();
    if (shift * count > N) fail("Packed vector must fit in a single ciphertext");
    auto outs = batch_outputs(c, B, slots, count * shift, a->scale);
    bool column = false;
    for (uint64_t i = 1; i < count; i++) column = column || (long long)(i * shift) * 2 >= (long long)N;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        u64 *rotator = nullptr;
        if (column) { // rotate_columns of every input (":1387-1394"); several are gathered so that one call serves all, one is read in place
            const u64 *in = vecs[0]->ptr(ch);
            if (B > 1) {
                u64 *g = c.ws_alloc((size_t)B * ctw);
                for (int b = 0; b < B; b++)
                    { CNHE_CUDA(cudaMemcpyAsync(g + (size_t)b * ctw, vecs[b]->ptr(ch), ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(g + (size_t)b * ctw, vecs[b]->ptr(ch)); }
                in = g;
            }
            rotator = c.ws_alloc((size_t)B * ctw);
            op_rotate_columns(c, ch, in, B, rotator, slots.data());
        }
        std::vector<RotateJob> jobs;
        std::vector<u64 *> pieces;
        for (int b = 0; b < B; b++) {
            u64 *res = outs[b]->ptr(ch);
            CNHE_CUDA(cudaMemcpyAsync(res, vecs[b]->ptr(ch), ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(res, vecs[b]->ptr(ch));
            for (uint64_t i = 1; i < count; i++) {
                long long target = (long long)(i * shift);
                const u64 *src = vecs[b]->ptr(ch);
                if (target * 2 >= (long long)N) {
                    src = rotator + (size_t)b * ctw;
                    target -= (long long)N / 2;
                }
                u64 *tmp = c.ws_alloc(ctw);
                jobs.push_back({src, -(int)target, tmp, slots[b]});
                pieces.push_back(tmp);
            }
        }
        op_rotate_rows_multi(c, ch, jobs);
        const size_t per = count > 0 ? count - 1 : 0;
        for (int b = 0; b < B; b++)
            for (size_t i = 0; i < per; i++) do_add(c, ch, outs[b]->ptr(ch), pieces[b * per + i], outs[b]->ptr(ch), ctw, 0);
    }
    for (int b = 0; b < B; b++) out[b] = outs[b].release();
}
extern "C" int cnhe_vec_duplicate(cnhe_ctx *h, const cnhe_vec *a, uint64_t count, cnhe_vec **out) {
    API_BEGIN(h)
    duplicate_vecs(c, &a, 1, count, out);
    API_END
}
extern "C" int cnhe_vecs_duplicate_batch(cnhe_ctx *h, const cnhe_vec *const *vecs, int B, uint64_t count, cnhe_vec **out) {
    API_BEGIN(h)
    duplicate_vecs(c, vecs, B, count, out);
    API_END
}
// Permute (AtomicSealBfvVector.cs:1436-1475) of B vectors (one per client) with the same n_perm permutations of n_sel selections each:
// out[b * n_perm + j] permutes vecs[b] with selections + j * n_sel and shifts + j * n_sel.  Per wave of clients the mask products are one
// outer product of the clients and the distinct selections, and every (client, permutation, selection) rotation goes into one
// op_rotate_rows_multi; then each output's sum in the reference's order (":1446-1461").
static void permute_vecs(Context &c, const cnhe_vec *const *vecs, int B, const cnhe_vec *const *selections, const int *shifts, int n_perm,
                         int n_sel, uint64_t output_dim, cnhe_vec **out) {
    const std::vector<int> slots = batch_inputs(c, vecs, B, out);
    if (!selections || !shifts || n_perm < 1 || n_sel < 1) fail("bad arguments");
    const cnhe_vec *a = vecs[0];
    if (a->format != CNHE_DENSE) fail("Permute works only on dense vectors");
    if (!a->enc) fail("can permute only encrypted vectors");
    if (a->blocks > 1) fail("can permute only a single block");
    std::vector<int> sel_index((size_t)n_perm * n_sel, -1); // each non-null selection's place among the distinct ones
    std::vector<const cnhe_vec *> distinct;
    std::vector<double> out_scale(n_perm);
    for (int j = 0; j < n_perm; j++) {
        const cnhe_vec *const *sel = selections + (size_t)j * n_sel;
        int first = -1;
        for (int i = 0; i < n_sel; i++) {
            if (!sel[i]) continue;
            same_ctx(c, sel[i]);
            if (first < 0) first = i;
            if (sel[i]->dim != a->dim) fail("dimension of selection vector does not match dimension of data vector");
            if (sel[i]->scale != sel[first]->scale) fail("scales of all selection vectors should be the same");
            if (sel[i]->enc) fail("encrypted size must be 2 (rotating the size-3 product of an encrypted selection is rejected by SEAL)");
            if (sel[i]->format != CNHE_DENSE) fail("selection vectors must be dense");
            const size_t d = std::find(distinct.begin(), distinct.end(), sel[i]) - distinct.begin();
            if (d == distinct.size()) distinct.push_back(sel[i]);
            sel_index[(size_t)j * n_sel + i] = (int)d;
        }
        if (first < 0) fail("permuting with no selected values is illigal");
        out_scale[j] = a->scale * sel[first]->scale;
    }
    const int S = (int)distinct.size(), terms = (int)std::count_if(sel_index.begin(), sel_index.end(), [](int s) { return s >= 0; });
    const size_t N = c.N, ctw = c.ct_words();
    std::vector<int> out_slot((size_t)B * n_perm);
    for (size_t o = 0; o < out_slot.size(); o++) out_slot[o] = slots[o / n_perm];
    auto outs = batch_outputs(c, B * n_perm, out_slot, output_dim, 0);
    for (int b = 0; b < B; b++)
        for (int j = 0; j < n_perm; j++) outs[(size_t)b * n_perm + j]->scale = out_scale[j];
    // clients per wave: their products and rotated terms stay under 8 GiB
    const int BW = (int)std::max<size_t>(1, ((size_t)1 << 30) / ((size_t)(S + terms) * ctw));
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        u64 *plains = c.ws_alloc((size_t)S * N);
        for (int s = 0; s < S; s++) CNHE_CUDA(cudaMemcpyAsync(plains + (size_t)s * N, distinct[s]->ptr(ch), N * 8, cudaMemcpyDeviceToDevice, c.stream));
        for (int b0 = 0; b0 < B; b0 += BW) {
            WsScope wave(c);
            const int nb = std::min(BW, B - b0);
            u64 *prod = c.ws_alloc((size_t)nb * S * ctw), *rot = c.ws_alloc((size_t)nb * terms * ctw);
            std::vector<const u64 *> cts(nb);
            for (int j = 0; j < nb; j++) cts[j] = vecs[b0 + j]->ptr(ch);
            op_multiply_plain_dense_outer(c, ch, cts, plains, S, prod);
            c.op_count[Context::OP_MULTIPLY_PLAIN] += (uint64_t)nb * (terms - S); // one per term, as the reference issues them
            std::vector<RotateJob> jobs; // (client, permutation, selection) in that order: the terms of an output are consecutive
            for (int bb = 0; bb < nb; bb++)
                for (size_t q = 0; q < sel_index.size(); q++)
                    if (sel_index[q] >= 0)
                        jobs.push_back({prod + ((size_t)bb * S + sel_index[q]) * ctw, shifts[q], rot + jobs.size() * ctw, slots[b0 + bb]});
            op_rotate_rows_multi(c, ch, jobs);
            const u64 *r = rot;
            for (int bb = 0; bb < nb; bb++)
                for (int j = 0; j < n_perm; j++) {
                    u64 *o = outs[(size_t)(b0 + bb) * n_perm + j]->ptr(ch);
                    for (int i = 0, have = 0; i < n_sel; i++) {
                        if (sel_index[(size_t)j * n_sel + i] < 0) continue;
                        if (!have) { CNHE_CUDA(cudaMemcpyAsync(o, r, ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(o, r); }
                        else do_add(c, ch, o, r, o, ctw, 0);
                        have = 1;
                        r += ctw;
                    }
                }
        }
    }
    for (size_t o = 0; o < outs.size(); o++) out[o] = outs[o].release();
}
extern "C" int cnhe_vec_permute(cnhe_ctx *h, const cnhe_vec *a, const cnhe_vec *const *selections, const int *shifts, int n, uint64_t output_dim,
                                cnhe_vec **out) {
    API_BEGIN(h)
    permute_vecs(c, &a, 1, selections, shifts, 1, n, output_dim, out);
    API_END
}
extern "C" int cnhe_vecs_permute_batch(cnhe_ctx *h, const cnhe_vec *const *vecs, int B, const cnhe_vec *const *selections, const int *shifts,
                                       int n_perm, int n_sel, uint64_t output_dim, cnhe_vec **out) {
    API_BEGIN(h)
    permute_vecs(c, vecs, B, selections, shifts, n_perm, n_sel, output_dim, out);
    API_END
}
// cnhe_vec_pointwise_multiply(vecs[i], plain) of n encrypted vectors and one plain dense vector, one outer product per channel and block:
// out[i] is bit-identical to the single call
extern "C" int cnhe_vecs_multiply_plain(cnhe_ctx *h, const cnhe_vec *const *vecs, int n, const cnhe_vec *plain, cnhe_vec **out) {
    API_BEGIN(h)
    const std::vector<int> slots = batch_inputs(c, vecs, n, out);
    same_ctx(c, plain);
    const cnhe_vec *a = vecs[0];
    if (!a->enc) fail("multiplying two plaintexts is not implemented");
    if (plain->enc || plain->format != CNHE_DENSE) fail("expecting a plain dense vector");
    check_pair(a, plain);
    if (a->blocks != plain->blocks) fail("Dimensions do not match");
    const int bl = a->blocks;
    const size_t ctw = c.ct_words();
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        big[ch] = c.alloc((size_t)n * bl * ctw);
    }
    std::vector<std::unique_ptr<cnhe_vec>> outs(n);
    for (int i = 0; i < n; i++) {
        outs[i].reset(slab_view(new_vec(c, a->dim, a->scale * plain->scale, a->format, true, bl), big, (size_t)i * bl));
        outs[i]->slot = slots[i];
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        for (int j = 0; j < bl; j++) {
            std::vector<const u64 *> cts(n);
            for (int i = 0; i < n; i++) cts[i] = vecs[i]->block(ch, j);
            u64 *dst = bl == 1 ? big[ch]->p : c.ws_alloc((size_t)n * ctw);
            op_multiply_plain_dense_outer(c, ch, cts, plain->block(ch, j), 1, dst);
            if (bl > 1)
                for (int i = 0; i < n; i++)
                    CNHE_CUDA(cudaMemcpyAsync(outs[i]->block(ch, j), dst + (size_t)i * ctw, ctw * 8, cudaMemcpyDeviceToDevice, c.stream));
        }
    }
    for (int i = 0; i < n; i++) out[i] = outs[i].release();
    API_END
}

// ---------------------------------------------------------------------------------------------------- matrix x vector, layers
struct RowHash {
    size_t operator()(const std::vector<int> &r) const {
        size_t hsh = 1469598103934665603ULL;
        for (int v : r) hsh = (hsh ^ (size_t)(unsigned)v) * 1099511628211ULL;
        return hsh;
    }
};
// ---- plan of a scalar-MAC layer for the wgmma kernel (mac_umma.cu): bundles of consecutive distinct gather rows
struct UmmaPlan {
    bool ok = false;
    std::vector<UmBundle> bundles;
    std::vector<int> chunk_rows;
    std::vector<unsigned char> wpack;
    std::vector<int> out_order;  // output index per (bundle, row)
    std::vector<int> extra_taps; // input index of every scratch-slab row (taps whose weights need the W2 part)
    int total_chunks = 0;
    // device copies (owned by the cache entry)
    UmBundle *d_bundles = nullptr;
    int *d_rows = nullptr;
    unsigned char *d_wpack = nullptr;
    ~UmmaPlan() {
        if (d_bundles) cudaFree(d_bundles);
        if (d_rows) cudaFree(d_rows);
        if (d_wpack) cudaFree(d_wpack);
    }
};
// bundles of `g` consecutive distinct rows; returns false when a bundle exceeds 128 outputs or a weight exceeds +-254
static bool umma_try(UmmaPlan &pl, int g, const std::vector<int> &grows, const std::vector<std::vector<int>> &row_outs, const std::vector<double> &wdh, int K) {
    const int R = (int)row_outs.size();
    std::unordered_map<std::string, int> seen;
    for (int start = 0; start < R; start += g) {
        const int end = std::min(R, start + g);
        std::vector<int> outs, out_row;
        int tmin = INT_MAX, tmax = -1;
        for (int r = start; r < end; r++) {
            for (int m : row_outs[r]) { outs.push_back(m); out_row.push_back(r); }
            for (int kk = 0; kk < K; kk++) {
                const int t = grows[(size_t)r * K + kk];
                if (t >= 0) { tmin = std::min(tmin, t); tmax = std::max(tmax, t); }
            }
        }
        if (outs.empty() || outs.size() > 128 || tmax < 0) return false;
        const int cols_main = ((tmax - tmin + 1) + 31) / 32 * 32;
        std::vector<int> wfull(outs.size() * (size_t)cols_main, 0);
        for (size_t i = 0; i < outs.size(); i++)
            for (int kk = 0; kk < K; kk++) {
                const int t = grows[(size_t)out_row[i] * K + kk];
                if (t >= 0) wfull[i * cols_main + (t - tmin)] += (int)wdh[(size_t)outs[i] * K + kk];
            }
        std::vector<int> extras; // columns that hold a weight beyond one signed byte
        for (int col = 0; col < cols_main; col++) {
            bool big = false;
            for (size_t i = 0; i < outs.size(); i++) {
                const int w = wfull[i * cols_main + col];
                if (w > 254 || w < -254) return false;
                big = big || w > 127 || w < -127;
            }
            if (big) extras.push_back(col);
        }
        const int cols = cols_main + ((int)extras.size() + 31) / 32 * 32;
        std::vector<signed char> w8(outs.size() * (size_t)cols, 0);
        for (size_t i = 0; i < outs.size(); i++) {
            for (int col = 0; col < cols_main; col++) w8[i * cols + col] = (signed char)std::max(-127, std::min(127, wfull[i * cols_main + col]));
            for (size_t j = 0; j < extras.size(); j++) {
                const int w = wfull[i * cols_main + extras[j]];
                w8[i * cols + cols_main + j] = (signed char)(w - std::max(-127, std::min(127, w)));
            }
        }
        std::string blob((size_t)cols / 32 * 4096, '\0');
        mac_umma_pack(w8.data(), (int)outs.size(), cols, reinterpret_cast<unsigned char *>(&blob[0]));
        UmBundle b;
        auto it = seen.find(blob);
        if (it == seen.end()) { // interior rows of a convolution share one matrix: the window slides with the bundle
            b.a_off = (int)pl.wpack.size();
            seen.emplace(blob, b.a_off);
            pl.wpack.insert(pl.wpack.end(), blob.begin(), blob.end());
        } else
            b.a_off = it->second;
        b.chunk0 = (int)pl.chunk_rows.size();
        b.n_chunks = cols / 32;
        b.n_out = (int)outs.size();
        b.out0 = (int)pl.out_order.size();
        for (int cch = 0; cch < cols_main / 32; cch++) pl.chunk_rows.push_back(tmin + 32 * cch);
        for (int cch = 0; cch < (cols - cols_main) / 32; cch++) pl.chunk_rows.push_back((1 << 30) | ((int)pl.extra_taps.size() + 32 * cch));
        for (int col : extras) pl.extra_taps.push_back(tmin + col);
        pl.out_order.insert(pl.out_order.end(), outs.begin(), outs.end());
        pl.bundles.push_back(b);
        pl.total_chunks += b.n_chunks;
    }
    return true;
}
// the search itself (host only): every bundle size g = 1, 2, ... rows; the plan with the fewest chunks per tile that fits in shared memory
static std::shared_ptr<UmmaPlan> umma_search(const std::vector<int> &grows, const std::vector<std::vector<int>> &row_outs, const std::vector<double> &wdh,
                                             int M, int K, int limbs) {
    std::shared_ptr<UmmaPlan> best;
    const int R = (int)row_outs.size();
    for (int g = 1; g <= R; g++) {
        auto pl = std::make_shared<UmmaPlan>();
        if (!umma_try(*pl, g, grows, row_outs, wdh, K)) {
            if (g > 1 && (size_t)g * row_outs[0].size() > 128) break; // larger groups only grow
            continue;
        }
        if (!mac_umma_fits((int)pl->wpack.size(), pl->total_chunks, M, (int)pl->bundles.size(), limbs)) continue;
        if (!best || pl->total_chunks < best->total_chunks) best = pl;
        if (g > 64) break;
    }
    return best;
}
// Planner probe for the CPU test suite (not part of include/cnhe.h, needs no GPU): gather[M][K] (-1 = padded tap), signed integer weights
// w[M][K]; out = {bundles, chunks per tile, weight bytes after de-duplication, extra (W2) taps}; returns 0 when no plan fits.
extern "C" int cnhe_debug_mac_plan(const int32_t *gather, const double *w, int M, int K, int limbs, int *out) {
    std::unordered_map<std::vector<int>, int, RowHash> index;
    std::vector<int> grows;
    std::vector<std::vector<int>> row_outs;
    for (int m = 0; m < M; m++) {
        std::vector<int> row(gather + (size_t)m * K, gather + (size_t)(m + 1) * K);
        auto it = index.find(row);
        if (it == index.end()) {
            index.emplace(row, (int)row_outs.size());
            grows.insert(grows.end(), row.begin(), row.end());
            row_outs.push_back({m});
        } else
            row_outs[it->second].push_back(m);
    }
    std::vector<double> wdh(w, w + (size_t)M * K);
    std::shared_ptr<UmmaPlan> pl = umma_search(grows, row_outs, wdh, M, K, limbs);
    if (!pl) return 0;
    out[0] = (int)pl->bundles.size(); out[1] = pl->total_chunks; out[2] = (int)pl->wpack.size(); out[3] = (int)pl->extra_taps.size();
    return 1;
}
// fewest chunks per tile over the bundle sizes that fit in shared memory; cached per layer (keyed by a hash of its gather table and weights)
static std::shared_ptr<UmmaPlan> umma_plan(Context &c, int ch, const std::vector<int> &grows, const std::vector<std::vector<int>> &row_outs,
                                           const std::vector<double> &wdh, int M, int K, int limbs) {
    u64 key = 0xcbf29ce484222325ULL ^ (u64)ch * 0x9e3779b97f4a7c15ULL ^ ((u64)M << 32) ^ (u64)K;
    auto mix = [&](const void *p, size_t bytes) {
        const u64 *w = reinterpret_cast<const u64 *>(p);
        for (size_t i = 0; i < bytes / 8; i++) { key ^= w[i]; key *= 0x100000001b3ULL; key ^= key >> 29; }
    };
    mix(wdh.data(), wdh.size() * 8);
    {
        std::vector<int> shape(grows); // the distinct gather rows, then which row every output reads
        shape.resize(grows.size() + (size_t)M + 1, -2);
        for (size_t r = 0; r < row_outs.size(); r++)
            for (int m : row_outs[r]) shape[grows.size() + (size_t)m] = (int)r;
        mix(shape.data(), shape.size() / 2 * 8);
    }
    auto hit = c.umma_plans.find(key);
    if (hit != c.umma_plans.end()) {
        if (c.rec) c.rec->keep.push_back(hit->second); // the cache may drop it; a graph that reads it keeps it
        return std::static_pointer_cast<UmmaPlan>(hit->second);
    }
    std::shared_ptr<UmmaPlan> best = umma_search(grows, row_outs, wdh, M, K, limbs);
    if (!best) best = std::make_shared<UmmaPlan>();
    else {
        best->ok = true;
        CNHE_CUDA(cudaMalloc((void **)&best->d_bundles, best->bundles.size() * sizeof(UmBundle)));
        CNHE_CUDA(cudaMalloc((void **)&best->d_rows, best->chunk_rows.size() * sizeof(int)));
        CNHE_CUDA(cudaMalloc((void **)&best->d_wpack, best->wpack.size()));
        // complete on return, on the upload stream: a plan built while recording must not touch the captured streams
        CNHE_CUDA(cudaMemcpyAsync(best->d_bundles, best->bundles.data(), best->bundles.size() * sizeof(UmBundle), cudaMemcpyHostToDevice,
                                  c.copy_stream));
        CNHE_CUDA(cudaMemcpyAsync(best->d_rows, best->chunk_rows.data(), best->chunk_rows.size() * sizeof(int), cudaMemcpyHostToDevice,
                                  c.copy_stream));
        CNHE_CUDA(cudaMemcpyAsync(best->d_wpack, best->wpack.data(), best->wpack.size(), cudaMemcpyHostToDevice, c.copy_stream));
        CNHE_CUDA(cudaStreamSynchronize(c.copy_stream));
    }
    if (c.umma_plans.size() > 64) c.umma_plans.clear();
    c.umma_plans[key] = best;
    if (c.rec) c.rec->keep.push_back(best);
    return best;
}
// A validated scalar-MAC layer: outputs that share a gather row in tiles of 8, and the key slot of every output.  The inputs are
// encrypted dense vectors (same block count), weights[m] plain sparse of dim K, bias[m] plain dense or null.
struct MacLayer {
    int n_in, M, K, bl, maxbits;
    const int32_t *gather;
    const cnhe_vec *const *weights, *const *bias;
    bool const_bias;
    std::vector<int> grows, out_slot;
    std::vector<MacTile> tiles;
    std::vector<std::vector<int>> row_outs; // outputs of every distinct gather row, in the order of `grows`
};
// in_scale: the scale of the ciphertexts the MAC sums (the inputs', or the activation's output scale when they are squared first); the
// bias must be at in_scale times the weights' scale
// keep_pending: leave pending inputs unrelinearised (the exact path of mac_layer)
static MacLayer mac_prepare(Context &c, const cnhe_vec *const *in, int n_in, double in_scale, const int32_t *gather, const cnhe_vec *const *weights,
                            const cnhe_vec *const *bias, int M, int K, bool keep_pending = false) {
    if (n_in < 1 || M < 1 || K < 1) fail("bad layer shape");
    MacLayer L;
    L.n_in = n_in; L.M = M; L.K = K; L.gather = gather; L.weights = weights; L.bias = bias;
    L.bl = in[0]->blocks;
    for (int i = 0; i < n_in; i++) {
        if (!keep_pending) same_ctx(c, in[i]);
        else if (!in[i] || in[i]->ctx != &c) fail(!in[i] ? "null vector" : "vector belongs to another context");
        if (!in[i]->enc || in[i]->format != CNHE_DENSE) fail("layer inputs must be encrypted dense vectors");
        if (in[i]->blocks != L.bl || in[i]->dim != in[0]->dim || in[i]->scale != in[0]->scale) fail("all layer inputs must share dimension and scale");
    }
    L.const_bias = bias != nullptr;
    for (int m = 0; m < M; m++) {
        same_ctx(c, weights[m]);
        if (weights[m]->enc || weights[m]->format != CNHE_SPARSE) fail("expecting a sparse vector");
        if (weights[m]->dim != (uint64_t)K) fail("dimensions do not match");
        if (weights[m]->scale != weights[0]->scale) fail("weight scales differ");
        if (bias) {
            if (!bias[m]) fail("null bias");
            same_ctx(c, bias[m]);
            if (bias[m]->enc || bias[m]->format != CNHE_DENSE || bias[m]->dim != in[0]->dim) fail("bias must be a plain dense vector of the input dimension");
            if (bias[m]->scale != in_scale * weights[0]->scale) fail("Scales do not match.");
            L.const_bias = L.const_bias && bias[m]->is_const;
        }
    }
    // The scalar MAC is key-independent, so one call may serve several clients (their images' columns side by side, each output's
    // gather row inside one client's columns): every output takes the key slot its taps share; taps of two slots in one output are refused
    const std::vector<int> in_slot = vec_slots(c, in, n_in, keep_pending);
    L.out_slot.assign(M, -1);
    for (int m = 0; m < M; m++) {
        for (int kk = 0; kk < (gather ? K : n_in); kk++) {
            const int g = gather ? gather[(size_t)m * K + kk] : kk;
            if (g < 0) continue;
            if (g >= n_in) fail("gather index out of range");
            if (L.out_slot[m] >= 0 && L.out_slot[m] != in_slot[g]) fail("encrypted operands belong to different key slots");
            L.out_slot[m] = in_slot[g];
        }
        if (L.out_slot[m] < 0) L.out_slot[m] = in_slot[0];
    }
    // 128-bit accumulator bound: K products of (q_l - 1)^2
    L.maxbits = 0;
    for (u64 q : c.q) L.maxbits = std::max(L.maxbits, hm::bit_length(q));
    if (2 * L.maxbits + hm::bit_length((u64)K) > 127) fail("layer too wide for the 128-bit accumulator with these coefficient moduli");
    // tiles: outputs that share a gather row, 8 at a time
    std::unordered_map<std::vector<int>, std::vector<int>, RowHash> groups;
    std::vector<std::vector<int>> order;
    for (int m = 0; m < M; m++) {
        std::vector<int> row(K);
        bool any = false;
        for (int kk = 0; kk < K; kk++) {
            row[kk] = gather ? gather[(size_t)m * K + kk] : kk;
            if (row[kk] >= n_in) fail("gather index out of range");
        }
        // The reference skips zero plaintexts per plaintext modulus (IsZero, AtomicSealBfvVector.cs:468) and sums what is left, so an
        // output whose taps are all = 0 modulo one of the t_c has an empty sum in that channel.  (Deviation, documented in DESIGN.md:
        // padded taps are skipped here, while the reference multiplies a fresh encryption of zero by their weight.)
        for (int ch = 0; ch < c.P; ch++) {
            bool any_ch = false;
            for (int kk = 0; kk < K; kk++) any_ch = any_ch || (row[kk] >= 0 && weights[m]->scalars[ch][kk] != 0);
            any = any || any_ch;
            if (!any_ch) fail("an output has no non-zero tap modulo one of the plaintext primes (the reference would sum an empty list)");
        }
        if (!any) fail("an output has no non-zero tap (the reference would sum an empty list)");
        auto it = groups.find(row);
        if (it == groups.end()) { order.push_back(row); groups[row] = {m}; }
        else it->second.push_back(m);
    }
    for (auto &row : order) {
        const int row_index = (int)(L.grows.size() / K);
        L.grows.insert(L.grows.end(), row.begin(), row.end());
        const std::vector<int> &ms = groups[row];
        L.row_outs.push_back(ms);
        for (size_t s = 0; s < ms.size(); s += 8) {
            MacTile t;
            memset(&t, 0, sizeof(t));
            t.gather_row = row_index;
            t.n_out = (int)std::min<size_t>(8, ms.size() - s);
            for (int j = 0; j < t.n_out; j++) t.out_index[j] = ms[s + j];
            L.tiles.push_back(t);
        }
    }
    return L;
}
// the layer's weights in channel ch as signed integers (centred mod t), and their largest magnitude
static std::vector<double> mac_weights(Context &c, const MacLayer &L, int ch, double &wmax) {
    const u64 t = c.t[ch], thr = (t + 1) >> 1;
    std::vector<double> wdh((size_t)L.M * L.K);
    wmax = 0;
    for (int m = 0; m < L.M; m++)
        for (int kk = 0; kk < L.K; kk++) {
            const u64 w = L.weights[m]->scalars[ch][kk];
            const double d = w >= thr ? -(double)(t - w) : (double)w;
            wdh[(size_t)m * L.K + kk] = d;
            wmax = std::max(wmax, std::fabs(d));
        }
    return wdh;
}
// the wgmma plan of channel ch, or null when the wgmma kernel cannot serve the layer: any layer whose inputs are evenly spaced rows of one
// slab (the previous layer's output, an imported batch) and whose weights stay within +-254; tap_stride: the rows' distance in words
static std::shared_ptr<UmmaPlan> mac_umma_plan(Context &c, const MacLayer &L, int ch, const std::vector<const u64 *> &ip_all, size_t ctw,
                                               const std::vector<double> &wdh, double wmax, long long &tap_stride) {
    const int n_in = L.n_in, M = L.M, maxbits = L.maxbits, limbs = (maxbits + 7) / 8;
    // (M >= 8: LoLa's per-map products come one output at a time -- a 128-row MMA per tile would be 99 % padding and the kernel's
    // per-tile latency more than the whole scalar-MAC launch)
    bool slab = L.bl == 1 && n_in >= 2 && M >= 8 && maxbits <= 50 && limbs >= 5 && limbs <= 7 && wmax <= 254.0 && !getenv("CNHE_MAC_NO_UMMA") &&
                !getenv("CNHE_MAC_NO_IMMA") && !getenv("CNHE_MAC_INT");
    tap_stride = 0;
    if (slab) {
        tap_stride = ip_all[1] - ip_all[0];
        slab = tap_stride >= (long long)ctw && tap_stride % 2 == 0;
        for (int i = 0; i < n_in && slab; i++) slab = ip_all[i] == ip_all[0] + (long long)i * tap_stride;
    }
    if (!slab) return nullptr;
    std::shared_ptr<UmmaPlan> plan = umma_plan(c, ch, L.grows, L.row_outs, wdh, M, L.K, limbs);
    return plan->ok && (double)plan->total_chunks * 32.0 * 127.0 * 255.0 < 2147483648.0 ? plan : nullptr;
}
// One channel of a prepared layer on ciphertexts of `polys` polynomials (2, or 3 for size-3 products: the sum is linear in each
// polynomial): ip[b * n_in + i] is block b of input i, op[m * bl + b] block b of output m; the blocks of one output lie consecutively,
// polys * k * N words apart.  The bias goes to c0.
// planes (exact path, DESIGN 4.15; size-3 inputs on the wgmma kernel only): the outputs get c0 and c1 alone (2kN words) and the digit
// sums of c2 go to planes[m][D][N] (int32) for the plane-source key switch
static void mac_channel(Context &c, const MacLayer &L, int ch, const std::vector<const u64 *> &ip_all, const std::vector<u64 *> &op_all, int polys,
                        int *planes = nullptr) {
    const int n_in = L.n_in, M = L.M, K = L.K, bl = L.bl, maxbits = L.maxbits;
    const int32_t *gather = L.gather;
    const cnhe_vec *const *weights = L.weights, *const *bias = L.bias;
    const std::vector<int> &grows = L.grows;
    const std::vector<MacTile> &tiles = L.tiles;
    const int order_rows = (int)(grows.size() / K);
    const size_t ctw = (size_t)polys * c.k * c.N;
    // every temporary lives on this channel's stream (stream-ordered frees must not overtake another channel's kernels)
    int *d_gather = (int *)c.ws_alloc((grows.size() + 1) / 2 + 1);
    c.h2d(d_gather, grows.data(), grows.size() * sizeof(int));
    MacTile *d_tiles = (MacTile *)c.ws_alloc((tiles.size() * sizeof(MacTile) + 7) / 8);
    c.h2d(d_tiles, tiles.data(), tiles.size() * sizeof(MacTile));
    std::vector<const u64 *> wp(M);
    for (int m = 0; m < M; m++) wp[m] = weights[m]->ptr(ch);
    const u64 *const *d_w = upload_ptrs(c, wp);
    // signed weights as doubles for the FP64 accumulate path, when they are small enough for it to be exact
    double wmax = 0;
    const std::vector<double> wdh = mac_weights(c, L, ch, wmax);
    const bool fp_mac = maxbits <= 50 && wmax < 131072.0 && (double)K * wmax * 67108864.0 < 4503599627370496.0 && !getenv("CNHE_MAC_INT");
    // dense layer (one gather row shared by every output, 8-bit weights): exact integer GEMM on the tensor cores (mac_imma.cu).  Both
    // tensor-core kernels join the limb sums in an FP64 epilogue that is exact only for moduli below 2^50 ((double)p, fcanon_u's
    // |x| < 2^51); wider moduli (N = 2048's 54-bit default, custom ones) take the 128-bit k_mac_layer
    const int limbs = (maxbits + 7) / 8;
    const bool imma = order_rows == 1 && wmax <= 254.0 && K >= 32 && M >= 8 && maxbits <= 50 && limbs >= 5 && limbs <= 7 &&
                      (double)K * 254.0 * 255.0 < 2147483648.0 && !getenv("CNHE_MAC_NO_IMMA") && !getenv("CNHE_MAC_INT");
    // ... or wgmma (mac_umma.cu), dense and convolution alike, under the same modulus bound
    long long tap_stride = 0;
    const std::shared_ptr<UmmaPlan> plan = mac_umma_plan(c, L, ch, ip_all, ctw, wdh, wmax, tap_stride);
    const bool umma = plan != nullptr;
    if (planes && !umma) throw Error(CNHE_ERR_INVALID, "internal error: the exact scalar-MAC path needs the wgmma kernel");
    const void *d_wfrag = nullptr, *d_wfrag2 = nullptr;
    if (!umma && imma) {
        const int mtiles = (M + 15) / 16, chunks = (K + 31) / 32;
        const size_t fwords = (size_t)mtiles * chunks * 32 * 4;
        std::vector<uint32_t> frag(2 * fwords, 0); // W1 = clamp(W, +-127) then the residual W2 = W - W1
        bool any2 = false;
        auto wq = [&](int m, int kk, int part) -> uint32_t { // signed weight of output m, tap kk (0 outside the matrix / on padded taps)
            if (m >= M || kk >= K || grows[kk] < 0) return 0;
            const int w = (int)wdh[(size_t)m * K + kk], w1 = std::max(-127, std::min(127, w));
            const int v = part ? w - w1 : w1;
            if (part && v) any2 = true;
            return (uint32_t)(uint8_t)(int8_t)v;
        };
        for (int part = 0; part < 2; part++)
            for (int mt = 0; mt < mtiles; mt++)
                for (int cch = 0; cch < chunks; cch++)
                    for (int lane = 0; lane < 32; lane++) {
                        const int g = lane >> 2, tig = lane & 3;
                        uint32_t *dst = &frag[part * fwords + (((size_t)mt * chunks + cch) * 32 + lane) * 4];
                        for (int r = 0; r < 4; r++) { // r: 0 (row g, k 0..15) 1 (row g+8) 2 (row g, k 16..31) 3 (row g+8, k 16..31)
                            const int row = mt * 16 + g + (r & 1) * 8, k0 = cch * 32 + tig * 4 + (r >> 1) * 16;
                            dst[r] = wq(row, k0, part) | (wq(row, k0 + 1, part) << 8) | (wq(row, k0 + 2, part) << 16) | (wq(row, k0 + 3, part) << 24);
                        }
                    }
        u64 *buf = c.ws_alloc((frag.size() * 4 + 7) / 8);
        c.h2d(buf, frag.data(), (any2 ? 2 : 1) * fwords * 4);
        d_wfrag = buf;
        if (any2) d_wfrag2 = reinterpret_cast<const uint32_t *>(buf) + fwords;
    }
    const double *d_wd = nullptr;
    if (fp_mac) {
        u64 *buf = c.ws_alloc(wdh.size());
        c.h2d(buf, wdh.data(), wdh.size() * 8);
        d_wd = reinterpret_cast<const double *>(buf);
    }
    const u64 *d_bias = nullptr;
    if (bias && L.const_bias) {
        std::vector<u64> bv(M);
        for (int m = 0; m < M; m++) bv[m] = bias[m]->const_val[ch];
        u64 *db = c.ws_alloc(M);
        c.h2d(db, bv.data(), (size_t)M * 8);
        d_bias = db;
    }
    for (int b = 0; b < bl; b++) {
        std::vector<const u64 *> ip(ip_all.begin() + (size_t)b * n_in, ip_all.begin() + (size_t)(b + 1) * n_in);
        std::vector<u64 *> op(M);
        for (int m = 0; m < M; m++) op[m] = op_all[(size_t)m * bl + b];
        double used = 0;
        for (auto &t : tiles) { int kk = 0; for (int j = 0; j < K; j++) kk += grows[(size_t)t.gather_row * K + j] >= 0; used += kk + t.n_out; }
        c.prof_begin(4, used * 8.0 * ctw);
        if (umma) {
            UmmaLaunch a;
            memset(&a, 0, sizeof(a));
            a.slab = ip[0];
            a.slab_stride_words = (size_t)tap_stride;
            a.slab_rows = (size_t)n_in;
            if (!plan->extra_taps.empty()) { // the taps that need the W2 part, side by side
                u64 *scratch = c.ws_alloc(plan->extra_taps.size() * ctw);
                for (size_t j = 0; j < plan->extra_taps.size(); j++)
                    CNHE_CUDA(cudaMemcpyAsync(scratch + j * ctw, ip[plan->extra_taps[j]], ctw * 8, cudaMemcpyDeviceToDevice, c.stream));
                a.scratch = scratch;
                a.scratch_rows = plan->extra_taps.size();
            }
            std::vector<u64 *> opo(M);
            for (int i = 0; i < M; i++) opo[i] = op[plan->out_order[i]];
            const u64 *d_bias_o = nullptr;
            if (d_bias) {
                std::vector<u64> bo(M);
                for (int i = 0; i < M; i++) bo[i] = bias[plan->out_order[i]]->const_val[ch];
                u64 *db = c.ws_alloc(M);
                c.h2d(db, bo.data(), (size_t)M * 8);
                d_bias_o = db;
            }
            a.bundles = plan->d_bundles; a.n_bundles = (int)plan->bundles.size();
            a.chunk_rows = plan->d_rows; a.total_chunks = plan->total_chunks;
            a.wpack = plan->d_wpack; a.a_bytes = (int)plan->wpack.size();
            a.out_ptrs = upload_ptrs_mut(c, opo); a.bias = d_bias_o; a.n_out_total = M;
            a.limbs = limbs; a.polys = polys; a.k = c.k; a.logn = c.logN; a.bc = c.d_bc; a.pc = c.ch[ch].pc;
            if (planes) { // digit planes in the key order of the relinearisation keys: digit d of residue src[d], bits shift[d] ..
                const DigitMap &dm = c.dm_relin;
                std::vector<int *> pp(M);
                for (int i = 0; i < M; i++) pp[i] = planes + (size_t)plan->out_order[i] * dm.D * c.N;
                u64 *dpp = c.ws_alloc(M);
                c.h2d(dpp, pp.data(), (size_t)M * 8);
                a.dig.planes = reinterpret_cast<int *const *>(dpp);
                a.dig.mask = (unsigned)dm.mask;
                a.dig.w = hm::bit_length(dm.mask);
                int most = 0;
                for (int d = 0; d < dm.D; d++) {
                    if (a.dig.count[dm.src[d]]++ == 0) a.dig.first[dm.src[d]] = (unsigned char)d;
                    most = std::max(most, (int)a.dig.count[dm.src[d]]);
                }
                a.dig.groups = (most + limbs / 2 - 1) / (limbs / 2);
            }
            c.check(launch_mac_umma(a, c.stream), "mac_umma");
        } else if (imma) {
            std::vector<const u64 *> ipg(K);
            for (int kk = 0; kk < K; kk++) ipg[kk] = ip[grows[kk] < 0 ? 0 : grows[kk]]; // padded taps carry weight 0
            c.check(launch_mac_dense_imma(upload_ptrs(c, ipg), d_wfrag, d_wfrag2, d_bias, K, M, limbs, upload_ptrs_mut(c, op), polys, c.k, c.logN, c.d_bc,
                                          c.ch[ch].pc, c.stream),
                    "mac_dense_imma");
        } else if (fp_mac)
            c.check(launch_mac_layer_fp(upload_ptrs(c, ip), d_gather, d_tiles, (int)tiles.size(), d_wd, d_bias, K, upload_ptrs_mut(c, op), polys, c.k,
                                        c.logN, c.d_bc, c.ch[ch].pc, c.stream),
                    "mac_layer_fp");
        else
            c.check(launch_mac_layer(upload_ptrs(c, ip), d_gather, d_tiles, (int)tiles.size(), d_w, d_bias, K, upload_ptrs_mut(c, op), polys, c.k, c.logN,
                                     c.d_bc, c.ch[ch].pc, c.stream),
                    "mac_layer");
        c.prof_end();
    }
    { // what the reference issues for this layer (AtomicSealBfvVector.cs:466-475, 497-505): MultiplyPlain per non-zero tap, AddMany per output
        uint64_t taps = 0;
        for (int m = 0; m < M; m++)
            for (int kk = 0; kk < K; kk++) taps += (!gather || gather[(size_t)m * K + kk] >= 0) && weights[m]->scalars[ch][kk] != 0;
        c.op_count[Context::OP_MULTIPLY_SCALAR] += taps * bl;
        c.op_count[Context::OP_ADD_MANY_ITEMS] += taps * bl;
        if (bias) c.op_count[Context::OP_ADD_PLAIN] += (uint64_t)M * bl;
        double ss = 0; // output 0: root-sum-square of its centred weights (the noise gain of the scalar MAC under independent inputs)
        for (int kk = 0; kk < K; kk++)
            if (!gather || gather[kk] >= 0) ss += wdh[kk] * wdh[kk];
        // (a size-3 sum has no noise budget of its own: its relinearised outputs are measured)
        c.note(Context::OP_ADD_MANY, ch, M * bl, polys == 2 && !planes ? op_all[0] : nullptr, ip_all[gather ? std::max(gather[0], 0) : 0], nullptr,
               ss > 0 ? 0.5 * std::log2(ss) : 0);
    }
    if (bias && !L.const_bias) // generic AddPlain per output, on c0 of each of its blocks
        for (int m = 0; m < M; m++) {
            u64 *o = op_all[(size_t)m * bl];
            c.check(launch_ct_add_plain(o, o, bl, planes ? 2 : polys, bias[m]->ptr(ch), c.N, (int)c.N, c.k, c.logN, c.d_bc, c.ch[ch].pc, 0, c.stream),
                    "ct_add_plain");
        }
}
// The exact path of mac_layer over pending squares (DESIGN 4.15): relinearising a size-3 product adds sum_d digit_d(c2) * rlk_d to
// (c0, c1), so the layer's output m is (sum_j W_mj (c0_j, c1_j) + bias) + sum_d S_md * rlk_d with the integer digit sums
// S_md = sum_j W_mj digit_d(c2_j) -- the same element of R_q, written canonical, as the layer over the relinearised squares: the same
// words and noise, for M key switches instead of one per input.  Taken when every input is pending, the context has the plane-source key
// switch, the wgmma kernel serves the layer in every channel and every |S| stays below min(2^31, min_l q_l); returns false (nothing
// done) otherwise.
static bool mac_layer_exact(Context &c, const cnhe_vec *const *in, int n_in, const int32_t *gather, const cnhe_vec *const *weights,
                            const cnhe_vec *const *bias, int M, int K, cnhe_vec **out) {
    if (n_in < 2 || !in || c.trace_noise || !relin_planes_built(c)) return false;
    const DigitMap &dm = c.dm_relin;
    const int w = hm::bit_length(dm.mask);
    if (w > 16) return false;
    for (int i = 0; i < n_in; i++) {
        if (!in[i] || in[i]->ctx != &c || !in[i]->pend) return false;
        for (int b = 0; b < in[i]->blocks; b++) // the square's key slot is the one its relinearisation would use
            if (in[i]->pend->ct_slot[in[i]->pend_ct + b] != in[i]->slot) return false;
    }
    const MacLayer L = mac_prepare(c, in, n_in, in[0]->scale, gather, weights, bias, M, K, true);
    if (L.bl != 1) return false;
    double bound = 2147483648.0;
    for (u64 q : c.q) bound = std::min(bound, (double)q);
    std::vector<std::vector<const u64 *>> ips(c.P);
    const size_t s3 = (size_t)3 * c.k * c.N, ctw = c.ct_words();
    for (int ch = 0; ch < c.P; ch++) {
        for (int i = 0; i < n_in; i++) ips[ch].push_back(in[i]->pending_block(ch, 0));
        double wmax = 0;
        const std::vector<double> wdh = mac_weights(c, L, ch, wmax);
        long long tap_stride = 0;
        if (!mac_umma_plan(c, L, ch, ips[ch], s3, wdh, wmax, tap_stride)) return false;
        for (int m = 0; m < M; m++) {
            double sum = 0;
            for (int kk = 0; kk < K; kk++)
                if (!gather || gather[(size_t)m * K + kk] >= 0) sum += std::fabs(wdh[(size_t)m * K + kk]);
            if (sum * (double)dm.mask >= bound) return false;
        }
    }
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        big[ch] = c.alloc((size_t)M * ctw);
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        u64 *y = c.ws_alloc((size_t)M * ctw);
        int *planes = reinterpret_cast<int *>(c.ws_alloc(((size_t)M * dm.D * c.N + 1) / 2));
        std::vector<u64 *> op(M);
        for (int m = 0; m < M; m++) op[m] = y + (size_t)m * ctw;
        mac_channel(c, L, ch, ips[ch], op, 3, planes);
        op_relinearize_planes(c, ch, planes, M, y, big[ch]->p, L.out_slot.data());
    }
    for (int m = 0; m < M; m++) out[m] = slab_output(c, big, (size_t)m, in[0], in[0]->scale * weights[0]->scale, L.out_slot[m]);
    return true;
}
// Shared body of DenseMatrixBySparseVectorMultiply (ciphertext columns x plain constants) and of the fused PoolLayer.
static void mac_layer(Context &c, const cnhe_vec *const *in, int n_in, const int32_t *gather, const cnhe_vec *const *weights, const cnhe_vec *const *bias,
                      int M, int K, cnhe_vec **out) {
    if (mac_layer_exact(c, in, n_in, gather, weights, bias, M, K, out)) return;
    const MacLayer L = mac_prepare(c, in, n_in, n_in > 0 ? in[0]->scale : 0.0, gather, weights, bias, M, K);
    const int bl = L.bl;
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        big[ch] = c.alloc((size_t)M * bl * c.ct_words());
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<const u64 *> ip((size_t)bl * n_in);
        for (int b = 0; b < bl; b++)
            for (int i = 0; i < n_in; i++) ip[(size_t)b * n_in + i] = in[i]->block(ch, b);
        std::vector<u64 *> op((size_t)M * bl);
        for (size_t j = 0; j < op.size(); j++) op[j] = big[ch]->p + j * c.ct_words();
        mac_channel(c, L, ch, ip, op, 2);
    }
    for (int m = 0; m < M; m++) out[m] = slab_output(c, big, (size_t)m * bl, in[0], in[0]->scale * weights[0]->scale, L.out_slot[m]);
}
extern "C" int cnhe_layer_conv_dense(cnhe_ctx *h, const cnhe_vec *const *in, int n_in, const int32_t *gather, const cnhe_vec *const *weights,
                                     const cnhe_vec *const *bias, int M, int K, cnhe_vec **out) {
    API_BEGIN(h)
    mac_layer(c, in, n_in, gather, weights, bias, M, K, out);
    API_END
}
// DenseMatrixBySparseVectorMultiply (AtomicSealBfvVector.cs:434-521)
extern "C" int cnhe_mat_mul_colmajor_sparse(cnhe_ctx *h, const cnhe_vec *const *cols, int K, const cnhe_vec *sparse, cnhe_vec **out) {
    API_BEGIN(h)
    if (K < 1) fail("empty matrix");
    same_ctx(c, sparse);
    for (int i = 0; i < K; i++) same_ctx(c, cols[i]);
    if ((uint64_t)K != sparse->dim) fail("dimensions do not match");
    if (sparse->format != CNHE_SPARSE) fail("expecting a sparse vector");
    if (!cols[0]->enc && !sparse->enc) fail("at least one parameter has to be encrypted");
    {
        std::vector<const cnhe_vec *> all(cols, cols + K);
        all.push_back(sparse);
        use_slot(c, all.data(), K + 1);
    }
    if (cols[0]->enc && !sparse->enc) {
        mac_layer(c, cols, K, nullptr, &sparse, nullptr, 1, K, out);
    } else {
        const int bl = cols[0]->blocks;
        const size_t ctw = c.ct_words();
        cnhe_vec *o = new_vec(c, cols[0]->dim, cols[0]->scale * sparse->scale, CNHE_DENSE, true, bl);
        std::unique_ptr<cnhe_vec> guard(o);
        alloc_channels(o);
        for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
            u64 *prod = c.ws_alloc((size_t)K * bl * ctw);
            if (cols[0]->enc) { // both encrypted: Multiply + Relinearize per (k, block)
                std::vector<const u64 *> a, b;
                for (int kk = 0; kk < K; kk++)
                    for (int i = 0; i < bl; i++) { a.push_back(cols[kk]->block(ch, i)); b.push_back(sparse->block(ch, kk)); }
                op_multiply_relin(c, ch, a, b, prod);
            } else { // plain columns x encrypted constants: MultiplyPlain(sparse.enc[k], denses[k].plain[i])
                for (int kk = 0; kk < K; kk++) {
                    u64 *rep = c.ws_alloc((size_t)bl * ctw);
                    for (int i = 0; i < bl; i++)
                        { CNHE_CUDA(cudaMemcpyAsync(rep + (size_t)i * ctw, sparse->block(ch, kk), ctw * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(rep + (size_t)i * ctw, sparse->block(ch, kk)); }
                    op_multiply_plain_dense(c, ch, rep, bl, cols[kk]->ptr(ch), true, prod + (size_t)kk * bl * ctw);
                }
            }
            for (int i = 0; i < bl; i++) {
                std::vector<const u64 *> terms;
                for (int kk = 0; kk < K; kk++) terms.push_back(prod + ((size_t)kk * bl + i) * ctw);
                do_add_many(c, ch, terms, o->block(ch, i));
            }
            c.host_fence();
        }
        *out = guard.release();
    }
    API_END
}
// cnhe_mat_mul_colmajor_sparse with both operands encrypted, the products' relinearisation deferred past their sum (DESIGN 4.14): per
// channel one op_multiply_sum over the K terms of every output block, which lifts and transforms each column block and each sparse element
// once, floors each chunk of at most K_c summed products once and relinearises each output block once
extern "C" int cnhe_mat_mul_colmajor_sparse_deferred(cnhe_ctx *h, const cnhe_vec *const *cols, int K, const cnhe_vec *sparse, cnhe_vec **out) {
    API_BEGIN(h)
    if (!cols || !out) fail("bad arguments");
    if (K < 1) fail("empty matrix");
    same_ctx(c, sparse);
    for (int i = 0; i < K; i++) same_ctx(c, cols[i]);
    if ((uint64_t)K != sparse->dim) fail("dimensions do not match");
    if (sparse->format != CNHE_SPARSE) fail("expecting a sparse vector");
    if (!cols[0]->enc && !sparse->enc) fail("at least one parameter has to be encrypted");
    for (int i = 0; i < K; i++)
        if (!cols[i]->enc || !sparse->enc)
            fail("the deferred product needs encrypted columns and an encrypted sparse vector (cnhe_mat_mul_colmajor_sparse serves the rest)");
    for (int i = 1; i < K; i++)
        if (cols[i]->dim != cols[0]->dim || cols[i]->blocks != cols[0]->blocks) fail("dimensions do not match");
    {
        std::vector<const cnhe_vec *> all(cols, cols + K);
        all.push_back(sparse);
        use_slot(c, all.data(), K + 1);
    }
    const int bl = cols[0]->blocks;
    cnhe_vec *o = new_vec(c, cols[0]->dim, cols[0]->scale * sparse->scale, CNHE_DENSE, true, bl);
    std::unique_ptr<cnhe_vec> guard(o);
    alloc_channels(o);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<const u64 *> a, b;
        for (int i = 0; i < bl; i++)
            for (int kk = 0; kk < K; kk++) a.push_back(cols[kk]->block(ch, i));
        for (int kk = 0; kk < K; kk++) b.push_back(sparse->block(ch, kk));
        op_multiply_sum(c, ch, a, b, K, bl, o->block(ch, 0));
        c.op_count[Context::OP_ADD_MANY_ITEMS] += (uint64_t)K * bl; // the sums, booked as the existing call books its AddMany items
    }
    *out = guard.release();
    API_END
}
extern "C" int cnhe_context_product_sum_terms(const cnhe_ctx *h, int *terms) {
    if (!h || !terms) return set_err(CNHE_ERR_INVALID, "null argument");
    *terms = h->c->sum_terms;
    return CNHE_OK;
}
// RowMajor matrix x vector (EncryptedSealBfvMatrix.cs:79-120): per row DotProduct(row, v) = PointwiseMultiply + SumAllSlots, then
// GenerateSparseOfArray, or (ForceDenseFormat) a one-hot mask per row and the sum of all rows.  All rows go through each stage
// together instead of one DotProduct per row.
// rows[i] is row first_row + i of a matrix with total_rows rows; vs are B encrypted vectors that may belong to different key slots (one
// inference per client), out[b] the product with vs[b].  The B * n_rows products are flattened (product p = b * n_rows + r) and go through
// each stage in waves -- whole clients when the rows fit in one wave, else slices of one client's rows: the plain products (one outer
// product of the wave's clients and rows when it holds several clients, else the broadcast product), one rotate-and-add ladder over
// `length` slots for the whole wave (every key switch of a step in one wave, each ciphertext under its own slot's keys), then per input the
// one-hot masks at the global columns first_row + r and the sum into its dense output of dimension total_rows, or its sparse elements.
// dot: no matrix output -- out[b * n_rows + r] is DotProduct(rows[r], vs[b], length) as cnhe_vec_dot_product returns it.
static void mat_mul_rowmajor(Context &c, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *const *vs, int B, bool force_dense, int first_row,
                             int total_rows, cnhe_vec **out, uint64_t length = CNHE_ALL_SLOTS, bool dot = false) {
    if (!rows || n_rows < 1 || !vs || B < 1 || !out) fail("bad arguments");
    for (int b = 0; b < B; b++) {
        same_ctx(c, vs[b]);
        if (!vs[b]->enc) fail("at least one parameter has to be encrypted");
        if (vs[b]->format != CNHE_DENSE) fail("Expecting dense vector format");
        if (vs[b]->blocks != 1) fail("row-major multiplication expects a single-block vector");
        if (vs[b]->dim != vs[0]->dim || vs[b]->scale != vs[0]->scale) fail("the input vectors must share dimension and scale");
    }
    for (int r = 0; r < n_rows; r++) {
        same_ctx(c, rows[r]);
        if (rows[r]->enc) fail("encrypted rows are not supported by the batched row-major product");
        if (rows[r]->dim != vs[0]->dim) fail("Dimensions do not match");
        if (rows[r]->format != CNHE_DENSE) fail("Format mismatch");
        if (rows[r]->scale != rows[0]->scale) fail("row scales differ");
    }
    if (length == 0) fail("Can't sum over less then one element");
    const size_t N = c.N, ctw = c.ct_words();
    if (force_dense && (size_t)total_rows > N) fail("column out of range");
    const std::vector<int> vslot = vec_slots(c, vs, B);
    const double out_scale = vs[0]->scale * rows[0]->scale;
    const int n_out = dot ? B * n_rows : B;
    std::vector<std::unique_ptr<cnhe_vec>> outs(n_out);
    for (int o = 0; o < n_out; o++) {
        if (dot) outs[o].reset(new_vec(c, vs[0]->dim, out_scale, CNHE_DENSE, true, 1));
        else outs[o].reset(new_vec(c, (uint64_t)(force_dense ? total_rows : n_rows), out_scale, force_dense ? CNHE_DENSE : CNHE_SPARSE, true,
                                   force_dense ? 1 : n_rows));
        outs[o]->slot = vslot[dot ? o / n_rows : o];
        if (force_dense) alloc_channels(outs[o].get());
    }
    std::vector<BufRef> big(c.P); // sparse outputs and dot products: one [B][n_rows] slab, product p lands in its place
    if (!force_dense) {
        for (int ch = 0; ch < c.P; ch++) {
            c.set_channel(ch);
            big[ch] = c.alloc((size_t)B * n_rows * ctw);
        }
        for (int o = 0; o < n_out; o++) slab_view(outs[o].get(), big, dot ? (size_t)o : (size_t)o * n_rows);
    }
    // products per wave: 1024, fewer when the wave's scratch (the products, the ladder's rotated copies and the masked products: three
    // ciphertexts per product) would pass 8 GiB -- the largest context, N = 16384 with nine primes, allows 1213
    const int total = B * n_rows, RC = (int)std::max<size_t>(16, std::min<size_t>(1024, ((size_t)1 << 30) / (3 * ctw)));
    struct Wave { int b0, nb, r0, nr; };
    std::vector<Wave> waves;
    if (n_rows <= RC)
        for (int b0 = 0; b0 < B; b0 += RC / n_rows) waves.push_back({b0, std::min(RC / n_rows, B - b0), 0, n_rows});
    else
        for (int b = 0; b < B; b++)
            for (int r0 = 0; r0 < n_rows; r0 += RC) waves.push_back({b, 1, r0, std::min(RC, n_rows - r0)});
    std::vector<int> pslot(total);
    for (int p = 0; p < total; p++) pslot[p] = vslot[p / n_rows];
    uint64_t len = length;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        std::vector<char> first(B, 1);
        for (const Wave &w : waves) {
            WsScope scope(c);
            const int p0 = w.b0 * n_rows + w.r0, m = w.nb * w.nr;
            u64 *prod = force_dense ? c.ws_alloc((size_t)m * ctw) : big[ch]->p + (size_t)p0 * ctw;
            u64 *plains = c.ws_alloc((size_t)w.nr * N);
            for (int i = 0; i < w.nr; i++)
                CNHE_CUDA(cudaMemcpyAsync(plains + (size_t)i * N, rows[w.r0 + i]->ptr(ch), N * 8, cudaMemcpyDeviceToDevice, c.stream));
            std::vector<const u64 *> cts(w.nb);
            for (int j = 0; j < w.nb; j++) cts[j] = vs[w.b0 + j]->ptr(ch);
            op_multiply_plain_dense_outer(c, ch, cts, plains, w.nr, prod);
            len = sum_slots_batched(c, ch, prod, m, length, pslot.data() + p0);
            if (force_dense) {
                // one-hot masks (EncryptedSealBfvMatrix.cs:96, AtomicSealBfvVector.cs:936-945), built on the device
                u64 *masks = c.ws_alloc((size_t)m * N);
                for (int j = 0; j < w.nb; j++) op_encode_onehot(c, ch, w.nr, first_row + w.r0, masks + (size_t)j * w.nr * N);
                op_multiply_plain_dense(c, ch, prod, m, masks, true, prod);
                for (int j = 0; j < w.nb; j++) {
                    const int b = w.b0 + j;
                    std::vector<const u64 *> terms;
                    if (!first[b]) terms.push_back(outs[b]->ptr(ch));
                    for (int i = 0; i < w.nr; i++) terms.push_back(prod + ((size_t)j * w.nr + i) * ctw);
                    do_add_many(c, ch, terms, outs[b]->ptr(ch));
                    first[b] = 0;
                }
                c.host_fence();
            }
        }
    }
    if (dot) // SumAllSlots' bookkeeping (AtomicSealBfvVector.cs:946-954)
        for (auto &o : outs) {
            o->dim = len >= N / 2 ? 1 : o->dim;
            o->format = len >= N ? CNHE_SPARSE : CNHE_DENSE;
        }
    for (int o = 0; o < n_out; o++) out[o] = outs[o].release();
}
extern "C" int cnhe_mat_mul_rowmajor(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *v, int force_dense, cnhe_vec **out) {
    API_BEGIN(h)
    mat_mul_rowmajor(c, rows, n_rows, &v, 1, force_dense != 0, 0, n_rows, out);
    API_END
}
// The same product for a contiguous SLICE of the matrix rows (rows[i] is global row first_row + i of a matrix with total_rows rows):
// the unit of the intra-inference multi-GPU split (SURVEY.md 8e: CIFAR's 5488 dense rows over 4 GPUs).  ForceDense: the one-hot masks sit
// at the global columns, so the partial results of the ranks add up to the full product (the reference sums the masked rows too,
// EncryptedSealBfvMatrix.cs:92-116); otherwise the output holds this slice's sparse elements only.
extern "C" int cnhe_mat_mul_rowmajor_shard(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *v, int force_dense, int first_row,
                                           int total_rows, cnhe_vec **out) {
    API_BEGIN(h)
    if (first_row < 0 || first_row + n_rows > total_rows) fail("row slice out of range");
    mat_mul_rowmajor(c, rows, n_rows, &v, 1, force_dense != 0, first_row, total_rows, out);
    API_END
}
// The row-major product of one plain matrix with B encrypted vectors (one inference per client): out[b] is what
// cnhe_mat_mul_rowmajor(rows, n_rows, vs[b], force_dense) returns, bit for bit.
extern "C" int cnhe_mat_mul_rowmajor_batch(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *const *vs, int B, int force_dense,
                                           cnhe_vec **out) {
    API_BEGIN(h)
    mat_mul_rowmajor(c, rows, n_rows, vs, B, force_dense != 0, 0, n_rows, out);
    API_END
}
// DotProduct(rows[r], vs[b], length) of every plain row with every encrypted vector (LLPackedDenseLayer's partial sums, one per client):
// out[b * n_rows + r] is bit-identical to cnhe_vec_dot_product(rows[r], vs[b], length, -1), the row-major product's waves without its
// final masks
extern "C" int cnhe_mat_dot_rows_batch(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, const cnhe_vec *const *vs, int B, uint64_t length,
                                       cnhe_vec **out) {
    API_BEGIN(h)
    mat_mul_rowmajor(c, rows, n_rows, vs, B, false, 0, n_rows, out, length, true);
    API_END
}
// The inputs of an activation layer: n encrypted vectors whose ciphertexts the layer takes as one flat batch, in[i]'s blocks from first[i]
// on (first[n]: the batch's size)
struct ActInputs {
    const cnhe_vec *const *in;
    int n;
    std::vector<int> first;
    std::vector<int> vslot, ct_slot; // the key slot of every vector and of every ciphertext (act_inputs)
    ActInputs(const cnhe_vec *const *in, int n) : in(in), n(n), first(n + 1, 0) {
        for (int i = 0; i < n; i++) first[i + 1] = first[i] + in[i]->blocks;
    }
    int total() const { return first[n]; }
    std::vector<const u64 *> blocks(int ch) const { // the batch's ciphertexts in channel ch
        std::vector<const u64 *> p;
        for (int i = 0; i < n; i++)
            for (int b = 0; b < in[i]->blocks; b++) p.push_back(in[i]->block(ch, b));
        return p;
    }
};
// The coefficients of an activation polynomial of degree 2, 3 or 4: cf[j] the coefficient of x^j (nullptr: 0), each a plain sparse vector
// of dimension 1; the leading one is required
struct ActCoeffs {
    int degree;
    const cnhe_vec *cf[5] = {};
    double out_scale = 0;                // W s^degree (read)
    std::vector<std::array<u64, 5>> res; // per channel the residues of cf[j] (read)
    ActCoeffs(Context &c, const cnhe_vec *const *coeffs, int degree, const char *lead_missing) : degree(degree) {
        if (!coeffs || !coeffs[degree]) fail(lead_missing);
        for (int j = 0; j <= degree; j++) {
            const cnhe_vec *p = cf[j] = coeffs[j];
            if (!p) continue;
            same_ctx(c, p);
            if (p->enc) fail("the coefficients must be plain");
            if (p->format != CNHE_SPARSE || p->dim != 1) fail("each coefficient must be a sparse vector of dimension 1");
        }
    }
    // for inputs at scale s: coefficient j at scale W s^(degree - j), W the leading coefficient's scale, the powers of s multiplied up one
    // factor at a time.  A leading coefficient that is 0 mod a plaintext prime only drops the square term of a quadratic there; degrees 3
    // and 4 divide by it
    void read(Context &c, double s) {
        double at[5];
        at[degree] = cf[degree]->scale;
        for (int j = degree - 1; j >= 0; j--) at[j] = at[j + 1] * s;
        for (int j = 0; j < degree; j++)
            if (cf[j] && cf[j]->scale != at[j]) fail("Scales do not match.");
        out_scale = at[0];
        res.assign(c.P, std::array<u64, 5>{});
        for (int ch = 0; ch < c.P; ch++) {
            const u64 t = c.ch[ch].t;
            for (int j = 0; j <= degree; j++) res[ch][j] = cf[j] ? cf[j]->scalars[ch][0] % t : 0;
            if (degree > 2 && res[ch][degree] == 0)
                fail(("the leading coefficient is 0 mod the plaintext prime " + std::to_string(t) + ": it has no inverse there").c_str());
        }
    }
};
// cnhe_layer_poly2's a x^2 + b x + c (b, c may be null)
static ActCoeffs quad_coeffs(Context &c, const cnhe_vec *a, const cnhe_vec *b, const cnhe_vec *cc) {
    const cnhe_vec *cf[3] = {cc, b, a};
    return ActCoeffs(c, cf, 2, "the quadratic coefficient is required");
}
// Validates an activation layer's inputs -- encrypted (else plain_msg), and at one scale when the layer has coefficients, which are then
// read at that scale -- and records their key slots: the vectors may belong to different key slots (several clients' layers in one
// call), each ciphertext is relinearised under its own
static ActInputs act_inputs(Context &c, const cnhe_vec *const *in, int n, const char *plain_msg, ActCoeffs *cf = nullptr) {
    for (int i = 0; i < n; i++) {
        same_ctx(c, in[i]);
        if (!in[i]->enc) fail(plain_msg);
        if (cf && in[i]->scale != in[0]->scale) fail("Scales do not match.");
    }
    if (cf) cf->read(c, in[0]->scale);
    ActInputs X(in, n);
    X.vslot = vec_slots(c, in, n);
    for (int i = 0; i < n; i++) X.ct_slot.insert(X.ct_slot.end(), in[i]->blocks, X.vslot[i]);
    return X;
}
// The constant term of an activation on a dense vector whose last block is only partly filled: Delta times the plaintext with C in the
// block's data slots and 0 in its padding slots ([k][N] canonical words, as add_plain scales it), so that padding stays zero as it does
// for the square -- rotating layers (Duplicate) add whole ciphertexts.  Returns the call's table of one entry per ciphertext (nullptr: the
// constant polynomial C, every slot a data slot), or nullptr when no ciphertext needs one.  Workspace memory of the call.
static const u64 *const *padded_constants(Context &c, int ch, const ActInputs &X, u64 C) {
    const size_t N = c.N;
    std::vector<const u64 *> tab(X.total(), nullptr);
    std::map<size_t, const u64 *> by_fill; // data slots of the last block -> its Delta-scaled plaintext
    bool any = false;
    for (int i = 0; i < X.n; i++) {
        const cnhe_vec *v = X.in[i];
        if (v->format != CNHE_DENSE || v->dim % N == 0) continue;
        const size_t fill = v->dim % N;
        const u64 *&cp = by_fill[fill];
        if (!cp) {
            std::vector<u64> vals(N, 0);
            std::fill(vals.begin(), vals.begin() + fill, C);
            u64 *dv = c.ws_alloc(N), *plain = c.ws_alloc(N), *scaled = c.ws_alloc((size_t)c.k * N);
            c.h2d(dv, vals.data(), N * 8);
            op_encode(c, ch, dv, 1, (int)N, plain);
            c.check(launch_fill_zero(scaled, (size_t)c.k * N, c.stream), "fill_zero");
            c.check(launch_ct_add_plain(scaled, scaled, 1, 1, plain, N, (int)N, c.k, c.logN, c.d_bc, c.ch[ch].pc, 0, c.stream), "ct_add_plain");
            cp = scaled;
        }
        tab[X.first[i + 1] - 1] = cp;
        any = true;
    }
    return any ? upload_ptrs(c, tab) : nullptr;
}
// The floor epilogue of one channel's activation wave over X (floor_epi): relinearize(A y^2) + B x + Delta C for the squared operand y,
// x read from the table x (nullptr: y itself), the constant padded where a dense vector's last block is partly filled.  book: count the
// terms' operations beyond the product (a term that is 0 mod t is skipped in that channel)
static FloorEpi act_epilogue(Context &c, int ch, const ActInputs &X, u64 A, u64 B, u64 C, const u64 *const *x = nullptr, bool book = true) {
    FloorEpi e = floor_epi(c, ch, A, B, C);
    e.x = x;
    if (C) e.c_poly = padded_constants(c, ch, X, C);
    if (book) {
        auto &ops = c.op_count;
        const uint64_t n = (uint64_t)X.total();
        if (A) ops[Context::OP_MULTIPLY_SCALAR] += n;
        if (B) {
            ops[Context::OP_MULTIPLY_SCALAR] += n;
            ops[Context::OP_ADD] += n;
        }
        if (C) ops[Context::OP_ADD_PLAIN] += n;
    }
    return e;
}
// cnhe_layer_square (cf == nullptr) and cnhe_layer_poly2 over validated inputs, in one wave per channel: relinearize(x^2), or with the
// quadratic's floor epilogue relinearize(A x^2) + B x + Delta C word for word
static void square_layer(Context &c, const ActInputs &X, const ActCoeffs *cf, cnhe_vec **out) {
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        FloorEpi epi;
        if (cf) epi = act_epilogue(c, ch, X, cf->res[ch][2], cf->res[ch][1], cf->res[ch][0]);
        big[ch] = c.alloc((size_t)X.total() * c.ct_words());
        const std::vector<const u64 *> xs = X.blocks(ch);
        op_multiply_relin(c, ch, xs, xs, big[ch]->p, X.ct_slot.data(), cf ? &epi : nullptr);
    }
    for (int i = 0; i < X.n; i++) {
        const double s = X.in[i]->scale;
        out[i] = slab_output(c, big, X.first[i], X.in[i], cf ? cf->out_scale : s * s, X.vslot[i]);
    }
}
// SquareActivation over a whole matrix: every column PointwiseMultiply'd with itself in one wave per channel; inputs of any scales
extern "C" int cnhe_layer_square(cnhe_ctx *h, const cnhe_vec *const *in, int n, cnhe_vec **out) {
    API_BEGIN(h)
    if (n < 1) fail("empty layer");
    bool chained = false; // a square of a pending square: a polynomial chain (x^4), not an activation that feeds a scalar-MAC layer
    for (int i = 0; i < n; i++) chained = chained || (in[i] && in[i]->pend);
    const ActInputs X = act_inputs(c, in, n, "multiplying two plaintexts is not implemented");
    const int total = X.total();
    // The products stay unrelinearised until something reads them (DESIGN 4.15): a scalar-MAC layer then key-switches its outputs instead
    // of these, with the same words.  Eager where that path can never run: with the noise trace (it measures every relinearised square),
    // without the plane-source key switch or with digits wider than 16 bits, when the size-3 slab would pass 8 GiB, and for a square of
    // squares, whose next consumer is another product rather than a scalar-MAC layer.
    const size_t s3 = (size_t)3 * c.k * c.N;
    if (!chained && !c.trace_noise && relin_planes_built(c) && hm::bit_length(c.dm_relin.mask) <= 16 && (size_t)total * s3 <= ((size_t)1 << 30)) {
        auto g = std::make_shared<PendingGroup>();
        g->total = total;
        g->ct_slot = X.ct_slot;
        g->slab3.resize(c.P);
        for (int ch = 0; ch < c.P; ch++) {
            c.set_channel(ch);
            (void)relin_keys(c, ch, total, X.ct_slot.data()); // a missing key fails here, as it does for the eager square
            g->slab3[ch] = c.alloc((size_t)total * s3);
            const std::vector<const u64 *> xs = X.blocks(ch);
            op_multiply(c, ch, xs, xs, g->slab3[ch]->p);
            c.op_count[Context::OP_RELINEARIZE] += (uint64_t)total; // booked here, as the eager square books it
        }
        for (int i = 0; i < n; i++) {
            out[i] = new_vec(c, in[i]->dim, in[i]->scale * in[i]->scale, in[i]->format, true, in[i]->blocks);
            out[i]->slot = X.vslot[i];
            out[i]->pend = g;
            out[i]->pend_ct = (size_t)X.first[i];
            g->members.push_back(out[i]);
        }
        return CNHE_OK;
    }
    square_layer(c, X, nullptr, out);
    API_END
}
// Chosen size-3 words as pending squares: n one-block vectors sharing one group in key slot `slot`, as cnhe_layer_square returns them, so
// that a test can place any digit in any plane of the exact scalar-MAC path.  Refused where the square would be eager, and for words that
// are not canonical residues.
extern "C" int cnhe_raw_import_products(cnhe_ctx *h, const uint64_t *words, int n, uint64_t dim, double scale, int slot, cnhe_vec **out) {
    API_BEGIN(h)
    not_recorded(c, "uploads host words");
    if (!words || n < 1 || !out || dim < 1 || dim > c.N) fail("bad arguments");
    if (!c.slot_live(slot)) fail("no such key slot");
    const size_t s3 = (size_t)3 * c.k * c.N;
    if (c.trace_noise || !relin_planes_built(c) || hm::bit_length(c.dm_relin.mask) > 16 || (size_t)n * s3 > ((size_t)1 << 30))
        fail("the context keeps no products pending (noise trace, no plane-source key switch, digits wider than 16 bits or over 8 GiB)");
    for (int ch = 0; ch < c.P; ch++)
        for (size_t j = 0; j < (size_t)n * 3 * c.k; j++) {
            const uint64_t *r = words + ((size_t)ch * n * 3 * c.k + j) * c.N, q = c.q[j % c.k];
            for (size_t i = 0; i < c.N; i++)
                if (r[i] >= q) fail("the words are not canonical residues");
        }
    auto g = std::make_shared<PendingGroup>();
    g->total = n;
    g->ct_slot.assign(n, slot);
    g->slab3.resize(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        (void)relin_keys(c, ch, n, g->ct_slot.data()); // a missing key fails here, as it does for the square
        g->slab3[ch] = c.alloc((size_t)n * s3);
        CNHE_CUDA(cudaMemcpyAsync(g->slab3[ch]->p, words + (size_t)ch * n * s3, (size_t)n * s3 * 8, cudaMemcpyHostToDevice, c.stream));
    }
    c.sync();
    for (int i = 0; i < n; i++) {
        out[i] = new_vec(c, dim, scale, CNHE_DENSE, true, 1);
        out[i]->slot = slot;
        out[i]->pend = g;
        out[i]->pend_ct = (size_t)i;
        g->members.push_back(out[i]);
    }
    API_END
}
// The quadratic activation a x^2 + b x + c over a whole matrix, in cnhe_layer_square's passes: the BEHZ floor kernel scales the size-3
// product by A and adds B x and Delta C (FloorEpi), so out[i] = relinearize(A (.) in[i]^2) + B (.) in[i] + C word for word
extern "C" int cnhe_layer_poly2(cnhe_ctx *h, const cnhe_vec *const *in, int n, const cnhe_vec *a, const cnhe_vec *b, const cnhe_vec *cc,
                                cnhe_vec **out) {
    API_BEGIN(h)
    if (n < 1) fail("empty layer");
    ActCoeffs cf = quad_coeffs(c, a, b, cc);
    square_layer(c, act_inputs(c, in, n, "the inputs must be encrypted", &cf), &cf, out);
    API_END
}
// The square (a == NULL) or quadratic activation followed by a scalar-MAC layer, relinearising the layer's outputs instead of its squared
// inputs: the scalar MAC is linear in each polynomial of a size-3 ciphertext, so per plaintext prime
//   P3(x)  = A (.) multiply(x, x) + (B x0 + Delta C, B x1, 0)       (cnhe_layer_poly2's floor epilogue on the unrelinearised product)
//   out[m] = relinearize(sum_k w[m][k] (.) P3(in[gather[m K + k]]) + add_plain(bias[m]))
// word for word, with M key switches per block instead of n_in.  All n_in size-3 products of a channel are held at once.
extern "C" int cnhe_layer_activation_conv_dense(cnhe_ctx *h, const cnhe_vec *const *in, int n_in, const cnhe_vec *a, const cnhe_vec *b,
                                                const cnhe_vec *cc, const int32_t *gather, const cnhe_vec *const *weights,
                                                const cnhe_vec *const *bias, int M, int K, cnhe_vec **out) {
    API_BEGIN(h)
    if (n_in < 1) fail("empty layer");
    std::optional<ActCoeffs> cf; // none: the square
    if (a || b || cc) cf = quad_coeffs(c, a, b, cc);
    same_ctx(c, in[0]);
    if (cf) cf->read(c, in[0]->scale);
    const double act_scale = cf ? cf->out_scale : in[0]->scale * in[0]->scale;
    const MacLayer L = mac_prepare(c, in, n_in, act_scale, gather, weights, bias, M, K);
    const ActInputs X(in, n_in);
    const int bl = L.bl, total = X.total();
    const size_t w3 = (size_t)3 * c.k * c.N;
    if ((size_t)total * w3 > ((size_t)1 << 30)) fail("the size-3 products of the layer's inputs exceed the 8 GiB scratch limit");
    std::vector<int> ct_slot; // relinearisation: every output under the key slot its taps share
    for (int m = 0; m < M; m++) ct_slot.insert(ct_slot.end(), bl, L.out_slot[m]);
    std::vector<BufRef> big(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        big[ch] = c.alloc((size_t)M * bl * c.ct_words());
    }
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c); // the size-3 slabs of this channel go back to its stream when its key switch is done
        u64 *x3 = c.ws_alloc((size_t)total * w3), *y3 = c.ws_alloc((size_t)M * bl * w3);
        FloorEpi epi;
        if (cf) epi = act_epilogue(c, ch, X, cf->res[ch][2], cf->res[ch][1], cf->res[ch][0]);
        const std::vector<const u64 *> xs = X.blocks(ch);
        op_multiply(c, ch, xs, xs, x3, cf ? &epi : nullptr);
        std::vector<const u64 *> ip((size_t)bl * n_in);
        for (int bb = 0; bb < bl; bb++)
            for (int i = 0; i < n_in; i++) ip[(size_t)bb * n_in + i] = x3 + ((size_t)i * bl + bb) * w3;
        std::vector<u64 *> op((size_t)M * bl);
        for (size_t j = 0; j < op.size(); j++) op[j] = y3 + j * w3;
        mac_channel(c, L, ch, ip, op, 3);
        op_relinearize(c, ch, y3, M * bl, big[ch]->p, ct_slot.data());
    }
    for (int m = 0; m < M; m++) out[m] = slab_output(c, big, (size_t)m * bl, in[0], act_scale * weights[0]->scale, L.out_slot[m]);
    API_END
}
// Quartic and cubic activations in two multiplicative levels built from squares only (DESIGN.md section 4.12).  Per plaintext prime t,
// with the coefficients c_j of x^j reduced mod t and A the leading one:
//   quartic (A, B, C, D, E): beta = B (2A)^-1, gamma = (C A^-1 - beta^2) 2^-1, D' = D - B gamma, E' = E - A gamma^2:
//     q = x^2 + beta x + gamma,  P(x) = A q^2 + D' x + E'
//   cubic (A, B, C, D): lambda = A 2^-1, gamma = (B lambda^-1 - 1) 2^-1, C' = C - A gamma, D' = D - lambda gamma^2:
//     u = x^2, q1 = u + x + gamma,  P(x) = lambda (q1^2 - u^2) + C' x + D'
struct PolyConsts {
    u64 lead, b, g, lin, cst; // quartic: A, beta, gamma, D', E'   cubic: lambda, -, gamma, C', D'
};
static PolyConsts poly_consts(u64 t, int degree, const u64 *cf /*degree + 1 residues, cf[j] of x^j*/) {
    const u64 inv2 = hm::inv(2, t);
    PolyConsts k{};
    if (degree == 4) {
        const u64 A = cf[4], B = cf[3], C = cf[2], D = cf[1], E = cf[0];
        k.lead = A;
        k.b = hm::mul(B, hm::inv(hm::add(A, A, t), t), t);
        k.g = hm::mul(hm::sub(hm::mul(C, hm::inv(A, t), t), hm::mul(k.b, k.b, t), t), inv2, t);
        k.lin = hm::sub(D, hm::mul(B, k.g, t), t);
        k.cst = hm::sub(E, hm::mul(A, hm::mul(k.g, k.g, t), t), t);
    } else {
        const u64 A = cf[3], B = cf[2], C = cf[1], D = cf[0];
        k.lead = hm::mul(A, inv2, t);
        k.g = hm::mul(hm::sub(hm::mul(B, hm::inv(k.lead, t), t), 1, t), inv2, t);
        k.lin = hm::sub(C, hm::mul(A, k.g, t), t);
        k.cst = hm::sub(D, hm::mul(k.lead, hm::mul(k.g, k.g, t), t), t);
    }
    return k;
}
// P(x) of degree 3 or 4 over a whole matrix.  Quartic: level 1 is cnhe_layer_poly2(x; 1, beta, gamma); level 2 squares q with the floor
// epilogue (A, D', E') reading the original input x.  Cubic: level 1 squares x (u) and forms q1 = u + x + gamma; level 2 squares q1 and u
// side by side in one wave, and the pair floor subtracts the two products and applies (lambda, C', D') before one key switch per output
extern "C" int cnhe_layer_poly(cnhe_ctx *h, const cnhe_vec *const *in, int n, const cnhe_vec *const *coeffs, int degree, cnhe_vec **out) {
    API_BEGIN(h)
    if (n < 1) fail("empty layer");
    if (degree != 3 && degree != 4) fail("the degree must be 3 or 4");
    ActCoeffs cf(c, coeffs, degree, "the leading coefficient is required");
    const ActInputs X = act_inputs(c, in, n, "the inputs must be encrypted", &cf);
    const int total = X.total();
    const size_t cw = c.ct_words();
    std::vector<BufRef> big(c.P);
    auto &ops = c.op_count;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        const PolyConsts k = poly_consts(c.ch[ch].t, degree, cf.res[ch].data());
        big[ch] = c.alloc((size_t)total * cw);
        const std::vector<const u64 *> xs = X.blocks(ch);
        const u64 *const *x_tab = upload_ptrs(c, xs);
        FloorEpi e2 = act_epilogue(c, ch, X, k.lead, k.lin, k.cst, x_tab);
        BufRef mid;
        std::vector<const u64 *> sq; // the second level's squared operands
        if (degree == 4) {
            // level 1: q = cnhe_layer_poly2(x; 1, beta, gamma)
            mid = c.alloc((size_t)total * cw);
            FloorEpi e1 = act_epilogue(c, ch, X, 1, k.b, k.g);
            op_multiply_relin(c, ch, xs, xs, mid->p, X.ct_slot.data(), &e1);
            for (int i = 0; i < total; i++) sq.push_back(mid->p + (size_t)i * cw);
            // level 2: relinearize(A (.) q^2) + D' x + E'
            op_multiply_relin(c, ch, sq, sq, big[ch]->p, X.ct_slot.data(), &e2);
        } else {
            // level 1: u = relinearize(x^2) in [0, total), q1 = u + x + gamma in [total, 2 total): an addition, not a floor epilogue
            mid = c.alloc((size_t)2 * total * cw);
            u64 *u = mid->p, *q1 = mid->p + (size_t)total * cw;
            op_multiply_relin(c, ch, xs, xs, u, X.ct_slot.data());
            FloorEpi e1 = act_epilogue(c, ch, X, 1, 1, k.g, x_tab, false);
            c.prof_begin(2, 24.0 * c.N * total * 2 * c.k);
            c.check(launch_ct_add_epi(u, q1, total, c.k, c.logN, c.d_bc, e1, c.stream), "ct_add_epi");
            c.prof_end();
            ops[Context::OP_ADD] += (uint64_t)total;
            if (k.g) ops[Context::OP_ADD_PLAIN] += (uint64_t)total;
            for (int i = 0; i < total; i++) {
                sq.push_back(q1 + (size_t)i * cw);
                sq.push_back(u + (size_t)i * cw);
            }
            // level 2: relinearize(lambda (.) (q1^2 - u^2)) + C' x + D', one key switch per output
            op_multiply_relin(c, ch, sq, sq, big[ch]->p, X.ct_slot.data(), &e2, true);
            ops[Context::OP_SUB] += (uint64_t)total;
        }
    }
    for (int i = 0; i < n; i++) out[i] = slab_output(c, big, X.first[i], in[i], cf.out_scale, X.vslot[i]);
    API_END
}

// ---------------------------------------------------------------------------------------------------- diagonal matrix-vector product
// A plain matrix prepared for the diagonal (Halevi-Shoup) product with baby-step / giant-step (DESIGN.md section 4.10, slot layout in
// diag.cu): its nonzero generalised diagonals (b, s = n1 g + h), each rotated right by n1 g and encoded, ordered by g, then b, then h.
// A folded matrix (cnhe_diag_prepare_folded) holds its nonzero wrapped diagonals of fold width W instead, as (0, g, h).
struct DiagEntry { int b, g, h; };
struct cnhe_diag {
    Context *ctx = nullptr;
    int n_rows = 0;
    uint64_t dim = 0;
    double scale = 1.0;
    int n1 = 1, n2 = 1;
    int fold = 0; // the fold width W of a folded matrix, else 0
    std::vector<DiagEntry> diags;
    std::vector<BufRef> plains; // per channel: [diags][N] plaintexts, coefficient form mod t
    // cnhe_diag_prepare_ntt: the first ntt_groups giant-step groups (ntt_diags diagonals) also held lifted into every q_l and in NTT form,
    // per channel [ntt_diags][k][N] canonical words -- what cnhe_mat_mul_diagonal would otherwise lift and transform on every call
    int ntt_groups = 0, ntt_diags = 0;
    std::vector<BufRef> ntt;
    uint64_t ntt_bytes() const { return (uint64_t)ntt.size() * ntt_diags * ctx->k * ctx->N * 8; }
};
// key switches of rotate_rows(steps), 0 <= steps < N/2, on a context holding the Galois elements c.galois_elts: one with the step's own
// key, else one per hop
static std::vector<int> rotation_hops(const Context &c) {
    const int half = (int)(c.N / 2);
    const u64 m = 2ULL * c.N;
    std::vector<int> hops(half, 0);
    u64 e = 1;
    for (int s = 1; s < half; s++) {
        e = (e * 3) & (m - 1);
        const bool own = std::find(c.galois_elts.begin(), c.galois_elts.end(), e) != c.galois_elts.end();
        hops[s] = own ? 1 : (int)naf_hops(c.N, s).size();
    }
    return hops;
}
// key switches per input vector with n1 baby steps: rotate_rows(h) of v -- and of rotate_columns(v), one more, when a diagonal has b = 1 --
// for every h a nonzero diagonal (b, n1 g + h) uses, and rotate_rows(n1 g) for every g that has one.  nz: [2][N/2] nonzero flags
static long diag_cost(const std::vector<char> &nz, const std::vector<int> &hops, int n1) {
    const int half = (int)hops.size();
    std::vector<char> baby(2 * (size_t)n1, 0), giant(half / n1, 0);
    for (int b = 0; b < 2; b++)
        for (int s = 0; s < half; s++)
            if (nz[(size_t)b * half + s]) { baby[(size_t)b * n1 + s % n1] = 1; giant[s / n1] = 1; }
    long cost = 0;
    for (int h = 0; h < n1; h++) {
        if (baby[h]) cost += hops[h];
        if (baby[n1 + h]) cost += hops[h];
    }
    for (int h = 0; h < n1; h++)
        if (baby[n1 + h]) { cost += 1; break; }
    for (int g = 1; g < half / n1; g++)
        if (giant[g]) cost += hops[(size_t)n1 * g];
    return cost;
}

// diagonals lifted and forward transformed per wave: their NTT forms stay under 8 GiB (the product's waves, and the prepare's)
static int diag_wave_cap(const Context &c) { return (int)std::max<size_t>(1, ((size_t)1 << 30) / ((size_t)c.k * c.N)); }

// fold < 0: the generalised diagonals (cnhe_diag_prepare); fold >= 0: the wrapped diagonals of fold width `fold`, 0 letting the planner
// choose it (cnhe_diag_prepare_folded)
static void diag_prepare(Context &c, const cnhe_vec *const *rows, int n_rows, int baby_steps, uint64_t max_ntt_bytes, int fold, cnhe_diag **out) {
    if (!rows || !out || n_rows < 1) fail("bad arguments");
    const size_t N = c.N;
    const int half = (int)(N / 2);
    for (int r = 0; r < n_rows; r++) {
        same_ctx(c, rows[r]);
        if (rows[r]->enc) fail("the diagonal product takes a plain matrix");
        if (rows[r]->format != CNHE_DENSE) fail("Expecting dense vector format");
        if (rows[r]->blocks != 1) fail("the diagonal product expects single-block rows");
        if (rows[r]->dim != rows[0]->dim) fail("Dimensions do not match");
        if (rows[r]->scale != rows[0]->scale) fail("row scales differ");
    }
    if ((size_t)n_rows > N) fail("more rows than slots");
    if (baby_steps < 0 || (baby_steps & (baby_steps - 1)) || baby_steps > half) fail("baby_steps must be 0 or a power of two dividing N/2");
    const bool folded = fold >= 0;
    if (folded) {
        if (n_rows > half) fail("the folded product takes at most N/2 rows");
        if ((fold & (fold - 1)) || (fold && (fold < n_rows || fold > half))) fail("fold_width must be 0 or a power of two in [n_rows, N/2]");
        if (fold && baby_steps > fold) fail("baby_steps must divide the fold width");
        if (rows[0]->dim > N) fail("the folded product takes at most N columns");
    }
    const int R = n_rows, dim = (int)rows[0]->dim;
    std::unique_ptr<cnhe_diag> d(new cnhe_diag());
    d->ctx = &c;
    d->n_rows = R;
    d->dim = rows[0]->dim;
    d->scale = rows[0]->scale;
    // every channel's rows decoded to slot values, and the diagonals with a nonzero weight in some channel
    std::vector<BufRef> vals(c.P), flags(c.P);
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        u64 *plain = c.ws_alloc((size_t)R * N);
        for (int r = 0; r < R; r++)
            CNHE_CUDA(cudaMemcpyAsync(plain + (size_t)r * N, rows[r]->ptr(ch), N * 8, cudaMemcpyDeviceToDevice, c.stream));
        vals[ch] = c.alloc((size_t)R * N);
        op_decode(c, ch, plain, R, vals[ch]->p);
        flags[ch] = c.alloc(N / 2); // N unsigned flags
        CNHE_CUDA(cudaMemsetAsync(flags[ch]->p, 0, N * sizeof(unsigned), c.stream));
        if (folded) c.check(launch_diag_flags_folded(vals[ch]->p, R, dim, c.logN, reinterpret_cast<unsigned *>(flags[ch]->p), c.stream), "diag_flags");
        else c.check(launch_diag_flags(vals[ch]->p, R, dim, c.logN, reinterpret_cast<unsigned *>(flags[ch]->p), c.stream), "diag_flags");
    }
    std::vector<char> nz(N, 0);
    {
        std::vector<unsigned> hf(N);
        for (int ch = 0; ch < c.P; ch++) {
            c.set_channel(ch);
            CNHE_CUDA(cudaMemcpyAsync(hf.data(), flags[ch]->p, N * sizeof(unsigned), cudaMemcpyDeviceToHost, c.stream));
            CNHE_CUDA(cudaStreamSynchronize(c.stream));
            for (size_t i = 0; i < N; i++) nz[i] |= hf[i] != 0;
        }
    }
    const std::vector<int> hops = rotation_hops(c);
    int n1 = baby_steps;
    if (folded) {
        // key switches per input of (W, n1): the BSGS rotations over the wrapped diagonals (b = 0 only), the column fold when the input
        // reaches the second row, and log2(N/2 / W) row folds.  The fewest win; on a tie the smaller W, then the smaller n1.
        int w_lo = fold, w_hi = fold;
        if (!fold) {
            for (w_lo = 1; w_lo < R; w_lo *= 2) {}
            w_hi = half;
        }
        std::vector<char> nzw(N, 0), best_nz;
        long best = -1;
        for (int w = w_lo; w <= w_hi; w *= 2) {
            std::fill(nzw.begin(), nzw.end(), 0);
            for (int s = 0; s < half; s++)
                if (nz[s]) nzw[s & (w - 1)] = 1;
            long fixed = dim > half ? 1 : 0;
            for (int v = w; v < half; v *= 2) fixed++;
            for (int t = baby_steps ? baby_steps : 1; t <= (baby_steps ? baby_steps : w) && t <= w; t *= 2) {
                const long cost = diag_cost(nzw, hops, t) + fixed;
                if (best < 0 || cost < best) { best = cost; n1 = t; d->fold = w; best_nz = nzw; }
            }
        }
        if (best < 0) fail("baby_steps must divide the fold width");
        nz.swap(best_nz);
    } else if (!n1) {
        long best = -1;
        for (int t = 1; t <= half; t *= 2) {
            const long cost = diag_cost(nz, hops, t);
            if (best < 0 || cost < best) { best = cost; n1 = t; }
        }
    }
    d->n1 = n1;
    d->n2 = (folded ? d->fold : half) / n1;
    for (int g = 0; g < d->n2; g++)
        for (int b = 0; b < 2; b++)
            for (int hh = 0; hh < n1; hh++)
                if (nz[(size_t)b * half + g * n1 + hh]) d->diags.push_back({b, g, hh});
    if (d->diags.empty()) d->diags.push_back({0, 0, 0}); // an all-zero matrix keeps one (zero) diagonal: its product is an encryption of 0
    const int nd = (int)d->diags.size();
    std::vector<int> desc((size_t)3 * nd);
    for (int j = 0; j < nd; j++) {
        desc[3 * j] = d->diags[j].b;
        desc[3 * j + 1] = n1 * d->diags[j].g;
        desc[3 * j + 2] = d->diags[j].h;
    }
    d->plains.resize(c.P);
    const int DW = 2048; // diagonals gathered per wave
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        d->plains[ch] = c.alloc((size_t)nd * N);
        int *ddesc = reinterpret_cast<int *>(c.ws_alloc(((size_t)3 * nd + 1) / 2));
        c.h2d(ddesc, desc.data(), desc.size() * sizeof(int));
        for (int j0 = 0; j0 < nd; j0 += DW) {
            WsScope wave(c);
            const int m = std::min(DW, nd - j0);
            u64 *dv = c.ws_alloc((size_t)m * N);
            c.check(launch_diag_gather(vals[ch]->p, R, dim, ddesc + 3 * j0, m, c.logN, d->fold, dv, c.stream), "diag_gather");
            op_encode(c, ch, dv, m, (int)N, d->plains[ch]->p + (size_t)j0 * N);
        }
    }
    // the longest prefix of whole giant-step groups whose NTT forms, over all channels, fit in max_ntt_bytes
    const uint64_t per_diag = (uint64_t)c.P * c.k * N * 8;
    const uint64_t fit = max_ntt_bytes / per_diag;
    for (int j = 0; j < nd; j++) {
        if (j + 1 < nd && d->diags[j + 1].g == d->diags[j].g) continue; // j ends its group
        if ((uint64_t)j + 1 > fit) break;
        d->ntt_groups++;
        d->ntt_diags = j + 1;
    }
    if (d->ntt_diags) {
        // exactly the product's words: launch_plain_lift, then the canonical forward transform
        const size_t kN = (size_t)c.k * N;
        const int cap = diag_wave_cap(c);
        d->ntt.resize(c.P);
        for (int ch = 0; ch < c.P; ch++) {
            c.set_channel(ch);
            d->ntt[ch] = c.alloc((size_t)d->ntt_diags * kN);
            for (int j0 = 0; j0 < d->ntt_diags; j0 += cap) {
                const int m = std::min(cap, d->ntt_diags - j0);
                u64 *L = d->ntt[ch]->p + (size_t)j0 * kN;
                c.check(launch_plain_lift(d->plains[ch]->p + (size_t)j0 * N, L, m, (int)N, c.k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "plain_lift");
                op_ntt(c, L, L, m * c.k, 0, c.k, false);
            }
        }
    }
    c.sync();
    *out = d.release();
}

extern "C" int cnhe_diag_prepare(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, int baby_steps, cnhe_diag **out) {
    API_BEGIN(h)
    not_recorded(c, "prepares a matrix (it reads device words back)");
    diag_prepare(c, rows, n_rows, baby_steps, 0, -1, out);
    API_END
}

extern "C" int cnhe_diag_prepare_ntt(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, int baby_steps, uint64_t max_ntt_bytes,
                                     cnhe_diag **out) {
    API_BEGIN(h)
    not_recorded(c, "prepares a matrix (it reads device words back)");
    diag_prepare(c, rows, n_rows, baby_steps, max_ntt_bytes, -1, out);
    API_END
}

extern "C" int cnhe_diag_prepare_folded(cnhe_ctx *h, const cnhe_vec *const *rows, int n_rows, int fold_width, int baby_steps,
                                        uint64_t max_ntt_bytes, cnhe_diag **out) {
    API_BEGIN(h)
    not_recorded(c, "prepares a matrix (it reads device words back)");
    if (fold_width < 0) fail("fold_width must be 0 or a power of two in [n_rows, N/2]");
    diag_prepare(c, rows, n_rows, baby_steps, max_ntt_bytes, fold_width, out);
    API_END
}

extern "C" int cnhe_diag_info(const cnhe_diag *d, int *n_rows, uint64_t *dim, int *n1, int *n2, int *n_diags, uint64_t *device_bytes) {
    if (!d) return set_err(CNHE_ERR_INVALID, "null matrix");
    if (n_rows) *n_rows = d->n_rows;
    if (dim) *dim = d->dim;
    if (n1) *n1 = d->n1;
    if (n2) *n2 = d->n2;
    if (n_diags) *n_diags = (int)d->diags.size();
    if (device_bytes) *device_bytes = (uint64_t)d->plains.size() * d->diags.size() * d->ctx->N * 8 + d->ntt_bytes();
    return CNHE_OK;
}

extern "C" int cnhe_diag_fold_width(const cnhe_diag *d, int *width) {
    if (!d || !width) return set_err(CNHE_ERR_INVALID, "null argument");
    *width = d->fold;
    return CNHE_OK;
}

extern "C" int cnhe_diag_ntt_info(const cnhe_diag *d, int *resident_giant_steps, int *resident_diags, uint64_t *ntt_bytes) {
    if (!d) return set_err(CNHE_ERR_INVALID, "null matrix");
    if (resident_giant_steps) *resident_giant_steps = d->ntt_groups;
    if (resident_diags) *resident_diags = d->ntt_diags;
    if (ntt_bytes) *ntt_bytes = d->ntt_bytes();
    return CNHE_OK;
}

extern "C" int cnhe_diag_export(cnhe_ctx *h, const cnhe_diag *d, int channel, int index, uint64_t *dst, size_t cap_words, int *bgh) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (!d || d->ctx != &c) fail("matrix belongs to another context");
    if (channel < 0 || channel >= c.P || index < 0 || index >= (int)d->diags.size()) fail("index out of range");
    if (dst) {
        if (cap_words < c.N) fail("buffer too small");
        c.set_channel(channel);
        CNHE_CUDA(cudaMemcpyAsync(dst, d->plains[channel]->p + (size_t)index * c.N, c.N * 8, cudaMemcpyDeviceToHost, c.stream));
        CNHE_CUDA(cudaStreamSynchronize(c.stream));
    }
    if (bgh) {
        bgh[0] = d->diags[index].b;
        bgh[1] = d->diags[index].g;
        bgh[2] = d->diags[index].h;
    }
    API_END
}

extern "C" int cnhe_diag_export_ntt(cnhe_ctx *h, const cnhe_diag *d, int channel, int index, uint64_t *dst, size_t cap_words) {
    API_BEGIN(h)
    not_recorded(c, "returns words to the host");
    if (!d || d->ctx != &c) fail("matrix belongs to another context");
    if (channel < 0 || channel >= c.P || index < 0 || index >= d->ntt_diags) fail("index outside the resident diagonals");
    const size_t kN = (size_t)c.k * c.N;
    if (!dst || cap_words < kN) fail("buffer too small");
    c.set_channel(channel);
    CNHE_CUDA(cudaMemcpyAsync(dst, d->ntt[channel]->p + (size_t)index * kN, kN * 8, cudaMemcpyDeviceToHost, c.stream));
    CNHE_CUDA(cudaStreamSynchronize(c.stream));
    API_END
}

extern "C" int cnhe_diag_destroy(cnhe_diag *d) {
    if (!d) return CNHE_OK;
    try {
        std::lock_guard<std::recursive_mutex> lock(d->ctx->mu);
        cudaSetDevice(d->ctx->device);
        delete d;
    } catch (...) { return set_err(CNHE_ERR_INVALID, "destroy failed"); }
    return CNHE_OK;
}

// y = sum_g rotate_rows(n1 g)( sum_{b,h} D'[g][b,h] (.) rotate_columns^b rotate_rows(h)(v) ) for B vectors at once (one per client; their key
// slots may differ).  Per channel: the baby-step rotations of every client in one op_rotate_rows_multi (after one column rotation per
// client when a diagonal has b = 1), their forward transforms, then waves of giant steps -- the wave's diagonals lifted and transformed
// (a matrix from cnhe_diag_prepare_ntt holds those words for its resident prefix of giant steps, which then takes one wave and
// k_diag_mac_resident), every client's inner sums in the NTT domain (k_diag_mac; dyadic products and additions off the FP64 path: the
// same residues), the inverse transforms -- and finally the giant-step rotations of every (g, client) in one op_rotate_rows_multi and
// each client's sum.
// Each inner sum equals the sum of the separate multiply_plain results, since the inverse transform is linear mod q_l.
// A folded matrix then folds every client's sum in one wave per step -- rotate_columns when its input reaches the second row, then
// rotate_rows by W, 2W, ..., N/4 (sum_slots_batched) -- so that slot i < n_rows holds row i's sum, and multiplies all B sums by one mask
// plaintext (1 in slots 0 .. n_rows - 1, 0 elsewhere) that clears the periodic copies beyond them.
extern "C" int cnhe_mat_mul_diagonal(cnhe_ctx *h, const cnhe_diag *d, const cnhe_vec *const *vs, int B, cnhe_vec **out) {
    API_BEGIN(h)
    if (!d || !vs || !out || B < 1) fail("bad arguments");
    if (d->ctx != &c) fail("matrix belongs to another context");
    for (int b = 0; b < B; b++) {
        same_ctx(c, vs[b]);
        if (!vs[b]->enc) fail("at least one parameter has to be encrypted");
        if (vs[b]->format != CNHE_DENSE) fail("Expecting dense vector format");
        if (vs[b]->blocks != 1) fail("the diagonal product expects a single-block vector");
        if (vs[b]->dim != d->dim) fail("Dimensions do not match");
        if (vs[b]->scale != vs[0]->scale) fail("the input vectors must share scale");
    }
    const std::vector<int> vslot = vec_slots(c, vs, B);
    const size_t N = c.N, ctw = c.ct_words(), kN = (size_t)c.k * N;
    const int k = c.k, n1 = d->n1, nd = (int)d->diags.size();
    // baby steps in use and their place in the baby-step buffer; giant steps in use and where their diagonals start
    std::vector<int> xidx(2 * (size_t)n1, -1), xsel(nd), gs, gstart;
    for (const DiagEntry &e : d->diags) xidx[(size_t)e.b * n1 + e.h] = 0;
    int nx = 0;
    for (int &x : xidx)
        if (x == 0) x = nx++;
    bool col = false;
    for (int j = 0; j < nd; j++) {
        const DiagEntry &e = d->diags[j];
        xsel[j] = xidx[(size_t)e.b * n1 + e.h];
        col = col || e.b == 1;
        if (j == 0 || e.g != d->diags[j - 1].g) { gs.push_back(e.g); gstart.push_back(j); }
    }
    gstart.push_back(nd);
    const int ng = (int)gs.size();
    bool fp = c.fp_elementwise;
    for (int l = 0; l < k; l++) fp = fp && c.h_tabs[l].fp_ok;
    const int fpq = fp ? 1 : 0;
    std::vector<std::unique_ptr<cnhe_vec>> outs(B);
    std::vector<BufRef> slab(c.P); // folded: the B outputs side by side, for the fold ladder and the mask
    for (int ch = 0; ch < c.P && d->fold; ch++) {
        c.set_channel(ch);
        slab[ch] = c.alloc((size_t)B * ctw);
    }
    for (int b = 0; b < B; b++) {
        outs[b].reset(new_vec(c, (uint64_t)d->n_rows, vs[0]->scale * d->scale, CNHE_DENSE, true, 1));
        outs[b]->slot = vslot[b];
        if (d->fold) slab_view(outs[b].get(), slab, (size_t)b);
        else alloc_channels(outs[b].get());
    }
    // diagonals per wave: their lifted NTT forms stay under 8 GiB (a wave always takes at least one giant step); the resident groups
    // (cnhe_diag_prepare_ntt) need no such scratch and go in one wave of their own
    const int cap = diag_wave_cap(c), nres = d->ntt_groups;
    for (int ch = 0; ch < c.P; ch++) {
        c.set_channel(ch);
        WsScope scope(c);
        // baby steps: X[xidx[b n1 + h]][client] = rotate_rows(h)(rotate_columns^b(v)), then their NTT forms
        u64 *X = c.ws_alloc((size_t)nx * B * ctw);
        u64 *kv = col ? c.ws_alloc((size_t)B * ctw) : nullptr;
        if (col)
            for (int b = 0; b < B; b++) op_rotate_columns(c, ch, vs[b]->ptr(ch), 1, kv + (size_t)b * ctw, &vslot[b]);
        {
            std::vector<RotateJob> jobs;
            for (int i = 0; i < 2 * n1; i++) {
                if (xidx[i] < 0) continue;
                for (int b = 0; b < B; b++)
                    jobs.push_back({i >= n1 ? kv + (size_t)b * ctw : vs[b]->ptr(ch), i % n1, X + ((size_t)xidx[i] * B + b) * ctw, vslot[b]});
            }
            op_rotate_rows_multi(c, ch, jobs);
        }
        op_ntt(c, X, X, nx * B * 2 * k, 0, k, false);
        u64 *acc = c.ws_alloc((size_t)ng * B * ctw); // [g][client], coefficient form once its wave is done
        const int *dxsel = nullptr;
        if (fp) {
            int *p = reinterpret_cast<int *>(c.ws_alloc(((size_t)nd + 1) / 2));
            c.h2d(p, xsel.data(), (size_t)nd * sizeof(int));
            dxsel = p;
        }
        for (int gi0 = 0; gi0 < ng;) {
            WsScope wave(c);
            const bool resident = gi0 < nres; // then gi0 = 0, and the wave is the whole resident prefix
            int gi1 = resident ? nres : gi0 + 1;
            while (!resident && gi1 < ng && gstart[gi1 + 1] - gstart[gi0] <= cap) gi1++;
            const int j0 = gstart[gi0], m = gstart[gi1] - j0, gw = gi1 - gi0;
            u64 *L;
            if (resident) {
                L = d->ntt[ch]->p;
            } else {
                L = c.ws_alloc((size_t)m * kN);
                c.prof_begin(5, 8.0 * m * (N + kN));
                c.check(launch_plain_lift(d->plains[ch]->p + (size_t)j0 * N, L, m, (int)N, k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "plain_lift");
                c.prof_end();
                op_ntt(c, L, L, m * k, 0, k, false);
            }
            u64 *A = acc + (size_t)gi0 * B * ctw;
            if (fp) {
                std::vector<int> st(gw + 1);
                for (int i = 0; i <= gw; i++) st[i] = gstart[gi0 + i] - j0;
                int *dst = reinterpret_cast<int *>(c.ws_alloc(((size_t)gw + 2) / 2));
                c.h2d(dst, st.data(), st.size() * sizeof(int));
                // HBM: the wave's diagonals once per 8 clients, the baby steps once (the giant steps share them through L2), the sums once
                c.prof_begin(4, 8.0 * ((double)((B + 7) / 8) * m * kN + (double)nx * B * ctw + (double)gw * B * ctw));
                if (resident)
                    c.check(launch_diag_mac_resident(L, X, dst, dxsel + j0, A, gw, B, k, c.logN, &c.h_bf, c.stream), "diag_mac_resident");
                else c.check(launch_diag_mac(L, X, dst, dxsel + j0, A, gw, B, k, c.logN, &c.h_bf, c.stream), "diag_mac");
                c.prof_end();
            } else {
                u64 *tmp = c.ws_alloc((size_t)B * ctw);
                for (int gi = gi0; gi < gi1; gi++) {
                    u64 *Ag = acc + (size_t)gi * B * ctw;
                    for (int j = gstart[gi]; j < gstart[gi + 1]; j++) {
                        const u64 *xs = X + (size_t)xsel[j] * B * ctw, *dj = L + (size_t)(j - j0) * kN;
                        if (j == gstart[gi]) { c.check(launch_dyadic_bcast(xs, dj, Ag, B, 2, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic"); continue; }
                        c.check(launch_dyadic_bcast(xs, dj, tmp, B, 2, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
                        c.check(launch_ct_add(Ag, tmp, Ag, (size_t)B * ctw, k, c.logN, c.d_bc, 0, c.stream), "ct_add");
                    }
                }
            }
            op_ntt(c, A, A, gw * B * 2 * k, 0, k, true);
            gi0 = gi1;
        }
        c.note(Context::OP_MULTIPLY_PLAIN, ch, B * nd);
        if (nd > ng) c.note(Context::OP_ADD, ch, B * (nd - ng));
        // giant steps, in place, then each client's sum over g
        {
            std::vector<RotateJob> jobs;
            for (int gi = 0; gi < ng; gi++)
                for (int b = 0; b < B; b++) {
                    u64 *p = acc + ((size_t)gi * B + b) * ctw;
                    jobs.push_back({p, n1 * gs[gi], p, vslot[b]});
                }
            op_rotate_rows_multi(c, ch, jobs);
        }
        for (int b = 0; b < B; b++) {
            if (ng == 1) {
                CNHE_CUDA(cudaMemcpyAsync(outs[b]->ptr(ch), acc + (size_t)b * ctw, ctw * 8, cudaMemcpyDeviceToDevice, c.stream));
                c.note_copy(outs[b]->ptr(ch), acc + (size_t)b * ctw);
                continue;
            }
            std::vector<const u64 *> terms;
            for (int gi = 0; gi < ng; gi++) terms.push_back(acc + ((size_t)gi * B + b) * ctw);
            do_add_many(c, ch, terms, outs[b]->ptr(ch));
        }
        if (d->fold) {
            u64 *y = slab[ch]->p;
            sum_slots_batched(c, ch, y, B, N / 2, vslot.data(), (uint64_t)d->fold, d->dim > N / 2);
            std::vector<u64> ones(N, 0);
            std::fill(ones.begin(), ones.begin() + d->n_rows, 1);
            u64 *mv = c.ws_alloc(N), *mask = c.ws_alloc(N);
            c.h2d(mv, ones.data(), N * 8);
            op_encode(c, ch, mv, 1, (int)N, mask);
            std::vector<const u64 *> cts(B);
            for (int b = 0; b < B; b++) cts[b] = y + (size_t)b * ctw;
            op_multiply_plain_dense_outer(c, ch, cts, mask, 1, y);
        }
    }
    for (int b = 0; b < B; b++) out[b] = outs[b].release();
    API_END
}
