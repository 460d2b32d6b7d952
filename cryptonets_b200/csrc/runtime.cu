// Host runtime of libcnhe (see runtime.h).  Product code: builds every table with hostmath.h, never touches oracle/.
#include "runtime.h"
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include <sys/random.h>

#include "hostmath.h"

namespace cnhe {

// 256-bit ChaCha20 key straight from the kernel CSPRNG (getrandom(2)); no fallback: a context without entropy must not encrypt
void rng_from_os(RngKey &rk) {
    memset(&rk, 0, sizeof(rk));
    unsigned char *p = reinterpret_cast<unsigned char *>(rk.key);
    size_t got = 0;
    while (got < sizeof(rk.key)) {
        const ssize_t r = getrandom(p + got, sizeof(rk.key) - got, 0);
        if (r <= 0) throw Error(-2, "getrandom() failed: no OS entropy for key generation / encryption");
        got += (size_t)r;
    }
    rk.secure = 1;
}
const char *op_kind_name(int kind) {
    static const char *names[] = {"Encryption", "Decryption", "Multiplication", "Relinarization", "PlainMultiplication", "ScalarMultiplication",
                                  "Addition", "PlainAddition", "Subtraction", "PlainSubtraction", "Rotation", "ColumnRotation", "AddMany",
                                  "AddManyItemCount"};
    return kind >= 0 && kind < Context::OP_COUNT ? names[kind] : "?";
}
void Context::note(OpKind kind, int channel, int n, const u64 *first_out, const u64 *in0, const u64 *in1, double aux) {
    op_count[kind] += (uint64_t)n;
    if (!trace_noise || kind == OP_ADD_MANY_ITEMS) return;
    int budget = -1;
    const int b0 = in0 ? known_budget(in0) : -1, b1 = in1 ? known_budget(in1) : -1; // before the output (possibly in place) is re-measured
    if (first_out && channel >= 0 && channel < P && ch[channel].have_sk && !foreign) { // other slots' ciphertexts: only slot 0's key is here
        budget = op_noise_budget(*this, channel, first_out);
        // the call wrote n ciphertexts starting here: whatever was recorded for these addresses (recycled blocks) is stale now
        budget_of.erase(budget_of.lower_bound(first_out), budget_of.lower_bound(first_out + (size_t)n * ct_words()));
        budget_of[first_out] = budget;
    }
    trace.push_back({(int)kind, channel, n, budget, b0, b1, (int)std::lround(aux * 1000.0), 0});
}

void cuda_check(cudaError_t e, const char *what) {
    if (e != cudaSuccess) throw Error(-2, std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}

// CNHE_TRACE_SLOW=<ms>: report host-side calls that take longer than that (diagnosing launch-path stalls)
static double trace_slow_ms() {
    static const double v = getenv("CNHE_TRACE_SLOW") ? atof(getenv("CNHE_TRACE_SLOW")) : 0.0;
    return v;
}
void Context::trace_gap(const char *what) {
    static thread_local std::chrono::steady_clock::time_point last = std::chrono::steady_clock::now();
    const auto now = std::chrono::steady_clock::now();
    const double ms = std::chrono::duration<double, std::milli>(now - last).count();
    if (ms > trace_ms && ms < 1000.0) fprintf(stderr, "[cnhe] %.2f ms of host time before/in launch of %s\n", ms, what);
    last = now;
}
DevBuf::DevBuf(size_t w, cudaStream_t s) : words(w), stream(s) {
    if (!w) return;
    if (trace_slow_ms() > 0) {
        const auto t0 = std::chrono::steady_clock::now();
        CNHE_CUDA(cudaMallocAsync((void **)&p, w * sizeof(u64), s));
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (ms > trace_slow_ms()) fprintf(stderr, "[cnhe] slow cudaMallocAsync: %.2f ms for %.1f MB\n", ms, w * 8.0 / 1e6);
        return;
    }
    CNHE_CUDA(cudaMallocAsync((void **)&p, w * sizeof(u64), s));
}
constexpr size_t RECYCLE_MIN_WORDS = (size_t)1 << 19;        // 4 MB
constexpr size_t RECYCLE_CAP_WORDS = (size_t)16 << 27;       // 16 GiB parked at most (a fifth of an 80 GB H100)
DevBuf::DevBuf(size_t w, cudaStream_t s, Context *ctx) : words(w), stream(s), owner(ctx) {
    if (!w) return;
    if (ctx && ctx->rec) { // recording: the graph's own memory
        arena = ctx->rec->arena;
        size_t got = 0;
        p = arena->take(w, s, got);
        if (p) words = got;
        else if (!(p = static_cast<u64 *>(arena->fresh(w * sizeof(u64)))))
            ctx->refuse("needs more device memory than a graph can own (recorded blocks are reused only by later allocations of a "
                        "similar size on the same stream)");
        return;
    }
    if (ctx && w >= RECYCLE_MIN_WORDS) {
        size_t got = 0;
        p = ctx->take_recycled(w, s, got);
        if (p) { words = got; return; }
    }
    if (ctx && !ctx->recycle.empty()) { // parked blocks of other sizes or streams are the first memory to give back when the device is full
        if (cudaMallocAsync((void **)&p, w * sizeof(u64), s) == cudaSuccess) return;
        p = nullptr;
        (void)cudaGetLastError();
        ctx->drop_recycled();
        CNHE_CUDA(cudaDeviceSynchronize()); // the frees complete, so that the pool can hand their memory to this stream
    }
    DevBuf fresh(w, s); // traced allocation path
    p = fresh.p;
    fresh.p = nullptr;
}
u64 *Context::take_recycled(size_t words, cudaStream_t s, size_t &got_words) {
    int best = -1;
    for (int i = 0; i < (int)recycle.size(); i++) {
        const Recycled &r = recycle[i];
        if (r.stream != s || r.words < words || r.words > words + words / 2) continue;
        if (best < 0 || r.words < recycle[best].words) best = i;
    }
    if (best < 0) return nullptr;
    u64 *p = recycle[best].p;
    got_words = recycle[best].words;
    recycle_words -= got_words;
    recycle.erase(recycle.begin() + best);
    return p;
}
bool Context::give_recycled(u64 *p, size_t words, cudaStream_t s) {
    if (!recycle_on || words < RECYCLE_MIN_WORDS || recycle_words + words > RECYCLE_CAP_WORDS || recycle.size() >= 256) return false;
    recycle.push_back({p, words, s});
    recycle_words += words;
    return true;
}
void Context::drop_recycled() {
    for (const Recycled &r : recycle) cudaFreeAsync(r.p, r.stream);
    recycle.clear();
    recycle_words = 0;
}
BufRef Context::alloc_upload(size_t words, cudaStream_t release_stream) {
    int pick = -1;
    for (int pass = 0; pass < 2 && pick < 0; pass++) // first a free slot whose last users are already done, else the longest-released one
        for (int i = 0; i < (int)upload_slots.size(); i++) {
            UploadSlot &u = upload_slots[i];
            if (u.busy || u.words < words || u.words > words + words / 2) continue;
            if (pass == 0 && cudaEventQuery(u.released) != cudaSuccess) continue;
            if (pick < 0 || u.stamp < upload_slots[pick].stamp) pick = i;
        }
    if (pick >= 0 && cudaEventQuery(upload_slots[pick].released) != cudaSuccess) { // grow to three slots of this size (enough for a
        int same = 0;                                                               // one-deep pipeline), then wait for the oldest
        for (const UploadSlot &u : upload_slots) same += u.words >= words && u.words <= words + words / 2;
        if (same < 3 * (int)streams.size()) pick = -1;
    }
    (void)cudaGetLastError(); // cudaEventQuery's cudaErrorNotReady is not an error
    if (pick < 0) { // first batch of this size: create the whole rotation at once (cudaMalloc of 0.5 GB costs ~50 ms; pay it up front)
        int same = 0;
        for (const UploadSlot &u : upload_slots) same += u.words >= words && u.words <= words + words / 2;
        const int want = same == 0 ? 3 * (int)streams.size() : same + 1;
        for (; same < want; same++) {
            UploadSlot u;
            u.words = words;
            u.busy = false;
            u.stamp = 0;
            CNHE_CUDA(cudaMalloc((void **)&u.p, words * sizeof(u64)));
            CNHE_CUDA(cudaEventCreateWithFlags(&u.released, cudaEventDisableTiming));
            upload_slots.push_back(u);
            if (pick < 0) pick = (int)upload_slots.size() - 1;
        }
    }
    UploadSlot &u = upload_slots[pick];
    u.busy = true;
    CNHE_CUDA(cudaStreamWaitEvent(copy_stream, u.released, 0)); // a never-recorded event is complete
    BufRef b = std::make_shared<DevBuf>(0, release_stream);
    b->p = u.p;
    b->words = u.words;
    b->owner = this;
    b->upload_slot = pick;
    return b;
}
void Context::release_upload(int slot, cudaStream_t s) {
    UploadSlot &u = upload_slots[slot];
    cudaEventRecord(u.released, s);
    u.busy = false;
    u.stamp = ++upload_stamp;
}
DevBuf::~DevBuf() {
    if (!p) return;
    if (arena) { arena->give(p, words, stream); return; }
    if (owner && owner->rec) { // a stream-ordered free now would be recorded into the graph: release it once the recording ends
        owner->rec->deferred.push_back({p, words, stream, upload_slot});
        return;
    }
    if (upload_slot >= 0) { owner->release_upload(upload_slot, stream); return; }
    if (owner && owner->give_recycled(p, words, stream)) return;
    cudaFreeAsync(p, stream);
}

u64 *GraphArena::take(size_t words, cudaStream_t s, size_t &got_words) { // the recycle list's fit rule
    int best = -1;
    for (int i = 0; i < (int)free.size(); i++) {
        const Free &f = free[i];
        if (f.stream != s || f.words < words || f.words > words + words / 2) continue;
        if (best < 0 || f.words < free[best].words) best = i;
    }
    if (best < 0) return nullptr;
    u64 *p = free[best].p;
    got_words = free[best].words;
    free.erase(free.begin() + best);
    return p;
}
void *GraphArena::fresh(size_t n) {
    void *p = nullptr;
    const cudaError_t e = cudaMalloc(&p, n); // not stream ordered: the block exists before the graph that uses it does
    if (e == cudaErrorMemoryAllocation) { (void)cudaGetLastError(); return nullptr; }
    CNHE_CUDA(e);
    blocks.push_back(p);
    bytes += n;
    return p;
}
const void *GraphArena::constant(const void *src, size_t n, cudaStream_t s) {
    const size_t need = (n + 255) & ~(size_t)255;
    if (const_off + need > const_cap) { // constants are small (pointer tables, masks, scalars): packed into 1 MB blocks
        const_cap = std::max<size_t>(need, (size_t)1 << 20);
        const_block = static_cast<unsigned char *>(fresh(const_cap));
        const_off = 0;
        if (!const_block) { const_cap = 0; throw Error(-3 /* CNHE_ERR_STATE */, "no device memory left for a graph's constants"); }
    }
    unsigned char *d = const_block + const_off;
    const_off += need;
    CNHE_CUDA(cudaMemcpyAsync(d, src, n, cudaMemcpyHostToDevice, s));
    CNHE_CUDA(cudaStreamSynchronize(s));
    return d;
}
GraphArena::~GraphArena() {
    for (void *p : blocks) cudaFree(p);
}
void release_deferred(Context &c, const std::vector<Recording::Deferred> &d) {
    for (const Recording::Deferred &x : d) {
        DevBuf b(0, x.stream, &c);
        b.p = x.p;
        b.words = x.words;
        b.upload_slot = x.upload_slot;
    }
}
cudaGraph_t end_capture(RecGroup &grp, bool keep) {
    const cudaStream_t s0 = grp.members[0]->streams[0];
    // every channel stream of every member joins the capturing stream 0 again (a capture cannot end with a stream left out); errors here
    // only mean the capture was already invalidated, which cudaStreamEndCapture reports
    for (Context *m : grp.members) {
        cudaSetDevice(m->device);
        for (cudaStream_t s : m->streams) {
            cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
            if (s != s0 && cudaStreamIsCapturing(s, &st) == cudaSuccess && st == cudaStreamCaptureStatusActive &&
                cudaEventRecord(m->ev_join, s) == cudaSuccess)
                cudaStreamWaitEvent(s0, m->ev_join, 0);
        }
    }
    cudaSetDevice(grp.members[0]->device);
    cudaGraph_t g = nullptr;
    if (cudaStreamEndCapture(s0, &g) != cudaSuccess) g = nullptr;
    for (Context *m : grp.members)
        for (cudaStream_t s : m->streams) { // a stream of an invalidated capture may still be in it
            cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
            if (cudaStreamIsCapturing(s, &st) == cudaSuccess && st != cudaStreamCaptureStatusNone) {
                cudaGraph_t stray = nullptr;
                if (cudaStreamEndCapture(s, &stray) == cudaSuccess && stray) cudaGraphDestroy(stray);
            }
        }
    (void)cudaGetLastError();
    if (g && !keep) { cudaGraphDestroy(g); g = nullptr; }
    return g;
}
void end_part(Context &c, std::vector<Recording::Deferred> *hold) {
    std::unique_ptr<Recording> r = std::move(c.rec);
    cudaSetDevice(c.device);
    for (int i = 0; i < Context::OP_COUNT; i++) c.op_count[i] = r->op0[i]; // recording runs nothing
    for (int i = 0; i < c.P; i++) c.ch[i].sanitized = r->sanitized0[i];
    c.launches = r->launches0;
    r->arena->recording = false;
    r->arena->free.clear();
    ws_release_all(c); // the last recorded call's temporaries go back to the graph's memory, not to the driver
    if (hold) *hold = std::move(r->deferred);
    else release_deferred(c, r->deferred);
}
void abort_recording(Context &c) {
    const std::shared_ptr<RecGroup> grp = c.rec->group;
    std::vector<Context *> locked;
    bool all = true;
    for (Context *m : grp->members) {
        if (m == &c) continue;
        if (!m->mu.try_lock()) { all = false; break; }
        locked.push_back(m);
    }
    if (all) {
        end_capture(*grp, false);
        for (Context *m : grp->members) end_part(*m);
    } else grp->abort_requested = true;
    for (Context *m : locked) m->mu.unlock();
    cudaSetDevice(c.device);
}

static std::vector<BufRef> &temps_of(Context &c) { return c.temps; } // per context, guarded by the context mutex

u64 *Context::ws_alloc(size_t words) {
    BufRef b = alloc(words ? words : 1);
    temps_of(*this).push_back(b);
    ws_used += words;
    return b->p;
}
void Context::sync() {
    if (rec) refuse("waits for the device");
    for (cudaStream_t s : streams) CNHE_CUDA(cudaStreamSynchronize(s));
}
void Context::join_streams() {
    for (size_t i = 1; i < streams.size(); i++) {
        CNHE_CUDA(cudaEventRecord(ev_join, streams[i]));
        CNHE_CUDA(cudaStreamWaitEvent(streams[0], ev_join, 0));
    }
}
void Context::fork_streams() {
    if (streams.size() < 2) return;
    CNHE_CUDA(cudaEventRecord(ev_join, streams[0]));
    for (size_t i = 1; i < streams.size(); i++) CNHE_CUDA(cudaStreamWaitEvent(streams[i], ev_join, 0));
}
void Context::refuse(const char *why) const {
    throw Error(-3 /* CNHE_ERR_STATE */, std::string(api) + " " + why + ": refused while the context records a graph");
}
void Context::upload(void *dst, const void *src, size_t bytes) {
    if (!bytes) return;
    if (rec) CNHE_CUDA(cudaMemcpyAsync(dst, rec->arena->constant(src, bytes, copy_stream), bytes, cudaMemcpyDeviceToDevice, stream));
    else CNHE_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
}
void Context::h2d(void *dst, const void *src, size_t bytes) {
    if (!bytes) return;
    if (rec) { upload(dst, src, bytes); return; } // the staging ring is overwritten by later calls: constants of a graph live in its memory
    if (!stage_buf) {
        stage_size = 64u << 20;
        CNHE_CUDA(cudaHostAlloc((void **)&stage_buf, stage_size, cudaHostAllocDefault));
        stage_ev.resize((size_t)STAGE_PARTS * streams.size());
        for (cudaEvent_t &e : stage_ev) CNHE_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        stage_ev_set.assign(STAGE_PARTS, 0);
    }
    const size_t part_size = stage_size / STAGE_PARTS;
    if (bytes > part_size) { // large: plain (staged by the driver) copy
        CNHE_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
        return;
    }
    const size_t need = (bytes + 255) & ~(size_t)255;
    size_t part = stage_off / part_size;
    if (stage_off + need > (part + 1) * part_size || stage_off + need > stage_size) { // move on to the next part
        // what was staged in the part being left is consumed once every channel stream has passed this point
        for (size_t s = 0; s < streams.size(); s++) CNHE_CUDA(cudaEventRecord(stage_ev[part * streams.size() + s], streams[s]));
        stage_ev_set[part] = 1;
        part = (part + 1) % STAGE_PARTS;
        if (stage_ev_set[part]) // its previous contents: staged STAGE_PARTS - 1 parts ago, long consumed in the steady state
            for (size_t s = 0; s < streams.size(); s++) CNHE_CUDA(cudaEventSynchronize(stage_ev[part * streams.size() + s]));
        stage_off = part * part_size;
    }
    memcpy(stage_buf + stage_off, src, bytes);
    CNHE_CUDA(cudaMemcpyAsync(dst, stage_buf + stage_off, bytes, cudaMemcpyHostToDevice, stream));
    stage_off += need;
}
void Context::prof_begin(int family, double bytes) {
    if (!prof) return;
    ProfRec r;
    r.family = family;
    r.bytes = bytes;
    for (cudaEvent_t *e : {&r.e0, &r.e1}) {
        if (!prof_pool.empty()) { *e = prof_pool.back(); prof_pool.pop_back(); }
        else CNHE_CUDA(cudaEventCreate(e));
    }
    CNHE_CUDA(cudaEventRecord(r.e0, stream));
    prof_recs.push_back(r);
}
void Context::prof_end() {
    if (!prof) return;
    CNHE_CUDA(cudaEventRecord(prof_recs.back().e1, stream));
    if (prof_recs.size() >= 4096) prof_flush();
}
void Context::prof_flush() {
    if (prof_recs.empty()) return;
    sync();
    for (auto &r : prof_recs) {
        float ms = 0;
        CNHE_CUDA(cudaEventElapsedTime(&ms, r.e0, r.e1));
        prof_ms[r.family] += ms;
        prof_bytes[r.family] += r.bytes;
        prof_n[r.family]++;
        prof_pool.push_back(r.e0);
        prof_pool.push_back(r.e1);
    }
    prof_recs.clear();
}
struct ProfScope {
    Context &c;
    ProfScope(Context &ctx, int family, double bytes) : c(ctx) { c.prof_begin(family, bytes); }
    ~ProfScope() { c.prof_end(); }
};
#define PROF(family, bytes) ProfScope prof_scope_##__LINE__(c, family, bytes)
Context::~Context() {
    cudaSetDevice(device);
    if (rec) abort_recording(*this);
    for (cudaStream_t s : streams) cudaStreamSynchronize(s);
    if (copy_stream) cudaStreamSynchronize(copy_stream);
    recycle_on = false; // buffers released from here on go straight back to the driver
    temps.clear();
    ch.clear();
    clients.clear(); // key slots: their buffers hold this context as owner, so they go before it does
    drop_recycled();
    if (d_bc) cudaFree(d_bc);
    if (d_bf) cudaFree(d_bf);
    if (d_tabs) cudaFree(d_tabs);
    if (d_table_mem) cudaFree(d_table_mem);
    if (d_index_map) cudaFree(d_index_map);
    if (d_sanitize_nonce) cudaFree(d_sanitize_nonce);
    for (auto &r : prof_recs) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    for (auto e : prof_pool) cudaEventDestroy(e);
    if (stage_buf) cudaFreeHost(stage_buf);
    for (cudaEvent_t e : stage_ev) cudaEventDestroy(e);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (ev_join) cudaEventDestroy(ev_join);
    for (cudaStream_t s : streams) cudaStreamDestroy(s);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    for (UploadSlot &u : upload_slots) { cudaFree(u.p); cudaEventDestroy(u.released); }
    if (ev_copy) cudaEventDestroy(ev_copy);
    for (cudaEvent_t e : ev_export) cudaEventDestroy(e);
}
// free the temporaries of the previous operation (stream ordered, so kernels still in flight keep their memory)
void ws_release_all(Context &c) {
    temps_of(c).clear();
    c.ws_used = 0;
}
WsScope::WsScope(Context &ctx) : c(ctx), mark(temps_of(ctx).size()) {}
WsScope::~WsScope() { temps_of(c).resize(mark); }

std::vector<u64> default_coeff_modulus(uint32_t N) {
    // DefaultParams.CoeffModulus128(N) of SEAL 3.2 ("HE Wrapper/AtomicSealBfvVector.cs:146"); values = the largest primes
    // congruent to 1 mod 2N with bit sizes 54 | 36,36,37 | 43,43,44,44,44 | 48x3,49x6 (checked by tests/test_tables.py)
    switch (N) {
    case 2048: return {0x3fffffff000001ULL};
    case 4096: return {0xffffee001ULL, 0xffffc4001ULL, 0x1ffffe0001ULL};
    case 8192: return {0x7fffffd8001ULL, 0x7fffffc8001ULL, 0xfffffffc001ULL, 0xffffff6c001ULL, 0xfffffebc001ULL};
    case 16384:
        return {0xfffffffd8001ULL,  0xfffffffa0001ULL,  0xfffffff00001ULL,  0x1fffffff68001ULL, 0x1fffffff50001ULL,
                0x1ffffffee8001ULL, 0x1ffffffea0001ULL, 0x1ffffffe88001ULL, 0x1ffffffe48001ULL};
    default: return {};
    }
}

static DMod make_dmod(u64 p) {
    DMod m;
    m.p = p;
    hm::barrett_ratio(p, m.r0, m.r1);
    return m;
}
// Decide whether the FP64 butterfly path is exact for this modulus and schedule its re-centring points.
// Magnitudes are tracked in units of p; every operand of a modular product must stay below 2^52 (limit L = 2^52/p, 10% margin).
static void fp_schedule(NttTab &tb, int logN, bool force_int) {
    tb.fp_ok = 0;
    tb.fwd_recenter = tb.inv_recenter = 0;
    const u64 p = tb.mod.p;
    if (force_int || hm::bit_length(p) > 49) return;
    const double L = 0.9 * 4503599627370496.0 / (double)p;
    auto c = [&](double a) { return 0.5 + 0.75 * a / (L / 0.9) + 1e-6; }; // bound of |a*w mod p| for |a| <= a*p, |w| <= p/2
    // forward schedule of a pass list; returns false when some pass overflows even after re-centring
    auto forward = [&](const int *rad, int np, unsigned &mask, double &A) {
        mask = 0;
        A = 1.0; // canonical input
        for (int i = 0; i < np; i++) {
            for (int attempt = 0; attempt < 2; attempt++) {
                double a = attempt ? 0.51 : A;
                bool ok = true;
                for (int s = 0; s < rad[i]; s++) { ok = ok && a < L; a += c(a); }
                ok = ok && a < L; // the canonicalisation / next pass consumes it
                if (ok) { A = a; if (attempt) mask |= 1u << i; break; }
                if (attempt) return false; // even a re-centred pass overflows
                if (i == 0) return false;  // the first pass reads straight from global memory: no re-centring slot
            }
        }
        return true;
    };
    int rad[4];
    const int np = ntt_pass_radices(logN, 0, rad);
    double A;
    if (!forward(rad, np, tb.fwd_recenter, A)) return;
    tb.fwd_recenter_split = 0;
    tb.split_ok = tb.split_out_rc = 0;
    // lazy forward output (|x| <= A p) feeds products of two such values (tensor) or of one with a canonical key word: both operands
    // of a modular product may be lazy only while A*A*p stays below 2^51
    auto out_rc = [&](double a) { return a * a * (double)p >= 0.9 * 2251799813685248.0; };
    if (logN >= 12) { // split form (CTA pairs at N = 16384, the fused key switch at 4096 / 8192): stage 0 rides on the first pass' loads
        const int split[3] = {logN - 8, 4, 4};
        double As;
        tb.split_ok = forward(split, 3, tb.fwd_recenter_split, As);
        if (logN == 14) {
            if (!tb.split_ok) return;
            A = std::max(A, As);
        } else if (tb.split_ok) {
            tb.split_out_rc = out_rc(As);
        }
    }
    tb.fwd_out_rc = out_rc(A);
    tb.fwd_out_bound = tb.fwd_out_rc ? 0.51 : A;
    // inverse: canonical or lazy input (tensor output: sum of two fresh products, <= 1.25 p); sums double every stage; bit v
    // re-centres the sums produced by stage v
    A = 1.25;
    for (int v = 0; v < logN; v++) {
        if (2 * A >= L) return;
        const double y = c(2 * A);
        double x = 2 * A;
        if (2 * x >= L) { tb.inv_recenter |= 1u << v; x = 0.51; }
        A = std::max(x, y);
    }
    if (A >= L) return;
    tb.fp_ok = 1;
}
static DigitMap make_digit_map(const std::vector<u64> &q, int w) {
    DigitMap dm;
    memset(&dm, 0, sizeof(dm));
    int d = 0;
    for (int i = 0; i < (int)q.size(); i++) {
        int bits = hm::bit_length(q[i]);
        for (int shift = 0; shift < bits; shift += w) {
            if (d >= 64) throw Error(-1, "decomposition bit count too small: more than 64 digits");
            dm.src[d] = (unsigned char)i;
            dm.shift[d] = (unsigned char)shift;
            d++;
        }
    }
    dm.D = d;
    dm.mask = w >= 64 ? ~0ULL : ((1ULL << w) - 1);
    return dm;
}

// Galois elements of KeyGenerator::galois_keys(dbc): 2N-1, then 3^(2^i), 3^-(2^i) for i < logN-1
std::vector<u64> standard_galois_elts(uint32_t N) {
    std::vector<u64> out;
    const u64 m2 = 2ULL * N;
    int logN = 0;
    while ((1u << logN) < N) logN++;
    out.push_back(m2 - 1);
    u64 p3 = 3, n3 = 0;
    for (u64 x = 1; x < m2; x += 2)
        if (((x * 3) & (m2 - 1)) == 1) { n3 = x; break; }
    for (int i = 0; i < logN - 1; i++) {
        out.push_back(p3);
        p3 = (p3 * p3) & (m2 - 1);
        out.push_back(n3);
        n3 = (n3 * n3) & (m2 - 1);
    }
    return out;
}

// ---- K_c (DESIGN 4.14).  A lifted word is x + c Q with |x + c Q| < Q (1 + k / m~) (c in {0, 1}; the centred m~ halves it), so a coefficient
// of a sum of K tensor products is below 2 K N Q^2 (1 + k / m~)^2 (d1 adds two negacyclic products of N terms each).  fast_floor returns
// y = floor(t X / Q) - e with 0 <= e < k, so |y| < 2 K N t Q (1 + k / m~)^2 + k + 1, and fastbconv_sk recovers y exactly while its alpha,
// which lies in (-|y| / B, na + |y| / B), stays inside the centred range of m_sk: |y| < B ((m_sk - 1) / 2 - na).  K_c is the largest K
// meeting both for the largest t, at least 1 (one product per floor is what op_multiply does) and at most INT32_MAX.
namespace {
typedef std::vector<u64> Big; // little-endian 64-bit limbs
Big big_of(u64 v) { return Big{v}; }
Big big_mul(const Big &a, u64 m) {
    Big r(a.size() + 1, 0);
    unsigned __int128 carry = 0;
    for (size_t i = 0; i < a.size(); i++) {
        const unsigned __int128 v = (unsigned __int128)a[i] * m + carry;
        r[i] = (u64)v;
        carry = v >> 64;
    }
    r[a.size()] = (u64)carry;
    while (r.size() > 1 && r.back() == 0) r.pop_back();
    return r;
}
Big big_sub(Big a, u64 v) { // a >= v
    for (size_t i = 0; i < a.size() && v; i++) {
        const u64 before = a[i];
        a[i] -= v;
        v = a[i] > before ? 1 : 0;
    }
    while (a.size() > 1 && a.back() == 0) a.pop_back();
    return a;
}
int big_cmp(const Big &a, const Big &b) {
    if (a.size() != b.size()) return a.size() < b.size() ? -1 : 1;
    for (size_t i = a.size(); i-- > 0;)
        if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return 0;
}
double big_log2(const Big &a) { return 64.0 * (double)(a.size() - 1) + std::log2((double)a.back()); }
} // namespace
static int product_sum_terms(const std::vector<u64> &q, const std::vector<u64> &bsk, const std::vector<u64> &t, uint32_t N) {
    const int k = (int)q.size(), na = (int)bsk.size() - 1;
    const u64 msk = bsk[na], MT = 1ULL << 32;
    u64 tmax = 0;
    for (u64 v : t) tmax = std::max(tmax, v);
    // limit = (B ((m_sk - 1) / 2 - na) - k - 1) m~^2,   per term = 2 N t Q (m~ + k)^2:   K_c = the largest K with K * per term < limit
    Big limit = big_of((msk - 1) / 2 - (u64)na);
    for (int j = 0; j < na; j++) limit = big_mul(limit, bsk[j]);
    limit = big_mul(big_mul(big_sub(limit, (u64)k + 1), MT), MT);
    Big per = big_of(2ULL * N);
    per = big_mul(big_mul(big_mul(per, tmax), MT + (u64)k), MT + (u64)k);
    for (u64 p : q) per = big_mul(per, p);
    if (big_log2(limit) - big_log2(per) > 32.0) return INT32_MAX;
    u64 lo = 0, hi = 1ULL << 33; // K * per < limit holds at lo and fails at hi
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) / 2;
        if (big_cmp(big_mul(per, mid), limit) < 0) lo = mid;
        else hi = mid;
    }
    return (int)std::max<u64>(1, std::min<u64>(lo, INT32_MAX));
}

Context *context_create(const u64 *plain_primes, int P, uint32_t N, const u64 *coeff, int k, int dbc_relin, int dbc_galois, int device) {
    if (P < 1 || P > 16) throw Error(-1, "need 1..16 plaintext primes");
    int logN = 0;
    while ((1u << logN) < N) logN++;
    if ((1u << logN) != N || logN < 10 || logN > 14) throw Error(-1, "PolyModulusDegree must be a power of two in [1024, 16384]");
    if (k < 1 || k > KMAX) throw Error(-1, "need 1..9 coefficient primes");
    if (dbc_relin < 1 || dbc_relin > 60 || dbc_galois < 1 || dbc_galois > 60) throw Error(-1, "decomposition bit count must be in [1,60]");
    int ndev = 0;
    cudaError_t de = cudaGetDeviceCount(&ndev);
    if (de != cudaSuccess || ndev == 0) throw Error(-2, "libcnhe needs a CUDA device (H100); none is visible -- there is no CPU fallback");
    if (device < 0 || device >= ndev) throw Error(-1, "bad device ordinal");
    std::unique_ptr<Context> cp(new Context());
    Context &c = *cp;
    static std::atomic<uint64_t> serials{0};
    c.serial = c.root = ++serials;
    c.device = device;
    CNHE_CUDA(cudaSetDevice(device));
    c.N = N; c.logN = logN; c.k = k; c.P = P; c.dbc_relin = dbc_relin; c.dbc_galois = dbc_galois;
    c.q.assign(coeff, coeff + k);
    c.t.assign(plain_primes, plain_primes + P);
    for (u64 p : c.q)
        if (!hm::is_prime(p) || (p - 1) % (2ULL * N) || hm::bit_length(p) > 61) throw Error(-1, "coefficient moduli must be primes = 1 mod 2N below 2^61");
    for (u64 p : c.t) {
        if (!hm::is_prime(p) || (p - 1) % (2ULL * N)) throw Error(-1, "plaintext moduli must be primes = 1 mod 2N (batching)");
        for (u64 qq : c.q)
            if (p >= qq) throw Error(-1, "plaintext modulus must be smaller than every coefficient prime");
    }
    // ---- BEHZ base Bsk = auxiliary primes then m_sk.
    // "seal" mode reproduces SEAL 3.2's choice: k auxiliary 61-bit primes (= 1 mod 2^18, descending, after m_sk and gamma)
    // and m_sk = 0x1fffffffffe00001.  The default "fast" mode picks 48-bit primes instead, as many as the exactness bound
    // needs (B*m_sk > 2^8 * N*t*q): every value BEHZ computes is an integer determined by (q, t, m~) alone -- the Bsk residues
    // only carry it -- so the multiply output is bit-identical in both modes (tests/test_gpu_kernels.py checks that), while
    // 48-bit moduli keep every NTT of the multiply on the FP64 butterfly path (DESIGN.md section 4).
    const u64 M_SK_SEAL = 0x1fffffffffe00001ULL, GAMMA = 0x1fffffffffc80001ULL;
    {
        const char *mode = getenv("CNHE_AUX_BASE");
        const bool seal = mode && std::string(mode) == "seal";
        if (seal) {
            u64 cand = (1ULL << 61) + 1;
            int skipped = 0;
            while ((int)c.bsk.size() < k) {
                cand -= 1ULL << 18;
                if (!hm::is_prime(cand)) continue;
                if (skipped < 2) { skipped++; continue; }
                c.bsk.push_back(cand);
            }
            c.bsk.push_back(M_SK_SEAL);
        } else {
            int need = logN + 8;
            u64 tmax = 0;
            for (u64 t : c.t) tmax = std::max(tmax, t);
            need += hm::bit_length(tmax);
            for (u64 p : c.q) need += hm::bit_length(p);
            const int count = (need + 46) / 47; // each 48-bit prime contributes more than 47 bits
            if (count > KBMAX) throw Error(-1, "parameters too large for the auxiliary base");
            u64 cand = (1ULL << 48) + 1;
            while ((int)c.bsk.size() < std::max(count, 2)) {
                cand -= 2ULL * N;
                if (!hm::is_prime(cand)) continue;
                bool clash = false;
                for (u64 p : c.q) clash = clash || p == cand;
                for (u64 p : c.t) clash = clash || p == cand;
                if (!clash) c.bsk.push_back(cand);
            }
            std::reverse(c.bsk.begin(), c.bsk.end()); // m_sk (last) = the largest
        }
    }
    // Decryption divides by q mod gamma and BEHZ by q mod each Bsk prime: a q holding one of them makes that inverse 0 and every result
    // garbage, with no error.  gamma and SEAL's base (61-bit, = 1 mod 2^18) are valid coefficient primes for every N; SEAL caps user
    // primes at 60 bits and never meets this, this library takes 61, so it refuses the collision.  (The fast base avoids q by choice.)
    for (u64 p : c.q) {
        if (p == GAMMA) throw Error(-1, "coefficient moduli must not contain gamma = 0x1fffffffffc80001, the decryption's auxiliary prime");
        for (u64 b : c.bsk)
            if (p == b) {
                char m[112];
                snprintf(m, sizeof(m), "coefficient moduli must not contain a prime of the BEHZ base Bsk (0x%llx)", (unsigned long long)b);
                throw Error(-1, m);
            }
    }
    const int kb = (int)c.bsk.size();
    const u64 M_SK = c.bsk[kb - 1];
    c.kb = kb;
    c.sum_terms = product_sum_terms(c.q, c.bsk, c.t, N);
    c.streams.resize(P);
    for (int i = 0; i < P; i++) CNHE_CUDA(cudaStreamCreateWithFlags(&c.streams[i], cudaStreamNonBlocking));
    c.stream = c.streams[0];
    c.trace_ms = trace_slow_ms();
    CNHE_CUDA(cudaStreamCreateWithFlags(&c.copy_stream, cudaStreamNonBlocking));
    CNHE_CUDA(cudaEventCreateWithFlags(&c.ev_copy, cudaEventDisableTiming));
    CNHE_CUDA(cudaEventCreateWithFlags(&c.ev_join, cudaEventDisableTiming));
    CNHE_CUDA(cudaEventCreate(&c.ev0));
    CNHE_CUDA(cudaEventCreate(&c.ev1));
    {
        cudaMemPool_t pool;
        CNHE_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        uint64_t thr = ~0ULL;
        CNHE_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    }
    // ---- NTT tables: ids 0..k-1 q, k..k+kb-1 Bsk, k+kb+c plain modulus c
    const int n_mod = k + kb + P;
    std::vector<u64> moduli;
    for (u64 p : c.q) moduli.push_back(p);
    for (u64 p : c.bsk) moduli.push_back(p);
    for (u64 p : c.t) moduli.push_back(p);
    // N-word tables per modulus: w, ws, iw, iws, wd, iwd, iwd_hi, wd_split, iwd_split, wd_split_grp, iwd_split_grp
    constexpr size_t TAB_WORDS = 11;
    std::vector<u64> host((size_t)n_mod * TAB_WORDS * N, 0);
    CNHE_CUDA(cudaMalloc((void **)&c.d_table_mem, host.size() * sizeof(u64)));
    c.h_tabs.resize(n_mod);
    for (int m = 0; m < n_mod; m++) {
        const u64 p = moduli[m];
        const u64 psi = hm::minimal_primitive_root(2ULL * N, p), ipsi = hm::inv(psi, p);
        u64 *w = &host[(size_t)m * TAB_WORDS * N], *ws = w + N, *iw = ws + N, *iws = iw + N;
        double *wd = reinterpret_cast<double *>(iws + N), *iwd = wd + N, *iwd_hi = iwd + N, *wd_split = iwd_hi + N, *iwd_split = wd_split + N;
        u64 a = 1, b = 1;
        for (u64 i = 0; i < N; i++) {
            const u64 r = hm::bit_reverse(i, logN);
            w[r] = a; ws[r] = hm::shoup(a, p);
            iw[r] = b; iws[r] = hm::shoup(b, p);
            wd[r] = a > p / 2 ? -(double)(p - a) : (double)a; // centred, exact below 2^53
            iwd[r] = b > p / 2 ? -(double)(p - b) : (double)b;
            a = hm::mul(a, psi, p);
            b = hm::mul(b, ipsi, p);
        }
        if (logN == 12 || logN == 13) { // transposed unit-stride inverse twiddles (see NttTab::iwd_hi)
            const u64 T = N / 16;
            for (u64 j = 0; j < T; j++) {
                for (int i = 0; i < 8; i++) iwd_hi[(u64)i * T + j] = iwd[(N >> 1) + (j << 3) + i];
                for (int i = 0; i < 4; i++) iwd_hi[(u64)(8 + i) * T + j] = iwd[(N >> 2) + (j << 2) + i];
                for (int i = 0; i < 2; i++) iwd_hi[(u64)(12 + i) * T + j] = iwd[(N >> 3) + (j << 1) + i];
                iwd_hi[(u64)14 * T + j] = iwd[(N >> 4) + j];
            }
        }
        if (logN >= 12) { // twiddle tables of the two half-size transforms (see NttTab::wd_split)
            const u64 H = N / 2;
            for (u64 h = 0; h < 2; h++)
                for (u64 i = 1; i < H; i++) {
                    u64 m2 = 1;
                    while (2 * m2 <= i) m2 *= 2; // stage of index i: [m2, 2 m2)
                    wd_split[h * H + i] = wd[i + m2 + h * m2];
                    iwd_split[h * H + i] = iwd[i + m2 + h * m2];
                }
        }
        if ((logN == 12 || logN == 13) && m < k + kb) { // per-thread twiddle groups of the fused kernels (see NttTab::wd_split_grp)
            const u64 H = N / 2, T = H / 16, S0 = logN - 5; // S0: first of the half's last four forward stages
            double *wd_grp = iwd_split + N, *iwd_grp = wd_grp + N;
            for (u64 h = 0; h < 2; h++)
                for (u64 j = 0; j < T; j++) {
                    double f[16] = {}, v[16] = {}; // word 2g + e goes to element e of group g
                    for (u64 u = 0; u < 4; u++) {
                        for (u64 i = 0; i < (1u << u); i++) f[(u ? 1u << u : 0) + i] = wd_split[h * H + (1u << (S0 + u)) + (j << u) + i];
                        for (u64 i = 0; i < (8u >> u); i++) v[16 - (16 >> u) + i] = iwd_split[h * H + (H >> (u + 1)) + (j << (3 - u)) + i];
                    }
                    for (u64 g = 0; g < 8; g++)
                        for (u64 e = 0; e < 2; e++) {
                            wd_grp[h * H + (g * T + j) * 2 + e] = f[2 * g + e];
                            iwd_grp[h * H + (g * T + j) * 2 + e] = v[2 * g + e];
                        }
                }
        }
        NttTab &tb = c.h_tabs[m];
        u64 *base = c.d_table_mem + (size_t)m * TAB_WORDS * N;
        tb.w = base; tb.ws = base + N; tb.iw = base + 2 * (size_t)N; tb.iws = base + 3 * (size_t)N;
        tb.wd = reinterpret_cast<const double *>(base + 4 * (size_t)N);
        tb.iwd = reinterpret_cast<const double *>(base + 5 * (size_t)N);
        tb.iwd_hi = reinterpret_cast<const double *>(base + 6 * (size_t)N);
        tb.wd_split = reinterpret_cast<const double *>(base + 7 * (size_t)N);
        tb.iwd_split = reinterpret_cast<const double *>(base + 8 * (size_t)N);
        tb.wd_split_grp = reinterpret_cast<const double *>(base + 9 * (size_t)N);
        tb.iwd_split_grp = reinterpret_cast<const double *>(base + 10 * (size_t)N);
        tb.inv_n = hm::inv(N % p, p);
        tb.inv_n_s = hm::shoup(tb.inv_n, p);
        tb.mod = make_dmod(p);
        tb.pd = (double)p;
        tb.pinv = 1.0 / (double)p;
        tb.inv_n_d = tb.inv_n > p / 2 ? -(double)(p - tb.inv_n) : (double)tb.inv_n;
        {
            const u64 nw = hm::mul(iw[1], tb.inv_n, p);
            tb.inv_n_w_d = nw > p / 2 ? -(double)(p - nw) : (double)nw;
        }
        fp_schedule(tb, logN, getenv("CNHE_NTT_INT") != nullptr);
    }
    CNHE_CUDA(cudaMemcpy(c.d_table_mem, host.data(), host.size() * sizeof(u64), cudaMemcpyHostToDevice));
    CNHE_CUDA(cudaMalloc((void **)&c.d_tabs, n_mod * sizeof(NttTab)));
    CNHE_CUDA(cudaMemcpy(c.d_tabs, c.h_tabs.data(), n_mod * sizeof(NttTab), cudaMemcpyHostToDevice));
    // ---- BatchEncoder index map (BatchEncoder::populate_matrix_reps_index_map)
    c.h_index_map.resize(N);
    {
        const u64 row = N >> 1, m2 = 2ULL * N;
        u64 pos = 1;
        for (u64 i = 0; i < row; i++) {
            c.h_index_map[i] = (u32)hm::bit_reverse((pos - 1) >> 1, logN);
            c.h_index_map[row | i] = (u32)hm::bit_reverse((m2 - pos - 1) >> 1, logN);
            pos = (pos * 3) & (m2 - 1);
        }
    }
    CNHE_CUDA(cudaMalloc((void **)&c.d_index_map, N * sizeof(u32)));
    CNHE_CUDA(cudaMemcpy(c.d_index_map, c.h_index_map.data(), N * sizeof(u32), cudaMemcpyHostToDevice));
    // ---- BEHZ constants (BaseConverter::generate)
    BehzConst &bc = c.h_bc;
    memset(&bc, 0, sizeof(bc));
    bc.k = k;
    bc.kb = kb;
    bc.centered_mtilde = 0;
    const int na = kb - 1;
    std::vector<u64> B(c.bsk.begin(), c.bsk.begin() + na);
    for (int i = 0; i < k; i++) bc.q[i] = make_dmod(c.q[i]);
    for (int j = 0; j < kb; j++) bc.bsk[j] = make_dmod(c.bsk[j]);
    const u64 MT = 1ULL << 32;
    u64 q_mod_mt = 1;
    for (int i = 0; i < k; i++) q_mod_mt = (q_mod_mt * (c.q[i] & 0xffffffffULL)) & 0xffffffffULL;
    {
        u64 x = q_mod_mt; // Newton iteration for the inverse modulo 2^32 (q is odd)
        for (int it = 0; it < 6; it++) x *= 2 - q_mod_mt * x;
        bc.inv_q_mod_mtilde = x & 0xffffffffULL;
    }
    for (int i = 0; i < k; i++) {
        const u64 qi = c.q[i];
        const u64 inv = hm::inv(hm::product_mod(c.q, i, qi), qi);
        bc.inv_qhat_mod_q[i] = inv;
        bc.mtilde_inv_qhat_mod_q[i] = hm::mul(inv, MT % qi, qi);
        u64 pm = 1;
        for (int l = 0; l < k; l++)
            if (l != i) pm = (pm * (c.q[l] & 0xffffffffULL)) & 0xffffffffULL;
        bc.qhat_mod_mtilde[i] = pm;
        bc.B_mod_q[i] = hm::product_mod(B, -1, qi);
        for (int j = 0; j < na; j++) bc.bhat_mod_q[i][j] = hm::product_mod(B, j, qi);
    }
    for (int j = 0; j < kb; j++) {
        const u64 bj = c.bsk[j];
        for (int i = 0; i < k; i++) bc.qhat_mod_bsk[j][i] = hm::product_mod(c.q, i, bj);
        bc.q_mod_bsk[j] = hm::product_mod(c.q, -1, bj);
        bc.inv_q_mod_bsk[j] = hm::inv(bc.q_mod_bsk[j], bj);
        bc.inv_mtilde_mod_bsk[j] = hm::inv(MT % bj, bj);
    }
    for (int j = 0; j < na; j++) {
        bc.inv_bhat_mod_b[j] = hm::inv(hm::product_mod(B, j, B[j]), B[j]);
        bc.bhat_mod_msk[j] = hm::product_mod(B, j, M_SK);
    }
    bc.inv_B_mod_msk = hm::inv(hm::product_mod(B, -1, M_SK), M_SK);
    CNHE_CUDA(cudaMalloc((void **)&c.d_bc, sizeof(BehzConst)));
    CNHE_CUDA(cudaMemcpy(c.d_bc, &bc, sizeof(BehzConst), cudaMemcpyHostToDevice));
    // FP64 twin of the constants (used on the FP64 element-wise path: fp_elementwise)
    {
        BehzConstF &f = c.h_bf;
        memset(&f, 0, sizeof(f));
        auto cen = [](u64 v, u64 p) { return v > p / 2 ? -(double)(p - v) : (double)v; };
        f.k = k; f.kb = kb; f.centered_mtilde = 0;
        c.fp_elementwise = getenv("CNHE_NTT_INT") == nullptr;
        for (int i = 0; i < k; i++) {
            const u64 p = c.q[i];
            c.fp_elementwise = c.fp_elementwise && hm::bit_length(p) <= 49;
            f.qd[i] = (double)p; f.qinv[i] = 1.0 / (double)p; f.q_u[i] = p;
            f.inv_qhat_mod_q[i] = cen(bc.inv_qhat_mod_q[i], p);
            f.mtilde_inv_qhat_mod_q[i] = cen(bc.mtilde_inv_qhat_mod_q[i], p);
            f.qhat_mod_mtilde[i] = bc.qhat_mod_mtilde[i];
            f.B_mod_q[i] = cen(bc.B_mod_q[i], p);
            for (int j = 0; j < na; j++) f.bhat_mod_q[i][j] = cen(bc.bhat_mod_q[i][j], p);
        }
        f.inv_q_mod_mtilde = bc.inv_q_mod_mtilde;
        for (int j = 0; j < kb; j++) {
            const u64 p = c.bsk[j];
            c.fp_elementwise = c.fp_elementwise && hm::bit_length(p) <= 48;
            f.bd[j] = (double)p; f.binv[j] = 1.0 / (double)p;
            for (int i = 0; i < k; i++) f.qhat_mod_bsk[j][i] = cen(bc.qhat_mod_bsk[j][i], p);
            f.q_mod_bsk[j] = cen(bc.q_mod_bsk[j], p);
            f.inv_q_mod_bsk[j] = cen(bc.inv_q_mod_bsk[j], p);
            f.inv_mtilde_mod_bsk[j] = cen(bc.inv_mtilde_mod_bsk[j], p);
        }
        for (int j = 0; j < na; j++) {
            f.inv_bhat_mod_b[j] = cen(bc.inv_bhat_mod_b[j], c.bsk[j]);
            f.bhat_mod_msk[j] = cen(bc.bhat_mod_msk[j], M_SK);
        }
        f.inv_B_mod_msk = cen(bc.inv_B_mod_msk, M_SK);
        f.msk_half = (double)(M_SK >> 1);
        // lazy-double intermediates between the kernels of a multiply / key switch: FP64 everywhere on the q and Bsk transforms
        for (int i = 0; i < k + kb; i++) c.fp_elementwise = c.fp_elementwise && c.h_tabs[i].fp_ok;
        CNHE_CUDA(cudaMalloc((void **)&c.d_bf, sizeof(BehzConstF)));
        CNHE_CUDA(cudaMemcpy(c.d_bf, &f, sizeof(BehzConstF), cudaMemcpyHostToDevice));
    }
    // ---- per plaintext modulus
    c.ch.resize(P);
    for (int ci = 0; ci < P; ci++) {
        Channel &ch = c.ch[ci];
        const u64 t = c.t[ci];
        ch.t = t;
        rng_from_os(ch.rng); // encryption randomness of a context that only imports a public key is unpredictable too
        ch.mod_id = k + kb + ci;
        PlainConst &pc = ch.pc;
        memset(&pc, 0, sizeof(pc));
        pc.t = t;
        pc.threshold = (t + 1) >> 1;
        pc.gamma = GAMMA;
        pc.tmod = make_dmod(t);
        pc.gmod = make_dmod(GAMMA);
        std::vector<u64> quot;
        u64 rem;
        hm::div_product(c.q, t, quot, rem);
        for (int i = 0; i < k; i++) {
            pc.delta[i] = hm::limbs_mod(quot, c.q[i]);
            pc.q_mod_t[i] = rem % c.q[i];
            pc.tgamma_mod_q[i] = hm::mul(t % c.q[i], GAMMA % c.q[i], c.q[i]);
            pc.qhat_mod_t[i] = hm::product_mod(c.q, i, t);
            pc.qhat_mod_gamma[i] = hm::product_mod(c.q, i, GAMMA);
        }
        { // folded constants of the floor kernel (FloorConstF)
            FloorConstF &ff = ch.floor_f;
            memset(&ff, 0, sizeof(ff));
            auto cen = [](u64 v, u64 p) { return v > p / 2 ? -(double)(p - v) : (double)v; };
            ff.k = k; ff.kb = kb;
            const int na_ = kb - 1;
            for (int i = 0; i < k; i++) {
                const u64 p = c.q[i];
                ff.qd[i] = (double)p; ff.qinv[i] = 1.0 / (double)p;
                ff.xq[i] = cen(hm::mul(t % p, bc.inv_qhat_mod_q[i], p), p);
                ff.B_mod_q[i] = cen(bc.B_mod_q[i], p);
                for (int j = 0; j < na_; j++) ff.bhat_mod_q[i][j] = cen(bc.bhat_mod_q[i][j], p);
            }
            for (int j = 0; j < kb; j++) {
                const u64 p = c.bsk[j];
                ff.bd[j] = (double)p; ff.binv[j] = 1.0 / (double)p;
                u64 post = bc.inv_q_mod_bsk[j];                                   // q^-1 mod p_j ...
                if (j < na_) post = hm::mul(post, bc.inv_bhat_mod_b[j], p);       // ... times B-hat_j^-1 for the base-B primes
                ff.xb[j] = cen(hm::mul(t % p, post, p), p);
                for (int i = 0; i < k; i++) ff.conv[j][i] = cen(hm::mul(bc.qhat_mod_bsk[j][i], post, p), p);
            }
            for (int j = 0; j < na_; j++) ff.bhat_mod_msk[j] = cen(bc.bhat_mod_msk[j], M_SK);
            ff.inv_B_mod_msk = cen(bc.inv_B_mod_msk, M_SK);
            ff.msk_half = (double)(M_SK >> 1);
        }
        pc.neg_inv_q_mod_t = hm::neg(hm::inv(hm::product_mod(c.q, -1, t), t), t);
        pc.neg_inv_q_mod_gamma = hm::neg(hm::inv(hm::product_mod(c.q, -1, GAMMA), GAMMA), GAMMA);
        pc.inv_gamma_mod_t = hm::inv(GAMMA % t, t);
    }
    c.dm_relin = make_digit_map(c.q, dbc_relin);
    c.dm_galois = make_digit_map(c.q, dbc_galois);
    c.galois_elts = standard_galois_elts(N);
    // ---- wrapper CRT data (EncryptedSealBfvEnvironment.PreCompute, "EncryptedSealBfvVector.cs:79-90")
    {
        unsigned __int128 big = 1;
        int bits = 0;
        for (u64 t : c.t) bits += hm::bit_length(t);
        if (bits > 126) throw Error(-1, "product of the plaintext moduli must stay below 2^126");
        for (u64 t : c.t) big *= t;
        c.big_factor = big;
        for (int i = 0; i < P; i++) {
            unsigned __int128 minor = big / c.t[i];
            u64 y = hm::inv((u64)(minor % c.t[i]), c.t[i]);
            c.crt_coeff.push_back(minor * y);
        }
    }
    CNHE_CUDA(cudaMalloc((void **)&c.d_sanitize_nonce, (size_t)P * 8));
    CNHE_CUDA(cudaMemset(c.d_sanitize_nonce, 0, (size_t)P * 8));
    CNHE_CUDA(cudaDeviceSynchronize());
    return cp.release();
}

// ---------------------------------------------------------------- pointer tables
const u64 *const *upload_ptrs(Context &c, const std::vector<const u64 *> &ptrs) {
    u64 *d = c.ws_alloc(ptrs.size());
    c.h2d(d, ptrs.data(), ptrs.size() * sizeof(u64 *));
    return reinterpret_cast<const u64 *const *>(d);
}
u64 *const *upload_ptrs_mut(Context &c, const std::vector<u64 *> &ptrs) {
    u64 *d = c.ws_alloc(ptrs.size());
    c.h2d(d, ptrs.data(), ptrs.size() * sizeof(u64 *));
    return reinterpret_cast<u64 *const *>(d);
}

// ---------------------------------------------------------------- core operations
static int fp_range(const Context &c, int mod_base, int mod_count) {
    for (int i = mod_base; i < mod_base + mod_count; i++)
        if (!c.h_tabs[i].fp_ok) return 0;
    return 1;
}
void op_ntt(Context &c, const u64 *src, u64 *dst, int n_polys, int mod_base, int mod_count, bool inverse) {
    PROF(inverse ? 1 : 0, 16.0 * c.N * n_polys);
    c.check(inverse ? launch_ntt_inverse(src, dst, n_polys, c.logN, c.d_tabs, mod_base, mod_count, fp_range(c, mod_base, mod_count), c.stream)
                    : launch_ntt_forward(src, dst, n_polys, c.logN, c.d_tabs, mod_base, mod_count, fp_range(c, mod_base, mod_count), c.stream),
            "ntt");
}

// Key switches of at least this many ciphertexts run fused (digit transforms and key product in one kernel, ntt.cu): the fused grid has
// 2k CTAs per ciphertext, each walking all D digits, so small calls leave most of the GPU idle where the digit path spreads n*D*k
// transforms over it.  tools/keyswitch_bench.py on one H100 SXM (700 W), N = 8192, k = 5, D = 25: fused / digit path 0.53 / 0.52 ms at
// 32 ciphertexts, 0.87 / 0.99 ms at 64, 11.9 / 14.1 ms at 945.  With the packed relinearisation keys (H100 SXM at 400 W) relinearisation
// crosses over lower, fused / digit path 0.41 / 0.52 ms at 32; Galois calls still read u64 keys and tie at 32, so the threshold stays
constexpr int KS_FUSED_MIN = 64;
// whether a key switch of n ciphertexts takes the fused path: N = 4096 / 8192 on the lazy FP64 path, n >= KS_FUSED_MIN.
// CNHE_KS_FUSED=0 / =1 forces the digit path / the fused path wherever it is built (read per call: tests compare both in one process)
static bool ks_fused_built(const Context &c) {
    if (c.logN != 12 && c.logN != 13) return false;
    if (!c.fp_elementwise) return false;
    for (int i = 0; i < c.k; i++)
        if (!c.h_tabs[i].split_ok) return false;
    return true;
}
static bool ks_fused(const Context &c, int n) {
    if (!ks_fused_built(c)) return false;
    const char *v = getenv("CNHE_KS_FUSED");
    if (v) return atoi(v) != 0;
    return n >= KS_FUSED_MIN;
}
static bool spans_overlap(const u64 *a, size_t a_words, const u64 *b, size_t b_words) { return a < b + b_words && b < a + a_words; }
// out[i] = (base_i + sum_d NTT^-1(NTT(digit_d(target_i)) * key_d)): ciphertext i's target polynomial (k residues) is at
// target + i * target_stride, its base (2 polynomials) at base + i * base_stride; out is packed [n][2][k][N]
const KeySet &Context::keys(int channel, int s) const {
    if (!slot_live(s)) throw Error(-1, "no such key slot");
    return s == 0 ? ch[channel] : clients[s - 1][channel];
}
const u64 *KeyBinding::ref(const u64 *base) {
    auto w = word.find(base);
    if (w == word.end()) {
        const auto k = seen.find(base);
        if (k == seen.end()) throw Error(-1, "internal error: a recorded key switch was given a key that no key slot holds");
        if (words.size() >= cap) throw Error(-1, "internal error: a recording read more keys than its key slots hold");
        w = word.emplace(base, words.size()).first;
        words.push_back(k->second);
    }
    return reinterpret_cast<const u64 *>(table + w->second);
}
// the pointer a kernel is given for key base p: while recording, its key reference (the graph reads the key through its binding)
static const u64 *key_arg(Context &c, const u64 *p) { return c.rec && p ? c.rec->keys->ref(p) : p; }
// ciphertexts c0 .. c0 + m of a per-ciphertext key table, as key_arg passes them, in workspace memory
static const u64 *const *key_table(Context &c, const std::vector<const u64 *> &tab, int c0, int m) {
    std::vector<const u64 *> part(tab.begin() + c0, tab.begin() + c0 + m);
    for (const u64 *&p : part) p = key_arg(c, p);
    return upload_ptrs(c, part);
}
KsKeys KsKeys::slice(int c0, int m) const {
    KsKeys r = *this;
    if (!per_ct()) return r;
    r.keys.assign(keys.begin() + c0, keys.begin() + c0 + m);
    if (!packs.empty()) r.packs.assign(packs.begin() + c0, packs.begin() + c0 + m);
    return r;
}
// collects each ciphertext's key set (per-ciphertext table or the call's slot) into KsKeys; a call of one slot stays uniform
// (kind, elt: which key pick takes, as a recording notes it)
template <class Pick>
static KsKeys pick_keys(Context &c, int ch, int n, const int *slots, int kind, u64 elt, Pick pick) {
    KsKeys r;
    auto take = [&](int s, const u64 *&key, const u64 *&pk) {
        pick(c.keys(ch, s), key, pk);
        if (!c.rec) return;
        c.rec->keys->seen[key] = {s, ch, kind, elt, c.rec->member};
        if (pk) c.rec->keys->seen[pk] = {s, ch, KeyBinding::RLK_PACKED, 0, c.rec->member};
    };
    if (slots) {
        bool uniform = true;
        for (int i = 0; i < n; i++) uniform = uniform && slots[i] == slots[0];
        if (!uniform) {
            bool packed = true;
            for (int i = 0; i < n; i++) {
                const u64 *key, *pk;
                take(slots[i], key, pk);
                r.keys.push_back(key);
                r.packs.push_back(pk);
                packed = packed && pk;
            }
            if (!packed) r.packs.clear();
            return r;
        }
    }
    take(slots && n ? slots[0] : c.slot, r.key, r.packed);
    return r;
}
KsKeys relin_keys(Context &c, int ch, int n, const int *slots) {
    return pick_keys(c, ch, n, slots, KeyBinding::RLK, 0, [](const KeySet &ks, const u64 *&key, const u64 *&pk) {
        if (!ks.have_rlk) throw Error(-3, "relinearization keys are missing");
        key = ks.rlk->p;
        pk = ks.rlk_packed ? ks.rlk_packed->p : nullptr;
    });
}
KsKeys galois_keys(Context &c, int ch, int n, const int *slots, u64 elt) {
    return pick_keys(c, ch, n, slots, KeyBinding::GALOIS, elt, [elt](const KeySet &ks, const u64 *&key, const u64 *&pk) {
        auto it = ks.glk.find(elt);
        if (it == ks.glk.end()) throw Error(-3, "Galois key not present");
        key = it->second->p;
        pk = nullptr;
    });
}
static KsKeys public_keys(Context &c, int ch, int n, const int *slots) {
    return pick_keys(c, ch, n, slots, KeyBinding::PK, 0, [](const KeySet &ks, const u64 *&key, const u64 *&pk) {
        if (!ks.have_pk || !ks.pk) throw Error(-3, "public key is missing");
        key = ks.pk->p;
        pk = nullptr;
    });
}
// whether every ciphertext's key slot holds the Galois key of elt
static bool has_galois(const Context &c, int ch, int n, const int *slots, u64 elt) {
    if (!slots) return c.keys(ch, c.slot).glk.count(elt) != 0;
    for (int i = 0; i < n; i++)
        if (!c.keys(ch, slots[i]).glk.count(elt)) return false;
    return true;
}
void op_key_switch(Context &c, const u64 *target, size_t target_stride, int n, const KsKeys &keys, const DigitMap &dm, const u64 *base,
                   size_t base_stride, u64 *out) {
    const int k = c.k;
    const u64 *key_packed = keys.per_ct() ? (keys.packs.empty() ? nullptr : keys.packs[0]) : keys.packed;
    const size_t N = c.N;
    // the FP64 path passes lazy doubles from the digit transforms to the product and from the product to the inverse transforms
    const int fwd = c.fp_elementwise ? NTT_FP | NTT_OUT_F : 0, inv = c.fp_elementwise ? NTT_FP | NTT_IN_F : 0;
    // the fused kernel writes `out` while other CTAs still read target and base words, so it serves only calls whose output overlaps
    // neither; every internal caller passes scratch, an in-place cnhe_raw_relinearize (out2 inside in3) takes the digit path
    const size_t out_words = (size_t)n * 2 * k * N;
    const bool fused = n > 0 && ks_fused(c, n) && !spans_overlap(out, out_words, target, (n - 1) * target_stride + k * N) &&
                       !spans_overlap(out, out_words, base, (n - 1) * base_stride + 2 * k * N);
    const int wave = c.wave(fused ? 0 : ((size_t)dm.D * k + 2 * k) * N);
    for (int c0 = 0; c0 < n; c0 += wave) {
        WsScope scope(c);
        const int m = std::min(wave, n - c0);
        // a call of several key slots passes one key base per ciphertext (the packed copies when every slot has one)
        const u64 *const *key_tab = nullptr;
        if (keys.per_ct()) key_tab = key_table(c, fused && key_packed ? keys.packs : keys.keys, c0, m);
        if (fused) {
            // HBM: the target residues once (the pair and the other residues' CTAs share them through L2), the keys once, the output.  The
            // base words the epilogue adds (another 8N bytes per output polynomial, mostly prefetched) are not booked: the figure keeps the
            // meaning it had when the kernel wrote an accumulator of the output's size
            PROF(3, 8.0 * N * ((double)m * k + (double)m * 2 * k) + (key_packed ? 6.0 : 8.0) * N * dm.D * 2 * k);
            c.check(launch_key_switch_fused(target + (size_t)c0 * target_stride, target_stride, key_arg(c, keys.key),
                                            reinterpret_cast<const uint4 *>(key_arg(c, key_packed)), key_tab, base + (size_t)c0 * base_stride, base_stride,
                                            out + (size_t)c0 * 2 * k * N, m, k, dm, c.logN, c.d_tabs, c.stream, c.rec != nullptr),
                    "key_switch_fused");
            continue;
        }
        u64 *acc = c.ws_alloc((size_t)m * 2 * k * N);
        {
            u64 *digits = c.ws_alloc((size_t)m * dm.D * k * N);
            {
                PROF(0, 16.0 * N * (double)m * dm.D * k); // SURVEY 8d: 16N bytes per transform (8N digit source read + 8N written)
                c.check(launch_ntt_forward_digits(target + (size_t)c0 * target_stride, target_stride, digits, m, k, dm, c.logN, c.d_tabs,
                                                  fwd, c.stream),
                        "ntt_forward_digits");
            }
            PROF(3, 8.0 * N * ((double)m * dm.D * k + (double)dm.D * 2 * k + (double)m * 2 * k));
            const u64 *key = key_arg(c, keys.key);
            if (c.fp_elementwise) c.check(launch_ks_mac_fp(digits, key, key_tab, acc, m, dm.D, k, c.logN, &c.h_bf, c.stream, c.rec != nullptr), "ks_mac_fp");
            else c.check(launch_ks_mac(digits, key, key_tab, acc, m, dm.D, k, c.logN, c.d_bc, c.stream, c.rec != nullptr), "ks_mac");
        }
        PROF(1, 24.0 * N * m * 2 * k);
        c.check(launch_ntt_inverse_add(acc, base + (size_t)c0 * base_stride, 2 * k, base_stride, out + (size_t)c0 * 2 * k * N, m * 2 * k, c.logN,
                                       c.d_tabs, 0, k, inv, c.stream),
                "ntt_inverse_add");
    }
}

// whether a product takes the fused square (forward transforms, tensor square and inverse transforms in one kernel, ntt.cu): every
// pair is a square (a[i] == b[i]), N = 4096 / 8192 on the lazy FP64 path, the split schedule exact on every modulus of q u Bsk.
// CNHE_MUL_FUSED=0 / =1 forces the separate kernels / the fused square wherever it applies (read per call: tests compare both in one process)
static bool mul_fused(const Context &c, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b) {
    if (c.logN != 12 && c.logN != 13) return false;
    const int kt = c.k + c.kb;
    if (!c.fp_elementwise) return false;
    for (int i = 0; i < kt; i++)
        if (!c.h_tabs[i].split_ok) return false;
    for (size_t i = 0; i < a.size(); i++)
        if (a[i] != b[i]) return false;
    const char *v = getenv("CNHE_MUL_FUSED");
    return v ? atoi(v) != 0 : true;
}
// scratch words per ciphertext of multiply_chunk
static size_t mul_words(const Context &c, bool fused) { return (size_t)(fused ? 2 * c.kb + 3 * (c.k + c.kb) : 7 * (c.k + c.kb)) * c.N; }
FloorEpi floor_epi(const Context &c, int ch, u64 A, u64 B, u64 C) {
    FloorEpi e;
    memset(&e, 0, sizeof(e));
    const PlainConst &pc = c.ch[ch].pc;
    auto cen = [](u64 v, u64 p) { return v > p / 2 ? -(double)(p - v) : (double)v; };
    for (int i = 0; i < c.k; i++) {
        const u64 q = c.q[i];
        auto lift = [&](u64 v) { return v >= pc.threshold ? v + (q - pc.t) : v; }; // multiply_plain's upper-half increment
        e.a[i] = lift(A);
        e.b[i] = lift(B);
        e.c[i] = hm::add(hm::mul(pc.delta[i], C, q), C >= pc.threshold ? pc.q_mod_t[i] : 0, q); // add_plain: Delta C (+ q mod t)
        e.a_d[i] = cen(e.a[i], q);
        e.b_d[i] = cen(e.b[i], q);
        e.c_d[i] = cen(e.c[i], q);
    }
    return e;
}
// epi: the call's FloorEpi, its x table (when the caller gave none: the squared operands, x_ptrs) and its c_poly table (one entry per
// output of the call) still to be pointed at the wave, whose first output is o0.  m products; pair: they make m / 2 outputs (2i, 2i + 1)
static void multiply_floor(Context &c, int ch, const u64 *D, int m, u64 *out3, const FloorEpi *epi = nullptr,
                           const u64 *const *x_ptrs = nullptr, int o0 = 0, bool pair = false) {
    FloorEpi e;
    if (epi) {
        e = *epi;
        e.x = epi->x ? epi->x + o0 : x_ptrs;
        e.c_poly = epi->c_poly ? epi->c_poly + o0 : nullptr;
    }
    const FloorEpi *ep = epi ? &e : nullptr;
    const int n_out = pair ? m / 2 : m;
    // the epilogue's read of the input's c0 and c1 (8N bytes per residue and polynomial) is booked with the family; the pair floor also
    // parks the second product's floor in the output and reads it back
    PROF(2, 8.0 * c.N * m * 3 * (c.k + c.kb) + 8.0 * c.N * n_out * 3 * c.k + (epi ? 8.0 * c.N * n_out * 2 * c.k : 0.0) +
                (pair ? 16.0 * c.N * n_out * 3 * c.k : 0.0));
    if (c.fp_elementwise) c.check(launch_behz_floor_fold_fp(D, out3, n_out, c.logN, &c.ch[ch].floor_f, c.stream, ep, pair), "behz_floor_fold_fp");
    else c.check(launch_behz_floor(D, out3, n_out, c.ch[ch].t, c.logN, c.d_bc, c.stream, ep, pair), "behz_floor");
}
// products c0 .. c0 + m - 1 of a x b; with an epilogue, o0 is the wave's first output (c0, or c0 / 2 for pairs)
static void multiply_chunk(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, int c0, int m, u64 *out3,
                           bool fused, const FloorEpi *epi = nullptr, bool pair = false) {
    const int o0 = pair ? c0 / 2 : c0;
    const int k = c.k, kt = k + c.kb;
    const size_t N = c.N;
    if (fused) {
        const u64 *const *ptrs = upload_ptrs(c, std::vector<const u64 *>(a.begin() + c0, a.begin() + c0 + m));
        u64 *L = c.ws_alloc((size_t)m * 2 * c.kb * N), *D = c.ws_alloc((size_t)m * 3 * kt * N);
        {
            PROF(2, 8.0 * N * m * 2 * (k + c.kb));
            c.check(launch_behz_lift_bsk_fp(ptrs, L, m, c.logN, &c.h_bf, c.stream), "behz_lift_bsk_fp");
        }
        {
            // HBM: both polynomials of every residue read once (the partner's reads are L2 hits), the three products written once
            PROF(0, 8.0 * N * m * (2 * kt + 3 * kt));
            c.check(launch_behz_square_fused(ptrs, L, D, m, k, kt, c.logN, c.d_tabs, c.stream), "behz_square_fused");
        }
        multiply_floor(c, ch, D, m, out3, epi, ptrs, o0, pair);
        return;
    }
    bool square = true;
    for (int i = 0; i < m; i++) square = square && a[c0 + i] == b[c0 + i];
    if (epi && !square) throw Error(-1, "the activation epilogue applies to squares only");
    std::vector<const u64 *> pa(a.begin() + c0, a.begin() + c0 + m);
    u64 *A = c.ws_alloc((size_t)m * 2 * kt * N);
    const int fmt = c.fp_elementwise ? NTT_FP | NTT_IN_F | NTT_OUT_F : 0;
    const u64 *const *pa_dev = upload_ptrs(c, pa);
    {
        PROF(2, 8.0 * N * m * 2 * (k + kt));
        if (c.fp_elementwise) c.check(launch_behz_lift_fp(pa_dev, A, m, c.logN, &c.h_bf, c.stream), "behz_lift_fp");
        else c.check(launch_behz_lift(pa_dev, A, m, c.logN, c.d_bc, c.stream), "behz_lift");
    }
    {
        PROF(0, 16.0 * N * m * 2 * kt);
        c.check(launch_ntt_forward(A, A, m * 2 * kt, c.logN, c.d_tabs, 0, kt, fmt, c.stream), "ntt_forward");
    }
    u64 *B = A;
    if (!square) {
        std::vector<const u64 *> pb(b.begin() + c0, b.begin() + c0 + m);
        B = c.ws_alloc((size_t)m * 2 * kt * N);
        if (c.fp_elementwise) c.check(launch_behz_lift_fp(upload_ptrs(c, pb), B, m, c.logN, &c.h_bf, c.stream), "behz_lift_fp");
        else c.check(launch_behz_lift(upload_ptrs(c, pb), B, m, c.logN, c.d_bc, c.stream), "behz_lift");
        c.check(launch_ntt_forward(B, B, m * 2 * kt, c.logN, c.d_tabs, 0, kt, fmt, c.stream), "ntt_forward");
    }
    u64 *D = c.ws_alloc((size_t)m * 3 * kt * N);
    {
        PROF(2, 8.0 * N * m * kt * (square ? 5 : 7));
        if (c.fp_elementwise) c.check(launch_behz_tensor_fp(A, B, D, m, kt, c.logN, &c.h_bf, c.stream), "behz_tensor_fp");
        else c.check(launch_behz_tensor(A, B, D, m, kt, c.logN, c.d_bc, c.stream), "behz_tensor");
    }
    {
        PROF(1, 16.0 * N * m * 3 * kt);
        c.check(launch_ntt_inverse(D, D, m * 3 * kt, c.logN, c.d_tabs, 0, kt, fmt, c.stream), "ntt_inverse");
    }
    multiply_floor(c, ch, D, m, out3, epi, pa_dev, o0, pair);
}
void op_multiply(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, u64 *out3, const FloorEpi *epi) {
    const int n = (int)a.size();
    const bool fused = mul_fused(c, a, b);
    const int wave = c.wave(mul_words(c, fused));
    for (int c0 = 0; c0 < n; c0 += wave) {
        WsScope scope(c);
        const int m = std::min(wave, n - c0);
        multiply_chunk(c, ch, a, b, c0, m, out3 + (size_t)c0 * 3 * c.k * c.N, fused, epi);
    }
    c.note(Context::OP_MULTIPLY, ch, n);
}
int multiply_sum_wave(const Context &c, int T) {
    const size_t N = c.N, kt = (size_t)c.k + c.kb, lifted = 2 * kt * N;
    // resident for the chunk: its T shared operands; per output: T lifted columns, the summed product and its floor
    const size_t fixed = (size_t)T * lifted, per = (size_t)T * lifted + 3 * kt * N + 3 * (size_t)c.k * N, cap = (size_t)1 << 30; // 8 GiB
    if (fixed + per > cap) return 0;
    return (int)std::min<size_t>((cap - fixed) / per, (size_t)INT32_MAX);
}
void op_multiply_sum(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, int T, int n_out, u64 *out2,
                     const int *slots) {
    if (T < 1 || n_out < 1 || a.size() != (size_t)n_out * T || b.size() != (size_t)T) throw Error(-1, "bad product-sum shape");
    const int Tc = std::min(T, c.sum_terms);
    const int wave = multiply_sum_wave(c, Tc);
    if (wave < 1) throw Error(-1, "a chunk of the product sum needs more than 8 GiB of scratch next to one output");
    (void)relin_keys(c, ch, n_out, slots); // a missing key fails before any launch
    const int k = c.k, kt = k + c.kb;
    const size_t N = c.N, lifted = (size_t)2 * kt * N, s3 = (size_t)3 * k * N;
    const int fmt = c.fp_elementwise ? NTT_FP | NTT_IN_F | NTT_OUT_F : 0;
    // BEHZ lift and forward transforms of n ciphertexts into [n][2][kt][N] (as multiply_chunk lifts its operands)
    auto lift = [&](const std::vector<const u64 *> &cts, u64 *dst) {
        const int n = (int)cts.size();
        const u64 *const *dev = upload_ptrs(c, cts);
        {
            PROF(2, 8.0 * N * n * 2 * (k + kt));
            if (c.fp_elementwise) c.check(launch_behz_lift_fp(dev, dst, n, c.logN, &c.h_bf, c.stream), "behz_lift_fp");
            else c.check(launch_behz_lift(dev, dst, n, c.logN, c.d_bc, c.stream), "behz_lift");
        }
        PROF(0, 16.0 * N * n * 2 * kt);
        c.check(launch_ntt_forward(dst, dst, n * 2 * kt, c.logN, c.d_tabs, 0, kt, fmt, c.stream), "ntt_forward");
    };
    WsScope scope(c);
    u64 *Y = c.ws_alloc((size_t)n_out * s3); // the floors of the chunks, summed
    for (int j0 = 0; j0 < T; j0 += Tc) {
        WsScope chunk(c);
        const int nt = std::min(Tc, T - j0);
        u64 *S = c.ws_alloc((size_t)nt * lifted);
        lift(std::vector<const u64 *>(b.begin() + j0, b.begin() + j0 + nt), S);
        for (int o0 = 0; o0 < n_out; o0 += wave) {
            WsScope w(c);
            const int m = std::min(wave, n_out - o0);
            std::vector<const u64 *> pa;
            for (int o = o0; o < o0 + m; o++) pa.insert(pa.end(), a.begin() + (size_t)o * T + j0, a.begin() + (size_t)o * T + j0 + nt);
            u64 *A = c.ws_alloc((size_t)m * nt * lifted), *D = c.ws_alloc((size_t)m * 3 * kt * N);
            lift(pa, A);
            {
                // HBM: every column word once, the shared words once (the outputs' CTAs of one tile read them out of L2), the sums written once
                PROF(2, 8.0 * N * ((double)m * nt * 2 * kt + (double)nt * 2 * kt + (double)m * 3 * kt));
                if (c.fp_elementwise) c.check(launch_behz_tensor_mac_fp(A, S, D, m, nt, kt, c.logN, &c.h_bf, c.stream), "behz_tensor_mac_fp");
                else c.check(launch_behz_tensor_mac(A, S, D, m, nt, kt, c.logN, c.d_bc, c.stream), "behz_tensor_mac");
            }
            {
                PROF(1, 16.0 * N * m * 3 * kt);
                c.check(launch_ntt_inverse(D, D, m * 3 * kt, c.logN, c.d_tabs, 0, kt, fmt, c.stream), "ntt_inverse");
            }
            u64 *dst = Y + (size_t)o0 * s3;
            if (j0 == 0) {
                multiply_floor(c, ch, D, m, dst);
            } else { // the chunk's floor added mod q to the earlier chunks' (the add kernel over the three polynomials)
                u64 *F = c.ws_alloc((size_t)m * s3);
                multiply_floor(c, ch, D, m, F);
                c.check(launch_ct_add(dst, F, dst, (size_t)m * s3, k, c.logN, c.d_bc, 0, c.stream), "ct_add");
            }
        }
    }
    c.op_count[Context::OP_MULTIPLY] += (uint64_t)n_out * T;
    c.op_count[Context::OP_ADD] += (uint64_t)n_out * (T - 1);
    op_relinearize(c, ch, Y, n_out, out2, slots);
}
void op_relinearize(Context &c, int ch, const u64 *in3, int n, u64 *out2, const int *slots, bool book) {
    const KsKeys keys = relin_keys(c, ch, n, slots);
    const int k = c.k;
    const size_t N = c.N;
    // the size-3 layout [c0 c1 c2] is consumed in place: c2 is the key-switch target, (c0, c1) the base it is added to
    const size_t s3 = (size_t)3 * k * N;
    op_key_switch(c, in3 + (size_t)2 * k * N, s3, n, keys, c.dm_relin, in3, s3, out2);
    if (book) c.note(Context::OP_RELINEARIZE, ch, n, out2);
}
bool relin_planes_built(const Context &c) { return ks_fused_built(c); }
void op_relinearize_planes(Context &c, int ch, const int *planes, int n, const u64 *base, u64 *out2, const int *slots) {
    if (!ks_fused_built(c)) throw Error(-1, "the plane-source key switch needs the fused key switch (N = 4096 / 8192, lazy FP64 path)");
    const KsKeys keys = relin_keys(c, ch, n, slots);
    const int k = c.k;
    const size_t N = c.N;
    const DigitMap &dm = c.dm_relin;
    const u64 *key_packed = keys.per_ct() ? (keys.packs.empty() ? nullptr : keys.packs[0]) : keys.packed;
    WsScope scope(c);
    const u64 *const *key_tab = nullptr;
    if (keys.per_ct()) key_tab = key_table(c, key_packed ? keys.packs : keys.keys, 0, n);
    // HBM: the digit planes once (every residue's CTAs of a ciphertext share them through L2), the keys once, the output
    PROF(3, 4.0 * N * n * dm.D + 8.0 * N * n * 2 * k + (key_packed ? 6.0 : 8.0) * N * dm.D * 2 * k);
    c.check(launch_key_switch_planes(planes, key_arg(c, keys.key), reinterpret_cast<const uint4 *>(key_arg(c, key_packed)), key_tab, base,
                                     (size_t)2 * k * N, out2, n, k, dm, c.logN, c.d_tabs, c.stream, c.rec != nullptr),
            "key_switch_planes");
}
void op_multiply_relin(Context &c, int ch, const std::vector<const u64 *> &a, const std::vector<const u64 *> &b, u64 *out2, const int *slots,
                       const FloorEpi *epi, bool pair) {
    if (pair && (!epi || !epi->x || a.size() % 2)) throw Error(-1, "the pair floor needs an epilogue with its own x table and whole pairs");
    const int per = pair ? 2 : 1, n = (int)a.size() / per, k = c.k;
    const KsKeys keys = relin_keys(c, ch, n, slots);
    const size_t N = c.N;
    const bool fused = mul_fused(c, a, b);
    const int wave = c.wave((ks_fused(c, n) ? 0 : (size_t)c.dm_relin.D * k * N) + per * mul_words(c, fused) + 5 * k * N);
    for (int c0 = 0; c0 < n; c0 += wave) {
        WsScope scope(c); // stream-ordered frees: the next wave reuses the memory once these kernels are done
        const int m = std::min(wave, n - c0);
        u64 *ct3 = c.ws_alloc((size_t)m * 3 * k * N);
        multiply_chunk(c, ch, a, b, c0 * per, m * per, ct3, fused, epi, pair);
        const size_t s3 = (size_t)3 * k * N;
        op_key_switch(c, ct3 + (size_t)2 * k * N, s3, m, keys.slice(c0, m), c.dm_relin, ct3, s3, out2 + (size_t)c0 * 2 * k * N);
    }
    c.op_count[Context::OP_MULTIPLY] += (uint64_t)a.size();
    c.note(Context::OP_RELINEARIZE, ch, n, out2, a[0], b[0]);
}

u64 galois_elt_from_step(const Context &c, int steps) { // Evaluator::galois_elt_from_step: positive = rotate left
    const u64 n = c.N, m = 2 * n;
    if (steps == 0) return m - 1;
    const bool neg = steps < 0;
    const u64 pos = neg ? (u64)(-(long long)steps) : (u64)steps;
    if (pos >= (n >> 1)) throw Error(-1, "step count too large");
    const u64 s = neg ? (n >> 1) - pos : pos;
    u64 e = 1;
    for (u64 i = 0; i < s; i++) e = (e * 3) & (m - 1);
    return e;
}
static u64 galois_inverse(uint32_t N, u64 elt) { // elt^-1 mod 2N
    const u64 m2 = 2ULL * N;
    for (u64 x = 1; x < m2; x += 2)
        if (((x * elt) & (m2 - 1)) == 1) return x;
    return 0;
}
void op_apply_galois(Context &c, int ch, const u64 *in, int n, u64 elt, u64 *out, bool add_back, const int *slots) {
    const KsKeys keys = galois_keys(c, ch, n, slots, elt);
    const int k = c.k;
    const size_t N = c.N;
    const u64 m2 = 2ULL * N, einv = galois_inverse(c.N, elt);
    for (int c0 = 0; c0 < n; c0 += c.chunk) {
        const int m = std::min(c.chunk, n - c0);
        u64 *base = c.ws_alloc((size_t)m * 2 * k * N), *p1 = c.ws_alloc((size_t)m * k * N);
        c.check(launch_galois(in + (size_t)c0 * 2 * k * N, base, p1, m, einv, k, c.logN, c.d_bc, c.stream, add_back ? 1 : 0), "galois");
        op_key_switch(c, p1, (size_t)k * N, m, keys.slice(c0, m), c.dm_galois, base, (size_t)2 * k * N, out + (size_t)c0 * 2 * k * N);
    }
    c.note(elt == m2 - 1 ? Context::OP_ROTATE_COLUMNS : Context::OP_ROTATE_ROWS_HOP, ch, n, out, in);
    if (add_back) c.note(Context::OP_ADD, ch, n, out, in, out); // the reference issues Rotate + Add: both are counted
}
// x + rotate(x) in one pass (in == out allowed): the permutation kernel folds the unrotated ciphertext into the key switch's base.  Returns
// false when the step has no key of its own (multi-hop rotation) or per-operation noise tracing wants the rotated ciphertext on its own.
bool op_rotate_add(Context &c, int ch, const u64 *in, int n, int steps, bool columns, u64 *out, const int *slots) {
    if (c.trace_noise) return false;
    const u64 elt = columns ? 2ULL * c.N - 1 : galois_elt_from_step(c, steps);
    if (!has_galois(c, ch, n, slots, elt)) return false;
    op_apply_galois(c, ch, in, n, elt, out, true, slots);
    return true;
}
std::vector<int> naf_hops(uint32_t N, int steps) {
    std::vector<int> res;
    const bool sign = steps < 0;
    int v = sign ? -steps : steps;
    for (int i = 0; v; i++) { // non-adjacent form, least significant term first (SEAL util::naf)
        const int zi = (v & 1) ? 2 - (v & 3) : 0;
        v = (v - zi) >> 1;
        if (zi && (1u << i) != N / 2) res.push_back((sign ? -zi : zi) * (1 << i));
    }
    return res;
}
// the row rotations a rotation by `steps` (!= 0) is made of: the step itself when every ciphertext's key slot holds its key, else its hops
static std::vector<int> row_hops(const Context &c, int ch, int n, const int *slots, int steps) {
    if (has_galois(c, ch, n, slots, galois_elt_from_step(c, steps))) return {steps};
    return naf_hops(c.N, steps);
}
void op_rotate_rows(Context &c, int ch, const u64 *in, int n, int steps, u64 *out, const int *slots) { // Evaluator::rotate_internal
    const size_t words = (size_t)n * c.ct_words();
    if (steps == 0) {
        if (in != out) { CNHE_CUDA(cudaMemcpyAsync(out, in, words * 8, cudaMemcpyDeviceToDevice, c.stream)); c.note_copy(out, in); }
        return;
    }
    // each hop takes its own Galois key: a missing one is CNHE_ERR_STATE
    const std::vector<int> hops = row_hops(c, ch, n, slots, steps);
    const u64 *cur = in;
    for (size_t h = 0; h < hops.size(); h++) {
        u64 *nxt = h + 1 == hops.size() ? out : c.ws_alloc(words);
        op_apply_galois(c, ch, cur, n, galois_elt_from_step(c, hops[h]), nxt, false, slots);
        cur = nxt;
    }
}
void op_rotate_columns(Context &c, int ch, const u64 *in, int n, u64 *out, const int *slots) {
    op_apply_galois(c, ch, in, n, 2ULL * c.N - 1, out, false, slots);
}

// apply_galois on n ciphertexts scattered in memory (pointer table) -> packed out[n]
static void apply_galois_gather(Context &c, int ch, const std::vector<const u64 *> &ins, u64 elt, u64 *out, const int *slots) {
    const int k = c.k, n = (int)ins.size();
    const KsKeys keys = galois_keys(c, ch, n, slots, elt);
    const size_t N = c.N;
    const u64 m2 = 2ULL * N, einv = galois_inverse(c.N, elt);
    for (int c0 = 0; c0 < n; c0 += c.chunk) {
        const int m = std::min(c.chunk, n - c0);
        std::vector<const u64 *> part(ins.begin() + c0, ins.begin() + c0 + m);
        u64 *base = c.ws_alloc((size_t)m * 2 * k * N), *p1 = c.ws_alloc((size_t)m * k * N);
        c.check(launch_galois_gather(upload_ptrs(c, part), base, p1, m, einv, k, c.logN, c.d_bc, c.stream), "galois");
        op_key_switch(c, p1, (size_t)k * N, m, keys.slice(c0, m), c.dm_galois, base, (size_t)2 * k * N, out + (size_t)c0 * 2 * k * N);
    }
    c.op_count[elt == m2 - 1 ? Context::OP_ROTATE_COLUMNS : Context::OP_ROTATE_ROWS_HOP] += (uint64_t)n;
    if (c.trace_noise) // one record per ciphertext, as the unbatched path would have written
        for (int i = 0; i < n; i++) {
            c.op_count[Context::OP_ROTATE_ROWS_HOP] -= 1; // note() counts it again
            c.note(Context::OP_ROTATE_ROWS_HOP, ch, 1, out + (size_t)i * 2 * k * N, ins[i]);
        }
}
void op_rotate_rows_multi(Context &c, int ch, const std::vector<RotateJob> &jobs) {
    const size_t ctw = c.ct_words();
    struct State { std::vector<int> hops; size_t next; const u64 *cur; };
    std::vector<State> st(jobs.size());
    std::vector<int> slots(jobs.size());
    for (size_t j = 0; j < jobs.size(); j++) slots[j] = jobs[j].slot < 0 ? c.slot : jobs[j].slot;
    for (size_t j = 0; j < jobs.size(); j++) {
        st[j].next = 0;
        st[j].cur = jobs[j].src;
        if (jobs[j].steps) st[j].hops = row_hops(c, ch, (int)slots.size(), slots.data(), jobs[j].steps);
    }
    for (;;) {
        // the hop value most jobs are waiting for next
        std::map<int, std::vector<size_t>> want;
        for (size_t j = 0; j < jobs.size(); j++)
            if (st[j].next < st[j].hops.size()) want[st[j].hops[st[j].next]].push_back(j);
        if (want.empty()) break;
        auto best = want.begin();
        for (auto it = want.begin(); it != want.end(); ++it)
            if (it->second.size() > best->second.size()) best = it;
        const std::vector<size_t> &js = best->second;
        std::vector<const u64 *> ins;
        std::vector<int> in_slots;
        for (size_t j : js) { ins.push_back(st[j].cur); in_slots.push_back(slots[j]); }
        u64 *out = c.ws_alloc(js.size() * ctw);
        apply_galois_gather(c, ch, ins, galois_elt_from_step(c, best->first), out, in_slots.data());
        for (size_t i = 0; i < js.size(); i++) {
            st[js[i]].cur = out + i * ctw;
            st[js[i]].next++;
        }
    }
    for (size_t j = 0; j < jobs.size(); j++)
        if (st[j].cur != jobs[j].dst) {
            CNHE_CUDA(cudaMemcpyAsync(jobs[j].dst, st[j].cur, ctw * 8, cudaMemcpyDeviceToDevice, c.stream));
            c.note_copy(jobs[j].dst, st[j].cur);
        }
}

void op_multiply_plain_dense(Context &c, int ch, const u64 *ct, int n, const u64 *plain, bool plain_per_ct, u64 *out) {
    const int k = c.k;
    const size_t N = c.N;
    const int np = plain_per_ct ? n : 1;
    u64 *lifted = c.ws_alloc((size_t)np * k * N);
    c.check(launch_plain_lift(plain, lifted, np, (int)N, k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "plain_lift");
    c.check(launch_ntt_forward(lifted, lifted, np * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
    u64 *tmp = c.ws_alloc((size_t)n * 2 * k * N);
    c.check(launch_ntt_forward(ct, tmp, n * 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
    c.check(launch_dyadic_bcast(tmp, lifted, tmp, n, 2, 1, plain_per_ct ? 1 : 0, k, c.logN, c.d_bc, c.stream), "dyadic");
    c.check(launch_ntt_inverse(tmp, out, n * 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
    c.note(Context::OP_MULTIPLY_PLAIN, ch, n, out, ct);
}
// one ciphertext times n dense plaintexts: out[i] = ct * plain[i]   (row-major matrix x vector: every row against the same input)
void op_multiply_plain_dense_bcast(Context &c, int ch, const u64 *ct, const u64 *plains, int n, u64 *out) {
    const int k = c.k;
    const size_t N = c.N;
    u64 *ctn = c.ws_alloc((size_t)2 * k * N);
    c.check(launch_ntt_forward(ct, ctn, 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
    for (int c0 = 0; c0 < n; c0 += 4 * c.chunk) {
        WsScope scope(c);
        const int m = std::min(4 * c.chunk, n - c0);
        u64 *lifted = c.ws_alloc((size_t)m * k * N);
        c.check(launch_plain_lift(plains + (size_t)c0 * N, lifted, m, (int)N, k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "plain_lift");
        c.check(launch_ntt_forward(lifted, lifted, m * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        u64 *dst = out + (size_t)c0 * 2 * k * N;
        c.check(launch_dyadic_bcast(ctn, lifted, dst, m, 2, 0, 1, k, c.logN, c.d_bc, c.stream), "dyadic");
        c.check(launch_ntt_inverse(dst, dst, m * 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
    }
    c.note(Context::OP_MULTIPLY_PLAIN, ch, n, out, ct);
}
// B ciphertexts times the same R dense plaintexts: out[b * R + r] = cts[b] * plains[r], each product the words
// op_multiply_plain_dense_bcast(cts[b], plains) gives.  Every ciphertext is transformed once and every plaintext once per wave of rows
// (R k (B - 1) forward transforms fewer than B broadcast calls); the FP64 path multiplies them in k_dyadic_outer, the integer path
// (CNHE_NTT_INT, a q_l >= 2^50) runs the broadcast kernel per ciphertext on the shared transforms.  One ciphertext is the broadcast call.
void op_multiply_plain_dense_outer(Context &c, int ch, const std::vector<const u64 *> &cts, const u64 *plains, int R, u64 *out) {
    const int k = c.k, B = (int)cts.size(), fpq = fp_range(c, 0, k);
    const size_t N = c.N, kN = (size_t)k * N, ctw = 2 * kN;
    if (B < 1 || R < 1) return;
    if (B == 1) return op_multiply_plain_dense_bcast(c, ch, cts[0], plains, R, out);
    WsScope scope(c);
    u64 *ctn = c.ws_alloc((size_t)B * ctw);
    bool packed = true;
    for (int b = 1; b < B && packed; b++) packed = cts[b] == cts[0] + (size_t)b * ctw;
    if (packed) c.check(launch_ntt_forward(cts[0], ctn, B * 2 * k, c.logN, c.d_tabs, 0, k, fpq, c.stream), "ntt_forward");
    else
        for (int b = 0; b < B; b++)
            c.check(launch_ntt_forward(cts[b], ctn + (size_t)b * ctw, 2 * k, c.logN, c.d_tabs, 0, k, fpq, c.stream), "ntt_forward");
    // rows per wave: their lifted transforms stay under 8 GiB
    const int RW = (int)std::max<size_t>(1, std::min<size_t>((size_t)R, ((size_t)1 << 30) / kN));
    for (int r0 = 0; r0 < R; r0 += RW) {
        WsScope wave(c);
        const int m = std::min(RW, R - r0);
        u64 *lifted = c.ws_alloc((size_t)m * kN);
        c.check(launch_plain_lift(plains + (size_t)r0 * N, lifted, m, (int)N, k, c.logN, c.d_bc, c.ch[ch].pc, c.stream), "plain_lift");
        c.check(launch_ntt_forward(lifted, lifted, m * k, c.logN, c.d_tabs, 0, k, fpq, c.stream), "ntt_forward");
        if (c.fp_elementwise) c.check(launch_dyadic_outer(ctn, lifted, out + (size_t)r0 * ctw, B, m, R, k, c.logN, &c.h_bf, c.stream), "dyadic_outer");
        else
            for (int b = 0; b < B; b++)
                c.check(launch_dyadic_bcast(ctn + (size_t)b * ctw, lifted, out + ((size_t)b * R + r0) * ctw, m, 2, 0, 1, k, c.logN, c.d_bc, c.stream),
                        "dyadic");
    }
    c.check(launch_ntt_inverse(out, out, B * R * 2 * k, c.logN, c.d_tabs, 0, k, fpq, c.stream), "ntt_inverse");
    for (int b = 0; b < B; b++) c.note(Context::OP_MULTIPLY_PLAIN, ch, R, out + (size_t)b * R * ctw, cts[b]);
}
void op_encode(Context &c, int ch, const u64 *values, int n, int count, u64 *plain) {
    c.check(launch_encode_scatter(values, plain, n, count, c.d_index_map, c.logN, c.stream), "encode_scatter");
    c.check(launch_ntt_inverse(plain, plain, n, c.logN, c.d_tabs, c.ch[ch].mod_id, 1, fp_range(c, c.ch[ch].mod_id, 1), c.stream), "ntt_inverse(t)");
}
void op_encode_values(Context &c, int ch, const double *values, int n, uint64_t dim, double scale, bool dense, u64 *plain, int *bad) {
    const int bl = dense ? (int)((dim + c.N - 1) / c.N) : 0;
    c.check(launch_split_scatter(values, plain, n * bl, bl, dim, scale, c.big_factor, c.t[ch], dense ? c.d_index_map : nullptr, c.logN, bad,
                                 c.stream),
            "split_scatter");
    if (dense)
        c.check(launch_ntt_inverse(plain, plain, n * bl, c.logN, c.d_tabs, c.ch[ch].mod_id, 1, fp_range(c, c.ch[ch].mod_id, 1), c.stream),
                "ntt_inverse(t)");
}
void op_encode_onehot(Context &c, int ch, int n, int first_col, u64 *plain) {
    c.check(launch_onehot_scatter(plain, n, first_col, c.d_index_map, c.logN, c.stream), "onehot_scatter");
    c.check(launch_ntt_inverse(plain, plain, n, c.logN, c.d_tabs, c.ch[ch].mod_id, 1, fp_range(c, c.ch[ch].mod_id, 1), c.stream), "ntt_inverse(t)");
}
void op_decode(Context &c, int ch, const u64 *plain, int n, u64 *values) {
    u64 *tmp = c.ws_alloc((size_t)n * c.N);
    c.check(launch_ntt_forward(plain, tmp, n, c.logN, c.d_tabs, c.ch[ch].mod_id, 1, fp_range(c, c.ch[ch].mod_id, 1), c.stream), "ntt_forward(t)");
    c.check(launch_decode_gather(tmp, values, n, c.d_index_map, c.logN, c.stream), "decode_gather");
}
u64 take_nonces(Context &c, int chi, u64 n) {
    if (c.rec) c.refuse("samples encryption randomness (a replay would reuse it for every input)");
    Channel &ch = c.ch[chi];
    if (n >= (1ULL << 31)) throw Error(-1, "too many encryptions in one call");
    if (ch.nonce + n >= (1ULL << 32)) { // the stream id carries 32 bits of the counter
        if (!ch.rng.secure) throw Error(-1, "deterministic (seeded, test-only) channel exhausted its 2^32 encryption nonces");
        rng_from_os(ch.rng);
        ch.nonce = 1;
    }
    const u64 n0 = ch.nonce;
    ch.nonce += n;
    return n0;
}
void op_encrypt(Context &c, int chi, const u64 *plain, size_t plain_stride, int n, int coeffs, u64 nonce0, u64 *ct) {
    Channel &ch = c.ch[chi];
    if (!ch.have_pk) throw Error(-3, "public key is missing");
    const int k = c.k;
    const size_t N = c.N;
    for (int c0 = 0; c0 < n; c0 += 4 * c.chunk) {
        const int m = std::min(4 * c.chunk, n - c0);
        u64 *u = c.ws_alloc((size_t)m * k * N);
        c.check(launch_sample(u, m, SAMPLE_TERNARY, ch.rng, stream_id(8, nonce0 + c0, 0), 1ULL << 16, k, c.logN, c.d_bc, c.stream), "sample");
        c.check(launch_ntt_forward(u, u, m * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        u64 *dst = ct + (size_t)c0 * 2 * k * N;
        c.check(launch_dyadic_bcast(ch.pk->p, u, dst, m, 2, 0, 1, k, c.logN, c.d_bc, c.stream), "dyadic");
        c.check(launch_ntt_inverse(dst, dst, m * 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
        c.check(launch_encrypt_finish(dst, plain ? plain + (size_t)c0 * plain_stride : nullptr, plain_stride, m, plain ? coeffs : 0, ch.rng,
                                      nonce0 + c0, k, c.logN, c.d_bc, ch.pc, c.stream),
                "encrypt_finish");
    }
    c.note(Context::OP_ENCRYPT, chi, n, ct);
}
// ---------------------------------------------------------------- sanitisation (DESIGN 4.18)
int sanitize_max_bits(const Context &c) {
    int best = 1 << 30;
    for (u64 t : c.t) {
        std::vector<u64> quot;
        u64 rem;
        hm::div_product(c.q, t, quot, rem); // floor(q / t): its bit length less one is floor(log2(q / t))
        int bits = 0;
        for (size_t i = quot.size(); i-- > 0;)
            if (quot[i]) { bits = 64 * (int)i + hm::bit_length(quot[i]); break; }
        best = std::min(best, bits - 1 - 2);
    }
    return best;
}
void sanitize_reserve(Context &c, int chi, u64 n) {
    Channel &ch = c.ch[chi];
    if (n > SANITIZE_NONCES - ch.sanitized)
        throw Error(-3, "the channel's sampler key has handed out its 2^48 sanitisation nonces (cnhe_keys_generate_secure re-keys it)");
    ch.sanitized += n;
}
void op_sanitize(Context &c, int chi, const std::vector<const u64 *> &in, const int *slots, int flood_bits, u64 *out) {
    Channel &ch = c.ch[chi];
    const int n = (int)in.size(), k = c.k;
    const size_t N = c.N, kN = (size_t)k * N;
    const KsKeys pks = public_keys(c, chi, n, slots);
    SanitizeConst S;
    memset(&S, 0, sizeof(S));
    S.k = k;
    S.words = flood_bits / 64 + 1; // ceil((b + 1) / 64)
    S.top_mask = (flood_bits + 1) % 64 ? (1ULL << ((flood_bits + 1) % 64)) - 1 : ~0ULL;
    for (int l = 0; l < k; l++) {
        S.q[l] = c.h_bc.q[l];
        S.pow2b[l] = hm::pw(2, (u64)flood_bits, c.q[l]);
    }
    sanitize_reserve(c, chi, (u64)n);
    const int wave = c.wave(3 * kN);
    for (int c0 = 0; c0 < n; c0 += wave) {
        WsScope scope(c);
        const int m = std::min(wave, n - c0);
        u64 *base = c.ws_alloc(1), *u = c.ws_alloc((size_t)m * kN), *dst = out + (size_t)c0 * 2 * kN;
        c.check(launch_sanitize_take(c.d_sanitize_nonce + chi, (u64)m, base, c.stream), "sanitize_take");
        c.check(launch_sanitize_u(u, m, base, ch.rng, k, c.logN, c.d_bc, c.stream), "sanitize_u");
        c.check(launch_ntt_forward(u, u, m * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        std::vector<const u64 *> tab(m);
        for (int i = 0; i < m; i++) tab[i] = pks.per_ct() ? pks.keys[c0 + i] : pks.key;
        c.check(launch_sanitize_upk(key_table(c, tab, 0, m), u, dst, m, k, c.logN, c.d_bc, c.rec != nullptr, c.stream), "sanitize_upk");
        c.check(launch_ntt_inverse(dst, dst, m * 2 * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
        const std::vector<const u64 *> part(in.begin() + c0, in.begin() + c0 + m);
        const u64 *const *in_tab = upload_ptrs(c, part);
        PROF(6, (double)m * 3 * 2 * kN * 8); // in and u pk read, out written: 48 k N bytes per ciphertext
        c.check(launch_sanitize_finish(in_tab, dst, m, base, ch.rng, S, c.logN, c.stream), "sanitize_finish");
    }
    c.note(Context::OP_ENCRYPT, chi, n, out);
    c.note(Context::OP_ADD, chi, n, out);
}
CompactShape compact_shape(const Context &c) {
    CompactShape sh;
    memset(&sh, 0, sizeof(sh));
    sh.k = c.k;
    sh.logn = c.logN;
    for (int l = 0; l < c.k; l++) {
        sh.bits[l] = 64 - __builtin_clzll(c.q[l]);
        sh.off[l + 1] = sh.off[l] + ((u64)c.N * sh.bits[l]) / 64; // N >= 64: every residue fills whole words
    }
    return sh;
}
CompactKey compact_key(Context &c, int chi, u64 nonce0) {
    const Channel &ch = c.ch[chi];
    CompactKey key;
    if (ch.rng.secure) {
        RngKey fresh;
        rng_from_os(fresh);
        memcpy(key.w, fresh.key, sizeof(key.w));
    } else {
        for (int i = 0; i < 4; i++) {
            const u64 w = rng64(ch.rng, stream_id(PURPOSE_COMPACT_KEY, nonce0, 0), (u64)i);
            key.w[2 * i] = (u32)w;
            key.w[2 * i + 1] = (u32)(w >> 32);
        }
    }
    return key;
}
// (c0, c1) = (-(a s) + e + Delta m, a): a from the expansion key (the server regenerates it), e fresh per ciphertext from the channel's sampler
void op_encrypt_compact(Context &c, int chi, const u64 *plain, int n, u64 nonce0, const CompactKey &key, u64 *packed) {
    Channel &ch = c.ch[chi];
    if (!ch.have_sk) throw Error(-3, "secret key is missing");
    const int k = c.k;
    const size_t N = c.N, kN = (size_t)k * N;
    const CompactShape sh = compact_shape(c);
    for (int c0 = 0; c0 < n; c0 += 4 * c.chunk) {
        WsScope scope(c);
        const int m = std::min(4 * c.chunk, n - c0);
        u64 *ct = c.ws_alloc((size_t)m * 2 * kN), *as = c.ws_alloc((size_t)m * kN);
        c.check(launch_compact_expand(ct, nullptr, key, PURPOSE_COMPACT_A, (u64)c0, m, sh, c.d_bc, c.stream), "compact_expand(a)");
        CNHE_CUDA(cudaMemcpy2DAsync(as, kN * 8, ct + kN, 2 * kN * 8, kN * 8, m, cudaMemcpyDeviceToDevice, c.stream));
        c.check(launch_ntt_forward(as, as, m * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        c.check(launch_dyadic_bcast(as, ch.sk->p, as, m, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
        c.check(launch_ntt_inverse(as, as, m * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
        c.check(launch_encrypt_finish_sk(ct, as, plain + (size_t)c0 * N, N, m, (int)N, ch.rng, nonce0 + c0, k, c.logN, c.d_bc, ch.pc, c.stream),
                "encrypt_finish_sk");
        c.check(launch_pack_residues(ct, packed + (size_t)c0 * sh.off[k], m, sh, c.stream), "pack_residues");
        if (c0 == 0) c.note(Context::OP_ENCRYPT, chi, n, ct); // the first ciphertext is alive only in this wave
    }
}
void op_compact_expand(Context &c, const u64 *packed, const CompactKey &key, int n, u64 *ct, cudaStream_t s) {
    const CompactShape sh = compact_shape(c);
    cudaStream_t keep = c.stream;
    c.stream = s; // the profiling events go on the stream the kernel runs on
    {
        ProfScope ps(c, 5, (double)n * (sh.off[c.k] + c.ct_words()) * 8);
        c.check(launch_compact_expand(ct, packed, key, PURPOSE_COMPACT_A, 0, n, sh, c.d_bc, s), "compact_expand");
    }
    c.stream = keep;
}
// x = c0 + c1 s (coefficient form) of the n ciphertexts whose parts are c0, c1 [n][kN]; c1 is overwritten
static void dot_parts(Context &c, int chi, const u64 *c0, u64 *c1, int n, u64 *x) {
    Channel &ch = c.ch[chi];
    if (!ch.have_sk) throw Error(-3, "secret key is missing");
    const int k = c.k;
    const size_t N = c.N;
    c.check(launch_ntt_forward(c1, c1, n * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
    c.check(launch_dyadic_bcast(c1, ch.sk->p, c1, n, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
    c.check(launch_ntt_inverse_add(c1, c0, 1, N, x, n * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse_add");
}
static void dot_with_secret(Context &c, int chi, const u64 *ct, int n, u64 *x) {
    const size_t kN = (size_t)c.k * c.N;
    u64 *c0 = c.ws_alloc((size_t)n * kN), *c1 = c.ws_alloc((size_t)n * kN);
    CNHE_CUDA(cudaMemcpy2DAsync(c0, kN * 8, ct, 2 * kN * 8, kN * 8, n, cudaMemcpyDeviceToDevice, c.stream));
    CNHE_CUDA(cudaMemcpy2DAsync(c1, kN * 8, ct + kN, 2 * kN * 8, kN * 8, n, cudaMemcpyDeviceToDevice, c.stream));
    dot_parts(c, chi, c0, c1, n, x);
}
void op_decrypt(Context &c, int chi, const u64 *ct, int n, u64 *plain) {
    u64 *x = c.ws_alloc((size_t)n * c.k * c.N);
    dot_with_secret(c, chi, ct, n, x);
    c.check(launch_decrypt_round(x, plain, n, c.k, c.logN, c.d_bc, c.ch[chi].pc, c.stream), "decrypt_round");
    c.op_count[Context::OP_DECRYPT] += (uint64_t)n;
}
void op_decrypt_many(Context &c, int chi, const std::vector<const u64 *> &cts, u64 *plain) {
    const int n = (int)cts.size();
    const size_t kN = (size_t)c.k * c.N;
    const int wave = c.wave(3 * kN);
    for (int c0 = 0; c0 < n; c0 += wave) {
        WsScope scope(c);
        const int m = std::min(wave, n - c0);
        u64 *p0 = c.ws_alloc((size_t)m * kN), *p1 = c.ws_alloc((size_t)m * kN), *x = c.ws_alloc((size_t)m * kN);
        const std::vector<const u64 *> part(cts.begin() + c0, cts.begin() + c0 + m);
        c.check(launch_split_parts(upload_ptrs(c, part), p0, p1, m, kN, c.stream), "split_parts");
        dot_parts(c, chi, p0, p1, m, x);
        c.check(launch_decrypt_round(x, plain + (size_t)c0 * c.N, m, c.k, c.logN, c.d_bc, c.ch[chi].pc, c.stream), "decrypt_round");
    }
    c.op_count[Context::OP_DECRYPT] += (uint64_t)n;
}
// Decryptor::invariant_noise_budget: bits(q) - bits(|t * (c0 + c1 s) mod q|_centred) - 1, composed on the host
int op_noise_budget(Context &c, int chi, const u64 *ct) {
    const int k = c.k;
    const size_t N = c.N;
    u64 *x = c.ws_alloc((size_t)k * N);
    dot_with_secret(c, chi, ct, 1, x);
    std::vector<u64> h((size_t)k * N);
    CNHE_CUDA(cudaMemcpyAsync(h.data(), x, h.size() * 8, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    typedef std::vector<u64> Big;
    auto mul_small = [](const Big &a, u64 b) {
        Big r(a.size() + 1, 0);
        u64 carry = 0;
        for (size_t i = 0; i < a.size(); i++) {
            unsigned __int128 v = (unsigned __int128)a[i] * b + carry;
            r[i] = (u64)v;
            carry = (u64)(v >> 64);
        }
        r[a.size()] = carry;
        return r;
    };
    auto add_to = [](Big &a, const Big &b) {
        if (a.size() < b.size() + 1) a.resize(b.size() + 1, 0);
        u64 carry = 0;
        for (size_t i = 0; i < a.size(); i++) {
            unsigned __int128 v = (unsigned __int128)a[i] + (i < b.size() ? b[i] : 0) + carry;
            a[i] = (u64)v;
            carry = (u64)(v >> 64);
        }
    };
    auto cmp = [](const Big &a, const Big &b) {
        size_t n = std::max(a.size(), b.size());
        for (size_t i = n; i-- > 0;) {
            u64 x = i < a.size() ? a[i] : 0, y = i < b.size() ? b[i] : 0;
            if (x != y) return x < y ? -1 : 1;
        }
        return 0;
    };
    auto sub_from = [](Big &a, const Big &b) {
        u64 borrow = 0;
        for (size_t i = 0; i < a.size(); i++) {
            u64 y = i < b.size() ? b[i] : 0;
            unsigned __int128 v = (unsigned __int128)a[i] - y - borrow;
            a[i] = (u64)v;
            borrow = (u64)(v >> 64) ? 1 : 0;
        }
    };
    auto bits = [](const Big &a) {
        for (size_t i = a.size(); i-- > 0;)
            if (a[i]) return (int)(i * 64 + 64 - __builtin_clzll(a[i]));
        return 0;
    };
    Big Q{1};
    for (u64 p : c.q) Q = mul_small(Q, p);
    std::vector<Big> qhat(k, Big{1});
    for (int i = 0; i < k; i++)
        for (int l = 0; l < k; l++)
            if (l != i) qhat[i] = mul_small(qhat[i], c.q[l]);
    Big half = Q;
    {
        unsigned __int128 r = 0;
        for (size_t i = half.size(); i-- > 0;) {
            unsigned __int128 cur = (r << 64) | half[i];
            half[i] = (u64)(cur / 2);
            r = cur % 2;
        }
    }
    int maxbits = 0;
    const u64 t = c.ch[chi].t;
    for (size_t n = 0; n < N; n++) {
        Big acc{0};
        for (int i = 0; i < k; i++) {
            u64 v = hm::mul(hm::mul(h[i * N + n], t % c.q[i], c.q[i]), c.h_bc.inv_qhat_mod_q[i], c.q[i]);
            add_to(acc, mul_small(qhat[i], v));
        }
        while (cmp(acc, Q) >= 0) sub_from(acc, Q);
        if (cmp(acc, half) > 0) {
            Big tmp = Q;
            tmp.resize(std::max(tmp.size(), acc.size()), 0);
            sub_from(tmp, acc);
            acc = tmp;
        }
        maxbits = std::max(maxbits, bits(acc));
    }
    int b = bits(Q) - maxbits - 1;
    return b < 0 ? 0 : b;
}

// ---------------------------------------------------------------- keys (KeyGenerator of SEAL 3.2, sampled on the device)
BufRef &key_slot(Context &c, int channel, int what, u64 arg, size_t &words, bool create) {
    if (channel < 0 || channel >= c.P) throw Error(-1, "bad channel");
    Channel &ch = c.ch[channel];
    const size_t kN = (size_t)c.k * c.N;
    BufRef *slot = nullptr;
    switch (what) {
    case 0: words = kN; slot = &ch.sk; break;
    case 1: words = 2 * kN; slot = &ch.pk; break;
    case 2: words = (size_t)c.dm_relin.D * 2 * kN; slot = &ch.rlk; break;
    case 3:
        words = (size_t)c.dm_galois.D * 2 * kN;
        if (!create && !ch.glk.count(arg)) throw Error(-3, "Galois key not present");
        slot = &ch.glk[arg];
        break;
    default: throw Error(-1, "bad key kind");
    }
    if (create && !*slot) *slot = c.alloc(words);
    if (!*slot) throw Error(-3, "key is missing");
    return *slot;
}
void rlk_ready(Context &c, int channel) { rlk_ready(c, c.ch[channel]); }
void rlk_ready(Context &c, KeySet &ch) {
    ch.have_rlk = true;
    ch.rlk_packed.reset();
    bool small = true;
    for (u64 q : c.q) small = small && q < (1ULL << 48);
    if (!ch.rlk || !small || !ks_fused_built(c)) return;
    const size_t polys = (size_t)c.dm_relin.D * 2 * c.k;
    ch.rlk_packed = c.alloc(polys * c.N * 6 / 8);
    c.check(launch_pack_keys48(ch.rlk->p, reinterpret_cast<uint4 *>(ch.rlk_packed->p), (int)polys, c.logN, c.stream), "pack_keys48");
    // the channel's key switches may run on another stream than this one: the copy is complete before any stream reads it
    CNHE_CUDA(cudaStreamSynchronize(c.stream));
}
// Randomness of D consecutive key pairs: pair d draws a from the channel's uniform sampler under stream a_stream0 + (d << 16), or -- with
// a_key set -- expands it from that key under stream_id(PURPOSE_KEYS_A, a_pair0 + d, l) (compact key sets); e under e_stream0 + (d << 16)
struct KeyRandom {
    const CompactKey *a_key = nullptr;
    u64 a_stream0 = 0, a_pair0 = 0, e_stream0 = 0;
};
// key-switching keys for `target` (k*N, NTT form): key (i,j) = (-(a s + e) + [residue i] 2^{jw} target, a) -> out [D][2][k][N];
// target == null: D = 1 and out = the public key (-(a s + e), a)
static void make_kskeys(Context &c, Channel &ch, const u64 *target_ntt, const DigitMap *dm, const KeyRandom &r, u64 *out) {
    const int k = c.k, D = target_ntt ? dm->D : 1;
    const size_t N = c.N, kN = (size_t)k * N;
    // c1 = a (uniform), written in place: key d part 1
    u64 *e = c.ws_alloc((size_t)D * kN), *as = c.ws_alloc((size_t)D * kN), *a = c.ws_alloc((size_t)D * kN);
    if (r.a_key) {
        c.check(launch_compact_expand(out, nullptr, *r.a_key, PURPOSE_KEYS_A, r.a_pair0, D, compact_shape(c), c.d_bc, c.stream), "compact_expand(a)");
        CNHE_CUDA(cudaMemcpy2DAsync(a, kN * 8, out + kN, 2 * kN * 8, kN * 8, D, cudaMemcpyDeviceToDevice, c.stream));
    } else {
        c.check(launch_sample(a, D, SAMPLE_UNIFORM, ch.rng, r.a_stream0, 1ULL << 16, k, c.logN, c.d_bc, c.stream), "sample");
    }
    c.check(launch_sample(e, D, SAMPLE_NOISE, ch.rng, r.e_stream0, 1ULL << 16, k, c.logN, c.d_bc, c.stream), "sample");
    c.check(launch_ntt_forward(e, e, D * k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
    c.check(launch_dyadic_bcast(a, ch.sk->p, as, D, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
    c.check(launch_ct_add(as, e, as, (size_t)D * kN, k, c.logN, c.d_bc, 0, c.stream), "ct_add");
    c.check(launch_ct_negate(as, as, (size_t)D * kN, k, c.logN, c.d_bc, c.stream), "ct_negate");
    // interleave into [D][2][k][N]
    CNHE_CUDA(cudaMemcpy2DAsync(out, 2 * kN * 8, as, kN * 8, kN * 8, D, cudaMemcpyDeviceToDevice, c.stream));
    CNHE_CUDA(cudaMemcpy2DAsync(out + kN, 2 * kN * 8, a, kN * 8, kN * 8, D, cudaMemcpyDeviceToDevice, c.stream));
    if (!target_ntt) return;
    // add 2^{jw} * target on residue src[d] of c0 of key d
    std::vector<u64> factors(D);
    for (int d = 0; d < D; d++) factors[d] = hm::pw(2, (u64)dm->shift[d], c.q[dm->src[d]]);
    u64 *dfac = c.ws_alloc(D);
    c.h2d(dfac, factors.data(), D * 8);
    c.check(launch_key_add_scaled(out, target_ntt, dfac, *dm, k, c.logN, c.d_bc, c.stream), "key_add_scaled");
}
static KeyRandom sampled(u64 purpose_a, u64 purpose_e, u64 key_tag) {
    KeyRandom r;
    r.a_stream0 = stream_id(purpose_a, key_tag * 256, 0);
    r.e_stream0 = stream_id(purpose_e, key_tag * 256, 0);
    return r;
}
// rs = NTT(s(x^elt)) from the coefficient-form secret key: the ciphertext Galois kernel on (sk_coeff, sk_coeff), whose perm_c1 output
// receives the permuted second part
static void galois_secret(Context &c, const u64 *sk_coeff, u64 elt, u64 *rs) {
    const size_t kN = (size_t)c.k * c.N;
    u64 *pair = c.ws_alloc(2 * kN), *base = c.ws_alloc(2 * kN);
    CNHE_CUDA(cudaMemcpyAsync(pair, sk_coeff, kN * 8, cudaMemcpyDeviceToDevice, c.stream));
    CNHE_CUDA(cudaMemcpyAsync(pair + kN, sk_coeff, kN * 8, cudaMemcpyDeviceToDevice, c.stream));
    c.check(launch_galois(pair, base, rs, 1, galois_inverse(c.N, elt), c.k, c.logN, c.d_bc, c.stream), "galois");
    c.check(launch_ntt_forward(rs, rs, c.k, c.logN, c.d_tabs, 0, c.k, fp_range(c, 0, c.k), c.stream), "ntt_forward");
}
static void keys_generate_impl(Context &c, bool secure, u64 seed) {
    const int k = c.k;
    const size_t N = c.N, kN = (size_t)k * N;
    for (int ci = 0; ci < c.P; ci++) {
        c.set_channel(ci);
        Channel &ch = c.ch[ci];
        if (secure) rng_from_os(ch.rng);
        else { memset(&ch.rng, 0, sizeof(ch.rng)); ch.rng.seed = seed + (u64)ci; }
        ch.nonce = 1;
        ch.sanitized = 0; // a new sampler key: its sanitisation nonces start again from 0
        CNHE_CUDA(cudaMemsetAsync(c.d_sanitize_nonce + ci, 0, 8, c.stream));
        size_t words;
        // secret key: ternary, kept in NTT form (and a coefficient-form copy for the Galois keys)
        BufRef &sk = key_slot(c, ci, 0, 0, words, true);
        u64 *sk_coeff = c.ws_alloc(kN);
        c.check(launch_sample(sk_coeff, 1, SAMPLE_TERNARY, ch.rng, stream_id(1, 0, 0), 0, k, c.logN, c.d_bc, c.stream), "sample");
        c.check(launch_ntt_forward(sk_coeff, sk->p, k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        ch.have_sk = true;
        // public key (-(a s + e), a)
        BufRef &pk = key_slot(c, ci, 1, 0, words, true);
        u64 *e = c.ws_alloc(kN), *as = c.ws_alloc(kN);
        c.check(launch_sample(pk->p + kN, 1, SAMPLE_UNIFORM, ch.rng, stream_id(2, 0, 0), 0, k, c.logN, c.d_bc, c.stream), "sample");
        c.check(launch_sample(e, 1, SAMPLE_NOISE, ch.rng, stream_id(3, 0, 0), 0, k, c.logN, c.d_bc, c.stream), "sample");
        c.check(launch_ntt_forward(e, e, k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_forward");
        c.check(launch_dyadic_bcast(pk->p + kN, sk->p, as, 1, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
        c.check(launch_ct_add(as, e, as, kN, k, c.logN, c.d_bc, 0, c.stream), "ct_add");
        c.check(launch_ct_negate(as, pk->p, kN, k, c.logN, c.d_bc, c.stream), "ct_negate");
        ch.have_pk = true;
        // relinearization keys for s^2
        BufRef &rlk = key_slot(c, ci, 2, 0, words, true);
        u64 *s2 = c.ws_alloc(kN);
        c.check(launch_dyadic_bcast(sk->p, sk->p, s2, 1, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
        make_kskeys(c, ch, s2, &c.dm_relin, sampled(4, 5, 0), rlk->p);
        rlk_ready(c, ci);
        // Galois keys: s(x^elt) in NTT form
        for (size_t gi = 0; gi < c.galois_elts.size(); gi++) {
            const u64 elt = c.galois_elts[gi];
            u64 *rs = c.ws_alloc(kN);
            galois_secret(c, sk_coeff, elt, rs);
            BufRef &gk = key_slot(c, ci, 3, elt, words, true);
            make_kskeys(c, ch, rs, &c.dm_galois, sampled(6, 7, gi + 1), gk->p);
        }
        c.sync();
        ws_release_all(c);
    }
}

// ---------------------------------------------------------------- compact key sets (format: compact.cu)
size_t compact_key_pairs(const Context &c, int sets, size_t n_galois) {
    return ((sets & 1) ? 1 : 0) + ((sets & 2) ? (size_t)c.dm_relin.D : 0) + n_galois * c.dm_galois.D;
}
void op_keys_save_compact(Context &c, int chi, int sets, const std::vector<u64> &elts, u64 nonce0, const CompactKey &key, u64 *packed) {
    Channel &ch = c.ch[chi];
    if (!ch.have_sk) throw Error(-3, "secret key is missing");
    const int k = c.k;
    const size_t kN = (size_t)k * c.N;
    const CompactShape sh = compact_shape(c);
    u64 *sk_coeff = c.ws_alloc(kN);
    c.check(launch_ntt_inverse(ch.sk->p, sk_coeff, k, c.logN, c.d_tabs, 0, k, fp_range(c, 0, k), c.stream), "ntt_inverse");
    u64 kappa = 0;
    // one key set: D pairs from kappa on, generated into scratch and packed into their place in the channel's payload
    auto emit = [&](const u64 *target, const DigitMap *dm) {
        WsScope scope(c);
        const int D = target ? dm->D : 1;
        KeyRandom r;
        r.a_key = &key;
        r.a_pair0 = kappa;
        r.e_stream0 = stream_id(PURPOSE_KEYS_E, nonce0 + kappa, 0);
        u64 *keys = c.ws_alloc((size_t)D * 2 * kN);
        make_kskeys(c, ch, target, dm, r, keys);
        c.check(launch_pack_residues(keys, packed + kappa * sh.off[k], D, sh, c.stream), "pack_residues");
        kappa += D;
    };
    if (sets & 1) emit(nullptr, nullptr);
    if (sets & 2) {
        WsScope scope(c);
        u64 *s2 = c.ws_alloc(kN);
        c.check(launch_dyadic_bcast(ch.sk->p, ch.sk->p, s2, 1, 1, 1, 0, k, c.logN, c.d_bc, c.stream), "dyadic");
        emit(s2, &c.dm_relin);
    }
    for (u64 elt : elts) {
        WsScope scope(c);
        u64 *rs = c.ws_alloc(kN);
        galois_secret(c, sk_coeff, elt, rs);
        emit(rs, &c.dm_galois);
    }
}
// pairs of one blob channel in order: public key, relinearisation digits, Galois digits of each element; `slot_of` gives each set's key buffer
template <class SlotOf>
static void keys_load_compact(Context &c, int sets, const std::vector<u64> &elts, const u64 *packed, const CompactKey &key, SlotOf slot_of) {
    const CompactShape sh = compact_shape(c);
    u64 kappa = 0;
    auto expand = [&](int what, u64 arg) {
        size_t words;
        BufRef &slot = slot_of(what, arg, words);
        const int D = (int)(words / c.ct_words());
        c.check(launch_compact_expand(slot->p, packed + kappa * sh.off[c.k], key, PURPOSE_KEYS_A, kappa, D, sh, c.d_bc, c.stream), "compact_expand");
        kappa += D;
    };
    if (sets & 1) expand(1, 0);
    if (sets & 2) expand(2, 0);
    for (u64 elt : elts) expand(3, elt);
}
void op_keys_load_compact(Context &c, int chi, int sets, const std::vector<u64> &elts, const u64 *packed, const CompactKey &key) {
    keys_load_compact(c, sets, elts, packed, key, [&](int what, u64 arg, size_t &words) -> BufRef & { return key_slot(c, chi, what, arg, words, true); });
    if (sets & 1) c.ch[chi].have_pk = true;
    if (sets & 2) rlk_ready(c, chi); // synchronises the channel's stream
}
void op_keys_load_compact(Context &c, KeySet &dst, int sets, const std::vector<u64> &elts, const u64 *packed, const CompactKey &key) {
    keys_load_compact(c, sets, elts, packed, key, [&](int what, u64 arg, size_t &words) -> BufRef & {
        BufRef &b = what == 1 ? dst.pk : what == 2 ? dst.rlk : dst.glk[arg];
        words = (size_t)(what == 1 ? 1 : what == 2 ? c.dm_relin.D : c.dm_galois.D) * c.ct_words();
        if (!b) b = c.alloc(words);
        return b;
    });
    if (sets & 1) dst.have_pk = true; // the key slot's sanitisation encrypts zero under it
    if (sets & 2) rlk_ready(c, dst); // synchronises the stream
}

void keys_generate(Context &c, u64 seed) { keys_generate_impl(c, false, seed); }
void keys_generate_secure(Context &c) { keys_generate_impl(c, true, 0); }

// ---------------------------------------------------------------- levels (DESIGN 4.17)
Context *context_derive(Context &p, int k) {
    if (k < 1 || k >= p.k) throw Error(-1, "a derived level needs 1 <= k < the parent's coefficient prime count");
    std::unique_ptr<Context> cp(context_create(p.t.data(), p.P, p.N, p.q.data(), k, p.dbc_relin, p.dbc_galois, p.device));
    Context &c = *cp;
    c.root = p.root;
    c.h_bc.centered_mtilde = c.h_bf.centered_mtilde = p.h_bc.centered_mtilde;
    CNHE_CUDA(cudaMemcpy(c.d_bc, &c.h_bc, sizeof(BehzConst), cudaMemcpyHostToDevice));
    CNHE_CUDA(cudaMemcpy(c.d_bf, &c.h_bf, sizeof(BehzConstF), cudaMemcpyHostToDevice));
    c.chunk = p.chunk;
    c.multi_stream = p.multi_stream;
    c.galois_elts = p.galois_elts;
    // a seeded (test) sampler is inherited, so that the child encrypts as a seeded context on q[:k] would; a secure channel keeps the
    // fresh OS key context_create drew, so parent and child never share encryption randomness
    for (int ci = 0; ci < p.P; ci++)
        if (!p.ch[ci].rng.secure) c.ch[ci].rng = p.ch[ci].rng;
    c.clients.resize(p.clients.size());
    for (int s = 0; s <= (int)p.clients.size(); s++) restrict_keys(c, p, s);
    return cp.release();
}
// Key (i, j) of a key-switching key is an encryption of 2^{jw} target on residue i only; its rows < k encrypt the same under q[:k], and the
// digits of residues < k are the first D' (residue-major): [D][2][k_src][N] -> [D'][2][k][N] is one strided copy
void restrict_keys(Context &dst, const Context &src, int s) {
    const size_t N = dst.N, kN = (size_t)dst.k * N, skN = (size_t)src.k * N;
    dst.keys_changed(s); // a graph recorded in dst against the slot's previous keys refuses to launch
    if (s > 0) {
        if ((size_t)s > dst.clients.size()) dst.clients.resize(s);
        dst.clients[s - 1].clear();
        if (!src.slot_live(s)) {
            dst.origin[s] = src.key_origin(s);
            return;
        }
        dst.clients[s - 1].resize(dst.P);
    }
    auto cut = [&](const BufRef &from, size_t rows) { // rows of k_src N words -> rows of k N words
        BufRef to = dst.alloc(rows * kN);
        CNHE_CUDA(cudaMemcpy2DAsync(to->p, kN * 8, from->p, skN * 8, kN * 8, rows, cudaMemcpyDeviceToDevice, dst.stream));
        return to;
    };
    for (int ci = 0; ci < dst.P; ci++) {
        dst.set_channel(ci);
        const KeySet &from = src.keys(ci, s);
        KeySet &to = s == 0 ? static_cast<KeySet &>(dst.ch[ci]) : dst.clients[s - 1][ci];
        to.have_rlk = false;
        to.rlk.reset();
        to.rlk_packed.reset();
        to.glk.clear();
        to.have_pk = from.have_pk && from.pk;
        to.pk = to.have_pk ? cut(from.pk, 2) : nullptr;
        if (s == 0) {
            const Channel &fc = src.ch[ci];
            Channel &tc = dst.ch[ci];
            tc.have_sk = fc.have_sk && fc.sk;
            tc.sk = tc.have_sk ? cut(fc.sk, 1) : nullptr;
        }
        for (const auto &g : from.glk) to.glk[g.first] = cut(g.second, (size_t)dst.dm_galois.D * 2);
        if (from.have_rlk && from.rlk) {
            to.rlk = cut(from.rlk, (size_t)dst.dm_relin.D * 2);
            rlk_ready(dst, to); // synchronises the stream
        }
        CNHE_CUDA(cudaStreamSynchronize(dst.stream));
    }
    dst.set_channel(0);
    dst.origin[s] = src.key_origin(s);
}
void op_mod_switch(Context &src, Context &dst, int ch, const std::vector<const u64 *> &in, u64 *out) {
    ModSwitchConst M;
    memset(&M, 0, sizeof(M));
    M.k = src.k;
    M.k_out = dst.k;
    for (int l = 0; l < src.k; l++) {
        M.q[l] = make_dmod(src.q[l]);
        M.half[l] = src.q[l] >> 1;
    }
    for (int j = dst.k; j < src.k; j++)
        for (int i = 0; i < j; i++) {
            const u64 qi = src.q[i];
            M.half_mod[j][i] = M.half[j] % qi;
            M.inv[j][i] = hm::inv(src.q[j] % qi, qi);
            M.inv_s[j][i] = hm::shoup(M.inv[j][i], qi);
        }
    const cudaStream_t ss = src.streams[src.multi_stream ? ch : 0];
    dst.set_channel(ch);
    cudaEvent_t ready, done;
    CNHE_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    CNHE_CUDA(cudaEventCreateWithFlags(&done, cudaEventDisableTiming));
    CNHE_CUDA(cudaEventRecord(ready, ss)); // the inputs are complete on the source's stream
    CNHE_CUDA(cudaStreamWaitEvent(dst.stream, ready, 0));
    const size_t in_words = (size_t)2 * src.k * dst.N, out_words = (size_t)2 * dst.k * dst.N;
    const int wave = dst.wave(in_words + out_words);
    for (int c0 = 0; c0 < (int)in.size(); c0 += wave) {
        const int m = std::min<int>(wave, (int)in.size() - c0);
        const std::vector<const u64 *> part(in.begin() + c0, in.begin() + c0 + m);
        dst.check(launch_mod_switch(upload_ptrs(dst, part), out + (size_t)c0 * out_words, m, dst.logN, M, dst.stream), "mod_switch");
    }
    CNHE_CUDA(cudaEventRecord(done, dst.stream)); // the source's later use (and release) of the inputs waits for the kernel
    CNHE_CUDA(cudaStreamWaitEvent(ss, done, 0));
    cudaEventDestroy(ready);
    cudaEventDestroy(done);
}

} // namespace cnhe
