// Internal header shared by the translation units that implement the C ABI (vec.cu: vectors, layers; wire.cu: wire formats).
#pragma once
#include <initializer_list>
#include <memory>
#include <string>
#include <vector>

#include "../../include/cnhe.h"
#include "runtime.h"

using namespace cnhe;

struct cnhe_ctx {
    Context *c;
};

struct cnhe_vec;
// The outputs of one cnhe_layer_square call before their relinearisation (DESIGN 4.15): the size-3 products of every ciphertext in one
// slab per channel.  A scalar-MAC layer that can key-switch its own outputs instead reads them as they are; any other use relinearises
// the whole group (materialise, vec.cu) and re-points every member at the result, which is the eager square's words.
struct PendingGroup {
    std::vector<BufRef> slab3;       // per channel: [total][3][k][N]
    std::vector<int> ct_slot;        // key slot of every ciphertext, as the square recorded it
    int total = 0;
    std::vector<cnhe_vec *> members; // the live vectors that still point into slab3
};
struct cnhe_vec {
    cnhe_vec() = default;
    cnhe_vec(const cnhe_vec &o); // an alias of a pending vector joins its group
    cnhe_vec &operator=(const cnhe_vec &) = delete;
    ~cnhe_vec();
    Context *ctx = nullptr;
    uint64_t dim = 0;
    double scale = 1.0;
    int format = CNHE_DENSE;
    bool enc = false;
    int slot = 0;   // encrypted: the key slot whose evaluation keys its key switches use (plain vectors ignore it)
    // made while recording a graph: that graph's key binding, which maps `slot` to the slot the graph is bound to (key_slot)
    std::shared_ptr<const KeyBinding> binding;
    int key_slot() const { return binding ? binding->slot(slot) : slot; }
    int blocks = 0; // ciphertexts / plaintexts per channel
    std::vector<BufRef> buf; // per channel: enc -> blocks*2kN words, plain dense -> blocks*N words, plain sparse -> `blocks` scalars
    std::vector<size_t> off;
    std::vector<std::vector<u64>> scalars; // plain sparse: host copy of the constants (mod t)
    bool is_const = false;                 // plain dense whose every plaintext is a constant polynomial
    std::vector<u64> const_val;            // per channel constant (mod t) when is_const

    std::shared_ptr<PendingGroup> pend; // set while this vector's ciphertexts are unrelinearised products in pend->slab3
    size_t pend_ct = 0;                 // ... starting at ciphertext pend_ct of the group

    u64 *ptr(int ch) const {
        if (pend) throw Error(CNHE_ERR_INVALID, "internal error: a squared vector was read before its relinearisation");
        return buf[ch]->p + off[ch];
    }
    const u64 *pending_block(int ch, int b) const { return pend->slab3[ch]->p + (pend_ct + (size_t)b) * 3 * ctx->k * ctx->N; }
    size_t unit() const { return enc ? ctx->ct_words() : (format == CNHE_DENSE ? (size_t)ctx->N : 1); }
    u64 *block(int ch, int b) const { return ptr(ch) + (size_t)b * unit(); }
};

int set_err(int code, const std::string &m); // thread-local last error (vec.cu)
// Graph recording (vec.cu).  api_enter: start of a public call on a context -- names the call for refusals and refuses calls from another
// thread than the recording one.  api_fail: a call failed; a failure while recording aborts the recording (the context stays usable).
// not_recorded: refuses the call while recording, saying why it cannot be part of a graph.
void api_enter(Context &c, const char *name);
int api_fail(Context &c, int code, const std::string &m);
static inline void not_recorded(Context &c, const char *why) { if (c.rec) c.refuse(why); }

#define API_BEGIN(CTX)                                                                                                 \
    if (!(CTX)) return set_err(CNHE_ERR_INVALID, "null context");                                                      \
    Context &c = *(CTX)->c;                                                                                            \
    try {                                                                                                              \
        std::lock_guard<std::recursive_mutex> lock(c.mu);                                                              \
        api_enter(c, __func__);                                                                                        \
        CNHE_CUDA(cudaSetDevice(c.device));                                                                            \
        c.set_channel(0);                                                                                              \
        c.slot = 0;                                                                                                    \
        c.foreign = false;                                                                                             \
        ws_release_all(c);
#define API_END                                                                                                        \
    }                                                                                                                  \
    catch (const Error &e) { return api_fail(c, e.code, e.what()); }                                                  \
    catch (const std::exception &e) { return api_fail(c, CNHE_ERR_INVALID, e.what()); }                               \
    return CNHE_OK;
static inline void fail(const char *m) { throw Error(CNHE_ERR_INVALID, m); }
cnhe_vec *new_vec(Context &c, uint64_t dim, double scale, int format, bool enc, int blocks); // bound to the call's key slot c.slot
// the key slot the encrypted vectors among vs share (plain and null entries have none), made the call's slot; CNHE_ERR_INVALID when two
// encrypted vectors belong to different slots or the slot was removed
int use_slot(Context &c, const cnhe_vec *const *vs, int n);
static inline int use_slot(Context &c, std::initializer_list<const cnhe_vec *> vs) { return use_slot(c, vs.begin(), (int)vs.size()); }
void alloc_channels(cnhe_vec *v);
void same_ctx(Context &c, const cnhe_vec *v); // also relinearises v's pending group (as use_slot and the layers' slot checks do)
void materialise(Context &c, const cnhe_vec *v);

