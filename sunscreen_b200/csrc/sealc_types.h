// sealc_types.h — handle types behind the SEAL-named C ABI (include/b200_sealc.h), shared by sealc_api.cpp
// (contexts, evaluator, keys, encryptor, decryptor, encoder), sealc_wire.cpp (Save/Load wire format) and
// sealc_polyarray.cpp (PolynomialArray).  Each struct mirrors the state the reference's C++ object carries
// (S/ciphertext.h:337-715, S/plaintext.h, S/kswitchkeys.h:340, S/publickey.h, S/secretkey.h, S/context.h).
#pragma once
#include "../../include/b200_bfv.h"
#include "host_ctx.h"
#include "sampling.h"
#include <algorithm>
#include <array>
#include <atomic>
#include <condition_variable>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <vector>
#include <string.h> // explicit_bzero

namespace b200c
{
typedef uint64_t u64;
typedef std::array<u64, 4> ParmsId;
static const ParmsId kZeroId = { { 0, 0, 0, 0 } };

static const long S_OK_ = 0L;
static const long E_POINTER_ = (long)0x80004003L;
static const long E_INVALIDARG_ = (long)0x80070057L;
static const long E_OUTOFMEMORY_ = (long)0x8007000EL;
static const long E_UNEXPECTED_ = (long)0x8000FFFFL;
static const long COR_E_INVALIDOPERATION_ = (long)0x80131509L;
static const long ERROR_INVALID_INDEX_ = (long)0x80070585L;

struct InvalidArg : std::runtime_error { using std::runtime_error::runtime_error; };
struct LogicErr : std::runtime_error { using std::runtime_error::runtime_error; };

struct Modulus_ { u64 value = 0; };

struct EncParams_
{
    uint8_t scheme = 1; // bfv
    u64 n = 0;
    std::vector<u64> coeff;
    u64 plain = 0;
};

// BFV default coefficient moduli for 128-bit security (values of S/util/globals.cpp:23-71) and the HE-standard
// total bit bounds (S/util/hestdparms.h).
static const u64 kDefault1024[] = { 0x7e00001 };
static const u64 kDefault2048[] = { 0x3fffffff000001 };
static const u64 kDefault4096[] = { 0xffffee001, 0xffffc4001, 0x1ffffe0001 };
static const u64 kDefault8192[] = { 0x7fffffd8001, 0x7fffffc8001, 0xfffffffc001, 0xffffff6c001, 0xfffffebc001 };
static const u64 kDefault16384[] = { 0xfffffffd8001, 0xfffffffa0001, 0xfffffff00001, 0x1fffffff68001, 0x1fffffff50001,
                              0x1ffffffee8001, 0x1ffffffea0001, 0x1ffffffe88001, 0x1ffffffe48001 };
static const u64 kDefault32768[] = { 0x7fffffffe90001, 0x7fffffffbf0001, 0x7fffffffbd0001, 0x7fffffffba0001, 0x7fffffffaa0001,
                              0x7fffffffa50001, 0x7fffffff9f0001, 0x7fffffff7e0001, 0x7fffffff770001, 0x7fffffff380001,
                              0x7fffffff330001, 0x7fffffff2d0001, 0x7fffffff170001, 0x7fffffff150001, 0x7ffffffef00001,
                              0xfffffffff70001 };
inline int max_bits_tc128(u64 n)
{
    switch (n)
    {
    case 1024: return 27;
    case 2048: return 54;
    case 4096: return 109;
    case 8192: return 218;
    case 16384: return 438;
    case 32768: return 881;
    default: return 0;
    }
}
inline int max_bits(u64 n, int sec)
{
    if (sec == 128)
        return max_bits_tc128(n);
    if (sec == 192)
    {
        switch (n) { case 1024: return 19; case 2048: return 37; case 4096: return 75; case 8192: return 152;
                     case 16384: return 305; case 32768: return 611; default: return 0; }
    }
    if (sec == 256)
    {
        switch (n) { case 1024: return 14; case 2048: return 29; case 4096: return 58; case 8192: return 118;
                     case 16384: return 237; case 32768: return 476; default: return 0; }
    }
    return 0;
}

// Shared ownership of the device context: data objects may outlive the SEALContext handle they were created with (Rust
// drops them in any order), and their device buffers must be returned to a context that still exists.
struct DevOwner
{
    b200_ctx *dev = nullptr;
    ~DevOwner()
    {
        if (dev)
            b200_ctx_destroy(dev);
    }
};

struct Ciphertext_;
struct KSwitchKeys_;
struct Context_
{
    EncParams_ parms;
    bool parameters_set = false;
    bool using_keyswitching = false;
    bool using_batching = false;
    b200_ctx *dev = nullptr;         // == owner->dev
    std::shared_ptr<DevOwner> owner; // keeps the device context alive for every object holding device memory
    int levels = 0, first_level = 0;
    std::vector<ParmsId> ids; // per level
    std::vector<int> level_k;
    std::mutex mu;            // serialises ENQUEUE (layer-1 caches, launch bookkeeping); never held while waiting for the GPU
    bool check_transparent = true;
    // Evaluator operations of different host threads run on different streams ("lanes") so that their small kernels
    // overlap on the GPU (sunscreen_runtime calls one Evaluator from rayon workers, run.rs:415-469).  A lane is owned by
    // one operation at a time; every operation completes before it returns, so results are visible to any thread.
    struct Lane
    {
        std::mutex m;
        bool ready = false;
        void *stream = nullptr;
        uint32_t *hflag = nullptr;    // transparent-result flag: pinned host memory the check kernel writes directly
        u64 **hptrs = nullptr;        // pinned pointer table of the combining layer: 3 * COMBINE_MAX entries the kernels read directly
        // CUDA graphs of the combining layer's launch sequences, one per (kind, level, batch size, key): every varying input
        // reaches the kernels through `hptrs` / `hflag`, whose addresses never change, so a graph is replayed as it is
        struct Graph
        {
            int kind, lv;
            size_t n;
            const void *key;
            void *exec;   // nullptr: seen once (caches are warm), capture on the next use
            uint64_t stamp;
            uint32_t elt; // Galois element (rotations)
        };
        std::vector<Graph> graphs;
        uint64_t clock = 0;
        void *ev = nullptr;     // blocking-sync event of the batch seams' waits (b200_stream_synchronize_blocking)
        u64 *pad_out = nullptr; // scratch destination of the pad items of a batch rounded up to a power of two
        size_t pad_words = 0;
    };
    static const int GRAPHS_PER_LANE = 48;
    bool use_graphs = true; // B200_NO_GRAPHS=1: enqueue the kernels one by one
    // what the combining layer did with each batch, summed over the lanes (B200_Context_GraphStatsDebug): a shape's first
    // sight (kernel by kernel), its capture, a capture that was refused, a replay, an LRU eviction, and a batch that ran
    // without a graph (graphs off, a reshaped alias, or a shape whose capture was refused before)
    enum { GS_FIRST, GS_CAPTURE, GS_REFUSED, GS_REPLAY, GS_EVICT, GS_NO_GRAPH, GS_COUNT };
    std::atomic<uint64_t> graph_stats[GS_COUNT] = {};
    // B200_BLOCKING_WAITS=1: the batch seams sleep on a blocking-sync event instead of spinning in cudaStreamSynchronize.  Off by
    // default: the sleeping wait was measured to halve the throughput of the chunked host-buffer pipeline (wake-up latency
    // of the order of a chunk's run time); it exists for hosts where caller threads outnumber the cores the process is granted.
    bool blocking_waits = false;
    static const int NLANE = 8;
    Lane lanes[NLANE];
    // Flat combining of concurrent per-handle calls (sealc_api.cpp: combine_submit): calls of the same kind that arrive
    // while one is executing are run TOGETHER as one batched launch sequence by whichever caller holds the combiner, so
    // N rayon workers cost one sequence of launches per round instead of N (sunscreen_runtime/src/run.rs:415-469).
    struct CombineReq
    {
        int kind = 0;             // index into Context_::comb
        Ciphertext_ *a = nullptr, *b = nullptr, *dst = nullptr;
        KSwitchKeys_ *keys = nullptr;
        size_t key_index = 0;
        uint32_t elt = 0;
        int lv = 0;
        bool done = false;
        std::exception_ptr err;
        bool compatible(const CombineReq &o) const
        {
            return kind == o.kind && lv == o.lv && keys == o.keys && key_index == o.key_index && elt == o.elt;
        }
    };
    struct Combiner
    {
        std::mutex m;
        std::condition_variable cv;
        std::vector<CombineReq *> pending;
        int active = 0; // leaders currently executing a batch
    };
    int combine_leaders = 4; // per kind: a caller that finds fewer leaders busy runs at once, on its own lane (B200_COMBINE_LEADERS)
    static const int NCOMB = 3;       // multiply (2,2) | relinearize (3 -> 2) | apply_galois
    static const int COMBINE_MAX = 64; // items per combined batch (= entries of a lane's pinned flag array)
    Combiner comb[NCOMB];
    bool combine = true;              // B200_NO_COMBINE=1 switches it off (every call runs alone, as before)
    // The SEALContext handle and every object created from it (Evaluator, Encryptor, Decryptor, KeyGenerator,
    // BatchEncoder) share the context, as the reference's objects share SEALContext's internals: it goes away with the
    // last of them, whichever order the caller destroys them in.
    std::atomic<int> refs{ 1 };
    static void release(Context_ *c)
    {
        if (c && c->refs.fetch_sub(1) == 1)
            delete c;
    }
    ~Context_()
    {
        if (dev)
        {
            for (auto &l : lanes)
            {
                if (l.stream)
                    b200_stream_destroy(dev, l.stream);
                if (l.hflag)
                    b200_free_host(l.hflag);
                if (l.hptrs)
                    b200_free_host(l.hptrs);
                for (auto &g : l.graphs)
                    if (g.exec)
                        b200_graph_destroy(dev, g.exec);
                if (l.pad_out)
                    b200_free(dev, l.pad_out);
                if (l.ev)
                    b200_event_destroy(dev, l.ev);
            }
            if (!owner)
                b200_ctx_destroy(dev);
        }
    }
    int level_of(const ParmsId &id) const
    {
        for (int i = 0; i < (int)ids.size(); i++)
            if (ids[i] == id)
                return i;
        return -1;
    }
};

inline void dev_check(int rc)
{
    if (rc == 0)
        return;
    if (rc == B200_E_INVALID)
        throw InvalidArg(b200_last_error());
    if (rc == B200_E_LOGIC)
        throw LogicErr(b200_last_error());
    if (rc == B200_E_NOMEM)
        throw std::bad_alloc();
    throw std::runtime_error(b200_last_error());
}

struct CtxHold
{
    Context_ *c = nullptr;
    void bind(Context_ *ctx)
    {
        if (c == ctx)
            return;
        Context_::release(c);
        c = ctx;
        if (c)
            c->refs.fetch_add(1);
    }
    ~CtxHold() { Context_::release(c); }
    CtxHold() = default;
    CtxHold(const CtxHold &) = delete;
    CtxHold &operator=(const CtxHold &) = delete;
};

// One Evaluator operation: owns a lane (stream) for its whole duration and the context mutex while it enqueues.
struct OpScope;
inline thread_local OpScope *tl_scope = nullptr;
struct OpScope
{
    Context_ *c;
    Context_::Lane *lane = nullptr;
    std::unique_lock<std::mutex> lane_lk, ctx_lk;
    OpScope *outer;
    bool blocking = false; // sleep instead of spinning while the GPU works (set by the batch seams: their waits are milliseconds)
    explicit OpScope(Context_ *ctx) : c(ctx), outer(tl_scope)
    {
        dev_check(b200_bind_thread(ctx->dev)); // worker threads of the caller never called cudaSetDevice themselves
        if (outer && outer->c == ctx)
        { // nested helper inside an operation of the same context: share its lane and its lock
            lane = outer->lane;
            tl_scope = this;
            return;
        }
        static std::atomic<unsigned> next{ 0 };
        static thread_local unsigned pref = next++;
        for (unsigned probe = 0;; probe++)
        {
            Context_::Lane &l = ctx->lanes[(pref + probe) % Context_::NLANE];
            std::unique_lock<std::mutex> lk(l.m, std::defer_lock);
            if (probe < (unsigned)Context_::NLANE ? lk.try_lock() : (lk.lock(), true))
            {
                lane = &l;
                lane_lk = std::move(lk);
                break;
            }
        }
        ctx_lk = std::unique_lock<std::mutex>(ctx->mu);
        if (!lane->ready)
        {
            lane->ready = true;
            dev_check(b200_stream_create(ctx->dev, &lane->stream));
            void *h = nullptr;
            dev_check(b200_malloc_host(sizeof(uint32_t) * Context_::COMBINE_MAX, &h));
            lane->hflag = (uint32_t *)h;
            h = nullptr;
            dev_check(b200_malloc_host(sizeof(u64 *) * 3 * Context_::COMBINE_MAX, &h));
            lane->hptrs = (u64 **)h;
        }
        tl_scope = this;
    }
    void *stream() const { return lane->stream; }
    // wait for everything this operation enqueued, without holding the context mutex
    void wait()
    {
        OpScope *root = this;
        while (root->outer && root->outer->c == c)
            root = root->outer;
        const bool held = root->ctx_lk.owns_lock();
        if (held)
            root->ctx_lk.unlock();
        int rc = blocking ? b200_stream_synchronize_blocking(c->dev, lane->stream, &lane->ev) : b200_stream_synchronize(c->dev, lane->stream);
        if (held)
            root->ctx_lk.lock();
        dev_check(rc);
    }
    ~OpScope()
    {
        tl_scope = outer;
        if (outer && outer->c == c)
            return;
        if (ctx_lk.owns_lock())
            ctx_lk.unlock();
        if (blocking)
            b200_stream_synchronize_blocking(c->dev, lane->stream, &lane->ev);
        else
            b200_stream_synchronize(c->dev, lane->stream); // the operation is complete when the call returns
    }
    OpScope(const OpScope &) = delete;
};
// stream of the Evaluator operation this thread is executing (the legacy default stream outside of one)
inline void *cur_stream() { return tl_scope ? tl_scope->stream() : nullptr; }

// Ciphertext: device-resident words with a lazily materialised host mirror.
struct Ciphertext_
{
    ParmsId parms_id = kZeroId;
    bool is_ntt_form = false;
    u64 size = 0, n = 0, k = 0;
    double scale = 1.0;
    u64 correction_factor = 1;
    Context_ *ctx = nullptr;          // context the device buffer belongs to (identity only: it may be gone already)
    std::shared_ptr<DevOwner> keep;   // ... and what keeps its device alive
    mutable std::vector<u64> host;
    mutable std::atomic<bool> host_valid{ true };
    mutable std::mutex mirror_mu; // the reference allows concurrent const reads: mirror materialisation is serialised
    u64 *dev = nullptr;
    size_t dev_words = 0;
    bool dev_valid = false;

    size_t words() const { return (size_t)(size * n * k); }
    ~Ciphertext_() { release_dev(); }
    void release_dev()
    {
        if (dev && keep && keep->dev)
        { // inside an operation the buffer may still be read by kernels enqueued on its stream: free in stream order
            if (tl_scope && tl_scope->c == ctx)
                b200_free_async(keep->dev, dev, tl_scope->stream());
            else
                b200_free(keep->dev, dev);
        }
        dev = nullptr;
        dev_words = 0;
        dev_valid = false;
    }
    void ensure_dev_capacity(Context_ *c)
    {
        if (ctx != c || dev_words < words() || !dev)
        {
            release_dev();
            ctx = c;
            keep = c->owner;
            void *p = nullptr;
            dev_check(b200_malloc(c->dev, std::max<size_t>(words(), 1) * sizeof(u64), &p));
            dev = (u64 *)p;
            dev_words = words();
        }
    }
    // make the device copy current (upload the host mirror if that is the valid one)
    const u64 *dev_ptr(Context_ *c)
    {
        if (!dev_valid || ctx != c)
        {
            if (!host_valid)
                sync_host();
            ensure_dev_capacity(c);
            if (words())
                dev_check(b200_memcpy_h2d(c->dev, dev, host.data(), words() * sizeof(u64), nullptr));
            dev_check(b200_stream_synchronize(c->dev, nullptr));
            dev_valid = true;
        }
        return dev;
    }
    void sync_host() const
    {
        if (host_valid.load(std::memory_order_acquire))
            return;
        std::lock_guard<std::mutex> lk(mirror_mu);
        if (host_valid.load(std::memory_order_relaxed))
            return;
        host.resize(words());
        if (words() && dev && keep)
        {
            dev_check(b200_memcpy_d2h(keep->dev, host.data(), dev, words() * sizeof(u64), nullptr));
            dev_check(b200_stream_synchronize(keep->dev, nullptr));
        }
        host_valid.store(true, std::memory_order_release);
    }
    // prepare as an output of shape (size, k) for context c; contents undefined, device copy becomes the valid one
    u64 *prepare_output(Context_ *c, const ParmsId &id, u64 new_size, u64 new_k)
    {
        parms_id = id;
        size = new_size;
        k = new_k;
        n = c->parms.n;
        is_ntt_form = false;
        scale = 1.0;
        correction_factor = 1;
        ensure_dev_capacity(c);
        dev_valid = true;
        host_valid = false;
        return dev;
    }
    void assign(const Ciphertext_ &o)
    {
        if (this == &o)
            return;
        o.sync_host();
        release_dev();
        parms_id = o.parms_id;
        is_ntt_form = o.is_ntt_form;
        size = o.size;
        n = o.n;
        k = o.k;
        scale = o.scale;
        correction_factor = o.correction_factor;
        ctx = o.ctx;
        host = o.host;
        host_valid = true;
    }
};

struct Plaintext_
{
    ParmsId parms_id = kZeroId;
    std::vector<u64> coeffs;
    double scale = 1.0;
};

// Secret material (secret-key residues, the sampled u / e, buffers derived from them) is zeroed before its memory goes back
// to the heap or the device pool — the reference keeps such data in clear-on-destruction pools (S/memorymanager.h, `clear_on_destruction`).
inline void wipe(std::vector<u64> &v)
{
    if (!v.empty())
        explicit_bzero(v.data(), v.size() * sizeof(u64));
}
struct WipeGuard
{
    std::vector<u64> &v;
    explicit WipeGuard(std::vector<u64> &x) : v(x) {}
    ~WipeGuard() { wipe(v); }
};
inline void wipe_dev_free(b200_ctx *dev, void *p, size_t bytes)
{
    if (!p || !dev)
        return;
    b200_memzero(dev, p, bytes, nullptr);
    b200_stream_synchronize(dev, nullptr);
    b200_free(dev, p);
}

struct PublicKey_ { Ciphertext_ data; };
struct SecretKey_ { Plaintext_ data; };

struct KSwitchKeys_
{
    ParmsId parms_id = kZeroId;
    std::vector<std::vector<PublicKey_ *>> keys; // owned
    // device cache of flattened key lists
    struct Flat { u64 *dev = nullptr; Context_ *ctx = nullptr; int count = 0; std::shared_ptr<DevOwner> keep; };
    std::vector<Flat> flat;
    ~KSwitchKeys_() { clear(); }
    void clear()
    {
        for (auto &l : keys)
            for (auto *p : l)
                delete p;
        keys.clear();
        drop_flat();
    }
    void drop_flat()
    {
        for (auto &f : flat)
            if (f.dev && f.keep && f.keep->dev)
                b200_free(f.keep->dev, f.dev);
        flat.clear();
    }
    // The cached buffer always holds EVERY component of the key list (the first level's decomposition count): a lower
    // level reads a prefix of it, so one key object can serve ciphertexts at any level in any order.
    const u64 *flat_dev(Context_ *c, size_t index, int decomp)
    {
        if (index >= keys.size() || keys[index].size() < (size_t)decomp)
            throw InvalidArg("kswitch_keys is not valid for encryption parameters");
        if (flat.size() <= index)
            flat.resize(index + 1);
        Flat &f = flat[index];
        if (f.dev && f.ctx == c && f.count >= decomp)
            return f.dev;
        if (f.dev && f.keep && f.keep->dev)
        {
            b200_free(f.keep->dev, f.dev);
            f.dev = nullptr;
        }
        const size_t K = c->parms.coeff.size(), n = c->parms.n;
        const size_t per = 2 * K * n;
        const int all = (int)keys[index].size();
        std::vector<u64> buf(per * all);
        for (int j = 0; j < all; j++)
        {
            Ciphertext_ &ct = keys[index][j]->data;
            ct.sync_host();
            if (ct.words() != per)
                throw InvalidArg("kswitch_keys is not valid for encryption parameters");
            std::memcpy(buf.data() + per * j, ct.host.data(), per * sizeof(u64));
        }
        void *p = nullptr;
        dev_check(b200_malloc(c->dev, buf.size() * sizeof(u64), &p));
        dev_check(b200_memcpy_h2d(c->dev, p, buf.data(), buf.size() * sizeof(u64), nullptr));
        dev_check(b200_stream_synchronize(c->dev, nullptr));
        f.dev = (u64 *)p;
        f.ctx = c;
        f.count = all;
        f.keep = c->owner;
        return f.dev;
    }
};


// PolynomialArray (S/polyarray.h:20-282): a stack of polynomials in RNS ([poly][residue][coeff]) or, after
// to_multiprecision, coefficient-major multi-precision form ([poly][coeff][word]).
struct PolynomialArray_
{
    std::vector<u64> moduli;
    size_t poly_size = 0, coeff_size = 0;
    std::vector<u64> data;
    std::vector<bool> filled;
    bool reserved = false, is_rns = true;
    size_t poly_len() const { return coeff_size * moduli.size(); }
    void reserve(size_t polys, size_t coeffs, const std::vector<u64> &base)
    {
        if (reserved)
            throw LogicErr("PolynomialArray can only be reserved once.");
        moduli = base;
        poly_size = polys;
        coeff_size = coeffs;
        data.assign(polys * poly_len(), 0);
        filled.assign(polys, false);
        reserved = true;
    }
    void insert(size_t index, const u64 *src)
    {
        if (index >= poly_size)
            throw LogicErr("Polynomial index greater than number of polynomials stored");
        if (filled[index])
            throw LogicErr("Attempted to overwrite a polynomial in PolynomialArray.");
        std::memcpy(data.data() + index * poly_len(), src, poly_len() * sizeof(u64));
        filled[index] = true;
    }
};

struct Evaluator_ { Context_ *ctx; CtxHold hold; };

struct BatchEncoder_
{
    Context_ *ctx;
    CtxHold hold;
    std::vector<size_t> index_map; // populate_matrix_reps_index_map (S/batchencoder.cpp:62-80)
};

struct Decryptor_
{
    Context_ *ctx;
    CtxHold hold;
    std::vector<u64> sk; // key level NTT form [K][n]
    // device cache: powers s^1..s^m packed per (level, terms)
    struct Pow { int level, terms; u64 *dev; size_t bytes; };
    std::vector<Pow> cache;
    std::shared_ptr<DevOwner> keep;
    ~Decryptor_();
    const u64 *powers(int level, int terms)
    {
        for (auto &p : cache)
            if (p.level == level && p.terms == terms)
                return p.dev;
        const size_t n = ctx->parms.n;
        const int k = ctx->level_k[level];
        std::vector<u64> buf((size_t)terms * k * n);
        WipeGuard wg(buf);
        for (int r = 0; r < k; r++)
        {
            const u64 q = ctx->parms.coeff[r];
            const u64 *s1 = sk.data() + (size_t)r * n;
            for (size_t c = 0; c < n; c++)
            {
                u64 cur = s1[c];
                for (int j = 0; j < terms; j++)
                {
                    buf[((size_t)j * k + r) * n + c] = cur;
                    cur = (u64)((unsigned __int128)cur * s1[c] % q);
                }
            }
        }
        void *p = nullptr;
        dev_check(b200_malloc(ctx->dev, buf.size() * sizeof(u64), &p));
        dev_check(b200_memcpy_h2d(ctx->dev, p, buf.data(), buf.size() * sizeof(u64), nullptr));
        dev_check(b200_stream_synchronize(ctx->dev, nullptr));
        keep = ctx->owner;
        cache.push_back({ level, terms, (u64 *)p, buf.size() * sizeof(u64) });
        return (u64 *)p;
    }
};

// ---- small device helpers for key generation / encryption (all arithmetic on the GPU through layer 1) ----
struct DevBuf
{
    Context_ *c;
    u64 *p = nullptr;
    size_t words;
    DevBuf(Context_ *ctx, size_t w) : c(ctx), words(w)
    {
        void *q = nullptr;
        dev_check(b200_malloc(c->dev, std::max<size_t>(w, 1) * 8, &q));
        p = (u64 *)q;
    }
    DevBuf(Context_ *ctx, const std::vector<u64> &h) : DevBuf(ctx, h.size()) { upload(h); }
    ~DevBuf()
    { // the E-row temporaries hold u, e and products with the secret key: always wiped
        b200_stream_synchronize(c->dev, nullptr);
        wipe_dev_free(c->dev, p, std::max<size_t>(words, 1) * 8);
    }
    void upload(const std::vector<u64> &h) { dev_check(b200_memcpy_h2d(c->dev, p, h.data(), h.size() * 8, nullptr)); }
    std::vector<u64> download()
    {
        std::vector<u64> h(words);
        dev_check(b200_memcpy_d2h(c->dev, h.data(), p, words * 8, nullptr));
        dev_check(b200_stream_synchronize(c->dev, nullptr));
        return h;
    }
    DevBuf(const DevBuf &) = delete;
};

// device-resident copies of key material (public key / secret key residues), created on first use, freed with their owner
struct DevCache
{
    std::shared_ptr<DevOwner> keep;
    std::vector<std::pair<int, u64 *>> bufs;
    std::vector<size_t> bytes;
    ~DevCache()
    {
        for (size_t i = 0; i < bufs.size(); i++)
            if (bufs[i].second && keep && keep->dev)
                wipe_dev_free(keep->dev, bufs[i].second, bytes[i]);
    }
    u64 *find(int key) const
    {
        for (auto &b : bufs)
            if (b.first == key)
                return b.second;
        return nullptr;
    }
    u64 *put(Context_ *c, int key, const std::vector<u64> &h)
    {
        void *p = nullptr;
        dev_check(b200_malloc(c->dev, std::max<size_t>(h.size(), 1) * sizeof(u64), &p));
        dev_check(b200_memcpy_h2d(c->dev, p, h.data(), h.size() * sizeof(u64), nullptr));
        dev_check(b200_stream_synchronize(c->dev, nullptr));
        keep = c->owner;
        bufs.emplace_back(key, (u64 *)p);
        bytes.push_back(std::max<size_t>(h.size(), 1) * sizeof(u64));
        return (u64 *)p;
    }
};

inline Decryptor_::~Decryptor_()
{
    for (auto &p : cache)
        if (p.dev && keep && keep->dev)
            wipe_dev_free(keep->dev, p.dev, p.bytes);
    wipe(sk);
}

// The samplers of sampling.h write one row per modulus; with this single zero "modulus" they return the small signed value
// itself (two's complement), which b200_expand_signed turns into residues on the device — n words cross PCIe instead of k n.
inline const std::vector<u64> &signed_only()
{
    static const std::vector<u64> z(1, 0);
    return z;
}
// host-side residues of such signed samples (only where the caller wants the components back: PolynomialArray)
inline std::vector<u64> expand_signed_host(const u64 *vals, size_t n, const std::vector<u64> &mods)
{
    std::vector<u64> out(mods.size() * n);
    for (size_t i = 0; i < mods.size(); i++)
        for (size_t c = 0; c < n; c++)
            out[i * n + c] = (int64_t)vals[c] < 0 ? vals[c] + mods[i] : vals[c];
    return out;
}

// encrypt_zero_symmetric at the key level, NTT form, no seed saving (S/util/rlwe.cpp:312-459): returns [2][K][n]
// c1 <- uniform (a fresh PRNG seeded from the bootstrap PRNG), c0 = -(s*c1 + e); dsk = the secret key on the device
inline std::vector<u64> encrypt_zero_symmetric_key_level(Context_ *c, const u64 *dsk, b200::Blake2xbPrng &bootstrap)
{
    const size_t n = c->parms.n, K = c->parms.coeff.size();
    b200::PrngSeed pub;
    bootstrap.generate(sizeof(pub), pub.data());
    b200::Blake2xbPrng ct_prng(pub);
    std::vector<u64> c1(K * n), noise(n);
    WipeGuard wg(noise);
    b200::sample_poly_uniform(ct_prng, n, c->parms.coeff, c1.data());
    b200::sample_poly_normal(bootstrap, n, signed_only(), noise.data());
    DevBuf d1(c, c1), dn(c, noise), de(c, K * n), d0(c, K * n);
    dev_check(b200_expand_signed(c->dev, 0, (const int64_t *)dn.p, 1, de.p, nullptr));
    dev_check(b200_dyadic_product(c->dev, 0, dsk, 1, d1.p, 1, d0.p, 1, nullptr)); // s (*) c1
    dev_check(b200_ntt_forward(c->dev, 0, de.p, 1, nullptr));                      // NTT(e)
    dev_check(b200_add(c->dev, 0, d0.p, de.p, d0.p, 1, 1, nullptr));
    dev_check(b200_negate(c->dev, 0, d0.p, d0.p, 1, 1, nullptr));
    std::vector<u64> out = d0.download();
    out.insert(out.end(), c1.begin(), c1.end());
    return out;
}

struct KeyGenerator_
{
    Context_ *ctx;
    CtxHold hold;
    std::vector<u64> sk; // key level, NTT form [K][n]
    DevCache dev_cache;
    ~KeyGenerator_() { wipe(sk); }
    const u64 *dev_sk()
    {
        u64 *p = dev_cache.find(0);
        return p ? p : dev_cache.put(ctx, 0, sk);
    }
    // generate_one_kswitch_key (S/keygenerator.cpp:303-337): new_key = [K][n] NTT form
    void one_kswitch_key(const std::vector<u64> &new_key, std::vector<PublicKey_ *> &dest)
    {
        Context_ *c = ctx;
        const size_t n = c->parms.n, K = c->parms.coeff.size();
        const int decomp = c->level_k[c->first_level];
        const u64 qsp = c->parms.coeff.back();
        b200::Blake2xbPrng bootstrap(b200::random_seed());
        for (int J = 0; J < decomp; J++)
        {
            std::vector<u64> w = encrypt_zero_symmetric_key_level(c, dev_sk(), bootstrap);
            const u64 qj = c->parms.coeff[J];
            const u64 factor = qsp % qj;
            const u64 factor_q = (u64)(((unsigned __int128)factor << 64) / qj); // Shoup quotient: no division per word
            for (size_t i = 0; i < n; i++)
            { // c0[J] += factor * new_key[J]  (S/keygenerator.cpp:330-334); all operands canonical
                const u64 nk = new_key[(size_t)J * n + i];
                u64 t = nk * factor - (u64)(((unsigned __int128)nk * factor_q) >> 64) * qj;
                t = t >= qj ? t - qj : t;
                u64 &d = w[(size_t)J * n + i];
                const u64 s = d + t;
                d = s >= qj ? s - qj : s;
            }
            auto *pk = new PublicKey_();
            pk->data.parms_id = c->ids[0];
            pk->data.size = 2;
            pk->data.k = K;
            pk->data.n = n;
            pk->data.is_ntt_form = true;
            pk->data.host = std::move(w);
            pk->data.host_valid = true;
            dest.push_back(pk);
        }
    }
};

struct Encryptor_
{
    Context_ *ctx;
    CtxHold hold;
    bool has_pk = false, has_sk = false;
    std::vector<u64> pk; // [2][K][n] NTT form, key level
    std::vector<u64> sk; // [K][n]
    ~Encryptor_() { wipe(sk); }
    DevCache dev_cache;  // key 0: secret key [K][n]; key 1 + level: the level's residues of both public-key polynomials
    const u64 *dev_sk()
    {
        u64 *p = dev_cache.find(0);
        return p ? p : dev_cache.put(ctx, 0, sk);
    }
    const u64 *dev_pk(int level)
    {
        if (u64 *p = dev_cache.find(1 + level))
            return p;
        const size_t n = ctx->parms.n, K = ctx->parms.coeff.size(), ke = (size_t)ctx->level_k[level];
        std::vector<u64> part(2 * ke * n);
        for (int j = 0; j < 2; j++)
            std::copy_n(pk.begin() + (size_t)j * K * n, ke * n, part.begin() + (size_t)j * ke * n);
        return dev_cache.put(ctx, 1 + level, part);
    }
};

template <class F>
long guard(F f)
{
    try
    {
        f();
        return S_OK_;
    }
    catch (const InvalidArg &)
    {
        return E_INVALIDARG_;
    }
    catch (const std::invalid_argument &)
    {
        return E_INVALIDARG_;
    }
    catch (const LogicErr &)
    {
        return COR_E_INVALIDOPERATION_;
    }
    catch (const std::logic_error &)
    {
        return COR_E_INVALIDOPERATION_;
    }
    catch (const std::bad_alloc &)
    {
        return E_OUTOFMEMORY_;
    }
    catch (...)
    {
        return E_UNEXPECTED_;
    }
}

#define NULLRET_THROW(p)                                                                                               \
    if (!(p))                                                                                                          \
    throw InvalidArg("null handle in batch")
#define NULLRET(p)                                                                                                     \
    if (!(p))                                                                                                          \
    return E_POINTER_

} // namespace b200c
