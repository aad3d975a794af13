// sealc_api.cpp — layer-2 C ABI (include/b200_sealc.h): SEAL's C export names over the B200 backend.
//
// Mirrors the behaviour (argument meaning, ownership, HRESULTs, validation order) of the reference's C export
// layer S/c/*.cpp and of the C++ methods it forwards to, for the BFV path that seal_fhe uses:
//   Evaluator_*      S/c/evaluator.cpp:31-700  -> S/evaluator.cpp (negate/add/sub/multiply/square/relinearize/
//                    mod_switch/multiply_plain/add_plain/sub_plain/apply_galois/rotate)
//   Ciphertext_*     S/c/ciphertext.cpp        -> S/ciphertext.h:337-715
//   KSwitchKeys_*    S/c/kswitchkeys.cpp       -> S/kswitchkeys.h:340
//   SEALContext_*    S/c/sealcontext.cpp       -> S/context.cpp:135-522
// No arithmetic happens here: every operation is a call into the layer-1 functions of b200_bfv.cu.
#include "../../include/b200_bfv.h"
#include "../../include/b200_sealc.h"
#include "host_ctx.h"
#include "sampling.h"
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <vector>

namespace
{
} // namespace
#include "sealc_types.h"
namespace
{
using namespace b200c;

// is_metadata_valid_for (S/valcheck.cpp:67-112): known data-level parms_id, matching shape
int data_level(Context_ *c, const Ciphertext_ &ct, const char *what)
{
    int lv = c->level_of(ct.parms_id);
    if (lv < 0 || (lv == 0 && c->first_level == 1) || ct.n != c->parms.n || ct.k != (u64)c->level_k[lv] || ct.size < 2 || ct.size > 16)
        throw InvalidArg(what);
    return lv;
}
// the level of a batch's items, which must be valid size-2 ciphertexts, not in NTT form, all at one level
int batch_level(Context_ *c, uint64_t count, void **cts)
{
    const int lv = data_level(c, *(Ciphertext_ *)cts[0], "encrypted is not valid for encryption parameters");
    for (uint64_t i = 0; i < count; i++)
    {
        auto &a = *(Ciphertext_ *)cts[i];
        if (data_level(c, a, "encrypted is not valid for encryption parameters") != lv || a.size != 2 || a.is_ntt_form)
            throw InvalidArg("batch items must be size-2 ciphertexts at the same level");
    }
    return lv;
}

void transparent_guard(Context_ *c, int level, Ciphertext_ &dst)
{
    OpScope *sc = tl_scope;
    if (!sc || sc->c != c)
        throw std::logic_error("internal: transparent_guard outside an operation scope");
    if (!c->check_transparent)
    {
        sc->wait();
        return;
    }
    // SEAL_THROW_ON_TRANSPARENT_CIPHERTEXT (seal_fhe/build.rs:37-42): "result ciphertext is transparent"
    // one kernel, writing "a nonzero word exists" straight into the lane's pinned flag
    *(volatile uint32_t *)sc->lane->hflag = 0;
    dev_check(b200_any_nonzero(c->dev, level, dst.dev, (int)dst.size, sc->lane->hflag, 1, sc->stream()));
    sc->wait(); // context mutex released while the GPU finishes this operation
    if (!*(volatile uint32_t *)sc->lane->hflag)
        throw LogicErr("result ciphertext is transparent");
}

// run `body(dst_ptr)` writing to `dst`; when dst aliases an input, go through a temporary
template <class F>
void with_output(Context_ *c, Ciphertext_ &dst, std::initializer_list<const Ciphertext_ *> inputs, const ParmsId &id, u64 size,
                 u64 k, F body)
{
    bool alias = false;
    for (auto *in : inputs)
        alias = alias || in == &dst;
    if (!alias)
    {
        body(dst.prepare_output(c, id, size, k));
        return;
    }
    Ciphertext_ tmp;
    body(tmp.prepare_output(c, id, size, k));
    // move tmp's buffer into dst
    dst.release_dev();
    dst.parms_id = id;
    dst.size = size;
    dst.k = k;
    dst.n = c->parms.n;
    dst.is_ntt_form = false;
    dst.scale = 1.0;
    dst.ctx = c;
    dst.keep = tmp.keep;
    dst.dev = tmp.dev;
    dst.dev_words = tmp.dev_words;
    dst.dev_valid = true;
    dst.host_valid = false;
    tmp.dev = nullptr;
    tmp.dev_words = 0;
}

void check_same(const Ciphertext_ &a, const Ciphertext_ &b)
{
    if (a.parms_id != b.parms_id)
        throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
    if (a.is_ntt_form != b.is_ntt_form)
        throw InvalidArg("NTT form mismatch");
    if (a.scale != b.scale)
        throw InvalidArg("scale mismatch");
}

void op_addsub(Context_ *c, Ciphertext_ &a, Ciphertext_ &b, Ciphertext_ &dst, int mode)
{
    OpScope scope(c);
    int lv = data_level(c, a, "encrypted1 is not valid for encryption parameters");
    data_level(c, b, "encrypted2 is not valid for encryption parameters");
    check_same(a, b);
    const u64 k = a.k, n = a.n;
    const u64 mx = std::max(a.size, b.size), mn = std::min(a.size, b.size);
    const u64 *pa = a.dev_ptr(c), *pb = b.dev_ptr(c);
    with_output(c, dst, { &a, &b }, a.parms_id, mx, k, [&](u64 *out) {
        dev_check((mode == 0 ? b200_add : b200_sub)(c->dev, lv, pa, pb, out, (int)mn, 1, cur_stream()));
        if (a.size > mn) // tail polys copied from the larger operand
            dev_check(b200_memcpy_d2d(c->dev, out + mn * k * n, pa + mn * k * n, (a.size - mn) * k * n * sizeof(u64), cur_stream()));
        else if (b.size > mn)
        {
            if (mode == 0)
                dev_check(b200_memcpy_d2d(c->dev, out + mn * k * n, pb + mn * k * n, (b.size - mn) * k * n * sizeof(u64), cur_stream()));
            else
                dev_check(b200_negate(c->dev, lv, pb + mn * k * n, out + mn * k * n, (int)(b.size - mn), 1, cur_stream()));
        }
    });
    dst.is_ntt_form = a.is_ntt_form;
    transparent_guard(c, lv, dst);
}

// ---------------------------------------------------------------------------------------------------------
// Flat combining (Context_::Combiner).  A caller validates its own arguments, then submits a request.  If nobody holds the
// combiner it becomes the leader: it repeatedly takes the compatible requests that are pending (its own included), runs
// them as ONE batch through the layer-1 batch entry points (gather -> compute -> scatter, one transparent-result check for
// all items), marks them done and wakes their owners; requests that arrive meanwhile form the next batch.  A batch of one
// runs the direct per-handle path (no gather / scatter).  Every call still completes before it returns and reports its
// own error (an item whose result is transparent fails alone).
// ---------------------------------------------------------------------------------------------------------
using CombineReq = Context_::CombineReq;

void multiply_direct(Context_ *c, Ciphertext_ &a, Ciphertext_ &b, Ciphertext_ &dst, bool square, int lv);
void relinearize_direct(Context_ *c, Ciphertext_ &a, KSwitchKeys_ &keys, Ciphertext_ &dst, int lv);
void op_galois(Context_ *c, Ciphertext_ &a, uint32_t elt, KSwitchKeys_ &keys, Ciphertext_ &dst);

static void combine_run_one(Context_ *c, CombineReq &r)
{
    try
    {
        if (r.kind == 0)
            multiply_direct(c, *r.a, *r.b, *r.dst, false, r.lv);
        else if (r.kind == 1)
            relinearize_direct(c, *r.a, *r.keys, *r.dst, r.lv);
        else
        {
            OpScope scope(c);
            op_galois(c, *r.a, r.elt, *r.keys, *r.dst);
        }
    }
    catch (...)
    {
        r.err = std::current_exception();
    }
}

static void combine_run_batch(Context_ *c, std::vector<CombineReq *> &batch)
{
    const size_t N = batch.size();
    if (N == 1 && !c->use_graphs)
    {
        c->graph_stats[Context_::GS_NO_GRAPH]++;
        return combine_run_one(c, *batch[0]);
    }
    CombineReq &r0 = *batch[0];
    try
    {
        OpScope scope(c);
        Context_::Lane &lane = *scope.lane;
        const int lv = r0.lv;
        const u64 k = (u64)c->level_k[lv], n = c->parms.n;
        const u64 in_polys = r0.kind == 1 ? 3 : 2, out_polys = r0.kind == 0 ? 3 : 2;
        const u64 win = in_polys * k * n, wout = out_polys * k * n;
        const size_t operands = r0.kind == 0 ? 2 : 1;
        // An upload may reallocate an operand's device buffer, whose size the alias test below reads: every operand's device
        // copy is made current first.
        for (auto *r : batch)
        {
            r->a->dev_ptr(c);
            if (operands == 2)
                r->b->dev_ptr(c);
        }
        // the gather must read an aliased operand before prepare_output may release its buffer: when a destination is also
        // an operand of DIFFERENT shape, fall back to the order gather -> prepare (no graph for that rare batch)
        bool reshaped_alias = false;
        for (size_t i = 0; i < N && !reshaped_alias; i++)
            for (size_t j = 0; j < N; j++)
                if ((batch[i]->dst == batch[j]->a || batch[i]->dst == batch[j]->b) && batch[i]->dst->dev_words < wout)
                    reshaped_alias = true;
        const bool graphs = c->use_graphs && !reshaped_alias;
        // With graphs the batch is padded to a power of two (the pad items repeat item 0 and write to a scratch destination):
        // far fewer distinct graph shapes per lane, at the price of a few wasted items in a latency-bound launch sequence.
        size_t count = N;
        if (graphs)
            for (count = 1; count < N; count <<= 1)
                ;
        // Everything that varies from call to call goes through the lane's pinned tables (addresses fixed for the lane's
        // lifetime, read directly by the kernels): operand pointers, destination pointers, transparent-result flags.
        u64 **tab = lane.hptrs, **dtab = tab + 2 * Context_::COMBINE_MAX;
        uint32_t *flags = lane.hflag;
        for (size_t i = 0; i < count; i++)
        {
            const size_t src = i < N ? i : 0;
            tab[i] = const_cast<u64 *>(batch[src]->a->dev_ptr(c));
            if (operands == 2)
                tab[count + i] = const_cast<u64 *>(batch[src]->b->dev_ptr(c));
        }
        if (count > N && lane.pad_words < wout)
        {
            if (lane.pad_out)
                b200_free_async(c->dev, lane.pad_out, cur_stream());
            void *pp = nullptr;
            dev_check(b200_malloc(c->dev, wout * sizeof(u64), &pp));
            lane.pad_out = (u64 *)pp;
            lane.pad_words = wout;
        }
        // destinations are only written by the final scatter, after every operand has been gathered: aliasing is harmless.
        // An operand that IS a destination keeps its buffer (prepare_output reuses it when the capacity suffices); when the
        // shapes differ the old buffer is released in stream order, after the gather that reads it.
        const u64 *key = r0.kind == 0 ? nullptr : r0.keys->flat_dev(c, r0.kind == 1 ? 0 : r0.key_index, (int)k);
        auto prepare = [&] {
            for (size_t i = 0; i < count; i++)
                dtab[i] = i < N ? batch[i]->dst->prepare_output(c, c->ids[lv], out_polys, k) : lane.pad_out;
        };
        // The launch sequence of the batch: allocate -> gather -> layer-1 call -> `place()` -> scatter -> transparent flags.
        // Its two slabs are freed in stream order on every exit.  Only `place` may throw: inside a stream capture, which must
        // always be ended, it does nothing.
        auto sequence = [&](auto place) -> int {
            struct Slabs
            {
                Context_ *c;
                void *in = nullptr, *out = nullptr;
                ~Slabs()
                {
                    if (in)
                        b200_free_async(c->dev, in, cur_stream());
                    if (out)
                        b200_free_async(c->dev, out, cur_stream());
                }
            } s{ c };
            int rc = b200_malloc_async(c->dev, operands * count * win * sizeof(u64), &s.in, cur_stream());
            if (!rc)
                rc = b200_malloc_async(c->dev, count * wout * sizeof(u64), &s.out, cur_stream());
            if (rc)
                return rc;
            u64 *in = (u64 *)s.in, *out = (u64 *)s.out;
            rc = b200_gather_scatter_table(c->dev, tab, operands * count, in, win, 1, cur_stream());
            if (!rc)
                rc = r0.kind == 0   ? b200_multiply(c->dev, lv, in, 2, in + count * win, 2, out, count, cur_stream())
                     : r0.kind == 1 ? b200_relinearize(c->dev, lv, in, key, out, count, cur_stream())
                                    : b200_apply_galois(c->dev, lv, in, r0.elt, key, out, count, cur_stream());
            place();
            if (!rc)
                rc = b200_gather_scatter_table(c->dev, dtab, count, out, wout, 0, cur_stream());
            if (!rc && c->check_transparent)
                rc = b200_any_nonzero(c->dev, lv, out, (int)out_polys, flags, count, cur_stream());
            return rc;
        };
        auto enqueue = [&] { return sequence([] {}); };
        if (c->check_transparent)
            for (size_t i = 0; i < count; i++)
                ((volatile uint32_t *)flags)[i] = 0;
        if (!graphs)
        {
            c->graph_stats[Context_::GS_NO_GRAPH]++;
            dev_check(sequence(prepare)); // prepared after the layer-1 call: an aliased operand is gathered before its release
        }
        else
        {
            prepare();
            Context_::Lane::Graph *g = nullptr;
            for (auto &e : lane.graphs)
                if ((e.kind == r0.kind || e.kind == -1 - r0.kind) && e.lv == lv && e.n == count && e.key == (const void *)key && e.elt == r0.elt)
                    g = &e;
            if (!g)
            { // first sight of this shape on this lane: run it kernel by kernel (this also warms every cache the sequence touches)
                c->graph_stats[Context_::GS_FIRST]++;
                if ((int)lane.graphs.size() >= Context_::GRAPHS_PER_LANE)
                {
                    c->graph_stats[Context_::GS_EVICT]++;
                    size_t old = 0;
                    for (size_t i = 1; i < lane.graphs.size(); i++)
                        if (lane.graphs[i].stamp < lane.graphs[old].stamp)
                            old = i;
                    if (lane.graphs[old].exec)
                        b200_graph_destroy(c->dev, lane.graphs[old].exec);
                    lane.graphs.erase(lane.graphs.begin() + (long)old);
                }
                lane.graphs.push_back({ r0.kind, lv, count, (const void *)key, nullptr, ++lane.clock, r0.elt });
                dev_check(enqueue());
            }
            else
            {
                g->stamp = ++lane.clock;
                if (g->exec)
                    c->graph_stats[Context_::GS_REPLAY]++;
                else if (g->kind < 0)
                    c->graph_stats[Context_::GS_NO_GRAPH]++;
                else
                { // second use: capture the sequence; from now on one graph launch replaces its ~10 kernel launches
                    if (b200_capture_begin(c->dev, cur_stream()) == 0)
                    {
                        const int rc = enqueue();
                        void *exec = nullptr;
                        const int rc2 = b200_capture_end(c->dev, cur_stream(), &exec);
                        if (rc || rc2)
                        { // not capturable here: this shape keeps the kernel-by-kernel path (nothing was executed yet)
                            if (exec)
                                b200_graph_destroy(c->dev, exec);
                            exec = nullptr;
                            g->kind = -1 - r0.kind;
                        }
                        g->exec = exec;
                    }
                    c->graph_stats[g->exec ? Context_::GS_CAPTURE : Context_::GS_REFUSED]++;
                }
                if (g->exec)
                    dev_check(b200_graph_launch(c->dev, g->exec, cur_stream()));
                else
                    dev_check(enqueue());
            }
        }
        scope.wait();
        if (c->check_transparent)
            for (size_t i = 0; i < N; i++)
                if (!((volatile uint32_t *)flags)[i])
                    batch[i]->err = std::make_exception_ptr(LogicErr("result ciphertext is transparent"));
    }
    catch (...)
    {
        for (auto *r : batch)
            if (!r->err)
                r->err = std::current_exception();
    }
}

// B200_Evaluator_CombinedBatchDebug: the requests its items' validation would submit are collected here instead
static thread_local std::vector<CombineReq> *tl_collect = nullptr;

static void combine_submit(Context_ *c, CombineReq &req)
{
    if (tl_collect)
        return tl_collect->push_back(req);
    Context_::Combiner &cb = c->comb[req.kind];
    std::unique_lock<std::mutex> lk(cb.m);
    cb.pending.push_back(&req);
    bool mine_pending = true; // still in cb.pending (nobody has taken it yet)
    while (!req.done)
    {
        if (mine_pending)
            mine_pending = std::find(cb.pending.begin(), cb.pending.end(), &req) != cb.pending.end();
        if (!mine_pending || cb.active >= c->combine_leaders)
        { // in flight with another leader, or all leaders busy: requests pile up and leave together with the next free leader
            cb.cv.wait(lk);
            continue;
        }
        // lead: my request and every compatible one that is waiting, as one batch, on a lane of its own
        cb.active++;
        std::vector<CombineReq *> batch{ &req }, rest;
        for (auto *r : cb.pending)
        {
            if (r == &req)
                continue;
            if ((int)batch.size() < Context_::COMBINE_MAX && r->compatible(req))
                batch.push_back(r);
            else
                rest.push_back(r);
        }
        cb.pending.swap(rest);
        lk.unlock();
        combine_run_batch(c, batch);
        lk.lock();
        for (auto *r : batch)
            r->done = true;
        cb.active--;
        cb.cv.notify_all();
    }
    lk.unlock();
    if (req.err)
        std::rethrow_exception(req.err);
}

void op_multiply(Context_ *c, Ciphertext_ &a, Ciphertext_ &b, Ciphertext_ &dst, bool square)
{
    int lv = data_level(c, a, "encrypted1 is not valid for encryption parameters");
    if (!square)
    {
        data_level(c, b, "encrypted2 is not valid for encryption parameters");
        if (a.parms_id != b.parms_id)
            throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
    }
    if (a.is_ntt_form || (!square && b.is_ntt_form))
        throw InvalidArg("encrypted1 or encrypted2 cannot be in NTT form");
    if (c->combine && !square && a.size == 2 && b.size == 2 && !tl_scope)
    {
        CombineReq r;
        r.kind = 0;
        r.a = &a;
        r.b = &b;
        r.dst = &dst;
        r.lv = lv;
        return combine_submit(c, r);
    }
    multiply_direct(c, a, b, dst, square, lv);
}

void multiply_direct(Context_ *c, Ciphertext_ &a, Ciphertext_ &b, Ciphertext_ &dst, bool square, int lv)
{
    OpScope scope(c);
    const u64 k = a.k;
    const u64 *pa = a.dev_ptr(c), *pb = square ? pa : b.dev_ptr(c);
    if (square && a.size != 2)
    { // the reference falls back to multiply for sizes other than 2 (S/evaluator.cpp:880-884)
        square = false;
        pb = pa;
    }
    const u64 sb = square ? a.size : (&a == &b ? a.size : b.size);
    const u64 ds = square ? 3 : a.size + sb - 1;
    if (ds > 16)
        throw InvalidArg("invalid size"); // Ciphertext::resize_internal, SEAL_CIPHERTEXT_SIZE_MAX (S/ciphertext.cpp:100-106)
    with_output(c, dst, { &a, &b }, a.parms_id, ds, k, [&](u64 *out) {
        if (square)
            dev_check(b200_square(c->dev, lv, pa, out, 1, cur_stream()));
        else
            dev_check(b200_multiply(c->dev, lv, pa, (int)a.size, pb, (int)sb, out, 1, cur_stream()));
    });
    transparent_guard(c, lv, dst);
}

void check_keys(Context_ *c, KSwitchKeys_ &keys, size_t index)
{
    if (!c->using_keyswitching)
        throw LogicErr("keyswitching is not supported by the context");
    if (keys.parms_id != c->ids[0])
        throw InvalidArg("parameter mismatch");
    if (index >= keys.keys.size() || keys.keys[index].empty())
        throw InvalidArg("key not present");
}

void op_relinearize(Context_ *c, Ciphertext_ &a, KSwitchKeys_ &keys, Ciphertext_ &dst)
{
    int lv = data_level(c, a, "encrypted is not valid for encryption parameters");
    if (keys.parms_id != c->ids[0])
        throw InvalidArg("relin_keys is not valid for encryption parameters");
    if (a.is_ntt_form)
        throw InvalidArg("BFV encrypted cannot be in NTT form");
    if (a.size == 2)
    { // nothing to do (S/evaluator.cpp:1131-1135)
        OpScope scope(c);
        dst.assign(a);
        return;
    }
    if (keys.keys.size() < a.size - 2)
        throw InvalidArg("not enough relinearization keys");
    if (c->combine && a.size == 3 && !tl_scope)
    {
        check_keys(c, keys, 0);
        if (keys.keys[0].size() < (size_t)a.k)
            throw InvalidArg("kswitch_keys is not valid for encryption parameters");
        CombineReq r;
        r.kind = 1;
        r.a = &a;
        r.dst = &dst;
        r.keys = &keys;
        r.lv = lv;
        return combine_submit(c, r);
    }
    relinearize_direct(c, a, keys, dst, lv);
}

void relinearize_direct(Context_ *c, Ciphertext_ &a, KSwitchKeys_ &keys, Ciphertext_ &dst, int lv)
{
    OpScope scope(c);
    const u64 k = a.k, n = a.n;
    const u64 *pa = a.dev_ptr(c);
    with_output(c, dst, { &a }, a.parms_id, 2, k, [&](u64 *out) {
        if (a.size == 3)
        {
            check_keys(c, keys, 0);
            const u64 *key = keys.flat_dev(c, 0, (int)k);
            dev_check(b200_relinearize(c->dev, lv, pa, key, out, 1, cur_stream()));
            return;
        }
        // size > 3: peel polynomials from the top, key index = power - 2 (S/evaluator.cpp:1143-1151)
        void *tmp = nullptr;
        dev_check(b200_malloc(c->dev, 3 * k * n * sizeof(u64), &tmp));
        u64 *t3 = (u64 *)tmp;
        dev_check(b200_memcpy_d2d(c->dev, out, pa, 2 * k * n * sizeof(u64), cur_stream()));
        int rc = 0;
        for (u64 s = a.size - 1; s >= 2 && !rc; s--)
        {
            check_keys(c, keys, s - 2);
            const u64 *key = keys.flat_dev(c, s - 2, (int)k);
            rc = b200_memcpy_d2d(c->dev, t3, out, 2 * k * n * sizeof(u64), cur_stream());
            if (!rc)
                rc = b200_memcpy_d2d(c->dev, t3 + 2 * k * n, pa + s * k * n, k * n * sizeof(u64), cur_stream());
            if (!rc)
                rc = b200_relinearize(c->dev, lv, t3, key, out, 1, cur_stream());
        }
        b200_stream_synchronize(c->dev, cur_stream());
        b200_free(c->dev, tmp);
        dev_check(rc);
    });
    transparent_guard(c, lv, dst);
}

bool has_galois_key(const KSwitchKeys_ &keys, uint32_t elt)
{
    const size_t idx = (elt - 1) >> 1;
    return idx < keys.keys.size() && !keys.keys[idx].empty();
}
// the key list's index of Galois element `elt`, whose key must be present
size_t galois_key_index(Context_ *c, KSwitchKeys_ &keys, uint32_t elt)
{
    if (!has_galois_key(keys, elt))
        throw InvalidArg("Galois key not present");
    const size_t idx = (elt - 1) >> 1;
    check_keys(c, keys, idx);
    return idx;
}
// the Galois element of a row rotation by `step`
uint32_t row_step_elt(Context_ *c, int step)
{
    uint32_t elt = 0;
    if (b200_galois_elt_from_step(c->dev, step, &elt))
        throw InvalidArg("step count too large");
    return elt;
}

// the checks of apply_galois (S/evaluator.cpp), in its order: returns the level of `a` and the key list's index of `elt`
std::pair<int, size_t> galois_checks(Context_ *c, Ciphertext_ &a, uint32_t elt, KSwitchKeys_ &keys)
{
    const int lv = data_level(c, a, "encrypted is not valid for encryption parameters");
    if (keys.parms_id != c->ids[0])
        throw InvalidArg("galois_keys is not valid for encryption parameters");
    if (!(elt & 1) || elt >= 2 * c->parms.n)
        throw InvalidArg("Galois element is not valid");
    if (a.size > 2)
        throw InvalidArg("encrypted size must be 2");
    return { lv, galois_key_index(c, keys, elt) };
}

void op_galois(Context_ *c, Ciphertext_ &a, uint32_t elt, KSwitchKeys_ &keys, Ciphertext_ &dst)
{
    // caller holds c->mu
    int lv;
    size_t index;
    std::tie(lv, index) = galois_checks(c, a, elt, keys);
    const u64 *pa = a.dev_ptr(c);
    const u64 *key = keys.flat_dev(c, index, (int)a.k);
    with_output(c, dst, { &a }, a.parms_id, 2, a.k, [&](u64 *out) {
        dev_check(b200_apply_galois(c->dev, lv, pa, elt, key, out, 1, cur_stream()));
    });
    transparent_guard(c, lv, dst);
}

// naf of an integer (S/util/numth.h: naf) — signed powers of two, least significant first
std::vector<int> naf(int value)
{
    std::vector<int> res;
    bool sign = value < 0;
    value = std::abs(value);
    for (int i = 0; value; i++)
    {
        int zi = (value & 1) ? 2 - (value & 3) : 0;
        value = (value - zi) >> 1;
        if (zi)
            res.push_back((sign ? -zi : zi) * (1 << i));
    }
    return res;
}

// The Galois elements rotate_internal (S/evaluator.cpp:2325-2380) applies for a row rotation by `steps` != 0: the step's own
// when its key is present, else those of its NAF parts, skipping the parts of +-n/2 (the identity on rows).  No part's
// magnitude exceeds n/2, so every remaining part has an element.
std::vector<uint32_t> row_rotation_elts(Context_ *c, const KSwitchKeys_ &keys, int steps)
{
    const uint32_t elt = row_step_elt(c, steps);
    if (has_galois_key(keys, elt))
        return { elt };
    const std::vector<int> parts = naf(steps);
    if (parts.size() == 1)
        throw InvalidArg("Galois key not present");
    std::vector<uint32_t> elts;
    for (int st : parts)
        if ((size_t)std::abs(st) != (c->parms.n >> 1))
            elts.push_back(row_step_elt(c, st));
    return elts;
}

// One application of a Galois automorphism whose key is present, through the combiner (same checks, same errors as op_galois);
// false: not combinable here (combining off, nested call) — the caller takes the direct path.
bool galois_combined(Context_ *c, Ciphertext_ &a, uint32_t elt, KSwitchKeys_ &keys, Ciphertext_ &dst)
{
    if (!c->combine || tl_scope)
        return false;
    int lv;
    size_t index;
    std::tie(lv, index) = galois_checks(c, a, elt, keys);
    if (keys.keys[index].size() < (size_t)a.k || a.is_ntt_form)
        return false; // let the direct path report it
    CombineReq r;
    r.kind = 2;
    r.a = &a;
    r.dst = &dst;
    r.keys = &keys;
    r.key_index = index;
    r.elt = elt;
    r.lv = lv;
    combine_submit(c, r);
    return true;
}

void op_rotate(Context_ *c, Ciphertext_ &a, int steps, KSwitchKeys_ &keys, Ciphertext_ &dst)
{
    // rotate_internal (S/evaluator.cpp:2325-2380)
    if (!c->using_batching)
        throw LogicErr("encryption parameters do not support batching");
    if (keys.parms_id != c->ids[0])
        throw InvalidArg("galois_keys is not valid for encryption parameters");
    if (steps == 0)
    {
        dst.assign(a);
        return;
    }
    // A plan of one element applies the step's own element: the NAF {x, +-n/2} rotates by x, whose element is the step's.
    const std::vector<uint32_t> elts = row_rotation_elts(c, keys, steps);
    if (elts.size() == 1)
    {
        op_galois(c, a, elts[0], keys, dst);
        return;
    }
    Ciphertext_ cur;
    cur.assign(a);
    for (uint32_t e : elts)
    {
        Ciphertext_ nxt;
        op_galois(c, cur, e, keys, nxt);
        cur.assign(nxt);
    }
    dst.assign(cur);
}

// Plaintext operand padded to n coefficients.  `check_values` mirrors WHICH reference entry points look at the
// coefficients: Encryptor::encrypt and BatchEncoder::decode call is_valid_for (metadata + every coefficient < t,
// S/valcheck.cpp:246-294), the Evaluator's plain operations only is_metadata_valid_for + is_buffer_valid
// (S/evaluator.cpp:1645-1660,1858-1870) and then compute with whatever 64-bit words they are given.
std::vector<u64> padded_plain(Context_ *c, const Plaintext_ &p, bool check_values = true)
{
    if (p.parms_id != kZeroId)
        throw InvalidArg("plain is not valid for encryption parameters");
    if (p.coeffs.size() > c->parms.n)
        throw InvalidArg("plain is not valid for encryption parameters");
    std::vector<u64> v(c->parms.n, 0);
    for (size_t i = 0; i < p.coeffs.size(); i++)
    {
        if (check_values && p.coeffs[i] >= c->parms.plain)
            throw InvalidArg("plain is not valid for encryption parameters");
        v[i] = p.coeffs[i];
    }
    return v;
}

// The plaintext operand of an Evaluator operation, padded to n coefficients; multiplying by zero gives a transparent result
std::vector<u64> plain_operand(Context_ *c, const Plaintext_ &p, bool multiply)
{
    std::vector<u64> v = padded_plain(c, p, false);
    if (multiply && c->check_transparent && std::all_of(v.begin(), v.end(), [](u64 x) { return x == 0; }))
        throw LogicErr("result ciphertext is transparent");
    return v;
}

void op_plain(Context_ *c, Ciphertext_ &a, const Plaintext_ &p, Ciphertext_ &dst, int which /*0 add 1 sub 2 mul*/)
{
    OpScope scope(c);
    int lv = data_level(c, a, "encrypted is not valid for encryption parameters");
    if (a.is_ntt_form)
        throw InvalidArg("BFV encrypted cannot be in NTT form");
    std::vector<u64> pv = plain_operand(c, p, which == 2);
    void *dp = nullptr;
    dev_check(b200_malloc(c->dev, pv.size() * sizeof(u64), &dp));
    int rc = b200_memcpy_h2d(c->dev, dp, pv.data(), pv.size() * sizeof(u64), cur_stream());
    const u64 *pa = a.dev_ptr(c);
    try
    {
        dev_check(rc);
        with_output(c, dst, { &a }, a.parms_id, a.size, a.k, [&](u64 *out) {
            if (which == 0)
                dev_check(b200_add_plain(c->dev, lv, pa, (int)a.size, (const u64 *)dp, 1, out, 1, cur_stream()));
            else if (which == 1)
                dev_check(b200_sub_plain(c->dev, lv, pa, (int)a.size, (const u64 *)dp, 1, out, 1, cur_stream()));
            else
                dev_check(b200_multiply_plain(c->dev, lv, pa, (int)a.size, (const u64 *)dp, 1, out, 1, cur_stream()));
        });
        b200_stream_synchronize(c->dev, cur_stream());
    }
    catch (...)
    {
        b200_stream_synchronize(c->dev, cur_stream());
        b200_free(c->dev, dp);
        throw;
    }
    b200_free(c->dev, dp);
    transparent_guard(c, lv, dst);
}

} // namespace

extern "C" {

// ---------------------------------------------------------------------------------------------------------
// Modulus / CoeffModulus
// ---------------------------------------------------------------------------------------------------------
long Modulus_Create1(uint64_t value, void **out)
{
    NULLRET(out);
    if (value == 1 || (value >> 61))
        return E_INVALIDARG_; // Modulus::set_value: "value can be at most 61 bits and cannot be 1"
    auto *m = new Modulus_();
    m->value = value;
    *out = m;
    return S_OK_;
}
long Modulus_Create2(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    *out = new Modulus_(*(Modulus_ *)copy);
    return S_OK_;
}
long Modulus_Destroy(void *p)
{
    NULLRET(p);
    delete (Modulus_ *)p;
    return S_OK_;
}
long Modulus_Value(void *p, uint64_t *v)
{
    NULLRET(p);
    NULLRET(v);
    *v = ((Modulus_ *)p)->value;
    return S_OK_;
}
long Modulus_BitCount(void *p, int *b)
{
    NULLRET(p);
    NULLRET(b);
    u64 v = ((Modulus_ *)p)->value;
    *b = v ? 64 - __builtin_clzll(v) : 0;
    return S_OK_;
}
long CoeffModulus_MaxBitCount(uint64_t n, int sec, int *bits)
{
    NULLRET(bits);
    *bits = sec == 0 ? 2147483647 : max_bits(n, sec);
    return S_OK_;
}
long CoeffModulus_BFVDefault(uint64_t n, int sec, uint64_t *length, void **coeffs)
{
    NULLRET(length);
    const u64 *tab = nullptr;
    size_t cnt = 0;
    if (sec != 128)
        return E_INVALIDARG_; // only the tc128 tables are carried (all Sunscreen uses: sunscreen/src/params.rs:137)
#define TAB(N)                                                                                                         \
    case N:                                                                                                            \
        tab = kDefault##N;                                                                                             \
        cnt = sizeof(kDefault##N) / sizeof(u64);                                                                       \
        break;
    switch (n)
    {
        TAB(1024) TAB(2048) TAB(4096) TAB(8192) TAB(16384) TAB(32768)
    default:
        return E_INVALIDARG_;
    }
#undef TAB
    *length = cnt;
    if (!coeffs)
        return S_OK_; // size query (S/c/modulus.cpp: BuildModulusPointers)
    for (size_t i = 0; i < cnt; i++)
    {
        auto *m = new Modulus_();
        m->value = tab[i];
        coeffs[i] = m;
    }
    return S_OK_;
}

long CoeffModulus_Create1(uint64_t n, uint64_t length, int *bit_sizes, void **coeffs)
{
    NULLRET(bit_sizes);
    NULLRET(coeffs);
    // CoeffModulus::Create (S/modulus.cpp:143-184): per distinct bit size the largest primes == 1 mod 2n, handed out
    // from the back of each list in the order the sizes were requested
    return guard([&] {
        if (n < 2 || n > 131072 || (n & (n - 1)))
            throw InvalidArg("poly_modulus_degree is invalid");
        if (length > 64)
            throw InvalidArg("bit_sizes is invalid");
        std::vector<std::pair<int, std::vector<b200::u64>>> tables;
        for (uint64_t i = 0; i < length; i++)
        {
            if (bit_sizes[i] > 60 || bit_sizes[i] < 2)
                throw InvalidArg("bit_sizes is invalid");
            bool found = false;
            for (auto &t : tables)
                found = found || t.first == bit_sizes[i];
            if (!found)
            {
                size_t cnt = 0;
                for (uint64_t j = 0; j < length; j++)
                    cnt += bit_sizes[j] == bit_sizes[i];
                tables.emplace_back(bit_sizes[i], b200::get_primes(2 * n, bit_sizes[i], cnt));
            }
        }
        for (uint64_t i = 0; i < length; i++)
            for (auto &t : tables)
                if (t.first == bit_sizes[i])
                {
                    auto *m = new Modulus_();
                    m->value = t.second.back();
                    t.second.pop_back();
                    coeffs[i] = m;
                }
    });
}

// ---------------------------------------------------------------------------------------------------------
// EncryptionParameters
// ---------------------------------------------------------------------------------------------------------
long EncParams_Create1(uint8_t scheme, void **out)
{
    NULLRET(out);
    if (scheme != 1)
        return E_INVALIDARG_; // only BFV is built by Sunscreen (seal_fhe/src/lib.rs:11-13)
    auto *p = new EncParams_();
    p->scheme = scheme;
    *out = p;
    return S_OK_;
}
long EncParams_Destroy(void *p)
{
    NULLRET(p);
    delete (EncParams_ *)p;
    return S_OK_;
}
long EncParams_GetPolyModulusDegree(void *p, uint64_t *d)
{
    NULLRET(p);
    NULLRET(d);
    *d = ((EncParams_ *)p)->n;
    return S_OK_;
}
long EncParams_SetPolyModulusDegree(void *p, uint64_t d)
{
    NULLRET(p);
    ((EncParams_ *)p)->n = d;
    return S_OK_;
}
long EncParams_GetCoeffModulus(void *p, uint64_t *length, void **coeffs)
{
    NULLRET(p);
    NULLRET(length);
    auto *e = (EncParams_ *)p;
    *length = e->coeff.size();
    if (!coeffs)
        return S_OK_;
    for (size_t i = 0; i < e->coeff.size(); i++)
    {
        auto *m = new Modulus_();
        m->value = e->coeff[i];
        coeffs[i] = m;
    }
    return S_OK_;
}
long EncParams_SetCoeffModulus(void *p, uint64_t length, void **coeffs)
{
    NULLRET(p);
    NULLRET(coeffs);
    auto *e = (EncParams_ *)p;
    if (length < 1 || length > 64)
        return E_INVALIDARG_;
    std::vector<u64> v;
    for (uint64_t i = 0; i < length; i++)
    {
        NULLRET(coeffs[i]);
        // only the COUNT is checked here (S/encryptionparams.h:188-207); widths are judged by SEALContext_Create
        v.push_back(((Modulus_ *)coeffs[i])->value);
    }
    e->coeff = v;
    return S_OK_;
}
long EncParams_GetScheme(void *p, uint8_t *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((EncParams_ *)p)->scheme;
    return S_OK_;
}
long EncParams_GetParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    auto *e = (EncParams_ *)p;
    std::vector<b200::u64> mods(e->coeff.begin(), e->coeff.end());
    b200::u64 out[4];
    b200::compute_parms_id((size_t)e->n, mods, e->plain, out);
    std::copy_n(out, 4, id);
    return S_OK_;
}
long EncParams_GetPlainModulus(void *p, void **m)
{
    NULLRET(p);
    NULLRET(m);
    auto *mm = new Modulus_();
    mm->value = ((EncParams_ *)p)->plain;
    *m = mm;
    return S_OK_;
}
long EncParams_SetPlainModulus1(void *p, void *m)
{
    NULLRET(p);
    NULLRET(m);
    ((EncParams_ *)p)->plain = ((Modulus_ *)m)->value;
    return S_OK_;
}
long EncParams_SetPlainModulus2(void *p, uint64_t v)
{
    NULLRET(p);
    if (v == 1 || (v >> 61))
        return COR_E_INVALIDOPERATION_; // Modulus::set_value throws; the C layer catches it as logic_error
                                        // (S/c/encryptionparameters.cpp:190-204)
    ((EncParams_ *)p)->plain = v;
    return S_OK_;
}

// ---------------------------------------------------------------------------------------------------------
// SEALContext
// ---------------------------------------------------------------------------------------------------------
long SEALContext_Create(void *parms, bool expand_mod_chain, int sec_level, void **out)
{
    NULLRET(parms);
    NULLRET(out);
    if (sec_level != 0 && sec_level != 128 && sec_level != 192 && sec_level != 256)
        return E_INVALIDARG_;
    auto *e = (EncParams_ *)parms;
    std::unique_ptr<Context_> c(new Context_());
    c->parms = *e;
    const char *nt = getenv("B200_SKIP_TRANSPARENT_CHECK");
    c->check_transparent = !(nt && nt[0] == '1');
    c->combine = !std::getenv("B200_NO_COMBINE");
    c->blocking_waits = std::getenv("B200_BLOCKING_WAITS") != nullptr;
    if (const char *cl = std::getenv("B200_COMBINE_LEADERS"))
        c->combine_leaders = std::max(1, std::min(4, atoi(cl)));
    c->use_graphs = !std::getenv("B200_NO_GRAPHS") && !std::getenv("B200_TRACE");
    // validation (S/context.cpp:135-420): anything failing leaves parameters_set = false, it is not an error here
    bool ok = e->n >= 2 && e->n <= 131072 && !(e->n & (e->n - 1)) && !e->coeff.empty() && e->plain >= 2;
    if (ok)
    {
        int total = 0;
        {
            b200::BigUInt Q(1);
            for (u64 q : e->coeff)
                Q.mul(q);
            total = Q.bit_length();
        }
        if (sec_level != 0 && total > max_bits(e->n, sec_level))
            ok = false;
        for (size_t i = 0; i < e->coeff.size() && ok; i++)
        {
            const int bits = e->coeff[i] ? 64 - __builtin_clzll(e->coeff[i]) : 0;
            if (bits < 2 || bits > 60) // SEAL_USER_MOD_BIT_COUNT_MIN / _MAX (S/context.cpp:166-177)
                ok = false;
            if ((e->coeff[i] - 1) % (2 * e->n))
                ok = false;
            if (e->plain >= e->coeff[i] && e->coeff.size() == 1)
                ok = false;
            if (std::__gcd(e->plain, e->coeff[i]) != 1)
                ok = false;
        }
    }
    if (ok)
    {
        const char *dv = getenv("B200_DEVICE");
        int device = dv ? atoi(dv) : 0;
        b200_ctx *dev = nullptr;
        int rc = b200_ctx_create(e->n, e->coeff.data(), e->coeff.size(), e->plain, device, &dev);
        if (rc == B200_E_CUDA || rc == B200_E_NOMEM)
            return E_UNEXPECTED_; // no CPU fallback: the backend cannot exist without its GPU
        if (rc)
            ok = false;
        else
        {
            c->dev = dev;
            c->owner = std::make_shared<DevOwner>();
            c->owner->dev = dev;
            b200_info info;
            b200_ctx_info(dev, &info);
            c->levels = info.levels;
            c->first_level = info.first_level;
            c->using_keyswitching = e->coeff.size() > 1;
            c->using_batching = info.using_batching != 0;
            for (int l = 0; l < info.levels; l++)
            {
                b200_level_info li;
                b200_ctx_level_info(dev, l, &li);
                ParmsId id;
                std::copy_n(li.parms_id, 4, id.begin());
                c->ids.push_back(id);
                c->level_k.push_back(li.k);
            }
            // the chain ends where the next parameter set would be invalid: the plain modulus must stay below the
            // coefficient modulus (S/context.cpp:207-215 via create_next_context_data, :478-497)
            {
                int keep = c->first_level + 1;
                for (int l = c->first_level + 1; l < c->levels; l++)
                {
                    b200::BigUInt Q(1);
                    for (int r = 0; r < c->level_k[l]; r++)
                        Q.mul(e->coeff[r]);
                    if (Q.w.size() == 1 && Q.w[0] <= e->plain)
                        break;
                    keep = l + 1;
                }
                if (!expand_mod_chain)
                    keep = c->first_level + 1; // only the key level and the first data level exist
                if (keep < c->levels)
                {
                    c->levels = keep;
                    c->ids.resize(keep);
                    c->level_k.resize(keep);
                }
            }
        }
    }
    c->parameters_set = ok;
    *out = c.release();
    return S_OK_;
}
long SEALContext_Destroy(void *p)
{
    NULLRET(p);
    Context_::release((Context_ *)p);
    return S_OK_;
}
static long ctx_id(void *p, uint64_t *out, int which)
{
    NULLRET(p);
    NULLRET(out);
    auto *c = (Context_ *)p;
    if (!c->parameters_set)
    {
        std::fill_n(out, 4, 0);
        return S_OK_;
    }
    int lv = which == 0 ? 0 : which == 1 ? c->first_level : c->levels - 1;
    std::copy_n(c->ids[lv].begin(), 4, out);
    return S_OK_;
}
long SEALContext_KeyParmsId(void *p, uint64_t *o) { return ctx_id(p, o, 0); }
long SEALContext_FirstParmsId(void *p, uint64_t *o) { return ctx_id(p, o, 1); }
long SEALContext_LastParmsId(void *p, uint64_t *o) { return ctx_id(p, o, 2); }
long SEALContext_ParametersSet(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    *b = ((Context_ *)p)->parameters_set;
    return S_OK_;
}
long SEALContext_UsingKeyswitching(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    *b = ((Context_ *)p)->using_keyswitching;
    return S_OK_;
}
long B200_SEALContext_Synchronize(void *p)
{
    NULLRET(p);
    auto *c = (Context_ *)p;
    return guard([&] {
        if (c->dev)
            dev_check(b200_stream_synchronize(c->dev, nullptr));
    });
}

// ---------------------------------------------------------------------------------------------------------
// Ciphertext
// ---------------------------------------------------------------------------------------------------------
long Ciphertext_Create1(void * /*pool*/, void **out)
{
    NULLRET(out);
    *out = new Ciphertext_();
    return S_OK_;
}
long Ciphertext_Create2(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    auto *c = new Ciphertext_();
    long hr = guard([&] { c->assign(*(Ciphertext_ *)copy); });
    if (hr)
    {
        delete c;
        return hr;
    }
    *out = c;
    return S_OK_;
}
long Ciphertext_Set(void *p, void *assign)
{
    NULLRET(p);
    NULLRET(assign);
    return guard([&] { ((Ciphertext_ *)p)->assign(*(Ciphertext_ *)assign); });
}
long Ciphertext_Destroy(void *p)
{
    NULLRET(p);
    delete (Ciphertext_ *)p;
    return S_OK_;
}
long Ciphertext_Size(void *p, uint64_t *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((Ciphertext_ *)p)->size;
    return S_OK_;
}
long Ciphertext_PolyModulusDegree(void *p, uint64_t *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((Ciphertext_ *)p)->n;
    return S_OK_;
}
long Ciphertext_CoeffModulusSize(void *p, uint64_t *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((Ciphertext_ *)p)->k;
    return S_OK_;
}
long Ciphertext_ParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(((Ciphertext_ *)p)->parms_id.begin(), 4, id);
    return S_OK_;
}
long Ciphertext_SetParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(id, 4, ((Ciphertext_ *)p)->parms_id.begin());
    return S_OK_;
}
long Ciphertext_Resize1(void *p, void *context, uint64_t *parms_id, uint64_t size)
{
    NULLRET(p);
    NULLRET(context);
    NULLRET(parms_id);
    auto *ct = (Ciphertext_ *)p;
    auto *c = (Context_ *)context;
    return guard([&] {
        if (!c->parameters_set)
            throw InvalidArg("encryption parameters are not set correctly");
        ParmsId id;
        std::copy_n(parms_id, 4, id.begin());
        int lv = c->level_of(id);
        if (lv < 0)
            throw InvalidArg("parms_id is not valid for encryption parameters");
        if ((size < 2 && size != 0) || size > 16)
            throw InvalidArg("invalid size");
        ct->sync_host();
        std::vector<u64> old = ct->host;
        const u64 ok = ct->k, on = ct->n, os = ct->size;
        ct->release_dev();
        ct->parms_id = id;
        ct->size = size;
        ct->k = c->level_k[lv];
        ct->n = c->parms.n;
        ct->ctx = c;
        ct->host.assign(ct->words(), 0);
        if (ok == ct->k && on == ct->n) // same shape per polynomial: existing polynomials are kept (DynArray::resize)
            std::copy_n(old.begin(), std::min(old.size(), ct->host.size()), ct->host.begin());
        (void)os;
        ct->host_valid = true;
    });
}
long Ciphertext_GetDataAt1(void *p, uint64_t index, uint64_t *data)
{
    NULLRET(p);
    NULLRET(data);
    auto *ct = (Ciphertext_ *)p;
    long hr = guard([&] { ct->sync_host(); });
    if (hr)
        return hr;
    if (index >= ct->host.size())
        return ERROR_INVALID_INDEX_;
    *data = ct->host[index];
    return S_OK_;
}
long Ciphertext_GetDataAt2(void *p, uint64_t poly, uint64_t coeff, uint64_t *data)
{
    NULLRET(p);
    NULLRET(data);
    auto *ct = (Ciphertext_ *)p;
    if (poly >= ct->size || coeff >= ct->k * ct->n)
        return ERROR_INVALID_INDEX_;
    return Ciphertext_GetDataAt1(p, poly * ct->k * ct->n + coeff, data);
}
long Ciphertext_SetDataAt(void *p, uint64_t index, uint64_t value)
{
    NULLRET(p);
    auto *ct = (Ciphertext_ *)p;
    long hr = guard([&] { ct->sync_host(); });
    if (hr)
        return hr;
    if (index >= ct->host.size())
        return ERROR_INVALID_INDEX_;
    ct->host[index] = value;
    ct->dev_valid = false;
    return S_OK_;
}
long Ciphertext_IsNTTForm(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    *b = ((Ciphertext_ *)p)->is_ntt_form;
    return S_OK_;
}
long Ciphertext_SetIsNTTForm(void *p, bool b)
{
    NULLRET(p);
    ((Ciphertext_ *)p)->is_ntt_form = b;
    return S_OK_;
}
long Ciphertext_Scale(void *p, double *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((Ciphertext_ *)p)->scale;
    return S_OK_;
}
long Ciphertext_IsTransparent(void *p, bool *r)
{
    NULLRET(p);
    NULLRET(r);
    auto *ct = (Ciphertext_ *)p;
    return guard([&] {
        // (!size || size < 2) || all polys from index 1 are zero (S/ciphertext.h:451-456)
        if (ct->size < 2)
        {
            *r = true;
            return;
        }
        ct->sync_host();
        bool nz = false;
        for (size_t i = (size_t)(ct->k * ct->n); i < ct->host.size() && !nz; i++)
            nz = ct->host[i] != 0;
        *r = !nz;
    });
}
long B200_Ciphertext_SetWords(void *p, void *context, uint64_t *parms_id, uint64_t size, bool ntt, const uint64_t *words)
{
    NULLRET(words);
    long hr = Ciphertext_Resize1(p, context, parms_id, size);
    if (hr)
        return hr;
    auto *ct = (Ciphertext_ *)p;
    std::memcpy(ct->host.data(), words, ct->words() * sizeof(u64));
    ct->is_ntt_form = ntt;
    ct->dev_valid = false;
    return S_OK_;
}
long B200_Ciphertext_GetWords(void *p, uint64_t *words, uint64_t cap)
{
    NULLRET(p);
    NULLRET(words);
    auto *ct = (Ciphertext_ *)p;
    long hr = guard([&] { ct->sync_host(); });
    if (hr)
        return hr;
    if (cap < ct->host.size())
        return E_INVALIDARG_;
    std::memcpy(words, ct->host.data(), ct->host.size() * sizeof(u64));
    return S_OK_;
}

// ---------------------------------------------------------------------------------------------------------
// Plaintext
// ---------------------------------------------------------------------------------------------------------
long Plaintext_Create1(void *, void **out)
{
    NULLRET(out);
    *out = new Plaintext_();
    return S_OK_;
}
long Plaintext_Create2(uint64_t count, void *, void **out)
{
    NULLRET(out);
    auto *p = new Plaintext_();
    p->coeffs.assign(count, 0);
    *out = p;
    return S_OK_;
}
// Plaintext(const std::string &hex_poly) (S/plaintext.cpp:88-203): "7FFx^3 + 1x^1 + 3" — hexadecimal coefficients,
// strictly decreasing decimal powers, terms separated by " + ", the constant term without "x^0"
long Plaintext_Create4(uint8_t *hex_poly, void *, void **out)
{
    NULLRET(out);
    NULLRET(hex_poly);
    const char *s = (const char *)hex_poly;
    const size_t len = std::strlen(s);
    auto is_hex = [](char ch) { return (ch >= '0' && ch <= '9') || (ch >= 'A' && ch <= 'F') || (ch >= 'a' && ch <= 'f'); };
    auto hex_val = [](char ch) -> u64 { return ch <= '9' ? (u64)(ch - '0') : (u64)((ch | 0x20) - 'a' + 10); };
    struct Term
    {
        u64 coeff;
        long power;
    };
    std::vector<Term> terms;
    size_t pos = 0;
    long last_power = 0x7fffffffL;
    long count = 0;
    int max_bits = 0;
    while (pos < len)
    {
        size_t cl = 0;
        while (is_hex(s[pos + cl]))
            cl++;
        if (!cl)
            return E_INVALIDARG_; // "unable to parse hex_poly"
        // significant bits of the coefficient (leading zeros do not count)
        size_t lead = 0;
        while (lead < cl && s[pos + lead] == '0')
            lead++;
        int bits = 0;
        if (lead < cl)
        {
            const u64 top = hex_val(s[pos + lead]);
            bits = (int)(4 * (cl - lead - 1)) + (64 - __builtin_clzll(top));
        }
        max_bits = std::max(max_bits, bits);
        u64 v = 0;
        if (bits <= 64)
            for (size_t i = lead; i < cl; i++)
                v = (v << 4) | hex_val(s[pos + i]);
        pos += cl;
        long power = 0;
        if (s[pos] != '\0')
        {
            if (s[pos] != 'x' || s[pos + 1] != '^')
                return E_INVALIDARG_;
            pos += 2;
            while (s[pos] >= '0' && s[pos] <= '9')
            {
                power = power * 10 + (s[pos] - '0');
                if (power > 0x7fffffffL)
                    return E_INVALIDARG_;
                pos++;
            }
        }
        if (power >= last_power)
            return E_INVALIDARG_;
        if (terms.empty())
            count = power + 1;
        last_power = power;
        terms.push_back({ v, power });
        if (s[pos] != '\0')
        {
            if (s[pos] != ' ' || s[pos + 1] != '+' || s[pos + 2] != ' ')
                return E_INVALIDARG_;
            pos += 3;
        }
    }
    auto *pl = new Plaintext_();
    if (count && max_bits)
    {
        if (max_bits > 64)
        {
            delete pl;
            return E_INVALIDARG_; // "hex_poly has too large coefficients"
        }
        pl->coeffs.assign((size_t)count, 0);
        for (auto &t : terms)
            pl->coeffs[(size_t)t.power] = t.coeff;
    }
    *out = pl;
    return S_OK_;
}
long Plaintext_Create5(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    *out = new Plaintext_(*(Plaintext_ *)copy);
    return S_OK_;
}
long Plaintext_Destroy(void *p)
{
    NULLRET(p);
    delete (Plaintext_ *)p;
    return S_OK_;
}
long Plaintext_CoeffCount(void *p, uint64_t *c)
{
    NULLRET(p);
    NULLRET(c);
    *c = ((Plaintext_ *)p)->coeffs.size();
    return S_OK_;
}
long Plaintext_CoeffAt(void *p, uint64_t i, uint64_t *c)
{
    NULLRET(p);
    NULLRET(c);
    auto *pl = (Plaintext_ *)p;
    if (i >= pl->coeffs.size())
        return ERROR_INVALID_INDEX_;
    *c = pl->coeffs[i];
    return S_OK_;
}
long Plaintext_SetCoeffAt(void *p, uint64_t i, uint64_t v)
{
    NULLRET(p);
    auto *pl = (Plaintext_ *)p;
    if (i >= pl->coeffs.size())
        return ERROR_INVALID_INDEX_;
    pl->coeffs[i] = v;
    return S_OK_;
}
long Plaintext_Resize(void *p, uint64_t c)
{
    NULLRET(p);
    auto *pl = (Plaintext_ *)p;
    if (pl->parms_id != kZeroId)
        return COR_E_INVALIDOPERATION_; // "cannot resize an NTT transformed Plaintext"
    pl->coeffs.resize(c, 0);
    return S_OK_;
}
long Plaintext_GetParmsId(void *p, uint64_t *parms_id)
{
    NULLRET(p);
    NULLRET(parms_id);
    std::copy_n(((Plaintext_ *)p)->parms_id.begin(), 4, parms_id);
    return S_OK_;
}
long Plaintext_SetParmsId(void *p, uint64_t *parms_id)
{
    NULLRET(p);
    NULLRET(parms_id);
    std::copy_n(parms_id, 4, ((Plaintext_ *)p)->parms_id.begin());
    return S_OK_;
}
long Plaintext_IsNTTForm(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    *b = ((Plaintext_ *)p)->parms_id != kZeroId;
    return S_OK_;
}
long Plaintext_IsZero(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    auto *pl = (Plaintext_ *)p;
    *b = std::all_of(pl->coeffs.begin(), pl->coeffs.end(), [](u64 x) { return x == 0; });
    return S_OK_;
}
long B200_Plaintext_SetCoeffs(void *p, uint64_t count, const uint64_t *coeffs)
{
    NULLRET(p);
    if (count)
        NULLRET(coeffs);
    ((Plaintext_ *)p)->coeffs.assign(coeffs, coeffs + count);
    return S_OK_;
}

// ---------------------------------------------------------------------------------------------------------
// PublicKey / SecretKey
// ---------------------------------------------------------------------------------------------------------
long PublicKey_Create1(void **out)
{
    NULLRET(out);
    *out = new PublicKey_();
    return S_OK_;
}
long PublicKey_Create2(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    auto *k = new PublicKey_();
    long hr = guard([&] { k->data.assign(((PublicKey_ *)copy)->data); });
    if (hr)
    {
        delete k;
        return hr;
    }
    *out = k;
    return S_OK_;
}
long PublicKey_Data(void *p, void **data)
{
    NULLRET(p);
    NULLRET(data);
    *data = &((PublicKey_ *)p)->data; // a view owned by the key, like the reference (S/c/publickey.cpp)
    return S_OK_;
}
long PublicKey_ParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(((PublicKey_ *)p)->data.parms_id.begin(), 4, id);
    return S_OK_;
}
long PublicKey_Destroy(void *p)
{
    NULLRET(p);
    delete (PublicKey_ *)p;
    return S_OK_;
}
long SecretKey_Create1(void **out)
{
    NULLRET(out);
    *out = new SecretKey_();
    return S_OK_;
}
long SecretKey_Create2(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    *out = new SecretKey_(*(SecretKey_ *)copy);
    return S_OK_;
}
long SecretKey_Data(void *p, void **data)
{
    NULLRET(p);
    NULLRET(data);
    *data = &((SecretKey_ *)p)->data;
    return S_OK_;
}
long SecretKey_ParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(((SecretKey_ *)p)->data.parms_id.begin(), 4, id);
    return S_OK_;
}
long SecretKey_Destroy(void *p)
{
    NULLRET(p);
    delete (SecretKey_ *)p;
    return S_OK_;
}
long B200_SecretKey_SetWords(void *p, void *context, const uint64_t *words)
{
    NULLRET(p);
    NULLRET(context);
    NULLRET(words);
    auto *c = (Context_ *)context;
    if (!c->parameters_set)
        return E_INVALIDARG_;
    auto *sk = (SecretKey_ *)p;
    sk->data.coeffs.assign(words, words + c->parms.coeff.size() * c->parms.n);
    sk->data.parms_id = c->ids[0];
    return S_OK_;
}

// ---------------------------------------------------------------------------------------------------------
// KSwitchKeys
// ---------------------------------------------------------------------------------------------------------
long KSwitchKeys_Create1(void **out)
{
    NULLRET(out);
    *out = new KSwitchKeys_();
    return S_OK_;
}
long KSwitchKeys_Create2(void *copy, void **out)
{
    NULLRET(copy);
    NULLRET(out);
    auto *src = (KSwitchKeys_ *)copy;
    auto *k = new KSwitchKeys_();
    long hr = guard([&] {
        k->parms_id = src->parms_id;
        for (auto &l : src->keys)
        {
            k->keys.emplace_back();
            for (auto *pk : l)
            {
                auto *n = new PublicKey_();
                n->data.assign(pk->data);
                k->keys.back().push_back(n);
            }
        }
    });
    if (hr)
    {
        delete k;
        return hr;
    }
    *out = k;
    return S_OK_;
}
long KSwitchKeys_Destroy(void *p)
{
    NULLRET(p);
    delete (KSwitchKeys_ *)p;
    return S_OK_;
}
long KSwitchKeys_Size(void *p, uint64_t *s)
{
    NULLRET(p);
    NULLRET(s);
    auto *k = (KSwitchKeys_ *)p;
    *s = (uint64_t)std::count_if(k->keys.begin(), k->keys.end(), [](const std::vector<PublicKey_ *> &v) { return !v.empty(); });
    return S_OK_;
}
long KSwitchKeys_RawSize(void *p, uint64_t *s)
{
    NULLRET(p);
    NULLRET(s);
    *s = ((KSwitchKeys_ *)p)->keys.size();
    return S_OK_;
}
long KSwitchKeys_GetKeyList(void *p, uint64_t index, uint64_t *count, void **list)
{
    NULLRET(p);
    NULLRET(count);
    auto *k = (KSwitchKeys_ *)p;
    if (index >= k->keys.size())
        return ERROR_INVALID_INDEX_;
    *count = k->keys[index].size();
    if (!list)
        return S_OK_;
    for (size_t i = 0; i < k->keys[index].size(); i++)
    { // copies owned by the caller (S/c/kswitchkeys.cpp: GetKeyFromVector)
        auto *n = new PublicKey_();
        n->data.assign(k->keys[index][i]->data);
        list[i] = n;
    }
    return S_OK_;
}
long KSwitchKeys_ClearDataAndReserve(void *p, uint64_t size)
{
    NULLRET(p);
    auto *k = (KSwitchKeys_ *)p;
    k->clear();
    k->keys.reserve(size);
    return S_OK_;
}
long KSwitchKeys_AddKeyList(void *p, uint64_t count, void **list)
{
    NULLRET(p);
    NULLRET(list);
    auto *k = (KSwitchKeys_ *)p;
    return guard([&] {
        k->keys.emplace_back();
        for (uint64_t i = 0; i < count; i++)
        {
            auto *n = new PublicKey_();
            n->data.assign(((PublicKey_ *)list[i])->data);
            k->keys.back().push_back(n);
        }
        k->drop_flat();
    });
}
long KSwitchKeys_GetParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(((KSwitchKeys_ *)p)->parms_id.begin(), 4, id);
    return S_OK_;
}
long KSwitchKeys_SetParmsId(void *p, uint64_t *id)
{
    NULLRET(p);
    NULLRET(id);
    std::copy_n(id, 4, ((KSwitchKeys_ *)p)->parms_id.begin());
    return S_OK_;
}
long RelinKeys_GetIndex(uint64_t key_power, uint64_t *index)
{
    NULLRET(index);
    if (key_power < 2)
        return E_INVALIDARG_;
    *index = key_power - 2;
    return S_OK_;
}
long GaloisKeys_GetIndex(uint32_t elt, uint64_t *index)
{
    NULLRET(index);
    if (!(elt & 1) || elt < 3)
        return E_INVALIDARG_; // GaloisTool::GetIndexFromElt (S/util/galois.h:139-147)
    *index = (elt - 1) >> 1;
    return S_OK_;
}
long B200_KSwitchKeys_SetKeyWords(void *p, void *context, uint64_t index, uint64_t decomp, const uint64_t *words)
{
    NULLRET(p);
    NULLRET(context);
    NULLRET(words);
    auto *k = (KSwitchKeys_ *)p;
    auto *c = (Context_ *)context;
    return guard([&] {
        if (!c->parameters_set)
            throw InvalidArg("encryption parameters are not set correctly");
        if (k->keys.size() <= index)
            k->keys.resize(index + 1);
        for (auto *pk : k->keys[index])
            delete pk;
        k->keys[index].clear();
        const size_t K = c->parms.coeff.size(), n = c->parms.n, per = 2 * K * n;
        for (uint64_t j = 0; j < decomp; j++)
        {
            auto *pk = new PublicKey_();
            pk->data.parms_id = c->ids[0];
            pk->data.size = 2;
            pk->data.k = K;
            pk->data.n = n;
            pk->data.is_ntt_form = true;
            pk->data.host.assign(words + per * j, words + per * (j + 1));
            pk->data.host_valid = true;
            k->keys[index].push_back(pk);
        }
        k->parms_id = c->ids[0];
        k->drop_flat();
    });
}

// ---------------------------------------------------------------------------------------------------------
// Evaluator
// ---------------------------------------------------------------------------------------------------------
long Evaluator_Create(void *context, void **out)
{
    NULLRET(context);
    NULLRET(out);
    auto *c = (Context_ *)context;
    if (!c->parameters_set)
        return E_INVALIDARG_; // "encryption parameters are not set correctly" (S/evaluator.cpp:66-71)
    auto *e = new Evaluator_();
    e->ctx = c;
    e->hold.bind(c);
    *out = e;
    return S_OK_;
}
long Evaluator_Destroy(void *p)
{
    NULLRET(p);
    delete (Evaluator_ *)p;
    return S_OK_;
}
long Evaluator_ContextUsingKeyswitching(void *p, bool *b)
{
    NULLRET(p);
    NULLRET(b);
    *b = ((Evaluator_ *)p)->ctx->using_keyswitching;
    return S_OK_;
}
long Evaluator_Negate(void *p, void *enc, void *dst)
{
    NULLRET(p);
    NULLRET(enc);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &a = *(Ciphertext_ *)enc;
    auto &d = *(Ciphertext_ *)dst;
    return guard([&] {
        OpScope scope(c);
        int lv = data_level(c, a, "encrypted is not valid for encryption parameters");
        const u64 *pa = a.dev_ptr(c);
        bool ntt = a.is_ntt_form;
        with_output(c, d, { &a }, a.parms_id, a.size, a.k,
                    [&](u64 *out) { dev_check(b200_negate(c->dev, lv, pa, out, (int)a.size, 1, cur_stream())); });
        d.is_ntt_form = ntt;
        transparent_guard(c, lv, d);
    });
}
long Evaluator_Add(void *p, void *a, void *b, void *dst)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(b);
    NULLRET(dst);
    return guard([&] { op_addsub(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Ciphertext_ *)b, *(Ciphertext_ *)dst, 0); });
}
long Evaluator_Sub(void *p, void *a, void *b, void *dst)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(b);
    NULLRET(dst);
    return guard([&] { op_addsub(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Ciphertext_ *)b, *(Ciphertext_ *)dst, 1); });
}
long Evaluator_AddMany(void *p, uint64_t count, void **encs, void *dst)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        if (count == 0)
            throw InvalidArg("encrypteds cannot be empty");
        for (uint64_t i = 0; i < count; i++)
            if (!encs[i] || encs[i] == dst)
                throw InvalidArg("encrypteds must be different from destination");
        // destination = encrypteds[0]; then add_inplace the rest in order (S/evaluator.cpp:319-350)
        auto &d = *(Ciphertext_ *)dst;
        d.assign(*(Ciphertext_ *)encs[0]);
        for (uint64_t i = 1; i < count; i++)
            op_addsub(c, d, *(Ciphertext_ *)encs[i], d, 0);
    });
}
long Evaluator_Multiply(void *p, void *a, void *b, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(b);
    NULLRET(dst);
    return guard([&] { op_multiply(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Ciphertext_ *)b, *(Ciphertext_ *)dst, false); });
}
long Evaluator_Square(void *p, void *a, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(dst);
    return guard([&] { op_multiply(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Ciphertext_ *)a, *(Ciphertext_ *)dst, true); });
}
long Evaluator_Relinearize(void *p, void *a, void *keys, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(keys);
    NULLRET(dst);
    return guard([&] { op_relinearize(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(KSwitchKeys_ *)keys, *(Ciphertext_ *)dst); });
}
long Evaluator_MultiplyMany(void *p, uint64_t count, void **encs, void *relin_keys, void *dst, void *)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(relin_keys);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)relin_keys;
    return guard([&] {
        // Evaluator::multiply_many (S/evaluator.cpp:1535-1605): pairwise products appended to a work list
        if (count == 0)
            throw InvalidArg("encrypteds vector must not be empty");
        for (uint64_t i = 0; i < count; i++)
            if (!encs[i] || encs[i] == dst)
                throw InvalidArg("encrypteds must be different from destination");
        auto &d = *(Ciphertext_ *)dst;
        if (count == 1)
        {
            d.assign(*(Ciphertext_ *)encs[0]);
            return;
        }
        std::vector<std::unique_ptr<Ciphertext_>> prod;
        auto mulrelin = [&](Ciphertext_ &x, Ciphertext_ &y, bool same) {
            std::unique_ptr<Ciphertext_> t(new Ciphertext_()), r(new Ciphertext_());
            op_multiply(c, x, same ? x : y, *t, same);
            op_relinearize(c, *t, keys, *r);
            prod.push_back(std::move(r));
        };
        for (uint64_t i = 0; i + 1 < count; i += 2)
            mulrelin(*(Ciphertext_ *)encs[i], *(Ciphertext_ *)encs[i + 1], encs[i] == encs[i + 1]);
        if (count & 1)
        {
            std::unique_ptr<Ciphertext_> t(new Ciphertext_());
            t->assign(*(Ciphertext_ *)encs[count - 1]);
            prod.push_back(std::move(t));
        }
        for (size_t i = 0; i + 1 < prod.size(); i += 2)
            mulrelin(*prod[i], *prod[i + 1], false);
        d.assign(*prod.back());
    });
}
long Evaluator_Exponentiate(void *p, void *a, uint64_t exponent, void *relin_keys, void *dst, void *pool)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(relin_keys);
    NULLRET(dst);
    if (exponent == 0)
        return E_INVALIDARG_;
    if (exponent == 1)
        return Ciphertext_Set(dst, a);
    // exponentiate_inplace: multiply_many over `exponent` copies (S/evaluator.cpp:1607-1643); the copies are
    // distinct objects there, so the square shortcut of multiply_many (same data pointer) does not trigger
    std::vector<std::unique_ptr<Ciphertext_>> copies;
    std::vector<void *> ptrs;
    long hr = guard([&] {
        for (uint64_t i = 0; i < exponent; i++)
        {
            copies.emplace_back(new Ciphertext_());
            copies.back()->assign(*(Ciphertext_ *)a);
            ptrs.push_back(copies.back().get());
        }
    });
    if (hr)
        return hr;
    Ciphertext_ tmp;
    hr = Evaluator_MultiplyMany(p, exponent, ptrs.data(), relin_keys, &tmp, pool);
    if (hr)
        return hr;
    return Ciphertext_Set(dst, &tmp);
}
long Evaluator_ModSwitchToNext1(void *p, void *a, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &x = *(Ciphertext_ *)a;
    auto &d = *(Ciphertext_ *)dst;
    return guard([&] {
        OpScope scope(c);
        int lv = data_level(c, x, "encrypted is not valid for encryption parameters");
        if (lv + 1 >= c->levels)
            throw InvalidArg("end of modulus switching chain reached");
        if (x.is_ntt_form)
            throw InvalidArg("BFV encrypted cannot be in NTT form");
        const u64 *px = x.dev_ptr(c);
        with_output(c, d, { &x }, c->ids[lv + 1], x.size, x.k - 1,
                    [&](u64 *out) { dev_check(b200_mod_switch_to_next(c->dev, lv, px, (int)x.size, out, 1, cur_stream())); });
        transparent_guard(c, lv + 1, d);
    });
}
// Evaluator::mod_switch_to_next(const Plaintext &, Plaintext &) (S/evaluator.h:380-407, evaluator.cpp:1307-1340):
// only NTT-form plaintexts can be switched; the last residue polynomial is dropped
long Evaluator_ModSwitchToNext2(void *p, void *plain, void *dst)
{
    NULLRET(p);
    NULLRET(plain);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &src = *(Plaintext_ *)plain;
    return guard([&] {
        Plaintext_ t(src);
        const size_t n = c->parms.n;
        // is_valid_for(plain) (S/valcheck.cpp:20-65,246-294)
        if (t.parms_id == kZeroId)
        {
            if (t.coeffs.size() > n)
                throw InvalidArg("plain is not valid for encryption parameters");
            for (u64 x : t.coeffs)
                if (x >= c->parms.plain)
                    throw InvalidArg("plain is not valid for encryption parameters");
            throw InvalidArg("plain is not in NTT form");
        }
        const int lv = c->level_of(t.parms_id);
        if (lv < c->first_level || t.coeffs.size() != (size_t)c->level_k[lv] * n)
            throw InvalidArg("plain is not valid for encryption parameters");
        for (int r = 0; r < c->level_k[lv]; r++)
            for (size_t i = 0; i < n; i++)
                if (t.coeffs[(size_t)r * n + i] >= c->parms.coeff[r])
                    throw InvalidArg("plain is not valid for encryption parameters");
        if (lv + 1 >= c->levels)
            throw InvalidArg("end of modulus switching chain reached");
        t.coeffs.resize((size_t)c->level_k[lv + 1] * n);
        t.parms_id = c->ids[lv + 1];
        *(Plaintext_ *)dst = std::move(t);
    });
}
long Evaluator_AddPlain(void *p, void *a, void *pl, void *dst)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(pl);
    NULLRET(dst);
    return guard([&] { op_plain(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Plaintext_ *)pl, *(Ciphertext_ *)dst, 0); });
}
long Evaluator_SubPlain(void *p, void *a, void *pl, void *dst)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(pl);
    NULLRET(dst);
    return guard([&] { op_plain(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Plaintext_ *)pl, *(Ciphertext_ *)dst, 1); });
}
long Evaluator_MultiplyPlain(void *p, void *a, void *pl, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(pl);
    NULLRET(dst);
    return guard([&] { op_plain(((Evaluator_ *)p)->ctx, *(Ciphertext_ *)a, *(Plaintext_ *)pl, *(Ciphertext_ *)dst, 2); });
}
long Evaluator_ApplyGalois(void *p, void *a, uint32_t elt, void *keys, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(keys);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        OpScope scope(c);
        op_galois(c, *(Ciphertext_ *)a, elt, *(KSwitchKeys_ *)keys, *(Ciphertext_ *)dst);
    });
}
long Evaluator_RotateRows(void *p, void *a, int steps, void *keys, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(keys);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        auto &K = *(KSwitchKeys_ *)keys;
        if (c->combine && c->using_batching && K.parms_id == c->ids[0] && steps != 0)
        { // a rotation whose key is present is one key switch: concurrent ones are combined like multiply / relinearize
            uint32_t elt = 0;
            if (b200_galois_elt_from_step(c->dev, steps, &elt) == 0 && has_galois_key(K, elt) &&
                galois_combined(c, *(Ciphertext_ *)a, elt, K, *(Ciphertext_ *)dst))
                return;
        }
        OpScope scope(c);
        op_rotate(c, *(Ciphertext_ *)a, steps, K, *(Ciphertext_ *)dst);
    });
}
long Evaluator_RotateColumns(void *p, void *a, void *keys, void *dst, void *)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(keys);
    NULLRET(dst);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        if (!c->using_batching)
            throw LogicErr("encryption parameters do not support batching");
        if (galois_combined(c, *(Ciphertext_ *)a, (uint32_t)(2 * c->parms.n - 1), *(KSwitchKeys_ *)keys, *(Ciphertext_ *)dst))
            return;
        OpScope scope(c);
        op_galois(c, *(Ciphertext_ *)a, (uint32_t)(2 * c->parms.n - 1), *(KSwitchKeys_ *)keys, *(Ciphertext_ *)dst);
    });
}
long B200_Evaluator_MultiplyRelinBatch(void *p, uint64_t count, void **e1, void **e2, void *relin_keys, void **dsts);

// The other DAG node kinds of sunscreen_runtime (run.rs:160-341) as batches of independent items: same results as the
// per-handle calls, one launch sequence per batch.  All items must be size-2 ciphertexts at one level.
namespace
{
struct BatchSlab
{
    Context_ *c;
    void *p = nullptr;
    BatchSlab(Context_ *ctx, size_t words) : c(ctx) { dev_check(b200_malloc(c->dev, std::max<size_t>(words, 1) * 8, &p)); }
    // freed in stream order (every use of the slab is on the operation's stream): no host synchronisation here, so the
    // context mutex is never held while the GPU works — batches of different caller threads overlap their copies and kernels
    ~BatchSlab() { b200_free_async(c->dev, p, cur_stream()); }
    u64 *w() const { return (u64 *)p; }
    BatchSlab(const BatchSlab &) = delete;
};
// every handle of a batch argument must be non-null BEFORE anything is read through it (E_INVALIDARG)
void batch_handles(uint64_t count, std::initializer_list<void **> arrays)
{
    for (void **arr : arrays)
        for (uint64_t i = 0; i < count; i++)
            NULLRET_THROW(arr[i]);
}
// A batch seam's operation scope.  B200_BLOCKING_WAITS=1: sleep instead of spinning while the batch completes.
struct SeamScope : OpScope
{
    explicit SeamScope(Context_ *c) : OpScope(c) { blocking = c->blocking_waits; }
};
// the Galois element of RotateRows(step) and its key list's index; a step without its own key is refused (no NAF parts)
size_t row_step_key(Context_ *c, KSwitchKeys_ &keys, int step, uint32_t *elt)
{
    return galois_key_index(c, keys, *elt = row_step_elt(c, step));
}
// the items (checked by batch_level) one after the other in `slab`: one launch for all of them
void batch_gather(Context_ *c, uint64_t count, void **cts, BatchSlab &slab)
{
    std::vector<u64 *> ptrs(count);
    for (uint64_t i = 0; i < count; i++)
        ptrs[i] = const_cast<u64 *>(((Ciphertext_ *)cts[i])->dev_ptr(c));
    dev_check(b200_gather_scatter(c->dev, ptrs.data(), count, slab.w(), ((Ciphertext_ *)cts[0])->words(), 1, cur_stream()));
}
void batch_scatter(Context_ *c, uint64_t count, void **dsts, const BatchSlab &slab, const ParmsId &id, u64 k, int level,
                   u64 size = 2)
{
    const u64 w = size * k * c->parms.n;
    std::vector<u64 *> ptrs(count);
    for (uint64_t i = 0; i < count; i++)
        ptrs[i] = ((Ciphertext_ *)dsts[i])->prepare_output(c, id, size, k);
    dev_check(b200_gather_scatter(c->dev, ptrs.data(), count, slab.w(), w, 0, cur_stream()));
    if (c->check_transparent)
    { // one flag per item
        BatchSlab flags(c, count);
        std::vector<uint32_t> h(count);
        dev_check(b200_is_transparent(c->dev, level, slab.w(), (int)size, (uint32_t *)flags.p, count, cur_stream()));
        dev_check(b200_memcpy_d2h(c->dev, h.data(), flags.p, count * 4, cur_stream()));
        tl_scope->wait(); // releases the context mutex while the batch completes
        for (uint32_t f : h)
            if (f)
                throw LogicErr("result ciphertext is transparent");
    }
}
} // namespace

// Bulk word access for a batch of handles: `words` is ONE contiguous host buffer [count][size][k][n] (pinned memory moves at
// link speed and asynchronously); one copy + one scatter/gather launch instead of a host memcpy and a transfer per handle.
// Same validation as B200_Ciphertext_SetWords.
long B200_Ciphertext_SetWordsBatch(void *context, uint64_t count, void **cts, uint64_t *parms_id, uint64_t size, bool ntt,
                                   const uint64_t *words)
{
    NULLRET(context);
    NULLRET(cts);
    NULLRET(parms_id);
    NULLRET(words);
    auto *c = (Context_ *)context;
    return guard([&] {
        if (!c->parameters_set)
            throw InvalidArg("encryption parameters are not set correctly");
        ParmsId id;
        std::copy_n(parms_id, 4, id.begin());
        const int lv = c->level_of(id);
        if (lv < 0)
            throw InvalidArg("parms_id is not valid for encryption parameters");
        if (size < 2 || size > 16)
            throw InvalidArg("invalid size");
        if (count == 0)
            return;
        batch_handles(count, { cts });
        SeamScope scope(c);
        const u64 k = (u64)c->level_k[lv];
        const u64 w = size * k * c->parms.n;
        BatchSlab S(c, count * w);
        dev_check(b200_memcpy_h2d(c->dev, S.p, words, count * w * sizeof(u64), cur_stream()));
        std::vector<u64 *> ptrs(count);
        for (uint64_t i = 0; i < count; i++)
        {
            auto *ct = (Ciphertext_ *)cts[i];
            ptrs[i] = ct->prepare_output(c, id, size, k);
            ct->is_ntt_form = ntt;
        }
        dev_check(b200_gather_scatter(c->dev, ptrs.data(), count, S.w(), w, 0, cur_stream()));
        scope.wait(); // the caller may reuse `words` when the call returns; context mutex released while the copy runs
    });
}
// all handles must have the same shape; `words` receives [count][size][k][n]
long B200_Ciphertext_GetWordsBatch(void *context, uint64_t count, void **cts, uint64_t *words, uint64_t cap)
{
    NULLRET(context);
    NULLRET(cts);
    NULLRET(words);
    auto *c = (Context_ *)context;
    return guard([&] {
        if (count == 0)
            return;
        batch_handles(count, { cts });
        auto &a0 = *(Ciphertext_ *)cts[0];
        const u64 w = a0.words();
        if (cap < count * w)
            throw InvalidArg("capacity too small");
        SeamScope scope(c);
        std::vector<u64 *> ptrs(count);
        for (uint64_t i = 0; i < count; i++)
        {
            auto &a = *(Ciphertext_ *)cts[i];
            if (a.size != a0.size || a.k != a0.k || a.n != a0.n)
                throw InvalidArg("batch items must have the same shape");
            ptrs[i] = const_cast<u64 *>(a.dev_ptr(c));
        }
        if (w == 0)
            return;
        BatchSlab S(c, count * w);
        dev_check(b200_gather_scatter(c->dev, ptrs.data(), count, S.w(), w, 1, cur_stream()));
        dev_check(b200_memcpy_d2h(c->dev, words, S.p, count * w * sizeof(u64), cur_stream()));
        scope.wait(); // context mutex released while the copy runs
    });
}

// Test aid: what a combiner leader runs for `count` per-handle calls that arrived together, on the calling thread and
// without thread timing.  Each item goes through its per-handle call's validation; the validated requests run as the
// leader would take them (compatible ones as one batch, in item order) and each item gets its own HRESULT.
long B200_Evaluator_CombinedBatchDebug(void *p, int kind, uint64_t count, void **a, void **b, void *keys, uint32_t galois_elt,
                                       void **dsts, long *hresults)
{
    NULLRET(p);
    NULLRET(a);
    NULLRET(dsts);
    NULLRET(hresults);
    auto *c = ((Evaluator_ *)p)->ctx;
    if (kind < 0 || kind >= Context_::NCOMB || count == 0 || count > (uint64_t)Context_::COMBINE_MAX || (kind == 0 && !b) ||
        (kind != 0 && !keys))
        return E_INVALIDARG_;
    if (!c->combine || tl_scope)
        return COR_E_INVALIDOPERATION_; // no combiner to drive
    std::vector<CombineReq> reqs;
    std::vector<uint64_t> owner; // item of each collected request
    reqs.reserve(count);
    for (uint64_t i = 0; i < count; i++)
    {
        if (!a[i] || !dsts[i] || (kind == 0 && !b[i]))
        {
            hresults[i] = E_POINTER_;
            continue;
        }
        auto &A = *(Ciphertext_ *)a[i], &D = *(Ciphertext_ *)dsts[i];
        const size_t before = reqs.size();
        tl_collect = &reqs;
        hresults[i] = guard([&] { // an item its per-handle call would not combine runs here, as that call does
            if (kind == 0)
                op_multiply(c, A, *(Ciphertext_ *)b[i], D, false);
            else if (kind == 1)
                op_relinearize(c, A, *(KSwitchKeys_ *)keys, D);
            else if (!galois_combined(c, A, galois_elt, *(KSwitchKeys_ *)keys, D))
            {
                OpScope scope(c);
                op_galois(c, A, galois_elt, *(KSwitchKeys_ *)keys, D);
            }
        });
        tl_collect = nullptr;
        if (reqs.size() > before)
            owner.push_back(i);
    }
    std::vector<CombineReq *> pending;
    for (auto &r : reqs)
        pending.push_back(&r);
    while (!pending.empty())
    {
        std::vector<CombineReq *> batch{ pending[0] }, rest;
        for (size_t j = 1; j < pending.size(); j++)
            (pending[j]->compatible(*pending[0]) ? batch : rest).push_back(pending[j]);
        combine_run_batch(c, batch);
        pending.swap(rest);
    }
    for (size_t j = 0; j < reqs.size(); j++)
        hresults[owner[j]] = guard([&] {
            if (reqs[j].err)
                std::rethrow_exception(reqs[j].err);
        });
    return S_OK_;
}
long B200_Context_GraphStatsDebug(void *context, uint64_t *out)
{
    NULLRET(context);
    NULLRET(out);
    auto *c = (Context_ *)context;
    for (int i = 0; i < Context_::GS_COUNT; i++)
        out[i] = c->graph_stats[i].load();
    return S_OK_;
}

long B200_Evaluator_MultiplyRelinBatch(void *p, uint64_t count, void **e1, void **e2, void *relin_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(e1);
    NULLRET(e2);
    NULLRET(relin_keys);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)relin_keys;
    return guard([&] {
        if (count == 0)
            return;
        batch_handles(count, { e1, e2, dsts });
        SeamScope scope(c);
        const int lv = batch_level(c, count, e1);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
        BatchSlab A(c, count * w), B(c, count * w), D(c, count * w);
        batch_gather(c, count, e1, A);
        if (batch_level(c, count, e2) != lv)
            throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
        batch_gather(c, count, e2, B);
        check_keys(c, keys, 0);
        dev_check(b200_multiply_relin(c->dev, lv, A.w(), B.w(), keys.flat_dev(c, 0, (int)k), D.w(), count, cur_stream()));
        batch_scatter(c, count, dsts, D, ((Ciphertext_ *)e1[0])->parms_id, k, lv);
    });
}
long B200_Evaluator_AddSubBatch(void *p, uint64_t count, void **e1, void **e2, bool subtract, void **dsts)
{
    NULLRET(p);
    NULLRET(e1);
    NULLRET(e2);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        if (count == 0)
            return;
        batch_handles(count, { e1, e2, dsts });
        SeamScope scope(c);
        const int lv = batch_level(c, count, e1);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
        BatchSlab A(c, count * w), B(c, count * w);
        batch_gather(c, count, e1, A);
        if (batch_level(c, count, e2) != lv)
            throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
        batch_gather(c, count, e2, B);
        dev_check((subtract ? b200_sub : b200_add)(c->dev, lv, A.w(), B.w(), A.w(), 2, count, cur_stream()));
        batch_scatter(c, count, dsts, A, ((Ciphertext_ *)e1[0])->parms_id, k, lv);
    });
}
// which: 0 add_plain, 1 sub_plain, 2 multiply_plain; one plaintext per item
long B200_Evaluator_PlainBatch(void *p, int which, uint64_t count, void **encs, void **plains, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(plains);
    NULLRET(dsts);
    if (which < 0 || which > 2)
        return E_INVALIDARG_;
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        if (count == 0)
            return;
        batch_handles(count, { encs, plains, dsts });
        SeamScope scope(c);
        const size_t n = c->parms.n;
        const int lv = batch_level(c, count, encs);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * n;
        BatchSlab A(c, count * w), O(c, count * w), P(c, count * n);
        batch_gather(c, count, encs, A);
        std::vector<u64> host(count * n);
        for (uint64_t i = 0; i < count; i++)
        {
            NULLRET_THROW(plains[i]);
            std::vector<u64> pv = plain_operand(c, *(Plaintext_ *)plains[i], which == 2);
            std::copy(pv.begin(), pv.end(), host.begin() + i * n);
        }
        dev_check(b200_memcpy_h2d(c->dev, P.p, host.data(), host.size() * 8, cur_stream()));
        if (which == 0)
            dev_check(b200_add_plain(c->dev, lv, A.w(), 2, P.w(), count, O.w(), count, cur_stream()));
        else if (which == 1)
            dev_check(b200_sub_plain(c->dev, lv, A.w(), 2, P.w(), count, O.w(), count, cur_stream()));
        else
            dev_check(b200_multiply_plain(c->dev, lv, A.w(), 2, P.w(), count, O.w(), count, cur_stream()));
        tl_scope->wait(); // `host` is read by the copy above
        batch_scatter(c, count, dsts, O, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
    });
}
// the same row rotation applied to every item (the Galois key for `steps` must be present: no NAF fallback here)
long B200_Evaluator_RotateRowsBatch(void *p, uint64_t count, void **encs, int steps, void *galois_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(galois_keys);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)galois_keys;
    return guard([&] {
        if (count == 0)
            return;
        if (!c->using_batching)
            throw LogicErr("encryption parameters do not support batching");
        batch_handles(count, { encs, dsts });
        SeamScope scope(c);
        const int lv = batch_level(c, count, encs);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
        BatchSlab A(c, count * w), O(c, count * w);
        batch_gather(c, count, encs, A);
        if (steps == 0)
        {
            batch_scatter(c, count, dsts, A, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
            return;
        }
        const uint32_t elt = row_step_elt(c, steps);
        if (keys.parms_id != c->ids[0])
            throw InvalidArg("galois_keys is not valid for encryption parameters");
        const size_t index = galois_key_index(c, keys, elt);
        dev_check(b200_apply_galois(c->dev, lv, A.w(), elt, keys.flat_dev(c, index, (int)k), O.w(), count, cur_stream()));
        batch_scatter(c, count, dsts, O, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
    });
}
// Plaintext matrix x ciphertext vector: destinations[i] <- the words of multiply_plain(encrypteds[0], plains[i * cols]) followed
// by add_inplace(multiply_plain(encrypteds[j], plains[i * cols + j])) for j = 1 ... cols - 1.  The ciphertexts are gathered
// once; the plaintexts go through b200_plain_to_ntt (multiply rule) in chunks of rows whose NTT-form scratch stays below
// B200_PLAIN_SUM_SCRATCH bytes (default 1 GiB), each chunk one b200_multiply_plain_sum.  Every operand is read before the
// first scatter, so destinations may alias encrypteds.
long B200_Evaluator_MultiplyPlainSum(void *p, uint64_t rows, uint64_t cols, void **encs, void **plains, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(plains);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    return guard([&] {
        if (rows == 0)
            return;
        if (cols == 0)
            throw InvalidArg("a sum needs at least one term");
        batch_handles(cols, { encs });
        batch_handles(rows, { dsts });
        batch_handles(rows * cols, { plains });
        SeamScope scope(c);
        const size_t n = c->parms.n;
        auto &a0 = *(Ciphertext_ *)encs[0];
        const int lv = data_level(c, a0, "encrypted is not valid for encryption parameters");
        const u64 size = a0.size, k = a0.k, w = size * k * n;
        const ParmsId id = a0.parms_id;
        std::vector<u64 *> ptrs(cols);
        for (uint64_t j = 0; j < cols; j++)
        {
            auto &a = *(Ciphertext_ *)encs[j];
            if (data_level(c, a, "encrypted is not valid for encryption parameters") != lv)
                throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
            if (a.is_ntt_form)
                throw InvalidArg("BFV encrypted cannot be in NTT form");
            if (a.size != size)
                throw InvalidArg("all encrypteds must have the same size");
            ptrs[j] = const_cast<u64 *>(a.dev_ptr(c));
        }
        // the plaintext checks of the chain's multiply_plain, all before any work
        std::vector<u64> host(rows * cols * n);
        for (uint64_t i = 0; i < rows * cols; i++)
        {
            std::vector<u64> pv = plain_operand(c, *(Plaintext_ *)plains[i], true);
            std::copy(pv.begin(), pv.end(), host.begin() + i * n);
        }
        BatchSlab X(c, cols * w);
        dev_check(b200_gather_scatter(c->dev, ptrs.data(), cols, X.w(), w, 1, cur_stream()));
        uint64_t cap = 1ull << 30;
        if (const char *e = std::getenv("B200_PLAIN_SUM_SCRATCH"))
            cap = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
        const uint64_t chunk = std::max<uint64_t>(1, std::min<uint64_t>(rows, cap / (cols * k * n * sizeof(u64))));
        BatchSlab Pc(c, chunk * cols * n), Pn(c, chunk * cols * k * n), O(c, chunk * w);
        for (uint64_t i0 = 0; i0 < rows; i0 += chunk)
        {
            const uint64_t r = std::min(chunk, rows - i0);
            dev_check(b200_memcpy_h2d(c->dev, Pc.p, host.data() + i0 * cols * n, r * cols * n * sizeof(u64), cur_stream()));
            dev_check(b200_plain_to_ntt(c->dev, lv, Pc.w(), r * cols, Pn.w(), B200_PLAIN_NTT_MULTIPLY, cur_stream()));
            dev_check(b200_multiply_plain_sum(c->dev, lv, X.w(), (int)size, cols, Pn.w(), r, O.w(), cur_stream()));
            scope.wait(); // `host` is read by the copy above
            batch_scatter(c, r, dsts + i0, O, id, k, lv, size);
        }
    });
}

// Encrypted inner products: destinations[i] receives the words of the chain
//     c = Relinearize(Multiply(e1[i cols], e2[i cols]));  c = Add(c, Relinearize(Multiply(e1[i cols + j], e2[i cols + j]))), j >= 1
// as one b200_multiply_relin_sum over the gathered operands.  Every term is checked in chain order before any work: Multiply's
// metadata, level and NTT-form checks, then Relinearize's key and size checks.  A term whose operands are both transparent
// (the chain's Multiply result is transparent) is found on the gathered slabs before the sum runs.  A transparent partial sum
// is not detected, only a transparent final result.  Operands are gathered before the first scatter, so destinations may
// alias them.
long B200_Evaluator_MultiplyRelinSum(void *p, uint64_t rows, uint64_t cols, void **e1, void **e2, void *relin_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(e1);
    NULLRET(e2);
    NULLRET(relin_keys);
    NULLRET(dsts);
    if (rows == 0)
        return 0;
    if (cols == 0)
        return E_INVALIDARG_;
    const uint64_t terms = rows * cols;
    for (uint64_t i = 0; i < terms; i++)
    {
        NULLRET(e1[i]);
        NULLRET(e2[i]);
    }
    for (uint64_t i = 0; i < rows; i++)
        NULLRET(dsts[i]);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)relin_keys;
    return guard([&] {
        const int lv = data_level(c, *(Ciphertext_ *)e1[0], "encrypted1 is not valid for encryption parameters");
        bool same = true; // every term a square of one handle: one gathered slab serves both operands
        for (uint64_t t = 0; t < terms; t++)
        {
            auto &a = *(Ciphertext_ *)e1[t];
            auto &b = *(Ciphertext_ *)e2[t];
            // Multiply
            const int la = data_level(c, a, "encrypted1 is not valid for encryption parameters");
            data_level(c, b, "encrypted2 is not valid for encryption parameters");
            if (a.parms_id != b.parms_id || la != lv)
                throw InvalidArg("encrypted1 and encrypted2 parameter mismatch");
            if (a.is_ntt_form || b.is_ntt_form)
                throw InvalidArg("encrypted1 or encrypted2 cannot be in NTT form");
            if (a.size + b.size - 1 > 16)
                throw InvalidArg("invalid size");
            // Relinearize of the size a.size + b.size - 1 product
            if (keys.parms_id != c->ids[0])
                throw InvalidArg("relin_keys is not valid for encryption parameters");
            if (a.size != 2 || b.size != 2 || keys.keys.empty())
                throw InvalidArg("not enough relinearization keys");
            check_keys(c, keys, 0);
            if (keys.keys[0].size() < (size_t)a.k)
                throw InvalidArg("kswitch_keys is not valid for encryption parameters");
            same = same && e1[t] == e2[t];
        }
        SeamScope scope(c);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
        BatchSlab A(c, terms * w);
        std::unique_ptr<BatchSlab> B;
        batch_gather(c, terms, e1, A);
        if (!same)
        {
            B.reset(new BatchSlab(c, terms * w));
            batch_gather(c, terms, e2, *B);
        }
        const u64 *pb = same ? A.w() : B->w();
        if (c->check_transparent)
        { // the chain's Multiply refuses a product of two transparent operands
            BatchSlab flags(c, (terms + 1) / 2);
            std::vector<uint32_t> fa(terms), fb(terms);
            dev_check(b200_is_transparent(c->dev, lv, A.w(), 2, (uint32_t *)flags.p, terms, cur_stream()));
            dev_check(b200_memcpy_d2h(c->dev, fa.data(), flags.p, terms * 4, cur_stream()));
            scope.wait();
            if (same)
                fb = fa;
            else
            {
                dev_check(b200_is_transparent(c->dev, lv, pb, 2, (uint32_t *)flags.p, terms, cur_stream()));
                dev_check(b200_memcpy_d2h(c->dev, fb.data(), flags.p, terms * 4, cur_stream()));
                scope.wait();
            }
            for (uint64_t t = 0; t < terms; t++)
                if (fa[t] && fb[t])
                    throw LogicErr("result ciphertext is transparent");
        }
        BatchSlab O(c, rows * w);
        dev_check(b200_multiply_relin_sum(c->dev, lv, A.w(), pb, keys.flat_dev(c, 0, (int)k), cols, O.w(), rows, cur_stream()));
        batch_scatter(c, rows, dsts, O, ((Ciphertext_ *)e1[0])->parms_id, k, lv);
    });
}

// Rotate-and-sum slot reduction: destinations[i] receives the words of the chain
//     c = encrypteds[i];  for s in steps: c = Add(c, RotateRows(c, s));  if columns: c = Add(c, RotateColumns(c))
// A step whose key is present is one b200_apply_galois_add.  A step without its own key goes through its NAF parts as
// op_rotate does (parts of +-n/2 skipped): the intermediate parts as b200_apply_galois, the last one fused with the add.  Step 0
// adds c to itself.  Every step and key is checked before any work.  The items are gathered into one slab and the steps
// ping-pong between two slabs, so destinations may alias encrypteds.  Only the final result is checked for transparency: a
// transparent intermediate the chain would refuse is not detected (a transparent input, c1 = 0, stays transparent and is
// reported).
long B200_Evaluator_RotateSumBatch(void *p, uint64_t count, void **encs, int nsteps, const int *steps, bool columns,
                                   void *galois_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(galois_keys);
    NULLRET(dsts);
    if (nsteps > 0)
        NULLRET(steps);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)galois_keys;
    return guard([&] {
        if (count == 0)
            return;
        if (!c->using_batching)
            throw LogicErr("encryption parameters do not support batching");
        if (nsteps < 0)
            throw InvalidArg("nsteps must not be negative");
        batch_handles(count, { encs, dsts });
        if (keys.parms_id != c->ids[0])
            throw InvalidArg("galois_keys is not valid for encryption parameters");
        const size_t n = c->parms.n;
        // per step, the Galois elements the chain applies (empty: c + c)
        std::vector<std::vector<uint32_t>> plan;
        for (int i = 0; i < nsteps; i++)
        {
            std::vector<uint32_t> elts;
            if (steps[i] != 0)
                elts = row_rotation_elts(c, keys, steps[i]);
            for (uint32_t x : elts)
                galois_key_index(c, keys, x);
            plan.push_back(std::move(elts));
        }
        if (columns)
        {
            galois_key_index(c, keys, (uint32_t)(2 * n - 1));
            plan.push_back({ (uint32_t)(2 * n - 1) });
        }
        SeamScope scope(c);
        const int lv = batch_level(c, count, encs);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * n;
        BatchSlab A(c, count * w), B(c, count * w);
        std::unique_ptr<BatchSlab> T; // third slab for NAF steps of three or more parts
        batch_gather(c, count, encs, A);
        BatchSlab *cur = &A, *other = &B;
        auto key = [&](uint32_t e) { return keys.flat_dev(c, galois_key_index(c, keys, e), (int)k); };
        for (const auto &elts : plan)
        {
            if (elts.empty())
            {
                dev_check(b200_add(c->dev, lv, cur->w(), cur->w(), cur->w(), 2, count, cur_stream()));
                continue;
            }
            if (elts.size() == 1)
            {
                dev_check(b200_apply_galois_add(c->dev, lv, cur->w(), elts[0], key(elts[0]), cur->w(), other->w(), count, cur_stream()));
                std::swap(cur, other);
                continue;
            }
            // NAF parts: the intermediates alternate between `other` and T; the last part adds into cur in place
            if (elts.size() > 2 && !T)
                T.reset(new BatchSlab(c, count * w));
            const u64 *src = cur->w();
            for (size_t j = 0; j + 1 < elts.size(); j++)
            {
                u64 *dst = src == other->w() ? T->w() : other->w();
                dev_check(b200_apply_galois(c->dev, lv, src, elts[j], key(elts[j]), dst, count, cur_stream()));
                src = dst;
            }
            dev_check(b200_apply_galois_add(c->dev, lv, src, elts.back(), key(elts.back()), cur->w(), cur->w(), count, cur_stream()));
        }
        batch_scatter(c, count, dsts, *cur, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
    });
}

// Row rotations by a step per item.  The items are gathered in the order of their Galois elements (step 0 last, a copy), so
// each element's items are one run of one key, and rotated by one b200_apply_galois_many; the results are scattered back to
// their destinations.  Every operand is gathered before the scatter, so destinations may alias encrypteds.
long B200_Evaluator_RotateRowsStepsBatch(void *p, uint64_t count, void **encs, const int *steps, void *galois_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(steps);
    NULLRET(galois_keys);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)galois_keys;
    return guard([&] {
        if (count == 0)
            return;
        if (!c->using_batching)
            throw LogicErr("encryption parameters do not support batching");
        batch_handles(count, { encs, dsts });
        const int lv = batch_level(c, count, encs);
        if (!c->using_keyswitching)
            throw LogicErr("keyswitching is not supported by the context");
        if (keys.parms_id != c->ids[0])
            throw InvalidArg("galois_keys is not valid for encryption parameters");
        std::vector<uint32_t> elt(count, 0);
        std::vector<size_t> idx(count, 0);
        for (uint64_t i = 0; i < count; i++)
            if (steps[i] != 0)
                idx[i] = row_step_key(c, keys, steps[i], &elt[i]);
        std::vector<uint64_t> order(count);
        for (uint64_t i = 0; i < count; i++)
            order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](uint64_t x, uint64_t y) {
            return (elt[x] ? elt[x] : UINT32_MAX) < (elt[y] ? elt[y] : UINT32_MAX);
        });
        std::vector<void *> src(count), dst(count);
        for (uint64_t i = 0; i < count; i++)
        {
            src[i] = encs[order[i]];
            dst[i] = dsts[order[i]];
        }
        uint64_t m = 0; // items with a rotation
        while (m < count && elt[order[m]])
            m++;
        SeamScope scope(c);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
        BatchSlab A(c, count * w), O(c, count * w);
        batch_gather(c, count, src.data(), A);
        if (m)
        {
            std::vector<uint32_t> el(m);
            std::vector<const uint64_t *> kp(m);
            for (uint64_t i = 0; i < m; i++)
            {
                el[i] = elt[order[i]];
                kp[i] = keys.flat_dev(c, idx[order[i]], (int)k);
            }
            dev_check(b200_apply_galois_many(c->dev, lv, A.w(), nullptr, el.data(), kp.data(), O.w(), m, cur_stream()));
        }
        if (m < count)
            dev_check(b200_memcpy_d2d(c->dev, O.w() + m * w, A.w() + m * w, (count - m) * w * sizeof(u64), cur_stream()));
        batch_scatter(c, count, dst.data(), O, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
    });
}

// Baby-step giant-step linear transform: the chain of B200_Evaluator_LinearTransform (b200_sealc.h) as one
// b200_linear_transform over the gathered ciphertexts, with the present plaintexts lifted to NTT form once per call.  Every
// plaintext, step and key is checked before any work; operands are gathered before the scatter, so destinations may alias
// encrypteds.
long B200_Evaluator_LinearTransform(void *p, uint64_t count, void **encs, uint64_t baby, uint64_t giant, void **plains,
                                    void *galois_keys, void **dsts)
{
    NULLRET(p);
    NULLRET(encs);
    NULLRET(plains);
    NULLRET(galois_keys);
    NULLRET(dsts);
    auto *c = ((Evaluator_ *)p)->ctx;
    auto &keys = *(KSwitchKeys_ *)galois_keys;
    return guard([&] {
        if (count == 0)
            return;
        if (baby == 0 || giant == 0 || baby > (1u << 20) || giant > (1u << 20))
            throw InvalidArg("baby and giant must be at least 1");
        if (!c->using_batching)
            throw LogicErr("encryption parameters do not support batching");
        batch_handles(count, { encs, dsts });
        // each item on its own: items at different levels are refused after the plaintexts (a zero one is a LogicErr)
        for (uint64_t i = 0; i < count; i++)
            batch_level(c, 1, encs + i);
        const size_t n = c->parms.n;
        const uint64_t terms = baby * giant;
        std::vector<uint8_t> present(terms, 0);
        std::vector<char> ub(baby, 0), ug(giant, 0);
        std::vector<u64> host(terms * n, 0);
        for (uint64_t t = 0; t < terms; t++)
        {
            if (!plains[t])
                continue;
            std::vector<u64> pv = plain_operand(c, *(Plaintext_ *)plains[t], true);
            std::copy(pv.begin(), pv.end(), host.begin() + t * n);
            present[t] = 1;
            ub[t % baby] = ug[t / baby] = 1;
        }
        if (std::find(present.begin(), present.end(), 1) == present.end())
            throw InvalidArg("every term is absent");
        const uint64_t ns = baby - 1 + giant - 1;
        std::vector<uint32_t> elts(std::max<uint64_t>(ns, 1), 0);
        std::vector<size_t> idx(std::max<uint64_t>(ns, 1), 0);
        bool rotates = false;
        for (uint64_t j = 1; j < baby; j++)
            rotates = rotates || ub[j];
        for (uint64_t g = 1; g < giant; g++)
            rotates = rotates || ug[g];
        if (rotates)
        {
            if (!c->using_keyswitching)
                throw LogicErr("keyswitching is not supported by the context");
            if (keys.parms_id != c->ids[0])
                throw InvalidArg("galois_keys is not valid for encryption parameters");
        }
        for (uint64_t j = 1; j < baby; j++)
            if (ub[j])
                idx[j - 1] = row_step_key(c, keys, (int)j, &elts[j - 1]);
        for (uint64_t g = 1; g < giant; g++)
            if (ug[g])
            {
                if (g * baby >= n / 2)
                    throw InvalidArg("step count too large");
                idx[baby - 1 + g - 1] = row_step_key(c, keys, (int)(g * baby), &elts[baby - 1 + g - 1]);
            }
        SeamScope scope(c);
        const int lv = batch_level(c, count, encs);
        const u64 k = (u64)c->level_k[lv], w = 2 * k * n;
        BatchSlab A(c, count * w), O(c, count * w);
        batch_gather(c, count, encs, A);
        std::vector<const uint64_t *> kp(std::max<uint64_t>(ns, 1), nullptr);
        for (uint64_t e = 0; e < ns; e++)
            if (elts[e])
                kp[e] = keys.flat_dev(c, idx[e], (int)k);
        BatchSlab Pc(c, terms * n), Pn(c, terms * k * n);
        dev_check(b200_memcpy_h2d(c->dev, Pc.p, host.data(), host.size() * sizeof(u64), cur_stream()));
        dev_check(b200_plain_to_ntt(c->dev, lv, Pc.w(), terms, Pn.w(), B200_PLAIN_NTT_MULTIPLY, cur_stream()));
        dev_check(b200_linear_transform(c->dev, lv, A.w(), count, (int)baby, (int)giant, elts.data(), kp.data(), Pn.w(),
                                        present.data(), O.w(), cur_stream()));
        scope.wait(); // `host` is read by the copy above
        batch_scatter(c, count, dsts, O, ((Ciphertext_ *)encs[0])->parms_id, k, lv);
    });
}

// ---------------------------------------------------------------------------------------------------------
// Decryptor
// ---------------------------------------------------------------------------------------------------------
long Decryptor_Create(void *context, void *secret_key, void **out)
{
    NULLRET(context);
    NULLRET(secret_key);
    NULLRET(out);
    auto *c = (Context_ *)context;
    auto *sk = (SecretKey_ *)secret_key;
    if (!c->parameters_set)
        return E_INVALIDARG_;
    if (sk->data.parms_id != c->ids[0] || sk->data.coeffs.size() != c->parms.coeff.size() * c->parms.n)
        return E_INVALIDARG_; // "secret key is not valid for encryption parameters" (S/decryptor.cpp:54-77)
    auto *d = new Decryptor_();
    d->ctx = c;
    d->hold.bind(c);
    d->sk = sk->data.coeffs;
    *out = d;
    return S_OK_;
}
long Decryptor_Destroy(void *p)
{
    NULLRET(p);
    delete (Decryptor_ *)p;
    return S_OK_;
}
long Decryptor_Decrypt(void *p, void *enc, void *dst)
{
    NULLRET(p);
    NULLRET(enc);
    NULLRET(dst);
    auto *d = (Decryptor_ *)p;
    auto *c = d->ctx;
    auto &ct = *(Ciphertext_ *)enc;
    auto &pl = *(Plaintext_ *)dst;
    return guard([&] {
        std::lock_guard<std::mutex> lk(c->mu);
        int lv = data_level(c, ct, "encrypted is not valid for encryption parameters");
        if (ct.is_ntt_form)
            throw InvalidArg("encrypted cannot be in NTT form");
        const size_t n = c->parms.n;
        const u64 *pc = ct.dev_ptr(c);
        const u64 *pw = d->powers(lv, (int)ct.size - 1);
        void *dp = nullptr;
        dev_check(b200_malloc(c->dev, n * 8, &dp));
        std::vector<u64> out(n);
        int rc = b200_decrypt(c->dev, lv, pc, (int)ct.size, pw, (u64 *)dp, 1, nullptr);
        if (!rc)
            rc = b200_memcpy_d2h(c->dev, out.data(), dp, n * 8, nullptr);
        if (!rc)
            rc = b200_stream_synchronize(c->dev, nullptr);
        b200_free(c->dev, dp);
        dev_check(rc);
        // trim leading zero coefficients (S/decryptor.cpp:186-193)
        size_t cnt = n;
        while (cnt > 0 && out[cnt - 1] == 0)
            cnt--;
        pl.coeffs.assign(out.begin(), out.begin() + std::max<size_t>(cnt, 1));
        pl.parms_id = kZeroId;
        pl.scale = 1.0;
    });
}
// Decryptor::invariant_noise_internal (S/decryptor.cpp:424-485): infinity norm of the centred t * (ct . sk) mod Q as
// a multi-precision integer (little-endian words); also returns the level's residue count and bit length of Q
static void noise_norm(Decryptor_ *d, Ciphertext_ &ct, std::vector<u64> &norm_out, int &k_out, int &q_bits_out)
{
    auto *c = d->ctx;
    {
        // Decryptor::invariant_noise_budget (S/decryptor.cpp:424-527): norm of t * (ct . sk) mod Q, centred
        std::lock_guard<std::mutex> lk(c->mu);
        int lv = data_level(c, ct, "encrypted is not valid for encryption parameters");
        if (ct.is_ntt_form)
            throw InvalidArg("encrypted cannot be in NTT form");
        const int k = c->level_k[lv];
        const u64 *pc = ct.dev_ptr(c);
        const u64 *pw = d->powers(lv, (int)ct.size - 1);
        // phase on the GPU, then per coefficient t * phase CRT-composed mod Q, centred, and the maximum — also on the GPU
        // (noise_norm_kernel); only the norm's words come back
        b200::BigUInt Q(1);
        for (int i = 0; i < k; i++)
            Q.mul(c->parms.coeff[i]);
        const size_t W = Q.w.size();
        std::vector<u64> norm(W + 1, 0);
        dev_check(b200_noise_norm(c->dev, lv, pc, (int)ct.size, pw, norm.data(), (int)norm.size(), 1, nullptr));
        norm_out = norm;
        k_out = k;
        q_bits_out = Q.bit_length();
    }
}
// Decryptor::invariant_noise_budget (S/decryptor.cpp:512-527): bits of Q left above the noise norm, at least 0
static int noise_budget(const u64 *norm, size_t words, int q_bits)
{
    int nb = 0;
    for (size_t i = words; i-- > 0;)
        if (norm[i])
        {
            nb = (int)(64 * i + 64 - __builtin_clzll(norm[i]));
            break;
        }
    return std::max(0, q_bits - nb - 1);
}
long Decryptor_InvariantNoiseBudget(void *p, void *enc, int *budget)
{
    NULLRET(p);
    NULLRET(enc);
    NULLRET(budget);
    return guard([&] {
        std::vector<u64> norm;
        int k = 0, qbits = 0;
        noise_norm((Decryptor_ *)p, *(Ciphertext_ *)enc, norm, k, qbits);
        *budget = noise_budget(norm.data(), norm.size(), qbits);
    });
}
// Decryptor::invariant_noise (S/decryptor.cpp:487-510, added by the Sunscreen fork): the same norm as a double,
// divided by Q; the floating-point operations are issued in the reference's order so that the result is identical
long Decryptor_InvariantNoise(void *p, void *enc, double *invariant_noise)
{
    NULLRET(p);
    NULLRET(enc);
    NULLRET(invariant_noise);
    auto *d = (Decryptor_ *)p;
    return guard([&] {
        std::vector<u64> norm;
        int k = 0, qbits = 0;
        noise_norm(d, *(Ciphertext_ *)enc, norm, k, qbits);
        double v = 0.0;
        for (int i = 0; i < k; i++)
            v += (double)((size_t)i < norm.size() ? norm[i] : 0) * std::exp2((double)(64 * i));
        double total = 1.0;
        for (int i = 0; i < k; i++)
            total *= (double)d->ctx->parms.coeff[i];
        *invariant_noise = v / total;
    });
}

// ---------------------------------------------------------------------------------------------------------
// KeyGenerator (S/c/keygenerator.cpp -> S/keygenerator.cpp)
// ---------------------------------------------------------------------------------------------------------
long KeyGenerator_Create1(void *context, void **out)
{
    NULLRET(context);
    NULLRET(out);
    auto *c = (Context_ *)context;
    if (!c->parameters_set)
        return E_INVALIDARG_;
    auto *kg = new KeyGenerator_();
    kg->ctx = c;
    kg->hold.bind(c);
    long hr = guard([&] {
        std::lock_guard<std::mutex> lk(c->mu);
        const size_t n = c->parms.n, K = c->parms.coeff.size();
        // generate_sk (S/keygenerator.cpp:57-92): ternary sample, then NTT at the key level
        b200::Blake2xbPrng prng(b200::random_seed());
        std::vector<u64> s(K * n);
        WipeGuard wg(s);
        b200::sample_poly_ternary(prng, n, c->parms.coeff, s.data());
        DevBuf d(c, s);
        dev_check(b200_ntt_forward(c->dev, 0, d.p, 1, nullptr));
        kg->sk = d.download();
    });
    if (hr)
    {
        delete kg;
        return hr;
    }
    *out = kg;
    return S_OK_;
}
long KeyGenerator_Create2(void *context, void *secret_key, void **out)
{
    NULLRET(context);
    NULLRET(secret_key);
    NULLRET(out);
    auto *c = (Context_ *)context;
    auto *sk = (SecretKey_ *)secret_key;
    if (!c->parameters_set || sk->data.parms_id != c->ids[0] || sk->data.coeffs.size() != c->parms.coeff.size() * c->parms.n)
        return E_INVALIDARG_;
    auto *kg = new KeyGenerator_();
    kg->ctx = c;
    kg->hold.bind(c);
    kg->sk = sk->data.coeffs;
    *out = kg;
    return S_OK_;
}
long KeyGenerator_Destroy(void *p)
{
    NULLRET(p);
    delete (KeyGenerator_ *)p;
    return S_OK_;
}
long KeyGenerator_SecretKey(void *p, void **out)
{
    NULLRET(p);
    NULLRET(out);
    auto *kg = (KeyGenerator_ *)p;
    auto *sk = new SecretKey_();
    sk->data.coeffs = kg->sk;
    sk->data.parms_id = kg->ctx->ids[0];
    *out = sk;
    return S_OK_;
}
long KeyGenerator_CreatePublicKey(void *p, bool /*save_seed*/, void **out)
{
    NULLRET(p);
    NULLRET(out);
    auto *kg = (KeyGenerator_ *)p;
    auto *c = kg->ctx;
    auto *pk = new PublicKey_();
    long hr = guard([&] {
        std::lock_guard<std::mutex> lk(c->mu);
        b200::Blake2xbPrng bootstrap(b200::random_seed());
        pk->data.host = encrypt_zero_symmetric_key_level(c, kg->dev_sk(), bootstrap); // generate_pk (S/keygenerator.cpp:94-122)
        pk->data.host_valid = true;
        pk->data.parms_id = c->ids[0];
        pk->data.size = 2;
        pk->data.k = c->parms.coeff.size();
        pk->data.n = c->parms.n;
        pk->data.is_ntt_form = true;
    });
    if (hr)
    {
        delete pk;
        return hr;
    }
    *out = pk;
    return S_OK_;
}
long KeyGenerator_CreateRelinKeys(void *p, bool /*save_seed*/, void **out)
{
    NULLRET(p);
    NULLRET(out);
    auto *kg = (KeyGenerator_ *)p;
    auto *c = kg->ctx;
    if (!c->using_keyswitching)
        return COR_E_INVALIDOPERATION_;
    auto *keys = new KSwitchKeys_();
    long hr = guard([&] {
        std::lock_guard<std::mutex> lk(c->mu);
        const size_t n = c->parms.n, K = c->parms.coeff.size();
        // s^2 in NTT form (compute_secret_key_array, S/keygenerator.cpp:245-300), then one key list (index 0)
        DevBuf ds(c, kg->sk), d2(c, K * n);
        dev_check(b200_dyadic_product(c->dev, 0, ds.p, 1, ds.p, 1, d2.p, 1, nullptr));
        std::vector<u64> s2 = d2.download();
        keys->keys.emplace_back();
        kg->one_kswitch_key(s2, keys->keys[0]);
        keys->parms_id = c->ids[0];
    });
    if (hr)
    {
        delete keys;
        return hr;
    }
    *out = keys;
    return S_OK_;
}
static long create_galois(KeyGenerator_ *kg, const std::vector<uint32_t> &elts, void **out)
{
    auto *c = kg->ctx;
    if (!c->using_keyswitching)
        return COR_E_INVALIDOPERATION_;
    auto *keys = new KSwitchKeys_();
    long hr = guard([&] {
        std::lock_guard<std::mutex> lk(c->mu);
        const size_t n = c->parms.n, K = c->parms.coeff.size();
        int logn = 0;
        while (((size_t)1 << logn) < n)
            logn++;
        keys->keys.resize(n);
        for (uint32_t elt : elts)
        {
            if (!(elt & 1) || elt >= 2 * n)
                throw InvalidArg("Galois element is not valid");
            const size_t index = (elt - 1) >> 1;
            if (!keys->keys[index].empty())
                continue;
            // apply_galois_ntt: a permutation of the NTT slots (S/util/galois.cpp:18-50,192-218)
            std::vector<u64> rot(K * n);
            for (size_t i = 0; i < n; i++)
            {
                const uint32_t rev = (uint32_t)b200::reverse_bits(n + i, logn + 1);
                const u64 raw = (((u64)elt * rev) >> 1) & (n - 1);
                const size_t src = (size_t)b200::reverse_bits(raw, logn);
                for (size_t r = 0; r < K; r++)
                    rot[r * n + i] = kg->sk[r * n + src];
            }
            kg->one_kswitch_key(rot, keys->keys[index]);
        }
        keys->parms_id = c->ids[0];
    });
    if (hr)
    {
        delete keys;
        return hr;
    }
    *out = keys;
    return S_OK_;
}
long KeyGenerator_CreateGaloisKeysFromElts(void *p, uint64_t count, uint32_t *elts, bool, void **out)
{
    NULLRET(p);
    NULLRET(elts);
    NULLRET(out);
    return create_galois((KeyGenerator_ *)p, std::vector<uint32_t>(elts, elts + count), out);
}
long KeyGenerator_CreateGaloisKeysFromSteps(void *p, uint64_t count, int *steps, bool, void **out)
{
    NULLRET(p);
    NULLRET(steps);
    NULLRET(out);
    auto *kg = (KeyGenerator_ *)p;
    if (!kg->ctx->using_batching)
        return COR_E_INVALIDOPERATION_;
    std::vector<uint32_t> elts;
    for (uint64_t i = 0; i < count; i++)
    {
        uint32_t e;
        if (b200_galois_elt_from_step(kg->ctx->dev, steps[i], &e))
            return E_INVALIDARG_;
        elts.push_back(e);
    }
    return create_galois(kg, elts, out);
}
long KeyGenerator_CreateGaloisKeysAll(void *p, bool, void **out)
{
    NULLRET(p);
    NULLRET(out);
    auto *kg = (KeyGenerator_ *)p;
    if (!kg->ctx->using_batching)
        return COR_E_INVALIDOPERATION_;
    // GaloisTool::get_elts_all (S/util/galois.cpp:106-131)
    const uint32_t m = (uint32_t)(2 * kg->ctx->parms.n);
    int logn = 0;
    while (((size_t)1 << logn) < kg->ctx->parms.n)
        logn++;
    std::vector<uint32_t> elts{ m - 1 };
    u64 pos = 3, neg = b200::inv_mod(3, m);
    for (int i = 0; i < logn - 1; i++)
    {
        elts.push_back((uint32_t)pos);
        pos = (pos * pos) & (m - 1);
        elts.push_back((uint32_t)neg);
        neg = (neg * neg) & (m - 1);
    }
    return create_galois(kg, elts, out);
}

// ---------------------------------------------------------------------------------------------------------
// Encryptor (S/c/encryptor.cpp -> S/encryptor.cpp:114-321)
// ---------------------------------------------------------------------------------------------------------
long Encryptor_Create(void *context, void *public_key, void *secret_key, void **out)
{
    NULLRET(context);
    NULLRET(out);
    auto *c = (Context_ *)context;
    if (!public_key && !secret_key)
        return E_POINTER_; // S/c/encryptor.cpp:46-49
    if (!c->parameters_set)
        return E_INVALIDARG_;
    auto *e = new Encryptor_();
    e->ctx = c;
    e->hold.bind(c);
    long hr = guard([&] {
        const size_t words = c->parms.coeff.size() * c->parms.n;
        if (public_key)
        {
            auto &d = ((PublicKey_ *)public_key)->data;
            d.sync_host();
            if (d.parms_id != c->ids[0] || d.host.size() != 2 * words)
                throw InvalidArg("public key is not valid for encryption parameters");
            e->pk = d.host;
            e->has_pk = true;
        }
        if (secret_key)
        {
            auto &d = ((SecretKey_ *)secret_key)->data;
            if (d.parms_id != c->ids[0] || d.coeffs.size() != words)
                throw InvalidArg("secret key is not valid for encryption parameters");
            e->sk = d.coeffs;
            e->has_sk = true;
        }
    });
    if (hr)
    {
        delete e;
        return hr;
    }
    *out = e;
    return S_OK_;
}
long Encryptor_Destroy(void *p)
{
    NULLRET(p);
    delete (Encryptor_ *)p;
    return S_OK_;
}

// Encryption (S/encryptor.cpp:160-321) in two steps: the host sampling (b200_sample_pk / b200_sample_sk), done before the
// operation scope so that it holds no lock of the context — threads that encrypt at the same time sample in parallel and
// serialise only for the device part — then one launch sequence for the batch (b200_encrypt_pk_samples / _sk_samples).  Every
// entry point, per-handle ones included, is a batch.  The key is checked before the plaintexts, as the reference checks them.
static void encrypt_key_check(Encryptor_ *e, bool symmetric)
{
    if (symmetric ? !e->has_sk : !e->has_pk)
        throw LogicErr(symmetric ? "secret key is not set" : "public key is not set");
}
// plains[i] padded to n coefficients, host [count][n], each checked as Encryptor::encrypt checks it (is_valid_for)
static std::vector<u64> encrypt_plains(Context_ *c, uint64_t count, void *const *plains)
{
    const size_t n = c->parms.n;
    std::vector<u64> host(count * n);
    for (uint64_t i = 0; i < count; i++)
    {
        std::vector<u64> v = padded_plain(c, *(const Plaintext_ *)plains[i]);
        std::copy(v.begin(), v.end(), host.begin() + i * n);
    }
    return host;
}
// a batch seam writes each destination once: a handle listed twice is refused (the scatter writes the items concurrently)
static void distinct_destinations(uint64_t count, void *const *dsts)
{
    std::vector<void *> v(dsts, dsts + count);
    std::sort(v.begin(), v.end());
    if (std::adjacent_find(v.begin(), v.end()) != v.end())
        throw InvalidArg("destinations must be distinct");
}
// The host samples of one call: pk u, e0, e1 ([count][3][n]) or sk e ([count][n]) and c1 ([count][k][n], public).  The small
// samples, and the seeds drawn for an unseeded call (which determine them), are wiped when the call is done.
struct EncSamples
{
    std::vector<int8_t> small;
    std::vector<u64> c1, seeds;
    ~EncSamples()
    {
        explicit_bzero(small.data(), small.size());
        wipe(seeds);
    }
};
// seeds: host [count][8], or NULL for a fresh random seed per item
static void encrypt_sample(Context_ *c, uint64_t count, const uint64_t *seeds, bool symmetric, EncSamples &S)
{
    const size_t n = c->parms.n, k = (size_t)c->level_k[c->first_level];
    if (!seeds)
    {
        S.seeds.resize(count * 8);
        for (uint64_t i = 0; i < count; i++)
        {
            b200::PrngSeed sd = b200::random_seed();
            std::copy(sd.begin(), sd.end(), S.seeds.begin() + i * 8);
            explicit_bzero(sd.data(), sizeof(sd));
        }
        seeds = S.seeds.data();
    }
    if (symmetric)
    {
        S.c1.resize(count * k * n);
        S.small.resize(count * n);
        dev_check(b200_sample_sk(c->dev, seeds, S.c1.data(), S.small.data(), count));
    }
    else
    {
        S.small.resize(count * 3 * n);
        dev_check(b200_sample_pk(c->dev, seeds, S.small.data(), count));
    }
}
// dsts[i] <- the encryption of plaintext row i of the device slab P [count][n] (checked) with the samples S, at the first data
// level.  Runs inside the caller's SeamScope; the caller waits before S goes away.
static void encrypt_device(Encryptor_ *e, uint64_t count, const BatchSlab &P, const EncSamples &S, bool symmetric, bool dsm,
                           void *const *dsts)
{
    Context_ *c = e->ctx;
    const int lv = c->first_level;
    const u64 k = (u64)c->level_k[lv], w = 2 * k * c->parms.n;
    // one item is encrypted straight into its destination; a batch into a slab, then scattered
    std::unique_ptr<BatchSlab> O(count > 1 ? new BatchSlab(c, count * w) : nullptr);
    u64 *out = O ? O->w() : ((Ciphertext_ *)dsts[0])->prepare_output(c, c->ids[lv], 2, k);
    if (symmetric)
        dev_check(b200_encrypt_sk_samples(c->dev, e->dev_sk(), S.c1.data(), S.small.data(), P.w(), out, count, cur_stream()));
    else
        dev_check(b200_encrypt_pk_samples(c->dev, e->dev_pk(), S.small.data(), P.w(), dsm ? 1 : 0, out, count, cur_stream()));
    if (!O)
        return;
    std::vector<u64 *> ptrs(count);
    for (uint64_t i = 0; i < count; i++)
        ptrs[i] = ((Ciphertext_ *)dsts[i])->prepare_output(c, c->ids[lv], 2, k);
    const uint64_t chunk = 65535; // items per b200_gather_scatter
    for (uint64_t i0 = 0; i0 < count; i0 += chunk)
        dev_check(b200_gather_scatter(c->dev, ptrs.data() + i0, std::min(chunk, count - i0), O->w() + i0 * w, w, 0, cur_stream()));
}
// plaintext handles -> ciphertexts, every item checked before any work; S receives the samples
static void encrypt_batch(Encryptor_ *e, uint64_t count, void *const *plains, const uint64_t *seeds, bool symmetric, bool dsm,
                          void *const *dsts, EncSamples &S)
{
    Context_ *c = e->ctx;
    encrypt_key_check(e, symmetric);
    const std::vector<u64> host = encrypt_plains(c, count, plains);
    if (count == 0)
        return;
    encrypt_sample(c, count, seeds, symmetric, S);
    SeamScope scope(c);
    BatchSlab P(c, host.size());
    dev_check(b200_memcpy_h2d(c->dev, P.p, host.data(), host.size() * sizeof(u64), cur_stream()));
    encrypt_device(e, count, P, S, symmetric, dsm, dsts);
    scope.wait(); // the device has read the samples
}

// Components of an encryption as the reference exports them (S/util/rlwe.cpp:243-288,403-407; S/util/scalingvariant.cpp:96-119)
struct EncComponents
{
    PolynomialArray_ *u = nullptr, *e = nullptr;
    Plaintext_ *remainder = nullptr;
};

// round(Q m / t) correction term of every plaintext coefficient: fix = floor(((Q mod t) m + floor((t+1)/2)) / t)
static void export_remainder(Context_ *c, const Plaintext_ &plain, Plaintext_ &dst)
{
    b200_level_info li;
    dev_check(b200_ctx_level_info(c->dev, c->first_level, &li));
    const u64 t = c->parms.plain, half = (t + 1) >> 1;
    Plaintext_ r;
    r.coeffs.resize(plain.coeffs.size());
    for (size_t i = 0; i < plain.coeffs.size(); i++)
        r.coeffs[i] = (u64)(((unsigned __int128)plain.coeffs[i] * li.q_mod_t + half) / t);
    dst = std::move(r);
}

// Encryptor_Encrypt{,Symmetric}ReturnComponents{,SetSeed} (S/c/encryptor.cpp:136-240,300-372): the fork's entry points
// that also hand back u, e and the rounding remainder; `seed8` == nullptr draws a fresh seed.  u and e are the residues, at
// the level the zero encryption is made at, of the samples layer 1 hands back.
static long encrypt_components(void *p, void *plaintext, bool asymmetric, bool disable_special_modulus, void *destination,
                               void *u_dst, void *e_dst, void *r_dst, const uint64_t *seed8)
{
    auto *e = (Encryptor_ *)p;
    return guard([&] {
        Context_ *c = e->ctx;
        EncComponents comp{ (PolynomialArray_ *)u_dst, (PolynomialArray_ *)e_dst, (Plaintext_ *)r_dst };
        // the component arrays must be fresh: reserve() refuses a second use, like the reference's
        if ((comp.u && comp.u->reserved) || (comp.e && comp.e->reserved))
            throw LogicErr("PolynomialArray can only be reserved once.");
        const size_t n = c->parms.n;
        EncSamples S;
        encrypt_batch(e, 1, &plaintext, seed8, !asymmetric, disable_special_modulus, &destination, S);
        const int8_t *smp = S.small.data();
        // pk: encrypted at the key level unless the special modulus is disabled (S/encryptor.cpp:160-163)
        const int enc_lv = asymmetric && c->first_level == 1 && !disable_special_modulus ? 0 : c->first_level;
        const std::vector<u64> mods(c->parms.coeff.begin(), c->parms.coeff.begin() + c->level_k[enc_lv]);
        if (comp.u)
        {
            comp.u->reserve(1, n, mods);
            comp.u->insert(0, expand_signed_host(smp, n, mods).data());
        }
        if (comp.e)
        {
            const size_t polys = asymmetric ? 2 : 1, first = asymmetric ? 1 : 0;
            comp.e->reserve(polys, n, mods);
            for (size_t j = 0; j < polys; j++)
                comp.e->insert(j, expand_signed_host(smp + (first + j) * n, n, mods).data());
        }
        if (comp.remainder)
            export_remainder(c, *(Plaintext_ *)plaintext, *comp.remainder);
    });
}
long Encryptor_EncryptReturnComponents(void *p, void *plaintext, bool disable_special_modulus, void *destination, void *u_dst,
                                       void *e_dst, void *r_dst, void *)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    NULLRET(u_dst);
    NULLRET(e_dst);
    NULLRET(r_dst);
    return encrypt_components(p, plaintext, true, disable_special_modulus, destination, u_dst, e_dst, r_dst, nullptr);
}
long Encryptor_EncryptReturnComponentsSetSeed(void *p, void *plaintext, bool disable_special_modulus, void *destination,
                                              void *u_dst, void *e_dst, void *r_dst, void *seed, void *)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    NULLRET(u_dst);
    NULLRET(e_dst);
    NULLRET(r_dst);
    NULLRET(seed);
    return encrypt_components(p, plaintext, true, disable_special_modulus, destination, u_dst, e_dst, r_dst, (const uint64_t *)seed);
}
long Encryptor_EncryptSymmetricReturnComponents(void *p, void *plaintext, void *destination, void *e_dst, void *r_dst, void *)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    NULLRET(e_dst);
    NULLRET(r_dst);
    return encrypt_components(p, plaintext, false, false, destination, nullptr, e_dst, r_dst, nullptr);
}
long Encryptor_EncryptSymmetricReturnComponentsSetSeed(void *p, void *plaintext, void *destination, void *e_dst, void *r_dst,
                                                       void *seed, void *)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    NULLRET(e_dst);
    NULLRET(r_dst);
    NULLRET(seed);
    return encrypt_components(p, plaintext, false, false, destination, nullptr, e_dst, r_dst, (const uint64_t *)seed);
}

long Encryptor_Encrypt(void *p, void *plaintext, void *destination, void *)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    return guard([&] {
        EncSamples S;
        encrypt_batch((Encryptor_ *)p, 1, &plaintext, nullptr, false, false, &destination, S);
    });
}
// deterministic variant: same stream as the reference's Encryptor_EncryptReturnComponentsSetSeed (S/c/encryptor.cpp:185-240)
long B200_Encryptor_EncryptSetSeed(void *p, void *plaintext, const uint64_t *seed8, void *destination)
{
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(seed8);
    NULLRET(destination);
    return guard([&] {
        EncSamples S;
        encrypt_batch((Encryptor_ *)p, 1, &plaintext, seed8, false, false, &destination, S);
    });
}
long Encryptor_EncryptSymmetric(void *p, void *plaintext, bool /*save_seed*/, void *destination, void *)
{
    // save_seed only changes how the result is later serialised (S/util/rlwe.cpp:441-457); the ciphertext handed
    // back here is always the expanded one, which every consumer accepts
    NULLRET(p);
    NULLRET(plaintext);
    NULLRET(destination);
    return guard([&] {
        EncSamples S;
        encrypt_batch((Encryptor_ *)p, 1, &plaintext, nullptr, true, false, &destination, S);
    });
}
long B200_Encryptor_EncryptBatch(void *encryptor, uint64_t count, void **plains, const uint64_t *seeds, bool symmetric,
                                 void **destinations)
{
    NULLRET(encryptor);
    NULLRET(plains);
    NULLRET(destinations);
    return guard([&] {
        batch_handles(count, { plains, destinations });
        distinct_destinations(count, destinations);
        EncSamples S;
        encrypt_batch((Encryptor_ *)encryptor, count, plains, seeds, symmetric, false, destinations, S);
    });
}
long B200_Encryptor_EncryptSlotsBatch(void *encryptor, void *encoder, uint64_t count, uint64_t values_per_item,
                                      const uint64_t *values, bool is_signed, const uint64_t *seeds, bool symmetric,
                                      void **destinations)
{
    NULLRET(encryptor);
    NULLRET(encoder);
    NULLRET(destinations);
    if (count && values_per_item)
        NULLRET(values);
    auto *e = (Encryptor_ *)encryptor;
    Context_ *c = e->ctx;
    if (((BatchEncoder_ *)encoder)->ctx != c)
        return E_INVALIDARG_;
    return guard([&] {
        batch_handles(count, { destinations });
        distinct_destinations(count, destinations);
        if (!c->using_batching)
            throw InvalidArg("encryption parameters are not valid for batching");
        encrypt_key_check(e, symmetric);
        if (values_per_item > c->parms.n)
            throw InvalidArg("values_matrix size is too large");
        if (count == 0)
            return;
        EncSamples S;
        encrypt_sample(c, count, seeds, symmetric, S);
        SeamScope scope(c);
        const size_t n = c->parms.n;
        BatchSlab V(c, count * values_per_item), P(c, count * n);
        if (values_per_item)
            dev_check(b200_memcpy_h2d(c->dev, V.p, values, count * values_per_item * sizeof(u64), cur_stream()));
        dev_check(b200_batch_encode(c->dev, V.w(), values_per_item, is_signed ? 1 : 0, P.w(), count, cur_stream()));
        encrypt_device(e, count, P, S, symmetric, false, destinations);
        scope.wait();
    });
}

// ---------------------------------------------------------------------------------------------------------
// BatchEncoder (S/c/batchencoder.cpp -> S/batchencoder.cpp): slot permutation and NTT mod t on the GPU (b200_batch_encode /
// b200_batch_decode); the per-handle calls are batches of one
// ---------------------------------------------------------------------------------------------------------
long BatchEncoder_Create(void *context, void **out)
{
    NULLRET(context);
    NULLRET(out);
    auto *c = (Context_ *)context;
    if (!c->parameters_set || !c->using_batching)
        return E_INVALIDARG_; // "encryption parameters are not valid for batching"
    auto *b = new BatchEncoder_();
    b->ctx = c;
    b->hold.bind(c);
    *out = b;
    return S_OK_;
}
long BatchEncoder_Destroy(void *p)
{
    NULLRET(p);
    delete (BatchEncoder_ *)p;
    return S_OK_;
}
long BatchEncoder_GetSlotCount(void *p, uint64_t *count)
{
    NULLRET(p);
    NULLRET(count);
    *count = ((BatchEncoder_ *)p)->ctx->parms.n;
    return S_OK_;
}
// dsts[i] <- the plaintext of row i of values [count][per] (host), one transfer each way.  The reference range-checks the
// values only in SEAL_DEBUG builds (S/batchencoder.cpp:110-193): unsigned values are reduced mod t, signed ones lifted first.
static void encode_rows(BatchEncoder_ *b, uint64_t count, uint64_t per, const u64 *values, bool is_signed, Plaintext_ *const *dsts)
{
    Context_ *c = b->ctx;
    const size_t n = c->parms.n;
    if (per > n)
        throw InvalidArg("values_matrix size is too large");
    if (count == 0)
        return;
    SeamScope scope(c);
    BatchSlab V(c, count * per), P(c, count * n);
    if (per)
        dev_check(b200_memcpy_h2d(c->dev, V.p, values, count * per * sizeof(u64), cur_stream()));
    dev_check(b200_batch_encode(c->dev, V.w(), per, is_signed ? 1 : 0, P.w(), count, cur_stream()));
    std::vector<u64> host(count * n);
    dev_check(b200_memcpy_d2h(c->dev, host.data(), P.p, host.size() * sizeof(u64), cur_stream()));
    scope.wait();
    for (uint64_t i = 0; i < count; i++)
    {
        Plaintext_ &dst = *dsts[i];
        dst.coeffs.assign(host.begin() + i * n, host.begin() + (i + 1) * n);
        dst.parms_id = kZeroId;
        dst.scale = 1.0;
    }
}
// out (host [count][n]) <- the slots of plains[i], every plaintext checked first as BatchEncoder::decode checks it; signed:
// centred (S/batchencoder.cpp:317-360)
static void decode_rows(BatchEncoder_ *b, uint64_t count, void *const *plains, bool is_signed, void *out)
{
    Context_ *c = b->ctx;
    const size_t n = c->parms.n;
    std::vector<u64> host(count * n);
    for (uint64_t i = 0; i < count; i++)
    {
        const Plaintext_ &pl = *(const Plaintext_ *)plains[i];
        if (pl.parms_id != kZeroId)
            throw InvalidArg("plain cannot be in NTT form");
        std::vector<u64> v = padded_plain(c, pl);
        std::copy(v.begin(), v.end(), host.begin() + i * n);
    }
    if (count == 0)
        return;
    SeamScope scope(c);
    BatchSlab P(c, count * n), S(c, count * n);
    dev_check(b200_memcpy_h2d(c->dev, P.p, host.data(), host.size() * sizeof(u64), cur_stream()));
    dev_check(b200_batch_decode(c->dev, P.w(), is_signed ? 1 : 0, S.w(), count, cur_stream()));
    dev_check(b200_memcpy_d2h(c->dev, out, S.p, count * n * sizeof(u64), cur_stream()));
    scope.wait();
}
long BatchEncoder_Encode1(void *p, uint64_t count, uint64_t *values, void *destination)
{
    NULLRET(p);
    NULLRET(destination);
    if (count)
        NULLRET(values);
    Plaintext_ *dst = (Plaintext_ *)destination;
    return guard([&] { encode_rows((BatchEncoder_ *)p, 1, count, values, false, &dst); });
}
long BatchEncoder_Encode2(void *p, uint64_t count, int64_t *values, void *destination)
{
    NULLRET(p);
    NULLRET(destination);
    if (count)
        NULLRET(values);
    Plaintext_ *dst = (Plaintext_ *)destination;
    return guard([&] { encode_rows((BatchEncoder_ *)p, 1, count, (const u64 *)values, true, &dst); });
}
long BatchEncoder_Decode1(void *p, void *plain, uint64_t *count, uint64_t *destination, void *)
{
    NULLRET(p);
    NULLRET(plain);
    NULLRET(count);
    NULLRET(destination);
    auto *b = (BatchEncoder_ *)p;
    return guard([&] {
        decode_rows(b, 1, &plain, false, destination);
        *count = b->ctx->parms.n;
    });
}
long BatchEncoder_Decode2(void *p, void *plain, uint64_t *count, int64_t *destination, void *)
{
    NULLRET(p);
    NULLRET(plain);
    NULLRET(count);
    NULLRET(destination);
    auto *b = (BatchEncoder_ *)p;
    return guard([&] {
        decode_rows(b, 1, &plain, true, destination);
        *count = b->ctx->parms.n;
    });
}
long B200_BatchEncoder_EncodeBatch(void *encoder, uint64_t count, uint64_t values_per_item, const uint64_t *values, bool is_signed,
                                   void **destinations)
{
    NULLRET(encoder);
    NULLRET(destinations);
    if (count && values_per_item)
        NULLRET(values);
    return guard([&] {
        batch_handles(count, { destinations });
        encode_rows((BatchEncoder_ *)encoder, count, values_per_item, values, is_signed, (Plaintext_ *const *)destinations);
    });
}
long B200_BatchEncoder_DecodeBatch(void *encoder, uint64_t count, void **plains, bool is_signed, void *slots_out)
{
    NULLRET(encoder);
    NULLRET(plains);
    NULLRET(slots_out);
    return guard([&] {
        batch_handles(count, { plains });
        decode_rows((BatchEncoder_ *)encoder, count, plains, is_signed, slots_out);
    });
}
long B200_Decryptor_DecryptSlotsBatch(void *decryptor, void *encoder, uint64_t count, void **encs, bool is_signed, void *slots_out,
                                      int *budgets)
{
    NULLRET(decryptor);
    NULLRET(encoder);
    NULLRET(encs);
    NULLRET(slots_out);
    auto *d = (Decryptor_ *)decryptor;
    auto *c = d->ctx;
    if (((BatchEncoder_ *)encoder)->ctx != c)
        return E_INVALIDARG_;
    return guard([&] {
        batch_handles(count, { encs });
        if (count == 0)
            return;
        const Ciphertext_ &first = *(const Ciphertext_ *)encs[0];
        int lv = -1;
        for (uint64_t i = 0; i < count; i++)
        {
            const Ciphertext_ &ct = *(const Ciphertext_ *)encs[i];
            const int l = data_level(c, ct, "encrypted is not valid for encryption parameters");
            if (ct.is_ntt_form)
                throw InvalidArg("encrypted cannot be in NTT form");
            if (i == 0)
                lv = l;
            else if (l != lv || ct.size != first.size)
                throw InvalidArg("batch items must be ciphertexts of one size at one level");
        }
        SeamScope scope(c);
        const size_t n = c->parms.n;
        const int size = (int)first.size, k = c->level_k[lv];
        const u64 *pw = d->powers(lv, size - 1);
        b200::BigUInt Q(1);
        for (int i = 0; i < k; i++)
            Q.mul(c->parms.coeff[i]);
        const size_t words = Q.w.size() + 1;
        std::vector<u64> norm(budgets ? count * words : 0);
        BatchSlab A(c, count * first.words()), S(c, count * n);
        batch_gather(c, count, encs, A);
        dev_check(b200_decrypt_slots(c->dev, lv, A.w(), size, pw, is_signed ? 1 : 0, S.w(), budgets ? norm.data() : nullptr,
                                     (int)words, count, cur_stream()));
        dev_check(b200_memcpy_d2h(c->dev, slots_out, S.p, count * n * sizeof(u64), cur_stream()));
        scope.wait();
        if (budgets)
            for (uint64_t i = 0; i < count; i++)
                budgets[i] = noise_budget(norm.data() + i * words, words, Q.bit_length());
    });
}

} // extern "C"
