"""The combining layer of the per-handle calls (sealc_api.cpp: combine_run_batch) against the unmodified reference.

Concurrent Evaluator_Multiply / Evaluator_Relinearize / Evaluator_RotateRows calls are run as one batch, padded to a power of
two NP, through per-lane pinned pointer tables; a batch shape (kind, level, NP, key, Galois element) runs kernel by kernel on
first sight, is captured as a CUDA graph on its second use and replayed after that, at most 48 shapes per lane (least
recently used evicted).  B200_Evaluator_CombinedBatchDebug runs exactly what a combiner leader runs, on the calling thread,
so every check here knows its batch size; B200_Context_GraphStatsDebug counts what happened to each batch, and every call
must show the transition a model of the per-lane graph list predicts.  Every call uses fresh operand words, and every item of
every call is compared word for word with the reference.

The GPU part (pytest -m gpu) also asserts that no capture is refused.  The emulation build has no graphs: there every capture
is refused, which still exercises the tables, the padding, the transparent-result flags and the fallback."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import refseal
from params import PARAMS
from sealc_checks import _libs
from sealc_driver import Sealc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MUL, RELIN, GALOIS = 0, 1, 2
KINDS = {"multiply": MUL, "relinearize": RELIN, "galois": GALOIS}
FIRST, CAPTURE, REFUSED, REPLAY, EVICT, NO_GRAPH = range(6)
GRAPHS_PER_LANE = 48  # Context_::GRAPHS_PER_LANE
COMBINE_MAX = 64      # Context_::COMBINE_MAX
S_OK, COR_E_INVALIDOPERATION = 0, 0x80131509
ELT = 3               # Galois element of RotateRows(1) (SEAL's generator 3)
_POOL = ThreadPoolExecutor(max_workers=max(1, min(32, len(os.sched_getaffinity(0)))))


def padded(N):
    return 1 << (N - 1).bit_length()


class ShapeModel:
    """What combine_run_batch's graph list of one lane does with the next graph-path batch of a shape: first sight, capture
    on the second use, replay after that; a first sight with 48 shapes listed evicts the least recently used one."""

    def __init__(self):
        self.uses, self.stamp, self.clock = {}, {}, 0

    def step(self, shape):
        self.clock += 1
        evicted = False
        if shape not in self.uses:
            if len(self.uses) >= GRAPHS_PER_LANE:
                old = min(self.stamp, key=self.stamp.get)
                del self.uses[old], self.stamp[old]
                evicted = True
            self.uses[shape] = 0
        self.uses[shape] += 1
        self.stamp[shape] = self.clock
        return ("first", "capture", "replay")[min(self.uses[shape], 3) - 1], evicted

    def forget(self, shape):
        self.uses.pop(shape, None)
        self.stamp.pop(shape, None)


class Rig:
    """One context of our library next to the reference's on chain `name`, with a relinearization key and a Galois key of
    random key-level words; operands are random words at a data level (0 = the first)."""

    def __init__(self, S, name, graphs, seed=1):
        n, moduli, t = PARAMS[name]
        self.S, self.n, self.moduli, self.graphs = S, n, moduli, graphs
        self.R = refseal.RefContext(n, moduli, t)
        self.O = S.context(n, moduli, t)
        self.RL, self.OL = _libs(self.R, self.O)
        self.pids = self.R.data_parms_ids()
        self.levels = len(self.pids)
        self.rng = np.random.default_rng(seed)
        self.model = ShapeModel()
        self.keys = {}
        for kind in (RELIN, GALOIS):
            self.set_key(kind, self.rand_key())

    # ---- operands and keys ----
    def k(self, L):
        return self.R.k - L

    def rand_words(self, size, L):
        return np.stack([self.rng.integers(0, q, size=(size, self.n), dtype=np.uint64) for q in self.moduli[:self.k(L)]], axis=1)

    def rand_key(self):
        """(k, 2, K, n) key-level words"""
        return np.stack([np.stack([self.rng.integers(0, q, size=(2, self.n), dtype=np.uint64) for q in self.moduli], axis=1)
                         for _ in range(self.R.k)])

    def set_key(self, kind, words, ours=None):
        """(re)place the key of `kind`: in a new handle, or inside our existing handle `ours` (B200_KSwitchKeys_SetKeyWords)"""
        index = 0 if kind == RELIN else (ELT - 1) >> 1
        if ours is None:
            ours = self.O.new_ksk({index: words})
        else:
            w = np.ascontiguousarray(words)
            self.S.call("B200_KSwitchKeys_SetKeyWords", ours, self.O.ctx, C.c_uint64(index), C.c_uint64(w.shape[0]),
                        w.ctypes.data_as(C.POINTER(C.c_uint64)))
        self.keys[kind] = (ours, self.R.new_ksk({index: words}))
        return ours

    def ours(self, words, L, into=None):
        h = into or self.O._dst()
        w = np.ascontiguousarray(words)
        self.S.call("B200_Ciphertext_SetWords", h, self.O.ctx, self.pids[L], C.c_uint64(w.shape[0]), C.c_bool(False),
                    w.ctypes.data_as(C.POINTER(C.c_uint64)))
        return h

    def load(self, words, L, into):
        """Ciphertext_Load of the reference's serialisation of `words` into our existing handle `into`"""
        r = self.R.new_ct(words, level=L)
        data = self.RL.save("Ciphertext", r, 0)
        self.R.free_ct(r)
        rc, used = self.OL.load_rc("Ciphertext", into, data)
        assert rc == 0 and used == len(data), hex(rc)
        return into

    def operands(self, kind, L, N, zero_at=()):
        A = [self.rand_words(3 if kind == RELIN else 2, L) for _ in range(N)]
        B = [self.rand_words(2, L) for _ in range(N)] if kind == MUL else None
        for i in zero_at:
            A[i][:] = 0
        return A, B

    def expect(self, kind, L, A, B, skip=()):
        R = self.R

        def one(i):
            if i in skip:
                return None
            hs = [R.new_ct(A[i], level=L)]
            if kind == MUL:
                hs.append(R.new_ct(B[i], level=L))
                hs.append(R.multiply(hs[0], hs[1]))
            elif kind == RELIN:
                hs.append(R.relinearize(hs[0], self.keys[RELIN][1]))
            else:
                hs.append(R.apply_galois(hs[0], ELT, self.keys[GALOIS][1]))
            out = R.ct_words(hs[-1])
            for h in hs:
                R.free_ct(h)
            return out
        return list(_POOL.map(one, range(len(A))))

    # ---- one combined call ----
    def run(self, kind, L, A, B, a=None, b=None, dsts=None):
        a = a or [self.ours(x, L) for x in A]
        b = b or ([self.ours(x, L) for x in B] if kind == MUL else None)
        before = self.O.graph_stats()
        dsts, hr = self.O.combined_batch(kind, a, b, self.keys[kind][0] if kind != MUL else None, ELT, dsts)
        return dsts, hr, self.O.graph_stats() - before, a, b

    def transition(self, step, evicted=False):
        d = np.zeros(6, dtype=np.int64)
        if step in ("capture", "replay") and not self.graphs:
            step = "refused"  # no graphs: every capture attempt is refused, and a shape never gets past it
        d[{"first": FIRST, "capture": CAPTURE, "refused": REFUSED, "replay": REPLAY, "none": NO_GRAPH}[step]] = 1
        d[EVICT] = int(evicted)
        return d

    def check(self, kind, L, A, B, dsts, hr, delta, step, zero_at=(), what=""):
        """every item's HRESULT and words, and the counters' transition (`step`: a ShapeModel step, "model" to ask the
        model, or "none" for a batch that must not use a graph)"""
        N = len(A)
        if step == "model":
            step, evicted = self.model.step((kind, L, padded(N), id(self.keys.get(kind, (None,))[0])))
        else:
            evicted = False
        exp = self.expect(kind, L, A, B, skip=zero_at)
        for i in range(N):
            if i in zero_at:
                assert hr[i] == COR_E_INVALIDOPERATION, f"{what} item {i}/{N}: transparent result gave 0x{hr[i]:08x}"
                continue
            assert hr[i] == S_OK, f"{what} item {i}/{N}: HRESULT 0x{hr[i]:08x}"
            got = self.O.ct_words(dsts[i])
            if not np.array_equal(got, exp[i]):
                bad = np.argwhere(got != exp[i])
                raise AssertionError(f"{what} item {i}/{N} (NP {padded(N)}, level {L}, {step}): {len(bad)} words differ, "
                                     f"first at {tuple(bad[0])}")
        want = self.transition(step, evicted)
        assert np.array_equal(delta, want), f"{what} N={N} level {L}: counters moved by {delta.tolist()}, expected {want.tolist()}"
        return exp

    def shape(self, kind, L, N, zero_at=(), calls=3, what=""):
        """`calls` combined calls of one shape, fresh operands each time, checked against the model"""
        for c in range(calls):
            A, B = self.operands(kind, L, N, zero_at)
            dsts, hr, delta, _, _ = self.run(kind, L, A, B)
            self.check(kind, L, A, B, dsts, hr, delta, "model", zero_at, f"{what} call {c}")

    def finish(self):
        st = self.O.graph_stats()
        # one lane: the graph list never holds more than 48 shapes
        assert st[FIRST] - st[EVICT] <= GRAPHS_PER_LANE, st.tolist()
        if self.graphs:
            assert st[REFUSED] == 0, f"refused captures: {st.tolist()}"
        else:
            assert st[CAPTURE] == 0 and st[REPLAY] == 0, st.tolist()
        return st


# ---------------------------------------------------------------------------------------------------------------------
# the checks (GPU and emulation)
# ---------------------------------------------------------------------------------------------------------------------
def chain_levels(S, graphs, name, N, levels=None):
    """All three kinds at the given data levels (default: every one), lowest first so that the lane's pad destination grows
    at each step, then one more replay of the lowest level's shapes after it has grown."""
    rig = Rig(S, name, graphs)
    levels = list(range(rig.levels)) if levels is None else levels
    order = sorted(levels, reverse=True)
    for L in order:
        for kind in (MUL, RELIN, GALOIS):
            rig.shape(kind, L, N, what=f"{name} kind {kind}")
    for kind in (MUL, RELIN, GALOIS):
        rig.shape(kind, order[0], N, calls=1, what=f"{name} kind {kind} after the pad destination grew")
    rig.finish()


def batch_sizes(S, graphs, name, kind, sizes):
    rig = Rig(S, name, graphs, seed=kind + 10)
    for N in sizes:
        rig.shape(kind, 0, N, what=f"batch {N}")
    rig.finish()


def operand_identity(S, graphs, name, kind, N=5, L=0):
    """Replays with operands in new handles (the old ones kept alive: new addresses), with the same handles reloaded by
    Ciphertext_Load and by SetWords, and in place (destination = operand)."""
    rig = Rig(S, name, graphs, seed=20 + kind)
    keep = []
    for c in range(3):  # new handles every call
        A, B = rig.operands(kind, L, N)
        dsts, hr, delta, a, b = rig.run(kind, L, A, B)
        rig.check(kind, L, A, B, dsts, hr, delta, "model", what=f"new handles, call {c}")
        keep.append((a, b, dsts))
    a, b, dsts = keep[-1]
    for how in ("Ciphertext_Load", "SetWords"):  # same handles, new words
        A, B = rig.operands(kind, L, N)
        put = (lambda w, h: rig.load(w, L, h)) if how == "Ciphertext_Load" else (lambda w, h: rig.ours(w, L, into=h))
        a = [put(w, h) for w, h in zip(A, a)]
        b = [put(w, h) for w, h in zip(B, b)] if kind == MUL else None
        dsts, hr, delta, _, _ = rig.run(kind, L, A, B, a=a, b=b, dsts=dsts)
        rig.check(kind, L, A, B, dsts, hr, delta, "model", what=f"reloaded by {how}")
    # in place: a size-3 product does not fit a size-2 operand's buffer, so an in-place multiply never takes a graph
    for c in range(3):
        A, B = rig.operands(kind, L, N)
        if c == 0:
            ip = [rig.ours(w, L) for w in A]
        else:
            ip = [rig.ours(w, L, into=h) for w, h in zip(A, ip)]
        dsts, hr, delta, _, _ = rig.run(kind, L, A, B, a=ip, dsts=ip)
        rig.check(kind, L, A, B, dsts, hr, delta, "none" if kind == MUL else "model", what=f"in place, call {c}")
    rig.finish()


def reshaped_alias(S, graphs, name, N=3, L=0):
    """A multiply whose destination is another item's size-2 operand: the batch runs gather -> prepare -> scatter without a
    graph (operand j is read before its buffer is replaced by item i's size-3 product); the shape's graph is unaffected."""
    rig = Rig(S, name, graphs, seed=30)
    rig.shape(MUL, L, N, calls=2, what="before the alias")
    A, B = rig.operands(MUL, L, N)
    a = [rig.ours(x, L) for x in A]
    dsts = [rig.O._dst() for _ in range(N)]
    dsts[N - 1] = a[0]
    dsts, hr, delta, _, _ = rig.run(MUL, L, A, B, a=a, dsts=dsts)
    rig.check(MUL, L, A, B, dsts, hr, delta, "none", what="reshaped alias")
    rig.shape(MUL, L, N, calls=1, what="after the alias")
    rig.finish()


def key_replaced(S, graphs, name, kind, N=3, L=0):
    """After a captured shape, the same key handle gets other words (B200_KSwitchKeys_SetKeyWords): its new device copy may
    come back at the same address and meet the cached graph.  Every word must be the reference's under the NEW key."""
    rig = Rig(S, name, graphs, seed=40 + kind)
    rig.shape(kind, L, N, what="first key")
    shape = (kind, L, padded(N), id(rig.keys[kind][0]))
    rig.set_key(kind, rig.rand_key(), ours=rig.keys[kind][0])
    for c in range(3):
        A, B = rig.operands(kind, L, N)
        dsts, hr, delta, _, _ = rig.run(kind, L, A, B)
        if c == 0 and delta[FIRST]:  # the new copy is elsewhere: a new shape (else the cached graph is replayed)
            rig.model.forget(shape)
        rig.check(kind, L, A, B, dsts, hr, delta, "model", what=f"replaced key, call {c}")
    rig.finish()


def eviction(S, graphs, name, extra=2):
    """More than 48 rotation shapes on one lane (one key object, 48 + extra Galois elements), then the first one again: an
    eviction and a fresh first sight, then its capture and replay."""
    rig = Rig(S, name, graphs, seed=50)
    words = rig.rand_key()
    elts = [2 * i + 1 for i in range(1, GRAPHS_PER_LANE + extra + 1)]
    ours = rig.O.new_ksk({(e - 1) >> 1: words for e in elts})
    ref = rig.R.new_ksk({(e - 1) >> 1: words for e in elts})
    R = rig.R
    seq = elts + [elts[0]] * 3
    for c, e in enumerate(seq):
        A = [rig.rand_words(2, 0)]
        a = [rig.ours(A[0], 0)]
        before = rig.O.graph_stats()
        dsts, hr = rig.O.combined_batch(GALOIS, a, None, ours, e)
        delta = rig.O.graph_stats() - before
        step, evicted = rig.model.step((GALOIS, 0, 1, e))
        assert hr[0] == S_OK, f"element {e}: 0x{hr[0]:08x}"
        ra = R.new_ct(A[0])
        rd = R.apply_galois(ra, e, ref)
        exp = R.ct_words(rd)
        R.free_ct(ra)
        R.free_ct(rd)
        assert np.array_equal(rig.O.ct_words(dsts[0]), exp), f"call {c}, element {e}"
        assert np.array_equal(delta, rig.transition(step, evicted)), f"call {c}, element {e}: {delta.tolist()}"
        st = rig.O.graph_stats()
        assert st[FIRST] - st[EVICT] <= GRAPHS_PER_LANE, st.tolist()
    st = rig.finish()
    assert st[EVICT] == extra + 1 and st[FIRST] == len(elts) + 1, st.tolist()


def transparent_items(S, graphs, name, kind, N=5, L=0):
    """One item whose result is transparent (an all-zero operand) at the first, a middle and the last real position before the
    pads: it alone gets COR_E_INVALIDOPERATION on first sight, capture and replay; then an all-valid replay succeeds for every
    item (the flags are cleared)."""
    rig = Rig(S, name, graphs, seed=60 + kind)
    for pos in (0, N // 2, N - 1):
        rig.shape(kind, L, N, zero_at=(pos,), what=f"transparent at {pos}")
    rig.shape(kind, L, N, calls=1, what="all valid after the transparent ones")
    rig.finish()


def condensed(S, graphs, combine=True):
    """A short sequence for the process-wide settings; returns a digest of every output word.  Without the combiner
    (B200_NO_COMBINE) the same items run as plain per-handle calls."""
    rig = Rig(S, "n8192", graphs, seed=70)
    h = hashlib.sha256()
    for L in (0, rig.levels - 1):
        for kind in (MUL, RELIN, GALOIS):
            for N in (3, 9, 17):
                for c in range(3):
                    A, B = rig.operands(kind, L, N)
                    if combine:
                        dsts, hr, delta, _, _ = rig.run(kind, L, A, B)
                        rig.check(kind, L, A, B, dsts, hr, delta, "model" if graphs else "none", what=f"kind {kind} N {N}")
                    else:
                        exp = rig.expect(kind, L, A, B)
                        dsts = []
                        for i in range(N):
                            a = rig.ours(A[i], L)
                            if kind == MUL:
                                d = rig.O.multiply(a, rig.ours(B[i], L))
                            elif kind == RELIN:
                                d = rig.O.relinearize(a, rig.keys[RELIN][0])
                            else:
                                d = rig.O.rotate_rows(a, 1, rig.keys[GALOIS][0])
                            assert np.array_equal(rig.O.ct_words(d), exp[i]), f"per-handle kind {kind} item {i}"
                            dsts.append(d)
                    for d in dsts:
                        h.update(rig.O.ct_words(d).tobytes())
    st = rig.finish()
    if not combine:
        assert not st.any(), st.tolist()
    return h.hexdigest()


def threaded_combiner(S, name, threads, rounds=6):
    """`threads` callers of Evaluator_Multiply -> Evaluator_Relinearize -> Evaluator_RotateRows(1) at the first and the last
    data level, new operand words every round; every result equals the reference's."""
    import threading
    rig = Rig(S, name, True, seed=80 + threads)
    levels = (0, rig.levels - 1)
    work = {}
    for r in range(rounds):
        for i in range(threads):
            L = levels[(i + r) & 1]
            A, B = rig.operands(MUL, L, 1)
            work[(r, i)] = (L, A[0], B[0])
    R, rrlk, rglk = rig.R, rig.keys[RELIN][1], rig.keys[GALOIS][1]

    def ref_one(key):
        L, a, b = work[key]
        hs = [R.new_ct(a, level=L), R.new_ct(b, level=L)]
        hs.append(R.multiply(hs[0], hs[1]))
        hs.append(R.relinearize(hs[-1], rrlk))
        hs.append(R.apply_galois(hs[-1], ELT, rglk))
        out = R.ct_words(hs[-1])
        for h in hs:
            R.free_ct(h)
        return out
    keys = sorted(work)
    exp = dict(zip(keys, _POOL.map(ref_one, keys)))
    ins = {key: (rig.ours(work[key][1], work[key][0]), rig.ours(work[key][2], work[key][0])) for key in keys}
    bad, errors = [], []
    barrier = threading.Barrier(threads)
    before = rig.O.graph_stats()

    def runner(i):
        try:
            for r in range(rounds):
                a, b = ins[(r, i)]
                barrier.wait()
                m = rig.O.multiply(a, b)
                m = rig.O.relinearize(m, rig.keys[RELIN][0])
                m = rig.O.rotate_rows(m, 1, rig.keys[GALOIS][0])
                if not np.array_equal(rig.O.ct_words(m), exp[(r, i)]):
                    bad.append((r, i))
        except Exception as e:  # pragma: no cover
            errors.append((i, repr(e)))
            barrier.abort()
    ts = [threading.Thread(target=runner, args=(i,)) for i in range(threads)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errors, errors
    assert not bad, f"results differ from the reference: {bad}"
    st = rig.O.graph_stats() - before
    assert st[REFUSED] == 0 and st[REPLAY] > 0, st.tolist()


# ---------------------------------------------------------------------------------------------------------------------
# emulation build (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_S(emu_lib):
    return Sealc(emu_lib.lib)


def test_emu_chain_levels(emu_S, ref):
    chain_levels(emu_S, False, "n4096", 3)


@pytest.mark.parametrize("kind", list(KINDS))
def test_emu_batch_sizes(emu_S, ref, kind):
    batch_sizes(emu_S, False, "n4096", KINDS[kind], [1, 2, 3, 5])


@pytest.mark.parametrize("kind", list(KINDS))
def test_emu_operand_identity(emu_S, ref, kind):
    operand_identity(emu_S, False, "n4096", KINDS[kind], N=3)


def test_emu_reshaped_alias(emu_S, ref):
    reshaped_alias(emu_S, False, "n4096")


@pytest.mark.parametrize("kind", ["relinearize", "galois"])
def test_emu_key_replaced(emu_S, ref, kind):
    key_replaced(emu_S, False, "n4096", KINDS[kind])


@pytest.mark.parametrize("kind", list(KINDS))
def test_emu_transparent_items(emu_S, ref, kind):
    transparent_items(emu_S, False, "n4096", KINDS[kind], N=3)


def test_emu_eviction(emu_S, ref):
    eviction(emu_S, False, "n4096")


def test_emu_hook_argument_checks(emu_S, ref):
    """the debug hook's own argument checks"""
    rig = Rig(emu_S, "n4096", False)
    A, _ = rig.operands(GALOIS, 0, 1)
    a = (C.c_void_p * 1)(rig.ours(A[0], 0))
    d = (C.c_void_p * 1)(rig.O._dst())
    hr = (C.c_long * 1)()
    rc = lambda kind, count, keys: emu_S.rc("B200_Evaluator_CombinedBatchDebug", rig.O.ev, C.c_int(kind), C.c_uint64(count),
                                            a, None, keys, C.c_uint32(ELT), d, hr)
    assert rc(GALOIS, 0, rig.keys[GALOIS][0]) == 0x80070057        # empty batch
    assert rc(GALOIS, COMBINE_MAX + 1, rig.keys[GALOIS][0]) == 0x80070057
    assert rc(MUL, 1, None) == 0x80070057                          # no second operands
    assert rc(3, 1, rig.keys[GALOIS][0]) == 0x80070057
    assert rc(GALOIS, 1, rig.keys[GALOIS][0]) == 0 and hr[0] == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu_S():
    from sunscreen_b200.lib import B200Lib
    lib = B200Lib.default()
    assert os.path.basename(lib.path) == "libb200bfv.so"
    return Sealc(lib.lib)


def dispatch_boundaries(name):
    """Batch sizes on both sides of the layer-1 rules NP crosses at the first data level (b200_bfv.cu): mul_cluster_kernel at
    4 (k + |Bsk|) NP > 2 sm_count, ks_cluster_kernel and the 512 / 256-thread NTT switch of the key switch's digits at
    k (k + 1) NP > 2 sm_count.  For each rule: the largest power of two NP below it and NP + 1 (which pads to 2 NP)."""
    from sunscreen_b200.lib import B200Context
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    li = ctx.level_info(ctx.first_level)
    k, sm = li["k"], ctx.sm_count
    ctx.close()
    out = set()
    for per_item in (4 * (k + li["nBsk"]), k * (k + 1)):
        NP = 1
        while per_item * 2 * NP <= 2 * sm:
            NP *= 2
        assert per_item * NP <= 2 * sm < per_item * 2 * NP
        if 2 * NP <= COMBINE_MAX:
            out |= {NP, NP + 1}
    return sorted(out)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_54", "n8192_60", "n16384", "n32768"])
def test_chain_levels(gpu_S, ref, name):
    if name == "n32768":  # the reference is slow here: the first and the lowest data level, two items
        chain_levels(gpu_S, True, name, 2, levels=[0, len(PARAMS[name][1]) - 2])
    else:
        chain_levels(gpu_S, True, name, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_batch_sizes(gpu_S, ref, kind):
    sizes = sorted({1, 2, 3, 5, 8, 9, 16, 17, 33, 64} | set(dispatch_boundaries("n8192")))
    assert {padded(N) for N in sizes} == {1, 2, 4, 8, 16, 32, 64}
    batch_sizes(gpu_S, True, "n8192", KINDS[kind], sizes)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("N", [5, 17])
def test_operand_identity(gpu_S, ref, kind, N):
    operand_identity(gpu_S, True, "n8192", KINDS[kind], N=N)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [3, 16])
def test_reshaped_alias(gpu_S, ref, N):
    reshaped_alias(gpu_S, True, "n8192", N=N)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["relinearize", "galois"])
@pytest.mark.parametrize("N", [3, 17])
def test_key_replaced(gpu_S, ref, kind, N):
    key_replaced(gpu_S, True, "n8192", KINDS[kind], N=N)


@pytest.mark.gpu
def test_eviction(gpu_S, ref):
    eviction(gpu_S, True, "n4096")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("N", [5, 33])
def test_transparent_items(gpu_S, ref, kind, N):
    transparent_items(gpu_S, True, "n8192", KINDS[kind], N=N)


_CONDENSED = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
from sunscreen_b200.lib import B200Lib
from sealc_driver import Sealc
import test_combined_graphs as T
print("digest", T.condensed(Sealc(B200Lib.default().lib), {graphs!r}, combine={combine!r}), flush=True)
"""


def _condensed_in_subprocess(setting):
    env = dict(os.environ)
    if setting:
        name, value = setting.split("=")
        env[name] = value
    graphs = setting != "B200_NO_GRAPHS=1"
    combine = setting != "B200_NO_COMBINE=1"
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _CONDENSED.format(root=ROOT, tests=HERE, graphs=graphs, combine=combine)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"{setting}: exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    return r.stdout.split()[-1]


@pytest.fixture(scope="module")
def default_digest(ref):
    return _condensed_in_subprocess(None)


@pytest.mark.gpu
@pytest.mark.parametrize("setting", ["B200_NO_GRAPHS=1", "B200_KS_CLUSTER=0", "B200_MUL_CLUSTER=0", "B200_NO_COMBINE=1"])
def test_process_wide_setting(ref, default_digest, setting):
    """the condensed sequence under each setting (words checked against the reference in the subprocess): the same bytes as
    under the defaults"""
    assert _condensed_in_subprocess(setting) == default_digest


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [16, 64])
def test_threaded_combiner(gpu_S, ref, threads):
    threaded_combiner(gpu_S, "n8192", threads)
