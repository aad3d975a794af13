"""Slot-wise linear transforms: b200_apply_galois_many (a key switch whose items carry their own Galois element and key) and
b200_linear_transform (the baby-step giant-step matrix x packed-vector product) against the reference's apply_galois /
rotate_rows, multiply_plain and add chain, word for word.  The same checks run on the CPU emulation build and, marked gpu, on
the CUDA library, where launch traces show ks_cluster_galois_multi_kernel and the new mod-downs."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from backends import CudaBackend, EmuBackend
from params import PARAMS
from sunscreen_b200.bsgs import apply_slotwise, bsgs_plain_vectors
from sunscreen_b200.lib import PLAIN_NTT_MULTIPLY, B200Error

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def level_k(P, j):
    return P.ctx.level_info(P.ctx.first_level + j)["k"]


def rule_batch(P, j, side):
    """a key-switch batch just below ("below") or just above ("at") the cluster rule k (k + 1) batch > 2 sm_count"""
    k = max(level_k(P, j), 2)
    last = (2 * P.ctx.sm_count) // (k * (k + 1))
    return max(1, last) if side == "below" else last + 1


def row_elt(n, step):
    return pow(3, step % (n // 2), 2 * n)


def keys_for(P, rng, elts):
    """one random key list per distinct element: {g: host words}"""
    return {g: pc.rand_ksk(rng, P.moduli, P.k, P.n) for g in sorted(set(elts))}


# ---- apply_galois_many ----

def many_vs_reference(P, j, batch, seed, src_map="random", elts=None, keys=None, cts=None):
    rng = np.random.default_rng(seed)
    lv, k, n = P.ctx.first_level + j, level_k(P, j), P.n
    if elts is None:
        pool = [3, 9, 243, 2 * n - 1, row_elt(n, n // 2 - 1)]
        elts = [pool[i % len(pool)] for i in range(batch)]
        elts = sorted(elts, key=pool.index)  # element-major, as a caller wanting few MAC runs orders them
    sources = batch if src_map == "identity" else max(1, batch // 2)
    if cts is None:
        cts = pc.rand_ct(rng, P.moduli, k, n, batch=sources)
    src = None if src_map == "identity" else [int(x) for x in rng.integers(0, sources, size=batch)]
    if keys is None:
        keys = keys_for(P, rng, elts)
    dkeys = {g: P.dev(v) for g, v in keys.items()}
    out = P.out(batch, 2, k, n)
    P.ctx.apply_galois_many(P.dev(cts), src, elts, [dkeys[g] for g in elts], out, level=lv)
    got = P.host(out).reshape(batch, 2, k, n)
    R = P.ref
    glk = R.new_ksk({(g - 1) // 2: v for g, v in keys.items()})
    for i in range(batch):
        h = R.new_ct(cts[src[i] if src else i], level=j)
        r = R.apply_galois(h, elts[i], glk)
        pc.eq(got[i], R.ct_words(r), f"item {i} of {batch} (element {elts[i]}), level {lv}")
        R.free_ct(r)
        R.free_ct(h)


# ---- linear_transform ----

def rand_plains(rng, n, t, G, b):
    return rng.integers(1, t, size=(G, b, n), dtype=np.uint64)


def ref_linear_transform(P, c, j, b, G, elts, glk, plains, present):
    """the reference's chain: baby rotations, multiply_plain + add per giant row, giant rotations added in order of g"""
    R = P.ref
    ct = R.new_ct(c, level=j)
    used = lambda g, jj: present is None or present[g][jj]
    rot = {0: ct}
    for jj in range(1, b):
        if any(used(g, jj) for g in range(G)):
            rot[jj] = R.apply_galois(ct, elts[jj - 1], glk)
    acc = None
    for g in range(G):
        inner = None
        for jj in range(b):
            if not used(g, jj):
                continue
            pt = R.new_pt(plains[g][jj])
            prod = R.multiply_plain(rot[jj], pt)
            R.free_pt(pt)
            if inner is None:
                inner = prod
            else:
                nxt = R.add(inner, prod)
                R.free_ct(inner)
                R.free_ct(prod)
                inner = nxt
        if inner is None:
            continue
        if g:
            r = R.apply_galois(inner, elts[b - 1 + g - 1], glk)
            R.free_ct(inner)
            inner = r
        if acc is None:
            acc = inner
        else:
            nxt = R.add(acc, inner)
            R.free_ct(acc)
            R.free_ct(inner)
            acc = nxt
    out = R.ct_words(acc)
    R.free_ct(acc)
    for h in rot.values():
        R.free_ct(h)
    return out


def bsgs_elts(n, b, G):
    return [row_elt(n, s) for s in range(1, b)] + [row_elt(n, g * b) for g in range(1, G)]


def lt_run(P, lv, cts, b, G, elts, dkeys, plains, present=None, out=None):
    V, _, k, n = cts.shape
    pn = P.out(G, b, k, n)
    P.ctx.plain_to_ntt(P.dev(plains.reshape(G * b, n)), G * b, pn, rule=PLAIN_NTT_MULTIPLY, level=lv)
    o = P.out(V, 2, k, n) if out is None else out
    P.ctx.linear_transform(P.dev(cts) if out is None else out, V, b, G, elts, [dkeys.get(g) for g in elts], pn, o,
                           present=present, level=lv)
    return P.host(o).reshape(V, 2, k, n)


def lt_vs_reference(P, j, V, b, G, seed, present=None, cts=None, keys=None, plains=None, check=None):
    rng = np.random.default_rng(seed)
    lv, k, n = P.ctx.first_level + j, level_k(P, j), P.n
    elts = bsgs_elts(n, b, G)
    if cts is None:
        cts = pc.rand_ct(rng, P.moduli, k, n, batch=V)
    if keys is None:
        keys = keys_for(P, rng, elts)
    if plains is None:
        plains = rand_plains(rng, n, P.t, G, b)
    dkeys = {g: P.dev(v) for g, v in keys.items()}
    got = lt_run(P, lv, cts, b, G, elts, dkeys, plains, present)
    glk = P.ref.new_ksk({(g - 1) // 2: v for g, v in keys.items()})
    for v in (range(V) if check is None else check):
        pc.eq(got[v], ref_linear_transform(P, cts[v], j, b, G, elts, glk, plains, present),
              f"b {b} G {G} vector {v} of {V}, level {lv}")


def absent_masks(b, G):
    col = np.ones((G, b), dtype=bool)
    col[:, b - 1] = False          # a whole baby column: that baby step is not rotated
    row = np.ones((G, b), dtype=bool)
    row[G - 1, :] = False          # a whole giant row: that giant step is dropped
    one = np.ones((G, b), dtype=bool)
    one[G // 2, b // 2] = False    # a single term
    first = np.ones((G, b), dtype=bool)
    first[0, :] = False            # no inner_0: the sum starts from the first giant term
    return {"column": col, "row": row, "single": one, "row0": first}


def check_errors(P, lib):
    from sunscreen_b200.lib import B200Context
    rng = np.random.default_rng(8)
    k, n = P.k, P.n
    key = P.dev(pc.rand_ksk(rng, P.moduli, P.k, n))
    buf = P.dev(pc.rand_ct(rng, P.moduli, k, n, batch=3))
    out = P.out(3, 2, k, n)

    def code(fn, *args, **kw):
        with pytest.raises(B200Error) as e:
            fn(*args, **kw)
        return e.value.code
    many = P.ctx.apply_galois_many
    assert code(many, buf, None, [3, 4], [key, key], out) == -1            # even element
    assert code(many, buf, None, [3, 2 * n + 1], [key, key], out) == -1    # element >= 2n
    assert code(many, buf, None, [3, 5], [key, None], out) == -4           # null key
    assert code(many, None, None, [3], [key], out) == -4
    assert code(many, buf, None, [3], [key], None) == -4
    assert code(many, buf, [0, 2], [3, 3], [key, key], buf[1:]) == -1      # out overlapping a source
    assert code(many, buf, None, [3], [key], out, level=0) == -2            # the key level: no key switching
    ctx1 = B200Context(n, [P.moduli[0]], P.t, lib=lib)
    assert code(ctx1.apply_galois_many, buf, None, [3], [key], out) == -2
    many(buf, None, [], [], out)                                              # batch 0
    lt = P.ctx.linear_transform
    pn = P.out(2, 2, k, n)
    elts = bsgs_elts(n, 2, 2)
    assert code(lt, buf, 1, 0, 1, [], [], pn, out) == -1                     # baby 0
    assert code(lt, buf, 1, 1, 0, [], [], pn, out) == -1                     # giant 0
    assert code(lt, buf, 1, 2, 2, elts, [key, key], pn, out, present=[[0, 0], [0, 0]]) == -1   # every term absent
    assert code(lt, buf, 1, 2, 2, [4, elts[1]], [key, key], pn, out) == -1   # invalid baby element
    assert code(lt, buf, 1, 2, 2, elts, [key, None], pn, out) == -4          # no key for a used giant step
    assert code(lt, None, 1, 2, 2, elts, [key, key], pn, out) == -4
    assert code(lt, buf, 1, 2, 2, elts, [key, key], None, out) == -4
    assert code(lt, buf, 2, 2, 2, elts, [key, key], pn, buf[1:]) == -1      # out partly overlapping cts
    assert code(lt, buf, 1, 2, 2, elts, [key, key], pn, out, level=0) == -2
    # a step no present term uses needs neither element nor key
    lt(buf, 1, 2, 2, [0, elts[1]], [None, key], pn, out, present=[[1, 0], [1, 0]])
    lt(buf, 0, 2, 2, elts, [key, key], pn, out)                              # V = 0


def check_against_existing_route(P, V, b, G, seed):
    """the fused op against b200_apply_galois per baby step, b200_multiply_plain_sum per vector and b200_apply_galois_add per
    giant step on the same device"""
    rng = np.random.default_rng(seed)
    k, n = P.k, P.n
    elts = bsgs_elts(n, b, G)
    keys = {g: P.dev(v) for g, v in keys_for(P, rng, elts).items()}
    cts = pc.rand_ct(rng, P.moduli, k, n, batch=V)
    plains = rand_plains(rng, n, P.t, G, b)
    got = lt_run(P, None, cts, b, G, elts, keys, plains)
    dc = P.dev(cts)
    pn = P.out(G, b, k, n)
    P.ctx.plain_to_ntt(P.dev(plains.reshape(G * b, n)), G * b, pn, rule=PLAIN_NTT_MULTIPLY)
    X = P.out(V, b, 2, k, n)
    inner = P.out(V, G, 2, k, n)
    exp = P.out(V, 2, k, n)
    for v in range(V):
        X[v, 0] = dc[v]
        for s in range(1, b):
            P.ctx.apply_galois(dc[v], elts[s - 1], keys[elts[s - 1]], X[v, s], 1)
        P.ctx.multiply_plain_sum(X[v], 2, b, pn, G, inner[v])
        exp[v] = inner[v, 0]
        for g in range(1, G):
            e = elts[b - 1 + g - 1]
            P.ctx.apply_galois_add(inner[v, g], e, keys[e], exp[v], exp[v], 1)
    pc.eq(got, P.host(exp).reshape(V, 2, k, n), f"V {V} b {b} G {G} vs the per-call route")


def check_decrypted(P, d, b, seed, banded=False, two=False):
    """real keys (KeyGenerator_CreateGaloisKeysFromSteps for the helper's steps), batch-encoded diagonals and a replicated
    input vector: each slot row decrypts to M v mod t"""
    R, n, t = P.ref, P.n, P.t
    rng = np.random.default_rng(seed)
    h = n // 2

    def mat():
        m = rng.integers(0, t, size=(d, d))
        if banded:
            m = np.where(np.abs(np.subtract.outer(np.arange(d), np.arange(d))) <= 2, m, 0)
        return m
    mats = (mat(), mat()) if two else mat()
    vecs, present, steps = bsgs_plain_vectors(mats, n, t, b)
    G = vecs.shape[0]
    kg = R.keygen()
    gk = R.galois_keys_steps(kg, steps)
    words = R.ksk_words(gk)
    enc, dec, be = R.encryptor(R.public_key(kg)), R.decryptor(R.secret_key(kg)), R.batch_encoder()
    x = rng.integers(0, t, size=(2, d), dtype=np.uint64)
    v = np.concatenate([np.tile(x[0], h // d), np.tile(x[1], h // d)])
    ct = R.ct_words(R.encrypt(enc, R.batch_encode(be, v)))
    plains = np.zeros((G, b, n), dtype=np.uint64)
    for g in range(G):
        for j in range(b):
            if present[g, j]:
                c = R.pt_coeffs(R.batch_encode(be, vecs[g, j]))
                plains[g, j, :c.size] = c
    elts = bsgs_elts(n, b, G)
    dkeys = {g: P.dev(words[(g - 1) // 2]) for g in set(elts) if (g - 1) // 2 in words}
    got = lt_run(P, None, ct[None], b, G, elts, dkeys, plains, present=present.tolist())
    hh = R.new_ct(got[0])
    slots = R.batch_decode(be, R.decrypt(dec, hh))
    assert np.array_equal(slots, apply_slotwise(mats, v, n, t)), (slots[:8], apply_slotwise(mats, v, n, t)[:8])


# ---- CPU emulation build ----

@pytest.fixture(scope="module")
def emu_pairs(emu_lib, ref):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.pair_for(EmuBackend(emu_lib), name)
        return cache[name]
    return get


@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_60", "n2048_2x27"])
def test_emu_apply_galois_many_levels(emu_pairs, name):
    P = emu_pairs(name)
    for j in range(len(P.ref.data_parms_ids())):
        many_vs_reference(P, j, 5, seed=j, src_map="random")
    many_vs_reference(P, 0, 3, seed=9, src_map="identity")


def test_emu_apply_galois_many_adversarial(emu_pairs):
    P = emu_pairs("n4096")
    K = len(P.moduli)
    pm1 = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        pm1[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    for kind in ("qm1", "alt"):
        c = pc.adversarial_ct(P, kind)[None]
        many_vs_reference(P, 0, 2, seed=5, src_map="random", elts=[3, 2 * P.n - 1], keys={3: pm1, 2 * P.n - 1: pm1}, cts=c)


@pytest.mark.parametrize("b,G", [(1, 1), (1, 4), (4, 1), (3, 5), (16, 16)])
def test_emu_linear_transform_shapes(emu_pairs, b, G):
    P = emu_pairs("n2048_2x27")
    lt_vs_reference(P, 0, 2, b, G, seed=b * 31 + G, check=[0, 1] if b * G < 256 else [1])


@pytest.mark.parametrize("name", ["n4096", "n8192_54"])
def test_emu_linear_transform_levels(emu_pairs, name):
    P = emu_pairs(name)
    for j in range(len(P.ref.data_parms_ids())):
        lt_vs_reference(P, j, 1, 3, 2, seed=40 + j)


@pytest.mark.parametrize("kind", ["column", "row", "single", "row0"])
def test_emu_linear_transform_absent_terms(emu_pairs, kind):
    P = emu_pairs("n2048_2x27")
    b, G = 3, 4
    lt_vs_reference(P, 0, 2, b, G, seed=60, present=absent_masks(b, G)[kind].tolist())


def test_emu_linear_transform_chunks(emu_pairs, monkeypatch):
    """a scratch bound of one vector: three chunks, the words of one call"""
    P = emu_pairs("n2048_2x27")
    monkeypatch.setenv("B200_LINEAR_SCRATCH", "1")
    lt_vs_reference(P, 0, 3, 2, 3, seed=70)


def test_emu_linear_transform_in_place(emu_pairs):
    P = emu_pairs("n2048_2x27")
    rng = np.random.default_rng(3)
    b, G, k, n = 2, 2, P.k, P.n
    elts = bsgs_elts(n, b, G)
    keys = {g: P.dev(v) for g, v in keys_for(P, rng, elts).items()}
    cts = pc.rand_ct(rng, P.moduli, k, n, batch=2)
    plains = rand_plains(rng, n, P.t, G, b)
    exp = lt_run(P, None, cts, b, G, elts, keys, plains)
    buf = P.dev(cts)
    got = lt_run(P, None, cts, b, G, elts, keys, plains, out=buf)
    pc.eq(got, exp, "out = cts")


def test_emu_errors(emu_pairs, emu_lib):
    check_errors(emu_pairs("n4096"), emu_lib)


@pytest.mark.parametrize("banded,two", [(False, False), (True, True)])
def test_emu_decrypted(emu_pairs, banded, two):
    check_decrypted(emu_pairs("n8192"), 16, 4, seed=90, banded=banded, two=two)


def test_bsgs_helper_plain_model():
    """the helper's vectors, applied slot by slot with plain rotations, give M v: the BSGS identity itself"""
    n, t, d, b = 64, 257, 8, 3
    rng = np.random.default_rng(1)
    mats = (rng.integers(0, t, size=(d, d)), rng.integers(0, t, size=(d, d)))
    vecs, present, steps = bsgs_plain_vectors(mats, n, t, b)
    G, h = vecs.shape[0], n // 2
    x = rng.integers(0, t, size=(2, d))
    v = np.concatenate([np.tile(x[0], h // d), np.tile(x[1], h // d)]).astype(object)
    rot = lambda a, s: np.concatenate([np.roll(a[:h], -s), np.roll(a[h:], -s)])
    out = np.zeros(n, dtype=object)
    for g in range(G):
        inner = sum(vecs[g, j].astype(object) * rot(v, j) for j in range(b) if present[g, j])
        out = out + rot(inner, g * b)
    assert np.array_equal(out % t, apply_slotwise(mats, v, n, t).astype(object))
    assert steps == [1, 2, 3, 6]


# ---- CUDA library ----

@pytest.fixture(scope="module")
def pairs(ref):
    be = CudaBackend()
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.pair_for(be, name)
        return cache[name]
    return get


GPU_SETS = ["n8192", "n8192_54", "n8192_60", "n16384", "n4096", "n4096_9x22", "n8192_9x24"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SETS)
def test_gpu_apply_galois_many_levels(pairs, name):
    """every data level, batches on both sides of the cluster rule, repeated and identity source maps"""
    P = pairs(name)
    for j in range(len(P.ref.data_parms_ids())):
        for side in ("below", "at"):
            many_vs_reference(P, j, rule_batch(P, j, side), seed=j, src_map="random")
    many_vs_reference(P, 0, rule_batch(P, 0, "at"), seed=7, src_map="identity")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n4096"])
def test_gpu_apply_galois_many_adversarial(pairs, name):
    P = pairs(name)
    K = len(P.moduli)
    pm1 = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        pm1[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    batch = rule_batch(P, 0, "at")
    for kind in ("qm1", "alt"):
        c = np.broadcast_to(pc.adversarial_ct(P, kind), (batch, 2, P.k, P.n)).copy()
        many_vs_reference(P, 0, batch, seed=5, src_map="identity", elts=[3, 2 * P.n - 1] * (batch // 2) + [3] * (batch % 2),
                          keys={3: pm1, 2 * P.n - 1: pm1}, cts=c)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SETS)
def test_gpu_linear_transform_levels(pairs, name):
    """b = 3, G = 5 at every data level: 2 V baby items and 4 V giant items, with V chosen so that both key switches are below
    the cluster rule, the baby steps below and the giant steps above it, and both above it"""
    P = pairs(name)
    for j in range(len(P.ref.data_parms_ids())):
        last = rule_batch(P, j, "below")  # the largest batch below the rule (1 where even one item is above it)
        below = max(1, last // 4)
        mixed = last // 2 if last // 2 >= 1 and 4 * (last // 2) > last else None
        above = -(-(last + 1) // 2)
        for V in [below, mixed, above]:
            if V is not None:
                lt_vs_reference(P, j, V, 3, 5, seed=j, check=[0, V - 1])


@pytest.mark.gpu
@pytest.mark.parametrize("b,G", [(1, 1), (1, 4), (4, 1), (3, 5), (16, 16)])
def test_gpu_linear_transform_shapes(pairs, b, G):
    P = pairs("n8192")
    lt_vs_reference(P, 0, 2, b, G, seed=b * 31 + G, check=[1])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["column", "row", "single", "row0"])
def test_gpu_linear_transform_absent_terms(pairs, kind):
    P = pairs("n8192")
    b, G = 4, 4
    lt_vs_reference(P, 0, 4, b, G, seed=60, present=absent_masks(b, G)[kind].tolist(), check=[0, 3])


@pytest.mark.gpu
def test_gpu_linear_transform_chunks(pairs, monkeypatch):
    P = pairs("n8192")
    monkeypatch.setenv("B200_LINEAR_SCRATCH", str(40 << 20))
    lt_vs_reference(P, 0, 5, 2, 3, seed=70, check=[0, 4])


@pytest.mark.gpu
@pytest.mark.parametrize("V,b,G", [(1, 16, 16), (64, 8, 8), (3, 4, 6)])
def test_gpu_matches_existing_route(pairs, V, b, G):
    check_against_existing_route(pairs("n8192"), V, b, G, seed=V + b)


@pytest.mark.gpu
def test_gpu_linear_transform_wide(pairs):
    P = pairs("n32768_60x6")
    lt_vs_reference(P, 0, 1, 2, 2, seed=5)


@pytest.mark.gpu
def test_gpu_errors(pairs):
    check_errors(pairs("n4096"), pairs("n4096").be.lib)


@pytest.mark.gpu
@pytest.mark.parametrize("banded,two", [(False, False), (True, True)])
def test_gpu_decrypted_n8192(pairs, banded, two):
    check_decrypted(pairs("n8192"), 256, 16, seed=91, banded=banded, two=two)


_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import parity_checks as pc
from backends import CudaBackend
from params import PARAMS
from sunscreen_b200.lib import B200Context, PLAIN_NTT_MULTIPLY
be = CudaBackend()
n, moduli, t = PARAMS["n8192"]
ctx = B200Context(n, moduli, t)
k, V, b, G = ctx.k(), {V}, {b}, {G}
rng = np.random.default_rng(1)
elts = [pow(3, s, 2 * n) for s in range(1, b)] + [pow(3, g * b, 2 * n) for g in range(1, G)]
keys = [be.to_dev(pc.rand_ksk(rng, moduli, k, n)) for _ in elts]
a = be.to_dev(pc.rand_ct(rng, moduli, k, n, batch=V))
pn = be.empty((G, b, k, n))
ctx.plain_to_ntt(be.to_dev(rng.integers(1, t, size=(G * b, n), dtype=np.uint64)), G * b, pn, rule=PLAIN_NTT_MULTIPLY)
o = be.empty((V, 2, k, n))
ctx.linear_transform(a, V, b, G, elts, keys, pn, o)
be.torch.cuda.synchronize()
c0 = ctx.launch_count()
ctx.linear_transform(a, V, b, G, elts, keys, pn, o)
be.torch.cuda.synchronize()
print("launches", ctx.launch_count() - c0, flush=True)
be.lib.lib.b200_trace_dump()
"""


def traced(V, b, G):
    env = dict(os.environ, B200_TRACE="1")
    for var in ("B200_KS_CLUSTER", "B200_KSMAC_TMA", "B200_LINEAR_SCRATCH"):
        env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _TRACE.format(root=ROOT, tests=HERE, V=V, b=b, G=G)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    per_call = int(re.search(r"launches (\d+)", r.stdout).group(1))
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    return per_call, launches


def count(launches, prefix):
    return sum(v for key, v in launches.items() if key.startswith(prefix))


@pytest.mark.gpu
def test_gpu_trace_cluster_path():
    """one vector, b = G = 16 at k = 4: 15 items per key switch, above the rule; two multi-element cluster launches (one per
    step group), the two new mod-downs, one masked MAC, and no addsub_kernel or galois_kernel"""
    per_call, launches = traced(1, 16, 16)
    assert count(launches, "ks_cluster_galois_multi_kernel") == 4, launches   # two calls
    assert count(launches, "ksmoddown_galois_many_kernel") == 2, launches
    assert count(launches, "moddown_galois_sum_kernel") == 2, launches
    assert count(launches, "plain_mac_multi_kernel") == 2, launches
    assert count(launches, "addsub_kernel") == 0 and count(launches, "galois_kernel") == 0, launches
    assert count(launches, "galois_many_kernel") == 0 and count(launches, "ks_cluster_kernel") == 0, launches
    # X[0] forward NTT, baby key switch + mod-down, forward NTT of the copies, MAC, inverse NTT, giant key switch + mod-down
    assert per_call == 8, (per_call, launches)


@pytest.mark.gpu
def test_gpu_trace_below_rule():
    """one vector, b = G = 2: one item per key switch, below the rule; the separate kernels run once per element group"""
    per_call, launches = traced(1, 2, 2)
    assert count(launches, "galois_many_kernel") == 4, launches
    assert count(launches, "ks_cluster") == 0, launches
    assert count(launches, "ksmoddown_galois_many_kernel") == 2, launches
    assert count(launches, "moddown_galois_sum_kernel") == 2, launches
    assert count(launches, "addsub_kernel") == 0, launches


# ---- layer 2: B200_Evaluator_RotateRowsStepsBatch, B200_Evaluator_LinearTransform ----

import ctypes as C  # noqa: E402

from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, E_POINTER  # noqa: E402
from sealc_checks import _libs  # noqa: E402
from sealc_driver import Sealc  # noqa: E402

vp, u64 = C.c_void_p, C.c_uint64
N4096_BATCHING = (4096, PARAMS["n4096"][1], 40961)  # the default n = 4096 chain with a batching plain modulus


def seam_setup(S, params, steps, count=3, seed=11):
    """reference and our contexts, Galois keys for `steps` (KeyGenerator_CreateGaloisKeysFromSteps) loaded into ours, and
    `count` fresh encryptions"""
    from refseal import RefContext
    n, moduli, t = params
    R = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = _libs(R, O)
    kg = R.keygen()
    gk = R.galois_keys_steps(kg, steps)
    ogk = OL.load("KSwitchKeys", RL.save("KSwitchKeys", gk, 0))
    enc = R.encryptor(R.public_key(kg))
    rng = np.random.default_rng(seed)
    rcts = [R.encrypt(enc, R.new_pt(rng.integers(0, t, size=n, dtype=np.uint64))) for _ in range(count)]
    octs = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts]
    return R, O, RL, OL, kg, gk, ogk, rcts, octs


def arr(x):
    return (vp * len(x))(*x) if x is not None else None


def steps_batch(S, O, hs, steps, glk, dsts, ev="default", count=None):
    st = (C.c_int * max(len(steps), 1))(*steps) if steps is not None else None
    return S.rc("B200_Evaluator_RotateRowsStepsBatch", O.ev if ev == "default" else ev, u64(len(hs) if count is None else count),
                arr(hs), st, glk, arr(dsts))


def lt_seam(S, O, hs, b, G, plains, glk, dsts, ev="default"):
    return S.rc("B200_Evaluator_LinearTransform", O.ev if ev == "default" else ev, u64(len(hs) if hs is not None else 1), arr(hs),
                u64(b), u64(G), arr(plains), glk, arr(dsts))


def chain(X, h, b, G, plains, glk):
    """the per-handle chain on X (ours or the reference): RotateRows, MultiplyPlain, Add"""
    rot = {0: h}
    for j in range(1, b):
        if any(plains[g * b + j] is not None for g in range(G)):
            rot[j] = X.rotate_rows(h, j, glk)
    acc = None
    for g in range(G):
        inner = None
        for j in range(b):
            p = plains[g * b + j]
            if p is None:
                continue
            prod = X.multiply_plain(rot[j], p)
            inner = prod if inner is None else X.add(inner, prod)
        if inner is None:
            continue
        if g:
            inner = X.rotate_rows(inner, g * b, glk)
        acc = inner if acc is None else X.add(acc, inner)
    return acc


def seam_checks(S, params):
    b, G = 3, 3
    steps = [1, 2, 3, 6, 5, -1]
    R, O, RL, OL, kg, gk, ogk, rcts, octs = seam_setup(S, params, steps)
    n, t = O.n, O.t
    words = lambda h: OL.save("Ciphertext", h, 0)
    rwords = lambda h: RL.save("Ciphertext", h, 0)
    fresh = lambda c=3: [OL.new("Ciphertext") for _ in range(c)]
    rng = np.random.default_rng(5)
    # RotateRowsStepsBatch: a step per item, 0 included, against per-handle RotateRows and the reference
    st = [5, 0, -1]
    d = fresh()
    assert steps_batch(S, O, octs, st, ogk, d) == 0
    for i in range(3):
        assert words(d[i]) == words(O.rotate_rows(octs[i], st[i], ogk)), f"item {i} step {st[i]} vs Evaluator_RotateRows"
        assert words(d[i]) == rwords(R.rotate_rows(rcts[i], st[i], gk)), f"item {i} step {st[i]} vs the reference"
    # LinearTransform against the per-handle chain and the reference, with and without absent terms
    coeffs = [rng.integers(0, t, size=n, dtype=np.uint64) for _ in range(b * G)]
    for absent in ([], [4], [2, 5, 8], [0, 1, 2]):
        op = [None if i in absent else O.new_pt(coeffs[i]) for i in range(b * G)]
        rp = [None if i in absent else R.new_pt(coeffs[i]) for i in range(b * G)]
        d = fresh()
        assert lt_seam(S, O, octs, b, G, op, ogk, d) == 0, absent
        for i in range(3):
            assert words(d[i]) == words(chain(O, octs[i], b, G, op, ogk)), f"absent {absent} item {i} vs the per-handle chain"
        assert words(d[0]) == rwords(chain(R, rcts[0], b, G, rp, gk)), f"absent {absent} vs the reference"
    op = [O.new_pt(c) for c in coeffs]
    # destinations aliasing encrypteds
    alias = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts]
    exp = [words(chain(O, h, b, G, op, ogk)) for h in alias]
    assert lt_seam(S, O, alias, b, G, op, ogk, alias[::-1]) == 0
    assert [words(h) for h in alias[::-1]] == exp
    alias = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts]
    exp = [words(O.rotate_rows(h, s, ogk)) for h, s in zip(alias, [1, 2, 3])]
    assert steps_batch(S, O, alias, [1, 2, 3], ogk, alias) == 0
    assert [words(h) for h in alias] == exp
    assert steps_batch(S, O, octs, [1], ogk, fresh(), count=0) == 0
    # HRESULTs
    assert steps_batch(S, O, octs, [1, 2, 4], ogk, fresh()) == E_INVALIDARG          # no key for 4 (the chain: NAF parts)
    assert lt_seam(S, O, octs, 4, 2, [op[0]] * 8, ogk, fresh()) == E_INVALIDARG     # giant step 4: no key
    assert steps_batch(S, O, octs, [1, n // 2, 1], ogk, fresh()) == E_INVALIDARG     # step too large
    assert lt_seam(S, O, octs, 1, n // 2, [op[0]] * (n // 2), ogk, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, octs, 0, 3, op, ogk, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, octs, 3, 0, op, ogk, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, octs, b, G, [None] * (b * G), ogk, fresh()) == E_INVALIDARG  # every term absent
    empty = OL.new("KSwitchKeys")
    assert steps_batch(S, O, octs, [1, 1, 1], empty, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, octs, b, G, op, empty, fresh()) == E_INVALIDARG
    size3 = O.multiply(octs[0], octs[1])
    assert steps_batch(S, O, [size3] + octs[1:], [1, 1, 1], ogk, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, [size3] + octs[1:], b, G, op, ogk, fresh()) == E_INVALIDARG
    ntt = O.new_ct(O.ct_words(octs[0]), ntt=True)
    assert steps_batch(S, O, [ntt] + octs[1:], [1, 1, 1], ogk, fresh()) == E_INVALIDARG
    assert lt_seam(S, O, [ntt] + octs[1:], b, G, op, ogk, fresh()) == E_INVALIDARG
    if len(R.data_parms_ids()) > 1:
        low = O.mod_switch_to_next(octs[0])
        assert steps_batch(S, O, [octs[0], low], [1, 1], ogk, fresh(2)) == E_INVALIDARG
        assert lt_seam(S, O, [octs[0], low], b, G, op, ogk, fresh(2)) == E_INVALIDARG
    assert steps_batch(S, O, octs, [1, 1, 1], ogk, fresh(), ev=None) == E_POINTER
    assert steps_batch(S, O, octs, None, ogk, fresh()) == E_POINTER
    assert steps_batch(S, O, octs, [1, 1, 1], None, fresh()) == E_POINTER
    assert steps_batch(S, O, octs, [1, 1, 1], ogk, None) == E_POINTER
    assert lt_seam(S, O, octs, b, G, op, ogk, fresh(), ev=None) == E_POINTER
    assert lt_seam(S, O, None, b, G, op, ogk, fresh()) == E_POINTER
    assert lt_seam(S, O, octs, b, G, None, ogk, fresh()) == E_POINTER
    assert lt_seam(S, O, octs, b, G, op, None, fresh()) == E_POINTER
    assert lt_seam(S, O, octs, b, G, op, ogk, None) == E_POINTER
    assert lt_seam(S, O, octs, b, G, op, ogk, [None] + fresh(2)) == E_INVALIDARG
    zero = O.new_pt(np.zeros(1, dtype=np.uint64))
    assert lt_seam(S, O, octs, b, G, [zero] + op[1:], ogk, fresh()) == COR_E_INVALIDOPERATION   # MultiplyPlain by zero
    # a trivial encryption (c1 = 0): the chain's rotations are transparent, the seam's final result too
    tr = O.ct_words(octs[0])
    tr[1] = 0
    trh = O.new_ct(tr)
    assert steps_batch(S, O, [trh], [1], ogk, fresh(1)) == COR_E_INVALIDOPERATION
    assert lt_seam(S, O, [trh], b, G, op, ogk, fresh(1)) == COR_E_INVALIDOPERATION


def seam_without_batching(S):
    n, moduli, t = PARAMS["n4096"]
    O = S.context(n, moduli, t)
    h = O.new_ct(np.zeros((2, O.k, n), dtype=np.uint64))
    keys = O.new_ksk({})
    p = O.new_pt(np.ones(1, dtype=np.uint64))
    assert steps_batch(S, O, [h], [1], keys, [O._dst()]) == COR_E_INVALIDOPERATION
    assert lt_seam(S, O, [h], 1, 2, [p, p], keys, [O._dst()]) == COR_E_INVALIDOPERATION


def seam_decrypted(S, params, d, b, seed, banded=False, two=False):
    """random (or banded, or one per slot row) d x d matrices through the layer-2 seam with keys from the helper's steps and
    batch-encoded diagonals: each slot row decrypts to M v mod t"""
    n, moduli, t = params
    rng = np.random.default_rng(seed)
    h = n // 2

    def mat():
        m = rng.integers(0, t, size=(d, d))
        if banded:
            m = np.where(np.abs(np.subtract.outer(np.arange(d), np.arange(d))) <= 2, m, 0)
        return m
    mats = (mat(), mat()) if two else mat()
    vecs, present, steps = bsgs_plain_vectors(mats, n, t, b)
    G = vecs.shape[0]
    R, O, RL, OL, kg, gk, ogk, _, _ = seam_setup(S, params, steps, count=0)
    enc, dec, be = R.encryptor(R.public_key(kg)), R.decryptor(R.secret_key(kg)), R.batch_encoder()
    x = rng.integers(0, t, size=(2, d), dtype=np.uint64)
    v = np.concatenate([np.tile(x[0], h // d), np.tile(x[1], h // d)])
    oct_ = OL.load("Ciphertext", RL.save("Ciphertext", R.encrypt(enc, R.batch_encode(be, v)), 0))
    plains = [OL.load("Plaintext", RL.save("Plaintext", R.batch_encode(be, vecs[g, j]), 0)) if present[g, j] else None
              for g in range(G) for j in range(b)]
    dst = [OL.new("Ciphertext")]
    assert lt_seam(S, O, [oct_], b, G, plains, ogk, dst) == 0
    got = RL.load("Ciphertext", OL.save("Ciphertext", dst[0], 0))
    slots = R.batch_decode(be, R.decrypt(dec, got))
    assert np.array_equal(slots, apply_slotwise(mats, v, n, t))


def test_emu_seams(emu_lib, ref):
    seam_checks(Sealc(emu_lib.lib), PARAMS["n8192"])


def test_emu_seams_without_batching(emu_lib):
    seam_without_batching(Sealc(emu_lib.lib))


@pytest.mark.parametrize("params,d,b", [(PARAMS["n8192"], 16, 4), (N4096_BATCHING, 16, 4)])
def test_emu_seam_decrypted(emu_lib, ref, params, d, b):
    seam_decrypted(Sealc(emu_lib.lib), params, d, b, seed=93)
    seam_decrypted(Sealc(emu_lib.lib), params, d, b, seed=94, banded=True, two=True)


@pytest.mark.gpu
@pytest.mark.parametrize("params", [PARAMS["n8192"], N4096_BATCHING])
def test_gpu_seams(ref, params):
    seam_checks(Sealc(CudaBackend().lib.lib), params)


@pytest.mark.gpu
def test_gpu_seams_without_batching():
    seam_without_batching(Sealc(CudaBackend().lib.lib))


@pytest.mark.gpu
@pytest.mark.parametrize("params,d,b", [(PARAMS["n8192"], 256, 16), (N4096_BATCHING, 128, 8)])
def test_gpu_seam_decrypted(ref, params, d, b):
    seam_decrypted(Sealc(CudaBackend().lib.lib), params, d, b, seed=95)
    seam_decrypted(Sealc(CudaBackend().lib.lib), params, d, b, seed=96, banded=True, two=True)
