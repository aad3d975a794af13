"""Rotate-and-sum slot reductions: b200_apply_galois_add and B200_Evaluator_RotateSumBatch against the reference's
apply_galois + add_inplace (rotate_rows / rotate_columns + add) chain, word for word.  The same checks run on the CPU emulation
build and, marked gpu, on the CUDA library, where the launch traces show the gather variant of the fused key switch
(ks_cluster_galois_kernel) and the rotate-add mod-down (ksmoddown_galois_add_kernel) replacing galois_kernel and addsub_kernel."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from backends import CudaBackend, EmuBackend
from params import PARAMS
from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, E_POINTER, SealError
from sealc_checks import _libs
from sealc_driver import Sealc

vp, u64 = C.c_void_p, C.c_uint64
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def row_elt(n, step):
    """the Galois element of rotate_rows(step) for 0 < step < n/2: 3^step mod 2n"""
    return pow(3, step, 2 * n)


def dot_prod_elts(n):
    """Sunscreen's dot_prod reduction: rotate_rows by 1, 2, 4, ..., n/4, then rotate_columns"""
    return [row_elt(n, 1 << i) for i in range((n // 4).bit_length())] + [2 * n - 1]


def level_k(P, j):
    return P.ctx.level_info(P.ctx.first_level + j)["k"]


def cluster_batch(P, j, side):
    """a batch just below ("below") or just above ("at") keyswitch_core's cluster rule k (k + 1) batch > 2 sm_count"""
    k = max(level_k(P, j), 2)
    last = (2 * P.ctx.sm_count) // (k * (k + 1))
    return max(1, last) if side == "below" else last + 1


def ref_rotate_add(P, c, j, elts, glk, addend=None):
    """the reference's chain c <- addend + apply_galois(c, g) for g in elts (addend None: c itself) at data level j"""
    R = P.ref
    cur = R.new_ct(c, level=j)
    for g in elts:
        rg = R.apply_galois(cur, g, glk)
        ra = cur if addend is None else R.new_ct(addend, level=j)
        nxt = R.add(ra, rg)
        R.free_ct(rg)
        if ra is not cur:
            R.free_ct(ra)
        R.free_ct(cur)
        cur = nxt
    out = R.ct_words(cur)
    R.free_ct(cur)
    return out


def chain_vs_reference(P, j, batch, elts, seed, key=None, cts=None):
    """c <- c + apply_galois(c, g) for g in elts over `batch` items at data level j, one b200_apply_galois_add per step with the
    addend equal to the input, item by item against the reference"""
    rng = np.random.default_rng(seed)
    lv, k = P.ctx.first_level + j, level_k(P, j)
    if key is None:
        key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    if cts is None:
        cts = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
    glk = P.ref.new_ksk({(g - 1) // 2: key for g in set(elts)})
    dK = P.dev(key)
    a, b = P.dev(cts), P.out(batch, 2, k, P.n)
    for g in elts:
        P.ctx.apply_galois_add(a, g, dK, a, b, batch, level=lv)
        a, b = b, a
    got = P.host(a).reshape(batch, 2, k, P.n)
    for i in range(batch):
        pc.eq(got[i], ref_rotate_add(P, cts[i], j, elts, glk), f"elements {elts} item {i} of {batch}, level {lv}")


def check_levels(P, elts, sides=("below",), seed=1):
    for j in range(len(P.ref.data_parms_ids())):
        for side in sides:
            chain_vs_reference(P, j, cluster_batch(P, j, side), elts, seed=seed + j)


def check_addend_modes(P, seed=3):
    """addend NULL (apply_galois alone), addend = in, addend = out (in place) and a separate addend"""
    rng = np.random.default_rng(seed)
    k, batch, g = P.k, 2, 3
    key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    glk = P.ref.new_ksk({(g - 1) // 2: key})
    cts = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
    X = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
    dK, dC = P.dev(key), P.dev(cts)
    R = P.ref
    only = []
    for i in range(batch):
        h = R.new_ct(cts[i])
        r = R.apply_galois(h, g, glk)
        only.append(R.ct_words(r))
    o = P.out(batch, 2, k, P.n)
    P.ctx.apply_galois_add(dC, g, dK, None, o, batch)
    pc.eq(P.host(o), np.stack(only), "addend NULL")
    o2 = P.out(batch, 2, k, P.n)
    P.ctx.apply_galois(dC, g, dK, o2, batch)
    pc.eq(P.host(o), P.host(o2), "addend NULL vs b200_apply_galois")
    P.ctx.apply_galois_add(dC, g, dK, dC, o, batch)
    pc.eq(P.host(o), np.stack([ref_rotate_add(P, cts[i], 0, [g], glk) for i in range(batch)]), "addend = in")
    exp_x = np.stack([ref_rotate_add(P, cts[i], 0, [g], glk, addend=X[i]) for i in range(batch)])
    P.ctx.apply_galois_add(dC, g, dK, P.dev(X), o, batch)
    pc.eq(P.host(o), exp_x, "separate addend")
    dX = P.dev(X)
    P.ctx.apply_galois_add(dC, g, dK, dX, dX, batch)
    pc.eq(P.host(dX), exp_x, "addend = out")


def check_adversarial(P):
    """all-(q - 1) and single-nonzero-word operands, random and all-(p - 1) keys"""
    K = len(P.moduli)
    pm1 = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        pm1[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    elts = [3, 2 * P.n - 1]
    for kind in ("qm1", "single", "alt"):
        c = pc.adversarial_ct(P, kind)[None]
        # (the reference refuses sigma_{2n-1} of the single word with the all-(p - 1) key: its result is transparent)
        chain_vs_reference(P, 0, 1, elts[:1] if kind == "single" else elts, seed=5, key=pm1, cts=c)
        chain_vs_reference(P, 0, 1, elts, seed=6, cts=c)


def check_errors(P, lib):
    from sunscreen_b200.lib import B200Context, B200Error
    rng = np.random.default_rng(8)
    k, n = P.k, P.n
    key = P.dev(pc.rand_ksk(rng, P.moduli, P.k, n))
    buf = P.dev(pc.rand_ct(rng, P.moduli, k, n, batch=3))
    out = P.out(3, 2, k, n)

    def code(*args, level=None, ctx=P.ctx):
        with pytest.raises(B200Error) as e:
            ctx.apply_galois_add(*args, level=level)
        return e.value.code
    assert code(buf, 4, key, buf, out, 2) == -1           # even element
    assert code(buf, 2 * n + 1, key, buf, out, 2) == -1   # element >= 2n
    assert code(None, 3, key, buf, out, 2) == -4
    assert code(buf, 3, None, buf, out, 2) == -4
    assert code(buf, 3, key, buf, None, 2) == -4
    assert code(buf, 3, key, None, buf, 2) == -1          # out == in
    assert code(buf, 3, key, None, buf[1:], 2) == -1      # out overlapping in
    assert code(buf[1:], 3, key, None, buf[:2], 2) == -1
    assert code(buf, 3, key, out[1:], out[:2], 2) == -1   # addend overlapping out without being out
    assert code(buf, 3, key, buf, out, 1, level=0) == -2   # the key level: no key switching below it
    ctx1 = B200Context(n, [P.moduli[0]], P.t, lib=lib)    # one prime: no key switching
    assert code(buf, 3, key, buf, out, 1, ctx=ctx1) == -2
    P.ctx.apply_galois_add(buf, 3, key, buf, buf, 0)      # batch 0: nothing to do, no overlap to report


# ---- layer 2 ----

def sealc_setup(S, name, count, seed=11):
    """reference and our contexts with the reference's keys, `count` fresh encryptions loaded into ours"""
    from refseal import RefContext
    n, moduli, t = PARAMS[name]
    R = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = _libs(R, O)
    kg = R.keygen()
    enc = R.encryptor(R.public_key(kg))
    rng = np.random.default_rng(seed)
    rcts = [R.encrypt(enc, R.new_pt(rng.integers(0, t, size=int(rng.integers(1, n)), dtype=np.uint64))) for _ in range(count)]
    octs = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts]
    return R, O, RL, OL, kg, rcts, octs


def own_chain(O, h, steps, columns, glk):
    cur = h
    for s in steps:
        cur = O.add(cur, O.rotate_rows(cur, s, glk))
    if columns:
        cur = O.add(cur, O.rotate_columns(cur, glk))
    return cur


def ref_chain(R, h, steps, columns, glk):
    cur = h
    for s in steps:
        cur = R.add(cur, R.rotate_rows(cur, s, glk))
    if columns:
        cur = R.add(cur, R.rotate_columns(cur, glk))
    return cur


def rotate_sum(S, O, hs, steps, columns, glk, dsts, ev="default", count=None):
    arr = lambda x: (vp * len(x))(*x) if x is not None else None
    st = (C.c_int * max(len(steps), 1))(*steps) if steps is not None else None
    return S.rc("B200_Evaluator_RotateSumBatch", O.ev if ev == "default" else ev, u64(len(hs) if count is None else count), arr(hs),
                C.c_int(len(steps) if steps is not None else 1), st, C.c_bool(columns), glk, arr(dsts))


def sealc_checks(S, name, count=3):
    R, O, RL, OL, kg, rcts, octs = sealc_setup(S, name, count)
    n = O.n
    words = lambda h: OL.save("Ciphertext", h, 0)
    rwords = lambda h: RL.save("Ciphertext", h, 0)
    fresh = lambda c=count: [OL.new("Ciphertext") for _ in range(c)]
    gall = R.galois_keys_all(kg)
    ogall = OL.load("KSwitchKeys", RL.save("KSwitchKeys", gall, 0))
    row_steps = [1 << i for i in range((n // 4).bit_length())]
    cases = [(row_steps, True), ([-1, -4, 0], False), ([3, -5, 7], True), ([0], False), ([], True), ([n // 2 - 1, 1 - n // 2], False)]
    for steps, columns in cases:
        d = fresh()
        assert rotate_sum(S, O, octs, steps, columns, ogall, d) == 0, (steps, columns)
        for i in range(count):
            exp = words(own_chain(O, octs[i], steps, columns, ogall))
            assert words(d[i]) == exp, f"{name}: steps {steps} columns {columns} item {i} vs the per-handle chain"
        assert words(d[0]) == rwords(ref_chain(R, rcts[0], steps, columns, gall)), f"{name}: steps {steps} vs the reference"
    # keys from steps: 3 has its own key, 5 = 4 + 1 goes through its NAF parts
    gst = R.galois_keys_steps(kg, [1, 3, 4])
    ogst = OL.load("KSwitchKeys", RL.save("KSwitchKeys", gst, 0))
    d = fresh()
    assert rotate_sum(S, O, octs, [3, 5, 1], False, ogst, d) == 0
    assert words(d[1]) == rwords(ref_chain(R, rcts[1], [3, 5, 1], False, gst))
    # destinations aliasing encrypteds, count 0
    alias = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts]
    exp = [words(own_chain(O, h, [1, 2], True, ogall)) for h in alias]
    assert rotate_sum(S, O, alias, [1, 2], True, ogall, alias[::-1]) == 0
    assert [words(h) for h in alias[::-1]] == exp
    assert rotate_sum(S, O, octs, [1], True, ogall, fresh(), count=0) == 0
    # HRESULTs, each against the chain's where the chain has one
    assert rotate_sum(S, O, octs, [2], False, ogst, fresh()) == E_INVALIDARG          # no key, no NAF decomposition
    with pytest.raises(SealError) as e:
        R.rotate_rows(rcts[0], 2, gst)
    assert e.value.code == E_INVALIDARG
    assert rotate_sum(S, O, octs, [1], True, ogst, fresh()) == E_INVALIDARG           # no key for 2n - 1
    assert rotate_sum(S, O, octs, [n // 2], False, ogall, fresh()) == E_INVALIDARG    # step too large
    with pytest.raises(SealError) as e:
        R.rotate_rows(rcts[0], n // 2, gall)
    assert e.value.code == E_INVALIDARG
    empty = OL.new("KSwitchKeys")
    assert rotate_sum(S, O, octs, [1], False, empty, fresh()) == E_INVALIDARG         # keys with another parms_id
    size3 = O.multiply(octs[0], octs[1])
    assert rotate_sum(S, O, [size3] + octs[1:], [1], False, ogall, fresh()) == E_INVALIDARG
    ntt = O.new_ct(O.ct_words(octs[0]), ntt=True)
    assert rotate_sum(S, O, [ntt] + octs[1:], [1], False, ogall, fresh()) == E_INVALIDARG
    if len(R.data_parms_ids()) > 1:
        low = O.mod_switch_to_next(octs[0])
        assert rotate_sum(S, O, [octs[0], low], [1], False, ogall, fresh(2)) == E_INVALIDARG
    assert rotate_sum(S, O, octs, [1], False, ogall, fresh(), ev=None) == E_POINTER
    assert rotate_sum(S, O, None, [1], False, ogall, fresh(), count=count) == E_POINTER
    assert rotate_sum(S, O, octs, [1], False, None, fresh()) == E_POINTER
    assert rotate_sum(S, O, octs, [1], False, ogall, None) == E_POINTER
    assert rotate_sum(S, O, octs, None, False, ogall, fresh()) == E_POINTER
    assert rotate_sum(S, O, octs, [1], False, ogall, [None] + fresh(count - 1)) == E_INVALIDARG
    # a trivial encryption (c1 = 0): the chain's first rotation is transparent, the seam's final result too
    tr = O.ct_words(octs[0])
    tr[1] = 0
    trh = O.new_ct(tr)
    assert rotate_sum(S, O, [trh], [1], True, ogall, fresh(1)) == COR_E_INVALIDOPERATION
    assert rotate_sum(S, O, [trh], [0], False, ogall, fresh(1)) == COR_E_INVALIDOPERATION
    with pytest.raises(SealError) as e:
        R.rotate_rows(R.new_ct(tr), 1, gall)
    assert e.value.code == COR_E_INVALIDOPERATION


def sealc_without_batching(S):
    n, moduli, t = PARAMS["n4096"]
    O = S.context(n, moduli, t)
    h = O.new_ct(np.zeros((2, O.k, n), dtype=np.uint64))
    keys = O.new_ksk({})
    assert rotate_sum(S, O, [h], [1], False, keys, [O._dst()]) == COR_E_INVALIDOPERATION


def dot_prod_replay(S):
    """Sunscreen's dot_prod at n = 8192: two Batched<4096> vectors (2 x 4096 slots), multiply + relinearize, the seam with steps
    1 ... 2048 and columns; every slot decrypts to the dot product, and the words are the reference chain's"""
    from refseal import RefContext
    n, moduli, t = PARAMS["n8192"]
    R = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = _libs(R, O)
    kg = R.keygen()
    sk, rlk, gk = R.secret_key(kg), R.relin_keys(kg), R.galois_keys_all(kg)
    enc, dec, be = R.encryptor(R.public_key(kg)), R.decryptor(sk), R.batch_encoder()
    rng = np.random.default_rng(21)
    a = rng.integers(0, 64, size=n, dtype=np.uint64)
    b = rng.integers(0, 64, size=n, dtype=np.uint64)
    ca, cb = R.encrypt(enc, R.batch_encode(be, a)), R.encrypt(enc, R.batch_encode(be, b))
    prod = R.relinearize(R.multiply(ca, cb), rlk)
    oprod = OL.load("Ciphertext", RL.save("Ciphertext", prod, 0))
    ogk = OL.load("KSwitchKeys", RL.save("KSwitchKeys", gk, 0))
    steps = [1 << i for i in range(12)]
    d = [OL.new("Ciphertext")]
    assert rotate_sum(S, O, [oprod], steps, True, ogk, d) == 0
    exp = ref_chain(R, prod, steps, True, gk)
    assert OL.save("Ciphertext", d[0], 0) == RL.save("Ciphertext", exp, 0)
    got = RL.load("Ciphertext", OL.save("Ciphertext", d[0], 0))
    slots = R.batch_decode(be, R.decrypt(dec, got))
    dot = int(sum(int(x) * int(y) for x, y in zip(a, b)) % t)
    assert np.all(slots == dot), (slots[:8], dot)


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
def test_emu_rotate_add_levels(emu_pairs, name):
    P = emu_pairs(name)
    check_levels(P, [3, 2 * P.n - 1])


def test_emu_dot_prod_elements(emu_pairs):
    P = emu_pairs("n2048_2x27")
    chain_vs_reference(P, 0, 2, dot_prod_elts(P.n), seed=4)


@pytest.mark.parametrize("name", ["n4096", "n8192_54"])
def test_emu_addend_modes(emu_pairs, name):
    check_addend_modes(emu_pairs(name))


def test_emu_adversarial(emu_pairs):
    check_adversarial(emu_pairs("n4096"))


def test_emu_errors(emu_pairs, emu_lib):
    check_errors(emu_pairs("n4096"), emu_lib)


def test_emu_sealc_rotate_sum(emu_lib, ref):
    sealc_checks(Sealc(emu_lib.lib), "n2048_2x27")


def test_emu_sealc_without_batching(emu_lib):
    sealc_without_batching(Sealc(emu_lib.lib))


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


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n8192_54", "n8192_60", "n16384", "n4096", "n4096_9x22", "n8192_9x24"])
def test_gpu_rotate_add_levels(pairs, name):
    """every data level, batches on both sides of the cluster rule, elements 3, 3^2, 3^5 and 2n - 1"""
    P = pairs(name)
    check_levels(P, [3, 9, 243, 2 * P.n - 1], sides=("below", "at"))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 16, 64])
def test_gpu_dot_prod_sequence(pairs, batch):
    """the dot_prod reduction's 13 elements at n = 8192, k = 4 (batch 16 and 64: the cluster path)"""
    P = pairs("n8192")
    chain_vs_reference(P, 0, batch, dot_prod_elts(P.n), seed=batch)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n8192_60", "n16384"])
def test_gpu_addend_modes(pairs, name):
    check_addend_modes(pairs(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n8192_54", "n4096"])
def test_gpu_adversarial(pairs, name):
    check_adversarial(pairs(name))


@pytest.mark.gpu
def test_gpu_adversarial_cluster_path(pairs):
    """all-(q - 1) and alternating 0 / (q - 1) operands with an all-(p - 1) key on the cluster path (16 items at k = 4)"""
    P = pairs("n8192")
    K = len(P.moduli)
    pm1 = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        pm1[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    c = np.broadcast_to(pc.adversarial_ct(P, "qm1"), (16, 2, P.k, P.n)).copy()
    c[1::2] = pc.adversarial_ct(P, "alt")
    chain_vs_reference(P, 0, 16, [3, 2 * P.n - 1], seed=9, key=pm1, cts=c)


@pytest.mark.gpu
def test_gpu_matches_apply_galois_then_add(pairs):
    """1024 items of the dot_prod sequence against b200_apply_galois + b200_add on the same device"""
    P = pairs("n8192")
    rng = np.random.default_rng(12)
    batch, k = 1024, P.k
    dK = P.dev(pc.rand_ksk(rng, P.moduli, P.k, P.n))
    cts = P.dev(pc.rand_ct(rng, P.moduli, k, P.n, batch=batch))
    a, b = cts.clone(), P.out(batch, 2, k, P.n)
    x, y = cts.clone(), P.out(batch, 2, k, P.n)
    for g in dot_prod_elts(P.n):
        P.ctx.apply_galois_add(a, g, dK, a, b, batch)
        a, b = b, a
        P.ctx.apply_galois(x, g, dK, y, batch)
        P.ctx.add(x, y, x, 2, batch)
    pc.eq(P.host(a), P.host(x), "1024 items vs apply_galois + add")


@pytest.mark.gpu
def test_gpu_errors(pairs):
    P = pairs("n4096")
    check_errors(P, P.be.lib)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n2048_2x27", "n8192"])
def test_gpu_sealc_rotate_sum(ref, name):
    sealc_checks(Sealc(CudaBackend().lib.lib), name)


@pytest.mark.gpu
def test_gpu_sealc_without_batching():
    sealc_without_batching(Sealc(CudaBackend().lib.lib))


@pytest.mark.gpu
def test_gpu_dot_prod_replay(ref):
    dot_prod_replay(Sealc(CudaBackend().lib.lib))


_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import parity_checks as pc
from backends import CudaBackend
from params import PARAMS
from sunscreen_b200.lib import B200Context
be = CudaBackend()
n, moduli, t = PARAMS["n8192"]
ctx = B200Context(n, moduli, t)
k, batch = ctx.k(), {batch}
rng = np.random.default_rng(1)
key = be.to_dev(pc.rand_ksk(rng, moduli, k, n))
a = be.to_dev(pc.rand_ct(rng, moduli, k, n, batch=batch))
o = be.empty((batch, 2, k, n))
ctx.apply_galois_add(a, 3, key, a, o, batch)
be.torch.cuda.synchronize()
c0 = ctx.launch_count()
ctx.apply_galois_add(o, 9, key, o, a, batch)
be.torch.cuda.synchronize()
print("launches", ctx.launch_count() - c0, flush=True)
be.lib.lib.b200_trace_dump()
"""


def traced(batch):
    env = dict(os.environ, B200_TRACE="1")
    for var in ("B200_KS_CLUSTER", "B200_KSMAC_TMA"):
        env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _TRACE.format(root=ROOT, tests=HERE, batch=batch)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    per_step = int(re.search(r"launches (\d+)", r.stdout).group(1))
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    return per_step, launches


def count(launches, prefix):
    return sum(v for key, v in launches.items() if key.startswith(prefix))


@pytest.mark.gpu
def test_gpu_trace_cluster_step():
    """16 items at k = 4 (above the cluster rule): the gather variant of the fused key switch and the rotate-add mod-down, two
    launches per step, no galois_kernel and no addsub_kernel"""
    per_step, launches = traced(16)
    assert per_step == 2, (per_step, launches)
    assert launches.get("ks_cluster_galois_kernel", 0) == 2, launches
    assert count(launches, "ksmoddown_galois_add_kernel") == 2, launches
    assert count(launches, "galois_kernel") == 0 and count(launches, "addsub_kernel") == 0, launches
    assert "ks_cluster_kernel" not in launches, launches


@pytest.mark.gpu
def test_gpu_trace_below_rule():
    """one item: the separate kernels, with galois_kernel writing sigma(c1) alone and no add"""
    per_step, launches = traced(1)
    assert count(launches, "galois_kernel") == 2, launches
    assert count(launches, "ksmoddown_galois_add_kernel") == 2, launches
    assert count(launches, "addsub_kernel") == 0 and count(launches, "ks_cluster") == 0, launches
    assert per_step == 5, (per_step, launches)  # galois_kernel, forward NTT, MAC, inverse NTT, mod-down
