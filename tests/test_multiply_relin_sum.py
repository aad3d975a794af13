"""Encrypted inner products: b200_multiply_relin_sum and B200_Evaluator_MultiplyRelinSum against the reference's multiply ->
relinearize -> add_inplace chain, word for word.  The same checks run on the CPU emulation build and, marked gpu, on the CUDA
library, where the launch traces show moddown_sum_kernel replacing the last kernel of one multiply_relin batch and every
addsub_kernel of the chain."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from backends import CudaBackend, EmuBackend
from params import PARAMS, WIDE
from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, E_POINTER, SealError
from sealc_checks import _libs
from sealc_driver import Sealc
from test_plain_sum import padded, signed_plain

vp, u64 = C.c_void_p, C.c_uint64
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def level_k(P, j):
    return P.ctx.level_info(P.ctx.first_level + j)["k"]


def ref_sum(P, a, b, rlk, j):
    """[R][2][k][n]: c = relin(mul(a[r][0], b[r][0])); c = c + relin(mul(a[r][i], b[r][i])) on the reference at data level j"""
    Rf = P.ref
    out = []
    for r in range(a.shape[0]):
        acc = None
        for i in range(a.shape[1]):
            ha = Rf.new_ct(a[r, i], level=j)
            hb = ha if b is a else Rf.new_ct(b[r, i], level=j)
            pm = Rf.multiply(ha, hb)
            t = Rf.relinearize(pm, rlk)
            for h in ([ha, pm] if hb is ha else [ha, hb, pm]):
                Rf.free_ct(h)
            if acc is None:
                acc = t
            else:
                nxt = Rf.add(acc, t)
                Rf.free_ct(acc)
                Rf.free_ct(t)
                acc = nxt
        out.append(Rf.ct_words(acc))
        Rf.free_ct(acc)
    return np.stack(out)


def mr_sum(P, a, b, dK, lv, square=False):
    """b200_multiply_relin_sum of host operands a, b [R][m][2][k][n] (square: b is a's device buffer itself)"""
    R, m, _, k, n = a.shape
    da = P.dev(a)
    db = da if square else P.dev(b)
    out = P.out(R, 2, k, n)
    P.ctx.multiply_relin_sum(da, db, dK, m, out, R, level=lv)
    return P.host(out).reshape(R, 2, k, n)


def chain_vs_reference(P, j, R, m, seed, key=None, a=None, b=None, square=False):
    rng = np.random.default_rng(seed)
    lv, k = P.ctx.first_level + j, level_k(P, j)
    if key is None:
        key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    if a is None:
        a = pc.rand_ct(rng, P.moduli, k, P.n, batch=R * m).reshape(R, m, 2, k, P.n)
    if b is None:
        b = a if square else pc.rand_ct(rng, P.moduli, k, P.n, batch=R * m).reshape(R, m, 2, k, P.n)
    rlk = P.ref.new_ksk({0: key})
    got = mr_sum(P, a, b, P.dev(key), lv, square=square)
    pc.eq(got, ref_sum(P, a, a if square else b, rlk, j), f"R = {R}, m = {m}, level {lv}{' (squares)' if square else ''}")
    return got


def check_levels(P, R=2, m=3, seed=1):
    for j in range(len(P.ref.data_parms_ids())):
        chain_vs_reference(P, j, R, m, seed=seed + j)


def check_m1(P, seed=2):
    """m = 1 is b200_multiply_relin word for word"""
    rng = np.random.default_rng(seed)
    k, R = P.k, 3
    key = P.dev(pc.rand_ksk(rng, P.moduli, P.k, P.n))
    a = pc.rand_ct(rng, P.moduli, k, P.n, batch=R)
    b = pc.rand_ct(rng, P.moduli, k, P.n, batch=R)
    o = P.out(R, 2, k, P.n)
    P.ctx.multiply_relin(P.dev(a), P.dev(b), key, o, R)
    pc.eq(mr_sum(P, a[:, None], b[:, None], key, None), P.host(o), "m = 1 vs multiply_relin")


def check_squares(P, seed=4):
    """b == a: the squares of a variance-style sum"""
    chain_vs_reference(P, 0, 1, 5, seed=seed, square=True)


def all_pm1_key(P):
    K = len(P.moduli)
    key = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        key[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    return key


def check_adversarial(P, R=1):
    """all-(q - 1) and single-word operands against random and all-(p - 1) keys"""
    qm1, single, alt = (pc.adversarial_ct(P, kind) for kind in ("qm1", "single", "alt"))
    a = np.stack([qm1, single, alt, qm1])[None].repeat(R, axis=0)
    b = np.stack([qm1, qm1, single, alt])[None].repeat(R, axis=0)
    for key in (None, all_pm1_key(P)):
        chain_vs_reference(P, 0, R, 4, seed=5, key=key, a=a, b=b)
        chain_vs_reference(P, 0, R, 4, seed=6, key=key, a=a, square=True)


def term_bytes(P, lv):
    """multiply_relin_sum's scratch estimate of one term (b200_bfv.cu)"""
    li = P.ctx.level_info(lv)
    k, R = li["k"], li["k"] + li["nBsk"]
    fp = max(int(q) for q in li["q"]).bit_length() <= 49
    keepD = fp and (k + 1) * (k + 2) <= 4 * R and k <= 8
    held = k + (3 * R if keepD else 2 * k)
    return (held + max(7 * R, (k + 1) * (k + 2))) * P.n * 8


def check_chunking(P, monkeypatch, seed=7):
    """B200_MR_SUM_SCRATCH of one output's terms (chunks of whole outputs) and of one term (each output's terms in chunks,
    the partial carried as the addend): the words of the unchunked sum"""
    rng = np.random.default_rng(seed)
    lv, k, R, m = P.ctx.first_level, P.k, 3, 3
    key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    a = pc.rand_ct(rng, P.moduli, k, P.n, batch=R * m).reshape(R, m, 2, k, P.n)
    b = pc.rand_ct(rng, P.moduli, k, P.n, batch=R * m).reshape(R, m, 2, k, P.n)
    dK = P.dev(key)
    whole = mr_sum(P, a, b, dK, lv)
    pc.eq(whole, ref_sum(P, a, b, P.ref.new_ksk({0: key}), 0), "unchunked")
    for cap in (m * term_bytes(P, lv), term_bytes(P, lv), 1):
        monkeypatch.setenv("B200_MR_SUM_SCRATCH", str(cap))
        pc.eq(mr_sum(P, a, b, dK, lv), whole, f"chunked at {cap} bytes")
    monkeypatch.delenv("B200_MR_SUM_SCRATCH")


def check_errors(P, lib):
    from sunscreen_b200.lib import B200Context, B200Error
    rng = np.random.default_rng(8)
    k, n = P.k, P.n
    key = P.dev(pc.rand_ksk(rng, P.moduli, P.k, n))
    buf = P.dev(pc.rand_ct(rng, P.moduli, k, n, batch=6))
    out = P.out(2, 2, k, n)

    def code(*args, level=None, ctx=P.ctx):
        with pytest.raises(B200Error) as e:
            ctx.multiply_relin_sum(*args, level=level)
        return e.value.code
    assert code(buf, buf, key, 0, out, 1) == -1            # m == 0
    assert code(None, buf, key, 2, out, 1) == -4
    assert code(buf, None, key, 2, out, 1) == -4
    assert code(buf, buf, None, 2, out, 1) == -4
    assert code(buf, buf, key, 2, None, 1) == -4
    assert code(buf, buf[4:], key, 2, buf[1:], 1) == -1    # out overlapping a
    assert code(buf[4:], buf, key, 2, buf[5:], 1) == -1    # out overlapping b
    assert code(buf, buf, key, 2, out, 1, level=0) == -2   # the key level: no key switching there
    ctx1 = B200Context(n, [P.moduli[0]], P.t, lib=lib)     # one prime: no key switching
    assert code(buf, buf, key, 2, out, 1, ctx=ctx1) == -2
    P.ctx.multiply_relin_sum(buf, buf, key, 2, buf, 0)     # rows == 0: no work, no overlap to report


# ---- layer 2 ----

def sealc_setup(S, name, count, seed=11):
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


def mr_seam(S, O, rows, cols, e1, e2, rlk, dsts, ev="default"):
    arr = lambda x: (vp * len(x))(*x) if x is not None else None
    return S.rc("B200_Evaluator_MultiplyRelinSum", O.ev if ev == "default" else ev, u64(rows), u64(cols), arr(e1), arr(e2), rlk,
                arr(dsts))


def chain(E, e1, e2, rlk):
    acc = None
    for x, y in zip(e1, e2):
        t = E.relinearize(E.multiply(x, y), rlk)
        acc = t if acc is None else E.add(acc, t)
    return acc


def sealc_checks(S, name, rows=2, cols=3):
    R, O, RL, OL, kg, rcts, octs = sealc_setup(S, name, 2 * rows * cols)
    words = lambda h: OL.save("Ciphertext", h, 0)
    rwords = lambda h: RL.save("Ciphertext", h, 0)
    fresh = lambda c=rows: [OL.new("Ciphertext") for _ in range(c)]
    rlk = R.relin_keys(kg)
    orlk = OL.load("KSwitchKeys", RL.save("KSwitchKeys", rlk, 0))
    T = rows * cols
    e1, e2 = octs[:T], octs[T:]
    d = fresh()
    assert mr_seam(S, O, rows, cols, e1, e2, orlk, d) == 0
    for i in range(rows):
        sl = slice(i * cols, (i + 1) * cols)
        assert words(d[i]) == words(chain(O, e1[sl], e2[sl], orlk)), f"{name}: row {i} vs the per-handle chain"
        assert words(d[i]) == rwords(chain(R, rcts[:T][sl], rcts[T:][sl], rlk)), f"{name}: row {i} vs the reference"
    # the same handle twice: squares
    d = fresh(1)
    assert mr_seam(S, O, 1, cols, e1[:cols], e1[:cols], orlk, d) == 0
    assert words(d[0]) == rwords(chain(R, rcts[:cols], rcts[:cols], rlk)), f"{name}: squares vs the reference"
    assert words(d[0]) == words(chain(O, e1[:cols], e1[:cols], orlk)), f"{name}: squares vs the per-handle chain"
    # destinations aliasing operands
    alias = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rcts[:cols]]
    exp = words(chain(O, alias, alias[::-1], orlk))
    assert mr_seam(S, O, 1, cols, alias, alias[::-1], orlk, [alias[1]]) == 0
    assert words(alias[1]) == exp
    assert mr_seam(S, O, 0, cols, e1, e2, orlk, fresh()) == 0
    # HRESULTs, each against the chain's
    assert mr_seam(S, O, rows, 0, e1, e2, orlk, fresh()) == E_INVALIDARG
    assert mr_seam(S, O, rows, cols, e1, e2, orlk, fresh(), ev=None) == E_POINTER
    assert mr_seam(S, O, rows, cols, None, e2, orlk, fresh()) == E_POINTER
    assert mr_seam(S, O, rows, cols, e1, None, orlk, fresh()) == E_POINTER
    assert mr_seam(S, O, rows, cols, e1, e2, None, fresh()) == E_POINTER
    assert mr_seam(S, O, rows, cols, e1, e2, orlk, None) == E_POINTER
    assert mr_seam(S, O, rows, cols, [None] + e1[1:], e2, orlk, fresh()) == E_POINTER
    assert mr_seam(S, O, rows, cols, e1, e2[:-1] + [None], orlk, fresh()) == E_POINTER
    assert mr_seam(S, O, rows, cols, e1, e2, orlk, [None] + fresh(rows - 1)) == E_POINTER
    ntt = O.new_ct(O.ct_words(e1[0]), ntt=True)
    assert mr_seam(S, O, rows, cols, [ntt] + e1[1:], e2, orlk, fresh()) == E_INVALIDARG
    size3 = O.multiply(e1[0], e1[1])
    assert mr_seam(S, O, rows, cols, [size3] + e1[1:], e2, orlk, fresh()) == E_INVALIDARG
    rsize3 = R.multiply(rcts[0], rcts[1])
    with pytest.raises(SealError) as e:
        R.relinearize(R.multiply(rsize3, rcts[2]), rlk)
    assert e.value.code == E_INVALIDARG
    if len(R.data_parms_ids()) > 1:
        low = O.mod_switch_to_next(e1[-1])
        assert mr_seam(S, O, rows, cols, e1[:-1] + [low], e2, orlk, fresh()) == E_INVALIDARG
        with pytest.raises(SealError) as e:
            R.multiply(rcts[0], R.mod_switch_to_next(rcts[1]))
        assert e.value.code == E_INVALIDARG
    empty = OL.new("KSwitchKeys")
    assert mr_seam(S, O, rows, cols, e1, e2, empty, fresh()) == E_INVALIDARG  # keys of another parms_id
    with pytest.raises(SealError) as e:
        R.relinearize(R.multiply(rcts[0], rcts[1]), R.new_ksk({}))
    assert e.value.code == E_INVALIDARG
    # a term of two transparent operands: the chain's Multiply refuses the product
    tr = O.ct_words(e1[0])
    tr[1] = 0
    trh = O.new_ct(tr)
    assert mr_seam(S, O, 1, 2, [e1[0], trh], [e2[0], trh], orlk, fresh(1)) == COR_E_INVALIDOPERATION
    with pytest.raises(SealError) as e:
        R.multiply(R.new_ct(tr), R.new_ct(tr))
    assert e.value.code == COR_E_INVALIDOPERATION
    # one transparent operand: the product is not transparent and the sum goes through
    d = fresh(1)
    assert mr_seam(S, O, 1, 2, [e1[0], trh], [e2[0], e2[1]], orlk, d) == 0
    assert words(d[0]) == words(chain(O, [e1[0], trh], [e2[0], e2[1]], orlk))


def sealc_without_keyswitching(S):
    """a one-prime chain: no key switching, so the chain's Relinearize throws logic_error"""
    n, moduli, t = 2048, [0x7fe6001], 12289
    O = S.context(n, moduli, t)
    h = O.new_ct(np.ones((2, 1, n), dtype=np.uint64))
    keys = O.new_ksk({0: np.zeros((1, 2, 1, n), dtype=np.uint64)})
    assert mr_seam(S, O, 1, 1, [h], [h], keys, [O._dst()]) == COR_E_INVALIDOPERATION


def decode_signed(coeffs, t):
    """Sunscreen's Signed decoding: sum of c_i 2^i with c_i > t / 2 read as c_i - t"""
    return sum((int(c) - t if int(c) > t // 2 else int(c)) << i for i, c in enumerate(coeffs))


def pir_replay(S, index=94):
    """Sunscreen's PIR example (10 x 10 database of 400 ... 499, Signed): stage 1 through MultiplyPlainSum, stage 2 through
    MultiplyRelinSum.  Decrypts to database[index]; the words are those of the reference's chain."""
    from refseal import RefContext
    n, moduli, t = PARAMS["n4096"]
    Rf = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = _libs(Rf, O)
    kg = Rf.keygen()
    sk, rlk = Rf.secret_key(kg), Rf.relin_keys(kg)
    enc, dec = Rf.encryptor(Rf.public_key(kg)), Rf.decryptor(sk)
    N = 10
    row, col = divmod(index, N)
    onehot = lambda i: [Rf.encrypt(enc, Rf.new_pt(padded(signed_plain(1 if j == i else 0, t), 1))) for j in range(N)]
    cq, rq = onehot(col), onehot(row)
    db = [[400 + i * N + j for j in range(N)] for i in range(N)]
    ocq = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in cq]
    orq = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in rq]
    orlk = OL.load("KSwitchKeys", RL.save("KSwitchKeys", rlk, 0))
    plains = [O.new_pt(signed_plain(db[i][j], t)) for i in range(N) for j in range(N)]
    cols = [O._dst() for _ in range(N)]
    assert S.rc("B200_Evaluator_MultiplyPlainSum", O.ev, u64(N), u64(N), (vp * N)(*ocq), (vp * (N * N))(*plains),
                (vp * N)(*cols)) == 0
    out = [O._dst()]
    assert mr_seam(S, O, 1, N, cols, orq, orlk, out) == 0
    # the reference's whole program
    rcols = []
    for i in range(N):
        acc = None
        for j in range(N):
            p = Rf.multiply_plain(cq[j], Rf.new_pt(signed_plain(db[i][j], t)))
            acc = p if acc is None else Rf.add(acc, p)
        rcols.append(acc)
    exp = chain(Rf, rcols, rq, rlk)
    assert OL.save("Ciphertext", out[0], 0) == RL.save("Ciphertext", exp, 0)
    got = RL.load("Ciphertext", OL.save("Ciphertext", out[0], 0))
    assert decode_signed(Rf.pt_coeffs(Rf.decrypt(dec, got)), t) == db[row][col] == 400 + index


def variance_replay(S, count=15):
    """a sum of 15 squares (mean_variance's numerator) decrypts to the sum of the squared values"""
    from refseal import RefContext
    n, moduli, t = PARAMS["n8192"]
    Rf = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = _libs(Rf, O)
    kg = Rf.keygen()
    rlk = Rf.relin_keys(kg)
    enc, dec, be = Rf.encryptor(Rf.public_key(kg)), Rf.decryptor(Rf.secret_key(kg)), Rf.batch_encoder()
    rng = np.random.default_rng(15)
    vals = rng.integers(0, 200, size=(count, n), dtype=np.uint64)
    hs = [Rf.encrypt(enc, Rf.batch_encode(be, v)) for v in vals]
    ohs = [OL.load("Ciphertext", RL.save("Ciphertext", h, 0)) for h in hs]
    orlk = OL.load("KSwitchKeys", RL.save("KSwitchKeys", rlk, 0))
    out = [O._dst()]
    assert mr_seam(S, O, 1, count, ohs, ohs, orlk, out) == 0
    assert OL.save("Ciphertext", out[0], 0) == RL.save("Ciphertext", chain(Rf, hs, hs, rlk), 0)
    got = RL.load("Ciphertext", OL.save("Ciphertext", out[0], 0))
    slots = Rf.batch_decode(be, Rf.decrypt(dec, got))
    exp = (vals.astype(object) ** 2).sum(axis=0) % t
    assert np.array_equal(slots.astype(object), exp)


# ---- CPU emulation build ----

@pytest.fixture(scope="module")
def emu_pairs(emu_lib, ref):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.pair_for(EmuBackend(emu_lib), name)
        return cache[name]
    return get


@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_49", "n8192_54", "n8192_60"])
def test_emu_chain_levels(emu_pairs, name):
    check_levels(emu_pairs(name))


def test_emu_chain_n16384(emu_pairs):
    """k = 8 and 7 take the separate scale (c0 / c1 from scratch), k <= 6 the scale inside the mod-down"""
    P = emu_pairs("n16384")
    for j in range(len(P.ref.data_parms_ids())):
        chain_vs_reference(P, j, 1, 2, seed=30 + j)


def test_emu_chain_long(emu_pairs):
    P = emu_pairs("n4096_9x22")
    check_levels(P, R=1, m=2)


def test_emu_m1_squares_adversarial(emu_pairs):
    P = emu_pairs("n4096")
    check_m1(P)
    check_squares(P)
    check_adversarial(P)


def test_emu_term_split(emu_pairs):
    """n = 1024, one output: 4 CTAs, below the emulation's 8, so the terms split into groups and a second pass sums them;
    three outputs fill it.  Every grouping gives the chain's words."""
    P = emu_pairs("n1024_2x27")
    for R, m in ((1, 1), (1, 2), (1, 7), (3, 5)):
        chain_vs_reference(P, 0, R, m, seed=40 + m)


def test_emu_pir_and_variance_shapes(emu_pairs):
    P = emu_pairs("n4096")
    chain_vs_reference(P, 0, 1, 10, seed=50)
    chain_vs_reference(P, 0, 1, 15, seed=51, square=True)


def test_emu_chunking(emu_pairs, monkeypatch):
    check_chunking(emu_pairs("n4096"), monkeypatch)


def test_emu_errors(emu_pairs, emu_lib):
    check_errors(emu_pairs("n4096"), emu_lib)


def test_emu_sealc_multiply_relin_sum(emu_lib, ref):
    sealc_checks(Sealc(emu_lib.lib), "n4096")


def test_emu_sealc_without_keyswitching(emu_lib):
    sealc_without_keyswitching(Sealc(emu_lib.lib))


def test_emu_pir_replay(emu_lib, ref):
    pir_replay(Sealc(emu_lib.lib))


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
@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_49", "n8192_54", "n8192_60", "n16384", "n8192_9x24", "n4096_9x22"])
def test_gpu_chain_levels(pairs, name):
    """every data level; on the nine-prime chains every cluster size of the key switch"""
    P = pairs(name)
    check_levels(P, R=1, m=3)
    check_levels(P, R=8, m=4, seed=20)


@pytest.mark.gpu
def test_gpu_chain_wide(pairs):
    P = pairs(WIDE[0])
    chain_vs_reference(P, 0, 1, 2, seed=60)


@pytest.mark.gpu
@pytest.mark.parametrize("R,m", [(1, 10), (1, 15), (1, 5), (1, 8), (1, 14), (2, 7), (64, 1), (64, 3), (1, 100)])
def test_gpu_shapes(pairs, R, m):
    """n = 8192, k = 4: PIR's R m = 10 runs the multiply's cluster (4 R_bsk 10 > 264) but not the key switch's (20 10 <= 264);
    R m = 5 runs neither, 14 both; R = 1 splits the terms, R = 64 does not"""
    chain_vs_reference(pairs("n8192"), 0, R, m, seed=R * 1000 + m)


@pytest.mark.gpu
def test_gpu_m1_squares_adversarial(pairs):
    P = pairs("n8192")
    check_m1(P)
    check_squares(P)
    check_adversarial(P)
    check_adversarial(P, R=16)


@pytest.mark.gpu
def test_gpu_chunking(pairs, monkeypatch):
    check_chunking(pairs("n8192"), monkeypatch)


@pytest.mark.gpu
def test_gpu_matches_multiply_relin_then_add(pairs):
    """256 outputs x 4 terms against b200_multiply_relin + b200_add on the same device"""
    P = pairs("n8192")
    rng = np.random.default_rng(12)
    R, m, k, n = 256, 4, P.k, P.n
    dK = P.dev(pc.rand_ksk(rng, P.moduli, P.k, n))
    a = P.dev(pc.rand_ct(rng, P.moduli, k, n, batch=R * m))
    b = P.dev(pc.rand_ct(rng, P.moduli, k, n, batch=R * m))
    o = P.out(R, 2, k, n)
    P.ctx.multiply_relin_sum(a, b, dK, m, o, R)
    prod = P.out(R * m, 2, k, n)
    P.ctx.multiply_relin(a, b, dK, prod, R * m)
    prod = prod.reshape(R, m, 2, k, n)
    acc = prod[:, 0].clone()
    for j in range(1, m):
        P.ctx.add(acc, prod[:, j].contiguous(), acc, 2, R)
    pc.eq(P.host(o), P.host(acc), "256 x 4 vs multiply_relin + add")


@pytest.mark.gpu
def test_gpu_errors(pairs):
    P = pairs("n4096")
    check_errors(P, P.be.lib)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n4096", "n8192"])
def test_gpu_sealc_multiply_relin_sum(ref, name):
    sealc_checks(Sealc(CudaBackend().lib.lib), name)


@pytest.mark.gpu
def test_gpu_sealc_without_keyswitching():
    sealc_without_keyswitching(Sealc(CudaBackend().lib.lib))


@pytest.mark.gpu
def test_gpu_pir_replay(ref):
    pir_replay(Sealc(CudaBackend().lib.lib))


@pytest.mark.gpu
def test_gpu_variance_replay(ref):
    variance_replay(Sealc(CudaBackend().lib.lib))


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
k, R, m = ctx.k(), {R}, {m}
rng = np.random.default_rng(1)
key = be.to_dev(pc.rand_ksk(rng, moduli, k, n))
a = be.to_dev(pc.rand_ct(rng, moduli, k, n, batch=R * m))
b = be.to_dev(pc.rand_ct(rng, moduli, k, n, batch=R * m))
o = be.empty((R, 2, k, n))
p = be.empty((R * m, 2, k, n))
ctx.{op}
be.torch.cuda.synchronize()
c0 = ctx.launch_count()
ctx.{op}
be.torch.cuda.synchronize()
print("launches", ctx.launch_count() - c0, flush=True)
be.lib.lib.b200_trace_dump()
"""


def traced(R, m, op):
    env = dict(os.environ, B200_TRACE="1")
    for var in ("B200_KS_CLUSTER", "B200_MUL_CLUSTER", "B200_KSMAC_TMA", "B200_MR_SPLIT", "B200_MR_SUM_SCRATCH"):
        env.pop(var, None)
    src = _TRACE.format(root=ROOT, tests=HERE, R=R, m=m, op=op)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", src]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    per_call = int(re.search(r"launches (\d+)", r.stdout).group(1))
    launches = {mm.group(1): int(mm.group(2)) for mm in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    return per_call, launches


def count(launches, prefix):
    return sum(v for key, v in launches.items() if key.startswith(prefix))


@pytest.mark.gpu
@pytest.mark.parametrize("R,m", [(1, 16), (16, 4)])
def test_gpu_trace(R, m):
    """above both cluster rules at n = 8192, k = 4: the sum's launches are one multiply_relin batch's with scale_moddown
    replaced by moddown_sum_kernel, plus its second pass where the terms split (one output: 32 CTAs; 16 outputs fill the GPU);
    no addsub_kernel.  (64 terms stay within the default 1 GiB scratch bound: one launch sequence.)"""
    fused, lf = traced(R, m, "multiply_relin_sum(a, b, key, m, o, R)")
    plain, lp = traced(R, m, "multiply_relin(a, b, key, p, R * m)")
    split = 1 if R == 1 else 0
    assert fused == plain + split, (fused, plain, lf, lp)
    assert count(lf, "moddown_sum_kernel") == 2 * (1 + split), lf
    assert count(lf, "scale_moddown_kernel_v2") == 0 and count(lf, "addsub_kernel") == 0, lf
    assert count(lp, "scale_moddown_kernel_v2") == 2, lp
    for name in ("mul_cluster_kernel", "ks_cluster_kernel"):
        assert lf.get(name, 0) == lp.get(name, 0) == 2, (name, lf, lp)
