"""Batched encryption: b200_encrypt_pk and b200_encrypt_sk, and the layer-2 seams B200_Encryptor_EncryptBatch and
B200_Encryptor_EncryptSlotsBatch, against the reference's seeded Encryptor_Encrypt{,Symmetric}ReturnComponentsSetSeed word for
word (ciphertexts, u and e), against our own per-handle calls, and through decryption.  The same checks run on the CPU
emulation build and, marked gpu, on the CUDA library."""
import ctypes as C

import numpy as np
import pytest

import parity_checks as pc
import sealc_checks as sc
from backends import CudaBackend, EmuBackend
from params import PARAMS, PLAIN_EDGE
from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, E_POINTER, RefContext
from sealc_driver import Sealc
from test_slots import _arr, value_rows

vp, u64 = C.c_void_p, C.c_uint64

# a chain without key switching: one prime, so the key level is the only data level
NO_KS = (8192, PARAMS["n8192"][1][:1], PARAMS["n8192"][2])
EMU_SETS = ["n4096", "n8192", "n4096_q_below_t"] + [p for p in PLAIN_EDGE if PARAMS[p][0] <= 8192] + ["no_ks"]
GPU_SETS = EMU_SETS + ["n16384", "n32768_60x6", "n16384_17x25"]


class NoKsPair(pc.Pair):
    """pc.Pair for NO_KS, whose single prime the appendix-B inputs of pc.Pair do not cover"""

    def __init__(self, be):
        from sunscreen_b200.lib import B200Context
        self.be = be
        self.n, self.moduli, self.t = NO_KS[0], list(NO_KS[1]), NO_KS[2]
        self.ref = RefContext(*NO_KS)
        self.ctx = B200Context(*NO_KS, lib=be.lib)
        self.k = self.ctx.k()


def pair(be, name):
    return NoKsPair(be) if name == "no_ks" else pc.pair_for(be, name)


def plaintexts(n, t, items, rng):
    """[items][n]: zero, all t - 1, a short plaintext (zero-padded), coefficients in the upper half, then uniform below t"""
    out = rng.integers(0, t, size=(items, n), dtype=np.uint64)
    kinds = [np.zeros(n, dtype=np.uint64), np.full(n, t - 1, dtype=np.uint64),
             np.concatenate([rng.integers(0, t, size=5, dtype=np.uint64), np.zeros(n - 5, dtype=np.uint64)]),
             rng.integers((t + 1) // 2, t, size=n, dtype=np.uint64)]
    for i in range(min(items, len(kinds))):
        out[i] = kinds[i]
    return out


def seed_rows(items, rng):
    s = rng.integers(0, 2**63, size=(items, 8), dtype=np.uint64)
    s[0] = np.arange(1, 9)
    return s


def residues(small, moduli):
    """[polys][n] small signed values -> [polys][len(moduli)][n] residues"""
    s = np.asarray(small, dtype=np.int64)
    return np.stack([np.where(s < 0, np.uint64(q) - (-s).astype(np.uint64), s.astype(np.uint64)) for q in moduli], axis=-2)


# ---- the reference's seeded component entry points ----

class RefKeys:
    def __init__(self, P):
        R, n = P.ref, P.n
        kg = R.keygen()
        self.sk, self.pk = R.secret_key(kg), R.public_key(kg)
        self.enc = R.encryptor(self.pk, self.sk)
        self.pk_words = sc._ref_pk_words(R, self.pk)                       # [2][K][n] NTT form
        h = vp()
        R.ref.call("SecretKey_Data", self.sk, C.byref(h))
        self.sk_words = R.pt_coeffs(h).reshape(-1, n)                      # [K][n] NTT form


def _pa(R):
    h = vp()
    R.ref.call("PolynomialArray_Create", None, C.byref(h))
    return h


def ref_components(P, keys, msg, seed, dsm):
    """(ciphertext words, u export, e export) of the reference's Encryptor_EncryptReturnComponentsSetSeed"""
    R = P.ref
    rct, pu, pe, rem = R.new_ct(), _pa(R), _pa(R), vp()
    R.ref.call("Plaintext_Create1", None, C.byref(rem))
    sd = (u64 * 8)(*[int(x) for x in seed])
    pt = R.new_pt(msg)
    R.ref.call("Encryptor_EncryptReturnComponentsSetSeed", keys.enc, pt, C.c_bool(dsm), rct, pu, pe, rem, sd, None)
    out = (R.ct_words(rct), sc._pa_export(R.ref, pu)[1], sc._pa_export(R.ref, pe)[1])
    for h in (pu, pe):
        R.ref.call("PolynomialArray_Destroy", h)
    R.free_pt(pt)
    R.free_pt(rem)
    R.free_ct(rct)
    return out


# ---- layer 1 ----

def check_layer1(P, batch_sizes=(1, 3), seed=71):
    """every item of b200_encrypt_pk (disable_special_modulus off and on) and b200_encrypt_sk equals the reference's seeded
    ReturnComponents ciphertext word for word, and samples_out / noise_out give its u and e"""
    n, t = P.n, P.t
    keys = RefKeys(P)
    rng = np.random.default_rng(seed)
    dpk, dsk = P.dev(keys.pk_words), P.dev(keys.sk_words)
    K, k1 = len(P.moduli), P.k
    for B in batch_sizes:
        msgs, seeds = plaintexts(n, t, B, rng), seed_rows(B, rng)
        dplain = P.dev(msgs)
        for dsm in (False, True):
            out, smp = P.out(B, 2, k1, n), np.zeros((B, 3, n), dtype=np.int8)
            P.ctx.encrypt_pk(dpk, seeds, dplain, out, B, disable_special_modulus=dsm, samples_out=smp)
            got = P.host(out).reshape(B, 2, k1, n)
            ke = k1 if dsm else K  # pk encryption is made at the key level unless the special modulus is disabled
            for i in range(B):
                what = f"encrypt_pk B={B} dsm={dsm} item {i}"
                ct, u, e = ref_components(P, keys, msgs[i], seeds[i], dsm)
                pc.eq(got[i], ct, what)
                pc.eq(residues(smp[i, :1], P.moduli[:ke]), u, what + " u")
                pc.eq(residues(smp[i, 1:], P.moduli[:ke]), e, what + " e")
        out, noise = P.out(B, 2, k1, n), np.zeros((B, n), dtype=np.int8)
        P.ctx.encrypt_sk(dsk, seeds, dplain, out, B, noise_out=noise)
        got = P.host(out).reshape(B, 2, k1, n)
        for i in range(B):
            check_sk_item(P, keys, got[i], noise[i], msgs[i], f"encrypt_sk B={B} item {i}")
        # the same seeds give the same words, without the sample output too; other seeds other words
        out2 = P.out(B, 2, k1, n)
        P.ctx.encrypt_sk(dsk, seeds, dplain, out2, B)
        pc.eq(P.host(out2), got, f"encrypt_sk B={B} without noise_out")
        # the two steps separately: the same samples and words
        c1, e1 = np.zeros((B, k1, n), dtype=np.uint64), np.zeros((B, n), dtype=np.int8)
        P.ctx.sample_sk(seeds, c1, e1, B)
        pc.eq(e1.view(np.uint8), noise.view(np.uint8), f"sample_sk B={B} noise")
        out3 = P.out(B, 2, k1, n)
        P.ctx.encrypt_sk_samples(dsk, c1, e1, dplain, out3, B)
        pc.eq(P.host(out3), got, f"sample_sk + encrypt_sk_samples B={B}")
        smp2, out4 = np.zeros((B, 3, n), dtype=np.int8), P.out(B, 2, k1, n)
        P.ctx.sample_pk(seeds, smp2, B)
        P.ctx.encrypt_pk_samples(dpk, smp2, dplain, out4, B)
        P.be.sync()
        P.ctx.encrypt_pk(dpk, seeds, dplain, out3, B)
        pc.eq(P.host(out4), P.host(out3), f"sample_pk + encrypt_pk_samples B={B}")
        seeds[:, 7] ^= np.uint64(1)
        P.ctx.encrypt_sk(dsk, seeds, dplain, out2, B)
        again = P.host(out2).reshape(B, 2, k1, n)
        assert all(not np.array_equal(again[i, 1], got[i, 1]) for i in range(B))


def check_sk_item(P, keys, ct, e, msg, what):
    """c0 == -(c1 s + e) + round(Q m / t) in every residue, with c1 and e as encrypt_sk gave them, the product taken with the
    reference's NTT.  (The reference's Encryptor_EncryptSymmetricReturnComponentsSetSeed does not forward the seed to
    encrypt_zero_symmetric, so its words are random: check_sk_golden holds the seeded stream to fixed words.)"""
    R, n, t, k1 = P.ref, P.n, P.t, P.k
    assert np.abs(e.astype(np.int64)).max() <= 19
    Q = 1
    for q in P.moduli[:k1]:
        Q *= int(q)
    m = [int(x) for x in msg]
    scaled = [(x * Q + (t + 1) // 2) // t for x in m]   # round(Q m / t), the rule of multiply_add_plain_with_scaling_variant
    for r in range(k1):
        q = int(P.moduli[r])
        c1 = ct[1, r]
        assert int(c1.max()) < q, what
        prod = R.ref.ntt_inverse(q, (R.ref.ntt_forward(q, c1[None]).astype(object) * keys.sk_words[r].astype(object) % q)
                                 .astype(np.uint64))[0]
        want = [(-(int(a) + int(b)) + sc_) % q for a, b, sc_ in zip(prod, e, scaled)]
        pc.eq(ct[0, r], np.array(want, dtype=np.uint64), f"{what} c0 residue {r}")


def check_launch_counts(P):
    """both calls issue as many launches for 257 items as for one"""
    n, k1, K = P.n, P.k, len(P.moduli)
    big = 257
    pk, sk = P.out(2, K, n), P.out(K, n)
    plain, out = P.out(big, n), P.out(big, 2, k1, n)
    seeds = np.zeros((big, 8), dtype=np.uint64)
    calls = {
        "encrypt_pk": lambda m: P.ctx.encrypt_pk(pk, seeds, plain, out, m),
        "encrypt_pk dsm": lambda m: P.ctx.encrypt_pk(pk, seeds, plain, out, m, disable_special_modulus=True),
        "encrypt_sk": lambda m: P.ctx.encrypt_sk(sk, seeds, plain, out, m),
    }
    for name, call in calls.items():
        deltas = []
        for m in (1, big, 1):
            before = P.ctx.launch_count()
            call(m)
            deltas.append(P.ctx.launch_count() - before)
        assert deltas[0] == deltas[1] == deltas[2] > 0, (name, deltas)


def check_arguments(P):
    from sunscreen_b200.lib import B200Error
    n, K, k1 = P.n, len(P.moduli), P.k
    buf, seeds = P.out(2, K, n), np.zeros((1, 8), dtype=np.uint64)
    for call in (lambda: P.ctx.encrypt_pk(None, seeds, buf, buf, 1), lambda: P.ctx.encrypt_pk(buf, None, buf, buf, 1),
                 lambda: P.ctx.encrypt_pk(buf, seeds, None, buf, 1), lambda: P.ctx.encrypt_pk(buf, seeds, buf, None, 1),
                 lambda: P.ctx.encrypt_sk(None, seeds, buf, buf, 1), lambda: P.ctx.encrypt_sk(buf, None, buf, buf, 1),
                 lambda: P.ctx.encrypt_sk(buf, seeds, None, buf, 1), lambda: P.ctx.encrypt_sk(buf, seeds, buf, None, 1)):
        with pytest.raises(B200Error) as e:
            call()
        assert e.value.code == -4
    out = P.out(1, 2, k1, n)
    P.ctx.encrypt_pk(buf, seeds, buf, out, 0)
    P.ctx.encrypt_sk(buf, seeds, buf, out, 0)
    assert not P.host(out).any()


# ---- layer 2 ----

def sealc_seams(S, name, seed=13, big=3):
    """EncryptBatch and EncryptSlotsBatch against the reference and our per-handle calls, the round trip through
    DecryptSlotsBatch, and every HRESULT"""
    n, moduli, t = PARAMS[name]
    R = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = sc._libs(R, O)
    rng = np.random.default_rng(seed)
    kg = R.keygen()
    rsk, rpk = R.secret_key(kg), R.public_key(kg)
    renc = R.encryptor(rpk, rsk)
    osk, opk = OL.load("SecretKey", RL.save("SecretKey", rsk, 0)), OL.load("PublicKey", RL.save("PublicKey", rpk, 0))
    obe, oenc, opk_only, osk_only, odec = vp(), vp(), vp(), vp(), vp()
    S.call("BatchEncoder_Create", O.ctx, C.byref(obe))
    S.call("Encryptor_Create", O.ctx, opk, osk, C.byref(oenc))
    S.call("Encryptor_Create", O.ctx, opk, None, C.byref(opk_only))
    S.call("Encryptor_Create", O.ctx, None, osk, C.byref(osk_only))
    S.call("Decryptor_Create", O.ctx, osk, C.byref(odec))

    def encrypt_batch(plains, seeds, symmetric, enc=None, dsts=None, count=None):
        dsts = [OL.new("Ciphertext") for _ in plains] if dsts is None else dsts
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64).ctypes.data_as(C.POINTER(u64))
        rc = S.rc("B200_Encryptor_EncryptBatch", oenc if enc is None else enc, u64(len(plains) if count is None else count),
                  _arr(plains), sd, C.c_bool(symmetric), _arr(dsts))
        return rc, dsts

    def slots_batch(vals, signed, seeds, symmetric, enc=None, be=None, dsts=None):
        vals = np.ascontiguousarray(vals)
        dsts = [OL.new("Ciphertext") for _ in range(vals.shape[0])] if dsts is None else dsts
        sd = None if seeds is None else np.ascontiguousarray(seeds, dtype=np.uint64).ctypes.data_as(C.POINTER(u64))
        rc = S.rc("B200_Encryptor_EncryptSlotsBatch", oenc if enc is None else enc, obe if be is None else be, u64(vals.shape[0]),
                  u64(vals.shape[1]), vals.ctypes.data_as(C.c_void_p), C.c_bool(signed), sd, C.c_bool(symmetric), _arr(dsts))
        return rc, dsts

    def per_handle(pt, sd, symmetric):
        h = OL.new("Ciphertext")
        s8 = (u64 * 8)(*[int(x) for x in sd])
        if symmetric:
            pe, rem = vp(), vp()
            S.call("PolynomialArray_Create", None, C.byref(pe))
            S.call("Plaintext_Create1", None, C.byref(rem))
            S.call("Encryptor_EncryptSymmetricReturnComponentsSetSeed", oenc, pt, h, pe, rem, s8, None)
        else:
            S.call("B200_Encryptor_EncryptSetSeed", oenc, pt, s8, h)
        return O.ct_words(h)

    def ref_seeded(msg, sd):
        rct, pu, pe, rem = R.new_ct(), vp(), vp(), vp()
        for h in (pu, pe):
            R.ref.call("PolynomialArray_Create", None, C.byref(h))
        R.ref.call("Plaintext_Create1", None, C.byref(rem))
        s8 = (u64 * 8)(*[int(x) for x in sd])
        R.ref.call("Encryptor_EncryptReturnComponentsSetSeed", renc, R.new_pt(msg), C.c_bool(False), rct, pu, pe, rem, s8, None)
        return R.ct_words(rct)

    # seeded EncryptBatch: the reference and B200_Encryptor_EncryptSetSeed / our symmetric SetSeed entry point, item by item
    msgs = plaintexts(n, t, 5, rng)
    msgs_short = [msgs[0][:0], msgs[2][:5]] + list(msgs[1:])
    plains = [O.new_pt(m) for m in msgs_short]
    seeds = seed_rows(len(plains), rng)
    for symmetric in (False, True):
        rc, dsts = encrypt_batch(plains, seeds, symmetric)
        assert rc == 0
        for i, h in enumerate(dsts):
            what = f"{name}: EncryptBatch symmetric={symmetric} item {i}"
            got = O.ct_words(h)
            if not symmetric:  # the reference's symmetric SetSeed path ignores the seed (see check_sk_item)
                pc.eq(got, ref_seeded(msgs_short[i], seeds[i]), what + " vs the reference")
            pc.eq(got, per_handle(plains[i], seeds[i], symmetric), what + " vs the per-handle call")
    # EncryptSlotsBatch == EncodeBatch then per-item seeded encryption
    for signed in (False, True):
        for per in (n, 7):
            vals = value_rows(t, per, signed, big, rng)
            seeds = seed_rows(big, rng)
            enc_pts = [OL.new("Plaintext") for _ in range(big)]
            S.call("B200_BatchEncoder_EncodeBatch", obe, u64(big), u64(per), np.ascontiguousarray(vals).ctypes.data_as(C.POINTER(u64)),
                   C.c_bool(signed), _arr(enc_pts))
            for symmetric in (False, True):
                rc, dsts = slots_batch(vals.view(np.uint64), signed, seeds, symmetric)
                assert rc == 0
                for i in range(big):
                    pc.eq(O.ct_words(dsts[i]), per_handle(enc_pts[i], seeds[i], symmetric),
                          f"{name}: EncryptSlotsBatch signed={signed} per={per} symmetric={symmetric} item {i}")
    # round trip: unseeded batches decrypt to the values with a positive budget; two calls give different words
    for signed in (False, True):
        vals = value_rows(t, n, signed, big, rng)
        for symmetric in (False, True):
            rc, dsts = slots_batch(vals.view(np.uint64), signed, None, symmetric)
            assert rc == 0
            rc, again = slots_batch(vals.view(np.uint64), signed, None, symmetric)
            assert rc == 0
            out = np.zeros((big, n), dtype=np.uint64)
            bud = (C.c_int * big)()
            S.call("B200_Decryptor_DecryptSlotsBatch", odec, obe, u64(big), _arr(dsts), C.c_bool(signed),
                   out.ctypes.data_as(C.c_void_p), bud)
            pc.eq(out, vals.view(np.uint64), f"{name}: round trip signed={signed} symmetric={symmetric}")
            assert min(bud) > 0, list(bud)
            for i in range(big):
                assert not np.array_equal(O.ct_words(dsts[i]), O.ct_words(again[i])), (signed, symmetric, i)
    # HRESULTs, each with the destinations left untouched
    keep = encrypt_batch(plains[:2], seeds[:2], False)[1]
    before = [O.ct_words(h) for h in keep]

    def untouched():
        for h, w in zip(keep, before):
            pc.eq(O.ct_words(h), w, f"{name}: destination after a refused call")

    big_pt = O.new_pt(np.full(3, t, dtype=np.uint64))                  # a coefficient not below t
    long_pt = O.new_pt(np.zeros(n + 1, dtype=np.uint64))               # more than n coefficients
    ntt_pt = vp()
    S.call("Plaintext_Create5", plains[1], C.byref(ntt_pt))
    S.call("Plaintext_SetParmsId", ntt_pt, O.first_id)
    for symmetric in (False, True):
        for bad in (big_pt, long_pt, ntt_pt):
            assert encrypt_batch([plains[0], bad], None, symmetric, dsts=keep)[0] == E_INVALIDARG
            untouched()
        assert encrypt_batch([plains[0], None], None, symmetric, dsts=keep)[0] == E_INVALIDARG
        assert encrypt_batch(plains[:2], None, symmetric, dsts=[keep[0], None])[0] == E_INVALIDARG
        untouched()
        # a destination listed twice (the items are written concurrently)
        assert encrypt_batch(plains[:3], None, symmetric, dsts=[keep[0], keep[1], keep[0]])[0] == E_INVALIDARG
        assert slots_batch(np.zeros((2, 4), dtype=np.uint64), False, None, symmetric, dsts=[keep[1], keep[1]])[0] == E_INVALIDARG
        untouched()
        # a missing key comes before the plaintext checks
        missing = osk_only if not symmetric else opk_only
        assert encrypt_batch([plains[0], big_pt], None, symmetric, enc=missing, dsts=keep)[0] == COR_E_INVALIDOPERATION
        assert slots_batch(np.zeros((2, 4), dtype=np.uint64), False, None, symmetric, enc=missing, dsts=keep)[0] == COR_E_INVALIDOPERATION
        untouched()
        # the per-handle calls agree
        h = OL.new("Ciphertext")
        if symmetric:
            assert S.rc("Encryptor_EncryptSymmetric", missing, plains[0], C.c_bool(False), h, None) == COR_E_INVALIDOPERATION
            assert S.rc("Encryptor_EncryptSymmetric", oenc, big_pt, C.c_bool(False), h, None) == E_INVALIDARG
        else:
            assert S.rc("Encryptor_Encrypt", missing, plains[0], h, None) == COR_E_INVALIDOPERATION
            assert S.rc("Encryptor_Encrypt", oenc, big_pt, h, None) == E_INVALIDARG
        assert slots_batch(np.zeros((2, n + 1), dtype=np.uint64), False, None, symmetric, dsts=keep)[0] == E_INVALIDARG
        untouched()
        assert encrypt_batch([], None, symmetric)[0] == 0
        assert slots_batch(np.zeros((0, 4), dtype=np.uint64), False, None, symmetric)[0] == 0
    assert encrypt_batch(plains, None, False, enc=vp())[0] == E_POINTER
    assert S.rc("B200_Encryptor_EncryptBatch", oenc, u64(1), None, None, C.c_bool(False), _arr(keep)) == E_POINTER
    assert S.rc("B200_Encryptor_EncryptBatch", oenc, u64(1), _arr(plains), None, C.c_bool(False), None) == E_POINTER
    vals = np.zeros((2, 4), dtype=np.uint64)
    assert slots_batch(vals, False, None, False, enc=vp())[0] == E_POINTER
    assert slots_batch(vals, False, None, False, be=vp())[0] == E_POINTER
    assert S.rc("B200_Encryptor_EncryptSlotsBatch", oenc, obe, u64(2), u64(4), None, C.c_bool(False), None, C.c_bool(False),
                _arr(keep)) == E_POINTER
    assert S.rc("B200_Encryptor_EncryptSlotsBatch", oenc, obe, u64(2), u64(4), vals.ctypes.data_as(C.c_void_p), C.c_bool(False),
                None, C.c_bool(False), None) == E_POINTER
    # an encoder of another context
    O2 = S.context(n, moduli, t)
    obe2 = vp()
    S.call("BatchEncoder_Create", O2.ctx, C.byref(obe2))
    assert slots_batch(vals, False, None, False, be=obe2, dsts=keep)[0] == E_INVALIDARG
    untouched()


def check_sk_golden(S):
    """seeded secret-key encryption reproduces tests/golden/encrypt_sk_n2048.npz, the words and noise the library gave when
    each call sampled and computed one item on its own (make_encrypt_sk_golden.py): the per-handle
    Encryptor_EncryptSymmetricReturnComponentsSetSeed and one EncryptBatch of all items"""
    import os
    from refseal import fnv1a64
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encrypt_sk_n2048.npz"))
    n, moduli, t = PARAMS["n2048_2x27"]
    R, O = RefContext(n, moduli, t), S.context(n, moduli, t)
    _, OL = sc._libs(R, O)
    osk, enc = OL.load("SecretKey", g["sk"].tobytes()), vp()
    S.call("Encryptor_Create", O.ctx, None, osk, C.byref(enc))
    plains = [O.new_pt(m) for m in g["msgs"]]
    for i, (p, sd) in enumerate(zip(plains, g["seeds"])):
        ct, e, rem = OL.new("Ciphertext"), vp(), OL.new("Plaintext")
        S.call("PolynomialArray_Create", None, C.byref(e))
        S.call("Encryptor_EncryptSymmetricReturnComponentsSetSeed", enc, p, ct, e, rem, (u64 * 8)(*[int(x) for x in sd]), None)
        assert fnv1a64(O.ct_words(ct)) == int(g["ct_fnv"][i]), f"per-handle item {i}"
        assert fnv1a64(sc._pa_export(OL, e)[1]) == int(g["e_fnv"][i]), f"noise of item {i}"
    dsts = [OL.new("Ciphertext") for _ in plains]
    seeds = np.ascontiguousarray(g["seeds"])
    S.call("B200_Encryptor_EncryptBatch", enc, u64(len(plains)), _arr(plains), seeds.ctypes.data_as(C.POINTER(u64)), C.c_bool(True),
           _arr(dsts))
    assert [fnv1a64(O.ct_words(h)) for h in dsts] == [int(x) for x in g["ct_fnv"]]


# ---- CPU emulation build ----

@pytest.mark.parametrize("name", EMU_SETS)
def test_layer1_words(emu_lib, ref, name):
    P = pair(EmuBackend(emu_lib), name)
    check_layer1(P, batch_sizes=(1, 3, 257) if name == "n4096" else (1, 3))


@pytest.mark.parametrize("name", ["n8192", "no_ks"])
def test_arguments_and_launch_counts(emu_lib, ref, name):
    P = pair(EmuBackend(emu_lib), name)
    check_arguments(P)
    check_launch_counts(P)


@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t"])
def test_sealc_seams(emu_lib, ref, name):
    sealc_seams(Sealc(emu_lib.lib), name)


def test_sk_golden(emu_lib, ref):
    check_sk_golden(Sealc(emu_lib.lib))


def test_resources_balance(emu_lib):
    """a context that encrypted batches (pk both ways, sk) gives back every allocation at destroy, and a second round of the
    same calls allocates nothing that stays behind"""
    import gc
    from sunscreen_b200.lib import B200Context
    fn = emu_lib.lib.b200_emu_live_resources
    fn.argtypes, fn.restype = [], C.c_longlong
    gc.collect()
    gc.disable()
    try:
        n, moduli, t = PARAMS["n4096"]
        before = fn()
        ctx = B200Context(n, moduli, t, lib=emu_lib)
        K, k1, B = len(moduli), ctx.k(), 3
        pk, sk = np.zeros((2, K, n), dtype=np.uint64), np.zeros((K, n), dtype=np.uint64)
        plain, out, seeds = np.zeros((B, n), dtype=np.uint64), np.zeros((B, 2, k1, n), dtype=np.uint64), np.zeros((B, 8), dtype=np.uint64)
        live = []
        for _ in range(2):
            ctx.encrypt_pk(pk, seeds, plain, out, B)
            ctx.encrypt_pk(pk, seeds, plain, out, B, disable_special_modulus=True)
            ctx.encrypt_sk(sk, seeds, plain, out, B)
            live.append(fn())
        assert live[0] == live[1], live
        del ctx
        gc.collect()
        assert fn() == before
    finally:
        gc.enable()


# ---- CUDA library ----

@pytest.fixture(scope="module")
def cuda_be():
    return CudaBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SETS)
def test_gpu_layer1_words(cuda_be, ref, name):
    check_layer1(pair(cuda_be, name), batch_sizes=(1, 3, 257))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "no_ks", "n16384_17x25"])
def test_gpu_arguments_and_launch_counts(cuda_be, ref, name):
    P = pair(cuda_be, name)
    check_arguments(P)
    check_launch_counts(P)


@pytest.mark.gpu
def test_gpu_sk_golden(cuda_be, ref):
    check_sk_golden(Sealc(cuda_be.lib.lib))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t"])
def test_gpu_sealc_seams(cuda_be, ref, name):
    sealc_seams(Sealc(cuda_be.lib.lib), name, big=257)
