"""Slots in and out: b200_batch_encode, b200_batch_decode and b200_decrypt_slots, and the layer-2 seams B200_BatchEncoder_EncodeBatch,
B200_BatchEncoder_DecodeBatch and B200_Decryptor_DecryptSlotsBatch, against the reference's BatchEncoder and Decryptor word for
word.  The same checks run on the CPU emulation build and, marked gpu, on the CUDA library."""
import ctypes as C
import math

import numpy as np
import pytest

import parity_checks as pc
import sealc_checks as sc
from backends import CudaBackend, EmuBackend
from params import PARAMS, PLAIN_EDGE
from refseal import E_INVALIDARG, E_POINTER, RefContext
from sealc_driver import Sealc
from sunscreen_b200.lib import PLAIN_NTT_MULTIPLY, PLAIN_NTT_TRANSFORM, B200Error
from test_plain_sum import data_levels, ref_transform_to_ntt, signed_plain

vp, u64 = C.c_void_p, C.c_uint64

EMU_SETS = ["n4096", "n8192", "n4096_q_below_t"] + [p for p in PLAIN_EDGE if PARAMS[p][0] <= 8192]
DECRYPT_SETS = ["n8192", "n8192_49", "n8192_54", "n8192_60"]


def batches(P):
    return P.t % (2 * P.n) == 1 and P.ctx.using_batching


# ---- the reference's BatchEncoder ----

def ref_encode(R, rbe, vals, signed):
    """BatchEncoder_Encode1 (Encode2 when signed) of the reference, padded to n coefficients"""
    p = vp()
    R.ref.call("Plaintext_Create1", None, C.byref(p))
    if signed:
        a = np.ascontiguousarray(vals, dtype=np.int64)
        R.ref.call("BatchEncoder_Encode2", rbe, u64(a.size), a.ctypes.data_as(C.POINTER(C.c_int64)), p)
    else:
        a = np.ascontiguousarray(vals, dtype=np.uint64)
        R.ref.call("BatchEncoder_Encode1", rbe, u64(a.size), a.ctypes.data_as(C.POINTER(u64)), p)
    c = R.pt_coeffs(p)
    R.free_pt(p)
    out = np.zeros(R.n, dtype=np.uint64)
    out[: c.size] = c
    return out


def ref_decode(R, rbe, pt, signed):
    """BatchEncoder_Decode1 (Decode2 when signed) of the reference plaintext handle `pt`, as uint64 words"""
    cnt = u64(R.n)
    if signed:
        out = np.zeros(R.n, dtype=np.int64)
        R.ref.call("BatchEncoder_Decode2", rbe, pt, C.byref(cnt), out.ctypes.data_as(C.POINTER(C.c_int64)), None)
        return out.view(np.uint64)
    out = np.zeros(R.n, dtype=np.uint64)
    R.ref.call("BatchEncoder_Decode1", rbe, pt, C.byref(cnt), out.ctypes.data_as(C.POINTER(u64)), None)
    return out


def value_rows(t, count, signed, items, rng):
    """[items][count] values: the classes batch_encoder_parity uses (uniform below t; signed, uniform in [-(t//2), t//2)),
    all zero, and with the edges 0, t - 1 (signed: 0, -(t-1)/2, (t-1)/2) at the first positions of every other item"""
    h = (t - 1) // 2
    rows = np.zeros((items, count), dtype=np.int64 if signed else np.uint64)
    edges = [0, -h, h] if signed else [0, t - 1]
    for i in range(items):
        if i % 3 == 1:
            continue  # all zero
        rows[i] = rng.integers(-(t // 2), t // 2, size=count) if signed else rng.integers(0, t, size=count, dtype=np.uint64)
        if i % 3 == 2:
            e = edges[: count]
            rows[i, : len(e)] = e
    return rows


# ---- layer 1 ----

def encode(P, vals, signed):
    items, count = vals.shape
    out = P.out(items, P.n)
    P.ctx.batch_encode(P.dev(vals.view(np.uint64)), count, out, items, signed=signed)
    return P.host(out).reshape(items, P.n)


def decode(P, plain, signed):
    items = plain.shape[0]
    d = P.dev(plain)
    out = P.out(items, P.n)
    P.ctx.batch_decode(d, out, items, signed=signed)
    assert np.array_equal(P.host(d).reshape(plain.shape), plain), "batch_decode modified its input"
    return P.host(out).reshape(items, P.n)


def check_encode_decode(P, seed=3, big=257):
    """encode and decode words against the reference for counts 0, 1, n/2, n - 1 and n, both signednesses, 1 and 3 items (and
    `big` items at count n); decode of encode gives the values back; random plaintexts below t decode as the reference's"""
    R, n, t = P.ref, P.n, P.t
    rbe = R.batch_encoder()
    rng = np.random.default_rng(seed)
    for signed in (False, True):
        for count in (0, 1, n // 2, n - 1, n):
            for items in (1, 3) + ((big,) if count == n else ()):
                vals = value_rows(t, count, signed, items, rng)
                got = encode(P, vals, signed)
                back = decode(P, got, signed)
                for i in range(items):
                    exp = ref_encode(R, rbe, vals[i], signed)
                    pc.eq(got[i], exp, f"encode signed={signed} count={count} items={items} item {i}")
                    want = np.zeros(n, dtype=vals.dtype)
                    want[:count] = vals[i]
                    pc.eq(back[i], want.view(np.uint64), f"decode(encode) signed={signed} count={count} item {i}")
        plains = rng.integers(0, t, size=(3, n), dtype=np.uint64)
        plains[1, 1:] = 0
        plains[2] = t - 1
        got = decode(P, plains, signed)
        for i in range(3):
            rp = R.new_pt(plains[i])
            pc.eq(got[i], ref_decode(R, rbe, rp, signed), f"decode of plaintext {i}, signed={signed}")
            R.free_pt(rp)
    with pytest.raises(B200Error) as e:
        encode(P, np.zeros((1, n + 1), dtype=np.uint64), False)
    assert e.value.code == -1


def check_refused_without_batching(P):
    """every slot entry point refuses parameters that do not batch (B200_E_INVALID), as the reference's BatchEncoder_Create does"""
    buf = P.out(4, P.ctx.k(), P.n)
    for call in (lambda: P.ctx.batch_encode(buf, 1, buf, 1), lambda: P.ctx.batch_decode(buf, buf, 1),
                 lambda: P.ctx.decrypt_slots(buf, 2, buf, buf, 1)):
        with pytest.raises(B200Error) as e:
            call()
        assert e.value.code == -1


def check_arguments(P):
    n = P.n
    buf = P.out(2, n)
    for call in (lambda: P.ctx.batch_encode(None, 1, buf, 1), lambda: P.ctx.batch_encode(buf, 1, None, 1),
                 lambda: P.ctx.batch_decode(None, buf, 1), lambda: P.ctx.batch_decode(buf, None, 1),
                 lambda: P.ctx.decrypt_slots(buf, 2, buf, None, 1), lambda: P.ctx.decrypt_slots(None, 2, buf, buf, 1)):
        with pytest.raises(B200Error) as e:
            call()
        assert e.value.code == -4
    with pytest.raises(B200Error) as e:
        P.ctx.decrypt_slots(buf, 1, buf, buf, 1)
    assert e.value.code == -1
    with pytest.raises(B200Error) as e:
        P.ctx.decrypt_slots(buf, 2, buf, buf, 1, level=P.ctx.levels)
    assert e.value.code == -1
    # zero items: no work, no error; count 0 takes no values
    P.ctx.batch_encode(None, 0, buf, 1)
    P.ctx.batch_encode(buf, n, buf, 0)
    P.ctx.batch_decode(buf, buf, 0)
    P.ctx.decrypt_slots(buf, 2, buf, buf, 0)


def check_multiply_ready(P, seed=5):
    """batch_encode -> plain_to_ntt(TRANSFORM) == the reference's Encode -> TransformToNTT1 at every data level;
    batch_encode -> plain_to_ntt(MULTIPLY) == plain_to_ntt(MULTIPLY) of the reference's Encode words"""
    R, n, t = P.ref, P.n, P.t
    rbe = R.batch_encoder()
    rng = np.random.default_rng(seed)
    vals = value_rows(t, n, False, 3, rng)
    coeffs = P.out(3, n)
    P.ctx.batch_encode(P.dev(vals), n, coeffs, 3)
    exp = np.stack([ref_encode(R, rbe, v, False) for v in vals])
    for lv, j, k in data_levels(P):
        out = P.out(3, k, n)
        P.ctx.plain_to_ntt(coeffs, 3, out, rule=PLAIN_NTT_TRANSFORM, level=lv)
        got = P.host(out).reshape(3, k, n)
        for i in range(3):
            pc.eq(got[i], ref_transform_to_ntt(P, exp[i], j), f"encode -> TRANSFORM level {lv} item {i}")
        out2, out3 = P.out(3, k, n), P.out(3, k, n)
        P.ctx.plain_to_ntt(coeffs, 3, out2, rule=PLAIN_NTT_MULTIPLY, level=lv)
        P.ctx.plain_to_ntt(P.dev(exp), 3, out3, rule=PLAIN_NTT_MULTIPLY, level=lv)
        pc.eq(P.host(out2), P.host(out3), f"encode -> MULTIPLY level {lv}")


def check_bsgs_plain_ntt(P, seed=6):
    """bsgs_plain_ntt (batch_encode -> plain_to_ntt(MULTIPLY) of the helper's slot vectors) == plain_to_ntt(MULTIPLY) of the
    reference's Encode of each vector"""
    from sunscreen_b200.bsgs import bsgs_plain_ntt, bsgs_plain_vectors
    R, n, t = P.ref, P.n, P.t
    rbe = R.batch_encoder()
    rng = np.random.default_rng(seed)
    d, b = 8, 3
    vecs, _, _ = bsgs_plain_vectors(rng.integers(0, t, size=(d, d)), n, t, b)
    G = vecs.shape[0]
    k = P.ctx.k()
    out, exp = P.out(G, b, k, n), P.out(G * b, k, n)
    bsgs_plain_ntt(P.ctx, P.dev(vecs), P.out(G * b, n), out)
    ref = np.stack([ref_encode(R, rbe, v, False) for v in vecs.reshape(G * b, n)])
    P.ctx.plain_to_ntt(P.dev(ref), G * b, exp, rule=PLAIN_NTT_MULTIPLY)
    pc.eq(P.host(out), P.host(exp), "bsgs_plain_ntt")


def check_launch_counts(P):
    """each of the three calls issues as many launches for 257 items as for one"""
    n, k = P.n, P.ctx.k()
    W = (math.prod(P.moduli[:k]).bit_length() + 63) // 64 + 1
    big = 257
    vals, plain, slots = P.out(big, n), P.out(big, n), P.out(big, n)
    ct, sk = P.out(big, 2, k, n), P.out(1, k, n)
    norm = np.zeros((big, W), dtype=np.uint64)
    calls = {
        "encode": lambda m: P.ctx.batch_encode(vals, n, plain, m),
        "decode": lambda m: P.ctx.batch_decode(plain, slots, m),
        "decrypt_slots": lambda m: P.ctx.decrypt_slots(ct, 2, sk, slots, m),
        "decrypt_slots with norms": lambda m: P.ctx.decrypt_slots(ct, 2, sk, slots, m, norm_out_host=norm, words=W),
    }
    for name, call in calls.items():
        deltas = []
        for m in (1, big, 1):
            before = P.ctx.launch_count()
            call(m)
            deltas.append(P.ctx.launch_count() - before)
        assert deltas[0] == deltas[1] == deltas[2] > 0, (name, deltas)


def check_decrypt_slots(P, seed=31, sizes=(2, 3)):
    """b200_decrypt_slots at every data level, sizes 2 and 3, with a real reference secret key, both signednesses, against
    b200_decrypt + b200_batch_decode and b200_noise_norm on the device and against the reference's Decrypt -> Decode and
    InvariantNoiseBudget.  The items: uniformly random ciphertexts (budget 0), a real encryption of slot values mod-switched
    down to the level, and (size 2) a ciphertext whose phase takes the crafted rounding-boundary values of check_decrypt."""
    R, n, t = P.ref, P.n, P.t
    rng = np.random.default_rng(seed)
    kg = R.keygen()
    sk = R.secret_key(kg)
    dec, enc, rbe = R.decryptor(sk), R.encryptor(R.public_key(kg)), R.batch_encoder()
    h = vp()
    R.ref.call("SecretKey_Data", sk, C.byref(h))
    s_ntt = R.pt_coeffs(h).reshape(-1, n)
    levels = data_levels(P)
    real = R.encrypt(enc, R.batch_encode(rbe, rng.integers(0, t, size=n, dtype=np.uint64)))
    reals = [real]
    for _ in levels[1:]:
        reals.append(R.mod_switch_to_next(reals[-1]))
    for lv, j, k in levels:
        q = [int(m) for m in P.moduli[:k]]
        Q = math.prod(q)
        W = (Q.bit_length() + 63) // 64 + 1
        dsk = P.dev(pc.key_powers(P, s_ntt, k, max(sizes) - 1))
        for size in sizes:
            B = 4
            ct = pc.rand_ct(rng, P.moduli, k, n, size=size, batch=B)
            ct[1] = 0
            ct[1, :2] = R.ct_words(reals[j])
            if size == 2:
                ct[2, 1] = 0
                ct[2, 0] = pc._residues(pc.crafted_phases(Q, t, rng), q, n, rng)[0]
            dct = P.dev(ct)
            for signed in (False, True):
                slots, norm = P.out(B, n), np.zeros((B, W), dtype=np.uint64)
                P.ctx.decrypt_slots(dct, size, dsk, slots, B, signed=signed, norm_out_host=norm, words=W, level=lv)
                got = P.host(slots).reshape(B, n)
                pt, chain = P.out(B, n), P.out(B, n)
                P.ctx.decrypt(dct, size, dsk, pt, B, level=lv)
                P.ctx.batch_decode(pt, chain, B, signed=signed)
                what = f"level {lv} size {size} signed={signed}"
                pc.eq(got, P.host(chain), f"decrypt_slots vs decrypt + batch_decode, {what}")
                norm2 = np.zeros((B, W), dtype=np.uint64)
                P.ctx.noise_norm(dct, size, dsk, norm2, W, B, level=lv)
                pc.eq(norm, norm2, f"decrypt_slots norms vs noise_norm, {what}")
                nonorm = P.out(B, n)
                P.ctx.decrypt_slots(dct, size, dsk, nonorm, B, signed=signed, level=lv)
                pc.eq(P.host(nonorm), got, f"decrypt_slots without norms, {what}")
                budgets = []
                for b in range(B):
                    rc = R.new_ct(ct[b], level=j)
                    rp = R.decrypt(dec, rc)
                    pc.eq(got[b], ref_decode(R, rbe, rp, signed), f"decrypt_slots vs the reference, {what}, item {b}")
                    nb = int.bit_length(sum(int(w) << (64 * i) for i, w in enumerate(norm[b])))
                    budgets.append(max(0, Q.bit_length() - nb - 1))
                    assert budgets[-1] == R.noise_budget(dec, rc), (what, b)
                    R.free_pt(rp)
                    R.free_ct(rc)
                assert budgets[0] == 0 and (j > 0 or budgets[1] > 0), budgets


def check_norm_edges(P, seed=37):
    """the norm edges of check_noise_norm_edges through b200_decrypt_slots: centring boundary, Q - 1 and word carries at
    coefficients 0, 127, 128 and n - 1, one all-zero item; norms == b200_noise_norm == Python integers, slots == the reference"""
    R, n, t, k = P.ref, P.n, P.t, P.k
    rng = np.random.default_rng(seed)
    rbe = R.batch_encoder()
    dec = R.decryptor(R.secret_key(R.keygen()))  # c1 = 0: the phase is c0 whatever the key
    q = [int(m) for m in P.moduli[:k]]
    Q = math.prod(q)
    W = (Q.bit_length() + 63) // 64 + 1
    tinv = pow(t, -1, Q)
    edges = [y for y in ((Q - 1) // 2, (Q + 1) // 2, Q - 1, 2**64 - 1, 2**64) if 0 < y < Q]
    centred = lambda y: Q - y if y >= (Q + 1) // 2 else y
    dsk = P.dev(np.zeros((1, k, n), dtype=np.uint64))
    for p, pos in enumerate((0, 127, 128, n - 1)):
        ct = np.zeros((5, 2, k, n), dtype=np.uint64)
        want = [0]
        for b in range(1, 5):
            Y = [int(v) for v in rng.integers(0, 2**20, size=n)]
            Y[pos] = edges[(p + b) % len(edges)]
            want.append(max(centred(y) for y in Y))
            ct[b, 0], _ = pc._residues([y * tinv % Q for y in Y], q, n, rng)
        dct = P.dev(ct)
        slots, norm, norm2 = P.out(5, n), np.zeros((5, W), dtype=np.uint64), np.zeros((5, W), dtype=np.uint64)
        P.ctx.decrypt_slots(dct, 2, dsk, slots, 5, norm_out_host=norm, words=W)
        P.ctx.noise_norm(dct, 2, dsk, norm2, W, 5)
        pc.eq(norm, norm2, f"norm edges at {pos}")
        got = P.host(slots).reshape(5, n)
        for b in range(5):
            assert sum(int(w) << (64 * i) for i, w in enumerate(norm[b])) == want[b], (pos, b)
            rc = R.new_ct(ct[b])
            rp = R.decrypt(dec, rc)
            pc.eq(got[b], ref_decode(R, rbe, rp, False), f"norm edges at {pos}, item {b} slots")
            R.free_pt(rp)
            R.free_ct(rc)
    with pytest.raises(B200Error) as e:
        P.ctx.decrypt_slots(dct, 2, dsk, slots, 5, norm_out_host=np.zeros((5, W - 1), dtype=np.uint64), words=W - 1)
    assert e.value.code == -1


# ---- layer 2 ----

def _arr(hs):
    return (vp * max(len(hs), 1))(*hs) if hs is not None else None


def sealc_seams(S, name, seed=11):
    """the three seams against the per-handle calls and the reference: words and budgets for real encryptions (Encryptor_Encrypt
    of batch-encoded values and of Sunscreen's Signed encodings) at two levels, and every HRESULT"""
    n, moduli, t = PARAMS[name]
    R = RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    RL, OL = sc._libs(R, O)
    rng = np.random.default_rng(seed)
    kg = R.keygen()
    rsk, rpk = R.secret_key(kg), R.public_key(kg)
    rdec, rbe = R.decryptor(rsk), R.batch_encoder()
    osk, opk = OL.load("SecretKey", RL.save("SecretKey", rsk, 0)), OL.load("PublicKey", RL.save("PublicKey", rpk, 0))
    obe, oenc, odec = vp(), vp(), vp()
    S.call("BatchEncoder_Create", O.ctx, C.byref(obe))
    S.call("Encryptor_Create", O.ctx, opk, None, C.byref(oenc))
    S.call("Decryptor_Create", O.ctx, osk, C.byref(odec))

    def encode_batch(vals, signed, count=None, be=None, dsts=None):
        vals = np.ascontiguousarray(vals)
        cnt = vals.shape[0] if count is None else count
        dsts = [OL.new("Plaintext") for _ in range(vals.shape[0])] if dsts is None else dsts
        rc = S.rc("B200_BatchEncoder_EncodeBatch", obe if be is None else be, u64(cnt), u64(vals.shape[1]),
                  vals.ctypes.data_as(C.POINTER(u64)), C.c_bool(signed), _arr(dsts))
        return rc, dsts

    def per_handle_encode(v, signed):
        p = OL.new("Plaintext")
        a = np.ascontiguousarray(v)
        S.call("BatchEncoder_Encode2" if signed else "BatchEncoder_Encode1", obe, u64(a.size), a.ctypes.data_as(C.c_void_p), p)
        return p

    def per_handle_decode(p, signed):
        out = np.zeros(n, dtype=np.uint64)
        cnt = u64()
        S.call("BatchEncoder_Decode2" if signed else "BatchEncoder_Decode1", obe, p, C.byref(cnt), out.ctypes.data_as(C.c_void_p), None)
        assert cnt.value == n
        return out

    def decode_batch(plains, signed, be=None, out=None):
        out = np.zeros((max(len(plains), 1), n), dtype=np.uint64) if out is None else out
        rc = S.rc("B200_BatchEncoder_DecodeBatch", obe if be is None else be, u64(len(plains)), _arr(plains), C.c_bool(signed),
                  out.ctypes.data_as(C.c_void_p))
        return rc, out

    def decrypt_batch(cts, signed, budgets=True, dec=None, be=None):
        out = np.zeros((max(len(cts), 1), n), dtype=np.uint64)
        bud = (C.c_int * max(len(cts), 1))() if budgets else None
        rc = S.rc("B200_Decryptor_DecryptSlotsBatch", odec if dec is None else dec, obe if be is None else be, u64(len(cts)),
                  _arr(cts), C.c_bool(signed), out.ctypes.data_as(C.c_void_p), bud)
        return rc, out, (list(bud)[: len(cts)] if budgets else None)

    # encode / decode against the per-handle calls and the reference
    for signed in (False, True):
        for per in (n, 7, 0):
            vals = value_rows(t, per, signed, 3, rng)
            rc, dsts = encode_batch(vals.view(np.uint64), signed)
            assert rc == 0
            for i in range(3):
                exp = ref_encode(R, rbe, vals[i], signed)
                pc.eq(O.pt_coeffs(dsts[i]), exp, f"{name}: EncodeBatch signed={signed} per={per} item {i}")
                pc.eq(O.pt_coeffs(per_handle_encode(vals[i], signed)), exp, f"{name}: Encode{2 if signed else 1} per={per}")
            rc, got = decode_batch(dsts, signed)
            assert rc == 0
            for i in range(3):
                want = np.zeros(n, dtype=vals.dtype)
                want[:per] = vals[i]
                pc.eq(got[i], want.view(np.uint64), f"{name}: DecodeBatch signed={signed} per={per} item {i}")
                pc.eq(got[i], per_handle_decode(dsts[i], signed), f"{name}: DecodeBatch vs Decode, item {i}")
    # real encryptions: batch-encoded values and Signed encodings, at the first level and one below
    plains = [per_handle_encode(rng.integers(0, t, size=n, dtype=np.uint64), False),
              per_handle_encode(rng.integers(-(t // 2), t // 2, size=n), True)]
    plains += [O.new_pt(signed_plain(v, t)) for v in (5, -123, 0)]
    cts = []
    for p in plains:
        h = OL.new("Ciphertext")
        S.call("Encryptor_Encrypt", oenc, p, h, None)
        cts.append(h)
    levels = [cts]
    if len(R.data_parms_ids()) > 1:
        low = []
        for h in cts:
            d = O._dst()
            S.call("Evaluator_ModSwitchToNext1", O.ev, h, d, None)
            low.append(d)
        levels.append(low)
    for hs in levels:
        for signed in (False, True):
            rc, got, bud = decrypt_batch(hs, signed)
            assert rc == 0
            rc, got_nb, none = decrypt_batch(hs, signed, budgets=False)
            assert rc == 0 and none is None
            pc.eq(got_nb, got, f"{name}: DecryptSlotsBatch without budgets")
            for i, h in enumerate(hs):
                pt = OL.new("Plaintext")
                S.call("Decryptor_Decrypt", odec, h, pt)
                pc.eq(got[i], per_handle_decode(pt, signed), f"{name}: DecryptSlotsBatch vs Decrypt + Decode, item {i}")
                b = C.c_int()
                S.call("Decryptor_InvariantNoiseBudget", odec, h, C.byref(b))
                assert bud[i] == b.value > 0, (i, bud[i], b.value)
                rh = RL.load("Ciphertext", OL.save("Ciphertext", h, 0))
                rp = R.decrypt(rdec, rh)
                pc.eq(got[i], ref_decode(R, rbe, rp, signed), f"{name}: DecryptSlotsBatch vs the reference, item {i}")
                assert bud[i] == R.noise_budget(rdec, rh)
    # HRESULTs
    ntt_pt = vp()  # an encoded plaintext marked as NTT form at the first level
    S.call("Plaintext_Create5", plains[0], C.byref(ntt_pt))
    S.call("Plaintext_SetParmsId", ntt_pt, O.first_id)
    assert decode_batch([plains[0], ntt_pt], False)[0] == E_INVALIDARG
    out = np.zeros(n, dtype=np.uint64)
    assert S.rc("BatchEncoder_Decode1", obe, ntt_pt, C.byref(u64()), out.ctypes.data_as(C.c_void_p), None) == E_INVALIDARG
    big = O.new_pt(np.full(3, t, dtype=np.uint64))  # a coefficient not below t
    assert decode_batch([plains[0], big], False)[0] == E_INVALIDARG
    assert decode_batch([plains[0], None], False)[0] == E_INVALIDARG
    assert decode_batch(plains, False, be=vp())[0] == E_POINTER
    assert S.rc("B200_BatchEncoder_DecodeBatch", obe, u64(1), None, C.c_bool(False), out.ctypes.data_as(C.c_void_p)) == E_POINTER
    assert decode_batch([], False)[0] == 0
    tall = np.zeros((2, n + 1), dtype=np.uint64)
    assert encode_batch(tall, False)[0] == E_INVALIDARG
    a = np.zeros(n + 1, dtype=np.uint64)
    assert S.rc("BatchEncoder_Encode1", obe, u64(n + 1), a.ctypes.data_as(C.c_void_p), OL.new("Plaintext")) == E_INVALIDARG
    assert encode_batch(np.zeros((2, 4), dtype=np.uint64), False, be=vp())[0] == E_POINTER
    assert encode_batch(np.zeros((2, 4), dtype=np.uint64), False, dsts=[OL.new("Plaintext"), None])[0] == E_INVALIDARG
    assert encode_batch(np.zeros((0, 4), dtype=np.uint64), False)[0] == 0
    assert decrypt_batch(cts, False, dec=vp())[0] == E_POINTER
    assert decrypt_batch(cts, False, be=vp())[0] == E_POINTER
    assert decrypt_batch([cts[0], None], False)[0] == E_INVALIDARG
    assert decrypt_batch([], False)[0] == 0
    if len(levels) > 1:
        assert decrypt_batch([cts[0], levels[1][1]], False)[0] == E_INVALIDARG
    k = O.k
    c3 = O.new_ct(pc.rand_ct(rng, moduli, k, n, size=3))
    assert decrypt_batch([cts[0], c3], False)[0] == E_INVALIDARG
    nct = O.new_ct(pc.rand_ct(rng, moduli, k, n), ntt=True)
    assert decrypt_batch([cts[0], nct], False)[0] == E_INVALIDARG
    assert S.rc("Decryptor_Decrypt", odec, nct, OL.new("Plaintext")) == E_INVALIDARG
    # a decryptor and an encoder of different contexts
    O2 = S.context(n, moduli, t)
    obe2 = vp()
    S.call("BatchEncoder_Create", O2.ctx, C.byref(obe2))
    assert decrypt_batch(cts, False, be=obe2)[0] == E_INVALIDARG
    # the size-3 batch alone decrypts as the per-handle calls do
    rc, got, bud = decrypt_batch([c3, c3], True)
    assert rc == 0
    pt = OL.new("Plaintext")
    S.call("Decryptor_Decrypt", odec, c3, pt)
    pc.eq(got[1], per_handle_decode(pt, True), f"{name}: size-3 DecryptSlotsBatch")
    assert bud == [0, 0]


# ---- CPU emulation build ----

@pytest.fixture(scope="module", params=EMU_SETS)
def emu_pair(request, emu_lib, ref):
    return pc.pair_for(EmuBackend(emu_lib), request.param)


def test_encode_decode_words(emu_pair):
    if not batches(emu_pair):
        check_refused_without_batching(emu_pair)
        return
    check_encode_decode(emu_pair)


def test_multiply_ready_operands(emu_pair):
    if batches(emu_pair):
        check_multiply_ready(emu_pair)


@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t"])
def test_arguments_and_launch_counts(emu_lib, ref, name):
    P = pc.pair_for(EmuBackend(emu_lib), name)
    check_arguments(P)
    check_launch_counts(P)
    check_bsgs_plain_ntt(P)


@pytest.mark.parametrize("name", DECRYPT_SETS)
def test_decrypt_slots(emu_lib, ref, name):
    check_decrypt_slots(pc.pair_for(EmuBackend(emu_lib), name))


def test_decrypt_slots_norm_edges(emu_lib, ref):
    check_norm_edges(pc.pair_for(EmuBackend(emu_lib), "n8192"))


@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t"])
def test_sealc_seams(emu_lib, ref, name):
    sealc_seams(Sealc(emu_lib.lib), name)


# ---- CUDA library ----

@pytest.fixture(scope="module")
def cuda_be():
    return CudaBackend()


@pytest.mark.gpu
@pytest.mark.parametrize("name", EMU_SETS + ["n32768"])
def test_gpu_encode_decode_words(cuda_be, ref, name):
    P = pc.pair_for(cuda_be, name)
    if not batches(P):
        check_refused_without_batching(P)
        return
    check_encode_decode(P)
    check_multiply_ready(P)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t", "n32768"])
def test_gpu_arguments_and_launch_counts(cuda_be, ref, name):
    P = pc.pair_for(cuda_be, name)
    check_arguments(P)
    check_launch_counts(P)
    check_bsgs_plain_ntt(P)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DECRYPT_SETS)
def test_gpu_decrypt_slots(cuda_be, ref, name):
    check_decrypt_slots(pc.pair_for(cuda_be, name))


@pytest.mark.gpu
def test_gpu_decrypt_slots_norm_edges(cuda_be, ref):
    check_norm_edges(pc.pair_for(cuda_be, "n8192"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n8192", "n4096_q_below_t"])
def test_gpu_sealc_seams(cuda_be, ref, name):
    sealc_seams(Sealc(cuda_be.lib.lib), name)
