"""Wide chains (tests/params.py WIDE) and the key level of the longest chains, against the unmodified reference.

- The key level of the 17-prime chains (n16384_17x25, n16384_49_16x24, n32768_49x17): public-key encryption works there and
  then drops the special prime with b200_mod_switch_to_next at 17 residues, the one k-templated kernel that takes 17.
  Encryption, key generation, decryption and the whole modulus-switching chain through layer 2, and the 17-residue mod
  switch at layer 1 against the big-integer rounding.
- n = 32768 beyond the default chain: 60-bit primes in the split transform (ntt_outer_kernel), 60-bit digits reduced mod
  30-bit primes, and the integer BEHZ kernels against a 47-bit auxiliary base with fewer primes than k (the split transform
  switches the FP64 path off).  The parity battery of test_gpu_parity.py on each, and on the default chain and the 60-bit
  chain with B200_NTT_SPLIT=1 (the one-stage split); the multiply's words with the narrow base equal those with the
  reference's 61-bit base; the launch traces show which kernels ran.
- 17 data residues (n16384_24x18), one beyond the library's limit: both libraries create the context, and every operation
  either gives the reference's words or refuses with E_INVALIDARG, never different words.

Tests without the gpu mark run the same checks on the CPU emulation build (tests/emu), one level or chain each."""
import ctypes as C
import math

import numpy as np
import pytest

import parity_checks as pc
import refseal
import sealc_checks as sc
from params import PARAMS
from refseal import E_INVALIDARG
from sealc_driver import Sealc, SealcError
from test_gpu_ks_cluster import keyswitch_vs_reference
from test_gpu_long_chains import count, traced_levels
from test_gpu_scale_moddown import mul_relin_three_ways

KEY17 = ["n16384_17x25", "n16384_49_16x24", "n32768_49x17"]     # 16 data residues, 17 primes at the key level
N32768 = ["n32768", "n32768_60x6", "n32768_30x5", "n32768_mixed", "n32768_49x17"]
B200_E_INVALID = -1
vp, u64 = C.c_void_p, C.c_uint64


@pytest.fixture(scope="module")
def cuda():
    from backends import CudaBackend
    return CudaBackend()


@pytest.fixture(scope="module")
def pairs(cuda, ref):
    cache = {}

    def get(name):
        if name not in cache:
            cache.clear()       # one n = 32768 context at a time
            cache[name] = pc.pair_for(cuda, name)
        return cache[name]
    return get


@pytest.fixture(scope="module")
def S_gpu():
    from sunscreen_b200.lib import B200Lib
    return Sealc(B200Lib.default().lib)


@pytest.fixture(scope="module")
def S_emu(emu_lib):
    return Sealc(emu_lib.lib)


def emu_pair(emu_lib, name):
    from backends import EmuBackend
    return pc.pair_for(EmuBackend(emu_lib), name)


# ---------------------------------------------------------------------------------------------------------------------
# what each chain reaches, on the library's own constants
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["n32768_60x6", "n32768_30x5", "n32768_mixed", "n32768_49x17", "n16384_24x18"] + KEY17[:2])
def test_library_reaches_the_cases(emu_lib, ref, name):
    """check_context against the reference, then what the set is there for: 17 primes at the key level; the auxiliary base
    of each n = 32768 set (61-bit when a prime is above 49 bits, else as wide as the widest prime, at least 47 bits), and
    nB < k on n32768_30x5; 17 data residues on n16384_24x18"""
    P = emu_pair(emu_lib, name)
    pc.check_context(P)
    key, top = P.ctx.level_info(0), P.ctx.level_info(P.ctx.first_level)
    assert key["k"] == len(P.moduli)
    widest = max(int(q).bit_length() for q in P.moduli)
    assert {p.bit_length() for p in top["bsk"]} == {61 if widest > 49 else max(47, widest)}, top["bsk"]
    if name in KEY17:
        assert key["k"] == 17 and top["k"] == 16
    if name == "n32768_30x5":
        assert top["nB"] < top["k"] == 4, (top["nB"], top["k"])
    if name == "n16384_24x18":
        assert top["k"] == 17


# ---------------------------------------------------------------------------------------------------------------------
# layer 1: the mod switch at 17 residues
# ---------------------------------------------------------------------------------------------------------------------
def modswitch_rounding(ct, q):
    """floor((X + q_last / 2) / q_last) mod q_i for the CRT value X of every coefficient of ct [..., K, n] (the reference's
    divide_and_round_q_last), with Python integers"""
    Q, half = math.prod(q), q[-1] >> 1
    X = sum(ct[..., i, :].astype(object) * ((Q // qi) * pow(Q // qi, -1, qi) % Q) for i, qi in enumerate(q)) % Q
    Y = (X + half) // q[-1]
    return np.stack([(Y % qi).astype(np.uint64) for qi in q[:-1]], axis=-2)


def check_modswitch_17(P, lv, batch=3, seed=61):
    """b200_mod_switch_to_next at level lv (17 residues) of ciphertexts of size 2 and 3, batch 3, with all-(q - 1), 0 and
    (q - 1) / 2 words in the first item, against the big-integer rounding"""
    rng = np.random.default_rng(seed)
    k = P.ctx.level_info(lv)["k"]
    assert k == 17
    q = [int(m) for m in P.moduli[:k]]
    for size in (2, 3):
        ct = pc.rand_ct(rng, P.moduli, k, P.n, size=size, batch=batch)
        for i, qi in enumerate(q):
            ct[0, 0, i, :8] = qi - 1
            ct[0, 0, i, 8:16] = 0
            ct[0, 0, i, 16:24] = (qi - 1) // 2
        o = P.out(batch, size, k - 1, P.n)
        P.ctx.mod_switch_to_next(P.dev(ct), size, o, batch, level=lv)
        pc.eq(P.host(o), modswitch_rounding(ct, q), f"mod_switch_to_next of 17 residues, level {lv}, size {size}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", KEY17)
def test_key_level_modswitch(pairs, name):
    check_modswitch_17(pairs(name), 0)


def test_key_level_modswitch_emulation(emu_lib, ref):
    check_modswitch_17(emu_pair(emu_lib, "n16384_17x25"), 0, batch=2)


# ---------------------------------------------------------------------------------------------------------------------
# layer 2: encryption, key generation and decryption on the 17-prime chains
# ---------------------------------------------------------------------------------------------------------------------
def key_level_layer2(S, name):
    args = PARAMS[name]
    sc.seeded_encryption_parity(S, *args)
    sc.encryption_components_parity(S, *args)
    sc.keygen_interop(S, *args)
    sc.simple_multiply_sequence(S, *args)      # decryption and noise budget at the first data level


@pytest.mark.gpu
@pytest.mark.parametrize("name", KEY17)
def test_key_level_encryption(S_gpu, ref, name):
    key_level_layer2(S_gpu, name)


@pytest.mark.gpu
def test_key_level_deep_chain(S_gpu, ref):
    """pk-encrypted ciphertexts through every data level of n16384_17x25, down to one residue"""
    sc.deep_chain_parity(S_gpu, *PARAMS["n16384_17x25"])


@pytest.mark.parametrize("name", KEY17[:2])
def test_key_level_encryption_emulation(S_emu, ref, name):
    key_level_layer2(S_emu, name)


# ---------------------------------------------------------------------------------------------------------------------
# n = 32768: the parity battery
# ---------------------------------------------------------------------------------------------------------------------
def check_modswitch_levels(P, levels, batch=2, seed=71):
    """b200_mod_switch_to_next at data levels `levels`: the reference's words where it switches, else the big-integer
    rounding"""
    rng = np.random.default_rng(seed)
    R = P.ref
    ref_levels = len(R.data_parms_ids())
    for j in levels:
        lv = P.ctx.first_level + j
        k = P.ctx.level_info(lv)["k"]
        if k < 2:
            continue
        ct = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
        o = P.out(batch, 2, k - 1, P.n)
        P.ctx.mod_switch_to_next(P.dev(ct), 2, o, batch, level=lv)
        got = P.host(o).reshape(batch, 2, k - 1, P.n)
        if j + 1 < ref_levels:
            for b in range(batch):
                rc = R.new_ct(ct[b], level=j)
                rn = R.mod_switch_to_next(rc)
                pc.eq(got[b], R.ct_words(rn), f"mod_switch_to_next, level {lv}, item {b}")
                R.free_ct(rc)
                R.free_ct(rn)
        else:
            pc.eq(got, modswitch_rounding(ct, [int(q) for q in P.moduli[:k]]), f"mod_switch_to_next, level {lv}")


def battery(P, every_level=True):
    """test_gpu_parity.py's checks at n = 32768: context constants, the NTT (random, delta, all-(q - 1), alternating, +-1),
    multiply with sizes, relinearize, the Galois elements, plain operands, the mod switch, decryption, the noise norm and the
    adversarial operands; every data level where the check walks them, else the top level and the next one"""
    pc.check_context(P)
    pc.check_ntt(P, items=6)
    m3, rm = pc.check_multiply(P, with_sizes=True)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_plain(P)
    levels = range(len(P.ref.data_parms_ids())) if every_level else (0, 1)
    pc.check_plain_operands(P, levels=levels)
    check_modswitch_levels(P, range(P.ctx.levels - P.ctx.first_level) if every_level else (0, 1))
    pc.check_decrypt(P, batch=2, levels=levels)
    pc.check_noise_norm(P, batch=2)
    pc.check_adversarial_multiply(P, with_size5=False, pairs=[("qm1", "qm1"), ("alt", "pm1"), ("single", "qm1")])
    pc.check_adversarial_keyswitch(P)
    for j in (1,) if not every_level else ():
        mul_relin_three_ways(P, j, 2, seed=90 + j)
        keyswitch_vs_reference(P, 2, seed=95 + j, j=j)


@pytest.mark.gpu
@pytest.mark.parametrize("name", N32768[1:])
def test_n32768_battery(pairs, name):
    P = pairs(name)
    assert P.ctx.level_info(P.ctx.first_level)["k"] == len(P.moduli) - 1
    battery(P, every_level=name != "n32768_49x17")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n32768", "n32768_60x6"])
def test_n32768_one_stage_split(cuda, ref, monkeypatch, name):
    """B200_NTT_SPLIT=1 (read when the context is created): one global stage and half-size sub-transforms"""
    monkeypatch.setenv("B200_NTT_SPLIT", "1")
    battery(pc.pair_for(cuda, name), every_level=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["n32768_30x5", "n32768_49x17"])
def test_n32768_aux_base_independence(cuda, ref, monkeypatch, name):
    """multiply / multiply_relin against the 47- or 49-bit auxiliary base equal the same under B200_FORCE_AUX61 (the
    reference's 61-bit base) and the reference's words, random and all-(q - 1) operands"""
    from sunscreen_b200.lib import B200Context
    P = pc.pair_for(cuda, name)
    n, moduli, t = PARAMS[name]
    monkeypatch.setenv("B200_FORCE_AUX61", "1")
    wide = B200Context(n, moduli, t, lib=cuda.lib)
    monkeypatch.delenv("B200_FORCE_AUX61")
    narrow_bsk = P.ctx.level_info(P.ctx.first_level)["bsk"]
    wide_bsk = wide.level_info(wide.first_level)["bsk"]
    assert max(p.bit_length() for p in narrow_bsk) <= 49 and {p.bit_length() for p in wide_bsk} == {61}
    rng = np.random.default_rng(5)
    batch = 2
    A = pc.rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    B = pc.rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    A[1] = pc.adversarial_ct(P, "qm1")
    B[1] = pc.adversarial_ct(P, "qm1")
    key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    dA, dB, dK = P.dev(A), P.dev(B), P.dev(key)
    got = {}
    for label, ctx in (("narrow", P.ctx), ("61-bit", wide)):
        o3, o2 = P.out(batch, 3, P.k, P.n), P.out(batch, 2, P.k, P.n)
        ctx.multiply(dA, 2, dB, 2, o3, batch)
        ctx.multiply_relin(dA, dB, dK, o2, batch)
        got[label] = (P.host(o3).reshape(batch, 3, P.k, P.n), P.host(o2).reshape(batch, 2, P.k, P.n))
    pc.eq(got["narrow"][0], got["61-bit"][0], "multiply, narrow vs 61-bit auxiliary base")
    pc.eq(got["narrow"][1], got["61-bit"][1], "multiply_relin, narrow vs 61-bit auxiliary base")
    R = P.ref
    rlk = R.new_ksk({0: key})
    for b in range(batch):
        ra, rb = R.new_ct(A[b]), R.new_ct(B[b])
        rm = R.multiply(ra, rb)
        pc.eq(got["narrow"][0][b], R.ct_words(rm), f"multiply item {b}")
        pc.eq(got["narrow"][1][b], R.ct_words(R.relinearize(rm, rlk)), f"multiply_relin item {b}")


@pytest.mark.gpu
def test_n32768_narrow_base_trace(ref):
    """on n32768_30x5 the multiply runs the integer lift_kernel / scale_kernel (not the FP64 _v2 ones) and the integer
    key-switch MAC, and every transform the split one (ntt_outer_kernel)"""
    recs = traced_levels("n32768_30x5", every=False)
    assert [(op, k) for op, _, k, _, _ in recs] == [("relinearize", 4), ("multiply_relin", 4)], recs
    for op, j, k, fused, launches in recs:
        assert count(launches, "ntt_outer_kernel") >= 2, (op, launches)
        assert count(launches, "ntt_fp") == 0, (op, launches)
        if op == "multiply_relin":
            assert count(launches, "lift_kernel<") == 1 and count(launches, "lift_kernel_v2") == 0, launches
            assert count(launches, "scale_kernel<") == 1 and count(launches, "scale_kernel_v2") == 0, launches
            assert count(launches, "scale_moddown_kernel_v2") == 0, launches


# ---------------------------------------------------------------------------------------------------------------------
# 17 data residues: the reference's words or E_INVALIDARG
# ---------------------------------------------------------------------------------------------------------------------
# what the library refuses on n16384_24x18, with B200_E_INVALID / E_INVALIDARG: everything that runs a kernel templated on
# the residue count other than the mod switch (the BEHZ multiply, the key switch, decryption) and, at the key level (18
# primes), the mod switch that public-key encryption ends with.  Every other operation gives the reference's words.
REFUSED_LAYER1 = {"multiply", "square", "relinearize", "multiply_relin", "apply_galois", "ct_sk_phase", "decrypt",
                  "mod_switch_to_next at the key level"}
REFUSED_LAYER2 = {"Evaluator_Multiply", "Evaluator_Square", "Evaluator_Relinearize", "Evaluator_RotateRows",
                  "Decryptor_Decrypt (fresh)", "Decryptor_Decrypt (product)", "Encryptor_Encrypt",
                  "Encryptor_EncryptReturnComponentsSetSeed"}


def beyond_limit_layer1(P):
    """every layer-1 operation at the first data level (k = 17) and the mod switch at the key level (18 primes): the
    reference's words (or, for the mod switch at the key level, the big-integer rounding) or B200_E_INVALID; returns the
    set of refused operations"""
    R, k, n = P.ref, P.k, P.n
    assert k == 17
    rng = np.random.default_rng(3)
    a, b = P.inp["a"], P.inp["b"]
    ra, rb = R.new_ct(a), R.new_ct(b)
    rm = R.multiply(ra, rb)
    m3 = R.ct_words(rm)
    rlk = R.new_ksk({0: P.inp["rlk"]})
    glk = R.new_ksk({1: P.inp["glk3"]})
    p = P.inp["p"]
    rp = R.new_pt(p)
    refused = set()

    def run(name, fn, shape, expect):
        """fn(o) writes the operation's words into o of `shape` (or, with shape None, into a buffer it returns)"""
        o = P.out(*shape) if shape else None
        try:
            o = fn(o) if o is None else (fn(o), o)[1]
        except Exception as e:      # B200Error
            assert getattr(e, "code", None) == B200_E_INVALID, (name, e)
            refused.add(name)
            return
        pc.eq(P.host(o), expect() if callable(expect) else expect, name)

    def ntt(_):
        d = P.dev(a[0])
        P.ctx.ntt_forward(d, 1)
        return d

    W = R.ct_words
    da, db = P.dev(a), P.dev(b)
    run("ntt_forward", ntt, None, lambda: np.stack([R.ref.ntt_forward(P.moduli[i], a[0, i]) for i in range(k)]))
    run("add", lambda o: P.ctx.add(da, db, o, 2, 1), (2, k, n), W(R.add(ra, rb)))
    run("sub", lambda o: P.ctx.sub(da, db, o, 2, 1), (2, k, n), W(R.sub(ra, rb)))
    run("negate", lambda o: P.ctx.negate(da, o, 2, 1), (2, k, n), W(R.negate(ra)))
    run("multiply", lambda o: P.ctx.multiply(da, 2, db, 2, o, 1), (3, k, n), m3)
    run("square", lambda o: P.ctx.square(da, o, 1), (3, k, n), lambda: W(R.square(ra)))
    exp_relin = W(R.relinearize(rm, rlk))
    run("relinearize", lambda o: P.ctx.relinearize(P.dev(m3), P.dev(P.inp["rlk"]), o, 1), (2, k, n), exp_relin)
    run("multiply_relin", lambda o: P.ctx.multiply_relin(da, db, P.dev(P.inp["rlk"]), o, 1), (2, k, n), exp_relin)
    run("apply_galois", lambda o: P.ctx.apply_galois(da, 3, P.dev(P.inp["glk3"]), o, 1), (2, k, n),
        lambda: W(R.rotate_rows(ra, 1, glk)))
    dp = P.dev(p)
    run("multiply_plain", lambda o: P.ctx.multiply_plain(da, 2, dp, 1, o, 1), (2, k, n), lambda: W(R.multiply_plain(ra, rp)))
    run("add_plain", lambda o: P.ctx.add_plain(da, 2, dp, 1, o, 1), (2, k, n), lambda: W(R.add_plain(ra, rp)))
    run("sub_plain", lambda o: P.ctx.sub_plain(da, 2, dp, 1, o, 1), (2, k, n), lambda: W(R.sub_plain(ra, rp)))
    run("mod_switch_to_next", lambda o: P.ctx.mod_switch_to_next(da, 2, o, 1), (2, k - 1, n),
        lambda: W(R.mod_switch_to_next(ra)))
    K = len(P.moduli)
    key_ct = pc.rand_ct(rng, P.moduli, K, n)
    run("mod_switch_to_next at the key level", lambda o: P.ctx.mod_switch_to_next(P.dev(key_ct), 2, o, 1, level=0),
        (2, K - 1, n), lambda: modswitch_rounding(key_ct, [int(q) for q in P.moduli]))
    # decryption with the reference's secret key (NTT form) and its square
    kg = R.keygen()
    sk = R.secret_key(kg)
    h = vp()
    R.ref.call("SecretKey_Data", sk, C.byref(h))
    s_ntt = R.pt_coeffs(h).reshape(-1, n)
    pows = pc.key_powers(P, s_ntt, k, 2)
    c3 = pc.rand_ct(rng, P.moduli, k, n, size=3)
    dec = R.decryptor(sk)

    def ref_decrypt():
        got = R.pt_coeffs(R.decrypt(dec, R.new_ct(c3)))
        out = np.zeros(n, dtype=np.uint64)
        out[: got.size] = got
        return out
    run("ct_sk_phase", lambda o: P.ctx.ct_sk_phase(P.dev(c3), 3, P.dev(pows), o, 1), (k, n),
        lambda: pc.independent_phase(P, c3, pows))
    run("decrypt", lambda o: P.ctx.decrypt(P.dev(c3), 3, P.dev(pows), o, 1), (n,), ref_decrypt)
    return refused


def check_beyond_limit_layer2(S, n, moduli, t):
    """every Evaluator / Encryptor / Decryptor / KeyGenerator call of the chain's first data level on both libraries: HRESULT
    0 with the reference's words, or E_INVALIDARG where the reference succeeds; returns the set of refused calls"""
    R = refseal.RefContext(n, moduli, t)
    O = S.context(n, moduli, t)
    assert O.parameters_set and list(O.first_id) == list(R.first_parms_id) and list(O.key_id) == list(R.key_parms_id)
    RL, OL = sc._libs(R, O)
    kg = R.keygen()
    sk, pk, rlk = R.secret_key(kg), R.public_key(kg), R.relin_keys(kg)
    glk = R.galois_keys_steps(kg, [1])
    enc, dec = R.encryptor(pk, sk), R.decryptor(sk)
    to_ours = lambda h, kind="Ciphertext": OL.load(kind, RL.save(kind, h, 0))
    orlk, oglk, osk, opk = to_ours(rlk, "KSwitchKeys"), to_ours(glk, "KSwitchKeys"), to_ours(sk, "SecretKey"), to_ours(pk, "PublicKey")
    odec, oenc = vp(), vp()
    O.S.call("Decryptor_Create", O.ctx, osk, C.byref(odec))
    O.S.call("Encryptor_Create", O.ctx, opk, osk, C.byref(oenc))
    rng = np.random.default_rng(11)
    ra = R.encrypt(enc, R.new_pt(rng.integers(0, t, size=n, dtype=np.uint64)))
    rb = R.encrypt(enc, R.new_pt(rng.integers(0, t, size=n, dtype=np.uint64)))
    oa, ob = to_ours(ra), to_ours(rb)
    pl = rng.integers(1, t, size=n, dtype=np.uint64)
    rm = R.multiply(ra, rb)
    om = to_ours(rm)
    refused = set()

    def call(name, fn, words):
        try:
            got = fn()
        except SealcError as e:
            assert e.code == E_INVALIDARG, (name, hex(e.code))
            refused.add(name)
            return
        assert got == words, f"{name}: different words from the reference's"

    ser = lambda L, h: L.save("Ciphertext", h, 0)
    both = lambda rfn, ofn: (lambda: ser(OL, ofn()), ser(RL, rfn()))
    for name, rfn, ofn in (
            ("Evaluator_Add", lambda: R.add(ra, rb), lambda: O.add(oa, ob)),
            ("Evaluator_Sub", lambda: R.sub(ra, rb), lambda: O.sub(oa, ob)),
            ("Evaluator_Negate", lambda: R.negate(ra), lambda: O.negate(oa)),
            ("Evaluator_Multiply", lambda: rm, lambda: O.multiply(oa, ob)),
            ("Evaluator_Square", lambda: R.square(ra), lambda: O.square(oa)),
            ("Evaluator_Relinearize", lambda: R.relinearize(rm, rlk), lambda: O.relinearize(om, orlk)),
            ("Evaluator_MultiplyPlain", lambda: R.multiply_plain(ra, R.new_pt(pl)), lambda: O.multiply_plain(oa, O.new_pt(pl))),
            ("Evaluator_AddPlain", lambda: R.add_plain(ra, R.new_pt(pl)), lambda: O.add_plain(oa, O.new_pt(pl))),
            ("Evaluator_SubPlain", lambda: R.sub_plain(ra, R.new_pt(pl)), lambda: O.sub_plain(oa, O.new_pt(pl))),
            ("Evaluator_RotateRows", lambda: R.rotate_rows(ra, 1, glk), lambda: O.rotate_rows(oa, 1, oglk)),
            ("Evaluator_ModSwitchToNext1", lambda: R.mod_switch_to_next(ra), lambda: O.mod_switch_to_next(oa))):
        call(name, *both(rfn, ofn))
    # decryption and noise budget of a fresh encryption and of a product
    for what, rh, oh in (("fresh", ra, oa), ("product", rm, om)):
        call(f"Decryptor_Decrypt ({what})", lambda: O.pt_coeffs(O.decrypt(odec, oh)).tobytes(),
             R.pt_coeffs(R.decrypt(dec, rh)).tobytes())
        call(f"Decryptor_InvariantNoiseBudget ({what})", lambda: O.noise_budget(odec, oh), R.noise_budget(dec, rh))
    # seeded public-key encryption: the same words for the same seed
    seed = (u64 * 8)(*range(1, 9))
    msg = rng.integers(0, t, size=n, dtype=np.uint64)

    def seeded(L, encryptor, new_pt):
        ct, u, e, rem = L.new("Ciphertext"), vp(), vp(), L.new("Plaintext")
        L.call("PolynomialArray_Create", None, C.byref(u))
        L.call("PolynomialArray_Create", None, C.byref(e))
        L.call("Encryptor_EncryptReturnComponentsSetSeed", encryptor, new_pt(msg), C.c_bool(False), ct, u, e, rem, seed, None)
        return L.save("Ciphertext", ct, 0)
    call("Encryptor_EncryptReturnComponentsSetSeed", lambda: seeded(OL, oenc, O.new_pt), seeded(RL, enc, R.new_pt))
    # unseeded encryption (public and secret key) and key generation: random words, so the reference decrypts ours
    def decrypts(fn):
        def run():
            ct = fn()
            back = R.pt_coeffs(R.decrypt(dec, R.new_ct(O.ct_words(ct))))
            return back.tobytes()
        return run
    small = msg[:16]
    expect = small[: np.flatnonzero(small)[-1] + 1].tobytes()

    def encrypt(fn_name, *extra):
        def go():
            d = O._dst()
            O.S.call(fn_name, oenc, O.new_pt(small), *extra, d, None)
            return d
        return go
    call("Encryptor_Encrypt", decrypts(encrypt("Encryptor_Encrypt")), expect)
    call("Encryptor_EncryptSymmetric", decrypts(encrypt("Encryptor_EncryptSymmetric", C.c_bool(False))), expect)
    # keys from our KeyGenerator (over the reference's secret key) work on the reference: it encrypts with our public key
    # and relinearizes with our relinearization keys, and decrypts both
    okg = vp()
    O.S.call("KeyGenerator_Create2", O.ctx, osk, C.byref(okg))

    def our_key(kind, fn_name):
        def make():
            h = vp()
            O.S.call(fn_name, okg, C.c_bool(False), C.byref(h))
            return RL.load(kind, OL.save(kind, h, 0))
        return make
    call("KeyGenerator_CreatePublicKey", lambda: R.pt_coeffs(R.decrypt(dec, R.encrypt(
        R.encryptor(our_key("PublicKey", "KeyGenerator_CreatePublicKey")()), R.new_pt(small)))).tobytes(), expect)
    call("KeyGenerator_CreateRelinKeys", lambda: R.pt_coeffs(R.decrypt(dec, R.relinearize(
        rm, our_key("KSwitchKeys", "KeyGenerator_CreateRelinKeys")()))).tobytes(), R.pt_coeffs(R.decrypt(dec, rm)).tobytes())
    return refused


@pytest.mark.gpu
def test_beyond_limit_layer1(pairs):
    assert beyond_limit_layer1(pairs("n16384_24x18")) == REFUSED_LAYER1


@pytest.mark.gpu
def test_beyond_limit_layer2(S_gpu, ref):
    assert check_beyond_limit_layer2(S_gpu, *PARAMS["n16384_24x18"]) == REFUSED_LAYER2


def test_beyond_limit_layer1_emulation(emu_lib, ref):
    assert beyond_limit_layer1(emu_pair(emu_lib, "n16384_24x18")) == REFUSED_LAYER1


def test_beyond_limit_layer2_emulation(S_emu, ref):
    assert check_beyond_limit_layer2(S_emu, *PARAMS["n16384_24x18"]) == REFUSED_LAYER2
