"""Word-for-word parity checks of the B200 path against the unmodified reference (shared by CPU-emu and GPU tests)."""
import math

import numpy as np

from refseal import COR_E_INVALIDOPERATION, E_INVALIDARG, SEC_TC128, RefContext, SealError, appendix_b_inputs, fnv1a64
from sunscreen_b200.lib import B200Context


class Pair:
    """Same parameters instantiated on the reference and on the B200 library."""

    def __init__(self, be, n, moduli, t, sec_level=SEC_TC128):
        self.be = be
        self.n, self.moduli, self.t = n, list(moduli), t
        self.ref = RefContext(n, moduli, t, sec_level)
        self.ctx = B200Context(n, moduli, t, lib=be.lib)
        self.k = self.ctx.k()
        self.inp = appendix_b_inputs(n, self.moduli, t)

    def dev(self, arr):
        return self.be.to_dev(arr)

    def host(self, x):
        return self.be.to_host(x)

    def out(self, *shape):
        return self.be.empty(shape)


def rand_ct(rng, moduli, k, n, size=2, batch=None):
    shape = (size, k, n) if batch is None else (batch, size, k, n)
    out = np.empty(shape, dtype=np.uint64)
    for i in range(k):
        out[..., i, :] = rng.integers(0, moduli[i], size=shape[:-2] + (n,), dtype=np.uint64)
    return out


def rand_ksk(rng, moduli, k, n):
    K = len(moduli)
    out = np.empty((k, 2, K, n), dtype=np.uint64)
    for i in range(K):
        out[:, :, i, :] = rng.integers(0, moduli[i], size=(k, 2, n), dtype=np.uint64)
    return out


def eq(got, exp, what):
    got = np.asarray(got).reshape(-1)
    exp = np.asarray(exp).reshape(-1)
    assert got.shape == exp.shape, f"{what}: shape {got.shape} vs {exp.shape}"
    if not np.array_equal(got, exp):
        bad = np.flatnonzero(got != exp)
        raise AssertionError(f"{what}: {bad.size} of {got.size} words differ; first at {bad[:4]}: "
                             f"{got[bad[:4]]} vs {exp[bad[:4]]}")


def pair_for(be, name):
    """Pair for a named parameter set of tests/params.py, at the security level the reference needs for it"""
    from params import PARAMS, SEC_NONE
    from refseal import SEC_NONE as NONE
    return Pair(be, *PARAMS[name], sec_level=NONE if name in SEC_NONE else SEC_TC128)


def check_context(P):
    li = P.ctx.level_info(P.ctx.first_level)
    ri = P.ref.rns_info()
    assert li["parms_id"] == list(P.ref.first_parms_id)
    assert P.ctx.level_info(0)["parms_id"] == list(P.ref.key_parms_id)
    assert li["gamma"] == ri["gamma"]
    if li["m_sk"] == ri["m_sk"]:
        # the reference's own auxiliary base (61-bit primes), |B| = k, plus one when 32 + bits(t) + bits(Q) >= 61 (k + 1)
        # (S/util/rns.cpp:617-624)
        assert li["bsk"] == ri["bsk_primes"] and (li["nB"], li["nBsk"]) == (ri["B"], ri["Bsk"])
        Q = math.prod(li["q"])
        assert li["nB"] == li["k"] + (32 + P.t.bit_length() + Q.bit_length() >= 61 * li["k"] + 61)
    else:
        # FP64-friendly auxiliary base: 47..49-bit NTT primes (as wide as the widest user prime), distinct from the user's
        # primes, with at least the reference's dynamic range condition
        # 32 + bits(t) + bits(Q) < bits(prod(B) * m_sk)   (S/util/rns.cpp:617-624); results are base-independent.
        width = max(47, max(int(m).bit_length() for m in P.moduli))
        assert width <= 49
        assert all(p < (1 << width) and p % (2 * P.n) == 1 for p in li["bsk"]) and len(set(li["bsk"])) == len(li["bsk"])
        assert not set(li["bsk"]) & set(int(m) for m in P.moduli) and P.t not in li["bsk"]
        Q = math.prod(li["q"])
        assert math.prod(li["bsk"]).bit_length() > 32 + P.t.bit_length() + Q.bit_length()
    pi = P.ref.plain_info()
    assert li["delta"] == pi["delta"]
    # the reference keeps Q mod t as RNS residues (S/context.cpp:309-326)
    Q = math.prod(li["q"])
    assert li["q_mod_t"] == Q % P.t
    assert pi["upper_half_increment"] == [li["q_mod_t"] % q for q in li["q"]]
    if all(q > P.t for q in li["q"]):
        # fast plain lift: the increment is q_i - t per residue
        assert pi["plain_upper_half_increment"] == [q - P.t for q in li["q"]]
    else:
        # a prime below t: the reference stores Q - t as one multi-word integer instead (S/context.cpp:341-346)
        words = pi["plain_upper_half_increment"]
        assert sum(w << (64 * i) for i, w in enumerate(words)) == Q - P.t
    for q, r in zip(li["q"], li["roots"]):
        assert P.ref.ref.ntt_root(q, P.n) == r


def check_ntt(P, items=6, seed=1):
    rng = np.random.default_rng(seed)
    x = rand_ct(rng, P.moduli, P.k, P.n, size=1, batch=items)[:, 0]
    x[0, :, :8] = 0
    x[0, 0, 0] = 1  # delta -> all-ones spectrum
    # magnitude extremes for the lazy (signed FP64 / Harvey) representations: every coefficient q-1, alternating 0 / q-1,
    # and a +-1 pattern (q-1 = -1) that makes the butterflies add up coherently
    qm1 = np.array([m - 1 for m in P.moduli[: P.k]], dtype=np.uint64)[:, None]
    if items >= 6:
        x[3] = np.broadcast_to(qm1, (P.k, P.n))
        x[4] = 0
        x[4, :, ::2] = qm1
        x[5] = 1
        x[5, :, 1::3] = qm1
    d = P.dev(x)
    P.ctx.ntt_forward(d, items)
    got = P.host(d)
    exp = np.stack([np.stack([P.ref.ref.ntt_forward(P.moduli[i], x[b, i]) for i in range(P.k)]) for b in range(items)])
    eq(got, exp, "ntt_forward")
    P.ctx.ntt_inverse(d, items)
    eq(P.host(d), x, "ntt round trip")
    # inverse alone against the reference
    d2 = P.dev(exp)
    P.ctx.ntt_inverse(d2, items)
    eq(P.host(d2), x, "ntt_inverse")


def check_elementwise(P):
    a, b = P.inp["a"], P.inp["b"]
    ra, rb = P.ref.new_ct(a), P.ref.new_ct(b)
    da, db = P.dev(a), P.dev(b)
    o = P.out(2, P.k, P.n)
    P.ctx.add(da, db, o, 2, 1)
    eq(P.host(o), P.ref.ct_words(P.ref.add(ra, rb)), "add")
    P.ctx.sub(da, db, o, 2, 1)
    eq(P.host(o), P.ref.ct_words(P.ref.sub(ra, rb)), "sub")
    P.ctx.negate(da, o, 2, 1)
    eq(P.host(o), P.ref.ct_words(P.ref.negate(ra)), "negate")
    # zero stays zero under negate
    z = np.zeros_like(a)
    P.ctx.negate(P.dev(z), o, 2, 1)
    eq(P.host(o), z, "negate(0)")


def check_multiply(P, with_sizes=True):
    a, b = P.inp["a"], P.inp["b"]
    ra, rb = P.ref.new_ct(a), P.ref.new_ct(b)
    da, db = P.dev(a), P.dev(b)
    o3 = P.out(3, P.k, P.n)
    P.ctx.multiply(da, 2, db, 2, o3, 1)
    rm = P.ref.multiply(ra, rb)
    m3 = P.ref.ct_words(rm)
    eq(P.host(o3), m3, "multiply(2,2)")
    P.ctx.square(da, o3, 1)
    eq(P.host(o3), P.ref.ct_words(P.ref.square(ra)), "square")
    if with_sizes:
        # (3,2) -> 4 : the general K x L convolution loop (S/evaluator.cpp:497-541)
        o4 = P.out(4, P.k, P.n)
        P.ctx.multiply(P.dev(m3), 3, db, 2, o4, 1)
        eq(P.host(o4), P.ref.ct_words(P.ref.multiply(rm, rb)), "multiply(3,2)")
    return m3, rm


def check_relin(P, m3=None, rm=None):
    if m3 is None:
        ra, rb = P.ref.new_ct(P.inp["a"]), P.ref.new_ct(P.inp["b"])
        rm = P.ref.multiply(ra, rb)
        m3 = P.ref.ct_words(rm)
    rlk = P.ref.new_ksk({0: P.inp["rlk"]})
    exp = P.ref.ct_words(P.ref.relinearize(rm, rlk))
    dk = P.dev(P.inp["rlk"])
    o2 = P.out(2, P.k, P.n)
    P.ctx.relinearize(P.dev(m3), dk, o2, 1)
    eq(P.host(o2), exp, "relinearize")
    o2b = P.out(2, P.k, P.n)
    P.ctx.multiply_relin(P.dev(P.inp["a"]), P.dev(P.inp["b"]), dk, o2b, 1)
    eq(P.host(o2b), exp, "multiply_relin")
    return exp


def check_galois(P):
    """Galois automorphisms 3 (rotate rows by 1) and 2n-1 (swap columns).  Without a batching plain modulus the reference
    refuses rotate_rows / rotate_columns, but Evaluator::apply_galois with the same elements and keys is still defined
    (S/evaluator.cpp:2217-2307): the comparison is then against that."""
    n = P.n
    a = P.inp["a"]
    ra = P.ref.new_ct(a)
    glk = P.ref.new_ksk({(3 - 1) // 2: P.inp["glk3"], (2 * n - 1 - 1) // 2: P.inp["glkc"]})
    da = P.dev(a)
    o2 = P.out(2, P.k, P.n)
    if P.ctx.using_batching:
        assert P.ctx.galois_elt_from_step(1) == 3 and P.ctx.galois_elt_from_step(0) == 2 * n - 1
        exp_rows, exp_cols = P.ref.rotate_rows(ra, 1, glk), P.ref.rotate_columns(ra, glk)
    else:
        exp_rows, exp_cols = P.ref.apply_galois(ra, 3, glk), P.ref.apply_galois(ra, 2 * n - 1, glk)
    P.ctx.apply_galois(da, 3, P.dev(P.inp["glk3"]), o2, 1)
    eq(P.host(o2), P.ref.ct_words(exp_rows), "galois 3 (rotate_rows(1))")
    P.ctx.apply_galois(da, 2 * n - 1, P.dev(P.inp["glkc"]), o2, 1)
    eq(P.host(o2), P.ref.ct_words(exp_cols), "galois 2n-1 (rotate_columns)")


def check_plain(P):
    a, p = P.inp["a"], P.inp["p"]
    ra, rp = P.ref.new_ct(a), P.ref.new_pt(p)
    da, dp = P.dev(a), P.dev(p)
    o2 = P.out(2, P.k, P.n)
    P.ctx.multiply_plain(da, 2, dp, 1, o2, 1)
    eq(P.host(o2), P.ref.ct_words(P.ref.multiply_plain(ra, rp)), "multiply_plain")
    P.ctx.add_plain(da, 2, dp, 1, o2, 1)
    eq(P.host(o2), P.ref.ct_words(P.ref.add_plain(ra, rp)), "add_plain")
    P.ctx.sub_plain(da, 2, dp, 1, o2, 1)
    eq(P.host(o2), P.ref.ct_words(P.ref.sub_plain(ra, rp)), "sub_plain")
    # monomial plaintext (the reference takes its fast path, S/evaluator.cpp:1885-1933): same words expected
    mono = np.zeros(P.n, dtype=np.uint64)
    mono[5] = 7 if 7 < (P.t + 1) // 2 else 1
    rm = P.ref.new_pt(mono[:6])
    P.ctx.multiply_plain(da, 2, P.dev(mono), 1, o2, 1)
    eq(P.host(o2), P.ref.ct_words(P.ref.multiply_plain(ra, rm)), "multiply_plain(monomial)")


def plain_operand_classes(n, t, rng):
    """(label, coefficients) of the plaintexts whose lift differs between the reference's paths: monomials m * x^e with m in
    {1, thr - 1, thr, t - 1, t, t + 5} (thr = (t+1)/2, the upper-half threshold; the Evaluator checks only metadata, so
    coefficients >= t are defined) at e in {0, 1, n - 1}; dense plaintexts in the upper half and in [t, t + 5]; and two
    nonzero coefficients, just off the monomial path.  Shuffled, so monomial and dense items alternate within a batch."""
    thr = (t + 1) // 2
    out = []
    for m in sorted({1, thr - 1, thr, t - 1, t, t + 5} - {0}):
        for e in (0, 1, n - 1):
            p = np.zeros(n, dtype=np.uint64)
            p[e] = m
            out.append((f"{m} * x^{e}", p))
    out.append(("dense upper half", rng.integers(thr, t, size=n, dtype=np.uint64)))
    out.append(("dense in [t, t + 5]", rng.integers(t, t + 6, size=n, dtype=np.uint64)))
    two = np.zeros(n, dtype=np.uint64)
    two[3], two[n - 1] = t - 1, thr
    out.append(("two nonzero", two))
    return [out[i] for i in rng.permutation(len(out))]


def check_plain_operands(P, seed=41, levels=None):
    """multiply_plain / add_plain / sub_plain with every plaintext class of plain_operand_classes, one per item of a batch
    (plain_batch == batch, so the monomial test is per item), at every data level of the reference's chain (or the data
    levels `levels`, 0 = the first) through layer 1's `level` argument, word for word against the reference's Evaluator;
    then one monomial broadcast to every item (plain_batch = 1).  Where the reference's product is transparent (a monomial
    t under a prime below t: Q - t + t = Q), it refuses it and the layer-1 words must be all zero."""
    rng = np.random.default_rng(seed)
    R = P.ref
    classes = plain_operand_classes(P.n, P.t, rng)
    labels = [c[0] for c in classes]
    plains = np.stack([c[1] for c in classes])
    B = len(classes)
    dpl = P.dev(plains)
    thr = (P.t + 1) // 2
    minus_one = np.zeros((1, P.n), dtype=np.uint64)
    minus_one[0, 0] = P.t - 1
    rpls = [R.new_pt(p) for p in plains]
    rp = R.new_pt(minus_one[0, :1])
    for j in range(len(R.data_parms_ids())) if levels is None else levels:
        lv = P.ctx.first_level + j
        k = P.ctx.level_info(lv)["k"]
        assert k == R.k - j
        moduli = P.moduli[:k]
        cts = rand_ct(rng, moduli, k, P.n, batch=B)
        dct = P.dev(cts)
        out = P.out(B, 2, k, P.n)
        rcts = [R.new_ct(cts[i], level=j) for i in range(B)]
        for op in ("multiply_plain", "add_plain", "sub_plain"):
            getattr(P.ctx, op)(dct, 2, dpl, B, out, B, level=lv)
            got = P.host(out).reshape(B, 2, k, P.n)
            for i in range(B):
                try:
                    rr = getattr(R, op)(rcts[i], rpls[i])
                except SealError as e:
                    assert op == "multiply_plain" and e.code == COR_E_INVALIDOPERATION, (op, labels[i], e)
                    eq(got[i], np.zeros_like(got[i]), f"{op} at level {lv}, item {i} ({labels[i]}): transparent")
                    continue
                eq(got[i], R.ct_words(rr), f"{op} at level {lv}, item {i} ({labels[i]})")
                R.free_ct(rr)
        # one plaintext for every item: the constant -1 (t - 1 >= thr whenever t > 1)
        assert P.t - 1 >= thr
        P.ctx.multiply_plain(dct, 2, P.dev(minus_one), 1, out, B, level=lv)
        got = P.host(out).reshape(B, 2, k, P.n)
        for i in range(B):
            rr = R.multiply_plain(rcts[i], rp)
            eq(got[i], R.ct_words(rr), f"multiply_plain by (t-1) * x^0 broadcast, level {lv}, item {i}")
            R.free_ct(rr)
        for h in rcts:
            R.free_ct(h)
    for h in rpls + [rp]:
        R.free_pt(h)


def check_modswitch(P):
    a = P.inp["a"]
    if P.k < 2:
        return
    ra = P.ref.new_ct(a)
    o = P.out(2, P.k - 1, P.n)
    P.ctx.mod_switch_to_next(P.dev(a), 2, o, 1)
    q = [int(m) for m in P.moduli[: P.k]]
    if math.prod(q[:-1]) > P.t:
        eq(P.host(o), P.ref.ct_words(P.ref.mod_switch_to_next(ra)), "mod_switch_to_next")
        return
    # the next level cannot hold t, so the reference's chain ends here and it refuses; the layer-1 kernel is still
    # defined: floor((X + q_last/2) / q_last) of the CRT value X, the reference's divide_and_round_q_last
    try:
        P.ref.mod_switch_to_next(ra)
    except SealError as e:
        assert e.code == E_INVALIDARG, e
    else:
        raise AssertionError("the reference switched to a level whose modulus is below t")
    got = P.host(o).reshape(2, P.k - 1, P.n)
    Q, half = math.prod(q), q[-1] >> 1
    for s in range(2):
        X = [sum(int(a[s, i, c]) * (Q // q[i]) * pow(Q // q[i], -1, q[i]) for i in range(P.k)) % Q for c in range(P.n)]
        want = np.array([[(x + half) // q[-1] % qi for x in X] for qi in q[:-1]], dtype=np.uint64)
        eq(got[s], want, f"mod_switch_to_next (component {s}) against the big-integer rounding")


def check_batch(P, batch=3, seed=7):
    """Distinct items in one launch: strides / item indexing."""
    rng = np.random.default_rng(seed)
    A = rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    B = rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    key = rand_ksk(rng, P.moduli, P.k, P.n)
    rlk = P.ref.new_ksk({0: key})
    glk = P.ref.new_ksk({1: key})
    dA, dB, dK = P.dev(A), P.dev(B), P.dev(key)
    o2 = P.out(batch, 2, P.k, P.n)
    o3 = P.out(batch, 3, P.k, P.n)
    P.ctx.multiply(dA, 2, dB, 2, o3, batch)
    got3 = P.host(o3)
    P.ctx.multiply_relin(dA, dB, dK, o2, batch)
    got2 = P.host(o2)
    og = P.out(batch, 2, P.k, P.n)
    P.ctx.apply_galois(dA, 3, dK, og, batch)
    gotg = P.host(og)
    for i in range(batch):
        ra, rb = P.ref.new_ct(A[i]), P.ref.new_ct(B[i])
        rm = P.ref.multiply(ra, rb)
        eq(got3[i], P.ref.ct_words(rm), f"batch multiply item {i}")
        eq(got2[i], P.ref.ct_words(P.ref.relinearize(rm, rlk)), f"batch multiply_relin item {i}")
        if P.ctx.using_batching:
            eq(gotg[i], P.ref.ct_words(P.ref.rotate_rows(ra, 1, glk)), f"batch rotate item {i}")
        for h in (ra, rb, rm):
            P.ref.free_ct(h)


def negacyclic_mul_mod(x, y, t):
    """x * y in Z_t[X] / (X^n + 1), coefficients of x, y below t < 2^60: the 20-bit limbs are convolved exactly in int64
    (sums below 2^55 for n <= 32768) and recombined with Python integers."""
    n = x.size
    limbs = lambda v: [((v >> np.uint64(20 * i)) & np.uint64(0xFFFFF)).astype(np.int64) for i in range(3)]
    X, Y = limbs(x), limbs(y)
    c = np.zeros(2 * n, dtype=object)
    for i in range(3):
        for j in range(3):
            if X[i].any() and Y[j].any():
                c[: 2 * n - 1] += np.convolve(X[i], Y[j]).astype(object) * (1 << (20 * (i + j)))
    return ((c[:n] - c[n:]) % t).astype(np.uint64)


def check_encrypted_roundtrip(P, seed=3):
    """Real keys + fresh encryptions from the reference; our multiply+relin output equals the reference's ciphertext word
    for word, and, where the reference's own product still has noise budget, decrypts on the reference to the product of
    the messages (slot-wise for a batching plain modulus, else the negacyclic product of coefficient plaintexts).  Chains
    without room for one multiplication only get the word comparison."""
    rng = np.random.default_rng(seed)
    R = P.ref
    kg = R.keygen()
    sk, pk, rk = R.secret_key(kg), R.public_key(kg), R.relin_keys(kg)
    enc, dec = R.encryptor(pk), R.decryptor(sk)
    v1 = rng.integers(0, P.t, size=P.n, dtype=np.uint64)
    v2 = rng.integers(0, P.t, size=P.n, dtype=np.uint64)
    if P.ctx.using_batching:
        be_ = R.batch_encoder()
        c1, c2 = R.encrypt(enc, R.batch_encode(be_, v1)), R.encrypt(enc, R.batch_encode(be_, v2))
    else:
        c1, c2 = R.encrypt(enc, R.new_pt(v1)), R.encrypt(enc, R.new_pt(v2))
    w1, w2 = R.ct_words(c1), R.ct_words(c2)
    key = R.ksk_words(rk)[0]
    exp_ct = R.relinearize(R.multiply(c1, c2), rk)
    o2 = P.out(2, P.k, P.n)
    P.ctx.multiply_relin(P.dev(w1), P.dev(w2), P.dev(key), o2, 1)
    got = P.host(o2)
    eq(got, R.ct_words(exp_ct), "multiply_relin on real ciphertexts")
    back = R.new_ct(got.reshape(2, P.k, P.n))
    if R.noise_budget(dec, exp_ct) == 0:
        return None
    assert R.noise_budget(dec, back) > 0
    if P.ctx.using_batching:
        vals = R.batch_decode(be_, R.decrypt(dec, back))
        expect = (v1.astype(object) * v2.astype(object)) % P.t
        assert np.array_equal(vals.astype(object), expect)
    else:
        coeffs = R.pt_coeffs(R.decrypt(dec, back))
        vals = np.zeros(P.n, dtype=np.uint64)
        vals[: coeffs.size] = coeffs
        eq(vals, negacyclic_mul_mod(v1, v2, P.t), "decrypted product")
    return dict(dec=dec, sk=sk, ct=got, expect_plain=R.pt_coeffs(R.decrypt(dec, back)))


def check_small_kernels(P, seed=29):
    """b200_is_transparent / b200_any_nonzero (the transparent-result guard, S/ciphertext.h:451-456) on a batch with one
    transparent item and one whose only nonzero word is the very last; b200_expand_signed (residues of the host-sampled
    ternary / clipped-normal values, S/util/rlwe.cpp:23-67) against v mod q_i."""
    rng = np.random.default_rng(seed)
    batch = 4
    ct = rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    ct[1, 1:] = 0                      # transparent: c1 == 0 (c0 arbitrary)
    ct[2, 1:] = 0
    ct[2, 1, P.k - 1, P.n - 1] = 1     # a single nonzero word at the very end
    d = P.dev(ct)
    words = (batch + 1) // 2
    flags = P.dev(np.zeros(words, dtype=np.uint64))
    P.ctx.is_transparent(d, 2, flags, batch)
    got = P.host(flags).view(np.uint32)[:batch]
    assert list(got) == [0, 1, 0, 0], f"is_transparent flags {list(got)}"
    flags = P.dev(np.zeros(words, dtype=np.uint64))
    P.ctx.any_nonzero(d, 2, flags, batch)
    got = P.host(flags).view(np.uint32)[:batch]
    assert list(got) == [1, 0, 1, 1], f"any_nonzero flags {list(got)}"
    vals = rng.integers(-19, 20, size=(3, P.n), dtype=np.int64)
    vals[0, :4] = (-1, 0, 1, -19)
    out = P.out(3, P.k, P.n)
    P.ctx.expand_signed(P.dev(vals.view(np.uint64)), 3, out)
    got = P.host(out).reshape(3, P.k, P.n)
    for i in range(P.k):
        want = (vals.astype(object) % int(P.moduli[i])).astype(np.uint64)
        eq(got[:, i, :], want, f"expand_signed residue {i}")


def independent_phase(P, ct, powers):
    """c0 + sum_j c_j * s^j in coefficient form for one ciphertext ct [size][k][n] and NTT-form key powers [size-1][k][n]:
    the reference's util-level NTT (S/util/ntt.cpp) and dyadic products with Python integers."""
    size, k = ct.shape[0], ct.shape[1]
    out = np.empty((k, P.n), dtype=np.uint64)
    for i in range(k):
        q = int(P.moduli[i])
        acc = np.zeros(P.n, dtype=object)
        for j in range(1, size):
            acc = (acc + P.ref.ref.ntt_forward(q, ct[j, i]).astype(object) * powers[j - 1, i].astype(object)) % q
        back = P.ref.ref.ntt_inverse(q, acc.astype(np.uint64))
        out[i] = ((back.astype(object) + ct[0, i].astype(object)) % q).astype(np.uint64)
    return out


def key_powers(P, s_ntt, k, count):
    """[count][k][n] NTT-form powers s, s^2, ... of the NTT-form key residues s_ntt [>= k][n], with Python integers."""
    out = np.empty((count, k, P.n), dtype=np.uint64)
    for i in range(k):
        q = int(P.moduli[i])
        s = s_ntt[i].astype(object)
        cur = s
        for j in range(count):
            out[j, i] = cur.astype(np.uint64)
            cur = cur * s % q
    return out


def check_noise_norm(P, batch=3, seed=23):
    """b200_noise_norm (the quantity behind invariant_noise_budget, S/decryptor.cpp:424-485): for random ciphertexts of
    size 2 and 3 and random key powers, the device's multi-precision infinity norm of the centred t * phase mod Q equals
    the same computed with Python integers from a phase computed independently of the library (independent_phase); the
    library's own b200_ct_sk_phase must equal that phase too."""
    from functools import reduce
    rng = np.random.default_rng(seed)
    q = [int(m) for m in P.moduli[: P.k]]
    Q = reduce(lambda a, b: a * b, q)
    words = (Q.bit_length() + 63) // 64 + 1
    for size in (2, 3):
        ct = rand_ct(rng, P.moduli, P.k, P.n, size=size, batch=batch)
        skp = np.stack([np.stack([rng.integers(0, q[i], size=P.n, dtype=np.uint64) for i in range(P.k)]) for _ in range(size - 1)])
        dct, dsk = P.dev(ct), P.dev(skp)
        ph = P.out(batch, P.k, P.n)
        P.ctx.ct_sk_phase(dct, size, dsk, ph, batch)
        phase = np.stack([independent_phase(P, ct[b], skp) for b in range(batch)])
        eq(P.host(ph), phase, f"ct_sk_phase, size {size}")
        got = np.zeros((batch, words), dtype=np.uint64)
        P.ctx.noise_norm(dct, size, dsk, got, words, batch)
        coef = [(Q // qi) * pow(Q // qi, -1, qi) * P.t % Q for qi in q]
        for b in range(batch):
            best = 0
            for c in range(P.n):
                v = sum(int(phase[b, i, c]) * coef[i] for i in range(P.k)) % Q
                v = Q - v if v >= (Q + 1) // 2 else v
                best = max(best, v)
            mine = sum(int(got[b, w]) << (64 * w) for w in range(words))
            assert mine == best, f"noise norm, size {size}, item {b}: {mine:#x} != {best:#x}"


def decrypt_branch(X, q, t, g):
    """(upper, zero) for a phase X mod Q = prod(q): whether the {t, gamma} correction of RNSTool::decrypt_scale_and_round
    (S/util/rns.cpp:1145-1213) takes its vg > gamma/2 branch, and whether the corrected value is 0 (the multiplication by
    gamma^-1 mod t is then skipped).  Used only to show that the crafted inputs reach every case, never as an expected value."""
    Q = math.prod(q)
    s = sum(X * t * g % qi * pow(Q // qi, -1, qi) % qi * (Q // qi) for qi in q)
    vt = s * -pow(Q, -1, t) % t
    vg = s * -pow(Q, -1, g) % g
    upper = vg > g >> 1
    return upper, ((vt + g - vg) if upper else (vt - vg)) % t == 0


def crafted_phases(Q, t, rng):
    """Phases at the edges of decryption: 0, 1, Q - 1, (Q -+ 1)/2; floor(jQ/t) + {-1, 0, 1} and the rounding boundaries
    floor((2j+1)Q/(2t)) + {-1, 0, 1, 2} for j in {0, 1, t/2, t - 1} and three random j."""
    js = {0, 1, t // 2, t - 1} | {int(rng.integers(0, t)) for _ in range(3)}
    X = [0, 1, Q - 1, (Q - 1) // 2, (Q + 1) // 2]
    for j in sorted(js):
        X += [j * Q // t + d for d in (-1, 0, 1)]
        X += [(2 * j + 1) * Q // (2 * t) + d for d in (-1, 0, 1, 2)]
    return [x % Q for x in X]


def _residues(X, q, n, rng):
    """[k][n] residues of the integers X (then uniformly random integers below prod(q) to fill n coefficients)."""
    import random
    Q = math.prod(q)
    fill = random.Random(int(rng.integers(0, 2**63)))
    X = list(X) + [fill.randrange(Q) for _ in range(n - len(X))]
    return np.array([[x % qi for x in X] for qi in q], dtype=np.uint64), X


def check_decrypt(P, batch=5, seed=31, levels=None):
    """b200_ct_sk_phase and b200_decrypt at every data level of the reference's chain (or the data levels `levels`, 0 = the
    first), with a real reference secret key
    (its NTT-form words; the powers s^2, s^3 come from Python integers):
    - uniformly random ciphertexts of size 2, 3 and 4, batch 5: the phase against independent_phase, the plaintext against
      the reference's Decryptor::decrypt (which accepts any ciphertext);
    - crafted phases (c1 = 0, so the phase is c0, set by CRT to chosen integers: crafted_phases): the plaintext against the
      reference's Decryptor and the plain-C oracle's decrypt; the inputs must reach both branches of the gamma correction
      and its m == 0 skip."""
    import ctypes as C
    from oracle_port import OraclePort
    rng = np.random.default_rng(seed)
    R = P.ref
    kg = R.keygen()
    sk = R.secret_key(kg)
    dec = R.decryptor(sk)
    h = C.c_void_p()
    R.ref.call("SecretKey_Data", sk, C.byref(h))
    s_ntt = R.pt_coeffs(h).reshape(-1, P.n)
    gamma = R.rns_info()["gamma"]
    port = OraclePort().context(P.n, P.moduli, P.t)

    def ref_decrypt(ct, j):
        c = R.new_ct(ct, level=j)
        got = R.pt_coeffs(R.decrypt(dec, c))
        R.free_ct(c)
        out = np.zeros(P.n, dtype=np.uint64)
        out[: got.size] = got
        return out

    for j in range(len(R.data_parms_ids())) if levels is None else levels:
        lv = P.ctx.first_level + j
        k = R.k - j
        assert P.ctx.level_info(lv)["k"] == k
        pows = key_powers(P, s_ntt, k, 3)
        dsk = P.dev(pows)
        for size in (2, 3, 4):
            ct = rand_ct(rng, P.moduli, k, P.n, size=size, batch=batch)
            dct = P.dev(ct)
            ph, pt = P.out(batch, k, P.n), P.out(batch, P.n)
            P.ctx.ct_sk_phase(dct, size, dsk, ph, batch, level=lv)
            P.ctx.decrypt(dct, size, dsk, pt, batch, level=lv)
            gph, gpt = P.host(ph).reshape(batch, k, P.n), P.host(pt).reshape(batch, P.n)
            for b in range(batch):
                eq(gph[b], independent_phase(P, ct[b], pows), f"ct_sk_phase, level {lv}, size {size}, item {b}")
                eq(gpt[b], ref_decrypt(ct[b], j), f"decrypt, level {lv}, size {size}, item {b}")
        q = [int(m) for m in P.moduli[:k]]
        Q = math.prod(q)
        X = crafted_phases(Q, P.t, rng)
        c0, _ = _residues(X, q, P.n, rng)
        ct = np.zeros((2, k, P.n), dtype=np.uint64)
        ct[0] = c0
        pt = P.out(P.n)
        P.ctx.decrypt(P.dev(ct), 2, dsk, pt, 1, level=lv)
        got = P.host(pt).reshape(P.n)
        eq(got, ref_decrypt(ct, j), f"decrypt of crafted phases, level {lv}")
        orc = np.zeros(P.n, dtype=np.uint64)
        assert port.L.orc_decrypt(C.byref(port.c), k, ct.ctypes.data_as(C.c_void_p), 2, np.ascontiguousarray(pows[0]).ctypes.data_as(C.c_void_p),
                                  orc.ctypes.data_as(C.c_void_p)) == 0
        eq(got, orc, f"decrypt of crafted phases against the oracle, level {lv}")
        cases = {decrypt_branch(x, q, P.t, gamma) for x in X}
        assert {u for u, _ in cases} == {True, False} and {z for _, z in cases} == {True, False}, cases


def check_noise_norm_edges(P, seed=37):
    """b200_noise_norm where its multi-precision arithmetic has edges: phases X with t X = Y (mod Q) for Y = 0, (Q -+ 1)/2
    (the centring boundary), Q - 1, 2^64 - 1 and 2^64 (a word carry), placed at coefficient 0, 127, 128 (a block boundary)
    or n - 1 over values below 2^20, in batches of five items, one of them all zero.  Each edge value is the item's largest
    centred value except Q - 1, whose centred value is 1; the expected norm is computed with Python integers.  `words` above W + 1 leaves the extra words zero; below W + 1 is refused."""
    rng = np.random.default_rng(seed)
    q = [int(m) for m in P.moduli[: P.k]]
    Q = math.prod(q)
    W = (Q.bit_length() + 63) // 64
    tinv = pow(P.t, -1, Q)
    edges = [y for y in ((Q - 1) // 2, (Q + 1) // 2, Q - 1, 2**64 - 1, 2**64) if 0 < y < Q]
    skp = np.zeros((1, P.k, P.n), dtype=np.uint64)  # c1 = 0: the key powers do not matter
    dsk = P.dev(skp)
    centred = lambda y: Q - y if y >= (Q + 1) // 2 else y
    for p, pos in enumerate((0, 127, 128, P.n - 1)):
        ct = np.zeros((5, 2, P.k, P.n), dtype=np.uint64)
        want = [0]
        for b in range(1, 5):
            Y = [int(v) for v in rng.integers(0, 2**20, size=P.n)]
            Y[pos] = edges[(p + b) % len(edges)]
            want.append(max(centred(y) for y in Y))
            ct[b, 0], _ = _residues([y * tinv % Q for y in Y], q, P.n, rng)
        dct = P.dev(ct)
        for words in (W + 1, W + 3):
            got = np.zeros((5, words), dtype=np.uint64)
            P.ctx.noise_norm(dct, 2, dsk, got, words, 5)
            for b in range(5):
                mine = sum(int(got[b, w]) << (64 * w) for w in range(words))
                assert mine == want[b], f"noise norm, maximum at {pos}, item {b}, {words} words: {mine:#x} != {want[b]:#x}"
    try:
        P.ctx.noise_norm(dct, 2, dsk, np.zeros((5, W), dtype=np.uint64), W, 5)
    except Exception as e:  # B200Error(B200_E_INVALID)
        assert getattr(e, "code", None) == -1, e
    else:
        raise AssertionError(f"noise_norm must refuse {W} words for a {Q.bit_length()}-bit modulus")


def check_host_pipeline(P, batch=5, seed=17):
    """b200_multiply_relin_host (host buffers in, host buffers out; chunked, overlapped, packed 6-byte transfers when the
    level's primes fit 48 bits) returns the same words as the device-resident entry point, also when the ring of staging
    slots wraps (chunk of 1 item, 5 items, 3 slots); a word that does not fit the residue width is rejected."""
    import os
    rng = np.random.default_rng(seed)
    A = rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    B = rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    key = rand_ksk(rng, P.moduli, P.k, P.n)
    dK = P.dev(key)
    o2 = P.out(batch, 2, P.k, P.n)
    P.ctx.multiply_relin(P.dev(A), P.dev(B), dK, o2, batch)
    want = P.host(o2)
    old = os.environ.get("B200_HOST_CHUNK")
    old_pack = os.environ.get("B200_HOST_PACK")
    try:
        for pack in ("0", "1"):
            os.environ["B200_HOST_PACK"] = pack
            for chunk in ("1", "2", "64"):
                os.environ["B200_HOST_CHUNK"] = chunk
                oh = np.zeros((batch, 2, P.k, P.n), dtype=np.uint64)
                P.ctx.multiply_relin_host(A, B, dK, oh, batch)
                eq(oh, want, f"multiply_relin_host, chunk {chunk}, pack {pack}")
        if max(P.moduli[: P.k]) < 2**48:
            bad = A.copy()
            bad[batch - 1, 1, P.k - 1, P.n - 1] = np.uint64(2**48)
            try:
                P.ctx.multiply_relin_host(bad, B, dK, np.zeros_like(want), batch)
            except Exception as e:  # B200Error(B200_E_INVALID)
                assert "residue width" in str(e) or "-1" in str(e), e
            else:
                raise AssertionError("an out-of-range ciphertext word must be rejected by the packed pipeline")
    finally:
        for name, val in (("B200_HOST_CHUNK", old), ("B200_HOST_PACK", old_pack)):
            if val is None:
                os.environ.pop(name, None)
            else:
                os.environ[name] = val


# ---------------------------------------------------------------------------------------------------------
# adversarial operands: the extremes of every lazy range (signed FP64 values up to 2^53, Harvey [0, 4q), the substituted
# 47..49-bit auxiliary base of the FP64 BEHZ path) — all q-1, alternating 0 / q-1, a +-1 pattern, a single nonzero word
# ---------------------------------------------------------------------------------------------------------
ADVERSARIAL = ("qm1", "alt", "pm1", "single", "one")


def adversarial_ct(P, kind, size=2):
    q = np.array([int(m) for m in P.moduli[: P.k]], dtype=np.uint64)[None, :, None]
    x = np.zeros((size, P.k, P.n), dtype=np.uint64)
    if kind == "qm1":
        x[:] = q - np.uint64(1)
    elif kind == "alt":
        x[:, :, ::2] = np.broadcast_to(q - np.uint64(1), (size, P.k, (P.n + 1) // 2))
    elif kind == "pm1":
        x[:] = 1
        x[:, :, 1::3] = np.broadcast_to(q - np.uint64(1), x[:, :, 1::3].shape)
    elif kind == "single":
        x[:, :, P.n - 1] = np.broadcast_to((q - np.uint64(1))[:, :, 0], (size, P.k))
    elif kind == "one":
        x[:, :, 0] = 1
    else:
        raise ValueError(kind)
    return x


def check_adversarial_multiply(P, pairs=None, with_size5=True):
    """multiply / square / multiply_relin of adversarial operands, word for word against the reference (which runs its own
    61-bit auxiliary base and integer arithmetic throughout)."""
    R = P.ref
    rlk = R.new_ksk({0: P.inp["rlk"]})
    dk = P.dev(P.inp["rlk"])
    pairs = pairs or [("qm1", "qm1"), ("qm1", "alt"), ("alt", "pm1"), ("pm1", "pm1"), ("single", "qm1"), ("single", "single"),
                      ("one", "qm1"), ("alt", "alt")]
    for ka, kb in pairs:
        a, b = adversarial_ct(P, ka), adversarial_ct(P, kb)
        ra, rb = R.new_ct(a), R.new_ct(b)
        da, db = P.dev(a), P.dev(b)
        rm = R.multiply(ra, rb)
        o3 = P.out(3, P.k, P.n)
        P.ctx.multiply(da, 2, db, 2, o3, 1)
        eq(P.host(o3), R.ct_words(rm), f"multiply({ka},{kb})")
        o2 = P.out(2, P.k, P.n)
        P.ctx.multiply_relin(da, db, dk, o2, 1)
        eq(P.host(o2), R.ct_words(R.relinearize(rm, rlk)), f"multiply_relin({ka},{kb})")
        if ka == kb:
            P.ctx.square(da, o3, 1)
            eq(P.host(o3), R.ct_words(R.square(ra)), f"square({ka})")
        for h in (ra, rb, rm):
            R.free_ct(h)
    if with_size5:
        for kind in ("qm1", "alt"):
            a3, b3 = adversarial_ct(P, kind, 3), adversarial_ct(P, "pm1" if kind == "alt" else "qm1", 3)
            o5 = P.out(5, P.k, P.n)
            P.ctx.multiply(P.dev(a3), 3, P.dev(b3), 3, o5, 1)
            ra, rb = R.new_ct(a3), R.new_ct(b3)
            eq(P.host(o5), R.ct_words(R.multiply(ra, rb)), f"multiply (3,3) -> 5 of {kind}")


def check_adversarial_keyswitch(P):
    """relinearize / rotate on adversarial targets with an all-(p-1) key: the key-switch accumulators at their largest."""
    R = P.ref
    K = len(P.moduli)
    key = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        key[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    rlk = R.new_ksk({0: key})
    dk = P.dev(key)
    for kind in ("qm1", "alt", "single"):
        m3 = adversarial_ct(P, kind, 3)
        o2 = P.out(2, P.k, P.n)
        P.ctx.relinearize(P.dev(m3), dk, o2, 1)
        eq(P.host(o2), R.ct_words(R.relinearize(R.new_ct(m3), rlk)), f"relinearize({kind}) with an all-(p-1) key")
    if P.ctx.using_batching:
        glk = R.new_ksk({1: key})
        a = adversarial_ct(P, "qm1")
        o2 = P.out(2, P.k, P.n)
        P.ctx.apply_galois(P.dev(a), 3, dk, o2, 1)
        eq(P.host(o2), R.ct_words(R.rotate_rows(R.new_ct(a), 1, glk)), "rotate_rows(qm1) with an all-(p-1) key")


def check_golden_appendix_b(be, g):
    """The library on the RNG-free App. B vectors against the unmodified reference's outputs stored in
    tests/golden/appendix_b.json (FNV-1a-64 of every output word; tests/golden/make_golden.py): no reference library needed."""
    n, moduli, t = g["n"], g["moduli"], g["t"]
    ctx = B200Context(n, moduli, t, lib=be.lib)
    k = ctx.k()
    assert k == g["k"]
    c = g["context"]
    li = ctx.level_info(ctx.first_level)
    assert li["parms_id"] == c["first_parms_id"] and ctx.level_info(0)["parms_id"] == c["key_parms_id"]
    assert li["gamma"] == c["gamma"] and li["delta"] == c["delta"]
    assert li["q_mod_t"] in (c["q_mod_t"] % t, c["q_mod_t"])
    assert li["roots"] == c["roots"][:k]
    inp = appendix_b_inputs(n, moduli, t)
    assert {name: "%016x" % fnv1a64(v) for name, v in inp.items()} == g["inputs"]
    H = lambda x: "%016x" % fnv1a64(be.to_host(x))
    a, b, p, rlk = (be.to_dev(inp[x]) for x in ("a", "b", "p", "rlk"))
    got = {}
    o2, o3 = be.empty((2, k, n)), be.empty((3, k, n))
    ctx.add(a, b, o2, 2, 1)
    got["add"] = H(o2)
    ctx.sub(a, b, o2, 2, 1)
    got["sub"] = H(o2)
    ctx.negate(a, o2, 2, 1)
    got["negate"] = H(o2)
    ctx.multiply(a, 2, b, 2, o3, 1)
    got["multiply"] = H(o3)
    ctx.relinearize(o3, rlk, o2, 1)
    got["relinearize"] = H(o2)
    ctx.multiply_relin(a, b, rlk, o2, 1)
    got["multiply_relin"] = H(o2)
    ctx.square(a, o3, 1)
    got["square"] = H(o3)
    ctx.multiply_plain(a, 2, p, 1, o2, 1)
    got["multiply_plain"] = H(o2)
    ctx.add_plain(a, 2, p, 1, o2, 1)
    got["add_plain"] = H(o2)
    ctx.sub_plain(a, 2, p, 1, o2, 1)
    got["sub_plain"] = H(o2)
    exp = dict(g["ops"], multiply_relin=g["ops"]["relinearize"])
    if k >= 2:
        om = be.empty((2, k - 1, n))
        ctx.mod_switch_to_next(a, 2, om, 1)
        got["mod_switch_to_next"] = H(om)
    if exp["rotate_rows_1"] is not None:
        assert ctx.galois_elt_from_step(1) == 3 and ctx.galois_elt_from_step(0) == 2 * n - 1
        ctx.apply_galois(a, 3, be.to_dev(inp["glk3"]), o2, 1)
        got["rotate_rows_1"] = H(o2)
        ctx.apply_galois(a, 2 * n - 1, be.to_dev(inp["glkc"]), o2, 1)
        got["rotate_columns"] = H(o2)
    else:
        got["rotate_rows_1"] = got["rotate_columns"] = None
    x = be.to_dev(inp["a"][0])
    ctx.ntt_forward(x, 1)
    got["ntt_a_p0_r0"] = "%016x" % fnv1a64(be.to_host(x)[0])
    assert got == {name: exp[name] for name in got}, {name: (got[name], exp[name]) for name in got if got[name] != exp[name]}
