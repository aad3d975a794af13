"""Word-for-word parity checks of the B200 path against the unmodified reference (shared by CPU-emu and GPU tests)."""
import numpy as np

from refseal import RefContext, appendix_b_inputs, fnv1a64
from sunscreen_b200.lib import B200Context


class Pair:
    """Same parameters instantiated on the reference and on the B200 library."""

    def __init__(self, be, n, moduli, t):
        self.be = be
        self.n, self.moduli, self.t = n, list(moduli), t
        self.ref = RefContext(n, moduli, t)
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


def check_context(P):
    li = P.ctx.level_info(P.ctx.first_level)
    ri = P.ref.rns_info()
    assert li["parms_id"] == list(P.ref.first_parms_id)
    assert P.ctx.level_info(0)["parms_id"] == list(P.ref.key_parms_id)
    assert li["gamma"] == ri["gamma"]
    if li["m_sk"] == ri["m_sk"]:
        # the reference's own auxiliary base (61-bit primes)
        assert li["bsk"] == ri["bsk_primes"] and (li["nB"], li["nBsk"]) == (ri["B"], ri["Bsk"])
    else:
        # FP64-friendly auxiliary base: 47..49-bit NTT primes (as wide as the widest user prime), distinct from the user's
        # primes, with at least the reference's dynamic range condition
        # 32 + bits(t) + bits(Q) < bits(prod(B) * m_sk)   (S/util/rns.cpp:617-624); results are base-independent.
        import math
        width = max(47, max(int(m).bit_length() for m in P.moduli))
        assert width <= 49
        assert all(p < (1 << width) and p % (2 * P.n) == 1 for p in li["bsk"]) and len(set(li["bsk"])) == len(li["bsk"])
        assert not set(li["bsk"]) & set(int(m) for m in P.moduli)
        Q = math.prod(li["q"])
        assert math.prod(li["bsk"]).bit_length() > 32 + P.t.bit_length() + Q.bit_length()
    pi = P.ref.plain_info()
    assert li["delta"] == pi["delta"]
    assert li["q_mod_t"] == pi["upper_half_increment"][0] % P.t or li["q_mod_t"] == pi["upper_half_increment"][0]
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
    mono[5] = 7
    rm = P.ref.new_pt(mono[:6])
    P.ctx.multiply_plain(da, 2, P.dev(mono), 1, o2, 1)
    eq(P.host(o2), P.ref.ct_words(P.ref.multiply_plain(ra, rm)), "multiply_plain(monomial)")


def check_modswitch(P):
    a = P.inp["a"]
    if P.k < 2:
        return
    ra = P.ref.new_ct(a)
    o = P.out(2, P.k - 1, P.n)
    P.ctx.mod_switch_to_next(P.dev(a), 2, o, 1)
    eq(P.host(o), P.ref.ct_words(P.ref.mod_switch_to_next(ra)), "mod_switch_to_next")


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
    """x * y in Z_t[X] / (X^n + 1), coefficients of x, y below t < 2^20 (exact in int64 for n <= 32768)."""
    n = x.size
    c = np.convolve(x.astype(np.int64), y.astype(np.int64))
    c = np.concatenate([c, np.zeros(1, dtype=np.int64)])
    return ((c[:n] % t - c[n:] % t) % t).astype(np.uint64)


def check_encrypted_roundtrip(P, seed=3):
    """Real keys + fresh encryptions from the reference; our multiply+relin output decrypts on the reference to the
    product of the messages (slot-wise for a batching plain modulus, else the negacyclic product of coefficient
    plaintexts), and equals the reference's ciphertext word for word."""
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


def check_noise_norm(P, batch=3, seed=23):
    """b200_noise_norm (the quantity behind invariant_noise_budget, S/decryptor.cpp:424-485): for random ciphertexts of
    size 2 and 3 and random key powers, the device's multi-precision infinity norm of the centred t * phase mod Q equals
    the same computed with Python integers from the phase words."""
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
        phase = P.host(ph).reshape(batch, P.k, P.n)
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
