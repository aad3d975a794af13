"""The parameter table itself: every chain is a list of distinct primes = 1 mod 2n, and each edge chain is exactly what
CoeffModulus::Create(n, bits) returns (the reference's prime search, restated here; compared with the reference library
itself where it is built)."""
import ctypes as C
import math

import pytest

from params import EDGE, EDGE_BITS, LONG, LONG_BITS, PARAMS, PLAIN_EDGE, PLAIN_EDGE_T, SEC_NONE, WIDE, WIDE_BITS


def is_prime(v):
    """Deterministic Miller-Rabin for v < 2^64."""
    if v < 2:
        return False
    bases = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    for p in bases:
        if v % p == 0:
            return v == p
    d, s = v - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in bases:
        x = pow(a, d, v)
        if x in (1, v - 1):
            continue
        for _ in range(s - 1):
            x = x * x % v
            if x == v - 1:
                break
        else:
            return False
    return True


def create_coeff_modulus(n, bit_sizes):
    """CoeffModulus::Create: per width, the `count` largest primes = 1 mod 2n below 2^width, descending; the requested
    widths are then served in order, each taking the SMALLEST prime left of its width."""
    table = {}
    for bits in set(bit_sizes):
        count, found = bit_sizes.count(bits), []
        v = ((1 << bits) - 1) // (2 * n) * (2 * n) + 1
        while count and v > 1 << (bits - 1):
            if is_prime(v):
                found.append(v)
                count -= 1
            v -= 2 * n
        table[bits] = found
    return [table[bits].pop() for bits in bit_sizes]


@pytest.mark.parametrize("name", sorted(PARAMS))
def test_chain_primes(name):
    n, moduli, t = PARAMS[name]
    assert len(set(moduli)) == len(moduli) >= 2
    for q in moduli:
        assert is_prime(q) and q % (2 * n) == 1 and q.bit_length() <= 60, hex(q)
    assert t < 1 << 60 and t not in moduli


@pytest.mark.parametrize("name", EDGE)
def test_edge_chain_is_create_output(name):
    n, bits = EDGE_BITS[name]
    _, moduli, _ = PARAMS[name]
    assert [q.bit_length() for q in moduli] == bits
    assert moduli == create_coeff_modulus(n, bits)


def test_edge_chains_reach_their_cases():
    """What each edge chain is there for (host_ctx.cpp: FP64 primes are <= 49 bits; fast plain lift needs every data prime
    above t; batching needs t prime and = 1 mod 2n)."""
    fp = lambda q: q.bit_length() <= 49
    n, m, t = PARAMS["n8192_sealfhe"]
    assert t == 1032193 and any(map(fp, m)) and not all(map(fp, m))
    n, m, t = PARAMS["n16384_mixed"]
    assert {q.bit_length() for q in m[:-1]} >= {48, 49, 50}
    n, m, t = PARAMS["n4096_narrow"]
    assert all(q.bit_length() <= 22 for q in m) and t < min(m) and is_prime(t) and t % (2 * n) == 1
    n, m, t = PARAMS["n4096_q_below_t"]
    assert min(m[:-1]) < t < max(m[:-1]) and is_prime(t) and t % (2 * n) == 1
    assert all(q.bit_length() == 60 for q in PARAMS["n8192_60"][1])
    assert all(q.bit_length() == 50 for q in PARAMS["n8192_50"][1])
    for name, logn in (("n2048_2x27", 11), ("n1024_2x27", 10)):
        n, m, t = PARAMS[name]
        assert n == 1 << logn and len(m) == 2 and t % (2 * n) == 1


@pytest.mark.parametrize("name", LONG)
def test_long_chain_is_create_output(name):
    n, bits = LONG_BITS[name]
    _, moduli, t = PARAMS[name]
    assert [q.bit_length() for q in moduli] == bits
    assert moduli == create_coeff_modulus(n, bits)
    assert t == {4096: 262144, 8192: 1032193, 16384: 786433}[n]     # the default plain modulus of each n


def test_long_chains_reach_their_cases():
    """What each long chain is there for (host_ctx.h: FP64 primes are <= 49 bits; the auxiliary base is as wide as the
    widest user prime, at least 47 bits; b200_bfv.cu: the key-switch cluster runs 2 <= k <= 8 at logn 12 and 13)."""
    assert all(q.bit_length() <= 49 for name in LONG for q in PARAMS[name][1])
    for name, logn in (("n8192_9x24", 13), ("n4096_9x22", 12)):
        n, m, t = PARAMS[name]
        assert n == 1 << logn and len(m) - 1 == 8                      # data levels k = 8 ... 1
    n, m, t = PARAMS["n8192_mixed_fp"]
    assert m[-1] < min(m[:-1]) and max(q.bit_length() for q in m) == 49 and len({q.bit_length() for q in m[:-1]}) == 3
    # the 20-bit prime Create would hand out as the special prime is the default t itself
    assert create_coeff_modulus(n, [20]) == [t]
    for name, widest in (("n16384_17x25", 25), ("n16384_49_16x24", 49)):
        n, m, t = PARAMS[name]
        assert len(m) - 1 == 16 and max(q.bit_length() for q in m) == widest


@pytest.mark.parametrize("name", WIDE)
def test_wide_chain_is_create_output(name):
    n, bits = WIDE_BITS[name]
    _, moduli, t = PARAMS[name]
    assert [q.bit_length() for q in moduli] == bits
    assert moduli == create_coeff_modulus(n, bits)
    assert t == {16384: 786433, 32768: 786433}[n]                 # the default plain modulus of each n


def test_wide_chains_reach_their_cases():
    """What each wide chain is there for (host_ctx.h: FP64 primes are <= 49 bits, and the auxiliary base is then as wide as
    the widest user prime, at least 47 bits, with enough primes that bits(prod(B) m_sk) > 32 + bits(t) + bits(Q); b200_bfv.cu:
    the k-templated kernels take at most 16 data residues, modswitch_kernel 17 at the key level)."""
    bits = lambda q: math.prod(q).bit_length()
    widths = lambda name: {q.bit_length() for q in PARAMS[name][1]}
    assert all(PARAMS[name][0] == 32768 for name in WIDE if name != "n16384_24x18")
    assert widths("n32768_60x6") == {60}
    assert widths("n32768_30x5") == {30}
    n, m, t = PARAMS["n32768_mixed"]
    assert [q.bit_length() for q in m] == [60, 30, 30, 30, 60] and m[0] < m[-1]        # the special prime is the widest
    # n32768_30x5: k 47-bit primes (k - 1 in B, and m_sk) already cover the first data level's range, so nB < k (asserted on
    # the library's own base by tests/test_gpu_wide_chains.py)
    n, m, t = PARAMS["n32768_30x5"]
    k = len(m) - 1
    assert 46 * k > 33 + t.bit_length() + bits(m[:k])
    # the 17-prime key levels: 16 data residues
    for name in ("n16384_17x25", "n16384_49_16x24", "n32768_49x17"):
        assert len(PARAMS[name][1]) == 17, name
    assert widths("n32768_49x17") == {49}
    # beyond the limit: 17 data residues, and still within 128-bit security at n = 16384 (438 bits)
    n, m, t = PARAMS["n16384_24x18"]
    assert len(m) - 1 == 17 and bits(m) <= 438 and sum(q.bit_length() for q in m) == 432


@pytest.mark.parametrize("name", WIDE)
def test_wide_chain_matches_reference_create(ref, name):
    reference_create_matches(ref, name, *WIDE_BITS[name])


def batching_plain_modulus(n, bits, skip=()):
    """PlainModulus::Batching(n, bits) = CoeffModulus::Create(n, {bits})[0], the largest prime = 1 mod 2n below 2^bits;
    with `skip`, the largest such prime not in it."""
    return max(p for p in create_coeff_modulus(n, [bits] * (len(skip) + 1)) if p not in skip)


@pytest.mark.parametrize("name", PLAIN_EDGE)
def test_plain_edge_modulus(name):
    base, rule = PLAIN_EDGE_T[name]
    n, moduli, t = PARAMS[name]
    assert (n, moduli) == PARAMS[base][:2]
    if isinstance(rule, tuple):
        assert rule[0] == "batching" and t.bit_length() == rule[1]
        assert t == batching_plain_modulus(n, rule[1], skip=moduli)
        assert is_prime(t) and t % (2 * n) == 1
    else:
        assert t == rule


def test_plain_edge_sets_reach_their_cases():
    """What each wide plain modulus is there for."""
    bits = lambda q: math.prod(q).bit_length()
    n, m, t = PARAMS["n8192_t47"]
    assert t == batching_plain_modulus(n, 47)      # the first candidate of the 47-bit FP64 auxiliary base
    assert max(q.bit_length() for q in m) < 47
    n, m, t = PARAMS["n8192_60_t60"]
    assert batching_plain_modulus(n, 60) in m and t not in m and all(q > t for q in m)
    n, m, t = PARAMS["n8192_54_t60"]
    k = len(m) - 1                                  # first data level: the reference's rule adds a B prime
    assert 32 + t.bit_length() + bits(m[:k]) >= 61 * k + 61
    assert PARAMS["n8192_t3p37"][2] % 2 == 1 and not is_prime(PARAMS["n8192_t3p37"][2])
    # the widest plain modulus the FP64 transform takes (host_ctx.h FP_PRIME_BITS; the kernel choice itself is asserted by
    # test_gpu_launch_shapes.py::test_plain_ntt_fp64_width_limit)
    assert PARAMS["n8192_t49"][2].bit_length() == 49
    # a 60-bit t on a chain whose primes all take the FP64 path (the auxiliary base's range margin is asserted by
    # test_emu_parity.py::test_wide_plain_modulus_auxiliary_base)
    n, m, t = PARAMS["n16384_t60"]
    assert t.bit_length() == 60 and max(q.bit_length() for q in m) == 49


@pytest.mark.parametrize("name", PLAIN_EDGE)
def test_plain_edge_matches_reference(ref, name):
    """The reference's own prime search gives the same batching t, and it accepts the set at 128-bit security."""
    import refseal
    base, rule = PLAIN_EDGE_T[name]
    n, moduli, t = PARAMS[name]
    if isinstance(rule, tuple):
        count = len(moduli) + 1
        arr = (C.c_int * count)(*([rule[1]] * count))
        out = (C.c_void_p * count)()
        ref.call("CoeffModulus_Create1", C.c_uint64(n), C.c_uint64(count), arr, out)
        got = []
        for h in out:
            v = C.c_uint64()
            ref.call("Modulus_Value", C.c_void_p(h), C.byref(v))
            got.append(v.value)
        assert t == max(p for p in got if p not in moduli)
    refseal.RefContext(n, moduli, t)


@pytest.mark.parametrize("name", LONG)
def test_long_chain_matches_reference_create(ref, name):
    reference_create_matches(ref, name, *LONG_BITS[name])


@pytest.mark.parametrize("name", EDGE)
def test_edge_chain_matches_reference_create(ref, name):
    reference_create_matches(ref, name, *EDGE_BITS[name])


def reference_create_matches(ref, name, n, bits):
    import refseal
    arr = (C.c_int * len(bits))(*bits)
    out = (C.c_void_p * len(bits))()
    ref.call("CoeffModulus_Create1", C.c_uint64(n), C.c_uint64(len(bits)), arr, out)
    got = []
    for h in out:
        v = C.c_uint64()
        ref.call("Modulus_Value", C.c_void_p(h), C.byref(v))
        got.append(v.value)
    assert got == PARAMS[name][1]
    # and the reference accepts the whole set, at 128-bit security unless the set is marked otherwise
    sec = refseal.SEC_NONE if name in SEC_NONE else refseal.SEC_TC128
    refseal.RefContext(n, PARAMS[name][1], PARAMS[name][2], sec)
    if name in SEC_NONE:
        with pytest.raises(ValueError):
            refseal.RefContext(n, PARAMS[name][1], PARAMS[name][2])
