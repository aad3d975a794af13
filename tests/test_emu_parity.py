"""CPU-side parity: the product sources compiled in the test-only emulation mode (tests/emu) against the
unmodified reference, on the RNG-free vectors of SURVEY.md App. B.  Covers host precompute, constant folding,
strides and the orchestration of every layer-1 entry point; the CUDA build itself is covered by test_gpu_parity."""
import json
import os

import pytest

import parity_checks as pc
from backends import EmuBackend
from params import EDGE, PARAMS, PLAIN_EDGE

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "appendix_b.json")))


@pytest.fixture(scope="module", params=["n4096", "n8192", "n8192_54", "n8192_49"] + EDGE + [p for p in PLAIN_EDGE if PARAMS[p][0] <= 8192])
def pair(request, emu_lib, ref):
    return pc.pair_for(EmuBackend(emu_lib), request.param)


@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_54", "n8192_49"])
def test_golden_appendix_b(emu_lib, name):
    pc.check_golden_appendix_b(EmuBackend(emu_lib), GOLD[name])


def test_context_constants(pair):
    pc.check_context(pair)


def test_ntt(pair):
    pc.check_ntt(pair)


def test_elementwise(pair):
    pc.check_elementwise(pair)


def test_multiply_and_relinearize(pair):
    m3, rm = pc.check_multiply(pair)
    pc.check_relin(pair, m3, rm)


def test_galois(pair):
    pc.check_galois(pair)


def test_plain_ops(pair):
    pc.check_plain(pair)


def test_plain_operands(pair):
    if pair.n > 8192:
        pytest.skip("plain operand classes run on n <= 8192 only (emulation speed)")
    pc.check_plain_operands(pair)


def test_mod_switch(pair):
    pc.check_modswitch(pair)


def test_adversarial_operands(pair):
    pc.check_adversarial_multiply(pair, with_size5=pair.n <= 4096,
                                  pairs=None if pair.n <= 4096 else [("qm1", "qm1"), ("alt", "pm1"), ("single", "qm1")])
    pc.check_adversarial_keyswitch(pair)


def test_batch_strides(pair):
    if pair.n > 4096:
        pytest.skip("batch stride test runs on the smallest set only (emulation speed)")
    pc.check_batch(pair)


def test_host_buffer_pipeline(pair):
    if pair.n > 4096:
        pytest.skip("host pipeline test runs on the smallest set only (emulation speed)")
    pc.check_host_pipeline(pair)


def test_small_kernels(pair):
    if pair.n > 4096:
        pytest.skip("runs on the smallest set only (emulation speed)")
    pc.check_small_kernels(pair)


def test_noise_norm(pair):
    if pair.n > 4096:
        pytest.skip("noise norm test runs on the smallest set only (emulation speed)")
    pc.check_noise_norm(pair)


def test_noise_norm_edges(pair):
    if pair.n > 8192:
        pytest.skip("noise norm edges run on n <= 8192 only (emulation speed)")
    pc.check_noise_norm_edges(pair)


def test_decrypt(pair):
    if pair.n > 8192:
        pytest.skip("decryption checks run on n <= 8192 only (emulation speed)")
    pc.check_decrypt(pair)


def test_encrypted_roundtrip(pair):
    pc.check_encrypted_roundtrip(pair)


def test_n32768_two_level_transform(emu_lib, ref):
    """BASELINE config 5 parameters (n=32768, 15 data residues + special): the two-level NTT and K=15 kernels."""
    n, moduli, t = PARAMS["n32768"]
    P = pc.Pair(EmuBackend(emu_lib), n, moduli, t)
    pc.check_context(P)
    pc.check_ntt(P, items=1)
    m3, rm = pc.check_multiply(P, with_sizes=False)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_plain(P)
    pc.check_modswitch(P)


def test_wide_plain_modulus_auxiliary_base(emu_lib):
    """n16384_t60: with a 60-bit t, the FP64 auxiliary base (49-bit primes) clears the range condition
    32 + bits(t) + bits(Q) < bits(prod(B) * m_sk) by less than one prime's width at every level, so a count rule one prime
    short would fail check_context there; with t = 786433 the same base has 47 to 49 bits to spare."""
    import math
    from sunscreen_b200.lib import B200Context

    def spare_bits(name):
        n, moduli, t = PARAMS[name]
        ctx = B200Context(n, moduli, t, lib=emu_lib)
        out = []
        for lv in range(ctx.levels):
            li = ctx.level_info(lv)
            assert max(b.bit_length() for b in li["bsk"]) == 49
            out.append(math.prod(li["bsk"]).bit_length() - (32 + t.bit_length() + math.prod(li["q"]).bit_length()))
        return out

    assert all(0 < s < 48 for s in spare_bits("n16384_t60")), spare_bits("n16384_t60")
    assert all(s >= 47 for s in spare_bits("n16384")), spare_bits("n16384")


def test_layer1_argument_checks(emu_lib):
    """Every layer-1 entry point answers bad arguments (NULL pointers, a level that does not exist, sizes outside the
    supported range, a NULL context) with its error code instead of touching memory."""
    import ctypes as C
    import numpy as np
    from sunscreen_b200.lib import B200Context
    n, moduli, t = PARAMS["n4096"]
    ctx = B200Context(n, moduli, t, lib=emu_lib)
    L, h = emu_lib.lib, ctx.h
    vp, u64, ci = C.c_void_p, C.c_uint64, C.c_int
    k = ctx.k()
    buf = np.zeros((3, k + 1, n), dtype=np.uint64)
    p = vp(buf.ctypes.data)
    E_INVALID, E_NULL = -1, -4
    lv = ctx.first_level
    cases = [
        ("ntt_forward null data", L.b200_ntt_forward, (h, ci(lv), None, u64(1), None), E_NULL),
        ("ntt_forward bad level", L.b200_ntt_forward, (h, ci(99), p, u64(1), None), E_INVALID),
        ("ntt_inverse negative level", L.b200_ntt_inverse, (h, ci(-1), p, u64(1), None), E_INVALID),
        ("ntt_forward null ctx", L.b200_ntt_forward, (None, ci(lv), p, u64(1), None), E_NULL),
        ("add null", L.b200_add, (h, ci(lv), p, None, p, ci(2), u64(1), None), E_NULL),
        ("multiply size 0", L.b200_multiply, (h, ci(lv), p, ci(0), p, ci(2), p, u64(1), None), E_INVALID),
        ("multiply sizes 9 x 9", L.b200_multiply, (h, ci(lv), p, ci(9), p, ci(9), p, u64(1), None), E_INVALID),
        ("multiply null out", L.b200_multiply, (h, ci(lv), p, ci(2), p, ci(2), None, u64(1), None), E_NULL),
        ("square bad level", L.b200_square, (h, ci(7), p, p, u64(1), None), E_INVALID),
        ("relinearize null key", L.b200_relinearize, (h, ci(lv), p, None, p, u64(1), None), E_NULL),
        ("multiply_relin null", L.b200_multiply_relin, (h, ci(lv), p, p, None, p, u64(1), None), E_NULL),
        ("apply_galois even element", L.b200_apply_galois, (h, ci(lv), p, C.c_uint32(4), p, p, u64(1), None), E_INVALID),
        ("apply_galois element too large", L.b200_apply_galois, (h, ci(lv), p, C.c_uint32(2 * n + 1), p, p, u64(1), None), E_INVALID),
        ("multiply_plain null plain", L.b200_multiply_plain, (h, ci(lv), p, ci(2), None, u64(1), p, u64(1), None), E_NULL),
        ("add_plain plain_batch mismatch", L.b200_add_plain, (h, ci(lv), p, ci(2), p, u64(3), p, u64(2), None), E_INVALID),
        ("mod_switch at the last level", L.b200_mod_switch_to_next, (h, ci(ctx.levels - 1), p, ci(2), p, u64(1), None), E_INVALID),
        ("decrypt null", L.b200_decrypt, (h, ci(lv), p, ci(2), None, p, u64(1), None), E_NULL),
        ("decrypt size 1", L.b200_decrypt, (h, ci(lv), p, ci(1), p, p, u64(1), None), E_INVALID),
        ("ct_sk_phase size 1", L.b200_ct_sk_phase, (h, ci(lv), p, ci(1), p, p, u64(1), None), E_INVALID),
        ("noise_norm null key", L.b200_noise_norm, (h, ci(lv), p, ci(2), None, p, ci(k + 1), u64(1), None), E_NULL),
        ("multiply_relin_host null", L.b200_multiply_relin_host, (h, ci(lv), None, p, p, p, u64(1)), E_NULL),
        ("level_info bad level", L.b200_ctx_level_info, (h, ci(50), p), E_INVALID),
        ("galois_elt_from_step too large", L.b200_galois_elt_from_step, (h, ci(n), p), E_INVALID),
    ]
    wrong = []
    for label, fn, args, want in cases:
        fn.restype = C.c_int
        fn.argtypes = None
        got = fn(*args)
        if got != want:
            wrong.append((label, got, want))
    assert not wrong, wrong
    # zero-sized batches are no-ops
    for fn, args in ((L.b200_ntt_forward, (h, ci(lv), p, u64(0), None)), (L.b200_multiply, (h, ci(lv), p, ci(2), p, ci(2), p, u64(0), None)),
                     (L.b200_multiply_relin, (h, ci(lv), p, p, p, p, u64(0), None))):
        fn.restype = C.c_int
        assert fn(*args) == 0


def test_n8192_with_the_reference_auxiliary_base(emu_lib, ref, monkeypatch):
    """The all-FP64 default chain with the reference's 61-bit auxiliary base (read when the context is created): the BEHZ
    jobs then mix FP64 data primes with integer-path auxiliary primes."""
    monkeypatch.setenv("B200_FORCE_AUX61", "1")
    P = pc.Pair(EmuBackend(emu_lib), *PARAMS["n8192"])
    assert P.ctx.level_info(P.ctx.first_level)["m_sk"] == P.ref.rns_info()["m_sk"]
    pc.check_context(P)
    pc.check_ntt(P)
    m3, rm = pc.check_multiply(P)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_adversarial_multiply(P, with_size5=False, pairs=[("qm1", "qm1"), ("alt", "pm1")])
    pc.check_adversarial_keyswitch(P)
