#!/usr/bin/env python
"""Regenerates tests/golden/appendix_b.json from the UNMODIFIED reference (oracle/_ref/libsealc_ref.so).

Run where the reference sources exist and `make -C oracle ref` has built oracle/_ref/libsealc_ref.so:
    python tests/golden/make_golden.py
For every parameter set of tests/params.py it fills ciphertexts / plaintext / key-switching keys with the RNG-free
splitmix64 stream of SURVEY.md App. B, runs each Evaluator entry point of the reference through its C export layer
and records the FNV-1a-64 of the output words (plus the context constants that pin the host precompute), and the
per-prime hashes of the full-size forward NTT of BASELINE config 2 (config2_ntt.json).
It also writes tests/golden/small_n64.npz: full input/output words at n=64 (sec_level none) for a word-level fixture.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import refseal  # noqa: E402
from params import PARAMS  # noqa: E402


def golden_for(n, moduli, t, sec=refseal.SEC_TC128, full=False):
    R = refseal.RefContext(n, moduli, t, sec_level=sec)
    inp = refseal.appendix_b_inputs(n, moduli, t)
    H = lambda h: "%016x" % refseal.fnv1a64(R.ct_words(h))
    a, b, p = R.new_ct(inp["a"]), R.new_ct(inp["b"]), R.new_pt(inp["p"])
    rlk = R.new_ksk({0: inp["rlk"]})
    out = {"n": n, "moduli": [int(m) for m in moduli], "t": t, "k": R.k}
    ri, pi = R.rns_info(), R.plain_info()
    out["context"] = {"roots": [R.ref.ntt_root(m, n) for m in moduli], "m_sk": ri["m_sk"], "gamma": ri["gamma"],
                      "bsk": ri["bsk_primes"], "nB": ri["B"], "delta": pi["delta"], "q_mod_t": pi["upper_half_increment"][0],
                      "first_parms_id": list(R.first_parms_id), "key_parms_id": list(R.key_parms_id)}
    words = {}
    ops = {}

    def rec(name, h):
        ops[name] = H(h)
        if full:
            words[name] = R.ct_words(h)

    out["inputs"] = {kk: "%016x" % refseal.fnv1a64(v) for kk, v in inp.items()}
    rec("add", R.add(a, b))
    rec("sub", R.sub(a, b))
    rec("negate", R.negate(a))
    m = R.multiply(a, b)
    rec("multiply", m)
    rec("relinearize", R.relinearize(m, rlk))
    rec("square", R.square(a))
    rec("multiply_plain", R.multiply_plain(a, p))
    rec("add_plain", R.add_plain(a, p))
    rec("sub_plain", R.sub_plain(a, p))
    if R.k >= 2:
        rec("mod_switch_to_next", R.mod_switch_to_next(a))
    try:
        glk = R.new_ksk({1: inp["glk3"], (2 * n - 2) // 2: inp["glkc"]})
        rec("rotate_rows_1", R.rotate_rows(a, 1, glk))
        rec("rotate_columns", R.rotate_columns(a, glk))
    except refseal.SealError:
        ops["rotate_rows_1"] = None  # t does not support batching -> logic_error in the reference
        ops["rotate_columns"] = None
    ops["ntt_a_p0_r0"] = "%016x" % refseal.fnv1a64(R.ref.ntt_forward(moduli[0], inp["a"][0, 0]))
    out["ops"] = ops
    return out, inp, words


def config2_hashes():
    """BASELINE config 2: FNV-1a-64, per prime, of the reference's forward NTT of 4096 polynomials whose residues are the
    splitmix64(0xB200) % q_i stream of SURVEY.md App. B (tests/test_gpu_parity.py::test_config2_all_16384_transforms_vs_reference)."""
    R = refseal.RefLib.get()
    out = {}
    for name in ("n8192", "n8192_54"):
        n, moduli, _ = PARAMS[name]
        items, state, hashes = 4096, 0xB200, []
        for i in range(4):
            w, state = refseal.splitmix64_words(items * n, int(moduli[i]), state)
            hashes.append("%016x" % refseal.fnv1a64(R.ntt_forward_mt(int(moduli[i]), w.reshape(items, n), os.cpu_count() or 1)))
        out[name] = hashes
    return out


def main():
    res = {}
    for name, (n, moduli, t) in PARAMS.items():
        print("generating", name, flush=True)
        res[name], _, _ = golden_for(n, moduli, t)
    with open(os.path.join(HERE, "appendix_b.json"), "w") as f:
        json.dump(res, f, indent=1)
    with open(os.path.join(HERE, "config2_ntt.json"), "w") as f:
        json.dump(config2_hashes(), f, indent=1)
    # small word-level fixture: n=64, two 30-bit data primes + one special prime, t = 257 (batching-friendly: 257 = 1 mod 128)
    n, t = 64, 257
    P = refseal.RefLib.get()
    moduli = []
    cand = (1 << 30) - ((1 << 30) - 1) % 128
    v = ((1 << 30) - 1) // 128 * 128 + 1
    port_dir = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "libbfv_oracle.so")
    import ctypes as C
    orc = C.CDLL(port_dir)
    orc.orc_is_prime.argtypes = [C.c_uint64]
    while len(moduli) < 3:
        if orc.orc_is_prime(v):
            moduli.append(v)
        v -= 128
    g, inp, words = golden_for(n, moduli, t, sec=refseal.SEC_NONE, full=True)
    np.savez_compressed(os.path.join(HERE, "small_n64.npz"), moduli=np.array(moduli, dtype=np.uint64), t=np.uint64(t),
                        **{"in_" + k: v for k, v in inp.items()}, **{"out_" + k: v for k, v in words.items()})
    with open(os.path.join(HERE, "small_n64.json"), "w") as f:
        json.dump(g, f, indent=1)
    print("done")


if __name__ == "__main__":
    main()
