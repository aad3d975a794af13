"""Slots in and out on one GPU at n = 8192 (the BFVDefault chain, t = 1032193, a 20-bit batching prime): each batched route
against the per-handle route it replaces, alternated in one process over five rounds (medians reported, host clock around
calls that return after completion):
  encode     B200_BatchEncoder_EncodeBatch of 4096 vectors  vs  4096 BatchEncoder_Encode1;
  decode     B200_BatchEncoder_DecodeBatch of 4096 plaintexts  vs  4096 BatchEncoder_Decode1;
  decrypt    B200_Decryptor_DecryptSlotsBatch of 1024 ciphertexts with budgets  vs  InvariantNoiseBudget + Decrypt + Decode1
             per ciphertext;
  diagonals  one linear_transform diagonal set (b = G = 64: 4096 slot vectors) as b200_batch_encode -> b200_plain_to_ntt on
             the device  vs  4096 BatchEncoder_Encode1 then the existing lift (one upload and b200_plain_to_ntt).
Each pair must give identical words.  Also the reference's per-handle CPU time per item (oracle/_ref, when built), and the GPU
name, power limit and SM clock.  Any number not taken is reported as "not measured".

    python tools/slots_probe.py
"""
import ctypes as C
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from params import PARAMS  # noqa: E402
from sealc_driver import Sealc  # noqa: E402
from sunscreen_b200.lib import PLAIN_NTT_MULTIPLY, B200Context, B200Lib  # noqa: E402

vp, u64 = C.c_void_p, C.c_uint64
ROUNDS = 5


def median_pair(a, b, rounds=ROUNDS):
    """alternate the two routes (one warm-up call each), returning (median, min, max) seconds of each"""
    a()
    b()
    ta, tb = [], []
    for _ in range(rounds):
        for fn, acc in ((a, ta), (b, tb)):
            t0 = time.perf_counter()
            fn()
            acc.append(time.perf_counter() - t0)
    return [(sorted(x)[len(x) // 2], min(x), max(x)) for x in (ta, tb)]


def report(case, items, batched, per_handle, same):
    (mb, lb, hb), (mp, lp, hp) = batched, per_handle
    print(f"{case} ({items} items): batched {mb * 1e3:.2f} ms (range {lb * 1e3:.2f}-{hb * 1e3:.2f})  per-handle {mp * 1e3:.2f} ms "
          f"(range {lp * 1e3:.2f}-{hp * 1e3:.2f})  per-handle/batched {mp / mb:.1f}x  words identical: {same}", flush=True)


def arr(hs):
    return (vp * len(hs))(*hs)


def reference_times(n, moduli, t, rng):
    """per-item CPU time of the reference's per-handle calls, or None when the reference library was not built"""
    import refseal
    if not refseal.have_ref():
        return None
    R = refseal.RefContext(n, moduli, t)
    kg = R.keygen()
    enc, dec, be = R.encryptor(R.public_key(kg)), R.decryptor(R.secret_key(kg)), R.batch_encoder()
    vals = [rng.integers(0, t, size=n, dtype=np.uint64) for _ in range(64)]
    t0 = time.perf_counter()
    pts = [R.batch_encode(be, v) for v in vals]
    t_enc = (time.perf_counter() - t0) / len(vals)
    t0 = time.perf_counter()
    for p in pts:
        R.batch_decode(be, p)
    t_dec = (time.perf_counter() - t0) / len(pts)
    cts = [R.encrypt(enc, p) for p in pts[:32]]
    t0 = time.perf_counter()
    for c in cts:
        R.noise_budget(dec, c)
        R.batch_decode(be, R.decrypt(dec, c))
    t_dcr = (time.perf_counter() - t0) / len(cts)
    return t_enc, t_dec, t_dcr


def main():
    assert torch.cuda.is_available(), "slots_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip().replace("\n", " | ")
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q}", flush=True)
    n, moduli, t = PARAMS["n8192"]
    rng = np.random.default_rng(7)
    S = Sealc(B200Lib.default().lib)
    O = S.context(n, moduli, t)
    be = vp()
    S.call("BatchEncoder_Create", O.ctx, C.byref(be))
    ok = True

    # ---- encode 4096 vectors ----
    E = 4096
    vals = rng.integers(0, t, size=(E, n), dtype=np.uint64)
    pb = []
    for _ in range(E):
        h = vp()
        S.call("Plaintext_Create1", None, C.byref(h))
        pb.append(h)
    ph = []
    for _ in range(E):
        h = vp()
        S.call("Plaintext_Create1", None, C.byref(h))
        ph.append(h)
    pb_arr = arr(pb)
    vptr = vals.ctypes.data_as(C.POINTER(u64))

    def enc_batched():
        S.call("B200_BatchEncoder_EncodeBatch", be, u64(E), u64(n), vptr, C.c_bool(False), pb_arr)

    def enc_per_handle():
        for i in range(E):
            S.call("BatchEncoder_Encode1", be, u64(n), vals[i].ctypes.data_as(C.POINTER(u64)), ph[i])

    tb, tp = median_pair(enc_batched, enc_per_handle)
    sb, sp = np.zeros((E, n), dtype=np.uint64), np.zeros((E, n), dtype=np.uint64)
    S.call("B200_BatchEncoder_DecodeBatch", be, u64(E), pb_arr, C.c_bool(False), sb.ctypes.data_as(C.c_void_p))
    S.call("B200_BatchEncoder_DecodeBatch", be, u64(E), arr(ph), C.c_bool(False), sp.ctypes.data_as(C.c_void_p))
    same = np.array_equal(sb, sp) and np.array_equal(sb, vals)
    ok &= same
    report("encode", E, tb, tp, same)

    # ---- decode 4096 plaintexts ----
    out_b = np.zeros((E, n), dtype=np.uint64)
    out_p = np.zeros((E, n), dtype=np.uint64)
    cnt = u64()

    def dec_batched():
        S.call("B200_BatchEncoder_DecodeBatch", be, u64(E), pb_arr, C.c_bool(False), out_b.ctypes.data_as(C.c_void_p))

    def dec_per_handle():
        for i in range(E):
            S.call("BatchEncoder_Decode1", be, pb[i], C.byref(cnt), out_p[i].ctypes.data_as(C.c_void_p), None)

    tb, tp = median_pair(dec_batched, dec_per_handle)
    same = np.array_equal(out_b, out_p)
    ok &= same
    report("decode", E, tb, tp, same)

    # ---- decrypt 1024 ciphertexts to slots with budgets ----
    D = 1024
    k = O.k
    sk = np.stack([rng.integers(0, m, size=n, dtype=np.uint64) for m in moduli])
    dec = O.decryptor(sk)
    cts = []
    for _ in range(D):
        w = np.stack([np.stack([rng.integers(0, m, size=n, dtype=np.uint64) for m in moduli[:k]]) for _ in range(2)])
        cts.append(O.new_ct(w))
    cts_arr = arr(cts)
    slots_b, slots_p = np.zeros((D, n), dtype=np.uint64), np.zeros((D, n), dtype=np.uint64)
    bud_b, bud_p = (C.c_int * D)(), [0] * D

    def dcr_batched():
        S.call("B200_Decryptor_DecryptSlotsBatch", dec, be, u64(D), cts_arr, C.c_bool(False), slots_b.ctypes.data_as(C.c_void_p), bud_b)

    pt = vp()
    S.call("Plaintext_Create1", None, C.byref(pt))

    def dcr_per_handle():
        b = C.c_int()
        for i in range(D):
            S.call("Decryptor_InvariantNoiseBudget", dec, cts[i], C.byref(b))
            bud_p[i] = b.value
            S.call("Decryptor_Decrypt", dec, cts[i], pt)
            S.call("BatchEncoder_Decode1", be, pt, C.byref(cnt), slots_p[i].ctypes.data_as(C.c_void_p), None)

    tb, tp = median_pair(dcr_batched, dcr_per_handle)
    same = np.array_equal(slots_b, slots_p) and list(bud_b) == bud_p
    ok &= same
    report("decrypt to slots + budget", D, tb, tp, same)

    # ---- one linear_transform diagonal set, b = G = 64 ----
    ctx = B200Context(n, moduli, t)
    kk = ctx.k()
    G = b = 64
    vecs = rng.integers(0, t, size=(G * b, n), dtype=np.uint64)
    dv = torch.from_numpy(vecs.view(np.int64)).cuda()
    coeffs = torch.empty((G * b, n), dtype=torch.int64, device="cuda")
    pn_b = torch.empty((G, b, kk, n), dtype=torch.int64, device="cuda")
    pn_p = torch.empty((G, b, kk, n), dtype=torch.int64, device="cuda")
    host = torch.empty((G * b, n), dtype=torch.int64).pin_memory()
    dhost = torch.empty((G * b, n), dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def diag_batched():
        ctx.batch_encode(dv, n, coeffs, G * b, stream=s)
        ctx.plain_to_ntt(coeffs, G * b, pn_b, rule=PLAIN_NTT_MULTIPLY, stream=s)
        torch.cuda.synchronize()

    def diag_per_handle():
        for i in range(G * b):
            S.call("BatchEncoder_Encode1", be, u64(n), vecs[i].ctypes.data_as(C.POINTER(u64)), ph[i])
        # the existing lift: the encoded coefficients (identical words: checked below) uploaded once and lifted
        dhost.copy_(host, non_blocking=True)
        ctx.plain_to_ntt(dhost, G * b, pn_p, rule=PLAIN_NTT_MULTIPLY, stream=s)
        torch.cuda.synchronize()

    diag_batched()
    host.copy_(coeffs.cpu())
    tb, tp = median_pair(diag_batched, diag_per_handle)
    same = torch.equal(pn_b, pn_p)
    for i in (0, G * b - 1):  # the per-handle plaintexts' own words against the device encode
        c = np.zeros(n, dtype=np.uint64)
        v = u64()
        for j in range(n):
            S.call("Plaintext_CoeffAt", ph[i], u64(j), C.byref(v))
            c[j] = v.value
        same &= np.array_equal(c, host[i].numpy().view(np.uint64))
    ok &= bool(same)
    report("diagonals encode -> plain_to_ntt", G * b, tb, tp, bool(same))

    ref = reference_times(n, moduli, t, rng)
    if ref is None:
        print("reference per-handle CPU time: not measured (oracle/_ref not built)")
    else:
        te, td, tr = ref
        print(f"reference per-handle CPU time per item: encode {te * 1e6:.1f} us, decode {td * 1e6:.1f} us, "
              f"InvariantNoiseBudget + Decrypt + Decode {tr * 1e6:.1f} us  (x4096 / x4096 / x1024: "
              f"{te * 4096 * 1e3:.1f} / {td * 4096 * 1e3:.1f} / {tr * 1024 * 1e3:.1f} ms)")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
