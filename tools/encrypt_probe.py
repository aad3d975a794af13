"""Batched encryption on one GPU at n = 8192 (the BFVDefault chain, t = 1032193): for 1, 64 and 1024 items,
  EncryptBatch      B200_Encryptor_EncryptBatch of encoded plaintexts (pk)
  EncryptSlotsBatch B200_Encryptor_EncryptSlotsBatch of slot vectors (pk)
against the per-handle route BatchEncoder_Encode1 + Encryptor_Encrypt per item, the routes alternated in one process over five
rounds (medians reported; host clock around calls that return after completion).  Seeded runs of both batched seams must give
the words of Encode1 + B200_Encryptor_EncryptSetSeed.  The split between host sampling and GPU work of one EncryptBatch call
is taken two ways: the host sampling step on its own clock (b200_sample_pk for the same items), and the call's kernels and copies
summed from a torch.profiler pass.  Concurrency: eight threads each encrypting items one by one (Encryptor_Encrypt), and the
latency of Evaluator_Multiply on another thread, idle and while a 1024-item encryption runs (EncryptBatch; with a library that
has no batch seam, eight threads of per-handle calls).  Also the reference's per-call CPU time (oracle/_ref, when built), and the
GPU name, power limit and SM clock.

    python tools/encrypt_probe.py [--lib other/libb200bfv.so]   (--lib: another build, e.g. an older one: per-handle and
                                                                  concurrency parts only when it lacks the batch seams)
"""
import argparse
import ctypes as C
import os
import threading
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
from sunscreen_b200.lib import B200Context, B200Lib  # noqa: E402

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


def arr(hs):
    return (vp * len(hs))(*hs)


def gpu_split(call):
    """(wall seconds, GPU seconds) of one call: kernels and copies summed from a torch.profiler pass"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        call()
        wall = time.perf_counter() - t0
    gpu_us = sum(e.device_time_total for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return wall, gpu_us * 1e-6


def reference_time(n, moduli, t, rng, items=32):
    """per-item CPU time of the reference's BatchEncoder_Encode1 + Encryptor_Encrypt, or None without oracle/_ref"""
    import refseal
    if not refseal.have_ref():
        return None
    R = refseal.RefContext(n, moduli, t)
    kg = R.keygen()
    enc, be = R.encryptor(R.public_key(kg)), R.batch_encoder()
    vals = [rng.integers(0, t, size=n, dtype=np.uint64) for _ in range(items)]
    R.encrypt(enc, R.batch_encode(be, vals[0]))
    t0 = time.perf_counter()
    for v in vals:
        R.encrypt(enc, R.batch_encode(be, v))
    return (time.perf_counter() - t0) / items


def concurrency(S, O, enc, be, n, t, rng, batched):
    """items/s of 8 threads x 32 per-handle encryptions; Evaluator_Multiply latency idle and during a 1024-item encryption"""
    T, M, BIG = 8, 32, 1024
    vals = rng.integers(0, t, size=n, dtype=np.uint64)
    pt = vp()
    S.call("Plaintext_Create1", None, C.byref(pt))
    S.call("BatchEncoder_Encode1", be, u64(n), vals.ctypes.data_as(C.POINTER(u64)), pt)

    def encrypt_many(m):
        h = vp()
        S.call("Ciphertext_Create1", None, C.byref(h))
        for _ in range(m):
            S.call("Encryptor_Encrypt", enc, pt, h, None)

    encrypt_many(2)
    th = [threading.Thread(target=encrypt_many, args=(M,)) for _ in range(T)]
    t0 = time.perf_counter()
    for x in th:
        x.start()
    for x in th:
        x.join()
    rate = T * M / (time.perf_counter() - t0)
    a, d = vp(), vp()
    S.call("Ciphertext_Create1", None, C.byref(a))
    S.call("Encryptor_Encrypt", enc, pt, a, None)
    S.call("Ciphertext_Create1", None, C.byref(d))

    def mul_latencies(stop=None, count=50):
        lat = []
        while (stop is None and len(lat) < count) or (stop is not None and not stop.is_set()):
            t1 = time.perf_counter()
            S.call("Evaluator_Multiply", O.ev, a, a, d, None)
            lat.append(time.perf_counter() - t1)
        return lat

    mul_latencies(count=5)
    idle = mul_latencies()
    pts = [pt] * BIG
    cts = []
    for _ in range(BIG):
        h = vp()
        S.call("Ciphertext_Create1", None, C.byref(h))
        cts.append(h)
    if batched:
        big = lambda: S.call("B200_Encryptor_EncryptBatch", enc, u64(BIG), arr(pts), None, C.c_bool(False), arr(cts))
    else:
        def big():
            ws = [threading.Thread(target=encrypt_many, args=(BIG // T,)) for _ in range(T)]
            for x in ws:
                x.start()
            for x in ws:
                x.join()
    stop = threading.Event()
    busy = []
    m = threading.Thread(target=lambda: busy.extend(mul_latencies(stop)))
    m.start()
    t0 = time.perf_counter()
    big()
    tbig = time.perf_counter() - t0
    stop.set()
    m.join()
    med = lambda x: sorted(x)[len(x) // 2] * 1e3
    print(f"concurrency: {T} threads x {M} per-handle Encryptor_Encrypt {rate:.0f} items/s;  Evaluator_Multiply latency idle "
          f"median {med(idle):.3f} ms, during a {BIG}-item encryption ({'EncryptBatch' if batched else f'{T} threads of Encrypt'}, "
          f"{tbig * 1e3:.0f} ms) median {med(busy):.3f} ms, max {max(busy) * 1e3:.2f} ms over {len(busy)} calls", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="another build of libb200bfv.so to measure instead of this tree's")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "encrypt_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip().replace("\n", " | ")
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q} | host CPUs: {os.cpu_count()}", flush=True)
    n, moduli, t = PARAMS["n8192"]
    rng = np.random.default_rng(9)
    lib = C.CDLL(os.path.abspath(args.lib), mode=os.RTLD_LOCAL) if args.lib else B200Lib.default().lib
    S = Sealc(lib)
    batched = hasattr(lib, "B200_Encryptor_EncryptBatch")
    print(f"library: {args.lib or 'this tree'}; batch seams: {batched}", flush=True)
    O = S.context(n, moduli, t)
    be, kg, pk, enc = vp(), vp(), vp(), vp()
    S.call("BatchEncoder_Create", O.ctx, C.byref(be))
    S.call("KeyGenerator_Create1", O.ctx, C.byref(kg))
    S.call("KeyGenerator_CreatePublicKey", kg, C.c_bool(False), C.byref(pk))
    S.call("Encryptor_Create", O.ctx, pk, None, C.byref(enc))
    ok = True

    def new(kind, count):
        hs = []
        for _ in range(count):
            h = vp()
            S.call(kind + "_Create1", None, C.byref(h))
            hs.append(h)
        return hs

    if not batched:
        for B in (1, 64, 1024):
            vals = rng.integers(0, t, size=(B, n), dtype=np.uint64)
            ph, cp = new("Plaintext", B), new("Ciphertext", B)

            def per_handle():
                for i in range(B):
                    S.call("BatchEncoder_Encode1", be, u64(n), vals[i].ctypes.data_as(C.POINTER(u64)), ph[i])
                    S.call("Encryptor_Encrypt", enc, ph[i], cp[i], None)

            tp, _ = median_pair(per_handle, lambda: None)
            print(f"{B} items: per-handle Encode1+Encrypt {tp[0] * 1e3:.2f} ms (range {tp[1] * 1e3:.2f}-{tp[2] * 1e3:.2f})", flush=True)
        concurrency(S, O, enc, be, n, t, rng, batched)
        return
    ctx = B200Context(n, moduli, t)
    for B in (1, 64, 1024):
        vals = rng.integers(0, t, size=(B, n), dtype=np.uint64)
        vptr = vals.ctypes.data_as(C.c_void_p)
        seeds = rng.integers(0, 2**63, size=(B, 8), dtype=np.uint64)
        sptr = seeds.ctypes.data_as(C.POINTER(u64))
        pts, cts_b, cts_s, cts_p = new("Plaintext", B), new("Ciphertext", B), new("Ciphertext", B), new("Ciphertext", B)
        S.call("B200_BatchEncoder_EncodeBatch", be, u64(B), u64(n), vals.ctypes.data_as(C.POINTER(u64)), C.c_bool(False), arr(pts))
        pts_a, cb_a, cs_a = arr(pts), arr(cts_b), arr(cts_s)

        def batch():
            S.call("B200_Encryptor_EncryptBatch", enc, u64(B), pts_a, None, C.c_bool(False), cb_a)

        def slots():
            S.call("B200_Encryptor_EncryptSlotsBatch", enc, be, u64(B), u64(n), vptr, C.c_bool(False), None, C.c_bool(False), cs_a)

        ph = new("Plaintext", B)

        def per_handle():
            for i in range(B):
                S.call("BatchEncoder_Encode1", be, u64(n), vals[i].ctypes.data_as(C.POINTER(u64)), ph[i])
                S.call("Encryptor_Encrypt", enc, ph[i], cts_p[i], None)

        tb, tp = median_pair(batch, per_handle)
        ts, tp2 = median_pair(slots, per_handle)
        # words: both seams seeded == Encode1 + B200_Encryptor_EncryptSetSeed
        S.call("B200_Encryptor_EncryptBatch", enc, u64(B), pts_a, sptr, C.c_bool(False), cb_a)
        S.call("B200_Encryptor_EncryptSlotsBatch", enc, be, u64(B), u64(n), vptr, C.c_bool(False), sptr, C.c_bool(False), cs_a)
        same = True
        for i in sorted({0, B // 2, B - 1}):
            S.call("BatchEncoder_Encode1", be, u64(n), vals[i].ctypes.data_as(C.POINTER(u64)), ph[i])
            S.call("B200_Encryptor_EncryptSetSeed", enc, ph[i], seeds[i].ctypes.data_as(C.POINTER(u64)), cts_p[i])
            w = O.ct_words(cts_p[i])
            same &= np.array_equal(O.ct_words(cts_b[i]), w) and np.array_equal(O.ct_words(cts_s[i]), w)
        ok &= bool(same)
        smp = np.zeros((B, 3, n), dtype=np.int8)
        ctx.sample_pk(seeds, smp, B)
        t0 = time.perf_counter()
        for _ in range(3):
            ctx.sample_pk(seeds, smp, B)
        tsample = (time.perf_counter() - t0) / 3
        wall, gpu = gpu_split(batch)
        fmt = lambda m: f"{m[0] * 1e3:.2f} ms (range {m[1] * 1e3:.2f}-{m[2] * 1e3:.2f})"
        print(f"{B} items: EncryptBatch {fmt(tb)}  EncryptSlotsBatch {fmt(ts)}  per-handle Encode1+Encrypt {fmt(tp)} / {fmt(tp2)}  "
              f"per-handle/EncryptBatch {tp[0] / tb[0]:.1f}x  per-handle/EncryptSlotsBatch {tp2[0] / ts[0]:.1f}x  "
              f"words identical: {same}", flush=True)
        print(f"  host sampling alone (b200_sample_pk, mean of 3): {tsample * 1e3:.2f} ms;  one profiled EncryptBatch: wall "
              f"{wall * 1e3:.2f} ms, GPU kernels+copies {gpu * 1e3:.3f} ms", flush=True)
    concurrency(S, O, enc, be, n, t, rng, batched)
    ref = reference_time(n, moduli, t, rng)
    if ref is None:
        print("reference per-call CPU time: not measured (oracle/_ref not built)")
    else:
        print(f"reference per-call CPU time (BatchEncoder_Encode1 + Encryptor_Encrypt): {ref * 1e3:.3f} ms per item")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
