"""Plaintext matrix x ciphertext vector on one GPU (R outputs, m terms, size-2 ciphertexts), timed with CUDA events after
warm-up:
  (a) b200_multiply_plain_sum with resident NTT-form plaintexts;
  (b) b200_plain_to_ntt (multiply rule) of the coefficient plaintexts, then (a);
  (c) today's route: b200_multiply_plain over the R * m items (one output row at a time), then R * (m - 1) b200_adds.
(a), (b) and (c) must give identical words.  The MAC kernel's own time comes from a separate torch.profiler run; its
algorithmic bytes (P once, X once, the output once) over that time are printed against the H100 SXM data sheet's 3.35 TB/s,
with the GPU name and power limit.

    python tools/plain_sum_probe.py [n8192:10 n8192:100 n32768:10 n32768:100 ...]
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from params import PARAMS  # noqa: E402
from sunscreen_b200.lib import PLAIN_NTT_MULTIPLY, B200Context  # noqa: E402

HBM_PEAK = 3.35e12


def rand_residues(shape, moduli, n, g):
    out = torch.empty(shape + (len(moduli), n), dtype=torch.int64, device="cuda")
    for i, q in enumerate(moduli):
        out[..., i, :] = torch.randint(0, q, shape + (n,), device="cuda", dtype=torch.int64, generator=g)
    return out


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def probe(name, R, m, iters):
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    k = ctx.k()
    g = torch.Generator(device="cuda")
    g.manual_seed(R * 1000 + m)
    s = torch.cuda.current_stream().cuda_stream
    cts = rand_residues((m, 2), moduli[:k], n, g)
    plains = torch.randint(0, t, (R, m, n), device="cuda", dtype=torch.int64, generator=g)
    pn = torch.empty((R, m, k, n), dtype=torch.int64, device="cuda")
    out_a = torch.empty((R, 2, k, n), dtype=torch.int64, device="cuda")
    out_b = torch.empty_like(out_a)
    out_c = torch.empty_like(out_a)

    def prep():
        ctx.plain_to_ntt(plains, R * m, pn, rule=PLAIN_NTT_MULTIPLY, stream=s)

    def run_a():
        ctx.multiply_plain_sum(cts, 2, m, pn, R, out_a, stream=s)

    def run_b():
        prep()
        ctx.multiply_plain_sum(cts, 2, m, pn, R, out_b, stream=s)

    prod = torch.empty((m, 2, k, n), dtype=torch.int64, device="cuda")

    def run_c():
        for i in range(R):
            ctx.multiply_plain(cts, 2, plains[i], m, prod, m, stream=s)
            if m == 1:
                out_c[i].copy_(prod[0])
                continue
            ctx.add(prod[0], prod[1], out_c[i], 2, 1, stream=s)
            for j in range(2, m):
                ctx.add(out_c[i], prod[j], out_c[i], 2, 1, stream=s)

    prep()
    for fn in (run_a, run_b, run_c):  # warm-up
        fn()
    torch.cuda.synchronize()
    same = torch.equal(out_a, out_b) and torch.equal(out_a, out_c)
    ta, tb, tc = timed(run_a, iters), timed(run_b, iters), timed(run_c, max(1, iters // 4))
    # the MAC kernel alone, in a profiled run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            run_a()
        torch.cuda.synchronize()
    mac_us = sum(e.device_time_total for e in prof.key_averages() if "plain_mac_kernel" in e.key) / iters
    mac_bytes = 8 * k * n * (R * m + 2 * m + 2 * R)
    bw = mac_bytes / (mac_us * 1e-6) if mac_us else float("nan")
    print(f"{name} n={n} k={k} R={R} m={m}: (a) {ta:.3f} ms  (b) {tb:.3f} ms  (c) {tc:.3f} ms  (c)/(a) {tc / ta:.1f}x  "
          f"(c)/(b) {tc / tb:.1f}x  words identical: {same}")
    print(f"    plain_mac_kernel {mac_us / 1e3:.3f} ms, {mac_bytes / 1e9:.3f} GB -> {bw / 1e12:.2f} TB/s = "
          f"{100 * bw / HBM_PEAK:.0f}% of 3.35 TB/s")
    del pn, plains, cts, prod
    ctx.close()
    torch.cuda.empty_cache()
    return same


def main():
    assert torch.cuda.is_available(), "plain_sum_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q}")
    cases = sys.argv[1:] or ["n8192:10", "n8192:100", "n32768:10", "n32768:100"]
    ok = True
    for c in cases:
        name, rm = c.split(":")
        R = m = int(rm)
        ok &= probe(name, R, m, iters=20 if R * m <= 100 else 5)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
