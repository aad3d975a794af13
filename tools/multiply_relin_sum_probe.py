"""Encrypted inner products on one GPU: out[r] = sum_j relinearize(multiply(a[r][j], b[r][j])), two routes on the same device
buffers, timed with CUDA events after warm-up, alternated over several rounds:
  fused  one b200_multiply_relin_sum (the adds inside the key switch's mod-down);
  chain  one b200_multiply_relin over all R m terms, then m - 1 b200_add (the multiply -> relinearize -> add chain).
Both routes must give identical words.  The GPU name, power limit and SM clock are printed with the numbers.

    python tools/multiply_relin_sum_probe.py [n8192:1:10 n8192:1:15 n8192:1:100 n8192:64:16 n8192:1024:4 n16384:64:8 n32768:4:8 ...]
(parameter set : outputs R : terms m; n16384 runs at its k = 8 level, n32768 at k = 15)
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from params import PARAMS  # noqa: E402
from sunscreen_b200.lib import B200Context  # noqa: E402


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


def probe(name, R, m, rounds=5):
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    k, K = ctx.k(), len(moduli)
    g = torch.Generator(device="cuda")
    g.manual_seed(R * 7 + m + n)
    s = torch.cuda.current_stream().cuda_stream
    key = torch.empty((k, 2, K, n), dtype=torch.int64, device="cuda")
    for i, q in enumerate(moduli):
        key[:, :, i, :] = torch.randint(0, q, (k, 2, n), device="cuda", dtype=torch.int64, generator=g)
    a = rand_residues((R, m, 2), moduli[:k], n, g)
    b = rand_residues((R, m, 2), moduli[:k], n, g)
    fo = torch.empty((R, 2, k, n), dtype=torch.int64, device="cuda")
    prod = torch.empty((R, m, 2, k, n), dtype=torch.int64, device="cuda")
    co = torch.empty_like(fo)

    def fused():
        ctx.multiply_relin_sum(a, b, key, m, fo, R, stream=s)
        return fo

    def chain():
        ctx.multiply_relin(a, b, key, prod, R * m, stream=s)
        co.copy_(prod[:, 0])
        for j in range(1, m):
            ctx.add(co, prod[:, j].contiguous(), co, 2, R, stream=s)
        return co

    res_f, res_c = fused(), chain()
    torch.cuda.synchronize()
    same = torch.equal(res_f, res_c)
    iters = max(1, min(50, 4000 // (R * m)))
    timed(fused, iters)  # warm-up of both shapes
    timed(chain, iters)
    tf, tc = [], []
    for _ in range(rounds):  # alternate the two routes
        tf.append(timed(fused, iters))
        tc.append(timed(chain, iters))
    tf.sort()
    tc.sort()
    mf, mc = tf[len(tf) // 2], tc[len(tc) // 2]
    print(f"{name} n={n} k={k} R={R} m={m}: fused {mf:.3f} ms (range {tf[0]:.3f}-{tf[-1]:.3f})  "
          f"chain {mc:.3f} ms (range {tc[0]:.3f}-{tc[-1]:.3f})  chain/fused {mc / mf:.2f}x  "
          f"per term: fused {1e3 * mf / (R * m):.2f} us, chain {1e3 * mc / (R * m):.2f} us  words identical: {same}", flush=True)
    del key, a, b, fo, prod, co
    ctx.close()
    torch.cuda.empty_cache()
    return same


def main():
    assert torch.cuda.is_available(), "multiply_relin_sum_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip().replace("\n", " | ")
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q}")
    cases = sys.argv[1:] or ["n8192:1:10", "n8192:1:15", "n8192:1:100", "n8192:64:16", "n8192:1024:4", "n16384:64:8",
                             "n32768:4:8"]
    ok = True
    for c in cases:
        name, R, m = c.split(":")
        ok &= probe(name, int(R), int(m))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
