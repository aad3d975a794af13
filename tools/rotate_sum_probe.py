"""Rotate-and-sum slot reductions on one GPU: c <- c + rotate(c) over a list of Galois elements, two routes on the same
device buffers, timed with CUDA events after warm-up, alternated over several rounds:
  fused  one b200_apply_galois_add per step (the automorphism inside the key switch, the add inside its mod-down);
  chain  b200_apply_galois then b200_add per step (the rotate_rows + add chain).
Both routes must give identical words.  The GPU name, power limit and SM clock are printed with the numbers.

    python tools/rotate_sum_probe.py [dotprod:n8192:1 dotprod:n8192:64 dotprod:n8192:1024 step:n16384:64 step:n32768:16 ...]
dotprod: rotate_rows by 1, 2, 4, ..., n/4 and rotate_columns (Sunscreen's dot_prod reduction); step: one rotate_rows(1).
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


def probe(kind, name, batch, rounds=5):
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    k, K = ctx.k(), len(moduli)
    elts = [pow(3, 1 << i, 2 * n) for i in range((n // 4).bit_length())] + [2 * n - 1] if kind == "dotprod" else [3]
    g = torch.Generator(device="cuda")
    g.manual_seed(batch * 7 + n)
    s = torch.cuda.current_stream().cuda_stream
    key = torch.empty((k, 2, K, n), dtype=torch.int64, device="cuda")
    for i, q in enumerate(moduli):
        key[:, :, i, :] = torch.randint(0, q, (k, 2, n), device="cuda", dtype=torch.int64, generator=g)
    c0 = rand_residues((batch, 2), moduli[:k], n, g)
    fa, fb = c0.clone(), torch.empty_like(c0)
    ca, cb = c0.clone(), torch.empty_like(c0)

    def fused():
        a, b = fa, fb
        for e in elts:
            ctx.apply_galois_add(a, e, key, a, b, batch, stream=s)
            a, b = b, a
        return a

    def chain():
        for e in elts:
            ctx.apply_galois(ca, e, key, cb, batch, stream=s)
            ctx.add(ca, cb, ca, 2, batch, stream=s)
        return ca

    # words: one pass of each route from the same input
    res_f, res_c = fused(), chain()
    torch.cuda.synchronize()
    same = torch.equal(res_f, res_c)
    iters = max(1, min(50, 2000 // (batch * len(elts))))
    timed(fused, iters)  # warm-up of both shapes
    timed(chain, iters)
    tf, tc = [], []
    for _ in range(rounds):  # alternate the two routes
        tf.append(timed(fused, iters))
        tc.append(timed(chain, iters))
    tf.sort()
    tc.sort()
    mf, mc = tf[len(tf) // 2], tc[len(tc) // 2]
    steps = len(elts)
    print(f"{kind} {name} n={n} k={k} batch={batch} steps={steps}: fused {mf:.3f} ms (range {tf[0]:.3f}-{tf[-1]:.3f})  "
          f"chain {mc:.3f} ms (range {tc[0]:.3f}-{tc[-1]:.3f})  chain/fused {mc / mf:.2f}x  "
          f"per step per item: fused {1e3 * mf / (steps * batch):.2f} us, chain {1e3 * mc / (steps * batch):.2f} us  "
          f"words identical: {same}")
    del key, c0, fa, fb, ca, cb
    ctx.close()
    torch.cuda.empty_cache()
    return same


def main():
    assert torch.cuda.is_available(), "rotate_sum_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip().replace("\n", " | ")
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q}")
    cases = sys.argv[1:] or ["dotprod:n8192:1", "dotprod:n8192:64", "dotprod:n8192:1024", "step:n16384:64", "step:n32768:16"]
    ok = True
    for c in cases:
        kind, name, batch = c.split(":")
        ok &= probe(kind, name, int(batch))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
