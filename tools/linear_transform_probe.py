"""Baby-step giant-step slot-wise linear transforms on one GPU, two routes on the same device buffers, timed with CUDA events
after warm-up, alternated over several rounds (medians reported):
  fused     one b200_linear_transform (one key switch per step group, the masked MAC of all vectors, the giant steps summed
            inside their mod-down);
  existing  b200_apply_galois per baby step, b200_multiply_plain_sum per vector and b200_apply_galois_add per giant step.
Both routes must give identical words.  The GPU name, power limit and SM clock are printed with the numbers.

    python tools/linear_transform_probe.py [n8192:1:16:16 n8192:1:64:64 n8192:64:8:8 n16384:1:16:16 ...]   (name:V:b:G)
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


def probe(name, V, b, G, rounds=5):
    n, moduli, t = PARAMS[name]
    ctx = B200Context(n, moduli, t)
    k, K = ctx.k(), len(moduli)
    g = torch.Generator(device="cuda")
    g.manual_seed(V * 131 + b * 7 + G)
    s = torch.cuda.current_stream().cuda_stream
    elts = [pow(3, j, 2 * n) for j in range(1, b)] + [pow(3, i * b, 2 * n) for i in range(1, G)]
    keys = {}
    for e in elts:
        key = torch.empty((k, 2, K, n), dtype=torch.int64, device="cuda")
        for i, q in enumerate(moduli):
            key[:, :, i, :] = torch.randint(0, q, (k, 2, n), device="cuda", dtype=torch.int64, generator=g)
        keys[e] = key
    klist = [keys[e] for e in elts]
    cts = rand_residues((V, 2), moduli[:k], n, g)
    plains = torch.randint(1, t, (G * b, n), device="cuda", dtype=torch.int64, generator=g)
    pn = torch.empty((G, b, k, n), dtype=torch.int64, device="cuda")
    ctx.plain_to_ntt(plains, G * b, pn, rule=PLAIN_NTT_MULTIPLY)
    fo = torch.empty((V, 2, k, n), dtype=torch.int64, device="cuda")
    X = torch.empty((V, b, 2, k, n), dtype=torch.int64, device="cuda")
    inner = torch.empty((V, G, 2, k, n), dtype=torch.int64, device="cuda")
    eo = torch.empty((V, 2, k, n), dtype=torch.int64, device="cuda")

    def fused():
        ctx.linear_transform(cts, V, b, G, elts, klist, pn, fo, stream=s)
        return fo

    def existing():
        for v in range(V):
            X[v, 0].copy_(cts[v])
            for j in range(1, b):
                ctx.apply_galois(cts[v], elts[j - 1], klist[j - 1], X[v, j], 1, stream=s)
            ctx.multiply_plain_sum(X[v], 2, b, pn, G, inner[v], stream=s)
            eo[v].copy_(inner[v, 0])
            for i in range(1, G):
                e = b - 1 + i - 1
                ctx.apply_galois_add(inner[v, i], elts[e], klist[e], eo[v], eo[v], 1, stream=s)
        return eo

    same = torch.equal(fused(), existing())
    torch.cuda.synchronize()
    per = timed(fused, 1)
    iters = max(2, min(30, int(200 / max(per, 0.01))))
    timed(fused, iters)  # warm-up of both routes
    timed(existing, iters)
    tf, te = [], []
    for _ in range(rounds):
        tf.append(timed(fused, iters))
        te.append(timed(existing, iters))
    tf.sort()
    te.sort()
    mf, me = tf[len(tf) // 2], te[len(te) // 2]
    print(f"{name} n={n} k={k} V={V} b={b} G={G}: fused {mf:.3f} ms (range {tf[0]:.3f}-{tf[-1]:.3f})  "
          f"existing {me:.3f} ms (range {te[0]:.3f}-{te[-1]:.3f})  existing/fused {me / mf:.2f}x  words identical: {same}",
          flush=True)
    del keys, klist, cts, plains, pn, fo, X, inner, eo
    ctx.close()
    torch.cuda.empty_cache()
    return same


def main():
    assert torch.cuda.is_available(), "linear_transform_probe needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip().replace("\n", " | ")
    print(f"GPU: {torch.cuda.get_device_name(0)} | nvidia-smi: {q}", flush=True)
    cases = sys.argv[1:] or ["n8192:1:16:16", "n8192:1:64:64", "n8192:64:8:8", "n16384:1:16:16"]
    ok = True
    for c in cases:
        name, V, b, G = c.split(":")
        ok &= probe(name, int(V), int(b), int(G))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
