"""Developer tool: time per transform inside the two cluster kernels of multiply+relinearize against the standalone FP64 NTT.

    python tools/cluster_probe.py [batch]

Runs multiply_relin (n = 8192, k = 4: bench.py's workload, both cluster kernels at their production grids) under the launch
trace and the batched forward / inverse NTT of bench.py's roofline (4096 polynomials x k residues, ntt_fp_kernel<13>) between
CUDA events, and prints each kernel's time divided by the transforms it runs: 7 per (item, row) in mul_cluster_kernel (4 forward
+ 3 inverse, k + |Bsk| rows), k + 2 per (item, key residue) in ks_cluster_kernel (k forward + 2 inverse, k + 1 residues), one per
polynomial and residue in the standalone transform.  Prints one JSON line, with the card's name, power limit and SM clocks."""
import json, os, re, subprocess, sys, tempfile
os.environ["B200_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sunscreen_b200.lib import B200Context
from bench import MODULI, PLAIN, N_POLY

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
POLYS, STEPS = 4096, 10
ctx = B200Context(N_POLY, MODULI, PLAIN)
k, n = ctx.k(), N_POLY
rows = k + len(ctx.level_info(ctx.first_level)["bsk"])


def rr(shape, mods):
    out = torch.empty(shape + (len(mods), n), dtype=torch.int64, device="cuda")
    for i, m in enumerate(mods):
        out[..., i, :] = torch.randint(0, m, shape + (n,), device="cuda", dtype=torch.int64)
    return out


def traced(fn):
    """per-kernel totals (ms) of STEPS calls of fn after 3 untimed ones"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            ctx.L.lib.b200_trace_dump()  # drop the warm-up launches
            for _ in range(STEPS):
                fn()
            torch.cuda.synchronize()
            ctx.L.lib.b200_trace_dump()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        text = f.read().split("[b200 trace] total")[-2]  # the block of the timed calls
    return {m.group(1): float(m.group(2)) / STEPS for m in re.finditer(r"\[b200 trace\] (\S+)\s+launches\s+\d+\s+total\s+([\d.]+) ms", text)}


a, b, rlk = rr((B, 2), MODULI[:k]), rr((B, 2), MODULI[:k]), rr((k, 2), MODULI)
out = torch.zeros_like(a)
s = torch.cuda.current_stream().cuda_stream
mr = traced(lambda: ctx.multiply_relin(a, b, rlk, out, B, stream=s))
del a, b, out
slab = rr((POLYS,), MODULI[:k])


def timed(fn):
    """ms per call (CUDA events: the NTT entry points launch outside the trace)"""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(STEPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / STEPS


fwd_ms = timed(lambda: ctx.ntt_forward(slab, POLYS, stream=s))
inv_ms = timed(lambda: ctx.ntt_inverse(slab, POLYS, stream=s))


def one(d, pat):
    hits = [v for name, v in d.items() if pat in name]
    assert len(hits) == 1, (pat, d)
    return hits[0]


gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()
mul_ms, ks_ms = one(mr, "mul_cluster"), one(mr, "ks_cluster")
res = {"gpu": gpu, "batch": B, "k": k, "rows": rows, "multiply_relin_kernels_ms": mr,
       "mul_cluster_ms": mul_ms, "mul_cluster_ns_per_transform": mul_ms * 1e6 / (B * rows * 7),
       "ks_cluster_ms": ks_ms, "ks_cluster_ns_per_transform": ks_ms * 1e6 / (B * (k + 1) * (k + 2)),
       "ntt_fwd_ms": fwd_ms, "ntt_fwd_ns_per_transform": fwd_ms * 1e6 / (POLYS * k),
       "ntt_inv_ms": inv_ms, "ntt_inv_ns_per_transform": inv_ms * 1e6 / (POLYS * k)}
print(json.dumps(res))
