"""Developer tool: forward / inverse NTT rate of a parameter set (tests/params.py name) against the measured HBM copy peak:
   python tools/ntt_roofline.py n8192_54 [polys]      (level 0 = all key-level primes, so the 54-bit set has 4 residues)
Algorithmic bytes: 16 n per residue transform (SURVEY.md 8(d))."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from params import PARAMS
from sunscreen_b200.lib import B200Context
name = sys.argv[1] if len(sys.argv) > 1 else "n8192_54"
n, moduli, t = PARAMS[name]
ctx = B200Context(n, moduli, t)
level = 0 if name.endswith("_54") else None
k = ctx.k(level)
items = int(sys.argv[2]) if len(sys.argv) > 2 else max(64, (1 << 25) // (n * k) // 8 * 8)  # ~2 GiB of words / 8
x = torch.empty((items, k, n), dtype=torch.int64, device="cuda")
for i in range(k):
    x[:, i, :] = torch.randint(0, moduli[i], (items, n), device="cuda", dtype=torch.int64)
s = torch.cuda.current_stream().cuda_stream
peak = 3350.0  # GB/s, HBM3 of the H100 SXM data sheet
def timed(fn, reps=5):
    best = 1e9
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best
for _ in range(2):
    ctx.ntt_forward(x, items, level=level, stream=s); ctx.ntt_inverse(x, items, level=level, stream=s)
f = timed(lambda: ctx.ntt_forward(x, items, level=level, stream=s))
i_ = timed(lambda: ctx.ntt_inverse(x, items, level=level, stream=s))
b = 16 * n * items * k
print(f"{name}: n={n}, {k} residues ({max(int(m).bit_length() for m in moduli[:k])}-bit primes), {items} polys: "
      f"fwd {f:.3f} ms {b/f/1e6:.0f} GB/s = {b/f/1e6/peak:.3f} of {peak:.0f} | inv {i_:.3f} ms {b/i_/1e6:.0f} GB/s = {b/i_/1e6/peak:.3f}")
