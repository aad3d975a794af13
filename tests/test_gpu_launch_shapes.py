"""Launch shapes and kernel variants the fixed-size parity tests do not pick on purpose (pytest -m gpu).

Every batch size here is derived from the device's SM count and the host-side launch formulas it targets, so the same
boundaries are hit on any H100 configuration:
  * n = 8192 static NTT: 512 threads per CTA while items * k <= 2 * sm_count, 256 above (b200_bfv.cu launch_ntt);
  * n = 16384 inverse NTT: the persistent variant runs min(blocks, per_sm * sm_count) CTAs, each prefetching the next
    polynomial it walks to, which may belong to another prime (ntt_fp_kernels.cu);
  * the key-switch MAC (ksmac_tma.cu launch): the batch is cut into chunks of `ipc` items whose last one is partial unless
    ipc divides the batch;
  * every correct FP64 NTT variant of every instantiated (size, CTA width), forced through b200_debug_ntt_variant;
  * settings read once per process (fused tensor inverse, the non-TMA key-switch MAC) in a subprocess each.
Every output word is compared with the unmodified reference."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from params import PARAMS

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def be():
    from backends import CudaBackend
    return CudaBackend()


@pytest.fixture(scope="module")
def pairs(be, ref):
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.Pair(be, *PARAMS[name])
        return cache[name]
    return get


def _threads():
    return max(1, min(64, len(os.sched_getaffinity(0))))


def persistent_ctas_per_sm(P, nt, var, forward=False):
    """resident CTAs per SM of an FP64 NTT kernel: the occupancy query the launcher makes to cap the persistent
    variant's grid (b200_debug_ntt_ctas_per_sm)"""
    per_sm = P.be.lib.lib.b200_debug_ntt_ctas_per_sm(P.n.bit_length() - 1, int(forward), nt, var)
    assert per_sm >= 1, per_sm
    return per_sm


def ksmac_items_per_chunk(n, k, batch, sm_count):
    """ksmac_tma.cu launch(): items per CTA of the key-switch MAC"""
    per_chunk = (n // 256) * (k + 1)
    ipc = batch
    while ipc > 8 and per_chunk * (-(-batch // ipc)) < 8 * sm_count:
        ipc = (ipc + 1) // 2
    return ipc


def mul_relin_vs_reference(P, batch, seed, also_relinearize=False):
    """multiply_relin (and optionally relinearize of our own size-3 product) of `batch` random pairs; every item equals
    the reference's relinearize(multiply(a, b))."""
    rng = np.random.default_rng(seed)
    A = pc.rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    B = pc.rand_ct(rng, P.moduli, P.k, P.n, batch=batch)
    key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    rlk = P.ref.new_ksk({0: key})
    exp = P.ref.mul_relin_batch(A, B, rlk, _threads())
    dK = P.dev(key)
    o2 = P.out(batch, 2, P.k, P.n)
    P.ctx.multiply_relin(P.dev(A), P.dev(B), dK, o2, batch)
    got = P.host(o2)
    for i in range(batch):
        if not np.array_equal(got[i], exp[i]):
            pc.eq(got[i], exp[i], f"multiply_relin item {i} of {batch}")
    if also_relinearize:
        o3 = P.out(batch, 3, P.k, P.n)
        P.ctx.multiply(P.dev(A), 2, P.dev(B), 2, o3, batch)
        o2r = P.out(batch, 2, P.k, P.n)
        P.ctx.relinearize(o3, dK, o2r, batch)
        got = P.host(o2r)
        for i in range(batch):
            if not np.array_equal(got[i], exp[i]):
                pc.eq(got[i], exp[i], f"relinearize item {i} of {batch}")


# ---------------------------------------------------------------------------------------------------------------------
# n = 8192: the 512 / 256 threads-per-CTA switch of the static NTT
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("side", ["at", "above"])
def test_n8192_ntt_thread_count_boundary(pairs, side):
    P = pairs("n8192")
    limit = 2 * P.ctx.sm_count                  # blocks <= limit -> 512 threads per CTA
    items = limit // P.k + (1 if side == "above" else 0)
    assert (items * P.k <= limit) == (side == "at")
    pc.check_ntt(P, items=items, seed=40 + items)


# ---------------------------------------------------------------------------------------------------------------------
# n = 16384: persistent inverse NTT at grids below, at and well above its CTA cap, and multiply_relin around it
# ---------------------------------------------------------------------------------------------------------------------
def _n16384_grid(P):
    return persistent_ctas_per_sm(P, 1024, 2064) * P.ctx.sm_count


@pytest.mark.parametrize("side", ["below", "at", "above"])
def test_n16384_persistent_inverse_ntt(pairs, side):
    P = pairs("n16384")
    G = _n16384_grid(P)
    items = {"below": (G - 1) // P.k, "at": -(-G // P.k), "above": 3 * (-(-G // P.k)) + 1}[side]
    blocks = items * P.k
    assert {"below": blocks < G, "at": G <= blocks < G + P.k, "above": blocks > 3 * G}[side]
    # above the cap, a CTA's next polynomial is in another slot (prime) whenever its stride G is not a multiple of items
    pc.check_ntt(P, items=items, seed=60 + items)


@pytest.mark.parametrize("side", ["below", "at", "above"])
def test_n16384_multiply_relin_around_persistent_grid(pairs, side):
    """The product's inverse NTT transforms every row of the size-3 tensor product in base q and in the auxiliary base
    Bsk (multiply_core: row_primes(..., with_bsk)), so 3 (k + |Bsk|) polynomials per item: batches around G / that."""
    P = pairs("n16384")
    G = _n16384_grid(P)
    rows = 3 * (P.k + len(P.ctx.level_info(P.ctx.first_level)["bsk"]))
    batch = {"below": (G - 1) // rows, "at": -(-G // rows), "above": 3 * (-(-G // rows)) + 1}[side]
    blocks = batch * rows
    assert batch >= 1 and {"below": blocks < G, "at": G <= blocks < G + rows, "above": blocks > 3 * G}[side], (G, rows, batch)
    mul_relin_vs_reference(P, batch, seed=70 + batch)


# ---------------------------------------------------------------------------------------------------------------------
# key-switch MAC: a partial last chunk of items
# ---------------------------------------------------------------------------------------------------------------------
def _partial_batches(P):
    sm = P.ctx.sm_count
    near = next(b for b in range(1000, 900, -1) if b % ksmac_items_per_chunk(P.n, P.k, b, sm))
    return [9, 17, near]


@pytest.mark.parametrize("which", [0, 1, 2])
def test_ksmac_partial_last_chunk(pairs, which):
    P = pairs("n8192")
    batch = _partial_batches(P)[which]
    ipc = ksmac_items_per_chunk(P.n, P.k, batch, P.ctx.sm_count)
    assert ipc < batch and batch % ipc, (batch, ipc)
    mul_relin_vs_reference(P, batch, seed=80 + batch, also_relinearize=True)


_KSMAC_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import parity_checks as pc
import test_gpu_launch_shapes as T
from backends import CudaBackend
from params import PARAMS
P = pc.Pair(CudaBackend(), *PARAMS["n8192"])
batch = T._partial_batches(P)[0]
T.mul_relin_vs_reference(P, batch, seed=80 + batch, also_relinearize=True)
P.be.lib.lib.b200_trace_dump()
"""


def test_ksmac_partial_last_chunk_runs_the_tma_kernel(ref):
    """The partial-chunk batches above only test the chunking if the key-switch MAC they reach is the TMA kernel (the
    launcher falls back to the item-major kernels when the tensor-map encoder is unavailable): with the launch trace on
    (B200_TRACE, read once per process) the same multiply_relin + relinearize must list ksmac_tma_kernel and no fallback."""
    env = dict(os.environ, B200_TRACE="1")
    env.pop("B200_KSMAC_TMA", None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _KSMAC_TRACE.format(root=ROOT, tests=HERE)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (\S+)\s+launches\s+(\d+)", r.stderr)}
    assert launches.get("ksmac_tma_kernel", 0) >= 2, launches
    assert not [name for name in launches if name.startswith("ksmac_kernel")], launches


# ---------------------------------------------------------------------------------------------------------------------
# every correct FP64 NTT variant, forced
# ---------------------------------------------------------------------------------------------------------------------
CORRECT_VARIANTS = (0, 1, 16, 2048, 2049, 2064)    # the others at (13, 256) are timing ablations with meaningless output
SIZE_SET = {12: "n4096", 13: "n8192", 14: "n16384"}


def instantiated_variants():
    """(logn, threads per CTA, variant) of every correct instantiation in ntt_fp_kernels.cu (B200_FP_KERNELS)"""
    src = open(os.path.join(ROOT, "sunscreen_b200", "csrc", "ntt_fp_kernels.cu")).read()
    block = src[src.index("#define B200_FP_KERNELS"):src.index("b200_ntt_fp_fn b200_ntt_fp_kernel")]
    found = sorted({tuple(map(int, m)) for m in re.findall(r"X\((\d+), (\d+), (\d+)\)", block)})
    return [f for f in found if f[2] in CORRECT_VARIANTS]


VARIANTS = instantiated_variants()


def test_variant_table_covers_every_size():
    assert {(l, nt) for l, nt, _ in VARIANTS} == {(12, 256), (13, 256), (13, 512), (14, 1024)}
    assert {v for _, _, v in VARIANTS} == set(CORRECT_VARIANTS)


@pytest.mark.parametrize("logn,nt,var", VARIANTS)
def test_forced_ntt_variant(be, pairs, logn, nt, var):
    P = pairs(SIZE_SET[logn])
    sm = P.ctx.sm_count
    if logn == 13 and nt == 512:
        items = max(6, (2 * sm) // P.k // 2)             # stays at or below 2 * sm_count blocks
        assert items * P.k <= 2 * sm
    elif var & 16:
        items = -(-3 * persistent_ctas_per_sm(P, nt, var) * sm // P.k) + 1   # every persistent CTA walks >= 3 polys
    else:
        items = 2 * sm // P.k + 3                         # above the 512-thread limit at n = 8192
    L = be.lib.lib
    old = L.b200_debug_ntt_variant(var)
    try:
        pc.check_ntt(P, items=items, seed=var + logn)
        pc.check_relin(P)
    finally:
        L.b200_debug_ntt_variant(old)


# ---------------------------------------------------------------------------------------------------------------------
# settings read once per process
# ---------------------------------------------------------------------------------------------------------------------
_SUBPROCESS_CHECKS = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import parity_checks as pc
from backends import CudaBackend
from params import PARAMS
be = CudaBackend()
for name in ("n4096", "n8192", "n16384"):
    P = pc.Pair(be, *PARAMS[name])
    pc.check_ntt(P, items=5)
    m3, rm = pc.check_multiply(P)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_batch(P, batch=5)
    pc.check_adversarial_multiply(P, with_size5=True)
    pc.check_adversarial_keyswitch(P)
    pc.check_encrypted_roundtrip(P)
    print("ok", name, flush=True)
"""


@pytest.mark.parametrize("setting", ["B200_TENSOR_FUSION=1", "B200_KSMAC_TMA=0"])
def test_process_wide_setting(ref, setting):
    name, value = setting.split("=")
    env = dict(os.environ, **{name: value})
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _SUBPROCESS_CHECKS.format(root=ROOT, tests=HERE)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"{setting}: exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    assert r.stdout.split() == ["ok", "n4096", "ok", "n8192", "ok", "n16384"], r.stdout


# ---------------------------------------------------------------------------------------------------------------------
# the plain-modulus NTT (BatchEncoder) on either side of the FP64 width limit
# ---------------------------------------------------------------------------------------------------------------------
_PLAIN_NTT_TRACE = """
import ctypes as C, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
from backends import CudaBackend
from sunscreen_b200.lib import B200Context, ptr
be = CudaBackend()
ctx = B200Context({n}, {moduli!r}, {t})
x = be.to_dev(np.arange(4 * {n}, dtype=np.uint64) % {t})
for inverse in (1, 0):
    assert ctx.L.lib.b200_plain_ntt(ctx.h, C.c_void_p(ptr(x)), C.c_uint64(4), C.c_int(inverse), None) == 0
assert np.array_equal(be.to_host(x).reshape(-1), np.arange(4 * {n}, dtype=np.uint64) % {t})
ctx.L.lib.b200_trace_dump()
"""


@pytest.mark.parametrize("bits", [49, 50])
def test_plain_ntt_fp64_width_limit(bits):
    """n8192_t49's plain modulus is the widest the FP64 transform takes (host_ctx.h FP_PRIME_BITS = 49): with the launch
    trace on, its BatchEncoder transforms run ntt_fp_kernel, and those of the 50-bit batching prime run the integer kernel."""
    from test_params import batching_plain_modulus
    from params import PARAMS
    n, moduli, t = PARAMS["n8192_t49"]
    if bits == 50:
        t = batching_plain_modulus(n, 50, skip=moduli)
    assert t.bit_length() == bits
    env = dict(os.environ, B200_TRACE="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _PLAIN_NTT_TRACE.format(root=ROOT, tests=HERE, n=n, moduli=moduli, t=t)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    names = [m.group(1) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+\d+", r.stderr)]
    fp = [nm for nm in names if nm.startswith("ntt_fp_kernel")]
    assert (len(fp) == 2) == (bits == 49) and (not fp) == (bits == 50), names
    assert ("kfn" in names) == (bits == 50), names
