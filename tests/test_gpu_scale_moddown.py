"""multiply_relin with the product's c0, c1 scaled inside the key switch's mod-down (scale_moddown_kernel_v2,
sunscreen_b200/csrc/b200_bfv.cu) against multiply followed by relinearize, which keep the separate scale and mod-down, and
against the unmodified reference (pytest -m gpu).

On FP64 levels multiply_relin scales only D2 before the key switch and keeps D0, D1 unscaled until the mod-down, which
scales them in registers and adds them.  Where holding D through a key switch on the separate kernels would raise the peak
scratch ((k + 1)(k + 2) > 4 (k + |Bsk|): k = 7, 8 at n = 16384), and on the integer path, the separate scale and mod-down
run."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from params import PARAMS
from test_gpu_launch_shapes import _threads

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

FP64_CHAINS = ["n4096", "n8192", "n8192_49", "n16384", "n4096_narrow", "n4096_q_below_t", "n2048_2x27", "n1024_2x27"]
# the same chains under other plain moduli: t enters every constant of the scale
FP64_PLAIN = ["n4096_t2", "n4096_t2p40", "n8192_t30", "n8192_t47", "n8192_t49", "n8192_t3p37", "n16384_t60"]


@pytest.fixture(scope="module")
def pairs(ref):
    from backends import CudaBackend
    be = CudaBackend()
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.pair_for(be, name)
        return cache[name]
    return get


def fused_expected(P, lv):
    """multiply_relin_one's rule: an FP64 level (every data and auxiliary prime within 49 bits) whose key-switch scratch
    fits beside D"""
    li = P.ctx.level_info(lv)
    k, R = li["k"], li["k"] + li["nBsk"]
    fp = all(q.bit_length() <= 49 for q in li["q"] + li["bsk"])
    return fp and (k + 1) * (k + 2) <= 4 * R


def qm1_ct(moduli, k, n, batch):
    q = np.array([int(m) for m in moduli[:k]], dtype=np.uint64)[None, None, :, None]
    return np.broadcast_to(q - np.uint64(1), (batch, 2, k, n)).copy()


def mul_relin_three_ways(P, j, batch, seed, adversarial=False):
    """multiply_relin of `batch` pairs at data level j (0: the first) equals multiply + relinearize word for word, and, on
    the levels of the reference's chain, the reference's relinearize(multiply(a, b)).  adversarial: every operand word
    q - 1 and an all-(p - 1) key."""
    R = P.ref
    rng = np.random.default_rng(seed)
    lv = P.ctx.first_level + j
    k = P.ctx.level_info(lv)["k"]
    if adversarial:
        A = B = qm1_ct(P.moduli, k, P.n, batch)
        key = np.empty((P.k, 2, len(P.moduli), P.n), dtype=np.uint64)
        for i, m in enumerate(P.moduli):
            key[:, :, i, :] = np.uint64(int(m) - 1)
    else:
        A = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
        B = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
        key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    dA, dB, dK = P.dev(A), P.dev(B), P.dev(key)
    o2 = P.out(batch, 2, k, P.n)
    P.ctx.multiply_relin(dA, dB, dK, o2, batch, level=lv)
    got = P.host(o2).reshape(batch, 2, k, P.n)
    o3 = P.out(batch, 3, k, P.n)
    P.ctx.multiply(dA, 2, dB, 2, o3, batch, level=lv)
    o2s = P.out(batch, 2, k, P.n)
    P.ctx.relinearize(o3, dK, o2s, batch, level=lv)
    pc.eq(got, P.host(o2s), f"multiply_relin vs multiply + relinearize, batch {batch}, level {lv}")
    if j >= len(R.data_parms_ids()):
        return got
    rlk = R.new_ksk({0: key})
    if j == 0 and batch > 64:
        exp = R.mul_relin_batch(A, B, rlk, _threads())
        for i in range(batch):
            if not np.array_equal(got[i], exp[i]):
                pc.eq(got[i], exp[i], f"multiply_relin item {i} of {batch}")
        return got
    for i in range(batch):
        ra, rb = R.new_ct(A[i], level=j), R.new_ct(B[i], level=j)
        rm = R.multiply(ra, rb)
        rr = R.relinearize(rm, rlk)
        pc.eq(got[i], R.ct_words(rr), f"multiply_relin item {i} of {batch}, level {lv}")
        for h in (ra, rb, rm, rr):
            R.free_ct(h)
    return got


def data_levels(P):
    return range(P.ctx.levels - P.ctx.first_level)


@pytest.mark.parametrize("name", FP64_CHAINS + FP64_PLAIN)
def test_every_level(pairs, name):
    P = pairs(name)
    assert fused_expected(P, P.ctx.first_level) or name.startswith("n16384")
    for j in data_levels(P):
        mul_relin_three_ways(P, j, 3, seed=200 + j)


@pytest.mark.parametrize("batch", [1, 17, 1024])
def test_n8192_batches(pairs, batch):
    """batch 1 runs the separate key-switch kernels, 17 and 1024 the cluster kernels"""
    mul_relin_three_ways(pairs("n8192"), 0, batch, seed=300 + batch)


@pytest.mark.parametrize("name", ["n4096", "n8192", "n8192_49", "n16384", "n4096_narrow"])
def test_adversarial_every_level(pairs, name):
    P = pairs(name)
    for j in data_levels(P):
        mul_relin_three_ways(P, j, 2, seed=0, adversarial=True)


def test_adversarial_n8192_clustered(pairs):
    mul_relin_three_ways(pairs("n8192"), 0, 17, seed=0, adversarial=True)


def test_mr_split_side_streams(ref, monkeypatch):
    """B200_MR_SPLIT=2 (read at context creation): the two halves of a batch run multiply_relin_one on side streams"""
    from backends import CudaBackend
    monkeypatch.setenv("B200_MR_SPLIT", "2")
    P = pc.pair_for(CudaBackend(), "n8192")
    mul_relin_three_ways(P, 0, 130, seed=400)


# ---------------------------------------------------------------------------------------------------------------------
# which kernels ran: launch trace (B200_TRACE is read once per process).  The subprocess runs multiply_relin alone; its
# words are checked by the tests above.
# ---------------------------------------------------------------------------------------------------------------------
_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import parity_checks as pc
import test_gpu_scale_moddown as T
from backends import CudaBackend
P = pc.pair_for(CudaBackend(), {name!r})
rng = np.random.default_rng(5)
lv = P.ctx.first_level + {j}
k = P.ctx.level_info(lv)["k"]
A = pc.rand_ct(rng, P.moduli, k, P.n, batch={batch})
B = pc.rand_ct(rng, P.moduli, k, P.n, batch={batch})
o2 = P.out({batch}, 2, k, P.n)
P.ctx.multiply_relin(P.dev(A), P.dev(B), P.dev(pc.rand_ksk(rng, P.moduli, P.k, P.n)), o2, {batch}, level=lv)
P.host(o2)
print("fused", int(T.fused_expected(P, lv)), flush=True)
P.be.lib.lib.b200_trace_dump()
"""


def traced_multiply_relin(name, j, batch):
    env = dict(os.environ, B200_TRACE="1")
    for var in ("B200_MR_SPLIT", "B200_KS_CLUSTER", "B200_MUL_CLUSTER"):
        env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _TRACE.format(root=ROOT, tests=HERE, name=name, j=j, batch=batch)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    fused = bool(int(re.search(r"fused (\d)", r.stdout).group(1)))
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    count = lambda prefix: sum(v for key, v in launches.items() if key.startswith(prefix))
    return fused, launches, count


@pytest.mark.parametrize("name,j,batch", [("n8192", 0, 17), ("n8192", 0, 1), ("n8192", 3, 2), ("n4096_narrow", 0, 40),
                                          ("n16384", 3, 2)])
def test_trace_fp64_levels_run_the_fused_kernel(ref, name, j, batch):
    fused, launches, count = traced_multiply_relin(name, j, batch)
    assert fused, launches
    assert count("scale_moddown_kernel_v2") == 1, launches
    assert count("ksmoddown_kernel_v2") == 0, launches
    assert count("scale_kernel_v2") == 1, launches        # D2 only


def test_trace_n16384_top_level_keeps_the_separate_scale(ref):
    """k = 8: D beside the separate key switch's ks1 + ks2 would exceed the multiply's ext + D"""
    fused, launches, count = traced_multiply_relin("n16384", 0, 2)
    assert not fused, launches
    assert count("scale_moddown_kernel_v2") == 0, launches
    assert count("ksmoddown_kernel_v2") == 1 and count("scale_kernel_v2") == 1, launches


def test_trace_integer_path_keeps_the_old_pair(ref):
    fused, launches, count = traced_multiply_relin("n8192_54", 0, 2)
    assert not fused, launches
    assert count("scale_moddown_kernel_v2") == 0 and count("scale_kernel_v2") == 0, launches
    assert count("scale_kernel<") == 1 and count("ksmoddown_kernel_v2") == 1, launches
