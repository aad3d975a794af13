"""Long modulus chains (tests/params.py LONG) against the unmodified reference: every cluster size of the fused key switch
and up to 16 data residues on the FP64 path.

At n <= 8192 the chains walk k = 8 ... 1 (n8192_9x24, n4096_9x22) or k = 5 ... 1 with a special prime narrower than the data
primes (n8192_mixed_fp), so ks_cluster_kernel runs with clusters of every size 2 ... 8, mul_cluster_kernel up to
k + |Bsk| = 14 rows, and multiply_relin's fused scale and mod-down ((k + 1)(k + 2) <= 4 (k + |Bsk|)) on both sides of its
rule.  At n = 16384 the FP64 BEHZ kernels and the FP64 key-switch MAC run with K = 16 data residues, against 47- and 49-bit
auxiliary primes: the widest FP64 inner products (DESIGN.md section 4 gives their bound).  Every comparison is word for word;
the launch traces show which kernels ran.  test_emulation_top_level runs without a GPU: the test-only emulation build (no
cluster kernels) on the same chains."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from params import LONG, PARAMS
from test_gpu_ks_cluster import keyswitch_vs_reference, side_batch
from test_gpu_launch_shapes import ksmac_items_per_chunk
from test_gpu_mul_cluster import adversarial_batch
from test_gpu_scale_moddown import fused_expected, mul_relin_three_ways

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SMALL = [name for name in LONG if PARAMS[name][0] <= 8192]   # the cluster kernels' range
BIG = [name for name in LONG if PARAMS[name][0] == 16384]


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


def data_levels(P):
    return range(P.ctx.levels - P.ctx.first_level)


def level_kr(P, j):
    """(k, k + |Bsk|) of data level j"""
    li = P.ctx.level_info(P.ctx.first_level + j)
    return li["k"], li["k"] + li["nBsk"]


def ks_batch(P, j, side):
    """a batch on `side` ("below" / "at") of keyswitch_accumulate's cluster rule k (k + 1) batch > 2 sm_count (k = 1: that of k = 2)"""
    return side_batch(max(level_kr(P, j)[0], 2), P.ctx.sm_count, side)


def mul_batch(P, j):
    """the first batch above multiply_core's cluster rule 4 (k + |Bsk|) batch > 2 sm_count"""
    return 2 * P.ctx.sm_count // (4 * level_kr(P, j)[1]) + 1


def above_both(P, j):
    return max(mul_batch(P, j), ks_batch(P, j, "at"))


def all_pm1_key(P):
    key = np.empty((P.k, 2, len(P.moduli), P.n), dtype=np.uint64)
    for i, m in enumerate(P.moduli):
        key[:, :, i, :] = np.uint64(int(m) - 1)
    return key


def test_long_chains_cover_the_cluster_sizes():
    """the chains at n <= 8192 reach every key-switch cluster size 2 ... 8 at both transform sizes (checked here on the
    parameters; the traces below show the launches)"""
    sizes = {}
    for name in SMALL:
        n, m, _ = PARAMS[name]
        sizes.setdefault(n, set()).update(range(2, len(m)))
    assert sizes == {4096: set(range(2, 9)), 8192: set(range(2, 9))}, sizes


# ---------------------------------------------------------------------------------------------------------------------
# n <= 8192: every data level, on both sides of the cluster thresholds
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("side", ["below", "at"])
@pytest.mark.parametrize("name", SMALL)
def test_keyswitch_every_level(pairs, name, side):
    """relinearize and apply_galois(3, 2n - 1) at every data level, with the batch just below and just above
    k (k + 1) batch > 2 sm_count"""
    P = pairs(name)
    for j in data_levels(P):
        k = level_kr(P, j)[0]
        batch = ks_batch(P, j, side)
        assert (max(k, 2) * (max(k, 2) + 1) * batch > 2 * P.ctx.sm_count) == (side == "at") or batch == 1
        keyswitch_vs_reference(P, batch, seed=500 + 10 * j + batch, j=j)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_multiply_relin_every_level(pairs, name):
    """multiply_relin = multiply + relinearize = the reference at every data level, with a batch above the multiply's and
    the key switch's cluster rules, random and adversarial operands; check_batch at the top level"""
    P = pairs(name)
    sides = set()
    for j in data_levels(P):
        batch = above_both(P, j)
        mul_relin_three_ways(P, j, batch, seed=600 + j)
        mul_relin_three_ways(P, j, batch, seed=0, adversarial=True)
        if level_kr(P, j)[0] >= 2:
            sides.add(fused_expected(P, P.ctx.first_level + j))
    assert sides == {True, False}, sides    # both sides of the fused scale-and-mod-down rule next to the cluster key switch
    pc.check_batch(P, batch=above_both(P, 0), seed=601)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_adversarial_top_level(pairs, name):
    """check_adversarial_keyswitch's targets with its all-(p - 1) key, and check_adversarial_multiply's operand pairs, over
    a batch above both cluster rules at the top level (the widest key-switch cluster of the chain)"""
    P = pairs(name)
    batch = above_both(P, 0)
    kinds = ("qm1", "alt", "single")
    C3 = np.stack([pc.adversarial_ct(P, kinds[i % 3], 3) for i in range(batch)])
    C2 = np.stack([pc.adversarial_ct(P, "qm1")] * batch)
    keyswitch_vs_reference(P, batch, seed=0, key=all_pm1_key(P), targets=(C3, C2), elts=(3,) if P.ctx.using_batching else ())
    adversarial_batch(P, batch)


# ---------------------------------------------------------------------------------------------------------------------
# n = 16384: 16 data residues on the FP64 BEHZ and key-switch kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", BIG)
def test_n16384_every_level(pairs, name):
    P = pairs(name)
    li = P.ctx.level_info(P.ctx.first_level)
    assert P.k == 16 and all(q.bit_length() <= 49 for q in li["q"] + li["bsk"])      # every prime on the FP64 path
    for j in data_levels(P):
        mul_relin_three_ways(P, j, 3, seed=700 + j)


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIG)
def test_n16384_top_level(pairs, name):
    """k = 16: multiply with sizes, relinearize, the Galois elements, the adversarial operands and the all-(p - 1) key"""
    P = pairs(name)
    m3, rm = pc.check_multiply(P)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_adversarial_multiply(P, with_size5=False)
    pc.check_adversarial_keyswitch(P)
    mul_relin_three_ways(P, 0, 2, seed=0, adversarial=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIG)
def test_n16384_ksmac_batch_walk(pairs, name):
    """ksmac_tma_kernel's items per CTA at the top levels: at k = 16 the grid ((n / 256) (k + 1) CTAs) already fills
    8 sm_count on an H100, so each CTA walks the whole batch; at the first level below that threshold the batch is cut into
    chunks, the last one partial"""
    P = pairs(name)
    sm = P.ctx.sm_count
    split = None
    for j in data_levels(P):
        k = level_kr(P, j)[0]
        if (P.n // 256) * (k + 1) < 8 * sm:
            split = j
            break
    assert split is not None
    k = level_kr(P, split)[0]
    batch = next(b for b in range(17, 64) if ksmac_items_per_chunk(P.n, k, b, sm) < b and b % ksmac_items_per_chunk(P.n, k, b, sm))
    for j in sorted({0, split}):
        ipc = ksmac_items_per_chunk(P.n, level_kr(P, j)[0], batch, sm)
        assert (ipc < batch) == (j == split), (j, ipc, batch)
        mul_relin_three_ways(P, j, batch, seed=800 + j)


@pytest.mark.gpu
def test_n32768_twelve_residues(pairs):
    """the default n = 32768 chain three levels down (k = 12, integer path): the key tile of ksmac_tma_kernel is then exactly
    the 48 KiB a launch gets without opting in, next to the kernel's static shared memory (the FP64 instantiation at k = 12
    runs in test_n16384_every_level)"""
    P = pairs("n32768")
    j = next(j for j in data_levels(P) if level_kr(P, j)[0] == 12)
    keyswitch_vs_reference(P, 1, seed=900, j=j)


# ---------------------------------------------------------------------------------------------------------------------
# which kernels ran: launch traces (B200_TRACE is read once per process), one section per operation
# ---------------------------------------------------------------------------------------------------------------------
_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import parity_checks as pc
import test_gpu_long_chains as T
from test_gpu_scale_moddown import fused_expected
from backends import CudaBackend
P = pc.pair_for(CudaBackend(), {name!r})
rng = np.random.default_rng(9)
key = P.dev(pc.rand_ksk(rng, P.moduli, P.k, P.n))
P.be.lib.lib.b200_trace_dump()
for j in (T.data_levels(P) if {every} else [0]):
    lv = P.ctx.first_level + j
    k = P.ctx.level_info(lv)["k"]
    batch = T.ks_batch(P, j, "at")
    C3 = P.dev(pc.rand_ct(rng, P.moduli, k, P.n, size=3, batch=batch))
    o2 = P.out(batch, 2, k, P.n)
    P.ctx.relinearize(C3, key, o2, batch, level=lv)
    P.host(o2)
    print("@@ relinearize", j, k, 0, file=sys.stderr, flush=True)
    P.be.lib.lib.b200_trace_dump()
    batch = T.above_both(P, j) if P.n <= 8192 else 2
    A = P.dev(pc.rand_ct(rng, P.moduli, k, P.n, batch=batch))
    B = P.dev(pc.rand_ct(rng, P.moduli, k, P.n, batch=batch))
    o2 = P.out(batch, 2, k, P.n)
    P.ctx.multiply_relin(A, B, key, o2, batch, level=lv)
    P.host(o2)
    print("@@ multiply_relin", j, k, int(fused_expected(P, lv)), file=sys.stderr, flush=True)
    P.be.lib.lib.b200_trace_dump()
"""


def traced_levels(name, every=True):
    """[(op, j, k, fused, launches)] of relinearize and multiply_relin at every data level (or the top one) of `name`"""
    env = dict(os.environ, B200_TRACE="1")
    for var in ("B200_KS_CLUSTER", "B200_MUL_CLUSTER", "B200_KSMAC_TMA", "B200_MR_SPLIT",
                "B200_FORCE_AUX61", "B200_NO_STATIC_NTT"):
        env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _TRACE.format(root=ROOT, tests=HERE, name=name, every=every)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    out = []
    for line in r.stderr.splitlines():
        m = re.match(r"@@ (\w+) (\d+) (\d+) (\d)", line)
        if m:   # the trace dump of this operation follows its line
            out.append((m.group(1), int(m.group(2)), int(m.group(3)), bool(int(m.group(4))), {}))
            continue
        m = re.match(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", line)
        if m and out:
            out[-1][4][m.group(1)] = int(m.group(2))
    return out


def count(launches, prefix):
    return sum(v for key, v in launches.items() if key.startswith(prefix))


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_trace_cluster_sizes(ref, name):
    """ks_cluster_kernel runs at every k >= 2 of the chain (cudaOccupancyMaxActiveClusters accepts every size from 2 to 8),
    mul_cluster_kernel at every level, and multiply_relin takes scale_moddown_kernel_v2 exactly where fused_expected holds"""
    K = len(PARAMS[name][1])
    recs = traced_levels(name)
    assert len(recs) == 2 * (K - 1), recs
    ks_sizes, fused_sides = set(), set()
    for op, j, k, fused, launches in recs:
        clustered = count(launches, "ks_cluster_kernel")
        assert clustered == (1 if k >= 2 else 0), (op, j, k, launches)
        if clustered:
            ks_sizes.add(k)
            assert count(launches, "ksmac") == 0, (op, j, k, launches)
        if op == "multiply_relin":
            assert count(launches, "mul_cluster_kernel") == 1 and count(launches, "tensor_kernel") == 0, (j, k, launches)
            assert count(launches, "scale_kernel_v2") == 1 and count(launches, "scale_kernel<") == 0, (j, k, launches)
            assert count(launches, "scale_moddown_kernel_v2") == int(fused), (j, k, fused, launches)
            assert count(launches, "ksmoddown_kernel_v2") == int(not fused), (j, k, fused, launches)
            if k >= 2:
                fused_sides.add(fused)
    assert ks_sizes == set(range(2, K)), ks_sizes
    assert fused_sides == {True, False}, recs


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIG)
def test_trace_fp64_behz_at_k16(ref, name):
    """k = 16 at n = 16384: the FP64 lift and scale (not the integer lift_kernel / scale_kernel) and the FP64 TMA MAC"""
    recs = traced_levels(name, every=False)
    assert [(op, k) for op, _, k, _, _ in recs] == [("relinearize", 16), ("multiply_relin", 16)], recs
    for op, j, k, fused, launches in recs:
        assert count(launches, "ks_cluster_kernel") == 0 and count(launches, "ksmac_tma_kernel") == 1, (op, launches)
        assert count(launches, "ksmac_kernel") == 0, (op, launches)
        if op == "multiply_relin":
            assert count(launches, "lift_kernel_v2") == 1 and count(launches, "lift_kernel<") == 0, launches
            assert count(launches, "scale_kernel_v2") + count(launches, "scale_moddown_kernel_v2") >= 1, launches
            assert count(launches, "scale_kernel<") == 0, launches


# ---------------------------------------------------------------------------------------------------------------------
# without a GPU: the emulation build (separate kernels) on the same chains
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", LONG)
def test_emulation_top_level(emu_lib, ref, name):
    """check_context, and at every level the FP64 auxiliary base: as wide as the widest user prime (at least 47 bits), the
    reference's range condition met, and at most k + 2 primes (the size of the FP64 BEHZ constant blocks); then the top
    level's multiply, relinearize, Galois elements and adversarial key switch"""
    from backends import EmuBackend
    P = pc.pair_for(EmuBackend(emu_lib), name)
    pc.check_context(P)
    width = max(47, max(int(m).bit_length() for m in P.moduli))
    for lv in range(P.ctx.first_level, P.ctx.levels):
        li = P.ctx.level_info(lv)
        assert {p.bit_length() for p in li["bsk"]} == {width}, (lv, li["bsk"])
        assert math.prod(li["bsk"]).bit_length() > 32 + P.t.bit_length() + math.prod(li["q"]).bit_length(), lv
        assert li["nBsk"] <= li["k"] + 2, (lv, li["nBsk"], li["k"])
    m3, rm = pc.check_multiply(P)
    pc.check_relin(P, m3, rm)
    pc.check_galois(P)
    pc.check_adversarial_keyswitch(P)
