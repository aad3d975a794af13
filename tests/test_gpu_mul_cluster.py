"""The fused tensor product of a size-2 x size-2 multiply (mul_cluster_kernel, sunscreen_b200/csrc/mul_cluster.cu) against the
unmodified reference, on either side of its dispatch rule, and the launch trace that shows which path ran (pytest -m gpu).

multiply_core runs forward NTTs, dyadic product and inverse NTTs as one 4-CTA cluster kernel for chains on the FP64 path at
n <= 8192 when the launch fills the GPU: 4 (k + |Bsk|) * batch > 2 * sm_count.  Below that, at n = 16384, for squares and
other sizes, and with B200_MUL_CLUSTER=0 the separate kernels run.  Every output word is compared with the reference."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import parity_checks as pc
from params import PARAMS
from test_gpu_launch_shapes import mul_relin_vs_reference

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FP_PRIME_BITS = 49  # host_ctx.h: primes up to this width take the FP64 kernels

# every parameter set at n <= 8192 whose data and auxiliary primes all take the FP64 path (asserted in fp_chain below)
CLUSTER_SETS = ["n4096", "n8192", "n8192_49", "n4096_narrow", "n4096_q_below_t"]


@pytest.fixture(scope="module")
def pairs(ref):
    from backends import CudaBackend
    be = CudaBackend()
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = pc.Pair(be, *PARAMS[name])
        return cache[name]
    return get


def rows(P):
    return P.k + len(P.ctx.level_info(P.ctx.first_level)["bsk"])


def last_separate_batch(P):
    """the largest batch that still runs the separate kernels (multiply_core's rule)"""
    return (2 * P.ctx.sm_count) // (4 * rows(P))


def fp_chain(P):
    li = P.ctx.level_info(P.ctx.first_level)
    return all(int(p).bit_length() <= FP_PRIME_BITS for p in li["q"] + li["bsk"] + [li["m_sk"]])


def side_batch(P, side):
    b = last_separate_batch(P)
    return {"below": max(1, b), "at": b + 1, "above": 3 * (b + 1) + 1}[side]


def adversarial_batch(P, batch):
    """multiply and multiply_relin of `batch` items cycling through check_adversarial_multiply's operand pairs"""
    kinds = [("qm1", "qm1"), ("qm1", "alt"), ("alt", "pm1"), ("pm1", "pm1"), ("single", "qm1"), ("single", "single"),
             ("one", "qm1"), ("alt", "alt")]
    R = P.ref
    rlk = R.new_ksk({0: P.inp["rlk"]})
    exp3, exp2, A, B = {}, {}, [], []
    for ka, kb in kinds:
        a, b = pc.adversarial_ct(P, ka), pc.adversarial_ct(P, kb)
        ra, rb = R.new_ct(a), R.new_ct(b)
        rm = R.multiply(ra, rb)
        exp3[(ka, kb)], exp2[(ka, kb)] = R.ct_words(rm), R.ct_words(R.relinearize(rm, rlk))
        for h in (ra, rb, rm):
            R.free_ct(h)
        A.append(a)
        B.append(b)
    idx = [i % len(kinds) for i in range(batch)]
    dA, dB = P.dev(np.stack([A[i] for i in idx])), P.dev(np.stack([B[i] for i in idx]))
    o3 = P.out(batch, 3, P.k, P.n)
    P.ctx.multiply(dA, 2, dB, 2, o3, batch)
    o2 = P.out(batch, 2, P.k, P.n)
    P.ctx.multiply_relin(dA, dB, P.dev(P.inp["rlk"]), o2, batch)
    got3, got2 = P.host(o3), P.host(o2)
    for j, i in enumerate(idx):
        pc.eq(got3[j], exp3[kinds[i]], f"multiply{kinds[i]} item {j} of {batch}")
        pc.eq(got2[j], exp2[kinds[i]], f"multiply_relin{kinds[i]} item {j} of {batch}")


@pytest.mark.parametrize("name", CLUSTER_SETS)
def test_cluster_sets_take_the_fp64_path(pairs, name):
    assert fp_chain(pairs(name))


@pytest.mark.parametrize("side", ["below", "at", "above"])
@pytest.mark.parametrize("name", CLUSTER_SETS)
def test_multiply_around_the_cluster_threshold(pairs, name, side):
    P = pairs(name)
    batch = side_batch(P, side)
    assert (4 * rows(P) * batch > 2 * P.ctx.sm_count) == (side != "below") or batch == 1
    pc.check_batch(P, batch=batch, seed=90 + batch)
    mul_relin_vs_reference(P, batch, seed=91 + batch, also_relinearize=True)
    adversarial_batch(P, batch)
    # batch-1 calls (separate kernels) in between: the two paths share the context's job tables and scratch pool
    m3, rm = pc.check_multiply(P)
    pc.check_relin(P, m3, rm)


def test_multiply_relin_n8192_batch_1024(pairs):
    mul_relin_vs_reference(pairs("n8192"), 1024, seed=1024)


def test_batch_seam_replayed(ref):
    """B200_Evaluator_MultiplyRelinBatch at batch 64 (cluster path) called repeatedly: every call gives, item by item, the
    words of the per-handle Evaluator_Multiply + Evaluator_Relinearize (separate kernels at batch 1)."""
    import refseal
    from sealc_driver import Sealc
    from sunscreen_b200.lib import B200Lib
    S = Sealc(B200Lib.default().lib)
    n, moduli, t = PARAMS["n8192"]
    O = S.context(n, moduli, t)
    rlk = O.new_ksk({0: refseal.appendix_b_inputs(n, moduli, t)["rlk"]})
    rng = np.random.default_rng(64)
    count = 64
    As, Bs, exp = [], [], []
    for _ in range(count):
        a = np.stack([rng.integers(0, moduli[r], size=(2, n), dtype=np.uint64) for r in range(O.k)], axis=1)
        b = np.stack([rng.integers(0, moduli[r], size=(2, n), dtype=np.uint64) for r in range(O.k)], axis=1)
        ha, hb = O.new_ct(a), O.new_ct(b)
        As.append(ha)
        Bs.append(hb)
        exp.append(O.ct_words(O.relinearize(O.multiply(ha, hb), rlk)))
    vp = C.c_void_p
    for rep in range(3):
        dsts = [O._dst() for _ in range(count)]
        O.S.call("B200_Evaluator_MultiplyRelinBatch", O.ev, C.c_uint64(count), (vp * count)(*As), (vp * count)(*Bs), rlk,
                 (vp * count)(*dsts))
        for i, (d, e) in enumerate(zip(dsts, exp)):
            assert np.array_equal(O.ct_words(d), e), f"call {rep}, item {i}"


# ---------------------------------------------------------------------------------------------------------------------
# which kernels ran: launch trace (B200_TRACE and B200_MUL_CLUSTER are read once per process)
# ---------------------------------------------------------------------------------------------------------------------
_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import parity_checks as pc
import test_gpu_mul_cluster as T
from test_gpu_launch_shapes import mul_relin_vs_reference
from backends import CudaBackend
from params import PARAMS
P = pc.Pair(CudaBackend(), *PARAMS[{name!r}])
batch = T.side_batch(P, {side!r})
mul_relin_vs_reference(P, batch, seed=5, also_relinearize=True)
print("rows", T.rows(P), flush=True)
P.be.lib.lib.b200_trace_dump()
"""


def traced_launches(name, side, **env_extra):
    env = dict(os.environ, B200_TRACE="1", **env_extra)
    for var in ("B200_MUL_CLUSTER",):
        if var not in env_extra:
            env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _TRACE.format(root=ROOT, tests=HERE, name=name, side=side)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    R = int(re.search(r"rows (\d+)", r.stdout).group(1))
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    # the separate path's product: tensor kernel + inverse NTT of the 3 R rows of D (multiply_relin + multiply: 2 each)
    separate = (sum(v for key, v in launches.items() if key.startswith("tensor_kernel")),
                launches.get(f"ntt_fp_kernel<inv> rows/item={3 * R}", 0))
    return launches, separate


def test_trace_above_threshold_runs_the_cluster_kernel(ref):
    launches, separate = traced_launches("n8192", "above")
    assert launches.get("mul_cluster_kernel", 0) == 2, launches
    assert separate == (0, 0), launches


@pytest.mark.parametrize("name,side", [("n8192", "below"), ("n16384", "above")])
def test_trace_separate_kernels(ref, name, side):
    launches, separate = traced_launches(name, side)
    assert "mul_cluster_kernel" not in launches, launches
    assert separate[0] == 2, launches


def test_mul_cluster_off_runs_the_separate_kernels(ref):
    """B200_MUL_CLUSTER=0: the same batch (words checked in the subprocess) runs the separate tensor and inverse kernels"""
    launches, separate = traced_launches("n8192", "above", B200_MUL_CLUSTER="0")
    assert "mul_cluster_kernel" not in launches, launches
    assert separate == (2, 2), launches
