"""The fused key switch (ks_cluster_kernel, sunscreen_b200/csrc/mul_cluster.cu) against the unmodified reference, on either
side of its dispatch rule, and the launch trace that shows which path ran (pytest -m gpu).

keyswitch_core runs the forward NTTs of the digits, the inner product with the key and the inverse NTTs as one k-CTA
cluster kernel for levels on the FP64 path at n <= 8192 with 2 <= k <= 8 when the launch fills the GPU:
k (k + 1) * batch > 2 * sm_count.  Below that, at k = 1, at n = 16384 and with B200_KS_CLUSTER=0 the separate kernels run.
relinearize, multiply_relin and apply_galois all go through keyswitch_core; every output word is compared with the
reference."""
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


def level_k(P, j):
    return P.ctx.level_info(P.ctx.first_level + j)["k"]


def last_separate_batch(k, sm_count):
    """the largest batch that still runs the separate kernels (keyswitch_core's rule)"""
    return (2 * sm_count) // (k * (k + 1))


def side_batch(k, sm_count, side):
    b = last_separate_batch(k, sm_count)
    return {"below": max(1, b), "at": b + 1, "above": 3 * (b + 1) + 1}[side]


def keyswitch_vs_reference(P, batch, seed, j=0, key=None, targets=None, elts=None):
    """relinearize of `batch` size-3 ciphertexts and apply_galois (default elements: 3 = rows, 2n - 1 = columns) of `batch`
    size-2 ciphertexts at data level j (0: the first level), item by item against the reference.  `targets` (optional):
    (size-3, size-2) word arrays replacing the random ones."""
    R = P.ref
    rng = np.random.default_rng(seed)
    lv = P.ctx.first_level + j
    k = level_k(P, j)
    if key is None:
        key = pc.rand_ksk(rng, P.moduli, P.k, P.n)
    if targets is None:
        C3 = pc.rand_ct(rng, P.moduli, k, P.n, size=3, batch=batch)
        C2 = pc.rand_ct(rng, P.moduli, k, P.n, batch=batch)
    else:
        C3, C2 = targets
    dK = P.dev(key)
    o2 = P.out(batch, 2, k, P.n)
    P.ctx.relinearize(P.dev(C3), dK, o2, batch, level=lv)
    got = P.host(o2).reshape(batch, 2, k, P.n)
    rlk = R.new_ksk({0: key})
    for i in range(batch):
        rc = R.new_ct(C3[i], level=j)
        rr = R.relinearize(rc, rlk)
        pc.eq(got[i], R.ct_words(rr), f"relinearize item {i} of {batch}, level {lv}")
        for h in (rc, rr):
            R.free_ct(h)
    dC2 = P.dev(C2)
    for elt in ((3, 2 * P.n - 1) if elts is None else elts):
        P.ctx.apply_galois(dC2, elt, dK, o2, batch, level=lv)
        got = P.host(o2).reshape(batch, 2, k, P.n)
        glk = R.new_ksk({(elt - 1) // 2: key})
        for i in range(batch):
            rc = R.new_ct(C2[i], level=j)
            rr = R.apply_galois(rc, elt, glk)
            pc.eq(got[i], R.ct_words(rr), f"apply_galois({elt}) item {i} of {batch}, level {lv}")
            for h in (rc, rr):
                R.free_ct(h)


@pytest.mark.parametrize("side", ["below", "at", "above"])
@pytest.mark.parametrize("name", ["n4096", "n8192"])
def test_keyswitch_around_the_cluster_threshold(pairs, name, side):
    P = pairs(name)
    sm = P.ctx.sm_count
    batch = side_batch(P.k, sm, side)
    assert (P.k * (P.k + 1) * batch > 2 * sm) == (side != "below")
    keyswitch_vs_reference(P, batch, seed=100 + batch)
    mul_relin_vs_reference(P, batch, seed=101 + batch, also_relinearize=True)


def test_multiply_relin_n8192_batch_1024(pairs):
    mul_relin_vs_reference(pairs("n8192"), 1024, seed=2048)


@pytest.mark.parametrize("j", [1, 2, 3])
def test_keyswitch_lower_levels_n8192(pairs, j):
    """k = 3 and k = 2 above their thresholds (cluster path); k = 1 has no cluster and takes the separate kernels"""
    P = pairs("n8192")
    k = level_k(P, j)
    assert k == P.k - j
    batch = side_batch(max(k, 2), P.ctx.sm_count, "above")
    keyswitch_vs_reference(P, batch, seed=110 + j, j=j)


@pytest.mark.parametrize("name", ["n4096_narrow", "n8192_49"])
def test_keyswitch_fp64_edge_chains(pairs, name):
    """~20-bit primes (k = 2) and 48/49-bit primes at the FP64 width limit (k = 3), above the threshold"""
    P = pairs(name)
    assert P.k == {"n4096_narrow": 2, "n8192_49": 3}[name]
    keyswitch_vs_reference(P, side_batch(P.k, P.ctx.sm_count, "above"), seed=120)


@pytest.mark.parametrize("name", ["n4096", "n8192"])
def test_adversarial_keyswitch_batched(pairs, name):
    """check_adversarial_keyswitch's cases with its all-(p-1) key, replicated over a batch above the threshold: relinearize
    of the qm1, alt and single targets, and (with a batching plain modulus) rotate_rows of qm1.  The accumulators are at
    their largest inside the cluster kernel."""
    P = pairs(name)
    K = len(P.moduli)
    key = np.empty((P.k, 2, K, P.n), dtype=np.uint64)
    for i in range(K):
        key[:, :, i, :] = np.uint64(int(P.moduli[i]) - 1)
    kinds = ("qm1", "alt", "single")
    batch = side_batch(P.k, P.ctx.sm_count, "above")
    C3 = np.stack([pc.adversarial_ct(P, kinds[i % 3], 3) for i in range(batch)])
    C2 = np.stack([pc.adversarial_ct(P, "qm1")] * batch)
    keyswitch_vs_reference(P, batch, seed=0, key=key, targets=(C3, C2), elts=(3,) if P.ctx.using_batching else ())


# ---------------------------------------------------------------------------------------------------------------------
# which kernels ran: launch trace (B200_TRACE and B200_KS_CLUSTER are read once per process)
# ---------------------------------------------------------------------------------------------------------------------
_TRACE = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import parity_checks as pc
import test_gpu_ks_cluster as T
from backends import CudaBackend
from params import PARAMS
P = pc.Pair(CudaBackend(), *PARAMS[{name!r}])
batch = T.side_batch(P.k, P.ctx.sm_count, {side!r})
T.keyswitch_vs_reference(P, batch, seed=7)
print("k", P.k, flush=True)
P.be.lib.lib.b200_trace_dump()
"""


def traced_launches(name, side, **env_extra):
    env = dict(os.environ, B200_TRACE="1", **env_extra)
    for var in ("B200_KS_CLUSTER", "B200_KSMAC_TMA"):
        if var not in env_extra:
            env.pop(var, None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _TRACE.format(root=ROOT, tests=HERE, name=name, side=side)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    k = int(re.search(r"k (\d+)", r.stdout).group(1))
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    # the separate path: forward NTT of k digits into k + 1 residues, the MAC, inverse NTT of 2 (k + 1) rows
    separate = (launches.get(f"ntt_fp_kernel<fwd> rows/item={k * (k + 1)}", 0),
                sum(v for key, v in launches.items() if key.startswith("ksmac")),
                launches.get(f"ntt_fp_kernel<inv> rows/item={2 * (k + 1)}", 0))
    return launches, separate


def test_trace_above_threshold_runs_the_cluster_kernel(ref):
    launches, separate = traced_launches("n8192", "above")
    assert launches.get("ks_cluster_kernel", 0) == 3, launches   # relinearize + two Galois elements
    assert separate == (0, 0, 0), launches


@pytest.mark.parametrize("name,side", [("n8192", "below"), ("n16384", "above")])
def test_trace_separate_kernels(ref, name, side):
    launches, separate = traced_launches(name, side)
    assert "ks_cluster_kernel" not in launches, launches
    assert separate[1] == 3, launches


def test_ks_cluster_off_runs_the_separate_kernels(ref):
    """B200_KS_CLUSTER=0: the same batch (words checked in the subprocess) runs the separate NTT, MAC and NTT kernels"""
    launches, separate = traced_launches("n8192", "above", B200_KS_CLUSTER="0")
    assert "ks_cluster_kernel" not in launches, launches
    assert separate == (3, 3, 3), launches


_PARTIAL = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import parity_checks as pc
import test_gpu_launch_shapes as T
from backends import CudaBackend
from params import PARAMS
P = pc.Pair(CudaBackend(), *PARAMS["n8192"])
batch = T._partial_batches(P)[{which}]
ipc = T.ksmac_items_per_chunk(P.n, P.k, batch, P.ctx.sm_count)
assert ipc < batch and batch % ipc, (batch, ipc)
T.mul_relin_vs_reference(P, batch, seed=80 + batch, also_relinearize=True)
P.be.lib.lib.b200_trace_dump()
"""


@pytest.mark.parametrize("which", [1, 2])
def test_ksmac_partial_last_chunk_without_cluster(ref, which):
    """the partial-last-chunk batches of test_ksmac_partial_last_chunk (17 and ~999) take the cluster kernel by default;
    with B200_KS_CLUSTER=0 they keep covering the TMA MAC's chunking"""
    env = dict(os.environ, B200_TRACE="1", B200_KS_CLUSTER="0")
    env.pop("B200_KSMAC_TMA", None)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
        ["-c", _PARTIAL.format(root=ROOT, tests=HERE, which=which)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"
    launches = {m.group(1): int(m.group(2)) for m in re.finditer(r"\[b200 trace\] (.+?)\s+launches\s+(\d+)", r.stderr)}
    assert launches.get("ksmac_tma_kernel", 0) >= 2, launches
    assert "ks_cluster_kernel" not in launches, launches
