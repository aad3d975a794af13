"""Host-side model of the group enumeration of the statically scheduled FP64 transform (sunscreen_b200/csrc/ntt_fp_body.cuh,
NttFpStaticPass: `gidx`, `WP_TG`, `WP_NG`) — the invariants the warp(-group)-private passes rely on, checked for every
instantiated shape without a GPU:
  * every pass enumerates each butterfly group exactly once;
  * after the first forward pass (before the last inverse pass) the groups a warp group handles touch ONLY the elements of that
    group's own block(s), in every remaining pass — which is why a __syncwarp / named barrier of that group is enough between them;
  * the write-out / copy-in of a group covers exactly its block(s).
The kernels themselves are compared bit for bit with the reference by the GPU parity tests, whose batch sizes reach every
shape through the launcher's automatic choice (tests/test_gpu_launch_shapes.py: both sides of the n = 8192 width switch and
of the n = 16384 persistent grid)."""
import pytest

SCHED = {12: (4, 4, 4), 13: (3, 3, 3, 4), 14: (3, 3, 4, 4)}   # NttSched<LOGN>: stages per forward pass
SHAPES = [(12, 256), (13, 256), (13, 512), (14, 1024)]          # (LOGN, threads per CTA) of the kernels (ntt_fp_kernels.cu)


def wp_geometry(logn, nt):
    blocks, warps = 1 << SCHED[logn][0], nt // 32
    tg = 32 * (warps // blocks) if warps > blocks else 32       # threads of one group
    ng = nt // tg                                               # groups in the CTA
    ok = blocks % ng == 0 and ng <= 15
    return tg, ng, ok


def group_elements(logn, done, L, g):
    """elements of butterfly group g of the pass that starts after `done` forward stages and spans L stages"""
    logs = logn - done - L
    i, o = g >> logs, g & ((1 << logs) - 1)
    base = (i << (logs + L)) + o
    return [base + (j << logs) for j in range(1 << L)]


@pytest.mark.parametrize("logn,nt", SHAPES)
def test_warp_private_passes_stay_inside_their_block(logn, nt):
    n = 1 << logn
    tg, ng, ok = wp_geometry(logn, nt)
    assert ok, "shape must qualify for the warp-private variant"
    sched = SCHED[logn]
    bs = n // ng                                                # elements owned by one thread group
    done = 0
    for pidx, L in enumerate(sched):
        ngroups = n >> L
        assert ngroups % nt == 0 or ngroups < nt
        iters = max(1, ngroups // nt)
        private = pidx >= 1                                     # forward: every pass after the first (the inverse mirrors it)
        seen = set()
        for tid in range(nt):
            grp, lane = tid // tg, tid % tg
            for it in range(iters):
                g = grp * (ngroups // ng) + lane + tg * it if private else tid + it * nt
                if g >= ngroups:
                    continue
                assert g not in seen
                seen.add(g)
                if private:
                    for e in group_elements(logn, done, L, g):
                        assert grp * bs <= e < (grp + 1) * bs, (logn, nt, pidx, tid, g, e)
        assert len(seen) == ngroups, "every group exactly once"
        done += L
    # write-out (forward) / copy-in (inverse) of a thread group covers exactly its block(s)
    for grp in range(ng):
        cover = sorted(grp * bs + lane + tg * r for lane in range(tg) for r in range(bs // tg))
        assert cover == list(range(grp * bs, (grp + 1) * bs))


def test_first_pass_mixes_all_blocks():
    """the reason ONE block-wide barrier per polynomial remains: a first-pass group has one element in every block"""
    logn, L0 = 13, SCHED[13][0]
    n, nblocks = 1 << logn, 1 << L0
    for g in (0, 1, 1023):
        owners = {e // (n // nblocks) for e in group_elements(logn, 0, L0, g)}
        assert owners == set(range(nblocks))
