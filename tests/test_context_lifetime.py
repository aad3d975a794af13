"""Resource lifetime of the layer-1 context (b200_ctx), on the emulation build (tests/emu): b200_ctx_destroy releases every
stream, event, memory pool and allocation that b200_ctx_create and the operations made, and a b200_ctx_create that fails
part-way releases what it had made before it returns.  The emulation counts those resources (b200_emu_live_resources) and
can fail every creation after a budget (b200_emu_alloc_budget)."""
import ctypes as C
import gc
import itertools

import numpy as np
import pytest

from params import PARAMS
from sunscreen_b200.lib import B200_E_CUDA, B200Context

N, MODULI, T = PARAMS["n4096"]


@pytest.fixture
def live(emu_lib):
    """Number of resources the emulation holds.  The garbage collector is held off so that no other test's context is
    destroyed while one is being counted."""
    fn = emu_lib.lib.b200_emu_live_resources
    fn.argtypes, fn.restype = [], C.c_longlong
    gc.collect()
    gc.disable()
    yield fn
    gc.enable()


@pytest.fixture
def budget(emu_lib):
    fn = emu_lib.lib.b200_emu_alloc_budget
    fn.argtypes, fn.restype = [C.c_longlong], None
    yield fn
    fn(-1)


def rand_ct(rng, k, batch):
    out = np.empty((batch, 2, k, N), dtype=np.uint64)
    for i in range(k):
        out[:, :, i, :] = rng.integers(0, MODULI[i], size=(batch, 2, N), dtype=np.uint64)
    return out


def rand_key(rng, k):
    out = np.empty((k, 2, len(MODULI), N), dtype=np.uint64)
    for i in range(len(MODULI)):
        out[:, :, i, :] = rng.integers(0, MODULI[i], size=(k, 2, N), dtype=np.uint64)
    return out


def test_destroy_releases_everything(emu_lib, live, monkeypatch):
    """A context that ran multiply_relin, multiply_relin_host (plain staging, grown once, and packed staging) and
    apply_galois gives back everything at destroy, the side streams and their events included."""
    before = live()
    ctx = B200Context(N, MODULI, T, lib=emu_lib)
    k, batch = ctx.k(), 2
    rng = np.random.default_rng(3)
    a, b, key = rand_ct(rng, k, batch), rand_ct(rng, k, batch), rand_key(rng, k)
    want = np.zeros_like(a)
    ctx.multiply_relin(a, b, key, want, batch)
    for pack, chunk in (("0", "1"), ("0", "2"), ("1", "2")):
        monkeypatch.setenv("B200_HOST_PACK", pack)
        monkeypatch.setenv("B200_HOST_CHUNK", chunk)
        got = np.zeros_like(a)
        ctx.multiply_relin_host(a, b, key, got, batch)
        assert np.array_equal(got, want), f"multiply_relin_host, pack {pack}, chunk {chunk}"
    ctx.apply_galois(a, 3, key, np.zeros_like(a), batch)
    assert live() > before
    ctx.close()
    assert live() == before


def test_failed_create_releases_what_it_made(emu_lib, live, budget):
    """b200_ctx_create failing at each of its creations in turn returns B200_E_CUDA and leaves nothing behind."""
    L = emu_lib.lib
    mods = (C.c_uint64 * len(MODULI))(*MODULI)
    before = live()
    for made in itertools.count():
        h = C.c_void_p()
        budget(made)
        rc = L.b200_ctx_create(N, mods, len(MODULI), T, 0, C.byref(h))
        budget(-1)
        if rc == 0:
            break
        assert rc == B200_E_CUDA and not h.value, (made, rc)
        assert live() == before, f"create failing after {made} creations leaves {live() - before} behind"
    assert live() - before == made  # every creation of a successful create is held by the context
    L.b200_ctx_destroy(h)
    assert live() == before
