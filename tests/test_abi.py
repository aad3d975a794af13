"""The product shared library loads on a CPU-only machine, exports every symbol include/*.h declares, and
refuses to compute without a CUDA device (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sunscreen_b200", "libb200bfv.so")


@pytest.fixture(scope="module")
def product_lib():
    subprocess.run(["make", "-C", os.path.join(ROOT, "sunscreen_b200", "csrc")], check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.PIPE)
    return C.CDLL(LIB, mode=os.RTLD_LOCAL)


def declared_symbols():
    names = set()
    for fn in sorted(os.listdir(os.path.join(ROOT, "include"))):
        if not fn.endswith(".h"):
            continue
        text = open(os.path.join(ROOT, "include", fn)).read()
        text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
        for m in re.finditer(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\(", text):
            name = m.group(1)
            if name.startswith("b200_") or re.match(r"^[A-Z][A-Za-z]+_[A-Z]", name):
                names.add(name)
    return sorted(names)


def test_exports_every_declared_symbol(product_lib):
    missing = [s for s in declared_symbols() if not hasattr(product_lib, s)]
    assert not missing, missing
    assert len(declared_symbols()) >= 30


def test_is_sm90a_cuda_build():
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-lelf", LIB], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_no_cpu_fallback(product_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present")
    ctx = C.c_void_p()
    mods = (C.c_uint64 * 3)(0xffffee001, 0xffffc4001, 0x1ffffe0001)
    product_lib.b200_ctx_create.argtypes = [C.c_uint64, C.POINTER(C.c_uint64), C.c_uint64, C.c_uint64, C.c_int,
                                            C.POINTER(C.c_void_p)]
    rc = product_lib.b200_ctx_create(4096, mods, 3, 262144, 0, C.byref(ctx))
    assert rc == -3  # B200_E_CUDA
    product_lib.b200_last_error.restype = C.c_char_p
    assert b"no CPU fallback" in product_lib.b200_last_error()


def test_package_refuses_emu_build(emu_lib):
    from sunscreen_b200.lib import B200Lib
    with pytest.raises(ImportError):
        B200Lib(emu_lib.path)
