"""sunscreen_b200 — an H100-native BFV ciphertext-arithmetic backend behind Sunscreen's `seal_fhe` FFI.

The product is the CUDA shared library `libb200bfv.so` (built in-tree from `csrc/`); the Python modules are plumbing:
    lib       ctypes binding of the layer-1 "slab" C ABI        (include/b200_bfv.h)
    seal_fhe  Python mirror of the seal_fhe Rust crate's API     (over include/b200_sealc.h)
    sharding  batch sharding across GPUs (scatter / per-rank compute / gather)
"""
from .lib import B200Context, B200Error, B200Lib  # noqa: F401
