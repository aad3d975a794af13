"""ctypes binding of the layer-1 C ABI (include/b200_bfv.h) — plumbing, not the product.

The product is sunscreen_b200/libb200bfv.so (CUDA, sm_90a).  This module only loads it, declares the
signatures and turns error codes into exceptions; buffers are raw device pointers (ints), typically
`torch.Tensor.data_ptr()` of a CUDA tensor.  There is no CPU fallback: if the shared library is missing or
was not built by nvcc for sm_90a, loading fails loudly.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200bfv.so")

B200_OK, B200_E_INVALID, B200_E_LOGIC, B200_E_CUDA, B200_E_NULL, B200_E_NOMEM = 0, -1, -2, -3, -4, -5
# lift rules of b200_plain_to_ntt
PLAIN_NTT_TRANSFORM, PLAIN_NTT_MULTIPLY = 0, 1

vp = C.c_void_p
u64 = C.c_uint64
u64p = C.POINTER(C.c_uint64)


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"b200 error {code}: {msg}")
        self.code = code


class Info(C.Structure):
    _fields_ = [("n", u64), ("plain_modulus", u64), ("key_primes", C.c_int32), ("levels", C.c_int32),
                ("first_level", C.c_int32), ("using_batching", C.c_int32), ("device", C.c_int32),
                ("sm_count", C.c_int32)]


class LevelInfo(C.Structure):
    _fields_ = [("k", C.c_int32), ("nB", C.c_int32), ("nBsk", C.c_int32), ("parms_id", u64 * 4), ("m_sk", u64),
                ("gamma", u64), ("q", u64 * 64), ("bsk", u64 * 66), ("roots", u64 * 64), ("delta", u64 * 64),
                ("q_mod_t", u64)]


_SIGS = {
    "b200_ctx_create": [u64, u64p, u64, u64, C.c_int, C.POINTER(vp)],
    "b200_ctx_info": [vp, C.POINTER(Info)],
    "b200_ctx_level_info": [vp, C.c_int, C.POINTER(LevelInfo)],
    "b200_galois_elt_from_step": [vp, C.c_int, C.POINTER(C.c_uint32)],
    "b200_malloc": [vp, C.c_size_t, C.POINTER(vp)],
    "b200_free": [vp, vp],
    "b200_malloc_host": [C.c_size_t, C.POINTER(vp)],
    "b200_free_host": [vp],
    "b200_memcpy_h2d": [vp, vp, vp, C.c_size_t, vp],
    "b200_memcpy_d2h": [vp, vp, vp, C.c_size_t, vp],
    "b200_memcpy_d2d": [vp, vp, vp, C.c_size_t, vp],
    "b200_memzero": [vp, vp, C.c_size_t, vp],
    "b200_debug_ntt_variant": [C.c_int],
    "b200_debug_ntt_ctas_per_sm": [C.c_int, C.c_int, C.c_int, C.c_int],
    "b200_debug_ntt_stagger": [C.c_int],
    "b200_gather_scatter_table": [vp, vp, u64, vp, u64, C.c_int, vp],
    "b200_malloc_async": [vp, C.c_size_t, C.POINTER(vp), vp],
    "b200_bind_thread": [vp],
    "b200_stream_synchronize_blocking": [vp, vp, C.POINTER(vp)],
    "b200_event_destroy": [vp, vp],
    "b200_capture_begin": [vp, vp],
    "b200_capture_end": [vp, vp, C.POINTER(vp)],
    "b200_graph_launch": [vp, vp, vp],
    "b200_graph_destroy": [vp, vp],
    "b200_stream_synchronize": [vp, vp],
    "b200_ntt_forward": [vp, C.c_int, vp, u64, vp],
    "b200_ntt_inverse": [vp, C.c_int, vp, u64, vp],
    "b200_add": [vp, C.c_int, vp, vp, vp, C.c_int, u64, vp],
    "b200_sub": [vp, C.c_int, vp, vp, vp, C.c_int, u64, vp],
    "b200_negate": [vp, C.c_int, vp, vp, C.c_int, u64, vp],
    "b200_multiply": [vp, C.c_int, vp, C.c_int, vp, C.c_int, vp, u64, vp],
    "b200_square": [vp, C.c_int, vp, vp, u64, vp],
    "b200_relinearize": [vp, C.c_int, vp, vp, vp, u64, vp],
    "b200_multiply_relin": [vp, C.c_int, vp, vp, vp, vp, u64, vp],
    "b200_apply_galois": [vp, C.c_int, vp, C.c_uint32, vp, vp, u64, vp],
    "b200_apply_galois_add": [vp, C.c_int, vp, C.c_uint32, vp, vp, vp, u64, vp],
    "b200_multiply_relin_sum": [vp, C.c_int, vp, vp, vp, u64, vp, u64, vp],
    "b200_multiply_plain": [vp, C.c_int, vp, C.c_int, vp, u64, vp, u64, vp],
    "b200_plain_to_ntt": [vp, C.c_int, vp, u64, vp, C.c_int, vp],
    "b200_multiply_plain_sum": [vp, C.c_int, vp, C.c_int, u64, vp, u64, vp, vp],
    "b200_apply_galois_many": [vp, C.c_int, vp, vp, vp, vp, vp, u64, vp],
    "b200_linear_transform": [vp, C.c_int, vp, u64, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp],
    "b200_add_plain": [vp, C.c_int, vp, C.c_int, vp, u64, vp, u64, vp],
    "b200_sub_plain": [vp, C.c_int, vp, C.c_int, vp, u64, vp, u64, vp],
    "b200_mod_switch_to_next": [vp, C.c_int, vp, C.c_int, vp, u64, vp],
    "b200_decrypt": [vp, C.c_int, vp, C.c_int, vp, vp, u64, vp],
    "b200_ct_sk_phase": [vp, C.c_int, vp, C.c_int, vp, vp, u64, vp],
    "b200_noise_norm": [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int, u64, vp],
    "b200_is_transparent": [vp, C.c_int, vp, C.c_int, vp, u64, vp],
    "b200_any_nonzero": [vp, C.c_int, vp, C.c_int, vp, u64, vp],
    "b200_expand_signed": [vp, C.c_int, vp, C.c_int, vp, vp],
    "b200_multiply_relin_host": [vp, C.c_int, vp, vp, vp, vp, u64],
    "b200_ntt_roundtrip_host": [vp, C.c_int, vp, vp, u64],
}

EXPORTS = sorted(list(_SIGS) + ["b200_last_error", "b200_device_count", "b200_ctx_destroy", "b200_launch_count"])


class B200Lib:
    """The loaded shared library.  `path` is only overridden by the test-suite (tests/emu)."""

    _default = None

    @classmethod
    def default(cls):
        if cls._default is None:
            cls._default = cls()
        return cls._default

    def __init__(self, path=None, _allow_emu=False):
        path = path or LIB_PATH
        if not os.path.exists(path):
            raise ImportError(
                f"{path} not found: build it with __graft_entry__.build() / make -C sunscreen_b200/csrc "
                "(the CUDA backend has no CPU fallback)")
        if not _allow_emu and "emu" in os.path.basename(path):
            raise ImportError("refusing to load a tests/emu build as the product library")
        self.path = path
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        for name, args in _SIGS.items():
            fn = getattr(self.lib, name)
            fn.argtypes = args
            fn.restype = C.c_int
        self.lib.b200_last_error.restype = C.c_char_p
        self.lib.b200_device_count.restype = C.c_int
        self.lib.b200_ctx_destroy.argtypes = [vp]
        self.lib.b200_ctx_destroy.restype = None
        self.lib.b200_launch_count.argtypes = [vp]
        self.lib.b200_launch_count.restype = u64

    def check(self, rc):
        if rc != 0:
            raise B200Error(rc, self.lib.b200_last_error().decode())

    def call(self, name, *args):
        self.check(getattr(self.lib, name)(*args))

    def device_count(self):
        return int(self.lib.b200_device_count())


def ptr(x):
    """Raw address of a torch tensor / numpy array / int."""
    if x is None:
        return None
    if isinstance(x, int):
        return x
    if hasattr(x, "data_ptr"):
        return x.data_ptr()
    if hasattr(x, "ctypes"):
        return x.ctypes.data
    raise TypeError(type(x))


class B200Context:
    """One BFV parameter set resident on one GPU (b200_ctx)."""

    def __init__(self, poly_modulus_degree, coeff_modulus, plain_modulus, device=0, lib=None):
        self.L = lib or B200Lib.default()
        arr = (u64 * len(coeff_modulus))(*[int(m) for m in coeff_modulus])
        h = vp()
        self.L.call("b200_ctx_create", u64(poly_modulus_degree), arr, u64(len(coeff_modulus)), u64(plain_modulus),
                    C.c_int(device), C.byref(h))
        self.h = h
        info = Info()
        self.L.call("b200_ctx_info", h, C.byref(info))
        self.n = int(info.n)
        self.t = int(info.plain_modulus)
        self.K = int(info.key_primes)
        self.levels = int(info.levels)
        self.first_level = int(info.first_level)
        self.using_batching = bool(info.using_batching)
        self.device = int(info.device)
        self.sm_count = int(info.sm_count)
        self.key_moduli = [int(m) for m in coeff_modulus]

    def close(self):
        if getattr(self, "h", None):
            self.L.lib.b200_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def level_info(self, level):
        li = LevelInfo()
        self.L.call("b200_ctx_level_info", self.h, C.c_int(level), C.byref(li))
        k = li.k
        return dict(k=k, nB=li.nB, nBsk=li.nBsk, parms_id=[int(x) for x in li.parms_id], m_sk=int(li.m_sk),
                    gamma=int(li.gamma), q=[int(x) for x in li.q[:k]], bsk=[int(x) for x in li.bsk[:li.nBsk]],
                    roots=[int(x) for x in li.roots[:k]], delta=[int(x) for x in li.delta[:k]], q_mod_t=int(li.q_mod_t))

    def k(self, level=None):
        return self.level_info(self.first_level if level is None else level)["k"]

    def galois_elt_from_step(self, steps):
        e = C.c_uint32()
        self.L.call("b200_galois_elt_from_step", self.h, C.c_int(steps), C.byref(e))
        return int(e.value)

    def launch_count(self):
        return int(self.L.lib.b200_launch_count(self.h))

    # raw memory helpers
    def malloc(self, nbytes):
        p = vp()
        self.L.call("b200_malloc", self.h, C.c_size_t(nbytes), C.byref(p))
        return p.value

    def free(self, p):
        self.L.call("b200_free", self.h, vp(p))

    def h2d(self, dst, src, nbytes, stream=None):
        self.L.call("b200_memcpy_h2d", self.h, vp(ptr(dst)), vp(ptr(src)), C.c_size_t(nbytes), vp(stream))

    def d2h(self, dst, src, nbytes, stream=None):
        self.L.call("b200_memcpy_d2h", self.h, vp(ptr(dst)), vp(ptr(src)), C.c_size_t(nbytes), vp(stream))

    def sync(self, stream=None):
        self.L.call("b200_stream_synchronize", self.h, vp(stream))

    # ops (device pointers)
    def _lv(self, level):
        return C.c_int(self.first_level if level is None else level)

    def ntt_forward(self, data, items, level=None, stream=None):
        self.L.call("b200_ntt_forward", self.h, self._lv(level), vp(ptr(data)), u64(items), vp(stream))

    def ntt_inverse(self, data, items, level=None, stream=None):
        self.L.call("b200_ntt_inverse", self.h, self._lv(level), vp(ptr(data)), u64(items), vp(stream))

    def add(self, a, b, out, size, batch, level=None, stream=None):
        self.L.call("b200_add", self.h, self._lv(level), vp(ptr(a)), vp(ptr(b)), vp(ptr(out)), C.c_int(size), u64(batch),
                    vp(stream))

    def sub(self, a, b, out, size, batch, level=None, stream=None):
        self.L.call("b200_sub", self.h, self._lv(level), vp(ptr(a)), vp(ptr(b)), vp(ptr(out)), C.c_int(size), u64(batch),
                    vp(stream))

    def negate(self, a, out, size, batch, level=None, stream=None):
        self.L.call("b200_negate", self.h, self._lv(level), vp(ptr(a)), vp(ptr(out)), C.c_int(size), u64(batch), vp(stream))

    def multiply(self, a, sa, b, sb, out, batch, level=None, stream=None):
        self.L.call("b200_multiply", self.h, self._lv(level), vp(ptr(a)), C.c_int(sa), vp(ptr(b)), C.c_int(sb), vp(ptr(out)),
                    u64(batch), vp(stream))

    def square(self, a, out, batch, level=None, stream=None):
        self.L.call("b200_square", self.h, self._lv(level), vp(ptr(a)), vp(ptr(out)), u64(batch), vp(stream))

    def relinearize(self, in3, rlk, out2, batch, level=None, stream=None):
        self.L.call("b200_relinearize", self.h, self._lv(level), vp(ptr(in3)), vp(ptr(rlk)), vp(ptr(out2)), u64(batch),
                    vp(stream))

    def multiply_relin(self, a, b, rlk, out2, batch, level=None, stream=None):
        self.L.call("b200_multiply_relin", self.h, self._lv(level), vp(ptr(a)), vp(ptr(b)), vp(ptr(rlk)), vp(ptr(out2)),
                    u64(batch), vp(stream))

    def multiply_relin_sum(self, a, b, rlk, m, out2, rows, level=None, stream=None):
        """out2[r] = sum_j relinearize(multiply(a[r][j], b[r][j])): a, b [rows][m][2][k][n] (b may be a: squares), out2
        [rows][2][k][n], which must not overlap a or b."""
        self.L.call("b200_multiply_relin_sum", self.h, self._lv(level), vp(ptr(a)), vp(ptr(b)), vp(ptr(rlk)), u64(m),
                    vp(ptr(out2)), u64(rows), vp(stream))

    def apply_galois(self, in2, elt, key, out2, batch, level=None, stream=None):
        self.L.call("b200_apply_galois", self.h, self._lv(level), vp(ptr(in2)), C.c_uint32(elt), vp(ptr(key)), vp(ptr(out2)),
                    u64(batch), vp(stream))

    def apply_galois_add(self, in2, elt, key, addend2, out2, batch, level=None, stream=None):
        """out2 = addend2 + apply_galois(in2, elt) (addend2 None: no addend); addend2 may be in2 or out2, out2 must not overlap in2."""
        self.L.call("b200_apply_galois_add", self.h, self._lv(level), vp(ptr(in2)), C.c_uint32(elt), vp(ptr(key)),
                    vp(ptr(addend2)), vp(ptr(out2)), u64(batch), vp(stream))

    def apply_galois_many(self, in2, src_idx, elts, keys, out2, level=None, stream=None):
        """out2[i] = apply_galois(in2[src_idx[i]], elts[i]) with key list keys[i] (src_idx None: item i), one key switch for
        all items; out2 must not overlap the sources."""
        batch = len(elts)
        src = (u64 * max(batch, 1))(*([int(x) for x in src_idx] if src_idx is not None else []))
        el = (C.c_uint32 * max(batch, 1))(*[int(e) for e in elts])
        ks = (vp * max(batch, 1))(*[ptr(key) for key in keys])
        self.L.call("b200_apply_galois_many", self.h, self._lv(level), vp(ptr(in2)), src if src_idx is not None else None, el, ks,
                    vp(ptr(out2)), u64(batch), vp(stream))

    def linear_transform(self, cts, V, baby, giant, elts, keys, plain_ntt, out, present=None, level=None, stream=None):
        """Baby-step giant-step slot-wise linear transform (see bsgs_plain_vectors): cts, out [V][2][k][n]; elts, keys the
        baby - 1 baby-step then giant - 1 giant-step elements and device key lists (None where no present term uses the step);
        plain_ntt [giant][baby][k][n] from plain_to_ntt(rule=PLAIN_NTT_MULTIPLY); present [giant][baby] booleans or None."""
        ns = baby - 1 + giant - 1
        el = (C.c_uint32 * max(ns, 1))(*[int(e or 0) for e in elts])
        ks = (vp * max(ns, 1))(*[ptr(key) for key in keys])
        pr = None
        if present is not None:
            flat = [1 if x else 0 for row in present for x in row]
            pr = (C.c_uint8 * len(flat))(*flat)
        self.L.call("b200_linear_transform", self.h, self._lv(level), vp(ptr(cts)), u64(V), C.c_int(baby), C.c_int(giant), el, ks,
                    vp(ptr(plain_ntt)), pr, vp(ptr(out)), vp(stream))

    def multiply_plain(self, a, size, plain, plain_batch, out, batch, level=None, stream=None):
        self.L.call("b200_multiply_plain", self.h, self._lv(level), vp(ptr(a)), C.c_int(size), vp(ptr(plain)),
                    u64(plain_batch), vp(ptr(out)), u64(batch), vp(stream))

    def plain_to_ntt(self, plain, plain_batch, out, rule=PLAIN_NTT_TRANSFORM, level=None, stream=None):
        """plain [plain_batch][n] -> out [plain_batch][k][n] in NTT form (rule: PLAIN_NTT_TRANSFORM or PLAIN_NTT_MULTIPLY)."""
        self.L.call("b200_plain_to_ntt", self.h, self._lv(level), vp(ptr(plain)), u64(plain_batch), vp(ptr(out)), C.c_int(rule),
                    vp(stream))

    def multiply_plain_sum(self, cts, size, m, plain_ntt, R, out, level=None, stream=None):
        """out[i] = sum_j multiply_plain(cts[j], plain i,j): cts [m][size][k][n], plain_ntt [R][m][k][n] from plain_to_ntt,
        out [R][size][k][n]."""
        self.L.call("b200_multiply_plain_sum", self.h, self._lv(level), vp(ptr(cts)), C.c_int(size), u64(m), vp(ptr(plain_ntt)),
                    u64(R), vp(ptr(out)), vp(stream))

    def add_plain(self, a, size, plain, plain_batch, out, batch, level=None, stream=None):
        self.L.call("b200_add_plain", self.h, self._lv(level), vp(ptr(a)), C.c_int(size), vp(ptr(plain)), u64(plain_batch),
                    vp(ptr(out)), u64(batch), vp(stream))

    def sub_plain(self, a, size, plain, plain_batch, out, batch, level=None, stream=None):
        self.L.call("b200_sub_plain", self.h, self._lv(level), vp(ptr(a)), C.c_int(size), vp(ptr(plain)), u64(plain_batch),
                    vp(ptr(out)), u64(batch), vp(stream))

    def mod_switch_to_next(self, a, size, out, batch, level=None, stream=None):
        self.L.call("b200_mod_switch_to_next", self.h, self._lv(level), vp(ptr(a)), C.c_int(size), vp(ptr(out)), u64(batch),
                    vp(stream))

    def decrypt(self, ct, size, sk_powers, plain_out, batch, level=None, stream=None):
        self.L.call("b200_decrypt", self.h, self._lv(level), vp(ptr(ct)), C.c_int(size), vp(ptr(sk_powers)),
                    vp(ptr(plain_out)), u64(batch), vp(stream))

    def ct_sk_phase(self, ct, size, sk_powers, phase_out, batch, level=None, stream=None):
        self.L.call("b200_ct_sk_phase", self.h, self._lv(level), vp(ptr(ct)), C.c_int(size), vp(ptr(sk_powers)),
                    vp(ptr(phase_out)), u64(batch), vp(stream))

    def noise_norm(self, ct, size, sk_powers, norm_out_host, words, batch, level=None, stream=None):
        """norm_out_host: HOST uint64 array [batch][words] (little-endian multi-precision)."""
        self.L.call("b200_noise_norm", self.h, self._lv(level), vp(ptr(ct)), C.c_int(size), vp(ptr(sk_powers)),
                    vp(ptr(norm_out_host)), C.c_int(words), u64(batch), vp(stream))

    def is_transparent(self, ct, size, flags, batch, level=None, stream=None):
        self.L.call("b200_is_transparent", self.h, self._lv(level), vp(ptr(ct)), C.c_int(size), vp(ptr(flags)), u64(batch),
                    vp(stream))

    def any_nonzero(self, ct, size, flags, batch, level=None, stream=None):
        """flags (uint32 per item, zeroed by the caller; device or pinned host memory) <- 1 where polys [1, size) are not all zero."""
        self.L.call("b200_any_nonzero", self.h, self._lv(level), vp(ptr(ct)), C.c_int(size), vp(ptr(flags)), u64(batch),
                    vp(stream))

    def expand_signed(self, vals, polys, out, level=None, stream=None):
        self.L.call("b200_expand_signed", self.h, self._lv(level), vp(ptr(vals)), C.c_int(polys), vp(ptr(out)), vp(stream))

    def multiply_relin_host(self, a_host, b_host, rlk_dev, out_host, batch, level=None):
        self.L.call("b200_multiply_relin_host", self.h, self._lv(level), vp(ptr(a_host)), vp(ptr(b_host)), vp(ptr(rlk_dev)),
                    vp(ptr(out_host)), u64(batch))

    def ntt_roundtrip_host(self, in_host, out_host, items, level=None):
        self.L.call("b200_ntt_roundtrip_host", self.h, self._lv(level), vp(ptr(in_host)), vp(ptr(out_host)), u64(items))
