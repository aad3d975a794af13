"""Drives the SEAL-named C ABI (include/b200_sealc.h) of OUR library the way seal_fhe's Rust wrappers do
(seal_fhe/src/{context,evaluator_base,bfv_evaluator,plaintext_ciphertext,key_generator}.rs), with keys / fresh
ciphertexts imported from the reference.  Test infrastructure."""
import ctypes as C

import numpy as np

vp, u64 = C.c_void_p, C.c_uint64


def hres(x):
    return x & 0xFFFFFFFF


class SealcError(RuntimeError):
    def __init__(self, name, code):
        super().__init__(f"{name} -> HRESULT 0x{hres(code):08x}")
        self.code = hres(code)


class Sealc:
    """ctypes view of the SEAL-named entry points of a library (ours: sunscreen_b200/libb200bfv.so or the emu build)."""

    def __init__(self, cdll):
        self.lib = cdll

    def rc(self, name, *args):
        fn = getattr(self.lib, name)
        fn.restype = C.c_long
        return hres(fn(*args))

    def call(self, name, *args):
        r = self.rc(name, *args)
        if r:
            raise SealcError(name, r)

    # --- the call sequence of seal_fhe::Context::new (context.rs) ---
    def context(self, n, moduli, t, sec=128):
        parms = vp()
        self.call("EncParams_Create1", C.c_uint8(1), C.byref(parms))
        self.call("EncParams_SetPolyModulusDegree", parms, u64(n))
        arr = (vp * len(moduli))()
        for i, m in enumerate(moduli):
            h = vp()
            self.call("Modulus_Create1", u64(m), C.byref(h))
            arr[i] = h
        self.call("EncParams_SetCoeffModulus", parms, u64(len(moduli)), arr)
        self.call("EncParams_SetPlainModulus2", parms, u64(t))
        ctx = vp()
        self.call("SEALContext_Create", parms, C.c_bool(True), C.c_int(sec), C.byref(ctx))
        return SealcContext(self, ctx, n, moduli, t)


class SealcContext:
    def __init__(self, S, ctx, n, moduli, t):
        self.S, self.ctx, self.n, self.moduli, self.t = S, ctx, n, list(moduli), t
        self.K = len(moduli)
        self.k = self.K - 1 if self.K > 1 else 1
        ok = C.c_bool()
        S.call("SEALContext_ParametersSet", ctx, C.byref(ok))
        self.parameters_set = ok.value
        self.first_id = (u64 * 4)()
        self.key_id = (u64 * 4)()
        S.call("SEALContext_FirstParmsId", ctx, self.first_id)
        S.call("SEALContext_KeyParmsId", ctx, self.key_id)
        self.ev = vp()
        if self.parameters_set:
            S.call("Evaluator_Create", ctx, C.byref(self.ev))

    def new_ct(self, words=None, ntt=False):
        h = vp()
        self.S.call("Ciphertext_Create1", None, C.byref(h))
        if words is not None:
            w = np.ascontiguousarray(words, dtype=np.uint64)
            self.S.call("B200_Ciphertext_SetWords", h, self.ctx, self.first_id, u64(w.shape[0]), C.c_bool(ntt),
                        w.ctypes.data_as(C.POINTER(u64)))
        return h

    def ct_words(self, h):
        size, k = u64(), u64()
        self.S.call("Ciphertext_Size", h, C.byref(size))
        self.S.call("Ciphertext_CoeffModulusSize", h, C.byref(k))
        out = np.zeros((size.value, k.value, self.n), dtype=np.uint64)
        self.S.call("B200_Ciphertext_GetWords", h, out.ctypes.data_as(C.POINTER(u64)), u64(out.size))
        return out

    def ct_words_key(self, h):
        """Words of a key-level ciphertext-shaped object (public key / key-switching key element)."""
        return self.ct_words(h)

    def new_pt(self, coeffs):
        h = vp()
        c = np.ascontiguousarray(coeffs, dtype=np.uint64)
        self.S.call("Plaintext_Create1", None, C.byref(h))
        self.S.call("B200_Plaintext_SetCoeffs", h, u64(c.size), c.ctypes.data_as(C.POINTER(u64)))
        return h

    def pt_coeffs(self, h):
        cnt = u64()
        self.S.call("Plaintext_CoeffCount", h, C.byref(cnt))
        out = np.zeros(cnt.value, dtype=np.uint64)
        for i in range(cnt.value):
            v = u64()
            self.S.call("Plaintext_CoeffAt", h, u64(i), C.byref(v))
            out[i] = v.value
        return out

    def new_ksk(self, key_lists):
        h = vp()
        self.S.call("KSwitchKeys_Create1", C.byref(h))
        for index, arr in sorted(key_lists.items()):
            a = np.ascontiguousarray(arr, dtype=np.uint64)
            self.S.call("B200_KSwitchKeys_SetKeyWords", h, self.ctx, u64(index), u64(a.shape[0]),
                        a.ctypes.data_as(C.POINTER(u64)))
        return h

    # evaluator_base.rs: destination is a fresh Ciphertext_Create1(NULL), pool is NULL
    def _dst(self):
        h = vp()
        self.S.call("Ciphertext_Create1", None, C.byref(h))
        return h

    def add(self, a, b):
        d = self._dst(); self.S.call("Evaluator_Add", self.ev, a, b, d); return d

    def sub(self, a, b):
        d = self._dst(); self.S.call("Evaluator_Sub", self.ev, a, b, d); return d

    def negate(self, a):
        d = self._dst(); self.S.call("Evaluator_Negate", self.ev, a, d); return d

    def multiply(self, a, b):
        d = self._dst(); self.S.call("Evaluator_Multiply", self.ev, a, b, d, None); return d

    def square(self, a):
        d = self._dst(); self.S.call("Evaluator_Square", self.ev, a, d, None); return d

    def relinearize(self, a, rlk):
        d = self._dst(); self.S.call("Evaluator_Relinearize", self.ev, a, rlk, d, None); return d

    def rotate_rows(self, a, steps, glk):
        d = self._dst(); self.S.call("Evaluator_RotateRows", self.ev, a, C.c_int(steps), glk, d, None); return d

    def rotate_columns(self, a, glk):
        d = self._dst(); self.S.call("Evaluator_RotateColumns", self.ev, a, glk, d, None); return d

    def multiply_plain(self, a, p):
        d = self._dst(); self.S.call("Evaluator_MultiplyPlain", self.ev, a, p, d, None); return d

    def add_plain(self, a, p):
        d = self._dst(); self.S.call("Evaluator_AddPlain", self.ev, a, p, d); return d

    def sub_plain(self, a, p):
        d = self._dst(); self.S.call("Evaluator_SubPlain", self.ev, a, p, d); return d

    def mod_switch_to_next(self, a):
        d = self._dst(); self.S.call("Evaluator_ModSwitchToNext1", self.ev, a, d, None); return d

    def multiply_many(self, cts, rlk):
        d = self._dst()
        arr = (vp * len(cts))(*cts)
        self.S.call("Evaluator_MultiplyMany", self.ev, u64(len(cts)), arr, rlk, d, None)
        return d

    def exponentiate(self, a, e, rlk):
        d = self._dst(); self.S.call("Evaluator_Exponentiate", self.ev, a, u64(e), rlk, d, None); return d

    def add_many(self, cts):
        d = self._dst()
        arr = (vp * len(cts))(*cts)
        self.S.call("Evaluator_AddMany", self.ev, u64(len(cts)), arr, d)
        return d

    # debug aids of include/b200_sealc.h
    def combined_batch(self, kind, a, b=None, keys=None, galois_elt=0, dsts=None):
        """B200_Evaluator_CombinedBatchDebug -> (destinations, per-item HRESULTs); the call's own HRESULT must be S_OK"""
        N = len(a)
        dsts = dsts or [self._dst() for _ in range(N)]
        hr = (C.c_long * N)()
        arr = lambda hs: (vp * N)(*hs)
        self.S.call("B200_Evaluator_CombinedBatchDebug", self.ev, C.c_int(kind), u64(N), arr(a), arr(b) if b else None, keys,
                    C.c_uint32(galois_elt), arr(dsts), hr)
        return dsts, [hres(x) for x in hr]

    def graph_stats(self):
        """B200_Context_GraphStatsDebug: first sights, captures, refused captures, replays, evictions, batches without a graph"""
        out = (u64 * 6)()
        self.S.call("B200_Context_GraphStatsDebug", self.ctx, out)
        return np.array(list(out), dtype=np.int64)

    def decryptor(self, sk_words):
        sk = vp()
        self.S.call("SecretKey_Create1", C.byref(sk))
        w = np.ascontiguousarray(sk_words, dtype=np.uint64)
        self.S.call("B200_SecretKey_SetWords", sk, self.ctx, w.ctypes.data_as(C.POINTER(u64)))
        d = vp()
        self.S.call("Decryptor_Create", self.ctx, sk, C.byref(d))
        return d

    def decrypt(self, dec, ct):
        p = vp()
        self.S.call("Plaintext_Create1", None, C.byref(p))
        self.S.call("Decryptor_Decrypt", dec, ct, p)
        return p

    def noise_budget(self, dec, ct):
        b = C.c_int()
        self.S.call("Decryptor_InvariantNoiseBudget", dec, ct, C.byref(b))
        return b.value
