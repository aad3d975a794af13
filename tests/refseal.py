"""ctypes driver for the UNMODIFIED reference (oracle/_ref/libsealc_ref.so) — test infrastructure.

Replays the FFI call sequences of seal_fhe (SURVEY.md §3: `seal_fhe/src/evaluator_base.rs:89-407`,
`bfv_evaluator.rs:143-247`) against the reference's own C export layer (`S/c/*.h`), with bulk word
access through the hooks in oracle/ref_shim.cpp.  Nothing in the product imports this module.
"""
import ctypes as C
import os

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(_ROOT, "oracle", "_ref", "libsealc_ref.so")

S_OK = 0
E_POINTER = 0x80004003
E_INVALIDARG = 0x80070057
COR_E_INVALIDOPERATION = 0x80131509

vp = C.c_void_p
u64 = C.c_uint64


def hres(x):
    return x & 0xFFFFFFFF


class SealError(RuntimeError):
    def __init__(self, name, code):
        super().__init__(f"{name} -> HRESULT 0x{hres(code):08x}")
        self.code = hres(code)


def have_ref():
    return os.path.exists(REF_SO)


def splitmix64_words(count, modulus, state):
    """SURVEY.md App. B generator: `count` words, each next() % modulus. Returns (array, new_state)."""
    # vectorised: state_i = state + (i+1)*gamma
    gamma = np.uint64(0x9E3779B97F4A7C15)
    idx = np.arange(1, count + 1, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(state) + idx * gamma
        new_state = int(z[-1]) if count else state
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z % np.uint64(modulus), new_state


def fnv1a64(words):
    """FNV-1a-64 over the little-endian bytes of a u64 array (SURVEY.md App. B)."""
    w = np.ascontiguousarray(words, dtype="<u8").reshape(-1)
    so = os.path.join(_ROOT, "oracle", "_ref", "libbfv_oracle.so")
    if os.path.exists(so):
        lib = C.CDLL(so)
        lib.orc_fnv1a64.restype = u64
        lib.orc_fnv1a64.argtypes = [vp, C.c_size_t]
        return int(lib.orc_fnv1a64(w.ctypes.data, w.size))
    h = 0xCBF29CE484222325
    data = w.tobytes()
    # pure-python loop is too slow for MBs; process with a small C-like loop via int ops on memoryview chunks
    prime = 0x100000001B3
    mask = 0xFFFFFFFFFFFFFFFF
    for b in data:
        h = ((h ^ b) * prime) & mask
    return h


class RefLib:
    """Loads the reference shared library and declares the handful of signatures we call."""

    _inst = None

    @classmethod
    def get(cls):
        if cls._inst is None:
            cls._inst = cls()
        return cls._inst

    def __init__(self, path=REF_SO):
        self.lib = C.CDLL(path, mode=os.RTLD_LOCAL)
        L = self.lib
        for name in ("refshim_ct_data", "refshim_pt_data", "refshim_ksk_data"):
            getattr(L, name).restype = C.POINTER(u64)
        for name in ("refshim_ct_words", "refshim_pt_coeff_count", "refshim_ksk_outer_size", "refshim_ksk_inner_size",
                     "refshim_ntt_root"):
            getattr(L, name).restype = u64
        L.refshim_ct_data.argtypes = [vp]
        L.refshim_ct_words.argtypes = [vp]
        L.refshim_pt_data.argtypes = [vp]
        L.refshim_pt_coeff_count.argtypes = [vp]
        L.refshim_ct_resize.argtypes = [vp, vp, C.POINTER(u64), u64, C.c_int]
        L.refshim_ksk_outer_size.argtypes = [vp]
        L.refshim_ksk_inner_size.argtypes = [vp, u64]
        L.refshim_ksk_data.argtypes = [vp, u64, u64]
        L.refshim_ksk_alloc.argtypes = [vp, vp, u64, u64]
        L.refshim_ntt_forward.argtypes = [u64, C.c_int, vp, u64]
        L.refshim_ntt_inverse.argtypes = [u64, C.c_int, vp, u64]
        L.refshim_ntt_root.argtypes = [u64, C.c_int]
        L.refshim_rns_info.argtypes = [vp, C.c_int, vp, u64]
        L.refshim_plain_info.argtypes = [vp, C.c_int, vp, u64]
        L.refshim_behz_lift.argtypes = [vp, vp, vp]
        L.refshim_behz_floor_sk.argtypes = [vp, vp, vp]
        L.refshim_time_mul_relin.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int]
        L.refshim_time_mul_relin.restype = C.c_double
        L.refshim_time_ntt_roundtrip.argtypes = [u64, C.c_int, vp, u64, C.c_int]
        L.refshim_time_ntt_roundtrip.restype = C.c_double
        if hasattr(L, "refshim_mul_relin_batch"):
            L.refshim_mul_relin_batch.argtypes = [vp, vp, vp, vp, vp, u64, C.c_int]
            L.refshim_ntt_forward_mt.argtypes = [u64, C.c_int, vp, u64, C.c_int]

    def call(self, name, *args):
        fn = getattr(self.lib, name)
        fn.restype = C.c_long
        rc = fn(*args)
        if rc != 0:
            raise SealError(name, rc)

    def call_rc(self, name, *args):
        fn = getattr(self.lib, name)
        fn.restype = C.c_long
        return hres(fn(*args))

    # --- low-level NTT (S/util/ntt.cpp:393-474) ---
    def ntt_forward(self, modulus, polys):
        a = np.ascontiguousarray(polys, dtype=np.uint64).copy()
        n = a.shape[-1]
        rc = self.lib.refshim_ntt_forward(modulus, n.bit_length() - 1, a.ctypes.data, a.size // n)
        assert rc == 0
        return a

    def ntt_forward_mt(self, modulus, polys, threads):
        a = np.ascontiguousarray(polys, dtype=np.uint64).copy()
        n = a.shape[-1]
        rc = self.lib.refshim_ntt_forward_mt(modulus, n.bit_length() - 1, a.ctypes.data, a.size // n, threads)
        assert rc == 0
        return a

    def ntt_inverse(self, modulus, polys):
        a = np.ascontiguousarray(polys, dtype=np.uint64).copy()
        n = a.shape[-1]
        rc = self.lib.refshim_ntt_inverse(modulus, n.bit_length() - 1, a.ctypes.data, a.size // n)
        assert rc == 0
        return a

    def ntt_root(self, modulus, n):
        return int(self.lib.refshim_ntt_root(modulus, n.bit_length() - 1))


SEC_NONE, SEC_TC128 = 0, 128
SCHEME_BFV = 1


class RefContext:
    """BFV context on the reference: EncParams_* + SEALContext_Create (S/c/encryptionparameters.h, sealcontext.h)."""

    def __init__(self, n, coeff_moduli, plain_modulus, sec_level=SEC_TC128, ref=None):
        self.ref = ref or RefLib.get()
        R = self.ref
        self.n = n
        self.key_moduli = [int(m) for m in coeff_moduli]
        self.t = int(plain_modulus)
        parms = vp()
        R.call("EncParams_Create1", C.c_uint8(SCHEME_BFV), C.byref(parms))
        R.call("EncParams_SetPolyModulusDegree", parms, u64(n))
        mods = (vp * len(coeff_moduli))()
        for i, m in enumerate(coeff_moduli):
            h = vp()
            R.call("Modulus_Create1", u64(m), C.byref(h))
            mods[i] = h
        R.call("EncParams_SetCoeffModulus", parms, u64(len(coeff_moduli)), mods)
        R.call("EncParams_SetPlainModulus2", parms, u64(plain_modulus))
        self.parms = parms
        ctx = vp()
        R.call("SEALContext_Create", parms, C.c_bool(True), C.c_int(sec_level), C.byref(ctx))
        ok = C.c_bool()
        R.call("SEALContext_ParametersSet", ctx, C.byref(ok))
        if not ok.value:
            raise ValueError("reference rejected parameters")
        self.ctx = ctx
        self.key_parms_id = (u64 * 4)()
        self.first_parms_id = (u64 * 4)()
        R.call("SEALContext_KeyParmsId", ctx, self.key_parms_id)
        R.call("SEALContext_FirstParmsId", ctx, self.first_parms_id)
        self.k = len(coeff_moduli) - 1 if len(coeff_moduli) > 1 else 1  # data-level residues
        self.data_moduli = self.key_moduli[: self.k]
        ev = vp()
        R.call("Evaluator_Create", ctx, C.byref(ev))
        self.ev = ev

    @staticmethod
    def bfv_default_moduli(n, ref=None):
        R = ref or RefLib.get()
        length = u64(0)
        R.call("CoeffModulus_BFVDefault", u64(n), C.c_int(SEC_TC128), C.byref(length), None)
        arr = (vp * length.value)()
        R.call("CoeffModulus_BFVDefault", u64(n), C.c_int(SEC_TC128), C.byref(length), arr)
        out = []
        for h in arr:
            v = u64()
            R.call("Modulus_Value", vp(h), C.byref(v))
            out.append(v.value)
        return out

    def data_parms_ids(self):
        """parms_id of every data level, the first data level first (its own chain: it ends before a modulus below t)."""
        R = self.ref
        out = []
        cd = vp()
        R.call("SEALContext_FirstContextData", self.ctx, C.byref(cd))
        while cd.value:
            parms = vp()
            R.call("ContextData_Parms", cd, C.byref(parms))
            pid = (u64 * 4)()
            R.call("EncParams_GetParmsId", parms, pid)
            R.call("EncParams_Destroy", parms)
            out.append(pid)
            nxt = vp()
            R.call("ContextData_NextContextData", cd, C.byref(nxt))
            cd = nxt
        return out

    # ---- data objects ----
    def new_ct(self, words=None, ntt=False, level=0):
        """words: (size, k, n) uint64 at data level `level` (0 = first_parms_id, 1 = after one modulus switch, ...; k of
        that level), or None for an empty destination."""
        R = self.ref
        h = vp()
        R.call("Ciphertext_Create1", None, C.byref(h))
        if words is not None:
            words = np.ascontiguousarray(words, dtype=np.uint64)
            assert words.shape[1:] == (self.k - level, self.n), words.shape
            pid = self.first_parms_id if level == 0 else self.data_parms_ids()[level]
            rc = R.lib.refshim_ct_resize(h, self.ctx, pid, words.shape[0], int(ntt))
            assert rc == 0
            C.memmove(R.lib.refshim_ct_data(h), words.ctypes.data, words.nbytes)
        return h

    def ct_words(self, h):
        R = self.ref
        size = u64()
        k = u64()
        R.call("Ciphertext_Size", h, C.byref(size))
        R.call("Ciphertext_CoeffModulusSize", h, C.byref(k))
        out = np.empty((size.value, k.value, self.n), dtype=np.uint64)
        assert R.lib.refshim_ct_words(h) == out.size
        if out.size:
            C.memmove(out.ctypes.data, R.lib.refshim_ct_data(h), out.nbytes)
        return out

    def ct_words_any(self, h):
        """Words of any ciphertext-shaped object (e.g. a public key at the key level)."""
        R = self.ref
        size, k = u64(), u64()
        R.call("Ciphertext_Size", h, C.byref(size))
        R.call("Ciphertext_CoeffModulusSize", h, C.byref(k))
        out = np.empty((size.value, k.value, self.n), dtype=np.uint64)
        C.memmove(out.ctypes.data, R.lib.refshim_ct_data(h), out.nbytes)
        return out

    def free_ct(self, h):
        self.ref.call("Ciphertext_Destroy", h)

    def new_pt(self, coeffs):
        R = self.ref
        coeffs = np.ascontiguousarray(coeffs, dtype=np.uint64)
        h = vp()
        R.call("Plaintext_Create2", u64(coeffs.size), None, C.byref(h))
        if coeffs.size:
            C.memmove(R.lib.refshim_pt_data(h), coeffs.ctypes.data, coeffs.nbytes)
        return h

    def free_pt(self, h):
        self.ref.call("Plaintext_Destroy", h)

    def pt_coeffs(self, h):
        R = self.ref
        cnt = int(R.lib.refshim_pt_coeff_count(h))
        out = np.zeros(cnt, dtype=np.uint64)
        if cnt:
            C.memmove(out.ctypes.data, R.lib.refshim_pt_data(h), out.nbytes)
        return out

    def new_ksk(self, key_lists):
        """key_lists: dict index -> array (decomp, 2, k+1, n) of key-level NTT-form words."""
        R = self.ref
        h = vp()
        R.call("KSwitchKeys_Create1", C.byref(h))
        for index, arr in sorted(key_lists.items()):
            arr = np.ascontiguousarray(arr, dtype=np.uint64)
            decomp = arr.shape[0]
            assert arr.shape[1:] == (2, len(self.key_moduli), self.n), arr.shape
            assert R.lib.refshim_ksk_alloc(h, self.ctx, index, decomp) == 0
            for j in range(decomp):
                C.memmove(R.lib.refshim_ksk_data(h, index, j), arr[j].ctypes.data, arr[j].nbytes)
        return h

    def ksk_words(self, h):
        """-> dict index -> array (decomp, 2, k+1, n)."""
        R = self.ref
        out = {}
        K = len(self.key_moduli)
        for index in range(int(R.lib.refshim_ksk_outer_size(h))):
            d = int(R.lib.refshim_ksk_inner_size(h, index))
            if not d:
                continue
            arr = np.empty((d, 2, K, self.n), dtype=np.uint64)
            for j in range(d):
                C.memmove(arr[j].ctypes.data, R.lib.refshim_ksk_data(h, index, j), arr[j].nbytes)
            out[index] = arr
        return out

    # ---- Evaluator (S/c/evaluator.h:16-79) ----
    def _op(self, name, *args):
        dest = self.new_ct()
        self.ref.call(name, self.ev, *args[:-1], dest, *([None] if args[-1] == "pool" else []))
        return dest

    def add(self, a, b):
        d = self.new_ct(); self.ref.call("Evaluator_Add", self.ev, a, b, d); return d

    def sub(self, a, b):
        d = self.new_ct(); self.ref.call("Evaluator_Sub", self.ev, a, b, d); return d

    def negate(self, a):
        d = self.new_ct(); self.ref.call("Evaluator_Negate", self.ev, a, d); return d

    def multiply(self, a, b):
        d = self.new_ct(); self.ref.call("Evaluator_Multiply", self.ev, a, b, d, None); return d

    def mul_relin_batch(self, A, B, rlk, threads):
        """relinearize(multiply(A[i], B[i])) for raw first-level words A, B: (count, 2, k, n) -> (count, 2, k, n)."""
        A = np.ascontiguousarray(A, dtype=np.uint64)
        B = np.ascontiguousarray(B, dtype=np.uint64)
        assert A.shape == B.shape and A.shape[1:] == (2, self.k, self.n)
        out = np.empty_like(A)
        rc = self.ref.lib.refshim_mul_relin_batch(self.ctx, A.ctypes.data, B.ctypes.data, rlk, out.ctypes.data, A.shape[0], threads)
        assert rc == 0
        return out

    def square(self, a):
        d = self.new_ct(); self.ref.call("Evaluator_Square", self.ev, a, d, None); return d

    def relinearize(self, a, rlk):
        d = self.new_ct(); self.ref.call("Evaluator_Relinearize", self.ev, a, rlk, d, None); return d

    def rotate_rows(self, a, steps, glk):
        d = self.new_ct(); self.ref.call("Evaluator_RotateRows", self.ev, a, C.c_int(steps), glk, d, None); return d

    def rotate_columns(self, a, glk):
        d = self.new_ct(); self.ref.call("Evaluator_RotateColumns", self.ev, a, glk, d, None); return d

    def apply_galois(self, a, elt, glk):
        d = self.new_ct(); self.ref.call("Evaluator_ApplyGalois", self.ev, a, C.c_uint32(elt), glk, d, None); return d

    def multiply_plain(self, a, p):
        d = self.new_ct(); self.ref.call("Evaluator_MultiplyPlain", self.ev, a, p, d, None); return d

    def add_plain(self, a, p):
        d = self.new_ct(); self.ref.call("Evaluator_AddPlain", self.ev, a, p, d); return d

    def sub_plain(self, a, p):
        d = self.new_ct(); self.ref.call("Evaluator_SubPlain", self.ev, a, p, d); return d

    def mod_switch_to_next(self, a):
        d = self.new_ct(); self.ref.call("Evaluator_ModSwitchToNext1", self.ev, a, d, None); return d

    # ---- keys / encryption (S/c/keygenerator.h, encryptor.h, decryptor.h, batchencoder.h) ----
    def keygen(self):
        R = self.ref
        kg = vp(); R.call("KeyGenerator_Create1", self.ctx, C.byref(kg))
        return kg

    def secret_key(self, kg):
        sk = vp(); self.ref.call("KeyGenerator_SecretKey", kg, C.byref(sk)); return sk

    def public_key(self, kg):
        pk = vp(); self.ref.call("KeyGenerator_CreatePublicKey", kg, C.c_bool(False), C.byref(pk)); return pk

    def relin_keys(self, kg):
        rk = vp(); self.ref.call("KeyGenerator_CreateRelinKeys", kg, C.c_bool(False), C.byref(rk)); return rk

    def galois_keys_all(self, kg):
        gk = vp(); self.ref.call("KeyGenerator_CreateGaloisKeysAll", kg, C.c_bool(False), C.byref(gk)); return gk

    def galois_keys_steps(self, kg, steps):
        gk = vp()
        arr = (C.c_int * len(steps))(*steps)
        self.ref.call("KeyGenerator_CreateGaloisKeysFromSteps", kg, u64(len(steps)), arr, C.c_bool(False), C.byref(gk))
        return gk

    def encryptor(self, pk, sk=None):
        e = vp(); self.ref.call("Encryptor_Create", self.ctx, pk, sk, C.byref(e)); return e

    def decryptor(self, sk):
        d = vp(); self.ref.call("Decryptor_Create", self.ctx, sk, C.byref(d)); return d

    def encrypt(self, enc, pt):
        d = self.new_ct(); self.ref.call("Encryptor_Encrypt", enc, pt, d, None); return d

    def decrypt(self, dec, ct):
        p = vp(); self.ref.call("Plaintext_Create1", None, C.byref(p))
        self.ref.call("Decryptor_Decrypt", dec, ct, p)
        return p

    def noise_budget(self, dec, ct):
        b = C.c_int(); self.ref.call("Decryptor_InvariantNoiseBudget", dec, ct, C.byref(b)); return b.value

    def batch_encoder(self):
        be = vp(); self.ref.call("BatchEncoder_Create", self.ctx, C.byref(be)); return be

    def batch_encode(self, be, values):
        values = np.ascontiguousarray(values, dtype=np.uint64)
        p = vp(); self.ref.call("Plaintext_Create1", None, C.byref(p))
        self.ref.call("BatchEncoder_Encode1", be, u64(values.size), values.ctypes.data_as(C.POINTER(u64)), p)
        return p

    def batch_decode(self, be, pt):
        out = np.zeros(self.n, dtype=np.uint64)
        cnt = u64(self.n)
        self.ref.call("BatchEncoder_Decode1", be, pt, C.byref(cnt), out.ctypes.data_as(C.POINTER(u64)), None)
        return out

    # ---- constants for pinning the host precompute ----
    def rns_info(self, key_level=False):
        buf = np.zeros(64, dtype=np.uint64)
        assert self.ref.lib.refshim_rns_info(self.ctx, int(key_level), buf.ctypes.data, buf.size) == 0
        nb, nbsk = int(buf[0]), int(buf[1])
        return dict(B=nb, Bsk=nbsk, m_sk=int(buf[2]), gamma=int(buf[3]), t=int(buf[4]),
                    bsk_primes=[int(x) for x in buf[5:5 + nbsk]])

    def plain_info(self, key_level=False):
        k = len(self.key_moduli) if key_level else self.k
        buf = np.zeros(3 * k + 1, dtype=np.uint64)
        assert self.ref.lib.refshim_plain_info(self.ctx, int(key_level), buf.ctypes.data, buf.size) == 0
        return dict(delta=[int(x) for x in buf[:k]], upper_half_increment=[int(x) for x in buf[k:2 * k]],
                    plain_upper_half_increment=[int(x) for x in buf[2 * k:3 * k]],
                    plain_upper_half_threshold=int(buf[3 * k]))

    def behz_lift(self, poly):
        poly = np.ascontiguousarray(poly, dtype=np.uint64)
        nbsk = self.rns_info()["Bsk"]
        out = np.empty((nbsk, self.n), dtype=np.uint64)
        assert self.ref.lib.refshim_behz_lift(self.ctx, poly.ctypes.data, out.ctypes.data) == 0
        return out

    def behz_floor_sk(self, poly_q_bsk):
        poly = np.ascontiguousarray(poly_q_bsk, dtype=np.uint64)
        out = np.empty((self.k, self.n), dtype=np.uint64)
        assert self.ref.lib.refshim_behz_floor_sk(self.ctx, poly.ctypes.data, out.ctypes.data) == 0
        return out

    def time_mul_relin(self, a, b, rlk, threads, iters, warmup=2):
        return float(self.ref.lib.refshim_time_mul_relin(self.ctx, a, b, rlk, threads, iters, warmup))


def appendix_b_inputs(n, key_moduli, t):
    """Deterministic RNG-free inputs of SURVEY.md App. B for one parameter set.

    Returns dict with a, b: (2,k,n); p: (n,); rlk: (k,2,k+1,n); glk3, glkc: (k,2,k+1,n)."""
    k = len(key_moduli) - 1
    state = 0xB200
    out = {}

    def poly(mods):
        nonlocal state
        rows = []
        for m in mods:
            w, state = splitmix64_words(n, m, state)
            rows.append(w)
        return np.stack(rows)

    data = key_moduli[:k]
    out["a"] = np.stack([poly(data), poly(data)])
    out["b"] = np.stack([poly(data), poly(data)])
    out["p"], state = splitmix64_words(n, t, state)

    def ksk():
        return np.stack([np.stack([poly(key_moduli), poly(key_moduli)]) for _ in range(k)])

    out["rlk"] = ksk()
    out["glk3"] = ksk()
    out["glkc"] = ksk()
    return out
