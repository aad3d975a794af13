"""Python mirror of the `seal_fhe` Rust crate's public API, bound to the SEAL-named C ABI of the CUDA backend.

The image has no Rust toolchain, so this module plays the role of `seal_fhe/src/*.rs`: the same type names, method names,
argument meaning and error behaviour, implemented with the same FFI calls the Rust wrappers make
(`bindgen::Evaluator_Multiply(...)` -> `lib.Evaluator_Multiply(...)`), so tests written against it read like the crate's
own (`seal_fhe/src/bfv_evaluator.rs:305-960`).  Every object is an opaque handle owned by the C side and released on
`__del__`, as the Rust `Drop` impls do.

    params = (BfvEncryptionParametersBuilder().set_poly_modulus_degree(8192)
              .set_coefficient_modulus(CoefficientModulus.create(8192, [50, 30, 30, 50, 50]))
              .set_plain_modulus(PlainModulus.batching(8192, 20)).build())
    ctx = Context(params, False, SecurityLevel.TC128)
    keygen = KeyGenerator(ctx)
    evaluator = BFVEvaluator(ctx)
    c = evaluator.relinearize(evaluator.multiply(a, b), keygen.create_relinearization_keys())
"""
import ctypes as C

from .lib import B200Lib

vp, u64 = C.c_void_p, C.c_uint64


class Error(RuntimeError):
    """seal_fhe::Error (seal_fhe/src/error.rs:9-62): the HRESULT classes the crate distinguishes."""
    NAMES = {0x80004003: "InvalidPointer", 0x80070057: "InvalidArgument", 0x8007000E: "OutOfMemory", 0x8000FFFF: "Unexpected",
             0x80131509: "InvalidOperation", 0x80070585: "InternalError(InvalidIndex)"}

    def __init__(self, fn, code):
        self.code = code & 0xFFFFFFFF
        self.kind = self.NAMES.get(self.code, f"Unknown(0x{self.code:08x})")
        super().__init__(f"{fn}: {self.kind}")


class SecurityLevel:
    NONE, TC128, TC192, TC256 = 0, 128, 192, 256


_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = B200Lib.default().lib
    return _lib


def use_library(cdll):
    """Bind the mirror to an explicit shared library (the test-suite passes its emulation build)."""
    global _lib
    _lib = cdll


def _call(name, *args):
    fn = getattr(_L(), name)
    fn.restype = C.c_long
    rc = fn(*args)
    if rc:
        raise Error(name, rc)


class _Handle:
    _destroy = None

    def __init__(self, handle):
        self.handle = handle

    def __del__(self):
        try:
            if self.handle and self._destroy:
                getattr(_L(), self._destroy)(self.handle)
                self.handle = None
        except Exception:
            pass


class CompressionType:
    """seal_fhe/src/lib.rs:39-45 (serialization::CompressionType)."""
    NONE, ZLIB, ZSTD = 0, 1, 2


class _Serializable:
    """ToBytes / FromBytes of seal_fhe (plaintext_ciphertext.rs:88-160,452-500; key_generator.rs:200-700): the crate
    always asks for Zstandard; `compression` is exposed here because byte-exact comparisons need NONE."""
    _prefix = None
    _create = None  # (function name, takes a pool argument)

    def as_bytes(self, compression=CompressionType.ZSTD):
        n = C.c_int64()
        _call(self._prefix + "_SaveSize", self.handle, C.c_uint8(compression), C.byref(n))
        buf = (C.c_uint8 * n.value)()
        out = C.c_int64()
        _call(self._prefix + "_Save", self.handle, buf, u64(n.value), C.c_uint8(compression), C.byref(out))
        return bytes(buf[: out.value])

    @classmethod
    def from_bytes(cls, ctx, data):
        name, pool = cls._create
        h = vp()
        _call(name, None, C.byref(h)) if pool else _call(name, C.byref(h))
        obj = cls(h)
        buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data if data else b"\0")
        n = C.c_int64()
        _call(cls._prefix + "_Load", h, ctx.handle, buf, u64(len(data)), C.byref(n))
        return obj


class Modulus(_Handle):
    _destroy = "Modulus_Destroy"

    def __init__(self, value=None, handle=None):
        if handle is None:
            handle = vp()
            _call("Modulus_Create1", u64(value), C.byref(handle))
        super().__init__(handle)

    def value(self):
        v = u64()
        _call("Modulus_Value", self.handle, C.byref(v))
        return v.value


class CoefficientModulus:
    @staticmethod
    def create(degree, bit_sizes):
        arr = (vp * len(bit_sizes))()
        _call("CoeffModulus_Create1", u64(degree), u64(len(bit_sizes)), (C.c_int * len(bit_sizes))(*bit_sizes), arr)
        return [Modulus(handle=vp(h)) for h in arr]

    @staticmethod
    def bfv_default(degree, security_level=SecurityLevel.TC128):
        n = u64()
        _call("CoeffModulus_BFVDefault", u64(degree), C.c_int(security_level), C.byref(n), None)
        arr = (vp * n.value)()
        _call("CoeffModulus_BFVDefault", u64(degree), C.c_int(security_level), C.byref(n), arr)
        return [Modulus(handle=vp(h)) for h in arr]

    @staticmethod
    def max_bit_count(degree, security_level=SecurityLevel.TC128):
        b = C.c_int()
        _call("CoeffModulus_MaxBitCount", u64(degree), C.c_int(security_level), C.byref(b))
        return b.value


class PlainModulus:
    @staticmethod
    def batching(degree, bit_size):
        return CoefficientModulus.create(degree, [bit_size])[0]

    @staticmethod
    def raw(value):
        return Modulus(value)


class EncryptionParameters(_Handle):
    _destroy = "EncParams_Destroy"

    def get_poly_modulus_degree(self):
        d = u64()
        _call("EncParams_GetPolyModulusDegree", self.handle, C.byref(d))
        return d.value

    def get_plain_modulus(self):
        h = vp()
        _call("EncParams_GetPlainModulus", self.handle, C.byref(h))
        return Modulus(handle=h)

    def get_coefficient_modulus(self):
        n = u64()
        _call("EncParams_GetCoeffModulus", self.handle, C.byref(n), None)
        arr = (vp * n.value)()
        _call("EncParams_GetCoeffModulus", self.handle, C.byref(n), arr)
        return [Modulus(handle=vp(h)) for h in arr]


class BfvEncryptionParametersBuilder:
    def __init__(self):
        self._degree = None
        self._coeff = None
        self._plain = None

    def set_poly_modulus_degree(self, degree):
        self._degree = degree
        return self

    def set_coefficient_modulus(self, moduli):
        self._coeff = moduli
        return self

    def set_plain_modulus(self, modulus):
        self._plain = modulus
        return self

    def set_plain_modulus_u64(self, value):
        self._plain = Modulus(value)
        return self

    def build(self):
        if self._degree is None:
            raise Error("BfvEncryptionParametersBuilder", 0x80070057)
        h = vp()
        _call("EncParams_Create1", C.c_uint8(1), C.byref(h))
        p = EncryptionParameters(h)
        _call("EncParams_SetPolyModulusDegree", h, u64(self._degree))
        if self._coeff is None or self._plain is None:
            raise Error("BfvEncryptionParametersBuilder", 0x80070057)
        _call("EncParams_SetCoeffModulus", h, u64(len(self._coeff)), (vp * len(self._coeff))(*[m.handle for m in self._coeff]))
        _call("EncParams_SetPlainModulus1", h, self._plain.handle)
        return p


class Context(_Handle):
    _destroy = "SEALContext_Destroy"

    def __init__(self, params, expand_mod_chain, security_level):
        h = vp()
        _call("SEALContext_Create", params.handle, C.c_bool(expand_mod_chain), C.c_int(security_level), C.byref(h))
        super().__init__(h)
        self.params = params

    def get_key_parms_id(self):
        a = (u64 * 4)()
        _call("SEALContext_KeyParmsId", self.handle, a)
        return list(a)

    def get_first_parms_id(self):
        a = (u64 * 4)()
        _call("SEALContext_FirstParmsId", self.handle, a)
        return list(a)


class Plaintext(_Handle, _Serializable):
    _destroy = "Plaintext_Destroy"
    _prefix, _create = "Plaintext", ("Plaintext_Create1", True)

    @classmethod
    def from_hex_string(cls, hex_str):
        """Plaintext::from_hex_string (plaintext_ciphertext.rs): "7FFx^3 + 1x^1 + 3"."""
        h = vp()
        _call("Plaintext_Create4", hex_str.encode(), None, C.byref(h))
        return cls(h)

    def __init__(self, handle=None):
        if handle is None:
            handle = vp()
            _call("Plaintext_Create1", None, C.byref(handle))
        super().__init__(handle)

    def get_coefficient(self, index):
        v = u64()
        _call("Plaintext_CoeffAt", self.handle, u64(index), C.byref(v))
        return v.value

    def set_coefficient(self, index, value):
        _call("Plaintext_SetCoeffAt", self.handle, u64(index), u64(value))

    def resize(self, count):
        _call("Plaintext_Resize", self.handle, u64(count))

    def len(self):
        n = u64()
        _call("Plaintext_CoeffCount", self.handle, C.byref(n))
        return n.value


class Ciphertext(_Handle, _Serializable):
    _destroy = "Ciphertext_Destroy"
    _prefix, _create = "Ciphertext", ("Ciphertext_Create1", True)

    def __init__(self, handle=None):
        if handle is None:
            handle = vp()
            _call("Ciphertext_Create1", None, C.byref(handle))
        super().__init__(handle)

    def num_polynomials(self):
        n = u64()
        _call("Ciphertext_Size", self.handle, C.byref(n))
        return n.value

    def coeff_modulus_size(self):
        n = u64()
        _call("Ciphertext_CoeffModulusSize", self.handle, C.byref(n))
        return n.value

    def get_data(self, index):
        v = u64()
        _call("Ciphertext_GetDataAt1", self.handle, u64(index), C.byref(v))
        return v.value

    def is_ntt_form(self):
        b = C.c_bool()
        _call("Ciphertext_IsNTTForm", self.handle, C.byref(b))
        return b.value

    def clone(self):
        h = vp()
        _call("Ciphertext_Create2", self.handle, C.byref(h))
        return Ciphertext(h)


class PublicKey(_Handle, _Serializable):
    _destroy = "PublicKey_Destroy"
    _prefix, _create = "PublicKey", ("PublicKey_Create1", False)


class SecretKey(_Handle, _Serializable):
    _destroy = "SecretKey_Destroy"
    _prefix, _create = "SecretKey", ("SecretKey_Create1", False)


class RelinearizationKeys(_Handle, _Serializable):
    _destroy = "KSwitchKeys_Destroy"
    _prefix, _create = "KSwitchKeys", ("KSwitchKeys_Create1", False)


class GaloisKeys(_Handle, _Serializable):
    _destroy = "KSwitchKeys_Destroy"
    _prefix, _create = "KSwitchKeys", ("KSwitchKeys_Create1", False)


class PolynomialArray(_Handle):
    """seal_fhe/src/poly_array.rs: the (u, e, key) polynomial container handed to the proof code."""
    _destroy = "PolynomialArray_Destroy"

    def __init__(self, handle=None):
        if handle is None:
            handle = vp()
            _call("PolynomialArray_Create", None, C.byref(handle))
        super().__init__(handle)

    @classmethod
    def _from(cls, fn, ctx, obj):
        h = vp()
        _call(fn, None, ctx.handle, obj.handle, C.byref(h))
        return cls(h)

    new_from_ciphertext = classmethod(lambda cls, ctx, ct: cls._from("PolynomialArray_CreateFromCiphertext", ctx, ct))
    new_from_public_key = classmethod(lambda cls, ctx, pk: cls._from("PolynomialArray_CreateFromPublicKey", ctx, pk))
    new_from_secret_key = classmethod(lambda cls, ctx, sk: cls._from("PolynomialArray_CreateFromSecretKey", ctx, sk))

    def _u64(self, name):
        v = u64()
        _call("PolynomialArray_" + name, self.handle, C.byref(v))
        return v.value

    def _bool(self, name):
        b = C.c_bool()
        _call("PolynomialArray_" + name, self.handle, C.byref(b))
        return b.value

    num_polynomials = lambda self: self._u64("PolySize")
    poly_modulus_degree = lambda self: self._u64("PolyModulusDegree")
    coeff_modulus_size = lambda self: self._u64("CoeffModulusSize")
    is_reserved = lambda self: self._bool("IsReserved")
    is_rns = lambda self: self._bool("IsRns")
    is_multiprecision = lambda self: not self._bool("IsRns")

    def to_rns(self):
        _call("PolynomialArray_ToRns", self.handle)

    def to_multiprecision(self):
        _call("PolynomialArray_ToMultiprecision", self.handle)

    def as_u64_slice(self):
        n = self._u64("ExportSize")
        buf = (u64 * max(n, 1))()
        if n:
            _call("PolynomialArray_PerformExport", self.handle, buf)
        return list(buf[:n])

    def drop(self):
        h = vp()
        _call("PolynomialArray_Drop", self.handle, C.byref(h))
        return PolynomialArray(h)

    def clone(self):
        h = vp()
        _call("PolynomialArray_Copy", self.handle, C.byref(h))
        return PolynomialArray(h)


class KeyGenerator(_Handle):
    _destroy = "KeyGenerator_Destroy"

    def __init__(self, ctx, secret_key=None):
        h = vp()
        if secret_key is None:
            _call("KeyGenerator_Create1", ctx.handle, C.byref(h))
        else:
            _call("KeyGenerator_Create2", ctx.handle, secret_key.handle, C.byref(h))
        super().__init__(h)
        self.ctx = ctx

    new_from_secret_key = classmethod(lambda cls, ctx, sk: cls(ctx, sk))

    def secret_key(self):
        h = vp()
        _call("KeyGenerator_SecretKey", self.handle, C.byref(h))
        return SecretKey(h)

    def create_public_key(self):
        h = vp()
        _call("KeyGenerator_CreatePublicKey", self.handle, C.c_bool(False), C.byref(h))
        return PublicKey(h)

    def create_relinearization_keys(self):
        h = vp()
        _call("KeyGenerator_CreateRelinKeys", self.handle, C.c_bool(False), C.byref(h))
        return RelinearizationKeys(h)

    def create_galois_keys(self):
        h = vp()
        _call("KeyGenerator_CreateGaloisKeysAll", self.handle, C.c_bool(False), C.byref(h))
        return GaloisKeys(h)


class Encryptor(_Handle):
    _destroy = "Encryptor_Destroy"

    def __init__(self, ctx, public_key=None, secret_key=None):
        h = vp()
        _call("Encryptor_Create", ctx.handle, public_key.handle if public_key else None,
              secret_key.handle if secret_key else None, C.byref(h))
        super().__init__(h)

    with_public_key = classmethod(lambda cls, ctx, pk: cls(ctx, public_key=pk))
    with_public_and_secret_key = classmethod(lambda cls, ctx, pk, sk: cls(ctx, pk, sk))

    def encrypt(self, plaintext):
        c = Ciphertext()
        _call("Encryptor_Encrypt", self.handle, plaintext.handle, c.handle, None)
        return c

    def encrypt_symmetric(self, plaintext):
        c = Ciphertext()
        _call("Encryptor_EncryptSymmetric", self.handle, plaintext.handle, C.c_bool(False), c.handle, None)
        return c

    def encrypt_return_components(self, plaintext, disable_special_modulus=False, seed=None):
        """encrypt_return_components{,_deterministic} (encryptor_decryptor.rs:250-420): (ciphertext, u, e, remainder)."""
        c, u_, e_, r = Ciphertext(), PolynomialArray(), PolynomialArray(), Plaintext()
        if seed is None:
            _call("Encryptor_EncryptReturnComponents", self.handle, plaintext.handle, C.c_bool(disable_special_modulus), c.handle,
                  u_.handle, e_.handle, r.handle, None)
        else:
            _call("Encryptor_EncryptReturnComponentsSetSeed", self.handle, plaintext.handle, C.c_bool(disable_special_modulus),
                  c.handle, u_.handle, e_.handle, r.handle, (u64 * 8)(*seed), None)
        return c, u_, e_, r

    def encrypt_deterministic(self, plaintext, seed):
        """encryptor_decryptor.rs:319-345 (feature "deterministic"): INSECURE, for tests and demonstrations only."""
        return self.encrypt_return_components(plaintext, False, seed)[0]

    def encrypt_symmetric_return_components(self, plaintext, seed=None):
        c, e_, r = Ciphertext(), PolynomialArray(), Plaintext()
        if seed is None:
            _call("Encryptor_EncryptSymmetricReturnComponents", self.handle, plaintext.handle, c.handle, e_.handle, r.handle, None)
        else:
            _call("Encryptor_EncryptSymmetricReturnComponentsSetSeed", self.handle, plaintext.handle, c.handle, e_.handle,
                  r.handle, (u64 * 8)(*seed), None)
        return c, e_, r


class Decryptor(_Handle):
    _destroy = "Decryptor_Destroy"

    def __init__(self, ctx, secret_key):
        h = vp()
        _call("Decryptor_Create", ctx.handle, secret_key.handle, C.byref(h))
        super().__init__(h)

    def decrypt(self, ciphertext):
        p = Plaintext()
        _call("Decryptor_Decrypt", self.handle, ciphertext.handle, p.handle)
        return p

    def invariant_noise_budget(self, ciphertext):
        b = C.c_int()
        _call("Decryptor_InvariantNoiseBudget", self.handle, ciphertext.handle, C.byref(b))
        return b.value

    def invariant_noise(self, ciphertext):
        d = C.c_double()
        _call("Decryptor_InvariantNoise", self.handle, ciphertext.handle, C.byref(d))
        return d.value


class BFVEncoder(_Handle):
    """seal_fhe::BFVEncoder (seal_fhe/src/encoder.rs): SIMD batching encoder."""
    _destroy = "BatchEncoder_Destroy"

    def __init__(self, ctx):
        h = vp()
        _call("BatchEncoder_Create", ctx.handle, C.byref(h))
        super().__init__(h)

    def get_slot_count(self):
        n = u64()
        _call("BatchEncoder_GetSlotCount", self.handle, C.byref(n))
        return n.value

    def encode_unsigned(self, data):
        p = Plaintext()
        _call("BatchEncoder_Encode1", self.handle, u64(len(data)), (u64 * len(data))(*[int(x) for x in data]), p.handle)
        return p

    def encode_signed(self, data):
        p = Plaintext()
        _call("BatchEncoder_Encode2", self.handle, u64(len(data)), (C.c_int64 * len(data))(*[int(x) for x in data]), p.handle)
        return p

    def decode_unsigned(self, plaintext):
        n = self.get_slot_count()
        out = (u64 * n)()
        cnt = u64(n)
        _call("BatchEncoder_Decode1", self.handle, plaintext.handle, C.byref(cnt), out, None)
        return list(out)

    def decode_signed(self, plaintext):
        n = self.get_slot_count()
        out = (C.c_int64 * n)()
        cnt = u64(n)
        _call("BatchEncoder_Decode2", self.handle, plaintext.handle, C.byref(cnt), out, None)
        return list(out)


class BFVEvaluator(_Handle):
    """seal_fhe::BFVEvaluator = `trait Evaluator` (seal_fhe/src/evaluator.rs:14-157) over EvaluatorBase
    (seal_fhe/src/evaluator_base.rs:89-407): out-of-place methods create a fresh destination, *_inplace pass dest == src."""
    _destroy = "Evaluator_Destroy"

    def __init__(self, ctx):
        h = vp()
        _call("Evaluator_Create", ctx.handle, C.byref(h))
        super().__init__(h)

    def _unary(self, fn, a, *extra, pool=True, inplace=False):
        d = a if inplace else Ciphertext()
        args = [self.handle, a.handle, *extra, d.handle] + ([None] if pool else [])
        _call(fn, *args)
        return d

    def negate(self, a):
        return self._unary("Evaluator_Negate", a, pool=False)

    def negate_inplace(self, a):
        self._unary("Evaluator_Negate", a, pool=False, inplace=True)

    def add(self, a, b):
        d = Ciphertext()
        _call("Evaluator_Add", self.handle, a.handle, b.handle, d.handle)
        return d

    def add_inplace(self, a, b):
        _call("Evaluator_Add", self.handle, a.handle, b.handle, a.handle)

    def add_many(self, cts):
        d = Ciphertext()
        _call("Evaluator_AddMany", self.handle, u64(len(cts)), (vp * len(cts))(*[c.handle for c in cts]), d.handle)
        return d

    def multiply_many(self, cts, relin_keys):
        d = Ciphertext()
        _call("Evaluator_MultiplyMany", self.handle, u64(len(cts)), (vp * len(cts))(*[c.handle for c in cts]), relin_keys.handle,
              d.handle, None)
        return d

    def sub(self, a, b):
        d = Ciphertext()
        _call("Evaluator_Sub", self.handle, a.handle, b.handle, d.handle)
        return d

    def sub_inplace(self, a, b):
        _call("Evaluator_Sub", self.handle, a.handle, b.handle, a.handle)

    def multiply(self, a, b):
        d = Ciphertext()
        _call("Evaluator_Multiply", self.handle, a.handle, b.handle, d.handle, None)
        return d

    def multiply_inplace(self, a, b):
        _call("Evaluator_Multiply", self.handle, a.handle, b.handle, a.handle, None)

    def square(self, a):
        return self._unary("Evaluator_Square", a)

    def square_inplace(self, a):
        self._unary("Evaluator_Square", a, inplace=True)

    def relinearize(self, a, relin_keys):
        return self._unary("Evaluator_Relinearize", a, relin_keys.handle)

    def relinearize_inplace(self, a, relin_keys):
        self._unary("Evaluator_Relinearize", a, relin_keys.handle, inplace=True)

    def mod_switch_to_next(self, a):
        return self._unary("Evaluator_ModSwitchToNext1", a)

    def exponentiate(self, a, exponent, relin_keys):
        return self._unary("Evaluator_Exponentiate", a, u64(exponent), relin_keys.handle)

    def add_plain(self, a, p):
        return self._unary("Evaluator_AddPlain", a, p.handle, pool=False)

    def sub_plain(self, a, p):
        return self._unary("Evaluator_SubPlain", a, p.handle, pool=False)

    def multiply_plain(self, a, p):
        return self._unary("Evaluator_MultiplyPlain", a, p.handle)

    def rotate_rows(self, a, steps, galois_keys):
        return self._unary("Evaluator_RotateRows", a, C.c_int(steps), galois_keys.handle)

    def rotate_rows_inplace(self, a, steps, galois_keys):
        self._unary("Evaluator_RotateRows", a, C.c_int(steps), galois_keys.handle, inplace=True)

    def rotate_columns(self, a, galois_keys):
        return self._unary("Evaluator_RotateColumns", a, galois_keys.handle)

    def rotate_columns_inplace(self, a, galois_keys):
        self._unary("Evaluator_RotateColumns", a, galois_keys.handle, inplace=True)
