"""Writes tests/golden/encrypt_sk_n2048.npz: seeded secret-key encryptions (Encryptor_EncryptSymmetricReturnComponentsSetSeed)
of the library as it was before encryption was batched, when each call sampled and computed one item on its own.  The
reference's own entry point ignores the seed, so these words are the fixed point that the batched sampling (public-seed
derivation, uniform c1, then e) is held to.  The secret key is the reference's, saved uncompressed.

    python tests/golden/make_encrypt_sk_golden.py <libb200bfv(.so or _emu.so) of that library>
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import sealc_checks as sc  # noqa: E402
from params import PARAMS  # noqa: E402
from refseal import RefContext, fnv1a64  # noqa: E402
from sealc_driver import Sealc  # noqa: E402

NAME = "n2048_2x27"


def main(lib_path):
    n, moduli, t = PARAMS[NAME]
    S = Sealc(C.CDLL(lib_path, mode=os.RTLD_LOCAL))
    R, O = RefContext(n, moduli, t), S.context(n, moduli, t)
    RL, OL = sc._libs(R, O)
    sk_bytes = RL.save("SecretKey", R.secret_key(R.keygen()), 0)
    osk, enc = OL.load("SecretKey", sk_bytes), C.c_void_p()
    S.call("Encryptor_Create", O.ctx, None, osk, C.byref(enc))
    rng = np.random.default_rng(23)
    msgs = rng.integers(0, t, size=(3, n), dtype=np.uint64)
    msgs[0] = 0
    msgs[1] = t - 1
    seeds = rng.integers(0, 2**63, size=(3, 8), dtype=np.uint64)
    ct_hash, e_hash = [], []
    for m, sd in zip(msgs, seeds):
        ct, e, rem = OL.new("Ciphertext"), C.c_void_p(), OL.new("Plaintext")
        S.call("PolynomialArray_Create", None, C.byref(e))
        S.call("Encryptor_EncryptSymmetricReturnComponentsSetSeed", enc, O.new_pt(m), ct, e, rem,
               (C.c_uint64 * 8)(*[int(x) for x in sd]), None)
        ct_hash.append(fnv1a64(O.ct_words(ct)))
        e_hash.append(fnv1a64(sc._pa_export(OL, e)[1]))
    np.savez_compressed(os.path.join(HERE, "encrypt_sk_n2048.npz"), sk=np.frombuffer(bytes(sk_bytes), dtype=np.uint8),
                        msgs=msgs, seeds=seeds, ct_fnv=np.array(ct_hash, dtype=np.uint64), e_fnv=np.array(e_hash, dtype=np.uint64))


if __name__ == "__main__":
    main(sys.argv[1])
