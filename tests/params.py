"""Parameter sets used by the parity tests and bench (SURVEY.md §8(d), BASELINE.json configs).
Moduli are the reference's BFVDefault tables (S/util/globals.cpp:23-71); t = PlainModulus::Batching(n, 20)
except n=4096 where Sunscreen's default t = 262144 is used (sunscreen/src/compiler.rs:155).  The edge chains at the end
come from CoeffModulus::Create instead."""

DEFAULT_MODULI = {
    4096: [0xffffee001, 0xffffc4001, 0x1ffffe0001],
    8192: [0x7fffffd8001, 0x7fffffc8001, 0xfffffffc001, 0xffffff6c001, 0xfffffebc001],
    16384: [0xfffffffd8001, 0xfffffffa0001, 0xfffffff00001, 0x1fffffff68001, 0x1fffffff50001, 0x1ffffffee8001,
            0x1ffffffea0001, 0x1ffffffe88001, 0x1ffffffe48001],
    32768: [0x7fffffffe90001, 0x7fffffffbf0001, 0x7fffffffbd0001, 0x7fffffffba0001, 0x7fffffffaa0001,
            0x7fffffffa50001, 0x7fffffff9f0001, 0x7fffffff7e0001, 0x7fffffff770001, 0x7fffffff380001,
            0x7fffffff330001, 0x7fffffff2d0001, 0x7fffffff170001, 0x7fffffff150001, 0x7ffffffef00001,
            0xfffffffff70001],
}

PARAMS = {
    # name: (n, key-level moduli, plain modulus)
    "n4096": (4096, DEFAULT_MODULI[4096], 262144),
    "n8192": (8192, DEFAULT_MODULI[8192], 1032193),
    "n8192_54": (8192, [0x3fffffffe64001, 0x3fffffffe7c001, 0x3fffffffeb8001, 0x3fffffffef8001], 1032193),
    # 48/49-bit primes: the widest the FP64 path takes (host_ctx.h FP_PRIME_BITS); 196 bits <= 218 (TC128 @ n=8192)
    "n8192_49": (8192, [0xffffffffc001, 0x1fffffff74001, 0x1fffffff68001, 0x1fffffff50001], 1032193),
    "n16384": (16384, DEFAULT_MODULI[16384], 786433),
    "n32768": (32768, DEFAULT_MODULI[32768], 786433),
}

# Edge chains: what CoeffModulus::Create(n, bits) returns for each, in its order (same-width primes are handed out
# smallest first); tests/test_params.py re-derives every list.  Each set reaches kernel choices the homogeneous
# BFVDefault chains above never make.
EDGE_BITS = {
    # seal_fhe's own evaluator tests (seal_fhe/src/bfv_evaluator.rs:305-960): 50-bit primes on the integer path, 30-bit
    # ones on FP64, so every NTT job is mixed and the BEHZ base is the reference's 61-bit one
    "n8192_sealfhe": (8192, [50, 30, 30, 50, 50]),
    # >= 50-bit and 48/49-bit primes in one chain: at logn 14 every transform of a mixed job, FP64-capable primes
    # included, runs the generic integer kernel, and the BEHZ base is the 61-bit one
    "n16384_mixed": (16384, [50, 49, 50, 48, 49, 50]),
    # ~20-bit primes under the 47-bit FP64 auxiliary base, t below all of them
    "n4096_narrow": (4096, [20, 21, 22]),
    # a 17-bit data prime below t: no fast plain lift (every q_i > t fails)
    "n4096_q_below_t": (4096, [17, 30, 30]),
    # the widest primes SEAL allows (60 bits: the 128-bit lazy sums at their largest), and the first integer width
    "n8192_60": (8192, [60, 60, 60]),
    "n8192_50": (8192, [50, 50, 50, 50]),
    # two-prime chains at logn 11 and 10: key switching with the generic 256-thread kernel (54 bits exceed 128-bit
    # security at n = 1024, so the reference accepts that one only without a security level: SEC_NONE below)
    "n2048_2x27": (2048, [27, 27]),
    "n1024_2x27": (1024, [27, 27]),
}

PARAMS.update({
    "n8192_sealfhe": (8192, [0x3ffffffef4001, 0x3ffe8001, 0x3fff4001, 0x3fffffffcc001, 0x3ffffffffc001], 1032193),
    "n16384_mixed": (16384, [0x3ffffffd20001, 0x1fffffff50001, 0x3ffffffd48001, 0xfffffffd8001, 0x1fffffff68001,
                             0x3ffffffdf0001], 786433),
    "n4096_narrow": (4096, [0xfc001, 0x1f6001, 0x3fa001], 40961),
    "n4096_q_below_t": (4096, [0x1c001, 0x3ffee001, 0x3fff4001], 786433),
    "n8192_60": (8192, [0xffffffffffd8001, 0xffffffffffe8001, 0xfffffffffffc001], 1032193),
    "n8192_50": (8192, [0x3ffffffe94001, 0x3ffffffef4001, 0x3fffffffcc001, 0x3ffffffffc001], 1032193),
    "n2048_2x27": (2048, [0x7fe6001, 0x7ff6001], 12289),
    "n1024_2x27": (1024, [0x7ffc801, 0x7fff801], 12289),
})
SEC_NONE = {"n1024_2x27"}   # sets the reference must be created for without a security level
EDGE = list(EDGE_BITS)

# Long chains (also from CoeffModulus::Create): every cluster size of the key switch and up to 16 data residues on the FP64
# path.  Kept out of EDGE, whose parametrisations they would slow down; tests/test_gpu_long_chains.py runs them.
LONG_BITS = {
    # data levels k = 8 ... 1 at logn 13: ks_cluster_kernel at every cluster size 2 ... 8, mul_cluster_kernel up to k + |Bsk| = 14,
    # and both sides of multiply_relin's fused scale-and-mod-down rule
    "n8192_9x24": (8192, [24] * 9),
    # the same walk at logn 12 (two chunks per round in the cluster's inner product); 198 bits exceed 128-bit security at
    # n = 4096 (SEC_NONE)
    "n4096_9x22": (4096, [22] * 9),
    # the special prime narrowest (21 bits: the 20-bit one Create hands out is t = 1032193 itself), a 49-bit data prime and so
    # the 49-bit auxiliary base, k = 5 at the top: mixed widths inside one cluster job
    "n8192_mixed_fp": (8192, [49, 36, 30, 30, 30, 21]),
    # 16 data residues on the FP64 BEHZ and key-switch kernels (47-bit auxiliary base)
    "n16384_17x25": (16384, [25] * 17),
    # 16 data residues against 49-bit auxiliary primes: the FP64 inner products at their largest
    "n16384_49_16x24": (16384, [49] + [24] * 16),
}
PARAMS.update({
    "n8192_9x24": (8192, [0xf34001, 0xf3c001, 0xf60001, 0xf84001, 0xfa0001, 0xfb4001, 0xfc0001, 0xfd0001, 0xffc001], 1032193),
    "n4096_9x22": (4096, [0x390001, 0x3ac001, 0x3c6001, 0x3d2001, 0x3dc001, 0x3e4001, 0x3ea001, 0x3ee001, 0x3fa001], 262144),
    "n8192_mixed_fp": (8192, [0x1fffffff74001, 0xffffc4001, 0x3ffc0001, 0x3ffe8001, 0x3fff4001, 0x1b4001], 1032193),
    "n16384_17x25": (16384, [0x1bf0001, 0x1c50001, 0x1c80001, 0x1cc8001, 0x1cf8001, 0x1d20001, 0x1d58001, 0x1d88001, 0x1de0001,
                             0x1df8001, 0x1e70001, 0x1e78001, 0x1ef0001, 0x1f60001, 0x1f68001, 0x1f98001, 0x1fc0001], 786433),
    "n16384_49_16x24": (16384, [0x1fffffff68001, 0xc18001, 0xc78001, 0xca0001, 0xcb8001, 0xcf0001, 0xd00001, 0xd08001, 0xd78001,
                                0xd80001, 0xe38001, 0xe40001, 0xee8001, 0xf60001, 0xfa0001, 0xfc0001, 0xfd0001], 786433),
})
SEC_NONE.add("n4096_9x22")
LONG = list(LONG_BITS)

# Wide chains (also from CoeffModulus::Create): n = 32768 beyond the default chain, and the key level of the longest chains.
# Kept out of EDGE and LONG; tests/test_gpu_wide_chains.py runs them.
WIDE_BITS = {
    # 60-bit primes through the n = 32768 split transform (ntt_outer_kernel): the Harvey lazy bounds at their tightest
    "n32768_60x6": (32768, [60] * 6),
    # 30-bit primes under a 47-bit auxiliary base that needs fewer primes than k (nB < k), on the integer BEHZ kernels
    # (the split transform switches the FP64 path off)
    "n32768_30x5": (32768, [30] * 5),
    # 60-bit digits reduced mod 30-bit primes (and back) in the split transform's input reduction, under the 61-bit base
    "n32768_mixed": (32768, [60, 30, 30, 30, 60]),
    # 16 data residues and 17 key-level primes at n = 32768 (833 bits <= 881), integer kernels against a 49-bit base
    "n32768_49x17": (32768, [49] * 17),
    # 17 data residues, one beyond the library's limit (432 bits <= 438): each op gives the reference's words or refuses
    "n16384_24x18": (16384, [24] * 18),
}
PARAMS.update({
    "n32768_60x6": (32768, [0xfffffffff330001, 0xfffffffff550001, 0xfffffffff5a0001, 0xfffffffff6a0001, 0xfffffffff840001,
                            0xffffffffffc0001], 786433),
    "n32768_30x5": (32768, [0x3fbb0001, 0x3fd20001, 0x3fde0001, 0x3fed0001, 0x3ffc0001], 786433),
    "n32768_mixed": (32768, [0xfffffffff840001, 0x3fde0001, 0x3fed0001, 0x3ffc0001, 0xffffffffffc0001], 786433),
    "n32768_49x17": (32768, [0x1ffffff0b0001, 0x1ffffff230001, 0x1ffffff330001, 0x1ffffff390001, 0x1ffffff510001,
                             0x1ffffff570001, 0x1ffffff5c0001, 0x1ffffff780001, 0x1ffffff890001, 0x1ffffffa10001,
                             0x1ffffffa20001, 0x1ffffffb00001, 0x1ffffffb40001, 0x1ffffffba0001, 0x1ffffffd40001,
                             0x1ffffffea0001, 0x1fffffff50001], 786433),
    "n16384_24x18": (16384, [0xbe0001, 0xbe8001, 0xc18001, 0xc78001, 0xca0001, 0xcb8001, 0xcf0001, 0xd00001, 0xd08001,
                             0xd78001, 0xd80001, 0xe38001, 0xe40001, 0xee8001, 0xf60001, 0xfa0001, 0xfc0001, 0xfd0001], 786433),
})
WIDE = list(WIDE_BITS)

# Plain moduli beyond 20 bits on chains above: name -> (chain, how t is chosen).  A batching t is what
# PlainModulus::Batching(n, bits) returns, the largest prime = 1 mod 2n below 2^bits (CoeffModulus::Create(n, {bits})),
# skipping the chain's own primes where noted; tests/test_params.py re-derives each.
PLAIN_EDGE_T = {
    "n4096_t2": ("n4096", 2),                       # the smallest t: threshold 1, every nonzero coefficient is upper half
    "n4096_t2p40": ("n4096", 1 << 40),              # a 41-bit power of two, not batching
    "n8192_t30": ("n8192", ("batching", 30)),
    "n8192_t49": ("n8192", ("batching", 49)),       # the FP64 plain NTT at its width limit
    "n8192_t47": ("n8192", ("batching", 47)),       # = the first 47-bit FP64 auxiliary candidate, which must be skipped
    "n8192_t3p37": ("n8192", 3 ** 37),              # odd composite, 59 bits
    "n8192_54_t60": ("n8192_54", ("batching", 60)),  # 32 + 60 + bits(Q) >= 61 (k + 1): the reference's nB = k + 1
    "n8192_60_t60": ("n8192_60", ("batching", 60)),  # the largest 60-bit batching prime is in the chain: the next one
    "n16384_t60": ("n16384", ("batching", 60)),     # the 49-bit FP64 auxiliary base less than one prime above its range bound
}
PARAMS.update({
    "n4096_t2": (4096, DEFAULT_MODULI[4096], 2),
    "n4096_t2p40": (4096, DEFAULT_MODULI[4096], 1 << 40),
    "n8192_t30": (8192, DEFAULT_MODULI[8192], 0x3fff4001),
    "n8192_t49": (8192, DEFAULT_MODULI[8192], 0x1fffffff74001),
    "n8192_t47": (8192, DEFAULT_MODULI[8192], 0x7ffffffec001),
    "n8192_t3p37": (8192, DEFAULT_MODULI[8192], 3 ** 37),
    "n8192_54_t60": (8192, PARAMS["n8192_54"][1], 0xfffffffffffc001),
    "n8192_60_t60": (8192, PARAMS["n8192_60"][1], 0xffffffffffc4001),
    "n16384_t60": (16384, DEFAULT_MODULI[16384], 0xffffffffffe8001),
})
PLAIN_EDGE = list(PLAIN_EDGE_T)
