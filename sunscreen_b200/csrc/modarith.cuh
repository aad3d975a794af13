// modarith.cuh — 64-bit modular arithmetic primitives for sm_90a (host/device).
//
// Everything here is exact unsigned integer arithmetic; "lazy" variants document their output range.
// Semantics follow the reference's scalar helpers (results, not code):
//   multiply_uint_mod_lazy / MultiplyUIntModOperand   S/util/uintarithsmallmod.h:300-426  (Shoup)
//   barrett_reduce_64 / barrett_reduce_128            S/util/uintarithsmallmod.h:167-262
// The host versions exist so tests/emu can run the kernel bodies on the CPU (test infrastructure
// only; the product library contains no CPU execution path).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif

typedef unsigned long long u64;
typedef unsigned int u32;

B200_HD u64 mulhi64(u64 a, u64 b)
{
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (u64)(((unsigned __int128)a * b) >> 64);
#endif
}

B200_HD void mul128(u64 a, u64 b, u64 &lo, u64 &hi)
{
    lo = a * b;
    hi = mulhi64(a, b);
}

// 128-bit accumulate: (lo,hi) += a*b
B200_HD void mac128(u64 a, u64 b, u64 &lo, u64 &hi)
{
    u64 pl = a * b, ph = mulhi64(a, b);
    lo += pl;
    hi += ph + (lo < pl);
}

// Shoup multiply: y * w mod q with wq = floor(w * 2^64 / q), w < q. Any 64-bit y. Output in [0, 2q).
B200_HD u64 shoup_mul_lazy(u64 y, u64 w, u64 wq, u64 q)
{
    u64 Q = mulhi64(wq, y);
    return w * y - Q * q;
}
B200_HD u64 shoup_mul(u64 y, u64 w, u64 wq, u64 q)
{
    u64 r = shoup_mul_lazy(y, w, wq, q);
    return r >= q ? r - q : r;
}

// Barrett for a single word: ratio1 = floor(2^64 / q) (the high word of floor(2^128/q) is what SEAL
// keeps in const_ratio[1]). Output canonical [0,q).
B200_HD u64 barrett64(u64 x, u64 q, u64 ratio1)
{
    u64 t = mulhi64(x, ratio1);
    u64 r = x - t * q;
    return r >= q ? r - q : r;
}

// Barrett for a 128-bit input (lo,hi) with the 2-word ratio floor(2^128/q) = (r0 low, r1 high).
// Valid for q < 2^63 and any 128-bit input whose quotient fits (inputs here are < 2^127).
B200_HD u64 barrett128(u64 lo, u64 hi, u64 q, u64 r0, u64 r1)
{
    // quotient estimate = floor( (hi*2^64+lo) * (r1*2^64+r0) / 2^128 ), dropping the lo*r0 low half
    u64 carry = mulhi64(lo, r0);
    u64 t_lo, t_hi;
    mul128(lo, r1, t_lo, t_hi);
    u64 s1 = t_lo + carry;
    u64 c1 = t_hi + (s1 < t_lo);
    mul128(hi, r0, t_lo, t_hi);
    u64 s2 = s1 + t_lo;
    u64 c2 = t_hi + (s2 < t_lo);
    u64 qhat = hi * r1 + c1 + c2;
    u64 r = lo - qhat * q;
    // estimate is low by at most 2
    r = r >= q ? r - q : r;
    return r >= q ? r - q : r;
}

B200_HD u64 add_mod(u64 a, u64 b, u64 q)
{
    u64 s = a + b;
    return s >= q ? s - q : s;
}
B200_HD u64 sub_mod(u64 a, u64 b, u64 q)
{
    return a >= b ? a - b : a + q - b;
}
B200_HD u64 neg_mod(u64 a, u64 q)
{
    return a ? q - a : 0;
}
