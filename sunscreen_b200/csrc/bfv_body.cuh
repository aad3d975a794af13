// bfv_body.cuh — per-coefficient bodies of the BFV hot path (everything that is not an NTT).
//
// Each body handles ONE coefficient index across all residues of one polynomial, with the residue loops
// fully unrolled (template<int K>) so the per-coefficient state stays in registers.  Thread mapping is
// always "consecutive threads -> consecutive coefficients" (coalesced 8-byte accesses per residue row;
// residue rows are n words apart).  The math is the reference's (SURVEY.md App. A.2/A.3/A.6/A.7), with
// constants pre-folded on the host (host_ctx.cpp); folded forms are exact modular identities, so the
// outputs are the same canonical residues the reference produces:
//   lift      = RNSTool::fastbconv_m_tilde + sm_mrq                       S/util/rns.cpp:991-1051,1098-1143
//   tensor    = bfv_multiply step (4)                                     S/evaluator.cpp:497-541
//   scale     = step (6) + RNSTool::fast_floor + fastbconv_sk             S/evaluator.cpp:549-566, rns.cpp:915-989,1053-1096
//   ks_mac    = switch_key_inplace accumulate                             S/evaluator.cpp:2475-2568
//   ks_moddown= switch_key_inplace mod-down, BFV branch                   S/evaluator.cpp:2618-2674
//   galois    = GaloisTool::apply_galois                                  S/util/galois.cpp:148-190
//   modswitch = RNSTool::divide_and_round_q_last_inplace                  S/util/rns.cpp:801-840
//   plain ops = multiply_add_plain_with_scaling_variant / plain lift      S/util/scalingvariant.cpp:69-188, S/evaluator.cpp:1939-1968
#pragma once
#include "modarith.cuh"
#include "ntt_fp_body.cuh"

#define B200_MAXK 16 // data residues per level (the reference's chain tops out at 15 data + 1 special for n=32768)

struct PrimeDev
{
    u64 p, r0, r1; // Barrett ratio floor(2^128/p) = r1:r0
};

// Device-side constants of one chain level (pointers into one device blob).
struct LevelDev
{
    int k, nB, nBsk;
    const PrimeDev *q;   // [k]
    const PrimeDev *bsk; // [nBsk] (B..., m_sk)
    u64 t;
    PrimeDev t_mod;
    PrimeDev gamma;
    // (the BEHZ lift and scale constants travel as kernel PARAMETERS: LiftIntC / ScaleIntC, LiftFpC / ScaleFpC below)
    // last-prime division (mod switch at this level)
    const u64 *inv_qlast;  // [2(k-1)]
    // plaintext
    const u64 *delta;      // [k]
    const u64 *plain_inc;  // [k]
    u64 q_mod_t, plain_thr;
    int fast_plain_lift;   // every q_i > t (ContextData::qualifiers().using_fast_plain_lift)
    // FP64 fast path (every prime of the level and of the aux base is below 2^47): the same constants as
    // integer-valued doubles, each entry {w, w/p_target}; primes as {p, 1/p}
    int fp;
    const double *dq;        // [2k]     {q_i, 1/q_i}
    const double *dbsk;      // [2nBsk]  {p_j, 1/p_j}
    // decrypt
    const u64 *dec_c;      // [2k]
    const u64 *dec_mat_t;  // [k]
    const u64 *dec_mat_g;  // [k]
    u64 inv_gamma_mod_t;
};

#if defined(__CUDA_ARCH__)
#define B200_LDG(ptr) __ldg(ptr)
#else
#define B200_LDG(ptr) (*(ptr))
#endif

B200_HD PrimeDev ld_prime(const PrimeDev *p)
{
    PrimeDev r;
    r.p = B200_LDG(&p->p);
    r.r0 = B200_LDG(&p->r0);
    r.r1 = B200_LDG(&p->r1);
    return r;
}

// ---------------------------------------------------------------------------------------------------------
// BEHZ lift: x (k residues, coeff form) -> z (nBsk residues, coeff form)
// ---------------------------------------------------------------------------------------------------------
// BEHZ constants of the integer path as kernel PARAMETERS (constant bank), like LiftFpC / ScaleFpC further down: the
// pointer-based tables cost one L1 transaction per use (up to ~550 per coefficient in scale at k = 15).
struct PrimeC
{
    u64 p, r0, r1;
};
template <int K>
struct LiftIntC
{
    int nBsk;
    u64 neg_inv_q_mod_mt;
    u64 q[K];                  // q_i
    u64 c[2 * K];              // Shoup pair of m~ (Q/q_i)^-1 mod q_i
    u64 mt[K];                 // (Q/q_i) mod m~
    PrimeC bsk[K + 2];
    u64 mat[(K + 2) * K];      // (Q/q_i) m~^-1 mod p_j
    u64 qm[K + 2];             // Q m~^-1 mod p_j
};
template <int K>
struct ScaleIntC
{
    int nB, nBsk;
    PrimeC q[K], bsk[K + 2];
    u64 c[2 * K];                  // Shoup pair of t (Q/q_i)^-1 mod q_i
    u64 tq[K + 2];                 // t Q^-1 mod p_j
    u64 mat[(K + 2) * K];          // -(Q/q_i) Q^-1 mod p_j
    u64 sk_c[2 * (K + 1)];         // Shoup pair of (B/b)^-1 mod b
    u64 sk_mat_q[K * (K + 1)];     // (B/b) mod q_i   (row i, column b; row stride K+1)
    u64 sk_mat_msk[K + 1];         // (B/b) mod m_sk
    u64 sk_prod_b_q[K];
    u64 sk_inv_b_msk;
};

template <int K>
B200_HD void lift_coeff(const LiftIntC<K> &L, const u64 *__restrict__ src /*[K][n]*/, u64 *__restrict__ dst /*[nBsk][n]*/,
                        long long n, long long c)
{
    u64 y[K];
    u64 ymt = 0;
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        y[i] = shoup_mul(src[i * n + c], L.c[2 * i], L.c[2 * i + 1], L.q[i]);
        ymt += y[i] * L.mt[i]; // only the low 32 bits matter (mod m~ = 2^32)
    }
    const u64 r = ((ymt & 0xffffffffULL) * L.neg_inv_q_mod_mt) & 0xffffffffULL;
#pragma unroll
    for (int j = 0; j < K + 2; j++)
    {
        if (j < L.nBsk)
        {
            const PrimeC P = L.bsk[j];
            // centred representative of r modulo p_j
            const u64 rc = (r >= 0x80000000ULL) ? r + P.p - 0x100000000ULL : r;
            u64 lo = 0, hi = 0;
#pragma unroll
            for (int i = 0; i < K; i++)
                mac128(y[i], L.mat[j * K + i], lo, hi);
            mac128(rc, L.qm[j], lo, hi);
            dst[j * n + c] = barrett128(lo, hi, P.p, P.r0, P.r1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// dyadic tensor product for one residue row: D_m = sum_{r+s=m} A_r * B_s  (sizes sa, sb <= 4)
// A, B point at residue row of poly 0; consecutive polys are `a_poly_stride` / `b_poly_stride` words apart.
// ---------------------------------------------------------------------------------------------------------
B200_HD void tensor_coeff(const PrimeDev &P, const u64 *__restrict__ A, long long a_poly_stride, int sa,
                          const u64 *__restrict__ B, long long b_poly_stride, int sb, u64 *__restrict__ D,
                          long long d_poly_stride, long long c)
{
    u64 a[4], b[4];
#pragma unroll
    for (int r = 0; r < 4; r++)
    {
        a[r] = r < sa ? A[r * a_poly_stride + c] : 0;
        b[r] = r < sb ? B[r * b_poly_stride + c] : 0;
    }
#pragma unroll
    for (int m = 0; m < 7; m++)
    {
        if (m < sa + sb - 1)
        {
            u64 lo = 0, hi = 0;
#pragma unroll
            for (int r = 0; r < 4; r++)
            {
                const int s = m - r;
                if (s >= 0 && s < 4 && r < sa && s < sb)
                    mac128(a[r], b[s], lo, hi);
            }
            D[m * d_poly_stride + c] = barrett128(lo, hi, P.p, P.r0, P.r1);
        }
    }
}

// operands of more than 4 polynomials (the reference allows any sizes with sa + sb - 1 <= 16, S/evaluator.cpp:395-567):
// plain loops over global memory — a rare shape, kept simple; works for every prime width
B200_HD void tensor_coeff_general(const PrimeDev &P, const u64 *__restrict__ A, long long a_poly_stride, int sa,
                                  const u64 *__restrict__ B, long long b_poly_stride, int sb, u64 *__restrict__ D,
                                  long long d_poly_stride, long long c)
{
    for (int m = 0; m < sa + sb - 1; m++)
    {
        u64 lo = 0, hi = 0;
        const int r0 = m - (sb - 1) > 0 ? m - (sb - 1) : 0;
        const int r1 = m < sa - 1 ? m : sa - 1;
        for (int r = r0; r <= r1; r++)
            mac128(A[r * a_poly_stride + c], B[(m - r) * b_poly_stride + c], lo, hi);
        D[m * d_poly_stride + c] = barrett128(lo, hi, P.p, P.r0, P.r1);
    }
}

// square of a size-2 ciphertext: D0 = A0^2, D1 = 2 A0 A1, D2 = A1^2  (S/evaluator.cpp:933-948)
B200_HD void square_coeff(const PrimeDev &P, const u64 *__restrict__ A, long long a_poly_stride, u64 *__restrict__ D,
                          long long d_poly_stride, long long c)
{
    const u64 a0 = A[c], a1 = A[a_poly_stride + c];
    u64 lo, hi;
    mul128(a0, a0, lo, hi);
    D[c] = barrett128(lo, hi, P.p, P.r0, P.r1);
    mul128(a0, a1, lo, hi);
    const u64 x = barrett128(lo, hi, P.p, P.r0, P.r1);
    D[d_poly_stride + c] = add_mod(x, x, P.p);
    mul128(a1, a1, lo, hi);
    D[2 * d_poly_stride + c] = barrett128(lo, hi, P.p, P.r0, P.r1);
}

// ---------------------------------------------------------------------------------------------------------
// BEHZ scale: (u in base q, v in base Bsk; coefficient form after INTT, canonical) -> out in base q
// src rows: [K q-rows][nBsk Bsk-rows], n words apart.
// ---------------------------------------------------------------------------------------------------------
template <int K>
B200_HD void scale_coeff(const ScaleIntC<K> &L, const u64 *__restrict__ src, u64 *__restrict__ dst, long long n, long long c)
{
    u64 y[K];
#pragma unroll
    for (int i = 0; i < K; i++)
        y[i] = shoup_mul(src[i * n + c], L.c[2 * i], L.c[2 * i + 1], L.q[i].p);
    // w_j = (t*v_j - FBC_{q->p_j}(t*u)) * Q^-1 mod p_j ; then y'_b = [w_b * (B/b)^-1]_b for b in B
    u64 yb[K + 1];
    u64 w_sk = 0;
    PrimeC MS = L.bsk[0];
#pragma unroll
    for (int j = 0; j < K + 2; j++)
    {
        if (j < L.nBsk)
        {
            const PrimeC P = L.bsk[j];
            u64 lo = 0, hi = 0;
            mac128(src[(K + j) * n + c], L.tq[j], lo, hi);
#pragma unroll
            for (int i = 0; i < K; i++)
                mac128(y[i], L.mat[j * K + i], lo, hi);
            const u64 w = barrett128(lo, hi, P.p, P.r0, P.r1);
            if (j < L.nB)
            {
                if (j < K + 1)
                    yb[j < K + 1 ? j : 0] = shoup_mul(w, L.sk_c[2 * (j < K + 1 ? j : 0)], L.sk_c[2 * (j < K + 1 ? j : 0) + 1], P.p);
            }
            else
            {
                w_sk = w;
                MS = P; // m_sk is the last prime of Bsk
            }
        }
    }
    // alpha_sk = (FBC_{B->m_sk}(w) - w_sk) * B^-1 mod m_sk
    u64 alpha;
    {
        u64 lo = 0, hi = 0;
#pragma unroll
        for (int b = 0; b < K + 1; b++)
            if (b < L.nB)
                mac128(yb[b], L.sk_mat_msk[b], lo, hi);
        mac128(MS.p - w_sk, L.sk_inv_b_msk, lo, hi);
        alpha = barrett128(lo, hi, MS.p, MS.r0, MS.r1);
    }
    const bool neg = alpha > (MS.p >> 1);
    const u64 mag = neg ? MS.p - alpha : alpha; // |centred alpha| < 2^60
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const PrimeC Q = L.q[i];
        u64 lo = 0, hi = 0;
#pragma unroll
        for (int b = 0; b < K + 1; b++)
            if (b < L.nB)
                mac128(yb[b], L.sk_mat_q[i * (K + 1) + b], lo, hi);
        const u64 pb = L.sk_prod_b_q[i];
        // alpha negative: + |alpha| * B ; alpha positive: + alpha * (q - B)
        mac128(mag, neg ? pb : Q.p - pb, lo, hi);
        dst[i * n + c] = barrett128(lo, hi, Q.p, Q.r0, Q.r1);
    }
}

// ---------------------------------------------------------------------------------------------------------
// key switch accumulate for one output residue I: acc_comp = sum_J op[J] * key[J][comp][key_res]  (mod p_I)
// ops: [K rows] (NTT_{p_I} of digit J), key: base pointer of key list, layout [J][comp(2)][Kkey][n].
// ---------------------------------------------------------------------------------------------------------
template <int K>
B200_HD void ksmac_coeff(const PrimeDev &P, const u64 *__restrict__ ops, long long op_stride, const u64 *__restrict__ key,
                         long long key_j_stride, long long key_comp_stride, u64 *__restrict__ out0,
                         u64 *__restrict__ out1, long long c)
{
    u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;
#pragma unroll
    for (int J = 0; J < K; J++)
    {
        const u64 x = ops[J * op_stride + c];
        mac128(x, B200_LDG(&key[J * key_j_stride + c]), lo0, hi0);
        mac128(x, B200_LDG(&key[J * key_j_stride + key_comp_stride + c]), lo1, hi1);
    }
    out0[c] = barrett128(lo0, hi0, P.p, P.r0, P.r1);
    out1[c] = barrett128(lo1, hi1, P.p, P.r0, P.r1);
}

// ---------------------------------------------------------------------------------------------------------
// divide-and-round by the last prime (BFV mod switch): rows [K] -> [K-1]
// ---------------------------------------------------------------------------------------------------------
// ld(i): canonical residue i of the coefficient (the last one is read first); st(i, v): result residue i < K - 1
template <int K, class Ld, class St>
B200_HD void modswitch_body(const PrimeDev *__restrict__ q, const u64 *__restrict__ inv_qlast, Ld ld, St st)
{
    const PrimeDev LP = ld_prime(&q[K - 1]);
    const u64 half = LP.p >> 1;
    u64 s = ld(K - 1) + half;
    s = s >= LP.p ? s - LP.p : s;
#pragma unroll
    for (int i = 0; i < K - 1; i++)
    {
        const PrimeDev Q = ld_prime(&q[i]);
        const u64 r = barrett64(s, Q.p, Q.r1);
        const u64 h = barrett64(half, Q.p, Q.r1);
        u64 v = ld(i) + (Q.p - r) + h;
        st(i, shoup_mul(v, B200_LDG(&inv_qlast[2 * i]), B200_LDG(&inv_qlast[2 * i + 1]), Q.p));
    }
}

template <int K>
B200_HD void modswitch_coeff(const PrimeDev *__restrict__ q, const u64 *__restrict__ inv_qlast, const u64 *__restrict__ src,
                             long long n, u64 *__restrict__ dst, long long c)
{
    modswitch_body<K>(q, inv_qlast, [&](int i) { return src[i * n + c]; }, [&](int i, u64 v) { dst[i * n + c] = v; });
}

// ---------------------------------------------------------------------------------------------------------
// Galois automorphism x -> x^g on one residue row (coefficient form), scatter form.
// ---------------------------------------------------------------------------------------------------------
B200_HD void galois_coeff(u64 p, const u64 *__restrict__ src, u64 *__restrict__ dst, int logn, u32 g, long long c)
{
    const u64 R = (u64)c * g;
    const u64 idx = R & ((1ULL << logn) - 1);
    const u64 v = src[c];
    dst[idx] = ((R >> logn) & 1) ? neg_mod(v, p) : v;
}

// ---------------------------------------------------------------------------------------------------------
// plaintext helpers
// ---------------------------------------------------------------------------------------------------------
// exact floor((a*b + add) / t) for a,b,add < t < 2^61: 128/64 division by the invariant t via Barrett + fix-up
B200_HD u64 div128_by_t(u64 lo, u64 hi, const PrimeDev &T)
{
    // qhat = floor(x * floor(2^128/t) / 2^128) is floor(x/t) or one less
    u64 carry = mulhi64(lo, T.r0);
    u64 t_lo, t_hi;
    mul128(lo, T.r1, t_lo, t_hi);
    u64 s1 = t_lo + carry;
    u64 c1 = t_hi + (s1 < t_lo);
    mul128(hi, T.r0, t_lo, t_hi);
    u64 s2 = s1 + t_lo;
    u64 c2 = t_hi + (s2 < t_lo);
    u64 qhat = hi * T.r1 + c1 + c2;
    u64 r = lo - qhat * T.p;
    if (r >= T.p)
    {
        r -= T.p;
        qhat++;
    }
    if (r >= T.p)
        qhat++;
    return qhat;
}

// scaled plaintext coefficient for add_plain/sub_plain: [m*Delta + fix]_{q_i}, fix = floor((Q mod t * m + floor((t+1)/2)) / t)
B200_HD u64 plain_scaled(const LevelDev &L, const PrimeDev &Q, int i, u64 m)
{
    u64 lo, hi;
    mul128(L.q_mod_t, m, lo, hi);
    const u64 thr = L.plain_thr;
    lo += thr;
    hi += lo < thr;
    const u64 fix = div128_by_t(lo, hi, L.t_mod);
    u64 l2, h2;
    mul128(m, B200_LDG(&L.delta[i]), l2, h2);
    l2 += fix;
    h2 += l2 < fix;
    return barrett128(l2, h2, Q.p, Q.r0, Q.r1);
}

// plain lift for multiply_plain: m -> m (+ plain_inc_i if m >= threshold), reduced mod q_i
B200_HD u64 plain_lift(const LevelDev &L, const PrimeDev &Q, int i, u64 m)
{
    u64 v = m >= L.plain_thr ? m + B200_LDG(&L.plain_inc[i]) : m;
    // fast lift: m < t < q_i and inc = q_i - t  =>  v < q_i already; general case needs a reduction
    return barrett64(v, Q.p, Q.r1);
}

// ---------------------------------------------------------------------------------------------------------
// decrypt scale-and-round: phase (k residues, coefficient form) -> plaintext coefficient mod t
// (RNSTool::decrypt_scale_and_round, S/util/rns.cpp:1145-1213)
// ---------------------------------------------------------------------------------------------------------
template <int K>
B200_HD u64 decrypt_coeff(const LevelDev &L, const u64 *__restrict__ src, long long n, long long c)
{
    u64 lt = 0, ht = 0, lg = 0, hg = 0;
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const u64 q = B200_LDG(&L.q[i].p);
        const u64 y = shoup_mul(src[i * n + c], B200_LDG(&L.dec_c[2 * i]), B200_LDG(&L.dec_c[2 * i + 1]), q);
        mac128(y, B200_LDG(&L.dec_mat_t[i]), lt, ht);
        mac128(y, B200_LDG(&L.dec_mat_g[i]), lg, hg);
    }
    const PrimeDev T = L.t_mod, G = L.gamma;
    const u64 vt = barrett128(lt, ht, T.p, T.r0, T.r1);
    const u64 vg = barrett128(lg, hg, G.p, G.r0, G.r1);
    u64 m;
    if (vg > (G.p >> 1))
        m = add_mod(vt, barrett64(G.p - vg, T.p, T.r1), T.p);
    else
        m = sub_mod(vt, barrett64(vg, T.p, T.r1), T.p);
    if (m)
    {
        u64 lo, hi;
        mul128(m, L.inv_gamma_mod_t, lo, hi);
        m = barrett128(lo, hi, T.p, T.r0, T.r1);
    }
    return m;
}


// =========================================================================================================
// FP64-pipe variants (the wide integer multiply is the slower pipe; see ntt_fp_body.cuh for the rationale and the exactness
// argument).  Same mathematics, same canonical outputs; used when LevelDev::fp is set.
// =========================================================================================================
B200_HD double fp_canon(double r, double p) // (-p, p) -> [0, p)
{
    return r < 0.0 ? B200_DADD(r, p) : r;
}
B200_HD u64 fp_to_u64(double r) // exact for 0 <= r < 2^52
{
#if defined(__CUDA_ARCH__)
    return (u64)__double_as_longlong(r + B200_TWO52) & 0x000FFFFFFFFFFFFFULL;
#else
    return (u64)(long long)r;
#endif
}
B200_HD double ldd(const double *p) { return B200_LDG(p); }

// BEHZ constants of the FP64 path, passed BY VALUE as a kernel parameter: they live in the constant bank, so each
// use is a constant operand of the DFMA/DMUL itself (or one uniform load) instead of a global load through L1 —
// with ~70 (lift) / ~140 (scale) constants per coefficient the pointer-based version kept L1TEX busy and starved the
// FP64 pipe.  Entries are {w, w/p_target} pairs, primes {p, 1/p}.
template <int K>
struct LiftFpC
{
    int nBsk;
    u64 neg_inv_q_mod_mt;
    u64 mt[K];                      // (Q/q_i) mod m~
    double dq[2 * K];               // {q_i, 1/q_i}
    double dbsk[2 * (K + 2)];       // {p_j, 1/p_j}
    double c[2 * K];                // m~ (Q/q_i)^-1 mod q_i
    double mat[2 * (K + 2) * K];    // (Q/q_i) m~^-1 mod p_j   (row j, column i)
    double qm[2 * (K + 2)];         // Q m~^-1 mod p_j
};
template <int K>
struct ScaleFpC
{
    int nB, nBsk;
    double dq[2 * K], dbsk[2 * (K + 2)];
    double c[2 * K];                     // t (Q/q_i)^-1 mod q_i
    double tq[2 * (K + 2)];              // t Q^-1 mod p_j
    double mat[2 * (K + 2) * K];         // -(Q/q_i) Q^-1 mod p_j
    double sk_c[2 * (K + 1)];            // (B/b)^-1 mod b
    double sk_mat_q[2 * K * (K + 1)];    // (B/b) mod q_i   (row i, column b)
    double sk_mat_msk[2 * (K + 1)];      // (B/b) mod m_sk
    double prod_b_q[2 * K], negprod_b_q[2 * K];
    double inv_b_msk[2];
};

template <int K>
B200_HD void lift_coeff_fp(const LiftFpC<K> &L, const u64 *__restrict__ src, u64 *__restrict__ dst, long long n, long long c)
{
    double y[K];
    u64 ymt = 0;
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const double q = L.dq[2 * i];
        y[i] = fp_canon(fp_mulmod(fp_from_u64(src[i * n + c]), L.c[2 * i], L.c[2 * i + 1], q), q);
        ymt += fp_to_u64(y[i]) * L.mt[i];
    }
    const u64 r = ((ymt & 0xffffffffULL) * L.neg_inv_q_mod_mt) & 0xffffffffULL;
    // centred representative of r (exact small integer)
    const double rc = (r >= 0x80000000ULL) ? -(double)(0x100000000ULL - r) : (double)r;
#pragma unroll
    for (int j = 0; j < K + 2; j++)
    {
        if (j < L.nBsk)
        {
            const double p = L.dbsk[2 * j], pinv = L.dbsk[2 * j + 1];
            double acc = fp_mulmod(rc, L.qm[2 * j], L.qm[2 * j + 1], p);
#pragma unroll
            for (int i = 0; i < K; i++)
                acc = B200_DADD(acc, fp_mulmod_term(i, y[i], L.mat[2 * (j * K + i)], L.mat[2 * (j * K + i) + 1], p));
            dst[j * n + c] = fp_to_canonical(acc, p, pinv);
        }
    }
}

B200_HD void tensor_coeff_fp(double p, double pinv, const u64 *__restrict__ A, long long a_poly_stride, int sa,
                             const u64 *__restrict__ B, long long b_poly_stride, int sb, u64 *__restrict__ D,
                             long long d_poly_stride, long long c)
{
    double a[4], b[4];
#pragma unroll
    for (int r = 0; r < 4; r++)
    {
        a[r] = r < sa ? fp_from_u64(A[r * a_poly_stride + c]) : 0.0;
        b[r] = r < sb ? fp_from_u64(B[r * b_poly_stride + c]) : 0.0;
    }
#pragma unroll
    for (int m = 0; m < 7; m++)
    {
        if (m < sa + sb - 1)
        {
            double acc = 0.0;
#pragma unroll
            for (int r = 0; r < 4; r++)
            {
                const int s = m - r;
                if (s >= 0 && s < 4 && r < sa && s < sb)
                    acc = B200_DADD(acc, fp_mulmod2(a[r], b[s], p, pinv));
            }
            D[m * d_poly_stride + c] = fp_to_canonical(acc, p, pinv);
        }
    }
}

B200_HD void square_coeff_fp(double p, double pinv, const u64 *__restrict__ A, long long a_poly_stride, u64 *__restrict__ D,
                             long long d_poly_stride, long long c)
{
    const double a0 = fp_from_u64(A[c]), a1 = fp_from_u64(A[a_poly_stride + c]);
    D[c] = fp_to_canonical(fp_mulmod2(a0, a0, p, pinv), p, pinv);
    const double x = fp_mulmod2(a0, a1, p, pinv);
    D[d_poly_stride + c] = fp_to_canonical(B200_DADD(x, x), p, pinv);
    D[2 * d_poly_stride + c] = fp_to_canonical(fp_mulmod2(a1, a1, p, pinv), p, pinv);
}

template <int K>
B200_HD void scale_coeff_fp(const ScaleFpC<K> &L, const u64 *__restrict__ src, u64 *__restrict__ dst, long long n, long long c)
{
    double y[K];
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const double q = L.dq[2 * i];
        y[i] = fp_canon(fp_mulmod(fp_from_u64(src[i * n + c]), L.c[2 * i], L.c[2 * i + 1], q), q);
    }
    double yb[K + 1];
    double w_sk = 0.0;
#pragma unroll
    for (int j = 0; j < K + 2; j++)
    {
        if (j < L.nBsk)
        {
            const double p = L.dbsk[2 * j], pinv = L.dbsk[2 * j + 1];
            double acc = fp_mulmod(fp_from_u64(src[(K + j) * n + c]), L.tq[2 * j], L.tq[2 * j + 1], p);
#pragma unroll
            for (int i = 0; i < K; i++)
                acc = B200_DADD(acc, fp_mulmod_term(i, y[i], L.mat[2 * (j * K + i)], L.mat[2 * (j * K + i) + 1], p));
            // canonical w_j
            double w = fp_renorm(acc, p, pinv);
            w = fp_canon(w, p);
            if (j < L.nB)
                yb[j < K + 1 ? j : 0] = fp_canon(fp_mulmod(w, L.sk_c[2 * (j < K + 1 ? j : 0)], L.sk_c[2 * (j < K + 1 ? j : 0) + 1], p), p);
            else
                w_sk = w;
        }
    }
    const int im = L.nB < K + 2 ? L.nB : K + 1; // index of m_sk in Bsk
    double ms = 0.0, msinv = 0.0;
#pragma unroll
    for (int j = 0; j < K + 2; j++) // constant-bank arrays want compile-time indices
        if (j == im)
        {
            ms = L.dbsk[2 * j];
            msinv = L.dbsk[2 * j + 1];
        }
    double alpha = fp_mulmod(-w_sk, L.inv_b_msk[0], L.inv_b_msk[1], ms);
#pragma unroll
    for (int b = 0; b < K + 1; b++)
        if (b < L.nB)
            alpha = B200_DADD(alpha, fp_mulmod_term(b, yb[b], L.sk_mat_msk[2 * b], L.sk_mat_msk[2 * b + 1], ms));
    alpha = fp_canon(fp_renorm(alpha, ms, msinv), ms);
    const bool neg = alpha > B200_DMUL(ms, 0.5); // m_sk odd: alpha > floor(m_sk/2)  <=>  alpha > m_sk/2
    const double mag = neg ? B200_DADD(ms, -alpha) : alpha;
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const double q = L.dq[2 * i], qinv = L.dq[2 * i + 1];
        const double pw = neg ? L.prod_b_q[2 * i] : L.negprod_b_q[2 * i];
        const double pwp = neg ? L.prod_b_q[2 * i + 1] : L.negprod_b_q[2 * i + 1];
        double acc = fp_mulmod(mag, pw, pwp, q);
#pragma unroll
        for (int b = 0; b < K + 1; b++)
            if (b < L.nB)
                acc = B200_DADD(acc, fp_mulmod_term(b, yb[b], L.sk_mat_q[2 * (i * (K + 1) + b)], L.sk_mat_q[2 * (i * (K + 1) + b) + 1], q));
        dst[i * n + c] = fp_to_canonical(acc, q, qinv);
    }
}

template <int K>
B200_HD void ksmac_coeff_fp(double p, double pinv, const u64 *__restrict__ ops, long long op_stride, const u64 *__restrict__ key,
                            long long key_j_stride, long long key_comp_stride, u64 *__restrict__ out0, u64 *__restrict__ out1,
                            long long c)
{
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int J = 0; J < K; J++)
    {
        const double x = fp_from_u64(ops[J * op_stride + c]);
        a0 = B200_DADD(a0, fp_mulmod2(x, fp_from_u64(B200_LDG(&key[J * key_j_stride + c])), p, pinv));
        a1 = B200_DADD(a1, fp_mulmod2(x, fp_from_u64(B200_LDG(&key[J * key_j_stride + key_comp_stride + c])), p, pinv));
    }
    out0[c] = fp_to_canonical(a0, p, pinv);
    out1[c] = fp_to_canonical(a1, p, pinv);
}
