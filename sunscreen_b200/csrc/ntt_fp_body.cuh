// ntt_fp_body.cuh — the FP64-pipe negacyclic NTT / INTT for primes below 2^47 (fast path for GPUs with a full-rate FP64 pipe).
//
// Why: the 64-bit integer butterfly is bound by the wide integer multiply (IMAD.WIDE.U32 / IMAD.HI chains; tools/ubench.cu
// measures the pipe rates), while H100 issues DFMA/DMUL/DADD at 64 lanes/clk/SM (its full-rate FP64 pipe).  A modular
// multiplication by a precomputed twiddle can be done EXACTLY in 6 double-precision operations:
//     h = y*w (rounded)            l = fma(y, w, -h)        (h + l == y*w exactly)
//     q = rint(h * (1/p))          (DMUL + FRND.F64; the rounding runs on the XU pipe, not the FP64 pipe)
//     r = fma(-q, p, h) + l        (== y*w - q*p exactly: an integer of magnitude <= p(1/2 + 3|y|/2^53))
// (the twiddle tables therefore hold w only: one 8-byte load per butterfly group instead of a {w, w/p} pair)
// All values are integer-valued doubles in a signed lazy range; every operation above is exact as long as every
// value stays an integer of magnitude <= 2^53 (p up to 49 bits: host_ctx.h FP_PRIME_BITS), so the transform computes
// the same residues as the integer path — the outputs are
// reduced to the canonical [0,p) before they leave the kernel and are bit-identical to the reference's
// ntt_negacyclic_harvey / inverse_ntt_negacyclic_harvey (S/util/ntt.cpp:393-474).
//
// Schedule: identical pass structure to ntt_body.cuh (radix-8/16 groups, padded shared memory), except that
// the FIRST pass reads its group straight from global memory (u64 -> double) and the LAST pass writes its
// group straight to global memory (double -> canonical u64), saving two shared-memory round trips.
// Magnitude bookkeeping (host, b200_bfv.cu build_device): a forward butterfly adds the product bound above to the
// magnitude, an inverse butterfly doubles it on the sum path; whenever a pass could exceed 2^53 its inputs are first
// renormalised (x -= rint(x/p)*p, 2 FP64 ops + FRND).
#pragma once
#include "ntt_body.cuh"
#include <type_traits>

#if defined(__CUDA_ARCH__)
#define B200_DMUL(a, b) __dmul_rn((a), (b))
#define B200_DADD(a, b) __dadd_rn((a), (b))
#define B200_DFMA(a, b, c) __fma_rn((a), (b), (c))
// round to nearest integer: FRND.F64 issues on the XU pipe (measured 14.6 lanes/clk/SM, tools/ubench.cu), i.e. it
// takes the rounding OFF the FP64 pipe that bounds these kernels (the magic-number add/sub costs two FP64 slots)
__device__ __forceinline__ double b200_rint(double x)
{
    double r;
    asm("cvt.rni.f64.f64 %0, %1;" : "=d"(r) : "d"(x));
    return r;
}
#define B200_RINT(x) b200_rint(x)
#else
#include <cmath>
// host (tests/emu): built with -ffp-contract=off so these stay separate IEEE operations
#define B200_DMUL(a, b) ((a) * (b))
#define B200_DADD(a, b) ((a) + (b))
#define B200_DFMA(a, b, c) std::fma((a), (b), (c))
#define B200_RINT(x) std::nearbyint(x)
#endif

#define B200_MAGIC 6755399441055744.0   /* 1.5 * 2^52 */
#define B200_TWO52 4503599627370496.0   /* 2^52 */

struct NttPrimeFp
{
    double p, pinv;
    double inv_n[2], inv_n_w[2]; // {w, w/p} (only [0] is used by the transform)
    const double *fwd;           // [n] w, bit-reversed order
    const double *inv;
    const double *fwd16;         // transposed twiddles of the sub-stride-1 radix-16 pass: [15][n/16]
    const double *inv16;
    unsigned renorm_fwd, renorm_inv; // bit i: renormalise inputs of pass i (pass order of the respective transform)
    int enabled;
};

B200_HD double fp_mulmod(double y, double w, double wp, double p)
{
    const double h = B200_DMUL(y, w);
    const double l = B200_DFMA(y, w, -h);
    // magic-number rounding (two FP64 slots): the element-wise BEHZ kernels that use this form issue almost nothing
    // but modular products, and routing all their roundings through the 16-lane XU pipe was measured slower
    const double q = B200_DADD(B200_DFMA(y, wp, B200_MAGIC), -B200_MAGIC);
    return B200_DADD(B200_DFMA(-q, p, h), l);
}
// the same with the rounding on the XU pipe (DMUL + FRND.F64 instead of DFMA + DADD): one FP64 slot less, one XU slot more.
// The BEHZ kernels alternate the two forms term by term (B200_BEHZ_XU_MIX): routing ALL their roundings through the 16-lane
// XU pipe measured slower, none leaves that pipe idle (ncu: 2-6 %) while the FP64 pipe and the issue slots are the bound.
B200_HD double fp_mulmod_x(double y, double w, double wp, double p)
{
    const double h = B200_DMUL(y, w);
    const double l = B200_DFMA(y, w, -h);
    const double q = B200_RINT(B200_DMUL(y, wp));
    return B200_DADD(B200_DFMA(-q, p, h), l);
}
#ifndef B200_BEHZ_XU_MIX
#define B200_BEHZ_XU_MIX 1
#endif
// term `i` of an inner product: odd terms round on the XU pipe
B200_HD double fp_mulmod_term(int i, double y, double w, double wp, double p)
{
    return (B200_BEHZ_XU_MIX && (i & 1)) ? fp_mulmod_x(y, w, wp, p) : fp_mulmod(y, w, wp, p);
}
// general product a*b mod p for |a|,|b| < 2^47 (no precomputed quotient): result in (-p, p)
B200_HD double fp_mulmod2(double a, double b, double p, double pinv)
{
    const double h = B200_DMUL(a, b);
    const double l = B200_DFMA(a, b, -h);
    const double q = B200_RINT(B200_DMUL(h, pinv));
    return B200_DADD(B200_DFMA(-q, p, h), l);
}
B200_HD double fp_renorm(double x, double p, double pinv)
{
    const double q = B200_DADD(B200_DFMA(x, pinv, B200_MAGIC), -B200_MAGIC);
    return B200_DFMA(-q, p, x);
}
// same with the rounding on the XU pipe (used inside the transform, where FP64 issue slots are the bound)
B200_HD double fp_renorm_x(double x, double p, double pinv)
{
    const double q = B200_RINT(B200_DMUL(x, pinv));
    return B200_DFMA(-q, p, x);
}
// any lazy value -> canonical [0,p) as u64
template <bool XU = false>
B200_HD u64 fp_to_canonical(double x, double p, double pinv)
{
    double r = XU ? fp_renorm_x(x, p, pinv) : fp_renorm(x, p, pinv); // |r| <= 0.76 p
    r = r < 0.0 ? B200_DADD(r, p) : r;
#if defined(__CUDA_ARCH__)
    return (u64)__double_as_longlong(r + B200_TWO52) & 0x000FFFFFFFFFFFFFULL; // exact: 0 <= r < 2^47
#else
    return (u64)(long long)r;
#endif
}
B200_HD double fp_from_u64(u64 v) // exact for v < 2^52
{
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)(v | 0x4330000000000000ULL)) - B200_TWO52;
#else
    return (double)v;
#endif
}

B200_HD double fp_load_tw(const double *__restrict__ tw, int idx)
{
#if defined(__CUDA_ARCH__)
    return __ldg(tw + idx);
#else
    return tw[idx];
#endif
}

// All R-1 twiddles of a radix-2^L group, loaded up front so that their (L2) latency is paid once per group and
// overlaps the data loads.  Slot order: forward stage l, sub-group grp -> (2^l - 1) + grp;
// inverse stage l, sub-group grp -> R - (R >> l) + grp  (the TW16 tables use the same slot order).
// TWSRC: 0 = read-only global path (__ldg), 1 = `tw` points at the CTA's shared-memory copy of the table's first 512
// entries (plain load), 2 = developer ablation (no load at all: a constant stands in; results are meaningless)
template <int TWSRC>
B200_HD double fp_load_tw_src(const double *__restrict__ tw, int idx, const NttPrimeFp &P)
{
    if (TWSRC == 2)
        return B200_DADD(P.inv_n[0], (double)(idx & 7));
    if (TWSRC == 1)
        return tw[idx];
    return fp_load_tw(tw, idx);
}
template <int L, bool FWD, bool TW16, int TWSRC = 0>
B200_HD void fp_load_group_tw(double (&tws)[(1 << L) - 1], const double *__restrict__ tw, int g, int i, int logs, int logn, int M,
                              int n16, const NttPrimeFp &P, bool last_inv)
{
    constexpr int R = 1 << L;
#pragma unroll
    for (int l = 0; l < L; l++)
    {
        if (FWD)
        {
            const int tw_base = (M << l) + (i << l);
#pragma unroll
            for (int grp = 0; grp < (1 << l); grp++)
            {
                const int slot = (1 << l) - 1 + grp;
                tws[slot] = fp_load_tw_src<TWSRC>(tw, TW16 ? slot * n16 + g : tw_base + grp, P);
            }
        }
        else
        {
            const int m = 1 << (logn - 1 - logs - l);
            const int tw_base = m + (i << (L - l - 1));
#pragma unroll
            for (int grp = 0; grp < (R >> (l + 1)); grp++)
            {
                const int slot = R - (R >> l) + grp;
                if (last_inv && l == L - 1)
                    tws[slot] = P.inv_n_w[0]; // final stage of the whole inverse: twiddle pre-multiplied by n^-1
                else
                    tws[slot] = fp_load_tw_src<TWSRC>(tw, TW16 ? slot * n16 + g : tw_base + grp, P);
            }
        }
    }
}

// one butterfly stage `l` of a radix-2^L group (compile-time stage index so everything stays in registers)
// ABL bit 0 (developer ablation): the modular product is replaced by one DMUL (results are meaningless)
template <int ABL>
B200_HD double fp_mulmod_abl(double a, double b, double p, double pinv)
{
    if (ABL & 1)
        return B200_DMUL(a, b);
    return fp_mulmod2(a, b, p, pinv);
}
template <int L, int l, bool FWD, int ABL = 0>
B200_HD void fp_stage(double (&x)[1 << L], const double (&tws)[(1 << L) - 1], const NttPrimeFp &P, bool last_inv)
{
    constexpr int R = 1 << L;
    const double p = P.p, pinv = P.pinv;
    if (FWD)
    {
        constexpr int half = 1 << (L - 1 - l);
#pragma unroll
        for (int grp = 0; grp < (1 << l); grp++)
        {
            const double w = tws[(1 << l) - 1 + grp];
#pragma unroll
            for (int jj = 0; jj < half; jj++)
            {
                const int j = grp * 2 * half + jj;
                const double T = fp_mulmod_abl<ABL>(x[j + half], w, p, pinv);
                const double X = x[j];
                x[j] = B200_DADD(X, T);
                x[j + half] = B200_DADD(X, -T);
            }
        }
    }
    else
    {
        constexpr int half = 1 << l;
        const bool fold = last_inv && (l == L - 1);
#pragma unroll
        for (int grp = 0; grp < (R >> (l + 1)); grp++)
        {
            const double w = tws[R - (R >> l) + grp];
#pragma unroll
            for (int jj = 0; jj < half; jj++)
            {
                const int j = grp * 2 * half + jj;
                const double X = x[j], Y = x[j + half];
                const double U = B200_DADD(X, Y);
                x[j + half] = fp_mulmod_abl<ABL>(B200_DADD(X, -Y), w, p, pinv);
                x[j] = fold ? fp_mulmod2(U, P.inv_n[0], p, pinv) : U;
            }
        }
    }
}

// padded shared-memory index of element j of a group: base + j*2^logs.  For sub-strides that are multiples of 16 the
// padding of j*2^logs is a constant, and for the sub-stride-1 radix-16 group (base = 16 g) it is g — so only one
// padded base per group is computed at run time and every element offset is a compile-time constant after inlining.
B200_HD int fp_elem_index(int pbase, int base, int j, int logs)
{
    if (logs >= 4)
        return pbase + j * ((1 << logs) + (1 << (logs - 4)));
    if (logs == 0)
        return pbase + j + (((base & 15) + j) >> 4);
    return ntt_pad(base + (j << logs));
}

template <int L, bool FWD, bool SRC_GLOBAL, bool DST_GLOBAL, bool TW16 = false, bool RENORM = true, bool REDUCE = true, bool PRELOADED = false,
          bool RAW_IN = false /* shared memory holds the raw input words (landed by cp.async): convert on read */,
          bool TW_PRE = false /* the group's twiddles were prefetched by the caller (twpre) */,
          int TWSRC = 0 /* fp_load_tw_src */, int ABL = 0 /* developer ablations: 1 cheap product, 2 no global loads, 4 no global stores */,
          bool REFILL = false /* streaming kernel, last inverse pass: once this group's inputs have been consumed, the NEXT
                                 polynomial's words for the same slots are requested (cp.async) from `refill` */>
B200_HD void ntt_fp_group(double *sm, const u64 *__restrict__ gsrc, u64 *__restrict__ gdst, int g, int logs, int logn, int M,
                          const NttPrimeFp &P, bool renorm, bool last_inv, bool reduce_input, u64 pint, u64 ratio1,
                          const u64 *pre = nullptr /* PRELOADED: the group's 2^L raw input words, already in registers */,
                          const double *twpre = nullptr, const double *stw = nullptr /* TWSRC == 1: shared-memory table */,
                          const u64 *refill = nullptr)
{
    constexpr int R = 1 << L;
    const int s = 1 << logs;
    const int i = g >> logs;
    const int o = g & (s - 1);
    const int base = (i << (logs + L)) + o;
    const int pbase = ntt_pad(base);
    const double p = P.p;
    const double *__restrict__ tw = TWSRC == 1 ? stw : TW16 ? (FWD ? P.fwd16 : P.inv16) : (FWD ? P.fwd : P.inv);
    const int n16 = 1 << (logn - 4); // groups of the radix-16 pass (TW16 layout: [slot][group])
    double tws[R - 1];
    if (TW_PRE)
    {
#pragma unroll
        for (int j = 0; j < R - 1; j++)
            tws[j] = twpre[j];
    }
    else
        fp_load_group_tw<L, FWD, TW16, TWSRC>(tws, tw, g, i, logs, logn, M, n16, P, last_inv);
    double x[R];
#pragma unroll
    for (int j = 0; j < R; j++)
    {
        if (SRC_GLOBAL)
        {
            u64 v = PRELOADED ? pre[j] : (ABL & 2) ? (u64)(base + j) : gsrc[base + (j << logs)];
            if (REDUCE && reduce_input)
                v = barrett64(v, pint, ratio1);
            x[j] = fp_from_u64(v);
        }
        else if (RAW_IN)
        {
#if defined(__CUDA_ARCH__)
            u64 v = (u64)__double_as_longlong(sm[fp_elem_index(pbase, base, j, logs)]);
            if (REDUCE && reduce_input)
                v = barrett64(v, pint, ratio1);
            x[j] = fp_from_u64(v);
#endif
        }
        else
        {
#if defined(__CUDA_ARCH__)
            if (PRELOADED) // shared-memory pass with the group's values fetched one group ahead by the caller (bit patterns)
                x[j] = __longlong_as_double((long long)pre[j]);
            else
#endif
                x[j] = sm[fp_elem_index(pbase, base, j, logs)];
        }
        if (RENORM && renorm)
            x[j] = fp_renorm_x(x[j], p, P.pinv);
    }
    fp_stage<L, 0, FWD, ABL>(x, tws, P, last_inv);
    if constexpr (L > 1)
        fp_stage<L, 1, FWD, ABL>(x, tws, P, last_inv);
    if constexpr (L > 2)
        fp_stage<L, 2, FWD, ABL>(x, tws, P, last_inv);
    if constexpr (L > 3)
        fp_stage<L, 3, FWD, ABL>(x, tws, P, last_inv);
#if defined(__CUDA_ARCH__)
    if (REFILL && !SRC_GLOBAL && refill)
    {
        // the slots this thread has just read are free (their values are in registers and have been used): land the next
        // polynomial's words in them while this one is finished and written out
#pragma unroll
        for (int j = 0; j < R; j++)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(sm + fp_elem_index(pbase, base, j, logs))),
                         "l"(refill + base + (j << logs))
                         : "memory");
    }
#endif
#pragma unroll
    for (int j = 0; j < R; j++)
    {
        if (DST_GLOBAL && (ABL & 4))
        {
            const u64 v = fp_to_canonical<true>(x[j], p, P.pinv);
            if (v == 0xFFFFFFFFFFFFFFFFULL) // never: keeps the value live without the store traffic
                gdst[base + (j << logs)] = v;
        }
        else if (DST_GLOBAL)
        {
#if defined(__CUDA_ARCH__)
            if (ABL & 8)
                __stcs(gdst + base + (j << logs), fp_to_canonical<true>(x[j], p, P.pinv));
            else
#endif
                gdst[base + (j << logs)] = fp_to_canonical<true>(x[j], p, P.pinv);
        }
        else
            sm[fp_elem_index(pbase, base, j, logs)] = x[j];
    }
}

template <int L, bool FWD, bool SG, bool DG>
B200_HD void ntt_fp_pass(double *sm, const u64 *gsrc, u64 *gdst, int n, int logs, int logn, int M, const NttPrimeFp &P,
                         bool renorm, bool last_inv, bool reduce_input, u64 pint, u64 ratio1, int tid, int nthreads)
{
    const int ngroups = n >> L;
    for (int g = tid; g < ngroups; g += nthreads)
        ntt_fp_group<L, FWD, SG, DG>(sm, gsrc, gdst, g, logs, logn, M, P, renorm, last_inv, reduce_input, pint, ratio1);
}

template <bool FWD, bool SG, bool DG>
B200_HD void ntt_fp_pass_dispatch(int L, double *sm, const u64 *gsrc, u64 *gdst, int n, int logs, int logn, int M,
                                  const NttPrimeFp &P, bool renorm, bool last_inv, bool reduce_input, u64 pint, u64 ratio1,
                                  int tid, int nthreads)
{
    switch (L)
    {
    case 1: ntt_fp_pass<1, FWD, SG, DG>(sm, gsrc, gdst, n, logs, logn, M, P, renorm, last_inv, reduce_input, pint, ratio1, tid, nthreads); break;
    case 2: ntt_fp_pass<2, FWD, SG, DG>(sm, gsrc, gdst, n, logs, logn, M, P, renorm, last_inv, reduce_input, pint, ratio1, tid, nthreads); break;
    case 3: ntt_fp_pass<3, FWD, SG, DG>(sm, gsrc, gdst, n, logs, logn, M, P, renorm, last_inv, reduce_input, pint, ratio1, tid, nthreads); break;
    default: ntt_fp_pass<4, FWD, SG, DG>(sm, gsrc, gdst, n, logs, logn, M, P, renorm, last_inv, reduce_input, pint, ratio1, tid, nthreads); break;
    }
}

// One CTA: FP64 transform of one residue polynomial. `smd` holds ntt_smem_words(n) doubles.
template <bool FWD>
B200_HD void ntt_fp_block_body(const NttJob &job, const NttPrimeFp &P, const NttPrime &PI, const u64 *src, u64 *dst, double *smd,
                               int tid, int nthreads)
{
    const int logn = job.logn;
    const int n = 1 << logn;
    const int np = job.npass;
    const bool red = job.reduce_input != 0;
    if (FWD)
    {
        int done = 0;
        for (int pi = 0; pi < np; pi++)
        {
            const int L = job.pass_L[pi];
            const int M = 1 << done;
            const int logs = logn - done - L;
            const bool rn = (P.renorm_fwd >> pi) & 1;
            const bool first = pi == 0, last = pi == np - 1;
            if (first && last)
                ntt_fp_pass_dispatch<true, true, true>(L, smd, src, dst, n, logs, logn, M, P, rn, false, red, PI.p, PI.ratio1, tid, nthreads);
            else if (first)
                ntt_fp_pass_dispatch<true, true, false>(L, smd, src, dst, n, logs, logn, M, P, rn, false, red, PI.p, PI.ratio1, tid, nthreads);
            else if (last)
                ntt_fp_pass_dispatch<true, false, true>(L, smd, src, dst, n, logs, logn, M, P, rn, false, false, 0, 0, tid, nthreads);
            else
                ntt_fp_pass_dispatch<true, false, false>(L, smd, src, dst, n, logs, logn, M, P, rn, false, false, 0, 0, tid, nthreads);
            B200_SYNC();
            done += L;
        }
    }
    else
    {
        int logs = 0;
        int step = 0;
        for (int pi = np - 1; pi >= 0; pi--, step++)
        {
            const int L = job.pass_L[pi];
            const bool rn = (P.renorm_inv >> step) & 1;
            const bool first = step == 0, last = pi == 0;
            if (first && last)
                ntt_fp_pass_dispatch<false, true, true>(L, smd, src, dst, n, logs, logn, 0, P, rn, true, red, PI.p, PI.ratio1, tid, nthreads);
            else if (first)
                ntt_fp_pass_dispatch<false, true, false>(L, smd, src, dst, n, logs, logn, 0, P, rn, false, red, PI.p, PI.ratio1, tid, nthreads);
            else if (last)
                ntt_fp_pass_dispatch<false, false, true>(L, smd, src, dst, n, logs, logn, 0, P, rn, true, false, 0, 0, tid, nthreads);
            else
                ntt_fp_pass_dispatch<false, false, false>(L, smd, src, dst, n, logs, logn, 0, P, rn, false, false, 0, 0, tid, nthreads);
            B200_SYNC();
            logs += L;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Statically scheduled variant (device fast path): compile-time pass schedule and thread count, group loops
// fully unrolled so that all global loads of the first pass are issued before the first butterfly.
// Same group routine as above (which the CPU emulation tests cover); only the control flow is specialised.
// ---------------------------------------------------------------------------------------------------------
#if defined(__CUDACC__)
template <int LOGN> struct NttSched;
template <> struct NttSched<12> { static constexpr int NP = 3; static constexpr int L0 = 4, L1 = 4, L2 = 4, L3 = 0; };
template <> struct NttSched<13> { static constexpr int NP = 4; static constexpr int L0 = 3, L1 = 3, L2 = 3, L3 = 4; };
template <> struct NttSched<14> { static constexpr int NP = 4; static constexpr int L0 = 3, L1 = 3, L2 = 4, L3 = 4; };

// the same schedules for the host's magnitude bookkeeping (renorm masks are per pass of the schedule that runs)
inline int ntt_static_schedule(int logn, int *L)
{
    auto fill = [&](int np, int a, int b, int c_, int d) { L[0] = a; L[1] = b; L[2] = c_; L[3] = d; return np; };
    if (logn == 12)
        return fill(NttSched<12>::NP, NttSched<12>::L0, NttSched<12>::L1, NttSched<12>::L2, NttSched<12>::L3);
    if (logn == 13)
        return fill(NttSched<13>::NP, NttSched<13>::L0, NttSched<13>::L1, NttSched<13>::L2, NttSched<13>::L3);
    if (logn == 14)
        return fill(NttSched<14>::NP, NttSched<14>::L0, NttSched<14>::L1, NttSched<14>::L2, NttSched<14>::L3);
    return 0;
}
template <int LOGN, int PI> struct NttSchedL
{
    static constexpr int value = PI == 0 ? NttSched<LOGN>::L0 : PI == 1 ? NttSched<LOGN>::L1 : PI == 2 ? NttSched<LOGN>::L2 : NttSched<LOGN>::L3;
};
template <int LOGN, int PI> struct NttSchedDone // stages completed before forward pass PI
{
    static constexpr int value = NttSchedDone<LOGN, PI - 1>::value + NttSchedL<LOGN, PI - 1>::value;
};
template <int LOGN> struct NttSchedDone<LOGN, 0> { static constexpr int value = 0; };

// VAR (bit mask): 1 = the table's first 512 twiddles (every stage whose butterflies span >= n/256 points) are copied into
// shared memory once per CTA and read from there (short latency, no L2 round trip per group); 2 / 4 / 8 = developer
// ablations for tools/ntt_ablate.py (no twiddle loads / one-DMUL products / no global traffic): results are meaningless,
// they only measure what each component costs.
// VAR & 8192 (forward only): the first pass reads sigma_g(src) instead of src, for the Galois automorphism X -> X^g of a
// coefficient-form row mod q: destination word e is source word i = e g^-1 mod 2n, negated mod q (gal_q) where i >= n.  `gal`
// is g^-1 mod 2n.  The negation happens mod q, before job.reduce_input reduces the word mod the transform's prime.
#define B200_NTT_TWS_ENTRIES 512
template <int LOGN, int NT, bool FWD, int STEP /*0..NP-1 in execution order*/, int VAR = 0>
struct NttFpStaticPass
{
    static __device__ __forceinline__ void run(const NttJob &job, const NttPrimeFp &P, const NttPrime &PI_, const u64 *src, u64 *dst,
                                               double *smd, int tid, long long item, int slot, const u64 *nsrc = nullptr,
                                               unsigned gal = 0, u64 gal_q = 0)
    {
#if defined(__CUDA_ARCH__)
        constexpr int N = 1 << LOGN;
        constexpr int NP = NttSched<LOGN>::NP;
        constexpr int PIDX = FWD ? STEP : NP - 1 - STEP;       // index into the forward schedule
        constexpr int L = NttSchedL<LOGN, PIDX>::value;
        constexpr int DONE = NttSchedDone<LOGN, PIDX>::value;  // forward stages before this pass
        constexpr int LOGS = LOGN - DONE - L;                  // log2 sub-stride (same for the mirrored inverse pass)
        constexpr int M = 1 << DONE;
        // Direct global I/O only where consecutive lanes touch consecutive words (large sub-stride).  The
        // sub-stride-1 pass would make every lane touch its own 128-byte line (32 L1 wavefronts per request), so
        // its global side is staged through shared memory with coalesced copies instead.
        constexpr bool EDGE_IN = STEP == 0, EDGE_OUT = STEP == NP - 1;
#ifndef B200_NTT_TW_PREFETCH
#define B200_NTT_TW_PREFETCH 1
#endif
#ifndef B200_NTT_DIRECT_IN
#define B200_NTT_DIRECT_IN 1
#endif
        // Direct global I/O only where consecutive lanes touch consecutive words (large sub-stride).  Staging the forward
        // input through cp.async instead (B200_NTT_DIRECT_IN=0) measures the same within noise (0.72 vs 0.71 ms for
        // 16384 polynomials): the per-CTA timeline (tools/ntt_timeline.py) shows the copy-in itself takes only 2.6 us of
        // a CTA's 18.4 us; the kernel is co-limited by the FP64 pipe (52 %) and the shared-memory pipe (55-58 %).
        // VAR & 16: streaming (persistent) kernel — the polynomial's raw words are ALREADY on their way into shared memory when a
        // pass sequence starts (requested during the previous polynomial's last pass, into slots that pass had finished with)
        constexpr bool STREAM = (VAR & 16) != 0;
        // VAR & 2048: warp-private sub-transforms.  After the first forward pass (radix 2^L0) the polynomial falls apart into 2^L0
        // independent blocks of N >> L0 points; with the blocks divided evenly among the warps each warp owns its block(s) for the remaining passes, so
        // those passes (and the write-out of the block) need only __syncwarp — one block-wide barrier per polynomial instead of
        // four — and the block's early-pass twiddles are warp-uniform.  The inverse mirrors it (warp-private until the last pass).
        // With more warps than blocks (n = 16384: 32 warps, 8 blocks) a block belongs to a GROUP of warps that synchronises on its
        // own named barrier: eight independent four-warp groups inside the one CTA an SM can hold.
        constexpr int WP_BLOCKS = 1 << NttSchedL<LOGN, 0>::value, WP_WARPS = NT / 32;
        constexpr int WP_TG = WP_WARPS > WP_BLOCKS ? 32 * (WP_WARPS / WP_BLOCKS) : 32; // threads of one group
        constexpr int WP_NG = NT / WP_TG;                                               // groups in the CTA (<= 15 named barriers)
        constexpr bool WP = (VAR & 2048) != 0 && (WP_BLOCKS % WP_NG) == 0 && WP_NG <= 15 && !(STREAM && FWD);
        constexpr bool WPSTEP = WP && (FWD ? STEP >= 1 : STEP + 1 < NP); // this pass runs group-private
        const int wlane = tid % WP_TG, wwarp = tid / WP_TG;                // position inside the group, group index
        auto wp_sync = [&]() {
            if constexpr (WP_TG == 32)
                __syncwarp();
            else
                asm volatile("bar.sync %0, %1;" ::"r"(1 + wwarp), "r"(WP_TG) : "memory");
        };
        // VAR & 4096: the polynomial stays in shared memory at the hand-off to / from the fused dyadic step (mul_cluster.cu): the
        // forward transform leaves its lazy result there (no copy-out), the inverse finds canonical values there (no copy-in)
        constexpr bool KEEP_OUT = (VAR & 4096) != 0 && FWD, SMEM_IN = (VAR & 4096) != 0 && !FWD;
        constexpr bool SG = EDGE_IN && LOGS >= 5 && B200_NTT_DIRECT_IN && !STREAM && !SMEM_IN,
                       DG = EDGE_OUT && LOGS >= 5 && !(VAR & 128) && !KEEP_OUT; // 128: always stage the output
        constexpr bool GATHER = (VAR & 8192) != 0 && FWD && EDGE_IN;
        static_assert(!GATHER || SG, "the Galois gather reads the first pass's words straight from global memory");
        auto gather_ld = [&](int e) -> u64 {
            const unsigned i = ((unsigned)e * gal) & (2u * N - 1u);
            const u64 x = src[i & (N - 1)];
            return i < (unsigned)N ? x : (x ? gal_q - x : 0);
        };
        constexpr bool TW16 = (L == 4 && LOGS == 0);
        constexpr int TWSRC = (VAR & 2) ? 2 : ((VAR & 1) && !TW16 && (1 << (DONE + L)) <= B200_NTT_TWS_ENTRIES) ? 1 : 0;
        constexpr int ABL = ((VAR & 4) ? 1 : 0) | ((VAR & (8 | 32)) ? 2 : 0) | ((VAR & (8 | 64)) ? 4 : 0) | ((VAR & 512) ? 8 : 0); // 32 / 64: loads / stores only; 512: streaming (evict-first) hints
        double *stw = smd + ntt_smem_words(N); // VAR & 1: B200_NTT_TWS_ENTRIES doubles behind the polynomial
        if (STEP == 0 && (VAR & 1))
        {
            const double *__restrict__ twg = FWD ? P.fwd : P.inv;
            for (int e = tid; e < B200_NTT_TWS_ENTRIES; e += NT)
                stw[e] = fp_load_tw(twg, e);
            if (SG)
                __syncthreads(); // (the staged copy-in below has its own barrier)
        }
        constexpr int NGROUPS = N >> L;
        constexpr int ITERS = (NGROUPS + NT - 1) / NT;
        const bool rn = (((FWD ? P.renorm_fwd : P.renorm_inv) >> STEP) & 1) || (!FWD && STEP == 0 && job.tensor_mode);
        const bool red = EDGE_IN && job.reduce_input != 0;
        const int ptid = ntt_pad(tid);              // NT is a multiple of 16: pad(tid + it*NT) = pad(tid) + it*(NT + NT/16)
        constexpr int PNT = NT + (NT >> 4);
        if constexpr (EDGE_IN && SMEM_IN)
            __syncthreads(); // the whole CTA's twiddle copy above is complete (the first pass may span other warps' values)
        else if (EDGE_IN && !SG)
        { // coalesced copy-in: u64 -> double
            if (!FWD && job.tensor_mode)
            {
                // fused BEHZ step (4): this slot is (m, row); operands are canonical NTT-form words
                const int R = job.t_rows;
                const int m = slot / R, row = slot - m * R;
                const int np_ = job.tensor_mode == 2 ? job.t_sa : job.t_sa + job.t_sb;
                const long long ps = (long long)R * N; // polynomial stride inside an item
                const u64 *A = job.tsrc + ((long long)item * np_ * R + row) * N;
                const u64 *B = job.tensor_mode == 2 ? A : A + (long long)job.t_sa * ps;
#pragma unroll
                for (int it = 0; it < N / NT; it++)
                {
                    const int e = tid + it * NT;
                    double acc = 0.0;
                    if (job.tensor_mode == 2)
                    {
                        const double a0 = fp_from_u64(A[e]), a1 = fp_from_u64(A[ps + e]);
                        if (m == 0)
                            acc = fp_mulmod2(a0, a0, P.p, P.pinv);
                        else if (m == 1)
                        {
                            acc = fp_mulmod2(a0, a1, P.p, P.pinv);
                            acc = B200_DADD(acc, acc);
                        }
                        else
                            acc = fp_mulmod2(a1, a1, P.p, P.pinv);
                    }
                    else
                    {
                        for (int r = 0; r < job.t_sa; r++)
                        {
                            const int s = m - r;
                            if (s >= 0 && s < job.t_sb)
                                acc = B200_DADD(acc, fp_mulmod2(fp_from_u64(A[r * ps + e]), fp_from_u64(B[s * ps + e]), P.p, P.pinv));
                        }
                    }
                    smd[ptid + it * PNT] = acc; // lazy, |acc| < 4p: the first pass renormalises if its bound needs it
                }
            }
            else if (STREAM)
                asm volatile("cp.async.wait_all;" ::: "memory"); // requested by the kernel prologue / the previous polynomial's last pass
            else
            {
                // asynchronous copy (LDGSTS): no registers are held, so all N/NT requests of a thread are in flight at
                // once; the words land raw and the first pass converts them when it reads (RAW_IN)
                const unsigned sbase = (unsigned)__cvta_generic_to_shared(smd + ptid);
                if (ABL & 2)
                {
#pragma unroll
                    for (int it = 0; it < N / NT; it++)
                        smd[ptid + it * PNT] = __longlong_as_double((long long)(tid + it * NT));
                }
                else if (WP && !FWD && !STREAM)
                { // warp-private: the warp lands its OWN block (the first passes of the inverse stay inside it)
                    constexpr int BS = N / WP_NG;
#pragma unroll
                    for (int r = 0; r < BS / WP_TG; r++)
                    {
                        const int e = wwarp * BS + wlane + WP_TG * r;
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smd + ntt_pad(e))), "l"(src + e)
                                     : "memory");
                    }
                    asm volatile("cp.async.commit_group;" ::: "memory");
                    asm volatile("cp.async.wait_group 0;" ::: "memory");
                }
                else
                {
#pragma unroll
                    for (int it = 0; it < N / NT; it++)
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sbase + (unsigned)(it * PNT * 8)), "l"(src + tid + it * NT)
                                     : "memory");
                    asm volatile("cp.async.commit_group;" ::: "memory");
                    asm volatile("cp.async.wait_group 0;" ::: "memory");
                }
            }
            if (WP && !FWD && !STREAM && !job.tensor_mode && !(ABL & 2)) // (streaming: the block was requested by other threads)
                wp_sync();
            else
                __syncthreads();
            if (job.timeline && tid == 0)
            {
                unsigned long long t;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                job.timeline[(unsigned long long)blockIdx.x * 8 + 6] = t; // copy-in complete
            }
        }
        constexpr bool RAW = EDGE_IN && !SG && !SMEM_IN; // (the tensor-fused copy-in writes doubles: handled by the run-time flag below)
        // renormalisation / input reduction are block-uniform run-time flags: branch ONCE to a compile-time variant
        // (as predicated code they cost 12 FP64 ops and ~10 IMADs per element whether needed or not)
        // group handled by this thread in iteration `it`: block-strided by default, inside the warp's own block when warp-private
        auto gidx = [&](int it) { return WPSTEP ? wwarp * (NGROUPS / WP_NG) + wlane + WP_TG * it : tid + it * NT; };
        auto groups = [&](auto RN, auto RD) {
            if constexpr (STREAM && FWD && EDGE_OUT && !DG)
            {
                // streaming forward transform, last (sub-stride-1) pass: the 32 groups a warp handles in one iteration are one
                // contiguous region of 32 R elements that no other warp touches in this pass, so the region is written out
                // (coalesced, canonical) by the warp itself as soon as its groups are done — no block-wide barrier — and
                // the NEXT polynomial's words for the same region are requested into the slots just read
                constexpr int R = 1 << L;
                static_assert(NGROUPS % NT == 0, "whole iterations");
                const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
                for (int it = 0; it < ITERS; it++)
                {
                    const int g = tid + it * NT;
                    ntt_fp_group<L, FWD, false, false, TW16, decltype(RN)::value, false, false, false, false, TWSRC, ABL>(
                        smd, src, dst, g, LOGS, LOGN, M, P, true, false, true, PI_.p, PI_.ratio1, nullptr, nullptr, stw);
                    __syncwarp();
                    const int e0 = ((warp << 5) + it * NT) << L;
#pragma unroll
                    for (int r = 0; r < R; r++)
                    {
                        const int e = e0 + lane + 32 * r;
                        const int pe = ntt_pad(e);
                        dst[e] = fp_to_canonical<true>(smd[pe], P.p, P.pinv);
                        if (nsrc)
                            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smd + pe)), "l"(nsrc + e)
                                         : "memory");
                    }
                }
            }
            else if constexpr (SG && NGROUPS % NT == 0 && ITERS > 1 && !GATHER)
            {
                // direct first pass, software-pipelined: the raw words of group it+1 are requested before group `it` is
                // transformed, so one DRAM latency is exposed per polynomial instead of one per group
                constexpr int R = 1 << L;
                u64 cur[R], nxt[R];
                {
                    const int g = tid, i0 = g >> LOGS, o0 = g & ((1 << LOGS) - 1);
                    const int b0 = (i0 << (LOGS + L)) + o0;
#pragma unroll
                    for (int j = 0; j < R; j++)
                        cur[j] = (ABL & 2) ? (u64)(b0 + j) : (ABL & 8) ? __ldcs(src + b0 + (j << LOGS)) : src[b0 + (j << LOGS)];
                }
#pragma unroll
                for (int it = 0; it < ITERS; it++)
                {
                    const int g = tid + it * NT;
                    if (it + 1 < ITERS)
                    {
                        const int gn = g + NT, in_ = gn >> LOGS, on = gn & ((1 << LOGS) - 1);
                        const int bn = (in_ << (LOGS + L)) + on;
#pragma unroll
                        for (int j = 0; j < R; j++)
                            nxt[j] = (ABL & 2) ? (u64)(bn + j) : (ABL & 8) ? __ldcs(src + bn + (j << LOGS)) : src[bn + (j << LOGS)];
                    }
                    ntt_fp_group<L, FWD, SG, DG, TW16, decltype(RN)::value, decltype(RD)::value, true, false, false, TWSRC, ABL>(
                        smd, src, dst, g, LOGS, LOGN, M, P, true, !FWD && EDGE_OUT, true, PI_.p, PI_.ratio1, cur, nullptr, stw);
#pragma unroll
                    for (int j = 0; j < R; j++)
                        cur[j] = nxt[j];
                }
            }
            else if constexpr (GATHER)
            {
                // the Galois gather: each group's words are loaded (scattered) right before it is transformed; no prefetch of
                // the next group, whose registers the index arithmetic needs (the prefetching form spills)
                constexpr int R = 1 << L;
                static_assert(NGROUPS % NT == 0, "whole iterations");
#pragma unroll
                for (int it = 0; it < ITERS; it++)
                {
                    const int g = tid + it * NT, i0 = g >> LOGS, o0 = g & ((1 << LOGS) - 1);
                    const int b0 = (i0 << (LOGS + L)) + o0;
                    u64 cur[R];
#pragma unroll
                    for (int j = 0; j < R; j++)
                        cur[j] = gather_ld(b0 + (j << LOGS));
                    ntt_fp_group<L, FWD, SG, DG, TW16, decltype(RN)::value, decltype(RD)::value, true, false, false, TWSRC, ABL>(
                        smd, src, dst, g, LOGS, LOGN, M, P, true, !FWD && EDGE_OUT, true, PI_.p, PI_.ratio1, cur, nullptr, stw);
                }
            }
            else
            {
                auto run = [&](auto RAWF) {
                    if constexpr ((VAR & 1024) != 0 && L <= 3 && NGROUPS % NT == 0 && ITERS > 1 && !decltype(RAWF)::value)
                    {
                        // VAR & 1024: the DATA of group it+1 is read from shared memory before group `it` is transformed (instead of
                        // prefetching twiddles): hides the shared-memory latency / queueing behind the butterflies
                        constexpr int R = 1 << L;
                        u64 xc[R], xn[R];
                        auto fetch = [&](u64(&dstv)[R], int g) {
                            const int i_ = g >> LOGS, o_ = g & ((1 << LOGS) - 1);
                            const int b_ = (i_ << (LOGS + L)) + o_;
                            const int pb_ = ntt_pad(b_);
#pragma unroll
                            for (int j = 0; j < R; j++)
                                dstv[j] = (u64)__double_as_longlong(smd[fp_elem_index(pb_, b_, j, LOGS)]);
                        };
                        fetch(xc, gidx(0));
#pragma unroll
                        for (int it = 0; it < ITERS; it++)
                        {
                            const int g = gidx(it);
                            if (it + 1 < ITERS)
                                fetch(xn, gidx(it + 1));
                            ntt_fp_group<L, FWD, false, DG, TW16, decltype(RN)::value, false, true, false, false, TWSRC, ABL, STREAM && !FWD && DG>(
                                smd, src, dst, g, LOGS, LOGN, M, P, true, !FWD && EDGE_OUT, true, PI_.p, PI_.ratio1, xc, nullptr, stw, nsrc);
#pragma unroll
                            for (int j = 0; j < R; j++)
                                xc[j] = xn[j];
                        }
                    }
                    else if constexpr (L <= 3 && NGROUPS % NT == 0 && ITERS > 1 && B200_NTT_TW_PREFETCH && TWSRC == 0)
                    {
                        // the twiddles of group it+1 are requested before group `it` is transformed: their L1/L2 latency
                        // (the kernel's largest stall reason when profiled) overlaps the butterflies
                        constexpr int R = 1 << L;
                        const double *__restrict__ twt = FWD ? P.fwd : P.inv;
                        double twc[R - 1], twn[R - 1];
                        fp_load_group_tw<L, FWD, false>(twc, twt, gidx(0), gidx(0) >> LOGS, LOGS, LOGN, M, 0, P, !FWD && EDGE_OUT);
#pragma unroll
                        for (int it = 0; it < ITERS; it++)
                        {
                            const int g = gidx(it);
                            if (it + 1 < ITERS)
                                fp_load_group_tw<L, FWD, false>(twn, twt, gidx(it + 1), gidx(it + 1) >> LOGS, LOGS, LOGN, M, 0, P, !FWD && EDGE_OUT);
                            ntt_fp_group<L, FWD, SG, DG, TW16, decltype(RN)::value, decltype(RD)::value, false, decltype(RAWF)::value, true, 0, ABL,
                                         STREAM && !FWD && DG>(
                                smd, src, dst, g, LOGS, LOGN, M, P, true, !FWD && EDGE_OUT, true, PI_.p, PI_.ratio1, nullptr, twc, nullptr, nsrc);
#pragma unroll
                            for (int j = 0; j < R - 1; j++)
                                twc[j] = twn[j];
                        }
                    }
                    else
                    {
#pragma unroll
                        for (int it = 0; it < ITERS; it++)
                        {
                            const int g = gidx(it);
                            if (NGROUPS % NT == 0 || g < NGROUPS)
                                ntt_fp_group<L, FWD, SG, DG, TW16, decltype(RN)::value, decltype(RD)::value, false, decltype(RAWF)::value, false, TWSRC, ABL,
                                             STREAM && !FWD && DG>(
                                    smd, src, dst, g, LOGS, LOGN, M, P, true, !FWD && EDGE_OUT, true, PI_.p, PI_.ratio1, nullptr, nullptr, stw, nsrc);
                        }
                    }
                };
                if constexpr (RAW)
                {
                    if (!FWD && job.tensor_mode)
                        run(std::false_type{});
                    else
                        run(std::true_type{});
                }
                else
                    run(std::false_type{});
            }
        };
        if (rn)
        {
            if ((SG || RAW) && red)
                groups(std::true_type{}, std::true_type{});
            else
                groups(std::true_type{}, std::false_type{});
        }
        else
        {
            if ((SG || RAW) && red)
                groups(std::false_type{}, std::true_type{});
            else
                groups(std::false_type{}, std::false_type{});
        }
        if (WPSTEP && (FWD || STEP + 2 < NP))
            wp_sync(); // the next pass (or the write-out) of this group touches only the group's own block(s)
        else if (!(STREAM && EDGE_OUT)) // (the streaming kernel's next polynomial starts with wait_all + barrier)
            __syncthreads();
        if (job.timeline && tid == 0)
        {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            job.timeline[(unsigned long long)blockIdx.x * 8 + 2 + STEP] = t;
        }
        if (EDGE_OUT && !DG && !(STREAM && FWD) && !KEEP_OUT)
        { // coalesced copy-out: lazy double -> canonical u64
            if constexpr ((VAR & 256) != 0)
            { // two adjacent words per thread: one 128-bit store (the pair never straddles a pad: even index, runs of 16)
#pragma unroll
                for (int it = 0; it < N / (2 * NT); it++)
                {
                    const int e = 2 * (tid + it * NT);
                    const int pe = ntt_pad(e);
                    const u64 v0 = fp_to_canonical<true>(smd[pe], P.p, P.pinv), v1 = fp_to_canonical<true>(smd[pe + 1], P.p, P.pinv);
                    __stcs(reinterpret_cast<ulonglong2 *>(dst + e), make_ulonglong2(v0, v1));
                }
            }
            else if constexpr (WP)
            { // the warp writes its own block out as soon as its last pass is done (no block-wide barrier before this)
                constexpr int BS = N / WP_NG;
#pragma unroll
                for (int r = 0; r < BS / WP_TG; r++)
                {
                    const int e = wwarp * BS + wlane + WP_TG * r;
                    dst[e] = fp_to_canonical<true>(smd[ntt_pad(e)], P.p, P.pinv);
                }
            }
            else
#pragma unroll
            for (int it = 0; it < N / NT; it++)
            {
                const u64 v = fp_to_canonical<true>(smd[ptid + it * PNT], P.p, P.pinv);
                if (!(ABL & 4) || v == 0xFFFFFFFFFFFFFFFFULL)
                    dst[tid + it * NT] = v;
            }
        }
        if (STEP + 1 < NP)
            NttFpStaticPass<LOGN, NT, FWD, (STEP + 1 < NP ? STEP + 1 : STEP), VAR>::run(job, P, PI_, src, dst, smd, tid, item, slot, nsrc, gal, gal_q);
#endif
    }
};
#endif // __CUDACC__
