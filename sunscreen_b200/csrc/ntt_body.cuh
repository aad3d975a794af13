// ntt_body.cuh — batched negacyclic NTT / INTT over one residue polynomial per CTA.
//
// Observable contract = the reference's (S/util/ntt.cpp:393-474, S/util/dwthandler.h:94-356; SURVEY.md App. A.1):
//   forward : natural-order input  -> bit-reversed-order output,  out[i] = sum_j in[j] * psi^((2*bitrev(i)+1) j)
//   inverse : exact inverse including n^-1
// psi = minimal primitive 2n-th root (host_ctx.cpp).  The internal schedule is our own: the polynomial
// lives in shared memory (padded, conflict-free), and each pass does 3 or 4 butterfly stages in
// registers (radix-8 / radix-16 groups) before the next block-wide exchange.  Butterflies are
// Harvey-lazy ([0,4p) forward, [0,2p) inverse) with Shoup twiddles (w, floor(w*2^64/p)).
//
// Twiddle tables (device, per prime):  fwd[idx] = psi^bitrev(idx) for idx in [1,n)  (same indexing as the
// reference's root_powers), inv[idx] = fwd[idx]^-1 (our own layout: the inverse of the forward twiddle of
// the same butterfly group), each stored as 2 words {w, wq}.
//
// The bodies are __host__ __device__ and written as strided loops over work items with B200_SYNC()
// between phases, so tests/emu can execute a CTA sequentially (tid=0,nthreads=1) on the CPU.
#pragma once
#include "modarith.cuh"

#if defined(__CUDA_ARCH__)
#define B200_SYNC() __syncthreads()
#else
#define B200_SYNC() ((void)0)
#endif

struct NttPrime
{
    u64 p;
    u64 ratio1;        // floor(2^64/p) (Barrett, single word)
    u64 inv_n, inv_n_q;      // n^-1 mod p and its Shoup quotient
    u64 inv_n_w, inv_n_w_q;  // n^-1 * inv[1] mod p (last inverse stage folded) and its Shoup quotient
    const u64 *fwd;    // [2n] words
    const u64 *inv;    // [2n] words
};

struct NttPrimeFp; // ntt_fp_body.cuh

// One item of a key switch whose items carry their own Galois element and key (b200_apply_galois_many, the BSGS linear
// transform): the source ciphertext [2][k][n], the key list [J][2][key_rows][n], where the per-item mod-down writes the
// result ([2][k][n]; unused by the summing mod-down), the element g and g^-1 mod 2n.
struct B200GalItem
{
    const u64 *ct;
    const u64 *key;
    u64 *dst;
    unsigned g, ginv;
};

// One launch = `items` x `slots` residue polynomials.
struct NttJob
{
    int logn;
    int slots;                 // residue polynomials per item
    const int *slot_prime;     // [slots] index into primes[]
    const long long *slot_src; // [slots] source offset (words) inside an item
    const long long *slot_dst; // [slots] destination offset (words) inside an item
    long long src_item_stride; // words
    long long dst_item_stride; // words
    const u64 *src;
    u64 *dst;
    const NttPrime *primes;
    const NttPrimeFp *fprimes; // FP64 fast-path descriptors, same indexing as primes[]
    int reduce_input;          // 1: inputs are arbitrary 64-bit words -> Barrett to [0,p) on load
    long long items;           // number of items in this launch
    int split;                 // 1: n is too large for one CTA: each CTA transforms one HALF (size n/2) as a sub-transform;
                               //    the remaining butterfly stage over the whole polynomial runs in ntt_outer_kernel
    int npass;                 // forward pass schedule (host: ntt_schedule); inverse runs it mirrored
    int pass_L[8];
    // up to two alternative sources: slots [0, alt_end[0]) read from alt_src[0], slots [alt_end[0], alt_end[1]) from
    // alt_src[1], the rest from `src` (one launch transforms rows that live in different buffers — the inputs of a
    // multiply and its lifted rows — instead of one latency-bound launch per buffer); alt_end = {0, 0}: off
    int alt_end[2];
    const u64 *alt_src[2];
    long long alt_stride[2];
};

B200_HD const u64 *ntt_src_ptr(const NttJob &job, long long item, int slot)
{
    if (slot < job.alt_end[0])
        return job.alt_src[0] + item * job.alt_stride[0] + job.slot_src[slot];
    if (slot < job.alt_end[1])
        return job.alt_src[1] + item * job.alt_stride[1] + job.slot_src[slot];
    return job.src + item * job.src_item_stride + job.slot_src[slot];
}

B200_HD int ntt_pad(int e) { return e + (e >> 4); }
B200_HD int ntt_smem_words(int n) { return n + (n >> 4); }

// pass schedules: stages per pass for the forward transform (the inverse uses the mirror image).
// Rule: the last forward pass is radix-16 so that the pass before it has sub-stride >= 16 (conflict-free).
inline int ntt_schedule(int logn, int *passes)
{
    int np = 0;
    int rem = logn;
    // number of radix-16 passes a, radix-8 passes b with 4a+3b = logn where possible
    int a = 0, b = 0;
    for (a = (rem >= 4 ? 1 : 0); a <= rem / 4; a++)
        if ((rem - 4 * a) % 3 == 0)
            break;
    if (a > rem / 4)
    { // not representable with a>=1 (logn in {1,2,3,5,6,9}): fall back to a greedy split
        int r = rem;
        while (r > 0)
        {
            int L = r >= 4 && r != 5 && r != 6 ? 4 : (r >= 3 ? 3 : r);
            passes[np++] = L;
            r -= L;
        }
        // order ascending so larger radices come last
        for (int i = 0; i < np; i++)
            for (int j = i + 1; j < np; j++)
                if (passes[j] < passes[i])
                {
                    int t = passes[i];
                    passes[i] = passes[j];
                    passes[j] = t;
                }
        return np;
    }
    // prefer more radix-16 passes when both decompositions exist (fewer exchanges)
    while (rem - 4 * (a + 3) >= 0 && (rem - 4 * (a + 3)) % 3 == 0)
        a += 3;
    b = (rem - 4 * a) / 3;
    for (int i = 0; i < b; i++)
        passes[np++] = 3;
    for (int i = 0; i < a; i++)
        passes[np++] = 4;
    return np;
}

// twiddle pair {w, floor(w 2^64 / p)} number idx of a table
B200_HD void ntt_load_tw(const u64 *__restrict__ tw, int idx, u64 &w, u64 &wq)
{
#if defined(__CUDA_ARCH__)
    const ulonglong2 t2 = __ldg(reinterpret_cast<const ulonglong2 *>(tw) + idx);
    w = t2.x;
    wq = t2.y;
#else
    w = tw[2 * idx];
    wq = tw[2 * idx + 1];
#endif
}

// One butterfly stage with a COMPILE-TIME stage index: every x[] index is a constant after unrolling, so the group stays
// in registers (with a run-time stage loop ptxas kept the inverse group's 16 words in local memory).
template <int L, int l>
B200_HD void ntt_fwd_stage(u64 (&x)[1 << L], const u64 *__restrict__ tw, int tw_base, u64 p, u64 two_p)
{
    constexpr int half = 1 << (L - 1 - l);
#pragma unroll
    for (int grp = 0; grp < (1 << l); grp++)
    {
        u64 w, wq;
        ntt_load_tw(tw, tw_base + grp, w, wq);
#pragma unroll
        for (int jj = 0; jj < half; jj++)
        {
            const int j = grp * 2 * half + jj;
            u64 X = x[j];
            X = X >= two_p ? X - two_p : X;
            const u64 T = shoup_mul_lazy(x[j + half], w, wq, p);
            x[j] = X + T;
            x[j + half] = X - T + two_p;
        }
    }
}
template <int L, int l>
B200_HD void ntt_inv_stage(u64 (&x)[1 << L], const u64 *__restrict__ tw, int tw_base, const NttPrime &P, u64 two_p, bool fold)
{
    constexpr int R = 1 << L;
    constexpr int half = 1 << l;
    const u64 p = P.p;
#pragma unroll
    for (int grp = 0; grp < (R >> (l + 1)); grp++)
    {
        u64 w, wq;
        if (fold)
        {
            w = P.inv_n_w;
            wq = P.inv_n_w_q;
        }
        else
            ntt_load_tw(tw, tw_base + grp, w, wq);
#pragma unroll
        for (int jj = 0; jj < half; jj++)
        {
            const int j = grp * 2 * half + jj;
            const u64 X = x[j], Y = x[j + half];
            u64 U = X + Y;
            U = U >= two_p ? U - two_p : U;
            const u64 V = shoup_mul_lazy(X - Y + two_p, w, wq, p);
            x[j] = fold ? shoup_mul_lazy(U, P.inv_n, P.inv_n_q, p) : U;
            x[j + half] = V;
        }
    }
}

// ---- forward: Cooley-Tukey group of 2^L elements, L stages -------------------------------------------
template <int L>
B200_HD void ntt_fwd_group(u64 *sm, int g, int logs /*log2 sub-stride*/, int M /*groups at first stage (times the
                           sub-transform multiplier 2+b when the CTA handles half b of a split transform)*/,
                           const u64 *__restrict__ tw, u64 p)
{
    constexpr int R = 1 << L;
    const int s = 1 << logs;
    const int i = g >> logs;
    const int o = g & (s - 1);
    const int base = (i << (logs + L)) + o;
    const u64 two_p = p << 1;
    u64 x[R];
#pragma unroll
    for (int j = 0; j < R; j++)
        x[j] = sm[ntt_pad(base + (j << logs))];
    ntt_fwd_stage<L, 0>(x, tw, M + i, p, two_p);
    if constexpr (L > 1)
        ntt_fwd_stage<L, 1>(x, tw, (M << 1) + (i << 1), p, two_p);
    if constexpr (L > 2)
        ntt_fwd_stage<L, 2>(x, tw, (M << 2) + (i << 2), p, two_p);
    if constexpr (L > 3)
        ntt_fwd_stage<L, 3>(x, tw, (M << 3) + (i << 3), p, two_p);
#pragma unroll
    for (int j = 0; j < R; j++)
        sm[ntt_pad(base + (j << logs))] = x[j];
}

// ---- inverse: Gentleman-Sande group of 2^L elements, L stages (gap grows) -----------------------------
// `last` marks the pass containing the final stage (m = 1), where n^-1 is folded in.
template <int L>
B200_HD void ntt_inv_group(u64 *sm, int g, int logs, int logn, const u64 *__restrict__ tw, const NttPrime &P,
                           bool last, int mult = 1)
{
    constexpr int R = 1 << L;
    const int s = 1 << logs;
    const int i = g >> logs;
    const int o = g & (s - 1);
    const int base = (i << (logs + L)) + o;
    const u64 two_p = P.p << 1;
    u64 x[R];
#pragma unroll
    for (int j = 0; j < R; j++)
        x[j] = sm[ntt_pad(base + (j << logs))];
    // stage l: global gap s*2^l, m = n/(2 gap) groups; twiddle index m*mult + (i << (L-l-1)) + grp
    const int m0 = 1 << (logn - 1 - logs);
    ntt_inv_stage<L, 0>(x, tw, m0 * mult + (i << (L - 1)), P, two_p, last && L == 1);
    if constexpr (L > 1)
        ntt_inv_stage<L, 1>(x, tw, (m0 >> 1) * mult + (i << (L - 2)), P, two_p, last && L == 2);
    if constexpr (L > 2)
        ntt_inv_stage<L, 2>(x, tw, (m0 >> 2) * mult + (i << (L - 3)), P, two_p, last && L == 3);
    if constexpr (L > 3)
        ntt_inv_stage<L, 3>(x, tw, (m0 >> 3) * mult + i, P, two_p, last && L == 4);
#pragma unroll
    for (int j = 0; j < R; j++)
        sm[ntt_pad(base + (j << logs))] = x[j];
}

template <bool FWD, int L>
B200_HD void ntt_pass(u64 *sm, int n, int logs, int logn, int M, const NttPrime &P, bool last, int tid, int nthreads)
{
    // M carries the sub-transform multiplier in both directions (forward: groups-at-first-stage * mult; inverse: mult)
    const int ngroups = n >> L;
    for (int g = tid; g < ngroups; g += nthreads)
    {
        if (FWD)
            ntt_fwd_group<L>(sm, g, logs, M, P.fwd, P.p);
        else
            ntt_inv_group<L>(sm, g, logs, logn, P.inv, P, last, M);
    }
}

template <bool FWD>
B200_HD void ntt_pass_dispatch(int L, u64 *sm, int n, int logs, int logn, int M, const NttPrime &P, bool last, int tid,
                               int nthreads)
{
    switch (L)
    {
    case 1: ntt_pass<FWD, 1>(sm, n, logs, logn, M, P, last, tid, nthreads); break;
    case 2: ntt_pass<FWD, 2>(sm, n, logs, logn, M, P, last, tid, nthreads); break;
    case 3: ntt_pass<FWD, 3>(sm, n, logs, logn, M, P, last, tid, nthreads); break;
    default: ntt_pass<FWD, 4>(sm, n, logs, logn, M, P, last, tid, nthreads); break;
    }
}

// One CTA: transform residue polynomial `block` of the job. sm holds ntt_smem_words(n) words.
template <bool FWD>
B200_HD void ntt_block_body(const NttJob &job, long long block, u64 *sm, int tid, int nthreads)
{
    // split transforms: CTA (poly, half) works on n/2 coefficients with twiddle multiplier 2 + half
    // job.split = log2 of the number of parts: 1 -> halves after one global stage, 2 -> quarters after two
    const int parts = 1 << job.split;
    const int half = (int)(block & (parts - 1));
    const long long poly = block >> job.split;
    const int logn = job.logn - job.split;
    const int n = 1 << logn;
    const int mult = job.split ? parts + half : 1; // part `half` of stage s covers groups [half*2^(s-split), ...)
    const long long item = poly / job.slots;
    const int slot = (int)(poly - item * job.slots);
    const NttPrime P = job.primes[job.slot_prime[slot]];
    const u64 *src = ntt_src_ptr(job, item, slot) + (long long)half * n;
    u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot] + (long long)half * n;
    const u64 p = P.p;

    for (int e = tid; e < n; e += nthreads)
    {
        u64 v = src[e];
        if (job.reduce_input)
            v = barrett64(v, p, P.ratio1);
        sm[ntt_pad(e)] = v;
    }
    B200_SYNC();

    const int np = job.npass;
    if (FWD)
    {
        int done = 0; // stages completed
        for (int pi = 0; pi < np; pi++)
        {
            const int L = job.pass_L[pi];
            const int M = 1 << done;
            const int logs = logn - done - L;
            ntt_pass_dispatch<true>(L, sm, n, logs, logn, M * mult, P, false, tid, nthreads);
            B200_SYNC();
            done += L;
        }
        const u64 two_p = p << 1;
        for (int e = tid; e < n; e += nthreads)
        {
            u64 v = sm[ntt_pad(e)];
            v = v >= two_p ? v - two_p : v;
            v = v >= p ? v - p : v;
            dst[e] = v;
        }
    }
    else
    {
        int logs = 0;
        for (int pi = np - 1; pi >= 0; pi--)
        {
            const int L = job.pass_L[pi];
            const bool last = (pi == 0) && !job.split; // a sub-transform leaves the final stage (and n^-1) to ntt_outer
            ntt_pass_dispatch<false>(L, sm, n, logs, logn, mult, P, last, tid, nthreads);
            B200_SYNC();
            logs += L;
        }
        for (int e = tid; e < n; e += nthreads)
        {
            u64 v = sm[ntt_pad(e)];
            v = v >= p ? v - p : v;
            dst[e] = v;
        }
    }
}


// The butterfly stage a split transform performs over the whole polynomial in global memory:
//   forward : first stage (m = 1, gap n/2, twiddle fwd[1]), canonical output, src -> dst
//   inverse : last stage (m = 1) with n^-1 folded in, in place on dst (input = the two inverse sub-transforms, < p)
// Two global stages at once for a transform split in four (n = 32768: the quarters then fit three CTAs per SM):
//   forward : stages m = 1 (gap n/2, twiddle 1) and m = 2 (gap n/4, twiddles 2 and 3), canonical output, src -> dst
//   inverse : the mirrored Gentleman-Sande stages with n^-1 folded into the last one, in place on dst
template <bool FWD>
B200_HD void ntt_outer_quad(const NttJob &job, long long poly, int j)
{
    const int n = 1 << job.logn, q4 = n >> 2;
    const long long item = poly / job.slots;
    const int slot = (int)(poly - item * job.slots);
    const NttPrime P = job.primes[job.slot_prime[slot]];
    const u64 p = P.p;
    u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
    if (FWD)
    {
        const u64 *src = ntt_src_ptr(job, item, slot);
        u64 a0 = src[j], a1 = src[j + q4], a2 = src[j + 2 * q4], a3 = src[j + 3 * q4];
        if (job.reduce_input)
        {
            a0 = barrett64(a0, p, P.ratio1);
            a1 = barrett64(a1, p, P.ratio1);
            a2 = barrett64(a2, p, P.ratio1);
            a3 = barrett64(a3, p, P.ratio1);
        }
        const u64 t2 = shoup_mul(a2, P.fwd[2], P.fwd[3], p), t3 = shoup_mul(a3, P.fwd[2], P.fwd[3], p);
        const u64 b0 = add_mod(a0, t2, p), b2 = sub_mod(a0, t2, p), b1 = add_mod(a1, t3, p), b3 = sub_mod(a1, t3, p);
        const u64 u1 = shoup_mul(b1, P.fwd[4], P.fwd[5], p), u3 = shoup_mul(b3, P.fwd[6], P.fwd[7], p);
        dst[j] = add_mod(b0, u1, p);
        dst[j + q4] = sub_mod(b0, u1, p);
        dst[j + 2 * q4] = add_mod(b2, u3, p);
        dst[j + 3 * q4] = sub_mod(b2, u3, p);
    }
    else
    {
        const u64 a0 = dst[j], a1 = dst[j + q4], a2 = dst[j + 2 * q4], a3 = dst[j + 3 * q4];
        const u64 b0 = add_mod(a0, a1, p), b1 = shoup_mul(sub_mod(a0, a1, p), P.inv[4], P.inv[5], p);
        const u64 b2 = add_mod(a2, a3, p), b3 = shoup_mul(sub_mod(a2, a3, p), P.inv[6], P.inv[7], p);
        dst[j] = shoup_mul(add_mod(b0, b2, p), P.inv_n, P.inv_n_q, p);
        dst[j + 2 * q4] = shoup_mul(sub_mod(b0, b2, p), P.inv_n_w, P.inv_n_w_q, p);
        dst[j + q4] = shoup_mul(add_mod(b1, b3, p), P.inv_n, P.inv_n_q, p);
        dst[j + 3 * q4] = shoup_mul(sub_mod(b1, b3, p), P.inv_n_w, P.inv_n_w_q, p);
    }
}

template <bool FWD>
B200_HD void ntt_outer_pair(const NttJob &job, long long poly, int j)
{
    const int n = 1 << job.logn;
    const long long item = poly / job.slots;
    const int slot = (int)(poly - item * job.slots);
    const NttPrime P = job.primes[job.slot_prime[slot]];
    const u64 p = P.p;
    if (FWD)
    {
        const u64 *src = ntt_src_ptr(job, item, slot);
        u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
        u64 X = src[j], Y = src[j + (n >> 1)];
        if (job.reduce_input)
        {
            X = barrett64(X, p, P.ratio1);
            Y = barrett64(Y, p, P.ratio1);
        }
        const u64 T = shoup_mul(Y, P.fwd[2], P.fwd[3], p);
        dst[j] = add_mod(X, T, p);
        dst[j + (n >> 1)] = sub_mod(X, T, p);
    }
    else
    {
        u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
        const u64 X = dst[j], Y = dst[j + (n >> 1)];
        dst[j] = shoup_mul(add_mod(X, Y, p), P.inv_n, P.inv_n_q, p);
        dst[j + (n >> 1)] = shoup_mul(sub_mod(X, Y, p), P.inv_n_w, P.inv_n_w_q, p);
    }
}
