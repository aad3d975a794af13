// b200_bfv.cu — CUDA kernels (sm_90a), device context and the layer-1 C ABI (include/b200_bfv.h).
//
// One process drives one GPU.  All work is enqueued on the caller's stream; temporaries come from the
// context-private stream-ordered pool (cudaMallocFromPoolAsync), so back-to-back calls never synchronise with the host.
// There is deliberately no CPU execution path in this library: if CUDA is unavailable every entry point
// returns B200_E_CUDA.
#include "../../include/b200_bfv.h"
#include "bfv_body.cuh"
#include "host_ctx.h"
#include "ntt_body.cuh"
#include "ntt_fp_body.cuh"
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#ifdef B200_EMU_HEADER
// Test-only build (tests/emu): the same sources compiled by g++ against a sequential CPU stand-in for
// the CUDA runtime, used by the CPU test-suite to check index math and orchestration without a GPU.
// The product library is never built this way and the package loader refuses to load such a build.
#include B200_EMU_HEADER
#else
#include <cuda_runtime.h>
#include <map>
#include <string>
#include <vector>
// Developer trace (B200_TRACE=1): CUDA events around every launch, summed per kernel name and printed by
// b200_trace_dump().  Off by default: the launch macro then costs one predictable branch.
struct B200TraceRec
{
    const char *name;
    cudaEvent_t e0, e1;
};
static int g_trace_on = -1;
static std::vector<B200TraceRec> g_trace;
static const char *g_trace_name = nullptr; // optional label for the next launch (function-pointer launches)
static inline bool trace_on()
{
    if (g_trace_on < 0)
        g_trace_on = getenv("B200_TRACE") ? 1 : 0;
    return g_trace_on == 1;
}
#define B200_LAUNCH(kernel, grid, block, smem, stream, ...)                                                            \
    do                                                                                                                 \
    {                                                                                                                  \
        if (trace_on())                                                                                                \
        {                                                                                                              \
            B200TraceRec r_{ g_trace_name ? g_trace_name : #kernel, nullptr, nullptr };                                \
            g_trace_name = nullptr;                                                                                    \
            cudaEventCreate(&r_.e0);                                                                                   \
            cudaEventCreate(&r_.e1);                                                                                   \
            cudaEventRecord(r_.e0, stream);                                                                            \
            kernel<<<grid, block, smem, stream>>>(__VA_ARGS__);                                                        \
            cudaEventRecord(r_.e1, stream);                                                                            \
            g_trace.push_back(r_);                                                                                     \
        }                                                                                                              \
        else                                                                                                           \
            kernel<<<grid, block, smem, stream>>>(__VA_ARGS__);                                                        \
    } while (0)
#endif
#include <condition_variable>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <sched.h>
#include <string>
#include <thread>
#include <vector>

using b200::BfvHostContext;
using b200::LevelHost;

static thread_local std::string g_err;
static int fail(int code, const std::string &msg)
{
    g_err = msg;
    return code;
}
#define CU_TRY(expr)                                                                                                   \
    do                                                                                                                 \
    {                                                                                                                  \
        cudaError_t _e = (expr);                                                                                       \
        if (_e != cudaSuccess)                                                                                         \
            return fail(B200_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));                              \
    } while (0)

// ---------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------
// MB = CTAs per SM the register allocation is sized for (the 64 KiB + pad of shared memory allow 3 at n = 8192; without a
// bound ptxas took 192 registers and a single 8-warp CTA ran per SM)
template <bool FWD, int NT, int MB = (NT <= 256 ? 3 : 1)>
__global__ void __launch_bounds__(NT, MB) ntt_kernel(const NttJob job)
{
#ifdef B200_EMU_HEADER
    u64 *ntt_sm = (u64 *)emu_shared;
#else
    extern __shared__ u64 ntt_sm[];
#endif
    const long long block = (long long)blockIdx.x;
    const long long item = block / job.slots;
    const int slot = (int)(block - item * job.slots);
#ifdef B200_EMU_HEADER
    // the emulation build has no statically scheduled FP64 kernel: FP64-capable primes take the generic FP64 body here, so
    // that the CPU-side tests cover its arithmetic
    const int pidx = job.slot_prime[slot];
    if (job.fprimes[pidx].enabled)
    {
        const u64 *src = ntt_src_ptr(job, item, slot);
        u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
        ntt_fp_block_body<FWD>(job, job.fprimes[pidx], job.primes[pidx], src, dst, reinterpret_cast<double *>(ntt_sm),
                               (int)threadIdx.x, (int)blockDim.x);
        return;
    }
#endif
    // integer Harvey / Shoup transform: valid for every prime up to 61 bits (jobs whose slots are all FP64-capable are
    // launched on ntt_fp_kernel instead; keeping the FP64 body out of this kernel saves ~60 registers)
    (void)item;
    (void)slot;
    ntt_block_body<FWD>(job, block, ntt_sm, (int)threadIdx.x, (int)blockDim.x);
}

// The FP64 statically scheduled kernels (ntt_fp_kernel<LOGN, FWD, NT, VAR>) live in their own translation unit,
// ntt_fp_kernels.cu; this file only fetches the function pointer of the instantiation it wants to launch.
#ifndef B200_EMU_HEADER
#include "ntt_fp_kernels.h"
#include "ksmac_tma.h"
#include "mul_cluster.h"
#endif

#define GLOBAL_IDX() ((long long)blockIdx.x * blockDim.x + threadIdx.x)

template <bool FWD>
__global__ void ntt_outer_kernel(const NttJob job, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    if (job.split == 2)
    {
        const int q4 = 1 << (job.logn - 2);
        ntt_outer_quad<FWD>(job, idx / q4, (int)(idx % q4));
        return;
    }
    const int halfn = 1 << (job.logn - 1);
    ntt_outer_pair<FWD>(job, idx / halfn, (int)(idx % halfn));
}

template <int K>
__global__ void lift_kernel(const LiftIntC<K> L, const u64 *a, int sa, const u64 *b, int sb, u64 *ext, long long n,
                            long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int P = sa + sb;
    const long long c = idx % n;
    const long long t = idx / n;
    const int p = (int)(t % P);
    const long long item = t / P;
    const int R = K + L.nBsk;
    const u64 *src = p < sa ? a + (item * sa + p) * K * n : b + (item * sb + (p - sa)) * K * n;
    u64 *dst = ext + ((item * P + p) * R + K) * n;
    lift_coeff<K>(L, src, dst, n, c); // integer path; the FP64 path is lift_kernel_v2
}

// rows: residue rows r in [0,R): r<K -> q[r], else bsk[r-K]
__global__ void tensor_kernel(const LevelDev L, const u64 *ext, int sa, int sb, u64 *D, long long n, long long total,
                              int square)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int R = L.k + L.nBsk;
    const long long c = idx % n;
    const long long t = idx / n;
    const int r = (int)(t % R);
    const long long item = t / R;
    const PrimeDev P = ld_prime(r < L.k ? &L.q[r] : &L.bsk[r - L.k]);
    const int Pn = square ? sa : sa + sb;
    const int Dn = square ? 3 : sa + sb - 1;
    const u64 *A = ext + ((item * Pn) * R + r) * n;
    u64 *Dp = D + ((item * Dn) * R + r) * n;
    if (!square && (sa > 4 || sb > 4))
    {
        tensor_coeff_general(P, A, R * n, sa, A + (long long)sa * R * n, R * n, sb, Dp, R * n, c);
        return;
    }
    if (L.fp)
    {
        const double *pd = r < L.k ? &L.dq[2 * r] : &L.dbsk[2 * (r - L.k)];
        const double p = __ldg(pd), pinv = __ldg(pd + 1);
        if (square)
            square_coeff_fp(p, pinv, A, R * n, Dp, R * n, c);
        else
            tensor_coeff_fp(p, pinv, A, R * n, sa, A + (long long)sa * R * n, R * n, sb, Dp, R * n, c);
        return;
    }
    if (square)
        square_coeff(P, A, R * n, Dp, R * n, c);
    else
        tensor_coeff(P, A, R * n, sa, A + (long long)sa * R * n, R * n, sb, Dp, R * n, c);
}

template <int K>
__global__ void scale_kernel(const ScaleIntC<K> L, const u64 *D, int Dn, u64 *dst0, int split, u64 *dst1, long long n,
                             long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int R = K + L.nBsk;
    const long long c = idx % n;
    const long long t = idx / n;
    const int m = (int)(t % Dn);
    const long long item = t / Dn;
    const u64 *src = D + ((item * Dn + m) * R) * n;
    u64 *dst = m < split ? dst0 + ((item * split + m) * K) * n : dst1 + ((item * (Dn - split) + (m - split)) * K) * n;
    scale_coeff<K>(L, src, dst, n, c); // integer path; the FP64 path is scale_kernel_v2
}

template <int K>
__global__ void ksmac_kernel(const PrimeDev *primes, const NttPrimeFp *fprimes, int use_fp, int special_idx, int key_rows,
                             const u64 *ks1, const u64 *key, u64 *ks2, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx % n;
    const long long t = idx / n;
    const int I = (int)(t % (K + 1));
    const long long item = t / (K + 1);
    const int prime_idx = I < K ? I : special_idx;
    const int key_res = I < K ? I : key_rows - 1;
    const PrimeDev P = ld_prime(&primes[prime_idx]);
    const u64 *ops = ks1 + ((item * (K + 1) + I) * K) * n;
    const u64 *kp = key + (long long)key_res * n;
    u64 *o0 = ks2 + ((item * 2 + 0) * (K + 1) + I) * n;
    u64 *o1 = ks2 + ((item * 2 + 1) * (K + 1) + I) * n;
    if (use_fp)
    {
        const double p = __ldg(&fprimes[prime_idx].p), pinv = __ldg(&fprimes[prime_idx].pinv);
        ksmac_coeff_fp<K>(p, pinv, ops, n, kp, 2LL * key_rows * n, (long long)key_rows * n, o0, o1, c);
        return;
    }
    ksmac_coeff<K>(P, ops, n, kp, 2LL * key_rows * n, (long long)key_rows * n, o0, o1, c);
}

// ---- FP64 element-wise kernels, two adjacent coefficients per thread (128-bit global accesses) ----
#ifdef B200_EMU_HEADER
struct b200_u64x2
{
    u64 x, y;
};
static inline b200_u64x2 ldg2(const u64 *p) { return b200_u64x2{ p[0], p[1] }; }
static inline void stg2(u64 *p, u64 a, u64 b)
{
    p[0] = a;
    p[1] = b;
}
#else
typedef ulonglong2 b200_u64x2;
__device__ __forceinline__ ulonglong2 ldg2(const u64 *p) { return __ldg(reinterpret_cast<const b200_u64x2 *>(p)); }
__device__ __forceinline__ void stg2(u64 *p, u64 a, u64 b) { *reinterpret_cast<ulonglong2 *>(p) = make_ulonglong2(a, b); }
#endif

template <int K>
__global__ void lift_kernel_v2(const LiftFpC<K> L, const u64 *a, int sa, const u64 *b, int sb, u64 *ext, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int P = sa + sb;
    const long long hn = n >> 1;
    const long long c = (idx % hn) * 2;
    const long long t = idx / hn;
    const int p = (int)(t % P);
    const long long item = t / P;
    const int R = K + L.nBsk;
    const u64 *src = p < sa ? a + (item * sa + p) * K * n : b + (item * sb + (p - sa)) * K * n;
    u64 *dst = ext + ((item * P + p) * R + K) * n;
    u64 xs[2][K], zs[2][K + 2];
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const b200_u64x2 v = ldg2(src + i * n + c);
        xs[0][i] = v.x;
        xs[1][i] = v.y;
    }
    lift_coeff_fp<K>(L, xs[0], zs[0], 1, 0);
    lift_coeff_fp<K>(L, xs[1], zs[1], 1, 0);
#pragma unroll
    for (int j = 0; j < K + 2; j++)
        if (j < L.nBsk)
            stg2(dst + j * n + c, zs[0][j], zs[1][j]);
}

__global__ void tensor_kernel_v2(const LevelDev L, const u64 *ext, u64 *D, long long n, long long total, int square)
{
    // size-2 x size-2 (or square of size 2) only: D0, D1, D2
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int R = L.k + L.nBsk;
    const long long hn = n >> 1;
    const long long c = (idx % hn) * 2;
    const long long t = idx / hn;
    const int r = (int)(t % R);
    const long long item = t / R;
    const double *pd = r < L.k ? &L.dq[2 * r] : &L.dbsk[2 * (r - L.k)];
    const double p = __ldg(pd), pinv = __ldg(pd + 1);
    const int Pn = square ? 2 : 4;
    const u64 *A = ext + ((item * Pn) * R + r) * n + c;
    u64 *Dp = D + ((item * 3) * R + r) * n + c;
    const long long ps = (long long)R * n;
    const b200_u64x2 a0 = ldg2(A), a1 = ldg2(A + ps);
    u64 in[2][4], out[2][3];
    in[0][0] = a0.x; in[1][0] = a0.y; in[0][1] = a1.x; in[1][1] = a1.y;
    if (!square)
    {
        const b200_u64x2 b0 = ldg2(A + 2 * ps), b1 = ldg2(A + 3 * ps);
        in[0][2] = b0.x; in[1][2] = b0.y; in[0][3] = b1.x; in[1][3] = b1.y;
    }
#pragma unroll
    for (int u = 0; u < 2; u++)
    {
        if (square)
            square_coeff_fp(p, pinv, in[u], 1, out[u], 1, 0);
        else
            tensor_coeff_fp(p, pinv, in[u], 1, 2, in[u] + 2, 1, 2, out[u], 1, 0);
    }
#pragma unroll
    for (int m = 0; m < 3; m++)
        stg2(Dp + m * ps, out[0][m], out[1][m]);
}

template <int K>
__global__ void scale_kernel_v2(const ScaleFpC<K> L, const u64 *D, int Dn, u64 *dst0, int split, u64 *dst1, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int R = K + L.nBsk;
    const long long hn = n >> 1;
    const long long c = (idx % hn) * 2;
    const long long t = idx / hn;
    const int m = (int)(t % Dn);
    const long long item = t / Dn;
    const u64 *src = D + ((item * Dn + m) * R) * n + c;
    u64 *dst = (m < split ? dst0 + ((item * split + m) * K) * n : dst1 + ((item * (Dn - split) + (m - split)) * K) * n) + c;
    u64 in[2][2 * K + 2], out[2][K];
#pragma unroll
    for (int i = 0; i < 2 * K + 2; i++)
        if (i < R)
        {
            const b200_u64x2 v = ldg2(src + i * n);
            in[0][i] = v.x;
            in[1][i] = v.y;
        }
    scale_coeff_fp<K>(L, in[0], out[0], 1, 0);
    scale_coeff_fp<K>(L, in[1], out[1], 1, 0);
#pragma unroll
    for (int i = 0; i < K; i++)
        stg2(dst + i * n, out[0][i], out[1][i]);
}

template <int K>
__global__ void ksmac_kernel_v2(const NttPrimeFp *fprimes, int special_idx, int key_rows, const u64 *ks1, const u64 *key, u64 *ks2,
                                long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long hn = n >> 1;
    const long long c = (idx % hn) * 2;
    const long long t = idx / hn;
    const int I = (int)(t % (K + 1));
    const long long item = t / (K + 1);
    const int prime_idx = I < K ? I : special_idx;
    const int key_res = I < K ? I : key_rows - 1;
    const double p = __ldg(&fprimes[prime_idx].p), pinv = __ldg(&fprimes[prime_idx].pinv);
    const u64 *ops = ks1 + ((item * (K + 1) + I) * K) * n + c;
    const u64 *kp = key + (long long)key_res * n + c;
    double acc[2][2] = { { 0.0, 0.0 }, { 0.0, 0.0 } };
#pragma unroll
    for (int J = 0; J < K; J++)
    {
        const b200_u64x2 x = ldg2(ops + J * n);
        const b200_u64x2 k0 = ldg2(kp + J * 2LL * key_rows * n), k1 = ldg2(kp + J * 2LL * key_rows * n + (long long)key_rows * n);
        const double x0 = fp_from_u64(x.x), x1 = fp_from_u64(x.y);
        acc[0][0] = B200_DADD(acc[0][0], fp_mulmod2(x0, fp_from_u64(k0.x), p, pinv));
        acc[0][1] = B200_DADD(acc[0][1], fp_mulmod2(x0, fp_from_u64(k1.x), p, pinv));
        acc[1][0] = B200_DADD(acc[1][0], fp_mulmod2(x1, fp_from_u64(k0.y), p, pinv));
        acc[1][1] = B200_DADD(acc[1][1], fp_mulmod2(x1, fp_from_u64(k1.y), p, pinv));
    }
    u64 *o0 = ks2 + ((item * 2 + 0) * (K + 1) + I) * n + c;
    u64 *o1 = ks2 + ((item * 2 + 1) * (K + 1) + I) * n + c;
    stg2(o0, fp_to_canonical(acc[0][0], p, pinv), fp_to_canonical(acc[1][0], p, pinv));
    stg2(o1, fp_to_canonical(acc[0][1], p, pinv), fp_to_canonical(acc[1][1], p, pinv));
}

template <int K>
__global__ void ksmoddown_kernel(const PrimeDev *primes, int special_idx, const u64 *inv_qsp, const u64 *ks2,
                                 const u64 *base0, long long base0_stride, const u64 *base1, long long base1_stride,
                                 u64 *dst, long long dst_item_stride, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx % n;
    const long long t = idx / n;
    const int comp = (int)(t & 1);
    const long long item = t >> 1;
    const PrimeDev SP = ld_prime(&primes[special_idx]);
    const u64 *acc = ks2 + ((item * 2 + comp) * (K + 1)) * n;
    const u64 *base = comp == 0 ? (base0 ? base0 + item * base0_stride : nullptr)
                                : (base1 ? base1 + item * base1_stride : nullptr);
    u64 *d = dst + item * dst_item_stride + (long long)comp * K * n;
    ksmoddown_coeff<K>(primes, SP, inv_qsp, acc, n, base, d, c);
}

// the same, two adjacent coefficients per thread: 128-bit loads / stores (the kernel is a pure stream of 2(k+1) + k rows in,
// 2k rows out per item)
template <int K>
__global__ void ksmoddown_kernel_v2(const PrimeDev *primes, int special_idx, const u64 *inv_qsp, const u64 *ks2,
                                    const u64 *base0, long long base0_stride, const u64 *base1, long long base1_stride,
                                    u64 *dst, long long dst_item_stride, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long hn = n >> 1;
    const long long c = (idx % hn) * 2;
    const long long t = idx / hn;
    const int comp = (int)(t & 1);
    const long long item = t >> 1;
    const PrimeDev SP = ld_prime(&primes[special_idx]);
    const u64 *acc = ks2 + ((item * 2 + comp) * (K + 1)) * n + c;
    const u64 *base = comp == 0 ? (base0 ? base0 + item * base0_stride : nullptr) : (base1 ? base1 + item * base1_stride : nullptr);
    u64 *d = dst + item * dst_item_stride + (long long)comp * K * n + c;
    const u64 half = SP.p >> 1;
    const b200_u64x2 sp = ldg2(acc + (long long)K * n);
    u64 s0 = sp.x + half, s1 = sp.y + half;
    s0 = s0 >= SP.p ? s0 - SP.p : s0;
    s1 = s1 >= SP.p ? s1 - SP.p : s1;
#pragma unroll
    for (int i = 0; i < K; i++)
    {
        const PrimeDev Q = ld_prime(&primes[i]);
        const u64 h = barrett64(half, Q.p, Q.r1);
        const u64 w = B200_LDG(&inv_qsp[2 * i]), wq = B200_LDG(&inv_qsp[2 * i + 1]);
        const b200_u64x2 a = ldg2(acc + (long long)i * n);
        u64 v0 = a.x + (Q.p - barrett64(s0, Q.p, Q.r1)) + h; // (a - r + h) mod q without underflow: < 3q
        u64 v1 = a.y + (Q.p - barrett64(s1, Q.p, Q.r1)) + h;
        v0 = shoup_mul(v0, w, wq, Q.p);
        v1 = shoup_mul(v1, w, wq, Q.p);
        if (base)
        {
            const b200_u64x2 b = ldg2(base + c + (long long)i * n);
            v0 = add_mod(v0, b.x, Q.p);
            v1 = add_mod(v1, b.y, Q.p);
        }
        stg2(d + (long long)i * n, v0, v1);
    }
}

template <int K>
__global__ void modswitch_kernel(const PrimeDev *primes, const u64 *inv_qlast, const u64 *src, u64 *dst, long long n,
                                 long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx % n;
    const long long poly = idx / n;
    modswitch_coeff<K>(primes, inv_qlast, src + poly * K * n, n, dst + poly * (K - 1) * n, c);
}

// out0 <- sigma(c0) (into dst poly 0), tmp <- sigma(c1)
__global__ void galois_kernel(const PrimeDev *primes, int k, const u64 *in2, u64 *out2, u64 *tmp, int logn, u32 g,
                              long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long n = 1LL << logn;
    const long long c = idx & (n - 1);
    const long long t = idx >> logn;
    const int r = (int)(t % k);
    const long long u = t / k;
    const int poly = (int)(u & 1);
    const long long item = u >> 1;
    const u64 p = __ldg(&primes[r].p);
    const u64 *src = in2 + ((item * 2 + poly) * k + r) * n;
    u64 *dst = poly == 0 ? out2 + ((item * 2) * k + r) * n : tmp + (item * k + r) * n;
    galois_coeff(p, src, dst, logn, g, c);
}

// mode 0: add, 1: sub, 2: negate (b unused)
__global__ void addsub_kernel(const PrimeDev *primes, int k, const u64 *a, const u64 *b, u64 *out, int logn, int mode,
                              long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const int r = (int)((idx >> logn) % k);
    const u64 p = __ldg(&primes[r].p);
    const u64 x = a[idx];
    u64 v;
    if (mode == 0)
        v = add_mod(x, b[idx], p);
    else if (mode == 1)
        v = sub_mod(x, b[idx], p);
    else
        v = neg_mod(x, p);
    out[idx] = v;
}

// small signed values (ternary secrets, clipped-normal noise: host samples, S/util/rlwe.cpp:23-67) -> their residues:
// out[poly][r][c] = v < 0 ? v + q_r : v
__global__ void expand_signed_kernel(const PrimeDev *primes, int k, const long long *vals, u64 *out, int logn, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx & ((1LL << logn) - 1);
    const long long row = idx >> logn;
    const int r = (int)(row % k);
    const long long poly = row / k;
    const long long v = vals[(poly << logn) + c];
    out[idx] = v < 0 ? __ldg(&primes[r].p) + (u64)v : (u64)v;
}

// dyadic out[item][poly][r][c] = x * y[(item % pb)][r][c] mod q_r   (x, y canonical)
__global__ void dyadic_plain_kernel(const PrimeDev *primes, int k, int size, const u64 *x, const u64 *y, long long pb,
                                    u64 *out, int logn, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long n = 1LL << logn;
    const long long c = idx & (n - 1);
    const long long t = idx >> logn;
    const int r = (int)(t % k);
    const long long u = t / k;
    const long long item = u / size;
    const PrimeDev P = ld_prime(&primes[r]);
    const u64 yv = y[((item % pb) * k + r) * n + c];
    u64 lo, hi;
    mul128(x[idx], yv, lo, hi);
    out[idx] = barrett128(lo, hi, P.p, P.r0, P.r1);
}

// mono[item] = 1 when plaintext `item` has exactly one nonzero coefficient (the monomial test of multiply_plain_normal,
// S/evaluator.cpp:1885).  One block per item: strided per-thread counts, summed in shared memory (blockDim a power of 2).
// The CPU emulation build runs kernels with dynamic shared memory as one thread per block, so only the CUDA build executes
// the tree reduction; the GPU parity tests (check_plain_operands, batches of monomial and dense items) cover it.
__global__ void plain_monomial_kernel(const u64 *plain, long long n, u32 *mono)
{
#ifdef B200_EMU_HEADER
    u64 *sm = (u64 *)emu_shared;
#else
    extern __shared__ u64 sm[];
#endif
    const u64 *p = plain + (long long)blockIdx.x * n;
    u64 cnt = 0;
    // four independent loads in flight per step; a thread that has seen two nonzero coefficients has decided that the item
    // is no monomial and stops, so a dense plaintext costs one step
    for (long long c = threadIdx.x; c < n && cnt < 2; c += 4LL * blockDim.x)
    {
        u64 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++)
        {
            const long long i = c + (long long)u * blockDim.x;
            v[u] = i < n ? p[i] : 0;
        }
#pragma unroll
        for (int u = 0; u < 4; u++)
            cnt += v[u] != 0;
    }
    sm[threadIdx.x] = cnt;
    B200_SYNC();
    for (int s = (int)blockDim.x >> 1; s > 0; s >>= 1)
    {
        if ((int)threadIdx.x < s)
            sm[threadIdx.x] += sm[threadIdx.x + s];
        B200_SYNC();
    }
    if (threadIdx.x == 0)
        mono[blockIdx.x] = sm[0] == 1;
}

// mono: per-item flags of plain_monomial_kernel, or null.  A monomial item is multiplied by its coefficient itself, the
// reference's monomial path (S/evaluator.cpp:1885-1933); the flags are only passed under the fast plain lift, where that
// differs from the general lift for a coefficient at or above the threshold (m instead of m + q_i - t).
__global__ void plain_lift_kernel(const LevelDev L, const u64 *plain, const u32 *mono, u64 *out, int logn, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long n = 1LL << logn;
    const long long c = idx & (n - 1);
    const long long t = idx >> logn;
    const int r = (int)(t % L.k);
    const long long item = t / L.k;
    const PrimeDev Q = ld_prime(&L.q[r]);
    const u64 m = plain[item * n + c];
    out[idx] = mono && mono[item] ? barrett64(m, Q.p, Q.r1) : plain_lift(L, Q, r, m);
}

// c0 +/- scaled plaintext; other polys copied.  sign: 0 add, 1 sub
__global__ void addsub_plain_kernel(const LevelDev L, int size, const u64 *a, const u64 *plain, long long pb, u64 *out,
                                    int logn, int sign, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long n = 1LL << logn;
    const long long c = idx & (n - 1);
    const long long t = idx >> logn;
    const int r = (int)(t % L.k);
    const long long u = t / L.k;
    const int poly = (int)(u % size);
    const long long item = u / size;
    u64 v = a[idx];
    if (poly == 0)
    {
        const PrimeDev Q = ld_prime(&L.q[r]);
        const u64 s = plain_scaled(L, Q, r, plain[(item % pb) * n + c]);
        v = sign ? sub_mod(v, s, Q.p) : add_mod(v, s, Q.p);
    }
    out[idx] = v;
}

// acc[item][r][c] = sum_{j>=1} X[item][j-1][r][c] * s[j-1][r][c] mod q_r
__global__ void dot_sk_kernel(const PrimeDev *primes, int k, int terms, const u64 *X, const u64 *sk, u64 *acc, int logn,
                              long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long n = 1LL << logn;
    const long long c = idx & (n - 1);
    const long long t = idx >> logn;
    const int r = (int)(t % k);
    const long long item = t / k;
    const PrimeDev P = ld_prime(&primes[r]);
    u64 lo = 0, hi = 0;
    for (int j = 0; j < terms; j++)
        mac128(X[((item * terms + j) * k + r) * n + c], sk[((long long)j * k + r) * n + c], lo, hi);
    acc[idx] = barrett128(lo, hi, P.p, P.r0, P.r1);
}

template <int K>
__global__ void decrypt_kernel(const LevelDev L, int size, const u64 *ct, u64 *phase /*in: dot, scratch*/, u64 *plain,
                               long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx % n;
    const long long item = idx / n;
    u64 *ph = phase + item * K * n;
    const u64 *c0 = ct + item * size * K * n;
#pragma unroll
    for (int i = 0; i < K; i++)
        ph[i * n + c] = add_mod(ph[i * n + c], c0[i * n + c], __ldg(&L.q[i].p));
    plain[item * n + c] = decrypt_coeff<K>(L, ph, n, c);
}

template <int K>
__global__ void phase_add_kernel(const PrimeDev *primes, int size, const u64 *ct, u64 *phase, long long n, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx >= total)
        return;
    const long long c = idx % n;
    const long long item = idx / n;
    u64 *ph = phase + item * K * n;
    const u64 *c0 = ct + item * size * K * n;
#pragma unroll
    for (int i = 0; i < K; i++)
        ph[i * n + c] = add_mod(ph[i * n + c], c0[i * n + c], __ldg(&primes[i].p));
}

// Decryptor::invariant_noise_internal (S/decryptor.cpp:424-485) on the device: per coefficient the phase c0 + dot, times t,
// CRT-composed to a multi-precision integer mod Q, centred (poly_infty_norm_coeffmod, S/util/polyarithsmallmod.cpp:292-322),
// and the maximum over the coefficients of a chunk.  One block = `chunk` consecutive coefficients of one item; the
// block maxima ([item][block][W + 1] little-endian words) are merged by the caller.
// consts: q[k] | c[k] | cq[k] | Q[W+1] | half[W+1] | punc[k][W]   with c_i = t (Q/q_i)^-1 mod q_i and its Shoup quotient
static const int NOISE_MAXW = 18;
B200_HD bool mp_ge(const u64 *a, const u64 *b, int words)
{
    for (int i = words; i-- > 0;)
        if (a[i] != b[i])
            return a[i] > b[i];
    return true;
}
__global__ void noise_norm_kernel(const u64 *consts, int k, int W, int size, const u64 *ct, const u64 *dot, long long n, int chunk,
                                  u64 *blockmax)
{
#ifdef B200_EMU_HEADER
    u64 *sm = (u64 *)emu_shared;
#else
    extern __shared__ u64 sm[];
#endif
    const int WW = W + 1;
    const u64 *q = consts, *cm = consts + k, *cq = consts + 2 * k, *Qw = consts + 3 * k, *half = Qw + WW, *punc = half + WW;
    const long long item = blockIdx.y;
    const u64 *c0 = ct + item * size * k * n;
    const u64 *dp = dot + item * k * n;
    u64 best[NOISE_MAXW], acc[NOISE_MAXW];
    for (int w = 0; w < WW; w++)
        best[w] = 0;
    for (int cc = (int)threadIdx.x; cc < chunk; cc += (int)blockDim.x)
    {
        const long long c = (long long)blockIdx.x * chunk + cc;
        if (c >= n)
            break;
        for (int w = 0; w < WW; w++)
            acc[w] = 0;
        for (int i = 0; i < k; i++)
        {
            const u64 qi = q[i];
            const u64 x = add_mod(dp[i * n + c], c0[i * n + c], qi);
            const u64 y = shoup_mul(x, cm[i], cq[i], qi);
            const u64 *pw = punc + (size_t)i * W;
            u64 carry = 0;
            for (int w = 0; w < W; w++)
            {
                u64 lo, hi;
                mul128(pw[w], y, lo, hi);
                lo += carry;
                hi += lo < carry;
                acc[w] += lo;
                hi += acc[w] < lo;
                carry = hi;
            }
            acc[W] += carry;
        }
        while (mp_ge(acc, Qw, WW))
        { // the sum is below k Q
            u64 borrow = 0;
            for (int w = 0; w < WW; w++)
            {
                const u64 b = Qw[w] + borrow;
                const u64 nb = (b < borrow) || (acc[w] < b);
                acc[w] -= b;
                borrow = nb;
            }
        }
        if (mp_ge(acc, half, WW))
        { // centred magnitude Q - acc
            u64 borrow = 0;
            for (int w = 0; w < WW; w++)
            {
                const u64 b = acc[w] + borrow;
                const u64 nb = (b < borrow) || (Qw[w] < b);
                acc[w] = Qw[w] - b;
                borrow = nb;
            }
        }
        if (mp_ge(acc, best, WW))
            for (int w = 0; w < WW; w++)
                best[w] = acc[w];
    }
    for (int w = 0; w < WW; w++)
        sm[(size_t)threadIdx.x * WW + w] = best[w];
    B200_SYNC();
    for (int s = (int)blockDim.x >> 1; s > 0; s >>= 1)
    {
        if ((int)threadIdx.x < s && mp_ge(sm + (size_t)(threadIdx.x + s) * WW, sm + (size_t)threadIdx.x * WW, WW))
            for (int w = 0; w < WW; w++)
                sm[(size_t)threadIdx.x * WW + w] = sm[(size_t)(threadIdx.x + s) * WW + w];
        B200_SYNC();
    }
    if (threadIdx.x == 0)
        for (int w = 0; w < WW; w++)
            blockmax[(item * gridDim.x + blockIdx.x) * WW + w] = sm[w];
}

__global__ void transparent_kernel(const u64 *ct, long long item_words, long long skip_words, u32 *flags)
{
    const long long item = blockIdx.y;
    const u64 *p = ct + item * item_words + skip_words;
    const long long cnt = item_words - skip_words;
    bool nz = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x)
        nz |= p[i] != 0;
    if (__syncthreads_or(nz) && threadIdx.x == 0)
        flags[item] = 0;
}

__global__ void fill_u32_kernel(u32 *p, u32 v, long long total)
{
    const long long idx = GLOBAL_IDX();
    if (idx < total)
        p[idx] = v;
}

// ---------------------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------------------
struct JobDesc
{
    int slots = 0;
    bool all_fp = false; // every slot's prime takes the FP64 path
    int *d_prime = nullptr;
    long long *d_src = nullptr;
    long long *d_dst = nullptr;
};

// host copies of the FP64 BEHZ constants of one level ({w, w/p} pairs), from which the kernel-parameter structs are filled
struct LevelFpHost
{
    std::vector<double> dq, dbsk, lift_c, lift_mat, lift_qm, scale_c, scale_tq, scale_mat, sk_c, sk_mat_q, sk_mat_msk, prod_b_q,
        negprod_b_q;
    std::vector<u64> lift_mt;
    u64 neg_inv_q_mod_mt = 0;
    double inv_b_msk[2] = { 0, 0 };
    int k = 0, nB = 0, nBsk = 0;
};

struct b200_ctx
{
    unsigned long long *ntt_timeline = nullptr; // developer aid, see b200_ntt_timeline()
    std::vector<LevelFpHost> fp_levels; // indexed like `levels`; empty tables when the level is not on the FP64 path
    std::unique_ptr<BfvHostContext> host;
    int device = 0;
    int sm_count = 0;
    int mul_clusters = 0; // 4-CTA clusters of mul_cluster_kernel the device holds at once (0: no cluster kernel for this size)
    size_t n = 0;
    int logn = 0;
    std::vector<void *> allocations; // everything freed at destroy
    NttPrime *d_ntt_primes = nullptr;
    NttPrimeFp *d_fp_primes = nullptr;
    bool fp_enabled = false;
    std::vector<bool> prime_fp;  // per device prime: takes the FP64 path
    int plain_prime_idx = -1;    // index of the plain modulus in the device prime tables (-1: no batching)
    PrimeDev *d_primes = nullptr;       // [all primes] key primes first
    std::vector<LevelDev> levels;       // device pointers inside
    std::vector<const u64 *> d_inv_qlast; // per level
    const u64 *d_inv_qsp = nullptr;     // key level's inv_qlast: q_sp^-1 mod q_i
    int npass = 0;
    int pass_L[8];
    std::map<std::string, JobDesc> jobs;
    std::map<int, std::pair<u64 *, int>> noise_consts; // per level: device constants of noise_norm_kernel, words of Q
    std::mutex mu;
    std::atomic<uint64_t> launches{ 0 };
    cudaStream_t s_h2d = nullptr, s_comp = nullptr, s_d2h = nullptr;
    cudaStream_t s_alloc = nullptr; // b200_malloc / b200_free order their pool operations on this stream
    cudaMemPool_t mempool = nullptr; // private stream-ordered pool of this context
    std::mutex alloc_mu;
    // side streams for intra-call concurrency: sub-batches of one call run on different streams so that the
    // FP64-bound NTT kernels of one overlap the HBM-bound element-wise kernels of another
    static const int NSIDE = 4;
    cudaStream_t s_side[NSIDE] = { nullptr, nullptr, nullptr, nullptr };
    cudaEvent_t ev_fork = nullptr, ev_join[NSIDE] = { nullptr, nullptr, nullptr, nullptr };
    int mr_split = 1;
    // staging ring of the *_host entry points (allocated on first use, reused afterwards)
    static const int NBUF = 3;
    u64 *hp_a[NBUF] = { nullptr, nullptr, nullptr }, *hp_b[NBUF] = { nullptr, nullptr, nullptr }, *hp_o[NBUF] = { nullptr, nullptr, nullptr };
    cudaEvent_t hp_in[NBUF], hp_comp[NBUF], hp_out[NBUF];
    size_t hp_words = 0;
    std::mutex hp_mu;
    // packed (6 bytes per word) PCIe staging of the host-buffer entry points: pinned host buffers and device landing zones
    uint8_t *hst_a[NBUF] = { nullptr, nullptr, nullptr }, *hst_b[NBUF] = { nullptr, nullptr, nullptr }, *hst_o[NBUF] = { nullptr, nullptr, nullptr };
    u64 *dpk_a[NBUF] = { nullptr, nullptr, nullptr }, *dpk_b[NBUF] = { nullptr, nullptr, nullptr }, *dpk_o[NBUF] = { nullptr, nullptr, nullptr };
    size_t pk_words = 0;
    struct HostPool *pool = nullptr;
    int ntt_threads = 256;
    size_t ntt_smem = 0;
    int ntt_split = 0; // n > 16384: two-level transform, ntt_outer_kernel + 2^split sub-transforms of n >> split points
};

template <class T>
static int upload(b200_ctx *ctx, const std::vector<T> &v, T **out)
{
    void *d = nullptr;
    size_t bytes = std::max<size_t>(v.size() * sizeof(T), 8);
    CU_TRY(cudaMalloc(&d, bytes));
    ctx->allocations.push_back(d);
    if (!v.empty())
        CU_TRY(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    *out = (T *)d;
    return 0;
}
#define UP(vec, ptr)                                                                                                   \
    do                                                                                                                 \
    {                                                                                                                  \
        int _rc = upload(ctx, vec, ptr);                                                                               \
        if (_rc)                                                                                                       \
            return _rc;                                                                                                \
    } while (0)

static std::vector<u64> flat(const std::vector<b200::Shoup> &v)
{
    std::vector<u64> o;
    for (auto &s : v)
    {
        o.push_back(s.w);
        o.push_back(s.wq);
    }
    return o;
}
static PrimeDev prime_dev(const b200::Modulus &m)
{
    PrimeDev p;
    p.p = m.p;
    p.r0 = m.r0;
    p.r1 = m.r1;
    return p;
}

static int build_device(b200_ctx *ctx)
{
    BfvHostContext &H = *ctx->host;
    const size_t n = H.n;
    // twiddle tables + per-prime descriptors; the plain modulus (when it supports batching) is appended as an
    // extra NTT prime for BatchEncoder (S/batchencoder.cpp:50-149)
    std::vector<b200::NttPrimeHost *> allp;
    for (auto &P : H.primes)
        allp.push_back(&P);
    ctx->plain_prime_idx = -1;
    if (H.using_batching)
    {
        ctx->plain_prime_idx = (int)allp.size();
        allp.push_back(&H.plain_ntt);
    }
    std::vector<NttPrime> np(allp.size());
    std::vector<PrimeDev> pd(allp.size());
    for (size_t i = 0; i < allp.size(); i++)
    {
        auto &P = *allp[i];
        u64 *dfwd = nullptr, *dinv = nullptr;
        UP(P.fwd, &dfwd);
        UP(P.inv, &dinv);
        np[i].p = P.mod.p;
        np[i].ratio1 = P.mod.r1;
        np[i].inv_n = P.inv_n.w;
        np[i].inv_n_q = P.inv_n.wq;
        np[i].inv_n_w = P.inv_n_w.w;
        np[i].inv_n_w_q = P.inv_n_w.wq;
        np[i].fwd = dfwd;
        np[i].inv = dinv;
        pd[i] = prime_dev(P.mod);
    }
    UP(np, &ctx->d_ntt_primes);
    UP(pd, &ctx->d_primes);
    {
        // FP64 fast path descriptors + magnitude bookkeeping (see ntt_fp_body.cuh).  All intermediates must stay
        // below 2^51; a forward stage adds < p to the bound, an inverse stage doubles it.
        const bool no_fp = std::getenv("B200_NO_FP64_NTT") != nullptr || ctx->ntt_split;
        ctx->fp_enabled = !no_fp;
        std::vector<NttPrimeFp> fp(allp.size());
        ctx->prime_fp.assign(allp.size(), false);
        for (size_t i = 0; i < allp.size(); i++)
        {
            auto &P = *allp[i];
            memset(&fp[i], 0, sizeof(NttPrimeFp));
            if (!P.fp || no_fp)
                continue;
            double *dfwd = nullptr, *dinv = nullptr;
            UP(P.dfwd, &dfwd);
            UP(P.dinv, &dinv);
            const double p = (double)P.mod.p;
            fp[i].p = p;
            fp[i].pinv = 1.0 / p;
            fp[i].inv_n[0] = P.inv_n_d[0];
            fp[i].inv_n[1] = P.inv_n_d[1];
            fp[i].inv_n_w[0] = P.inv_n_w_d[0];
            fp[i].inv_n_w[1] = P.inv_n_w_d[1];
            fp[i].fwd = dfwd;
            fp[i].inv = dinv;
            fp[i].enabled = 1;
            ctx->prime_fp[i] = true;
            if (ctx->logn >= 4)
            { // transposed tables for the sub-stride-1 radix-16 pass (lanes read consecutive entries)
                const int n16 = (int)(n >> 4), lg = ctx->logn;
                std::vector<double> f16((size_t)15 * n16), i16((size_t)15 * n16);
                for (int g = 0; g < n16; g++)
                    for (int l = 0; l < 4; l++)
                    {
                        for (int grp = 0; grp < (1 << l); grp++)
                        { // forward: M = n/16 groups at the first stage of the pass
                            const size_t idx = ((size_t)n16 << l) + ((size_t)g << l) + grp;
                            const size_t slot = (size_t)((1 << l) - 1 + grp) * n16 + g;
                            f16[slot] = P.dfwd[idx];
                        }
                        for (int grp = 0; grp < (8 >> l); grp++)
                        { // inverse: stage l has m = n/2 >> l groups
                            const size_t idx = ((size_t)1 << (lg - 1 - l)) + ((size_t)g << (3 - l)) + grp;
                            const size_t slot = (size_t)(16 - (16 >> l) + grp) * n16 + g;
                            i16[slot] = P.dinv[idx];
                        }
                    }
                double *d16 = nullptr;
                UP(f16, &d16);
                fp[i].fwd16 = d16;
                UP(i16, &d16);
                fp[i].inv16 = d16;
            }
            // Magnitude bookkeeping.  Every stored value must stay an exactly representable integer (|x| <= 2^53), and a
            // modular product y*w - rint(fl(fl(y*w) * fl(1/p))) * p of an input |y| <= 2^53 has magnitude at most
            // p * (1/2 + 3 * 2^-53 * |y|)  (three roundings of relative size 2^-53 in the quotient, one rint), computed
            // exactly (ntt_fp_body.cuh).  Forward butterfly: X +- T.  Inverse butterfly: X + Y and (X - Y) * w.
            const double LIMIT = 9007199254740992.0; // 2^53
            auto prod_bound = [&](double y) { return p * (0.5 + 3.0 * y / LIMIT) + 1.0; };
            const double RENORMED = 0.76 * p;       // |x - rint(x/p) p| after fp_renorm / fp_renorm_x
            auto fwd_pass = [&](double b, int L, bool &ok) {
                for (int s = 0; s < L; s++)
                {
                    b += prod_bound(b);
                    ok = ok && b <= LIMIT;
                }
                return b;
            };
            auto inv_pass = [&](double b, int L, bool &ok) {
                for (int s = 0; s < L; s++)
                {
                    ok = ok && 2.0 * b <= LIMIT;
                    b = std::max(2.0 * b, prod_bound(2.0 * b));
                }
                return b;
            };
            // the pass schedule that will run: the statically scheduled kernel's where it is used, else the generic one
            int sched_np = ctx->npass, sched_L[8];
            for (int pi = 0; pi < ctx->npass; pi++)
                sched_L[pi] = ctx->pass_L[pi];
#ifndef B200_EMU_HEADER
            if (ctx->logn >= 12 && ctx->logn <= 14 && !std::getenv("B200_NO_STATIC_NTT"))
                sched_np = ntt_static_schedule(ctx->logn, sched_L);
#endif
            double B = p; // canonical (or Barrett-reduced) input
            for (int pi = 0; pi < sched_np; pi++)
            {
                bool ok = true;
                double nb = fwd_pass(B, sched_L[pi], ok);
                if (!ok)
                {
                    fp[i].renorm_fwd |= 1u << pi;
                    ok = true;
                    nb = fwd_pass(RENORMED, sched_L[pi], ok);
                    if (!ok)
                        return fail(B200_E_LOGIC, "internal: FP64 NTT bound analysis failed (forward)");
                }
                B = nb;
            }
            B = p;
            int step = 0;
            for (int pi = sched_np - 1; pi >= 0; pi--, step++)
            {
                bool ok = true;
                double nb = inv_pass(B, sched_L[pi], ok);
                if (!ok)
                {
                    fp[i].renorm_inv |= 1u << step;
                    ok = true;
                    nb = inv_pass(RENORMED, sched_L[pi], ok);
                    if (!ok)
                        return fail(B200_E_LOGIC, "internal: FP64 NTT bound analysis failed (inverse)");
                }
                B = nb;
            }
        }
        UP(fp, &ctx->d_fp_primes);
    }
    for (auto &Lh : H.levels)
    {
        LevelDev L;
        memset(&L, 0, sizeof(L));
        L.k = Lh.k;
        L.nB = Lh.nB;
        L.nBsk = Lh.nBsk;
        L.q = ctx->d_primes; // q_idx is always the prefix 0..k-1
        std::vector<PrimeDev> bsk;
        for (int idx : Lh.bsk_idx)
            bsk.push_back(pd[idx]);
        PrimeDev *dbsk = nullptr;
        UP(bsk, &dbsk);
        L.bsk = dbsk;
        L.m_sk = H.primes[H.aux0].mod.p;
        L.t = H.t;
        L.t_mod = prime_dev(H.t_mod);
        L.gamma = pd[Lh.gamma_idx];
        u64 *d = nullptr;
#define UPF(field, vec)                                                                                                \
    do                                                                                                                 \
    {                                                                                                                  \
        std::vector<u64> _v = vec;                                                                                     \
        UP(_v, &d);                                                                                                    \
        L.field = d;                                                                                                   \
    } while (0)
        UPF(lift_c, flat(Lh.lift_c));
        UPF(lift_mat, Lh.lift_mat);
        UPF(lift_mt, Lh.lift_mt);
        UPF(lift_qm, Lh.lift_qm);
        L.neg_inv_q_mod_mt = Lh.neg_inv_q_mod_mt;
        UPF(scale_c, flat(Lh.scale_c));
        UPF(scale_tq, Lh.scale_tq);
        UPF(scale_mat, Lh.scale_mat);
        UPF(sk_c, flat(Lh.sk_c));
        UPF(sk_mat_q, Lh.sk_mat_q);
        UPF(sk_mat_msk, Lh.sk_mat_msk);
        UPF(sk_prod_b_q, Lh.sk_prod_b_q);
        L.sk_inv_b_msk = Lh.sk_inv_b_msk;
        UPF(inv_qlast, flat(Lh.inv_qlast));
        UPF(delta, Lh.delta);
        UPF(plain_inc, Lh.plain_upper_half_inc);
        L.q_mod_t = Lh.q_mod_t;
        L.plain_thr = Lh.plain_upper_half_threshold;
        L.fast_plain_lift = Lh.fast_plain_lift ? 1 : 0;
        LevelFpHost fp_level;
        {
            bool lfp = ctx->fp_enabled && H.aux_bits <= b200::FP_PRIME_BITS;
            for (int idx : Lh.q_idx)
                lfp = lfp && H.primes[idx].fp;
            for (int idx : Lh.bsk_idx)
                lfp = lfp && H.primes[idx].fp;
            L.fp = lfp ? 1 : 0;
            if (lfp)
            {
                std::vector<double> qd, bd;
                std::vector<u64> qv, bv;
                for (int idx : Lh.q_idx)
                    qv.push_back(H.primes[idx].mod.p);
                for (int idx : Lh.bsk_idx)
                    bv.push_back(H.primes[idx].mod.p);
                auto primes_d = [](const std::vector<u64> &v) {
                    std::vector<double> o;
                    for (u64 p : v)
                    {
                        o.push_back((double)p);
                        o.push_back(1.0 / (double)p);
                    }
                    return o;
                };
                // {w, w/p} with p = target[row] (rows of `cols` entries)
                auto pairs = [](const std::vector<u64> &w, const std::vector<u64> &target, int cols) {
                    std::vector<double> o;
                    for (size_t i = 0; i < w.size(); i++)
                    {
                        const double p = (double)target[i / (size_t)cols];
                        o.push_back((double)w[i]);
                        o.push_back((double)w[i] / p);
                    }
                    return o;
                };
                auto shoup_w = [](const std::vector<b200::Shoup> &v) {
                    std::vector<u64> o;
                    for (auto &s : v)
                        o.push_back(s.w);
                    return o;
                };
                double *dd = nullptr;
#define UPD(field, vec)                                                                                                \
    do                                                                                                                 \
    {                                                                                                                  \
        std::vector<double> _v = vec;                                                                                  \
        UP(_v, &dd);                                                                                                   \
        L.field = dd;                                                                                                  \
    } while (0)
                const int k = Lh.k, nB = Lh.nB;
                UPD(dq, primes_d(qv));
                UPD(dbsk, primes_d(bv));
                LevelFpHost F;
                F.k = k;
                F.nB = nB;
                F.nBsk = Lh.nBsk;
                F.dq = primes_d(qv);
                F.dbsk = primes_d(bv);
                F.lift_c = pairs(shoup_w(Lh.lift_c), qv, 1);
                F.lift_mat = pairs(Lh.lift_mat, bv, k);
                F.lift_qm = pairs(Lh.lift_qm, bv, 1);
                F.lift_mt = Lh.lift_mt;
                F.neg_inv_q_mod_mt = Lh.neg_inv_q_mod_mt;
                F.scale_c = pairs(shoup_w(Lh.scale_c), qv, 1);
                F.scale_tq = pairs(Lh.scale_tq, bv, 1);
                F.scale_mat = pairs(Lh.scale_mat, bv, k);
                F.sk_c = pairs(shoup_w(Lh.sk_c), bv, 1);
                F.sk_mat_q = pairs(Lh.sk_mat_q, qv, nB);
                std::vector<u64> msk_t(1, bv[nB]);
                F.sk_mat_msk = pairs(Lh.sk_mat_msk, msk_t, nB > 0 ? nB : 1);
                F.prod_b_q = pairs(Lh.sk_prod_b_q, qv, 1);
                std::vector<u64> negpb;
                for (int i = 0; i < k; i++)
                    negpb.push_back((qv[i] - Lh.sk_prod_b_q[i]) % qv[i]);
                F.negprod_b_q = pairs(negpb, qv, 1);
                F.inv_b_msk[0] = (double)Lh.sk_inv_b_msk;
                F.inv_b_msk[1] = (double)Lh.sk_inv_b_msk / (double)bv[nB];
                fp_level = F;
#undef UPD
            }
        }
        UPF(dec_c, flat(Lh.dec_c));
        UPF(dec_mat_t, Lh.dec_mat_t);
        UPF(dec_mat_g, Lh.dec_mat_g);
        L.inv_gamma_mod_t = Lh.inv_gamma_mod_t;
#undef UPF
        ctx->levels.push_back(L);
        ctx->fp_levels.push_back(fp_level);
    }
    ctx->d_inv_qsp = ctx->levels[0].inv_qlast;
    (void)n;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// launch helpers
// ---------------------------------------------------------------------------------------------------------
struct Scratch
{
    cudaStream_t s;
    cudaMemPool_t pool;
    std::vector<void *> ptrs;
    Scratch(b200_ctx *ctx, cudaStream_t st) : s(st), pool(ctx->mempool) {}
    int get(size_t words, u64 **out)
    {
        void *p = nullptr;
        cudaError_t e = cudaMallocFromPoolAsync(&p, std::max<size_t>(words, 1) * sizeof(u64), pool, s);
        if (e != cudaSuccess)
            return fail(B200_E_NOMEM, std::string("cudaMallocAsync: ") + cudaGetErrorString(e));
        ptrs.push_back(p);
        *out = (u64 *)p;
        return 0;
    }
    ~Scratch()
    {
        for (void *p : ptrs)
            cudaFreeAsync(p, s);
    }
};

static inline unsigned blocks_for(long long total, int bs) { return (unsigned)((total + bs - 1) / bs); }

static int get_job(b200_ctx *ctx, const std::string &key, const std::vector<int> &prime, const std::vector<long long> &src,
                   const std::vector<long long> &dst, JobDesc *out)
{
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->jobs.find(key);
    if (it != ctx->jobs.end())
    {
        *out = it->second;
        return 0;
    }
    JobDesc j;
    j.slots = (int)prime.size();
    j.all_fp = ctx->fp_enabled;
    for (int pi : prime)
        j.all_fp = j.all_fp && ctx->prime_fp[pi];
    UP(prime, &j.d_prime);
    UP(src, &j.d_src);
    UP(dst, &j.d_dst);
    ctx->jobs[key] = j;
    *out = j;
    return 0;
}

struct TensorArgs
{
    int mode = 0, sa = 0, sb = 0, rows = 0;
    const u64 *src = nullptr;
};

#ifndef B200_EMU_HEADER
// FP64 NTT kernel variant (ntt_fp_body.cuh: NttFpStaticPass VAR); B200_NTT_VAR or b200_debug_ntt_variant() override the default
static std::atomic<int> g_ntt_stagger{ std::getenv("B200_NTT_STAGGER") ? atoi(std::getenv("B200_NTT_STAGGER")) : 0 };
static std::atomic<int> g_ntt_var{ std::getenv("B200_NTT_VAR") ? atoi(std::getenv("B200_NTT_VAR")) : B200_NTT_DEFAULT_VAR };
#endif
static bool static_fp_ok(b200_ctx *ctx, const JobDesc &jd)
{
#ifdef B200_EMU_HEADER
    (void)ctx;
    (void)jd;
    return false;
#else
    return jd.all_fp && ctx->logn >= 12 && ctx->logn <= 14 && !std::getenv("B200_NO_STATIC_NTT");
#endif
}

// alternative sources of the leading slots (NttJob::alt_*)
struct NttAlt
{
    int end[2] = { 0, 0 };
    const u64 *src[2] = { nullptr, nullptr };
    long long stride[2] = { 0, 0 };
};

template <bool FWD>
static int launch_ntt(b200_ctx *ctx, const JobDesc &jd, const u64 *src, long long src_stride, u64 *dst, long long dst_stride,
                      long long items, int reduce_input, cudaStream_t s, const TensorArgs *ta = nullptr, const NttAlt *alt = nullptr)
{
    if (items == 0 || jd.slots == 0)
        return 0;
    NttJob job;
    for (int i = 0; i < 2; i++)
    {
        job.alt_end[i] = alt ? alt->end[i] : 0;
        job.alt_src[i] = alt ? alt->src[i] : nullptr;
        job.alt_stride[i] = alt ? alt->stride[i] : 0;
    }
    job.logn = ctx->logn;
    job.slots = jd.slots;
    job.slot_prime = jd.d_prime;
    job.slot_src = jd.d_src;
    job.slot_dst = jd.d_dst;
    job.src_item_stride = src_stride;
    job.dst_item_stride = dst_stride;
    job.src = src;
    job.dst = dst;
    job.primes = ctx->d_ntt_primes;
    job.fprimes = ctx->d_fp_primes;
    job.reduce_input = reduce_input;
    job.items = items;
    static const int pf = std::getenv("B200_NTT_PREFETCH") ? atoi(std::getenv("B200_NTT_PREFETCH")) : 0;
    job.prefetch_dist = pf;
    job.timeline = ctx->ntt_timeline;
    static const int slot_major = std::getenv("B200_NTT_ITEM_MAJOR") ? 0 : 1;
    job.slot_major = slot_major;
#ifndef B200_EMU_HEADER
    job.stagger = g_ntt_stagger.load(std::memory_order_relaxed);
#else
    job.stagger = 0;
#endif
    job.sm_count = ctx->sm_count;
    job.tensor_mode = ta ? ta->mode : 0;
    job.t_sa = ta ? ta->sa : 0;
    job.t_sb = ta ? ta->sb : 0;
    job.t_rows = ta ? ta->rows : 0;
    job.tsrc = ta ? ta->src : nullptr;
    if (ta && ta->mode && !static_fp_ok(ctx, jd))
        return fail(B200_E_LOGIC, "internal: fused tensor source needs the static FP64 NTT kernel");
    job.split = ctx->ntt_split;
    job.npass = ctx->npass;
    for (int i = 0; i < 8; i++)
        job.pass_L[i] = ctx->pass_L[i];
    const long long blocks = items * jd.slots * (1LL << ctx->ntt_split);
    if (ctx->ntt_split)
    {
        // two-level transform: the stage over the whole polynomial runs in global memory, the halves in shared memory
        const long long pairs = items * jd.slots * (long long)(ctx->n >> ctx->ntt_split); // butterflies (split 1) / quads (2)
        void (*kin)(const NttJob) = ctx->ntt_threads == 512 ? ntt_kernel<FWD, 512> : ntt_kernel<FWD, 256>;
        if (FWD)
        {
            B200_LAUNCH(ntt_outer_kernel<true>, blocks_for(pairs, 256), 256, 0, s, job, pairs);
            NttJob inner = job; // sub-transforms run in place on the destination
            inner.alt_end[0] = inner.alt_end[1] = 0;
            inner.src = job.dst;
            inner.slot_src = job.slot_dst;
            inner.src_item_stride = job.dst_item_stride;
            inner.reduce_input = 0;
            B200_LAUNCH(kin, (unsigned)blocks, ctx->ntt_threads, ctx->ntt_smem, s, inner);
        }
        else
        {
            B200_LAUNCH(kin, (unsigned)blocks, ctx->ntt_threads, ctx->ntt_smem, s, job);
            B200_LAUNCH(ntt_outer_kernel<false>, blocks_for(pairs, 256), 256, 0, s, job, pairs);
        }
        ctx->launches += 2;
        CU_TRY(cudaGetLastError());
        return 0;
    }
    if (blocks > 0x7fffffffLL)
        return fail(B200_E_INVALID, "batch too large for one NTT launch");
#ifndef B200_EMU_HEADER
    if (static_fp_ok(ctx, jd))
    {
        // n = 8192: 256 threads x 3 CTAs/SM is the throughput configuration; a launch that cannot fill the SMs anyway (the
        // per-handle path: at most 36 polynomials) is latency-bound and finishes sooner with 512 threads per polynomial
        static const int nt_env = std::getenv("B200_NTT_NT") ? atoi(std::getenv("B200_NTT_NT")) : 0;
        int var_env = g_ntt_var.load(std::memory_order_relaxed);
        if (var_env < 0)
        { // automatic: what measured fastest per size and direction (tools/ntt_ablate.py).  2048 = warp(-group)-private
          // sub-transforms, +1 = first 512 twiddles in shared memory, +16 = streaming (persistent) kernel
            if (ctx->logn == 14)
                var_env = FWD ? 2049 : 2064;
            else if (ctx->logn == 13)
                var_env = FWD ? 2048 : 2049;
            else
                var_env = 2048;
        }
        const int nt13 = nt_env ? nt_env : (blocks <= 2LL * ctx->sm_count ? 512 : 256);
        const int nt = ctx->logn == 12 ? 256 : ctx->logn == 13 ? (nt13 == 256 ? 256 : 512) : 1024;
        int var = ta && ta->mode ? (var_env & 1) : var_env; // the fused-tensor copy-in exists in the plain variants only
        if ((var & 16) && nt == 512)
            var &= ~16; // the streaming variant exists for the throughput configuration; small launches stay latency-optimised
        b200_ntt_fp_fn sfn = b200_ntt_fp_kernel(ctx->logn, FWD, nt, var);
        if (!sfn)
        {
            var &= 1;
            sfn = b200_ntt_fp_kernel(ctx->logn, FWD, nt, var);
        }
        if (!sfn)
        {
            var = 0;
            sfn = b200_ntt_fp_kernel(ctx->logn, FWD, nt, 0);
        }
        if (!sfn)
            return fail(B200_E_LOGIC, "internal: no FP64 NTT kernel for this size");
        const size_t smem = ctx->ntt_smem + ((var & 1) ? B200_NTT_TWS_ENTRIES * sizeof(double) : 0);
        if (trace_on())
        {
            static char labels[2][128][40];
            const int sl = jd.slots < 128 ? jd.slots : 127;
            snprintf(labels[FWD ? 1 : 0][sl], sizeof(labels[0][0]), "ntt_fp_kernel<%s> rows/item=%d%s", FWD ? "fwd" : "inv", jd.slots,
                     job.tensor_mode ? " +tensor" : "");
            g_trace_name = labels[FWD ? 1 : 0][sl];
        }
        unsigned grid = (unsigned)blocks;
        if (var & 16)
        { // persistent: one CTA per resident slot, each walking its share of the polynomials
            static std::map<b200_ntt_fp_fn, int> occ;
            static std::mutex occ_mu;
            int per_sm;
            {
                std::lock_guard<std::mutex> lk(occ_mu);
                auto it = occ.find(sfn);
                if (it == occ.end())
                    it = occ.emplace(sfn, b200_ntt_fp_ctas_per_sm(sfn, nt, smem)).first;
                per_sm = it->second;
            }
            grid = (unsigned)std::min<long long>(blocks, (long long)per_sm * ctx->sm_count);
        }
        B200_LAUNCH(sfn, grid, nt, smem, s, job);
        ctx->launches++;
        CU_TRY(cudaGetLastError());
        return 0;
    }
#endif
    static const int mb = std::getenv("B200_NTT_INT_MB") ? atoi(std::getenv("B200_NTT_INT_MB")) : 3;
    void (*kfn)(const NttJob) = ctx->ntt_threads == 512   ? ntt_kernel<FWD, 512>
                                : ctx->ntt_threads == 256 ? (mb == 2 ? ntt_kernel<FWD, 256, 2> : mb == 1 ? ntt_kernel<FWD, 256, 1> : ntt_kernel<FWD, 256>)
                                                          : ntt_kernel<FWD, 64>;
    B200_LAUNCH(kfn, (unsigned)blocks, ctx->ntt_threads, ctx->ntt_smem, s, job);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

#define DISPATCH_K(kval, ...)                                                                                         \
    switch (kval)                                                                                                      \
    {                                                                                                                  \
    case 1: { constexpr int KK = 1; __VA_ARGS__; } break;                                                                     \
    case 2: { constexpr int KK = 2; __VA_ARGS__; } break;                                                                     \
    case 3: { constexpr int KK = 3; __VA_ARGS__; } break;                                                                     \
    case 4: { constexpr int KK = 4; __VA_ARGS__; } break;                                                                     \
    case 5: { constexpr int KK = 5; __VA_ARGS__; } break;                                                                     \
    case 6: { constexpr int KK = 6; __VA_ARGS__; } break;                                                                     \
    case 7: { constexpr int KK = 7; __VA_ARGS__; } break;                                                                     \
    case 8: { constexpr int KK = 8; __VA_ARGS__; } break;                                                                     \
    case 9: { constexpr int KK = 9; __VA_ARGS__; } break;                                                                     \
    case 10: { constexpr int KK = 10; __VA_ARGS__; } break;                                                                   \
    case 11: { constexpr int KK = 11; __VA_ARGS__; } break;                                                                   \
    case 12: { constexpr int KK = 12; __VA_ARGS__; } break;                                                                   \
    case 13: { constexpr int KK = 13; __VA_ARGS__; } break;                                                                   \
    case 14: { constexpr int KK = 14; __VA_ARGS__; } break;                                                                   \
    case 15: { constexpr int KK = 15; __VA_ARGS__; } break;                                                                   \
    case 16: { constexpr int KK = 16; __VA_ARGS__; } break;                                                                   \
    default: return fail(B200_E_INVALID, "unsupported residue count (max 16 data residues)");                          \
    }

template <int K>
static LiftIntC<K> make_lift_intc(const b200_ctx *ctx, int level)
{
    const auto &Lh = ctx->host->levels[level];
    LiftIntC<K> C;
    memset(&C, 0, sizeof(C));
    C.nBsk = Lh.nBsk;
    C.neg_inv_q_mod_mt = Lh.neg_inv_q_mod_mt;
    for (int i = 0; i < K; i++)
    {
        C.q[i] = ctx->host->primes[Lh.q_idx[i]].mod.p;
        C.c[2 * i] = Lh.lift_c[i].w;
        C.c[2 * i + 1] = Lh.lift_c[i].wq;
        C.mt[i] = Lh.lift_mt[i];
    }
    for (int j = 0; j < Lh.nBsk; j++)
    {
        const auto &M = ctx->host->primes[Lh.bsk_idx[j]].mod;
        C.bsk[j] = PrimeC{ M.p, M.r0, M.r1 };
        C.qm[j] = Lh.lift_qm[j];
        for (int i = 0; i < K; i++)
            C.mat[j * K + i] = Lh.lift_mat[(size_t)j * K + i];
    }
    return C;
}
template <int K>
static ScaleIntC<K> make_scale_intc(const b200_ctx *ctx, int level)
{
    const auto &Lh = ctx->host->levels[level];
    ScaleIntC<K> C;
    memset(&C, 0, sizeof(C));
    C.nB = Lh.nB;
    C.nBsk = Lh.nBsk;
    for (int i = 0; i < K; i++)
    {
        const auto &M = ctx->host->primes[Lh.q_idx[i]].mod;
        C.q[i] = PrimeC{ M.p, M.r0, M.r1 };
        C.c[2 * i] = Lh.scale_c[i].w;
        C.c[2 * i + 1] = Lh.scale_c[i].wq;
        C.sk_prod_b_q[i] = Lh.sk_prod_b_q[i];
        for (int b = 0; b < Lh.nB; b++)
            C.sk_mat_q[i * (K + 1) + b] = Lh.sk_mat_q[(size_t)i * Lh.nB + b];
    }
    for (int j = 0; j < Lh.nBsk; j++)
    {
        const auto &M = ctx->host->primes[Lh.bsk_idx[j]].mod;
        C.bsk[j] = PrimeC{ M.p, M.r0, M.r1 };
        C.tq[j] = Lh.scale_tq[j];
        for (int i = 0; i < K; i++)
            C.mat[j * K + i] = Lh.scale_mat[(size_t)j * K + i];
    }
    for (int b = 0; b < Lh.nB; b++)
    {
        C.sk_c[2 * b] = Lh.sk_c[b].w;
        C.sk_c[2 * b + 1] = Lh.sk_c[b].wq;
        C.sk_mat_msk[b] = Lh.sk_mat_msk[b];
    }
    C.sk_inv_b_msk = Lh.sk_inv_b_msk;
    return C;
}
template <int K>
static LiftFpC<K> make_lift_fpc(const b200_ctx *ctx, int level)
{
    const LevelFpHost &H = ctx->fp_levels[level];
    LiftFpC<K> C;
    memset(&C, 0, sizeof(C));
    C.nBsk = H.nBsk;
    C.neg_inv_q_mod_mt = H.neg_inv_q_mod_mt;
    for (int i = 0; i < K; i++)
        C.mt[i] = H.lift_mt[i];
    std::copy(H.dq.begin(), H.dq.end(), C.dq);
    std::copy(H.dbsk.begin(), H.dbsk.end(), C.dbsk);
    std::copy(H.lift_c.begin(), H.lift_c.end(), C.c);
    std::copy(H.lift_mat.begin(), H.lift_mat.end(), C.mat); // rows of K pairs, as in the struct
    std::copy(H.lift_qm.begin(), H.lift_qm.end(), C.qm);
    return C;
}
template <int K>
static ScaleFpC<K> make_scale_fpc(const b200_ctx *ctx, int level)
{
    const LevelFpHost &H = ctx->fp_levels[level];
    ScaleFpC<K> C;
    memset(&C, 0, sizeof(C));
    C.nB = H.nB;
    C.nBsk = H.nBsk;
    std::copy(H.dq.begin(), H.dq.end(), C.dq);
    std::copy(H.dbsk.begin(), H.dbsk.end(), C.dbsk);
    std::copy(H.scale_c.begin(), H.scale_c.end(), C.c);
    std::copy(H.scale_tq.begin(), H.scale_tq.end(), C.tq);
    std::copy(H.scale_mat.begin(), H.scale_mat.end(), C.mat);
    std::copy(H.sk_c.begin(), H.sk_c.end(), C.sk_c);
    for (int i = 0; i < K; i++) // host rows have nB columns, the struct K+1
        for (int b = 0; b < H.nB; b++)
        {
            C.sk_mat_q[2 * (i * (K + 1) + b)] = H.sk_mat_q[2 * (i * H.nB + b)];
            C.sk_mat_q[2 * (i * (K + 1) + b) + 1] = H.sk_mat_q[2 * (i * H.nB + b) + 1];
        }
    std::copy(H.sk_mat_msk.begin(), H.sk_mat_msk.end(), C.sk_mat_msk);
    std::copy(H.prod_b_q.begin(), H.prod_b_q.end(), C.prod_b_q);
    std::copy(H.negprod_b_q.begin(), H.negprod_b_q.end(), C.negprod_b_q);
    C.inv_b_msk[0] = H.inv_b_msk[0];
    C.inv_b_msk[1] = H.inv_b_msk[1];
    return C;
}

static const int EB = 256; // element-wise block size

static int check_level(b200_ctx *ctx, int level)
{
    if (!ctx)
        return fail(B200_E_NULL, "null context");
    if (level < 0 || level >= (int)ctx->levels.size())
        return fail(B200_E_INVALID, "level out of range");
    return 0;
}

// slots over a dense [items][slots][n] slab with per-slot prime
static int dense_job(b200_ctx *ctx, const std::string &key, const std::vector<int> &prime, JobDesc *jd)
{
    std::vector<long long> off(prime.size());
    for (size_t i = 0; i < prime.size(); i++)
        off[i] = (long long)i * (long long)ctx->n;
    return get_job(ctx, key, prime, off, off, jd);
}

static std::vector<int> row_primes(b200_ctx *ctx, int level, bool with_bsk)
{
    const LevelHost &Lh = ctx->host->levels[level];
    std::vector<int> r(Lh.q_idx);
    if (with_bsk)
        r.insert(r.end(), Lh.bsk_idx.begin(), Lh.bsk_idx.end());
    return r;
}

// ---- multiply core: writes polys [0,split) to dst0 and [split,Dn) to dst1 ----
static int multiply_core(b200_ctx *ctx, int level, const u64 *a, int sa, const u64 *b, int sb, bool square, u64 *dst0,
                         int split, u64 *dst1, long long batch, cudaStream_t s)
{
    const LevelDev &L = ctx->levels[level];
    const LevelHost &Lh = ctx->host->levels[level];
    const long long n = (long long)ctx->n;
    const int k = L.k, R = k + L.nBsk;
    const int P = square ? sa : sa + sb;
    const int Dn = square ? 3 : sa + sb - 1;
    Scratch scr(ctx, s);
    u64 *ext = nullptr, *D = nullptr;
    int rc;
    if ((rc = scr.get((size_t)batch * P * R * n, &ext)))
        return rc;
    if ((rc = scr.get((size_t)batch * Dn * R * n, &D)))
        return rc;
    bool clustered = false; // (3)-(5) ran as mul_cluster_kernel
    // (1)-(2) lift to Bsk
    {
        if (L.fp)
        {
            const long long total = batch * P * (n >> 1);
            DISPATCH_K(k, B200_LAUNCH(lift_kernel_v2<KK>, blocks_for(total, EB), EB, 0, s, make_lift_fpc<KK>(ctx, level), a, sa,
                                      square ? a : b, square ? 0 : sb, ext, n, total));
        }
        else
        {
            const long long total = batch * P * n;
            DISPATCH_K(k, B200_LAUNCH(lift_kernel<KK>, blocks_for(total, EB), EB, 0, s, make_lift_intc<KK>(ctx, level), a, sa,
                                      square ? a : b, square ? 0 : sb, ext, n, total));
        }
        ctx->launches++;
    }
#ifndef B200_EMU_HEADER
    // (3)-(5) in one kernel for a size-2 x size-2 product on the FP64 static path (mul_cluster.cu): the NTT-form operands and
    // products stay in the shared memory of a 4-CTA cluster.  Taken where the launch fills the GPU (the rule of the 256/512
    // thread switch in launch_ntt); B200_MUL_CLUSTER=0 selects the separate kernels below, B200_TENSOR_FUSION=1 their fused
    // inverse copy-in.
    static const bool want_cluster = !(std::getenv("B200_MUL_CLUSTER") && std::getenv("B200_MUL_CLUSTER")[0] == '0') &&
                                     !std::getenv("B200_TENSOR_FUSION");
    if (want_cluster && !square && sa == 2 && sb == 2 && L.fp && ctx->mul_clusters > 0 && ctx->logn <= 13 &&
        4LL * R * batch > 2LL * ctx->sm_count)
    {
        JobDesc jd;
        if ((rc = get_job(ctx, "mulcl:" + std::to_string(level), row_primes(ctx, level, true), {}, {}, &jd)))
            return rc;
        if (static_fp_ok(ctx, jd))
        {
            if (4LL * R * batch > 0x7fffffffLL)
                return fail(B200_E_INVALID, "batch too large for one multiply launch");
            NttJob job;
            memset(&job, 0, sizeof(job));
            job.logn = ctx->logn;
            job.slots = R;
            job.slot_prime = jd.d_prime;
            job.primes = ctx->d_ntt_primes;
            job.fprimes = ctx->d_fp_primes;
            job.items = batch;
            cudaEvent_t t0 = nullptr, t1 = nullptr;
            if (trace_on())
            {
                cudaEventCreate(&t0);
                cudaEventCreate(&t1);
                cudaEventRecord(t0, s);
            }
            const int crc = b200_mul_cluster(ctx->logn, job, a, b, ext, D, k, s);
            if (crc)
                return fail(B200_E_CUDA, std::string("mul_cluster_kernel: ") + cudaGetErrorString((cudaError_t)crc));
            if (t0)
            {
                cudaEventRecord(t1, s);
                g_trace.push_back(B200TraceRec{ "mul_cluster_kernel", t0, t1 });
            }
            ctx->launches++;
            clustered = true;
        }
    }
#endif
    // (3) forward NTTs in ONE launch: q rows straight from the inputs (alternative sources a, b), Bsk rows in place in ext
    if (!clustered)
    {
        std::vector<int> prime;
        std::vector<long long> so, dof;
        NttAlt alt;
        for (int which = 0; which < (square ? 1 : 2); which++)
        {
            const int sz = which == 0 ? sa : sb;
            const int p0 = which == 0 ? 0 : sa;
            for (int p = 0; p < sz; p++)
                for (int r = 0; r < k; r++)
                {
                    prime.push_back(Lh.q_idx[r]);
                    so.push_back(((long long)p * k + r) * n);
                    dof.push_back(((long long)(p0 + p) * R + r) * n);
                }
            alt.end[which] = (int)prime.size();
            alt.src[which] = which == 0 ? a : b;
            alt.stride[which] = (long long)sz * k * n;
        }
        if (square)
            alt.end[1] = alt.end[0];
        for (int p = 0; p < P; p++)
            for (int j = 0; j < L.nBsk; j++)
            {
                prime.push_back(Lh.bsk_idx[j]);
                so.push_back(((long long)p * R + k + j) * n);
                dof.push_back(((long long)p * R + k + j) * n);
            }
        JobDesc jd;
        std::string key = "mulfwd:" + std::to_string(level) + ":" + std::to_string(sa) + ":" + std::to_string(square ? 0 : sb);
        if ((rc = get_job(ctx, key, prime, so, dof, &jd)))
            return rc;
        if ((rc = launch_ntt<true>(ctx, jd, ext, (long long)P * R * n, ext, (long long)P * R * n, batch, 0, s, nullptr, &alt)))
            return rc;
    }
    // (4) tensor + (5) inverse NTTs.  Optionally (FP64 path) the dyadic products are formed inside the inverse
    // transform's coalesced copy-in (D never materialised in NTT form); by default a separate tensor kernel runs.
    if (!clustered)
    {
        std::vector<int> rows = row_primes(ctx, level, true), prime;
        for (int m = 0; m < Dn; m++)
            prime.insert(prime.end(), rows.begin(), rows.end());
        JobDesc jd;
        if ((rc = dense_job(ctx, "muld:" + std::to_string(level) + ":" + std::to_string(Dn), prime, &jd)))
            return rc;
        // measured on B200 (round 1): the fused variant is SLOWER (10.9 vs 8.9 ms per 1024 ops) — the extra strided
        // loads sit on the transform's latency-critical copy-in — so it stays opt-in (B200_TENSOR_FUSION=1)
        static const bool want_fuse = std::getenv("B200_TENSOR_FUSION") != nullptr;
        const bool fuse = want_fuse && L.fp && static_fp_ok(ctx, jd);
        TensorArgs ta;
        if (fuse)
        {
            ta.mode = square ? 2 : 1;
            ta.sa = sa;
            ta.sb = sb;
            ta.rows = R;
            ta.src = ext;
        }
        else
        {
            if (L.fp && (square || (sa == 2 && sb == 2)))
            {
                const long long total = batch * R * (n >> 1);
                B200_LAUNCH(tensor_kernel_v2, blocks_for(total, EB), EB, 0, s, L, ext, D, n, total, square ? 1 : 0);
            }
            else
            {
                const long long total = batch * R * n;
                B200_LAUNCH(tensor_kernel, blocks_for(total, EB), EB, 0, s, L, ext, sa, sb, D, n, total, square ? 1 : 0);
            }
            ctx->launches++;
        }
        if ((rc = launch_ntt<false>(ctx, jd, D, (long long)Dn * R * n, D, (long long)Dn * R * n, batch, 0, s, fuse ? &ta : nullptr)))
            return rc;
    }
    // (6)-(8) scale
    {
        if (L.fp)
        {
            const long long total = batch * Dn * (n >> 1);
            DISPATCH_K(k, B200_LAUNCH(scale_kernel_v2<KK>, blocks_for(total, EB), EB, 0, s, make_scale_fpc<KK>(ctx, level), D, Dn,
                                      dst0, split, dst1, n, total));
        }
        else
        {
            const long long total = batch * Dn * n;
            DISPATCH_K(k, B200_LAUNCH(scale_kernel<KK>, blocks_for(total, EB), EB, 0, s, make_scale_intc<KK>(ctx, level), D, Dn, dst0,
                                      split, dst1, n, total));
        }
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---- key switch core: target d (k rows per item, stride d_stride), key list; dst_c = base_c + moddown(acc_c) ----
static int keyswitch_core(b200_ctx *ctx, int level, const u64 *d, long long d_stride, const u64 *key, const u64 *base0,
                          long long base0_stride, const u64 *base1, long long base1_stride, u64 *dst,
                          long long dst_stride, long long batch, cudaStream_t s)
{
    if (!ctx->host->using_keyswitching || level < 1)
        return fail(B200_E_LOGIC, "keyswitching is not supported by the context");
    const LevelDev &L = ctx->levels[level];
    const LevelHost &Lh = ctx->host->levels[level];
    const long long n = (long long)ctx->n;
    const int k = L.k;
    const int Kkey = ctx->host->K;
    const int special = Kkey - 1;
    Scratch scr(ctx, s);
    u64 *ks1 = nullptr, *ks2 = nullptr;
    int rc;
    if ((rc = scr.get((size_t)batch * (k + 1) * k * n, &ks1)))
        return rc;
    if ((rc = scr.get((size_t)batch * 2 * (k + 1) * n, &ks2)))
        return rc;
    {
        std::vector<int> prime;
        std::vector<long long> so, dof;
        for (int I = 0; I <= k; I++)
            for (int J = 0; J < k; J++)
            {
                prime.push_back(I < k ? Lh.q_idx[I] : special);
                so.push_back((long long)J * n);
                dof.push_back(((long long)I * k + J) * n);
            }
        JobDesc jd;
        if ((rc = get_job(ctx, "ks1:" + std::to_string(level), prime, so, dof, &jd)))
            return rc;
        if ((rc = launch_ntt<true>(ctx, jd, d, d_stride, ks1, (long long)(k + 1) * k * n, batch, 1, s)))
            return rc;
    }
    {
        bool done = false;
#ifndef B200_EMU_HEADER
        // key tile resident in shared memory (one tiled TMA load per CTA), batch walked inside the CTA: the key is read from
        // HBM once per batch chunk instead of once per item (B200_KSMAC_TMA=0 selects the item-major kernels below)
        static const bool want_tma = !(std::getenv("B200_KSMAC_TMA") && std::getenv("B200_KSMAC_TMA")[0] == '0');
        if (want_tma && b200_ksmac_tma_supported(n, k))
        {
            if (trace_on())
                g_trace_name = "ksmac_tma_kernel";
            cudaEvent_t t0 = nullptr, t1 = nullptr;
            if (trace_on())
            {
                cudaEventCreate(&t0);
                cudaEventCreate(&t1);
                cudaEventRecord(t0, s);
            }
            const int rc2 = b200_ksmac_tma(k, L.fp ? 1 : 0, ctx->d_primes, ctx->d_fp_primes, special, Kkey, ks1, key, ks2, n, batch,
                                           ctx->sm_count, s);
            if (rc2 > 0)
                return fail(B200_E_CUDA, std::string("ksmac_tma_kernel: ") + cudaGetErrorString((cudaError_t)rc2));
            if (rc2 == 0)
            {
                done = true;
                if (t0)
                {
                    cudaEventRecord(t1, s);
                    g_trace.push_back(B200TraceRec{ "ksmac_tma_kernel", t0, t1 });
                    g_trace_name = nullptr;
                }
            }
        }
#endif
        if (done)
            ;
        else if (L.fp)
        {
            const long long total = batch * (k + 1) * (n >> 1);
            DISPATCH_K(k, B200_LAUNCH(ksmac_kernel_v2<KK>, blocks_for(total, EB), EB, 0, s, ctx->d_fp_primes, special, Kkey, ks1, key,
                                      ks2, n, total));
        }
        else
        {
            const long long total = batch * (k + 1) * n;
            DISPATCH_K(k, B200_LAUNCH(ksmac_kernel<KK>, blocks_for(total, EB), EB, 0, s, ctx->d_primes, ctx->d_fp_primes,
                                      (int)(L.fp != 0), special, Kkey, ks1, key, ks2, n, total));
        }
        ctx->launches++;
    }
    {
        std::vector<int> prime;
        for (int comp = 0; comp < 2; comp++)
            for (int I = 0; I <= k; I++)
                prime.push_back(I < k ? Lh.q_idx[I] : special);
        JobDesc jd;
        if ((rc = dense_job(ctx, "ks2:" + std::to_string(level), prime, &jd)))
            return rc;
        if ((rc = launch_ntt<false>(ctx, jd, ks2, 2LL * (k + 1) * n, ks2, 2LL * (k + 1) * n, batch, 0, s)))
            return rc;
    }
    {
        const long long total = batch * 2 * (n >> 1);
        DISPATCH_K(k, B200_LAUNCH(ksmoddown_kernel_v2<KK>, blocks_for(total, EB), EB, 0, s, ctx->d_primes, special, ctx->d_inv_qsp, ks2,
                                                                                base0, base0_stride, base1, base1_stride,
                                                                                dst, dst_stride, n, total));
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------
extern "C" {

const char *b200_last_error(void) { return g_err.c_str(); }

int b200_device_count(void)
{
    int c = 0;
    if (cudaGetDeviceCount(&c) != cudaSuccess)
        return 0;
    return c;
}

int b200_ctx_create(uint64_t n, const uint64_t *coeff_modulus, uint64_t count, uint64_t plain_modulus, int device,
                    b200_ctx **out)
{
    if (!coeff_modulus || !out)
        return fail(B200_E_NULL, "null argument");
    *out = nullptr;
    std::unique_ptr<b200_ctx> ctx(new b200_ctx());
    try
    {
        std::vector<b200::u64> mods(coeff_modulus, coeff_modulus + count);
        ctx->host.reset(new BfvHostContext((size_t)n, mods, plain_modulus));
    }
    catch (const std::invalid_argument &e)
    {
        return fail(B200_E_INVALID, e.what());
    }
    catch (const std::logic_error &e)
    {
        return fail(B200_E_LOGIC, e.what());
    }
    catch (const std::exception &e)
    {
        return fail(B200_E_INVALID, e.what());
    }
    ctx->n = ctx->host->n;
    ctx->logn = ctx->host->logn;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(B200_E_CUDA, "no CUDA device available: the CUDA backend has no CPU fallback");
    if (device < 0 || device >= ndev)
        return fail(B200_E_INVALID, "device index out of range");
    CU_TRY(cudaSetDevice(device));
    ctx->device = device;
    cudaDeviceProp prop;
    CU_TRY(cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    // NTT launch configuration
    // n = 32768: two global stages + quarter-size sub-transforms (69.6 KB of shared memory: three CTAs per SM); B200_NTT_SPLIT=1
    // selects the older one-stage / half-size split (139 KB: one CTA per SM)
    ctx->ntt_split = ctx->logn >= 15 ? (std::getenv("B200_NTT_SPLIT") ? atoi(std::getenv("B200_NTT_SPLIT")) : 2) : 0;
    if (ctx->ntt_split < 1 && ctx->logn >= 15)
        ctx->ntt_split = 1;
    if (ctx->ntt_split > 2)
        ctx->ntt_split = 2;
    if (ctx->logn > 15)
        return fail(B200_E_INVALID, "poly_modulus_degree above 32768 is not supported");
    const int local_logn = ctx->logn - ctx->ntt_split;
    ctx->npass = ntt_schedule(local_logn, ctx->pass_L);
    ctx->ntt_smem = (size_t)ntt_smem_words(1 << local_logn) * sizeof(u64);
    if (ctx->ntt_smem > (size_t)prop.sharedMemPerBlockOptin)
        return fail(B200_E_INVALID, "poly_modulus_degree too large for the shared-memory NTT");
    ctx->ntt_threads = local_logn >= 14 ? 512 : (local_logn >= 10 ? 256 : 64);
#ifndef B200_EMU_HEADER
    {
        const int frc = b200_ntt_fp_setup((int)prop.sharedMemPerBlockOptin);
        if (frc)
            return fail(B200_E_CUDA, std::string("cudaFuncSetAttribute (FP64 NTT kernels): ") + cudaGetErrorString((cudaError_t)frc));
        const int crc = b200_mul_cluster_setup(ctx->logn, &ctx->mul_clusters);
        if (crc)
            return fail(B200_E_CUDA, std::string("mul_cluster_kernel setup: ") + cudaGetErrorString((cudaError_t)crc));
    }
#endif
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 512>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
#ifndef B200_EMU_HEADER
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 256, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 256, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 256, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 256, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 256>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 256>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 256, 2>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 256, 2>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
#endif
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<true, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    CU_TRY(cudaFuncSetAttribute(ntt_kernel<false, 64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)prop.sharedMemPerBlockOptin));
    // A PRIVATE stream-ordered pool (the device's default pool is shared with every other user of the process, e.g. torch:
    // its attributes are not ours to change).  Freed scratch stays cached in it instead of returning to the OS.
    cudaMemPool_t pool;
    {
        cudaMemPoolProps props;
        std::memset(&props, 0, sizeof(props));
        props.allocType = cudaMemAllocationTypePinned;
        props.handleTypes = cudaMemHandleTypeNone;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = device;
        CU_TRY(cudaMemPoolCreate(&pool, &props));
        ctx->mempool = pool;
        unsigned long long thr = ~0ULL;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        // a block freed on one stream must not be handed to another stream by making that stream WAIT for the first one:
        // the per-handle path runs one operation per lane stream, and such a wait would chain independent operations
        if (!std::getenv("B200_POOL_INTERNAL_DEPS"))
        {
            int off = 0;
            cudaMemPoolSetAttribute(pool, cudaMemPoolReuseAllowInternalDependencies, &off);
        }
    }
    int rc = build_device(ctx.get());
    if (rc)
        return rc;
    CU_TRY(cudaStreamCreateWithFlags(&ctx->s_alloc, cudaStreamNonBlocking));
    CU_TRY(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
    CU_TRY(cudaStreamCreateWithFlags(&ctx->s_comp, cudaStreamNonBlocking));
    CU_TRY(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
    for (int i = 0; i < b200_ctx::NSIDE; i++)
    {
        CU_TRY(cudaStreamCreateWithFlags(&ctx->s_side[i], cudaStreamNonBlocking));
        CU_TRY(cudaEventCreateWithFlags(&ctx->ev_join[i], cudaEventDisableTiming));
    }
    CU_TRY(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    if (const char *sp = getenv("B200_MR_SPLIT"))
        ctx->mr_split = std::max(1, std::min((int)b200_ctx::NSIDE, atoi(sp)));
    CU_TRY(cudaDeviceSynchronize());
    *out = ctx.release();
    return 0;
}

static void host_pool_destroy(b200_ctx *ctx);
void b200_ctx_destroy(b200_ctx *ctx)
{
    if (!ctx)
        return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (void *p : ctx->allocations)
        cudaFree(p);
    for (int i = 0; i < b200_ctx::NBUF; i++)
        if (ctx->hst_a[i])
        {
            cudaFreeHost(ctx->hst_a[i]);
            cudaFreeHost(ctx->hst_b[i]);
            cudaFreeHost(ctx->hst_o[i]);
            cudaFree(ctx->dpk_a[i]);
            cudaFree(ctx->dpk_b[i]);
            cudaFree(ctx->dpk_o[i]);
        }
    host_pool_destroy(ctx); // (HostPool is defined further down: deleting it here would delete an incomplete type)
    for (int i = 0; i < b200_ctx::NBUF; i++)
        if (ctx->hp_a[i])
        {
            cudaFree(ctx->hp_a[i]);
            cudaFree(ctx->hp_b[i]);
            cudaFree(ctx->hp_o[i]);
            cudaEventDestroy(ctx->hp_in[i]);
            cudaEventDestroy(ctx->hp_comp[i]);
            cudaEventDestroy(ctx->hp_out[i]);
        }
    if (ctx->s_alloc)
        cudaStreamDestroy(ctx->s_alloc);
    if (ctx->s_h2d)
        cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_comp)
        cudaStreamDestroy(ctx->s_comp);
    if (ctx->s_d2h)
        cudaStreamDestroy(ctx->s_d2h);
    if (ctx->mempool)
        cudaMemPoolDestroy(ctx->mempool);
    delete ctx;
}

int b200_ctx_info(const b200_ctx *ctx, b200_info *out)
{
    if (!ctx || !out)
        return fail(B200_E_NULL, "null argument");
    out->n = ctx->n;
    out->plain_modulus = ctx->host->t;
    out->key_primes = ctx->host->K;
    out->levels = (int)ctx->host->levels.size();
    out->first_level = ctx->host->first_level();
    out->using_batching = ctx->host->using_batching;
    out->device = ctx->device;
    out->sm_count = ctx->sm_count;
    return 0;
}

int b200_ctx_level_info(const b200_ctx *ctx, int level, b200_level_info *out)
{
    if (!ctx || !out)
        return fail(B200_E_NULL, "null argument");
    if (level < 0 || level >= (int)ctx->host->levels.size())
        return fail(B200_E_INVALID, "level out of range");
    const LevelHost &L = ctx->host->levels[level];
    memset(out, 0, sizeof(*out));
    out->k = L.k;
    out->nB = L.nB;
    out->nBsk = L.nBsk;
    memcpy(out->parms_id, L.parms_id, sizeof(L.parms_id));
    out->m_sk = ctx->host->primes[ctx->host->aux0].mod.p;
    out->gamma = ctx->host->primes[L.gamma_idx].mod.p;
    for (int i = 0; i < L.k && i < 64; i++)
    {
        out->q[i] = ctx->host->primes[L.q_idx[i]].mod.p;
        out->roots[i] = ctx->host->primes[L.q_idx[i]].root;
        out->delta[i] = L.delta[i];
    }
    for (int j = 0; j < L.nBsk && j < 66; j++)
        out->bsk[j] = ctx->host->primes[L.bsk_idx[j]].mod.p;
    out->q_mod_t = L.q_mod_t;
    return 0;
}

int b200_galois_elt_from_step(const b200_ctx *ctx, int steps, uint32_t *elt)
{
    if (!ctx || !elt)
        return fail(B200_E_NULL, "null argument");
    try
    {
        *elt = ctx->host->galois_elt_from_step(steps);
    }
    catch (const std::exception &e)
    {
        return fail(B200_E_INVALID, e.what());
    }
    return 0;
}

// Device memory comes from the stream-ordered pool (release threshold = infinity, set at context creation): an
// allocation is a pool lookup, not a driver call, and a free does not synchronise the device — the per-handle FFI path
// allocates a destination per operation, and several host threads do so at once (sunscreen_runtime's rayon workers).
int b200_malloc(b200_ctx *ctx, size_t bytes, void **dptr)
{
    if (!ctx || !dptr)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> lk(ctx->alloc_mu);
    CU_TRY(cudaMallocFromPoolAsync(dptr, bytes ? bytes : 8, ctx->mempool, ctx->s_alloc));
    CU_TRY(cudaStreamSynchronize(ctx->s_alloc)); // usable from every stream on return
    return 0;
}
// the caller guarantees that no work using the buffer is still in flight (every layer-2 operation completes before it returns)
int b200_free(b200_ctx *ctx, void *dptr)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    if (!dptr)
        return 0;
    std::lock_guard<std::mutex> lk(ctx->alloc_mu);
    CU_TRY(cudaFreeAsync(dptr, ctx->s_alloc));
    return 0;
}
// free ordered after the work already enqueued on `stream` (an operation replacing a buffer it has just read)
int b200_free_async(b200_ctx *ctx, void *dptr, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    if (!dptr)
        return 0;
    CU_TRY(cudaFreeAsync(dptr, (cudaStream_t)stream));
    return 0;
}
int b200_stream_create(b200_ctx *ctx, void **stream)
{
    if (!ctx || !stream)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaSetDevice(ctx->device));
    cudaStream_t s;
    CU_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    *stream = (void *)s;
    return 0;
}
int b200_stream_destroy(b200_ctx *ctx, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    if (stream)
        CU_TRY(cudaStreamDestroy((cudaStream_t)stream));
    return 0;
}
int b200_malloc_host(size_t bytes, void **hptr)
{
    if (!hptr)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaMallocHost(hptr, bytes ? bytes : 8));
    return 0;
}
int b200_free_host(void *hptr)
{
    CU_TRY(cudaFreeHost(hptr));
    return 0;
}
int b200_memcpy_h2d(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return 0;
}
int b200_memcpy_d2h(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return 0;
}
int b200_memcpy_d2d(b200_ctx *ctx, void *dst, const void *src, size_t bytes, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return 0;
}
int b200_memzero(b200_ctx *ctx, void *dst, size_t bytes, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    if (!dst || !bytes)
        return 0;
    CU_TRY(cudaMemsetAsync(dst, 0, bytes, (cudaStream_t)stream));
    return 0;
}
int b200_stream_synchronize(b200_ctx *ctx, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}

// developer aid: attach a device buffer of 8 u64 per CTA that the NEXT static NTT launches fill with
// {smid, t_start, t_after_each_pass (<=5), t_end} (globaltimer ns); pass nullptr to detach
int b200_debug_ntt_stagger(int cycles)
{
#ifndef B200_EMU_HEADER
    return g_ntt_stagger.exchange(cycles);
#else
    (void)cycles;
    return 0;
#endif
}
int b200_debug_ntt_variant(int variant)
{
#ifndef B200_EMU_HEADER
    return g_ntt_var.exchange(variant);
#else
    (void)variant;
    return 0;
#endif
}
int b200_debug_ntt_ctas_per_sm(int logn, int forward, int threads, int variant)
{
#ifndef B200_EMU_HEADER
    // the query launch_ntt makes for the grid of the persistent variant (same kernel, same dynamic shared memory)
    b200_ntt_fp_fn sfn = b200_ntt_fp_kernel(logn, forward != 0, threads, variant);
    if (!sfn)
        return fail(B200_E_INVALID, "no FP64 NTT kernel for this (size, direction, CTA width, variant)");
    const size_t smem = (size_t)ntt_smem_words(1 << logn) * sizeof(u64) + ((variant & 1) ? B200_NTT_TWS_ENTRIES * sizeof(double) : 0);
    return b200_ntt_fp_ctas_per_sm(sfn, threads, smem);
#else
    (void)logn;
    (void)forward;
    (void)threads;
    (void)variant;
    return fail(B200_E_INVALID, "the emulation build has no FP64 NTT kernels");
#endif
}
void b200_ntt_timeline(b200_ctx *ctx, unsigned long long *device_buffer)
{
    if (ctx)
        ctx->ntt_timeline = device_buffer;
}

void b200_trace_dump(void)
{
#ifndef B200_EMU_HEADER
    cudaDeviceSynchronize();
    std::map<std::string, std::pair<double, int>> acc;
    std::vector<std::string> order;
    double total = 0;
    for (auto &r : g_trace)
    {
        float ms = 0;
        cudaEventElapsedTime(&ms, r.e0, r.e1);
        cudaEventDestroy(r.e0);
        cudaEventDestroy(r.e1);
        if (!acc.count(r.name))
            order.push_back(r.name);
        acc[r.name].first += ms;
        acc[r.name].second++;
        total += ms;
    }
    for (auto &nm : order)
        fprintf(stderr, "[b200 trace] %-44s launches %5d  total %9.3f ms  avg %8.4f ms  %5.1f%%\n", nm.c_str(), acc[nm].second,
                acc[nm].first, acc[nm].first / acc[nm].second, 100.0 * acc[nm].first / total);
    fprintf(stderr, "[b200 trace] total %.3f ms\n", total);
    g_trace.clear();
#endif
}

// dst[i*words .. ) <- *srcs[i]   (gather = 1)   or   *ptrs[i] <- slab[i*words ..)   (gather = 0); ptrs is a DEVICE array
__global__ void gather_scatter_kernel(u64 *const *ptrs, u64 *slab, long long words, int gather)
{
    const long long i = blockIdx.y;
    u64 *p = ptrs[i];
    u64 *s = slab + i * words;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < words; e += (long long)gridDim.x * blockDim.x)
    {
        if (gather)
            s[e] = p[e];
        else
            p[e] = s[e];
    }
}
// Move `count` equally sized word arrays between individually allocated device buffers (host array of device pointers)
// and one contiguous slab, in ONE launch: the batch seams of the SEAL-named layer gather operands and scatter results
// this way instead of issuing a memcpy per ciphertext.
int b200_gather_scatter(b200_ctx *ctx, uint64_t *const *host_ptrs, uint64_t count, uint64_t *slab, uint64_t words, int gather,
                        void *stream)
{
    if (!ctx || !host_ptrs || !slab)
        return fail(B200_E_NULL, "null argument");
    if (count == 0 || words == 0)
        return 0;
    if (count > 65535)
        return fail(B200_E_INVALID, "at most 65535 items per gather/scatter");
    cudaStream_t s = (cudaStream_t)stream;
    void *dptrs = nullptr;
    CU_TRY(cudaMallocFromPoolAsync(&dptrs, count * sizeof(void *), ctx->mempool, s));
    CU_TRY(cudaMemcpyAsync(dptrs, host_ptrs, count * sizeof(void *), cudaMemcpyHostToDevice, s));
    dim3 grid((unsigned)std::min<long long>(64, (long long)(words + 255) / 256), (unsigned)count);
    B200_LAUNCH(gather_scatter_kernel, grid, 256, 0, s, (u64 *const *)dptrs, (u64 *)slab, (long long)words, gather);
    ctx->launches++;
    CU_TRY(cudaFreeAsync(dptrs, s));
    CU_TRY(cudaGetLastError());
    return 0;
}

// Same, with the pointer table already in device-ACCESSIBLE memory (e.g. pinned host memory, which kernels read directly under
// unified addressing): no staging copy, no allocation — the combining layer's per-batch cost is then one launch.
int b200_gather_scatter_table(b200_ctx *ctx, uint64_t *const *table, uint64_t count, uint64_t *slab, uint64_t words, int gather,
                              void *stream)
{
    if (!ctx || !table || !slab)
        return fail(B200_E_NULL, "null argument");
    if (count == 0 || words == 0)
        return 0;
    if (count > 65535)
        return fail(B200_E_INVALID, "at most 65535 items per gather/scatter");
    dim3 grid((unsigned)std::min<long long>(64, (long long)(words + 255) / 256), (unsigned)count);
    B200_LAUNCH(gather_scatter_kernel, grid, 256, 0, (cudaStream_t)stream, (u64 *const *)table, (u64 *)slab, (long long)words, gather);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}
// ---- CUDA graphs for fixed launch sequences (the combining layer of the SEAL-named ABI replays one graph per batch) ----
// Everything enqueued on `stream` between begin and end becomes a graph: kernels with their parameters BY VALUE and the
// stream-ordered allocations / frees as memory nodes, so a replay touches the same addresses.  The caller guarantees that
// the captured sequence only reads its varying inputs through fixed locations (pinned pointer tables).
int b200_capture_begin(b200_ctx *ctx, void *stream)
{
#ifdef B200_EMU_HEADER
    (void)ctx;
    (void)stream;
    return fail(B200_E_LOGIC, "graphs are not available in the emulation build");
#else
    if (!ctx || !stream)
        return fail(B200_E_NULL, "null argument");
    if (trace_on())
        return fail(B200_E_LOGIC, "no graph capture while tracing");
    CU_TRY(cudaStreamBeginCapture((cudaStream_t)stream, cudaStreamCaptureModeRelaxed));
    return 0;
#endif
}
int b200_capture_end(b200_ctx *ctx, void *stream, void **graph_exec)
{
#ifdef B200_EMU_HEADER
    (void)ctx;
    (void)stream;
    (void)graph_exec;
    return fail(B200_E_LOGIC, "graphs are not available in the emulation build");
#else
    if (!ctx || !stream || !graph_exec)
        return fail(B200_E_NULL, "null argument");
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture((cudaStream_t)stream, &g);
    if (e != cudaSuccess || !g)
    {
        cudaGetLastError();
        return fail(B200_E_CUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(e));
    }
    cudaGraphExec_t x = nullptr;
    e = cudaGraphInstantiate(&x, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess)
        return fail(B200_E_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e));
    *graph_exec = x;
    return 0;
#endif
}
int b200_graph_launch(b200_ctx *ctx, void *graph_exec, void *stream)
{
#ifdef B200_EMU_HEADER
    (void)ctx;
    (void)graph_exec;
    (void)stream;
    return fail(B200_E_LOGIC, "graphs are not available in the emulation build");
#else
    if (!ctx || !graph_exec)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaGraphLaunch((cudaGraphExec_t)graph_exec, (cudaStream_t)stream));
    ctx->launches++;
    return 0;
#endif
}
int b200_graph_destroy(b200_ctx *ctx, void *graph_exec)
{
#ifndef B200_EMU_HEADER
    if (ctx && graph_exec)
        cudaGraphExecDestroy((cudaGraphExec_t)graph_exec);
#else
    (void)ctx;
    (void)graph_exec;
#endif
    return 0;
}

// Wait for `stream` WITHOUT spinning: the calling thread sleeps on a blocking-sync event until the work is done.  For waits of
// milliseconds (the batch seams: transfers of tens of MiB) — many caller threads that spin in cudaStreamSynchronize burn one core each,
// and on a CPU-quota'd host that gets the whole process throttled.  `*event_slot` caches the event (created on first use).
int b200_stream_synchronize_blocking(b200_ctx *ctx, void *stream, void **event_slot)
{
    if (!ctx || !event_slot)
        return fail(B200_E_NULL, "null argument");
    cudaEvent_t ev = (cudaEvent_t)*event_slot;
    if (!ev)
    {
        CU_TRY(cudaEventCreateWithFlags(&ev, cudaEventBlockingSync | cudaEventDisableTiming));
        *event_slot = ev;
    }
    CU_TRY(cudaEventRecord(ev, (cudaStream_t)stream));
    CU_TRY(cudaEventSynchronize(ev));
    return 0;
}
int b200_event_destroy(b200_ctx *ctx, void *event)
{
    (void)ctx;
    if (event)
        cudaEventDestroy((cudaEvent_t)event);
    return 0;
}
// make the context's GPU the calling thread's current device (a new host thread starts on device 0: the SEAL-named layer
// calls this at the start of every operation, so worker threads of a multi-GPU process need no CUDA calls of their own)
int b200_bind_thread(b200_ctx *ctx)
{
    if (!ctx)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaSetDevice(ctx->device)); // (a no-op when it already is the current device)
    return 0;
}
// stream-ordered allocation usable by work enqueued on `stream` after this call (no host synchronisation)
int b200_malloc_async(b200_ctx *ctx, size_t bytes, void **dptr, void *stream)
{
    if (!ctx || !dptr)
        return fail(B200_E_NULL, "null argument");
    CU_TRY(cudaMallocFromPoolAsync(dptr, bytes ? bytes : 8, ctx->mempool, (cudaStream_t)stream));
    return 0;
}

uint64_t b200_launch_count(const b200_ctx *ctx) { return ctx ? ctx->launches.load() : 0; }

// ---- NTT ----
static int ntt_slab(b200_ctx *ctx, int level, u64 *data, uint64_t items, void *stream, bool fwd)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!data)
        return fail(B200_E_NULL, "null data");
    JobDesc jd;
    if ((rc = dense_job(ctx, "slab:" + std::to_string(level), row_primes(ctx, level, false), &jd)))
        return rc;
    const long long stride = (long long)ctx->levels[level].k * (long long)ctx->n;
    if (fwd)
        return launch_ntt<true>(ctx, jd, data, stride, data, stride, (long long)items, 0, (cudaStream_t)stream);
    return launch_ntt<false>(ctx, jd, data, stride, data, stride, (long long)items, 0, (cudaStream_t)stream);
}
int b200_ntt_forward(b200_ctx *ctx, int level, uint64_t *data, uint64_t items, void *stream)
{
    return ntt_slab(ctx, level, (u64 *)data, items, stream, true);
}
int b200_ntt_inverse(b200_ctx *ctx, int level, uint64_t *data, uint64_t items, void *stream)
{
    return ntt_slab(ctx, level, (u64 *)data, items, stream, false);
}

// negacyclic NTT modulo the PLAIN modulus t over [items][n] (BatchEncoder's transform, S/batchencoder.cpp:129,149)
int b200_plain_ntt(b200_ctx *ctx, uint64_t *data, uint64_t items, int inverse, void *stream)
{
    if (!ctx)
        return fail(B200_E_NULL, "null context");
    if (!data)
        return fail(B200_E_NULL, "null data");
    if (ctx->plain_prime_idx < 0)
        return fail(B200_E_INVALID, "encryption parameters are not valid for batching");
    JobDesc jd;
    int rc = dense_job(ctx, "plain", std::vector<int>(1, ctx->plain_prime_idx), &jd);
    if (rc)
        return rc;
    const long long stride = (long long)ctx->n;
    if (inverse)
        return launch_ntt<false>(ctx, jd, (u64 *)data, stride, (u64 *)data, stride, (long long)items, 0, (cudaStream_t)stream);
    return launch_ntt<true>(ctx, jd, (u64 *)data, stride, (u64 *)data, stride, (long long)items, 0, (cudaStream_t)stream);
}

// ---- add / sub / negate ----
static int addsub(b200_ctx *ctx, int level, const u64 *a, const u64 *b, u64 *out, int size, uint64_t batch, void *stream,
                  int mode)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !out || (mode != 2 && !b))
        return fail(B200_E_NULL, "null ciphertext pointer");
    if (size < 1)
        return fail(B200_E_INVALID, "size");
    const LevelDev &L = ctx->levels[level];
    const long long total = (long long)batch * size * L.k * (long long)ctx->n;
    if (total == 0)
        return 0;
    B200_LAUNCH(addsub_kernel, blocks_for(total, EB), EB, 0, (cudaStream_t)stream, ctx->d_primes, L.k, a, b, out, ctx->logn, mode,
                                                                         total);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}
int b200_add(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, uint64_t *out, int size, uint64_t batch,
             void *stream)
{
    return addsub(ctx, level, (const u64 *)a, (const u64 *)b, (u64 *)out, size, batch, stream, 0);
}
int b200_sub(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, uint64_t *out, int size, uint64_t batch,
             void *stream)
{
    return addsub(ctx, level, (const u64 *)a, (const u64 *)b, (u64 *)out, size, batch, stream, 1);
}
int b200_negate(b200_ctx *ctx, int level, const uint64_t *a, uint64_t *out, int size, uint64_t batch, void *stream)
{
    return addsub(ctx, level, (const u64 *)a, nullptr, (u64 *)out, size, batch, stream, 2);
}

// residues of small signed host samples: vals [polys][n] (int64, device) -> out [polys][k][n]
int b200_expand_signed(b200_ctx *ctx, int level, const int64_t *vals, int polys, uint64_t *out, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!vals || !out)
        return fail(B200_E_NULL, "null pointer");
    if (polys < 1)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const int k = ctx->levels[level].k;
    const long long total = (long long)polys * k * (long long)ctx->n;
    B200_LAUNCH(expand_signed_kernel, blocks_for(total, EB), EB, 0, (cudaStream_t)stream, ctx->d_primes, k, (const long long *)vals,
                (u64 *)out, ctx->logn, total);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---- multiply / square ----
int b200_multiply(b200_ctx *ctx, int level, const uint64_t *a, int sa, const uint64_t *b, int sb, uint64_t *out,
                  uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !b || !out)
        return fail(B200_E_NULL, "null ciphertext pointer");
    if (sa < 1 || sb < 1 || sa + sb - 1 > 16)
        return fail(B200_E_INVALID, "ciphertext sizes must be >= 1 with a destination size of at most 16");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const int Dn = sa + sb - 1;
    return multiply_core(ctx, level, (const u64 *)a, sa, (const u64 *)b, sb, false, (u64 *)out, Dn, nullptr,
                         (long long)batch, (cudaStream_t)stream);
}

int b200_square(b200_ctx *ctx, int level, const uint64_t *a, uint64_t *out, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !out)
        return fail(B200_E_NULL, "null ciphertext pointer");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    return multiply_core(ctx, level, (const u64 *)a, 2, nullptr, 0, true, (u64 *)out, 3, nullptr, (long long)batch,
                         (cudaStream_t)stream);
}

int b200_relinearize(b200_ctx *ctx, int level, const uint64_t *in3, const uint64_t *relin_key, uint64_t *out2,
                     uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!in3 || !relin_key || !out2)
        return fail(B200_E_NULL, "null pointer");
    if (batch == 0)
        return 0;
    if ((const void *)in3 == (const void *)out2 && batch != 1)
        return fail(B200_E_INVALID, "in-place relinearize is only defined for batch == 1");
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const int k = ctx->levels[level].k;
    const u64 *c = (const u64 *)in3;
    return keyswitch_core(ctx, level, c + 2LL * k * n, 3LL * k * n, (const u64 *)relin_key, c, 3LL * k * n, c + (long long)k * n,
                          3LL * k * n, (u64 *)out2, 2LL * k * n, (long long)batch, (cudaStream_t)stream);
}

static int multiply_relin_one(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, const uint64_t *relin_key,
                             uint64_t *out2, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !b || !relin_key || !out2)
        return fail(B200_E_NULL, "null pointer");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const int k = ctx->levels[level].k;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *c2 = nullptr;
    if ((rc = scr.get((size_t)batch * k * n, &c2)))
        return rc;
    // c0,c1 go straight into out2; c2 into scratch
    if ((rc = multiply_core(ctx, level, (const u64 *)a, 2, (const u64 *)b, 2, false, (u64 *)out2, 2, c2, (long long)batch, s)))
        return rc;
    u64 *o = (u64 *)out2;
    return keyswitch_core(ctx, level, c2, (long long)k * n, (const u64 *)relin_key, o, 2LL * k * n, o + (long long)k * n,
                          2LL * k * n, o, 2LL * k * n, (long long)batch, s);
}

int b200_multiply_relin(b200_ctx *ctx, int level, const uint64_t *a, const uint64_t *b, const uint64_t *relin_key,
                        uint64_t *out2, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    const int parts = (ctx->mr_split > 1 && batch >= 64) ? ctx->mr_split : 1;
    if (parts == 1)
        return multiply_relin_one(ctx, level, a, b, relin_key, out2, batch, stream);
    // fork: sub-batches on side streams, ordered after everything already enqueued on the caller's stream
    CU_TRY(cudaSetDevice(ctx->device));
    cudaStream_t us = (cudaStream_t)stream;
    const size_t w = (size_t)2 * ctx->levels[level].k * ctx->n;
    CU_TRY(cudaEventRecord(ctx->ev_fork, us));
    for (int p = 0; p < parts && !rc; p++)
    {
        const uint64_t lo = batch * p / parts, hi = batch * (p + 1) / parts;
        CU_TRY(cudaStreamWaitEvent(ctx->s_side[p], ctx->ev_fork, 0));
        rc = multiply_relin_one(ctx, level, a + lo * w, b + lo * w, relin_key, out2 + lo * w, hi - lo, ctx->s_side[p]);
        CU_TRY(cudaEventRecord(ctx->ev_join[p], ctx->s_side[p]));
        CU_TRY(cudaStreamWaitEvent(us, ctx->ev_join[p], 0));
    }
    return rc;
}

int b200_apply_galois(b200_ctx *ctx, int level, const uint64_t *in2, uint32_t galois_elt, const uint64_t *galois_key,
                      uint64_t *out2, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!in2 || !galois_key || !out2)
        return fail(B200_E_NULL, "null pointer");
    if (!(galois_elt & 1) || galois_elt >= 2 * ctx->n)
        return fail(B200_E_INVALID, "Galois element is not valid");
    if ((const void *)in2 == (const void *)out2)
        return fail(B200_E_INVALID, "apply_galois cannot run in place at this layer");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const LevelDev &L = ctx->levels[level];
    const int k = L.k;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *tmp = nullptr;
    if ((rc = scr.get((size_t)batch * k * n, &tmp)))
        return rc;
    const long long total = (long long)batch * 2 * k * n;
    B200_LAUNCH(galois_kernel, blocks_for(total, EB), EB, 0, s, ctx->d_primes, k, (const u64 *)in2, (u64 *)out2, tmp, ctx->logn,
                                                       galois_elt, total);
    ctx->launches++;
    u64 *o = (u64 *)out2;
    return keyswitch_core(ctx, level, tmp, (long long)k * n, (const u64 *)galois_key, o, 2LL * k * n, nullptr, 0, o,
                          2LL * k * n, (long long)batch, s);
}

int b200_multiply_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t pb,
                        uint64_t *out, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !plain || !out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 1 || (pb != 1 && pb != batch))
        return fail(B200_E_INVALID, "size / plain_batch");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const LevelDev &L = ctx->levels[level];
    const int k = L.k;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *pl = nullptr;
    if ((rc = scr.get((size_t)pb * k * n, &pl)))
        return rc;
    u32 *mono = nullptr;
    if (L.fast_plain_lift)
    {
        u64 *flags = nullptr;
        if ((rc = scr.get((size_t)(pb + 1) / 2, &flags)))
            return rc;
        mono = (u32 *)flags;
        B200_LAUNCH(plain_monomial_kernel, (unsigned)pb, 1024, 1024 * sizeof(u64), s, (const u64 *)plain, n, mono);
        ctx->launches++;
    }
    {
        const long long total = (long long)pb * k * n;
        B200_LAUNCH(plain_lift_kernel, blocks_for(total, EB), EB, 0, s, L, (const u64 *)plain, (const u32 *)mono, pl, ctx->logn,
                                                                total);
        ctx->launches++;
    }
    JobDesc jd;
    if ((rc = dense_job(ctx, "slab:" + std::to_string(level), row_primes(ctx, level, false), &jd)))
        return rc;
    if ((rc = launch_ntt<true>(ctx, jd, pl, (long long)k * n, pl, (long long)k * n, (long long)pb, 0, s)))
        return rc;
    // ct polys: forward (out of place), dyadic, inverse
    if ((rc = launch_ntt<true>(ctx, jd, (const u64 *)a, (long long)k * n, (u64 *)out, (long long)k * n, (long long)batch * size, 0,
                               s)))
        return rc;
    {
        const long long total = (long long)batch * size * k * n;
        B200_LAUNCH(dyadic_plain_kernel, blocks_for(total, EB), EB, 0, s, ctx->d_primes, k, size, (const u64 *)out, pl, (long long)pb,
                                                                 (u64 *)out, ctx->logn, total);
        ctx->launches++;
    }
    if ((rc = launch_ntt<false>(ctx, jd, (const u64 *)out, (long long)k * n, (u64 *)out, (long long)k * n,
                                (long long)batch * size, 0, s)))
        return rc;
    CU_TRY(cudaGetLastError());
    return 0;
}

// out[item][poly][r][c] = x[item][poly][r][c] * y[item % y_batch][r][c] mod q_r  (dyadic_product_coeffmod,
// S/util/polyarithsmallmod.cpp:226-284); any domain, canonical in/out
int b200_dyadic_product(b200_ctx *ctx, int level, const uint64_t *x, int size, const uint64_t *y, uint64_t y_batch,
                        uint64_t *out, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!x || !y || !out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 1 || y_batch < 1)
        return fail(B200_E_INVALID, "size / y_batch");
    if (batch == 0)
        return 0;
    const int k = ctx->levels[level].k;
    const long long total = (long long)batch * size * k * (long long)ctx->n;
    B200_LAUNCH(dyadic_plain_kernel, blocks_for(total, EB), EB, 0, (cudaStream_t)stream, ctx->d_primes, k, size, (const u64 *)x,
                (const u64 *)y, (long long)y_batch, (u64 *)out, ctx->logn, total);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

static int addsub_plain(b200_ctx *ctx, int level, const u64 *a, int size, const u64 *plain, uint64_t pb, u64 *out,
                        uint64_t batch, void *stream, int sign)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !plain || !out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 1 || (pb != 1 && pb != batch))
        return fail(B200_E_INVALID, "size / plain_batch");
    if (batch == 0)
        return 0;
    const LevelDev &L = ctx->levels[level];
    const long long total = (long long)batch * size * L.k * (long long)ctx->n;
    B200_LAUNCH(addsub_plain_kernel, blocks_for(total, EB), EB, 0, (cudaStream_t)stream, L, size, a, plain, (long long)pb, out,
                                                                               ctx->logn, sign, total);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}
int b200_add_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t pb, uint64_t *out,
                   uint64_t batch, void *stream)
{
    return addsub_plain(ctx, level, (const u64 *)a, size, (const u64 *)plain, pb, (u64 *)out, batch, stream, 0);
}
int b200_sub_plain(b200_ctx *ctx, int level, const uint64_t *a, int size, const uint64_t *plain, uint64_t pb, uint64_t *out,
                   uint64_t batch, void *stream)
{
    return addsub_plain(ctx, level, (const u64 *)a, size, (const u64 *)plain, pb, (u64 *)out, batch, stream, 1);
}

int b200_mod_switch_to_next(b200_ctx *ctx, int level, const uint64_t *a, int size, uint64_t *out, uint64_t batch,
                            void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a || !out)
        return fail(B200_E_NULL, "null pointer");
    const LevelDev &L = ctx->levels[level];
    if (L.k < 2 || level + 1 >= (int)ctx->levels.size())
        return fail(B200_E_INVALID, "end of modulus switching chain reached");
    if (batch == 0)
        return 0;
    const long long n = (long long)ctx->n;
    const long long total = (long long)batch * size * n;
    DISPATCH_K(L.k, B200_LAUNCH(modswitch_kernel<KK>, blocks_for(total, EB), EB, 0, (cudaStream_t)stream, 
                        ctx->d_primes, L.inv_qlast, (const u64 *)a, (u64 *)out, n, total));
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

int b200_decrypt(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *plain_out,
                 uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!ct || !sk_powers_ntt || !plain_out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 2)
        return fail(B200_E_INVALID, "ciphertext size must be >= 2");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const LevelDev &L = ctx->levels[level];
    const LevelHost &Lh = ctx->host->levels[level];
    const int k = L.k, terms = size - 1;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *X = nullptr, *acc = nullptr;
    if ((rc = scr.get((size_t)batch * terms * k * n, &X)))
        return rc;
    if ((rc = scr.get((size_t)batch * k * n, &acc)))
        return rc;
    {
        std::vector<int> prime;
        std::vector<long long> so, dof;
        for (int j = 0; j < terms; j++)
            for (int r = 0; r < k; r++)
            {
                prime.push_back(Lh.q_idx[r]);
                so.push_back(((long long)(j + 1) * k + r) * n);
                dof.push_back(((long long)j * k + r) * n);
            }
        JobDesc jd;
        if ((rc = get_job(ctx, "dec:" + std::to_string(level) + ":" + std::to_string(size), prime, so, dof, &jd)))
            return rc;
        if ((rc = launch_ntt<true>(ctx, jd, (const u64 *)ct, (long long)size * k * n, X, (long long)terms * k * n,
                                   (long long)batch, 0, s)))
            return rc;
    }
    {
        const long long total = (long long)batch * k * n;
        B200_LAUNCH(dot_sk_kernel, blocks_for(total, EB), EB, 0, s, ctx->d_primes, k, terms, X, (const u64 *)sk_powers_ntt, acc,
                                                           ctx->logn, total);
        ctx->launches++;
    }
    JobDesc jd;
    if ((rc = dense_job(ctx, "slab:" + std::to_string(level), row_primes(ctx, level, false), &jd)))
        return rc;
    if ((rc = launch_ntt<false>(ctx, jd, acc, (long long)k * n, acc, (long long)k * n, (long long)batch, 0, s)))
        return rc;
    {
        const long long total = (long long)batch * n;
        DISPATCH_K(k, B200_LAUNCH(decrypt_kernel<KK>, blocks_for(total, EB), EB, 0, s, L, size, (const u64 *)ct, acc,
                                                                              (u64 *)plain_out, n, total));
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

// phase = c0 + sum_{j>=1} c_j * s^j  (coefficient form, canonical), [batch][k][n]
int b200_ct_sk_phase(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *phase_out,
                     uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!ct || !sk_powers_ntt || !phase_out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 2)
        return fail(B200_E_INVALID, "ciphertext size must be >= 2");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const LevelDev &L = ctx->levels[level];
    const LevelHost &Lh = ctx->host->levels[level];
    const int k = L.k, terms = size - 1;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *X = nullptr;
    u64 *acc = (u64 *)phase_out;
    if ((rc = scr.get((size_t)batch * terms * k * n, &X)))
        return rc;
    {
        std::vector<int> prime;
        std::vector<long long> so, dof;
        for (int j = 0; j < terms; j++)
            for (int r = 0; r < k; r++)
            {
                prime.push_back(Lh.q_idx[r]);
                so.push_back(((long long)(j + 1) * k + r) * n);
                dof.push_back(((long long)j * k + r) * n);
            }
        JobDesc jd;
        if ((rc = get_job(ctx, "dec:" + std::to_string(level) + ":" + std::to_string(size), prime, so, dof, &jd)))
            return rc;
        if ((rc = launch_ntt<true>(ctx, jd, (const u64 *)ct, (long long)size * k * n, X, (long long)terms * k * n,
                                   (long long)batch, 0, s)))
            return rc;
    }
    {
        const long long total = (long long)batch * k * n;
        B200_LAUNCH(dot_sk_kernel, blocks_for(total, EB), EB, 0, s, ctx->d_primes, k, terms, X, (const u64 *)sk_powers_ntt, acc,
                    ctx->logn, total);
        ctx->launches++;
    }
    JobDesc jd;
    if ((rc = dense_job(ctx, "slab:" + std::to_string(level), row_primes(ctx, level, false), &jd)))
        return rc;
    if ((rc = launch_ntt<false>(ctx, jd, acc, (long long)k * n, acc, (long long)k * n, (long long)batch, 0, s)))
        return rc;
    {
        const long long total = (long long)batch * n;
        DISPATCH_K(k, B200_LAUNCH(phase_add_kernel<KK>, blocks_for(total, EB), EB, 0, s, ctx->d_primes, size, (const u64 *)ct, acc, n,
                                  total));
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

// infinity norm of the centred t * (c0 + sum_j c_j s^j) mod Q of each item as a little-endian multi-precision integer
// (Decryptor::invariant_noise_internal, S/decryptor.cpp:424-485).  norm_out: HOST array [batch][words]; the call returns
// after the result has arrived.
int b200_noise_norm(b200_ctx *ctx, int level, const uint64_t *ct, int size, const uint64_t *sk_powers_ntt, uint64_t *norm_out,
                    int words, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!ct || !sk_powers_ntt || !norm_out)
        return fail(B200_E_NULL, "null pointer");
    if (size < 2)
        return fail(B200_E_INVALID, "ciphertext size must be >= 2");
    CU_TRY(cudaSetDevice(ctx->device));
    const long long n = (long long)ctx->n;
    const LevelDev &L = ctx->levels[level];
    const LevelHost &Lh = ctx->host->levels[level];
    const int k = L.k, terms = size - 1;
    u64 *consts = nullptr;
    int W = 0;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        auto it = ctx->noise_consts.find(level);
        if (it == ctx->noise_consts.end())
        {
            std::vector<u64> q(k);
            for (int i = 0; i < k; i++)
                q[i] = ctx->host->primes[Lh.q_idx[i]].mod.p;
            b200::BigUInt Q(1);
            for (u64 v : q)
                Q.mul(v);
            W = (int)Q.w.size();
            if (W + 1 > NOISE_MAXW)
                return fail(B200_E_INVALID, "coefficient modulus too wide for the noise-norm kernel");
            std::vector<u64> h((size_t)3 * k + 2 * (W + 1) + (size_t)k * W, 0);
            for (int i = 0; i < k; i++)
            {
                h[i] = q[i];
                h[k + i] = Lh.scale_c[i].w;
                h[2 * k + i] = Lh.scale_c[i].wq;
                b200::BigUInt P(1);
                for (int j = 0; j < k; j++)
                    if (j != i)
                        P.mul(q[j]);
                std::copy(P.w.begin(), P.w.end(), h.begin() + 3 * k + 2 * (W + 1) + (size_t)i * W);
            }
            u64 *Qw = h.data() + 3 * k, *half = Qw + W + 1;
            std::copy(Q.w.begin(), Q.w.end(), Qw);
            { // half = (Q + 1) / 2: value >= half  <=>  centred negative
                std::vector<u64> tmp(Qw, Qw + W + 1);
                u64 carry = 1;
                for (auto &x : tmp)
                {
                    const u64 s = x + carry;
                    carry = s < x;
                    x = s;
                }
                for (int i = 0; i <= W; i++)
                    half[i] = (tmp[i] >> 1) | (i < W ? tmp[i + 1] << 63 : 0);
            }
            if ((rc = upload(ctx, h, &consts)))
                return rc;
            ctx->noise_consts[level] = std::make_pair(consts, W);
        }
        else
        {
            consts = it->second.first;
            W = it->second.second;
        }
    }
    if (words < W + 1)
        return fail(B200_E_INVALID, "norm_out holds fewer words than the coefficient modulus");
    for (size_t i = 0; i < (size_t)batch * words; i++)
        norm_out[i] = 0;
    if (batch == 0)
        return 0;
    cudaStream_t s = (cudaStream_t)stream;
    Scratch scr(ctx, s);
    u64 *X = nullptr, *acc = nullptr, *bm = nullptr;
    const int NT = 128, CHUNK = 128, WW = W + 1;
    const int blocks = (int)((n + CHUNK - 1) / CHUNK);
    if ((rc = scr.get((size_t)batch * terms * k * n, &X)))
        return rc;
    if ((rc = scr.get((size_t)batch * k * n, &acc)))
        return rc;
    if ((rc = scr.get((size_t)batch * blocks * WW, &bm)))
        return rc;
    {
        std::vector<int> prime;
        std::vector<long long> so, dof;
        for (int j = 0; j < terms; j++)
            for (int r = 0; r < k; r++)
            {
                prime.push_back(Lh.q_idx[r]);
                so.push_back(((long long)(j + 1) * k + r) * n);
                dof.push_back(((long long)j * k + r) * n);
            }
        JobDesc jd;
        if ((rc = get_job(ctx, "dec:" + std::to_string(level) + ":" + std::to_string(size), prime, so, dof, &jd)))
            return rc;
        if ((rc = launch_ntt<true>(ctx, jd, (const u64 *)ct, (long long)size * k * n, X, (long long)terms * k * n,
                                   (long long)batch, 0, s)))
            return rc;
    }
    {
        const long long total = (long long)batch * k * n;
        B200_LAUNCH(dot_sk_kernel, blocks_for(total, EB), EB, 0, s, ctx->d_primes, k, terms, X, (const u64 *)sk_powers_ntt, acc,
                    ctx->logn, total);
        ctx->launches++;
    }
    JobDesc jd;
    if ((rc = dense_job(ctx, "slab:" + std::to_string(level), row_primes(ctx, level, false), &jd)))
        return rc;
    if ((rc = launch_ntt<false>(ctx, jd, acc, (long long)k * n, acc, (long long)k * n, (long long)batch, 0, s)))
        return rc;
    {
        dim3 grid((unsigned)blocks, (unsigned)batch);
        B200_LAUNCH(noise_norm_kernel, grid, NT, (size_t)NT * WW * 8, s, (const u64 *)consts, k, W, size, (const u64 *)ct,
                    (const u64 *)acc, n, CHUNK, bm);
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    std::vector<u64> hb((size_t)batch * blocks * WW);
    CU_TRY(cudaMemcpyAsync(hb.data(), bm, hb.size() * 8, cudaMemcpyDeviceToHost, s));
    CU_TRY(cudaStreamSynchronize(s));
    for (uint64_t b = 0; b < batch; b++)
    {
        u64 *best = (u64 *)norm_out + b * words;
        for (int j = 0; j < blocks; j++)
        {
            const u64 *v = hb.data() + (b * blocks + j) * WW;
            if (mp_ge(v, best, WW))
                std::copy(v, v + WW, best);
        }
    }
    return 0;
}

int b200_is_transparent(b200_ctx *ctx, int level, const uint64_t *ct, int size, uint32_t *flags_out, uint64_t batch,
                        void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!ct || !flags_out)
        return fail(B200_E_NULL, "null pointer");
    if (batch == 0)
        return 0;
    const long long n = (long long)ctx->n;
    const int k = ctx->levels[level].k;
    cudaStream_t s = (cudaStream_t)stream;
    B200_LAUNCH(fill_u32_kernel, blocks_for((long long)batch, EB), EB, 0, s, flags_out, 1u, (long long)batch);
    ctx->launches++;
    if (size >= 2)
    {
        dim3 grid(8, (unsigned)batch);
        B200_LAUNCH(transparent_kernel, grid, 256, 0, s, (const u64 *)ct, (long long)size * k * n, (long long)k * n, flags_out);
        ctx->launches++;
    }
    CU_TRY(cudaGetLastError());
    return 0;
}

// flags[item] = 1 when polys [1, size) of the item hold a nonzero word; flags are NOT cleared here (the caller zeroes them)
// and may live in pinned host memory (b200_malloc_host; device-accessible under UVA), which saves the per-call path a fill
// kernel and a device-to-host copy per operation
__global__ void any_nonzero_kernel(const u64 *ct, long long item_words, long long skip_words, u32 *flags)
{
    const long long item = blockIdx.y;
    const u64 *p = ct + item * item_words + skip_words;
    const long long cnt = item_words - skip_words;
    bool nz = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (long long)gridDim.x * blockDim.x)
        nz |= p[i] != 0;
    if (nz)
        flags[item] = 1; // every writer stores the same value
}
int b200_any_nonzero(b200_ctx *ctx, int level, const uint64_t *ct, int size, uint32_t *flags, uint64_t batch, void *stream)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!ct || !flags)
        return fail(B200_E_NULL, "null pointer");
    if (batch == 0 || size < 2)
        return 0;
    const long long n = (long long)ctx->n;
    const int k = ctx->levels[level].k;
    const long long words = (long long)(size - 1) * k * n;
    dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(64, words / 512)), (unsigned)batch);
    B200_LAUNCH(any_nonzero_kernel, grid, 256, 0, (cudaStream_t)stream, (const u64 *)ct, (long long)size * k * n, (long long)k * n,
                flags);
    ctx->launches++;
    CU_TRY(cudaGetLastError());
    return 0;
}

// ---- host-buffer variants ----
static int host_ring(b200_ctx *ctx, size_t words_per_slot)
{
    if (ctx->hp_words >= words_per_slot)
        return 0;
    for (int i = 0; i < b200_ctx::NBUF; i++)
    {
        if (ctx->hp_a[i])
        {
            cudaFree(ctx->hp_a[i]);
            cudaFree(ctx->hp_b[i]);
            cudaFree(ctx->hp_o[i]);
        }
        else
        {
            CU_TRY(cudaEventCreateWithFlags(&ctx->hp_in[i], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&ctx->hp_comp[i], cudaEventDisableTiming));
            CU_TRY(cudaEventCreateWithFlags(&ctx->hp_out[i], cudaEventDisableTiming));
        }
        CU_TRY(cudaMalloc((void **)&ctx->hp_a[i], words_per_slot * sizeof(u64)));
        CU_TRY(cudaMalloc((void **)&ctx->hp_b[i], words_per_slot * sizeof(u64)));
        CU_TRY(cudaMalloc((void **)&ctx->hp_o[i], words_per_slot * sizeof(u64)));
    }
    ctx->hp_words = words_per_slot;
    return 0;
}


// ---------------------------------------------------------------------------------------------------------
// Packed PCIe transfers for the host-buffer entry points (OPT-IN, see level_packs).  A canonical residue of a level
// whose primes are all below 2^48 carries at most 6 significant bytes, and the end-to-end rate of
// multiply+relinearize is set by PCIe (1 MiB in + 0.5 MiB out per op against ~7 us of GPU time), so the words can
// cross the link as 6 bytes each: host threads pack into pinned staging while the previous chunk is in flight, the
// GPU expands after landing (and packs the result before it leaves).  Bit-exact: every word is checked to fit
// before it is narrowed.
// ---------------------------------------------------------------------------------------------------------
static const u64 PACK_MASK = 0x0000FFFFFFFFFFFFULL;

// 4 words <- 3 u64 (24 bytes)
__global__ void unpack48_kernel(const u64 *packed, u64 *out, long long groups)
{
    const long long g = GLOBAL_IDX();
    if (g >= groups)
        return;
    const u64 a = packed[3 * g], b = packed[3 * g + 1], c = packed[3 * g + 2];
    out[4 * g] = a & PACK_MASK;
    out[4 * g + 1] = ((a >> 48) | (b << 16)) & PACK_MASK;
    out[4 * g + 2] = ((b >> 32) | (c << 32)) & PACK_MASK;
    out[4 * g + 3] = c >> 16;
}
__global__ void pack48_kernel(const u64 *in, u64 *packed, long long groups)
{
    const long long g = GLOBAL_IDX();
    if (g >= groups)
        return;
    const u64 w0 = in[4 * g], w1 = in[4 * g + 1], w2 = in[4 * g + 2], w3 = in[4 * g + 3];
    packed[3 * g] = w0 | (w1 << 48);
    packed[3 * g + 1] = (w1 >> 16) | (w2 << 32);
    packed[3 * g + 2] = (w2 >> 32) | (w3 << 16);
}

// minimal fork-join pool (the packing loops are pure streaming work; 8-16 threads saturate what PCIe can take)
struct HostPool
{
    std::vector<std::thread> th;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::function<void(int, int)> task;
    long long generation = 0;
    int pending = 0;
    bool stop = false;
    int nth = 1;
    explicit HostPool(int n) : nth(n < 1 ? 1 : n)
    {
        for (int i = 1; i < nth; i++)
            th.emplace_back([this, i] { loop(i); });
    }
    ~HostPool()
    {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv_work.notify_all();
        for (auto &t : th)
            t.join();
    }
    void loop(int id)
    {
        long long seen = 0;
        for (;;)
        {
            std::function<void(int, int)> fn;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv_work.wait(lk, [&] { return stop || generation != seen; });
                if (stop)
                    return;
                seen = generation;
                fn = task;
            }
            fn(id, nth);
            {
                std::lock_guard<std::mutex> lk(mu);
                if (--pending == 0)
                    cv_done.notify_one();
            }
        }
    }
    void run(const std::function<void(int, int)> &fn)
    {
        if (nth == 1)
        {
            fn(0, 1);
            return;
        }
        {
            std::lock_guard<std::mutex> lk(mu);
            task = fn;
            pending = nth - 1;
            generation++;
        }
        cv_work.notify_all();
        fn(0, nth);
        std::unique_lock<std::mutex> lk(mu);
        cv_done.wait(lk, [&] { return pending == 0; });
    }
};

static void host_pool_destroy(b200_ctx *ctx)
{
    delete ctx->pool;
    ctx->pool = nullptr;
}
static HostPool *host_pool(b200_ctx *ctx)
{
    if (!ctx->pool)
    {
        int n = 0;
        if (const char *e = getenv("B200_HOST_THREADS"))
            n = atoi(e);
        if (n <= 0)
        {
            cpu_set_t set;
            CPU_ZERO(&set);
            int avail = sched_getaffinity(0, sizeof(set), &set) == 0 ? CPU_COUNT(&set) : (int)std::thread::hardware_concurrency();
            n = std::max(1, std::min(16, avail / 2));
        }
        ctx->pool = new HostPool(n);
    }
    return ctx->pool;
}

// src[words] -> dst[6*words (+2 slack)]; returns the OR of all words (to verify that they fit 48 bits)
static u64 cpu_pack48(HostPool *pool, const u64 *src, uint8_t *dst, size_t words)
{
    std::vector<u64> ors((size_t)pool->nth, 0);
    pool->run([&](int id, int nth) {
        const size_t lo = words * (size_t)id / (size_t)nth, hi = words * (size_t)(id + 1) / (size_t)nth;
        if (lo >= hi)
            return;
        u64 m = 0;
        uint8_t *d = dst + 6 * lo;
        for (size_t i = lo; i + 1 < hi; i++, d += 6)
        {
            const u64 w = src[i];
            m |= w;
            std::memcpy(d, &w, 8); // the two spill bytes are overwritten by the next word of this range
        }
        const u64 w = src[hi - 1];
        m |= w;
        std::memcpy(d, &w, 6);
        ors[(size_t)id] = m;
    });
    u64 m = 0;
    for (u64 x : ors)
        m |= x;
    return m;
}
static void cpu_unpack48(HostPool *pool, const uint8_t *src, u64 *dst, size_t words)
{
    pool->run([&](int id, int nth) {
        const size_t lo = words * (size_t)id / (size_t)nth, hi = words * (size_t)(id + 1) / (size_t)nth;
        const uint8_t *s = src + 6 * lo;
        for (size_t i = lo; i < hi; i++, s += 6)
        {
            u64 w;
            std::memcpy(&w, s, 8); // staging buffers carry 8 bytes of slack
            dst[i] = w & PACK_MASK;
        }
    });
}

static bool level_packs(const b200_ctx *ctx, int level)
{
    // Opt-in (B200_HOST_PACK=1).  Narrowing on the CPU costs more host memory traffic (~5 GiB per 1024 ops instead of 1.5)
    // than PCIe saves, so the default is the plain pipeline.
    const char *e = getenv("B200_HOST_PACK");
    if (!e || atoi(e) == 0 || (ctx->n & 3))
        return false;
    const auto &Lh = ctx->host->levels[level];
    for (int idx : Lh.q_idx)
        if (ctx->host->primes[idx].mod.p >> 48)
            return false;
    return true;
}

static int pack_ring(b200_ctx *ctx, size_t words_per_slot)
{
    if (ctx->pk_words >= words_per_slot)
        return 0;
    const size_t bytes = words_per_slot * 6 + 16;
    for (int i = 0; i < b200_ctx::NBUF; i++)
    {
        if (ctx->hst_a[i])
        {
            cudaFreeHost(ctx->hst_a[i]);
            cudaFreeHost(ctx->hst_b[i]);
            cudaFreeHost(ctx->hst_o[i]);
            cudaFree(ctx->dpk_a[i]);
            cudaFree(ctx->dpk_b[i]);
            cudaFree(ctx->dpk_o[i]);
        }
        CU_TRY(cudaMallocHost((void **)&ctx->hst_a[i], bytes));
        CU_TRY(cudaMallocHost((void **)&ctx->hst_b[i], bytes));
        CU_TRY(cudaMallocHost((void **)&ctx->hst_o[i], bytes));
        CU_TRY(cudaMalloc((void **)&ctx->dpk_a[i], bytes));
        CU_TRY(cudaMalloc((void **)&ctx->dpk_b[i], bytes));
        CU_TRY(cudaMalloc((void **)&ctx->dpk_o[i], bytes));
    }
    ctx->pk_words = words_per_slot;
    return 0;
}

// multiply+relinearize over host buffers with packed transfers (see above); same contract as the plain pipeline
static int multiply_relin_host_packed(b200_ctx *ctx, int level, const u64 *a_host, const u64 *b_host, const u64 *relin_key_dev,
                                      u64 *out_host, uint64_t batch, long long chunk, size_t ct_words)
{
    int rc = 0;
    if ((rc = host_ring(ctx, (size_t)chunk * ct_words)) || (rc = pack_ring(ctx, (size_t)chunk * ct_words)))
        return rc;
    HostPool *pool = host_pool(ctx);
    const int NBUF = b200_ctx::NBUF, LAG = NBUF - 1;
    std::vector<uint64_t> offs;
    for (uint64_t off = 0; off < batch; off += (uint64_t)chunk)
        offs.push_back(off);
    const int iters = (int)offs.size();
    auto drain = [&](int j) { // bring the result of iteration j home
        const int sl = j % NBUF;
        const size_t words = (size_t)std::min<uint64_t>((uint64_t)chunk, batch - offs[j]) * ct_words;
        cudaEventSynchronize(ctx->hp_out[sl]);
        cpu_unpack48(pool, ctx->hst_o[sl], out_host + offs[j] * ct_words, words);
    };
    u64 ormask = 0;
    for (int it = 0; it < iters && rc == 0; it++)
    {
        const int sl = it % NBUF;
        const uint64_t off = offs[it];
        const long long cnt = (long long)std::min<uint64_t>((uint64_t)chunk, batch - off);
        const size_t words = (size_t)cnt * ct_words, pbytes = words * 6, groups = words / 4;
        if (it >= NBUF)
            cudaEventSynchronize(ctx->hp_in[sl]); // the staging buffers of this slot have left the host
        ormask |= cpu_pack48(pool, a_host + off * ct_words, ctx->hst_a[sl], words);
        ormask |= cpu_pack48(pool, b_host + off * ct_words, ctx->hst_b[sl], words);
        if (ormask >> 48)
        {
            rc = fail(B200_E_INVALID, "ciphertext word does not fit the residue width of this level");
            break;
        }
        if (it >= NBUF)
            cudaStreamWaitEvent(ctx->s_h2d, ctx->hp_out[sl], 0); // device slot free once its previous output left
        cudaMemcpyAsync(ctx->dpk_a[sl], ctx->hst_a[sl], pbytes, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaMemcpyAsync(ctx->dpk_b[sl], ctx->hst_b[sl], pbytes, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaEventRecord(ctx->hp_in[sl], ctx->s_h2d);
        cudaStreamWaitEvent(ctx->s_comp, ctx->hp_in[sl], 0);
        B200_LAUNCH(unpack48_kernel, blocks_for((long long)groups, 256), 256, 0, ctx->s_comp, (const u64 *)ctx->dpk_a[sl], ctx->hp_a[sl],
                    (long long)groups);
        B200_LAUNCH(unpack48_kernel, blocks_for((long long)groups, 256), 256, 0, ctx->s_comp, (const u64 *)ctx->dpk_b[sl], ctx->hp_b[sl],
                    (long long)groups);
        ctx->launches += 2;
        rc = b200_multiply_relin(ctx, level, (const uint64_t *)ctx->hp_a[sl], (const uint64_t *)ctx->hp_b[sl],
                                 (const uint64_t *)relin_key_dev, (uint64_t *)ctx->hp_o[sl], (uint64_t)cnt, ctx->s_comp);
        B200_LAUNCH(pack48_kernel, blocks_for((long long)groups, 256), 256, 0, ctx->s_comp, (const u64 *)ctx->hp_o[sl], ctx->dpk_o[sl],
                    (long long)groups);
        ctx->launches++;
        cudaEventRecord(ctx->hp_comp[sl], ctx->s_comp);
        cudaStreamWaitEvent(ctx->s_d2h, ctx->hp_comp[sl], 0);
        cudaMemcpyAsync(ctx->hst_o[sl], ctx->dpk_o[sl], pbytes, cudaMemcpyDeviceToHost, ctx->s_d2h);
        cudaEventRecord(ctx->hp_out[sl], ctx->s_d2h);
        if (it >= LAG)
            drain(it - LAG);
    }
    cudaError_t e1 = cudaStreamSynchronize(ctx->s_h2d);
    cudaError_t e2 = cudaStreamSynchronize(ctx->s_comp);
    cudaError_t e3 = cudaStreamSynchronize(ctx->s_d2h);
    if (rc)
        return rc;
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)
        return fail(B200_E_CUDA, std::string("host pipeline: ") +
                                     cudaGetErrorString(e1 != cudaSuccess ? e1 : (e2 != cudaSuccess ? e2 : e3)));
    for (int j = std::max(0, iters - LAG); j < iters; j++)
        drain(j);
    return 0;
}

int b200_multiply_relin_host(b200_ctx *ctx, int level, const uint64_t *a_host, const uint64_t *b_host,
                             const uint64_t *relin_key_dev, uint64_t *out_host, uint64_t batch)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!a_host || !b_host || !relin_key_dev || !out_host)
        return fail(B200_E_NULL, "null pointer");
    if (batch == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> lk(ctx->hp_mu);
    const long long n = (long long)ctx->n;
    const int k = ctx->levels[level].k;
    const size_t ct_words = (size_t)2 * k * n;
    const char *env = getenv("B200_HOST_CHUNK");
    long long chunk = env ? atoll(env) : 64;
    if (chunk < 1)
        chunk = 1;
    if ((uint64_t)chunk > batch)
        chunk = (long long)batch;
    if (level_packs(ctx, level))
        return multiply_relin_host_packed(ctx, level, (const u64 *)a_host, (const u64 *)b_host, (const u64 *)relin_key_dev,
                                          (u64 *)out_host, batch, chunk, ct_words);
    if ((rc = host_ring(ctx, (size_t)chunk * ct_words)))
        return rc;
    const int NBUF = b200_ctx::NBUF;
    int it = 0;
    for (uint64_t off = 0; off < batch && rc == 0; off += (uint64_t)chunk, it++)
    {
        const int sl = it % NBUF;
        const long long cnt = (long long)std::min<uint64_t>((uint64_t)chunk, batch - off);
        const size_t bytes = (size_t)cnt * ct_words * sizeof(u64);
        if (it >= NBUF)
            cudaStreamWaitEvent(ctx->s_h2d, ctx->hp_out[sl], 0); // slot free once its previous output left
        cudaMemcpyAsync(ctx->hp_a[sl], a_host + off * ct_words, bytes, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaMemcpyAsync(ctx->hp_b[sl], b_host + off * ct_words, bytes, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaEventRecord(ctx->hp_in[sl], ctx->s_h2d);
        cudaStreamWaitEvent(ctx->s_comp, ctx->hp_in[sl], 0);
        rc = b200_multiply_relin(ctx, level, (const uint64_t *)ctx->hp_a[sl], (const uint64_t *)ctx->hp_b[sl], relin_key_dev,
                                 (uint64_t *)ctx->hp_o[sl], (uint64_t)cnt, ctx->s_comp);
        cudaEventRecord(ctx->hp_comp[sl], ctx->s_comp);
        cudaStreamWaitEvent(ctx->s_d2h, ctx->hp_comp[sl], 0);
        cudaMemcpyAsync(out_host + off * ct_words, ctx->hp_o[sl], bytes, cudaMemcpyDeviceToHost, ctx->s_d2h);
        cudaEventRecord(ctx->hp_out[sl], ctx->s_d2h);
    }
    cudaError_t e1 = cudaStreamSynchronize(ctx->s_h2d);
    cudaError_t e2 = cudaStreamSynchronize(ctx->s_comp);
    cudaError_t e3 = cudaStreamSynchronize(ctx->s_d2h);
    if (rc)
        return rc;
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)
        return fail(B200_E_CUDA, std::string("host pipeline: ") +
                                     cudaGetErrorString(e1 != cudaSuccess ? e1 : (e2 != cudaSuccess ? e2 : e3)));
    return 0;
}

int b200_ntt_roundtrip_host(b200_ctx *ctx, int level, const uint64_t *in_host, uint64_t *out_host, uint64_t items)
{
    int rc = check_level(ctx, level);
    if (rc)
        return rc;
    if (!in_host || !out_host)
        return fail(B200_E_NULL, "null pointer");
    if (items == 0)
        return 0;
    CU_TRY(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> lk(ctx->hp_mu);
    const size_t words = (size_t)ctx->levels[level].k * ctx->n;
    long long chunk = 512;
    if ((uint64_t)chunk > items)
        chunk = (long long)items;
    if ((rc = host_ring(ctx, (size_t)chunk * words)))
        return rc;
    const int NBUF = b200_ctx::NBUF;
    int it = 0;
    for (uint64_t off = 0; off < items && rc == 0; off += (uint64_t)chunk, it++)
    {
        const int sl = it % NBUF;
        const long long cnt = (long long)std::min<uint64_t>((uint64_t)chunk, items - off);
        const size_t bytes = (size_t)cnt * words * sizeof(u64);
        if (it >= NBUF)
            cudaStreamWaitEvent(ctx->s_h2d, ctx->hp_out[sl], 0);
        cudaMemcpyAsync(ctx->hp_a[sl], in_host + off * words, bytes, cudaMemcpyHostToDevice, ctx->s_h2d);
        cudaEventRecord(ctx->hp_in[sl], ctx->s_h2d);
        cudaStreamWaitEvent(ctx->s_comp, ctx->hp_in[sl], 0);
        rc = b200_ntt_forward(ctx, level, (uint64_t *)ctx->hp_a[sl], (uint64_t)cnt, ctx->s_comp);
        if (!rc)
            rc = b200_ntt_inverse(ctx, level, (uint64_t *)ctx->hp_a[sl], (uint64_t)cnt, ctx->s_comp);
        cudaEventRecord(ctx->hp_comp[sl], ctx->s_comp);
        cudaStreamWaitEvent(ctx->s_d2h, ctx->hp_comp[sl], 0);
        cudaMemcpyAsync(out_host + off * words, ctx->hp_a[sl], bytes, cudaMemcpyDeviceToHost, ctx->s_d2h);
        cudaEventRecord(ctx->hp_out[sl], ctx->s_d2h);
    }
    cudaError_t e1 = cudaStreamSynchronize(ctx->s_h2d);
    cudaError_t e2 = cudaStreamSynchronize(ctx->s_comp);
    cudaError_t e3 = cudaStreamSynchronize(ctx->s_d2h);
    if (rc)
        return rc;
    if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)
        return fail(B200_E_CUDA, "host pipeline failed");
    return 0;
}

} // extern "C"
