// tools/ubench.cu — developer microbenchmarks (not part of the product): integer pipe rates on sm_90a that
// decide the NTT butterfly design. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench ubench.cu
#include <cstdio>
#include <cuda_runtime.h>
typedef unsigned long long u64;
typedef unsigned int u32;
#define ITERS 4096

__device__ __forceinline__ u64 madwide(u32 a, u32 b, u64 c)
{
    u64 d;
    asm volatile("mad.wide.u32 %0, %1, %2, %3;" : "=l"(d) : "r"(a), "r"(b), "l"(c));
    return d;
}
__device__ __forceinline__ u32 madlo(u32 a, u32 b, u32 c)
{
    u32 d;
    asm volatile("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

template <int MODE>
__global__ void k_pipe(u64 *out, u32 a0, u32 b0)
{
    u64 acc[8];
    u32 r[8];
    u32 a = a0 + threadIdx.x, b = b0;
#pragma unroll
    for (int i = 0; i < 8; i++)
    {
        acc[i] = i + threadIdx.x;
        r[i] = i * 3 + threadIdx.x;
    }
    for (int it = 0; it < ITERS; it++)
    {
#pragma unroll
        for (int i = 0; i < 8; i++)
        {
            if (MODE == 0)
                acc[i] = madwide(a, (u32)acc[i], acc[i]); // IMAD.WIDE.U32
            else if (MODE == 1)
                r[i] = madlo(a, r[i], b);                  // IMAD
            else if (MODE == 2)
            {
                asm volatile("add.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(a)); // IADD3
            }
            else if (MODE == 3)
            { // 1 wide + 1 add (dual pipe)
                acc[i] = madwide(a, (u32)acc[i], acc[i]);
                asm volatile("add.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(a));
            }
            else if (MODE == 4)
            { // 1 wide + 2 adds
                acc[i] = madwide(a, (u32)acc[i], acc[i]);
                asm volatile("add.u32 %0, %0, %1;" : "+r"(r[i]) : "r"(a));
                asm volatile("xor.b32 %0, %0, %1;" : "+r"(r[i]) : "r"(b));
            }
            else if (MODE == 5)
            { // 1 wide + 1 lo
                acc[i] = madwide(a, (u32)acc[i], acc[i]);
                r[i] = madlo(a, r[i], b);
            }
        }
    }
    u64 s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        s += acc[i] + r[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---- butterfly variants, register resident ----
__device__ __forceinline__ u64 shoup_lazy(u64 y, u64 w, u64 wq, u64 q)
{
    u64 Q = __umul64hi(wq, y);
    return w * y - Q * q;
}
// hand-limb lazy butterfly: X' = X + W*Y + Q*nq ; Y' = 2X + 2p - X'   (nq = -q mod 2^64), approximate quotient (drops lo*lo)
__device__ __forceinline__ void bf_limb(u64 &X, u64 &Y, u64 w, u64 wq, u64 nq, u64 twop2 /*unused*/, u64 twop)
{
    u32 yl = (u32)Y, yh = (u32)(Y >> 32), ql = (u32)wq, qh = (u32)(wq >> 32);
    // Q ~ hi64(wq*Y) without the lo*lo term
    u64 t1 = madwide(qh, yl, 0);
    u64 t2 = madwide(ql, yh, (u64)(u32)t1);
    u64 hs = (t1 >> 32) + (t2 >> 32);
    u64 Q = madwide(qh, yh, hs);
    u32 Ql = (u32)Q, Qh = (u32)(Q >> 32);
    u32 wl = (u32)w, wh = (u32)(w >> 32), nl = (u32)nq, nh = (u32)(nq >> 32);
    u64 acc = madwide(wl, yl, X);
    acc = madwide(Ql, nl, acc);
    u32 hi = (u32)(acc >> 32);
    hi = madlo(wl, yh, hi);
    hi = madlo(wh, yl, hi);
    hi = madlo(Ql, nh, hi);
    hi = madlo(Qh, nl, hi);
    u64 Xn = ((u64)hi << 32) | (u32)acc;
    Y = X + X + twop - Xn;
    X = Xn;
}

template <int MODE>
__global__ void k_bf(u64 *out, const u64 *tw, u64 p)
{
    u64 x[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
        x[i] = out[(blockIdx.x * blockDim.x + threadIdx.x) * 8 + i];
    const u64 twop = p << 1, nq = 0 - p;
    u64 w = tw[threadIdx.x & 7], wq = tw[8 + (threadIdx.x & 7)];
    for (int it = 0; it < ITERS / 8; it++)
    {
#pragma unroll
        for (int s = 0; s < 3; s++)
        {
            const int half = 4 >> s;
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (!(j & half))
                {
                    if (MODE == 0)
                    { // Harvey, compiler
                        u64 X = x[j];
                        X = X >= twop ? X - twop : X;
                        u64 T = shoup_lazy(x[j + half], w, wq, p);
                        x[j] = X + T;
                        x[j + half] = X - T + twop;
                    }
                    else if (MODE == 1)
                    { // lazy, compiler
                        u64 X = x[j];
                        u64 T = shoup_lazy(x[j + half], w, wq, p);
                        x[j] = X + T;
                        x[j + half] = X - T + twop;
                    }
                    else
                        bf_limb(x[j], x[j + half], w, wq, nq, 0, twop);
                }
            w += wq; // keep the twiddle changing so nothing is hoisted
        }
    }
    u64 s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        s ^= x[i];
    out[(blockIdx.x * blockDim.x + threadIdx.x) * 8] = s;
}

// ---- FP64 pipe ----
template <int MODE>
__global__ void k_fp(double *out, double a0, double b0)
{
    double acc[8];
    double a = a0 + threadIdx.x, b = b0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        acc[i] = i + threadIdx.x;
    for (int it = 0; it < ITERS; it++)
    {
#pragma unroll
        for (int i = 0; i < 8; i++)
        {
            if (MODE == 0)
                acc[i] = fma(acc[i], a, b);
            else if (MODE == 1)
                acc[i] = acc[i] * a;
            else if (MODE == 2)
                acc[i] = acc[i] + a;
            else if (MODE == 3)
                asm volatile("cvt.rni.f64.f64 %0, %0;" : "+d"(acc[i]));
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// FP64 butterfly: signed lazy representation, values are integer-valued doubles.
// T = y*w - rint(y*wp)*p  (wp = w/p), exact via FMA splitting; X' = X + T, Y' = X - T.
__device__ __forceinline__ void bf_fp(double &X, double &Y, double w, double wp, double p)
{
    const double MAGIC = 6755399441055744.0; // 1.5 * 2^52
    double h = Y * w;
    double l = fma(Y, w, -h);
    double q = fma(Y, wp, MAGIC) - MAGIC;
    double r = fma(-q, p, h) + l;
    Y = X - r;
    X = X + r;
}
// variant: q = rint(h * pinv) with the rounding done by FRND (cvt.rni.f64.f64) instead of the magic add/sub
__device__ __forceinline__ void bf_fp_rnd(double &X, double &Y, double w, double pinv, double p)
{
    double h = Y * w;
    double l = fma(Y, w, -h);
    double q = h * pinv;
    asm("cvt.rni.f64.f64 %0, %0;" : "+d"(q));
    double r = fma(-q, p, h) + l;
    Y = X - r;
    X = X + r;
}
template <int MODE>
__global__ void k_bf_fp(double *out, const double *tw, double p)
{
    double x[8];
#pragma unroll
    for (int i = 0; i < 8; i++)
        x[i] = out[(blockIdx.x * blockDim.x + threadIdx.x) * 8 + i];
    double w = tw[threadIdx.x & 7], wp = w / p;
    for (int it = 0; it < ITERS / 8; it++)
    {
#pragma unroll
        for (int s = 0; s < 3; s++)
        {
            const int half = 4 >> s;
#pragma unroll
            for (int j = 0; j < 8; j++)
                if (!(j & half))
                {
                    if (MODE == 2)
                        bf_fp_rnd(x[j], x[j + half], w, 1.0 / p, p);
                    else
                        bf_fp(x[j], x[j + half], w, wp, p);
                }
            w = w * 0.999 + 1.0;
            wp = w / p;
        }
        if (MODE == 1)
        { // renormalise every 3 stages (keeps magnitudes bounded for the benchmark)
#pragma unroll
            for (int j = 0; j < 8; j++)
            {
                double q = fma(x[j], 1.0 / p, 6755399441055744.0) - 6755399441055744.0;
                x[j] = fma(-q, p, x[j]);
            }
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 8; i++)
        s += x[i];
    out[(blockIdx.x * blockDim.x + threadIdx.x) * 8] = s;
}

// mixed: half the warps do FP64 butterflies, the other half integer limb butterflies (both pipes busy)
__global__ void k_bf_mixed(u64 *out, const u64 *tw, u64 p)
{
    const int warp = threadIdx.x >> 5;
    if (warp & 1)
    {
        double x[8];
#pragma unroll
        for (int i = 0; i < 8; i++)
            x[i] = (double)(out[(blockIdx.x * blockDim.x + threadIdx.x) * 8 + i] & 0xfffffffffffULL);
        double pd = (double)p;
        double w = (double)(tw[threadIdx.x & 7] & 0xfffffffffffULL), wp = w / pd;
        for (int it = 0; it < ITERS / 8; it++)
        {
#pragma unroll
            for (int s = 0; s < 3; s++)
            {
                const int half = 4 >> s;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (!(j & half))
                        bf_fp(x[j], x[j + half], w, wp, pd);
                w = w * 0.999 + 1.0;
                wp = w / pd;
            }
#pragma unroll
            for (int j = 0; j < 8; j++)
            {
                double q = fma(x[j], 1.0 / pd, 6755399441055744.0) - 6755399441055744.0;
                x[j] = fma(-q, pd, x[j]);
            }
        }
        double s = 0;
#pragma unroll
        for (int i = 0; i < 8; i++)
            s += x[i];
        out[(blockIdx.x * blockDim.x + threadIdx.x) * 8] = (u64)(long long)s;
    }
    else
    {
        u64 x[8];
#pragma unroll
        for (int i = 0; i < 8; i++)
            x[i] = out[(blockIdx.x * blockDim.x + threadIdx.x) * 8 + i];
        const u64 twop = p << 1, nq = 0 - p;
        u64 w = tw[threadIdx.x & 7], wq = tw[8 + (threadIdx.x & 7)];
        for (int it = 0; it < ITERS / 8; it++)
        {
#pragma unroll
            for (int s = 0; s < 3; s++)
            {
                const int half = 4 >> s;
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (!(j & half))
                        bf_limb(x[j], x[j + half], w, wq, nq, 0, twop);
                w += wq;
            }
        }
        u64 s = 0;
#pragma unroll
        for (int i = 0; i < 8; i++)
            s ^= x[i];
        out[(blockIdx.x * blockDim.x + threadIdx.x) * 8] = s;
    }
}

// ---- distributed shared memory (DSMEM) across a 4-CTA cluster: the hand-off of mul_cluster.cu ----
// Every CTA holds one padded n = 8192 polynomial (the NTT kernels' shared-memory footprint, 3 CTAs/SM); each pass every thread
// touches its 32 words once, in the CTA `pass % 3 + 1` ranks ahead (MODE 0: local ld.shared, 1: remote ld.shared::cluster,
// 2: remote st.shared::cluster).
#define DS_N 8192
#define DS_WORDS (DS_N + DS_N / 16)
template <int MODE>
__global__ void __launch_bounds__(256, 3) k_dsmem(double *out, int passes)
{
    extern __shared__ double ds[];
    unsigned rank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    for (int e = threadIdx.x; e < DS_WORDS; e += 256)
        ds[e] = e + rank;
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    double acc = 0.0;
    for (int ps = 0; ps < passes; ps++)
    {
        const unsigned peer = MODE == 0 ? rank : (rank + 1 + ps % 3) & 3;
#pragma unroll 8
        for (int it = 0; it < DS_N / 256; it++)
        {
            const int e = threadIdx.x + it * 256;
            const unsigned la = (unsigned)__cvta_generic_to_shared(ds + e + (e >> 4));
            unsigned ra;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(peer));
            if (MODE == 2)
                asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(acc + e) : "memory");
            else
            {
                double v;
                asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra) : "memory");
                acc += v;
            }
        }
    }
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <int MODE>
static float dsmem_run(double *out, int clusters, int passes)
{
    const size_t smem = DS_WORDS * sizeof(double);
    cudaFuncSetAttribute(k_dsmem<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 4;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(4 * clusters);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = smem;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    if (MODE == 0)
    {
        int active = 0;
        cudaOccupancyMaxActiveClusters(&active, k_dsmem<MODE>, &cfg);
        printf("dsmem: %d active 4-CTA clusters (%d CTAs), %zu B shared memory per CTA\n", active, 4 * active, smem);
    }
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    cudaLaunchKernelEx(&cfg, k_dsmem<MODE>, out, passes);
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    cudaLaunchKernelEx(&cfg, k_dsmem<MODE>, out, passes);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        printf("dsmem: %s\n", cudaGetErrorString(e));
    return ms;
}

template <class F>
float timeit(F f)
{
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    f();
    cudaDeviceSynchronize();
    cudaEventRecord(a);
    f();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    return ms;
}

int main()
{
    cudaDeviceProp pr;
    cudaGetDeviceProperties(&pr, 0);
    int sms = pr.multiProcessorCount;
    int khz;
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("SMs %d, clock attr %d kHz\n", sms, khz);
    u64 *out, *tw;
    const int blocks = sms * 8, threads = 256;
    cudaMalloc(&out, (size_t)blocks * threads * 8 * sizeof(u64));
    cudaMemset(out, 1, (size_t)blocks * threads * 8 * sizeof(u64));
    cudaMalloc(&tw, 64 * sizeof(u64));
    cudaMemset(tw, 3, 64 * sizeof(u64));
    const char *names[] = { "IMAD.WIDE.U32", "IMAD(lo)", "IADD", "WIDE+ADD", "WIDE+2ALU", "WIDE+IMADlo" };
    const double per_iter[] = { 8, 8, 8, 16, 24, 16 };
#define RUNP(M)                                                                                                        \
    {                                                                                                                  \
        float ms = timeit([&] { k_pipe<M><<<blocks, threads>>>(out, 12345u, 777u); });                                 \
        double ops = (double)blocks * threads * ITERS * per_iter[M];                                                   \
        printf("%-14s %8.3f ms  %8.2f Tlane-instr/s  (%.1f lane-instr/clk/SM @1.9GHz)\n", names[M], ms,              \
               ops / ms / 1e9, ops / ms / 1e3 / 1.9e6 / sms / 1e3 * 1e3 / 1e3);                                        \
    }
    RUNP(0) RUNP(1) RUNP(2) RUNP(3) RUNP(4) RUNP(5)
    const char *bn[] = { "bf harvey(compiler)", "bf lazy(compiler)", "bf limb(hand)" };
#define RUNB(M)                                                                                                        \
    {                                                                                                                  \
        float ms = timeit([&] { k_bf<M><<<blocks, threads>>>(out, tw, 0x7fffffd8001ULL); });                           \
        double bfs = (double)blocks * threads * (ITERS / 8) * 12;                                                      \
        printf("%-20s %8.3f ms  %8.2f G butterflies/s -> %.2f M NTT(8192)/s\n", bn[M], ms, bfs / ms / 1e6,             \
               bfs / ms / 1e3 / 53248.0);                                                                              \
    }
    RUNB(0) RUNB(1) RUNB(2)
    const char *fn[] = { "DFMA", "DMUL", "DADD", "FRND.F64" };
#define RUNF(M)                                                                                                        \
    {                                                                                                                  \
        float ms = timeit([&] { k_fp<M><<<blocks, threads>>>((double *)out, 1.0000001, 0.5); });                       \
        double ops = (double)blocks * threads * ITERS * 8;                                                             \
        printf("%-14s %8.3f ms  %8.2f Tlane-instr/s (%.1f lanes/clk/SM @1.9GHz)\n", fn[M], ms, ops / ms / 1e9,       \
               ops / ms / 1e3 / 1.9e9 / sms * 1e3);                                                                    \
    }
    RUNF(0) RUNF(1) RUNF(2) RUNF(3)
    cudaMemset(out, 0, (size_t)blocks * threads * 8 * sizeof(u64));
    const char *bfn[] = { "bf fp64 (no renorm)", "bf fp64 (+renorm/3)", "bf fp64 (FRND quotient)" };
#define RUNBF(M)                                                                                                       \
    {                                                                                                                  \
        float ms = timeit([&] { k_bf_fp<M><<<blocks, threads>>>((double *)out, (const double *)tw, 8796092858369.0); }); \
        double bfs = (double)blocks * threads * (ITERS / 8) * 12;                                                      \
        printf("%-20s %8.3f ms  %8.2f G butterflies/s -> %.2f M NTT(8192)/s\n", bfn[M], ms, bfs / ms / 1e6,          \
               bfs / ms / 1e3 / 53248.0);                                                                              \
    }
    RUNBF(0) RUNBF(1) RUNBF(2)
    {
        float ms = timeit([&] { k_bf_mixed<<<blocks, threads>>>(out, tw, 0x7fffffd8001ULL); });
        double bfs = (double)blocks * threads * (ITERS / 8) * 12;
        printf("%-20s %8.3f ms  %8.2f G butterflies/s -> %.2f M NTT(8192)/s\n", "bf mixed int+fp64", ms, bfs / ms / 1e6,
               bfs / ms / 1e3 / 53248.0);
    }
    {
        // 3 CTAs per SM, whole clusters: 99 clusters on 132 SMs
        const int clusters = sms * 3 / 4, passes = 256;
        double *dout;
        cudaMalloc(&dout, (size_t)clusters * 4 * 256 * sizeof(double));
        const char *dn[] = { "dsmem local ld", "dsmem remote ld", "dsmem remote st" };
        float ms[3] = { dsmem_run<0>(dout, clusters, passes), dsmem_run<1>(dout, clusters, passes), dsmem_run<2>(dout, clusters, passes) };
        for (int m = 0; m < 3; m++)
        {
            const double bytes = (double)clusters * 4 * passes * DS_N * sizeof(double);
            printf("%-20s %8.3f ms  %8.2f TB/s aggregate\n", dn[m], ms[m], bytes / ms[m] / 1e9);
        }
        cudaFree(dout);
    }
    return 0;
}
