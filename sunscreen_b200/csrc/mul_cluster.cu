// mul_cluster.cu — BEHZ steps (3)-(5) of a size-2 x size-2 multiply in one kernel: forward NTTs, dyadic product and inverse
// NTTs of one residue row, with the NTT-form operands never leaving the chip.
//
// The product D = (a0 + a1 y)(b0 + b1 y) of residue row r needs the four NTT-form rows a0, a1, b0, b1 at once: 4 x 64 KiB at
// n = 8192, more than one CTA's shared memory but within a 4-CTA thread-block cluster's.  CTA c of the cluster transforms
// operand c in its own shared memory (NttFpStaticPass, VAR & 4096: no copy-out), the dyadic step reads the operands of each
// coefficient through distributed shared memory and writes D0, D1, D2 into the buffers of CTAs 0, 1, 2, which transform them
// back from there (VAR & 4096: no copy-in) and write D in coefficient form.  The separate path moves the same rows through
// HBM three more times (forward write, tensor read + write, inverse read: 126 of its 264 rows per item at k = 4, |Bsk| = 5).
//
// Every intermediate word equals the separate path's: the operands are brought to canonical form before the products (the
// words the forward transform would have written), the products are formed by the arithmetic of tensor_coeff_fp
// (bfv_body.cuh) and brought to canonical form again (the words the tensor kernel would have written), so the inverse
// transform starts from the inputs, and the magnitude bounds (renorm masks), it has today.
#include "mul_cluster.h"
#include "ntt_fp_body.cuh"
#include <cuda_runtime.h>

namespace
{
constexpr int NT = 256;        // threads per CTA: the n = 8192 throughput configuration (3 CTAs per SM)
constexpr int CLUSTER = 4;     // CTAs per cluster: operands a0, a1, b0, b1
constexpr int FWD_VAR = 2048 | 4096;     // warp-private passes, result stays in shared memory
constexpr int INV_VAR = 2048 | 1 | 4096; // + first 512 twiddles in shared memory, input already in shared memory

template <int LOGN>
constexpr size_t smem_bytes()
{
    return (size_t)(ntt_smem_words(1 << LOGN) + B200_NTT_TWS_ENTRIES) * sizeof(double);
}

__device__ __forceinline__ void cluster_sync()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__device__ __forceinline__ double to_canonical(double x, double p, double pinv) // any lazy value -> [0, p), as a double
{
    const double r = fp_renorm(x, p, pinv);
    return r < 0.0 ? B200_DADD(r, p) : r;
}

// this CTA's place: rank c in the cluster, residue row r, item.  Read afresh from the special registers at every use, so that
// nothing of it stays live (in registers) across the transforms, which use all 80 of them
struct Place
{
    unsigned c;
    int r;
    long long item;
};
__device__ __forceinline__ Place place(const NttJob &job)
{
    unsigned c, blk;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(c));
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(blk));
    const unsigned cl = blk / CLUSTER, items = (unsigned)job.items; // row-major: all items of row r adjacent (its twiddles stay hot)
    const unsigned r = cl / items;
    return Place{ c, (int)r, (long long)(cl - r * items) };
}

template <int LOGN>
__global__ void __launch_bounds__(NT, 3) mul_cluster_kernel(const NttJob job, const u64 *a, const u64 *b, const u64 *ext, u64 *D, int k)
{
    extern __shared__ u64 mc_sm[];
    constexpr int N = 1 << LOGN;
    double *smd = reinterpret_cast<double *>(mc_sm);
    const int tid = (int)threadIdx.x;
    const int R = job.slots;
    Place w = place(job);
    const NttPrimeFp PF = job.fprimes[job.slot_prime[w.r]];
    const NttPrime PI_ = job.primes[job.slot_prime[w.r]];
    // operand c (a0, a1, b0, b1): q rows straight from the ciphertexts, Bsk rows from the lifted rows
    const u64 *src = w.r < k ? (w.c < 2 ? a : b) + ((w.item * 2 + (w.c & 1)) * k + w.r) * N : ext + ((w.item * CLUSTER + w.c) * R + w.r) * N;
    NttFpStaticPass<LOGN, NT, true, 0, FWD_VAR>::run(job, PF, PI_, src, nullptr, smd, tid, w.item, w.r);
    cluster_sync(); // all four operands transformed
    w = place(job);

    // dyadic step: CTA c owns coefficients [c N/4, (c+1) N/4); each of them is read (4 CTAs) and written (CTAs 0-2) by one
    // thread only, so the in-place overwrite of a0, a1, b0 by D0, D1, D2 has no hazard
    {
        const double p = PF.p, pinv = PF.pinv;
        const unsigned base = (unsigned)__cvta_generic_to_shared(smd);
        unsigned rb[CLUSTER];
#pragma unroll
        for (int q = 0; q < CLUSTER; q++)
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb[q]) : "r"(base), "r"(q));
        // U coefficients per round: their 4 U remote loads are in flight together (n = 4096: one, a wider round makes ptxas spill)
        constexpr int QN = N / CLUSTER, U = LOGN >= 13 ? 4 : 1;
#pragma unroll 1
        for (int it = 0; it < QN / NT; it += U)
        {
            unsigned off[U];
            double x[U][CLUSTER];
#pragma unroll
            for (int u = 0; u < U; u++)
            {
                off[u] = (unsigned)ntt_pad((int)w.c * QN + tid + (it + u) * NT) * 8u;
#pragma unroll
                for (int q = 0; q < CLUSTER; q++)
                    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(x[u][q]) : "r"(rb[q] + off[u]) : "memory");
            }
#pragma unroll
            for (int u = 0; u < U; u++)
            {
#pragma unroll
                for (int q = 0; q < CLUSTER; q++)
                    x[u][q] = to_canonical(x[u][q], p, pinv);
                // tensor_coeff_fp's sums, term order included
                const double d0 = B200_DADD(0.0, fp_mulmod2(x[u][0], x[u][2], p, pinv));
                const double d1 = B200_DADD(B200_DADD(0.0, fp_mulmod2(x[u][0], x[u][3], p, pinv)), fp_mulmod2(x[u][1], x[u][2], p, pinv));
                const double d2 = B200_DADD(0.0, fp_mulmod2(x[u][1], x[u][3], p, pinv));
                asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(rb[0] + off[u]), "d"(to_canonical(d0, p, pinv)) : "memory");
                asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(rb[1] + off[u]), "d"(to_canonical(d1, p, pinv)) : "memory");
                asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(rb[2] + off[u]), "d"(to_canonical(d2, p, pinv)) : "memory");
            }
        }
    }
    cluster_sync(); // D0, D1, D2 in place; nothing reads CTA 3's shared memory after this
    w = place(job);
    if (w.c == CLUSTER - 1)
        return;
    u64 *dst = D + ((w.item * 3 + w.c) * R + w.r) * N;
    const NttPrimeFp PFi = job.fprimes[job.slot_prime[w.r]]; // (loaded again: nothing of the forward phase stays live)
    NttFpStaticPass<LOGN, NT, false, 0, INV_VAR>::run(job, PFi, job.primes[job.slot_prime[w.r]], nullptr, dst, smd, tid, w.item, w.r);
}

template <int LOGN>
cudaLaunchConfig_t config(long long clusters, cudaLaunchAttribute *at, cudaStream_t s)
{
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CLUSTER;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(clusters * CLUSTER));
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = smem_bytes<LOGN>();
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    return cfg;
}

template <int LOGN>
int setup(int *active)
{
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(mul_cluster_kernel<LOGN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<LOGN>())) != cudaSuccess)
        return (int)e;
    if ((e = cudaFuncSetAttribute(mul_cluster_kernel<LOGN>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)) != cudaSuccess)
        return (int)e;
    cudaLaunchAttribute at[1];
    const cudaLaunchConfig_t cfg = config<LOGN>(1, at, nullptr);
    return (int)cudaOccupancyMaxActiveClusters(active, mul_cluster_kernel<LOGN>, &cfg);
}
} // namespace

int b200_mul_cluster_setup(int logn, int *active)
{
    *active = 0;
    if (logn == 12)
        return setup<12>(active);
    if (logn == 13)
        return setup<13>(active);
    return 0;
}

int b200_mul_cluster(int logn, const NttJob &job, const u64 *a, const u64 *b, const u64 *ext, u64 *D, int k, void *stream)
{
    cudaLaunchAttribute at[1];
    const long long clusters = job.items * job.slots;
    if (logn == 12)
    {
        const cudaLaunchConfig_t cfg = config<12>(clusters, at, (cudaStream_t)stream);
        return (int)cudaLaunchKernelEx(&cfg, mul_cluster_kernel<12>, job, a, b, ext, D, k);
    }
    if (logn == 13)
    {
        const cudaLaunchConfig_t cfg = config<13>(clusters, at, (cudaStream_t)stream);
        return (int)cudaLaunchKernelEx(&cfg, mul_cluster_kernel<13>, job, a, b, ext, D, k);
    }
    return (int)cudaErrorInvalidValue;
}
