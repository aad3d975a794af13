// mul_cluster.cu — BEHZ steps (3)-(5) of a size-2 x size-2 multiply in one kernel: forward NTTs, dyadic product and inverse
// NTTs of one residue row, with the NTT-form operands never leaving the chip.
//
// The product D = (a0 + a1 y)(b0 + b1 y) of residue row r needs the four NTT-form rows a0, a1, b0, b1 at once: 4 x 64 KiB at
// n = 8192, more than one CTA's shared memory but within a 4-CTA thread-block cluster's.  CTA c of the cluster transforms
// operand c in its own shared memory (NttFpStaticPass with the HANDOFF option: no copy-out), the dyadic step reads the operands of each
// coefficient through distributed shared memory and writes D0, D1, D2 into the buffers of CTAs 0, 1, 2, which transform them
// back from there (HANDOFF: no copy-in) and write D in coefficient form.  The separate path moves the same rows through
// HBM three more times (forward write, tensor read + write, inverse read: 126 of its 264 rows per item at k = 4, |Bsk| = 5).
//
// Every intermediate word equals the separate path's: the operands are brought to canonical form before the products (the
// words the forward transform would have written), the products are formed by the arithmetic of tensor_coeff_fp
// (bfv_body.cuh) and brought to canonical form again (the words the tensor kernel would have written), so the inverse
// transform starts from the inputs, and the magnitude bounds (renorm masks), it has today.
//
// ks_cluster_kernel gives the key switch the same treatment: a k-CTA cluster per (item, key residue I) transforms the k digits
// mod p_I, forms the two inner products with the key and transforms them back, instead of the ks1 NTT, the MAC and the ks2 NTT
// of keyswitch_accumulate.  Its hand-offs are canonical as well: the digits before the products (the words of ks1), the accumulators
// (the words of ks2, formed by the FP64 branch of ksmac_tma_kernel), so every word and every renorm bound equals the separate path's.
#include "mul_cluster.h"
#include "ntt_fp_body.cuh"
#include <algorithm>
#include <cuda_runtime.h>

namespace
{
constexpr int NT = 256;        // threads per CTA: the n = 8192 throughput configuration (3 CTAs per SM)
constexpr int CLUSTER = 4;     // CTAs per cluster: operands a0, a1, b0, b1
using FwdOpt = NttFpOpt<false, false, true>;            // result stays in shared memory
using GalOpt = NttFpOpt<false, false, true, true>;      // the same, first pass gathers sigma_g(src)
using InvOpt = NttFpOpt<true, false, true>;             // first twiddles in shared memory, input already in shared memory

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
    NttFpStaticPass<LOGN, NT, true, 0, FwdOpt>::run(job, PF, PI_, src, nullptr, smd, tid);
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
    NttFpStaticPass<LOGN, NT, false, 0, InvOpt>::run(job, PFi, job.primes[job.slot_prime[w.r]], nullptr, dst, smd, tid);
}

// ks_cluster_kernel's place: rank J in the cluster (digit J), key residue I in [0, k] (k: the special prime), item.  Items
// outermost: the k + 1 clusters of an item run together, so its k digit rows come from HBM once and from L2 the other k times
struct KsPlace
{
    int J, I;
    long long item;
};
__device__ __forceinline__ KsPlace ks_place(int k)
{
    unsigned J, blk;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(J));
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(blk));
    const unsigned cl = blk / (unsigned)k, item = cl / (unsigned)(k + 1);
    return KsPlace{ (int)J, (int)(cl - item * (unsigned)(k + 1)), (long long)item };
}

// The key switch's NTT-domain half for one (item, key residue I): forward transforms of the k digits mod p_I, inner product
// with the key, inverse transforms of the two accumulators into ks2 [item][2][k + 1][n] (coefficient form, canonical).
// GAL: the target is sigma_g(d) for the Galois element g with g^-1 mod 2n = ginv.  Digit J is gathered from d by the first
// forward pass and negated mod q_J where the automorphism flips the sign, before its reduction mod p_I: the digits are the
// integers the separate galois_kernel would have written, so every later word is unchanged.
// MULTI (with GAL): item i's target is sigma_{g_i}(c1) of tab[i].ct with tab[i]'s key; d, d_stride, key and ginv are unused.
template <int LOGN, bool GAL, bool MULTI = false>
__device__ __forceinline__ void ks_cluster_body(const NttJob &job, const u64 *d, long long d_stride, const u64 *key, int key_rows,
                                                u64 *ks2, int k, unsigned ginv, const B200GalItem *tab = nullptr)
{
    extern __shared__ u64 mc_sm[];
    constexpr int N = 1 << LOGN;
    double *smd = reinterpret_cast<double *>(mc_sm);
    const int tid = (int)threadIdx.x;
    KsPlace w = ks_place(k);
    {
        const NttPrimeFp PF = job.fprimes[job.slot_prime[w.I]];
        const NttPrime PI_ = job.primes[job.slot_prime[w.I]];
        // digit J of the target, reduced mod p_I by the first pass (job.reduce_input)
        const u64 *dj = MULTI ? nullptr : d + w.item * d_stride + (long long)w.J * N;
        if constexpr (MULTI)
            NttFpStaticPass<LOGN, NT, true, 0, GalOpt>::run(job, PF, PI_, tab[w.item].ct + (long long)(k + w.J) * N, nullptr, smd, tid,
                                                            nullptr, tab[w.item].ginv, job.primes[job.slot_prime[w.J]].p);
        else if constexpr (GAL)
            NttFpStaticPass<LOGN, NT, true, 0, GalOpt>::run(job, PF, PI_, dj, nullptr, smd, tid, nullptr, ginv,
                                                            job.primes[job.slot_prime[w.J]].p);
        else
            NttFpStaticPass<LOGN, NT, true, 0, FwdOpt>::run(job, PF, PI_, dj, nullptr, smd, tid);
    }
    cluster_sync(); // all k digits transformed
    w = ks_place(k);

    // inner product: CTA J owns the chunks of NT coefficients J, J + k, J + 2k, ...; each coefficient is read (k CTAs) and
    // written (CTAs 0, 1) by one thread only, so the in-place overwrite of digits 0 and 1 by acc_0 and acc_1 has no hazard
    {
        const NttPrimeFp PF = job.fprimes[job.slot_prime[w.I]];
        const double p = PF.p, pinv = PF.pinv;
        const unsigned base = (unsigned)__cvta_generic_to_shared(smd);
        unsigned r0, r1;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r0) : "r"(base), "r"(0));
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r1) : "r"(base), "r"(1));
        // key[J][c][residue][coeff]: the special prime's row is the last key residue
        const long long kstride = (long long)key_rows * N;
        const u64 *kr = (MULTI ? tab[w.item].key : key) + (long long)(w.I < k ? w.I : key_rows - 1) * N + tid;
        // U chunks per round: their k remote loads and 2k key loads are issued per digit together (n = 4096: two, as in
        // mul_cluster_kernel a wider round makes ptxas spill)
        constexpr int CH = N / NT, U = LOGN >= 13 ? 4 : 2;
#pragma unroll 1
        for (int ch = w.J; ch < CH; ch += U * k)
        {
            unsigned off[U];
            int e[U];
            double a0[U], a1[U];
#pragma unroll
            for (int u = 0; u < U; u++)
            {
                e[u] = (ch + u * k) * NT;
                off[u] = (unsigned)ntt_pad(e[u] + tid) * 8u;
                a0[u] = 0.0;
                a1[u] = 0.0;
            }
#pragma unroll 1
            for (int J = 0; J < k; J++)
            {
                unsigned rj;
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rj) : "r"(base), "r"(J));
                const u64 *k0 = kr + (long long)(2 * J) * kstride, *k1 = k0 + kstride;
                double x[U];
                u64 y0[U], y1[U];
#pragma unroll
                for (int u = 0; u < U; u++)
                    if (ch + u * k < CH)
                    {
                        asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(x[u]) : "r"(rj + off[u]) : "memory");
                        y0[u] = __ldg(k0 + e[u]);
                        y1[u] = __ldg(k1 + e[u]);
                    }
#pragma unroll
                for (int u = 0; u < U; u++)
                    if (ch + u * k < CH)
                    {
                        // the FP64 branch of ksmac_tma_kernel, term order included, on the words the forward NTT would have written
                        const double xc = to_canonical(x[u], p, pinv);
                        a0[u] = B200_DADD(a0[u], fp_mulmod2(xc, fp_from_u64(y0[u]), p, pinv));
                        a1[u] = B200_DADD(a1[u], fp_mulmod2(xc, fp_from_u64(y1[u]), p, pinv));
                    }
            }
#pragma unroll
            for (int u = 0; u < U; u++)
                if (ch + u * k < CH)
                {
                    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(r0 + off[u]), "d"(to_canonical(a0[u], p, pinv)) : "memory");
                    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(r1 + off[u]), "d"(to_canonical(a1[u], p, pinv)) : "memory");
                }
        }
    }
    cluster_sync(); // acc_0, acc_1 in place; nothing reads the shared memory of CTAs 2 .. k-1 after this
    w = ks_place(k);
    if (w.J >= 2)
        return;
    u64 *dst = ks2 + ((w.item * 2 + w.J) * (k + 1) + w.I) * N;
    const int pi = job.slot_prime[w.I]; // (loaded again: nothing of the inner product stays live)
    NttFpStaticPass<LOGN, NT, false, 0, InvOpt>::run(job, job.fprimes[pi], job.primes[pi], nullptr, dst, smd, tid);
}

template <int LOGN>
__global__ void __launch_bounds__(NT, 3) ks_cluster_kernel(const NttJob job, const u64 *d, long long d_stride, const u64 *key, int key_rows,
                                                           u64 *ks2, int k)
{
    ks_cluster_body<LOGN, false>(job, d, d_stride, key, key_rows, ks2, k, 0);
}

template <int LOGN>
__global__ void __launch_bounds__(NT, 3) ks_cluster_galois_kernel(const NttJob job, const u64 *d, long long d_stride, const u64 *key,
                                                                  int key_rows, u64 *ks2, int k, unsigned ginv)
{
    ks_cluster_body<LOGN, true>(job, d, d_stride, key, key_rows, ks2, k, ginv);
}

template <int LOGN>
__global__ void __launch_bounds__(NT, 3) ks_cluster_galois_multi_kernel(const NttJob job, const B200GalItem *tab, int key_rows, u64 *ks2,
                                                                        int k)
{
    ks_cluster_body<LOGN, true, true>(job, nullptr, 0, nullptr, key_rows, ks2, k, 0, tab);
}

template <int LOGN>
cudaLaunchConfig_t config(long long clusters, cudaLaunchAttribute *at, cudaStream_t s, int csize = CLUSTER)
{
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = csize;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(clusters * csize));
    cfg.blockDim = dim3(NT);
    cfg.dynamicSmemBytes = smem_bytes<LOGN>();
    cfg.stream = s;
    // let the hardware balance a cluster's CTAs over the SMs of its GPC: 4 % more multiply+relinearize throughput at n = 8192,
    // k = 4 than the default placement, which measured the same as cudaClusterSchedulingPolicySpread (DESIGN.md §5)
    at[1].id = cudaLaunchAttributeClusterSchedulingPolicyPreference;
    at[1].val.clusterSchedulingPolicyPreference = cudaClusterSchedulingPolicyLoadBalancing;
    cfg.attrs = at;
    cfg.numAttrs = 2;
    return cfg;
}

// shared-memory attributes of a cluster kernel, and how many clusters of `csize` CTAs of it the device holds at once
template <int LOGN, typename KERNEL>
int setup(KERNEL kernel, int csize, int *active)
{
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<LOGN>())) != cudaSuccess)
        return (int)e;
    if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100)) != cudaSuccess)
        return (int)e;
    cudaLaunchAttribute at[2];
    const cudaLaunchConfig_t cfg = config<LOGN>(1, at, nullptr, csize);
    return (int)cudaOccupancyMaxActiveClusters(active, kernel, &cfg);
}
} // namespace

int b200_mul_cluster_setup(int logn, int *active)
{
    *active = 0;
    if (logn == 12)
        return setup<12>(mul_cluster_kernel<12>, CLUSTER, active);
    if (logn == 13)
        return setup<13>(mul_cluster_kernel<13>, CLUSTER, active);
    return 0;
}

int b200_mul_cluster(int logn, const NttJob &job, const u64 *a, const u64 *b, const u64 *ext, u64 *D, int k, void *stream)
{
    cudaLaunchAttribute at[2];
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

int b200_ks_cluster_setup(int logn, int k, int *active)
{
    *active = 0;
    if (k < 2 || k > 8)
        return 0;
    // all three variants: the same shared memory, and the register bound of __launch_bounds__; the smallest count of them
    int plain = 0, gal = 0, multi = 0, rc = 0;
    if (logn == 12 && !(rc = setup<12>(ks_cluster_kernel<12>, k, &plain)) && !(rc = setup<12>(ks_cluster_galois_kernel<12>, k, &gal)))
        rc = setup<12>(ks_cluster_galois_multi_kernel<12>, k, &multi);
    if (logn == 13 && !(rc = setup<13>(ks_cluster_kernel<13>, k, &plain)) && !(rc = setup<13>(ks_cluster_galois_kernel<13>, k, &gal)))
        rc = setup<13>(ks_cluster_galois_multi_kernel<13>, k, &multi);
    *active = rc ? 0 : std::min(plain, std::min(gal, multi));
    return rc;
}

int b200_ks_cluster_multi(int logn, const NttJob &job, const B200GalItem *tab, int key_rows, u64 *ks2, int k, void *stream)
{
    cudaLaunchAttribute at[2];
    const long long clusters = job.items * (k + 1);
    if (k < 2 || k > 8)
        return (int)cudaErrorInvalidValue;
    if (logn == 12)
    {
        const cudaLaunchConfig_t cfg = config<12>(clusters, at, (cudaStream_t)stream, k);
        return (int)cudaLaunchKernelEx(&cfg, ks_cluster_galois_multi_kernel<12>, job, tab, key_rows, ks2, k);
    }
    if (logn == 13)
    {
        const cudaLaunchConfig_t cfg = config<13>(clusters, at, (cudaStream_t)stream, k);
        return (int)cudaLaunchKernelEx(&cfg, ks_cluster_galois_multi_kernel<13>, job, tab, key_rows, ks2, k);
    }
    return (int)cudaErrorInvalidValue;
}

int b200_ks_cluster(int logn, const NttJob &job, const u64 *d, long long d_stride, const u64 *key, int key_rows, u64 *ks2, int k,
                    unsigned galois_inv, void *stream)
{
    cudaLaunchAttribute at[2];
    const long long clusters = job.items * (k + 1);
    if (k < 2 || k > 8)
        return (int)cudaErrorInvalidValue;
    if (logn == 12)
    {
        const cudaLaunchConfig_t cfg = config<12>(clusters, at, (cudaStream_t)stream, k);
        if (galois_inv)
            return (int)cudaLaunchKernelEx(&cfg, ks_cluster_galois_kernel<12>, job, d, d_stride, key, key_rows, ks2, k, galois_inv);
        return (int)cudaLaunchKernelEx(&cfg, ks_cluster_kernel<12>, job, d, d_stride, key, key_rows, ks2, k);
    }
    if (logn == 13)
    {
        const cudaLaunchConfig_t cfg = config<13>(clusters, at, (cudaStream_t)stream, k);
        if (galois_inv)
            return (int)cudaLaunchKernelEx(&cfg, ks_cluster_galois_kernel<13>, job, d, d_stride, key, key_rows, ks2, k, galois_inv);
        return (int)cudaLaunchKernelEx(&cfg, ks_cluster_kernel<13>, job, d, d_stride, key, key_rows, ks2, k);
    }
    return (int)cudaErrorInvalidValue;
}
