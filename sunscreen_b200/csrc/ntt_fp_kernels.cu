// ntt_fp_kernels.cu — the statically scheduled FP64-pipe NTT / INTT kernels (ntt_fp_body.cuh) as their own translation
// unit: every (size, direction, CTA width) kernel is compiled here once; b200_bfv.cu launches them through
// the function pointers returned by b200_ntt_fp_kernel().
#include "ntt_fp_kernels.h"
#include "ntt_fp_body.cuh"
#include <cuda_runtime.h>

// The options each transform ships with, per (log2 n, direction): every pass after the first forward (before the last inverse)
// one is warp-private; the n = 8192 inverse and the n = 16384 forward read the first twiddles from shared memory, and the
// n = 16384 inverse is the persistent kernel whose input streams in during the previous polynomial's last pass.
template <int LOGN, bool FWD>
using KernelOpt = NttFpOpt<(LOGN == 13 && !FWD) || (LOGN == 14 && FWD), LOGN == 14 && !FWD>;

// FP64-only statically scheduled kernel (all slots of the job use FP-capable primes).  Blocks run slot-major (all items of
// slot 0, then slot 1, ...): CTAs that run at the same time work on the same prime, so the early-pass twiddles stay in L1.
template <int LOGN, bool FWD, int NT>
__global__ void __launch_bounds__(NT, (LOGN <= 13 ? (NT <= 256 ? 3 : 2) : 1)) ntt_fp_kernel(const NttJob job)
{
    using OPT = KernelOpt<LOGN, FWD>;
    extern __shared__ u64 ntt_sm[];
    if constexpr (OPT::STREAM)
    {
        // Persistent CTAs walk blockIdx.x, blockIdx.x + gridDim.x, ... ; while one polynomial's LAST pass runs, the next
        // polynomial's words are already requested (cp.async) into the shared-memory slots that pass has finished with, so no
        // CTA ever sits idle waiting for its input (with global traffic removed the same kernel needed 0.49 ms instead of
        // 0.70 ms for 16384 transforms — that wait is what this kernel hides).
        constexpr int N = 1 << LOGN;
        const long long total = job.items * (long long)job.slots;
        long long b = (long long)blockIdx.x;
        if (b >= total)
            return;
        const int tid = (int)threadIdx.x;
        double *smd = reinterpret_cast<double *>(ntt_sm);
        int slot = (int)(b / job.items);
        long long item = b - (long long)slot * job.items;
        const u64 *src = ntt_src_ptr(job, item, slot);
        {
            const int ptid = ntt_pad(tid);
            constexpr int PNT = NT + (NT >> 4);
            const unsigned sbase = (unsigned)__cvta_generic_to_shared(smd + ptid);
#pragma unroll
            for (int it = 0; it < N / NT; it++)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(sbase + (unsigned)(it * PNT * 8)), "l"(src + tid + it * NT) : "memory");
        }
        for (;;)
        {
            const int pidx = job.slot_prime[slot];
            const NttPrimeFp PF = job.fprimes[pidx];
            const NttPrime PI_ = job.primes[pidx];
            u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
            const long long nb = b + (long long)gridDim.x;
            const u64 *nsrc = nullptr;
            int nslot = 0;
            long long nitem = 0;
            if (nb < total)
            {
                nslot = (int)(nb / job.items);
                nitem = nb - (long long)nslot * job.items;
                nsrc = ntt_src_ptr(job, nitem, nslot);
            }
            NttFpStaticPass<LOGN, NT, FWD, 0, OPT>::run(job, PF, PI_, src, dst, smd, tid, nsrc);
            if (!nsrc)
                break;
            b = nb;
            slot = nslot;
            item = nitem;
            src = nsrc;
        }
        return;
    }
    const long long block = (long long)blockIdx.x;
    const int slot = (int)(block / job.items);
    const long long item = block - (long long)slot * job.items;
    const int pidx = job.slot_prime[slot];
    const NttPrimeFp PF = job.fprimes[pidx];
    const NttPrime PI_ = job.primes[pidx];
    const u64 *src = ntt_src_ptr(job, item, slot);
    u64 *dst = job.dst + item * job.dst_item_stride + job.slot_dst[slot];
    NttFpStaticPass<LOGN, NT, FWD, 0, OPT>::run(job, PF, PI_, src, dst, reinterpret_cast<double *>(ntt_sm), (int)threadIdx.x);
}

// (log2 n, threads per CTA) of every kernel, each in both directions: the n = 8192 transform has a 256-thread (throughput)
// and a 512-thread (latency) width
#define B200_FP_KERNELS(X) X(12, 256) X(13, 256) X(13, 512) X(14, 1024)

b200_ntt_fp_fn b200_ntt_fp_kernel(int logn, bool fwd, int nt)
{
#define X(LOGN, NT)                                                                                                    \
    if (logn == LOGN && nt == NT)                                                                                      \
        return fwd ? ntt_fp_kernel<LOGN, true, NT> : ntt_fp_kernel<LOGN, false, NT>;
    B200_FP_KERNELS(X)
#undef X
    return nullptr;
}

template <int LOGN, bool FWD>
static B200NttFpLayout fp_layout()
{
    using OPT = KernelOpt<LOGN, FWD>;
    const size_t words = (size_t)ntt_smem_words(1 << LOGN) + (OPT::SMEM_TW ? B200_NTT_TWS_ENTRIES : 0);
    return B200NttFpLayout{ words * sizeof(double), OPT::STREAM };
}

B200NttFpLayout b200_ntt_fp_layout(int logn, bool fwd)
{
    if (logn == 12)
        return fwd ? fp_layout<12, true>() : fp_layout<12, false>();
    if (logn == 13)
        return fwd ? fp_layout<13, true>() : fp_layout<13, false>();
    return fwd ? fp_layout<14, true>() : fp_layout<14, false>();
}

int b200_ntt_fp_ctas_per_sm(b200_ntt_fp_fn fn, int nt, size_t smem)
{
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fn, nt, smem) != cudaSuccess || nb < 1)
        nb = 1;
    return nb;
}

int b200_ntt_fp_setup(int smem_optin)
{
    cudaError_t e;
#define X(LOGN, NT)                                                                                                    \
    if ((e = cudaFuncSetAttribute(ntt_fp_kernel<LOGN, true, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin)) != cudaSuccess) return (int)e; \
    if ((e = cudaFuncSetAttribute(ntt_fp_kernel<LOGN, false, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin)) != cudaSuccess) return (int)e; \
    if ((e = cudaFuncSetAttribute(ntt_fp_kernel<LOGN, true, NT>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)) != cudaSuccess) return (int)e; \
    if ((e = cudaFuncSetAttribute(ntt_fp_kernel<LOGN, false, NT>, cudaFuncAttributePreferredSharedMemoryCarveout, 100)) != cudaSuccess) return (int)e;
    B200_FP_KERNELS(X)
#undef X
    return 0;
}
