// ksmac_tma.cu — key-switch inner product with TMA-tiled key streaming (sm_90a).
//
// What it computes (reference: the MAC loop of switch_key_inplace, S/evaluator.cpp:2517-2541, key layout S/kswitchkeys.h:340):
//     acc_c[I][coeff] = sum_J  NTT_{p_I}(digit_J)[coeff] * key[J][c][I][coeff]   (mod p_I),   c in {0,1}, I in [0,k] (I = k: special prime)
// for every item of a batch.  The key is the same for all items; at n = 32768, k = 15 one Galois key is 120 MiB — as large as
// the whole L2 — so an item-major kernel re-streams it from HBM for every item.
//
// Schedule here: the CTA owns one (I, 256-coefficient tile) of the KEY.  One elected thread issues a single 3-D tiled TMA load
// (cp.async.bulk.tensor, box = 256 coefficients x 1 residue x 2k (J, c) rows) that lands the whole key tile in shared memory
// and signals an mbarrier; while it is in flight every thread already requests the first item's digit rows.  The CTA then walks
// its share of the batch with the key tile resident, so each key byte is read from HBM once per batch chunk instead of once
// per item.  Digit rows are read with 128-bit coalesced loads, software-pipelined one item ahead.
#include "ksmac_tma.h"
#include "bfv_body.cuh"
#include "ntt_fp_body.cuh"
#include <cuda.h>
#include <cuda_runtime.h>
#include <mutex>

namespace
{
constexpr int TILE = 256; // coefficients per key tile (TMA box dimension limit)
constexpr int NT = 128;   // threads: two adjacent coefficients each

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int K, bool FP>
__global__ void __launch_bounds__(NT) ksmac_tma_kernel(const __grid_constant__ CUtensorMap tmap, const PrimeDev *__restrict__ primes,
                                                       const NttPrimeFp *__restrict__ fprimes, int special_idx, int key_rows,
                                                       const u64 *__restrict__ ks1, u64 *__restrict__ ks2, long long n, long long batch,
                                                       int items_per_cta)
{
    extern __shared__ __align__(1024) unsigned char ks_smem[];
    __shared__ __align__(8) unsigned long long mbar;
    u64 *ktile = reinterpret_cast<u64 *>(ks_smem); // [2K][TILE]
    const int tile = blockIdx.x, I = blockIdx.y;
    const long long item0 = (long long)blockIdx.z * items_per_cta;
    const long long item1 = item0 + items_per_cta < batch ? item0 + items_per_cta : batch;
    const int tid = threadIdx.x;
    const int prime_idx = I < K ? I : special_idx;
    const int key_res = I < K ? I : key_rows - 1;
    if (tid == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0)
    {
        const unsigned bytes = 2u * K * TILE * (unsigned)sizeof(u64);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                         smem_u32(ktile)),
                     "l"(reinterpret_cast<unsigned long long>(&tmap)), "r"(smem_u32(&mbar)), "r"(tile * TILE), "r"(key_res), "r"(0)
                     : "memory");
    }
    const long long c = (long long)tile * TILE + 2 * tid;
    // digit rows of one item: ks1[item][I][J][coeff]
    auto rows = [&](long long item) { return ks1 + ((item * (K + 1) + I) * K) * n + c; };
    ulonglong2 x[K], xn[K];
    if (item0 < item1)
    {
        const u64 *r = rows(item0);
#pragma unroll
        for (int J = 0; J < K; J++)
            x[J] = __ldg(reinterpret_cast<const ulonglong2 *>(r + J * n));
    }
    // wait for the key tile (phase 0 of the barrier)
    {
        unsigned done = 0;
        while (!done)
            asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                         : "=r"(done)
                         : "r"(smem_u32(&mbar)), "r"(0)
                         : "memory");
    }
    PrimeDev P;
    double p = 0.0, pinv = 0.0;
    if (FP)
    {
        p = __ldg(&fprimes[prime_idx].p);
        pinv = __ldg(&fprimes[prime_idx].pinv);
    }
    else
        P = ld_prime(&primes[prime_idx]);
    const ulonglong2 *kt = reinterpret_cast<const ulonglong2 *>(ktile) + tid; // row r of the tile: kt[r * TILE / 2]
    for (long long item = item0; item < item1; item++)
    {
        if (item + 1 < item1)
        {
            const u64 *r = rows(item + 1);
#pragma unroll
            for (int J = 0; J < K; J++)
                xn[J] = __ldg(reinterpret_cast<const ulonglong2 *>(r + J * n));
        }
        u64 o00, o01, o10, o11; // o[coefficient][component]
        if (FP)
        {
            double a00 = 0.0, a01 = 0.0, a10 = 0.0, a11 = 0.0;
#pragma unroll
            for (int J = 0; J < K; J++)
            {
                const ulonglong2 k0 = kt[(2 * J) * (TILE / 2)], k1 = kt[(2 * J + 1) * (TILE / 2)];
                const double x0 = fp_from_u64(x[J].x), x1 = fp_from_u64(x[J].y);
                a00 = B200_DADD(a00, fp_mulmod2(x0, fp_from_u64(k0.x), p, pinv));
                a01 = B200_DADD(a01, fp_mulmod2(x0, fp_from_u64(k1.x), p, pinv));
                a10 = B200_DADD(a10, fp_mulmod2(x1, fp_from_u64(k0.y), p, pinv));
                a11 = B200_DADD(a11, fp_mulmod2(x1, fp_from_u64(k1.y), p, pinv));
            }
            o00 = fp_to_canonical(a00, p, pinv);
            o01 = fp_to_canonical(a01, p, pinv);
            o10 = fp_to_canonical(a10, p, pinv);
            o11 = fp_to_canonical(a11, p, pinv);
        }
        else
        {
            u64 l00 = 0, h00 = 0, l01 = 0, h01 = 0, l10 = 0, h10 = 0, l11 = 0, h11 = 0; // 128-bit lazy sums (k <= 16 terms of < 2^122)
#pragma unroll
            for (int J = 0; J < K; J++)
            {
                const ulonglong2 k0 = kt[(2 * J) * (TILE / 2)], k1 = kt[(2 * J + 1) * (TILE / 2)];
                mac128(x[J].x, k0.x, l00, h00);
                mac128(x[J].x, k1.x, l01, h01);
                mac128(x[J].y, k0.y, l10, h10);
                mac128(x[J].y, k1.y, l11, h11);
            }
            o00 = barrett128(l00, h00, P.p, P.r0, P.r1);
            o01 = barrett128(l01, h01, P.p, P.r0, P.r1);
            o10 = barrett128(l10, h10, P.p, P.r0, P.r1);
            o11 = barrett128(l11, h11, P.p, P.r0, P.r1);
        }
        u64 *out0 = ks2 + ((item * 2 + 0) * (K + 1) + I) * n + c;
        u64 *out1 = ks2 + ((item * 2 + 1) * (K + 1) + I) * n + c;
        *reinterpret_cast<ulonglong2 *>(out0) = make_ulonglong2(o00, o10);
        *reinterpret_cast<ulonglong2 *>(out1) = make_ulonglong2(o01, o11);
#pragma unroll
        for (int J = 0; J < K; J++)
            x[J] = xn[J];
    }
}

typedef CUresult (*encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                              CUtensorMapFloatOOBfill);
encode_fn get_encode()
{
    static encode_fn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (encode_fn)p;
    });
    return fn;
}

template <int K>
int launch(bool fp, const CUtensorMap &tm, const PrimeDev *primes, const NttPrimeFp *fprimes, int special_idx, int key_rows, const u64 *ks1,
           u64 *ks2, long long n, long long batch, int sm_count, cudaStream_t s)
{
    const int tiles = (int)(n / TILE);
    // items per CTA: enough CTAs to fill the machine several times over, but every CTA amortises its key tile over >= 8 items
    long long ipc = batch;
    const long long per_chunk = (long long)tiles * (K + 1);
    while (ipc > 8 && per_chunk * ((batch + ipc - 1) / ipc) < 8LL * sm_count)
        ipc = (ipc + 1) / 2;
    const unsigned chunks = (unsigned)((batch + ipc - 1) / ipc);
    const size_t smem = 2 * (size_t)K * TILE * sizeof(u64);
    dim3 grid((unsigned)tiles, (unsigned)(K + 1), chunks);
    cudaError_t e;
    if (fp)
    {
        if (smem > 48 * 1024 && (e = cudaFuncSetAttribute(ksmac_tma_kernel<K, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return (int)e;
        ksmac_tma_kernel<K, true><<<grid, NT, smem, s>>>(tm, primes, fprimes, special_idx, key_rows, ks1, ks2, n, batch, (int)ipc);
    }
    else
    {
        if (smem > 48 * 1024 && (e = cudaFuncSetAttribute(ksmac_tma_kernel<K, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess)
            return (int)e;
        ksmac_tma_kernel<K, false><<<grid, NT, smem, s>>>(tm, primes, fprimes, special_idx, key_rows, ks1, ks2, n, batch, (int)ipc);
    }
    return (int)cudaGetLastError();
}
} // namespace

int b200_ksmac_tma_supported(long long n, int K)
{
    return n >= TILE && n % TILE == 0 && K >= 1 && K <= 16 && get_encode() != nullptr;
}

int b200_ksmac_tma(int K, int fp, const void *primes, const void *fprimes, int special_idx, int key_rows, const unsigned long long *ks1,
                   const unsigned long long *key, unsigned long long *ks2, long long n, long long batch, int sm_count, void *stream)
{
    encode_fn enc = get_encode();
    if (!enc)
        return -1;
    // the key list as a 3-D tensor: (coefficient n | key residue key_rows | (J, component) 2K), 8-byte elements
    CUtensorMap tm;
    const cuuint64_t dims[3] = { (cuuint64_t)n, (cuuint64_t)key_rows, (cuuint64_t)(2 * K) };
    const cuuint64_t strides[2] = { (cuuint64_t)n * 8, (cuuint64_t)n * 8 * (cuuint64_t)key_rows };
    const cuuint32_t box[3] = { (cuuint32_t)TILE, 1, (cuuint32_t)(2 * K) };
    const cuuint32_t estr[3] = { 1, 1, 1 };
    CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, const_cast<unsigned long long *>(key), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return -2;
    const PrimeDev *pd = (const PrimeDev *)primes;
    const NttPrimeFp *fd = (const NttPrimeFp *)fprimes;
    cudaStream_t s = (cudaStream_t)stream;
#define CASE(KK)                                                                                                        \
    case KK:                                                                                                            \
        return launch<KK>(fp != 0, tm, pd, fd, special_idx, key_rows, ks1, ks2, n, batch, sm_count, s);
    switch (K)
    {
        CASE(1) CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10) CASE(11) CASE(12) CASE(13) CASE(14) CASE(15) CASE(16)
    default:
        return -3;
    }
#undef CASE
}
