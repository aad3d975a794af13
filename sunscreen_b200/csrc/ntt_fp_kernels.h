// ntt_fp_kernels.h — entry points of the translation unit that holds the statically scheduled FP64 NTT kernels.
#pragma once
#include "ntt_body.cuh"
#include <cstddef>
typedef void (*b200_ntt_fp_fn)(const NttJob);
// the kernel for (log2 n, direction, threads per CTA) or nullptr when there is none
b200_ntt_fp_fn b200_ntt_fp_kernel(int logn, bool fwd, int nt);
// how the kernels of (log2 n in [12, 14], direction) are launched; the same for every CTA width, since the options they are
// compiled with depend on size and direction only
struct B200NttFpLayout
{
    size_t smem;     // dynamic shared memory per CTA, bytes
    bool persistent; // grid of at most the resident CTAs, each walking polynomials blockIdx.x, blockIdx.x + gridDim.x, ...
};
B200NttFpLayout b200_ntt_fp_layout(int logn, bool fwd);
// resident CTAs per SM of a kernel (grid size of a persistent one)
int b200_ntt_fp_ctas_per_sm(b200_ntt_fp_fn fn, int nt, size_t smem);
// raises the dynamic shared-memory limit of every kernel; returns 0 or a cudaError_t
int b200_ntt_fp_setup(int smem_optin);
