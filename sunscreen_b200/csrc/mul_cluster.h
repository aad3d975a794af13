// mul_cluster.h — launcher of the fused BEHZ tensor-product kernel (mul_cluster.cu).
#pragma once
#include "ntt_body.cuh"

// Sets the kernel's shared-memory attribute and returns (in *active) how many 4-CTA clusters of it the device can hold at
// once (cudaOccupancyMaxActiveClusters); *active = 0 for sizes without a cluster kernel.  Returns a cudaError_t.
int b200_mul_cluster_setup(int logn, int *active);
// The size-2 x size-2 product over `job.items` items and job.slots = R = k + |Bsk| residue rows (job.slot_prime), FP64 primes
// only: forward transforms of a0, a1, b0, b1 (q rows from a/b [item][2][k][n], Bsk rows from ext [item][4][R][n]), dyadic
// product, inverse transforms of D0, D1, D2 into D [item][3][R][n] (coefficient form, canonical).  Returns a cudaError_t.
int b200_mul_cluster(int logn, const NttJob &job, const u64 *a, const u64 *b, const u64 *ext, u64 *D, int k, void *stream);
