// mul_cluster.h — launchers of the thread-block cluster kernels (mul_cluster.cu): the fused BEHZ tensor product and the fused
// NTT-domain half of the key switch.
#pragma once
#include "ntt_body.cuh"

// Sets the kernel's shared-memory attribute and returns (in *active) how many 4-CTA clusters of it the device can hold at
// once (cudaOccupancyMaxActiveClusters); *active = 0 for sizes without a cluster kernel.  Returns a cudaError_t.
int b200_mul_cluster_setup(int logn, int *active);
// The size-2 x size-2 product over `job.items` items and job.slots = R = k + |Bsk| residue rows (job.slot_prime), FP64 primes
// only: forward transforms of a0, a1, b0, b1 (q rows from a/b [item][2][k][n], Bsk rows from ext [item][4][R][n]), dyadic
// product, inverse transforms of D0, D1, D2 into D [item][3][R][n] (coefficient form, canonical).  Returns a cudaError_t.
int b200_mul_cluster(int logn, const NttJob &job, const u64 *a, const u64 *b, const u64 *ext, u64 *D, int k, void *stream);
// Same for ks_cluster_kernel and ks_cluster_galois_kernel with clusters of k CTAs (*active = 0 outside 2 <= k <= 8 and n = 4096,
// 8192).
int b200_ks_cluster_setup(int logn, int k, int *active);
// The NTT-domain half of a key switch over `job.items` items, FP64 primes only: job.slot_prime = the k + 1 key residues
// (q_0 .. q_{k-1}, special), job.reduce_input = 1.  Digit J of item i is d + i d_stride + J n; the key is key[J][2][key_rows][n]
// (special prime: residue key_rows - 1).  Forward transforms of the digits mod every p_I, inner products with the key, inverse
// transforms into ks2 [item][2][k + 1][n] (coefficient form, canonical), as the ks1 NTT, the MAC and the ks2 NTT of the
// separate path produce them.  galois_inv != 0: the target is sigma_g(d) for the Galois element g = galois_inv^-1 mod 2n, each
// digit gathered from d and negated mod q_J as galois_kernel does (ks_cluster_galois_kernel).  Returns a cudaError_t.
int b200_ks_cluster(int logn, const NttJob &job, const u64 *d, long long d_stride, const u64 *key, int key_rows, u64 *ks2, int k,
                    unsigned galois_inv, void *stream);
// The same with a Galois element and a key per item (ks_cluster_galois_multi_kernel): item i's target is sigma_{g_i}(c1) of
// tab[i].ct ([2][k][n]), its key list tab[i].key; tab [job.items] is in device memory.  Returns a cudaError_t.
int b200_ks_cluster_multi(int logn, const NttJob &job, const B200GalItem *tab, int key_rows, u64 *ks2, int k, void *stream);
