// tests/emu/cuda_emu.h — TEST INFRASTRUCTURE ONLY.
// A sequential CPU stand-in for the small slice of the CUDA runtime that sunscreen_b200/csrc uses, so the
// CPU test-suite (`pytest -m "not gpu"`) can execute the library's host orchestration and kernel bodies
// (index math, constant folding, strides) without a GPU.  A "launch" runs every CTA one after another with
// blockDim forced to 1 thread for kernels that use shared memory phases (all bodies are written as strided
// loops, see ntt_body.cuh).  Nothing here is compiled into sunscreen_b200/libb200bfv.so.
#pragma once
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#define __global__ static
#define __launch_bounds__(...)
#define __restrict__

typedef int cudaError_t;
static const cudaError_t cudaSuccess = 0;
inline const char *cudaGetErrorString(cudaError_t) { return "emu error"; }
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
typedef void *cudaMemPool_t;
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaEventBlockingSync = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8,
       cudaMemPoolReuseAllowInternalDependencies = 3, cudaMemPoolAttrReleaseThreshold = 4 };
struct cudaDeviceProp { int multiProcessorCount = 1; size_t sharedMemPerBlockOptin = 232448; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };

static thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;
static thread_local void *emu_shared = nullptr;

// Resource accounting for tests/test_context_lifetime.py.  Streams, events and memory pools are distinct non-null handles;
// emu_live counts them together with every cudaMalloc, cudaMallocHost and pool allocation not yet released.  A budget
// n >= 0 lets n more of these creations succeed and fails every later one, as an exhausted device would (-1: no limit).
static std::atomic<long long> emu_live{ 0 }, emu_budget{ -1 };
static std::atomic<uintptr_t> emu_next_handle{ 0 };
extern "C" long long b200_emu_live_resources(void) { return emu_live; }
extern "C" void b200_emu_alloc_budget(long long n) { emu_budget = n; }
inline bool emu_acquire()
{
    if (emu_budget == 0)
        return false;
    if (emu_budget > 0)
        emu_budget--;
    emu_live++;
    return true;
}
inline cudaError_t emu_create(void **h)
{
    if (!emu_acquire())
        return 2;
    *h = (void *)(++emu_next_handle * 16);
    return 0;
}
inline cudaError_t emu_destroy(void *h)
{
    if (!h)
        return 1; // the runtime rejects a null handle
    emu_live--;
    return 0;
}

inline cudaError_t cudaGetDeviceCount(int *c) { *c = 1; return 0; }
inline cudaError_t cudaSetDevice(int) { return 0; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { *p = cudaDeviceProp(); return 0; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F, int, int) { return 0; }
inline cudaError_t cudaDeviceGetDefaultMemPool(cudaMemPool_t *p, int) { *p = nullptr; return 0; }
inline cudaError_t cudaMemPoolSetAttribute(cudaMemPool_t, int, void *) { return 0; }
enum { cudaMemAllocationTypePinned = 1, cudaMemHandleTypeNone = 0, cudaMemLocationTypeDevice = 1 };
struct cudaMemPoolProps { int allocType, handleTypes; struct { int type, id; } location; };
inline cudaError_t cudaMemPoolCreate(cudaMemPool_t *p, const cudaMemPoolProps *) { return emu_create(p); }
inline cudaError_t cudaMemPoolDestroy(cudaMemPool_t p) { return emu_destroy(p); }
inline cudaError_t cudaDeviceSynchronize() { return 0; }
inline cudaError_t cudaGetLastError() { return 0; }
inline cudaError_t cudaMalloc(void **p, size_t b)
{
    if (!emu_acquire())
        return 2;
    *p = std::malloc(b ? b : 8);
    return *p ? 0 : 2;
}
inline cudaError_t cudaFree(void *p)
{
    if (p)
        emu_live--;
    std::free(p);
    return 0;
}
inline cudaError_t cudaMallocHost(void **p, size_t b) { return cudaMalloc(p, b); }
inline cudaError_t cudaFreeHost(void *p) { return cudaFree(p); }
inline cudaError_t cudaMallocAsync(void **p, size_t b, cudaStream_t) { return cudaMalloc(p, b); }
inline cudaError_t cudaMallocFromPoolAsync(void **p, size_t b, cudaMemPool_t, cudaStream_t) { return cudaMalloc(p, b); }
inline cudaError_t cudaFreeAsync(void *p, cudaStream_t) { return cudaFree(p); }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t b, cudaMemcpyKind) { std::memmove(d, s, b); return 0; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t b, cudaMemcpyKind, cudaStream_t) { std::memmove(d, s, b); return 0; }
inline cudaError_t cudaMemsetAsync(void *d, int v, size_t b, cudaStream_t) { std::memset(d, v, b); return 0; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, int) { return emu_create(s); }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { return emu_destroy(s); }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, int) { return 0; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, int) { return emu_create(e); }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return 0; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { return emu_destroy(e); }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
inline unsigned long long __ldg(const unsigned long long *p) { return *p; }
inline double __ldg(const double *p) { return *p; }
inline int __syncthreads_or(int v) { return v; }

template <class F>
inline void emu_launch(dim3 grid, dim3 block, size_t smem, bool single_thread, F body)
{
    std::vector<unsigned char> sm(smem + 16);
    emu_shared = sm.data();
    gridDim = grid;
    blockDim = single_thread ? dim3(1, 1, 1) : block;
    for (unsigned by = 0; by < grid.y; by++)
        for (unsigned bx = 0; bx < grid.x; bx++)
        {
            blockIdx = dim3(bx, by, 0);
            for (unsigned tx = 0; tx < blockDim.x; tx++)
            {
                threadIdx = dim3(tx, 0, 0);
                body();
            }
        }
    emu_shared = nullptr;
}
// kernels with shared memory (or block-wide votes) run as ONE thread per CTA; the rest thread by thread
#define B200_LAUNCH(kernel, grid, block, smem, stream, ...)                                                            \
    emu_launch(dim3(grid), dim3(block), (size_t)(smem), (smem) != 0 || std::strcmp(#kernel, "transparent_kernel") == 0, \
               [&]() { kernel(__VA_ARGS__); })
