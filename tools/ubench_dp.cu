// Developer microbenchmark: FP64 pipe throughput on sm_90a as a function of resident warps per SM sub-partition and of
// the number of independent dependency chains per thread (how much parallelism the NTT kernels need to fill the pipe).
#include <cstdio>
#include <cuda_runtime.h>
template <int ILP, int MODE>
__global__ void k(double *out, double a, double b, int iters)
{
    double acc[ILP];
#pragma unroll
    for (int i = 0; i < ILP; i++)
        acc[i] = threadIdx.x + i;
    for (int it = 0; it < iters; it++)
    {
#pragma unroll
        for (int i = 0; i < ILP; i++)
        {
            if (MODE == 0)
                acc[i] = fma(acc[i], a, b);
            else
            { // the modular product's chain: DMUL -> DMUL -> FRND -> DFMA -> DADD (+ independent DFMA)
                double h = acc[i] * a;
                double l = fma(acc[i], a, -h);
                double q = h * b;
                asm("cvt.rni.f64.f64 %0, %0;" : "+d"(q));
                acc[i] = fma(-q, 1.0e13, h) + l;
            }
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < ILP; i++)
        s += acc[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
template <int ILP, int MODE>
void run(int sms, int warps_per_smsp, double *out)
{
    const int iters = 4096;
    const int threads = 32 * 4 * warps_per_smsp; // one CTA per SM
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    k<ILP, MODE><<<sms, threads>>>(out, 1.0000001, 1e-13, 16);
    cudaEventRecord(e0);
    k<ILP, MODE><<<sms, threads>>>(out, 1.0000001, 1e-13, iters);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    const double dp_per_iter = MODE == 0 ? 1 : 6;
    const double ops = (double)sms * threads * iters * ILP * dp_per_iter;
    printf("mode %d  warps/SMSP %2d  ILP %2d : %6.1f FP64 lanes/clk/SM (@1.9 GHz)\n", MODE, warps_per_smsp, ILP, ops / (ms * 1e-3) / 1.9e9 / sms);
}
int main()
{
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    double *out;
    cudaMalloc(&out, (size_t)p.multiProcessorCount * 1024 * 8);
    for (int mode = 0; mode < 2; mode++)
        for (int w : { 1, 2, 4, 6, 8 })
        {
            run<1, 0>(p.multiProcessorCount, w, out);
            if (mode == 0)
            {
                run<2, 0>(p.multiProcessorCount, w, out);
                run<4, 0>(p.multiProcessorCount, w, out);
                run<8, 0>(p.multiProcessorCount, w, out);
            }
            else
            {
                run<1, 1>(p.multiProcessorCount, w, out);
                run<2, 1>(p.multiProcessorCount, w, out);
                run<4, 1>(p.multiProcessorCount, w, out);
                run<8, 1>(p.multiProcessorCount, w, out);
            }
        }
    return 0;
}
