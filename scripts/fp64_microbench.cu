// FP64 pipe microbenchmark (tuning aid, not part of the library): DFMA throughput as a function of resident warps per SM and
// independent chains per thread, plus the mixed case DFMA + integer ALU work.  nvcc -O3 -arch=sm_90a -o /tmp/fp64_microbench
#include <cstdio>
#include <cuda_runtime.h>

template <int C>
__global__ void k(double* out, int iters, double m, double c) {
    double a[C];
#pragma unroll
    for (int i = 0; i < C; ++i) a[i] = 1.0 + 1e-9 * (threadIdx.x + i);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < C; ++i) a[i] = fma(a[i], m, c);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < C; ++i) s += a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// each DFMA accompanied by K dependent integer ops on a separate chain (models address / bit-manipulation work)
template <int C, int K>
__global__ void kmix(double* out, int iters, double m, double c) {
    double a[C];
    unsigned u[C];
#pragma unroll
    for (int i = 0; i < C; ++i) { a[i] = 1.0 + 1e-9 * (threadIdx.x + i); u[i] = threadIdx.x + i; }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < C; ++i) {
            a[i] = fma(a[i], m, c);
#pragma unroll
            for (int q = 0; q < K; ++q) u[i] = (u[i] ^ (u[i] >> 3)) + 0x9e3779b9u;
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < C; ++i) s += a[i] + (double)u[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <class F>
double timeit(F f) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    f();
    cudaEventRecord(e0);
    f();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

int main() {
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int sms = p.multiProcessorCount;
    double* out; cudaMalloc(&out, (size_t)sms * 2048 * 8);
    const int iters = 20000;
    printf("device %s, %d SMs, clock %d kHz\n", p.name, sms, p.clockRate);
    printf("warps/SM chains  TFLOP/s  cycles per DFMA per warp-chain (latency if < peak)\n");
    for (int wps : {4, 8, 16, 32, 64}) {
        const int threads = wps >= 8 ? 256 : wps * 32, blocks = sms * (wps * 32 / threads);
#define RUN(C) { double ms = timeit([&] { k<C><<<blocks, threads>>>(out, iters, 0.999999999, 1e-9); }); \
        double fl = 2.0 * C * iters * (double)blocks * threads; \
        double cyc = ms * 1e-3 * p.clockRate * 1e3 / ((double)iters); \
        printf("%5d %6d  %8.2f   %6.2f clk per loop trip (%d dfma)\n", wps, C, fl / ms / 1e9, cyc, C); }
        RUN(1) RUN(2) RUN(4) RUN(8)
    }
    printf("mixed: DFMA + K int ops, 16 warps/SM, 2 chains\n");
    {
        const int threads = 256, blocks = sms * 2;
#define RUNM(K) { double ms = timeit([&] { kmix<2, K><<<blocks, threads>>>(out, iters, 0.999999999, 1e-9); }); \
        double fl = 2.0 * 2 * iters * (double)blocks * threads; printf("K=%d  %8.2f TFLOP/s\n", K, fl / ms / 1e9); }
        RUNM(0) RUNM(1) RUNM(2) RUNM(4)
    }
    return 0;
}
