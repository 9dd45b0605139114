// FP64 latency / throughput of this GPU, as the kernels of this repo see it (-fmad=false does not matter here: explicit intrinsics).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench/fp64 tools/microbench/fp64.cu && tools/microbench/fp64
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void chain(double* out, long long* cyc, int iters, double seed) {
    double x = seed + threadIdx.x * 1e-9, y = 1.000000001;
    const long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (OP == 0) x = __dadd_rn(x, y);
            if (OP == 1) x = __dmul_rn(x, y);
            if (OP == 2) x = __fma_rn(x, y, y);
            if (OP == 3) x = __ddiv_rn(y, x) + 1.5;   // division + one add, dependent
            if (OP == 4) x = __dsqrt_rn(x) + 1.5;
        }
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
    out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}
// throughput: every thread runs 8 independent chains
__global__ void tput(double* out, long long* cyc, int iters, double seed) {
    double x[8];
    for (int k = 0; k < 8; ++k) x[k] = seed + k + threadIdx.x * 1e-9;
    const double y = 1.000000001;
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 1
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = __fma_rn(x[k], y, y);
    }
    __syncthreads();
    const long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
    double s = 0;
    for (int k = 0; k < 8; ++k) s += x[k];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
    double* out; long long* cyc; long long h;
    cudaMalloc(&out, 1 << 24); cudaMalloc(&cyc, 8);
    const char* names[5] = {"DADD", "DMUL", "DFMA", "DDIV+DADD", "DSQRT+DADD"};
    const int iters = 2000;
    for (int warps = 1; warps <= 8; warps *= 2) {
        printf("dependent chain, one block of %d warp(s) on one SM: cycles per operation\n", warps);
#define RUN(OP) chain<OP><<<1, 32 * warps>>>(out, cyc, iters, 1.25); chain<OP><<<1, 32 * warps>>>(out, cyc, iters, 1.25); cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost); printf("  %-11s %7.1f\n", names[OP], (double)h / (iters * 16.0));
        RUN(0) RUN(1) RUN(2) RUN(3) RUN(4)
    }
    for (int threads = 128; threads <= 1024; threads *= 2) {
        tput<<<1, threads>>>(out, cyc, iters, 1.25); tput<<<1, threads>>>(out, cyc, iters, 1.25);
        cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("independent DFMA, one SM, %4d threads x 8 chains: %.2f DFMA lanes per cycle per SM\n", threads, (double)threads * 32.0 * iters / (double)h);
    }
    int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("SM clock (attribute) %d kHz; cudaGetLastError: %s\n", clk, cudaGetErrorString(cudaGetLastError()));
    return 0;
}
