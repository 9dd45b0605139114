// Latency micro-benchmarks behind the design of the 18x18 solve.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o lat lat.cu && ./lat
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_lat(double* out, long long* cyc, double a, double b, int n) {
    double x = a;
    long long t0 = clock64();
    for (int i = 0; i < n; ++i) x = x + b;            // dependent DADD
    long long t1 = clock64();
    double y = a;
    for (int i = 0; i < n; ++i) y = y * b;            // dependent DMUL
    long long t2 = clock64();
    double z = a;
    for (int i = 0; i < n; ++i) z = z / b;            // dependent DDIV
    long long t3 = clock64();
    double w = a;
    for (int i = 0; i < n; ++i) w = (w > b) ? w - b : w + a;   // compare + select + add
    long long t4 = clock64();
    float f = (float)a;
    for (int i = 0; i < n; ++i) f = f + (float)b;     // dependent FADD
    long long t5 = clock64();
    double s = a;
    for (int i = 0; i < n; ++i) s = __shfl_xor_sync(0xffffffffu, s, 1) + b;   // shuffle(f64) + DADD
    long long t6 = clock64();
    for (int i = 0; i < n; ++i) __syncthreads();
    long long t7 = clock64();
    if (threadIdx.x == 0) {
        cyc[0] = t1 - t0; cyc[1] = t2 - t1; cyc[2] = t3 - t2; cyc[3] = t4 - t3; cyc[4] = t5 - t4; cyc[5] = t6 - t5; cyc[6] = t7 - t6;
    }
    out[threadIdx.x] = x + y + z + w + f + s;
}

int main() {
    double* d_out; long long* d_c;
    cudaMalloc(&d_out, 1024 * 8); cudaMalloc(&d_c, 64);
    const int n = 2000;
    const char* names[7] = {"DADD dep", "DMUL dep", "DDIV dep", "DSETP+SEL+DADD dep", "FADD dep", "SHFL64+DADD dep", "__syncthreads"};
    for (int threads : {32, 128, 672}) {
        k_lat<<<1, threads>>>(d_out, d_c, 1.0000001, 1.0000002, n);
        cudaDeviceSynchronize();
        k_lat<<<1, threads>>>(d_out, d_c, 1.0000001, 1.0000002, n);
        cudaDeviceSynchronize();
        long long c[8];
        cudaMemcpy(c, d_c, 56, cudaMemcpyDeviceToHost);
        printf("threads=%d:", threads);
        for (int i = 0; i < 7; ++i) printf("  %s=%.1f", names[i], (double)c[i] / n);
        printf("  (cycles per op)\n");
    }
    return 0;
}
