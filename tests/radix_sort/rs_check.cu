// TEST INFRASTRUCTURE (not product code): the stable radix sort of immesh_b200/csrc/radix_sort.cuh run twice on the same pairs --
// with the count on the host (grids cover the count), and with the count read on the device over a larger capacity and a grid of
// dev_grid blocks (0: the grid covers the capacity), as the plane-map markers of the scan feed and the mesh's change feed run it.
#include <cuda_runtime.h>

#define IM_LAUNCH(KERN, GRID, BLOCK, SMEM, STREAM, ...) KERN<<<dim3(GRID), dim3(BLOCK), (SMEM), (STREAM)>>>(__VA_ARGS__)
namespace {
#include "../../immesh_b200/csrc/radix_sort.cuh"
}

namespace {
struct Bufs {
    unsigned int* k[2] = {nullptr, nullptr};
    unsigned int* v[2] = {nullptr, nullptr};
    int* hist = nullptr;
    int* n = nullptr;
    ~Bufs() {
        for (int i = 0; i < 2; ++i) { cudaFree(k[i]); cudaFree(v[i]); }
        cudaFree(hist);
        cudaFree(n);
    }
    cudaError_t alloc(int len) {
        const size_t tiles = (size_t)(len + VG_TILE - 1) / VG_TILE + 1;
        cudaError_t e = cudaSuccess;
        for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
            if ((e = cudaMalloc(&k[i], (size_t)(len + 1) * 4)) == cudaSuccess) e = cudaMalloc(&v[i], (size_t)(len + 1) * 4);
        }
        if (e == cudaSuccess) e = cudaMalloc(&hist, tiles * 256 * sizeof(int));
        if (e == cudaSuccess) e = cudaMalloc(&n, sizeof(int));
        return e;
    }
};
// the n pairs (keys, values) into b's first buffers, sorted over `passes` digits; the sorted pairs back to the host
cudaError_t run(Bufs& b, const unsigned int* keys, int n, int len, int passes, bool on_device, int dev_grid, unsigned int* ko, unsigned int* vo) {
    cudaError_t e = b.alloc(len);
    if (e != cudaSuccess) return e;
    unsigned int* iota = new unsigned int[n + 1];
    for (int i = 0; i < n; ++i) iota[i] = (unsigned int)i;
    if (n > 0) {
        if ((e = cudaMemcpy(b.k[0], keys, (size_t)n * 4, cudaMemcpyHostToDevice)) == cudaSuccess) e = cudaMemcpy(b.v[0], iota, (size_t)n * 4, cudaMemcpyHostToDevice);
    }
    delete[] iota;
    if (e == cudaSuccess) e = cudaMemcpy(b.n, &n, sizeof(int), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return e;
    const int cur = on_device ? rs_sort_passes(0, b.k, b.v, 0, len, passes, b.hist, b.n, dev_grid) : rs_sort_passes(0, b.k, b.v, 0, n, passes, b.hist);
    if ((e = cudaGetLastError()) != cudaSuccess || (e = cudaDeviceSynchronize()) != cudaSuccess) return e;
    if (n > 0) {
        if ((e = cudaMemcpy(ko, b.k[cur], (size_t)n * 4, cudaMemcpyDeviceToHost)) == cudaSuccess) e = cudaMemcpy(vo, b.v[cur], (size_t)n * 4, cudaMemcpyDeviceToHost);
    }
    return e;
}
}  // namespace

extern "C" {
// 0, or the CUDA error.  n >= 1 for the host-count sort (its grids cover n); the device-count sort takes any n <= cap.
int rs_check_host(const unsigned int* keys, int n, int passes, unsigned int* keys_out, unsigned int* vals_out) {
    Bufs b;
    return (int)run(b, keys, n, n, passes, false, 0, keys_out, vals_out);
}
int rs_check_dev(const unsigned int* keys, int n, int cap, int passes, int dev_grid, unsigned int* keys_out, unsigned int* vals_out) {
    Bufs b;
    return (int)run(b, keys, n, cap, passes, true, dev_grid, keys_out, vals_out);
}
}
