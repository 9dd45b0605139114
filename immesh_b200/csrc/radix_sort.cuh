// immesh_b200 -- the one-block scan of a buffer and the stable LSD radix sort of (u32 key, u32 value) pairs, 8-bit digits, 2048-element tiles;
// ranks inside a tile from __match_any_sync (warp) + per-warp digit counts in shared memory.  Used by the pcl::VoxelGrid front-end
// (cell index -> point), the IMU undistortion (time stamp -> point), the plane-map publisher, the viewer's region buffers, the
// batched frame and the mesh's change feed.  Include inside an anonymous namespace of a translation unit that includes common_host.hpp (IM_LAUNCH).
#pragma once
#define VG_TILE 2048
#define VG_THREADS 256
#include "block_scan.cuh"

// ---- stable LSD radix sort, 8-bit digits.  hist is digit-major: hist[d * ntiles + t].  Each kernel has a variant (_dev) that reads
// the count from the device: block b takes tiles b, b + gridDim.x, ... of the count's tiles, so that any grid gives the same result
// (a grid that covers a capacity gives each block at most one tile; a smaller one keeps the cost with the count).
__device__ __forceinline__ void rs_hist_tile(const unsigned int* __restrict__ keys, int n, int shift, int* hist, int ntiles, int tile) {
    __shared__ int h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int base = tile * VG_TILE;
    for (int r = 0; r < VG_TILE / VG_THREADS; ++r) {
        const int i = base + r * VG_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255u], 1);
    }
    __syncthreads();
    hist[threadIdx.x * ntiles + tile] = h[threadIdx.x];   // each thread reads back only its own digit before the next tile clears it
}
__global__ void __launch_bounds__(VG_THREADS) k_rs_hist(const unsigned int* __restrict__ keys, int n, int shift, int* hist, int nblocks) {
    rs_hist_tile(keys, n, shift, hist, nblocks, blockIdx.x);
}
__global__ void __launch_bounds__(VG_THREADS) k_rs_hist_dev(const unsigned int* __restrict__ keys, const int* n_dev, int shift, int* hist) {
    const int n = *n_dev, nb = (n + VG_TILE - 1) / VG_TILE;
    for (int t = blockIdx.x; t < nb; t += gridDim.x) rs_hist_tile(keys, n, shift, hist, nb, t);
}
// exclusive scan of `len` ints in place by ONE block (len <= a few 100 k); total -> *total_out if not null
__device__ __forceinline__ void rs_scan_block(int* a, int len, int* total_out) {
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < len; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < len ? a[i] : 0;
        const int excl = block_scan_1024(v) + s_carry;
        if (i < len) a[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total_out) *total_out = s_carry;
}
__global__ void __launch_bounds__(1024) k_rs_scan(int* a, int len, int* total_out) { rs_scan_block(a, len, total_out); }
__global__ void __launch_bounds__(1024) k_rs_scan_dev(int* a, const int* n_dev) { rs_scan_block(a, 256 * ((*n_dev + VG_TILE - 1) / VG_TILE), nullptr); }
__device__ __forceinline__ void rs_scatter_tile(const unsigned int* __restrict__ kin, const unsigned int* __restrict__ vin, unsigned int* kout, unsigned int* vout,
                                                int n, int shift, const int* __restrict__ hist, int ntiles, int tile) {
    __shared__ int run[256];                      // next free slot of every digit for this tile (global position)
    __shared__ int wcnt[VG_THREADS / 32][256];    // per-warp digit counts of the current round
    run[threadIdx.x] = hist[threadIdx.x * ntiles + tile];   // (the previous tile's last read of run[] is behind its final barrier)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int base = tile * VG_TILE;
    for (int r = 0; r < VG_TILE / VG_THREADS; ++r) {
        for (int w = 0; w < VG_THREADS / 32; ++w) wcnt[w][threadIdx.x] = 0;
        __syncthreads();
        const int i = base + r * VG_THREADS + threadIdx.x;
        const bool valid = i < n;
        unsigned int key = 0, val = 0;
        if (valid) { key = kin[i]; val = vin[i]; }
        const unsigned int d = valid ? ((key >> shift) & 255u) : (256u + (unsigned)lane);   // invalid lanes: singleton groups
        const unsigned int peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) wcnt[warp][d] = __popc(peers);
        __syncthreads();
        if (valid) {
            int off = run[d];
            for (int w = 0; w < warp; ++w) off += wcnt[w][d];
            kout[off + rank] = key;
            vout[off + rank] = val;
        }
        __syncthreads();
        int tot = 0;
        for (int w = 0; w < VG_THREADS / 32; ++w) tot += wcnt[w][threadIdx.x];
        run[threadIdx.x] += tot;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(VG_THREADS) k_rs_scatter(const unsigned int* __restrict__ kin, const unsigned int* __restrict__ vin, unsigned int* kout, unsigned int* vout,
                                                            int n, int shift, const int* __restrict__ hist, int nblocks) {
    rs_scatter_tile(kin, vin, kout, vout, n, shift, hist, nblocks, blockIdx.x);
}
__global__ void __launch_bounds__(VG_THREADS) k_rs_scatter_dev(const unsigned int* __restrict__ kin, const unsigned int* __restrict__ vin, unsigned int* kout,
                                                                unsigned int* vout, const int* n_dev, int shift, const int* __restrict__ hist) {
    const int n = *n_dev, nb = (n + VG_TILE - 1) / VG_TILE;
    for (int t = blockIdx.x; t < nb; t += gridDim.x) rs_scatter_tile(kin, vin, kout, vout, n, shift, hist, nb, t);
}
// the LSD passes over the low `passes` 8-bit digits of the n keys in k[cur] (values in v[cur]), each from one buffer of the pairs into
// the other; hist holds 256 * ceil(n / VG_TILE) ints.  Returns the index of the buffers that hold the sorted pairs.  n_dev: the count
// is read on the device (*n_dev <= n), and n is the capacity; the grids cover it, or have dev_grid blocks when dev_grid > 0.
inline int rs_sort_passes(cudaStream_t st, unsigned int* const k[2], unsigned int* const v[2], int cur, int n, int passes, int* hist, const int* n_dev = nullptr,
                          int dev_grid = 0) {
    const int nb = (n + VG_TILE - 1) / VG_TILE;
    const int gd = dev_grid > 0 ? dev_grid : nb;
    for (int pass = 0; pass < passes; ++pass) {
        if (n_dev) {
            IM_LAUNCH(k_rs_hist_dev, gd, VG_THREADS, 0, st, (const unsigned int*)k[cur], n_dev, 8 * pass, hist);
            IM_LAUNCH(k_rs_scan_dev, 1, 1024, 0, st, hist, n_dev);
            IM_LAUNCH(k_rs_scatter_dev, gd, VG_THREADS, 0, st, (const unsigned int*)k[cur], (const unsigned int*)v[cur], k[cur ^ 1], v[cur ^ 1], n_dev, 8 * pass, (const int*)hist);
        } else {
            IM_LAUNCH(k_rs_hist, nb, VG_THREADS, 0, st, (const unsigned int*)k[cur], n, 8 * pass, hist, nb);
            IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, hist, 256 * nb, (int*)nullptr);
            IM_LAUNCH(k_rs_scatter, nb, VG_THREADS, 0, st, (const unsigned int*)k[cur], (const unsigned int*)v[cur], k[cur ^ 1], v[cur ^ 1], n, 8 * pass, (const int*)hist, nb);
        }
        cur ^= 1;
    }
    return cur;
}
