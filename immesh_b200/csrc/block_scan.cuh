// immesh_b200 -- the one-block exclusive scans (device functions only: a translation unit can use them without the radix sort's kernels)
#pragma once

// exclusive scan of v over a block of 1024 threads, which all call it: warp shuffle, then a scan of the 32 warp totals in warp 0
__device__ __forceinline__ int block_scan_1024(int v) {
    __shared__ int s_warp[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += u;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int wv = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, wv, o);
            if (lane >= o) wv += u;
        }
        s_warp[lane] = wv;
    }
    __syncthreads();
    return (warp ? s_warp[warp - 1] : 0) + x - v;
}
// exclusive scan of n items by one block of 1024 threads in ONE pass: thread t owns a contiguous chunk of ceil(n/1024) items.
// count(c) is item c's value; emit(c, run) stores item c's offset run and returns its value.  Returns the offset after the thread's
// chunk (thread 1023: the total).
template <class Count, class Emit>
__device__ __forceinline__ int chunk_scan_1024(int n, Count count, Emit emit) {
    const int per = (n + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(lo + per, n);
    int mine = 0;
    for (int c = lo; c < hi; ++c) mine += count(c);
    int run = block_scan_1024(mine);
    for (int c = lo; c < hi; ++c) run += emit(c, run);
    return run;
}
