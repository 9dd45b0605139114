// immesh_b200 -- front-end in front of the hot path (SURVEY 8f-1): pcl::VoxelGrid centroid down-sampling of a scan on the
// device, replacing  m_downSizeFilterSurf.setInputCloud(m_feats_undistort); m_downSizeFilterSurf.filter(*m_feats_down_body);
// (/root/reference/src/voxel_mapping.cpp:1715, :1888-1889; mesher copy: src/ImMesh_mesh_reconstruction.cpp:335-338).
// Semantics = published algorithm of pcl::VoxelGrid<PointT>::applyFilter with default parameters (restated in
// oracle/orc_frontend.hpp, which this path matches bit for bit): float inverse leaf, float min/max box, int cell index
// idx = ijk . (1, dx, dx*dy), points grouped by idx in ascending order, float centroid per group with the points summed in
// ascending scan order (PCL's std::sort leaves that order unspecified; both sides define it as the stable order).
//
// Kernels (all HBM-streaming, 12 B in per point per pass):
//   k_vg_minmax   block min/max of the finite points -> ordered-int atomics               12 n bytes in
//   k_vg_setup    one thread: box -> min_b, div_b, multipliers, PCL's INT_MAX overflow test
//   k_vg_keys     idx per point (0xFFFFFFFF for non-finite points, sorted last and dropped)  12 n in, 8 n out
//   k_rs_hist / k_rs_scan / k_rs_scatter  x4   stable LSD radix sort of (idx, point index), 8-bit digits, 2048-element tiles;
//                 ranks inside a tile from __match_any_sync (warp) + per-warp digit counts (shared memory)   16 n in+out per pass
//   k_vg_heads / k_rs_scan / k_vg_head_pos   run heads -> output slots (tile counts + scan) -> start of every run
//   k_vg_centroid_warp   one warp per run: serial float sums in run order
// There is no CPU path: the entry points need a CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"

using immesh::im_fail;

namespace {

#include "radix_sort.cuh"
#include "depth_kernels.cuh"

struct VgGrid {
    int mn[3], mx[3];        // ordered-int encodings of the float box (atomicMin / atomicMax targets)
    int min_b[3], div_b[3];
    int mul[3];
    int too_small;           // PCL: "Leaf size is too small for the input dataset" -> output = input
    int n_finite;
    int m_out;
};

__device__ __forceinline__ int f2ord(float f) { const int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

__global__ void k_vg_reset(VgGrid* g) {
    if (threadIdx.x < 3) { g->mn[threadIdx.x] = 0x7fffffff; g->mx[threadIdx.x] = (int)0x80000000; }
    if (threadIdx.x == 0) { g->too_small = 0; g->n_finite = 0; g->m_out = 0; }
}
// n_dev (or null): the kernels from k_vg_minmax to k_vg_copy_if_small read the count there; n is then its upper bound, which sizes the grids
__global__ void __launch_bounds__(VG_THREADS) k_vg_minmax(const float* __restrict__ pts, int n, const int* n_dev, VgGrid* g) {
    if (n_dev) n = *n_dev;
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    int cnt = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        if (!finite3(x, y, z)) continue;
        mn[0] = fminf(mn[0], x); mn[1] = fminf(mn[1], y); mn[2] = fminf(mn[2], z);
        mx[0] = fmaxf(mx[0], x); mx[1] = fmaxf(mx[1], y); mx[2] = fmaxf(mx[2], z);
        ++cnt;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0 && cnt > 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { atomicMin(&g->mn[a], f2ord(mn[a])); atomicMax(&g->mx[a], f2ord(mx[a])); }
        atomicAdd(&g->n_finite, cnt);
    }
}
// applyFilter: box -> grid (float arithmetic exactly as PCL: products with the float inverse leaf, floor, int casts)
__global__ void k_vg_setup(VgGrid* g, float inv) {
    if (threadIdx.x != 0) return;
    if (g->n_finite == 0) { g->div_b[0] = g->div_b[1] = g->div_b[2] = 0; return; }
    float mn[3], mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = ord2f(g->mn[a]); mx[a] = ord2f(g->mx[a]); }
    const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1, dz = (long long)((mx[2] - mn[2]) * inv) + 1;
    if (dx * dy * dz > 2147483647LL) { g->too_small = 1; return; }
    for (int a = 0; a < 3; ++a) {
        g->min_b[a] = (int)floorf(mn[a] * inv);
        const int max_b = (int)floorf(mx[a] * inv);
        g->div_b[a] = max_b - g->min_b[a] + 1;
    }
    g->mul[0] = 1; g->mul[1] = g->div_b[0]; g->mul[2] = g->div_b[0] * g->div_b[1];
}
__global__ void __launch_bounds__(VG_THREADS) k_vg_keys(const float* __restrict__ pts, int n, const int* n_dev, const VgGrid* g, float inv, unsigned int* keys,
                                                         unsigned int* vals) {
    if (n_dev) n = *n_dev;
    const int mb0 = g->min_b[0], mb1 = g->min_b[1], mb2 = g->min_b[2], m1 = g->mul[1], m2 = g->mul[2];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
        unsigned int key = 0xFFFFFFFFu;
        if (finite3(x, y, z)) {
            const int i0 = (int)(floorf(x * inv) - (float)mb0), i1 = (int)(floorf(y * inv) - (float)mb1), i2 = (int)(floorf(z * inv) - (float)mb2);
            key = (unsigned int)(i0 + i1 * m1 + i2 * m2);
        }
        keys[i] = key;
        vals[i] = (unsigned int)i;
    }
}

// ---- runs of equal idx -> centroids
__global__ void __launch_bounds__(VG_THREADS) k_vg_heads(const unsigned int* __restrict__ keys, int n, const int* n_dev, int* tile_heads) {
    if (n_dev) n = *n_dev;
    __shared__ int s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    const int base = blockIdx.x * VG_TILE;
    int c = 0;
    for (int r = 0; r < VG_TILE / VG_THREADS; ++r) {
        const int i = base + r * VG_THREADS + threadIdx.x;
        if (i < n) {
            const unsigned int k = keys[i];
            if (k != 0xFFFFFFFFu && (i == 0 || keys[i - 1] != k)) ++c;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) tile_heads[blockIdx.x] = s_cnt;
}
// record where every run starts: head_pos[slot] (the sums are then taken by k_vg_centroid_warp)
__global__ void __launch_bounds__(VG_THREADS) k_vg_head_pos(const unsigned int* __restrict__ keys, int n, const int* n_dev, const int* __restrict__ tile_base,
                                                             int* head_pos) {
    if (n_dev) n = *n_dev;
    __shared__ int s_warp[VG_THREADS / 32];
    __shared__ int s_run;
    if (threadIdx.x == 0) s_run = tile_base[blockIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int base = blockIdx.x * VG_TILE;
    for (int r = 0; r < VG_TILE / VG_THREADS; ++r) {
        const int i = base + r * VG_THREADS + threadIdx.x;
        unsigned int k = 0xFFFFFFFFu;
        bool head = false;
        if (i < n) { k = keys[i]; head = k != 0xFFFFFFFFu && (i == 0 || keys[i - 1] != k); }
        const unsigned int hb = __ballot_sync(0xffffffffu, head);
        if (lane == 0) s_warp[warp] = __popc(hb);
        __syncthreads();
        int slot = s_run + __popc(hb & ((1u << lane) - 1u));
        for (int w = 0; w < warp; ++w) slot += s_warp[w];
        if (head) head_pos[slot] = i;
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < VG_THREADS / 32; ++w) t += s_warp[w]; s_run += t; }
        __syncthreads();
    }
}
// one warp per run: the lanes fetch 32 points of the run at once (the loads are what makes a thread-per-run loop slow: a dense
// leaf near the sensor holds hundreds of points, ~1 us of dependent misses each), then every lane adds the 32 values in
// run order from shuffles -- the float sum keeps the serial order of CentroidPoint, only the memory latency is taken off the chain.
__global__ void __launch_bounds__(VG_THREADS) k_vg_centroid_warp(const float* __restrict__ pts, const unsigned int* __restrict__ vals, const int* __restrict__ head_pos,
                                                                  const int* __restrict__ total_heads, const VgGrid* g, float* out,
                                                                  const float* __restrict__ inten, float* out_i) {
    const int lane = threadIdx.x & 31;
    const int m = *total_heads, n_valid = g->n_finite;
    const int nwarps = gridDim.x * (blockDim.x >> 5);
    for (int slot = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); slot < m; slot += nwarps) {
        const int b = head_pos[slot], e = (slot + 1 < m) ? head_pos[slot + 1] : n_valid;
        float sx = 0.f, sy = 0.f, sz = 0.f, si = 0.f;
        for (int c = b; c < e; c += 32) {
            const int i = c + lane;
            float x = 0.f, y = 0.f, z = 0.f, w = 0.f;
            if (i < e) {
                const unsigned int p = vals[i];
                x = pts[3 * (size_t)p]; y = pts[3 * (size_t)p + 1]; z = pts[3 * (size_t)p + 2];
                if (inten) w = inten[p];
            }
            const int cnt = min(32, e - c);
            if (inten) {
                for (int t = 0; t < cnt; ++t) {
                    sx += __shfl_sync(0xffffffffu, x, t); sy += __shfl_sync(0xffffffffu, y, t); sz += __shfl_sync(0xffffffffu, z, t);
                    si += __shfl_sync(0xffffffffu, w, t);
                }
            } else {
                for (int t = 0; t < cnt; ++t) {
                    sx += __shfl_sync(0xffffffffu, x, t); sy += __shfl_sync(0xffffffffu, y, t); sz += __shfl_sync(0xffffffffu, z, t);
                }
            }
        }
        if (lane == 0) {
            const float cnt = (float)(e - b);
            out[3 * (size_t)slot] = sx / cnt; out[3 * (size_t)slot + 1] = sy / cnt; out[3 * (size_t)slot + 2] = sz / cnt;
            if (inten) out_i[slot] = si / cnt;
        }
    }
}
__global__ void k_vg_finish(VgGrid* g, const int* total_heads, int n, const int* n_dev) {
    if (threadIdx.x == 0) g->m_out = g->too_small ? (n_dev ? *n_dev : n) : *total_heads;
}
__global__ void __launch_bounds__(VG_THREADS) k_vg_copy_if_small(const float* __restrict__ pts, int n, const int* n_dev, const VgGrid* g, float* out,
                                                                  const float* __restrict__ inten, float* out_i) {
    if (!g->too_small) return;
    if (n_dev) n = *n_dev;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < 3 * (size_t)n; i += (size_t)gridDim.x * blockDim.x) {
        out[i] = pts[i];
        if (inten && i < (size_t)n) out_i[i] = inten[i];
    }
}

// front of the front-end: strided input (x y z in the first three of `stride` floats) -> packed [n][3], with the KITTI laser
// calibration (voxel_mapping.cpp:1844-1859) applied on the way when preprocess/calib_laser is set.  dst_i != nullptr: the
// intensity isrc[i * istride] is packed into dst_i[i] beside it (the calibration copies the whole point, intensity included).
__global__ void __launch_bounds__(VG_THREADS) k_frontend_pack(const float* __restrict__ src, int n, int stride, int calib, float* __restrict__ dst,
                                                               const float* __restrict__ isrc, int istride, float* __restrict__ dst_i) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float x = src[(size_t)i * stride], y = src[(size_t)i * stride + 1], z = src[(size_t)i * stride + 2];
        if (calib) immesh::kitti_calib_point(&x, &y, &z);
        dst[3 * (size_t)i] = x; dst[3 * (size_t)i + 1] = y; dst[3 * (size_t)i + 2] = z;
        if (dst_i) dst_i[i] = isrc[(size_t)i * istride];
    }
}
// the depth IMU chain's undistorted cloud, x y z t -> packed [n][3]: *n_src points (the cloud in branches 2 and 3, else 0); block 0 sets
// the ring slot's count to *n_keep (the cloud in branch 3 only: the frame the mesher is handed)
__global__ void __launch_bounds__(VG_THREADS) k_dimu_pack(const float4* __restrict__ src, const int* n_src, const int* n_keep, float* __restrict__ dst, int* n_dst) {
    const int n = *n_src;
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_dst = *n_keep;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = src[i];
        dst[3 * (size_t)i] = p.x; dst[3 * (size_t)i + 1] = p.y; dst[3 * (size_t)i + 2] = p.z;
    }
}

}  // namespace

struct immesh_voxelgrid {
    int max_points = 0, nblocks_max = 0, n_sm = 132;
    cudaStream_t stream = nullptr;
    float* d_in = nullptr;       // staging for host input / packed (calibrated) cloud of immesh_frontend_prepare: the current slot of
    float* d_in_ring[8] = {};   // a ring of 8 (a mesh frame may still be reading the cloud of up to IM_SLOTS + 1 scans ago)
    int in_idx = 0;
    float* d_raw = nullptr;      // [max_points][4] strided input of immesh_frontend_prepare
    float* h_raw = nullptr;      // pinned staging for it
    cudaEvent_t ev_raw = nullptr; // the H2D copy out of h_raw has completed
    int raw_pending = 0;
    float* d_out = nullptr;      // [max_points][3]
    unsigned int *d_k[2] = {nullptr, nullptr}, *d_v[2] = {nullptr, nullptr};
    int* d_hist = nullptr;       // [256 * nblocks_max]
    int* d_tile = nullptr;       // [nblocks_max + 1]
    int* d_head = nullptr;       // [max_points] start of every run in the sorted order
    VgGrid* d_grid = nullptr;
    VgGrid* h_grid = nullptr;    // pinned
    float* h_pts = nullptr;      // pinned staging [max_points][3]
    int last_m = 0;
    int raw_stride = 4;          // floats per point that d_raw / h_raw hold (widened by the first _i call with wider host records)
    // intensity of the _i entry points, allocated by the first of them
    float* d_in_i_ring[8] = {};  // intensity of the cloud in d_in_ring[k], same order
    float* d_out_i = nullptr;    // [max_points] intensity of the down-sampled cloud d_out
    float* h_out_i = nullptr;    // pinned [max_points]
    long long calls = 0;         // calls that queued work on the handle (immesh_lio_frontend_cloud: has vg run another call since)
    // depth images (immesh_frontend_prepare_depth, immesh_lio_step_async_depth), allocated by the first of them: per ring slot, the
    // image's DepthFrame and the count of the filtered cloud the kernels write into d_in_ring[k]
    struct Depth {
        immesh::DepthFrame* d_df = nullptr;   // [8]
        immesh::DepthFrame* h_df = nullptr;   // pinned [8]
        int* d_n = nullptr;                   // [8] (immesh_voxelgrid_input_count)
        int* h_n = nullptr;                   // pinned: a count read back by immesh_frontend_prepare_depth
        int *blk = nullptr, *kblk = nullptr;  // [nb + 1] valid and kept samples per block of DF_BLOCK sampled pixels, scanned in place
        int has_n[8] = {};                    // 1: d_in_ring[k] holds a depth cloud, counted in d_n[k]
    } dep;
    immesh::MemSet dev, pinned{immesh::MemSet::Pinned};   // every buffer above
};

extern "C" {

int immesh_voxelgrid_create(int max_points, immesh_voxelgrid_t** out) {
    if (!out || max_points < 1) return im_fail(IMMESH_E_INVALID, "bad argument");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path"); }
    immesh::Building<immesh_voxelgrid> owner(new immesh_voxelgrid(), immesh_voxelgrid_destroy);   // every failure below releases what was created
    immesh_voxelgrid* h = owner.get();
    h->max_points = max_points;
    h->nblocks_max = (max_points + VG_TILE - 1) / VG_TILE;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    const size_t n = (size_t)max_points;
    for (int i = 0; i < 8; ++i) IM_CUDA(h->dev.alloc(&h->d_in_ring[i], n * 3));
    h->d_in = h->d_in_ring[0];
    IM_CUDA(h->dev.alloc(&h->d_out, n * 3));
    IM_CUDA(h->dev.alloc(&h->d_raw, n * 4));
    IM_CUDA(h->pinned.alloc(&h->h_raw, n * 4));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_raw, cudaEventDisableTiming));
    for (int i = 0; i < 2; ++i) {
        IM_CUDA(h->dev.alloc(&h->d_k[i], n));
        IM_CUDA(h->dev.alloc(&h->d_v[i], n));
    }
    IM_CUDA(h->dev.alloc(&h->d_hist, (size_t)256 * h->nblocks_max));
    IM_CUDA(h->dev.alloc(&h->d_tile, (size_t)h->nblocks_max + 1));
    IM_CUDA(h->dev.alloc(&h->d_head, n));
    IM_CUDA(h->dev.alloc(&h->d_grid, 1));
    IM_CUDA(h->pinned.alloc(&h->h_grid, 1));
    IM_CUDA(h->pinned.alloc(&h->h_pts, n * 3));
    *out = owner.release();
    return IMMESH_OK;
}

int immesh_voxelgrid_destroy(immesh_voxelgrid_t* h) {
    if (!h) return IMMESH_OK;
    cudaStreamSynchronize(h->stream);
    if (h->ev_raw) cudaEventDestroy(h->ev_raw);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return IMMESH_OK;
}

// the intensity buffers of the _i entry points, and host staging for records of `host_stride` floats (0: device input only).
// Allocated on first use, so that a handle that never carries intensity keeps the footprint it has at create.  Each of the two
// steps is all or nothing: after a failure the handle is as it was.
static int vg_intensity_alloc(immesh_voxelgrid* h, int host_stride) {
    const size_t n = (size_t)h->max_points;
    if (!h->d_out_i) {
        immesh::MemSet dev, pinned(immesh::MemSet::Pinned);
        float *ring[8], *d_out_i, *h_out_i;
        for (int i = 0; i < 8; ++i) IM_CUDA(dev.alloc(&ring[i], n));
        IM_CUDA(dev.alloc(&d_out_i, n));
        IM_CUDA(pinned.alloc(&h_out_i, n));
        std::copy(ring, ring + 8, h->d_in_i_ring);
        h->d_out_i = d_out_i;
        h->h_out_i = h_out_i;
        h->dev.take(std::move(dev));
        h->pinned.take(std::move(pinned));
    }
    if (host_stride > h->raw_stride) {
        immesh::MemSet dev, pinned(immesh::MemSet::Pinned);
        float *d_raw, *h_raw;
        IM_CUDA(dev.alloc(&d_raw, n * host_stride));
        IM_CUDA(pinned.alloc(&h_raw, n * host_stride));
        IM_CUDA(cudaDeviceSynchronize());   // no queued copy or pack still uses the narrower staging
        h->raw_pending = 0;
        h->dev.free(h->d_raw); h->pinned.free(h->h_raw);
        h->d_raw = d_raw; h->h_raw = h_raw; h->raw_stride = host_stride;
        h->dev.take(std::move(dev));
        h->pinned.take(std::move(pinned));
    }
    return IMMESH_OK;
}
// the point records the _i entry points take: `stride` floats, x y z in 0..2, intensity (and the time stamp, tcol >= 0) in columns
// of their own beyond them
static bool records_ok(int stride, int icol, int tcol) {
    if (stride < 4 || stride > 16 || icol < 3 || icol >= stride) return false;
    return tcol < 0 || (tcol >= 3 && tcol < stride && tcol != icol);
}

// queue the filter's launch sequence for the packed device cloud d_pts on stream st (no host synchronisation); inten != nullptr:
// the points' intensity ([n]), averaged into d_out_i.  n_dev != nullptr: the count is read on the device (*n_dev <= n; the grids and
// the sort's scratch cover n)
static int vg_enqueue(immesh_voxelgrid* h, const float* d_pts, int n, float leaf, cudaStream_t st, const float* inten = nullptr, const int* n_dev = nullptr) {
    ++h->calls;
    float* out_i = inten ? h->d_out_i : nullptr;
    const float inv = 1.0f / leaf;
    const int nb = (n + VG_TILE - 1) / VG_TILE;
    const int gs = std::min(nb * (VG_TILE / VG_THREADS), h->n_sm * 8);
    IM_LAUNCH(k_vg_reset, 1, 32, 0, st, h->d_grid);
    IM_LAUNCH(k_vg_minmax, gs, VG_THREADS, 0, st, d_pts, n, n_dev, h->d_grid);
    IM_LAUNCH(k_vg_setup, 1, 32, 0, st, h->d_grid, inv);
    IM_LAUNCH(k_vg_keys, gs, VG_THREADS, 0, st, d_pts, n, n_dev, (const VgGrid*)h->d_grid, inv, h->d_k[0], h->d_v[0]);
    const int cur = rs_sort_passes(st, h->d_k, h->d_v, 0, n, 4, h->d_hist, n_dev);
    IM_LAUNCH(k_vg_heads, nb, VG_THREADS, 0, st, (const unsigned int*)h->d_k[cur], n, n_dev, h->d_tile);
    IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, h->d_tile, nb, h->d_tile + h->nblocks_max);
    IM_LAUNCH(k_vg_head_pos, nb, VG_THREADS, 0, st, (const unsigned int*)h->d_k[cur], n, n_dev, (const int*)h->d_tile, h->d_head);
    IM_LAUNCH(k_vg_centroid_warp, h->n_sm * 4, VG_THREADS, 0, st, d_pts, (const unsigned int*)h->d_v[cur], (const int*)h->d_head,
              (const int*)(h->d_tile + h->nblocks_max), (const VgGrid*)h->d_grid, h->d_out, inten, out_i);
    IM_LAUNCH(k_vg_finish, 1, 32, 0, st, h->d_grid, (const int*)(h->d_tile + h->nblocks_max), n, n_dev);
    IM_LAUNCH(k_vg_copy_if_small, gs, VG_THREADS, 0, st, d_pts, n, n_dev, (const VgGrid*)h->d_grid, h->d_out, inten, out_i);
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}

int immesh_voxelgrid_filter(immesh_voxelgrid_t* h, const float* xyz, int n, int on_device, float leaf, float* out_xyz, int* m_out, int* leaf_too_small) {
    if (!h || (!xyz && n > 0) || n < 0 || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    if (m_out) *m_out = 0;
    if (leaf_too_small) *leaf_too_small = 0;
    h->last_m = 0;
    if (n == 0) return IMMESH_OK;
    cudaStream_t st = h->stream;
    const float* d_pts = xyz;
    if (!on_device) {
        std::memcpy(h->h_pts, xyz, (size_t)n * 3 * sizeof(float));
        IM_CUDA(cudaMemcpyAsync(h->d_in, h->h_pts, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
        d_pts = h->d_in;
    }
    const int rc = vg_enqueue(h, d_pts, n, leaf, st);
    if (rc) return rc;
    IM_CUDA(cudaMemcpyAsync(h->h_grid, h->d_grid, sizeof(VgGrid), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int m = h->h_grid->m_out;
    h->last_m = m;
    if (m_out) *m_out = m;
    if (leaf_too_small) *leaf_too_small = h->h_grid->too_small;
    if (out_xyz && m > 0) {
        IM_CUDA(cudaMemcpyAsync(h->h_pts, h->d_out, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
        std::memcpy(out_xyz, h->h_pts, (size_t)m * 3 * sizeof(float));
    }
    return IMMESH_OK;
}

// PCL's "leaf size too small" decision (k_vg_setup's index-overflow test) on a cloud of any size: the box of its finite points is reduced
// max_points at a time (host input through the handle's staging) by k_vg_minmax, whose order-free atomics accumulate across chunks, so
// the decision equals immesh_voxelgrid_filter's on the whole cloud.  Used by immesh_mesh_reconstruct_from_pointcloud_batched.
int immesh_voxelgrid_leaf_too_small(immesh_voxelgrid_t* h, const float* xyz, int64_t n, int on_device, float leaf, int* too_small) {
    if (!h || (!xyz && n > 0) || n < 0 || !(leaf > 0.f) || !too_small) return im_fail(IMMESH_E_INVALID, "bad argument");
    cudaStream_t st = h->stream;
    ++h->calls;
    IM_LAUNCH(k_vg_reset, 1, 32, 0, st, h->d_grid);
    for (int64_t c0 = 0; c0 < n; c0 += h->max_points) {
        const int m = (int)std::min<int64_t>(h->max_points, n - c0);
        const float* d = xyz + (size_t)c0 * 3;
        if (!on_device) {
            IM_CUDA(cudaStreamSynchronize(st));   // the previous chunk's copy out of the staging buffer is done
            std::memcpy(h->h_pts, d, (size_t)m * 3 * sizeof(float));
            IM_CUDA(cudaMemcpyAsync(h->d_in, h->h_pts, (size_t)m * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
            d = h->d_in;
        }
        const int gs = std::min(((m + VG_TILE - 1) / VG_TILE) * (VG_TILE / VG_THREADS), h->n_sm * 8);
        IM_LAUNCH(k_vg_minmax, gs, VG_THREADS, 0, st, d, m, (const int*)nullptr, h->d_grid);
    }
    IM_LAUNCH(k_vg_setup, 1, 32, 0, st, h->d_grid, 1.0f / leaf);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_grid, h->d_grid, sizeof(VgGrid), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    *too_small = h->h_grid->too_small;
    return IMMESH_OK;
}

// upload (host input) + pack / calibrate into d_in on stream st.  Intensity, packed into the ring slot beside d_in: column icol of
// the records (icol >= 0), or the separate device array isep ([n]).
static int frontend_pack(immesh_voxelgrid* h, const float* pts, int n, int stride, int on_device, int calib_laser, cudaStream_t st, int icol = -1,
                         const float* isep = nullptr) {
    const bool with_i = icol >= 0 || isep;
    if (with_i) {
        const int rc = vg_intensity_alloc(h, on_device ? 0 : stride);
        if (rc) return rc;
    }
    ++h->calls;
    h->in_idx = (h->in_idx + 1) & 7;
    h->d_in = h->d_in_ring[h->in_idx];
    h->dep.has_n[h->in_idx] = 0;
    const float* d_src = pts;
    if (!on_device) {
        const float* src = pts;
        if (!immesh::host_ptr_is_pinned(pts)) {
            if (h->raw_pending) { IM_CUDA(cudaEventSynchronize(h->ev_raw)); h->raw_pending = 0; }   // the previous copy out of the staging buffer
            std::memcpy(h->h_raw, pts, (size_t)n * stride * sizeof(float));
            src = h->h_raw;
        }
        IM_CUDA(cudaMemcpyAsync(h->d_raw, src, (size_t)n * stride * sizeof(float), cudaMemcpyHostToDevice, st));
        if (src == h->h_raw) { IM_CUDA(cudaEventRecord(h->ev_raw, st)); h->raw_pending = 1; }
        d_src = h->d_raw;
    }
    const float* isrc = icol >= 0 ? d_src + icol : isep;
    IM_LAUNCH(k_frontend_pack, std::min((n + VG_THREADS - 1) / VG_THREADS, h->n_sm * 8), VG_THREADS, 0, st, d_src, n, stride, calib_laser, h->d_in,
              isrc, icol >= 0 ? stride : 1, with_i ? h->d_in_i_ring[h->in_idx] : (float*)nullptr);
    return IMMESH_OK;
}

int immesh_frontend_prepare(immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float* out_xyz) {
    if (!h || (!pts && n > 0) || n < 0 || (stride != 3 && stride != 4)) return im_fail(IMMESH_E_INVALID, "bad argument (stride must be 3 or 4)");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    if (n == 0) return IMMESH_OK;
    int rc = frontend_pack(h, pts, n, stride, on_device, calib_laser, h->stream);
    if (rc) return rc;
    IM_CUDA(cudaGetLastError());
    if (out_xyz) {
        IM_CUDA(cudaMemcpyAsync(h->h_pts, h->d_in, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        IM_CUDA(cudaStreamSynchronize(h->stream));
        std::memcpy(out_xyz, h->h_pts, (size_t)n * 3 * sizeof(float));
    } else {
        IM_CUDA(cudaStreamSynchronize(h->stream));
    }
    return IMMESH_OK;
}
const float* immesh_voxelgrid_input_points(immesh_voxelgrid_t* h) { return h ? h->d_in : nullptr; }
const int* immesh_voxelgrid_input_count(immesh_voxelgrid_t* h) { return h && h->dep.has_n[h->in_idx] ? h->dep.d_n + h->in_idx : nullptr; }

// ---- depth images into the localization (immesh_frontend_prepare_depth, immesh_lio_step_async_depth): the image checked, then the
// kernels of depth_kernels.cuh queued on st into the next input ring slot -- the filtered sensor-frame cloud and its count, both on the
// device.  *n_sampled: the sampled pixels, the upper bound of the count.
// The argument checks of a depth frame, nothing queued: *d set up from the image, *n_sampled its sampled pixels.
static int depth_check(immesh_voxelgrid* h, const immesh_depth_frame* f, const void* img, int point_filter_num, double blind, immesh::DepthFrame* d,
                       long long* pitch, int* bpp, int* n_sampled) {
    if (point_filter_num < 1) return im_fail(IMMESH_E_INVALID, "depth frame: point_filter_num must be >= 1");
    if (!(blind >= 0.0 && std::isfinite(blind))) return im_fail(IMMESH_E_INVALID, "depth frame: blind must be finite and >= 0");
    if (const char* bad = immesh::depth_frame_setup(f, img, d, pitch, bpp)) return im_fail(IMMESH_E_INVALID, bad);
    if ((long long)d->sw * d->sh > h->max_points) return im_fail(IMMESH_E_CAPACITY, "depth frame: more sampled pixels than the VoxelGrid's max_points");
    *n_sampled = d->sw * d->sh;
    return IMMESH_OK;
}
// wait_ms (or null): the host time spent waiting for the previous image's copy out of the staging buffer is added there
static int depth_pack(immesh_voxelgrid* h, const immesh_depth_frame* f, const void* img, int on_device, int point_filter_num, double blind, cudaStream_t st,
                      int* n_sampled, double* wait_ms = nullptr) {
    immesh::DepthFrame d;
    long long pitch = 0;
    int bpp = 0, ns = 0;
    if (const int rc = depth_check(h, f, img, point_filter_num, blind, &d, &pitch, &bpp, &ns)) return rc;
    auto& D = h->dep;
    if (!D.d_n) {   // all or nothing: after a failure the handle is as it was
        const size_t nb = (size_t)(h->max_points + DF_BLOCK - 1) / DF_BLOCK;
        immesh::MemSet dev, pinned(immesh::MemSet::Pinned);
        immesh_voxelgrid::Depth b;
        IM_CUDA(dev.alloc(&b.d_df, 8));
        IM_CUDA(pinned.alloc(&b.h_df, 8));
        IM_CUDA(dev.alloc(&b.d_n, 8, 0));
        IM_CUDA(pinned.alloc(&b.h_n, 1));
        IM_CUDA(dev.alloc(&b.blk, nb + 1));
        IM_CUDA(dev.alloc(&b.kblk, nb + 1));
        D.d_df = b.d_df; D.h_df = b.h_df; D.d_n = b.d_n; D.h_n = b.h_n; D.blk = b.blk; D.kblk = b.kblk;
        h->dev.take(std::move(dev));
        h->pinned.take(std::move(pinned));
    }
    ++h->calls;
    h->in_idx = (h->in_idx + 1) & 7;
    const int k = h->in_idx;
    h->d_in = h->d_in_ring[k];
    if (!on_device) {   // the sampled grid, tight, through the pinned staging (sw * sh * bpp <= 4 max_points bytes, within h_raw)
        if (h->raw_pending) {   // the previous copy out of the staging buffer
            const auto t0 = std::chrono::steady_clock::now();
            IM_CUDA(cudaEventSynchronize(h->ev_raw));
            if (wait_ms) *wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            h->raw_pending = 0;
        }
        unsigned char* hb = reinterpret_cast<unsigned char*>(h->h_raw);
        immesh::depth_stage_grid(d, static_cast<const unsigned char*>(img), pitch, bpp, hb);
        IM_CUDA(cudaMemcpyAsync(h->d_raw, hb, (size_t)ns * bpp, cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaEventRecord(h->ev_raw, st));
        h->raw_pending = 1;
        d.img = reinterpret_cast<const unsigned char*>(h->d_raw);
        d.row_bytes = (long long)d.sw * bpp;
        d.col_bytes = bpp;
    }
    // the pinned slot k was last copied from 8 calls ago, behind which the localization's staging slots have since been waited on
    D.h_df[k] = d;
    IM_CUDA(cudaMemcpyAsync(D.d_df + k, D.h_df + k, sizeof(immesh::DepthFrame), cudaMemcpyHostToDevice, st));
    const int nb = (ns + DF_BLOCK - 1) / DF_BLOCK;
    const bool filter = point_filter_num > 1 || blind > 0.0;
    const immesh::DepthFrame* df = D.d_df + k;
    IM_LAUNCH(k_depth_count, nb, DF_BLOCK, 0, st, df, D.blk);
    IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, D.blk, nb, D.blk + nb);
    if (filter) {
        IM_LAUNCH(k_depth_keep, nb, DF_BLOCK, 0, st, df, (const int*)D.blk, point_filter_num, blind, D.kblk);
        IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, D.kblk, nb, D.kblk + nb);
    }
    IM_LAUNCH(k_depth_emit, nb, DF_BLOCK, 0, st, df, (const int*)D.blk, (const int*)(filter ? D.kblk : D.blk), nb, point_filter_num, blind, 0,
              (immesh::FrameDyn*)nullptr, h->d_in, D.d_n + k);
    D.has_n[k] = 1;
    *n_sampled = ns;
    return IMMESH_OK;
}

int immesh_frontend_prepare_depth(immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num, double blind,
                                  float* out_xyz, int cap, int* n_out) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !out_xyz)) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    int ns = 0;
    int rc = depth_pack(h, f, depth, on_device, point_filter_num, blind, h->stream, &ns);
    if (rc) return rc;
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->dep.h_n, h->dep.d_n + h->in_idx, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    const int n = *h->dep.h_n;
    *n_out = n;
    if (cap == 0) return IMMESH_OK;
    if (n > cap) return im_fail(IMMESH_E_CAPACITY, "more filtered points than cap");
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(h->h_pts, h->d_in, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        IM_CUDA(cudaStreamSynchronize(h->stream));
        std::memcpy(out_xyz, h->h_pts, (size_t)n * 3 * sizeof(float));
    }
    return IMMESH_OK;
}

int immesh_voxelgrid_filter_i(immesh_voxelgrid_t* h, const float* pts, int n, int stride, int intensity_col, int on_device, float leaf, float* out_xyzi, int* m_out,
                              int* leaf_too_small) {
    if (!h || (!pts && n > 0) || n < 0 || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!records_ok(stride, intensity_col, -1)) return im_fail(IMMESH_E_INVALID, "bad records (stride <= 16; intensity_col >= 3 and < stride)");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    if (m_out) *m_out = 0;
    if (leaf_too_small) *leaf_too_small = 0;
    h->last_m = 0;
    if (n == 0) return IMMESH_OK;
    cudaStream_t st = h->stream;
    int rc = frontend_pack(h, pts, n, stride, on_device, 0, st, intensity_col);
    if (rc) return rc;
    rc = vg_enqueue(h, h->d_in, n, leaf, st, h->d_in_i_ring[h->in_idx]);
    if (rc) return rc;
    IM_CUDA(cudaMemcpyAsync(h->h_grid, h->d_grid, sizeof(VgGrid), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int m = h->h_grid->m_out;
    h->last_m = m;
    if (m_out) *m_out = m;
    if (leaf_too_small) *leaf_too_small = h->h_grid->too_small;
    if (out_xyzi && m > 0) {
        IM_CUDA(cudaMemcpyAsync(h->h_pts, h->d_out, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaMemcpyAsync(h->h_out_i, h->d_out_i, (size_t)m * sizeof(float), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
        for (int j = 0; j < m; ++j) {
            std::memcpy(out_xyzi + 4 * (size_t)j, h->h_pts + 3 * (size_t)j, 3 * sizeof(float));
            out_xyzi[4 * (size_t)j + 3] = h->h_out_i[j];
        }
    }
    return IMMESH_OK;
}

// The device-resident front-end chain of one scan (SURVEY 8f-1), queued on the localization handle's stream with no host round
// trip: [KITTI laser calibration] -> pcl::VoxelGrid -> predict + IESKF iterations + map update.  The down-sampled cloud and its
// size never leave the device (the step reads the count from the filter's result block).
// internal (also immesh_lio_step_async_imu): the chain with the intensity of column icol of the records, or of the separate device
// array isep, carried beside the clouds; then the step is what immesh_lio_frontend_cloud publishes from
int immesh_frontend_step_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float leaf,
                               double dt, double cov_gyr, double cov_acc, int icol, const float* isep) {
    const bool with_i = icol >= 0 || isep;
    lio->fe_vg = nullptr;
    cudaStream_t st = lio->stream;
    int rc = frontend_pack(h, pts, n, stride, on_device, calib_laser, st, icol, isep);
    if (rc) return rc;
    rc = vg_enqueue(h, h->d_in, n, leaf, st, with_i ? h->d_in_i_ring[h->in_idx] : nullptr);
    if (rc) return rc;
    // the scan feed's full scan (registered source 2): the calibrated input cloud immesh_voxelgrid_input_points returns, with its
    // intensity on the _i chains; the IMU chain has set its own kind and branch
    immesh_lio::FeedNext& nx = lio->feed_next;
    if (nx.kind < 0) { nx.kind = with_i ? IMMESH_FEED_KIND_RAW_I : IMMESH_FEED_KIND_RAW; nx.branch = 0; }
    nx.pts = h->d_in;
    nx.inten = with_i ? h->d_in_i_ring[h->in_idx] : nullptr;
    nx.n = n;
    rc = immesh_lio_step_async_dev_n(lio, h->d_out, n < lio->max_scan ? n : lio->max_scan, &h->d_grid->m_out, dt, cov_gyr, cov_acc);
    lio->feed_next = immesh_lio::FeedNext();
    if (rc || !with_i) return rc;
    lio->fe_vg = h;
    lio->fe_uploads = lio->uploads;
    lio->fe_vg_calls = h->calls;
    lio->fe_n = n;
    return IMMESH_OK;
}
int immesh_lio_step_async_raw(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* pts, int n, int stride, int on_device, int calib_laser, float leaf,
                              double dt, double cov_gyr, double cov_acc) {
    if (!lio || !h || (!pts && n > 0) || n < 1 || (stride != 3 && stride != 4) || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    return immesh_frontend_step_async(lio, h, pts, n, stride, on_device, calib_laser, leaf, dt, cov_gyr, cov_acc, -1, nullptr);
}
// The chain of one depth image (the reference's lidar_type 4, imu_en false): unproject + filter -> pcl::VoxelGrid -> predict + IESKF +
// map update, every count on the device.  A frame with no point left is predicted only (the step's *d_n == 0 path).
int immesh_lio_step_async_depth(immesh_lio_t* lio, immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num,
                                double blind, float leaf, double dt, double cov_gyr, double cov_acc) {
    if (!lio || !h || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_depth runs on a single GPU: the localization handle is sharded");
    lio->fe_vg = nullptr;
    cudaStream_t st = lio->stream;
    int ns = 0;
    int rc = depth_pack(h, f, depth, on_device, point_filter_num, blind, st, &ns);
    if (rc) return rc;
    const int* d_n = h->dep.d_n + h->in_idx;
    rc = vg_enqueue(h, h->d_in, ns, leaf, st, nullptr, d_n);
    if (rc) return rc;
    immesh_lio::FeedNext& nx = lio->feed_next;   // the scan feed's full scan (registered source 2): the filtered cloud, counted on the device
    nx.kind = IMMESH_FEED_KIND_DEPTH;
    nx.branch = 0;
    nx.pts = h->d_in;
    nx.inten = nullptr;
    nx.n = ns;
    nx.n_dev = d_n;
    rc = immesh_lio_step_async_dev_n(lio, h->d_out, ns < lio->max_scan ? ns : lio->max_scan, &h->d_grid->m_out, dt, cov_gyr, cov_acc);
    lio->feed_next = immesh_lio::FeedNext();
    return rc;
}
int immesh_lio_step_async_raw_i(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* pts, int n, int stride, int intensity_col, int on_device, int calib_laser,
                                float leaf, double dt, double cov_gyr, double cov_acc) {
    if (!lio || !h || !pts || n < 1 || !(leaf > 0.f)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!records_ok(stride, intensity_col, -1)) return im_fail(IMMESH_E_INVALID, "bad records (stride <= 16; intensity_col >= 3 and < stride)");
    if (lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_step_async_raw_i runs on a single GPU: the localization handle is sharded");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    return immesh_frontend_step_async(lio, h, pts, n, stride, on_device, calib_laser, leaf, dt, cov_gyr, cov_acc, intensity_col, nullptr);
}

int immesh_lio_registered_cloud_sep(immesh_lio_t* h, const float* d_xyz, const float* d_inten, int n, int point_skip, float* rows, int cap, int* n_out);   // lio_capi.cu
int immesh_lio_frontend_cloud(immesh_lio_t* lio, immesh_voxelgrid_t* vg, int dense, int point_skip, float* rows, int cap, int* n_out) {
    if (!lio || !vg || !n_out || cap < 0 || (cap > 0 && !rows) || point_skip <= 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    if (lio->P.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_lio_frontend_cloud: the localization handle is sharded");
    if (lio->fe_vg != vg || lio->fe_uploads != lio->uploads || lio->fe_vg_calls != vg->calls)
        return im_fail(IMMESH_E_INVALID, "immesh_lio_frontend_cloud: the last step on the localization handle was not an intensity-carrying (_i) front-end chain "
                                         "through this VoxelGrid handle, or the VoxelGrid handle has run another call since");
    if (dense) return immesh_lio_registered_cloud_sep(lio, vg->d_in, vg->d_in_i_ring[vg->in_idx], lio->fe_n, point_skip, rows, cap, n_out);
    return immesh_lio_registered_cloud_sep(lio, nullptr, vg->d_out_i, 0, point_skip, rows, cap, n_out);
}

const float* immesh_voxelgrid_device_points(immesh_voxelgrid_t* h) { return h ? h->d_out : nullptr; }

// internal (immesh_lio_step_async_imu): capacity of the handle, and voxel_map_init queued on the localization stream from a device
// cloud -- [calibration] + repack into the input ring (immesh_voxelgrid_input_points), then the build kernels on the packed full scan
int immesh_voxelgrid_max_points(immesh_voxelgrid_t* h) { return h ? h->max_points : 0; }
int immesh_voxelmap_build_async_dev(immesh_lio_t* lio, const float* d_body_xyz, int n);   // lio_capi.cu
// internal (immesh_lio_step_async_depth_imu): the depth frame's checks (*n_sampled: its sampled pixels), and its cloud queued on the
// localization stream into the next input ring slot (*d_xyz, count *d_n on the device)
int immesh_frontend_depth_check(immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int point_filter_num, double blind, int* n_sampled) {
    immesh::DepthFrame d;
    long long pitch = 0;
    int bpp = 0;
    return depth_check(h, f, depth, point_filter_num, blind, &d, &pitch, &bpp, n_sampled);
}
int immesh_frontend_depth_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const immesh_depth_frame* f, const void* depth, int on_device, int point_filter_num,
                                double blind, const float** d_xyz, const int** d_n) {
    lio->fe_vg = nullptr;
    int ns = 0;
    const int rc = depth_pack(h, f, depth, on_device, point_filter_num, blind, lio->stream, &ns, &lio->host_wait_ms);   // staging back-pressure
    if (rc) return rc;
    *d_xyz = h->d_in;
    *d_n = h->dep.d_n + h->in_idx;
    return IMMESH_OK;
}
// internal (immesh_lio_step_async_depth_imu): the chain behind UndistortPcl, every branch launched and every count read on the device.
// d_xyzt: the undistorted cloud, *d_und points (0 unless branch 2 or 3); *d_b2 / *d_b3: the cloud's count in branch 2 / 3, else 0.
//   pack        -> back into the input ring slot immesh_frontend_depth_async unprojected into (one slot per call, as on every chain: a
//                  mesh frame may still read the slot of up to IM_SLOTS + 1 calls ago), its count *d_b3 (the mesher's frame)
//   voxel_map_init of *d_b2 points (builds nothing unless branch 2; records no scan)
//   VoxelGrid(leaf) of *d_b3 points -> predict (dt 0: none) + IESKF + map update of the down-sampled cloud: nothing unless branch 3.  Its
//   scan is the frame's one scan-feed record, with the device branch.
int immesh_voxelmap_build_async_dev_n(immesh_lio_t* h, const float* d_body_xyz, int n_max, const int* d_n);   // lio_capi.cu
int immesh_frontend_depth_imu_tail(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* d_xyzt, int n_max, const int* d_und, const int* d_b2, const int* d_b3,
                                   const int* d_branch, float leaf) {
    cudaStream_t st = lio->stream;
    lio->fe_vg = nullptr;
    const int k = h->in_idx;   // the k_dimu_expand of the same call has read the unprojected cloud out of it
    IM_LAUNCH(k_dimu_pack, std::min((n_max + VG_THREADS - 1) / VG_THREADS, h->n_sm * 8), VG_THREADS, 0, st, (const float4*)d_xyzt, d_und, d_b3, h->d_in,
              h->dep.d_n + k);
    int rc = immesh_voxelmap_build_async_dev_n(lio, h->d_in, n_max, d_b2);
    if (rc) return rc;
    rc = vg_enqueue(h, h->d_in, n_max, leaf, st, nullptr, d_b3);
    if (rc) return rc;
    immesh_lio::FeedNext& nx = lio->feed_next;   // the scan feed's full scan (registered source 2): the undistorted cloud, as for the IMU chain
    nx.kind = IMMESH_FEED_KIND_DEPTH_IMU;
    nx.branch = 0;
    nx.branch_dev = d_branch;
    nx.pts = h->d_in;
    nx.inten = nullptr;
    nx.n = n_max;
    nx.n_dev = d_b3;
    rc = immesh_lio_step_async_dev_n(lio, h->d_out, n_max < lio->max_scan ? n_max : lio->max_scan, &h->d_grid->m_out, 0.0, 0.0, 0.0);
    lio->feed_next = immesh_lio::FeedNext();
    return rc;
}

int immesh_frontend_build_async(immesh_lio_t* lio, immesh_voxelgrid_t* h, const float* d_pts, int n, int stride, int calib_laser, const float* d_inten) {
    if (!lio || !h || !d_pts || n < 1 || (stride != 3 && stride != 4)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_points) return im_fail(IMMESH_E_CAPACITY, "cloud larger than max_points");
    const int rc = frontend_pack(h, d_pts, n, stride, 1, calib_laser, lio->stream, -1, d_inten);
    if (rc) return rc;
    const int brc = immesh_voxelmap_build_async_dev(lio, h->d_in, n);   // takes the IMU chain's feed_next (branch 2)
    lio->feed_next = immesh_lio::FeedNext();
    return brc;
}

}  // extern "C"
