// immesh_b200 -- the kernels that turn one depth image into its points in ascending pixel order (depth_frame.cuh's bodies), shared by
// the mesh's depth frames (mesh_capi.cu: world points, the frame's FrameDyn set from the count) and the localization's front-end
// (frontend_capi.cu: sensor-frame points, filtered as Preprocess::l515_handler does, into the VoxelGrid handle's input ring).
//   k_depth_count  the valid samples per block of DF_BLOCK consecutive sampled pixels
//   (scan)         their offsets, total behind them: the one-block exclusive scan (k_rf_scan in mesh_capi.cu, k_rs_scan elsewhere)
//   k_depth_keep   with a filter only: each valid sample's global index (block offset + rank), so that the decimation and blind can be
//                  evaluated; the kept samples per block, then the scan again for their offsets
//   k_depth_emit   each kept sample's point at its block's offset plus its rank in the block; block 0 writes the count
// point_filter_num = 1 and blind = 0 keep every valid sample: then the keep pass is not launched and valid_off serves as keep_off.
// Include inside the anonymous namespace of a translation unit, after handles.hpp (depth_frame.cuh, mesh_core.cuh) and radix_sort.cuh
// (block_scan_1024).
#pragma once

#define DF_BLOCK 1024

__global__ void __launch_bounds__(DF_BLOCK) k_depth_count(const immesh::DepthFrame* df, int* blk) {
    const immesh::DepthFrame& D = *df;
    const int k = blockIdx.x * DF_BLOCK + threadIdx.x;
    float p[3];
    const int c = __syncthreads_count(k < D.sw * D.sh && immesh::depth_point(D, k, p));
    if (threadIdx.x == 0) blk[blockIdx.x] = c;
}
__global__ void __launch_bounds__(DF_BLOCK) k_depth_keep(const immesh::DepthFrame* df, const int* valid_off, int point_filter_num, double blind, int* kblk) {
    const immesh::DepthFrame& D = *df;
    const int k = blockIdx.x * DF_BLOCK + threadIdx.x;
    float p[3];
    const bool ok = k < D.sw * D.sh && immesh::depth_point(D, k, p);
    const int i = valid_off[blockIdx.x] + block_scan_1024(ok ? 1 : 0);
    const int c = __syncthreads_count(ok && immesh::depth_keep(i, p, point_filter_num, blind));
    if (threadIdx.x == 0) kblk[blockIdx.x] = c;
}
// keep_off[nb] is the count: to *n_out, and with dyn (a mesh frame) the frame's n, step, m and cmask (frame_append_dims)
__global__ void __launch_bounds__(DF_BLOCK) k_depth_emit(const immesh::DepthFrame* df, const int* valid_off, const int* keep_off, int nb, int point_filter_num,
                                                         double blind, int append_target, immesh::FrameDyn* dyn, float* pts, int* n_out) {
    const immesh::DepthFrame& D = *df;
    const int k = blockIdx.x * DF_BLOCK + threadIdx.x;
    float p[3];
    const bool ok = k < D.sw * D.sh && immesh::depth_point(D, k, p);
    bool keep = ok;
    if (point_filter_num > 1 || blind > 0.0) {   // uniform
        const int i = valid_off[blockIdx.x] + block_scan_1024(ok ? 1 : 0);
        keep = ok && immesh::depth_keep(i, p, point_filter_num, blind);
        __syncthreads();   // block_scan_1024's shared words are read by every thread before the next scan writes them
    }
    const int j = keep_off[blockIdx.x] + block_scan_1024(keep ? 1 : 0);
    if (keep) { pts[(size_t)j * 3 + 0] = p[0]; pts[(size_t)j * 3 + 1] = p[1]; pts[(size_t)j * 3 + 2] = p[2]; }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const int n = keep_off[nb];
        *n_out = n;
        if (dyn) {
            dyn->n = n;
            immesh::frame_append_dims(n, append_target, &dyn->step, &dyn->m, &dyn->cmask);
        }
    }
}
