// immesh_b200 -- the batched frame (one frame of any size: append in chunks, per-voxel stage in batches) and the offline reconstruction
// of a point cloud.  CUDA kernels (sm_90a) and their host orchestration; the stages shared with the queued frame are in mesh_capi.cu.
#include <cmath>

#include "handles.hpp"

using namespace immesh;

// ---- the batched frame (immesh_mesh_push_frame_batched): one frame, append in chunks, per-voxel stage in batches.  The frame-level
// counters of the per-frame path are accumulated across chunks / batches in the IM_MC_BAT_* slots and written back by k_bat_frame_end.
__global__ void k_bat_chunk_begin(MeshDev M, FrameBuf F) {   // the candidate grid of one append chunk after the first
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (unsigned int i = tid; i <= F.cmask; i += nt) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    if (tid == 0) mesh_cnt_bat_chunk_begin(M);
}
__global__ void k_bat_chunk_end(MeshDev M) { mesh_cnt_bat_chunk_end(M); }
// activation rule over every activated voxel of the frame (after the last chunk); the meshed ones with their keys
__global__ void __launch_bounds__(128) k_bat_select(MeshDev M, FrameBuf F, int* sel, unsigned long long* key) {
    const int na = min(M.cnt[IM_MC_ACT], F.max_act);
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < na; a += gridDim.x * blockDim.x) {
        const int vs = F.act[a];
        if (!voxel_activate(M, F, vs)) continue;
        const int k = atomicAdd(&M.cnt[IM_MC_BAT_SELECTED], 1);
        sel[k] = vs;
        key[k] = M.vkeys[vs];
    }
}
// sort word of position i: half 0 / 1 = low / high 32 bits of the key (LSD order)
__global__ void __launch_bounds__(128) k_bat_word(int n, int half, const unsigned long long* key, const unsigned int* vin, unsigned int* kout, unsigned int* vout) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vin ? vin[i] : (unsigned int)i;
        kout[i] = (unsigned int)(key[v] >> (32 * half));
        vout[i] = v;
    }
}
__global__ void k_bat_reset(MeshDev M, FrameBuf F, int clear_fset) {   // the per-batch lists
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    if (clear_fset) for (unsigned int i = tid; i <= F.fset_mask; i += nt) F.fset[i] = -1;
    if (tid == 0) mesh_cnt_bat_reset(M);
}
// meshed voxels [lo, hi) in key order -> the batch's work list; the rank is the flip priority
__global__ void __launch_bounds__(128) k_bat_fill(MeshDev M, FrameBuf F, const int* sel, const unsigned int* order, int lo, int hi, int* rank) {
    for (int r = lo + blockIdx.x * blockDim.x + threadIdx.x; r < hi; r += gridDim.x * blockDim.x) {
        const int w = voxel_enqueue(M, F, sel[order[r]]);
        if (w >= 0) rank[w] = r;
    }
}
// the batch's additions, pushed at once; marked so that later batches' pulls and commits do not see them as pre-frame triangles
__global__ void __launch_bounds__(128) k_bat_push_add(MeshDev M, FrameBuf F) {
    const int n = min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const int t = tri_add(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
        if (t >= 0) F.tri_mark[t] = IM_TRI_BORN;
    }
}
__global__ void k_bat_batch_end(MeshDev M) { mesh_cnt_bat_batch_end(M); }
// after the last batch: the deferred removals; every mark cleared for the next frame
__global__ void __launch_bounds__(128) k_bat_sweep(MeshDev M, FrameBuf F) {
    const int n = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const unsigned char m = F.tri_mark[t];
        if (!m) continue;
        if (m == IM_TRI_REMOVE) tri_remove(M, t);
        F.tri_mark[t] = 0;
    }
}
__global__ void k_bat_frame_end(MeshDev M) { mesh_cnt_bat_frame_end(M); }

// reconstruct_mesh_from_pointcloud (src/ImMesh_mesh_reconstruction.cpp:328-345, the offline entry of config/offline_pointcloud.yaml):
// the whole cloud is down-sampled by a pcl::VoxelGrid with leaf = minimum_pts_distance and meshed as ONE frame with the identity pose
// (Eigen::Quaterniond::Identity(), vec_3::Zero(), frame 0).  Both steps run on the device; the down-sampled cloud never leaves it.
int immesh_mesh_reconstruct_from_pointcloud(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int n, int on_device, double minimum_pts_distance, int* n_downsampled) {
    if (!h || !vg || (!xyz && n > 0) || n < 0 || !(minimum_pts_distance > 0)) return im_fail(IMMESH_E_INVALID, "bad argument");
    int m = 0, small = 0;
    int rc = immesh_voxelgrid_filter(vg, xyz, n, on_device, (float)minimum_pts_distance, nullptr, &m, &small);
    if (rc) return rc;
    if (n_downsampled) *n_downsampled = m;
    const double zero[3] = {0.0, 0.0, 0.0};
    return mesh_push_dev(h, immesh_voxelgrid_device_points(vg), m, zero, IMMESH_MFEED_KIND_RECONSTRUCT);
}

// scratch of the batched frame: sized by max_voxels, max_work, max_triangles and max_list, never by the frame
// (all or nothing: after a failure the handle has none of it)
static cudaError_t mesh_batched_scratch(immesh_mesh* h) {
    if (h->b_fp) return cudaSuccess;
    const size_t nv = (size_t)std::max(h->max_vox, 1), fcap = pow2_at_least((size_t)h->F.max_list * 2);
    immesh::MemSet b;
    int *act, *sel, *hist, *rank, *fset;
    unsigned long long* key;
    unsigned int *ku, *vu;
    unsigned char* mark;
    FramePose* fp;
    cudaError_t e;
    if ((e = b.alloc(&act, nv)) != cudaSuccess || (e = b.alloc(&sel, nv)) != cudaSuccess || (e = b.alloc(&key, nv)) != cudaSuccess ||
        (e = b.alloc(&ku, 2 * nv)) != cudaSuccess || (e = b.alloc(&vu, 2 * nv)) != cudaSuccess || (e = b.alloc(&hist, mesh_sort_hist_ints(nv))) != cudaSuccess ||
        (e = b.alloc(&rank, (size_t)h->F.max_work)) != cudaSuccess || (e = b.alloc(&mark, (size_t)h->M.max_t, 0)) != cudaSuccess ||
        (e = b.alloc(&fset, fcap, 0xFF)) != cudaSuccess || (e = b.alloc(&fp, 1)) != cudaSuccess)
        return e;
    // the initialising memsets ran on the legacy stream, which the handle's non-blocking streams do not wait for
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return e;
    h->b_act = act; h->b_sel = sel; h->b_key = key; h->b_ku = ku; h->b_vu = vu; h->b_hist = hist; h->b_rank = rank; h->b_mark = mark; h->b_fset = fset; h->b_fp = fp;
    h->b_fset_mask = (unsigned int)(fcap - 1);
    h->batch = std::move(b);
    return cudaSuccess;
}

// incremental_mesh_reconstruction (src/ImMesh_mesh_reconstruction.cpp:92-267) as ONE frame of any size: append in chunks of <= B
// candidates, then the per-voxel stage in batches of <= V meshed voxels (DESIGN.md, batched frame).  Blocking.
static int mesh_push_batched(immesh_mesh* h, const float* xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels, int64_t* stats,
                             int kind) {
    if (!h || (!xyz && n > 0) || n < 0 || !pose_t || batch_points < 0 || batch_points > h->max_frame_points || batch_voxels < 0 || batch_voxels > h->F.max_work)
        return im_fail(IMMESH_E_INVALID, "bad argument (batch_points in [0, max_frame_points], batch_voxels in [0, the frame's work capacity])");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "push_frame_batched: a sharded handle is not supported");
    const int prev = mesh_wait_impl(h, false);   // frames queued before this one
    if (prev) return prev;
    {   // growth before the frame only (m candidates at most); an overflow inside it stays IMMESH_E_CAPACITY
        const int64_t st0 = std::max<int64_t>(1, (int64_t)std::llround((double)(n / (int64_t)h->P.append_target)));
        const int grc = mesh_growth_check(h, n > 0 ? (n + st0 - 1) / st0 : 0);
        if (grc) return grc;
    }
    IM_CUDA(mesh_batched_scratch(h));
    const MeshParams& P = h->P;
    const int B = batch_points ? batch_points : h->max_frame_points, V = batch_voxels ? batch_voxels : h->F.max_work;
    // append_point_step = max(1, round(N / appending_pts_frame)), integer division first (ImMesh_mesh_reconstruction.cpp:111), 64-bit
    const int64_t step = std::max<int64_t>(1, (int64_t)std::llround((double)(n / (int64_t)P.append_target)));
    if (step > 0x7fffffff) return im_fail(IMMESH_E_INVALID, "push_frame_batched: append step out of range");
    const int64_t m_total = n > 0 ? (n + step - 1) / step : 0;
    cudaStream_t st = h->stream;
    FrameBuf F = h->F;
    F.dyn = nullptr;
    F.epoch = 0;
    F.act = h->b_act; F.max_act = h->max_vox;
    F.work_rank = h->b_rank; F.tri_mark = h->b_mark;
    F.fset = h->b_fset; F.fset_mask = h->b_fset_mask;
    F.fp = h->b_fp;
    F.frame = ++h->frame_counter;   // one frame: one frame number, one vox_frame stamp
    FramePose fp;
    for (int j = 0; j < 3; ++j) { fp.pose_t[j] = pose_t[j]; fp.prio_origin[j] = 0; }
    IM_CUDA(cudaMemcpyAsync(h->b_fp, &fp, sizeof(FramePose), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(h->M.cnt + IM_MC_BAT_VERTICES, 0, (IM_MC_BAT_SELECTED + 1 - IM_MC_BAT_VERTICES) * sizeof(int), st));
    const bool fd_on = h->feed.on != 0;   // a header and the pose: the reinforcement and the view do not follow batched frames
    if (fd_on) {
        const int rc = mesh_feed_stage(h, F.frame & (IM_SLOTS - 1), F.frame, n, (int)step, kind, pose_t, false, false);
        if (rc) return rc;
        mesh_feed_begin_launch(h, st);
    }
    // ---- append, chunk c = candidates [c B, (c + 1) B), candidate i = point i step.  Host input: gathered into the pinned slot c & 1
    // while the device works on the other one
    const size_t slot_pts = (size_t)h->max_frame_points * 3;
    int64_t chunks = 0;
    for (int64_t c0 = 0; c0 < m_total || chunks == 0; c0 += B, ++chunks) {
        const int m = (int)std::min<int64_t>(B, m_total - c0);
        FrameBuf Fc = F;
        Fc.m = m; Fc.n = m;
        Fc.cmask = (unsigned)(pow2_at_least((size_t)std::max(m, 1) * 2) - 1);
        const int s = (int)(chunks & 1);
        if (m > 0 && !on_device) {
            float* hs = h->h_pts + s * slot_pts;
            float* ds = h->d_pts + s * slot_pts;
            if (chunks >= 2) IM_CUDA(cudaEventSynchronize(h->ev_up[s]));   // the slot's previous upload has left the pinned buffer
            if (step == 1) std::memcpy(hs, xyz + (size_t)c0 * 3, (size_t)m * 3 * sizeof(float));
            else for (int i = 0; i < m; ++i) std::memcpy(hs + (size_t)i * 3, xyz + (size_t)(c0 + i) * step * 3, 3 * sizeof(float));
            if (chunks >= 2) IM_CUDA(cudaStreamWaitEvent(h->stream_up, h->ev_in[s], 0));   // the chunk that read the slot has finished
            IM_CUDA(upload_async(ds, hs, (size_t)m * 3 * sizeof(float), nullptr, h->stream_up, h->ev_up[s], st));
            Fc.pts = ds; Fc.step = 1;
        } else {
            Fc.pts = xyz ? xyz + (size_t)c0 * step * 3 : nullptr;
            Fc.step = (int)step;
        }
        if (chunks == 0) mesh_frame_begin_launch(h, Fc, st, false);
        else IM_LAUNCH(k_bat_chunk_begin, h->n_sm * 8, 256, 0, st, h->M, Fc);
        if (m > 0) mesh_append_launch(h, Fc, mesh_grid(h, m, 128), st, false);
        IM_LAUNCH(k_bat_chunk_end, 1, 1, 0, st, h->M);
        if (m > 0 && !on_device) IM_CUDA(cudaEventRecord(h->ev_in[s], st));
    }
    if (m_total == 0) chunks = 0;
    // ---- the activation rule after the last chunk; the meshed voxels in ascending key order
    IM_LAUNCH(k_bat_select, mesh_grid(h, h->max_vox, 128), 128, 0, st, h->M, F, h->b_sel, h->b_key);
    int nsel = 0;
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(&nsel, h->M.cnt + IM_MC_BAT_SELECTED, sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    unsigned int* ku[2] = {h->b_ku, h->b_ku + h->max_vox};
    unsigned int* vu[2] = {h->b_vu, h->b_vu + h->max_vox};
    int cur = 0;
    if (nsel > 0) {
        const int g = mesh_grid(h, nsel, 128);
        for (int half = 0; half < 2; ++half) {
            IM_LAUNCH(k_bat_word, g, 128, 0, st, nsel, half, (const unsigned long long*)h->b_key, half == 0 ? (const unsigned int*)nullptr : (const unsigned int*)vu[cur],
                      ku[cur ^ 1], vu[cur ^ 1]);
            cur = mesh_sort_passes(st, ku, vu, cur ^ 1, nsel, 4, h->b_hist);
        }
    }
    const unsigned int* order = vu[cur];
    const int nbat = (nsel + V - 1) / V;
    const int g_fill = mesh_grid(h, V, 128);
    // ---- pass 0: every dilation of the frame, with its smoothing store, before any orientation.  Pass 1: the dilation lists again
    // (the smoothing reads raw positions: the re-store writes the same bits), triangulation, pull + commit against the pre-frame store,
    // the batch's additions pushed at once
    for (int pass = 0; pass < 2; ++pass) {
        for (int b = 0; b < nbat; ++b) {
            IM_LAUNCH(k_bat_reset, pass ? h->n_sm * 8 : 1, pass ? 256 : 32, 0, st, h->M, F, pass);
            IM_LAUNCH(k_bat_fill, g_fill, 128, 0, st, h->M, F, (const int*)h->b_sel, order, b * V, std::min(nsel, (b + 1) * V), h->b_rank);
            mesh_dilate_launch(h, F, st, false);
            if (!pass) continue;
            if (const int rc = mesh_tri_launch(h, F, st, false)) return rc;
            IM_LAUNCH(k_bat_push_add, h->n_sm * 2, 128, 0, st, h->M, F);
            IM_LAUNCH(k_bat_batch_end, 1, 1, 0, st, h->M);
        }
    }
    IM_LAUNCH(k_bat_sweep, h->n_sm * 8, 128, 0, st, h->M, F);
    IM_LAUNCH(k_bat_frame_end, 1, 1, 0, st, h->M);
    if (h->chg.on) {
        mesh_changes_launch(h, F, st, true);
        h->chg.last_frame = F.frame;
    }
    if (fd_on) mesh_feed_launch(h, st, false, false);
    IM_CUDA(cudaGetLastError());
    if (fd_on) IM_CUDA(mesh_feed_commit(h, F.frame));
    int cnt[IM_MC_HOST];
    IM_CUDA(cudaMemcpyAsync(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    std::memcpy(h->last_cnt, cnt, sizeof(cnt));
    if (h->grow_max_bytes > 0) mesh_note(h, cnt, F.frame);
    if (stats) { stats[0] = chunks; stats[1] = nbat; stats[2] = (int64_t)h->batch.bytes(); stats[3] = cnt[IM_MC_ADD]; }
    return mesh_status(cnt[IM_MC_ERR]);
}

int immesh_mesh_push_frame_batched(immesh_mesh_t* h, const float* world_xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels,
                                   int64_t* stats) {
    return mesh_push_batched(h, world_xyz, n, on_device, pose_t, batch_points, batch_voxels, stats, IMMESH_MFEED_KIND_BATCHED);
}

extern "C" int immesh_voxelgrid_leaf_too_small(immesh_voxelgrid_t* h, const float* xyz, int64_t n, int on_device, float leaf, int* too_small);   // frontend_capi.cu

int immesh_mesh_reconstruct_from_pointcloud_batched(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int64_t n, int on_device, double minimum_pts_distance,
                                                    int batch_points, int batch_voxels, int64_t* n_meshed_points) {
    if (!h || !vg || (!xyz && n > 0) || n < 0 || !(minimum_pts_distance > 0)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reconstruct_from_pointcloud_batched: a sharded handle is not supported");
    if (batch_points < 0 || batch_points > h->max_frame_points || batch_voxels < 0 || batch_voxels > h->F.max_work)
        return im_fail(IMMESH_E_INVALID, "bad argument (batch_points in [0, max_frame_points], batch_voxels in [0, the frame's work capacity])");
    if (n_meshed_points) *n_meshed_points = 0;
    const double zero[3] = {0.0, 0.0, 0.0};
    int small = 0;
    if (n > 0) {
        const int rc = immesh_voxelgrid_leaf_too_small(vg, xyz, n, on_device, (float)minimum_pts_distance, &small);
        if (rc) return rc;
    }
    if (small || n == 0) {   // PCL passes the cloud through: every raw point goes into the frame, whatever the VoxelGrid handle holds
        if (n_meshed_points) *n_meshed_points = n;
        return mesh_push_batched(h, xyz, n, on_device, zero, batch_points, batch_voxels, nullptr, IMMESH_MFEED_KIND_RECONSTRUCT_BATCHED);
    }
    int m = 0, small2 = 0;
    const int rc = n > 0x7fffffff ? IMMESH_E_CAPACITY : immesh_voxelgrid_filter(vg, xyz, (int)n, on_device, (float)minimum_pts_distance, nullptr, &m, &small2);
    if (rc == IMMESH_E_CAPACITY)
        return im_fail(IMMESH_E_CAPACITY, "reconstruct_from_pointcloud_batched: PCL down-samples this cloud and it holds more points than the VoxelGrid handle's max_points");
    if (rc) return rc;
    if (n_meshed_points) *n_meshed_points = m;
    return mesh_push_batched(h, immesh_voxelgrid_device_points(vg), m, 1, zero, batch_points, batch_voxels, nullptr, IMMESH_MFEED_KIND_RECONSTRUCT_BATCHED);
}

