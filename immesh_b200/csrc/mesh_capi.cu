// immesh_b200 -- the mesher's handle and frame chain (create / destroy, mesh_enqueue and the push entry points, growth, sharding,
// counters): CUDA kernels (sm_90a, bodies in mesh_core.cuh / mesh_voxel.cuh) and C-ABI host orchestration.  No CPU path.
#include <chrono>
#include <cmath>
#include <cstdlib>

#include "block_scan.cuh"
#include "handles.hpp"
#include "nccl_api.hpp"
#include "pdl.cuh"
#include "pool_growth.cuh"

using namespace immesh;

// ------------------------------------------------------------------ kernels
__global__ void k_frame_begin(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (unsigned int i = tid; i <= F.cmask; i += nt) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    for (unsigned int i = tid; i <= F.fset_mask; i += nt) F.fset[i] = -1;
    if (tid == 0) mesh_cnt_frame_begin(M);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_init(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_init(M, P, F, c);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_conflicts(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_conflicts(M, P, F, c);
    pdl_trigger();
}
// Priority polling: candidate c waits only on candidates with a smaller index.  Blocks take tickets so that the
// block holding the smallest undecided candidate is always resident; a poll cap turns a (never observed) livelock
// into an error flag instead of a hang.
__global__ void __launch_bounds__(128) k_cand_resolve(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ int s_ticket;
    const int nblocks = (F.m + blockDim.x - 1) / blockDim.x;
    while (true) {
        if (threadIdx.x == 0) s_ticket = atomicAdd(&M.cnt[IM_MC_RESOLVE_TICKET], 1);
        __syncthreads();
        const int b = s_ticket;
        __syncthreads();
        if (b >= nblocks) break;
        const int c = b * blockDim.x + threadIdx.x;
        if (c < F.m && F.cand_status[c] == CAND_UNDECIDED) {
            int polls = 0;
            while (!cand_poll(M, P, F, c)) {
                if (++polls > (1 << 22)) { atomicOr(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); atomicAdd(&M.cnt[IM_MC_UNDECIDED], 1); break; }
                __nanosleep(64);
            }
            __threadfence();
        }
    }
    pdl_trigger();
}

// the accept flags into the candidates' output ranks
__global__ void __launch_bounds__(1024) k_cand_scan(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    chunk_scan_1024(F.m, [&](int c) { return F.cand_status[c] == CAND_ACCEPT ? 1 : 0; },
                    [&](int c, int run) { F.cand_scan[c] = run; return F.cand_status[c] == CAND_ACCEPT ? 1 : 0; });
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_commit(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[IM_MC_VERTICES];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_commit(M, P, F, c, base);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_place(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[IM_MC_VERTICES];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_place(M, F, c, base);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_voxel_select(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int na = min(M.cnt[IM_MC_ACT], F.max_act);
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < na; a += gridDim.x * blockDim.x) voxel_select(M, F, a);
    pdl_trigger();
}
// stage A: dilation (exact 20-NN of the in-voxel vertices + smoothing); one block per (voxel, group of <= 8 queries)
__global__ void __launch_bounds__(128) k_voxel_dilate(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ DilateSmem S;
    __shared__ int s_item;
    const int ni = min(M.cnt[IM_MC_DITEMS], F.max_ditem);
    while (true) {
        if (threadIdx.x == 0) s_item = atomicAdd(&M.cnt[IM_MC_DILATE_TICKET], 1);
        __syncthreads();
        const int i = s_item;
        __syncthreads();
        if (i >= ni) break;
        voxel_dilate(M, P, F, F.ditem[i], &S, threadIdx.x, blockDim.x);
        __syncthreads();
    }
    pdl_trigger();
}
// stage B, small dilated sets: one warp per voxel (four independent voxels per block), voxels claimed dynamically
#define IM_WARP_NMAX 96
__global__ void __launch_bounds__(128) k_voxel_tri_warp(MeshDev M, MeshParams P, FrameBuf F_, int n_max) {
    const FrameBuf F = frame_load_dyn(F_);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    MeshWarpSmem<128>* S = reinterpret_cast<MeshWarpSmem<128>*>(smem_raw) + warp;
    const int nw = work_total(M, F);
    IM_STAMP(30, nw);
    int n_done = 0;
    while (true) {
        int i = 0;
        if (lane == 0) i = atomicAdd(&M.cnt[IM_MC_TRI_TICKET], 1);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= nw) break;
        voxel_mesh_warp<128>(M, P, F, work_slot(M, F, i), S, lane, 32, n_max);
        __syncwarp();
        ++n_done;
    }
    IM_STAMP(31, n_done);
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0 && (immesh_stamp_store(41, n_done), true), 42, nw);
}
// stage C (flat): after every voxel's smoothing is final
__global__ void __launch_bounds__(128) k_commit_faces(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int nf = min(M.cnt[IM_MC_FACES], F.max_list);
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += gridDim.x * blockDim.x) commit_face(M, P, F, f);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_pull_vertices(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int nr = min(M.cnt[IM_MC_VREFS], F.max_vref);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) pull_vertex(M, P, F, r);
}
__global__ void __launch_bounds__(128) k_pull_check(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int ne = min(M.cnt[IM_MC_PULLED], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < ne; e += gridDim.x * blockDim.x) pull_check(M, F, e);
    pdl_trigger();
}
template <int MAXD>
__global__ void __launch_bounds__(128) k_voxel_mesh(MeshDev M, MeshParams P, FrameBuf F_, int lo, int store_only) {
    const FrameBuf F = frame_load_dyn(F_);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MeshSmem<MAXD>* S = reinterpret_cast<MeshSmem<MAXD>*>(smem_raw);
    const int nw = work_total(M, F);
    for (int i = blockIdx.x; i < nw; i += gridDim.x) {
        const int w = work_slot(M, F, i);
        const int n = F.work_n_ids[w];
        const int na = n < 0 ? -n : n;
        if ((n < 0 && !store_only) || (n > 0 && na > lo && na <= MAXD)) voxel_mesh<MAXD>(M, P, F, w, S, threadIdx.x, blockDim.x, store_only);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(128) k_push_remove(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[IM_MC_REMOVE], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) tri_remove(M, F.rem_tri[e]);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_push_add(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x)
        tri_add(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
    pdl_trigger();
}
__global__ void k_frame_end(MeshDev M) {
    pdl_wait();
    mesh_cnt_frame_end(M);
}

// ---- depth-camera frames (immesh_mesh_push_depth): the kernels of depth_kernels.cuh without a filter; block 0 of k_depth_emit sets the
// frame's n, step, m and cmask in its FrameDyn, and the kernels after it read the device count.  Grids cover max_frame_points samples.
namespace {
#include "depth_kernels.cuh"
}

// ---- growth of the mesh pools (immesh_mesh_reserve): the three open-addressed tables rebuilt into tables of the new size
#define MGROW_THREADS 256
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_xi(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.gmask; s += gridDim.x * blockDim.x) rehash_xi_slot(from, to, s);
}
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_voxels(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.vmask; s += gridDim.x * blockDim.x) rehash_voxel_slot(from, to, s);
}
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_tris(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.tmask; s += gridDim.x * blockDim.x) rehash_tri_slot(from, to, s);
}

// ------------------------------------------------------------------ host side

#if defined(IM_DEBUG_STAMPS)
extern "C" int immesh_debug_stamps_mesh(long long* out64) {   // debug variant only (tools/debug/build_stamps.sh); not declared in include/
    return cudaMemcpyFromSymbol(out64, immesh::g_stamps, 64 * sizeof(long long)) == cudaSuccess ? 0 : -1;
}
#endif

int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    if (!cfg || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    if (!(cfg->points_minimum_scale > 0) || !(cfg->voxel_resolution > 0) || cfg->number_of_pts_append_to_map < 1) return im_fail(IMMESH_E_INVALID, "bad mesh configuration");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path");
    immesh::Building<immesh_mesh> owner(new immesh_mesh(), immesh_mesh_destroy);   // every failure below releases what was created
    immesh_mesh* h = owner.get();
    h->F.shard_rank = 0; h->F.shard_n = 1; h->F.x_cap = 0;
    h->F.work_rank = nullptr; h->F.tri_mark = nullptr;   // the per-frame path
    // dilated sets up to warp_nmax vertices are triangulated by one warp each (side stream), larger ones by a thread block each
    // (main stream, concurrently): the split balances the two kernels' longest serial insertion chains
    h->warp_nmax = std::getenv("IMMESH_WARP_NMAX") ? std::atoi(std::getenv("IMMESH_WARP_NMAX")) : IM_WARP_NMAX;
    if (h->warp_nmax < 3) h->warp_nmax = 3;
    if (h->warp_nmax > 128) h->warp_nmax = 128;
    h->use_graph = std::getenv("IMMESH_GRAPH") ? std::atoi(std::getenv("IMMESH_GRAPH")) : 1;
    MeshParams& P = h->P;
    P.xi = cfg->points_minimum_scale;
    P.res = cfg->voxel_resolution;
    P.accept = cfg->voxel_resolution * 1.25;
    P.knn_max = P.accept * 2 * 1.000001;
    P.inv_q = 4194304.0 / cfg->voxel_resolution;
    P.append_target = cfg->number_of_pts_append_to_map;
    const int max_v = cfg->max_vertices ? cfg->max_vertices : (8 << 20);
    const int max_t = cfg->max_triangles ? cfg->max_triangles : (32 << 20);
    const int max_vox = cfg->max_voxels ? cfg->max_voxels : (2 << 20);
    h->max_frame_points = cfg->max_frame_points ? cfg->max_frame_points : (2 << 20);
    h->max_vox = max_vox;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& e : h->ev) IM_CUDA(cudaEventCreate(&e));
    MeshDev& M = h->M;
    M.max_v = max_v;
    M.max_t = max_t;
    IM_CUDA(h->dev.alloc(&M.vpos, (size_t)max_v));
    IM_CUDA(h->dev.alloc(&M.vsmooth, (size_t)max_v * 3));
    IM_CUDA(h->dev.alloc(&M.vsmoothed, (size_t)max_v, 0));
    IM_CUDA(h->dev.alloc(&M.v_tri_head, (size_t)max_v, 0xFF));
    const size_t gcap = pow2_at_least((size_t)max_v * 2);
    IM_CUDA(h->dev.alloc(&M.gkeys, gcap, 0xFF));
    IM_CUDA(h->dev.alloc(&M.gval, gcap, 0xFF));
    M.gmask = (unsigned)(gcap - 1);
    const size_t vcap = pow2_at_least((size_t)max_vox * 2);
    IM_CUDA(h->dev.alloc(&M.vkeys, vcap, 0xFF));
    M.vmask = (unsigned)(vcap - 1);
    IM_CUDA(h->dev.alloc(&M.vox_chunk, vcap * IM_VCHUNKS, 0xFF));
    M.max_vchunks = max_v / 4 + 1024;
    IM_CUDA(h->dev.alloc(&M.vchunk_pts, (size_t)M.max_vchunks * 16));
    IM_CUDA(h->dev.alloc(&M.vox_count, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_meshing_times, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_new_added, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_frame, vcap, 0xFF));
    M.vox_short_axis = nullptr;
    IM_CUDA(h->dev.alloc(&M.tri, (size_t)max_t));
    IM_CUDA(h->dev.alloc(&M.tri_next, (size_t)max_t * 3));
    IM_CUDA(h->dev.alloc(&M.tri_flip, (size_t)max_t));
    const size_t tcap = pow2_at_least((size_t)max_t * 2);
    IM_CUDA(h->dev.alloc(&M.thash, tcap, 0xFF));
    M.tmask = (unsigned)(tcap - 1);
    IM_CUDA(h->dev.alloc(&M.cnt, IM_MC_ALLOC, 0));
    {
        int init[IM_MC_HOST] = {};
        mesh_cnt_init(init);
        IM_CUDA(cudaMemcpy(M.cnt, init, sizeof(init), cudaMemcpyHostToDevice));
    }
    FrameBuf& F = h->F;
    const size_t mc = (size_t)h->max_frame_points;  // candidates <= points
    F.max_cand = (int)mc;
    F.max_work = max_vox < (1 << 16) ? max_vox : std::min(std::max(max_vox / 16, 1 << 16), 1 << 18);   // voxels (re)meshed per frame; 4 KB of id list each
    F.max_act = (int)std::min<size_t>((size_t)max_vox, mc);
    F.max_list = 4 << 20;
    IM_CUDA(h->dev.alloc(&h->d_pts, IM_SLOTS * mc * 3));
    IM_CUDA(h->dev.alloc(&h->d_body, IM_SLOTS * mc * 3));   // staging of body-frame scans handed over by the localization handle (not allocated lazily: an allocation inside a frame stalls the pipeline)
    F.pts = h->d_pts;
    IM_CUDA(h->dev.alloc(&h->d_fp, IM_SLOTS));
    for (int i = 0; i < IM_SLOTS; ++i) { IM_CUDA(cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming)); IM_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming)); }
    IM_CUDA(h->dev.alloc(&F.cand_gkey, mc));
    IM_CUDA(h->dev.alloc(&F.cand_vslot, mc));
    IM_CUDA(h->dev.alloc(&F.cand_status, mc));
    IM_CUDA(h->dev.alloc(&F.cand_scan, mc));
    IM_CUDA(h->dev.alloc(&F.cand_conf, mc * IM_CONF_K));
    IM_CUDA(h->dev.alloc(&F.cand_nconf, mc));
    IM_CUDA(h->dev.alloc(&F.cand_next, mc));
    IM_CUDA(h->dev.alloc(&F.cand_pos, mc));
    h->ccap = pow2_at_least(mc * 2);
    IM_CUDA(h->dev.alloc(&F.ckeys, h->ccap));
    IM_CUDA(h->dev.alloc(&F.chead, h->ccap));
    F.scan_block = nullptr;
    IM_CUDA(h->dev.alloc(&F.act, (size_t)F.max_act));
    IM_CUDA(h->dev.alloc(&F.work, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_n_ids, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_ids, (size_t)F.max_work * IM_MAXD));
    IM_CUDA(h->dev.alloc(&F.work_nfaces, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_bits, (size_t)F.max_work * (IM_MAXG / 32), 0));
    IM_CUDA(h->dev.alloc(&F.work_ring, (size_t)F.max_work, 0));
    IM_CUDA(h->dev.alloc(&F.work_done, (size_t)F.max_work, 0));
    F.max_ditem = F.max_work * 4;
    IM_CUDA(h->dev.alloc(&F.ditem, (size_t)F.max_ditem));
    F.max_vref = 8 << 20;
    IM_CUDA(h->dev.alloc(&F.all_faces, (size_t)F.max_list));
    IM_CUDA(h->dev.alloc(&F.all_vref, (size_t)F.max_vref));
    IM_CUDA(h->dev.alloc(&F.pulled, (size_t)F.max_list * 2));
    F.fset_mask = (1u << 21) - 1;
    IM_CUDA(h->dev.alloc(&F.fset, (size_t)F.fset_mask + 1, 0xFF));
    IM_CUDA(h->dev.alloc(&F.work_axes, (size_t)F.max_work * 9));
    IM_CUDA(h->dev.alloc(&F.add_tri, (size_t)F.max_list * 3));
    IM_CUDA(h->dev.alloc(&F.add_flip, (size_t)F.max_list));
    IM_CUDA(h->dev.alloc(&F.rem_tri, (size_t)F.max_list));
    IM_CUDA(h->pinned.alloc(&h->h_pts, IM_SLOTS * mc * 3));
    IM_CUDA(h->pinned.alloc(&h->h_cnt, IM_SLOTS * IM_MC_HOST));
    IM_CUDA(h->pinned.alloc(&h->h_fp, IM_SLOTS));
    IM_CUDA(h->pinned.alloc(&h->h_dyn, IM_SLOTS));
    IM_CUDA(h->dev.alloc(&h->d_dyn, 1, 0));
    IM_CUDA(h->dev.alloc(&h->cam_ring, IM_RF_RING, 0));
    IM_CUDA(h->dev.alloc(&h->cam_ring_frame, IM_RF_RING, 0));
    F.dyn = h->d_dyn;
    F.epoch = 0;
    IM_CUDA(cudaFuncSetAttribute(k_voxel_mesh<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<1024>)));
    IM_CUDA(cudaFuncSetAttribute(k_voxel_tri_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(4 * sizeof(MeshWarpSmem<128>))));
    IM_CUDA(cudaFuncSetAttribute(k_voxel_mesh<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<256>)));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream3, cudaStreamNonBlocking));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream_up, cudaStreamNonBlocking));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CUDA(cudaEventCreateWithFlags(&h->ev_up[i], cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_join3, cudaEventDisableTiming));
    std::memset(h->last_cnt, 0, sizeof(h->last_cnt));
    IM_CUDA(cudaDeviceSynchronize());
    *out = owner.release();
    return IMMESH_OK;
}

int immesh_mesh_destroy(immesh_mesh_t* h) {
    if (!h) return IMMESH_OK;
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->graph.destroy();
    mesh_feed_free(h);   // after the drain: no queued kernel still writes the done word
    if (h->win.local) immesh::peer_window_close(h->win);
    if (h->nccl_comm && immesh::nccl().CommDestroy) immesh::nccl().CommDestroy(h->nccl_comm);
    for (int i = 0; i < IM_SLOTS; ++i) { if (h->ev_in[i]) cudaEventDestroy(h->ev_in[i]); if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]); }
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->stream2) cudaStreamDestroy(h->stream2);
    if (h->stream3) cudaStreamDestroy(h->stream3);
    if (h->stream_up) cudaStreamDestroy(h->stream_up);
    for (int i = 0; i < IM_SLOTS; ++i) if (h->ev_up[i]) cudaEventDestroy(h->ev_up[i]);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->ev_join3) cudaEventDestroy(h->ev_join3);
    delete h;
    return IMMESH_OK;
}

// resident blocks per SM of the persistent per-voxel kernels (headroom for the kernels on the other streams)
#define MESH_TRI_BPS 3      // k_voxel_tri_warp, k_voxel_mesh<256>
#define MESH_DILATE_BPS 3   // k_voxel_dilate

extern "C" {   // the kernels of the localization hand-off and the shard exchange: profiles and tools name them without a signature
// transformLidar of the full-resolution scan with the converged state (ImMesh_mesh_reconstruction.cpp:413 ->
// voxel_mapping_common.cpp:709-726): p_w = (float)( R (R_ext p + t_ext) + t ).  First kernel of a frame handed over by the
// localization handle: the pose is the one that scan converged to (LioCtrl::pose_ring, written by the last kernel of the
// scan's sequence; the localization stream may already be working on later scans).  Block 0 also derives the frame's sensor
// position + the origin of the flip-priority rank, and records the pose in the handle's camera ring (reinforce.cuh, rf_avr_pose).
// A count read on the device (FrameDyn::n_dev, immesh_mesh_push_frame_from_lio_async_dev_n): every block reads it there, and block 0 sets
// the frame's n, step, m and cmask from it (frame_append_dims) for the kernels after this one.
__global__ void __launch_bounds__(128) k_transform_full(LioParams P, const LioCtrl* ctrl, FrameBuf F_, double res, double (*cam_ring)[12], int* cam_ring_frame,
                                                        int append_target) {
    __shared__ double s[12];
    const FrameDyn d = *F_.dyn;
    const int n = d.n_dev ? *d.n_dev : d.n;
    if (d.n_dev && blockIdx.x == 0 && threadIdx.x == 0) {
        FrameDyn* w = const_cast<FrameDyn*>(F_.dyn);
        w->n = n;
        frame_append_dims(n, append_target, &w->step, &w->m, &w->cmask);
    }
    if (threadIdx.x < 12) s[threadIdx.x] = ctrl->pose_ring[d.pose_idx][threadIdx.x];
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < 3) {
        const double t = s[9 + threadIdx.x];
        d.fp->pose_t[threadIdx.x] = t;
        d.fp->prio_origin[threadIdx.x] = (long long)floor(t / res) - 1024;
    }
    if (blockIdx.x == 0 && threadIdx.x < 12) {
        cam_ring[d.frame % IM_RF_RING][threadIdx.x] = s[threadIdx.x];
        if (threadIdx.x == 0) cam_ring_frame[d.frame % IM_RF_RING] = d.frame;
    }
    const float* body = d.body;
    float* world = const_cast<float*>(d.pts);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double pb[3] = {(double)body[(size_t)i * 3 + 0], (double)body[(size_t)i * 3 + 1], (double)body[(size_t)i * 3 + 2]};
        double pw[3];
        body_to_world(P, s, s + 9, pb, pw);
        world[(size_t)i * 3 + 0] = (float)pw[0]; world[(size_t)i * 3 + 1] = (float)pw[1]; world[(size_t)i * 3 + 2] = (float)pw[2];
    }
}
// blocking localization calls (immesh_lio_estimate, set_state, ...) do not publish a pose: done on request, on the localization stream
__global__ void k_pose_publish(LioCtrl* ctrl, int idx) {
    if (threadIdx.x < 12) ctrl->pose_ring[idx][threadIdx.x] = ctrl->state[threadIdx.x];
}

// ---- multi-GPU exchange of the per-voxel stage (sharded mesher).  A segment = [16-B header: counts][entries, x_cap each].
struct XHeader { int n_smooth, n_face, n_rem, pad; };
__global__ void k_xhdr(MeshDev M, FrameBuf F_, XHeader* hdr) {
    const FrameBuf F = frame_load_dyn(F_);
    if (threadIdx.x == 0) {
        hdr->n_smooth = min(M.cnt[IM_MC_X_SMOOTHS], F.x_cap);
        hdr->n_face = min(M.cnt[IM_MC_X_FACES], F.x_cap);
        hdr->n_rem = min(M.cnt[IM_MC_X_REMS], F.x_cap);
        hdr->pad = 0;
    }
}
// ---- the same exchange over peer windows (peer_win.cuh): k_xpush stores the USED part of this rank's segment straight into
// slot `rank` of every rank's receive area (its own included) and the last block raises the epoch flag; the apply kernels
// wait on the flags of their peers.  Window: flag[2][8] u64 | pad to 256 | recv1[n][seg1_bytes] | recv2[n][seg2_bytes].
struct MeshPeers {
    unsigned char* w[IM_MAX_RANKS];
    int rank, n;          // n == 0: NCCL transport (no waiting inside the apply kernels)
    unsigned long long recv_off[2], seg_bytes[2];
};
__device__ __forceinline__ unsigned long long* meshwin_flag(unsigned char* w, int which, int src) { return (unsigned long long*)w + which * IM_MAX_RANKS + src; }
__device__ __forceinline__ void copy16(unsigned char* dst, const unsigned char* src, size_t n16, int tid, int nt) {
    for (size_t i = tid; i < n16; i += nt) ((uint4*)dst)[i] = ((const uint4*)src)[i];
}
__global__ void __launch_bounds__(256) k_xpush(MeshDev M, FrameBuf F_, const unsigned char* seg, int which, MeshPeers pe, int* done) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    __shared__ int s_last;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    const int n_smooth = min(M.cnt[IM_MC_X_SMOOTHS], F.x_cap), n_face = min(M.cnt[IM_MC_X_FACES], F.x_cap), n_rem = min(M.cnt[IM_MC_X_REMS], F.x_cap);
    for (int r = 0; r < pe.n; ++r) {
        unsigned char* dst = pe.w[r] + pe.recv_off[which] + (size_t)pe.rank * pe.seg_bytes[which];
        if (tid == 0) *(int4*)dst = make_int4(n_smooth, n_face, n_rem, 0);
        if (which == 0) {
            copy16(dst + 16, seg + 16, (size_t)n_smooth * 2, tid, nt);
        } else {
            copy16(dst + 16, seg + 16, (size_t)n_face, tid, nt);
            const size_t woff = 16 + (size_t)F.x_cap * 16, roff = 16 + (size_t)F.x_cap * 24;
            copy16(dst + woff, seg + woff, ((size_t)n_face + 1) / 2, tid, nt);
            copy16(dst + roff, seg + roff, (size_t)n_rem, tid, nt);
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(done, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (s_last) {
        if (threadIdx.x == 0) *done = 0;
        __threadfence_system();
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) immesh::st_release_sys(meshwin_flag(pe.w[threadIdx.x], which, pe.rank), epoch);
    }
}
__device__ __forceinline__ void mesh_wait_peers(const MeshPeers& pe, int which, unsigned long long epoch, int* err) {
    if (pe.n > 0) {
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) {
            immesh::wait_epoch(meshwin_flag(pe.w[pe.rank], which, threadIdx.x), epoch, err, IM_MERR_PEER_TIMEOUT);
        }
        __syncthreads();
    }
}
// smoothed positions written by the other ranks' dilations -> this rank's replica
__global__ void __launch_bounds__(256) k_apply_smooth(MeshDev M, FrameBuf F_, const unsigned char* recv, size_t seg_bytes, MeshPeers pe) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    mesh_wait_peers(pe, 0, epoch, &M.cnt[IM_MC_ERR]);
    for (int r = 0; r < F.shard_n; ++r) {
        if (r == F.shard_rank) continue;
        const unsigned char* seg = recv + (size_t)r * seg_bytes;
        const int n = __ldcg((const int*)seg);
        const double2* e = (const double2*)(seg + 16);
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            const double2 a = __ldcg(e + 2 * (size_t)i), b = __ldcg(e + 2 * (size_t)i + 1);   // {id|pad, x}, {y, z}
            const int id = (int)(__double_as_longlong(a.x) & 0xffffffffLL);
            store_smooth(M, id, a.y, b.x, b.y);
        }
    }
}
// facets / removals of ALL ranks (own segment included) -> add / remove lists of this rank's replica
__global__ void __launch_bounds__(256) k_apply_lists(MeshDev M, FrameBuf F_, const unsigned char* recv, size_t seg_bytes, MeshPeers pe) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    mesh_wait_peers(pe, 1, epoch, &M.cnt[IM_MC_ERR]);
    for (int r = 0; r < F.shard_n; ++r) {
        const unsigned char* seg = recv + (size_t)r * seg_bytes;
        const int4 h = __ldcg((const int4*)seg);   // n_smooth, n_face, n_rem, -
        const int4* face = (const int4*)(seg + 16);
        const unsigned long long* word = (const unsigned long long*)(seg + 16 + (size_t)F.x_cap * 16);
        const int4* rem = (const int4*)(seg + 16 + (size_t)F.x_cap * 24);
        const int nf = h.y, nr = h.z;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf + nr; i += gridDim.x * blockDim.x) {
            if (i < nf) { const int4 f = __ldcg(face + i); apply_face(M, F, f.x, f.y, f.z, __ldcg(word + i)); }
            else { const int4 t = __ldcg(rem + (i - nf)); apply_remove(M, F, t.x, t.y, t.z); }
        }
    }
}
}  // extern "C"

int mesh_status(int err) {
    if (err & (IM_MERR_VERT_POOL | IM_MERR_TRI_POOL | IM_MERR_HASH_FULL | IM_MERR_LIST_CAP | IM_MERR_VOXEL_CAP)) {
        // name every flag that fired: the caller can tell a full pool from a per-voxel working set over its cap
        std::string m = "mesh pool / per-voxel working-set overflow (flags:";
        if (err & IM_MERR_VERT_POOL) m += " VERT_POOL";
        if (err & IM_MERR_TRI_POOL) m += " TRI_POOL";
        if (err & IM_MERR_HASH_FULL) m += " HASH_FULL";
        if (err & IM_MERR_LIST_CAP) m += " LIST_CAP";
        if (err & IM_MERR_VOXEL_CAP) m += " VOXEL_CAP";
        m += ")";
        return im_fail(IMMESH_E_CAPACITY, m.c_str());
    }
    if (err & (IM_MERR_KEY_RANGE | IM_MERR_PRIO_RANGE)) return im_fail(IMMESH_E_RANGE, "mesh key out of range");
    if (err & IM_MERR_PEER_TIMEOUT) return im_fail(IMMESH_E_CUDA, "sharded mesher: a peer rank did not publish its segment in time (peer window epoch flag)");
    if (err & IM_MERR_FEED_INDEX) return im_fail(IMMESH_E_CUDA, "frame feed: internal error (a record slot outside its ring; nothing was written)");
    return IMMESH_OK;
}
// wait for the frame queued in slot s and take over its counters
static int mesh_harvest(immesh_mesh* h, int s) {
    if (!h->inflight[s]) return IMMESH_OK;
    if (cudaEventQuery(h->ev_done[s]) != cudaSuccess) {
        cudaGetLastError();
        const auto t0 = std::chrono::steady_clock::now();
        IM_CUDA(cudaEventSynchronize(h->ev_done[s]));
        h->host_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    h->inflight[s] = 0;
    std::memcpy(h->last_cnt, h->h_cnt + IM_MC_HOST * s, sizeof(h->last_cnt));
    if (h->grow_max_bytes > 0) mesh_note(h, h->last_cnt, h->h_dyn[s].frame);
    const int rc = mesh_status(h->last_cnt[IM_MC_ERR]);
    if (rc && !h->pending_rc) h->pending_rc = rc;
    return rc;
}

// ---- growth of the mesh pools.  Device bytes per record: vertex 109 (vpos 16, vsmooth 24, m_smoothed 1, incidence head 4, its
// share of the vertex chunks 64 at max_v / 4 chunks of 16 float4), plus the xi-grid at 12 B per slot over 2 max_v rounded up to a
// power of two; triangle 36 (record 16, incidence links 12, flip word 8) plus the triple hash at 4 B per slot over 2 max_t; mesh
// voxel 88 B per slot (key 8, 16 chunk ids 64, count / meshing_times / new_added / frame 16) over 2 max_voxels.  Every pool stops at
// IM_MPOOL_LIMIT records.
static size_t mesh_pool_bytes(const immesh_mesh* h, long long v, long long t, long long x) {
    const size_t gcap = pow2_at_least((size_t)v * 2), tcap = pow2_at_least((size_t)t * 2), vcap = pow2_at_least((size_t)x * 2);
    const size_t act = std::min<size_t>((size_t)x, (size_t)h->max_frame_points);
    return (size_t)v * 45 + gcap * 12 + ((size_t)v / 4 + 1024) * 16 * sizeof(float4) + (size_t)t * 36 + tcap * 4 + vcap * (8 + IM_VCHUNKS * 4 + 16) + act * 4;
}
// counters of frame number `frame`, finished (see note_counters of the localization handle)
void mesh_note(immesh_mesh* h, const int* c, int frame) {
    if (frame <= h->known_frame) return;
    h->max_step_tris = std::max(h->max_step_tris, c[IM_MC_TRIS_ALLOC] - h->known[IM_MC_TRIS_ALLOC]);   // over several frames: an upper bound of one
    std::memcpy(h->known, c, sizeof(h->known));
    h->known_frame = frame;
}
// Enlarge the pools to (vertices, triangles, voxels), each >= the current one: as lio_grow (lio_capi.cu) -- drain, allocate all,
// migrate on the stream, free the old buffers, drop the captured launch sequence.  The batched frame's scratch (sized by max_voxels
// and max_triangles) is freed, and allocated again at the new sizes by the next batched frame.
static int mesh_grow(immesh_mesh* h, long long verts, long long tris, long long vox) {
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "a sharded mesh handle cannot grow (its replicas would have to grow in lockstep)");
    if (verts > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "vertex pool: more than 2^30 vertices (32-bit vertex ids)");
    if (tris > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "triangle pool: more than 2^30 triangles (32-bit triangle ids)");
    if (vox > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "voxel hash: more than 2^30 mesh voxels (32-bit voxel ids)");
    MeshDev& M = h->M;
    const long long v0 = M.max_v, t0 = M.max_t, x0 = h->max_vox;
    const bool gv = verts > v0, gt = tris > t0, gx = vox > x0;
    if (!gv && !gt && !gx) return IMMESH_OK;
    verts = std::max(verts, v0); tris = std::max(tris, t0); vox = std::max(vox, x0);
    // the batched frame's scratch (h->batch) goes, so it is not part of the sum
    const size_t bytes = h->dev.bytes() - mesh_pool_bytes(h, v0, t0, x0) + mesh_pool_bytes(h, verts, tris, vox);
    if (h->grow_max_bytes > 0 && bytes > (size_t)h->grow_max_bytes) {
        const std::string pools = std::string(gv ? " vertex pool" : "") + (gt ? " triangle pool" : "") + (gx ? " voxel hash" : "");
        return im_fail(IMMESH_E_CAPACITY, ("growth of the" + pools + " to " + std::to_string(bytes) + " device bytes is above the ceiling of " +
                                           std::to_string(h->grow_max_bytes) + " (immesh_mesh_set_growth)").c_str());
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, c));
    const int nv = std::min(c[IM_MC_VERTICES], M.max_v), nt = std::min(c[IM_MC_TRIS_ALLOC], M.max_t), nch = std::min(c[IM_MC_VERT_CHUNKS], M.max_vchunks);
    MeshDev nm = M;
    FrameBuf nf = h->F;
    immesh::MemSet fresh;   // the new buffers, freed on every failure below
    const char* pool = "";
    const size_t gcap = pow2_at_least((size_t)verts * 2), tcap = pow2_at_least((size_t)tris * 2), vcap = pow2_at_least((size_t)vox * 2);
    const int vch = (int)(verts / 4 + 1024), act = (int)std::min<long long>(vox, h->max_frame_points);
    cudaError_t e = cudaSuccess;
    if (gv) {
        pool = "vertex pool";
        if ((e = fresh.alloc(&nm.vpos, verts)) == cudaSuccess && (e = fresh.alloc(&nm.vsmooth, verts * 3)) == cudaSuccess && (e = fresh.alloc(&nm.vsmoothed, verts)) == cudaSuccess &&
            (e = fresh.alloc(&nm.v_tri_head, verts)) == cudaSuccess && (e = fresh.alloc(&nm.vchunk_pts, (size_t)vch * 16)) == cudaSuccess && gcap > (size_t)M.gmask + 1 &&
            (e = fresh.alloc(&nm.gkeys, gcap)) == cudaSuccess)
            e = fresh.alloc(&nm.gval, gcap);
    }
    if (gt && e == cudaSuccess) {
        pool = "triangle pool";
        if ((e = fresh.alloc(&nm.tri, tris)) == cudaSuccess && (e = fresh.alloc(&nm.tri_next, tris * 3)) == cudaSuccess && (e = fresh.alloc(&nm.tri_flip, tris)) == cudaSuccess &&
            tcap > (size_t)M.tmask + 1)
            e = fresh.alloc(&nm.thash, tcap);
    }
    if (gx && e == cudaSuccess) {
        pool = "voxel hash";
        if (vcap > (size_t)M.vmask + 1 && (e = fresh.alloc(&nm.vkeys, vcap)) == cudaSuccess && (e = fresh.alloc(&nm.vox_chunk, vcap * IM_VCHUNKS)) == cudaSuccess &&
            (e = fresh.alloc(&nm.vox_count, vcap)) == cudaSuccess && (e = fresh.alloc(&nm.vox_meshing_times, vcap)) == cudaSuccess &&
            (e = fresh.alloc(&nm.vox_new_added, vcap)) == cudaSuccess)
            e = fresh.alloc(&nm.vox_frame, vcap);
        if (e == cudaSuccess && act > h->F.max_act) e = fresh.alloc(&nf.act, act);
    }
    // the change feed's per-triangle stamp and published byte follow the triangle pool
    immesh::MemSet cfresh;
    int* c_stamp = h->F.chg_stamp;
    unsigned char* c_pub = h->chg.C.pub;
    if (gt && h->chg.on && e == cudaSuccess) {
        pool = "triangle pool (change feed)";
        if ((e = cfresh.alloc(&c_stamp, tris)) == cudaSuccess) e = cfresh.alloc(&c_pub, tris);
    }
    auto fail = [&](cudaError_t err, const char* what) {
        return im_fail_alloc(err, (std::string(what) + ": " + cudaGetErrorString(err) + " during the growth; the handle is unchanged").c_str());
    };
    if (e != cudaSuccess) return fail(e, pool);
    cudaStream_t st = h->stream;
    const int g = h->n_sm * 16;
    auto migrate = [&]() -> cudaError_t {
        cudaError_t r = cudaSuccess;
#define MG(x) do { if ((r = (x)) != cudaSuccess) return r; } while (0)
        if (gv) {
            MG(cudaMemsetAsync(nm.vsmoothed, 0, (size_t)verts, st));
            MG(cudaMemsetAsync(nm.v_tri_head, 0xFF, (size_t)verts * 4, st));
            if (nv > 0) {
                MG(cudaMemcpyAsync(nm.vpos, M.vpos, (size_t)nv * sizeof(float4), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.vsmooth, M.vsmooth, (size_t)nv * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.vsmoothed, M.vsmoothed, (size_t)nv, cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.v_tri_head, M.v_tri_head, (size_t)nv * 4, cudaMemcpyDeviceToDevice, st));
            }
            if (nch > 0) MG(cudaMemcpyAsync(nm.vchunk_pts, M.vchunk_pts, (size_t)nch * 16 * sizeof(float4), cudaMemcpyDeviceToDevice, st));
            nm.max_v = (int)verts;
            nm.max_vchunks = vch;
            if (nm.gkeys != M.gkeys) {
                MG(cudaMemsetAsync(nm.gkeys, 0xFF, gcap * 8, st));
                MG(cudaMemsetAsync(nm.gval, 0xFF, gcap * 4, st));
                nm.gmask = (unsigned)(gcap - 1);
                IM_LAUNCH(k_rehash_xi, g, MGROW_THREADS, 0, st, M, nm);
            }
        }
        if (gt) {
            if (nt > 0) {
                MG(cudaMemcpyAsync(nm.tri, M.tri, (size_t)nt * sizeof(int4), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.tri_next, M.tri_next, (size_t)nt * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.tri_flip, M.tri_flip, (size_t)nt * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
            }
            if (c_pub != h->chg.C.pub) {
                MG(cudaMemsetAsync(c_stamp, 0xFF, (size_t)tris * 4, st));
                MG(cudaMemsetAsync(c_pub, 0, (size_t)tris, st));
                if (nt > 0) {
                    MG(cudaMemcpyAsync(c_stamp, h->F.chg_stamp, (size_t)nt * 4, cudaMemcpyDeviceToDevice, st));
                    MG(cudaMemcpyAsync(c_pub, h->chg.C.pub, (size_t)nt, cudaMemcpyDeviceToDevice, st));
                }
            }
            nm.max_t = (int)tris;
            if (nm.thash != M.thash) {
                MG(cudaMemsetAsync(nm.thash, 0xFF, tcap * 4, st));
                nm.tmask = (unsigned)(tcap - 1);
                IM_LAUNCH(k_rehash_tris, g, MGROW_THREADS, 0, st, M, nm);
            }
        }
        if (gx && nm.vkeys != M.vkeys) {
            MG(cudaMemsetAsync(nm.vkeys, 0xFF, vcap * 8, st));
            MG(cudaMemsetAsync(nm.vox_chunk, 0xFF, vcap * IM_VCHUNKS * 4, st));
            for (int* q : {nm.vox_count, nm.vox_meshing_times, nm.vox_new_added}) MG(cudaMemsetAsync(q, 0, vcap * 4, st));
            MG(cudaMemsetAsync(nm.vox_frame, 0xFF, vcap * 4, st));
            nm.vmask = (unsigned)(vcap - 1);
            IM_LAUNCH(k_rehash_voxels, g, MGROW_THREADS, 0, st, M, nm);
        }
        MG(cudaGetLastError());
        MG(cudaStreamSynchronize(st));
#undef MG
        return r;
    };
    e = migrate();
    if (e != cudaSuccess) return fail(e, "mesh migration");   // the old buffers were only read: the handle is as it was
    // the replaced buffers go; the new ones join the handle's device memory
    const std::pair<const void*, const void*> replaced[] = {   // (old, new)
        {M.vpos, nm.vpos}, {M.vsmooth, nm.vsmooth}, {M.vsmoothed, nm.vsmoothed}, {M.v_tri_head, nm.v_tri_head}, {M.vchunk_pts, nm.vchunk_pts},
        {M.gkeys, nm.gkeys}, {M.gval, nm.gval}, {M.tri, nm.tri}, {M.tri_next, nm.tri_next}, {M.tri_flip, nm.tri_flip}, {M.thash, nm.thash},
        {M.vkeys, nm.vkeys}, {M.vox_chunk, nm.vox_chunk}, {M.vox_count, nm.vox_count}, {M.vox_meshing_times, nm.vox_meshing_times},
        {M.vox_new_added, nm.vox_new_added}, {M.vox_frame, nm.vox_frame}, {h->F.act, nf.act}};
    for (const auto& r : replaced)
        if (r.first != r.second) h->dev.free(r.first);
    h->dev.take(std::move(fresh));
    if (c_pub != h->chg.C.pub) {
        h->chg.dev.free(h->F.chg_stamp);
        h->chg.dev.free(h->chg.C.pub);
        h->chg.dev.take(std::move(cfresh));
        h->F.chg_stamp = c_stamp;
        h->chg.C.pub = c_pub;
    }
    if (h->b_fp) {   // batched-frame scratch: allocated again at the new sizes by the next batched frame
        h->batch = immesh::MemSet();
        h->b_act = h->b_sel = h->b_rank = h->b_hist = h->b_fset = nullptr;
        h->b_key = nullptr; h->b_ku = h->b_vu = nullptr; h->b_mark = nullptr; h->b_fp = nullptr;
    }
    nf.max_act = std::max(h->F.max_act, act);
    M = nm;
    h->F.act = nf.act;
    h->F.max_act = nf.max_act;
    h->max_vox = (int)vox;
    h->growths++;
    h->graph.destroy();
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}
// Automatic growth (immesh_mesh_set_growth) before a frame of m candidates: mesh_growth_targets (pool_growth.cuh) on the counters of
// the last frame known to have finished; the handle is drained only when a pool is short.
int mesh_growth_check(immesh_mesh* h, long long m) {
    if (h->grow_max_bytes <= 0) return IMMESH_OK;
    long long steps = 1, m_max = m;
    for (int i = 1; i <= IM_SLOTS; ++i) {   // oldest frame first: consecutive frames give one frame's use each
        const int s = (h->frame_counter + i) & (IM_SLOTS - 1);
        if (!h->inflight[s]) continue;
        if (cudaEventQuery(h->ev_done[s]) == cudaSuccess) {
            mesh_note(h, h->h_cnt + IM_MC_HOST * s, h->h_dyn[s].frame);
        } else {
            ++steps;
            m_max = std::max<long long>(m_max, h->h_dyn[s].m);
        }
    }
    cudaGetLastError();   // cudaErrorNotReady of the queries
    for (int pass = 0; pass < 2; ++pass) {
        long long v = h->M.max_v, t = h->M.max_t, x = h->max_vox;
        mesh_growth_targets(h->known, steps, m_max, h->max_step_tris, &v, &t, &x);
        if (v == h->M.max_v && t == h->M.max_t && x == h->max_vox) return IMMESH_OK;
        if (pass == 1) return mesh_grow(h, v, t, x);
        IM_CUDA(cudaStreamSynchronize(h->stream));
        for (int i = 1; i <= IM_SLOTS; ++i) {
            const int s = (h->frame_counter + i) & (IM_SLOTS - 1);
            if (h->inflight[s]) mesh_note(h, h->h_cnt + IM_MC_HOST * s, h->h_dyn[s].frame);
        }
        steps = 1;
        m_max = m;
    }
    return IMMESH_OK;
}


// ---- the stages of the frame chain the batched frame shares (pdl: a programmatic dependent launch, see mesh_enqueue)
void mesh_frame_begin_launch(const immesh_mesh* h, const FrameBuf& F, cudaStream_t st, bool pdl) {
    IM_LAUNCH_PDL(pdl, k_frame_begin, h->n_sm * 8, 256, 0, st, h->M, F);
}
// the append of F.m candidates: grid g over the candidates
void mesh_append_launch(const immesh_mesh* h, const FrameBuf& F, int g, cudaStream_t st, bool pdl) {
    const MeshParams& P = h->P;
    IM_LAUNCH_PDL(pdl, k_cand_init, g, 128, 0, st, h->M, P, F);
    IM_LAUNCH_PDL(pdl, k_cand_conflicts, g, 128, 0, st, h->M, P, F);
    IM_LAUNCH_PDL(pdl, k_cand_resolve, h->n_sm * 4, 128, 0, st, h->M, P, F);
    IM_LAUNCH_PDL(pdl, k_cand_scan, 1, 1024, 0, st, h->M, F);
    IM_LAUNCH_PDL(pdl, k_cand_commit, g, 128, 0, st, h->M, P, F);
    IM_LAUNCH_PDL(pdl, k_cand_place, g, 128, 0, st, h->M, F);
}
void mesh_dilate_launch(const immesh_mesh* h, const FrameBuf& F, cudaStream_t st, bool pdl) {
    IM_LAUNCH_PDL(pdl, k_voxel_dilate, h->n_sm * MESH_DILATE_BPS, 128, 0, st, h->M, h->P, F);
}
// triangulation: small dilated sets warp-level on the side stream, mid-size ones block-level on the main stream, concurrently; then
// the rare large / handed-over ones (monolithic: triangulate + commit in shared memory), the commit and the pull check.  A failed
// fork or join returns before anything else is queued.
int mesh_tri_launch(const immesh_mesh* h, const FrameBuf& F, cudaStream_t st, bool pdl) {
    const MeshParams& P = h->P;
    IM_CUDA(cudaEventRecord(h->ev_fork, st));
    IM_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
    IM_CUDA(cudaStreamWaitEvent(h->stream3, h->ev_fork, 0));
    IM_LAUNCH(k_voxel_tri_warp, h->n_sm * MESH_TRI_BPS, 128, 4 * sizeof(MeshWarpSmem<128>), h->stream2, h->M, P, F, h->warp_nmax);
    IM_CUDA(cudaEventRecord(h->ev_join, h->stream2));
    IM_LAUNCH(k_pull_vertices, h->n_sm * 8, 128, 0, h->stream3, h->M, P, F);   // incidence-list walk: only needs the dilation
    IM_CUDA(cudaEventRecord(h->ev_join3, h->stream3));
    IM_LAUNCH((k_voxel_mesh<256>), h->n_sm * MESH_TRI_BPS, 128, sizeof(MeshSmem<256>), st, h->M, P, F, h->warp_nmax, 1);
    IM_CUDA(cudaStreamWaitEvent(st, h->ev_join, 0));
    IM_CUDA(cudaStreamWaitEvent(st, h->ev_join3, 0));
    IM_LAUNCH((k_voxel_mesh<1024>), h->n_sm * 2, 128, sizeof(MeshSmem<1024>), st, h->M, P, F, 256, 0);
    IM_LAUNCH_PDL(pdl, k_commit_faces, h->n_sm * 8, 128, 0, st, h->M, P, F);
    IM_LAUNCH_PDL(pdl, k_pull_check, h->n_sm * 8, 128, 0, st, h->M, F);
    return IMMESH_OK;
}

// A frame's input (the kind is part of the graph signature): world points xyz at the sensor position pose_t; body points at the
// localization handle's converged pose (n_dev: their count on the device, n its bound); or a depth image at pose_t, n its sampled
// pixels (host_img: the image with its pitch and bytes per pixel, staged through the pinned slot; null: df.img is on the device).
enum class FrameSrcKind : unsigned { HostWorld = 0, DevWorld = 1, HostBody = 2, DevBody = 3, Depth = 4 };
struct FrameSrc {
    FrameSrcKind kind;
    const float* xyz = nullptr;
    int n = 0;
    const double* pose_t = nullptr;
    immesh_lio* lio = nullptr;
    const int* n_dev = nullptr;
    DepthFrame df = {};
    const unsigned char* host_img = nullptr;
    long long pitch = 0;
    int bpp = 0;
};

// Queues one frame (no host synchronisation except when both staging slots are still busy): validate, stage the source, stage the
// optional stages, launch, commit.  Host work per frame in the pipelined form: (memcpy into the pinned slot unless the caller's buffer
// is pinned) + H2D scan + H2D FrameDyn + one stream wait + ONE cudaGraphLaunch (no node is touched: every per-frame value is read
// from the FrameDyn) + one D2H of the counters.
static int mesh_enqueue(immesh_mesh* h, const FrameSrc& in, int kind, bool allow_graph = false) {
    const FrameSrcKind src = in.kind;
    const bool from_lio = src == FrameSrcKind::HostBody || src == FrameSrcKind::DevBody, depth = src == FrameSrcKind::Depth;
    const bool dev_dims = depth || in.n_dev;   // n, step, m and cmask are set on the device
    const int n = in.n;
    immesh_lio* lio = in.lio;
    if (!h || (!in.xyz && n > 0 && !depth) || n < 0 || (!from_lio && !in.pose_t)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_frame_points) return im_fail(IMMESH_E_CAPACITY, "frame larger than max_frame_points");
    FrameBuf& F = h->F;
    const MeshParams& P = h->P;
    // a depth frame's n, step, m and cmask are set by its kernels from the valid count, a device-count hand-off's by k_transform_full:
    // the host holds n = the upper bound and the most candidates it can give, for the growth check and for the grids, which cover
    // max_frame_points anyway
    int step, m;
    unsigned int cmask;
    frame_append_dims(n, P.append_target, &step, &m, &cmask);
    if (dev_dims) m = frame_append_max_m(n, P.append_target);
    const int grc = mesh_growth_check(h, m);
    if (grc) return grc;
    F.n = n;
    F.step = step;
    F.m = m;
    F.frame = ++h->frame_counter;
    const int s = F.frame & (IM_SLOTS - 1);
    mesh_harvest(h, s);   // the frame IM_SLOTS calls ago used this slot
    FramePose* d_fp = h->d_fp + s;
    F.fp = d_fp;
    F.cmask = cmask;
    cudaStream_t st = h->stream;
    const bool graphed = allow_graph && h->use_graph && !profiler().enabled && (F.shard_n <= 1 || h->win.ok);
    if (!graphed) IM_CUDA(cudaEventRecord(h->ev[0], st));
    // the frame's points into slot s (host inputs on the upload stream), the body points k_transform_full reads, the pose ring index
    const size_t slot_pts = (size_t)h->max_frame_points * 3, bytes = (size_t)n * 3 * sizeof(float);
    float* d_pts = h->d_pts + s * slot_pts;
    float* h_pts = h->h_pts + s * slot_pts;
    const float* d_body = nullptr;
    int pose_idx = 0;
    F.pts = d_pts;
    if (!from_lio) {
        FramePose* hp = h->h_fp + s;
        for (int j = 0; j < 3; ++j) { hp->pose_t[j] = in.pose_t[j]; hp->prio_origin[j] = (long long)std::floor(in.pose_t[j] / P.res) - 1024; }
        IM_CUDA(cudaMemcpyAsync(d_fp, hp, sizeof(FramePose), cudaMemcpyHostToDevice, st));
        if (depth) {
            F.pts = h->dep.pts;
            DepthFrame* hd = h->dep.h_df + s;
            *hd = in.df;
            if (in.host_img) {   // the sampled grid, tight, through the pinned slot (sw * sh * bpp <= 4 max_frame_points bytes)
                unsigned char* hb = reinterpret_cast<unsigned char*>(h_pts);
                const size_t rowb = (size_t)hd->sw * in.bpp;
                depth_stage_grid(*hd, in.host_img, in.pitch, in.bpp, hb);
                unsigned char* db = reinterpret_cast<unsigned char*>(h->d_body + s * slot_pts);
                IM_CUDA(upload_async(db, hb, rowb * hd->sh, nullptr, h->stream_up, h->ev_up[s], st));
                hd->img = db;
                hd->row_bytes = (long long)rowb;
                hd->col_bytes = in.bpp;
            }
            IM_CUDA(cudaMemcpyAsync(h->dep.d_df, hd, sizeof(DepthFrame), cudaMemcpyHostToDevice, st));
        } else if (n > 0) {
            if (src == FrameSrcKind::HostWorld) IM_CUDA(upload_async(d_pts, in.xyz, bytes, h_pts, h->stream_up, h->ev_up[s], st));
            else F.pts = in.xyz;
        }
    } else {   // the body-frame scan does not depend on the localization: it is uploaded right away
        d_body = in.xyz;
        if (src == FrameSrcKind::HostBody && n > 0) {
            float* dst = h->d_body + s * slot_pts;
            IM_CUDA(upload_async(dst, in.xyz, bytes, h_pts, h->stream_up, h->ev_up[s], st));
            d_body = dst;
        }
        // the pose: published by the last kernel of the scan's sequence (step entry points), else on request
        if (lio->pose_pub_idx < 0) {
            lio->pose_pub_idx = ++lio->scan_counter;
            IM_LAUNCH(k_pose_publish, 1, 32, 0, lio->stream, lio->d_ctrl, lio->pose_pub_idx & (IM_POSE_RING - 1));
        }
        pose_idx = lio->pose_pub_idx & (IM_POSE_RING - 1);
        IM_CUDA(cudaEventRecord(lio->ev_pose, lio->stream));
        IM_CUDA(cudaStreamWaitEvent(st, lio->ev_pose, 0));
    }
    MeshPeers pe = {};
    unsigned long long epoch = 0;
    if (F.shard_n > 1 && h->win.ok) {   // one epoch per frame; the two exchanges have separate flag rows
        for (int r = 0; r < IM_MAX_RANKS; ++r) pe.w[r] = h->win.peer[r];
        pe.rank = h->win.rank; pe.n = h->win.n;
        pe.recv_off[0] = 256; pe.recv_off[1] = 256 + (unsigned long long)h->seg1_bytes * h->win.n;
        pe.seg_bytes[0] = h->seg1_bytes; pe.seg_bytes[1] = h->seg2_bytes;
        epoch = ++h->win.epoch;
    }
    F.epoch = epoch;
    {   // the frame's device-resident inputs
        FrameDyn& d = h->h_dyn[s];
        d.pts = F.pts; d.body = d_body; d.fp = d_fp;
        d.n = F.n; d.step = F.step; d.m = F.m; d.frame = F.frame; d.cmask = F.cmask; d.pose_idx = pose_idx; d.epoch = epoch; d.n_dev = in.n_dev;
        IM_CUDA(cudaMemcpyAsync(h->d_dyn, &d, sizeof(FrameDyn), cudaMemcpyHostToDevice, st));
    }
    // the inputs of the stages queued behind the frame
    const bool rf_on = h->rf.on != 0, chg_on = h->chg.on != 0, vw_on = h->vw.on != 0;
    const bool fd_on = h->feed.on != 0, fd_img = fd_on && vw_on && h->feed.max_images > 0;
    int rc = rf_on ? queued_cam_stage(h, h->rf, s) : IMMESH_OK;
    if (!rc && fd_on) rc = mesh_feed_stage(h, s, F.frame, dev_dims ? -1 : F.n, F.step, kind, from_lio ? nullptr : in.pose_t, rf_on, fd_img);
    if (!rc && vw_on) rc = queued_cam_stage(h, h->vw, s);
    if (rc) return rc;
    // the frame's launch sequence (fixed grids: grid-stride loops over the counts the kernels read on the device)
    bool nccl_failed = false;
    const int g_pts = mesh_grid_fixed(h, h->max_frame_points, 128);
    const int g_cand = mesh_grid_fixed(h, std::min<long long>(h->max_frame_points, 2LL * P.append_target), 128);
    // Graph-replayed and not sharded: a kernel that directly follows another kernel on `st` is a programmatic dependent launch.  The
    // first kernel after a copy, an event wait or the triangulation's join keeps an ordinary edge, as do the change feed's kernels.
    const bool pdl_frame = F.shard_n <= 1;
    auto exchange = [&](int which, unsigned char* seg, unsigned char* recv, size_t bytes) {   // this rank's segment to every rank
        if (h->win.ok) {   // pushed into the other ranks' windows
            IM_LAUNCH(k_xpush, h->n_sm, 256, 0, st, h->M, F, (const unsigned char*)seg, which, pe, h->d_xdone + which);
        } else {           // NCCL transport
            IM_LAUNCH(k_xhdr, 1, 32, 0, st, h->M, F, (XHeader*)seg);
            if (immesh::nccl().AllGather(seg, recv, bytes, immesh::kNcclUint8, h->nccl_comm, st)) nccl_failed = true;
        }
    };
    auto launch_frame = [&](bool timing) {
        const bool pdl = pdl_frame && !timing;
        if (fd_on) mesh_feed_begin_launch(h, st);
        if (from_lio) IM_LAUNCH(k_transform_full, g_pts, 128, 0, st, lio->P, (const LioCtrl*)lio->d_ctrl, F, P.res, h->cam_ring, h->cam_ring_frame, P.append_target);
        if (depth) {
            auto& D = h->dep;
            IM_LAUNCH(k_depth_count, D.nb, DF_BLOCK, 0, st, (const DepthFrame*)D.d_df, D.blk);
            rf_scan_launch(st, D.blk, D.nb, D.blk_off);
            IM_LAUNCH(k_depth_emit, D.nb, DF_BLOCK, 0, st, (const DepthFrame*)D.d_df, (const int*)D.blk_off, (const int*)D.blk_off, D.nb, 1, 0.0, P.append_target,
                      h->d_dyn, D.pts, D.n);
        }
        mesh_frame_begin_launch(h, F, st, pdl && src >= FrameSrcKind::HostBody);
        if (timing) cudaEventRecord(h->ev[1], st);
        mesh_append_launch(h, F, g_cand, st, pdl);
        IM_LAUNCH_PDL(pdl, k_voxel_select, g_cand, 128, 0, st, h->M, F);
        if (timing) cudaEventRecord(h->ev[2], st);
        mesh_dilate_launch(h, F, st, pdl);
        if (F.shard_n > 1) {   // smoothed positions of the other ranks' voxels
            exchange(0, h->d_seg1, h->d_recv1, h->seg1_bytes);
            IM_LAUNCH(k_apply_smooth, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv1, h->seg1_bytes, pe);
        }
        mesh_tri_launch(h, F, st, pdl);
        if (F.shard_n > 1) {   // every rank applies the facets / removals of all ranks to its replica of the store
            exchange(1, h->d_seg2, h->d_recv2, h->seg2_bytes);
            IM_LAUNCH(k_apply_lists, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv2, h->seg2_bytes, pe);
        }
        if (timing) cudaEventRecord(h->ev[3], st);
        IM_LAUNCH_PDL(pdl, k_push_remove, h->n_sm * 2, 128, 0, st, h->M, F);
        IM_LAUNCH_PDL(pdl, k_push_add, h->n_sm * 2, 128, 0, st, h->M, F);
        if (chg_on) mesh_changes_launch(h, F, st, false);
        IM_LAUNCH_PDL(pdl && !chg_on, k_frame_end, 1, 1, 0, st, h->M);
        if (rf_on) mesh_reinforce_launch(h, st);
        if (vw_on) mesh_view_launch(h, st);
        if (fd_on) mesh_feed_launch(h, st, rf_on, fd_img);
    };
    bool queued = false;
    if (graphed) {
        // signature: everything that changes the sequence or its (static) arguments
        const unsigned long long lp = (unsigned long long)(uintptr_t)lio;
        const unsigned sig = (h->win.ok ? 2u : 0u) | 1u | ((unsigned)src << 2) | ((unsigned)F.shard_n << 5) | ((unsigned)((lp >> 4) ^ (lp >> 36)) << 9);
        queued = immesh::run_graphed_static(h->graph, sig, st, [&] { launch_frame(false); }) == cudaSuccess;
        if (!queued) { h->use_graph = 0; IM_CUDA(cudaEventRecord(h->ev[0], st)); }
    }
    if (!queued) launch_frame(true);
    if (nccl_failed) return im_fail(IMMESH_E_CUDA, "ncclAllGather failed");
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_cnt + IM_MC_HOST * s, h->M.cnt, IM_MC_HOST * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!queued) IM_CUDA(cudaEventRecord(h->ev[4], st));
    IM_CUDA(cudaEventRecord(h->ev_done[s], st));
    h->inflight[s] = 1;
    h->timed_last = queued ? 0 : 1;
    if (rf_on) h->rf.last_frame = F.frame;
    if (vw_on) h->vw.last_frame = F.frame;
    if (chg_on) h->chg.last_frame = F.frame;
    if (depth) h->dep.last_frame = F.frame;
    if (dev_dims) h->dev_dims_frame = F.frame;
    if (fd_on) IM_CUDA(mesh_feed_commit(h, F.frame));
    return IMMESH_OK;
}
// drain the queue; returns the status of the frames harvested since the last call
int mesh_wait_impl(immesh_mesh* h, bool timings) {
    for (int i = 1; i <= IM_SLOTS; ++i) mesh_harvest(h, (h->frame_counter + i) & (IM_SLOTS - 1));   // oldest frame first: last_cnt ends as the newest frame's
    if (profiler().enabled) {
        cudaStreamSynchronize(h->stream);
        profiler().collect();
    }
    if (timings && h->timed_last) {
        float a = 0, b = 0, c = 0, d = 0;
        cudaEventElapsedTime(&a, h->ev[0], h->ev[4]);
        cudaEventElapsedTime(&b, h->ev[1], h->ev[2]);
        cudaEventElapsedTime(&c, h->ev[2], h->ev[3]);
        cudaEventElapsedTime(&d, h->ev[3], h->ev[4]);
        h->last_ms[0] = a; h->last_ms[1] = b; h->last_ms[2] = c; h->last_ms[3] = d;
    }
    const int rc = h->pending_rc;
    h->pending_rc = 0;
    return rc;
}

int immesh_mesh_push_frame(immesh_mesh_t* h, const float* world_xyz, int n, const double* pose_t, int frame_idx) {
    (void)frame_idx;
    int rc = mesh_enqueue(h, {FrameSrcKind::HostWorld, world_xyz, n, pose_t}, IMMESH_MFEED_KIND_PUSH);
    return rc ? rc : mesh_wait_impl(h, true);
}
int mesh_push_dev(immesh_mesh* h, const float* d_world_xyz, int n, const double* pose_t, int kind) {
    int rc = mesh_enqueue(h, {FrameSrcKind::DevWorld, d_world_xyz, n, pose_t}, kind);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_dev(immesh_mesh_t* h, const float* d_world_xyz, int n, const double* pose_t, int frame_idx) {
    (void)frame_idx;
    return mesh_push_dev(h, d_world_xyz, n, pose_t, IMMESH_MFEED_KIND_PUSH_DEV);
}
int immesh_mesh_push_frame_from_lio(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    int rc = mesh_enqueue(h, {on_device ? FrameSrcKind::DevBody : FrameSrcKind::HostBody, body_xyz, n, nullptr, lio}, IMMESH_MFEED_KIND_FROM_LIO);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_from_lio_async(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    return mesh_enqueue(h, {on_device ? FrameSrcKind::DevBody : FrameSrcKind::HostBody, body_xyz, n, nullptr, lio}, IMMESH_MFEED_KIND_FROM_LIO_ASYNC, true);
}
int immesh_mesh_push_frame_from_lio_async_dev_n(immesh_mesh_t* h, immesh_lio_t* lio, const float* d_body_xyz, int n_max, const int* d_n) {
    if (!h || !lio || !d_body_xyz || !d_n || n_max < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_push_frame_from_lio_async_dev_n: the mesh handle is sharded");
    return mesh_enqueue(h, {FrameSrcKind::DevBody, d_body_xyz, n_max, nullptr, lio, d_n}, IMMESH_MFEED_KIND_FROM_LIO_ASYNC_DEV_N, true);
}

// ---- depth-camera frames (include/immesh_b200.h, immesh_depth_frame)
// the image and camera of f checked and turned into a frame source; the handle's depth buffers allocated by the first frame
static int depth_source(immesh_mesh* h, const immesh_depth_frame* f, const void* img, int on_device, FrameSrc* src) {
    if (!h) return im_fail(IMMESH_E_INVALID, "depth frame: null argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "depth frame: a sharded mesh handle takes world-frame points only");
    if (const char* bad = depth_frame_setup(f, img, &src->df, &src->pitch, &src->bpp)) return im_fail(IMMESH_E_INVALID, bad);
    const int sw = src->df.sw, sh = src->df.sh;
    if ((long long)sw * sh > h->max_frame_points) return im_fail(IMMESH_E_CAPACITY, "depth frame: more sampled pixels than max_frame_points");
    auto& D = h->dep;
    if (!D.pts) {
        immesh::MemSet dev, pinned{immesh::MemSet::Pinned};
        const int nb = (h->max_frame_points + DF_BLOCK - 1) / DF_BLOCK;
        cudaError_t e = dev.alloc(&D.d_df, 1);
        if (e == cudaSuccess) e = pinned.alloc(&D.h_df, IM_SLOTS);
        if (e == cudaSuccess) e = dev.alloc(&D.pts, (size_t)h->max_frame_points * 3);
        if (e == cudaSuccess) e = dev.alloc(&D.n, 1, 0);
        if (e == cudaSuccess) e = dev.alloc(&D.blk, (size_t)nb);
        if (e == cudaSuccess) e = dev.alloc(&D.blk_off, (size_t)nb + 1);
        if (e != cudaSuccess) {
            cudaGetLastError();
            D = immesh_mesh::Depth();
            return im_fail(IMMESH_E_CAPACITY, "depth frame: out of device or pinned memory for its buffers");
        }
        D.nb = nb;
        D.dev = std::move(dev);
        D.pinned = std::move(pinned);
    }
    src->host_img = on_device ? nullptr : static_cast<const unsigned char*>(img);
    src->n = sw * sh;
    src->pose_t = f->cam_t;
    return IMMESH_OK;
}
int immesh_mesh_push_depth(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device) {
    FrameSrc src{FrameSrcKind::Depth};
    int rc = depth_source(h, f, depth, on_device, &src);
    if (!rc) rc = mesh_enqueue(h, src, IMMESH_MFEED_KIND_DEPTH);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_depth_async(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device) {
    FrameSrc src{FrameSrcKind::Depth};
    const int rc = depth_source(h, f, depth, on_device, &src);
    return rc ? rc : mesh_enqueue(h, src, IMMESH_MFEED_KIND_DEPTH, true);
}
int immesh_mesh_depth_points(immesh_mesh_t* h, float* xyz, int cap, int* n) {
    if (!h || !n || cap < 0 || (cap > 0 && !xyz)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!h->dep.last_frame) return im_fail(IMMESH_E_INVALID, "no depth frame was pushed");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c = 0;
    IM_CUDA(cudaMemcpy(&c, h->dep.n, sizeof(int), cudaMemcpyDeviceToHost));
    *n = c;
    if (cap == 0) return IMMESH_OK;
    if (c > cap) return im_fail(IMMESH_E_CAPACITY, "more depth points than cap");
    if (c > 0) IM_CUDA(cudaMemcpy(xyz, h->dep.pts, (size_t)c * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    return IMMESH_OK;
}
// device-side timing of a pipelined batch: begin mark on the localization stream, end mark behind BOTH streams
int immesh_pipeline_mark_begin(immesh_lio_t* lio) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null handle");
    if (!lio->ev_mark) IM_CUDA(cudaEventCreate(&lio->ev_mark));
    IM_CUDA(cudaEventRecord(lio->ev_mark, lio->stream));
    return IMMESH_OK;
}
int immesh_pipeline_mark_end(immesh_lio_t* lio, immesh_mesh_t* h, double* ms) {
    if (!lio || !h || !ms || !lio->ev_mark) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!h->ev_mark) { IM_CUDA(cudaEventCreate(&h->ev_mark)); IM_CUDA(cudaEventCreateWithFlags(&h->ev_sync, cudaEventDisableTiming)); }
    IM_CUDA(cudaEventRecord(h->ev_sync, lio->stream));
    IM_CUDA(cudaStreamWaitEvent(h->stream, h->ev_sync, 0));
    IM_CUDA(cudaEventRecord(h->ev_mark, h->stream));
    IM_CUDA(cudaEventSynchronize(h->ev_mark));
    float t = 0.f;
    IM_CUDA(cudaEventElapsedTime(&t, lio->ev_mark, h->ev_mark));
    *ms = t;
    return IMMESH_OK;
}
int immesh_mesh_shard(immesh_mesh_t* h, int rank, int nranks, const char* unique_id128) {
    if (!h || !unique_id128 || nranks < 1 || rank < 0 || rank >= nranks) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (nranks == 1) { h->F.shard_rank = 0; h->F.shard_n = 1; return IMMESH_OK; }
    if (h->grow_max_bytes > 0) return im_fail(IMMESH_E_INVALID, "a mesh handle with automatic growth cannot be sharded (immesh_mesh_set_growth(h, 0) first)");
    if (h->rf.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the reinforcement enabled cannot be sharded (immesh_mesh_reinforce_enable(h, NULL, ...) first)");
    if (h->chg.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the change feed enabled cannot be sharded (immesh_mesh_changes_enable(h, 0, 0) first)");
    if (h->feed.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the frame feed enabled cannot be sharded (immesh_mesh_feed_enable(h, NULL) first)");
    if (h->vw.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the queued view enabled cannot be sharded (immesh_mesh_view_enable(h, NULL, ...) first)");
    if (!immesh::nccl().load()) return im_fail(IMMESH_E_CUDA, "libnccl.so.2 not found");
    immesh::nccl_uid_t id;
    std::memcpy(id.internal, unique_id128, 128);
    immesh::nccl_comm_t comm = nullptr;
    const int rc = immesh::nccl().CommInitRank(&comm, nranks, id, rank);
    if (rc) return im_fail(IMMESH_E_CUDA, immesh::nccl().GetErrorString ? immesh::nccl().GetErrorString(rc) : "ncclCommInitRank failed");
    h->nccl_comm = comm;
    FrameBuf& F = h->F;
    F.shard_rank = rank;
    F.shard_n = nranks;
    F.x_cap = 1 << 16;
    // segment 1: header + smoothed positions; segment 2: header + facets + words + removals
    h->seg1_bytes = 16 + (size_t)F.x_cap * sizeof(immesh::XSmooth);
    h->seg2_bytes = 16 + (size_t)F.x_cap * (16 + 8 + 16);
    unsigned char *s1 = nullptr, *s2 = nullptr;
    IM_CUDA(h->dev.alloc(&s1, h->seg1_bytes, 0));
    IM_CUDA(h->dev.alloc(&s2, h->seg2_bytes, 0));
    // receive areas: inside a peer window (other ranks store into it over NVLink) or, with NCCL transport, private buffers
    const char* force_nccl = std::getenv("IMMESH_SHARD_NCCL");
    if (!(force_nccl && force_nccl[0] == '1')) {
        const cudaError_t e = immesh::peer_window_open(h->win, 256 + (h->seg1_bytes + h->seg2_bytes) * (size_t)nranks, rank, nranks, comm, h->stream);
        if (e != cudaSuccess) {
            std::fprintf(stderr, "[immesh_b200] rank %d: peer window unavailable (%s); sharded mesher falls back to NCCL all-gathers\n", rank, cudaGetErrorString(e));
            cudaGetLastError();
        }
    }
    if (h->win.ok) {
        h->d_recv1 = h->win.local + 256;
        h->d_recv2 = h->win.local + 256 + h->seg1_bytes * (size_t)nranks;
        IM_CUDA(h->dev.alloc(&h->d_xdone, 2, 0));
    } else {
        IM_CUDA(h->dev.alloc(&h->d_recv1, h->seg1_bytes * nranks, 0));
        IM_CUDA(h->dev.alloc(&h->d_recv2, h->seg2_bytes * nranks, 0));
    }
    h->d_seg1 = s1; h->d_seg2 = s2;
    F.x_smooth = (immesh::XSmooth*)(s1 + 16);
    F.x_face = (int4*)(s2 + 16);
    F.x_word = (unsigned long long*)(s2 + 16 + (size_t)F.x_cap * 16);
    F.x_rem = (int4*)(s2 + 16 + (size_t)F.x_cap * 24);
    return IMMESH_OK;
}
int immesh_mesh_shard_transport(immesh_mesh_t* h) {
    if (!h || h->F.shard_n <= 1) return 0;
    return h->win.ok ? 2 : 1;
}
int immesh_graph_stats(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 6; ++i) out[i] = 0;
    if (lio) { out[0] = lio->graph.captures; out[1] = lio->graph.replays; out[2] = lio->graph.failures; }
    if (mesh) { out[3] = mesh->graph.captures; out[4] = mesh->graph.replays; out[5] = mesh->graph.failures; }
    return IMMESH_OK;
}
int immesh_graph_pdl_edges(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    out[0] = lio ? lio->graph.pdl_edges : 0;
    out[1] = mesh ? mesh->graph.pdl_edges : 0;
    return IMMESH_OK;
}
// host time (ms) the enqueue calls spent blocked on busy staging slots since the last call of this function: [lio, mesh].
// Queueing a scan costs (wall time of the call) - (this): the rest is back-pressure from the device.
int immesh_host_wait_ms(immesh_lio_t* lio, immesh_mesh_t* mesh, double* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    out[0] = lio ? lio->host_wait_ms : 0.0;
    out[1] = mesh ? mesh->host_wait_ms : 0.0;
    if (lio) lio->host_wait_ms = 0;
    if (mesh) mesh->host_wait_ms = 0;
    return IMMESH_OK;
}
int immesh_mesh_wait(immesh_mesh_t* h) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    return mesh_wait_impl(h, false);
}

int immesh_mesh_capacity(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, c));
    out[0] = h->M.max_v; out[1] = c[IM_MC_VERTICES];
    out[2] = h->M.max_t; out[3] = c[IM_MC_TRIS_ALLOC];
    out[4] = h->max_vox; out[5] = c[IM_MC_VOXELS];
    out[6] = (int64_t)(h->dev.bytes() + h->batch.bytes()); out[7] = h->growths;
    return IMMESH_OK;
}
int immesh_mesh_reserve(immesh_mesh_t* h, int64_t vertices, int64_t triangles, int64_t voxels) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_reserve: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    const int rc = mesh_grow(h, std::max<long long>(vertices, h->M.max_v), std::max<long long>(triangles, h->M.max_t), std::max<long long>(voxels, h->max_vox));
    if (rc == IMMESH_OK) return rc;
    return im_fail(rc, (std::string("immesh_mesh_reserve: ") + immesh::last_error_storage()).c_str());
}
int immesh_mesh_set_growth(immesh_mesh_t* h, int64_t max_bytes) {
    if (!h || max_bytes < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (max_bytes > 0 && h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_set_growth: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    if (max_bytes > 0 && h->grow_max_bytes <= 0) {   // growth starts from the mesh as it is now
        IM_CUDA(cudaStreamSynchronize(h->stream));
        IM_CUDA(mesh_read_counters(h, h->known));
        h->known_frame = h->frame_counter;
    }
    h->grow_max_bytes = max_bytes;
    return IMMESH_OK;
}
int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    out[0] = c[IM_MC_VERTICES]; out[1] = c[IM_MC_TRIS_LIVE]; out[2] = c[IM_MC_NEW_VERTICES]; out[3] = c[IM_MC_WORK_FRONT] + c[IM_MC_WORK_BACK];
    out[4] = c[IM_MC_ADD]; out[5] = c[IM_MC_REMOVE]; out[6] = c[IM_MC_VOXELS]; out[7] = c[IM_MC_ACT];
    return IMMESH_OK;
}

int immesh_mesh_work_stats(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    int m = h->F.m;
    if (h->dev_dims_frame && h->dev_dims_frame == h->frame_counter) {   // the newest frame's m is set on the device
        FrameDyn d;
        IM_CUDA(cudaStreamSynchronize(h->stream));
        IM_CUDA(cudaMemcpy(&d, h->d_dyn, sizeof(d), cudaMemcpyDeviceToHost));
        m = d.m;
    }
    out[0] = m; out[1] = c[IM_MC_STAT_GATHERED]; out[2] = c[IM_MC_STAT_QUERIES]; out[3] = c[IM_MC_STAT_DILATED]; out[4] = c[IM_MC_STAT_FACETS];
    out[5] = c[IM_MC_WORK_FRONT] + c[IM_MC_WORK_BACK]; out[6] = c[IM_MC_ADD]; out[7] = c[IM_MC_REMOVE];
    return IMMESH_OK;
}

int immesh_mesh_last_timing(immesh_mesh_t* h, double* ms) {
    if (!h || !ms) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 4; ++i) ms[i] = h->last_ms[i];
    return IMMESH_OK;
}

