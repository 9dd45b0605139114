// immesh_b200 -- handle definitions shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>

#include "common_host.hpp"
#include "lio_core.cuh"
#include "mesh_voxel.cuh"
#include "peer_win.cuh"
#include "reinforce.cuh"

using immesh::LioParams; using immesh::VoxelMapDev; using immesh::ScanBuf; using immesh::LioCtrl;
using immesh::MeshParams; using immesh::MeshDev; using immesh::FrameBuf; using immesh::FramePose;

// staging depth of the pipelined entry points: the host may queue this many scans / frames ahead of the device before it has to wait
// (2 was enough for the device, but a host hiccup of ~1 ms then drained the pipeline: seen as single ranks of an 8-rank run falling
// back to the blocking-call rate)
#define IM_SLOTS 4
// immesh_lio::h_ints (pinned, 64 ints) past its copy of the counter block: the iteration count of a blocking estimate, the count a
// publisher reads back (the plane markers' four counters behind it)
constexpr int IM_HINT_ITERS = 32, IM_HINT_PUB = 40, IM_HINT_SIZE = 64;
static_assert(immesh::IM_LC_SIZE <= IM_HINT_ITERS && IM_HINT_PUB + 5 <= IM_HINT_SIZE, "immesh_lio::h_ints layout");

struct immesh_lio {
    LioParams P;
    VoxelMapDev map;
    ScanBuf sb;
    LioCtrl* d_ctrl = nullptr;
    int* d_counters = nullptr;  // [IM_LC_SIZE] the counter block, slots IM_LC_*
    // grow-only scratch of the publishers, in `scratch`
    int* d_pub_scratch = nullptr;    // immesh_voxelmap_plane_markers: key sort, per-root row counts / offsets
    size_t pub_scratch_ints = 0;
    double* d_pub_rows = nullptr;    // immesh_voxelmap_plane_markers: the rows of one call
    size_t pub_rows_doubles = 0;
    // immesh_lio_effect_cloud / immesh_lio_registered_cloud
    float4* d_spub_rows = nullptr;   // x y z intensity rows of one call
    size_t spub_rows_cap = 0;
    int* d_spub_idx = nullptr;       // scan index of each effect row
    size_t spub_idx_cap = 0;
    int* d_spub_tiles = nullptr;     // per-tile match counts, scanned in place into offsets; the total behind them
    size_t spub_tiles_cap = 0;
    float* d_spub_in = nullptr;      // staging of a host dense cloud (never the scan slots, which hold the localised scan)
    size_t spub_in_cap = 0;
    int scan_rows = 0;                      // per-scan buffers: 0 no IESKF run since create / voxelmap_build, 1 last run's, -1 overwritten
    const char* scan_rows_overwritten_by = nullptr;
    long long uploads = 0;                  // scans placed in the per-scan buffers (upload_scan), by any call
    // immesh_lio_frontend_cloud: the front-end that fed the last step, when it was an intensity-carrying (_i) chain
    const void* fe_vg = nullptr;            // its VoxelGrid handle (nullptr: the last step was not such a chain)
    long long fe_uploads = 0;               // `uploads` right after that step
    long long fe_vg_calls = 0;              // the VoxelGrid's call count right after it
    int fe_n = 0;                           // points of its full-resolution scan
    int* d_sorted = nullptr;
    int* d_complex = nullptr;   // touched root voxels left to the general warp-per-voxel kernel (the others are finished by k_grow_simple)
    double* d_ptpl = nullptr;
    float* d_body_own = nullptr;  // scan buffers owned by the handle, IM_SLOTS slots of max_scan*3 (sb.body points into them unless the caller passed a device pointer)
    cudaStream_t stream_up = nullptr;   // upload stream: the H2D copy of scan k+1 overlaps the kernels of scan k
    cudaEvent_t ev_up[IM_SLOTS] = {};
    float* h_body = nullptr;   // pinned staging, IM_SLOTS slots
    double* h_state = nullptr; // pinned, IM_STATE_DOUBLES + 64
    cudaEvent_t ev_slot[IM_SLOTS] = {};  // completion of the step that used staging slot s
    int slot_busy[IM_SLOTS] = {};
    int step_counter = 0;
    immesh::ScanDyn* h_dyn = nullptr;   // pinned, IM_SLOTS slots: per-scan inputs of the launch sequence (one H2D per scan)
    immesh::ScanDyn dyn_last = {};         // host copy of the block last uploaded
    immesh::LioOut* h_out = nullptr;    // pinned, IM_SLOTS slots: what a scan returns to the host (one D2H per scan)
    const int* next_n_dev = nullptr;    // device-resident point count for the next upload (immesh_lio_step_async_dev_n)
    int scan_counter = 0;               // scans queued through the step entry points; pose ring slot = scan_counter & 7
    int pose_pub_idx = -1;              // scan index whose converged pose is in LioCtrl::pose_ring (-1: not published)
    int timed_last = 0;                 // the last step recorded its stage timing events
    double host_wait_ms = 0;            // host time spent blocked on a busy staging slot inside the enqueue calls (back-pressure, not work)
    cudaEvent_t ev_pose = nullptr;      // "pose of the last scan published" (the mesher's stream waits on it)
    cudaEvent_t ev_mark = nullptr;   // pipeline timing mark (begin)
    void* nccl_comm = nullptr;       // ncclComm_t when the VoxelMap is sharded over several GPUs
    unsigned int* d_bits = nullptr;  // [2][words] exists / matched-in-own-voxel bit words of the sharded residual pass
    immesh::PeerWindow win;          // peer window of the sharded residual pass (NVLink peer memory, replaces the NCCL all-reduces)
    int words_cap = 0;
    int* h_ints = nullptr;     // pinned, IM_HINT_SIZE: a copy of the counter block, a count read back at IM_HINT_ITERS or IM_HINT_PUB
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t cap = 0;
    int max_nodes = 0, max_chunks = 0, max_scan = 0;
    int n_sm = 132;
    int last_n = 0;
    immesh::GraphCtx graph;   // replay of the per-scan launch sequence (pipelined API)
    int use_graph = 1;
    double last_ms[3] = {0, 0, 0};
    immesh::MemSet dev;           // device memory counted in immesh_lio_capacity: the create-time buffers, the map pools, d_ptpl, d_bits
    immesh::MemSet scratch;       // device memory not counted: the publishers' scratch
    immesh::MemSet pinned{immesh::MemSet::Pinned};
    // growth of the map pools (immesh_lio_reserve / immesh_lio_set_growth)
    long long growths = 0;        // calls that enlarged at least one pool
    int64_t grow_max_bytes = 0;   // automatic growth before every step: 0 off, > 0 ceiling on dev.bytes()
    int known[immesh::IM_LC_SIZE] = {};   // counters (IM_LC_* slots) of the last step known to have finished
    long long known_step = 0;     // its number among the map-growing steps (0: the empty map at create)
    long long map_steps = 0;      // map-growing steps queued so far
    long long slot_step[IM_SLOTS] = {};   // number of the step that used staging slot s
    int max_step_nodes = 0, max_step_chunks = 0;   // largest node / chunk use between two noted steps (finished blocks are noted in step order)
};

// the device buffers of one depth image of the tiled rasteriser (mesh_capi.cu: rf_image_alloc, rf_image_launch): the camera, the tile
// counters and offsets, the bins, misc[0] (the bins overflowed), the valid pixels per block and their offsets, the depth bits, and
// result buffers 0 and 1 (image, points, pixels, count; the pose is the queued reinforcement's own)
struct RfOut { float* depth; float* pts; int* pix; int* n; double* pose; };
struct RfImage {
    int ntiles = 0, nb = 0, bin_cap = 0;
    immesh::DepthCam* cam = nullptr;
    int *tile_cnt = nullptr, *tile_off = nullptr, *bin = nullptr, *misc = nullptr, *blk = nullptr, *blk_off = nullptr;
    unsigned int* depth_bits = nullptr;
    RfOut out[2] = {};
};

struct immesh_mesh {
    MeshParams P;
    MeshDev M;
    FrameBuf F;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    float* d_pts = nullptr;   // IM_SLOTS slots of max_frame_points*3
    float* d_body = nullptr;  // IM_SLOTS slots, staging for body-frame scans handed over by the localization handle
    float* h_pts = nullptr;   // pinned, IM_SLOTS slots
    int* h_cnt = nullptr;     // pinned, IM_SLOTS slots of IM_MC_HOST
    FramePose* d_fp = nullptr;  // IM_SLOTS slots
    FramePose* h_fp = nullptr;  // pinned, IM_SLOTS slots
    immesh::FrameDyn* h_dyn = nullptr;  // pinned, IM_SLOTS slots: per-frame inputs of the launch sequence
    immesh::FrameDyn* d_dyn = nullptr;  // device copy read by every kernel of the frame (F.dyn)
    int timed_last = 0;
    double host_wait_ms = 0;
    cudaEvent_t ev_in[IM_SLOTS] = {};    // inputs of slot s ready (recorded on the producer stream)
    cudaEvent_t ev_done[IM_SLOTS] = {};  // frame of slot s finished (mesh stream)
    int inflight[IM_SLOTS] = {};
    cudaEvent_t ev_mark = nullptr, ev_sync = nullptr;  // pipeline timing mark (end) / cross-stream join
    cudaStream_t stream2 = nullptr;   // side stream: warp-level triangulation, concurrent with the block-level one
    cudaStream_t stream3 = nullptr;   // side stream: pull (incidence-list walk), concurrent with the triangulation
    cudaStream_t stream_up = nullptr; // upload stream: the H2D copy of frame k+1 overlaps the kernels of frame k
    cudaEvent_t ev_up[IM_SLOTS] = {};
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_join3 = nullptr;
    int pending_rc = 0;
    void* nccl_comm = nullptr;        // ncclComm_t when the per-voxel stage is sharded over several GPUs
    unsigned char *d_seg1 = nullptr, *d_seg2 = nullptr, *d_recv1 = nullptr, *d_recv2 = nullptr;   // exchange segments
    immesh::PeerWindow win;           // peer window: [flags][recv1 x n][recv2 x n] when the segments are pushed over NVLink
    int* d_xdone = nullptr;           // block-done counters of the two push kernels
    size_t seg1_bytes = 0, seg2_bytes = 0;
    int* d_snap_tri = nullptr;
    int* d_snap_flip = nullptr;
    int* d_snap_n = nullptr;
    int max_frame_points = 0;
    immesh::GraphCtx graph;   // replay of the per-frame launch sequence (pipelined API)
    int use_graph = 1;
    int frame_counter = 0;
    int warp_nmax = 96;       // largest dilated set triangulated by a single warp
    int n_sm = 132;
    size_t ccap = 0;
    double last_ms[4] = {0, 0, 0, 0};
    int last_cnt[immesh::IM_MC_HOST];
    immesh::MemSet dev;       // device memory counted in immesh_mesh_capacity (with `batch`): the create-time buffers, the pools and the shard segments
    immesh::MemSet scratch;   // device memory not counted: the region buffers' scratch
    immesh::MemSet pinned{immesh::MemSet::Pinned};
    unsigned char* region_scratch[16] = {};   // immesh_mesh_region_buffers, grow-only, in `scratch`
    size_t region_scratch_cap[16] = {};
    // batched frame (immesh_mesh_push_frame_batched), allocated by its first call into `batch`, sized by the handle's capacities only
    immesh::MemSet batch;
    int max_vox = 0;
    int* b_act = nullptr;             // [max_vox] the frame's activated voxels (all append chunks)
    int* b_sel = nullptr;             // [max_vox] the voxels the frame meshes
    unsigned long long* b_key = nullptr;   // [max_vox] their keys
    unsigned int *b_ku = nullptr, *b_vu = nullptr;   // [2][max_vox] radix-sort ping-pong (key order -> rank)
    int* b_hist = nullptr;
    int* b_rank = nullptr;            // [max_work] rank of the batch's work voxels
    unsigned char* b_mark = nullptr;  // [max_t] triangle marks (FrameBuf::tri_mark)
    int* b_fset = nullptr;            // facet set of a batch, 2 x max_list slots
    unsigned int b_fset_mask = 0;
    immesh::FramePose* b_fp = nullptr;
    // growth of the mesh pools (immesh_mesh_reserve / immesh_mesh_set_growth)
    long long growths = 0;
    int64_t grow_max_bytes = 0;
    int known[immesh::IM_MC_HOST] = {};   // counters (IM_MC_* slots) of the last frame known to have finished
    int known_frame = 0;          // its frame number (0: the empty mesh at create)
    int max_step_tris = 0;        // largest triangle allocation between two noted frames (noted oldest first)
    // LiDAR point-cloud reinforcement (immesh_mesh_reinforce_enable)
    double (*cam_ring)[12] = nullptr;   // [IM_RF_RING] rot_end, pos_end of the frames handed over by the localization handle
    int* cam_ring_frame = nullptr;      // [IM_RF_RING] frame number each ring entry belongs to (0: none)
    struct Reinforce {
        int on = 0, win = 1;
        int last_frame = 0;               // newest frame queued with the reinforcement (0: none since enable)
        int explicit_pose = 0;            // immesh_mesh_reinforce_pose: the caller's pose from the next frame on
        double R[9] = {}, t[3] = {};
        immesh::DepthCam base = {};       // intrinsics, z range and image size; the pose is filled in on the device per frame
        void* rd = nullptr;               // RfDyn, written per frame from the pinned slot
        void* h_rd = nullptr;             // pinned, IM_SLOTS RfDyn
        RfImage img;                      // result buffer (frame & 1) holds the frame's image and pose
        immesh::MemSet dev, pinned{immesh::MemSet::Pinned};   // the buffers above, freed by disable / destroy (not counted)
    } rf;
};
