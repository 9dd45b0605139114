// immesh_b200 -- handle definitions shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>

#include "common_host.hpp"
#include "depth_frame.cuh"
#include "lio_core.cuh"
#include "lio_feed.cuh"
#include "mesh_changes.cuh"
#include "mesh_feed.cuh"
#include "mesh_voxel.cuh"
#include "peer_win.cuh"
#include "view_overlay.cuh"

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
    // local map (immesh_lio_local_map / immesh_voxelmap_evict_boxes); map.node_free is allocated by the first of them, in `dev`
    int lm_on = 0;                // the box rule and the eviction sweep are queued with every step
    long long lm_purges = 0;      // rebuilds of the root hash that dropped tombstones (lio_purge_check)
    int tombs_known = 0;          // tombstones after the last step known to have finished
    float* d_lm_boxes = nullptr;  // the caller's boxes of immesh_voxelmap_evict_boxes, in `scratch`
    size_t lm_boxes_cap = 0;
    // the scan the next lio_enqueue / immesh_voxelmap_build_async_dev records in the scan feed, when the front-end or the IMU chain
    // queues it (set around their inner step call; kind < 0: the entry point's own kind, no full scan)
    struct FeedNext {
        int kind = -1, branch = 0, n = 0;
        const float* pts = nullptr;     // the full scan (registered source 2)
        const float* inten = nullptr;   // its intensity, or null
        const int* n_dev = nullptr;     // its count when that is device resident (n: the upper bound)
    } feed_next;
    // scan feed (immesh_lio_feed_enable)
    struct Feed {
        int on = 0, effect = 0, registered = 0, skip = 1;
        long long max_scans = 0, max_rows = 0;
        long long queued = 0;             // scans recorded since enable: the newest one's number
        int nb = 0;                       // tiles of the effect count (max_scan points)
        immesh::LioFeedDev* dev = nullptr;
        long long* hdr = nullptr;         // [max_scans][IMMESH_LIO_FEED_HDR]
        double* states = nullptr;         // [max_scans][IM_STATE_DOUBLES]
        float4* rows = nullptr;           // [max_rows]
        int* idx = nullptr;               // [max_rows] scan index of the effect rows (effect = 1)
        int* tiles = nullptr;             // [nb + 1] the effect count's tiles and total
        immesh::FeedDyn* h_dyn = nullptr; // pinned ring of IM_FEED_DYN_RING: the per-scan inputs
        long long* h_done = nullptr;      // pinned, written by k_feed_done: the newest scan whose record is complete
        long long* d_done = nullptr;      // its device address
        cudaStream_t stream = nullptr;    // the reader's copies (never the handle's stream)
        cudaEvent_t ev = nullptr;         // recorded behind the newest scan's record
        immesh::MemSet dev_mem, pinned{immesh::MemSet::Pinned};
        // plane-map markers (immesh_lio_feed_markers_enable): on while mk_rows > 0
        long long mk_rows = 0;            // marker ring, rows of IMMESH_PLANE_MARKER_COLS doubles
        immesh::LioMarkDev* mk_dev = nullptr;
        long long* mk_hdr = nullptr;      // [max_scans][IMMESH_LIO_FEED_MARKER_HDR]
        double* mk_ring = nullptr;        // [mk_rows][IMMESH_PLANE_MARKER_COLS]
        unsigned int* mk_sort = nullptr;  // [4][mk_cap]: the key sort's two buffer pairs; then the roots' slots and row offsets
        int* mk_hist = nullptr;           // [256 * tiles of mk_cap]
        size_t mk_cap = 0;                // root slots the sort scratch covers (the hash capacity when it was sized)
        immesh::MemSet mk_mem, mk_scratch;
    } feed;
};
#define IM_FEED_DYN_RING 64

// the device buffers of one depth image of the tiled rasteriser (mesh_render.cu: rf_image_alloc, rf_image_launch): the camera, the tile
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
    unsigned char* region_scratch[12] = {};   // immesh_mesh_region_buffers, grow-only, in `scratch`
    size_t region_scratch_cap[12] = {};
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
    // a camera queued behind every frame: the reinforcement (immesh_mesh_reinforce_enable) and the view (immesh_mesh_view_enable)
    struct QueuedCam {
        int on = 0, win = 1;
        int last_frame = 0;               // newest frame queued with it (0: none since enable)
        int mode = 0;                     // the camera source (RfDyn::mode): 0 sensor-bound, 1 the caller's fixed pose, 2 the follow camera
        double R[9] = {}, t[3] = {};
        immesh::DepthCam base = {};       // intrinsics, z range and image size; the pose is filled in on the device per frame
        void* rd = nullptr;               // RfDyn, written per frame from the pinned slot
        void* h_rd = nullptr;             // pinned, IM_SLOTS RfDyn
        RfImage img;                      // result buffer (frame & 1) holds the frame's image and pose
        immesh::MemSet dev, pinned{immesh::MemSet::Pinned};   // the buffers above, freed by disable / destroy (not counted)
    } rf;                                 // LiDAR point-cloud reinforcement: the caller's pose (mode 1) from immesh_mesh_reinforce_pose
    // the viewer's shaded image (immesh_mesh_view_enable queues it behind every frame; immesh_mesh_render_view builds one for a call)
    struct View : QueuedCam {
        int pos = 0, color = 0, auto_range = 0;   // immesh_view_style: positions, color_by_height, z range from the mesh
        uchar4* rgba[2] = {};             // the colour image of result buffer b
        float* zr = nullptr;              // [2] the height colour's z range (the caller's, or k_view_zrange's)
        unsigned int* zr_part = nullptr;  // [2 zr_blocks] k_view_zrange's per-block partials
        int* zr_done = nullptr;           // k_view_zrange's finished-block counter (0 between launches)
        int zr_blocks = 1;
        immesh::ViewOverlay ov = {};      // immesh_mesh_view_overlay (ov.on = 0: none)
        immesh::MemSet ov_dev;            // its keys, trajectory and frustum, freed by the next overlay call, disable or destroy (not counted)
    } vw;
    // change feed (immesh_mesh_changes_enable); its per-frame pointers are in F (chg_stamp, chg_list, chg_cnt, chg_cap)
    struct Changes {
        int on = 0;
        int enable_frame = 0;             // frame_counter at enable: the frames after it are recorded
        int last_frame = 0;               // newest frame queued with the feed
        immesh::ChgDev C = {};
        unsigned int *ku = nullptr, *vu = nullptr;   // [2][chg_cap] radix-sort ping-pong of the frame's rows
        int* hist = nullptr;
        immesh::MemSet dev;               // every buffer of the feed, freed by disable / destroy (not counted)
    } chg;
    // frame feed (immesh_mesh_feed_enable, mesh_feed.cuh).  Every buffer here is freed only by immesh_mesh_feed_enable and
    // immesh_mesh_destroy, after the stream is drained and the graph dropped; the image ring also by immesh_mesh_view_enable.
    struct Feed {
        int on = 0, depth = 0;
        long long max_frames = 0, max_rows = 0, max_images = 0;   // max_images = 0: no image recording
        long long npx = 0;                // pixels of one image (the view's w * h at the enable)
        long long enable_frame = 0;       // frame_counter at the enable: the frames after it are recorded
        long long queued = 0;             // newest frame recorded
        immesh::MeshFeedDev* dev = nullptr;
        long long* hdr = nullptr;         // [max_frames][IMMESH_MESH_FEED_HDR]
        double* poses = nullptr;          // [max_frames][IMMESH_MESH_FEED_POSE]
        float* pts = nullptr;             // [max_rows][3]
        int* pix = nullptr;               // [max_rows]
        uchar4* rgba = nullptr;           // [max_images][npx]
        float* depth_ring = nullptr;      // [max_images][npx] (depth = 1)
        immesh::MeshFeedDyn* h_dyn = nullptr;   // pinned, IM_SLOTS slots: the per-frame inputs
        long long* h_done = nullptr;      // pinned, written by k_mfeed_done: the newest frame whose record is complete
        long long* d_done = nullptr;      // its device address
        cudaStream_t stream = nullptr;    // the reader's copies (never the handle's stream)
        cudaEvent_t ev = nullptr;         // recorded behind the newest frame's record
        immesh::MemSet dev_mem, img_mem, pinned{immesh::MemSet::Pinned};
    } feed;
    // depth-camera frames (immesh_mesh_push_depth, depth_frame.cuh), allocated by the first of them and kept until destroy.  The points
    // buffer holds the newest depth frame's world points (one buffer: every frame's kernels run in stream order on `stream`).
    struct Depth {
        immesh::DepthFrame* d_df = nullptr;   // the frame's image and camera, written per frame from the pinned slot
        immesh::DepthFrame* h_df = nullptr;   // pinned, IM_SLOTS slots
        float* pts = nullptr;                 // [max_frame_points][3] the valid samples' world points (FrameDyn::pts of a depth frame)
        int* n = nullptr;                     // their count
        int *blk = nullptr, *blk_off = nullptr;   // valid samples per block of DF_BLOCK sampled pixels, their offsets [nb + 1]
        int nb = 0;                           // blocks covering max_frame_points sampled pixels
        int last_frame = 0;                   // newest depth frame queued (0: none)
        immesh::MemSet dev, pinned{immesh::MemSet::Pinned};   // not counted in immesh_mesh_capacity
    } dep;
    int dev_dims_frame = 0;   // newest frame whose n, step and m were set on the device (a depth frame, a device-count hand-off)
};

// The live triangles in one defined order, for immesh_mesh_snapshot, _region_stream, _region_buffers and immesh_mesh_evaluate
// (mesh_tri_order, mesh_query.cu): the live records compacted (w = the slot) and sorted by the triple (a, b, c); with a region size
// first by the region of tri_region_key, either every region by its key (ascending x, y, z) or, with qkeys, only the regions of the
// table qkeys / qval by the caller's index.  The caller provides the buffers for `cap` records.  A key outside +-1048000 sets `range`.
struct TriOrder {
    int cap;
    int4* rec;                         // [cap] the kept records
    int* reg;                          // [3 cap] the keys (all regions) or [cap] the caller's index (requested regions)
    unsigned int *k[2], *v[2];         // [cap] each: the sort's ping-pong
    int* hist;                         // 256 * ceil(cap / VG_TILE) ints
    int* misc;                         // [8] on the device: count, range flag, minimum and maximum of each region word
    const unsigned long long* qkeys;   // requested regions: packed keys (qmask + 1 slots) and each slot's index
    const int* qval;
    unsigned int qmask;
    int n, range;                      // out: the records kept, the range flag
    const unsigned int* order;         // out: the kept records' indices into rec, in order
};
int mesh_tri_order(immesh_mesh* h, const int* cnt, double region_size, TriOrder& o);

// ---- what the mesher's translation units call in one another, by the file that defines it: mesh_capi.cu (the handle's bookkeeping and
// the frame chain's stages the batched frame shares), mesh_render.cu, mesh_feeds.cu, mesh_query.cu (rs_sort_passes of radix_sort.cuh,
// whose kernels the mesher compiles once, and the ints of its hist for n keys)
#define IM_MPOOL_LIMIT (1LL << 30)   // ids are 32-bit: every mesh pool (and the change feed's ring) stops at 2^30 records

inline size_t pow2_at_least(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}
inline int mesh_grid(const immesh_mesh* h, int n, int threads, int waves = 8) {
    int g = (n + threads - 1) / threads;
    if (g > h->n_sm * waves) g = h->n_sm * waves;
    return g < 1 ? 1 : g;
}
inline int mesh_grid_fixed(const immesh_mesh* h, long long n_cap, int threads, int waves = 8) {
    long long g = (n_cap + threads - 1) / threads;
    if (g > (long long)h->n_sm * waves) g = (long long)h->n_sm * waves;
    return g < 1 ? 1 : (int)g;
}
inline int rb_passes(unsigned long long max_value) {   // 8-bit radix passes that cover max_value
    int b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return std::max(1, (b + 7) / 8);
}

int mesh_status(int err);
void mesh_note(immesh_mesh* h, const int* c, int frame);
// the host's copy of the counters (the first IM_MC_HOST slots), blocking: the caller has drained what it needs
inline cudaError_t mesh_read_counters(const immesh_mesh* h, int (&c)[immesh::IM_MC_HOST]) { return cudaMemcpy(c, h->M.cnt, sizeof(c), cudaMemcpyDeviceToHost); }
int mesh_growth_check(immesh_mesh* h, long long m);
int mesh_wait_impl(immesh_mesh* h, bool timings);
int mesh_push_dev(immesh_mesh* h, const float* d_world_xyz, int n, const double* pose_t, int kind);
void mesh_frame_begin_launch(const immesh_mesh* h, const immesh::FrameBuf& F, cudaStream_t st, bool pdl);
void mesh_append_launch(const immesh_mesh* h, const immesh::FrameBuf& F, int g, cudaStream_t st, bool pdl);
void mesh_dilate_launch(const immesh_mesh* h, const immesh::FrameBuf& F, cudaStream_t st, bool pdl);
int mesh_tri_launch(const immesh_mesh* h, const immesh::FrameBuf& F, cudaStream_t st, bool pdl);
int queued_cam_stage(immesh_mesh* h, immesh_mesh::QueuedCam& c, int s);
void mesh_reinforce_launch(immesh_mesh* h, cudaStream_t st);
void mesh_view_launch(immesh_mesh* h, cudaStream_t st);
void rf_scan_launch(cudaStream_t st, const int* cnt, int n, int* off);
void mesh_changes_launch(immesh_mesh* h, const immesh::FrameBuf& F, cudaStream_t st, bool batched);
void mesh_feed_begin_launch(immesh_mesh* h, cudaStream_t st);
int mesh_feed_stage(immesh_mesh* h, int s, long long frame, long long n, int step, int kind, const double* pose_t, bool rf, bool img);
void mesh_feed_launch(immesh_mesh* h, cudaStream_t st, bool rf, bool img);
cudaError_t mesh_feed_commit(immesh_mesh* h, long long frame);
void mesh_feed_free(immesh_mesh* h);
int mesh_sort_passes(cudaStream_t st, unsigned int* const k[2], unsigned int* const v[2], int cur, int n, int passes, int* hist, const int* n_dev = nullptr);
size_t mesh_sort_hist_ints(size_t n);
