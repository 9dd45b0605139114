// immesh_b200 -- device-resident voxel-wise incremental mesher.
//
// Reference semantics being reproduced (all /root/reference):
//   append_points_to_global_map      src/meshing/r3live/pointcloud_rgbd.cpp:411-552
//   KD_TREE::Nearest_Search (exact kNN, float)   include/ikd-Tree/ikd_Tree.cpp:441-476, 1097-1279, 1722-1727
//   retrieve_pts_in_voxels / retrieve_neighbor_pts_kdtree   pointcloud_rgbd.cpp:397-407, mesh_rec_geometry.cpp:336-377
//   delaunay_triangulation + is_face_is_ok   src/meshing/mesh_rec_geometry.cpp:24-57, 174-295
//   find_relative_triangulation_combination (pull)   src/meshing/r3live/triangle.hpp:223-246
//   triangle_compare (commit), correct_triangle_index   mesh_rec_geometry.cpp:137-172, 399-433
//   remove_triangle_list / insert_triangle (push)    triangle.hpp:164-221, 330-395
//   incremental_mesh_reconstruction (driver)         src/ImMesh_mesh_reconstruction.cpp:92-267
//
// Data layout in HBM: vertex SoA (float4 position, double3 smoothed position, intrusive per-voxel list,
// incidence-list head), two open-addressed hashes (xi-cell -> vertex, mesh voxel -> voxel record; the slot
// index IS the voxel id), triangle pool (sorted id triple + alive flag, 3 intrusive incidence links, flip
// word) with an open-addressed triple hash.  Per frame: candidate arrays, activated / work voxel lists,
// per-voxel dilated id lists, add / remove lists.
//
// Parallel decomposition: vertex append = lexicographically-first maximal independent set in scan order,
// resolved by priority polling (identical to the sequential greedy loop of the reference); dilation / kNN,
// PCA + Delaunay (Bowyer-Watson with block-wide conflict search and exact integer predicates) and
// pull/commit = one thread block per activated voxel; push = one thread per list entry.
#pragma once
#include <cuda_runtime.h>  // vector types (float4, int4, int2); host-only builds use the same headers
#include <cstring>

#include "hd_math.cuh"
#include "voxelmap.cuh"  // atomics + key packing helpers

#if defined(__CUDA_ARCH__)
#define IM_SYNCBLOCK_M() __syncthreads()
#else
#define IM_SYNCBLOCK_M()
#endif

namespace immesh {

struct MeshParams {
    double xi;         // m_minimum_pts_size
    double res;        // m_voxel_resolution
    double accept;     // g_kd_tree_accept_pt_dis = 1.25 * res (mesh_rec_geometry.cpp:343)
    double knn_max;    // 2 * accept * (1 + 1e-6): beyond this both filters of the dilation ignore a neighbour
    double inv_q;      // 2^22 / res: snapping factor of the exact Delaunay predicates
    int append_target; // appending_pts_frame
};

enum : int { CAND_UNDECIDED = 0, CAND_ACCEPT = 1, CAND_REJECT = 2 };
#define IM_MAXD 1024        // max dilated vertices per voxel
#define IM_MAXG 2048        // max gathered kNN candidates per voxel neighbourhood
#define IM_MAXT (3 * IM_MAXD + 8)
#define IM_MAXPULL 4096
#define IM_MAXF 512         // facets of a voxel with <= 256 dilated vertices (2n - 5 at most)
#define IM_MAXIN 256        // max in-voxel vertices
#define IM_CONF_K 24        // stored earlier-conflict candidates per candidate
#define IM_VCHUNKS 16        // 16 chunks x 16 vertices = IM_MAXIN vertices per mesh voxel

enum : int {
    IM_MERR_VERT_POOL = 1,
    IM_MERR_TRI_POOL = 2,
    IM_MERR_HASH_FULL = 4,
    IM_MERR_VOXEL_CAP = 8,   // a per-voxel working set exceeded IM_MAXD / IM_MAXG / IM_MAXPULL / IM_MAXIN
    IM_MERR_LIST_CAP = 16,   // add/remove/work list overflow
    IM_MERR_KEY_RANGE = 32,
    IM_MERR_PRIO_RANGE = 64, // activated voxel farther than 1024 voxels from the sensor (flip priority)
    IM_MERR_PEER_TIMEOUT = 128,   // sharded mode: a peer rank's epoch flag did not arrive (peer_win.cuh)
    IM_MERR_FEED_INDEX = 256,     // the frame feed computed a slot outside its ring (mesh_feed.cuh): an internal error, nothing written
};

struct MeshDev {
    // vertices
    float4* vpos;        // xyz, w unused
    double* vsmooth;     // [max_v][3]
    unsigned char* vsmoothed;  // [max_v] RGB_pts::m_smoothed: cleared at append, set by every store_smooth (null: not kept)
    int* v_tri_head;     // head of the incidence list
    int max_v;
    // xi-grid hash: cell -> vertex id
    unsigned long long* gkeys;
    int* gval;
    unsigned int gmask;
    // mesh-voxel hash (slot = voxel id)
    unsigned long long* vkeys;
    unsigned int vmask;
    int* vox_chunk;      // [cap][IM_VCHUNKS] ids of the voxel's vertex chunks (-1 = none); vertex k of a voxel lives in
                         // vchunk_pts[vox_chunk[k / 16] * 16 + k % 16] -> a voxel's vertices are fetched with a few wide, independent loads
    float4* vchunk_pts;  // [max_vchunks][16] xyz + vertex id (bit-cast in w)
    int max_vchunks;
    int* vox_count;
    int* vox_meshing_times;
    int* vox_new_added;
    int* vox_frame;
    double* vox_short_axis;  // [cap][3]
    // triangles
    int4* tri;            // a<b<c, alive
    int* tri_next;        // [max_t][3]
    unsigned long long* tri_flip;
    int* thash;           // open addressing on the triple, value = triangle index
    unsigned int tmask;
    int max_t;
    int* cnt;             // [IM_MC_ALLOC] the counter block, slots IM_MC_*
};

// Slots of MeshDev::cnt: name, writer, reset.  "Frame begin" is k_frame_begin (mesh_cnt_frame_begin); "batch" is k_bat_reset
// (mesh_cnt_bat_reset); "chunk" is k_bat_chunk_begin.  The host copies the first IM_MC_HOST slots after every frame.
enum : int {
    IM_MC_VERTICES = 0,        // vertices: the id base of the frame's new ones; += IM_MC_NEW_VERTICES at frame / chunk end; never reset
    IM_MC_TRIS_ALLOC = 1,      // triangle records allocated (tri_add); never reset
    IM_MC_TRIS_LIVE = 2,       // live triangles (tri_add / tri_remove); never reset
    IM_MC_ERR = 3,             // IM_MERR_* flags, or-ed by every stage; never reset
    IM_MC_VOXELS = 4,          // mesh voxels created (cand_init); never reset
    IM_MC_ACT = 5,             // activated voxels of the frame (cand_init); frame begin
    IM_MC_WORK_FRONT = 6,      // front end of the two-ended work list (voxel_enqueue); frame begin, batch; batched frame end: its meshed total
    IM_MC_ADD = 7,             // add-list entries (apply_face); frame begin, batch; batched frame end: its total
    IM_MC_REMOVE = 8,          // remove-list entries (emit_remove, apply_remove); frame begin
    IM_MC_UNDECIDED = 9,       // candidates left undecided by the resolve's poll cap (k_cand_resolve); frame begin, chunk
    IM_MC_NEW_VERTICES = 10,   // vertices the frame appends (cand_commit); frame begin, chunk end; batched frame end: its total
    IM_MC_BBOX_MIN_X = 11,     // key bounding box of the mesh voxels (cand_init), minimum x, y, z; set to +0x7fffffff at create
    IM_MC_BBOX_MIN_Y = 12,
    IM_MC_BBOX_MIN_Z = 13,
    IM_MC_BBOX_MAX_X = 14,     // maximum x, y, z; set to -0x7fffffff at create
    IM_MC_BBOX_MAX_Y = 15,
    IM_MC_BBOX_MAX_Z = 16,
    IM_MC_WORK_BACK = 17,      // back end of the two-ended work list (voxel_enqueue); frame begin, batch, batched frame end
    IM_MC_RESOLVE_TICKET = 18, // block ticket of k_cand_resolve; frame begin, chunk
    IM_MC_TRI_TICKET = 19,     // voxel ticket of k_voxel_tri_warp; frame begin, batch
    IM_MC_STAT_GATHERED = 20,  // work statistics (voxel_dilate, triangulation): kNN candidates gathered, kNN queries, dilated
    IM_MC_STAT_QUERIES = 21,   //   vertices, facets produced; frame begin
    IM_MC_STAT_DILATED = 22,
    IM_MC_STAT_FACETS = 23,
    IM_MC_DILATE_TICKET = 24,  // item ticket of k_voxel_dilate; frame begin, batch
    IM_MC_FACES = 25,          // entries of FrameBuf::all_faces (triangulation); frame begin, batch
    IM_MC_VREFS = 26,          // entries of FrameBuf::all_vref (voxel_dilate); frame begin, batch
    IM_MC_VERT_CHUNKS = 27,    // vertex chunks allocated (cand_commit); never reset
    IM_MC_PULLED = 28,         // entries of FrameBuf::pulled (pull_vertex); frame begin, batch
    IM_MC_DITEMS = 29,         // dilation items (voxel_enqueue); frame begin, batch
    IM_MC_X_FACES = 30,        // sharded frame: entries of FrameBuf::x_face, x_rem, x_smooth (emit_face, emit_remove, emit_smooth); frame begin
    IM_MC_X_REMS = 31,
    IM_MC_X_SMOOTHS = 32,
    IM_MC_BAT_VERTICES = 33,   // batched frame: its new vertices (chunk end), add entries and meshed voxels (batch end), set to
    IM_MC_BAT_ADD = 34,        //   zero with IM_MC_BAT_SELECTED when the batched frame starts
    IM_MC_BAT_MESHED = 35,
    IM_MC_BAT_SELECTED = 36,   // batched frame: voxels its activation rule meshes (k_bat_select)
    IM_MC_HOST = 32,           // slots the host copies back: [0, IM_MC_HOST)
    IM_MC_ALLOC = 64,          // ints allocated
};
// every slot the host reads from its copy (counts, work_stats, capacity, snapshot, growth, the frame's error flags)
static_assert(IM_MC_VERTICES < IM_MC_HOST && IM_MC_TRIS_ALLOC < IM_MC_HOST && IM_MC_TRIS_LIVE < IM_MC_HOST && IM_MC_ERR < IM_MC_HOST &&
              IM_MC_VOXELS < IM_MC_HOST && IM_MC_ACT < IM_MC_HOST && IM_MC_WORK_FRONT < IM_MC_HOST && IM_MC_ADD < IM_MC_HOST &&
              IM_MC_REMOVE < IM_MC_HOST && IM_MC_NEW_VERTICES < IM_MC_HOST && IM_MC_WORK_BACK < IM_MC_HOST &&
              IM_MC_STAT_GATHERED < IM_MC_HOST && IM_MC_STAT_QUERIES < IM_MC_HOST && IM_MC_STAT_DILATED < IM_MC_HOST &&
              IM_MC_STAT_FACETS < IM_MC_HOST && IM_MC_VERT_CHUNKS < IM_MC_HOST, "a slot the host reads lies outside its copy");
static_assert(IM_MC_BAT_SELECTED < IM_MC_ALLOC, "mesh counter block too small");

// ---- the counter bookkeeping of the frame stages (one thread of the kernels in mesh_capi.cu and mesh_batched.cu; the host emulation of the tests)
IM_HD void mesh_cnt_init(int* c) {   // create: c holds IM_MC_HOST zeros
    c[IM_MC_BBOX_MIN_X] = c[IM_MC_BBOX_MIN_Y] = c[IM_MC_BBOX_MIN_Z] = 0x7fffffff;
    c[IM_MC_BBOX_MAX_X] = c[IM_MC_BBOX_MAX_Y] = c[IM_MC_BBOX_MAX_Z] = -0x7fffffff;
}
IM_HD void mesh_cnt_frame_begin(const MeshDev& M) {
    M.cnt[IM_MC_ACT] = 0; M.cnt[IM_MC_WORK_FRONT] = 0; M.cnt[IM_MC_ADD] = 0; M.cnt[IM_MC_REMOVE] = 0; M.cnt[IM_MC_UNDECIDED] = 0;
    M.cnt[IM_MC_NEW_VERTICES] = 0; M.cnt[IM_MC_WORK_BACK] = 0; M.cnt[IM_MC_RESOLVE_TICKET] = 0; M.cnt[IM_MC_TRI_TICKET] = 0;
    M.cnt[IM_MC_STAT_GATHERED] = 0; M.cnt[IM_MC_STAT_QUERIES] = 0; M.cnt[IM_MC_STAT_DILATED] = 0; M.cnt[IM_MC_STAT_FACETS] = 0;
    M.cnt[IM_MC_DILATE_TICKET] = 0; M.cnt[IM_MC_FACES] = 0; M.cnt[IM_MC_VREFS] = 0; M.cnt[IM_MC_PULLED] = 0; M.cnt[IM_MC_DITEMS] = 0;
    M.cnt[IM_MC_X_FACES] = 0; M.cnt[IM_MC_X_REMS] = 0; M.cnt[IM_MC_X_SMOOTHS] = 0;
}
IM_HD void mesh_cnt_frame_end(const MeshDev& M) { M.cnt[IM_MC_VERTICES] += M.cnt[IM_MC_NEW_VERTICES]; }
// batched frame: the start of an append chunk after the first, its end (the chunk's vertices are in the map before the next chunk
// is examined), the per-batch lists, the end of a batch, the end of the frame (the per-frame totals written back)
IM_HD void mesh_cnt_bat_chunk_begin(const MeshDev& M) { M.cnt[IM_MC_UNDECIDED] = 0; M.cnt[IM_MC_RESOLVE_TICKET] = 0; }
IM_HD void mesh_cnt_bat_chunk_end(const MeshDev& M) {
    M.cnt[IM_MC_VERTICES] += M.cnt[IM_MC_NEW_VERTICES];
    M.cnt[IM_MC_BAT_VERTICES] += M.cnt[IM_MC_NEW_VERTICES];
    M.cnt[IM_MC_NEW_VERTICES] = 0;
}
IM_HD void mesh_cnt_bat_reset(const MeshDev& M) {
    M.cnt[IM_MC_WORK_FRONT] = 0; M.cnt[IM_MC_ADD] = 0; M.cnt[IM_MC_WORK_BACK] = 0; M.cnt[IM_MC_TRI_TICKET] = 0;
    M.cnt[IM_MC_DILATE_TICKET] = 0; M.cnt[IM_MC_FACES] = 0; M.cnt[IM_MC_VREFS] = 0; M.cnt[IM_MC_PULLED] = 0; M.cnt[IM_MC_DITEMS] = 0;
}
IM_HD void mesh_cnt_bat_batch_end(const MeshDev& M) {
    M.cnt[IM_MC_BAT_ADD] += M.cnt[IM_MC_ADD];
    M.cnt[IM_MC_BAT_MESHED] += M.cnt[IM_MC_WORK_FRONT] + M.cnt[IM_MC_WORK_BACK];
}
IM_HD void mesh_cnt_bat_frame_end(const MeshDev& M) {
    M.cnt[IM_MC_NEW_VERTICES] = M.cnt[IM_MC_BAT_VERTICES];
    M.cnt[IM_MC_ADD] = M.cnt[IM_MC_BAT_ADD];
    M.cnt[IM_MC_WORK_FRONT] = M.cnt[IM_MC_BAT_MESHED];
    M.cnt[IM_MC_WORK_BACK] = 0;
}

struct FramePose {        // per-frame sensor position (device resident so that a frame can be queued behind the localization)
    double pose_t[3];
    long long prio_origin[3];  // floor(pose_t / res) - 1024: origin of the 11-bit-per-axis voxel rank used by the flip priority
};
struct XSmooth { int id, pad; double x, y, z; };   // 32 B
// Per-frame inputs of the launch sequence, device resident (one small H2D per frame): the captured CUDA graph of a frame is
// replayed without touching its nodes, every kernel takes the frame's values from here (frame_load_dyn).
struct FrameDyn {
    const float* pts;     // world-frame scan of this frame (staging slot, or the caller's device buffer)
    const float* body;    // body-frame scan when the frame is handed over by the localization handle (transformed into pts first)
    FramePose* fp;
    int n, step, m, frame;
    unsigned int cmask;
    int pose_idx;         // slot of LioCtrl::pose_ring holding the pose the scan converged to
    unsigned long long epoch;   // peer-window epoch of this frame (sharded mode)
    const int* n_dev;     // a handed-over frame whose count is device resident: n is read here, and n, step, m, cmask set (k_transform_full)
};
struct FrameBuf {
    const float* pts;     // [n][3] world-frame scan
    int n, step, m;       // m = number of candidates = ceil(n / step)
    int frame;            // internal monotonically increasing frame counter
    const FramePose* fp;
    const FrameDyn* dyn;  // device: the seven per-frame fields above + cmask + epoch are taken from here by the kernels
    unsigned long long epoch;
    // candidates
    unsigned long long* cand_gkey;
    int* cand_vslot;
    int* cand_status;
    int* cand_scan;       // exclusive scan of accept flags
    int* cand_conf;       // [m][IM_CONF_K]
    int* cand_nconf;      // count, or -1 when the list overflowed
    int* cand_next;       // next candidate in the same xi-cell (per-frame candidate grid)
    int* cand_pos;        // position of an accepted candidate inside its mesh voxel
    unsigned long long* ckeys;  // per-frame candidate grid
    int* chead;
    unsigned int cmask;
    int* scan_block;      // block sums for the scan
    // voxel lists
    int* act;             // activated voxel slots
    int* work;            // voxels to (re)mesh this frame
    int* work_n_ids;      // dilated set sizes
    int* work_ids;        // [max_work][IM_MAXD] ascending vertex ids
    unsigned int* work_bits;  // [max_work][IM_MAXG/32] dilation-member bitmap shared by the groups of a voxel
    int* work_ring;       // largest ring any group of the voxel gathered
    int* work_done;       // groups of the voxel that have finished
    int* ditem;           // dilation items: work slot << 5 | query group
    int max_ditem;
    int* work_nfaces;     // facets produced by the fused dilate+triangulate stage (-1: left to the large variant)
    int4* all_faces;      // compact list of this frame's new facets: (a, b, c, work slot)   [max_list]
    int* all_vref;        // compact list of (work slot << 10 | index into its dilated id list) [max_vref]
    int* pulled;          // [max_list][2] (work slot, triangle) pairs found by the pull stage
    int* fset;            // open-addressed set over all_faces (value = facet index), cleared per frame
    unsigned int fset_mask;
    int max_vref;
    double* work_axes;    // [max_work][9] short / mid / long axis of the voxel's PCA frame
    // push lists
    int* add_tri;         // [max_list][3]
    unsigned long long* add_flip;
    int* rem_tri;         // [max_list] triangle indices
    int max_cand, max_act, max_work, max_list;
    // multi-GPU: the per-voxel stage of a frame is sharded by mesh-voxel owner; what a rank produces is recorded in these
    // exchange lists (all-gathered, then applied by every rank to its replica of the store) instead of being applied
    int shard_rank, shard_n;
    int x_cap;            // capacity of each exchange list (entries)
    XSmooth* x_smooth;    // smoothed positions written by this rank's dilations
    int4* x_face;         // new facets (a, b, c, -) of this rank's voxels
    unsigned long long* x_word;   // their flip-priority words
    int4* x_rem;          // triangles (a, b, c, -) this rank's voxels want removed
    // batched frame (immesh_mesh_push_frame_batched: one frame's per-voxel stage in several batches); null on the per-frame path
    const int* work_rank; // [max_work] flip priority of the work voxel: its rank among the frame's meshed voxels in (x, y, z) key order
    unsigned char* tri_mark;   // [max_t] IM_TRI_BORN: made live by an earlier batch of this frame; IM_TRI_REMOVE: removal deferred to the frame's end
    // change feed (immesh_mesh_changes_enable; chg_stamp null: off): the frame number of each triangle slot's first touch, the
    // frame's touched slots and the feed's counter block (slots IM_CH_*)
    int* chg_stamp;       // [max_t]
    int* chg_list;        // [chg_cap]
    int* chg_cnt;
    int chg_cap;
};
enum : unsigned char { IM_TRI_BORN = 1, IM_TRI_REMOVE = 2 };
// Slots of FrameBuf::chg_cnt: name, writer.  All three are reset by chg_frame_end (mesh_changes.cuh) and at enable.
enum : int {
    IM_CH_TOUCHED = 0,   // touched slots listed (chg_touch); may exceed chg_cap: the frame then falls back to a sweep
    IM_CH_SWEPT = 1,     // slots listed by the sweep (chg_sweep_slot)
    IM_CH_ROWS = 2,      // rows of the frame (k_chg_rows)
    IM_CH_SIZE = 4,
};
// a live triangle that was live before the frame began (the only ones the frame's pull and commit see)
IM_HD bool tri_pre_frame(const FrameBuf& F, int t) { return !F.tri_mark || F.tri_mark[t] != IM_TRI_BORN; }

IM_HD FrameBuf frame_load_dyn(const FrameBuf& F) {
    FrameBuf o = F;
    if (F.dyn) {
        const FrameDyn d = *F.dyn;
        o.pts = d.pts; o.n = d.n; o.step = d.step; o.m = d.m; o.frame = d.frame; o.fp = d.fp; o.cmask = d.cmask; o.epoch = d.epoch;
    }
    return o;
}

// ------------------------------------------------------------------ keys
IM_HD int round_key(float x, double cell) { return (int)round((double)x / cell); }  // std::round, pointcloud_rgbd.cpp:467-472
IM_HD unsigned long long pack_ikey(int x, int y, int z) {
    return ((unsigned long long)(unsigned int)(x + 1048576) << 42) | ((unsigned long long)(unsigned int)(y + 1048576) << 21) | (unsigned long long)(unsigned int)(z + 1048576);
}
IM_HD bool ikey_ok(int x, int y, int z) { return x > -1048000 && x < 1048000 && y > -1048000 && y < 1048000 && z > -1048000 && z < 1048000; }
IM_HD void unpack_ikey(unsigned long long k, int* x, int* y, int* z) {
    *x = (int)((k >> 42) & 0x1FFFFF) - 1048576;
    *y = (int)((k >> 21) & 0x1FFFFF) - 1048576;
    *z = (int)(k & 0x1FFFFF) - 1048576;
}
IM_HD int table_find(const unsigned long long* keys, unsigned int mask, unsigned long long key) {
    unsigned int s = hash_key(key) & mask;
    for (unsigned int probe = 0; probe <= mask; ++probe) {
        const unsigned long long k = keys[s];
        if (k == key) return (int)s;
        if (k == IM_EMPTY_KEY) return -1;
        s = (s + 1) & mask;
    }
    return -1;
}
IM_HD int table_insert(unsigned long long* keys, unsigned int mask, unsigned long long key, int* created) {
    unsigned int s = hash_key(key) & mask;
    *created = 0;
    for (unsigned int probe = 0; probe <= mask; ++probe) {
        unsigned long long k = keys[s];
        if (k == key) return (int)s;
        if (k == IM_EMPTY_KEY) {
            k = im_atomic_cas64(&keys[s], IM_EMPTY_KEY, key);
            if (k == IM_EMPTY_KEY) { *created = 1; return (int)s; }
            if (k == key) return (int)s;
        }
        s = (s + 1) & mask;
    }
    return -1;
}
IM_HD int im_atomic_exch(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicExch(p, v);
#else
    const int o = *p; *p = v; return o;
#endif
}
IM_HD int im_atomic_cas32(int* p, int cmp, int v) {
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, cmp, v);
#else
    const int o = *p; if (o == cmp) *p = v; return o;
#endif
}
IM_HD int im_atomic_min(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicMin(p, v);
#else
    const int o = *p; if (v < o) *p = v; return o;
#endif
}
IM_HD int im_atomic_max(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicMax(p, v);
#else
    const int o = *p; if (v > o) *p = v; return o;
#endif
}
IM_HD unsigned long long im_atomic_max64(unsigned long long* p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    return atomicMax(p, v);
#else
    const unsigned long long o = *p; if (v > o) *p = v; return o;
#endif
}
IM_HD int im_vload(const int* p) {
#if defined(__CUDA_ARCH__)
    return *(const volatile int*)p;
#else
    return *p;
#endif
}
IM_HD void im_fence() {
#if defined(__CUDA_ARCH__)
    __threadfence();
#endif
}
// change feed: the first touch of triangle slot t in this frame puts it on the frame's list (once, whichever writer comes first)
IM_HD void chg_touch(const FrameBuf& F, int t) {
    if (!F.chg_stamp || im_atomic_exch(&F.chg_stamp[t], F.frame) == F.frame) return;
    const int e = im_atomic_add(&F.chg_cnt[IM_CH_TOUCHED], 1);
    if (e < F.chg_cap) F.chg_list[e] = t;
}
// float squared distance exactly as KD_TREE::calc_dist (ikd_Tree.cpp:1722-1727): ((dx*dx + dy*dy) + dz*dz), no FMA
IM_HD float dist2f(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = ax - bx, dy = ay - by, dz = az - bz;
    return (dx * dx + dy * dy) + dz * dz;
}

// ------------------------------------------------------------------ M1: candidates (thread per candidate)
// pointcloud_rgbd.cpp:464-517: grid / voxel keys, voxel get-or-create + activation, rejection against the
// vertices of earlier frames (occupied xi-cell, or an existing vertex closer than xi).
IM_HDN inline void cand_init(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int c) {
    IM_STAMP(53, 0);
    const float* p = F.pts + (size_t)c * F.step * 3;
    const float px = p[0], py = p[1], pz = p[2];
    IM_STAMP(54, __float_as_int(px + py + pz));
    const int gx = round_key(px, P.xi), gy = round_key(py, P.xi), gz = round_key(pz, P.xi);
    const int bx = round_key(px, P.res), by = round_key(py, P.res), bz = round_key(pz, P.res);
    F.cand_status[c] = CAND_REJECT;
    F.cand_vslot[c] = -1;
    F.cand_nconf[c] = 0;
    F.cand_next[c] = -1;
    if (!ikey_ok(gx, gy, gz) || !ikey_ok(bx, by, bz)) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_KEY_RANGE); return; }
    const unsigned long long gkey = pack_ikey(gx, gy, gz);
    F.cand_gkey[c] = gkey;
    // voxel get-or-create (:482-495); every examined point activates its voxel, accepted or not
    int created = 0;
    const int vs = table_insert(M.vkeys, M.vmask, pack_ikey(bx, by, bz), &created);
    if (vs < 0) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); return; }
    IM_STAMP(55, vs);
    if (created) {
        im_atomic_add(&M.cnt[IM_MC_VOXELS], 1);
        im_atomic_min(&M.cnt[IM_MC_BBOX_MIN_X], bx); im_atomic_min(&M.cnt[IM_MC_BBOX_MIN_Y], by); im_atomic_min(&M.cnt[IM_MC_BBOX_MIN_Z], bz);
        im_atomic_max(&M.cnt[IM_MC_BBOX_MAX_X], bx); im_atomic_max(&M.cnt[IM_MC_BBOX_MAX_Y], by); im_atomic_max(&M.cnt[IM_MC_BBOX_MAX_Z], bz);
    }
    F.cand_vslot[c] = vs;
    if (im_atomic_exch(&M.vox_frame[vs], F.frame) != F.frame) {
        const int a = im_atomic_add(&M.cnt[IM_MC_ACT], 1);
        if (a < F.max_act) F.act[a] = vs; else im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP);
    }
    IM_STAMP(56, 0);
    // occupied xi-cell (:473-481)
    const int occupied = table_find(M.gkeys, M.gmask, gkey);
    IM_STAMP(57, occupied);
    if (occupied >= 0) return;
    // nearest existing vertex closer than xi (:507-517): any vertex with sqrtf(d2) < xi lies in the 27 surrounding cells.
    // The 27 first-probe loads are issued together (independent addresses) before any of them is consumed.
    {
        unsigned long long want[27], got[27];
        unsigned int slot[27];
#pragma unroll
        for (int q = 0; q < 27; ++q) {
            want[q] = pack_ikey(gx + (q / 9 - 1), gy + ((q / 3) % 3 - 1), gz + (q % 3 - 1));
            slot[q] = hash_key(want[q]) & M.gmask;
        }
#pragma unroll
        for (int q = 0; q < 27; ++q) got[q] = M.gkeys[slot[q]];
        int vid[27];
#pragma unroll
        for (int q = 0; q < 27; ++q) {
            int s = -1;
            if (got[q] == want[q]) s = (int)slot[q];
            else if (got[q] != IM_EMPTY_KEY) s = table_find(M.gkeys, M.gmask, want[q]);  // collision chain: rare
            vid[q] = s >= 0 ? M.gval[s] : -1;
        }
        IM_STAMP(58, vid[0] + vid[13] + vid[26]);
        bool close = false;
#pragma unroll
        for (int q = 0; q < 27; ++q) {
            if (vid[q] < 0) continue;
            const float4 v = M.vpos[vid[q]];
            if ((double)sqrtf(dist2f(px, py, pz, v.x, v.y, v.z)) < P.xi) close = true;
        }
        IM_STAMP(59, close);
        if (close) return;
    }
    // survives the old map: enters the per-frame candidate grid, decided in cand_resolve
    F.cand_status[c] = CAND_UNDECIDED;
    int cc = 0;
    const int cs = table_insert(F.ckeys, F.cmask, gkey, &cc);
    if (cs < 0) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); F.cand_status[c] = CAND_REJECT; return; }
    // push onto the cell's candidate list
#if defined(__CUDA_ARCH__)
    // The lists are only walked by the kernels after this one, so the moment in which the head already names c while c's link is not
    // stored yet is never observed: one exchange, no fence, no retry.  (A next-store / fence / compare-and-swap loop stood here; the
    // stamps put most of this function's cycles into it.)
    F.cand_next[c] = atomicExch(&F.chead[cs], c);
#else
    F.cand_next[c] = F.chead[cs];
    F.chead[cs] = c;
#endif
    IM_STAMP(60, 0);
}

// earlier candidates that conflict with c: same xi-cell (:473-481 on a vertex accepted earlier in this frame) or
// closer than xi (:507-517).  Fills cand_conf (or marks overflow).
IM_HDN inline void cand_conflicts(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int c) {
    if (F.cand_status[c] != CAND_UNDECIDED) return;
    const float* p = F.pts + (size_t)c * F.step * 3;
    int gx, gy, gz;
    unpack_ikey(F.cand_gkey[c], &gx, &gy, &gz);
    int n = 0;
    bool overflow = false;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dz = -1; dz <= 1; ++dz) {
                const int cs = table_find(F.ckeys, F.cmask, pack_ikey(gx + dx, gy + dy, gz + dz));
                if (cs < 0) continue;
                const bool same = (dx == 0 && dy == 0 && dz == 0);
                for (int j = F.chead[cs]; j >= 0; j = F.cand_next[j]) {
                    if (j >= c) continue;
                    const float* q = F.pts + (size_t)j * F.step * 3;
                    if (same || (double)sqrtf(dist2f(p[0], p[1], p[2], q[0], q[1], q[2])) < P.xi) {
                        if (n < IM_CONF_K) F.cand_conf[(size_t)c * IM_CONF_K + n] = j;
                        else overflow = true;
                        ++n;
                    }
                }
            }
    F.cand_nconf[c] = overflow ? -1 : n;
}

// one polling pass for candidate c: accepted iff every earlier conflicting candidate is rejected, rejected iff one
// of them is accepted.  Returns true when decided.  (Sequential greedy semantics of :464-545.)
IM_HDN inline bool cand_poll(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int c) {
    bool pending = false;
    const int nc = F.cand_nconf[c];
    if (nc >= 0) {
        for (int k = 0; k < nc; ++k) {
            const int s = im_vload(&F.cand_status[F.cand_conf[(size_t)c * IM_CONF_K + k]]);
            if (s == CAND_ACCEPT) { F.cand_status[c] = CAND_REJECT; return true; }
            if (s == CAND_UNDECIDED) pending = true;
        }
    } else {
        const float* p = F.pts + (size_t)c * F.step * 3;
        int gx, gy, gz;
        unpack_ikey(F.cand_gkey[c], &gx, &gy, &gz);
        for (int dx = -1; dx <= 1; ++dx)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dz = -1; dz <= 1; ++dz) {
                    const int cs = table_find(F.ckeys, F.cmask, pack_ikey(gx + dx, gy + dy, gz + dz));
                    if (cs < 0) continue;
                    const bool same = (dx == 0 && dy == 0 && dz == 0);
                    for (int j = F.chead[cs]; j >= 0; j = F.cand_next[j]) {
                        if (j >= c) continue;
                        const float* q = F.pts + (size_t)j * F.step * 3;
                        if (same || (double)sqrtf(dist2f(p[0], p[1], p[2], q[0], q[1], q[2])) < P.xi) {
                            const int s = im_vload(&F.cand_status[j]);
                            if (s == CAND_ACCEPT) { F.cand_status[c] = CAND_REJECT; return true; }
                            if (s == CAND_UNDECIDED) pending = true;
                        }
                    }
                }
    }
    if (pending) return false;
    F.cand_status[c] = CAND_ACCEPT;
    return true;
}

// accepted candidate -> vertex (pointcloud_rgbd.cpp:518-540); id = vertices before the frame + accepted before c
IM_HDN inline void cand_commit(const MeshDev& M, const MeshParams& P, const FrameBuf& F, int c, int base) {
    if (F.cand_status[c] != CAND_ACCEPT) return;
    const int id = base + F.cand_scan[c];
    if (id >= M.max_v) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VERT_POOL); return; }
    const float* p = F.pts + (size_t)c * F.step * 3;
    M.vpos[id] = make_float4(p[0], p[1], p[2], 0.f);
    M.vsmooth[(size_t)id * 3 + 0] = (double)p[0];
    M.vsmooth[(size_t)id * 3 + 1] = (double)p[1];
    M.vsmooth[(size_t)id * 3 + 2] = (double)p[2];
    if (M.vsmoothed) M.vsmoothed[id] = 0;
    M.v_tri_head[id] = -1;
    int created = 0;
    const int gs = table_insert(M.gkeys, M.gmask, F.cand_gkey[c], &created);
    if (gs < 0) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); return; }
    M.gval[gs] = id;
    const int vs = F.cand_vslot[c];
    const int pos = im_atomic_add(&M.vox_count[vs], 1);
    F.cand_pos[c] = pos;
    if (pos >= IM_VCHUNKS * 16) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VOXEL_CAP); F.cand_pos[c] = -1; }
    else if ((pos & 15) == 0) {   // first vertex of a chunk: allocate it (published for the placement kernel that follows)
        const int ch = im_atomic_add(&M.cnt[IM_MC_VERT_CHUNKS], 1);
        if (ch >= M.max_vchunks) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_VERT_POOL); F.cand_pos[c] = -1; }
        else M.vox_chunk[(size_t)vs * IM_VCHUNKS + (pos >> 4)] = ch;
    }
    im_atomic_add(&M.vox_new_added[vs], 1);
    M.vox_meshing_times[vs] = 0;
    im_atomic_add(&M.cnt[IM_MC_NEW_VERTICES], 1);
}

// chunk id of a voxel's chunk table entry for the readers: an entry left at -1 by a chunk-pool overflow (the frame fails with
// VERT_POOL) reads chunk 0 instead of memory before the pool
IM_HD int im_chunk_or0(int ch) { return ch < 0 ? 0 : ch; }
// second half of the append: the vertex goes into its voxel's chunk (the chunk table is complete after cand_commit)
IM_HDN inline void cand_place(const MeshDev& M, const FrameBuf& F, int c, int base) {
    if (F.cand_status[c] != CAND_ACCEPT || F.cand_pos[c] < 0) return;
    const int id = base + F.cand_scan[c];
    if (id >= M.max_v) return;
    const int vs = F.cand_vslot[c], pos = F.cand_pos[c];
    const int ch = M.vox_chunk[(size_t)vs * IM_VCHUNKS + (pos >> 4)];
    if (ch < 0) return;   // the chunk pool overflowed in cand_commit (VERT_POOL raised): nowhere to put the vertex
    const float* p = F.pts + (size_t)c * F.step * 3;
    float4 v;
    v.x = p[0]; v.y = p[1]; v.z = p[2];
    int idb = id;
    memcpy(&v.w, &idb, 4);
    M.vchunk_pts[(size_t)ch * 16 + (pos & 15)] = v;
}

// activation test of ImMesh_mesh_reconstruction.cpp:132-151 on activated voxel vs: true when this rank meshes it in this frame
IM_HD bool voxel_activate(const MeshDev& M, const FrameBuf& F, int vs) {
    if (M.vox_meshing_times[vs] >= 1 || M.vox_new_added[vs] < 0) return false;
    M.vox_meshing_times[vs] += 1;
    M.vox_new_added[vs] = 0;
    if (M.vox_count[vs] < 3) return false;
    if (F.shard_n > 1 && voxel_owner(M.vkeys[vs], F.shard_n) != F.shard_rank) return false;   // another rank meshes this voxel
    return true;
}
// voxel vs -> work list + dilation items; returns its work slot (-1: the work list is full)
IM_HDN inline int voxel_enqueue(const MeshDev& M, const FrameBuf& F, int vs) {
    // two-ended work list: populous voxels (the expensive ones) from the front, the rest from the back, so that the
    // per-voxel stages start the long jobs first (IM_MC_WORK_FRONT counts from the front, IM_MC_WORK_BACK from the back)
    int w;
    if (M.vox_count[vs] >= 20) w = im_atomic_add(&M.cnt[IM_MC_WORK_FRONT], 1);
    else w = F.max_work - 1 - im_atomic_add(&M.cnt[IM_MC_WORK_BACK], 1);
    if (w >= 0 && w < F.max_work && M.cnt[IM_MC_WORK_FRONT] + M.cnt[IM_MC_WORK_BACK] <= F.max_work) F.work[w] = vs; else { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); return -1; }
    // dilation items: groups of up to 8 of the voxel's vertices (the kNN queries), so that a populous voxel is spread over
    // several thread blocks instead of serialising on one
    int nq = M.vox_count[vs];
    if (nq > IM_MAXIN) nq = IM_MAXIN;
    const int ng = (nq + 7) >> 3;
    const int base = im_atomic_add(&M.cnt[IM_MC_DITEMS], ng);
    if (base + ng > F.max_ditem) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); return w; }
    for (int g = 0; g < ng; ++g) F.ditem[base + g] = (w << 5) | g;
    return w;
}
// thread per activated voxel
IM_HDN inline void voxel_select(const MeshDev& M, const FrameBuf& F, int a) {
    const int vs = F.act[a];
    if (voxel_activate(M, F, vs)) voxel_enqueue(M, F, vs);
}
// Flip-priority field (33 bits) of the facets of work voxel w: the frame word keeps the largest, so among a frame's voxels the last
// in ascending (x, y, z) key order wins.  Per-frame path: the key relative to prio_origin, 11 bits per axis (IM_MERR_PRIO_RANGE
// beyond 1024 voxels from the sensor).  Batched frame: the voxel's rank among the frame's meshed voxels in the same order -- the same
// winner wherever the 11-bit field is in range, and no range limit.
IM_HD unsigned long long voxel_prio(const MeshDev& M, const FrameBuf& F, int w, bool report) {
    if (F.work_rank) return (unsigned long long)(unsigned int)F.work_rank[w];
    int kx, ky, kz;
    unpack_ikey(M.vkeys[F.work[w]], &kx, &ky, &kz);
    const long long lx = kx - F.fp->prio_origin[0], ly = ky - F.fp->prio_origin[1], lz = kz - F.fp->prio_origin[2];
    if (report && (lx < 0 || lx >= 2048 || ly < 0 || ly >= 2048 || lz < 0 || lz >= 2048)) im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_PRIO_RANGE);
    return ((unsigned long long)(lx & 2047) << 22) | ((unsigned long long)(ly & 2047) << 11) | (unsigned long long)(lz & 2047);
}

// i-th work item (0 <= i < IM_MC_WORK_FRONT + IM_MC_WORK_BACK entries) -> slot in the two-ended work arrays
IM_HD int work_slot(const MeshDev& M, const FrameBuf& F, int i) {
    const int na = M.cnt[IM_MC_WORK_FRONT];
    return i < na ? i : F.max_work - 1 - (i - na);
}
IM_HD int work_total(const MeshDev& M, const FrameBuf& F) {
    const int t = M.cnt[IM_MC_WORK_FRONT] + M.cnt[IM_MC_WORK_BACK];
    return t < F.max_work ? t : F.max_work;
}

// ------------------------------------------------------------------ exact integer predicates
IM_HD int orient2d_i(int ax, int ay, int bx, int by, int cx, int cy) {
    const long long d = (long long)(bx - ax) * (long long)(cy - ay) - (long long)(by - ay) * (long long)(cx - ax);
    return (d > 0) - (d < 0);
}
// > 0 iff d strictly inside the circumcircle of the counter-clockwise triangle (a,b,c).
// double filter on exactly representable integers, exact __int128 fallback.
IM_HDN inline int incircle_i(int ax, int ay, int bx, int by, int cx, int cy, int dx, int dy) {
    const long long adx = (long long)ax - dx, ady = (long long)ay - dy, bdx = (long long)bx - dx, bdy = (long long)by - dy, cdx = (long long)cx - dx, cdy = (long long)cy - dy;
    const long long al = adx * adx + ady * ady, bl = bdx * bdx + bdy * bdy, cl = cdx * cdx + cdy * cdy;
    const long long m1 = bdx * cdy - bdy * cdx, m2 = cdx * ady - cdy * adx, m3 = adx * bdy - ady * bdx;
    // |coordinates| < 2^25 => lifts and minors < 2^52: exact in double; three products are rounded once each
    const double t1 = (double)al * (double)m1, t2 = (double)bl * (double)m2, t3 = (double)cl * (double)m3;
    const double det = (t1 + t2) + t3;
    const double bound = ((fabs(t1) + fabs(t2)) + fabs(t3)) * 1.0e-15;
    if (det > bound) return 1;
    if (det < -bound) return -1;
    const __int128 ex = (__int128)al * (__int128)m1 + (__int128)bl * (__int128)m2 + (__int128)cl * (__int128)m3;
    return (ex > 0) - (ex < 0);
}

struct DTri { short v[3]; short alive; };  // local vertex indices, -1 = ghost vertex
#define IM_GHOST (-1)

// conflict test of the Bowyer-Watson step: finite triangle -> strict in-circle; ghost (u,v,inf) -> strictly left of
// u->v, or on the open segment uv
IM_HDN inline bool dt_conflict(const DTri& t, const int2* P, int p) {
    const int px = P[p].x, py = P[p].y;
    for (int i = 0; i < 3; ++i)
        if (t.v[i] == IM_GHOST) {
            const int u = t.v[(i + 1) % 3], v = t.v[(i + 2) % 3];
            const int o = orient2d_i(P[u].x, P[u].y, P[v].x, P[v].y, px, py);
            if (o > 0) return true;
            if (o < 0) return false;
            const long long dx = (long long)P[v].x - P[u].x, dy = (long long)P[v].y - P[u].y;
            const long long t1 = ((long long)px - P[u].x) * dx + ((long long)py - P[u].y) * dy;
            const long long t2 = ((long long)px - P[v].x) * dx + ((long long)py - P[v].y) * dy;
            return t1 > 0 && t2 < 0;
        }
    return incircle_i(P[t.v[0]].x, P[t.v[0]].y, P[t.v[1]].x, P[t.v[1]].y, P[t.v[2]].x, P[t.v[2]].y, px, py) > 0;
}

// float circumcircle (centre, padded squared radius) used only to prune the exact in-circle tests
IM_HD void circumcircle_f(const int2* P, int a, int b, int c, float* out) {
    const double bx = (double)(P[b].x - P[a].x), by = (double)(P[b].y - P[a].y);
    const double cx = (double)(P[c].x - P[a].x), cy = (double)(P[c].y - P[a].y);
    const double d = 2.0 * (bx * cy - by * cx);
    const double b2 = bx * bx + by * by, c2 = cx * cx + cy * cy;
    // one float reciprocal refined by a Newton step instead of two double divisions (this is only a pruning filter;
    // the 0.2 % padding below dwarfs the ~1e-14 relative error); d == 0 gives inf/nan -> the guard below disables the filter
    double inv = (double)(1.0f / (float)d);
    inv = inv * (2.0 - d * inv);
    const double ux = (cy * b2 - by * c2) * inv, uy = (bx * c2 - cx * b2) * inv;
    const double r2 = ux * ux + uy * uy;
    const double ccx = (double)P[a].x + ux, ccy = (double)P[a].y + uy;
    if (!(fabs(ccx) < 1.0e9) || !(fabs(ccy) < 1.0e9) || !(r2 < 1.0e18)) { out[0] = 0.f; out[1] = 0.f; out[2] = INFINITY; return; }
    out[0] = (float)ccx; out[1] = (float)ccy;
    out[2] = (float)(r2 * 1.002) + 64.0f;   // conservative: float rounding of centre/radius is ~1e-6 relative
}

// Block-cooperative Delaunay triangulation of n snapped points (Bowyer-Watson, exact predicates, insertion in
// index order after a non-degenerate seed).  tris/ntri: triangle pool in shared memory.  scratch: >= 784 ints
// (scratch[4] = seed found, scratch[6] = capacity overflow).
// Returns (via *ntri) the pool size; dead slots have alive == 0.  ok=false when all points are collinear.
IM_HDN inline void delaunay_block(const int2* P, int n, DTri* tris, int max_tris, int* ntri, int* scratch, int tid, int nthreads, float (*circ)[3] = nullptr) {
    int* s_cav_n = scratch;        // [0]
    int* s_edge_n = scratch + 1;   // [1]
    int* s_seed = scratch + 2;     // [2..4] i1, i2, ok
    int* s_new_n = scratch + 5;
    int* s_ovf = scratch + 6;      // [6] cavity / pool overflow flag
    int* s_cav = scratch + 8;      // [256] cavity triangle indices
    int* s_edges = scratch + 264;  // [260*2] boundary edges (a,b)
    if (tid == 0) {
        *s_ovf = 0;
        int i1 = -1, i2 = -1;
        for (int i = 1; i < n; ++i)
            if (P[i].x != P[0].x || P[i].y != P[0].y) { i1 = i; break; }
        if (i1 >= 0)
            for (int i = 1; i < n; ++i)
                if (i != i1 && orient2d_i(P[0].x, P[0].y, P[i1].x, P[i1].y, P[i].x, P[i].y) != 0) { i2 = i; break; }
        s_seed[0] = i1; s_seed[1] = i2; s_seed[2] = (i1 >= 0 && i2 >= 0) ? 1 : 0;
        *ntri = 0;
        if (s_seed[2]) {
            int a = 0, b = i1, c = i2;
            if (orient2d_i(P[a].x, P[a].y, P[b].x, P[b].y, P[c].x, P[c].y) < 0) { const int t = b; b = c; c = t; }
            const short tv[4][3] = {{(short)a, (short)b, (short)c}, {(short)c, (short)b, IM_GHOST}, {(short)a, (short)c, IM_GHOST}, {(short)b, (short)a, IM_GHOST}};
            for (int k = 0; k < 4; ++k) { tris[k].v[0] = tv[k][0]; tris[k].v[1] = tv[k][1]; tris[k].v[2] = tv[k][2]; tris[k].alive = 1; }
            if (circ) circumcircle_f(P, a, b, c, circ[0]);
            *ntri = 4;
        }
    }
    IM_SYNCBLOCK_M();
    if (!s_seed[2]) return;
    const int i1 = s_seed[0], i2 = s_seed[1];
    for (int p = 1; p < n; ++p) {
        if (p == i1 || p == i2) continue;
        if (tid == 0) { *s_cav_n = 0; *s_edge_n = 0; *s_new_n = 0; }
        IM_SYNCBLOCK_M();
        const int nt = *ntri;
        const float pxf = (float)P[p].x, pyf = (float)P[p].y;
        for (int t = tid; t < nt; t += nthreads) {
            if (!tris[t].alive) continue;
            if (circ && tris[t].v[0] != IM_GHOST && tris[t].v[1] != IM_GHOST && tris[t].v[2] != IM_GHOST) {
                const float dx = pxf - circ[t][0], dy = pyf - circ[t][1];
                if (dx * dx + dy * dy > circ[t][2]) continue;   // certainly outside the circumcircle
            }
            if (dt_conflict(tris[t], P, p)) {
                const int k = im_atomic_add(s_cav_n, 1);
                if (k < 256) s_cav[k] = t;
            }
        }
        IM_SYNCBLOCK_M();
        int nc = *s_cav_n;
        if (nc > 256) { nc = 256; *s_ovf = 1; }
        // boundary edges: directed edge (a,b) of a cavity triangle whose reverse is not a cavity edge
        for (int e = tid; e < nc * 3; e += nthreads) {
            const DTri& t = tris[s_cav[e / 3]];
            const int a = t.v[(e % 3 + 1) % 3], b = t.v[(e % 3 + 2) % 3];
            bool interior = false;
            for (int f = 0; f < nc * 3 && !interior; ++f) {
                const DTri& u = tris[s_cav[f / 3]];
                if (u.v[(f % 3 + 1) % 3] == b && u.v[(f % 3 + 2) % 3] == a) interior = true;
            }
            if (!interior) {
                const int k = im_atomic_add(s_edge_n, 1);
                if (k < 260) { s_edges[2 * k] = a; s_edges[2 * k + 1] = b; }
            }
        }
        IM_SYNCBLOCK_M();
        int ne = *s_edge_n;
        if (ne > 260) { ne = 260; *s_ovf = 1; }
        // kill the cavity, write (a,b,p) per boundary edge: reuse cavity slots first, then grow the pool
        for (int k = tid; k < nc; k += nthreads) tris[s_cav[k]].alive = 0;
        IM_SYNCBLOCK_M();
        for (int k = tid; k < ne; k += nthreads) {
            const int slot = (k < nc) ? s_cav[k] : (nt + (k - nc));
            if (slot < max_tris) {
                tris[slot].v[0] = (short)s_edges[2 * k];
                tris[slot].v[1] = (short)s_edges[2 * k + 1];
                tris[slot].v[2] = (short)p;
                tris[slot].alive = 1;
                if (circ && s_edges[2 * k] != IM_GHOST && s_edges[2 * k + 1] != IM_GHOST) circumcircle_f(P, s_edges[2 * k], s_edges[2 * k + 1], p, circ[slot]);
            }
        }
        if (tid == 0 && ne > nc) {
            if (nt + (ne - nc) <= max_tris) *ntri = nt + (ne - nc);
            else { *ntri = max_tris; *s_ovf = 1; }
        }
        IM_SYNCBLOCK_M();
    }
}

// smallest double c with !(acos(c) * 57.3 > 150) under glibc: a face is dropped iff cos < this (and cos >= -1)
#define IM_COS150 (-8.65928972248464878803e-01)
IM_HD bool angle_bad(double ax, double ay, double bx, double by, double cx, double cy) {  // compute_angle at apex a
    const double abx = bx - ax, aby = by - ay, acx = cx - ax, acy = cy - ay;
    const double cosv = (abx * acx + aby * acy) / (sqrt(abx * abx + aby * aby) * sqrt(acx * acx + acy * acy));
    return cosv < IM_COS150 && cosv >= -1.0;
}

// correct_triangle_index, mesh_rec_geometry.cpp:399-433 (smoothed vertex positions)
IM_HDN inline int compute_flip(const MeshDev& M, int ia, int ib, int ic, const double* cam, const double* short_axis) {
    const double* a = M.vsmooth + (size_t)ia * 3;
    const double* b = M.vsmooth + (size_t)ib * 3;
    const double* c = M.vsmooth + (size_t)ic * 3;
    const double ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]};
    const double ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
    const double tc[3] = {cam[0] - a[0], cam[1] - a[1], cam[2] - a[2]};
    double nrm[3] = {ab[1] * ac[2] - ab[2] * ac[1], ab[2] * ac[0] - ab[0] * ac[2], ab[0] * ac[1] - ab[1] * ac[0]};
    const double nn = sqrt(dot3(nrm, nrm));
    if (nn != 0) { nrm[0] = nrm[0] / nn; nrm[1] = nrm[1] / nn; nrm[2] = nrm[2] / nn; }
    else { nrm[0] = 0; nrm[1] = 0; nrm[2] = 1; }
    double sa[3] = {short_axis[0], short_axis[1], short_axis[2]};
    if (dot3(sa, tc) < 0) { sa[0] = -sa[0]; sa[1] = -sa[1]; sa[2] = -sa[2]; }
    return (dot3(sa, nrm) < 0) ? 0 : 1;
}

// ------------------------------------------------------------------ triangle store
IM_HD unsigned int tri_hash(int a, int b, int c) {
    unsigned long long k = ((unsigned long long)(unsigned int)a * 0x9E3779B97F4A7C15ull) ^ ((unsigned long long)(unsigned int)b * 0xC2B2AE3D27D4EB4Full) ^
                           ((unsigned long long)(unsigned int)c * 0x165667B19E3779F9ull);
    k ^= k >> 31; k *= 0xff51afd7ed558ccdull; k ^= k >> 33;
    return (unsigned int)k;
}
IM_HDN inline int tri_find(const MeshDev& M, int a, int b, int c) {
    unsigned int s = tri_hash(a, b, c) & M.tmask;
    for (unsigned int probe = 0; probe <= M.tmask; ++probe) {
        const int t = im_vload(&M.thash[s]);
        if (t < 0) return -1;
        const int4 r = M.tri[t];
        if (r.x == a && r.y == b && r.z == c) return t;
        s = (s + 1) & M.tmask;
    }
    return -1;
}
// insert_triangle (triangle.hpp:330-395): find-or-create, mark alive, link into the three incidence lists on creation; returns the
// triangle's index (-1 on a full pool or hash)
IM_HDN inline int tri_add(const MeshDev& M, int a, int b, int c, unsigned long long flipword) {
    unsigned int s = tri_hash(a, b, c) & M.tmask;
    int mine = -1;
    int t = -1;
    for (unsigned int probe = 0; probe <= M.tmask; ++probe) {
        int cur = im_vload(&M.thash[s]);
        if (cur < 0) {
            if (mine < 0) {
                mine = im_atomic_add(&M.cnt[IM_MC_TRIS_ALLOC], 1);
                if (mine >= M.max_t) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_TRI_POOL); return -1; }
                M.tri[mine] = make_int4(a, b, c, 0);
                M.tri_flip[mine] = 0ull;
                M.tri_next[(size_t)mine * 3 + 0] = -1; M.tri_next[(size_t)mine * 3 + 1] = -1; M.tri_next[(size_t)mine * 3 + 2] = -1;
                im_fence();
            }
            cur = im_atomic_cas32(&M.thash[s], -1, mine);
            if (cur < 0) { t = mine; break; }
        }
        const int4 r = M.tri[cur];
        if (r.x == a && r.y == b && r.z == c) { t = cur; break; }
        s = (s + 1) & M.tmask;
    }
    if (t < 0) { im_atomic_or(&M.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); return -1; }
    if (t == mine) {
        const int vs[3] = {a, b, c};
#if defined(__CUDA_ARCH__)
        // three independent list insertions.  The incidence lists are walked by other kernels only (pull, remove: before or after
        // this one in stream order), so head-before-link is never observed: one exchange per list, no fence, no retry loop.
        int prev[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) prev[k] = atomicExch(&M.v_tri_head[vs[k]], t);
#pragma unroll
        for (int k = 0; k < 3; ++k) M.tri_next[(size_t)t * 3 + k] = prev[k];
#else
        for (int k = 0; k < 3; ++k) {
            M.tri_next[(size_t)t * 3 + k] = M.v_tri_head[vs[k]];
            M.v_tri_head[vs[k]] = t;
        }
#endif
    }
    // (a record allocated by a thread that lost the publication race stays unused: a leaked slot, never linked)
    if (im_atomic_exch(&M.tri[t].w, 1) == 0) im_atomic_add(&M.cnt[IM_MC_TRIS_LIVE], 1);
    im_atomic_max64(&M.tri_flip[t], flipword);
    return t;
}
IM_HD void tri_remove(const MeshDev& M, int t) {  // erase_triangle, triangle.hpp:164-210
    if (im_atomic_exch(&M.tri[t].w, 0) == 1) im_atomic_add(&M.cnt[IM_MC_TRIS_LIVE], -1);
}

// ------------------------------------------------------------------ smoothed positions and the viewer's region sets
// RGB_pts::set_smooth_pos (pointcloud_rgbd.cpp:68-75): the smoothed position and m_smoothed.  Every writer of vsmooth except the
// append goes through here.
IM_HD void store_smooth(const MeshDev& M, int v, double x, double y, double z) {
    M.vsmooth[(size_t)v * 3 + 0] = x; M.vsmooth[(size_t)v * 3 + 1] = y; M.vsmooth[(size_t)v * 3 + 2] = z;
    if (M.vsmoothed) M.vsmoothed[v] = 1;
}
// Global_map::smooth_pts (pointcloud_rgbd.cpp:932-958) of vertex v from its k nearest vertices (ascending; the first is v itself and
// is skipped, a -1 id ends the list): those with sqrt(d2) < max_dis are averaged from their RAW positions (get_pos()), so the result
// does not depend on which vertices were smoothed before;  r = p (1 - f) + sum f / valid  (valid == 0 divides by zero like the reference)
IM_HD void smooth_vertex(const MeshDev& M, int v, int k, const int* idx, const float* d2, double sf, double max_dis, double* r) {
    const float4 p = M.vpos[v];
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, valid = 0.0;
    for (int j = 1; j < k; ++j) {
        const int id = idx[j];
        if (id < 0) break;
        if ((double)sqrtf(d2[j]) < max_dis) {
            const float4 q = M.vpos[id];
            s0 = s0 + (double)q.x; s1 = s1 + (double)q.y; s2 = s2 + (double)q.z;
            valid += 1.0;
        }
    }
    r[0] = (double)p.x * (1.0 - sf) + s0 * sf / valid;
    r[1] = (double)p.y * (1.0 - sf) + s1 * sf / valid;
    r[2] = (double)p.z * (1.0 - sf) + s2 * sf / valid;
}
// Triangle_manager::insert_triangle_to_list (triangle.cpp:35-53): region = round(centre / region_size), centre = mean of the three
// raw vertex positions (get_triangle_center)
IM_HD void tri_region_key(const MeshDev& M, const int4& r, double region_size, int* key) {
    const float4 a = M.vpos[r.x], b = M.vpos[r.y], c = M.vpos[r.z];
    key[0] = (int)round((((double)a.x + (double)b.x) + (double)c.x) / 3.0 / region_size);
    key[1] = (int)round((((double)a.y + (double)b.y) + (double)c.y) / 3.0 / region_size);
    key[2] = (int)round((((double)a.z + (double)b.z) + (double)c.z) / 3.0 / region_size);
}
// unparse_triangle_set_to_vector (mesh_rec_display.cpp:78-104): get_pos(1).cast<float>() of the three vertices, ascending ids
IM_HD void region_row(const MeshDev& M, const int4& r, float* xyz9) {
    const int v[3] = {r.x, r.y, r.z};
    for (int j = 0; j < 3; ++j)
        for (int d = 0; d < 3; ++d) xyz9[j * 3 + d] = (float)M.vsmooth[(size_t)v[j] * 3 + d];
}
// get_axis_min_max (mesh_rec_display.cpp:105-137) as an order-free reduction.  The reference walks the emitted floats in order and
// replaces the bound on a strict < / >: it ends at the FIRST occurrence of the extreme value (+0 and -0 compare equal) when that
// beats the bound, and NaN never replaces it.  So per axis the accumulator keeps (extreme value, lowest position among its equals),
// which any reduction order reproduces; axis_apply then makes the reference's single comparison against the caller's bound.
struct AxisAcc { float v[6]; int p[6]; };   // min x y z, max x y z; p = 0x7fffffff: nothing seen
IM_HD void axis_init(AxisAcc& a) {
    for (int j = 0; j < 6; ++j) { a.v[j] = 0.f; a.p[j] = 0x7fffffff; }
}
IM_HD void axis_take(AxisAcc& a, int j, float v, int p) {
    if (!(v == v) || p == 0x7fffffff) return;
    const bool lo = j < 3;
    if (a.p[j] == 0x7fffffff || (lo ? v < a.v[j] : v > a.v[j]) || (v == a.v[j] && p < a.p[j])) { a.v[j] = v; a.p[j] = p; }
}
IM_HD void axis_merge(AxisAcc& a, const AxisAcc& b) {
    for (int j = 0; j < 6; ++j) axis_take(a, j, b.v[j], b.p[j]);
}
IM_HD void axis_apply(const AxisAcc& a, float* box) {
    for (int j = 0; j < 3; ++j) {
        if (a.p[j] != 0x7fffffff && box[j] > a.v[j]) box[j] = a.v[j];
        if (a.p[j + 3] != 0x7fffffff && box[j + 3] < a.v[j + 3]) box[j + 3] = a.v[j + 3];
    }
}

}  // namespace immesh
