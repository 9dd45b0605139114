// TEST INFRASTRUCTURE (not product code): executes the __host__ __device__ bodies of the CUDA
// localization path (immesh_b200/csrc/*.cuh) on the CPU, one lane / one thread at a time, so
// that the host-side logic (state machines, pool bookkeeping, numerics contract) can be checked
// against the oracle in the CPU-only test tier.  The shipped library (libimmesh_b200.so) never
// links or calls this; it has no CPU path.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "../../immesh_b200/csrc/lio_core.cuh"

using namespace immesh;

struct immesh_lio {
    LioParams P;
    VoxelMapDev map;
    ScanBuf sb;
    LioCtrl ctrl;
    std::vector<unsigned long long> keys;
    std::vector<int> root_node, avail, pending, ints;
    std::vector<NodeRec> nodes;
    std::vector<PlaneRec> planes;
    std::vector<Chunk> chunks;
    std::vector<float> body, pw;
    std::vector<double> body_cov, p_imu, bv_imu, var, sortkey;
    std::vector<int> match_node, match_layer, slot, seg, seg2, slot_count, slot_offset, slot_cursor, touched;
    int counters[IM_LC_SIZE];
    int max_scan;
    std::vector<unsigned int> bits;   // sharded mode: [exists words | ok words]
};

static void fill_params(const immesh_lio_config* c, LioParams& P) {
    P.voxel_size = c->voxel_size;
    P.voxel_size_f = (float)c->voxel_size;
    P.voxel_size_ins = (double)P.voxel_size_f;
    P.max_layer = c->max_layer;
    for (int i = 0; i < 5; ++i) P.layer_init[i] = c->layer_init_size[i];
    P.max_points = c->max_points_size;
    P.planer_threshold = (float)c->min_eigen_value;
    P.dept_err = (float)c->dept_err;
    const float be = (float)c->beam_err;
    const double s = std::sin((double)be * 0.017453293);
    P.dir_var = s * s;
    const double sc = std::sin((double)(float)0.01 * 0.017453293);
    P.dir_var_calib = sc * sc;
    P.calib_laser = c->calib_laser;
    P.max_iter = c->max_iteration;
    for (int i = 0; i < 9; ++i) P.extR[i] = c->ext_R[i];
    for (int i = 0; i < 3; ++i) P.extT[i] = c->ext_T[i];
}

extern "C" {
int immesh_lio_create(const immesh_lio_config* cfg, immesh_lio_t** out) {
    immesh_lio* h = new immesh_lio();
    fill_params(cfg, h->P);
    const int caplog = cfg->hash_capacity_log2 ? cfg->hash_capacity_log2 : 18;
    const int max_nodes = cfg->max_nodes ? cfg->max_nodes : (1 << 18);
    const int max_chunks = cfg->max_chunks ? cfg->max_chunks : (1 << 19);
    h->max_scan = cfg->max_scan_points ? cfg->max_scan_points : (1 << 20);
    const size_t cap = (size_t)1 << caplog;
    h->keys.assign(cap, IM_EMPTY_KEY);
    h->root_node.assign(cap, -1);
    h->nodes.resize(max_nodes);
    h->planes.resize(max_nodes);
    h->chunks.resize(max_chunks);
    h->avail.assign(max_chunks, 0);
    h->pending.assign(max_chunks, 0);
    std::memset(h->counters, 0, sizeof(h->counters));
    VoxelMapDev& m = h->map;
    m.keys = h->keys.data(); m.root_node = h->root_node.data(); m.cap_mask = (unsigned)(cap - 1);
    m.nodes = h->nodes.data(); m.planes = h->planes.data(); m.node_count = &h->counters[IM_LC_NODES]; m.max_nodes = max_nodes;
    m.chunks = h->chunks.data(); m.chunk_bump = &h->counters[IM_LC_CHUNK_BUMP]; m.max_chunks = max_chunks;
    m.avail = h->avail.data(); m.avail_top = &h->counters[IM_LC_AVAIL_TOP]; m.pending = h->pending.data(); m.pending_n = &h->counters[IM_LC_PENDING];
    m.err = &h->counters[IM_LC_ERR]; m.n_roots = &h->counters[IM_LC_ROOTS]; m.stat = nullptr;
    const int ms = h->max_scan;
    h->body.resize((size_t)ms * 3); h->pw.resize((size_t)ms * 3);
    h->body_cov.resize((size_t)ms * 6); h->p_imu.resize((size_t)ms * 3); h->bv_imu.resize((size_t)ms * 6); h->var.resize((size_t)ms * 6); h->sortkey.resize(ms);
    h->match_node.assign(ms, -1); h->match_layer.assign(ms, 0); h->slot.resize(ms); h->seg.resize(ms); h->seg2.resize(ms); h->touched.resize(ms);
    h->slot_count.assign(cap, 0); h->slot_offset.assign(cap, 0); h->slot_cursor.assign(cap, 0);
    ScanBuf& sb = h->sb;
    sb.dyn = nullptr;
    sb.n = 0; sb.body = h->body.data(); sb.body_cov = h->body_cov.data(); sb.p_imu = h->p_imu.data(); sb.bv_imu = h->bv_imu.data();
    sb.match_node = h->match_node.data(); sb.match_layer = h->match_layer.data(); sb.pw = h->pw.data(); sb.var = h->var.data();
    sb.sortkey = h->sortkey.data(); sb.slot = h->slot.data(); sb.seg = h->seg.data();
    sb.slot_count = h->slot_count.data(); sb.slot_offset = h->slot_offset.data(); sb.slot_cursor = h->slot_cursor.data();
    sb.touched = h->touched.data(); sb.n_touched = &h->counters[IM_LC_TOUCHED]; sb.seg_top = &h->counters[IM_LC_SEG_TOP];
    std::memset(&h->ctrl, 0, sizeof(LioCtrl));
    double* s = h->ctrl.state;
    s[0] = s[4] = s[8] = 1.0;
    for (int i = 0; i < 18; ++i) s[24 + i * 18 + i] = 0.0000001;
    *out = h;
    return 0;
}
int immesh_lio_destroy(immesh_lio_t* h) { delete h; return 0; }
int immesh_lio_set_state(immesh_lio_t* h, const double* s) { std::memcpy(h->ctrl.state, s, 348 * 8); return 0; }
int immesh_lio_get_state(immesh_lio_t* h, double* s) { std::memcpy(s, h->ctrl.state, 348 * 8); return 0; }
int immesh_lio_predict(immesh_lio_t* h, double dt, double cg, double ca) {
    std::vector<double> T(324), Fx(324);
    predict_const_vel(h->ctrl.state, dt, cg, ca, T.data(), Fx.data(), 0, 1);
    return 0;
}
static void load_scan(immesh_lio* h, const float* body, int n) {
    std::memcpy(h->body.data(), body, (size_t)n * 12);
    h->sb.n = n;
}
static void grow(immesh_lio* h, int mode) {
    const int n = h->sb.n;
    *h->sb.n_touched = 0;
    *h->sb.seg_top = 0;
    for (int i = 0; i < n; ++i) grow_point(h->map, h->P, h->sb, h->ctrl.state, i, mode);
    const int nt = *h->sb.n_touched;
    for (int t = 0; t < nt; ++t) grow_segment(h->sb, t);
    for (int i = 0; i < n; ++i) grow_scatter(h->sb, i);
    for (int t = 0; t < nt; ++t) grow_voxel(h->map, h->P, h->sb, t, mode, 0, 1, h->seg2.data());
    recycle_chunks(h->map, 0, 1);
}
int immesh_voxelmap_build(immesh_lio_t* h, const float* body, int n) {
    load_scan(h, body, n);
    grow(h, 1);
    return (*h->map.err) ? IMMESH_E_CAPACITY : 0;
}
}  // extern "C"

// ---- host emulation of the 8-lanes-per-point match (k_match).  The lanes of a point meet at `combine`; the emulation replays the
// lane function: every pass runs the 8 lanes up to the first merge point that is not known yet (their results are recorded and the
// lane is told `ok` so that it stops), merges the records in lane order with the strict '>' -- the rule the device's shuffle
// butterfly implements (MatchCombine8, lio_capi.cu) -- and hands the merged pairs to the next pass.
namespace {
struct LaneReplay {
    int n_known = 0;
    bool known_ok[2] = {false, false};
    MatchResult known_best[2];
    int call = 0;
    bool recorded = false;
    bool rec_ok = false;
    MatchResult rec_best;
};
struct LaneCombine {
    LaneReplay* r;
    void operator()(bool* ok, MatchResult* best) const {
        const int c = r->call++;
        if (c < r->n_known) { *ok = r->known_ok[c]; *best = r->known_best[c]; return; }
        if (c == r->n_known) { r->recorded = true; r->rec_ok = *ok; r->rec_best = *best; }
        *ok = true;   // nothing after this merge point is evaluated in this pass
    }
};
void match_lanes_point(immesh_lio* h, const double* state, int i) {
    LaneReplay known;
    for (int pass = 0; pass < 3; ++pass) {
        bool any_rec = false, m_ok = false;
        MatchResult m_best;
        m_best.node = -1; m_best.layer = 0; m_best.prob = 0.0;
        for (int lane = 0; lane < 8; ++lane) {   // lane 0 stores the match of the point; the store of the last pass is the final one
            LaneReplay r = known;
            r.call = 0; r.recorded = false;
            residual_match_lanes(h->map, h->P, h->sb, state, i, lane, 8, LaneCombine{&r});
            if (!r.recorded) continue;
            any_rec = true;
            if (r.rec_ok) m_ok = true;
            if (r.rec_best.prob > m_best.prob) m_best = r.rec_best;
        }
        if (!any_rec) return;   // every merge point was known already
        known.known_ok[known.n_known] = m_ok;
        known.known_best[known.n_known] = m_best;
        known.n_known++;
    }
}
int g_split = 1;
}  // namespace

extern "C" {
// small numerical bodies of the kernels, exposed one by one for tests/test_kernel_math_emu.py
void emu_jacobi3(const double* a6, double* d, double* V) { jacobi3(a6, d, V); }
void emu_lu_inverse6(const double* A, double* Ainv) {
    double a[36];
    int piv[6];
    for (int i = 0; i < 36; ++i) a[i] = A[i];
    lu_factor6(a, piv);
    for (int c = 0; c < 6; ++c) lu_solve_col6(a, piv, c, Ainv);
}
void emu_order3(const double* ev, int* o) { order3(ev, o); }
int emu_lio_set_split(int mode) { g_split = mode; return 0; }   // 0: k_residual body, 1: k_match with 8 lanes + k_terms, 2: k_match with 1 lane + k_terms
// The same per first-level child (the 8-lane split of k_match): out[i*24 + j*3 + {0,1,2}] = nodes visited, planes evaluated, planes
// past the range gate in the subtree below child j of the point's root voxel (zeros for plane roots: lane 0 evaluates the root).
int emu_match_lane_stats(immesh_lio_t* h, int* out, int n) {
    const VoxelMapDev& m = h->map;
    for (int i = 0; i < n && i < h->sb.n; ++i) {
        int* o = out + (size_t)i * 24;
        for (int q = 0; q < 24; ++q) o[q] = 0;
        double pwd[3], pw[3], var6[6];
        residual_world(h->P, h->sb, h->ctrl.state, i, pwd, pw, var6);
        long long k[3];
        float loc[3];
        if (!voxel_key3_loc(pw, h->P.voxel_size, k, loc)) continue;
        const int slot = hash_find(m, pack_key(k[0], k[1], k[2]));
        if (slot < 0 || m.root_node[slot] < 0) continue;
        const int root = m.root_node[slot];
        if (m.planes[root].is_plane) { o[0] = 1; o[1] = 1; o[2] = 1; continue; }
        if (h->P.max_layer < 1) continue;
        for (int j = 0; j < 8; ++j) {
            if (m.nodes[root].children[j] < 0) continue;
            std::vector<std::pair<int, int>> st{{m.nodes[root].children[j], 1}};
            while (!st.empty()) {
                const auto [nd, layer] = st.back();
                st.pop_back();
                ++o[j * 3];
                const PlaneRec& pl = m.planes[nd];
                if (pl.is_plane) {
                    ++o[j * 3 + 1];
                    const float dp = (float)fabs(((pl.normal[0] * pw[0] + pl.normal[1] * pw[1]) + pl.normal[2] * pw[2]) + (double)pl.d);
                    const float dc = (float)(((pl.center[0] - pw[0]) * (pl.center[0] - pw[0]) + (pl.center[1] - pw[1]) * (pl.center[1] - pw[1])) + (pl.center[2] - pw[2]) * (pl.center[2] - pw[2]));
                    if ((double)sqrtf(dc - dp * dp) <= 3.0 * (double)pl.radius) ++o[j * 3 + 2];
                    continue;
                }
                if (layer >= h->P.max_layer) continue;
                for (int c = 0; c < 8; ++c)
                    if (m.nodes[nd].children[c] >= 0) st.push_back({m.nodes[nd].children[c], layer + 1});
            }
        }
    }
    return 0;
}
// Work statistics of the match walk of the loaded scan at the current state (kernel design aid, tools/debug/match_stats.py):
// per point out[i*4 + {0,1,2,3}] = root kind (0 no voxel, 1 plane root, 2 split root), nodes visited, planes evaluated, planes that
// pass the range gate (and so run the 6x6 sigma + exp chain); root voxel only (no neighbour retry).
int emu_match_walk_stats(immesh_lio_t* h, int* out, int n) {
    const VoxelMapDev& m = h->map;
    for (int i = 0; i < n && i < h->sb.n; ++i) {
        int* o = out + (size_t)i * 4;
        o[0] = o[1] = o[2] = o[3] = 0;
        double pwd[3], pw[3], var6[6];
        residual_world(h->P, h->sb, h->ctrl.state, i, pwd, pw, var6);
        long long k[3];
        float loc[3];
        if (!voxel_key3_loc(pw, h->P.voxel_size, k, loc)) continue;
        const int slot = hash_find(m, pack_key(k[0], k[1], k[2]));
        if (slot < 0 || m.root_node[slot] < 0) continue;
        const int root = m.root_node[slot];
        o[0] = m.planes[root].is_plane ? 1 : 2;
        std::vector<std::pair<int, int>> st{{root, 0}};
        while (!st.empty()) {
            const auto [nd, layer] = st.back();
            st.pop_back();
            ++o[1];
            const PlaneRec& pl = m.planes[nd];
            if (pl.is_plane) {
                ++o[2];
                const float dp = (float)fabs(((pl.normal[0] * pw[0] + pl.normal[1] * pw[1]) + pl.normal[2] * pw[2]) + (double)pl.d);
                const float dc = (float)(((pl.center[0] - pw[0]) * (pl.center[0] - pw[0]) + (pl.center[1] - pw[1]) * (pl.center[1] - pw[1])) + (pl.center[2] - pw[2]) * (pl.center[2] - pw[2]));
                if ((double)sqrtf(dc - dp * dp) <= 3.0 * (double)pl.radius) ++o[3];
                continue;
            }
            if (layer >= h->P.max_layer) continue;
            for (int c = 0; c < 8; ++c)
                if (m.nodes[nd].children[c] >= 0) st.push_back({m.nodes[nd].children[c], layer + 1});
        }
    }
    return 0;
}
int immesh_lio_estimate(immesh_lio_t* h, const float* body, int n, int* iters_run) {
    load_scan(h, body, n);
    LioCtrl& c = h->ctrl;
    std::memcpy(c.state_prop, c.state, 348 * 8);
    std::memset(c.acc, 0, sizeof(c.acc));
    c.stop = 0; c.iters_run = 0; c.rematch_num = 0;
    for (int i = 0; i < n; ++i) prepare_point(h->P, h->sb, i);
    SolveScratch S;
    for (int it = 0; it < h->P.max_iter && !c.stop; ++it) {
        long long hi[IM_NTERMS], lo[IM_NTERMS];   // each term split into its 32-bit halves as it is added: no partial sum can wrap
        for (int k = 0; k < IM_NTERMS; ++k) hi[k] = lo[k] = 0;
        if (g_split == 1)
            for (int i = 0; i < n; ++i) match_lanes_point(h, c.state, i);   // k_match, 8 lanes per point
        else if (g_split == 2)
            for (int i = 0; i < n; ++i) residual_match_lanes(h->map, h->P, h->sb, c.state, i, 0, 1, [](bool*, MatchResult*) {});   // k_match, large scans: 1 lane
        for (int i = 0; i < n; ++i) {
            long long t[IM_NTERMS];
            const bool hit = g_split ? residual_point_matched(h->map, h->P, h->sb, c.state, i, t, h->map.err)   // k_terms
                                     : residual_point(h->map, h->P, h->sb, c.state, i, t, h->map.err);            // k_residual
            if (hit)
                for (int k = 0; k < IM_NTERMS; ++k) { hi[k] += t[k] >> 32; lo[k] += t[k] & 0xffffffffLL; }
        }
        for (int k = 0; k < IM_NTERMS; ++k) {
            c.acc[it][2 * k] += (unsigned long long)hi[k];
            c.acc[it][2 * k + 1] += (unsigned long long)lo[k];
        }
        ieskf_solve(h->P, &c, it, &S, 0, 1);
    }
    if (iters_run) *iters_run = c.iters_run;
    return 0;
}
int immesh_voxelmap_update(immesh_lio_t* h) {
    grow(h, 0);
    return (*h->map.err) ? IMMESH_E_CAPACITY : 0;
}
int immesh_lio_iter_stats(immesh_lio_t* h, int it, double* out) {
    const IterStats& s = h->ctrl.stats[it];
    std::memcpy(out, s.HTH, 36 * 8);
    std::memcpy(out + 36, s.HTz, 6 * 8);
    out[42] = s.n_match; out[43] = s.total_residual;
    std::memcpy(out + 44, s.solution, 18 * 8);
    out[62] = s.converged;
    return 0;
}
int immesh_lio_matches(immesh_lio_t* h, int* plane_layer, int n) {
    for (int i = 0; i < n; ++i) plane_layer[i] = h->match_node[i] >= 0 ? h->match_layer[i] : -1;
    return 0;
}
}  // extern "C"

// canonical dump shared with the CUDA library's host-side dump (same traversal on host copies of the pools)
#include "../../immesh_b200/csrc/map_dump.hpp"
extern "C" {
int64_t immesh_voxelmap_dump(immesh_lio_t* h, double* rows, int64_t cap_rows) {
    return dump_voxelmap(h->keys.data(), h->root_node.data(), h->keys.size(), h->nodes.data(), h->planes.data(), rows, cap_rows);
}
int immesh_voxelmap_counts(immesh_lio_t* h, int64_t* out) {
    out[0] = h->counters[IM_LC_ROOTS]; out[1] = h->counters[IM_LC_NODES]; out[2] = h->counters[IM_LC_CHUNK_BUMP]; out[3] = h->counters[IM_LC_ERR];
    return 0;
}
}

// ------------------------------------------------------------------ sharded VoxelMap, split-phase (test-only entry points)
// The CUDA library runs these phases back to back on one stream with ncclAllReduce in between; here the test does the two
// all-reduces with torch.distributed (gloo) on the exposed host buffers.
extern "C" {
int emu_lio_set_shard(immesh_lio_t* h, int rank, int n) { h->P.shard_rank = rank; h->P.shard_n = n; return 0; }
int emu_shard_begin(immesh_lio_t* h, const float* body, int n) {
    load_scan(h, body, n);
    LioCtrl& c = h->ctrl;
    std::memcpy(c.state_prop, c.state, 348 * 8);
    std::memset(c.acc, 0, sizeof(c.acc));
    c.stop = 0; c.iters_run = 0; c.rematch_num = 0;
    for (int i = 0; i < n; ++i) prepare_point(h->P, h->sb, i);
    h->bits.assign(2 * ((size_t)(n + 31) / 32) + 2, 0u);
    return 0;
}
unsigned int* emu_shard_bits(immesh_lio_t* h, int* nwords) { *nwords = (int)h->bits.size(); return h->bits.data(); }
int emu_shard_pass1(immesh_lio_t* h) {
    const int n = h->sb.n;
    const size_t w = (size_t)(n + 31) / 32 + 1;
    std::fill(h->bits.begin(), h->bits.end(), 0u);
    for (int i = 0; i < n; ++i) shard_pass1_point(h->map, h->P, h->sb, h->ctrl.state, i, h->bits.data(), h->bits.data() + w);
    return 0;
}
int emu_shard_pass2(immesh_lio_t* h, int it) {
    const int n = h->sb.n;
    const size_t w = (size_t)(n + 31) / 32 + 1;
    long long hi[IM_NTERMS], lo[IM_NTERMS];
    for (int k = 0; k < IM_NTERMS; ++k) hi[k] = lo[k] = 0;
    for (int i = 0; i < n; ++i) {
        long long t[IM_NTERMS];
        if (shard_pass2_point(h->map, h->P, h->sb, h->ctrl.state, i, h->bits.data(), h->bits.data() + w, t, h->map.err))
            for (int k = 0; k < IM_NTERMS; ++k) { hi[k] += t[k] >> 32; lo[k] += t[k] & 0xffffffffLL; }
    }
    for (int k = 0; k < IM_NTERMS; ++k) {
        h->ctrl.acc[it][2 * k] = (unsigned long long)hi[k];
        h->ctrl.acc[it][2 * k + 1] = (unsigned long long)lo[k];
    }
    return 0;
}
unsigned long long* emu_shard_acc(immesh_lio_t* h, int it) { return h->ctrl.acc[it]; }
int emu_shard_solve(immesh_lio_t* h, int it) {
    SolveScratch S;
    ieskf_solve(h->P, &h->ctrl, it, &S, 0, 1);
    return h->ctrl.stop;
}
}

// ---- IMU front-end (imu_core.cuh bodies, one thread): same entry points as immesh_b200/csrc/imu_capi.cu
#include "../../immesh_b200/csrc/imu_core.cuh"
struct immesh_imu {
    ImuParams P;
    double last_imu[7] = {0, 0, 0, 0, 0, 0, 0};
    double last_lidar_end_time = -1.0, last_update_time = 0.0;
    double run[IM_IMU_RUN];
    std::vector<double> poses;
    std::vector<float> out;
    int last_poses = 0;
};
extern "C" {
int immesh_imu_create(const immesh_imu_config* c, immesh_imu_t** out) {
    immesh_imu* h = new immesh_imu();
    for (int i = 0; i < 3; ++i) { h->P.cov_gyr[i] = c->cov_gyr[i]; h->P.cov_acc[i] = c->cov_acc[i]; h->P.cov_bias_gyr[i] = c->cov_bias_gyr[i]; h->P.cov_bias_acc[i] = c->cov_bias_acc[i]; h->P.lid_T[i] = c->lid_T[i]; }
    for (int i = 0; i < 9; ++i) h->P.lid_R[i] = c->lid_R[i];
    h->P.mean_acc_norm = c->mean_acc_norm;
    for (int i = 0; i < IM_IMU_RUN; ++i) h->run[i] = 0.0;
    *out = h;
    return 0;
}
int immesh_imu_destroy(immesh_imu_t* h) { delete h; return 0; }
int immesh_imu_reset(immesh_imu_t* h, const double* last_imu7, double last_lidar_end_time, double last_update_time, const double* acc_s_last, const double* angvel_last) {
    std::memcpy(h->last_imu, last_imu7, 56);
    h->last_lidar_end_time = last_lidar_end_time; h->last_update_time = last_update_time;
    for (int i = 0; i < 3; ++i) { h->run[i] = acc_s_last ? acc_s_last[i] : 0.0; h->run[3 + i] = angvel_last ? angvel_last[i] : 0.0; }
    return 0;
}
int immesh_imu_undistort(immesh_imu_t* h, immesh_lio_t* lio, const double* imu, int n_imu, const float* pts, int n, int, double lidar_beg_time, float* out_xyzt) {
    std::vector<const double*> v;
    v.push_back(h->last_imu);
    for (int i = 0; i < n_imu; ++i) v.push_back(imu + 7 * (size_t)i);
    const double imu_end_time = v.back()[0];
    const double pcl_beg_time = std::max(lidar_beg_time, h->last_update_time);
    const double pcl_end_time = lidar_beg_time + (double)pts[4 * (size_t)(n - 1) + 3] / double(1000);
    h->last_update_time = pcl_end_time;
    std::vector<ImuStep> steps;
    for (size_t k = 0; k + 1 < v.size(); ++k) {
        const double *head = v[k], *tail = v[k + 1];
        if (tail[0] < h->last_lidar_end_time) continue;
        ImuStep s;
        for (int i = 0; i < 3; ++i) { s.gyr_avg[i] = 0.5 * (head[1 + i] + tail[1 + i]); s.acc_avg[i] = 0.5 * (head[4 + i] + tail[4 + i]); }
        s.dt = (head[0] < h->last_lidar_end_time) ? tail[0] - h->last_lidar_end_time : tail[0] - head[0];
        s.offs_t = tail[0] - pcl_beg_time;
        steps.push_back(s);
    }
    double note, dt_end;
    if (imu_end_time > pcl_beg_time) { note = pcl_end_time > imu_end_time ? 1.0 : -1.0; dt_end = note * (pcl_end_time - imu_end_time); }
    else { note = pcl_end_time > pcl_beg_time ? 1.0 : -1.0; dt_end = note * (pcl_end_time - pcl_beg_time); }
    double last[7];
    std::memcpy(last, v.back(), 56);
    std::memcpy(h->last_imu, last, 56);
    h->last_lidar_end_time = pcl_end_time;
    double* st = lio->ctrl.state;
    for (int i = 0; i < 3; ++i) { h->run[6 + i] = st[12 + i]; h->run[9 + i] = st[9 + i]; }
    for (int i = 0; i < 9; ++i) h->run[12 + i] = st[i];
    h->poses.assign((steps.size() + 1) * IM_POSE_DOUBLES, 0.0);
    imu_write_pose(h->poses.data(), 0.0, h->run);
    std::vector<double> Fx(324), T(324);
    for (size_t k = 0; k < steps.size(); ++k) imu_forward_step(h->P, st, h->run, steps[k], h->poses.data() + (k + 1) * IM_POSE_DOUBLES, Fx.data(), T.data(), 0, 1);
    imu_predict_end(st, h->run, note, dt_end);
    std::vector<int> order(n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return pts[4 * (size_t)a + 3] < pts[4 * (size_t)b + 3]; });
    h->out.resize(4 * (size_t)n);
    for (int i = 0; i < n; ++i)
        for (int c = 0; c < 4; ++c) h->out[4 * (size_t)i + c] = pts[4 * (size_t)order[i] + c];
    const int n_pose = (int)steps.size() + 1;
    for (int s = 0; s < n; ++s) imu_undistort_point(h->P, st, h->poses.data(), n_pose, h->out.data(), s);
    h->last_poses = n_pose;
    if (out_xyzt) std::memcpy(out_xyzt, h->out.data(), 4 * (size_t)n * sizeof(float));
    return 0;
}
const float* immesh_imu_device_points(immesh_imu_t* h) { return h->out.data(); }
int immesh_imu_get_poses(immesh_imu_t* h, double* out, int cap) {
    const int m = std::min(cap, h->last_poses);
    std::memcpy(out, h->poses.data(), (size_t)m * IM_POSE_DOUBLES * sizeof(double));
    return h->last_poses;
}
}  // extern "C"
