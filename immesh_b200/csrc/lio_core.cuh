// immesh_b200 -- per-scan localization path on the device-resident VoxelMap:
//   K1 scan preparation        (m_body_cov_list / m_cross_mat_list, voxel_mapping.cpp:1302-1316)
//   K2+K3 residual + Jacobian row + normal-equation terms, one thread per scan point
//                              (voxel_mapping.cpp:1344-1392, :1487-1586)
//   K4 IESKF solve             (voxel_mapping.cpp:1586-1650), one thread block
//   K5 map growth              (ImMesh_mesh_reconstruction.cpp:387-408 + updateVoxelMap)
// The bodies are __host__ __device__ so that tests/emu can execute the very same source on the
// CPU (single lane / single thread) for logic tests; the product only ever runs them on the GPU.
#pragma once
#include "voxelmap.cuh"

#if defined(__CUDA_ARCH__)
#define IM_SYNCBLOCK() __syncthreads()
#else
#define IM_SYNCBLOCK()
#endif

namespace immesh {

#define IM_MAX_ITER 8
#define IM_STATE_DOUBLES 348  // rot 9, pos 3, vel 3, bg 3, ba 3, grav 3, cov 324
#define IM_NTERMS 30          // 21 HTH + 6 HTz + sum|r| + match count + spare

struct IterStats {
    double HTH[36];
    double HTz[6];
    double n_match;
    double total_residual;
    double solution[18];
    double converged;
};

// Per-scan inputs of the launch sequence.  They live in device memory (one small H2D per scan) instead of kernel arguments so
// that the captured CUDA graph of a scan is replayed WITHOUT touching any of its nodes: kernel arguments, grids and
// dependencies are constant from scan to scan.
struct ScanDyn {
    const float* body;        // [n][3] body-frame scan (device pointer)
    int n;
    int scan_idx;             // running scan counter; the converged pose goes to LioCtrl::pose_ring[scan_idx & 7]
    double dt, cov_gyr, cov_acc;   // Forward_without_imu inputs; dt <= 0: no prediction
    unsigned long long epoch; // peer-window epoch base of this scan (sharded mode)
    int mode, pad_;
    const int* n_dev;         // when not null: the number of points is read from here at execution time (a device-resident
                              // front-end produced the scan: no host round trip of the count)
};
// Slots of the localization's counter block (immesh_lio::d_counters), wired into VoxelMapDev and ScanBuf at create: name, writer, reset
enum : int {
    IM_LC_NODES = 0,         // VoxelMapDev::node_count: node records allocated (alloc_node); never reset
    IM_LC_CHUNK_BUMP = 1,    // VoxelMapDev::chunk_bump: chunks ever taken from the pool (alloc_chunk); never reset
    IM_LC_AVAIL_TOP = 2,     // VoxelMapDev::avail_top: recycled chunks on the free stack (alloc_chunk, recycle_chunks)
    IM_LC_PENDING = 3,       // VoxelMapDev::pending_n: chunks freed this scan (node_free_points); recycle_chunks
    IM_LC_ERR = 4,           // VoxelMapDev::err: IM_ERR_* flags; never reset
    IM_LC_ROOTS = 5,         // VoxelMapDev::n_roots: root voxels; never reset
    IM_LC_TOUCHED = 6,       // ScanBuf::n_touched: root voxels the scan touched (grow_point); k_grow_finish
    IM_LC_SEG_TOP = 7,       // ScanBuf::seg_top: points placed into the touched voxels' segments; k_grow_finish
    IM_LC_WORK = 8,          // voxel ticket of k_grow_voxel; k_grow_finish
    IM_LC_REFITS = 9,        // VoxelMapDev::stat[0]: plane refits of the scan; k_grow_finish
    IM_LC_REFIT_POINTS = 10, // VoxelMapDev::stat[1]: points read by the refits; k_grow_finish
    IM_LC_COMPLEX = 11,      // touched root voxels left to k_grow_voxel (k_grow_simple); k_grow_finish
    IM_LC_PUB_N = 12,        // VoxelMapDev::pub_n: entries of the plane-map publisher's pending list; immesh_voxelmap_plane_markers
    IM_LC_SIZE = 16,         // ints allocated, read back and copied into LioOut::counters
};

// what the host reads back after a scan, one D2H copy
struct LioOut {
    double state[IM_STATE_DOUBLES];
    int iters_run;
    int scan_idx;
    int counters[IM_LC_SIZE];
    int pad_[2];
};
#define IM_POSE_RING 8

struct LioCtrl {
    double state[IM_STATE_DOUBLES];
    double state_prop[IM_STATE_DOUBLES];
    double pose_ring[IM_POSE_RING][12];   // rot_end, pos_end each scan converged to (read by the mesher's frame, which runs behind)
    LioOut out;
    ScanDyn dyn;
    unsigned long long acc[IM_MAX_ITER][IM_NTERMS * 2];  // (hi, lo) pairs, two's complement sums
    IterStats stats[IM_MAX_ITER];
    int stop;
    int iters_run;
    int rematch_num;
    int pad_;
    int blocks_done[IM_MAX_ITER];  // residual blocks that have published their sums (the last one runs the solve)
    int shard_cnt[2];              // peer-window exchange: blocks of pass 1 / pass 2 that have finished (reset by the last one)
    int pad2_[2];
};

struct ScanBuf {
    int n;
    const float* body;   // [n][3] body-frame (LiDAR) points, float like pcl::PointXYZI
    const ScanDyn* dyn;  // device: n / body of the current scan are taken from here (scan_load_dyn), see ScanDyn
    double* body_cov;    // [n][6]
    double* p_imu;       // [n][3]  R_ext p + t_ext (z==0 -> 0.001 rule applied first, :1305-1312)
    double* bv_imu;      // [n][6]  calcBodyVar at the IMU-frame point of the raw scan point (weights, :1498-1521); state independent
    int* match_node;     // [n] plane node of the accepted match, -1 otherwise (last residual pass)
    int* match_layer;    // [n]
    float* wsqrt;        // [n] (float)sqrt(R_inv) of the matched points of the last residual pass: the IESKF weight the reference writes
                         // into m_laserCloudOri's intensity (:1527), kept for immesh_lio_effect_cloud; null: not kept
    float* pw;           // [n][3] world points of the growth pass
    double* var;         // [n][6]
    double* sortkey;     // [n]
    int* slot;           // [n]
    int* seg;            // [n] point indices grouped by root voxel
    // per-slot scratch (size = hash capacity)
    int* slot_count;
    int* slot_offset;
    int* slot_cursor;
    // touched root voxels of this scan
    int* touched;
    int* n_touched;
    int* seg_top;
};

// kernels work on a copy of their ScanBuf argument whose per-scan fields come from the device-resident block
IM_HD ScanBuf scan_load_dyn(const ScanBuf& sb) {
    ScanBuf o = sb;
    if (sb.dyn) { o.n = sb.dyn->n_dev ? *sb.dyn->n_dev : sb.dyn->n; o.body = sb.dyn->body; }
    return o;
}

// ------------------------------------------------------------------ K1
IM_HDN inline void prepare_point(const LioParams& P, const ScanBuf& sb, int i) {
    double p[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    if (p[2] == 0) p[2] = 0.001;
    calc_body_var(p, P.dept_err, P.dir_var, sb.body_cov + (size_t)i * 6);
    double q[3];
    m3_vec(P.extR, p, q);
    sb.p_imu[(size_t)i * 3 + 0] = q[0] + P.extT[0];
    sb.p_imu[(size_t)i * 3 + 1] = q[1] + P.extT[1];
    sb.p_imu[(size_t)i * 3 + 2] = q[2] + P.extT[2];
    // measurement covariance used by the IESKF weights: evaluated at R_ext p + t_ext of the RAW point (:1496-1521)
    const double pr[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    double qi[3];
    m3_vec(P.extR, pr, qi);
    qi[0] = qi[0] + P.extT[0]; qi[1] = qi[1] + P.extT[1]; qi[2] = qi[2] + P.extT[2];
    calc_body_var(qi, P.dept_err, P.calib_laser ? P.dir_var_calib : P.dir_var, sb.bv_imu + (size_t)i * 6);
}

// world covariance for matching: R S_b R^T + (-[p]x) S_R (-[p]x)^T + S_t   (voxel_mapping.cpp:1356)
IM_HDN inline void world_cov(const double* A, const double* body_cov6, const double* p_imu, const double* cov18, double* out6) {
    double Sb[9], C[9], nC[9], rot_var[9], T1[6], T2[6];
    s6_full(body_cov6, Sb);
    congr6(A, Sb, T1);
    skew3(p_imu, C);
    for (int k = 0; k < 9; ++k) nC[k] = -C[k];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) rot_var[a * 3 + b] = cov18[a * 18 + b];
    congr6(nC, rot_var, T2);
    for (int a = 0; a < 3; ++a)
        for (int b = a; b < 3; ++b) out6[s6(a, b)] = (T1[s6(a, b)] + T2[s6(a, b)]) + cov18[(3 + a) * 18 + (3 + b)];
}

// ------------------------------------------------------------------ K2 + K3 (one scan point)
// terms[0..20] = upper triangle of w h h^T, [21..26] = w h z, [27] = |r|, [28] = 1 (match count); as 2^-20 fixed point.
// returns true when the point is matched.
// world point (float-rounded, as transformLidar stores it) + its covariance for the matching step (:1344-1359)
IM_HDN inline void residual_world(const LioParams& P, const ScanBuf& sb, const double* state, int i, double* pwd, double* pw, double* var6) {
    const double* R = state;
    const double* t = state + 9;
    const double* cov = state + 24;
    const double pb[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    body_to_world(P, R, t, pb, pwd);
    pw[0] = (double)(float)pwd[0]; pw[1] = (double)(float)pwd[1]; pw[2] = (double)(float)pwd[2];
    world_cov(R, sb.body_cov + (size_t)i * 6, sb.p_imu + (size_t)i * 3, cov, var6);
}
// residual, Jacobian row, weight and the 29 fixed-point normal-equation terms of point i matched to plane `node`
// (voxel_mapping.cpp:1372-1392, :1487-1586)
IM_HDN inline bool residual_terms(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, int node, const double* pwd, long long* terms, int* err) {
    const double* R = state;
    const double* t = state + 9;
    const double pb[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    const PlaneRec& pl = map.planes[node];
    // float-rounded normal / residual through the PCL point structs (voxel_mapping.cpp:1377-1389)
    const float nf[3] = {(float)pl.normal[0], (float)pl.normal[1], (float)pl.normal[2]};
    const float dis = (float)(((pwd[0] * (double)nf[0] + pwd[1] * (double)nf[1]) + pwd[2] * (double)nf[2]) + (double)pl.d);
    // Jacobian row and weight (voxel_mapping.cpp:1496-1569)
    double p_imu[3];
    m3_vec(P.extR, pb, p_imu);
    p_imu[0] = p_imu[0] + P.extT[0]; p_imu[1] = p_imu[1] + P.extT[1]; p_imu[2] = p_imu[2] + P.extT[2];
    double C[9];
    skew3(p_imu, C);
    const double nv[3] = {(double)nf[0], (double)nf[1], (double)nf[2]};
    double pw2[3];
    m3_vec(R, p_imu, pw2);
    pw2[0] = pw2[0] + t[0]; pw2[1] = pw2[1] + t[1]; pw2[2] = pw2[2] + t[2];
    double Sb[9], RRe[9], wv[6];
    s6_full(sb.bv_imu + (size_t)i * 6, Sb);  // calcBodyVar at the IMU-frame point (:1498-1521), precomputed in prepare_point
    m3_mul(R, P.extR, RRe);
    congr6(RRe, Sb, wv);
    const double sigma_l = plane_sigma(pw2, pl.center, pl.normal, pl.pv);
    const double R_inv = 1.0 / (sigma_l + quad6(nv, wv));
    // stored here, not recomputed at publish time: the weight depends on this iteration's pose and on the planes before the map update
    if (sb.wsqrt) sb.wsqrt[i] = (float)sqrt(R_inv);
    double CRt[9], A[3];
    m3_mul_bt(C, R, CRt);
    m3_vec(CRt, nv, A);
    const double h[6] = {A[0], A[1], A[2], nv[0], nv[1], nv[2]};
    const double z = -(double)dis;
    double hw[6];
    for (int a = 0; a < 6; ++a) hw[a] = h[a] * R_inv;
    int e = 0;
    bool range_ok = true;
    for (int a = 0; a < 6; ++a)
        for (int b = a; b < 6; ++b, ++e) {
            const double term = hw[a] * h[b];
            if (!(fabs(term) < 1.0e10)) range_ok = false;
            terms[e] = im_llrint(term * IM_FX_SCALE);
        }
    for (int a = 0; a < 6; ++a) {
        const double term = hw[a] * z;
        if (!(fabs(term) < 1.0e10)) range_ok = false;
        terms[21 + a] = im_llrint(term * IM_FX_SCALE);
    }
    terms[27] = im_llrint(fabs((double)dis) * IM_FX_SCALE);
    terms[28] = 1;
    terms[29] = 0;
    if (!range_ok) {
        im_atomic_or(err, IM_ERR_FX_RANGE);
        for (int k = 0; k < IM_NTERMS; ++k) terms[k] = 0;
        return false;
    }
    return true;
}
IM_HDN inline bool residual_point(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, long long* terms, int* err) {
    double pwd[3], pw[3], var6[6];
    residual_world(P, sb, state, i, pwd, pw, var6);
    const MatchResult mr = match_point(map, P, pw, var6);
    sb.match_node[i] = mr.node;
    sb.match_layer[i] = mr.layer;
    if (mr.node < 0) return false;
    return residual_terms(map, P, sb, state, i, mr.node, pwd, terms, err);
}

// The same in two steps (one GPU, k_match + k_terms): the match with each root voxel's walk split over nl lanes (8 or 1), then the terms of
// the matched points.  match_point_lanes returns what match_point returns (voxelmap.cuh), the second step repeats residual_point's tail.
template <class Combine>
IM_HDN inline void residual_match_lanes(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, int lane, int nl, Combine combine) {
    double pwd[3], pw[3], var6[6];
    residual_world(P, sb, state, i, pwd, pw, var6);
    IM_STAMP(3, __double_as_longlong(var6[5] + pw[2]));
    const MatchResult mr = match_point_lanes(map, P, pw, var6, lane, nl, combine);
    if (lane == 0) {
        sb.match_node[i] = mr.node;
        sb.match_layer[i] = mr.layer;
    }
}
IM_HDN inline bool residual_point_matched(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, long long* terms, int* err) {
    const int node = sb.match_node[i];
    if (node < 0) return false;
    const double pb[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    double pwd[3];
    body_to_world(P, state, state + 9, pb, pwd);
    return residual_terms(map, P, sb, state, i, node, pwd, terms, err);
}

// ------------------------------------------------------------------ sharded VoxelMap (multi-GPU): split residual pass
// The scan is replicated, root voxels are owned by voxel_owner(key).  Pass 1: the owner of a point's root voxel matches it
// there and publishes two bits (root voxel exists / matched there); the owner of the point's retry neighbour voxel
// evaluates that match speculatively.  The bit words of all ranks are summed (bits are disjoint: one owner per point), then
// pass 2 lets exactly one rank contribute the point's normal-equation terms.  Integer sums => the all-reduced
// accumulators, hence the state, are bit-identical to the single-GPU run for any number of ranks.
//   sb.slot[i] : speculative neighbour match node (-1 none)      sb.seg[i] : its layer
// core of pass 1: returns the two bits of point i through *exists / *ok1 (false unless this rank owns the point's root voxel)
IM_HDN inline void shard_pass1_flags(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, bool* exists, bool* ok1) {
    double pwd[3], pw[3], var6[6];
    *exists = false;
    *ok1 = false;
    sb.match_node[i] = -1;
    sb.match_layer[i] = 0;
    sb.slot[i] = -1;
    sb.seg[i] = 0;
    // owner-computes: the world point alone decides which ranks need this point (its root voxel's owner and the owner of the
    // one retry neighbour); everybody else is done after ~40 flops, without the covariance propagation and without a probe
    {
        const double pb[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
        body_to_world(P, state, state + 9, pb, pwd);
        pw[0] = (double)(float)pwd[0]; pw[1] = (double)(float)pwd[1]; pw[2] = (double)(float)pwd[2];
    }
    long long k[3];
    float loc[3];
    if (!voxel_key3_loc(pw, P.voxel_size, k, loc)) return;
    const unsigned long long key = pack_key(k[0], k[1], k[2]);
    long long nk[3];
    neighbour_key(P, k, loc, nk);
    const bool nk_ok = nk[0] > -1048000 && nk[0] < 1048000 && nk[1] > -1048000 && nk[1] < 1048000 && nk[2] > -1048000 && nk[2] < 1048000;
    const unsigned long long nkey = nk_ok ? pack_key(nk[0], nk[1], nk[2]) : 0ull;
    const int o1 = voxel_owner(key, P.shard_n);
    const int o2 = nk_ok ? voxel_owner(nkey, P.shard_n) : -1;
    if (o1 != P.shard_rank && o2 != P.shard_rank) return;
    world_cov(state, sb.body_cov + (size_t)i * 6, sb.p_imu + (size_t)i * 3, state + 24, var6);
    if (o1 == P.shard_rank) {
        const int slot = hash_find(map, key);
        const int root = slot >= 0 ? map.root_node[slot] : -1;
        if (root >= 0) {
            *exists = true;
            MatchResult best; best.node = -1; best.layer = 0; best.prob = 0.0;
            bool ok = false;
            match_in_voxel(map, P, root, pw, var6, &ok, &best);
            if (ok) {
                *ok1 = true;
                sb.match_node[i] = best.node;
                sb.match_layer[i] = best.layer;
            } else if (o2 == P.shard_rank) {
                const int s2 = hash_find(map, nkey);
                if (s2 >= 0 && map.root_node[s2] >= 0) match_in_voxel(map, P, map.root_node[s2], pw, var6, &ok, &best);
                if (ok) { sb.match_node[i] = best.node; sb.match_layer[i] = best.layer; }
            }
        }
    } else if (o2 == P.shard_rank) {
        const int s2 = hash_find(map, nkey);
        if (s2 >= 0 && map.root_node[s2] >= 0) {
            MatchResult best; best.node = -1; best.layer = 0; best.prob = 0.0;
            bool ok = false;
            match_in_voxel(map, P, map.root_node[s2], pw, var6, &ok, &best);
            if (ok) { sb.slot[i] = best.node; sb.seg[i] = best.layer; }
        }
    }
}
// bit-word form (NCCL all-reduce / gloo variant): the two bits are OR-ed into per-scan words
IM_HDN inline void shard_pass1_point(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, unsigned int* bits_exists, unsigned int* bits_ok) {
    bool ex, ok1;
    shard_pass1_flags(map, P, sb, state, i, &ex, &ok1);
#if defined(__CUDA_ARCH__)
    if (ex) atomicOr(&bits_exists[i >> 5], 1u << (i & 31));
    if (ok1) atomicOr(&bits_ok[i >> 5], 1u << (i & 31));
#else
    if (ex) bits_exists[i >> 5] |= 1u << (i & 31);
    if (ok1) bits_ok[i >> 5] |= 1u << (i & 31);
#endif
}
// pass 2: after the bits of all ranks have been combined (ex / ok1 = the point's two global bits)
IM_HDN inline bool shard_pass2_flags(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, bool ex, bool ok1, long long* terms, int* err) {
    int node = sb.match_node[i];
    if (node < 0 && sb.slot[i] >= 0) {
        if (ex && !ok1) { node = sb.slot[i]; sb.match_node[i] = node; sb.match_layer[i] = sb.seg[i]; }
    }
    if (node < 0) return false;
    double pwd[3];
    const double pb[3] = {(double)sb.body[i * 3 + 0], (double)sb.body[i * 3 + 1], (double)sb.body[i * 3 + 2]};
    body_to_world(P, state, state + 9, pb, pwd);
    return residual_terms(map, P, sb, state, i, node, pwd, terms, err);
}
IM_HDN inline bool shard_pass2_point(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, const unsigned int* bits_exists, const unsigned int* bits_ok, long long* terms, int* err) {
    const bool ex = (bits_exists[i >> 5] >> (i & 31)) & 1u, ok1 = (bits_ok[i >> 5] >> (i & 31)) & 1u;
    return shard_pass2_flags(map, P, sb, state, i, ex, ok1, terms, err);
}

// ------------------------------------------------------------------ K4: IESKF update
// The reference forms K1 = (H^T R^-1 H (+) 0_12 + P^-1)^-1 with two 18x18 inverses per iteration (voxel_mapping.cpp:1588-1592).
// H^T R^-1 H is non-zero only in its 6x6 pose block A, and K1 is only ever used through its first six columns, for which the
// matrix inversion lemma gives
//     K1[:, :6] = P[:, :6] (I6 + A P11)^-1,          P11 = P[:6, :6]
// (G = K1[:, :6] A, solution = K1[:, :6] H^T z + v - G v[:6], final P = P - G[:, :6] P[:6, :]).  One 6x6 partial-pivot LU instead
// of two 18x18 ones, no P^-1 at all; better conditioned than the double inversion.  The oracle evaluates the same expressions
// in the same order (orc_lio.hpp, solve_mode 0) and bounds the distance to the literal reference form (solve_mode 1).
struct SolveScratch {
    double HTH[36];
    double HTz[6];
    double B[36];     // I + A P11, LU-factorised in place
    double S[36];     // its inverse
    double K1c[108];  // K1[:, :6]
    double G6[108];   // G[:, :6]
    double vec[18];
    double sol[18];
    double ncov[324];
    int piv[6];
    int flags[2];
};

// 6x6 partial-pivot LU (one thread) + substitution (one thread per column); same operation order as orc::lu_inverse<6>.
// The factorisation runs on a register copy, every loop unrolled through the step template (a row exchange is a chain of selects, no
// indexed access -- plain `#pragma unroll` loops with a conditional swap left the copy in local memory):
// through shared memory, as first written, the one thread's dependent load/store chain was a large share of the IESKF update.
template <int K>
IM_HD void lu_step6(double (&a)[36], int (&piv)[6]) {
    int best = K;
    double bv = fabs(a[K * 6 + K]);
#pragma unroll
    for (int i = K + 1; i < 6; ++i) {
        const double v = fabs(a[i * 6 + K]);
        if (v > bv) { bv = v; best = i; }
    }
#pragma unroll
    for (int i = K + 1; i < 6; ++i) {   // exchange rows K and `best`
        const bool sw = (best == i);
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const double x = a[K * 6 + j], y = a[i * 6 + j];
            a[K * 6 + j] = sw ? y : x;
            a[i * 6 + j] = sw ? x : y;
        }
        const int p = piv[K], q = piv[i];
        piv[K] = sw ? q : p;
        piv[i] = sw ? p : q;
    }
    const double pivv = a[K * 6 + K];
#pragma unroll
    for (int i = K + 1; i < 6; ++i) a[i * 6 + K] = a[i * 6 + K] / pivv;
#pragma unroll
    for (int i = K + 1; i < 6; ++i) {
        const double lik = a[i * 6 + K];
#pragma unroll
        for (int j = K + 1; j < 6; ++j) a[i * 6 + j] = a[i * 6 + j] - lik * a[K * 6 + j];
    }
}
IM_HDN inline void lu_factor6(double* a_io, int* piv_io) {
    double a[36];
    int piv[6];
#pragma unroll
    for (int i = 0; i < 36; ++i) a[i] = a_io[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) piv[i] = i;
    lu_step6<0>(a, piv); lu_step6<1>(a, piv); lu_step6<2>(a, piv); lu_step6<3>(a, piv); lu_step6<4>(a, piv); lu_step6<5>(a, piv);
#pragma unroll
    for (int i = 0; i < 36; ++i) a_io[i] = a[i];
#pragma unroll
    for (int i = 0; i < 6; ++i) piv_io[i] = piv[i];
}
IM_HDN inline void lu_solve_col6(const double* a, const int* piv, int c, double* inv) {
    double y[6];
    for (int i = 0; i < 6; ++i) {
        double s = (piv[i] == c) ? 1.0 : 0.0;
        for (int j = 0; j < i; ++j) s = s - a[i * 6 + j] * y[j];
        y[i] = s;
    }
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
        for (int j = i + 1; j < 6; ++j) s = s - a[i * 6 + j] * y[j];
        y[i] = s / a[i * 6 + i];
    }
    for (int i = 0; i < 6; ++i) inv[i * 6 + c] = y[i];
}

// state_propagat (-) state, include/common_lib.h:249-260
IM_HDN inline void state_minus(const double* a, const double* b, double* out) {
    double rotd[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) rotd[i * 3 + j] = (b[0 * 3 + i] * a[0 * 3 + j] + b[1 * 3 + i] * a[1 * 3 + j]) + b[2 * 3 + i] * a[2 * 3 + j];
    so3_log3(rotd, out);
    for (int i = 0; i < 15; ++i) out[3 + i] = a[9 + i] - b[9 + i];
}
// state (+)= delta, include/common_lib.h:238-247
IM_HDN inline void state_plus(double* s, const double* add) {
    double E[9], Rn[9];
    so3_exp3(add[0], add[1], add[2], E);
    m3_mul(s, E, Rn);
    for (int i = 0; i < 9; ++i) s[i] = Rn[i];
    for (int i = 0; i < 15; ++i) s[9 + i] = s[9 + i] + add[3 + i];
}

// one IESKF update (voxel_mapping.cpp:1586-1650) executed by one thread block (>= 32 threads; 1 thread in the host emulation)
IM_HDN inline void ieskf_solve(const LioParams& P, LioCtrl* ctrl, int iter, SolveScratch* S, int tid, int nthreads) {
    double* state = ctrl->state;
    double* cov = state + 24;
    // normal equations from the fixed-point accumulators
    for (int e = tid; e < 29; e += nthreads) {
#if defined(__CUDA_ARCH__)
        const long long hi = (long long)*(volatile unsigned long long*)&ctrl->acc[iter][2 * e];
        const long long lo = (long long)*(volatile unsigned long long*)&ctrl->acc[iter][2 * e + 1];
#else
        const long long hi = (long long)ctrl->acc[iter][2 * e], lo = (long long)ctrl->acc[iter][2 * e + 1];
#endif
        // hi/lo were accumulated from block sums: total = hi * 2^32 + lo (two's complement, exact)
        const double v = fx_value(hi, lo);
        if (e < 21) {
            int ei = 0, base = 0;
            while (e >= base + (6 - ei)) { base += 6 - ei; ++ei; }
            const int ej = ei + (e - base);
            S->HTH[ei * 6 + ej] = v;
            S->HTH[ej * 6 + ei] = v;
        } else if (e < 27) {
            S->HTz[e - 21] = v;
        } else if (e == 27) {
            ctrl->stats[iter].total_residual = v;
        } else {
            ctrl->stats[iter].n_match = (double)((hi << 32) + lo);
        }
    }
    // v = state_propagat (-) state: independent of the gain, done by the last thread while thread 0 factorises
    IM_STAMP_IF(tid == 0, 20, 0);
    if (tid == nthreads - 1) state_minus(ctrl->state_prop, state, S->vec);
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 21, 0);
    for (int idx = tid; idx < 36; idx += nthreads) {
        const int i = idx / 6, j = idx % 6;
        double s = (i == j) ? 1.0 : 0.0;
        for (int k = 0; k < 6; ++k) s = s + S->HTH[i * 6 + k] * cov[k * 18 + j];
        S->B[idx] = s;
    }
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 22, 0);
    if (tid == 0) lu_factor6(S->B, S->piv);
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 23, 0);
    for (int c = tid; c < 6; c += nthreads) lu_solve_col6(S->B, S->piv, c, S->S);
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 24, 0);
    for (int idx = tid; idx < 108; idx += nthreads) {
        const int i = idx / 6, j = idx % 6;
        double s = 0.0;
        for (int k = 0; k < 6; ++k) s = s + cov[i * 18 + k] * S->S[k * 6 + j];
        S->K1c[idx] = s;
    }
    IM_SYNCBLOCK();
    for (int idx = tid; idx < 108; idx += nthreads) {
        const int i = idx / 6, j = idx % 6;
        double s = 0.0;
        for (int k = 0; k < 6; ++k) s = s + S->K1c[i * 6 + k] * S->HTH[k * 6 + j];
        S->G6[idx] = s;
    }
    IM_SYNCBLOCK();
    for (int i = tid; i < 18; i += nthreads) {
        double s1 = 0.0, s2 = 0.0;
        for (int k = 0; k < 6; ++k) s1 = s1 + S->K1c[i * 6 + k] * S->HTz[k];
        for (int k = 0; k < 6; ++k) s2 = s2 + S->G6[i * 6 + k] * S->vec[k];
        S->sol[i] = (s1 + S->vec[i]) - s2;
    }
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 25, 0);
    if (tid == 0) {
        const double* sol = S->sol;
        const double rn = sqrt((sol[0] * sol[0] + sol[1] * sol[1]) + sol[2] * sol[2]);
        const double tn = sqrt((sol[3] * sol[3] + sol[4] * sol[4]) + sol[5] * sol[5]);
        const int converged = ((rn * 57.3 < 0.01) && (tn * 100 < 0.015)) ? 1 : 0;
        int rematch = ctrl->rematch_num;
        if (converged || ((rematch == 0) && (iter == P.max_iter - 2))) rematch++;
        ctrl->rematch_num = rematch;
        ctrl->iters_run = iter + 1;
        S->flags[0] = (rematch >= 2 || iter == P.max_iter - 1) ? 1 : 0;
        S->flags[1] = converged;
    }
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 26, 0);
    // state (+)= solution by thread 0 while the other warps (all threads when the block is a single warp / the host emulation) do the
    // covariance update and the diagnostics: neither reads the state vector's first 24 entries
    const bool split_tail = nthreads > 32;
    if (tid == 0) state_plus(state, S->sol);
    if (!split_tail || tid >= 32) {
        const int t2 = split_tail ? tid - 32 : tid, n2 = split_tail ? nthreads - 32 : nthreads;
        IterStats& st = ctrl->stats[iter];   // diagnostics of the iteration (parity tests)
        for (int i = t2; i < 36; i += n2) st.HTH[i] = S->HTH[i];
        for (int i = t2; i < 6; i += n2) st.HTz[i] = S->HTz[i];
        for (int i = t2; i < 18; i += n2) st.solution[i] = S->sol[i];
        if (t2 == 0) st.converged = S->flags[1];
        if (S->flags[0]) {
            // cov = (I - G) cov = cov - G[:, :6] cov[:6, :]  (rows 0-5 of cov are operands of every element: staged, then stored)
            for (int idx = t2; idx < 324; idx += n2) {
                const int i = idx / 18, j = idx % 18;
                double s = 0.0;
                for (int k = 0; k < 6; ++k) s = s + S->G6[i * 6 + k] * cov[k * 18 + j];
                S->ncov[idx] = cov[idx] - s;
            }
        }
    }
    IM_SYNCBLOCK();
    if (S->flags[0]) {
        for (int idx = tid; idx < 324; idx += nthreads) cov[idx] = S->ncov[idx];
        if (tid == 0) ctrl->stop = 1;
    }
    IM_SYNCBLOCK();
    IM_STAMP_IF(tid == 0, 27, 0);
}

// Forward_without_imu (constant-velocity prediction), src/IMU_Processing.cpp:486-553
IM_HDN inline void predict_const_vel(double* state, double dt, double cov_gyr, double cov_acc, double* T /*324*/, double* Fx /*324*/, int tid, int nthreads) {
    double* cov = state + 24;
    if (tid == 0) {
        for (int i = 0; i < 324; ++i) Fx[i] = 0.0;
        for (int i = 0; i < 18; ++i) Fx[i * 18 + i] = 1.0;
        double En[9];
        so3_exp_dt(state + 15, -dt, En);
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) Fx[a * 18 + b] = En[a * 3 + b];
        for (int a = 0; a < 3; ++a) { Fx[a * 18 + 9 + a] = dt; Fx[(3 + a) * 18 + 6 + a] = dt; }
    }
    IM_SYNCBLOCK();
    for (int idx = tid; idx < 324; idx += nthreads) {
        const int i = idx / 18, j = idx % 18;
        double s = 0.0;
        for (int k = 0; k < 18; ++k) s = s + Fx[i * 18 + k] * cov[k * 18 + j];
        T[idx] = s;
    }
    IM_SYNCBLOCK();
    for (int idx = tid; idx < 324; idx += nthreads) {
        const int i = idx / 18, j = idx % 18;
        double s = 0.0;
        for (int k = 0; k < 18; ++k) s = s + T[i * 18 + k] * Fx[j * 18 + k];
        double cw = 0.0;
        if (i == j && i >= 9 && i < 12) cw = cov_gyr * dt * dt;
        if (i == j && i >= 6 && i < 9) cw = cov_acc * dt * dt;
        cov[idx] = s + cw;
    }
    IM_SYNCBLOCK();
    if (tid == 0) {
        double Ef[9], Rn[9];
        so3_exp_dt(state + 15, dt, Ef);
        m3_mul(state, Ef, Rn);
        for (int i = 0; i < 9; ++i) state[i] = Rn[i];
        for (int i = 0; i < 3; ++i) state[9 + i] = state[9 + i] + state[12 + i] * dt;
    }
    IM_SYNCBLOCK();
}

// ------------------------------------------------------------------ K5: map growth
// pass 1 (thread / point): world point + covariance with the converged state, sort key, root-voxel insert, count
//   mode 0: map_incremental_grow (ImMesh_mesh_reconstruction.cpp:393-404)   cov uses (R R_ext) and [p_imu]x
//   mode 1: voxel_map_init       (voxel_mapping.cpp:1249-1265)              cov uses R and [p_lidar]x, input order kept
//   mode | 2: world points (sb.pw) and covariances (sb.var) were supplied by the caller (Point_with_var lists of
//             updateVoxelMap / buildVoxelMap, voxel_mapping.hpp:80-92), caller's order is kept
IM_HDN inline void grow_point(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, const double* state, int i, int mode) {
    const double* R = state;
    const double* t = state + 9;
    const double* cov = state + 24;
    float wx, wy, wz;
    double* v6 = sb.var + (size_t)i * 6;
    double pb[3] = {0.0, 0.0, 0.0};
    if (mode & 2) {
        wx = sb.pw[(size_t)i * 3 + 0]; wy = sb.pw[(size_t)i * 3 + 1]; wz = sb.pw[(size_t)i * 3 + 2];
    } else {
        pb[0] = (double)sb.body[i * 3 + 0]; pb[1] = (double)sb.body[i * 3 + 1]; pb[2] = (double)sb.body[i * 3 + 2];
        double pwd[3];
        body_to_world(P, R, t, pb, pwd);
        wx = (float)pwd[0]; wy = (float)pwd[1]; wz = (float)pwd[2];
        sb.pw[(size_t)i * 3 + 0] = wx; sb.pw[(size_t)i * 3 + 1] = wy; sb.pw[(size_t)i * 3 + 2] = wz;
    }
    // the root voxel (and with it the owning rank) follows from the world point alone: a sharded rank is done with the points of
    // other ranks' voxels here, before the covariance propagation
    const double pw[3] = {(double)wx, (double)wy, (double)wz};
    long long k[3];
    sb.slot[i] = -1;
    if (!voxel_key3(pw, P.voxel_size_ins, k)) { im_atomic_or(map.err, IM_ERR_KEY_RANGE); return; }
    const unsigned long long key = pack_key(k[0], k[1], k[2]);
    if (P.shard_n > 1 && voxel_owner(key, P.shard_n) != P.shard_rank) return;   // another rank owns this root voxel
    if (mode & 2) {
        sb.sortkey[i] = (double)i;
    } else if (mode == 0) {
        double RRe[9];
        m3_mul(R, P.extR, RRe);
        world_cov(RRe, sb.body_cov + (size_t)i * 6, sb.p_imu + (size_t)i * 3, cov, v6);
        sb.sortkey[i] = sqrt((v6[0] * v6[0] + v6[3] * v6[3]) + v6[5] * v6[5]);  // var_contrast, voxel_mapping.cpp:49
    } else {
        double pt[3] = {pb[0], pb[1], pb[2]};
        double bv[6];
        calc_body_var(pt, P.dept_err, P.dir_var, bv);
        world_cov(R, bv, pt, cov, v6);
        sb.sortkey[i] = (double)i;
    }
    int created = 0;
    const int slot = hash_insert(map, key, &created);
    if (slot < 0) return;
    if (created) {
        map.root_node[slot] = make_root(map, P, key, slot);
        im_atomic_add(map.n_roots, 1);
    }
    sb.slot[i] = slot;
    if (im_atomic_add(&sb.slot_count[slot], 1) == 0) {
        const int ti = im_atomic_add(sb.n_touched, 1);
        sb.touched[ti] = slot;
    }
}
// pass 2 (thread / touched voxel): claim a segment
IM_HD void grow_segment(const ScanBuf& sb, int ti) {
    const int slot = sb.touched[ti];
    sb.slot_offset[slot] = im_atomic_add(sb.seg_top, sb.slot_count[slot]);
    sb.slot_cursor[slot] = 0;
}
// pass 3 (thread / point): scatter point indices into the voxel's segment
IM_HD void grow_scatter(const ScanBuf& sb, int i) {
    const int slot = sb.slot[i];
    if (slot < 0) return;
    const int pos = sb.slot_offset[slot] + im_atomic_add(&sb.slot_cursor[slot], 1);
    sb.seg[pos] = i;
}
// pass 4 (warp / touched voxel): order the segment like std::sort(var_contrast) would, then apply the points
IM_HDN inline void grow_voxel(const VoxelMapDev& map, const LioParams& P, const ScanBuf& sb, int ti, int mode, int lane, int nlanes, int* sorted_scratch) {
    const int slot = sb.touched[ti];
    const int cnt = sb.slot_count[slot];
    const int off = sb.slot_offset[slot];
    // rank sort on (key, index): rank = number of strictly smaller elements
    for (int a = lane; a < cnt; a += nlanes) {
        const int ia = sb.seg[off + a];
        const double ka = sb.sortkey[ia];
        int rank = 0;
        for (int b = 0; b < cnt; ++b) {
            const int ib = sb.seg[off + b];
            const double kb = sb.sortkey[ib];
            if (kb < ka || (kb == ka && ib < ia)) ++rank;
        }
        sorted_scratch[off + rank] = ia;
    }
    IM_SYNCWARP();
    const int root = map.root_node[slot];
    if (root >= 0) {
        if ((mode & 1) == 0) {
            for (int a = 0; a < cnt; ++a) {
                const int i = sorted_scratch[off + a];
                update_octo_tree(map, P, root, sb.pw[(size_t)i * 3 + 0], sb.pw[(size_t)i * 3 + 1], sb.pw[(size_t)i * 3 + 2], sb.var + (size_t)i * 6, lane, nlanes);
            }
        } else {
            // buildVoxelMap: append everything, then one init_octo_tree (voxel_mapping.cpp:115-150)
            for (int a = 0; a < cnt; ++a) {
                const int i = sorted_scratch[off + a];
                const float px = sb.pw[(size_t)i * 3 + 0], py = sb.pw[(size_t)i * 3 + 1], pz = sb.pw[(size_t)i * 3 + 2];
                if (lane == 0) {
                    node_append(map, root, px, py, pz, sb.var + (size_t)i * 6);
                    map.nodes[root].new_points += 1;
                }
                node_moments_add(map, root, px, py, pz, sb.var + (size_t)i * 6, lane, nlanes);
            }
            IM_SYNCWARP();
            init_octo_tree(map, P, root, lane, nlanes);
        }
    }
    IM_SYNCWARP();
    if (lane == 0) {
        sb.slot_count[slot] = 0;
        sb.slot_cursor[slot] = 0;
    }
}
// between scans: recycle chunks freed during the scan
IM_HD void recycle_chunks(const VoxelMapDev& map, int tid, int nthreads) {
    int top = *map.avail_top;
    if (top < 0) top = 0;
    const int np = *map.pending_n < map.max_chunks ? *map.pending_n : map.max_chunks;
    for (int i = tid; i < np; i += nthreads) map.avail[top + i] = map.pending[i];
    IM_SYNCBLOCK();
    if (tid == 0) {
        *map.avail_top = top + np;
        *map.pending_n = 0;
    }
}

// ------------------------------------------------------------------ scan publishers (immesh_lio_effect_cloud / _registered_cloud)
// one published point: RGBpointBodyToWorld (voxel_mapping_common.cpp:168-189) with `state`, x y z stored as the float PointType holds
IM_HD void scan_pub_row(const LioParams& P, const double* state, const float* p, float intensity, float* row) {
    const double pb[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double pw[3];
    body_to_world(P, state, state + 9, pb, pw);
    row[0] = (float)pw[0]; row[1] = (float)pw[1]; row[2] = (float)pw[2]; row[3] = intensity;
}

}  // namespace immesh
