// ORACLE (test infrastructure, NOT product code): C entry points for the ctypes harness in
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
// Parity status: "parity unpinned" (see orc_math.hpp).
#include <chrono>
#include <cstring>

#include "orc_lio.hpp"
#include "orc_mesh.hpp"
#include "orc_frontend.hpp"
#include "orc_imu.hpp"

using namespace orc;

static void pack_state(const State& s, double* o) {
    std::memcpy(o, s.rot, 9 * 8);
    std::memcpy(o + 9, s.pos, 24);
    std::memcpy(o + 12, s.vel, 24);
    std::memcpy(o + 15, s.bg, 24);
    std::memcpy(o + 18, s.ba, 24);
    std::memcpy(o + 21, s.grav, 24);
    std::memcpy(o + 24, s.cov, 324 * 8);
}
static void unpack_state(const double* o, State& s) {
    std::memcpy(s.rot, o, 9 * 8);
    std::memcpy(s.pos, o + 9, 24);
    std::memcpy(s.vel, o + 12, 24);
    std::memcpy(s.bg, o + 15, 24);
    std::memcpy(s.ba, o + 18, 24);
    std::memcpy(s.grav, o + 21, 24);
    std::memcpy(s.cov, o + 24, 324 * 8);
}

extern "C" {

// cfg_d: [voxel_size, min_eigen_value, dept_err, beam_err, extR[9], extT[3]]  (16)
// cfg_i: [max_layer, layer_init_size[5], max_points_size, max_iteration, calib_laser, sum_mode, omp_threads, solve_mode, plane_var_mode] (13)
void* orc_lio_create(const double* cfg_d, const int* cfg_i) {
    LioCfg c;
    c.voxel_size = cfg_d[0];
    c.min_eigen_value = cfg_d[1];
    c.dept_err = cfg_d[2];
    c.beam_err = cfg_d[3];
    for (int i = 0; i < 9; ++i) c.extR[i] = cfg_d[4 + i];
    for (int i = 0; i < 3; ++i) c.extT[i] = cfg_d[13 + i];
    c.max_layer = cfg_i[0];
    for (int i = 0; i < 5; ++i) c.layer_init_size[i] = cfg_i[1 + i];
    c.max_points_size = cfg_i[6];
    c.max_iteration = cfg_i[7];
    c.calib_laser = cfg_i[8];
    c.sum_mode = cfg_i[9];
    c.omp_threads = cfg_i[10];
    c.solve_mode = cfg_i[11];
    c.plane_var_mode = cfg_i[12];
    return new LioOracle(c);
}
void orc_lio_destroy(void* h) { delete (LioOracle*)h; }
void orc_lio_set_state(void* h, const double* s) { unpack_state(s, ((LioOracle*)h)->state); }
void orc_lio_get_state(void* h, double* s) { pack_state(((LioOracle*)h)->state, s); }
void orc_lio_map_init(void* h, const float* body, int n) { ((LioOracle*)h)->voxel_map_init(body, n); }
int orc_lio_estimate(void* h, const float* body, int n, const double* state_prop) {
    LioOracle* o = (LioOracle*)h;
    State sp;
    unpack_state(state_prop, sp);
    o->lio_state_estimation(body, n, sp);
    return o->iters_run;
}
// out: HTH[36], HTz[6], n_match, total_residual, solution[18], converged  (63)
void orc_lio_iter_stats(void* h, int it, double* out) {
    const IterStats& s = ((LioOracle*)h)->iter_stats[it];
    std::memcpy(out, s.HTH, 36 * 8);
    std::memcpy(out + 36, s.HTz, 6 * 8);
    out[42] = s.n_match;
    out[43] = s.total_residual;
    std::memcpy(out + 44, s.solution, 18 * 8);
    out[62] = s.converged;
}
int orc_lio_last_matches(void* h, int* idx, int* layer, int cap) {
    LioOracle* o = (LioOracle*)h;
    const int n = (int)o->last_match_idx.size();
    for (int i = 0; i < n && i < cap; ++i) { idx[i] = o->last_match_idx[i]; layer[i] = o->last_match_layer[i]; }
    return n;
}
void orc_lio_map_grow(void* h, const float* body, int n) { ((LioOracle*)h)->map_incremental_grow(body, n); }
void orc_lio_predict(void* h, double dt, double cov_gyr, double cov_acc) { ((LioOracle*)h)->forward_without_imu(dt, cov_gyr, cov_acc); }
long orc_lio_dump_map(void* h, double* out, long cap_rows) {
    std::vector<double> d;
    ((LioOracle*)h)->dump_map(d);
    const long rows = (long)(d.size() / LioOracle::kDumpCols);
    if (out && rows <= cap_rows) std::memcpy(out, d.data(), d.size() * 8);
    return rows;
}
long orc_lio_num_root_voxels(void* h) { return (long)((LioOracle*)h)->feat_map.size(); }

// Stand-alone residual list at the CURRENT state (BuildResidualListOMP, voxel_mapping.cpp:153-245), for the
// drop-in immesh_residual_build() parity test.  Outputs per match: src index, layer, point[3], normal[3],
// center[3], d, plane_var[21]  -> 2 ints + 31 doubles.
int orc_lio_residual_list(void* h, const float* body, int n, int* idx_layer, double* vals, int cap) {
    LioOracle* o = (LioOracle*)h;
    o->prepare_scan(body, n);
    std::vector<PV> pv(n);
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < 3; ++j) pv[i].pb[j] = (double)body[i * 3 + j];
        o->body_to_world_f(o->state.rot, o->state.pos, pv[i].pb, pv[i].pw);
        o->world_cov_match(o->state.rot, o->state.cov, i, pv[i].var);
    }
    std::vector<Ptpl> out;
    o->build_residual_list(pv, 3.0, out);
    const int m = (int)out.size();
    for (int i = 0; i < m && i < cap; ++i) {
        idx_layer[2 * i] = out[i].src_index;
        idx_layer[2 * i + 1] = out[i].layer;
        double* v = vals + (size_t)i * 31;
        for (int j = 0; j < 3; ++j) { v[j] = out[i].point[j]; v[3 + j] = out[i].normal[j]; v[6 + j] = out[i].center[j]; }
        v[9] = out[i].d;
        for (int j = 0; j < 21; ++j) v[10 + j] = out[i].plane_var[j];
    }
    return m;
}

// transformLidar of a full-resolution scan with the current state (ImMesh_mesh_reconstruction.cpp:413 -> voxel_mapping_common.cpp:709-726)
void orc_lio_transform_full(void* h, const float* body, int n, float* world) {
    LioOracle* o = (LioOracle*)h;
    for (int i = 0; i < n; ++i) {
        const double pb[3] = {(double)body[i * 3 + 0], (double)body[i * 3 + 1], (double)body[i * 3 + 2]};
        double pw[3];
        o->body_to_world_f(o->state.rot, o->state.pos, pb, pw);
        for (int j = 0; j < 3; ++j) world[i * 3 + j] = (float)pw[j];
    }
}
// The three free functions of voxel_mapping.hpp:80-105 on caller-built Point_with_var lists (parity tests of the *_pv entry points)
static void fill_pv(std::vector<PV>& pv, const double* pts_body, const double* pts_world, const double* var9, int n) {
    pv.resize(n);
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < 3; ++j) { pv[i].pb[j] = pts_body[i * 3 + j]; pv[i].pw[j] = pts_world[i * 3 + j]; }
        const double* v = var9 + (size_t)i * 9;
        pv[i].var[0] = v[0]; pv[i].var[1] = v[1]; pv[i].var[2] = v[2]; pv[i].var[3] = v[4]; pv[i].var[4] = v[5]; pv[i].var[5] = v[8];
    }
}
void orc_lio_build_pv(void* h, const double* pts_world, const double* var9, int n) {
    std::vector<PV> pv;
    fill_pv(pv, pts_world, pts_world, var9, n);   // insert path: m_point carries the world point
    ((LioOracle*)h)->build_voxel_map(pv);
}
void orc_lio_update_pv(void* h, const double* pts_world, const double* var9, int n) {
    std::vector<PV> pv;
    fill_pv(pv, pts_world, pts_world, var9, n);
    ((LioOracle*)h)->update_voxel_map(pv);
}
int orc_lio_residual_pv(void* h, const double* pts_body, const double* pts_world, const double* var9, int n, int* idx_layer, double* vals, int cap) {
    std::vector<PV> pv;
    fill_pv(pv, pts_body, pts_world, var9, n);
    std::vector<Ptpl> out;
    ((LioOracle*)h)->build_residual_list(pv, 3.0, out);
    const int m = (int)out.size();
    for (int i = 0; i < m && i < cap; ++i) {
        idx_layer[2 * i] = out[i].src_index;
        idx_layer[2 * i + 1] = out[i].layer;
        double* v = vals + (size_t)i * 31;
        for (int j = 0; j < 3; ++j) { v[j] = out[i].point[j]; v[3 + j] = out[i].normal[j]; v[6 + j] = out[i].center[j]; }
        v[9] = out[i].d;
        for (int j = 0; j < 21; ++j) v[10 + j] = out[i].plane_var[j];
    }
    return m;
}
// per-point world covariance lists exactly as the reference builds them before calling the free functions (tests build their
// Point_with_var inputs from these): mode 0 = map_incremental_grow (ImMesh_mesh_reconstruction.cpp:393-404), 1 = matching (:1344-1359)
void orc_lio_pv_lists(void* h, const float* body, int n, int mode, double* pts_world, double* var9) {
    LioOracle* o = (LioOracle*)h;
    o->prepare_scan(body, n);
    double RRe[9];
    mat3_mul(o->state.rot, o->cfg.extR, RRe);
    for (int i = 0; i < n; ++i) {
        const double pb[3] = {(double)body[i * 3 + 0], (double)body[i * 3 + 1], (double)body[i * 3 + 2]};
        double pw[3], v6[6];
        o->body_to_world_f(o->state.rot, o->state.pos, pb, pw);
        if (mode == 1) {
            o->world_cov_match(o->state.rot, o->state.cov, i, v6);
        } else {
            double Sb[9], T1[6], T2[6], C[9], nC[9], rot_var[9];
            sym6_to_full(&o->body_cov[(size_t)i * 6], Sb);
            congr_sym6(RRe, Sb, T1);
            for (int k = 0; k < 9; ++k) { C[k] = o->cross_mat[(size_t)i * 9 + k]; nC[k] = -C[k]; }
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) rot_var[a * 3 + b] = o->state.cov[a * 18 + b];
            congr_sym6(nC, rot_var, T2);
            for (int a = 0; a < 3; ++a)
                for (int b = a; b < 3; ++b) v6[sym6_idx(a, b)] = (T1[sym6_idx(a, b)] + T2[sym6_idx(a, b)]) + o->state.cov[(3 + a) * 18 + (3 + b)];
        }
        for (int j = 0; j < 3; ++j) pts_world[i * 3 + j] = pw[j];
        double* v = var9 + (size_t)i * 9;
        v[0] = v6[0]; v[1] = v6[1]; v[2] = v6[2]; v[3] = v6[1]; v[4] = v6[3]; v[5] = v6[4]; v[6] = v6[2]; v[7] = v6[4]; v[8] = v6[5];
    }
}

// ------------------------------------------------------------------ mesh
void* orc_mesh_create(double minimum_pts, double voxel_res, int append_target, int threads) {
    MeshCfg c;
    c.minimum_pts = minimum_pts;
    c.voxel_resolution = voxel_res;
    c.append_target = append_target;
    c.threads = threads;
    return new MeshOracle(c);
}
void orc_mesh_destroy(void* h) { delete (MeshOracle*)h; }
void orc_mesh_push_frame(void* h, const float* pts, int n, const double* pose_t) { ((MeshOracle*)h)->push_frame(pts, n, pose_t); }
// counts: [n_vertices, n_live_tris, frame_new_vertices, frame_voxels_meshed, frame_added, frame_removed (summed over voxels), n_voxels, n_activated]
void orc_mesh_counts(void* h, long* c) {
    MeshOracle* m = (MeshOracle*)h;
    c[0] = (long)m->vpos.size();
    c[1] = (long)m->live.size();
    c[2] = m->frame_new_vertices;
    c[3] = m->frame_voxels_meshed;
    c[4] = m->frame_added_mult;
    c[5] = m->frame_removed_mult;
    c[6] = (long)m->voxels.size();
    c[7] = (long)m->activated.size();
}
void orc_mesh_get_vertices(void* h, float* pos, double* smooth) {
    MeshOracle* m = (MeshOracle*)h;
    for (size_t i = 0; i < m->vpos.size(); ++i)
        for (int j = 0; j < 3; ++j) {
            if (pos) pos[i * 3 + j] = m->vpos[i][j];
            if (smooth) smooth[i * 3 + j] = m->vsmooth[i][j];
        }
}
void orc_mesh_get_tris(void* h, int* tris, int* flips) {  // ascending (i,j,k)
    MeshOracle* m = (MeshOracle*)h;
    size_t i = 0;
    for (const Tri& t : m->live) {
        tris[i * 3] = t[0]; tris[i * 3 + 1] = t[1]; tris[i * 3 + 2] = t[2];
        if (flips) flips[i] = m->flip.at(t);
        ++i;
    }
}
void orc_mesh_get_frame_delta(void* h, int* added, int* removed) {
    MeshOracle* m = (MeshOracle*)h;
    for (size_t i = 0; i < m->frame_added.size(); ++i)
        for (int j = 0; j < 3; ++j) added[i * 3 + j] = m->frame_added[i][j];
    for (size_t i = 0; i < m->frame_removed.size(); ++i)
        for (int j = 0; j < 3; ++j) removed[i * 3 + j] = m->frame_removed[i][j];
}
// voxel keys (x,y,z) + vertex count, ascending key
long orc_mesh_get_voxels(void* h, int* out, long cap) {
    MeshOracle* m = (MeshOracle*)h;
    std::vector<std::array<int, 4>> rows;
    for (auto& v : m->voxels) rows.push_back({v.key.x, v.key.y, v.key.z, (int)v.pts.size()});
    std::sort(rows.begin(), rows.end());
    if (out && (long)rows.size() <= cap)
        for (size_t i = 0; i < rows.size(); ++i)
            for (int j = 0; j < 4; ++j) out[i * 4 + j] = rows[i][j];
    return (long)rows.size();
}
// per voxel meshed in the last frame, ascending key: x, y, z, dilated-set size, largest cavity, seed found, in-circle ties, duplicates
long orc_mesh_frame_voxel_stats(void* h, long* out, long cap) {
    MeshOracle* m = (MeshOracle*)h;
    const long n = (long)m->frame_stats.size();
    if (out && n <= cap)
        for (long i = 0; i < n; ++i) {
            const MeshOracle::VoxStat& s = m->frame_stats[i];
            const long row[8] = {s.key[0], s.key[1], s.key[2], s.n, s.max_cav, s.seeded, s.n_ties, s.n_dup};
            std::memcpy(out + i * 8, row, sizeof(row));
        }
    return n;
}
void orc_mesh_smooth_all(void* h, double smooth_factor, int knn, double* out) {
    std::vector<std::array<double, 3>> r;
    ((MeshOracle*)h)->smooth_all(smooth_factor, knn, r);
    for (size_t i = 0; i < r.size(); ++i) { out[3 * i] = r[i][0]; out[3 * i + 1] = r[i][1]; out[3 * i + 2] = r[i][2]; }
}
long orc_mesh_region_keys(void* h, double region_size, int* out) {   // one key per live triangle, in ascending-triple order
    std::vector<std::array<int, 3>> r;
    ((MeshOracle*)h)->region_keys(region_size, r);
    if (out)
        for (size_t i = 0; i < r.size(); ++i) { out[3 * i] = r[i][0]; out[3 * i + 1] = r[i][1]; out[3 * i + 2] = r[i][2]; }
    return (long)r.size();
}
long orc_mesh_render_depth(void* h, const double* K4, int w, int ht, double z_near, double z_far, const double* R, const double* t, float* depth, float* pts, int* pix) {
    std::vector<float> d;
    std::vector<std::array<float, 3>> p;
    std::vector<int> px;
    ((MeshOracle*)h)->render_depth(K4, w, ht, z_near, z_far, R, t, d, p, px);
    std::memcpy(depth, d.data(), d.size() * 4);
    for (size_t i = 0; i < p.size(); ++i) { pts[3 * i] = p[i][0]; pts[3 * i + 1] = p[i][1]; pts[3 * i + 2] = p[i][2]; pix[i] = px[i]; }
    return (long)p.size();
}
void orc_mesh_knn(void* h, const float* q, int nq, int k, double max_dist, int* idx, float* d2) {
    MeshOracle* m = (MeshOracle*)h;
    std::vector<std::pair<float, int>> nn;
    for (int i = 0; i < nq; ++i) {
        m->knn(q + 3 * i, k, max_dist, nn);
        for (int j = 0; j < k; ++j) {
            idx[i * k + j] = j < (int)nn.size() ? nn[j].second : -1;
            d2[i * k + j] = j < (int)nn.size() ? nn[j].first : INFINITY;
        }
    }
}
// raw exact Delaunay of integer points (no angle filter): returns #faces, CCW vertex triples
int orc_delaunay2d_int(const int64_t* pts, int n, int* faces, int cap) {
    Delaunay2D dt;
    if (!dt.run(pts, n)) return 0;
    int c = 0;
    for (const auto& t : dt.tris) {
        if (!t.alive || t.v[0] < 0 || t.v[1] < 0 || t.v[2] < 0) continue;
        if (c < cap) { faces[3 * c] = t.v[0]; faces[3 * c + 1] = t.v[1]; faces[3 * c + 2] = t.v[2]; }
        ++c;
    }
    return c;
}
// per-voxel mesher on explicit 3-D points (ids 0..n-1): PCA projection + Delaunay + 150-degree filter
int orc_voxel_triangulate(const float* pts, int n, double voxel_res, int* faces, int cap, double* short_axis) {
    MeshCfg c{0.1, voxel_res, 10000, 1};
    MeshOracle m(c);
    std::vector<long> ids(n);
    for (int i = 0; i < n; ++i) {
        m.vpos.push_back({pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]});
        ids[i] = i;
    }
    std::vector<Tri> f;
    m.triangulate(ids, short_axis, f);
    for (size_t i = 0; i < f.size() && (int)i < cap; ++i)
        for (int j = 0; j < 3; ++j) faces[i * 3 + j] = f[i][j];
    return (int)f.size();
}

// ------------------------------------------------------------------ math probes for unit tests
void orc_math_probe(const double* x, int n, double* s, double* c, double* e, double* ac) {
    for (int i = 0; i < n; ++i) {
        det_sincos(x[i], &s[i], &c[i]);
        e[i] = det_exp(-std::fabs(x[i]));
        ac[i] = det_acos(std::fmax(-1.0, std::fmin(1.0, x[i])));
    }
}
// ImuProcess::UndistortPcl restatement (orc_imu.hpp).  cfg: cov_gyr 3, cov_acc 3, cov_bias_gyr 3, cov_bias_acc 3, mean_acc_norm, lid_R 9, lid_T 3 (25)
void* orc_imu_create(const double* cfg) {
    ImuOracle* o = new ImuOracle();
    for (int i = 0; i < 3; ++i) { o->cov_gyr[i] = cfg[i]; o->cov_acc[i] = cfg[3 + i]; o->cov_bias_gyr[i] = cfg[6 + i]; o->cov_bias_acc[i] = cfg[9 + i]; o->lid_T[i] = cfg[22 + i]; }
    o->mean_acc_norm = cfg[12];
    for (int i = 0; i < 9; ++i) o->lid_R[i] = cfg[13 + i];
    return o;
}
void orc_imu_destroy(void* h) { delete (ImuOracle*)h; }
void orc_imu_reset(void* h, const double* last_imu7, double last_lidar_end_time, double last_update_time, const double* acc_s_last, const double* angvel_last) {
    ImuOracle* o = (ImuOracle*)h;
    o->last_imu.t = last_imu7[0];
    for (int i = 0; i < 3; ++i) { o->last_imu.gyr[i] = last_imu7[1 + i]; o->last_imu.acc[i] = last_imu7[4 + i]; o->acc_s_last[i] = acc_s_last ? acc_s_last[i] : 0.0; o->angvel_last[i] = angvel_last ? angvel_last[i] : 0.0; }
    o->last_lidar_end_time = last_lidar_end_time;
    o->last_update_time = last_update_time;
}
// state348 in/out; pts [n][4] in/out (sorted + compensated); returns the number of IMUpose records, copied to poses (22 doubles each)
int orc_imu_undistort(void* h, double* state348, const double* imu, int n_imu, float* pts, int n, double lidar_beg_time, double* poses, int cap_poses) {
    ImuOracle* o = (ImuOracle*)h;
    State st;
    unpack_state(state348, st);
    std::vector<ImuSample> v(n_imu);
    for (int i = 0; i < n_imu; ++i) { v[i].t = imu[7 * i]; for (int k = 0; k < 3; ++k) { v[i].gyr[k] = imu[7 * i + 1 + k]; v[i].acc[k] = imu[7 * i + 4 + k]; } }
    o->undistort_pcl(st, v, pts, n, lidar_beg_time);
    pack_state(st, state348);
    const int m = (int)o->IMUpose.size();
    for (int i = 0; i < m && i < cap_poses; ++i) {
        const Pose6D& p = o->IMUpose[i];
        double* q = poses + 22 * (size_t)i;
        q[0] = p.offset_time;
        for (int k = 0; k < 3; ++k) { q[1 + k] = p.acc[k]; q[4 + k] = p.gyr[k]; q[7 + k] = p.vel[k]; q[10 + k] = p.pos[k]; }
        for (int k = 0; k < 9; ++k) q[13 + k] = p.rot[k];
    }
    return m;
}
// pcl::VoxelGrid restatement (orc_frontend.hpp).  out: [cap][3]; returns m (or -m-1 when PCL's leaf-too-small branch copied the input)
int orc_voxel_grid(const float* pts, int n, float leaf, float* out, int cap, int* grid6) {
    const VoxelGridResult r = voxel_grid_filter(pts, n, leaf);
    const int m = (int)(r.out.size() / 3);
    for (int i = 0; i < m && i < cap; ++i) { out[3 * i] = r.out[3 * i]; out[3 * i + 1] = r.out[3 * i + 1]; out[3 * i + 2] = r.out[3 * i + 2]; }
    if (grid6) { for (int a = 0; a < 3; ++a) { grid6[a] = r.min_b[a]; grid6[3 + a] = r.div_b[a]; } }
    return r.leaf_too_small ? -m - 1 : m;
}
void orc_kitti_calib(float* pts, int n) { kitti_calib(pts, n); }
void orc_jacobi_eig3(const double* a6, double* d, double* V) { jacobi_eig3(a6, d, V); }
void orc_lu_inverse18(const double* A, double* Ainv) { lu_inverse<18>(A, Ainv); }
void orc_lu_inverse6(const double* A, double* Ainv) { lu_inverse<6>(A, Ainv); }
void orc_calc_body_var(const double* pb, double dept_err, double beam_err, double* var6) {
    double p[3] = {pb[0], pb[1], pb[2]};
    const double s = std::sin((double)(float)beam_err * 0.017453293);
    LioOracle::calc_body_var(p, (float)dept_err, s * s, var6);
}
void orc_voxel_key(const double* p, double vs, long* out) {
    const VoxelKey k = voxel_key(p, vs);
    out[0] = k.x; out[1] = k.y; out[2] = k.z;
}

}  // extern "C"
