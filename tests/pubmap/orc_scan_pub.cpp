// ORACLE EXTENSION (test infrastructure, NOT product code): publish_effect_world and publish_frame_world
// (src/voxel_mapping_common.cpp:535-547, :595-614) on the CPU oracle, which it does not change.
// The oracle keeps the match set of the last IESKF iteration (last_match_idx) but not its weights.  orc_eff_estimate runs the
// oracle's lio_state_estimation, then rebuilds the state the last iteration started from -- the start state plus the solutions of
// the iterations before it, applied with the oracle's own state_plus as its loop applies them (the covariance changes only after
// the last iteration) -- forms the last residual list again there with the oracle's own functions, and evaluates R_inv with the
// loop's expression (orc_lio.hpp, lio_state_estimation (c)-(e); voxel_mapping.cpp:1496-1527).  That the rebuilt match set equals
// last_match_idx, and that the weights reproduce the iteration's H^T R^-1 H, are checked by the tests.
#include "../../oracle/orc_capi.cpp"

#include <unordered_map>

namespace {
struct EffState {
    std::vector<float> body;     // the down-sampled body-frame scan of the last estimation (m_feats_down_body)
    std::vector<int> idx;        // matches of the last iteration, ptpl order (ascending scan index)
    std::vector<double> r_inv;   // their R_inv
    std::vector<double> normal;  // their normals as the loop uses them (float-rounded, :1377-1389)
    int replay_ok = 1;           // the rebuilt match set equals the oracle's last_match_idx
};
std::unordered_map<void*, EffState> g_eff;

// RGBpointBodyToWorld (voxel_mapping_common.cpp:168-189): pointBodyToWorld in double, the identity _gravity_correct_rotM applied
// as the reference applies it (Eigen's coefficient-wise product), then the float PointType
void rgb_body_to_world(const LioOracle& o, const float* p, float intensity, float* row) {
    const double pb[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double pw[3];
    o.body_to_world_d(o.state.rot, o.state.pos, pb, pw);
    const double G[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int r = 0; r < 3; ++r) row[r] = (float)((G[r * 3 + 0] * pw[0] + G[r * 3 + 1] * pw[1]) + G[r * 3 + 2] * pw[2]);
    row[3] = intensity;
}
}  // namespace

extern "C" {
int orc_eff_estimate(void* h, const float* body, int n, const double* state_prop) {
    LioOracle* o = (LioOracle*)h;
    const State s0 = o->state;
    const int iters = orc_lio_estimate(h, body, n, state_prop);
    EffState& e = g_eff[h];
    e = EffState();
    e.body.assign(body, body + (size_t)n * 3);
    if (iters == 0) return 0;
    State s = s0;
    for (int it = 0; it + 1 < iters; ++it) LioOracle::state_plus(s, o->iter_stats[it].solution);
    std::vector<PV> pv(n);
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < 3; ++j) pv[i].pb[j] = (double)body[i * 3 + j];
        o->body_to_world_f(s.rot, s.pos, pv[i].pb, pv[i].pw);
        o->world_cov_match(s.rot, s.cov, i, pv[i].var);
    }
    std::vector<Ptpl> ptpl;
    o->build_residual_list(pv, 3.0, ptpl);
    double RRe[9];
    mat3_mul(s.rot, o->cfg.extR, RRe);
    for (const Ptpl& pt : ptpl) {
        const double pbf[3] = {(double)(float)pt.point[0], (double)(float)pt.point[1], (double)(float)pt.point[2]};
        const double nv[3] = {(double)(float)pt.normal[0], (double)(float)pt.normal[1], (double)(float)pt.normal[2]};
        double p_imu[3], pw2[3];
        mat3_vec(o->cfg.extR, pbf, p_imu);
        for (int j = 0; j < 3; ++j) p_imu[j] = p_imu[j] + o->cfg.extT[j];
        mat3_vec(s.rot, p_imu, pw2);
        for (int j = 0; j < 3; ++j) pw2[j] = pw2[j] + s.pos[j];
        double bv[6], Sb[9], var6[6];
        double p_for_var[3] = {p_imu[0], p_imu[1], p_imu[2]};
        LioOracle::calc_body_var(p_for_var, o->dept_err_f, o->cfg.calib_laser ? o->dir_var_calib : o->dir_var, bv);
        sym6_to_full(bv, Sb);
        congr_sym6(RRe, Sb, var6);
        const double sigma_l = LioOracle::plane_sigma(pw2, pt.center, pt.normal, pt.plane_var);
        e.idx.push_back(pt.src_index);
        e.r_inv.push_back(1.0 / (sigma_l + LioOracle::quad_sym6(nv, var6)));
        for (int j = 0; j < 3; ++j) e.normal.push_back(nv[j]);
    }
    e.replay_ok = e.idx == o->last_match_idx ? 1 : 0;
    return iters;
}
int orc_eff_replay_ok(void* h) { return g_eff[h].replay_ok; }
// publish_effect_world: m_effct_feat_num rows (0 before any estimation), with the handle's current state.  Any output may be NULL.
int orc_eff_cloud(void* h, float* rows, int* scan_index, double* r_inv, double* normal) {
    const LioOracle* o = (const LioOracle*)h;
    const EffState& e = g_eff[h];
    const int m = (int)e.idx.size();
    for (int k = 0; k < m; ++k) {
        const int i = e.idx[k];
        float row[4];
        rgb_body_to_world(*o, &e.body[(size_t)i * 3], (float)std::sqrt(e.r_inv[k]), row);   // intensity = sqrt(R_inv(i)), :1527
        if (rows) std::memcpy(rows + (size_t)k * 4, row, sizeof(row));
        if (scan_index) scan_index[k] = i;
        if (r_inv) r_inv[k] = e.r_inv[k];
        if (normal) for (int j = 0; j < 3; ++j) normal[(size_t)k * 3 + j] = e.normal[(size_t)k * 3 + j];
    }
    return m;
}
// publish_frame_world: every point of pts ([n][stride], intensity from column intensity_col, 0 when < 0) to the world frame, then
// points 0, skip, 2 skip, ... (the reference's two loops); returns the row count
int orc_frame_world(void* h, const float* pts, int n, int stride, int intensity_col, int point_skip, float* rows) {
    const LioOracle* o = (const LioOracle*)h;
    std::vector<float> world((size_t)n * 4);
    for (int i = 0; i < n; ++i) {
        const float* p = pts + (size_t)i * stride;
        rgb_body_to_world(*o, p, intensity_col >= 0 ? p[intensity_col] : 0.0f, &world[(size_t)i * 4]);
    }
    int m = 0;
    for (int i = 0; i < n; i += point_skip) std::memcpy(rows + (size_t)(m++) * 4, &world[(size_t)i * 4], 4 * sizeof(float));
    return m;
}
// the down-sampled scan of the last estimation (pts == NULL of immesh_lio_registered_cloud)
int orc_eff_scan(void* h, float* body) {
    const EffState& e = g_eff[h];
    if (body) std::memcpy(body, e.body.data(), e.body.size() * sizeof(float));
    return (int)(e.body.size() / 3);
}
void orc_eff_forget(void* h) { g_eff.erase(h); }
}  // extern "C"
