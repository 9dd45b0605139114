// ORACLE EXTENSION (test infrastructure, NOT product code): pubPlaneMap (src/voxel_mapping.cpp:947-1159) on the CPU oracle.
// The oracle's Plane has no m_is_update / m_p_center, so this file keeps them beside the oracle's tree, per node, with the
// reference's semantics (voxel_loc.cpp:111-118, :136): every init_plane sets the flag, a planar one also sets m_p_center to the
// float centre and normal.  The fits are observed, not re-implemented: map growth feeds the oracle's own update_voxel_map ONE
// point at a time, in the order map_incremental_grow gives it, and after each point the point's root voxel is compared with the
// previous look -- a node was fitted exactly when its points_size changed (a refit needs > 5 new points; a first fit goes from 0
// to n > 0).  buildVoxelMap fits every node once, so after voxel_map_init every node with points_size > 0 has its flag set.
// pub_plane_map is the reference's walk over the WHOLE map, with no pending-set bookkeeping (roots in ascending key).
#include "../../oracle/orc_capi.cpp"

#include <unordered_map>

namespace {
struct Pub {
    int seen_points = 0;
    bool is_update = false;
    float p_center[6] = {0, 0, 0, 0, 0, 0};
};
struct PubState {
    std::unordered_map<const OctoTree*, Pub> node;
    std::vector<double> rows;
};
std::unordered_map<void*, PubState> g_state;

void observe(PubState& s, const OctoTree* nd) {
    Pub& p = s.node[nd];
    if (nd->plane.points_size != p.seen_points) {
        p.seen_points = nd->plane.points_size;
        p.is_update = true;
        if (nd->plane.is_plane)
            for (int i = 0; i < 3; ++i) { p.p_center[i] = (float)nd->plane.center[i]; p.p_center[3 + i] = (float)nd->plane.normal[i]; }
    }
    for (const OctoTree* l : nd->leaves)
        if (l) observe(s, l);
}
std::vector<VoxelKey> sorted_keys(const LioOracle& o) {
    std::vector<VoxelKey> keys;
    for (auto& kv : o.feat_map) keys.push_back(kv.first);
    std::sort(keys.begin(), keys.end(), [](const VoxelKey& a, const VoxelKey& b) {
        if (a.x != b.x) return a.x < b.x;
        if (a.y != b.y) return a.y < b.y;
        return a.z < b.z;
    });
    return keys;
}
// one pubPlane call: kx ky kz path layer id(m_id) | p_center xyz normal xyz | radius (the float pubPlane takes) min_eig trace alpha
void row(PubState& s, const VoxelKey& k, const OctoTree* nd, int64_t path, float radius, float alpha) {
    const Plane& p = nd->plane;
    std::vector<double>& out = s.rows;
    out.push_back((double)k.x); out.push_back((double)k.y); out.push_back((double)k.z);
    out.push_back((double)path); out.push_back(nd->layer); out.push_back(p.id);
    for (int i = 0; i < 6; ++i) out.push_back(s.node[nd].p_center[i]);
    out.push_back(radius);
    out.push_back(p.min_eigen_value);
    out.push_back((p.plane_var[pv21_idx(0, 0)] + p.plane_var[pv21_idx(1, 1)]) + p.plane_var[pv21_idx(2, 2)]);   // block<3,3>(0,0).diagonal().sum()
    out.push_back(alpha);
}
}  // namespace

extern "C" {
void orc_pub_map_init(void* h, const float* body, int n) {
    LioOracle* o = (LioOracle*)h;
    o->voxel_map_init(body, n);
    PubState& s = g_state[h];
    for (auto& kv : o->feat_map) observe(s, kv.second);
}
// map_incremental_grow (orc_lio.hpp), the sorted point list handed to update_voxel_map one point at a time
void orc_pub_map_grow(void* h, const float* body, int n) {
    LioOracle* o = (LioOracle*)h;
    PubState& s = g_state[h];
    const State& st = o->state;
    std::vector<PV> pv_list(n);
    double RRe[9];
    mat3_mul(st.rot, o->cfg.extR, RRe);
    for (int i = 0; i < n; ++i) {
        PV& pv = pv_list[i];
        const double pb[3] = {(double)body[i * 3 + 0], (double)body[i * 3 + 1], (double)body[i * 3 + 2]};
        double pw[3];
        o->body_to_world_f(st.rot, st.pos, pb, pw);
        for (int j = 0; j < 3; ++j) { pv.pb[j] = pw[j]; pv.pw[j] = pw[j]; }
        double Sb[9], T1[6], T2[6], C[9], nC[9], rot_var[9];
        sym6_to_full(&o->body_cov[(size_t)i * 6], Sb);
        congr_sym6(RRe, Sb, T1);
        for (int k = 0; k < 9; ++k) { C[k] = o->cross_mat[(size_t)i * 9 + k]; nC[k] = -C[k]; }
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) rot_var[a * 3 + b] = st.cov[a * 18 + b];
        congr_sym6(nC, rot_var, T2);
        for (int a = 0; a < 3; ++a)
            for (int b = a; b < 3; ++b) pv.var[sym6_idx(a, b)] = (T1[sym6_idx(a, b)] + T2[sym6_idx(a, b)]) + st.cov[(3 + a) * 18 + (3 + b)];
    }
    std::vector<std::pair<double, int>> keyed(n);
    for (int i = 0; i < n; ++i) {
        const double* v = pv_list[i].var;
        keyed[i] = {std::sqrt((v[0] * v[0] + v[3] * v[3]) + v[5] * v[5]), i};
    }
    std::sort(keyed.begin(), keyed.end());
    const double vs = (double)(float)o->cfg.voxel_size;
    for (int i = 0; i < n; ++i) {
        const PV& pv = pv_list[keyed[i].second];
        o->update_voxel_map(std::vector<PV>(1, pv));
        observe(s, o->feat_map.at(voxel_key(pv.pb, vs)));
    }
}
// pubPlaneMap over the whole map; returns the number of rows (orc_pub_rows copies them), counts = plane, sub-plane,
// sub-sub-plane, update counts of the reference's log lines (:1154-1158)
long orc_pub_plane_markers(void* h, long* counts) {
    LioOracle* o = (LioOracle*)h;
    PubState& s = g_state[h];
    s.rows.clear();
    long plane_count = 0, sub_plane_count = 0, sub_sub_plane_count = 0, update_count = 0;
    for (const VoxelKey& k : sorted_keys(*o)) {
        OctoTree* t = o->feat_map.at(k);
        if (s.node[t].is_update) {
            row(s, k, t, 0, 1.25 * t->plane.radius, t->plane.is_plane ? 1.0f : 0.0f);
            s.node[t].is_update = false;
            update_count++;
            plane_count++;
        } else {
            for (int i = 0; i < 8; i++) {
                OctoTree* c = t->leaves[i];
                if (c == nullptr) continue;
                if (s.node[c].is_update) {
                    row(s, k, c, i + 1, 1.25 * c->plane.radius, c->plane.is_plane ? 1.0f : 0.0f);
                    s.node[c].is_update = false;
                    update_count++;
                    sub_plane_count++;
                } else {
                    for (int j = 0; j < 8; j++) {
                        OctoTree* g = c->leaves[j];
                        if (g == nullptr) continue;
                        if (g->octo_state == 0 && s.node[g].is_update) {
                            if (g->plane.is_plane) {
                                row(s, k, g, (int64_t)(i + 1) * 9 + (j + 1), g->plane.radius, 1.0f);
                                s.node[g].is_update = false;
                                update_count++;
                            }
                            sub_sub_plane_count++;
                        }
                    }
                }
            }
        }
    }
    counts[0] = plane_count; counts[1] = sub_plane_count; counts[2] = sub_sub_plane_count; counts[3] = update_count;
    return (long)(s.rows.size() / 16);
}
void orc_pub_rows(void* h, double* out) {
    const PubState& s = g_state[h];
    std::memcpy(out, s.rows.data(), s.rows.size() * 8);
}
// per node in orc_lio_dump_map's order (roots by key, pre-order): is_update, octo_state, p_center[6]
long orc_pub_dump(void* h, double* out, long cap_rows) {
    LioOracle* o = (LioOracle*)h;
    PubState& s = g_state[h];
    std::vector<double> d;
    std::vector<const OctoTree*> st;
    for (const VoxelKey& k : sorted_keys(*o)) {
        st.push_back(o->feat_map.at(k));
        while (!st.empty()) {
            const OctoTree* nd = st.back();
            st.pop_back();
            const Pub& p = s.node[nd];
            d.push_back(p.is_update);
            d.push_back(nd->octo_state);
            for (int i = 0; i < 6; ++i) d.push_back(p.p_center[i]);
            for (int l = 7; l >= 0; --l)
                if (nd->leaves[l]) st.push_back(nd->leaves[l]);
        }
    }
    const long rows = (long)(d.size() / 8);
    if (out && rows <= cap_rows) std::memcpy(out, d.data(), d.size() * 8);
    return rows;
}
void orc_pub_forget(void* h) { g_state.erase(h); }
}  // extern "C"
