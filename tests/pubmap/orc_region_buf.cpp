// ORACLE EXTENSION (test infrastructure, NOT product code): the mesh viewer's region buffers -- synchronize_triangle_list_for_disp
// -> unparse_triangle_set_to_vector + get_axis_min_max (src/meshing/mesh_rec_display.cpp:78-137, :220-258) -- on the CPU oracle,
// which it does not change.  It keeps RGB_pts::m_smoothed beside the oracle's vsmooth:
//   * a frame's new vertices start clear;
//   * the in-voxel vertices of every voxel the frame meshed are set: retrieve_neighbor_pts_kdtree (mesh_rec_geometry.cpp:336-377)
//     calls set_smooth_pos on each of them.  Which voxels were meshed is read from the oracle's own voxel records: the frame's
//     activation test (ImMesh_mesh_reconstruction.cpp:132-151) is evaluated on their state before the frame plus the vertices
//     the frame appended to them;
//   * smooth_all_pts sets all of them.
// The walk itself is the reference's, literally: regions in order, triangles in order, a vertex with the flag clear smoothed by
// Global_map::smooth_pts (pointcloud_rgbd.cpp:932-958) on the oracle's kNN, rows from the smoothed positions, the axis box with
// the strict comparisons, one region after the other.
#include "../../oracle/orc_capi.cpp"

#include <unordered_map>

namespace {
std::unordered_map<void*, std::vector<char>> g_flag;

// Global_map::smooth_pts(pt, smooth_factor, knn, maximum_smooth_dis), literally
void smooth_pts(MeshOracle* m, int v, double smooth_factor, int knn, double maximum_smooth_dis) {
    std::vector<std::pair<float, int>> nn;
    const float q[3] = {m->vpos[v][0], m->vpos[v][1], m->vpos[v][2]};
    m->knn(q, knn, std::numeric_limits<double>::infinity(), nn);
    const double pt_vec[3] = {(double)m->vpos[v][0], (double)m->vpos[v][1], (double)m->vpos[v][2]};
    double nb[3] = {0, 0, 0};
    double valid_size = 0.0;
    const int size = (int)nn.size();
    for (int k = 1; k < size; k++) {
        if (std::sqrt(nn[k].first) < maximum_smooth_dis) {
            for (int j = 0; j < 3; ++j) nb[j] += (double)m->vpos[nn[k].second][j];
            valid_size += 1.0;
        }
    }
    for (int j = 0; j < 3; ++j) m->vsmooth[v][j] = pt_vec[j] * (1.0 - smooth_factor) + nb[j] * smooth_factor / valid_size;
    g_flag[m][v] = 1;   // set_smooth_pos
}
}  // namespace

extern "C" {
void orc_view_push_frame(void* h, const float* pts, int n, const double* pose_t) {
    MeshOracle* m = (MeshOracle*)h;
    const size_t nvox0 = m->voxels.size();
    std::vector<long> mt0(nvox0), na0(nvox0);
    std::vector<size_t> np0(nvox0);
    for (size_t i = 0; i < nvox0; ++i) { mt0[i] = m->voxels[i].meshing_times; na0[i] = m->voxels[i].new_added; np0[i] = m->voxels[i].pts.size(); }
    m->push_frame(pts, n, pose_t);
    std::vector<char>& f = g_flag[h];
    f.resize(m->vpos.size(), 0);
    for (int vi : m->activated) {
        const auto& vx = m->voxels[vi];
        const bool old = (size_t)vi < nvox0;
        const long added = (long)vx.pts.size() - (long)(old ? np0[vi] : 0);
        const long mt = added > 0 ? 0 : (old ? mt0[vi] : 0);   // append_points_to_global_map resets m_meshing_times on a new vertex
        const long na = (old ? na0[vi] : 0) + added;
        if (mt >= 1 || na < 0 || vx.pts.size() < 3) continue;
        for (int v : vx.pts) f[v] = 1;
    }
}
void orc_view_smooth_all(void* h, double smooth_factor, int knn, double* out) {
    orc_mesh_smooth_all(h, smooth_factor, knn, out);
    std::vector<char>& f = g_flag[h];
    f.assign(((MeshOracle*)h)->vpos.size(), 1);
}
int orc_view_flags(void* h, unsigned char* out) {
    const std::vector<char>& f = g_flag[h];
    for (size_t i = 0; i < f.size(); ++i) out[i] = (unsigned char)f[i];
    return (int)f.size();
}
// keys == NULL: every region in ascending key order, else the listed ones in that order.  Outputs sized by the caller for all live
// triangles and nk (or n_live) + 1 regions.  Returns the row count; *n_regions, *n_smoothed.
int orc_view_region_buffers(void* h, double region_size, const int* keys, int nk, double smooth_factor, int knn, float* xyz, int* ids, int* rkeys,
                            int* roff, float* axis_min_max, int* n_regions, int* n_smoothed) {
    MeshOracle* m = (MeshOracle*)h;
    std::vector<char>& f = g_flag[h];
    f.resize(m->vpos.size(), 0);
    const double accept = m->cfg.voxel_resolution * 1.25;   // g_kd_tree_accept_pt_dis
    std::map<std::array<int, 3>, std::vector<Tri>> sets;
    std::vector<std::array<int, 3>> tk;
    m->region_keys(region_size, tk);
    size_t i = 0;
    for (const Tri& t : m->live) sets[tk[i++]].push_back(t);
    std::vector<std::array<int, 3>> order;
    if (keys) for (int r = 0; r < nk; ++r) order.push_back({keys[3 * r], keys[3 * r + 1], keys[3 * r + 2]});
    else for (auto& kv : sets) order.push_back(kv.first);
    int row = 0, smoothed = 0;
    for (size_t r = 0; r < order.size(); ++r) {
        for (int j = 0; j < 3; ++j) rkeys[r * 3 + j] = order[r][j];
        roff[r] = row;
        auto it = sets.find(order[r]);
        if (it == sets.end()) continue;
        std::vector<std::array<float, 3>> vec;   // m_triangle_pt_vec of the region
        for (const Tri& t : it->second) {
            for (int p = 0; p < 3; ++p)
                if (!f[t[p]]) { smooth_pts(m, t[p], smooth_factor, knn, accept); ++smoothed; }
            for (int p = 0; p < 3; ++p) vec.push_back({(float)m->vsmooth[t[p]][0], (float)m->vsmooth[t[p]][1], (float)m->vsmooth[t[p]][2]});
            for (int p = 0; p < 3; ++p) ids[(size_t)row * 3 + p] = t[p];
            ++row;
        }
        std::memcpy(xyz + ((size_t)row - it->second.size()) * 9, vec.data(), vec.size() * 3 * sizeof(float));
        if (axis_min_max)   // get_axis_min_max
            for (const auto& v : vec)
                for (int a = 0; a < 3; ++a) {
                    if (axis_min_max[a] > v[a]) axis_min_max[a] = v[a];
                    if (axis_min_max[3 + a] < v[a]) axis_min_max[3 + a] = v[a];
                }
    }
    roff[order.size()] = row;
    *n_regions = (int)order.size();
    *n_smoothed = smoothed;
    return row;
}
}  // extern "C"
