// ORACLE EXTENSION (test infrastructure, NOT product code): the local map of Voxel_mapping on the CPU oracle.
// laser_map_fov_segment (src/voxel_mapping_common.cpp:214-288) written from the reference's code with its types -- m_cube_len
// double, DETECTION_RANGE / MOV_THRESHOLD float, BoxPointType float, dist_to_map_edge float -- and the deletion of the boxes it
// leaves behind applied to the oracle's feat_map: a root voxel whose voxel centre passes Delete_Point_Boxes' half-open test
// (include/ikd-Tree/ikd_Tree.cpp:826-827) is erased with its tree.  The reference runs this rule only on its ikd-Tree; the library
// applies it to the VoxelMap, and this is the oracle of that.
#include "../../oracle/orc_capi.cpp"

#include <unordered_map>

namespace {
struct BoxPointType { float vertex_min[3], vertex_max[3]; };
struct LocalMap {
    double m_cube_len = 0;
    float DETECTION_RANGE = 300.0f;
    float MOV_THRESHOLD = 1.5f;
    bool m_localmap_Initialized = false;
    BoxPointType m_LocalMap_Points = {};
    std::vector<BoxPointType> m_cub_need_rm;
    long moves = 0;
};
std::unordered_map<void*, LocalMap> g_lm;

// the reference's function body, pos_LiD = state.pos_end
void laser_map_fov_segment(LocalMap& lm, const double* pos_LiD) {
    lm.m_cub_need_rm.clear();
    if (!lm.m_localmap_Initialized) {
        for (int i = 0; i < 3; i++) {
            lm.m_LocalMap_Points.vertex_min[i] = pos_LiD[i] - lm.m_cube_len / 2.0;
            lm.m_LocalMap_Points.vertex_max[i] = pos_LiD[i] + lm.m_cube_len / 2.0;
        }
        lm.m_localmap_Initialized = true;
        return;
    }
    const float MOV_THRESHOLD = lm.MOV_THRESHOLD, DETECTION_RANGE = lm.DETECTION_RANGE;
    float dist_to_map_edge[3][2];
    bool need_move = false;
    for (int i = 0; i < 3; i++) {
        dist_to_map_edge[i][0] = fabs(pos_LiD[i] - lm.m_LocalMap_Points.vertex_min[i]);
        dist_to_map_edge[i][1] = fabs(pos_LiD[i] - lm.m_LocalMap_Points.vertex_max[i]);
        if (dist_to_map_edge[i][0] <= MOV_THRESHOLD * DETECTION_RANGE || dist_to_map_edge[i][1] <= MOV_THRESHOLD * DETECTION_RANGE) need_move = true;
    }
    if (!need_move) return;
    BoxPointType New_LocalMap_Points, tmp_boxpoints;
    New_LocalMap_Points = lm.m_LocalMap_Points;
    float mov_dist = std::max((lm.m_cube_len - 2.0 * MOV_THRESHOLD * DETECTION_RANGE) * 0.5 * 0.9, double(DETECTION_RANGE * (MOV_THRESHOLD - 1)));
    for (int i = 0; i < 3; i++) {
        tmp_boxpoints = lm.m_LocalMap_Points;
        if (dist_to_map_edge[i][0] <= MOV_THRESHOLD * DETECTION_RANGE) {
            New_LocalMap_Points.vertex_max[i] -= mov_dist;
            New_LocalMap_Points.vertex_min[i] -= mov_dist;
            tmp_boxpoints.vertex_min[i] = lm.m_LocalMap_Points.vertex_max[i] - mov_dist;
            lm.m_cub_need_rm.push_back(tmp_boxpoints);
        } else if (dist_to_map_edge[i][1] <= MOV_THRESHOLD * DETECTION_RANGE) {
            New_LocalMap_Points.vertex_max[i] += mov_dist;
            New_LocalMap_Points.vertex_min[i] += mov_dist;
            tmp_boxpoints.vertex_max[i] = lm.m_LocalMap_Points.vertex_min[i] + mov_dist;
            lm.m_cub_need_rm.push_back(tmp_boxpoints);
        }
    }
    lm.m_LocalMap_Points = New_LocalMap_Points;
    ++lm.moves;
}

bool in_box(const BoxPointType& b, const double* c) {
    return b.vertex_min[0] <= c[0] && b.vertex_max[0] > c[0] && b.vertex_min[1] <= c[1] && b.vertex_max[1] > c[1] && b.vertex_min[2] <= c[2] &&
           b.vertex_max[2] > c[2];
}
long delete_boxes(LioOracle* o, const std::vector<BoxPointType>& boxes) {
    long n = 0;
    for (auto it = o->feat_map.begin(); it != o->feat_map.end();) {
        bool hit = false;
        for (const auto& b : boxes) hit = hit || in_box(b, it->second->voxel_center);
        if (hit) {
            delete it->second;
            it = o->feat_map.erase(it);
            ++n;
        } else {
            ++it;
        }
    }
    return n;
}
void to_rows(const std::vector<BoxPointType>& v, float* rows) {
    for (size_t k = 0; k < v.size(); ++k)
        for (int i = 0; i < 3; ++i) { rows[6 * k + i] = v[k].vertex_min[i]; rows[6 * k + 3 + i] = v[k].vertex_max[i]; }
}
}  // namespace

extern "C" {
void orc_lm_set(void* h, double cube_len, float det_range, float mov_threshold) {
    LocalMap& lm = g_lm[h];
    lm = LocalMap();
    lm.m_cube_len = cube_len; lm.DETECTION_RANGE = det_range; lm.MOV_THRESHOLD = mov_threshold;
}
// the rule at the oracle's pos_end and the deletion of its boxes: returns the number of boxes (written to rm [3][6]); box [6], *evicted
int orc_lm_segment(void* h, float* box, float* rm, long* evicted) {
    LocalMap& lm = g_lm[h];
    LioOracle* o = (LioOracle*)h;
    laser_map_fov_segment(lm, o->state.pos);
    to_rows({lm.m_LocalMap_Points}, box);
    to_rows(lm.m_cub_need_rm, rm);
    *evicted = lm.m_cub_need_rm.empty() ? 0 : delete_boxes(o, lm.m_cub_need_rm);
    return (int)lm.m_cub_need_rm.size();
}
long orc_lio_evict_boxes(void* h, const float* rows, int n) {
    std::vector<BoxPointType> v(n);
    for (int k = 0; k < n; ++k)
        for (int i = 0; i < 3; ++i) { v[k].vertex_min[i] = rows[6 * k + i]; v[k].vertex_max[i] = rows[6 * k + 3 + i]; }
    return delete_boxes((LioOracle*)h, v);
}
// the rule alone on a caller-held box: placed / box in-out, returns the number of removal boxes (rm [3][6])
int orc_lm_rule(double cube_len, float det_range, float mov_threshold, int* placed, float* box, const double* pos, float* rm) {
    LocalMap lm;
    lm.m_cube_len = cube_len; lm.DETECTION_RANGE = det_range; lm.MOV_THRESHOLD = mov_threshold;
    lm.m_localmap_Initialized = *placed != 0;
    for (int i = 0; i < 3; ++i) { lm.m_LocalMap_Points.vertex_min[i] = box[i]; lm.m_LocalMap_Points.vertex_max[i] = box[3 + i]; }
    laser_map_fov_segment(lm, pos);
    *placed = 1;
    to_rows({lm.m_LocalMap_Points}, box);
    to_rows(lm.m_cub_need_rm, rm);
    return (int)lm.m_cub_need_rm.size();
}
}  // extern "C"
