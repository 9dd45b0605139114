// immesh_b200 -- local map of the device VoxelMap (immesh_lio_local_map / immesh_voxelmap_evict_boxes): a cube that follows the
// sensor, and the eviction of the root voxels it leaves behind.  Bodies shared by the CUDA kernels (lio_capi.cu: k_local_map_box,
// k_evict_roots) and the host emulation of the tests.
//
// Box rule: Voxel_mapping::laser_map_fov_segment (src/voxel_mapping_common.cpp:214-288) in the reference's own types -- the pose
// pos_end is double, the box vertex_min / vertex_max is float (BoxPointType), dist_to_map_edge is float, the threshold is
// MOV_THRESHOLD * DETECTION_RANGE in float, and mov_dist = (float)max((cube_len - 2.0 mov det) * 0.5 * 0.9, (double)(det (mov - 1)))
// (:256).  The first evaluation only places the box around the pose (:227-239).  Each later evaluation that moves the box removes,
// for every axis that moved, the old box with that axis narrowed to the slab it gave up (:257-278): at most three removal boxes.
//
// Eviction: a root voxel whose centre (NodeRec::vc of the root, double) lies in a removal box, tested half-open with the float edges
// widened to double as ikd-Tree's Delete_Point_Boxes does (include/ikd-Tree/ikd_Tree.cpp:826-827: min <= c < max), is removed with
// its whole octree: every node's chunks go through node_free_points (the pending list, recycled at the end of the scan), every node
// id goes onto the node free stack that alloc_node pops before it bumps, and the slot becomes a tombstone (IM_TOMB_KEY,
// root_node = -1, pub_mark cleared).  hash_find and hash_insert step over a tombstone as over any other key, so a root created again
// later takes a fresh slot and is a fresh root, exactly as on its first visit.  Tombstones leave the table when it is rebuilt
// (rehash_root_slot skips them): by a growth of the root hash, or by the purge that rebuilds it at the same capacity once they
// exceed an eighth of the slots.
#pragma once
#include "voxelmap.cuh"

namespace immesh {

#define IM_LM_MAX_BOXES 3

// the local map's device state, in LioCtrl (written by the host only while the handle is drained)
struct LocalMapCtrl {
    double cube_len;            // cube_side_length
    float det_range;            // DETECTION_RANGE
    float mov_threshold;        // MOV_THRESHOLD
    int on;                     // the automatic rule is evaluated once per scan (k_local_map_box)
    int placed;                 // m_localmap_Initialized
    float box[6];               // m_LocalMap_Points: vertex_min xyz, vertex_max xyz
    float rm[IM_LM_MAX_BOXES][6];   // m_cub_need_rm of this scan's evaluation
    int n_rm;                   // its size (0: k_evict_roots exits at once)
    int pad_;
    unsigned long long moves;   // evaluations that moved the box
    unsigned long long roots;   // root voxels evicted
    unsigned long long nodes;   // node records freed
    unsigned long long chunks;  // point chunks freed
};

// laser_map_fov_segment at pos_end `pos`: places or moves L.box and writes the removal boxes of this evaluation into L.rm / L.n_rm
IM_HD void local_map_rule(LocalMapCtrl& L, const double* pos) {
    L.n_rm = 0;
    if (!L.placed) {
        for (int i = 0; i < 3; ++i) {
            L.box[i] = (float)(pos[i] - L.cube_len / 2.0);
            L.box[3 + i] = (float)(pos[i] + L.cube_len / 2.0);
        }
        L.placed = 1;
        return;
    }
    const float thr = L.mov_threshold * L.det_range;
    float dist[3][2];
    bool need_move = false;
    for (int i = 0; i < 3; ++i) {
        dist[i][0] = (float)fabs(pos[i] - (double)L.box[i]);
        dist[i][1] = (float)fabs(pos[i] - (double)L.box[3 + i]);
        if (dist[i][0] <= thr || dist[i][1] <= thr) need_move = true;
    }
    if (!need_move) return;
    const double a = (L.cube_len - 2.0 * (double)L.mov_threshold * (double)L.det_range) * 0.5 * 0.9;
    const double b = (double)(L.det_range * (L.mov_threshold - 1));
    const float mov_dist = (float)(a < b ? b : a);   // std::max(a, b)
    float nb[6];
    for (int k = 0; k < 6; ++k) nb[k] = L.box[k];
    for (int i = 0; i < 3; ++i) {
        float tmp[6];
        for (int k = 0; k < 6; ++k) tmp[k] = L.box[k];
        if (dist[i][0] <= thr) {
            nb[3 + i] -= mov_dist;
            nb[i] -= mov_dist;
            tmp[i] = L.box[3 + i] - mov_dist;
        } else if (dist[i][1] <= thr) {
            nb[3 + i] += mov_dist;
            nb[i] += mov_dist;
            tmp[3 + i] = L.box[i] + mov_dist;
        } else {
            continue;
        }
        for (int k = 0; k < 6; ++k) L.rm[L.n_rm][k] = tmp[k];
        ++L.n_rm;
    }
    for (int k = 0; k < 6; ++k) L.box[k] = nb[k];
    L.moves += 1;
}

// Delete_Point_Boxes' test of one point against one box (ikd_Tree.cpp:826-827), the float edges widened to double
IM_HD bool local_map_in_box(const double* c, const float* b) {
    return (double)b[0] <= c[0] && (double)b[3] > c[0] && (double)b[1] <= c[1] && (double)b[4] > c[1] && (double)b[2] <= c[2] && (double)b[5] > c[2];
}

// deepest octree under a root: max_layer <= 4 (immesh_lio_create), so a depth-first walk holds at most 1 + 4 x 7 + 8 ids
#define IM_LM_STACK 40

// slot s against the removal boxes: evicts its root when the root's centre lies in one.  Returns 1 when it did, and the node records
// and chunks it freed through *nodes / *chunks.
IM_HD int evict_root_slot(const VoxelMapDev& m, unsigned int s, const float* boxes, int n_boxes, int* nodes, int* chunks) {
    *nodes = 0;
    *chunks = 0;
    if (m.keys[s] >> 63) return 0;   // empty or tombstone
    const int root = m.root_node[s];
    if (root < 0) return 0;
    bool hit = false;
    for (int b = 0; b < n_boxes && !hit; ++b) hit = local_map_in_box(m.nodes[root].vc, boxes + 6 * b);
    if (!hit) return 0;
    int stack[IM_LM_STACK];
    int top = 0;
    stack[top++] = root;
    while (top > 0) {
        const int nd = stack[--top];
        for (int c = 0; c < 8; ++c) {
            const int ch = m.nodes[nd].children[c];
            if (ch >= 0 && top < IM_LM_STACK) stack[top++] = ch;
        }
        *chunks += node_free_points(m, nd);
        const int i = im_atomic_add(m.node_free_top, 1);
        m.node_free[i] = nd;
        ++*nodes;
    }
    m.root_node[s] = -1;
    m.keys[s] = IM_TOMB_KEY;
    if (m.pub_mark) m.pub_mark[s] = 0;
    im_atomic_add(m.n_roots, -1);
    im_atomic_add(m.n_tombs, 1);
    return 1;
}

}  // namespace immesh
