// immesh_b200 -- migration bodies of a VoxelMap growth (immesh_lio_reserve), shared by the CUDA kernels (lio_capi.cu) and the
// host emulation of the tests.
//
// The node, plane, PubRec and chunk pools are copied as they are: their indices are stored elsewhere (children, chunk lists,
// match_node, avail / pending) and stay valid.  The root hash is rebuilt into a larger table: every occupied slot is inserted
// again by its key, its root_node and pub_mark move with it, and the two back-pointers to slots -- NodeRec::root_slot and the
// pub_list entries -- are rewritten through the old-slot -> new-slot map the rebuild leaves behind.
//
// Slot placement after a concurrent rebuild depends on the order of the inserts, exactly as it does for the inserts of a step
// (grow_point).  No output of the library depends on it: the map dump and the plane markers are ordered by root key, and the
// match and update walks reach a root through its key.
#pragma once
#include "lio_core.cuh"
#include "mesh_core.cuh"

namespace immesh {

// old slot s of `from` into `to`; slot_map[s] = its new slot (-1: empty, or `to` full, with IM_ERR_HASH_FULL raised)
IM_HD void rehash_root_slot(const VoxelMapDev& from, const VoxelMapDev& to, unsigned int s, int* slot_map) {
    const unsigned long long key = from.keys[s];
    if (key >> 63) { slot_map[s] = -1; return; }   // empty, or a tombstone of the local map (dropped)
    int created = 0;
    const int ns = hash_insert(to, key, &created);
    slot_map[s] = ns;
    if (ns < 0) return;
    to.root_node[ns] = from.root_node[s];
    if (to.pub_mark) to.pub_mark[ns] = from.pub_mark[s];
}
// node nd of the (copied) pool in `to`: its root's slot in the rebuilt table
IM_HD void remap_node_root_slot(const VoxelMapDev& to, int nd, const int* slot_map) {
    NodeRec& n = to.nodes[nd];
    if (n.root_slot >= 0) n.root_slot = slot_map[n.root_slot];   // < 0: a record freed with an evicted root
}
// entry i of the plane-map publisher's pending list
IM_HD void remap_pub_entry(const int* from_list, const VoxelMapDev& to, int i, const int* slot_map) {
    to.pub_list[i] = slot_map[from_list[i]];
}

// ---- the mesh handle (immesh_mesh_reserve).  Vertex, vertex-chunk and triangle records are copied as they are; the three open-
// addressed tables are rebuilt into tables of the new size.
// xi-grid: old slot s (cell key -> vertex id) into `to`
IM_HD void rehash_xi_slot(const MeshDev& from, const MeshDev& to, unsigned int s) {
    const unsigned long long key = from.gkeys[s];
    if (key == IM_EMPTY_KEY) return;
    int created = 0;
    const int ns = table_insert(to.gkeys, to.gmask, key, &created);
    if (ns < 0) { im_atomic_or(&to.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); return; }
    to.gval[ns] = from.gval[s];
}
// mesh-voxel hash: the slot IS the voxel id, so every per-voxel array row moves with its key
IM_HD void rehash_voxel_slot(const MeshDev& from, const MeshDev& to, unsigned int s) {
    const unsigned long long key = from.vkeys[s];
    if (key == IM_EMPTY_KEY) return;
    int created = 0;
    const int ns = table_insert(to.vkeys, to.vmask, key, &created);
    if (ns < 0) { im_atomic_or(&to.cnt[IM_MC_ERR], IM_MERR_HASH_FULL); return; }
    for (int k = 0; k < IM_VCHUNKS; ++k) to.vox_chunk[(size_t)ns * IM_VCHUNKS + k] = from.vox_chunk[(size_t)s * IM_VCHUNKS + k];
    to.vox_count[ns] = from.vox_count[s];
    to.vox_meshing_times[ns] = from.vox_meshing_times[s];
    to.vox_new_added[ns] = from.vox_new_added[s];
    to.vox_frame[ns] = from.vox_frame[s];
}
// triangle triple hash: every index the old table holds -- every triple ever published, live or not, so that a re-added triple
// keeps reusing its record (tri_add) -- inserted by its triple; `to.tri` holds the records (copied first)
IM_HD void rehash_tri_slot(const MeshDev& from, const MeshDev& to, unsigned int s) {
    const int t = from.thash[s];
    if (t < 0) return;
    const int4 r = to.tri[t];
    unsigned int p = tri_hash(r.x, r.y, r.z) & to.tmask;
    for (unsigned int probe = 0; probe <= to.tmask; ++probe) {
        if (im_atomic_cas32(&to.thash[p], -1, t) < 0) return;
        p = (p + 1) & to.tmask;
    }
    im_atomic_or(&to.cnt[IM_MC_ERR], IM_MERR_HASH_FULL);
}

// Automatic growth (immesh_lio_set_growth): the capacities the next `steps` steps need (the steps still in flight and the one
// being queued), each of at most n_max points, from the counters c (IM_LC_* slots) of the last step known to have finished.
// *cap, *nodes, *chunks hold the current capacities on entry; a pool is doubled until
//   root hash : load factor <= 1/2 after the steps, each adding at most n_max roots (one per point at most: a sound bound); the
//               local map's tombstones count as occupied slots
//   nodes     : free >= max(capacity / 4, steps x max(2 x the largest per-step use seen, n_max)), with nodes in use =
//               node_count - the records on the local map's node free stack
//   chunks    : the same, with chunks in use = chunk_bump - avail_top
// The node and chunk bounds are not sound (a plane fit that splits a node redistributes its points): a step that overflows anyway
// returns IMMESH_E_CAPACITY as it does without growth.
inline void growth_targets(const int* c, long long steps, long long n_max, int max_step_nodes, int max_step_chunks, long long* cap,
                           long long* nodes, long long* chunks) {
    while (((long long)c[IM_LC_ROOTS] + c[IM_LC_TOMBS] + steps * n_max) * 2 > *cap) *cap *= 2;
    const long long per_node = 2LL * max_step_nodes > n_max ? 2LL * max_step_nodes : n_max;
    const long long per_chunk = 2LL * max_step_chunks > n_max ? 2LL * max_step_chunks : n_max;
    const long long used_chunks = (long long)c[IM_LC_CHUNK_BUMP] - (c[IM_LC_AVAIL_TOP] > 0 ? c[IM_LC_AVAIL_TOP] : 0);
    auto need = [&](long long capacity, long long used, long long per) {
        const long long q = capacity / 4;
        return capacity - used < (q > steps * per ? q : steps * per);
    };
    const long long used_nodes = (long long)c[IM_LC_NODES] - (c[IM_LC_NODE_FREE] > 0 ? c[IM_LC_NODE_FREE] : 0);
    while (need(*nodes, used_nodes, per_node)) *nodes *= 2;
    while (need(*chunks, used_chunks, per_chunk)) *chunks *= 2;
}

// Automatic growth of the mesh handle (immesh_mesh_set_growth), the same scheme before a frame of at most m candidates: a frame
// appends at most m vertices, xi-cells, mesh voxels and vertex chunks (one per candidate at most: sound bounds); its facets are
// bounded by twice the largest per-frame use seen, and by 8 m (neither is sound).  c: the mesh counters (IM_MC_* slots) of the last frame known to have
// finished; *vertices, *triangles, *voxels hold the current capacities on entry and are doubled until
//   vertices, voxels : free >= max(capacity / 4, steps x m), for the vertices and for the vertex chunks that come with them   (the xi-grid and the voxel hash keep a load factor <= 1/2: they are
//                      sized at twice these capacities)
//   triangles        : free >= max(capacity / 4, steps x max(2 x the largest per-frame use seen, 8 m))
inline void mesh_growth_targets(const int* c, long long steps, long long m, int max_step_tris, long long* vertices, long long* triangles,
                                long long* voxels) {
    auto need = [&](long long capacity, long long used, long long per) {
        const long long q = capacity / 4;
        return capacity - used < (q > steps * per ? q : steps * per);
    };
    const long long per_tri = 2LL * max_step_tris > 8 * m ? 2LL * max_step_tris : 8 * m;
    while (need(*vertices, c[IM_MC_VERTICES], m) || need(*vertices / 4 + 1024, c[IM_MC_VERT_CHUNKS], m)) *vertices *= 2;   // vertex chunks: max_v / 4 + 1024
    while (need(*voxels, c[IM_MC_VOXELS], m)) *voxels *= 2;
    while (need(*triangles, c[IM_MC_TRIS_ALLOC], per_tri)) *triangles *= 2;
}

}  // namespace immesh
