// TEST INFRASTRUCTURE (not product code): the host emulation of the localization kernels (tests/emu/emu_lio.cpp) with the local
// map's bodies of the CUDA library (immesh_b200/csrc/local_map.cuh): the box rule of k_local_map_box, the eviction sweep of
// k_evict_roots one slot at a time (in a seeded pseudo-random order, as the device's concurrent sweep may visit them), and the
// purge, which rebuilds the root hash at its size through the growth's rehash bodies (pool_growth.cuh).
#include "../emu/emu_lio.cpp"
#include "../../immesh_b200/csrc/pool_growth.cuh"

#include <numeric>
#include <random>
#include <unordered_map>

namespace {
std::unordered_map<immesh_lio*, std::vector<int>> g_free;
unsigned g_seed = 0;
std::vector<unsigned> visit_order(size_t n) {
    std::vector<unsigned> o(n);
    std::iota(o.begin(), o.end(), 0u);
    if (g_seed) std::shuffle(o.begin(), o.end(), std::mt19937(g_seed));
    return o;
}
}  // namespace

extern "C" {
// local_map_rule on a caller-held box: returns the number of removal boxes (rm [3][6]); *placed, box [6] in / out
int emu_lm_rule(double cube_len, float det_range, float mov_threshold, int* placed, float* box, const double* pos, float* rm) {
    LocalMapCtrl L;
    std::memset(&L, 0, sizeof(L));
    L.cube_len = cube_len; L.det_range = det_range; L.mov_threshold = mov_threshold; L.on = 1; L.placed = *placed;
    for (int k = 0; k < 6; ++k) L.box[k] = box[k];
    local_map_rule(L, pos);
    *placed = L.placed;
    for (int k = 0; k < 6; ++k) box[k] = L.box[k];
    for (int b = 0; b < L.n_rm; ++b)
        for (int k = 0; k < 6; ++k) rm[6 * b + k] = L.rm[b][k];
    return L.n_rm;
}
int emu_lm_set_order(unsigned seed) { g_seed = seed; return 0; }
// the node free stack and the tombstone counter wired into the map, as the library does on the first eviction
int emu_lm_enable(immesh_lio_t* h) {
    std::vector<int>& f = g_free[h];
    f.assign(h->nodes.size(), -1);
    h->map.node_free = f.data();
    h->map.node_free_top = &h->counters[IM_LC_NODE_FREE];
    h->map.n_tombs = &h->counters[IM_LC_TOMBS];
    return 0;
}
// k_local_map_box's clamp, then k_evict_roots over every slot: stats = [roots, nodes, chunks]
int emu_lm_evict(immesh_lio_t* h, const float* boxes, int n, long long* stats) {
    if (*h->map.node_free_top < 0) *h->map.node_free_top = 0;
    stats[0] = stats[1] = stats[2] = 0;
    for (unsigned s : visit_order(h->keys.size())) {
        int nn = 0, nc = 0;
        stats[0] += evict_root_slot(h->map, s, boxes, n, &nn, &nc);
        stats[1] += nn;
        stats[2] += nc;
    }
    return 0;
}
// the purge: the root hash rebuilt at its size by rehash_root_slot (tombstones dropped), the node back-pointers remapped
int emu_lm_purge(immesh_lio_t* h) {
    const size_t cap = h->keys.size();
    std::vector<unsigned long long> keys(cap, IM_EMPTY_KEY);
    std::vector<int> roots(cap, -1), slot_map(cap, -1);
    VoxelMapDev nm = h->map;
    nm.keys = keys.data();
    nm.root_node = roots.data();
    for (unsigned s : visit_order(cap)) rehash_root_slot(h->map, nm, s, slot_map.data());
    const int nn = std::min<int>(h->counters[IM_LC_NODES], (int)h->nodes.size());
    for (int i = 0; i < nn; ++i) remap_node_root_slot(nm, i, slot_map.data());
    h->keys = keys;
    h->root_node = roots;
    h->map.keys = h->keys.data();
    h->map.root_node = h->root_node.data();
    h->counters[IM_LC_TOMBS] = 0;
    return 0;
}
// the table: keys [cap] and root ids [cap]; returns cap
long long emu_lm_table(immesh_lio_t* h, unsigned long long* keys, int* roots) {
    if (keys) std::memcpy(keys, h->keys.data(), h->keys.size() * 8);
    if (roots) std::memcpy(roots, h->root_node.data(), h->root_node.size() * 4);
    return (long long)h->keys.size();
}
int emu_lm_find(immesh_lio_t* h, unsigned long long key) { return hash_find(h->map, key); }
int emu_lm_counter(immesh_lio_t* h, int slot) { return h->counters[slot]; }
// every node's root_slot: its root's slot (or -1 for a freed record) -- the back-pointer the growth and the publisher follow
int emu_lm_root_slots(immesh_lio_t* h, int* out) {
    const int nn = std::min<int>(h->counters[IM_LC_NODES], (int)h->nodes.size());
    for (int i = 0; i < nn; ++i) out[i] = h->nodes[i].root_slot;
    return nn;
}
}  // extern "C"
