// TEST INFRASTRUCTURE (not product code): the host emulation of the localization kernels with the plane-map publisher's state
// (tests/pubmap/emu_pub.cpp), plus immesh_lio_reserve / immesh_lio_capacity running the migration bodies of the CUDA library
// (immesh_b200/csrc/pool_growth.cuh) one slot / node at a time, and immesh_lio_set_growth with the library's policy
// (growth_targets) checked before every map insert.  The old slots are visited in a seeded pseudo-random order, so
// that the rebuilt table's placement differs from an ascending rebuild the way a concurrent one on the device does.
#define immesh_voxelmap_build emu_base_voxelmap_build
#define immesh_voxelmap_update emu_base_voxelmap_update
#include "../pubmap/emu_pub.cpp"
#undef immesh_voxelmap_build
#undef immesh_voxelmap_update
#include "../../immesh_b200/csrc/pool_growth.cuh"

#include <numeric>
#include <random>

namespace {
unsigned g_order_seed = 0;
long long g_growths = 0;

std::vector<unsigned> visit_order(size_t n) {
    std::vector<unsigned> o(n);
    std::iota(o.begin(), o.end(), 0u);
    if (g_order_seed) std::shuffle(o.begin(), o.end(), std::mt19937(g_order_seed));
    return o;
}
// root hash of `cap` slots rebuilt from m (cap > the current one); slot_map filled; the caller owns the new arrays
void rebuild_roots(const VoxelMapDev& m, VoxelMapDev& nm, size_t cap0, std::vector<int>& slot_map, int n_nodes, const int* old_list, int n_pub) {
    slot_map.assign(cap0, -1);
    for (unsigned s : visit_order(cap0)) rehash_root_slot(m, nm, s, slot_map.data());
    for (int i = 0; i < n_nodes; ++i) remap_node_root_slot(nm, i, slot_map.data());
    for (int i = 0; i < n_pub; ++i) remap_pub_entry(old_list, nm, i, slot_map.data());
}
struct GrowState {
    int64_t max_bytes = 0;
    int known[IM_LC_SIZE] = {};
    int max_step_nodes = 0, max_step_chunks = 0;
};
std::unordered_map<immesh_lio*, GrowState> g_grow;
}  // namespace

extern "C" {
int emu_growth_set_order(unsigned seed) { g_order_seed = seed; return 0; }
int immesh_lio_reserve(immesh_lio_t* h, int64_t root_slots, int64_t nodes, int64_t chunks);

int immesh_lio_set_growth(immesh_lio_t* h, int64_t max_bytes) { g_grow[h].max_bytes = max_bytes; return 0; }
// the library's check before a step of n points, on the emulation's (always exact) counters
static int growth_check(immesh_lio* h, long long n) {
    auto it = g_grow.find(h);
    if (it == g_grow.end() || it->second.max_bytes <= 0) return 0;
    GrowState& g = it->second;
    const int* c = h->counters;
    g.max_step_nodes = std::max(g.max_step_nodes, c[IM_LC_NODES] - g.known[IM_LC_NODES]);
    g.max_step_chunks = std::max(g.max_step_chunks, c[IM_LC_CHUNK_BUMP] - g.known[IM_LC_CHUNK_BUMP]);
    std::memcpy(g.known, c, sizeof(g.known));
    long long cap = (long long)h->keys.size(), nodes = (long long)h->nodes.size(), chunks = (long long)h->chunks.size();
    growth_targets(g.known, 1, n, g.max_step_nodes, g.max_step_chunks, &cap, &nodes, &chunks);
    return immesh_lio_reserve(h, cap, nodes, chunks);
}
int immesh_voxelmap_build(immesh_lio_t* h, const float* body, int n) {
    const int rc = growth_check(h, n);
    return rc ? rc : emu_base_voxelmap_build(h, body, n);
}
int immesh_voxelmap_update(immesh_lio_t* h) {
    const int rc = growth_check(h, h->sb.n);
    return rc ? rc : emu_base_voxelmap_update(h);
}

int immesh_lio_reserve(immesh_lio_t* h, int64_t root_slots, int64_t nodes, int64_t chunks) {
    PubStore* ps = g_pub[h];
    VoxelMapDev& m = h->map;
    const size_t cap0 = h->keys.size();
    size_t cap = cap0;
    while ((int64_t)cap < root_slots) cap *= 2;
    bool grew = false;
    if (nodes > (int64_t)h->nodes.size()) {
        h->nodes.resize(nodes); h->planes.resize(nodes); ps->pub.resize(nodes);
        grew = true;
    }
    if (chunks > (int64_t)h->chunks.size()) {
        h->chunks.resize(chunks); h->avail.resize(chunks); h->pending.resize(chunks);
        grew = true;
    }
    m.nodes = h->nodes.data(); m.planes = h->planes.data(); m.pub = ps->pub.data(); m.max_nodes = (int)h->nodes.size();
    m.chunks = h->chunks.data(); m.avail = h->avail.data(); m.pending = h->pending.data(); m.max_chunks = (int)h->chunks.size();
    if (cap > cap0) {
        std::vector<unsigned long long> keys(cap, IM_EMPTY_KEY);
        std::vector<int> root(cap, -1), mark(cap, 0), list(cap, 0), slot_map;
        VoxelMapDev nm = m;
        nm.keys = keys.data(); nm.root_node = root.data(); nm.pub_mark = mark.data(); nm.pub_list = list.data(); nm.cap_mask = (unsigned)(cap - 1);
        rebuild_roots(m, nm, cap0, slot_map, std::min(*m.node_count, m.max_nodes), ps->list.data(), *m.pub_n);
        h->keys.swap(keys); h->root_node.swap(root); ps->mark.swap(mark); ps->list.swap(list);
        h->slot_count.assign(cap, 0); h->slot_offset.assign(cap, 0); h->slot_cursor.assign(cap, 0);
        m = nm;
        m.keys = h->keys.data(); m.root_node = h->root_node.data(); m.pub_mark = ps->mark.data(); m.pub_list = ps->list.data();
        h->sb.slot_count = h->slot_count.data(); h->sb.slot_offset = h->slot_offset.data(); h->sb.slot_cursor = h->slot_cursor.data();
        grew = true;
    }
    if (grew) ++g_growths;
    return 0;
}
int immesh_lio_capacity(immesh_lio_t* h, int64_t* out) {
    const int* c = h->counters;
    out[0] = (int64_t)h->keys.size(); out[1] = c[IM_LC_ROOTS];
    out[2] = (int64_t)h->nodes.size(); out[3] = c[IM_LC_NODES];
    out[4] = (int64_t)h->chunks.size(); out[5] = (int64_t)c[IM_LC_CHUNK_BUMP] - std::max(c[IM_LC_AVAIL_TOP], 0);
    out[6] = 0; out[7] = g_growths;
    return 0;
}

// the two growth policies of the library (pool_growth.cuh), with any number of steps in flight: caps = {cap, nodes, chunks} or
// {vertices, triangles, voxels} in, grown capacities out
int emu_growth_targets(const int* c, long long steps, long long n, int max_a, int max_b, long long* caps) {
    growth_targets(c, steps, n, max_a, max_b, &caps[0], &caps[1], &caps[2]);
    return 0;
}
int emu_mesh_growth_targets(const int* c, long long steps, long long m, int max_tris, long long* caps) {
    mesh_growth_targets(c, steps, m, max_tris, &caps[0], &caps[1], &caps[2]);
    return 0;
}

int emu_hash_home(unsigned long long key, int log2_cap) { return (int)(hash_key(key) & ((1u << log2_cap) - 1u)); }

// A table of 2^log2_old slots filled from keys[n] in order: slot of key i holds root_node i and pub_mark marks[i]; node record i
// has root_slot = that slot; pub_list = the slots of the marked keys, listed in key index order.  The table is rebuilt into
// 2^log2_new slots with the migration bodies, then every key is looked up in the new table with hash_find:
//   out_slot[i] (-1: not found), out_root[i] / out_mark[i] = what that slot holds, out_node_slot[i] = node i's root_slot,
//   out_list[j] = pub_list entry j, list_key[j] = the key index that entry held before.  Returns the number of list entries.
int emu_rehash_check(const unsigned long long* keys, const int* marks, int n, int log2_old, int log2_new, int* out_slot, int* out_root,
                     int* out_mark, int* out_node_slot, int* out_list, int* list_key) {
    const size_t cap0 = (size_t)1 << log2_old, cap = (size_t)1 << log2_new;
    int counters[IM_LC_SIZE] = {};
    std::vector<unsigned long long> k0(cap0, IM_EMPTY_KEY), k1(cap, IM_EMPTY_KEY);
    std::vector<int> r0(cap0, -1), m0(cap0, 0), l0(cap0, 0), r1(cap, -1), m1(cap, 0), l1(cap, 0), slot_map;
    std::vector<NodeRec> nodes(n > 0 ? n : 1);
    VoxelMapDev m{};
    m.keys = k0.data(); m.root_node = r0.data(); m.cap_mask = (unsigned)(cap0 - 1); m.nodes = nodes.data(); m.max_nodes = n;
    m.err = &counters[IM_LC_ERR]; m.pub_mark = m0.data(); m.pub_list = l0.data(); m.pub_n = &counters[IM_LC_PUB_N];
    for (int i = 0; i < n; ++i) {
        int created = 0;
        const int s = hash_insert(m, keys[i], &created);
        if (s < 0 || !created) return -1;
        m.root_node[s] = i;
        m.pub_mark[s] = marks[i];
        nodes[i].root_slot = s;
        if (marks[i]) { list_key[*m.pub_n] = i; m.pub_list[(*m.pub_n)++] = s; }
    }
    VoxelMapDev nm = m;
    nm.keys = k1.data(); nm.root_node = r1.data(); nm.pub_mark = m1.data(); nm.pub_list = l1.data(); nm.cap_mask = (unsigned)(cap - 1);
    rebuild_roots(m, nm, cap0, slot_map, n, l0.data(), *m.pub_n);
    if (counters[IM_LC_ERR]) return -2;
    for (int i = 0; i < n; ++i) {
        const int s = hash_find(nm, keys[i]);
        out_slot[i] = s;
        out_root[i] = s >= 0 ? nm.root_node[s] : -9;
        out_mark[i] = s >= 0 ? nm.pub_mark[s] : -9;
        out_node_slot[i] = nodes[i].root_slot;
    }
    for (int j = 0; j < *m.pub_n; ++j) out_list[j] = nm.pub_list[j];
    return *m.pub_n;
}

// The mesh tables: n voxel keys into a voxel hash of 2^log2_old slots (per-voxel rows derived from the key index), and n triangles
// (triples from tris[n][3], the odd ones removed again) into a triple hash of 2^log2_old slots; both rebuilt into 2^log2_new slots
// with the migration bodies.  Returns the number of keys whose rows did not follow them plus the number of triples tri_find does
// not map to their old index (0 when the rebuild is right); -1 when the set-up overflowed.
int emu_mesh_rehash_check(const unsigned long long* vkeys, int n, const int* tris, int nt, int log2_old, int log2_new) {
    const size_t c0 = (size_t)1 << log2_old, c1 = (size_t)1 << log2_new;
    std::vector<int> cnt(IM_MC_ALLOC, 0);
    std::vector<unsigned long long> k0(c0, IM_EMPTY_KEY), k1(c1, IM_EMPTY_KEY);
    std::vector<int> ch0(c0 * IM_VCHUNKS, -1), ch1(c1 * IM_VCHUNKS, -1), r0[4], r1[4];
    for (int a = 0; a < 4; ++a) { r0[a].assign(c0, 0); r1[a].assign(c1, 0); }
    std::vector<int4> tri(nt > 0 ? nt : 1);
    std::vector<int> tnext((size_t)(nt > 0 ? nt : 1) * 3), head(1 << 20, -1), th0(c0, -1), th1(c1, -1);
    std::vector<unsigned long long> flip(nt > 0 ? nt : 1);
    MeshDev m{};
    m.vkeys = k0.data(); m.vmask = (unsigned)(c0 - 1); m.vox_chunk = ch0.data();
    m.vox_count = r0[0].data(); m.vox_meshing_times = r0[1].data(); m.vox_new_added = r0[2].data(); m.vox_frame = r0[3].data();
    m.tri = tri.data(); m.tri_next = tnext.data(); m.tri_flip = flip.data(); m.v_tri_head = head.data(); m.max_t = nt;
    m.thash = th0.data(); m.tmask = (unsigned)(c0 - 1); m.cnt = cnt.data();
    for (int i = 0; i < n; ++i) {
        int created = 0;
        const int s = table_insert(m.vkeys, m.vmask, vkeys[i], &created);
        if (s < 0 || !created) return -1;
        for (int k = 0; k < IM_VCHUNKS; ++k) m.vox_chunk[(size_t)s * IM_VCHUNKS + k] = i * 16 + k;
        m.vox_count[s] = i + 1; m.vox_meshing_times[s] = 3 * i + 2; m.vox_new_added[s] = 5 * i + 3; m.vox_frame[s] = 7 * i + 4;
    }
    for (int i = 0; i < nt; ++i) {
        const int t = tri_add(m, tris[3 * i], tris[3 * i + 1], tris[3 * i + 2], 1ull);
        if (t != i) return -1;
        if (i & 1) tri_remove(m, t);
    }
    MeshDev nm = m;
    nm.vkeys = k1.data(); nm.vmask = (unsigned)(c1 - 1); nm.vox_chunk = ch1.data();
    nm.vox_count = r1[0].data(); nm.vox_meshing_times = r1[1].data(); nm.vox_new_added = r1[2].data(); nm.vox_frame = r1[3].data();
    nm.thash = th1.data(); nm.tmask = (unsigned)(c1 - 1);
    for (unsigned s : visit_order(c0)) rehash_voxel_slot(m, nm, s);
    for (unsigned s : visit_order(c0)) rehash_tri_slot(m, nm, s);
    if (cnt[IM_MC_ERR]) return -1;
    int bad = 0;
    for (int i = 0; i < n; ++i) {
        const int s = table_find(nm.vkeys, nm.vmask, vkeys[i]);
        if (s < 0) { ++bad; continue; }
        bool ok = nm.vox_count[s] == i + 1 && nm.vox_meshing_times[s] == 3 * i + 2 && nm.vox_new_added[s] == 5 * i + 3 && nm.vox_frame[s] == 7 * i + 4;
        for (int k = 0; k < IM_VCHUNKS; ++k) ok = ok && nm.vox_chunk[(size_t)s * IM_VCHUNKS + k] == i * 16 + k;
        if (!ok) ++bad;
    }
    for (int i = 0; i < nt; ++i)
        if (tri_find(nm, tris[3 * i], tris[3 * i + 1], tris[3 * i + 2]) != i) ++bad;
    return bad;
}
}  // extern "C"
