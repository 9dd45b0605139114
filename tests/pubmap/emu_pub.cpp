// TEST INFRASTRUCTURE (not product code): the host emulation of the localization kernels (tests/emu/emu_lio.cpp) with the
// plane-map publisher's device state attached -- VoxelMapDev::pub (per node), pub_mark / pub_list / pub_n (per hash slot) -- and
// immesh_voxelmap_plane_markers running the same __host__ __device__ walk as the CUDA library (voxelmap.cuh: plane_pub_root,
// plane_pub_commit).  Built as its own library: the handles it creates carry the publisher state from the start.
#define immesh_lio_create emu_base_lio_create
#define immesh_lio_destroy emu_base_lio_destroy
#include "../emu/emu_lio.cpp"
#undef immesh_lio_create
#undef immesh_lio_destroy

#include <unordered_map>

namespace {
struct PubStore {
    std::vector<PubRec> pub;
    std::vector<int> mark, list;
    int n = 0;
};
std::unordered_map<immesh_lio*, PubStore*> g_pub;
}  // namespace

extern "C" {
int immesh_lio_create(const immesh_lio_config* cfg, immesh_lio_t** out) {
    const int rc = emu_base_lio_create(cfg, out);
    if (rc) return rc;
    immesh_lio* h = *out;
    PubStore* s = new PubStore();
    s->pub.resize(h->nodes.size());
    s->mark.assign(h->keys.size(), 0);
    s->list.assign(h->keys.size(), 0);
    g_pub[h] = s;
    VoxelMapDev& m = h->map;
    m.pub = s->pub.data(); m.pub_mark = s->mark.data(); m.pub_list = s->list.data(); m.pub_n = &s->n;
    return 0;
}
int immesh_lio_destroy(immesh_lio_t* h) {
    auto it = g_pub.find(h);
    if (it != g_pub.end()) { delete it->second; g_pub.erase(it); }
    return emu_base_lio_destroy(h);
}
// the CUDA library's contract: the listed roots in ascending packed key, rows counted first, nothing consumed when they do not fit
int immesh_voxelmap_plane_markers(immesh_lio_t* h, double* rows, int cap, int* n_out, int64_t* counts) {
    if (!h || !n_out || cap < 0 || (cap > 0 && !rows)) return IMMESH_E_INVALID;
    const VoxelMapDev& m = h->map;
    const int n = *m.pub_n;
    std::vector<int> slots(m.pub_list, m.pub_list + n);
    std::sort(slots.begin(), slots.end(), [&](int a, int b) { return m.keys[a] < m.keys[b]; });
    int c[4] = {0, 0, 0, 0};
    std::vector<int> off(n + 1, 0);
    for (int i = 0; i < n; ++i) {
        const int root = m.root_node[slots[i]];
        off[i + 1] = off[i] + (root >= 0 ? plane_pub_root(m, root, m.keys[slots[i]], nullptr, c) : 0);
    }
    *n_out = off[n];
    if (counts) {
        for (int k = 0; k < 4; ++k) counts[k] = c[k];
        counts[4] = n;
    }
    if (off[n] > cap) return IMMESH_E_CAPACITY;
    std::vector<double> buf((size_t)off[n] * IM_PUB_COLS + 1);   // the device writes its rows to a buffer of its own too
    *m.pub_n = 0;
    for (int i = 0; i < n; ++i)
        if (plane_pub_commit(m, slots[i], buf.data() + (size_t)off[i] * IM_PUB_COLS)) m.pub_list[(*m.pub_n)++] = slots[i];
    if (off[n] > 0) std::memcpy(rows, buf.data(), (size_t)off[n] * IM_PUB_COLS * sizeof(double));
    return 0;
}
}  // extern "C"
