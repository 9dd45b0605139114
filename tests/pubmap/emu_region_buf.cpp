// TEST INFRASTRUCTURE (not product code): the host emulation of the mesher (tests/emu/emu_mesh.cpp) with the m_smoothed flags
// (MeshDev::vsmoothed) attached, and immesh_mesh_region_buffers / immesh_mesh_smooth_all on the emulated buffers with the CUDA
// library's contract: the same __host__ __device__ bodies (mesh_core.cuh: tri_region_key, smooth_vertex, store_smooth, region_row,
// axis_take / axis_apply), the same (region, triple) order, claim-once smoothing, capacity and argument rules.  The kNN is k_knn's
// exact ring search run by one lane.  Built as its own library: the handles it creates keep the flags from the start.
#define immesh_mesh_create emu_base_mesh_create
#define immesh_mesh_destroy emu_base_mesh_destroy
#define emu_mesh_xapply_smooth emu_base_mesh_xapply_smooth
#include "../emu/emu_mesh.cpp"
#undef immesh_mesh_create
#undef immesh_mesh_destroy
#undef emu_mesh_xapply_smooth

#include <map>
#include <unordered_map>

namespace {
std::unordered_map<immesh_mesh*, std::vector<unsigned char>*> g_flags;

// k_knn for one query: exact k nearest vertices by float squared distance (dist2f), ascending, ties to the lower id, ring
// expansion over the mesh-voxel hash with k_knn's stopping rules
void emu_knn(const MeshDev& M, const MeshParams& P, const float* q, int k, double max_dist, int* out_idx, float* out_d2) {
    const int cx = round_key(q[0], P.res), cy = round_key(q[1], P.res), cz = round_key(q[2], P.res);
    const double max_d2 = max_dist * max_dist;
    std::vector<std::pair<float, int>> best;
    int far = -1;
    if (M.cnt[4] > 0) {
        far = std::max(std::abs(cx - M.cnt[11]), std::abs(cx - M.cnt[14]));
        far = std::max(far, std::max(std::abs(cy - M.cnt[12]), std::abs(cy - M.cnt[15])));
        far = std::max(far, std::max(std::abs(cz - M.cnt[13]), std::abs(cz - M.cnt[16])));
    }
    for (int ring = 0; ring <= far; ++ring) {
        if (ring >= 1) {
            const double lb = (double)(ring - 1) * P.res;
            if (lb > max_dist) break;
            if ((int)best.size() >= k && (double)best[k - 1].first < lb * lb * 0.999999) break;
        }
        for (int dx = -ring; dx <= ring; ++dx)
            for (int dy = -ring; dy <= ring; ++dy)
                for (int dz = -ring; dz <= ring; ++dz) {
                    if (std::max(std::abs(dx), std::max(std::abs(dy), std::abs(dz))) != ring) continue;
                    if (!ikey_ok(cx + dx, cy + dy, cz + dz)) continue;
                    const int s = table_find(M.vkeys, M.vmask, pack_ikey(cx + dx, cy + dy, cz + dz));
                    if (s < 0) continue;
                    const int cntv = std::min(M.vox_count[s], IM_VCHUNKS * 16);
                    for (int kk = 0; kk < cntv; ++kk) {
                        const float4 p = M.vchunk_pts[(size_t)M.vox_chunk[(size_t)s * IM_VCHUNKS + (kk >> 4)] * 16 + (kk & 15)];
                        int v;
                        std::memcpy(&v, &p.w, 4);
                        const float d2 = dist2f(q[0], q[1], q[2], p.x, p.y, p.z);
                        if (!((double)d2 <= max_d2)) continue;
                        best.push_back({d2, v});
                    }
                }
        std::sort(best.begin(), best.end());
        if ((int)best.size() > k) best.resize(k);
    }
    for (int r = 0; r < k; ++r) {
        out_idx[r] = r < (int)best.size() ? best[r].second : -1;
        out_d2[r] = r < (int)best.size() ? best[r].first : INFINITY;
    }
}
void emu_smooth_list(immesh_mesh* h, const std::vector<int>& list, int knn, double sf) {
    std::vector<int> idx((size_t)knn);
    std::vector<float> d2((size_t)knn);
    for (int v : list) {   // k_knn over the list, then k_rb_smooth / k_smooth_all: the result reads raw positions only
        const float4 p = h->M.vpos[v];
        const float q[3] = {p.x, p.y, p.z};
        emu_knn(h->M, h->P, q, knn, INFINITY, idx.data(), d2.data());
        double r[3];
        smooth_vertex(h->M, v, knn, idx.data(), d2.data(), sf, h->P.accept, r);
        store_smooth(h->M, v, r[0], r[1], r[2]);
    }
}
}  // namespace

extern "C" {
int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    const int rc = emu_base_mesh_create(cfg, out);
    if (rc) return rc;
    immesh_mesh* h = *out;
    auto* f = new std::vector<unsigned char>((size_t)h->M.max_v, 0);
    g_flags[h] = f;
    h->M.vsmoothed = f->data();
    return 0;
}
int immesh_mesh_destroy(immesh_mesh_t* h) {
    auto it = g_flags.find(h);
    if (it != g_flags.end()) { delete it->second; g_flags.erase(it); }
    return emu_base_mesh_destroy(h);
}
// k_apply_smooth's per-entry store
int emu_mesh_xapply_smooth(immesh_mesh_t* h, const void* smooth32, int n) {
    const XSmooth* e = (const XSmooth*)smooth32;
    for (int i = 0; i < n; ++i) store_smooth(h->M, e[i].id, e[i].x, e[i].y, e[i].z);
    return 0;
}
// the flags and smoothed positions of the first n vertices (test access)
int emu_mesh_smooth_state(immesh_mesh_t* h, unsigned char* flags, double* smooth) {
    const int nv = h->M.cnt[0];
    if (flags) std::memcpy(flags, h->M.vsmoothed, (size_t)nv);
    if (smooth) std::memcpy(smooth, h->M.vsmooth, (size_t)nv * 3 * sizeof(double));
    return nv;
}
int immesh_mesh_smooth_all(immesh_mesh_t* h, double smooth_factor, int knn, double* smoothed) {
    if (!h || knn < 1 || knn > 32) return IMMESH_E_INVALID;
    const int nv = h->M.cnt[0];
    std::vector<int> all((size_t)nv);
    for (int v = 0; v < nv; ++v) all[v] = v;
    emu_smooth_list(h, all, knn, smooth_factor);
    if (smoothed) std::memcpy(smoothed, h->M.vsmooth, (size_t)nv * 3 * sizeof(double));
    return 0;
}
int immesh_mesh_region_buffers(immesh_mesh_t* h, double region_size, const int32_t* keys, int n_keys, double smooth_factor, int knn,
                               float* tri_xyz, int32_t* tri_ids, int cap, int32_t* region_keys, int32_t* region_offsets, int cap_regions,
                               float* axis_min_max, int* n_regions, int* n_tris, int* n_smoothed) {
    if (!h || !n_regions || !n_tris || !(region_size > 0) || knn < 1 || knn > 32 || cap < 0 || cap_regions < 0 || (keys && n_keys < 0)) return IMMESH_E_INVALID;
    *n_regions = 0;
    *n_tris = 0;
    if (n_smoothed) *n_smoothed = 0;
    const MeshDev& M = h->M;
    const bool use_keys = keys != nullptr;
    const int nk = use_keys ? n_keys : 0;
    std::map<unsigned long long, int> req;
    for (int i = 0; i < nk; ++i) {
        for (int j = 0; j < i; ++j)
            if (keys[3 * i] == keys[3 * j] && keys[3 * i + 1] == keys[3 * j + 1] && keys[3 * i + 2] == keys[3 * j + 2]) return IMMESH_E_INVALID;
        if (ikey_ok(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2])) req[pack_ikey(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2])] = i;
    }
    // k_rb_select + the radix sort's result: (region word, i, j, k) ascending
    struct Kept { unsigned long long word; int a, b, c, slot; };
    std::vector<Kept> kept;
    const int nalloc = std::min(M.cnt[1], M.max_t);
    for (int t = 0; t < nalloc; ++t) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        int k[3];
        tri_region_key(M, r, region_size, k);
        if (!ikey_ok(k[0], k[1], k[2])) return IMMESH_E_RANGE;
        unsigned long long word = pack_ikey(k[0], k[1], k[2]);
        if (use_keys) {
            auto it = req.find(word);
            if (it == req.end()) continue;
            word = (unsigned long long)it->second;
        }
        kept.push_back({word, r.x, r.y, r.z, t});
    }
    std::sort(kept.begin(), kept.end(), [](const Kept& x, const Kept& y) {
        if (x.word != y.word) return x.word < y.word;
        if (x.a != y.a) return x.a < y.a;
        if (x.b != y.b) return x.b < y.b;
        return x.c < y.c;
    });
    const int n = (int)kept.size();
    std::vector<int> rkeys, roff;
    if (use_keys) {
        roff.assign((size_t)nk + 1, n);
        for (int r = nk - 1; r >= 0; --r) {
            int i = roff[r + 1];
            while (i > 0 && (int)kept[i - 1].word >= r) --i;
            roff[r] = i;
        }
        rkeys.assign(keys, keys + (size_t)nk * 3);
    } else {
        for (int i = 0; i < n; ++i)
            if (i == 0 || kept[i].word != kept[i - 1].word) {
                int x, y, z;
                unpack_ikey(kept[i].word, &x, &y, &z);
                rkeys.insert(rkeys.end(), {x, y, z});
                roff.push_back(i);
            }
        roff.push_back(n);
    }
    const int nr = (int)roff.size() - 1;
    *n_tris = n;
    *n_regions = nr;
    if (n > cap || nr > cap_regions) return IMMESH_E_CAPACITY;
    // k_rb_claim + k_knn + k_rb_smooth
    std::vector<unsigned char> claimed((size_t)M.cnt[0], 0);
    std::vector<int> list;
    for (const Kept& e : kept)
        for (int v : {e.a, e.b, e.c})
            if (!M.vsmoothed[v] && !claimed[v]) { claimed[v] = 1; list.push_back(v); }
    emu_smooth_list(h, list, knn, smooth_factor);
    if (n_smoothed) *n_smoothed = (int)list.size();
    // k_rb_emit + k_rb_axis
    AxisAcc acc;
    axis_init(acc);
    for (int i = 0; i < n; ++i) {
        const int4 r = make_int4(kept[i].a, kept[i].b, kept[i].c, 1);
        float row[9];
        region_row(M, r, row);
        if (tri_xyz) std::memcpy(tri_xyz + (size_t)i * 9, row, sizeof(row));
        if (tri_ids) { tri_ids[(size_t)i * 3] = r.x; tri_ids[(size_t)i * 3 + 1] = r.y; tri_ids[(size_t)i * 3 + 2] = r.z; }
        for (int j = 0; j < 3; ++j)
            for (int d = 0; d < 3; ++d) { axis_take(acc, d, row[j * 3 + d], i * 3 + j); axis_take(acc, d + 3, row[j * 3 + d], i * 3 + j); }
    }
    if (axis_min_max) axis_apply(acc, axis_min_max);
    if (region_keys && nr > 0) std::memcpy(region_keys, rkeys.data(), (size_t)nr * 3 * sizeof(int));
    if (region_offsets) std::memcpy(region_offsets, roff.data(), ((size_t)nr + 1) * sizeof(int));
    return 0;
}
}  // extern "C"
