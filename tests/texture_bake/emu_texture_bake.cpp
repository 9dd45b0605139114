// TEST INFRASTRUCTURE (not product code): immesh_mesh_texture_bake's bodies (immesh_b200/csrc/texture_bake_core.cuh) and its argument
// check run on the CPU with the device call's orchestration: per row the class and key (k_bake_class) and the class histogram, the rows
// sorted stably by key (the radix sort's order), the class table (k_bake_table), each textured position's cell, slot, page and atlas uv
// (k_bake_place), then the slots grouped stably by camera and each slot's owned texels written (k_bake_texels).  The shipped library
// never links or calls this.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../immesh_b200/csrc/texture_bake_core.cuh"

using namespace immesh;

static std::string g_err;

extern "C" {
const char* emu_texture_bake_error() { return g_err.c_str(); }

// as immesh_mesh_texture_bake without a handle: returns IMMESH_OK, IMMESH_E_INVALID or IMMESH_E_CAPACITY with the same outputs
int emu_texture_bake(const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device, const int32_t* facet_cam,
                     const float* facet_uv, int64_t n_facets, const immesh_texture_atlas_config* cfg, uint8_t* pages, int cap_pages, int32_t* facet_page,
                     float* atlas_uv, int* n_pages, int64_t* counts) {
    long long n_tex = 0;
    std::vector<unsigned char> used;
    g_err = bake_check(cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, cfg, cap_pages, n_pages, &n_tex, used);
    if (!g_err.empty()) return IMMESH_E_INVALID;
    const int n = (int)n_facets, P = cfg->page_size;
    int page_lg = 0;
    while ((8 << page_lg) < P) ++page_lg;
    // k_bake_class
    std::vector<unsigned int> key(n);
    std::vector<int> hist(IM_BAKE_CLASSES, 0);
    std::vector<double> scaled((size_t)n * 6);
    for (int r = 0; r < n; ++r) {
        const int k = facet_cam[r];
        if (k < 0) { key[r] = IM_BAKE_UNTEXTURED; continue; }
        bake_scaled(facet_uv + 6 * (size_t)r, images[k].width, images[k].height, cams[k].width, cams[k].height, &scaled[6 * (size_t)r]);
        const int c = bake_class(&scaled[6 * (size_t)r], cfg->max_cell);
        key[r] = bake_key(c, k);
        ++hist[IM_BAKE_MAX_CLASS - c];
    }
    // the stable sort by key
    std::vector<int> order(n);
    for (int r = 0; r < n; ++r) order[r] = r;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key[a] < key[b]; });
    // k_bake_table
    std::vector<int> row_start(IM_BAKE_CLASSES, 0);
    std::vector<long long> unit_base(IM_BAKE_CLASSES, 0);
    long long units = 0, cells = 0, texels = 0;
    for (int b = 0; b < IM_BAKE_CLASSES; ++b) {
        const int S = 1 << (IM_BAKE_MAX_CLASS - b);
        row_start[b] = b ? row_start[b - 1] + hist[b - 1] : 0;
        unit_base[b] = units;
        units += (long long)((hist[b] + 1) / 2) << (2 * (IM_BAKE_MAX_CLASS - b - IM_BAKE_MIN_CLASS));
        cells += (hist[b] + 1) / 2;
        texels += (long long)((hist[b] + 1) / 2) * bake_owned(S, 0) + (long long)(hist[b] / 2) * bake_owned(S, 1);
    }
    const long long U = 1LL << (2 * page_lg), np = (units + U - 1) / U;
    *n_pages = (int)np;
    if (pages && np > cap_pages) { g_err = "more pages than cap_pages"; return IMMESH_E_CAPACITY; }
    // k_bake_place
    struct Slot { int row, page, ox, oy, cls, slot, cam; };
    std::vector<Slot> slots(n_tex);
    std::vector<int> page_of(n, -1);
    std::vector<float> auv((size_t)n * 6);
    for (int p = 0; p < n_tex; ++p) {
        const int row = order[p], b = bake_key_bin(key[row]), cls = IM_BAKE_MAX_CLASS - b, S = 1 << cls, q = p - row_start[b];
        const long long off = unit_base[b] + ((long long)(q >> 1) << (2 * (cls - IM_BAKE_MIN_CLASS)));
        int ux, uy;
        bake_morton(off & (U - 1), &ux, &uy);
        Slot s{row, (int)(off >> (2 * page_lg)), 8 * ux, 8 * uy, cls, q & 1, bake_key_cam(key[row])};
        slots[p] = s;
        page_of[row] = s.page;
        for (int k = 0; k < 3; ++k) {
            int x, y;
            bake_corner(S, s.slot, k, &x, &y);
            auv[6 * (size_t)row + 2 * k] = (float)(s.ox + x);
            auv[6 * (size_t)row + 2 * k + 1] = (float)(s.oy + y);
        }
    }
    // the slots grouped by camera, then k_bake_texels (pages zeroed first)
    if (pages && np > 0) {
        std::stable_sort(slots.begin(), slots.end(), [](const Slot& a, const Slot& b) { return a.cam < b.cam; });
        std::memset(pages, 0, (size_t)np * P * P * 3);
        for (const Slot& s : slots) {
            const immesh_texture_image& im = images[s.cam];
            const BakeImg I{im.data, im.width, im.height, (long long)im.pitch};
            const int S = 1 << s.cls;
            for (int j = 0; j < S; ++j)
                for (int i = 0; i < S; ++i) {
                    if (bake_owner(S, i, j) != s.slot) continue;
                    bake_texel(I, &scaled[6 * (size_t)s.row], S, s.slot, i, j, pages + ((size_t)s.page * P * P + (size_t)(s.oy + j) * P + s.ox + i) * 3);
                }
        }
    }
    for (int r = 0; r < n; ++r) {
        if (facet_page) facet_page[r] = page_of[r];
        if (atlas_uv && page_of[r] >= 0) std::memcpy(atlas_uv + 6 * (size_t)r, &auv[6 * (size_t)r], 6 * sizeof(float));
    }
    if (counts) { counts[0] = n_tex; counts[1] = n - n_tex; counts[2] = cells; counts[3] = texels; }
    return IMMESH_OK;
}
}  // extern "C"
