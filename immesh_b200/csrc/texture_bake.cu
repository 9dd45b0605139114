// immesh_b200 -- the texture atlas of a texture selection (immesh_mesh_texture_bake; the rule is stated in include/immesh_b200.h) and the
// uncompressed PNG writer of its pages.  CUDA kernels (sm_90a, bodies in texture_bake_core.cuh) and their C-ABI host orchestration.
//   Layout: one thread per row (k_bake_class) scales the corners, picks the class and writes the sort key and the class histogram; the
// stable radix sort (mesh_sort_passes) orders the rows by key; one block scans the 11 classes (k_bake_table); one thread per textured
// row (k_bake_place) writes its page, its atlas uv and its slot, with the slot's camera as the key of a second stable sort that groups
// the slots by camera (k_bake_ranges marks each camera's range).
//   Bake: one warp per slot (k_bake_texels), lanes striding over the cell's texels and writing the slot's own.  Device images: one launch
// over every slot.  Host images: whole images in camera order, batched into two alternating arenas on an upload stream, each batch's
// launch behind its copies and each copy behind the launch that last read its arena.
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "block_scan.cuh"
#include "handles.hpp"
#include "texture_bake_core.cuh"

using namespace immesh;

namespace {

// the per-class table of k_bake_table, bin b = class IM_BAKE_MAX_CLASS - b
struct BakeTable {
    int rows[IM_BAKE_CLASSES];             // textured rows of the class
    int row_start[IM_BAKE_CLASSES];        // its first sorted position
    long long unit_base[IM_BAKE_CLASSES];  // the unit offset of its first cell
    long long units, cells, texels;        // totals
};
// a textured row's slot, at its sorted position
struct BakeSlot { int row, page, ox, oy, cls, slot; };

// per row: the class of the scaled corners and the key (untextured rows: IM_BAKE_UNTEXTURED); the class histogram
__global__ void __launch_bounds__(256) k_bake_class(const int* cam, const float* uv, const int4* wh, int n, int max_cell, unsigned int* key, unsigned int* val,
                                                    int* hist) {
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
        const int k = cam[r];
        val[r] = (unsigned int)r;
        if (k < 0) { key[r] = IM_BAKE_UNTEXTURED; continue; }
        const int4 s = wh[k];
        double p[6];
        bake_scaled(uv + 6 * (size_t)r, s.x, s.y, s.z, s.w, p);
        const int c = bake_class(p, max_cell);
        key[r] = bake_key(c, k);
        atomicAdd(&hist[IM_BAKE_MAX_CLASS - c], 1);
    }
}

// one block of 1024: each class's first sorted row (a block scan of the histogram), cells and unit base; units per page U = 4^lg
__global__ void __launch_bounds__(1024) k_bake_table(const int* hist, BakeTable* T) {
    const int b = threadIdx.x;
    const int rows = b < IM_BAKE_CLASSES ? hist[b] : 0;
    const int start = block_scan_1024(rows);
    if (b >= IM_BAKE_CLASSES) return;
    T->rows[b] = rows;
    T->row_start[b] = start;
    // the unit base: the cells of the larger classes before it, each (S / 8)^2 units (11 terms, in 64 bits)
    long long base = 0;
    for (int c = 0; c < b; ++c) base += (long long)((hist[c] + 1) / 2) << (2 * (IM_BAKE_MAX_CLASS - c - IM_BAKE_MIN_CLASS));
    T->unit_base[b] = base;
    if (b == IM_BAKE_CLASSES - 1) {
        long long cells = 0, texels = 0;
        for (int c = 0; c < IM_BAKE_CLASSES; ++c) {
            const int S = 1 << (IM_BAKE_MAX_CLASS - c);
            cells += (hist[c] + 1) / 2;
            texels += (long long)((hist[c] + 1) / 2) * bake_owned(S, 0) + (long long)(hist[c] / 2) * bake_owned(S, 1);
        }
        T->units = base + ((long long)((rows + 1) / 2) << (2 * (IM_BAKE_MAX_CLASS - b - IM_BAKE_MIN_CLASS)));
        T->cells = cells;
        T->texels = texels;
    }
}

// per sorted textured position p: the cell and slot (rule 3), the page and origin (rule 5), the row's page and atlas uv; the slot's
// camera and position as the camera sort's pairs
__global__ void __launch_bounds__(256) k_bake_place(const unsigned int* key, const unsigned int* val, int n_tex, const BakeTable* T, int page_lg,
                                                    int* facet_page, float* atlas_uv, BakeSlot* slots, unsigned int* cam_key, unsigned int* cam_val) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_tex; p += gridDim.x * blockDim.x) {
        const unsigned int kk = key[p];
        const int b = bake_key_bin(kk), cls = IM_BAKE_MAX_CLASS - b, S = 1 << cls, q = p - T->row_start[b], row = (int)val[p];
        const long long off = T->unit_base[b] + ((long long)(q >> 1) << (2 * (cls - IM_BAKE_MIN_CLASS)));
        int ux, uy;
        bake_morton(off & ((1LL << (2 * page_lg)) - 1), &ux, &uy);
        BakeSlot s;
        s.row = row; s.page = (int)(off >> (2 * page_lg)); s.ox = 8 * ux; s.oy = 8 * uy; s.cls = cls; s.slot = q & 1;
        slots[p] = s;
        facet_page[row] = s.page;
        for (int k = 0; k < 3; ++k) {
            int x, y;
            bake_corner(S, s.slot, k, &x, &y);
            atlas_uv[6 * (size_t)row + 2 * k] = (float)(s.ox + x);
            atlas_uv[6 * (size_t)row + 2 * k + 1] = (float)(s.oy + y);
        }
        cam_key[p] = (unsigned int)bake_key_cam(kk);
        cam_val[p] = (unsigned int)p;
    }
}

// the slots sorted by camera: camera k's slots are [lo[k], hi[k]) (lo = hi = 0 for an unused camera, from the memset)
__global__ void __launch_bounds__(256) k_bake_ranges(const unsigned int* cam, int n_tex, int* lo, int* hi) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_tex; i += gridDim.x * blockDim.x) {
        if (i == 0 || cam[i] != cam[i - 1]) lo[cam[i]] = i;
        if (i == n_tex - 1 || cam[i] != cam[i + 1]) hi[cam[i]] = i + 1;
    }
}

// one warp per slot of the camera-ordered positions [lo, hi): lanes stride over the cell's S x S texels and write the slot's own
__global__ void __launch_bounds__(256) k_bake_texels(const BakeSlot* slots, const unsigned int* by_cam, int lo, int hi, const int* cam, const float* uv,
                                                     const int4* wh, const BakeImg* imgs, unsigned char* pages, int P) {
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long w = lo + (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < hi; w += warps) {
        const BakeSlot s = slots[by_cam[w]];
        const int k = cam[s.row], S = 1 << s.cls;
        const int4 d = wh[k];
        const BakeImg I = imgs[k];
        double p[6];
        bake_scaled(uv + 6 * (size_t)s.row, d.x, d.y, d.z, d.w, p);
        unsigned char* base = pages + ((size_t)s.page * P * P + (size_t)s.oy * P + s.ox) * 3;
        for (int t = lane; t < S * S; t += 32) {
            const int i = t % S, j = t / S;
            if (bake_owner(S, i, j) != s.slot) continue;
            unsigned char c[3];
            bake_texel(I, p, S, s.slot, i, j, c);
            unsigned char* o = base + ((size_t)j * P + i) * 3;
            o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
        }
    }
}

// the call's upload stream and events, released on every return
struct BakeStreams {
    cudaStream_t up = nullptr;
    cudaEvent_t ev_up[2] = {}, ev_done[2] = {};
    cudaError_t create() {
        cudaError_t e = cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking);
        for (int a = 0; a < 2 && e == cudaSuccess; ++a) {
            e = cudaEventCreateWithFlags(&ev_up[a], cudaEventDisableTiming);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_done[a], cudaEventDisableTiming);
        }
        return e;
    }
    ~BakeStreams() {
        if (up) cudaStreamSynchronize(up);
        for (int a = 0; a < 2; ++a) {
            if (ev_up[a]) cudaEventDestroy(ev_up[a]);
            if (ev_done[a]) cudaEventDestroy(ev_done[a]);
        }
        if (up) cudaStreamDestroy(up);
    }
};

int bake_sort_passes(long long max_key) {
    int passes = 0;
    while (passes < 4 && (max_key >> (8 * passes)) != 0) ++passes;
    return passes;
}

}  // namespace

// Host images in camera order through two alternating device arenas (the batches of bake_batches, batch_start ending with n_cams):
// each batch's images are copied on an upload stream into arena[batch & 1], their entries of himg / d_img [n_cams] point there
// (pitch 3 width), and run(first, last) -- the batch's first and last wanted camera -- queues the batch's work on st behind its
// copies; a copy into an arena waits for the work that last read it.  Shared by immesh_mesh_texture_bake and
// immesh_mesh_render_textured.
int tex_upload_batches(cudaStream_t st, const immesh_texture_image* images, const unsigned char* want, const std::vector<int>& batch_start,
                       unsigned char* const arena[2], std::vector<BakeImg>& himg, BakeImg* d_img, const std::function<void(int, int)>& run) {
    BakeStreams S;
    IM_CUDA(S.create());
    for (size_t bi = 0; bi + 1 < batch_start.size(); ++bi) {
        const int a = (int)(bi & 1), k0 = batch_start[bi], k1 = batch_start[bi + 1];
        if (bi >= 2) IM_CUDA(cudaStreamWaitEvent(S.up, S.ev_done[a], 0));   // the work that last read this arena
        long long off = 0;
        int first = -1, last = -1;
        for (int k = k0; k < k1; ++k) {
            if (!want[k]) continue;
            const immesh_texture_image& im = images[k];
            IM_CUDA(cudaMemcpy2DAsync(arena[a] + off, (size_t)im.width * 3, im.data, (size_t)im.pitch, (size_t)im.width * 3, (size_t)im.height,
                                      cudaMemcpyHostToDevice, S.up));
            himg[k] = BakeImg{arena[a] + off, im.width, im.height, 3LL * im.width};
            off += bake_image_bytes(im);
            if (first < 0) first = k;
            last = k;
        }
        IM_CUDA(cudaMemcpyAsync(d_img + k0, himg.data() + k0, (size_t)(k1 - k0) * sizeof(BakeImg), cudaMemcpyHostToDevice, S.up));
        IM_CUDA(cudaEventRecord(S.ev_up[a], S.up));
        IM_CUDA(cudaStreamWaitEvent(st, S.ev_up[a], 0));
        run(first, last);
        IM_CUDA(cudaEventRecord(S.ev_done[a], st));
    }
    return IMMESH_OK;
}

int immesh_mesh_texture_bake(immesh_mesh_t* h, const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device,
                             const int32_t* facet_cam, const float* facet_uv, int64_t n_facets, const immesh_texture_atlas_config* cfg, uint8_t* pages,
                             int cap_pages, int32_t* facet_page, float* atlas_uv, int* n_pages, int64_t* counts) {
    long long n_tex = 0;
    std::vector<unsigned char> used;
    if (!h) return im_fail(IMMESH_E_INVALID, "texture_bake: bad argument (NULL h)");
    {
        const std::string why = bake_check(cams, n_cams, images, on_device, facet_cam, facet_uv, n_facets, cfg, cap_pages, n_pages, &n_tex, used);
        if (!why.empty()) return im_fail(IMMESH_E_INVALID, ("texture_bake: " + why).c_str());
    }
    const int n = (int)n_facets, nt = (int)n_tex, P = cfg->page_size;
    int page_lg = 0;
    while ((8 << page_lg) < P) ++page_lg;   // U = 4^page_lg units of 8 x 8 texels per page
    cudaStream_t st = h->stream;
    IM_CUDA(cudaStreamSynchronize(st));   // the frames already queued, the pipelined ones included

    std::vector<int4> hwh(n_cams);
    std::vector<BakeImg> himg(n_cams);
    for (int k = 0; k < n_cams; ++k) {
        hwh[k] = used[k] ? make_int4(images[k].width, images[k].height, cams[k].width, cams[k].height) : make_int4(1, 1, 1, 1);
        himg[k] = BakeImg{used[k] ? images[k].data : nullptr, images[k].width, images[k].height, (long long)images[k].pitch};
    }
    const size_t n1 = (size_t)std::max(n, 1), t1 = (size_t)std::max(nt, 1);
    MemSet mem;   // every buffer of the call, released on every return
    int *d_cam = nullptr, *hist = nullptr, *d_page = nullptr, *lo = nullptr, *hi = nullptr, *sort_hist = nullptr;
    float *d_uv = nullptr, *d_auv = nullptr;
    int4* d_wh = nullptr;
    BakeImg* d_img = nullptr;
    BakeTable* d_tab = nullptr;
    BakeSlot* slots = nullptr;
    unsigned int *ku[2] = {}, *vu[2] = {}, *ck[2] = {}, *cv[2] = {};
    {
        cudaError_t e = cudaSuccess;
        auto add = [&e, &mem](auto** p, size_t count) { if (e == cudaSuccess) e = mem.alloc(p, std::max<size_t>(count, 1)); };
        add(&d_cam, n1); add(&d_uv, 6 * n1); add(&d_wh, (size_t)n_cams); add(&d_img, (size_t)n_cams);
        add(&hist, IM_BAKE_CLASSES); add(&d_tab, 1); add(&d_page, n1); add(&d_auv, 6 * n1); add(&slots, t1);
        add(&lo, (size_t)n_cams); add(&hi, (size_t)n_cams);
        for (int b = 0; b < 2; ++b) { add(&ku[b], n1); add(&vu[b], n1); add(&ck[b], t1); add(&cv[b], t1); }
        add(&sort_hist, mesh_sort_hist_ints(n1));
        if (e != cudaSuccess) return im_fail_alloc(e, "texture_bake: allocation of the call's layout buffers failed");
    }
    BakeTable tab = {};
    std::vector<int> hlo(n_cams, 0), hhi(n_cams, 0), hpage;
    std::vector<float> hauv;
    if (n > 0) {
        IM_CUDA(cudaMemcpyAsync(d_cam, facet_cam, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaMemcpyAsync(d_uv, facet_uv, (size_t)n * 6 * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    IM_CUDA(cudaMemcpyAsync(d_wh, hwh.data(), (size_t)n_cams * sizeof(int4), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(hist, 0, IM_BAKE_CLASSES * sizeof(int), st));
    IM_CUDA(cudaMemsetAsync(d_page, 0xff, n1 * sizeof(int), st));
    IM_CUDA(cudaMemsetAsync(lo, 0, (size_t)n_cams * sizeof(int), st));
    IM_CUDA(cudaMemsetAsync(hi, 0, (size_t)n_cams * sizeof(int), st));
    if (n > 0) IM_LAUNCH(k_bake_class, mesh_grid(h, n, 256), 256, 0, st, (const int*)d_cam, (const float*)d_uv, (const int4*)d_wh, n, cfg->max_cell, ku[0], vu[0], hist);
    IM_LAUNCH(k_bake_table, 1, 1024, 0, st, (const int*)hist, d_tab);
    int by_cam = 0;   // the buffer of the camera sort's values
    if (nt > 0) {
        const int cur = mesh_sort_passes(st, ku, vu, 0, n, 4, sort_hist);
        IM_LAUNCH(k_bake_place, mesh_grid(h, nt, 256), 256, 0, st, (const unsigned int*)ku[cur], (const unsigned int*)vu[cur], nt, (const BakeTable*)d_tab, page_lg,
                  d_page, d_auv, slots, ck[0], cv[0]);
        by_cam = mesh_sort_passes(st, ck, cv, 0, nt, bake_sort_passes(n_cams - 1), sort_hist);
        IM_LAUNCH(k_bake_ranges, mesh_grid(h, nt, 256), 256, 0, st, (const unsigned int*)ck[by_cam], nt, lo, hi);
    }
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(&tab, d_tab, sizeof(tab), cudaMemcpyDeviceToHost, st));
    if (n > 0) {
        hpage.resize(n);
        hauv.resize((size_t)n * 6);
        IM_CUDA(cudaMemcpyAsync(hpage.data(), d_page, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaMemcpyAsync(hauv.data(), d_auv, (size_t)n * 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    IM_CUDA(cudaMemcpyAsync(hlo.data(), lo, (size_t)n_cams * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaMemcpyAsync(hhi.data(), hi, (size_t)n_cams * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const long long U = 1LL << (2 * page_lg), np = (tab.units + U - 1) / U;
    if (np > INT_MAX) return im_fail(IMMESH_E_CAPACITY, "texture_bake: the atlas needs more than 2^31 - 1 pages");
    *n_pages = (int)np;
    if (pages && np > cap_pages)
        return im_fail(IMMESH_E_CAPACITY, "texture_bake: more pages than cap_pages (*n_pages holds the number needed; nothing was written)");

    if (pages && np > 0) {
        const size_t page_bytes = (size_t)P * P * 3;
        unsigned char* d_pages = nullptr;
        unsigned char* arena[2] = {nullptr, nullptr};
        // host images: batches of whole used images in camera order, each at most max_image_bytes
        std::vector<int> batch_start;   // the first camera of every batch, then n_cams
        long long arena_bytes = 0;
        if (!on_device) batch_start = bake_batches(images, used.data(), n_cams, bake_arena_bytes(cfg->max_image_bytes), &arena_bytes);
        {
            cudaError_t e = mem.alloc(&d_pages, (size_t)np * page_bytes);
            for (int a = 0; a < 2 && e == cudaSuccess && arena_bytes > 0 && (a == 0 || batch_start.size() > 2); ++a) e = mem.alloc(&arena[a], (size_t)arena_bytes);
            if (e != cudaSuccess) return im_fail_alloc(e, "texture_bake: allocation of the pages or the image arenas failed");
        }
        IM_CUDA(cudaMemsetAsync(d_pages, 0, (size_t)np * page_bytes, st));
        auto bake = [&](int a, int b) {   // the camera-ordered slots [a, b)
            if (b > a) IM_LAUNCH(k_bake_texels, mesh_grid(h, (b - a) * 32, 256), 256, 0, st, (const BakeSlot*)slots, (const unsigned int*)cv[by_cam], a, b,
                                 (const int*)d_cam, (const float*)d_uv, (const int4*)d_wh, (const BakeImg*)d_img, d_pages, P);
        };
        if (on_device) {
            IM_CUDA(cudaMemcpyAsync(d_img, himg.data(), (size_t)n_cams * sizeof(BakeImg), cudaMemcpyHostToDevice, st));
            bake(0, nt);
        } else if (const int rc = tex_upload_batches(st, images, used.data(), batch_start, arena, himg, d_img,
                                                     [&](int first, int last) { bake(hlo[first], hhi[last]); })) {
            return rc;
        }
        IM_CUDA(cudaGetLastError());
        IM_CUDA(cudaMemcpyAsync(pages, d_pages, (size_t)np * page_bytes, cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
    }
    for (int r = 0; r < n; ++r) {   // the rows of untextured facets keep the caller's atlas_uv
        if (facet_page) facet_page[r] = hpage[r];
        if (atlas_uv && hpage[r] >= 0) std::memcpy(atlas_uv + 6 * (size_t)r, hauv.data() + 6 * (size_t)r, 6 * sizeof(float));
    }
    if (counts) {
        counts[0] = nt; counts[1] = n - nt; counts[2] = tab.cells; counts[3] = tab.texels;
    }
    return IMMESH_OK;
}

// An 8-bit RGB PNG with stored (uncompressed) deflate blocks.  Host-side only.
namespace {
unsigned int png_crc(const unsigned char* p, size_t n, unsigned int c = 0xffffffffu) {
    static unsigned int table[256];
    static bool ready = false;
    if (!ready) {
        for (unsigned int i = 0; i < 256; ++i) {
            unsigned int x = i;
            for (int k = 0; k < 8; ++k) x = (x & 1u) ? 0xedb88320u ^ (x >> 1) : x >> 1;
            table[i] = x;
        }
        ready = true;
    }
    for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 255u] ^ (c >> 8);
    return c;
}
void png_be32(std::vector<unsigned char>& v, unsigned int x) {
    for (int s = 24; s >= 0; s -= 8) v.push_back((unsigned char)(x >> s));
}
bool png_chunk(FILE* f, const char* type, const unsigned char* data, size_t n) {
    std::vector<unsigned char> head;
    png_be32(head, (unsigned int)n);
    head.insert(head.end(), type, type + 4);
    unsigned int c = png_crc(head.data() + 4, 4);
    c = png_crc(data, n, c) ^ 0xffffffffu;
    std::vector<unsigned char> tail;
    png_be32(tail, c);
    return std::fwrite(head.data(), 1, head.size(), f) == head.size() && (n == 0 || std::fwrite(data, 1, n, f) == n) &&
           std::fwrite(tail.data(), 1, tail.size(), f) == tail.size();
}
}  // namespace

int immesh_write_png(const char* path, const uint8_t* rgb, int width, int height) {
    if (!path || !rgb || width < 1 || height < 1 || (long long)width * 3 + 1 > INT_MAX)
        return im_fail(IMMESH_E_INVALID, "write_png: bad argument (NULL path or rgb; a size below 1)");
    const size_t row = (size_t)width * 3 + 1, raw = row * (size_t)height;
    // the zlib stream: header, stored blocks of at most 65535 bytes of the filtered rows (filter 0), Adler-32 of those rows
    std::vector<unsigned char> z;
    z.reserve(2 + raw + 5 * (raw / 65535 + 1) + 4);
    z.push_back(0x78); z.push_back(0x01);
    unsigned int s1 = 1, s2 = 0;
    size_t left = raw, y = 0, x = 0;   // the next byte: row y, position x (0: the filter byte)
    while (left > 0) {
        const size_t len = std::min<size_t>(left, 65535);
        left -= len;
        z.push_back(left == 0 ? 1 : 0);
        z.push_back((unsigned char)(len & 255)); z.push_back((unsigned char)(len >> 8));
        z.push_back((unsigned char)(~len & 255)); z.push_back((unsigned char)((~len >> 8) & 255));
        for (size_t i = 0; i < len; ++i) {
            const unsigned char b = x == 0 ? 0 : rgb[y * (row - 1) + x - 1];
            z.push_back(b);
            s1 = (s1 + b) % 65521u;
            s2 = (s2 + s1) % 65521u;
            if (++x == row) { x = 0; ++y; }
        }
    }
    png_be32(z, (s2 << 16) | s1);
    FILE* f = std::fopen(path, "wb");
    if (!f) return im_fail(IMMESH_E_INVALID, "write_png: cannot open the file");
    static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    std::vector<unsigned char> ihdr;
    png_be32(ihdr, (unsigned int)width);
    png_be32(ihdr, (unsigned int)height);
    const unsigned char rest[5] = {8, 2, 0, 0, 0};   // 8 bits, RGB, deflate, adaptive filtering, no interlace
    ihdr.insert(ihdr.end(), rest, rest + 5);
    bool ok = std::fwrite(sig, 1, 8, f) == 8 && png_chunk(f, "IHDR", ihdr.data(), ihdr.size());
    for (size_t o = 0; ok && o < z.size(); o += (size_t)1 << 30) ok = png_chunk(f, "IDAT", z.data() + o, std::min<size_t>(z.size() - o, (size_t)1 << 30));
    ok = ok && png_chunk(f, "IEND", nullptr, 0);
    if (std::fclose(f) != 0 || !ok) return im_fail(IMMESH_E_INVALID, "write_png: writing the file failed");
    return IMMESH_OK;
}
