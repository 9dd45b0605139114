// immesh_b200 -- the texture atlas of immesh_mesh_texture_bake (texture_bake.cu; the rule is stated in include/immesh_b200.h): a row's
// corners in its image, its cell class and sort key, the slots' triangles and texel ownership, the Morton placement of a cell and the
// value of one texel.  __host__ __device__ bodies shared by the kernels and the host emulation of the tests; float64 in the written
// order (built with -fmad=false on the device and -ffp-contract=off on the host).  Also the call's argument check, host code shared
// with the emulation so that both refuse the same inputs.
#pragma once
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/immesh_b200.h"
#include "hd_math.cuh"

namespace immesh {

#define IM_BAKE_MIN_CLASS 3    // S = 8
#define IM_BAKE_MAX_CLASS 13   // S = 8192, the largest page
#define IM_BAKE_CLASSES (IM_BAKE_MAX_CLASS - IM_BAKE_MIN_CLASS + 1)
#define IM_BAKE_CAM_BITS 27
#define IM_BAKE_UNTEXTURED 0xffffffffu   // the sort key of an untextured row: after every textured one

// one camera's image as the kernels read it: packed rows of 3 channels at `pitch` bytes
struct BakeImg { const unsigned char* data; int w, h; long long pitch; };

// rule 1: the corners (u0' v0' u1' v1' u2' v2') of a row's uv in a w x h image selected at ws x hs
IM_HD void bake_scaled(const float* uv, int w, int h, int ws, int hs, double* p) {
    for (int k = 0; k < 3; ++k) {
        p[2 * k] = (((double)uv[2 * k] + 0.5) * (double)w) / (double)ws - 0.5;
        p[2 * k + 1] = (((double)uv[2 * k + 1] + 0.5) * (double)h) / (double)hs - 0.5;
    }
}

// rule 2: the class log2 S of scaled corners p
IM_HD int bake_class(const double* p, int max_cell) {
    double L = 0.0;
    for (int k = 0; k < 3; ++k) {
        const int e = k == 2 ? 0 : k + 1;
        const double du = p[2 * e] - p[2 * k], dv = p[2 * e + 1] - p[2 * k + 1];
        const double l = sqrt(du * du + dv * dv);
        if (l > L) L = l;
    }
    const double need = ceil(L) + 4.0;
    int S = 1 << IM_BAKE_MIN_CLASS, c = IM_BAKE_MIN_CLASS;
    while (S < max_cell && (double)S < need) { S <<= 1; ++c; }
    return c;
}

// rule 3: the sort key (class descending, camera ascending); bin = IM_BAKE_MAX_CLASS - class, the key's top bits
IM_HD unsigned int bake_key(int cls, int cam) { return ((unsigned int)(IM_BAKE_MAX_CLASS - cls) << IM_BAKE_CAM_BITS) | (unsigned int)cam; }
IM_HD int bake_key_bin(unsigned int key) { return (int)(key >> IM_BAKE_CAM_BITS); }
IM_HD int bake_key_cam(unsigned int key) { return (int)(key & ((1u << IM_BAKE_CAM_BITS) - 1u)); }

// rule 4: corner k of slot `slot`'s triangle in a cell of side S, and the slot that owns texel (i, j)
IM_HD void bake_corner(int S, int slot, int k, int* x, int* y) {
    const int t = S - 4;
    if (slot == 0) { *x = k == 1 ? t : 0; *y = k == 2 ? t : 0; }
    else { *x = k == 1 ? 2 : S - 2; *y = k == 2 ? 2 : S - 2; }
}
IM_HD int bake_owner(int S, int i, int j) { return i + j <= S - 2 ? 0 : 1; }
// the texels a slot owns: slot 0 the (S - 1) S / 2 on or above the anti-diagonal i + j = S - 2, slot 1 the other S (S + 1) / 2
IM_HD long long bake_owned(int S, int slot) { return slot == 0 ? (long long)(S - 1) * S / 2 : (long long)S * (S + 1) / 2; }

// rule 5: the Morton decode of a unit offset inside a page: x from the even bits, y from the odd bits
IM_HD void bake_morton(long long off, int* x, int* y) {
    int ux = 0, uy = 0;
    for (int b = 0; b < IM_BAKE_MAX_CLASS; ++b) {   // a page holds at most (8192 / 8)^2 = 2^20 units
        ux |= (int)((off >> (2 * b)) & 1LL) << b;
        uy |= (int)((off >> (2 * b + 1)) & 1LL) << b;
    }
    *x = ux; *y = uy;
}

// rule 6's sample: the point (x, y) clamped to [0, W - 1] x [0, H - 1], then each channel bilinear from x0 = floor(x), x1 = min(x0 + 1,
// W - 1), fx = x - x0 (y likewise), written as floor(value + 0.5)
IM_HD void bake_bilinear(const BakeImg& I, double x, double y, unsigned char* out) {
    const double xm = (double)(I.w - 1), ym = (double)(I.h - 1);
    x = x < 0.0 ? 0.0 : (x > xm ? xm : x);
    y = y < 0.0 ? 0.0 : (y > ym ? ym : y);
    const int x0 = (int)floor(x), y0 = (int)floor(y);
    const int x1 = x0 + 1 < I.w ? x0 + 1 : I.w - 1, y1 = y0 + 1 < I.h ? y0 + 1 : I.h - 1;
    const double fx = x - (double)x0, fy = y - (double)y0;
    const unsigned char* r0 = I.data + (long long)y0 * I.pitch;
    const unsigned char* r1 = I.data + (long long)y1 * I.pitch;
    for (int c = 0; c < 3; ++c) {
        const double top = (1.0 - fx) * (double)r0[3 * x0 + c] + fx * (double)r0[3 * x1 + c];
        const double bot = (1.0 - fx) * (double)r1[3 * x0 + c] + fx * (double)r1[3 * x1 + c];
        const double v = (1.0 - fy) * top + fy * bot;
        out[c] = (unsigned char)floor(v + 0.5);
    }
}

// rule 6: texel (i, j) of slot `slot` in a cell of side S for scaled corners p, sampled bilinearly with clamp to edge from image I
IM_HD void bake_texel(const BakeImg& I, const double* p, int S, int slot, int i, int j, unsigned char* out) {
    const double T = (double)(S - 4);
    const double w1 = (double)(slot ? S - 2 - i : i) / T, w2 = (double)(slot ? S - 2 - j : j) / T;
    double a = w1 > 0.0 ? w1 : 0.0, b = w2 > 0.0 ? w2 : 0.0;
    if (a + b > 1.0) {
        const double s = a + b;
        a = a / s;
        b = b / s;
    }
    const double w0 = (1.0 - a) - b;
    bake_bilinear(I, (w0 * p[0] + a * p[2]) + b * p[4], (w0 * p[1] + a * p[3]) + b * p[5], out);
}

// host code
inline bool bake_pow2_in(long long v, long long lo, long long hi) { return v >= lo && v <= hi && (v & (v - 1)) == 0; }
inline long long bake_image_bytes(const immesh_texture_image& im) { return 3LL * im.width * im.height; }
inline long long bake_arena_bytes(long long max_image_bytes) { return max_image_bytes > 0 ? max_image_bytes : 512LL << 20; }

// the rows' part of the argument check: facet_cam in [-1, n_cams), finite uv on every textured row.  *n_tex: the textured rows;
// used [n_cams]: 1 for a camera some row uses.  An empty string when the rows are valid, else the reason.
inline std::string bake_check_rows(int n_cams, const int32_t* facet_cam, const float* facet_uv, int64_t n_facets, long long* n_tex,
                                   std::vector<unsigned char>& used) {
    used.assign((size_t)n_cams, 0);
    *n_tex = 0;
    for (int64_t r = 0; r < n_facets; ++r) {
        const int k = facet_cam[r];
        if (k < -1 || k >= n_cams) return "facet_cam outside [-1, n_cams) in row " + std::to_string(r);
        if (k < 0) continue;
        for (int c = 0; c < 6; ++c)
            if (!std::isfinite(facet_uv[6 * r + c])) return "a textured row with a non-finite uv: row " + std::to_string(r);
        used[k] = 1;
        ++*n_tex;
    }
    return std::string();
}
// the image part for camera k, which some row uses: an image, image and camera sizes >= 1, a pitch >= 3 width, and for host images
// at most `arena` bytes
inline std::string bake_check_image(const immesh_texture_camera* cams, const immesh_texture_image* images, int on_device, long long arena, int k) {
    const immesh_texture_image& im = images[k];
    if (!im.data || im.width < 1 || im.height < 1 || im.pitch < 3LL * im.width || cams[k].width < 1 || cams[k].height < 1)
        return "camera " + std::to_string(k) + " is used: it needs an image, image and camera sizes >= 1 and a pitch >= 3 width";
    if (!on_device && bake_image_bytes(im) > arena) return "camera " + std::to_string(k) + "'s image is larger than max_image_bytes";
    return std::string();
}

// Host images: the cameras with want[k] in index order, batched into whole images of at most `arena` bytes each (packed 3 width
// height).  Returns the first camera of every batch, then n_cams; *fill_max: the bytes of the largest batch.
inline std::vector<int> bake_batches(const immesh_texture_image* images, const unsigned char* want, int n_cams, long long arena, long long* fill_max) {
    std::vector<int> start;
    long long fill = arena + 1;
    *fill_max = 0;
    for (int k = 0; k < n_cams; ++k) {
        if (!want[k]) continue;
        const long long b = bake_image_bytes(images[k]);
        if (fill + b > arena) { start.push_back(k); fill = 0; }
        fill += b;
        *fill_max = std::max(*fill_max, fill);
    }
    start.push_back(n_cams);
    return start;
}

// the argument check of immesh_mesh_texture_bake (everything but h): an empty string when the call may proceed, else the reason.
// *n_tex: the textured rows.  used [n_cams]: 1 for a camera some row uses.
inline std::string bake_check(const immesh_texture_camera* cams, int n_cams, const immesh_texture_image* images, int on_device, const int32_t* facet_cam,
                              const float* facet_uv, int64_t n_facets, const immesh_texture_atlas_config* cfg, int cap_pages, const int* n_pages,
                              long long* n_tex, std::vector<unsigned char>& used) {
    if (!cams || !images || !cfg || !n_pages || n_cams < 1 || n_cams >= (1 << IM_BAKE_CAM_BITS) || n_facets < 0 || n_facets > 0x7fffffffLL ||
        (n_facets > 0 && (!facet_cam || !facet_uv)) || (on_device != 0 && on_device != 1) || cap_pages < 0)
        return "bad argument (NULL cams, images, cfg or n_pages; n_cams outside [1, 2^27); n_facets outside [0, 2^31) or rows NULL; on_device "
               "not 0 / 1; cap_pages < 0)";
    if (!bake_pow2_in(cfg->page_size, 256, 8192) || !bake_pow2_in(cfg->max_cell, 8, cfg->page_size) || cfg->max_image_bytes < 0)
        return "bad config (page_size a power of two in [256, 8192]; max_cell a power of two in [8, page_size]; max_image_bytes >= 0)";
    std::string why = bake_check_rows(n_cams, facet_cam, facet_uv, n_facets, n_tex, used);
    for (int k = 0; k < n_cams && why.empty(); ++k)
        if (used[k]) why = bake_check_image(cams, images, on_device, bake_arena_bytes(cfg->max_image_bytes), k);
    return why;
}

}  // namespace immesh
