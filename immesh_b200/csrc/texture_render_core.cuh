// immesh_b200 -- the textured mesh at a camera (immesh_mesh_render_textured, texture_render.cu; the pixel rule is stated in
// include/immesh_b200.h): the winner's weights in the face order of its row, the source point in its image, and one pixel's error
// against the truth image.  __host__ __device__ bodies shared by the kernels and the host emulation of the tests; float64 in the written
// order (built with -fmad=false on the device and -ffp-contract=off on the host).  The sample itself is bake_bilinear
// (texture_bake_core.cuh).  Also the call's argument check, host code shared with the emulation so that both refuse the same inputs.
#pragma once
#include <climits>
#include <cmath>
#include <string>
#include <vector>

#include "texture_bake_core.cuh"
#include "texture_core.cuh"

namespace immesh {

// steps 3-4: the winner's perspective-correct weights w_i = e_i (1 / z_i) at pixel (x, y) of its set-up T (corners in stored order),
// permuted into the face order of tex_corners: o0 = w0, o1 = flip ? w1 : w2, o2 = flip ? w2 : w1
IM_HD void trv_weights(const DepthTri& T, int x, int y, int flip, double* o) {
    double e[3];
    depth_edges(T, x, y, e);
    const double w0 = e[0] * T.iz0, w1 = e[1] * T.iz1, w2 = e[2] * T.iz2;
    o[0] = w0;
    o[1] = flip ? w1 : w2;
    o[2] = flip ? w2 : w1;
}
// step 5: the source point of face-order weights o and scaled corners p (bake_scaled)
IM_HD void trv_source(const double* o, const double* p, double* x, double* y) {
    const double s = (o[0] + o[1]) + o[2];
    *x = ((o[0] * p[0] + o[1] * p[2]) + o[2] * p[4]) / s;
    *y = ((o[0] * p[1] + o[1] * p[3]) + o[2] * p[5]) / s;
}
// the score of one textured pixel: squared differences per channel into sse[3], absolute differences into *sad
IM_HD void trv_error(const unsigned char* a, const unsigned char* b, long long* sse, long long* sad) {
    for (int c = 0; c < 3; ++c) {
        const long long d = (long long)a[c] - (long long)b[c];
        sse[c] += d * d;
        *sad += d < 0 ? -d : d;
    }
}

// the argument check of immesh_mesh_render_textured before the view is resolved (n_live: the live triangle count; shard_n: the
// handle's shards): an empty string when the call may proceed, else the reason.  used [n_cams]: 1 for a camera some row uses.  A NULL
// image of a camera the view samples is refused once the view is resolved (trv_check_needed).
inline std::string trv_check(const immesh_texture_camera* view, const immesh_texture_view_config* cfg, const immesh_texture_camera* cams, int n_cams,
                             const immesh_texture_image* images, int on_device, const int32_t* facet_cam, const float* facet_uv, int64_t n_facets,
                             const immesh_texture_image* truth, const uint8_t* rgb, int64_t n_live, int shard_n, std::vector<unsigned char>& used) {
    if (!view || !cfg || !cams || n_cams < 1 || n_facets < 0 || n_facets > INT_MAX || (n_facets > 0 && (!facet_cam || !facet_uv)) ||
        (on_device != 0 && on_device != 1))
        return "bad argument (NULL view, cfg or cams; n_cams < 1; n_facets outside [0, 2^31) or rows NULL; on_device not 0 / 1)";
    if (!tex_camera_ok(*view)) return "bad view (1 <= width * height <= 2^26; finite intrinsics and pose; fx, fy != 0)";
    if (!(cfg->z_near > 0) || !(cfg->z_far > cfg->z_near) || !std::isfinite(cfg->z_far) || (cfg->positions != 0 && cfg->positions != 1) ||
        cfg->max_image_bytes < 0)
        return "bad config (0 < z_near < z_far < inf; positions 0 or 1; max_image_bytes >= 0)";
    if (!images && (rgb || truth)) return "rgb and truth need images (images = NULL is the query)";
    if (truth && (!truth->data || truth->width != view->width || truth->height != view->height || truth->pitch < 3LL * truth->width))
        return "truth must be an image of the view's size with a pitch >= 3 width";
    if (shard_n > 1) return "a sharded mesh handle is not supported";
    if (n_facets != n_live) return "n_facets (" + std::to_string(n_facets) + ") is not the live triangle count (" + std::to_string(n_live) + ")";
    long long n_tex = 0;
    std::string why = bake_check_rows(n_cams, facet_cam, facet_uv, n_facets, &n_tex, used);
    for (int k = 0; images && k < n_cams && why.empty(); ++k)
        if (used[k] && images[k].data) why = bake_check_image(cams, images, on_device, bake_arena_bytes(cfg->max_image_bytes), k);
    return why;
}
// after the view is resolved: every camera it samples has an image
inline std::string trv_check_needed(const immesh_texture_image* images, const unsigned char* needed, int n_cams) {
    for (int k = 0; images && k < n_cams; ++k)
        if (needed[k] && !images[k].data) return "camera " + std::to_string(k) + " is sampled by the view: it needs an image";
    return std::string();
}
// each camera's image and selection sizes (W, H, Ws, Hs) as bake_scaled reads them; (1, 1, 1, 1) where no image is given
inline void trv_sizes(const immesh_texture_camera* cams, const immesh_texture_image* images, int n_cams, int* wh /*[n_cams][4]*/) {
    for (int k = 0; k < n_cams; ++k) {
        const bool img = images && images[k].data;
        wh[4 * k] = img ? images[k].width : 1; wh[4 * k + 1] = img ? images[k].height : 1;
        wh[4 * k + 2] = img ? cams[k].width : 1; wh[4 * k + 3] = img ? cams[k].height : 1;
    }
}

}  // namespace immesh
