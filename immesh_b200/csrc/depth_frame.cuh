// immesh_b200 -- depth-camera frames (immesh_mesh_push_depth, immesh_lio_step_async_depth): the unprojection of one sampled pixel of a
// depth image into a point, the localization's point filter (Preprocess::l515_handler), and the append step rule of a frame whose point
// count is known on the device only.  __host__ __device__, so that the host emulations (tests/depth_frame/emu_depth_frame.cpp,
// tests/depth_lio/emu_depth_lio.cpp) run the same bodies as the kernels of depth_kernels.cuh.  depth_frame_setup is the one check of a
// caller's immesh_depth_frame for both entry-point families.
//
// Arithmetic (include/immesh_b200.h, immesh_depth_frame): float64 in the written order under -fmad=false, so that a numpy restatement
// reproduces every point bit for bit.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#include "../../include/immesh_b200.h"
#include "hd_math.cuh"

namespace immesh {

// One frame's image and camera as the kernels read them (one H2D per frame).  The image is read on the sampled grid only: sampled pixel
// (su, sv) -- image pixel (su * stride, sv * stride) -- lies at img + sv * row_bytes + su * col_bytes.  A device image is read in place
// (row_bytes = stride * pitch, col_bytes = stride * bytes per pixel); a host image is staged as its sampled grid, tight.
struct DepthFrame {
    const unsigned char* img;
    long long row_bytes, col_bytes;
    int sw, sh;            // sampled grid: ceil(width / stride) x ceil(height / stride)
    int stride, format, kind, pad_;
    double depth_scale, fx, fy, cx, cy, z_min, z_max;
    double R[9], t[3];     // camera to world, OpenCV axes (x right, y down, z forward)
};

IM_HD int depth_bytes_per_pixel(int format) { return format == IMMESH_DEPTH_U16 ? 2 : 4; }
IM_HD int depth_sampled(int len, int stride) { return (len + stride - 1) / stride; }

// Sampled pixel k (row-major over the sampled grid, so ascending k is ascending pixel order): true and its world point when valid.
IM_HD bool depth_point(const DepthFrame& D, int k, float out[3]) {
    const int sv = k / D.sw, su = k - sv * D.sw;
    const unsigned char* p = D.img + (long long)sv * D.row_bytes + (long long)su * D.col_bytes;
    double d;
    if (D.format == IMMESH_DEPTH_U16) {
        unsigned short raw;
        memcpy(&raw, p, sizeof(raw));
        if (raw == 0) return false;
        d = (double)raw * D.depth_scale;
    } else {
        float raw;
        memcpy(&raw, p, sizeof(raw));
        unsigned int bits;
        memcpy(&bits, &raw, sizeof(bits));
        if ((bits & 0x7f800000u) == 0x7f800000u) return false;   // inf or NaN
        d = (double)raw;
    }
    const double u = (double)(su * D.stride), v = (double)(sv * D.stride);
    const double a = (u - D.cx) / D.fx, b = (v - D.cy) / D.fy;
    const double z = D.kind == IMMESH_DEPTH_RANGE ? d / sqrt((a * a + b * b) + 1.0) : d;
    if (!(D.z_min <= z && z <= D.z_max)) return false;
    const double x = a * z, y = b * z;
    for (int i = 0; i < 3; ++i) out[i] = (float)(((D.R[i * 3 + 0] * x + D.R[i * 3 + 1] * y) + D.R[i * 3 + 2] * z) + D.t[i]);
    return true;
}

// The localization's filter of the valid samples (Preprocess::l515_handler, preprocess.cpp:250-256): valid sample i (numbered 0, 1, 2,
// ... in ascending pixel order) with point p is kept iff i % point_filter_num == 0 and not closer than blind:
// r = (x*x + y*y) + z*z in float32 (no FMA), dropped iff (double)r < blind * blind.  point_filter_num = 1, blind = 0 keeps every one.
IM_HD bool depth_keep(int i, const float p[3], int point_filter_num, double blind) {
    if (i % point_filter_num != 0) return false;
    const float r = (p[0] * p[0] + p[1] * p[1]) + p[2] * p[2];
    return !((double)r < blind * blind);
}

// append_point_step = max(1, round(n / appending_pts_frame)) with the integer division first (ImMesh_mesh_reconstruction.cpp:111),
// m = ceil(n / step) candidates, and the candidate grid's mask: one rule for the host (world-frame and handed-over frames) and the
// device (depth frames, whose n is counted there)
IM_HD void frame_append_dims(int n, int append_target, int* step, int* m, unsigned int* cmask) {
    const int s = (int)lround((double)(n / append_target));
    *step = s > 1 ? s : 1;
    *m = n > 0 ? (n + *step - 1) / *step : 0;
    unsigned long long c = 1;
    while (c < 2ULL * (unsigned long long)(*m > 1 ? *m : 1)) c <<= 1;
    *cmask = (unsigned int)(c - 1);
}
// the most candidates any n <= n_max gives: m = n below 2 appending_pts_frame, fewer than 2 appending_pts_frame above it
IM_HD int frame_append_max_m(int n_max, int append_target) {
    const long long cap = 2LL * append_target;
    return (int)(n_max < cap ? n_max : cap);
}

// A caller's immesh_depth_frame and image checked (the error rules of include/immesh_b200.h) and turned into the kernels' DepthFrame,
// read in place at the caller's pitch; *pitch and *bpp for staging a host image.  Returns null, or what is wrong (IMMESH_E_INVALID).
inline const char* depth_frame_setup(const immesh_depth_frame* f, const void* img, DepthFrame* d, long long* pitch, int* bpp) {
    if (!f || !img) return "depth frame: null argument";
    if (f->format != IMMESH_DEPTH_F32 && f->format != IMMESH_DEPTH_U16) return "depth frame: unknown format";
    if (f->kind != IMMESH_DEPTH_PLANAR && f->kind != IMMESH_DEPTH_RANGE) return "depth frame: unknown kind";
    const int b = depth_bytes_per_pixel(f->format);
    if (f->width < 1 || f->height < 1 || f->stride < 1) return "depth frame: width, height and stride must be >= 1";
    const long long p = f->pitch_bytes ? f->pitch_bytes : (long long)f->width * b;
    if (p < (long long)f->width * b || p % b || (uintptr_t)img % b)
        return "depth frame: the pitch is below the row's bytes, or the pitch or the image is not aligned to the pixel size";
    bool finite = std::isfinite(f->fx) && std::isfinite(f->fy) && f->fx != 0.0 && f->fy != 0.0 && std::isfinite(f->cx) && std::isfinite(f->cy);
    for (int i = 0; i < 9; ++i) finite = finite && std::isfinite(f->cam_R[i]);
    for (int i = 0; i < 3; ++i) finite = finite && std::isfinite(f->cam_t[i]);
    if (!finite) return "depth frame: fx and fy must be finite and non-zero, cx, cy, cam_R and cam_t finite";
    if (!(0.0 <= f->z_min && f->z_min < f->z_max && f->z_max < INFINITY)) return "depth frame: needs 0 <= z_min < z_max < inf";
    if (f->format == IMMESH_DEPTH_U16 && !(f->depth_scale > 0.0 && std::isfinite(f->depth_scale)))
        return "depth frame: a u16 image needs a positive, finite depth_scale";
    std::memset(d, 0, sizeof(*d));
    d->img = static_cast<const unsigned char*>(img);
    d->row_bytes = (long long)f->stride * p;
    d->col_bytes = (long long)f->stride * b;
    d->sw = depth_sampled(f->width, f->stride); d->sh = depth_sampled(f->height, f->stride);
    d->stride = f->stride; d->format = f->format; d->kind = f->kind;
    d->depth_scale = f->depth_scale; d->fx = f->fx; d->fy = f->fy; d->cx = f->cx; d->cy = f->cy; d->z_min = f->z_min; d->z_max = f->z_max;
    std::memcpy(d->R, f->cam_R, sizeof(d->R));
    std::memcpy(d->t, f->cam_t, sizeof(d->t));
    *pitch = p;
    *bpp = b;
    return nullptr;
}
// a host image's sampled grid, tight (row_bytes = sw * bpp), into dst: what the kernels read of it, staged through pinned memory
inline void depth_stage_grid(const DepthFrame& d, const unsigned char* img, long long pitch, int bpp, unsigned char* dst) {
    const size_t rowb = (size_t)d.sw * bpp;
    for (int sv = 0; sv < d.sh; ++sv) {
        const unsigned char* row = img + (size_t)sv * d.stride * pitch;
        if (d.stride == 1) { std::memcpy(dst + sv * rowb, row, rowb); continue; }
        for (int su = 0; su < d.sw; ++su) std::memcpy(dst + sv * rowb + (size_t)su * bpp, row + (size_t)su * d.stride * bpp, bpp);
    }
}

}  // namespace immesh
