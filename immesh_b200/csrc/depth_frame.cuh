// immesh_b200 -- depth-camera frames (immesh_mesh_push_depth): the unprojection of one sampled pixel of a depth image into a world point,
// and the append step rule of a frame whose point count is known on the device only.  __host__ __device__, so that the host emulation
// (tests/depth_frame/emu_depth_frame.cpp) runs the same bodies as the kernels of mesh_capi.cu (k_depth_count, k_depth_emit).
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

}  // namespace immesh
