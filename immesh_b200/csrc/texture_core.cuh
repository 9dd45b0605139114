// immesh_b200 -- the texture selection of immesh_mesh_texture_select (texture_capi.cu; the rule is stated in include/immesh_b200.h):
// the caller's OpenCV camera as the rasteriser's, a facet's corners in the PLY face order, the "seen by camera k" test, the nearest
// camera and the texture coordinates.  __host__ __device__ bodies shared by the kernels and the host emulation of the tests; float64
// in the written order (built with -fmad=false on the device and -ffp-contract=off on the host).
#pragma once
#include <cmath>

#include "../../include/immesh_b200.h"
#include "reinforce.cuh"

namespace immesh {

// the rasteriser's camera of an OpenCV camera (x right, y down, z forward; world = cam_R p + cam_t): the rasteriser maps
// world = R diag(1, -1, -1) p + t, so R is cam_R with columns 1 and 2 negated (exact: depth_project's u, v, z are unchanged bits)
IM_HD DepthCam tex_camera(const immesh_texture_camera& c, double z_near, double z_far) {
    DepthCam C;
    C.fx = c.fx; C.fy = c.fy; C.cx = c.cx; C.cy = c.cy; C.z_near = z_near; C.z_far = z_far;
    for (int r = 0; r < 3; ++r) {
        C.R[r * 3 + 0] = c.cam_R[r * 3 + 0];
        C.R[r * 3 + 1] = -c.cam_R[r * 3 + 1];
        C.R[r * 3 + 2] = -c.cam_R[r * 3 + 2];
    }
    for (int i = 0; i < 3; ++i) C.t[i] = c.cam_t[i];
    C.w = c.width; C.h = c.height;
    return C;
}

// the corners q0 q1 q2 of the stored triple's positions p0 p1 p2 in immesh_write_ply's face order: flip != 0 p0 p1 p2, else p0 p2 p1
IM_HD void tex_corners(const float4& p0, const float4& p1, const float4& p2, int flip, float4* q) {
    q[0] = p0;
    q[1] = flip ? p1 : p2;
    q[2] = flip ? p2 : p1;
}

// The rule's per-camera settings (immesh_texture_config) in the form the test reads them.
struct TexRule { double min_cos2; int permille, two_sided; };
IM_HD TexRule tex_rule(const immesh_texture_config& cfg) { return TexRule{cfg.min_cos * cfg.min_cos, cfg.min_visible_permille, cfg.two_sided}; }

// Facet q (corners in face order) seen by camera C with won / covered pixels: every corner projects into [0, w-1] x [0, h-1], won >= 1,
// 1000 won >= permille covered, and the angle test on s = n . e (n = (q1 - q0) x (q2 - q0), e = cam_t - g, g the centroid):
// s > 0 (two-sided: s != 0) and s s >= min_cos^2 (|n|^2 |e|^2).  *e2 = |e|^2, the distance the nearest camera is chosen by.
IM_HD bool tex_seen(const DepthCam& C, const float4* q, int won, int covered, const TexRule& r, double* e2) {
    for (int k = 0; k < 3; ++k) {
        double u, v, z;
        depth_project(C, q[k], &u, &v, &z);
        if (!(u >= 0.0 && u <= (double)(C.w - 1) && v >= 0.0 && v <= (double)(C.h - 1))) return false;
    }
    if (won < 1 || 1000LL * won < (long long)r.permille * covered) return false;
    const double P[3][3] = {{q[0].x, q[0].y, q[0].z}, {q[1].x, q[1].y, q[1].z}, {q[2].x, q[2].y, q[2].z}};
    double g[3], e[3];
    for (int k = 0; k < 3; ++k) {
        g[k] = ((P[0][k] + P[1][k]) + P[2][k]) / 3.0;
        e[k] = C.t[k] - g[k];
    }
    const double a[3] = {P[1][0] - P[0][0], P[1][1] - P[0][1], P[1][2] - P[0][2]};
    const double b[3] = {P[2][0] - P[0][0], P[2][1] - P[0][1], P[2][2] - P[0][2]};
    const double n[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    const double s = (n[0] * e[0] + n[1] * e[1]) + n[2] * e[2];
    if (r.two_sided ? !(s != 0.0) : !(s > 0.0)) return false;
    const double nn = (n[0] * n[0] + n[1] * n[1]) + n[2] * n[2], ee = (e[0] * e[0] + e[1] * e[1]) + e[2] * e[2];
    if (!(s * s >= r.min_cos2 * (nn * ee))) return false;
    *e2 = ee;
    return true;
}

// the texture coordinates of the corners in the chosen camera: (float) of the float64 pixel coordinates, u0 v0 u1 v1 u2 v2
IM_HD void tex_uv(const DepthCam& C, const float4* q, float* uv) {
    for (int k = 0; k < 3; ++k) {
        double u, v, z;
        depth_project(C, q[k], &u, &v, &z);
        uv[2 * k] = (float)u;
        uv[2 * k + 1] = (float)v;
    }
}

}  // namespace immesh
