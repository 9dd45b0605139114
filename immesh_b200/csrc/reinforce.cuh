// immesh_b200 -- the LiDAR point-cloud reinforcement (src/ImMesh_node.cpp:302-329 with g_if_depth_bind_cam): the depth camera's pose
// from the last meshed frames (get_last_avr_pose, :169-206) and the depth rasterisation of the live mesh, as __host__ __device__
// bodies shared by the kernels of mesh_render.cu and the host emulation of the tests.
#pragma once
#include <cuda_runtime.h>
#include <cmath>
#include <cstring>

#include "hd_math.cuh"

namespace immesh {

// ---- depth camera (immesh_mesh_render_depth's sampling rule, include/immesh_b200.h): camera frame x right / y down / z forward,
// world = R diag(1,-1,-1) p + t, pixel (u, v) = (fx x / z + cx, fy y / z + cy), samples at integer pixel coordinates.
struct DepthCam { double fx, fy, cx, cy, z_near, z_far; double R[9], t[3]; int w, h; };
IM_HD void depth_project(const DepthCam& C, const float4& p, double* u, double* v, double* z) {
    const double d[3] = {(double)p.x - C.t[0], (double)p.y - C.t[1], (double)p.z - C.t[2]};
    const double xc = (C.R[0] * d[0] + C.R[3] * d[1]) + C.R[6] * d[2];     // R^T d
    const double yc = -((C.R[1] * d[0] + C.R[4] * d[1]) + C.R[7] * d[2]);
    const double zc = -((C.R[2] * d[0] + C.R[5] * d[1]) + C.R[8] * d[2]);
    *z = zc;
    *u = C.fx * xc / zc + C.cx;
    *v = C.fy * yc / zc + C.cy;
}
// one projected triangle: screen vertices, 1/z at the vertices, twice the signed area, pixel box clipped to the image
struct DepthTri { double u0, v0, u1, v1, u2, v2, iz0, iz1, iz2, area; int x_lo, x_hi, y_lo, y_hi; };
// false: the triangle is skipped (a vertex outside (z_near, z_far), zero area, or no sample inside the image)
IM_HD bool depth_tri_setup(const DepthCam& C, const float4& p0, const float4& p1, const float4& p2, DepthTri* T) {
    double z0, z1, z2;
    depth_project(C, p0, &T->u0, &T->v0, &z0);
    depth_project(C, p1, &T->u1, &T->v1, &z1);
    depth_project(C, p2, &T->u2, &T->v2, &z2);
    if (!(z0 > C.z_near && z0 < C.z_far && z1 > C.z_near && z1 < C.z_far && z2 > C.z_near && z2 < C.z_far)) return false;
    const double u0 = T->u0, v0 = T->v0, u1 = T->u1, v1 = T->v1, u2 = T->u2, v2 = T->v2;
    T->area = (u1 - u0) * (v2 - v0) - (v1 - v0) * (u2 - u0);
    if (T->area == 0.0) return false;
    const int xl = (int)ceil(fmin(u0, fmin(u1, u2))), xh = (int)floor(fmax(u0, fmax(u1, u2)));
    const int yl = (int)ceil(fmin(v0, fmin(v1, v2))), yh = (int)floor(fmax(v0, fmax(v1, v2)));
    T->x_lo = xl > 0 ? xl : 0; T->x_hi = xh < C.w - 1 ? xh : C.w - 1;
    T->y_lo = yl > 0 ? yl : 0; T->y_hi = yh < C.h - 1 ? yh : C.h - 1;
    T->iz0 = 1.0 / z0; T->iz1 = 1.0 / z1; T->iz2 = 1.0 / z2;
    return T->x_lo <= T->x_hi && T->y_lo <= T->y_hi;
}
// the sample at pixel (x, y) inside the triangle's box: covered when the three edge functions share a sign (zero included); the
// depth is 1 / (1/z interpolated affinely).  Returns whether the sample writes *zf (> 0).
IM_HD void depth_edges(const DepthTri& T, int x, int y, double* e) {
    const double px = (double)x, py = (double)y;
    e[0] = (T.u2 - T.u1) * (py - T.v1) - (T.v2 - T.v1) * (px - T.u1);   // weight of vertex 0
    e[1] = (T.u0 - T.u2) * (py - T.v2) - (T.v0 - T.v2) * (px - T.u2);
    e[2] = (T.u1 - T.u0) * (py - T.v0) - (T.v1 - T.v0) * (px - T.u0);
}
IM_HD bool depth_sample(const DepthTri& T, int x, int y, float* zf) {
    double e[3];
    depth_edges(T, x, y, e);
    const double e0 = e[0], e1 = e[1], e2 = e[2];
    if (!((e0 >= 0 && e1 >= 0 && e2 >= 0) || (e0 <= 0 && e1 <= 0 && e2 <= 0))) return false;
    const double iz = ((e0 * T.iz0 + e1 * T.iz1) + e2 * T.iz2) / T.area;
    *zf = (float)(1.0 / iz);
    return *zf > 0.f;
}

// convert_depth_buffer_to_truth_depth's validity rule (val < 0.99 z_far) and unproject_point (openGL_camera_view.cpp:407-414):
// m_camera_intrinsic_inv (x, y, 1) scaled to depth val, GL camera axes (x, -y, -z), then R p + t
IM_HD bool depth_valid(const DepthCam& C, float val) { return (double)val < C.z_far * 0.99; }
IM_HD void depth_unproject(const DepthCam& C, int x, int y, float val, float* out) {
    const double sx = ((double)x - C.cx) / C.fx, sy = ((double)y - C.cy) / C.fy;
    const double g[3] = {sx * (double)val, -(sy * (double)val), -(double)val};
    for (int a = 0; a < 3; ++a) out[a] = (float)(((C.R[a * 3 + 0] * g[0] + C.R[a * 3 + 1] * g[1]) + C.R[a * 3 + 2] * g[2]) + C.t[a]);
}

// ---- tiled rasteriser: square screen tiles of IM_RT_TILE pixels a side, one thread block (one thread per pixel) per tile
#define IM_RT_TILE 16
#define IM_RT_THREADS (IM_RT_TILE * IM_RT_TILE)
// the nearest surface over triangles tris[0, n) at pixel (x, y), as the bits of a positive float (+inf: none); unsigned order of
// the bits is the order of the floats, so the result is the nearest sample whatever the order of the triangles
IM_HD unsigned int rt_pixel_min(const DepthTri* tris, int n, int x, int y, unsigned int acc) {
    for (int j = 0; j < n; ++j) {
        const DepthTri& T = tris[j];
        if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
        float zf;
        if (depth_sample(T, x, y, &zf)) {
            unsigned int b;
            memcpy(&b, &zf, 4);
            acc = b < acc ? b : acc;
        }
    }
    return acc;
}

// ---- the shaded view (immesh_mesh_render_view's image rule, include/immesh_b200.h): the viewer's facet shader (if_light, face mode)
// at the winning sample of the same rasteriser.
// the vertex position drawn: pos_mode 0 the raw position; 1 the stored smoothed position (as float) where m_smoothed is set
IM_HD float4 view_vertex(const float4* vpos, const double* vsmooth, const unsigned char* vsmoothed, int pos_mode, int v) {
    if (pos_mode == 1 && vsmoothed && vsmoothed[v])
        return make_float4((float)vsmooth[(size_t)v * 3 + 0], (float)vsmooth[(size_t)v * 3 + 1], (float)vsmooth[(size_t)v * 3 + 2], 0.f);
    return vpos[v];
}
// the visibility order: the nearer sample (smaller depth bits) wins; on equal bits the lower (a, b, c) triple
IM_HD bool view_better(unsigned int bits, int a, int b, int c, unsigned int best_bits, int ba, int bb, int bc) {
    if (bits != best_bits) return bits < best_bits;
    if (a != ba) return a < ba;
    if (b != bb) return b < bb;
    return c < bc;
}
// the height colour of one vertex: t = (z - lo) / (hi - lo) in float (0 when hi == lo), s = clamp(1 - t, 0, 1) at 4 s on the ramp
// blue, cyan, green, yellow, red (linear between neighbouring stops), each channel truncated to a byte
IM_HD void view_heat(float z, float lo, float hi, unsigned char* rgb) {
    const float val = hi == lo ? 0.0f : (z - lo) / (hi - lo);
    double s = 1.0 - (double)val;
    s = s < 0.0 ? 0.0 : (s > 1.0 ? 1.0 : s);
    const double a = s * 4.0, i = floor(a), f = a - i;
    // the five stops, channel by channel (r, g, b)
    const double stop[5][3] = {{0, 0, 1}, {0, 1, 1}, {0, 1, 0}, {1, 1, 0}, {1, 0, 0}};
    const int i0 = (int)i, i1 = (int)ceil(a);
    for (int k = 0; k < 3; ++k) rgb[k] = (unsigned char)(((1.0 - f) * stop[i0][k] + f * stop[i1][k]) * 255.0);
}
// a colour channel in [0, 1] to a byte (NaN and below 0 give 0)
IM_HD unsigned char view_byte(double c) {
    const double k = c > 0.0 ? (c < 1.0 ? c : 1.0) : 0.0;
    return (unsigned char)floor(k * 255.0 + 0.5);
}
// the shaded colour of the winning triangle (p[3] in stored order, colours col[3][3] in [0, 1]) at pixel (x, y) of its set-up T,
// lit from the camera position cam_t: face normal, perspective-correct weights e_i / z_i, two-sided diffuse 0.2 + 0.5 |n . l|
IM_HD uchar4 view_shade(const DepthTri& T, int x, int y, const float4* p, const double (*col)[3], const double* cam_t) {
    const double P[3][3] = {{p[0].x, p[0].y, p[0].z}, {p[1].x, p[1].y, p[1].z}, {p[2].x, p[2].y, p[2].z}};
    const double a[3] = {P[1][0] - P[0][0], P[1][1] - P[0][1], P[1][2] - P[0][2]};
    const double b[3] = {P[2][0] - P[0][0], P[2][1] - P[0][1], P[2][2] - P[0][2]};
    const double n[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
    double e[3];
    depth_edges(T, x, y, e);
    const double w0 = e[0] * T.iz0, w1 = e[1] * T.iz1, w2 = e[2] * T.iz2, ws = (w0 + w1) + w2;
    double l[3], c[3];
    for (int k = 0; k < 3; ++k) {
        l[k] = cam_t[k] - ((w0 * P[0][k] + w1 * P[1][k]) + w2 * P[2][k]) / ws;
        c[k] = ((w0 * col[0][k] + w1 * col[1][k]) + w2 * col[2][k]) / ws;
    }
    const double nn = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]), ln = sqrt((l[0] * l[0] + l[1] * l[1]) + l[2] * l[2]);
    const double d = ((n[0] / nn) * (l[0] / ln) + (n[1] / nn) * (l[1] / ln)) + (n[2] / nn) * (l[2] / ln);
    const double s = 0.2 + 0.5 * fabs(d);
    return make_uchar4(view_byte(s * c[0]), view_byte(s * c[1]), view_byte(s * c[2]), 255);
}
// a vertex's colour: white, or the height colour of its z
IM_HD void view_color(int color, float z, float lo, float hi, double* out) {
    if (!color) { out[0] = out[1] = out[2] = 1.0; return; }
    unsigned char rgb[3];
    view_heat(z, lo, hi, rgb);
    for (int k = 0; k < 3; ++k) out[k] = (double)rgb[k] / 255.0;
}
// float min / max through integer atomics: an order-preserving map of the float bits to unsigned int
IM_HD unsigned int view_ordered(float f) {
    unsigned int u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
IM_HD float view_unordered(unsigned int u) {
    u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// ---- get_last_avr_pose (src/ImMesh_node.cpp:169-206) on the poses the mesher's frames used.  Quaternions are (w, x, y, z).
// Eigen::Quaterniond(const Matrix3d&) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl)
IM_HD void rf_quat_from_rot(const double* m /*row-major*/, double* q) {
    const double t = (m[0] + m[4]) + m[8];
    if (t > 0.0) {
        double s = sqrt(t + 1.0);
        q[0] = 0.5 * s;
        s = 0.5 / s;
        q[1] = (m[7] - m[5]) * s;
        q[2] = (m[2] - m[6]) * s;
        q[3] = (m[3] - m[1]) * s;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 4]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        double s = sqrt(((m[i * 4] - m[j * 4]) - m[k * 4]) + 1.0);
        q[1 + i] = 0.5 * s;
        s = 0.5 / s;
        q[0] = (m[k * 3 + j] - m[j * 3 + k]) * s;
        q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * s;
        q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * s;
    }
}
IM_HD void rf_quat_normalize(double* q) {
    const double n = sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
    for (int i = 0; i < 4; ++i) q[i] = q[i] / n;
}
IM_HD void rf_quat_mul(const double* a, const double* b, double* o) {
    const double w = ((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2]) - a[3] * b[3];
    const double x = ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2];
    const double y = ((a[0] * b[2] + a[2] * b[0]) + a[3] * b[1]) - a[1] * b[3];
    const double z = ((a[0] * b[3] + a[3] * b[0]) + a[1] * b[2]) - a[2] * b[1];
    o[0] = w; o[1] = x; o[2] = y; o[3] = z;
}
// Sophus::SO3d(q).log() (src/tools/lib_sophus/so3.hpp:247-290; the constructor normalises q)
IM_HD void rf_so3_log(const double* q_in, double* r) {
    double q[4] = {q_in[0], q_in[1], q_in[2], q_in[3]};
    rf_quat_normalize(q);
    const double sn = (q[1] * q[1] + q[2] * q[2]) + q[3] * q[3], w = q[0], eps = 1e-10;
    double f;
    if (sn < eps * eps) {
        f = 2.0 / w - (2.0 / 3.0) * sn / (w * (w * w));
    } else {
        const double n = sqrt(sn);
        if (fabs(w) < eps) f = (w > 0.0 ? 3.141592653589793 : -3.141592653589793) / n;
        else f = 2.0 * atan(n / w) / n;
    }
    for (int i = 0; i < 3; ++i) r[i] = f * q[1 + i];
}
// Sophus::SO3d::exp(omega).unit_quaternion() (so3.hpp:585-621)
IM_HD void rf_so3_exp(const double* o, double* q) {
    const double th2 = (o[0] * o[0] + o[1] * o[1]) + o[2] * o[2], eps = 1e-10;
    double im, re;
    if (th2 < eps * eps) {
        const double th4 = th2 * th2;
        im = (0.5 - (1.0 / 48.0) * th2) + (1.0 / 3840.0) * th4;
        re = (1.0 - (1.0 / 8.0) * th2) + (1.0 / 384.0) * th4;
    } else {
        const double th = sqrt(th2);
        im = sin(0.5 * th) / th;
        re = cos(0.5 * th);
    }
    q[0] = re; q[1] = im * o[0]; q[2] = im * o[1]; q[3] = im * o[2];
}
// QuaternionBase::toRotationMatrix, row-major
IM_HD void rf_quat_to_rot(const double* q, double* R) {
    const double tx = 2.0 * q[1], ty = 2.0 * q[2], tz = 2.0 * q[3];
    const double twx = tx * q[0], twy = ty * q[0], twz = tz * q[0];
    const double txx = tx * q[1], txy = ty * q[1], txz = tz * q[1];
    const double tyy = ty * q[2], tyz = tz * q[2], tzz = tz * q[3];
    R[0] = 1.0 - (tyy + tzz); R[1] = txy - twz; R[2] = txz + twy;
    R[3] = txy + twz; R[4] = 1.0 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy; R[7] = tyz + twx; R[8] = 1.0 - (txx + tyy);
}
// Poses of the frames the mesher has run: frame f (1-based, the handle's frame counter) left rot_end (row-major) and pos_end in
// ring[f % IM_RF_RING] with ring_frame[f % IM_RF_RING] = f; a frame that had no rotation (world-frame input) left nothing.
#define IM_RF_RING 64
// The camera pose of frame `frame`: frames [max(1, frame - win), frame) with a pose -- the reference's [max(0, cur - win), cur) with
// cur = frame - 1 -- q_first exp(mean log(q_first^-1 q)) lidar_frame_to_camera_frame and the mean translation.  The first frame
// (cur < 1) gets the identity pose, as the reference returns it; so does a window without any pose (the reference divides by zero).
IM_HD void rf_avr_pose(const double (*ring)[12], const int* ring_frame, int frame, int win, double* R, double* t) {
    double q_first[4] = {1, 0, 0, 0}, inv_first[4] = {1, 0, 0, 0}, acc[3] = {0, 0, 0}, ts[3] = {0, 0, 0};
    int count = 0;
    for (int f = frame - win > 1 ? frame - win : 1; f < frame; ++f) {
        const int s = f % IM_RF_RING;
        if (ring_frame[s] != f) continue;
        double q[4];
        rf_quat_from_rot(ring[s], q);
        rf_quat_normalize(q);
        if (count == 0) {
            for (int i = 0; i < 4; ++i) q_first[i] = q[i];
            // Quaternion::inverse(): the conjugate over the squared norm
            const double n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3];
            inv_first[0] = q[0] / n2; inv_first[1] = -q[1] / n2; inv_first[2] = -q[2] / n2; inv_first[3] = -q[3] / n2;
        }
        double d[4], l[3];
        rf_quat_mul(inv_first, q, d);
        rf_so3_log(d, l);
        for (int i = 0; i < 3; ++i) { acc[i] += l[i]; ts[i] += ring[s][9 + i]; }
        ++count;
    }
    if (count == 0) {
        for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
        t[0] = t[1] = t[2] = 0.0;
        return;
    }
    double m[3], e[4], q[4], qc[4];
    for (int i = 0; i < 3; ++i) { t[i] = ts[i] / (double)count; m[i] = acc[i] / (double)count; }
    rf_so3_exp(m, e);
    rf_quat_mul(q_first, e, q);
    rf_quat_normalize(q);
    const double l2c[9] = {0, 0, -1, -1, 0, 0, 0, 1, 0};   // lidar_frame_to_camera_frame (:172-174)
    double c[4];
    rf_quat_from_rot(l2c, c);
    rf_quat_mul(q, c, qc);
    rf_quat_to_rot(qc, R);
}
// A queued image's camera for frame `frame` by its per-frame source: mode 0 the sensor-bound pose (rf_avr_pose); 1 the caller's
// (R_in, t_in); 2 the follow camera (g_follow_cam with tracking_camera(Identity, t_last_avr), ImMesh_node.cpp:434-440): the fixed
// rotation R_in at the window's mean translation plus the offset t_in (a window without a pose: a zero mean translation).
IM_HD void rf_frame_pose(const double (*ring)[12], const int* ring_frame, int frame, int win, int mode, const double* R_in, const double* t_in,
                         double* R, double* t) {
    if (mode == 1) {
        for (int i = 0; i < 9; ++i) R[i] = R_in[i];
        for (int i = 0; i < 3; ++i) t[i] = t_in[i];
        return;
    }
    rf_avr_pose(ring, ring_frame, frame, win, R, t);
    if (mode == 2) {
        for (int i = 0; i < 9; ++i) R[i] = R_in[i];
        for (int i = 0; i < 3; ++i) t[i] = t[i] + t_in[i];
    }
}

}  // namespace immesh
