// immesh_b200 -- the overlays of the queued mesh view (immesh_mesh_view_overlay, include/immesh_b200.h): what the reference's main
// loop draws into the viewer's window besides the faces (src/ImMesh_node.cpp:422-470) -- the current scan, the reinforced points,
// the axis, the ground grid, the wireframe, the sensor's camera frustum and the trajectory -- as __host__ __device__ bodies shared by
// the kernels of mesh_render.cu and the host emulation of the tests.  Everything is float64 in the order written, without fused
// multiply-adds (the library is built with -fmad=false).
#pragma once
#include "reinforce.cuh"

namespace immesh {

// the layers in the reference's draw order: on equal depth bits the earlier layer wins (GL_LESS)
enum { OV_SCAN = 0, OV_REINFORCED = 1, OV_AXIS = 2, OV_GRID = 3, OV_MESH = 4, OV_CAMERA = 5, OV_PATH = 6 };
#define OV_AXIS_WIDTH 10       // g_axis_shader's m_pts_size
#define OV_GRID_WIDTH 1        // g_ground_plane_shader's m_pts_size
#define OV_CAMERA_WIDTH 5      // draw_camera_pose: set_point_attr(5, ...)
#define OV_WIRE_WIDTH 1        // draw_triangle with g_display_face = 0
#define OV_N_AXIS 3
#define OV_N_GRID 42           // init(SHADER_DIR, 10, 10): 21 lines along y, 21 along x, 10 m apart, from -100 m to 100 m
#define OV_N_CAMERA 10         // the frustum's 11-vertex line strip
#define OV_IDX_BITS 29         // the primitive index inside a layer in the overlay key
#define OV_NONE 0xffffffffffffffffull

// a point in the depth camera's frame (depth_project's arithmetic on float64 input)
IM_HD void ov_cam_point(const DepthCam& C, const double* p, double* c) {
    const double d[3] = {p[0] - C.t[0], p[1] - C.t[1], p[2] - C.t[2]};
    c[0] = (C.R[0] * d[0] + C.R[3] * d[1]) + C.R[6] * d[2];
    c[1] = -((C.R[1] * d[0] + C.R[4] * d[1]) + C.R[7] * d[2]);
    c[2] = -((C.R[2] * d[0] + C.R[5] * d[1]) + C.R[8] * d[2]);
}

// ---- points: a point of size s at (u, v) covers the integer pixels u - s/2 <= x < u + s/2, v - s/2 <= y < v + s/2 (cut to the
// image), drawn when z_near < z < z_far, its depth the camera z as float.  emit(x, y, zf) once per covered pixel.
template <class Emit>
IM_HD void ov_point_raster(const DepthCam& C, const double* p, int size, Emit emit) {
    double c[3];
    ov_cam_point(C, p, c);
    if (!(c[2] > C.z_near && c[2] < C.z_far)) return;
    const double u = C.fx * c[0] / c[2] + C.cx, v = C.fy * c[1] / c[2] + C.cy, hs = (double)size * 0.5;
    const double x0 = ceil(u - hs), y0 = ceil(v - hs);
    const float zf = (float)c[2];
    for (double y = y0 > 0.0 ? y0 : 0.0; y < v + hs && y < (double)C.h; y += 1.0)
        for (double x = x0 > 0.0 ? x0 : 0.0; x < u + hs && x < (double)C.w; x += 1.0) emit((int)x, (int)y, zf);
}

// ---- segments: clipped in camera space to [z_near, z_far], then projected.  u, v the pixel coordinates and iz = 1/z of the ends.
struct OvSeg { double u0, v0, iz0, u1, v1, iz1; };
// the end a moved along a -> b to the plane z = zp
IM_HD void ov_clip_end(double* a, const double* b, double zp) {
    const double s = (zp - a[2]) / (b[2] - a[2]);
    a[0] = a[0] + s * (b[0] - a[0]);
    a[1] = a[1] + s * (b[1] - a[1]);
    a[2] = zp;
}
IM_HD void ov_project(const DepthCam& C, const double* c, double* u, double* v, double* iz) {
    *u = C.fx * c[0] / c[2] + C.cx;
    *v = C.fy * c[1] / c[2] + C.cy;
    *iz = 1.0 / c[2];
}
// false: nothing of the segment p0 -> p1 lies in [z_near, z_far]
IM_HD bool ov_seg_setup(const DepthCam& C, const double* p0, const double* p1, OvSeg* S) {
    double a[3], b[3];
    ov_cam_point(C, p0, a);
    ov_cam_point(C, p1, b);
    if (!(a[2] >= C.z_near || b[2] >= C.z_near) || !(a[2] <= C.z_far || b[2] <= C.z_far)) return false;   // wholly outside (or NaN)
    if (a[2] < C.z_near) ov_clip_end(a, b, C.z_near);
    else if (b[2] < C.z_near) ov_clip_end(b, a, C.z_near);
    if (a[2] > C.z_far) ov_clip_end(a, b, C.z_far);
    else if (b[2] > C.z_far) ov_clip_end(b, a, C.z_far);
    ov_project(C, a, &S->u0, &S->v0, &S->iz0);
    ov_project(C, b, &S->u1, &S->v1, &S->iz1);
    return true;
}
// GL's wide non-antialiased line of width w: x-major when |du| >= |dv|, covering the integer columns min(u0, u1) <= x < max(u0, u1);
// in a column, t = (x - u0) / (u1 - u0), v = v0 + t (v1 - v0), the rows v - w/2 <= y < v + w/2; 1/z = iz0 + t (iz1 - iz0).  A
// y-major line swaps the axes.  (Major axis m, minor axis n below.)
IM_HD bool ov_seg_xmajor(const OvSeg& S) { return fabs(S.u1 - S.u0) >= fabs(S.v1 - S.v0); }
// the fragment at major coordinate m: its parameter, minor coordinate and float depth
IM_HD void ov_seg_at(const OvSeg& S, bool xm, double m, double* t, double* n, float* zf) {
    const double m0 = xm ? S.u0 : S.v0, m1 = xm ? S.u1 : S.v1, n0 = xm ? S.v0 : S.u0, n1 = xm ? S.v1 : S.u1;
    *t = (m - m0) / (m1 - m0);
    *n = n0 + *t * (n1 - n0);
    *zf = (float)(1.0 / (S.iz0 + *t * (S.iz1 - S.iz0)));
}
// every covered pixel inside the image: emit(x, y, zf, t); the major coordinates first, first + step, ... of the covered ones (a
// warp's lanes split them)
template <class Emit>
IM_HD void ov_seg_raster(const DepthCam& C, const OvSeg& S, int width, int first, int step, Emit emit) {
    const bool xm = ov_seg_xmajor(S);
    const double hw = (double)width * 0.5;
    const double m0 = xm ? S.u0 : S.v0, m1 = xm ? S.u1 : S.v1, mlim = (double)(xm ? C.w : C.h), nlim = (double)(xm ? C.h : C.w);
    const double lo = fmin(m0, m1), hi = fmax(m0, m1), mstart = ceil(lo);
    for (double m = (mstart > 0.0 ? mstart : 0.0) + (double)first; m < hi && m < mlim; m += (double)step) {
        double t, n;
        float zf;
        ov_seg_at(S, xm, m, &t, &n, &zf);
        const double nstart = ceil(n - hw);
        for (double k = nstart > 0.0 ? nstart : 0.0; k < n + hw && k < nlim; k += 1.0)
            xm ? emit((int)m, (int)k, zf, t) : emit((int)k, (int)m, zf, t);
    }
}
// the same rule for one pixel (the wireframe, evaluated per pixel of a tile): whether (x, y) is covered, with its depth and parameter
IM_HD bool ov_seg_pixel(const OvSeg& S, int width, int x, int y, float* zf, double* t) {
    const bool xm = ov_seg_xmajor(S);
    const double m = (double)(xm ? x : y), k = (double)(xm ? y : x), hw = (double)width * 0.5;
    const double m0 = xm ? S.u0 : S.v0, m1 = xm ? S.u1 : S.v1;
    if (!(m >= fmin(m0, m1) && m < fmax(m0, m1))) return false;
    double n;
    ov_seg_at(S, xm, m, t, &n, zf);
    return k >= n - hw && k < n + hw;
}

// ---- the overlay key: per pixel, the 64-bit minimum over the overlay fragments of (depth bits, layer, index in the layer) -- the
// nearest fragment, on equal bits the earlier layer, then the lower index.  Positive float depths order as their bits.
IM_HD unsigned long long ov_key(float zf, int layer, unsigned int idx) {
    unsigned int bits;
    memcpy(&bits, &zf, 4);
    return ((unsigned long long)bits << 32) | ((unsigned long long)layer << OV_IDX_BITS) | idx;
}
// whether the overlay fragment of key k is drawn over the mesh's best sample (depth bits mesh_bits; 0x7f800000: none): nearer, or
// as near and from a layer drawn before the mesh
IM_HD bool ov_over_mesh(unsigned long long k, unsigned int mesh_bits) {
    if (k == OV_NONE) return false;
    const unsigned int bits = (unsigned int)(k >> 32);
    return bits < mesh_bits || (bits == mesh_bits && (int)((k >> OV_IDX_BITS) & 7u) < OV_MESH);
}
// the colour of an overlay fragment by its key: scan and camera and path white, reinforced points magenta, the axes red / green /
// blue, the grid grey 0.45 (view_byte: 115); opaque
IM_HD uchar4 ov_color(unsigned long long k) {
    const int layer = (int)((k >> OV_IDX_BITS) & 7u), idx = (int)(k & ((1u << OV_IDX_BITS) - 1));
    if (layer == OV_REINFORCED) return make_uchar4(255, 0, 255, 255);
    if (layer == OV_AXIS) return make_uchar4(idx == 0 ? 255 : 0, idx == 1 ? 255 : 0, idx == 2 ? 255 : 0, 255);
    if (layer == OV_GRID) { const unsigned char g = view_byte(0.45); return make_uchar4(g, g, g, 255); }
    return make_uchar4(255, 255, 255, 255);
}

// ---- the fixed geometry
// axis k (g_axis_shader, init(SHADER_DIR, 1)): from the origin 1 m along x, y, z
IM_HD void ov_axis(int k, double* p0, double* p1) {
    for (int i = 0; i < 3; ++i) { p0[i] = 0.0; p1[i] = i == k ? 1.0 : 0.0; }
}
// grid line k (Ground_plane_shader::init_pts(10, 10)): i = k / 2 - 10; k even (10 i, -100, 0) -> (10 i, 100, 0), odd (-100, 10 i, 0)
// -> (100, 10 i, 0)
IM_HD void ov_grid(int k, double* p0, double* p1) {
    const double c = (double)(k / 2 - 10) * 10.0;
    if (k % 2 == 0) { p0[0] = c; p0[1] = -100.0; p1[0] = c; p1[1] = 100.0; }
    else { p0[0] = -100.0; p0[1] = c; p1[0] = 100.0; p1[1] = c; }
    p0[2] = p1[2] = 0.0;
}
// The sensor's camera frustum (draw_camera_pose, mesh_rec_display.cpp:297-313; Camera_pose_shader::init_camera_frustum_vertex with the
// hard-coded K and 1440 x 1080 at scale 1.5): the 11 vertices of its line strip in the world, from rot_end R (row-major) and pos_end t
// of the frame, camera size cs: with fu = 1 / fx, u0 = -cx / fx (fv, v0 likewise), xl = 1.5 u0, xh = 1.5 (1440 fu + u0), yl = 1.5 v0,
// yh = 1.5 (1080 fv + v0), the local vertices (xl,yl,1.5) (xh,yl,1.5) (xh,yh,1.5) (xl,yh,1.5) (xl,yl,1.5) 0 (xh,yl,1.5) 0 (xl,yh,1.5) 0
// (xh,yh,1.5), and world_k = t_k + cs ((M_k0 x + M_k1 y) + M_k2 z) with M = R [0 0 1; -1 0 0; 0 -1 0] = [-R_1 -R_2 R_0] by columns.
IM_HD void ov_frustum(const double* R, const double* t, double cs, double (*out)[3]) {
    const double fx = 704.504153913163, cx = 708.8501128392297, fy = 703.6790228113778, cy = 562.7041625276061, s = 1.5;
    const double fu = 1.0 / fx, u0 = -cx / fx, fv = 1.0 / fy, v0 = -cy / fy;
    const double xl = s * u0, xh = s * (1440.0 * fu + u0), yl = s * v0, yh = s * (1080.0 * fv + v0);
    const double loc[11][3] = {{xl, yl, s}, {xh, yl, s}, {xh, yh, s}, {xl, yh, s}, {xl, yl, s}, {0, 0, 0},
                               {xh, yl, s}, {0, 0, 0}, {xl, yh, s}, {0, 0, 0}, {xh, yh, s}};
    for (int i = 0; i < 11; ++i)
        for (int k = 0; k < 3; ++k) {
            const double m0 = -R[k * 3 + 1], m1 = -R[k * 3 + 2], m2 = R[k * 3 + 0];
            out[i][k] = t[k] + cs * ((m0 * loc[i][0] + m1 * loc[i][1]) + m2 * loc[i][2]);
        }
}

// the overlays of a queued view (immesh_mesh_view_overlay; on = 0: none), passed to the kernels by value
struct ViewOverlay {
    int on, wire, scan_size, reinforced_size, axis_and_grid, path_width, path_cap, npx;
    double camera_size;
    double (*path)[3];          // [path_cap] the trajectory's positions, position k in path[k % path_cap]
    int* path_n;                // positions recorded since the overlay was set
    double (*frustum)[3];       // [11] the frame's camera frustum
    int* frustum_on;            // the frame has one
    unsigned long long* key;    // [npx] the per-pixel overlay key (OV_NONE: no fragment)
};
// the segments of the line layers in draw order: axis (3) and grid (42) with axis_and_grid, the frustum's 10 when the frame has one,
// the trajectory's n - 1 over its n kept positions (oldest first).  Segment i -> its layer, index in the layer and ends; false past the end.
IM_HD int ov_path_kept(const ViewOverlay& O, int path_n) { return O.path_width > 0 ? (path_n < O.path_cap ? path_n : O.path_cap) : 0; }
IM_HD bool ov_line(const ViewOverlay& O, int frustum_on, int path_n, int i, int* layer, int* idx, int* width, double* p0, double* p1) {
    if (O.axis_and_grid) {
        if (i < OV_N_AXIS) { *layer = OV_AXIS; *idx = i; *width = OV_AXIS_WIDTH; ov_axis(i, p0, p1); return true; }
        i -= OV_N_AXIS;
        if (i < OV_N_GRID) { *layer = OV_GRID; *idx = i; *width = OV_GRID_WIDTH; ov_grid(i, p0, p1); return true; }
        i -= OV_N_GRID;
    }
    if (frustum_on) {
        if (i < OV_N_CAMERA) {
            *layer = OV_CAMERA; *idx = i; *width = OV_CAMERA_WIDTH;
            for (int k = 0; k < 3; ++k) { p0[k] = O.frustum[i][k]; p1[k] = O.frustum[i + 1][k]; }
            return true;
        }
        i -= OV_N_CAMERA;
    }
    const int kept = ov_path_kept(O, path_n);
    if (i < kept - 1) {
        const int first = path_n - kept;
        *layer = OV_PATH; *idx = i; *width = O.path_width;
        for (int k = 0; k < 3; ++k) { p0[k] = O.path[(first + i) % O.path_cap][k]; p1[k] = O.path[(first + i + 1) % O.path_cap][k]; }
        return true;
    }
    return false;
}

// k_ov_begin's per-frame step: the frame's position (a localization frame's pos_end, a world-frame push's pose_t: both are its
// FramePose::pose_t) appended to the trajectory, and the frame's camera frustum from the camera ring (a world-frame push carries no
// rotation: none)
IM_HD void ov_begin_frame(const ViewOverlay& O, int frame, const double* pose_t, const double (*ring)[12], const int* ring_frame) {
    if (O.path_width > 0) {
        const int n = *O.path_n;
        for (int k = 0; k < 3; ++k) O.path[n % O.path_cap][k] = pose_t[k];
        *O.path_n = n + 1;
    }
    const int s = frame % IM_RF_RING;
    const int on = O.camera_size > 0.0 && ring_frame[s] == frame;
    if (on) ov_frustum(ring[s], ring[s] + 9, O.camera_size, O.frustum);
    *O.frustum_on = on;
}

// ---- the wireframe (draw_triangle with g_display_face = 0): the three edges (a, b), (b, c), (a, c) of each triangle the face rule
// would rasterise with every vertex inside (z_near, z_far), each from its lower vertex id to its higher one, width OV_WIRE_WIDTH.
// The set-up keeps the face's values (T: screen vertices, 1/z, area) with the pixel box widened to every pixel an edge can cover,
// and the face's own pixel box in *face (empty when the face rule skips the triangle: zero area, or no sample in the image).
IM_HD bool view_wire_setup(const DepthCam& C, const float4& p0, const float4& p1, const float4& p2, DepthTri* T, int4* face) {
    double z0, z1, z2;
    depth_project(C, p0, &T->u0, &T->v0, &z0);
    depth_project(C, p1, &T->u1, &T->v1, &z1);
    depth_project(C, p2, &T->u2, &T->v2, &z2);
    *face = make_int4(1, 0, 1, 0);
    if (!(z0 > C.z_near && z0 < C.z_far && z1 > C.z_near && z1 < C.z_far && z2 > C.z_near && z2 < C.z_far)) return false;
    const double u0 = T->u0, v0 = T->v0, u1 = T->u1, v1 = T->v1, u2 = T->u2, v2 = T->v2;
    T->area = (u1 - u0) * (v2 - v0) - (v1 - v0) * (u2 - u0);
    T->iz0 = 1.0 / z0; T->iz1 = 1.0 / z1; T->iz2 = 1.0 / z2;
    const double ul = fmin(u0, fmin(u1, u2)), uh = fmax(u0, fmax(u1, u2)), vl = fmin(v0, fmin(v1, v2)), vh = fmax(v0, fmax(v1, v2));
    if (T->area != 0.0) {
        const int xl = (int)ceil(ul), xh = (int)floor(uh), yl = (int)ceil(vl), yh = (int)floor(vh);
        const int4 f = make_int4(xl > 0 ? xl : 0, xh < C.w - 1 ? xh : C.w - 1, yl > 0 ? yl : 0, yh < C.h - 1 ? yh : C.h - 1);
        if (f.x <= f.y && f.z <= f.w) *face = f;
    }
    // an edge fragment lies within half the width of the edge's box; one pixel more covers the rounding of v = v0 + t (v1 - v0)
    const double pad = (double)OV_WIRE_WIDTH * 0.5 + 1.0;
    const double bx0 = floor(ul - pad), bx1 = ceil(uh + pad), by0 = floor(vl - pad), by1 = ceil(vh + pad);
    if (bx1 < 0.0 || by1 < 0.0 || bx0 > (double)(C.w - 1) || by0 > (double)(C.h - 1)) return false;
    T->x_lo = bx0 > 0.0 ? (int)bx0 : 0; T->x_hi = bx1 < (double)(C.w - 1) ? (int)bx1 : C.w - 1;
    T->y_lo = by0 > 0.0 ? (int)by0 : 0; T->y_hi = by1 < (double)(C.h - 1) ? (int)by1 : C.h - 1;
    return true;
}
// edge e (0: (a, b), 1: (b, c), 2: (a, c)) of a set-up triangle as a segment
IM_HD OvSeg view_wire_edge(const DepthTri& T, int e) {
    OvSeg S;
    const int i = e == 1 ? 1 : 0, j = e == 0 ? 1 : 2;
    S.u0 = i == 0 ? T.u0 : T.u1; S.v0 = i == 0 ? T.v0 : T.v1; S.iz0 = i == 0 ? T.iz0 : T.iz1;
    S.u1 = j == 1 ? T.u1 : T.u2; S.v1 = j == 1 ? T.v1 : T.v2; S.iz1 = j == 1 ? T.iz1 : T.iz2;
    return S;
}
// the edge order on equal depth bits: the lower (a, b, c) triple, then the lower edge
IM_HD bool view_wire_better(unsigned int bits, int a, int b, int c, int e, unsigned int best_bits, int ba, int bb, int bc, int be) {
    if (bits != best_bits || a != ba || b != bb || c != bc) return view_better(bits, a, b, c, best_bits, ba, bb, bc);
    return e < be;
}
// the wireframe's pixel best over one triangle: its face sample (into *face_bits, the depth image's minimum) and its three edges
IM_HD void view_wire_pixel(const DepthTri& T, const int4& fb, int a, int b, int c, int slot, int x, int y, unsigned int* face_bits,
                           unsigned int* best, int* ba, int* bb, int* bc, int* be, int* bs) {
    if (x >= fb.x && x <= fb.y && y >= fb.z && y <= fb.w) {
        float zf;
        if (depth_sample(T, x, y, &zf)) {
            unsigned int u;
            memcpy(&u, &zf, 4);
            if (u < *face_bits) *face_bits = u;
        }
    }
    for (int e = 0; e < 3; ++e) {
        float zf;
        double t;
        if (!ov_seg_pixel(view_wire_edge(T, e), OV_WIRE_WIDTH, x, y, &zf, &t)) continue;
        unsigned int u;
        memcpy(&u, &zf, 4);
        if (u < 0x7f800000u && view_wire_better(u, a, b, c, e, *best, *ba, *bb, *bc, *be)) { *best = u; *ba = a; *bb = b; *bc = c; *be = e; *bs = slot; }
    }
}
// the colour of the winning edge e of the triangle p[3] (stored order) at (x, y): the vertex colours col of its two ends mixed
// perspective-correctly, w0 = (1 - t) iz0, w1 = t iz1, c = (w0 c0 + w1 c1) / (w0 + w1), unlit, bytes by view_byte
IM_HD uchar4 view_wire_color(const DepthCam& C, const float4* p, const double (*col)[3], int e, int x, int y) {
    DepthTri T;
    int4 fb;
    view_wire_setup(C, p[0], p[1], p[2], &T, &fb);
    const OvSeg S = view_wire_edge(T, e);
    float zf;
    double t = 0.0;
    ov_seg_pixel(S, OV_WIRE_WIDTH, x, y, &zf, &t);
    const int i = e == 1 ? 1 : 0, j = e == 0 ? 1 : 2;
    const double w0 = (1.0 - t) * S.iz0, w1 = t * S.iz1;
    unsigned char ch[3];
    for (int k = 0; k < 3; ++k) ch[k] = view_byte((w0 * col[i][k] + w1 * col[j][k]) / (w0 + w1));
    return make_uchar4(ch[0], ch[1], ch[2], 255);
}

}  // namespace immesh
