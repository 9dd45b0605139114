// immesh_b200 -- the texture selection of immesh_mesh_texture_select (texture_capi.cu) and of the texturing queued behind every frame
// (texture_online.cu; both rules are stated in include/immesh_b200.h): the caller's OpenCV camera as the rasteriser's, a facet's
// corners in the PLY face order, the "seen by camera k" test, the nearest camera and the texture coordinates, a frame's texture camera
// and a record's update.  __host__ __device__ bodies shared by the kernels and the host emulation of the tests; float64 in the written
// order (built with -fmad=false on the device and -ffp-contract=off on the host).  The tile kernel both callers share is device-only.
#pragma once
#include <cmath>

#include "../../include/immesh_b200.h"
#include "reinforce.cuh"
#ifdef __CUDACC__
#include <climits>

#include "mesh_core.cuh"
#endif

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

// the camera and config checks of immesh_mesh_texture_select (host side)
inline bool tex_camera_ok(const immesh_texture_camera& c) {
    if (c.width < 1 || c.height < 1 || (long long)c.width * c.height > (1 << 26)) return false;
    const double k[4] = {c.fx, c.fy, c.cx, c.cy};
    for (double v : k) if (!std::isfinite(v)) return false;
    for (double v : c.cam_R) if (!std::isfinite(v)) return false;
    for (double v : c.cam_t) if (!std::isfinite(v)) return false;
    return c.fx != 0.0 && c.fy != 0.0;
}
inline bool tex_config_ok(const immesh_texture_config& c) {
    return c.z_near > 0 && c.z_far > c.z_near && std::isfinite(c.z_far) && c.min_cos >= 0.0 && c.min_cos <= 1.0 && c.min_visible_permille >= 0 &&
           c.min_visible_permille <= 1000 && (c.two_sided == 0 || c.two_sided == 1) && (c.positions == 0 || c.positions == 1);
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


// ---- the texturing queued behind every frame (immesh_mesh_texture_enable)
// Frame f's texture camera: the caller's camera (R_in, t_in) as it is, or the rig (rig.cam_R, rig.cam_t: the colour camera in the frame's
// sensor frame) composed with the frame's sensor pose (R_f, t_f): R = R_f R_rig, t = ((R_f0 t_rig0 + R_f1 t_rig1) + R_f2 t_rig2) + t_f
// per row, every entry summed left to right.  The rig's size and intrinsics in both cases.
IM_HD immesh_texture_camera txo_camera(const immesh_texture_camera& rig, const double* R_f, const double* t_f) {
    immesh_texture_camera c = rig;
    for (int r = 0; r < 3; ++r) {
        for (int k = 0; k < 3; ++k)
            c.cam_R[r * 3 + k] = (R_f[r * 3 + 0] * rig.cam_R[k] + R_f[r * 3 + 1] * rig.cam_R[3 + k]) + R_f[r * 3 + 2] * rig.cam_R[6 + k];
        c.cam_t[r] = ((R_f[r * 3 + 0] * rig.cam_t[0] + R_f[r * 3 + 1] * rig.cam_t[1]) + R_f[r * 3 + 2] * rig.cam_t[2]) + t_f[r];
    }
    return c;
}
IM_HD immesh_texture_camera txo_fixed_camera(const immesh_texture_camera& rig, const double* R_in, const double* t_in) {
    immesh_texture_camera c = rig;
    for (int i = 0; i < 9; ++i) c.cam_R[i] = R_in[i];
    for (int i = 0; i < 3; ++i) c.cam_t[i] = t_in[i];
    return c;
}
// A record's state: the frame that textures it (-1: none), its |e|^2, won and covered pixels there, and the texture coordinates of
// its corners in stored (ascending-id) order, so that a later flip only permutes them.
struct TxoRecord { int frame; double e2; int won, cov; float uv[6]; };
// Frame `frame` at camera C with a live record's stored positions p and current flip, its won / covered pixels: the "seen" test on the
// corners in face order, and a strictly nearer camera replaces the record's choice (a tie keeps the earlier frame).
IM_HD void txo_observe(const DepthCam& C, const float4* p, int flip, int won, int cov, const TexRule& r, int frame, TxoRecord* s) {
    if (won < 1) return;
    float4 q[3];
    tex_corners(p[0], p[1], p[2], flip, q);
    double e2;
    if (!tex_seen(C, q, won, cov, r, &e2) || !(e2 < s->e2)) return;
    s->frame = frame; s->e2 = e2; s->won = won; s->cov = cov;
    tex_uv(C, p, s->uv);
}
// the stored-order coordinates uv_s in the face order of flip (tex_corners): q0 = p0, q1 = flip ? p1 : p2, q2 = flip ? p2 : p1
IM_HD void txo_face_uv(const float* uv_s, int flip, float* uv) {
    const int c[3] = {0, flip ? 1 : 2, flip ? 2 : 1};
    for (int k = 0; k < 3; ++k) { uv[2 * k] = uv_s[2 * c[k]]; uv[2 * k + 1] = uv_s[2 * c[k] + 1]; }
}

#ifdef __CUDACC__
__device__ __forceinline__ float4 tex_vertex(const MeshDev& M, int pos_mode, int v) { return view_vertex(M.vpos, M.vsmooth, M.vsmoothed, pos_mode, v); }
// k_tex_tile counts a slot's pixels at an index of the caller's (immesh_mesh_texture_select: the live record's; texture_gains: the
// snapshot row's)
struct TexRowOf {
    const int* row_of;
    __device__ __forceinline__ int operator()(int slot) const { return row_of[slot]; }
};

// one block per tile, one thread per pixel (k_view_tile's shape and visibility): the bin's set-ups staged IM_RT_THREADS at a time in
// shared memory; a covered sample is counted for its facet (ballot per warp, shared sum per block, one atomic per facet and batch), the
// pixel's winner (depth bits, then the lower triple) gets one won pixel.  Bins over capacity (misc[0]): every triangle slot instead.
// Counts go to index row(slot): the live record's row of immesh_mesh_texture_select, or the slot itself for the queued texturing.
template <class Row>
__global__ void __launch_bounds__(IM_RT_THREADS) k_tex_tile(MeshDev M, int pos_mode, const DepthCam* cam, const int* tile_off, const int* bin, const int* misc,
                                                            Row row, int* won, int* cov) {
    __shared__ DepthTri S[IM_RT_THREADS];
    __shared__ int4 Q[IM_RT_THREADS];   // a b c, row
    __shared__ int s_cov[IM_RT_THREADS];
    const DepthCam C = *cam;
    const int ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE, lane = threadIdx.x & 31;
    const int x = (blockIdx.x % ntx) * IM_RT_TILE + (int)(threadIdx.x % IM_RT_TILE), y = (blockIdx.x / ntx) * IM_RT_TILE + (int)(threadIdx.x / IM_RT_TILE);
    const bool all = misc[0] != 0;
    const int lo = all ? 0 : tile_off[blockIdx.x], hi = all ? min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t) : tile_off[blockIdx.x + 1];
    unsigned int best = 0x7f800000u;   // +inf: nothing drawn
    int ba = INT_MAX, bb = INT_MAX, bc = INT_MAX, brow = -1;
    for (int b = lo; b < hi; b += IM_RT_THREADS) {
        const int i = b + (int)threadIdx.x;
        bool ok = false;
        if (i < hi) {
            const int slot = all ? i : bin[i];
            const int4 r = M.tri[slot];
            ok = r.w && depth_tri_setup(C, tex_vertex(M, pos_mode, r.x), tex_vertex(M, pos_mode, r.y), tex_vertex(M, pos_mode, r.z), &S[threadIdx.x]);
            Q[threadIdx.x] = make_int4(r.x, r.y, r.z, ok ? row(slot) : -1);
        }
        if (!ok) { S[threadIdx.x].x_lo = 1; S[threadIdx.x].x_hi = 0; }   // an empty box
        s_cov[threadIdx.x] = 0;
        __syncthreads();
        const int n = min(IM_RT_THREADS, hi - b);
        for (int j = 0; j < n; ++j) {   // uniform over the block: every lane reaches the ballot
            const DepthTri& T = S[j];
            bool c = false;
            unsigned int bits = 0;
            if (x >= T.x_lo && x <= T.x_hi && y >= T.y_lo && y <= T.y_hi) {
                float zf;
                if (depth_sample(T, x, y, &zf)) { bits = __float_as_uint(zf); c = bits < 0x7f800000u; }
            }
            const unsigned int m = __ballot_sync(0xffffffffu, c);
            if (lane == 0 && m) atomicAdd(&s_cov[j], __popc(m));
            const int4 q = Q[j];
            if (c && view_better(bits, q.x, q.y, q.z, best, ba, bb, bc)) { best = bits; ba = q.x; bb = q.y; bc = q.z; brow = q.w; }
        }
        __syncthreads();
        if ((int)threadIdx.x < n && s_cov[threadIdx.x]) atomicAdd(&cov[Q[threadIdx.x].w], s_cov[threadIdx.x]);
        __syncthreads();
    }
    if (brow >= 0) atomicAdd(&won[brow], 1);
}

#endif

}  // namespace immesh
