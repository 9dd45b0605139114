// immesh_b200 -- the mesher's rasteriser outputs: the depth image, the queued reinforcement, the shaded view (a call's or queued) and
// its overlays.  CUDA kernels (sm_90a, bodies in reinforce.cuh / view_overlay.cuh) and their C-ABI host orchestration.
#include <climits>
#include <cmath>

#include "block_scan.cuh"
#include "handles.hpp"

using namespace immesh;

// ---- depth rasterisation of the live mesh ("LiDAR point-cloud reinforcement", src/ImMesh_node.cpp:305-329: draw_triangle into a depth
// camera, Cam_view::read_depth, convert_depth_buffer_to_truth_depth + unproject_point, src/tools/openGL_libs/openGL_camera_view.cpp:316-
// 418).  The reference lets OpenGL rasterise; here a CUDA rasteriser with a defined sampling rule produces the metric depth directly:
// camera frame x right / y down / z forward (the frame unproject_point inverts: world = R diag(1,-1,-1) p + t), pixel (u, v) =
// (fx x / z + cx, fy y / z + cy), samples at integer pixel coordinates, a sample is covered when the three edge functions have one
// sign (zero included), depth interpolated perspective-correctly (1/z is affine in the image), nearest surface wins.  Triangles with a
// vertex outside (z_near, z_far) are skipped (GL would clip them).  DepthCam, the triangle set-up and the sample are in reinforce.cuh.
// One image (rf_image_launch): the tiled rasteriser (k_rf_count -> k_rf_scan -> k_rf_fill -> k_rf_tile) and the compaction of the
// valid pixels in ascending pixel order (k_rf_fcount -> k_rf_scan -> k_rf_emit).  The blocking immesh_mesh_render_depth runs it at the
// caller's pose; the queued reinforcement (immesh_mesh_reinforce_enable) runs it behind every frame, on the mesh stream and inside its
// graph, after the camera pose (k_rf_pose), into result buffer (frame & 1).
struct RfDyn { int mode, pad; double R[9], t[3]; };   // per frame: rf_frame_pose's source (1 = the caller's pose, 2 = the view's follow camera)
// one block: the frame's camera (sensor-bound or the caller's), the tile counters cleared
__global__ void __launch_bounds__(256) k_rf_pose(const double (*ring)[12], const int* ring_frame, const FrameDyn* dyn, const RfDyn* rd, int win, DepthCam base,
                                                 DepthCam* cam, RfOut o0, RfOut o1, int* tile_cnt, int ntiles) {
    for (int i = threadIdx.x; i < ntiles; i += blockDim.x) tile_cnt[i] = 0;
    if (threadIdx.x != 0) return;
    const int frame = dyn->frame;
    double R[9], t[3];
    rf_frame_pose(ring, ring_frame, frame, win, rd->mode, rd->R, rd->t, R, t);
    for (int i = 0; i < 9; ++i) base.R[i] = R[i];
    for (int i = 0; i < 3; ++i) base.t[i] = t[i];
    *cam = base;
    double* pose = (frame & 1) ? o1.pose : o0.pose;
    for (int i = 0; i < 9; ++i) pose[i] = R[i];
    for (int i = 0; i < 3; ++i) pose[9 + i] = t[i];
}
// the position a binning pass reads (view_vertex; pos_mode 0, the depth image's, is M.vpos)
__device__ __forceinline__ float4 rf_vertex(const MeshDev& M, int pos_mode, int v) { return view_vertex(M.vpos, M.vsmooth, M.vsmoothed, pos_mode, v); }
// the screen tiles a triangle's pixel box touches
__device__ __forceinline__ void rf_tiles(const DepthTri& T, int* tx0, int* tx1, int* ty0, int* ty1) {
    *tx0 = T.x_lo / IM_RT_TILE; *tx1 = T.x_hi / IM_RT_TILE; *ty0 = T.y_lo / IM_RT_TILE; *ty1 = T.y_hi / IM_RT_TILE;
}
// a triangle's set-up for the bins: the face rule's (depth_tri_setup), or with `wire` the wireframe's widened box (view_wire_setup)
__device__ __forceinline__ bool rf_bin_setup(const DepthCam& C, const MeshDev& M, int pos_mode, int wire, const int4& r, DepthTri* T) {
    const float4 p0 = rf_vertex(M, pos_mode, r.x), p1 = rf_vertex(M, pos_mode, r.y), p2 = rf_vertex(M, pos_mode, r.z);
    if (!wire) return depth_tri_setup(C, p0, p1, p2, T);
    int4 fb;
    return view_wire_setup(C, p0, p1, p2, T, &fb);
}
// count pass: bin entries per tile (positions by pos_mode; boxes of the wireframe with `wire`)
__global__ void __launch_bounds__(128) k_rf_count(MeshDev M, int pos_mode, int wire, const DepthCam* cam, int* tile_cnt) {
    const DepthCam C = *cam;
    const int n_alloc = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t), ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        DepthTri T;
        if (!rf_bin_setup(C, M, pos_mode, wire, r, &T)) continue;
        int tx0, tx1, ty0, ty1;
        rf_tiles(T, &tx0, &tx1, &ty0, &ty1);
        for (int ty = ty0; ty <= ty1; ++ty)
            for (int tx = tx0; tx <= tx1; ++tx) atomicAdd(&tile_cnt[ty * ntx + tx], 1);
    }
}
// one block: exclusive scan of cnt[0, n) into off[0, n] (off[n] = total); cur (or null, or cnt itself) gets a copy of the offsets,
// the fill cursors; misc[0] (or null) = total > cap, the bins' overflow flag
__global__ void __launch_bounds__(1024) k_rf_scan(const int* cnt, int n, int* off, int* cur, int cap, int* misc) {
    const int total = chunk_scan_1024(n, [&](int c) { return cnt[c]; }, [&](int c, int run) {
        const int k = cnt[c];
        off[c] = run;
        if (cur) cur[c] = run;
        return k;
    });
    if (threadIdx.x == 1023) {
        off[n] = total;
        if (misc) misc[0] = total > cap ? 1 : 0;
    }
}
// fill pass: triangle slots into the bins (order inside a bin is free: the tile takes the minimum)
__global__ void __launch_bounds__(128) k_rf_fill(MeshDev M, int pos_mode, int wire, const DepthCam* cam, int* cur, int* bin, const int* misc) {
    if (misc[0]) return;
    const DepthCam C = *cam;
    const int n_alloc = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t), ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        DepthTri T;
        if (!rf_bin_setup(C, M, pos_mode, wire, r, &T)) continue;
        int tx0, tx1, ty0, ty1;
        rf_tiles(T, &tx0, &tx1, &ty0, &ty1);
        for (int ty = ty0; ty <= ty1; ++ty)
            for (int tx = tx0; tx <= tx1; ++tx) bin[atomicAdd(&cur[ty * ntx + tx], 1)] = t;
    }
}
// one block per tile, one thread per pixel: the bin's triangles are set up IM_RT_THREADS at a time into shared memory, each thread
// keeps its pixel's nearest sample in a register and writes it once.  Bins over capacity (misc[0]): every triangle slot instead.
__global__ void __launch_bounds__(IM_RT_THREADS) k_rf_tile(MeshDev M, const DepthCam* cam, const int* tile_off, const int* bin, const int* misc, unsigned int* depth) {
    __shared__ DepthTri S[IM_RT_THREADS];
    const DepthCam C = *cam;
    const int ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    const int x = (blockIdx.x % ntx) * IM_RT_TILE + (int)(threadIdx.x % IM_RT_TILE), y = (blockIdx.x / ntx) * IM_RT_TILE + (int)(threadIdx.x / IM_RT_TILE);
    const bool all = misc[0] != 0;
    const int lo = all ? 0 : tile_off[blockIdx.x], hi = all ? min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t) : tile_off[blockIdx.x + 1];
    unsigned int acc = 0x7f800000u;   // +inf
    for (int b = lo; b < hi; b += IM_RT_THREADS) {
        const int i = b + (int)threadIdx.x;
        bool ok = false;
        if (i < hi) {
            const int4 r = M.tri[all ? i : bin[i]];
            ok = r.w && depth_tri_setup(C, M.vpos[r.x], M.vpos[r.y], M.vpos[r.z], &S[threadIdx.x]);
        }
        if (!ok) { S[threadIdx.x].x_lo = 1; S[threadIdx.x].x_hi = 0; }   // an empty box
        __syncthreads();
        acc = rt_pixel_min(S, min(IM_RT_THREADS, hi - b), x, y, acc);
        __syncthreads();
    }
    if (x < C.w && y < C.h) depth[(size_t)y * C.w + x] = acc;
}
#define RF_FIN 1024
// valid pixels per block of RF_FIN consecutive pixels
__global__ void __launch_bounds__(RF_FIN) k_rf_fcount(const DepthCam* cam, const unsigned int* depth, int* blk) {
    const DepthCam C = *cam;
    const int i = blockIdx.x * RF_FIN + threadIdx.x;
    const int c = __syncthreads_count(i < C.w * C.h && depth_valid(C, __uint_as_float(depth[i])));
    if (threadIdx.x == 0) blk[blockIdx.x] = c;
}
// depth image and the valid pixels' points in ascending pixel order: block offset + rank inside the block
__global__ void __launch_bounds__(RF_FIN) k_rf_emit(const DepthCam* cam, const FrameDyn* dyn, const unsigned int* depth, const int* blk_off, int nb, RfOut o0, RfOut o1) {
    __shared__ int s_warp[RF_FIN / 32];
    const DepthCam C = *cam;
    const RfOut o = (dyn->frame & 1) ? o1 : o0;
    const int i = blockIdx.x * RF_FIN + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float val = i < C.w * C.h ? __uint_as_float(depth[i]) : 0.f;
    const bool ok = i < C.w * C.h && depth_valid(C, val);
    const unsigned int ball = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[warp] = __popc(ball);
    __syncthreads();
    if (warp == 0) {
        const int mine = s_warp[lane];
        int v = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d) v += u;
        }
        s_warp[lane] = v - mine;   // exclusive
    }
    __syncthreads();
    if (i < C.w * C.h) o.depth[i] = ok ? val : -1.0f;
    if (ok) {
        const int k = blk_off[blockIdx.x] + s_warp[warp] + __popc(ball & ((1u << lane) - 1u));
        depth_unproject(C, i % C.w, i / C.w, val, o.pts + (size_t)k * 3);
        o.pix[k] = i;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *o.n = blk_off[nb];
}

// ---- the viewer's shaded image of the live mesh (draw_triangle with the facet shader, mesh_rec_display.cpp:273-282; the rule is
// immesh_mesh_render_view's, include/immesh_b200.h).  The binning passes of the depth image (k_rf_count -> k_rf_scan -> k_rf_fill,
// with the view's positions), the z range of the height colour when it is automatic (k_view_zrange), then one block per tile
// (k_view_tile): the nearest sample with the triple tie-break per pixel, shaded from the winning triangle.  The blocking
// immesh_mesh_render_view runs it at the caller's camera; the queued view (immesh_mesh_view_enable) behind every frame after the
// reinforcement, its camera from k_rf_pose, into result buffer (frame & 1).
struct ViewOut { uchar4* rgba; float* depth; };
#define VIEW_ZR_THREADS 128
// min / max z (view_ordered) over the vertices of the live triangles: per-block partials, reduced by the last block to finish into
// zr[0], zr[1]; the last block resets the done counter for the next launch
__global__ void __launch_bounds__(VIEW_ZR_THREADS) k_view_zrange(MeshDev M, int pos_mode, unsigned int* part, int* done, float* zr) {
    __shared__ unsigned int s_lo[VIEW_ZR_THREADS / 32], s_hi[VIEW_ZR_THREADS / 32];
    __shared__ bool s_last;
    const int n_alloc = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned int lo = 0xffffffffu, hi = 0u;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        const int v[3] = {r.x, r.y, r.z};
        for (int k = 0; k < 3; ++k) {
            const unsigned int u = view_ordered(rf_vertex(M, pos_mode, v[k]).z);
            lo = min(lo, u); hi = max(hi, u);
        }
    }
    auto block_reduce = [&](unsigned int& a, unsigned int& b) {
        a = __reduce_min_sync(0xffffffffu, a); b = __reduce_max_sync(0xffffffffu, b);
        if (lane == 0) { s_lo[warp] = a; s_hi[warp] = b; }
        __syncthreads();
        if (threadIdx.x == 0)
            for (int w = 1; w < VIEW_ZR_THREADS / 32; ++w) { a = min(a, s_lo[w]); b = max(b, s_hi[w]); }
    };
    block_reduce(lo, hi);
    if (threadIdx.x == 0) {
        part[2 * blockIdx.x] = lo; part[2 * blockIdx.x + 1] = hi;
        __threadfence();
        s_last = atomicAdd(done, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    lo = 0xffffffffu; hi = 0u;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) {
        lo = min(lo, __ldcg(part + 2 * b)); hi = max(hi, __ldcg(part + 2 * b + 1));
    }
    __syncthreads();   // s_lo / s_hi are reused
    block_reduce(lo, hi);
    if (threadIdx.x == 0) { zr[0] = view_unordered(lo); zr[1] = view_unordered(hi); *done = 0; }
}
// one block per tile, one thread per pixel (k_rf_tile's shape): the bin's set-ups and (a, b, c, slot) records staged IM_RT_THREADS at
// a time in shared memory; each thread keeps its pixel's best (depth bits, triple, slot) in registers, then shades the winner and
// writes the pixel's colour and depth.  Bins over capacity (misc[0]): every triangle slot instead, the same image.  With the
// overlays' keys (ov, or null), an overlay fragment drawn over the winner (ov_over_mesh) gives the pixel its colour instead.
__global__ void __launch_bounds__(IM_RT_THREADS) k_view_tile(MeshDev M, int pos_mode, int color, const float* zr, const DepthCam* cam, const int* tile_off,
                                                             const int* bin, const int* misc, const FrameDyn* dyn, ViewOut o0, ViewOut o1,
                                                             const unsigned long long* ov) {
    __shared__ DepthTri S[IM_RT_THREADS];
    __shared__ int4 Q[IM_RT_THREADS];
    const DepthCam C = *cam;
    const int ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    const int x = (blockIdx.x % ntx) * IM_RT_TILE + (int)(threadIdx.x % IM_RT_TILE), y = (blockIdx.x / ntx) * IM_RT_TILE + (int)(threadIdx.x / IM_RT_TILE);
    const bool all = misc[0] != 0;
    const int lo = all ? 0 : tile_off[blockIdx.x], hi = all ? min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t) : tile_off[blockIdx.x + 1];
    unsigned int best = 0x7f800000u;   // +inf: nothing drawn
    int ba = INT_MAX, bb = INT_MAX, bc = INT_MAX, bs = -1;
    for (int b = lo; b < hi; b += IM_RT_THREADS) {
        const int i = b + (int)threadIdx.x;
        bool ok = false;
        if (i < hi) {
            const int slot = all ? i : bin[i];
            const int4 r = M.tri[slot];
            ok = r.w && depth_tri_setup(C, rf_vertex(M, pos_mode, r.x), rf_vertex(M, pos_mode, r.y), rf_vertex(M, pos_mode, r.z), &S[threadIdx.x]);
            Q[threadIdx.x] = make_int4(r.x, r.y, r.z, slot);
        }
        if (!ok) { S[threadIdx.x].x_lo = 1; S[threadIdx.x].x_hi = 0; }   // an empty box
        __syncthreads();
        const int n = min(IM_RT_THREADS, hi - b);
        for (int j = 0; j < n; ++j) {
            const DepthTri& T = S[j];
            if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
            float zf;
            if (!depth_sample(T, x, y, &zf)) continue;
            const unsigned int bits = __float_as_uint(zf);
            const int4 q = Q[j];
            if (bits < 0x7f800000u && view_better(bits, q.x, q.y, q.z, best, ba, bb, bc)) { best = bits; ba = q.x; bb = q.y; bc = q.z; bs = q.w; }
        }
        __syncthreads();
    }
    if (x >= C.w || y >= C.h) return;
    const ViewOut o = (dyn->frame & 1) ? o1 : o0;
    const size_t px = (size_t)y * C.w + x;
    const float val = __uint_as_float(best);
    o.depth[px] = depth_valid(C, val) ? val : -1.0f;
    uchar4 c = make_uchar4(0, 0, 0, 255);
    const unsigned long long k = ov ? ov[px] : OV_NONE;
    if (ov_over_mesh(k, best)) {
        c = ov_color(k);
    } else if (bs >= 0) {
        const int4 r = M.tri[bs];
        const float4 p[3] = {rf_vertex(M, pos_mode, r.x), rf_vertex(M, pos_mode, r.y), rf_vertex(M, pos_mode, r.z)};
        DepthTri T;
        depth_tri_setup(C, p[0], p[1], p[2], &T);
        const float zlo = color ? zr[0] : 0.f, zhi = color ? zr[1] : 0.f;
        double col[3][3];
        for (int k = 0; k < 3; ++k) view_color(color, p[k].z, zlo, zhi, col[k]);
        c = view_shade(T, x, y, p, col, C.t);
    }
    o.rgba[px] = c;
}

// The wireframe (immesh_mesh_view_overlay with wireframe): k_view_tile's shape over the bins of the wireframe's widened boxes.  Per
// pixel, the nearest face sample (the depth image, as in face mode) and the best edge fragment by (depth bits, triple, edge); the
// winning edge coloured from its ends (view_wire_color), unless an overlay fragment is drawn over it.
__global__ void __launch_bounds__(IM_RT_THREADS) k_view_wire_tile(MeshDev M, int pos_mode, int color, const float* zr, const DepthCam* cam, const int* tile_off,
                                                                  const int* bin, const int* misc, const FrameDyn* dyn, ViewOut o0, ViewOut o1,
                                                                  const unsigned long long* ov) {
    __shared__ DepthTri S[IM_RT_THREADS];
    __shared__ int4 Q[IM_RT_THREADS];
    __shared__ int4 FB[IM_RT_THREADS];
    const DepthCam C = *cam;
    const int ntx = (C.w + IM_RT_TILE - 1) / IM_RT_TILE;
    const int x = (blockIdx.x % ntx) * IM_RT_TILE + (int)(threadIdx.x % IM_RT_TILE), y = (blockIdx.x / ntx) * IM_RT_TILE + (int)(threadIdx.x / IM_RT_TILE);
    const bool all = misc[0] != 0;
    const int lo = all ? 0 : tile_off[blockIdx.x], hi = all ? min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t) : tile_off[blockIdx.x + 1];
    unsigned int face = 0x7f800000u, best = 0x7f800000u;
    int ba = INT_MAX, bb = INT_MAX, bc = INT_MAX, be = 3, bs = -1;
    for (int b = lo; b < hi; b += IM_RT_THREADS) {
        const int i = b + (int)threadIdx.x;
        bool ok = false;
        if (i < hi) {
            const int slot = all ? i : bin[i];
            const int4 r = M.tri[slot];
            ok = r.w && view_wire_setup(C, rf_vertex(M, pos_mode, r.x), rf_vertex(M, pos_mode, r.y), rf_vertex(M, pos_mode, r.z), &S[threadIdx.x], &FB[threadIdx.x]);
            Q[threadIdx.x] = make_int4(r.x, r.y, r.z, slot);
        }
        if (!ok) { S[threadIdx.x].x_lo = 1; S[threadIdx.x].x_hi = 0; }
        __syncthreads();
        const int n = min(IM_RT_THREADS, hi - b);
        for (int j = 0; j < n; ++j) {
            const DepthTri& T = S[j];
            if (x < T.x_lo || x > T.x_hi || y < T.y_lo || y > T.y_hi) continue;
            const int4 q = Q[j];
            view_wire_pixel(T, FB[j], q.x, q.y, q.z, q.w, x, y, &face, &best, &ba, &bb, &bc, &be, &bs);
        }
        __syncthreads();
    }
    if (x >= C.w || y >= C.h) return;
    const ViewOut o = (dyn->frame & 1) ? o1 : o0;
    const size_t px = (size_t)y * C.w + x;
    const float val = __uint_as_float(face);
    o.depth[px] = depth_valid(C, val) ? val : -1.0f;
    uchar4 c = make_uchar4(0, 0, 0, 255);
    const unsigned long long k = ov ? ov[px] : OV_NONE;
    if (ov_over_mesh(k, best)) {
        c = ov_color(k);
    } else if (bs >= 0) {
        const int4 r = M.tri[bs];
        const float4 p[3] = {rf_vertex(M, pos_mode, r.x), rf_vertex(M, pos_mode, r.y), rf_vertex(M, pos_mode, r.z)};
        const float zlo = color ? zr[0] : 0.f, zhi = color ? zr[1] : 0.f;
        double col[3][3];
        for (int v = 0; v < 3; ++v) view_color(color, p[v].z, zlo, zhi, col[v]);
        c = view_wire_color(C, p, col, be, x, y);
    }
    o.rgba[px] = c;
}

// ---- the overlays of the queued view (immesh_mesh_view_overlay; the rule is in include/immesh_b200.h): k_ov_begin clears the
// per-pixel keys, appends the frame's sensor position to the trajectory and places the frame's camera frustum; k_ov_points rasterises
// the scan and reinforced points, k_ov_lines the axis, grid, frustum and trajectory segments (a warp per segment), each fragment an
// atomicMin of its 64-bit key (ov_key); the tile kernels then resolve the keys against the mesh.
__global__ void __launch_bounds__(256) k_ov_begin(ViewOverlay O, const FrameDyn* dyn, const double (*ring)[12], const int* ring_frame) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < O.npx; i += gridDim.x * blockDim.x) O.key[i] = OV_NONE;
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    const FrameDyn d = *dyn;
    ov_begin_frame(O, d.frame, d.fp->pose_t, ring, ring_frame);
}
__global__ void __launch_bounds__(128) k_ov_points(ViewOverlay O, const DepthCam* cam, const FrameDyn* dyn, RfOut r0, RfOut r1, int rf_on) {
    const DepthCam C = *cam;
    const FrameDyn d = *dyn;
    const int n_scan = O.scan_size > 0 && d.frame >= 2 ? d.n : 0;
    const RfOut r = (d.frame & 1) ? r1 : r0;
    const int n_rf = O.reinforced_size > 0 && rf_on ? *r.n : 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_scan + n_rf; i += gridDim.x * blockDim.x) {
        const bool scan = i < n_scan;
        const int j = scan ? i : i - n_scan, layer = scan ? OV_SCAN : OV_REINFORCED;
        const float* q = (scan ? d.pts : r.pts) + (size_t)j * 3;
        const double p[3] = {(double)q[0], (double)q[1], (double)q[2]};
        ov_point_raster(C, p, scan ? O.scan_size : O.reinforced_size,
                        [&](int x, int y, float zf) { atomicMin(&O.key[(size_t)y * C.w + x], ov_key(zf, layer, (unsigned)j)); });
    }
}
__global__ void __launch_bounds__(128) k_ov_lines(ViewOverlay O, const DepthCam* cam) {
    const DepthCam C = *cam;
    const int frustum_on = *O.frustum_on, path_n = O.path_width > 0 ? *O.path_n : 0, lane = threadIdx.x & 31;
    const int nseg = (O.axis_and_grid ? OV_N_AXIS + OV_N_GRID : 0) + (frustum_on ? OV_N_CAMERA : 0) + max(ov_path_kept(O, path_n) - 1, 0);
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nseg; i += (gridDim.x * blockDim.x) >> 5) {
        int layer, idx, width;
        double p0[3], p1[3];
        OvSeg S;
        if (!ov_line(O, frustum_on, path_n, i, &layer, &idx, &width, p0, p1) || !ov_seg_setup(C, p0, p1, &S)) continue;
        ov_seg_raster(C, S, width, lane, 32,
                      [&](int x, int y, float zf, double) { atomicMin(&O.key[(size_t)y * C.w + x], ov_key(zf, layer, (unsigned)idx)); });
    }
}

// the buffers of one w x h depth image and `nout` result buffers (image, points, pixels, count) into dev; stops at the first failure
static cudaError_t rf_image_alloc(immesh::MemSet& dev, int w, int h, int nout, RfImage* im) {
    const size_t n = (size_t)w * h;
    im->ntiles = ((w + IM_RT_TILE - 1) / IM_RT_TILE) * ((h + IM_RT_TILE - 1) / IM_RT_TILE);
    im->nb = (int)((n + RF_FIN - 1) / RF_FIN);
    im->bin_cap = std::max(1 << 22, 16 * im->ntiles);   // beyond it an image's tiles walk every triangle slot (same image, slower)
    cudaError_t e = cudaSuccess;
    auto add = [&e, &dev](auto** p, size_t count) { if (e == cudaSuccess) e = dev.alloc(p, std::max<size_t>(count, 1)); };
    add(&im->cam, 1);
    add(&im->tile_cnt, (size_t)im->ntiles); add(&im->tile_off, (size_t)im->ntiles + 1); add(&im->bin, (size_t)im->bin_cap); add(&im->misc, 4);
    add(&im->blk, (size_t)im->nb); add(&im->blk_off, (size_t)im->nb + 1); add(&im->depth_bits, n);
    for (int b = 0; b < nout; ++b) { RfOut& o = im->out[b]; add(&o.depth, n); add(&o.pts, n * 3); add(&o.pix, n); add(&o.n, 1); }
    return e;
}
// the binning passes of an image: the triangles at positions pos_mode (view_vertex) into the tiles' bins
static void rf_bin_launch(const immesh_mesh* h, const RfImage& im, int pos_mode, cudaStream_t st, int wire = 0) {
    const int g = h->n_sm * 8;
    IM_LAUNCH(k_rf_count, g, 128, 0, st, h->M, pos_mode, wire, (const DepthCam*)im.cam, im.tile_cnt);
    IM_LAUNCH(k_rf_scan, 1, 1024, 0, st, (const int*)im.tile_cnt, im.ntiles, im.tile_off, im.tile_cnt, im.bin_cap, im.misc);
    IM_LAUNCH(k_rf_fill, g, 128, 0, st, h->M, pos_mode, wire, (const DepthCam*)im.cam, im.tile_cnt, im.bin, (const int*)im.misc);
}
// the exclusive scan of cnt[0, n) into off[0, n] by k_rf_scan (the valid pixels per block of an image, or of a depth frame)
void rf_scan_launch(cudaStream_t st, const int* cnt, int n, int* off) {
    IM_LAUNCH(k_rf_scan, 1, 1024, 0, st, cnt, n, off, (int*)nullptr, 0, (int*)nullptr);
}
// the image of the camera in im.cam, with the tile counters zeroed, into result buffer (dyn->frame & 1) (fixed grids: every
// per-image value is read on the device)
static void rf_image_launch(const immesh_mesh* h, const RfImage& im, const FrameDyn* dyn, cudaStream_t st) {
    const DepthCam* cam = im.cam;
    rf_bin_launch(h, im, 0, st);
    IM_LAUNCH(k_rf_tile, im.ntiles, IM_RT_THREADS, 0, st, h->M, cam, (const int*)im.tile_off, (const int*)im.bin, (const int*)im.misc, im.depth_bits);
    IM_LAUNCH(k_rf_fcount, im.nb, RF_FIN, 0, st, cam, (const unsigned int*)im.depth_bits, im.blk);
    rf_scan_launch(st, im.blk, im.nb, im.blk_off);
    IM_LAUNCH(k_rf_emit, im.nb, RF_FIN, 0, st, cam, dyn, (const unsigned int*)im.depth_bits, (const int*)im.blk_off, im.nb, im.out[0], im.out[1]);
}

// ---- the queued cameras (immesh_mesh::QueuedCam): the reinforcement and the view
// the camera of intrinsics K (fx, fy, cx, cy) and the pose R, t when given (a queued camera's is set on the device per frame) into C;
// false for bad arguments (a queued camera also needs finite intrinsics with fx, fy != 0, a finite z_far and its pose window)
static bool depth_cam(DepthCam* C, const double* K, int width, int height, double z_near, double z_far, bool queued, int win, const double* R = nullptr,
                      const double* t = nullptr) {
    if (!K || width < 1 || height < 1 || (long long)width * height > (1 << 26) || !(z_near > 0) || !(z_far > z_near)) return false;
    if (queued && !(std::isfinite(z_far) && win >= 1 && win <= IM_RF_RING - 1 && std::isfinite(K[0]) && std::isfinite(K[1]) && std::isfinite(K[2]) &&
                    std::isfinite(K[3]) && K[0] != 0.0 && K[1] != 0.0))
        return false;
    *C = DepthCam{K[0], K[1], K[2], K[3], z_near, z_far, {}, {}, width, height};
    for (int i = 0; R && i < 9; ++i) C->R[i] = R[i];
    for (int i = 0; t && i < 3; ++i) C->t[i] = t[i];
    return true;
}
// the per-frame camera source (RfDyn) and its pinned slots; stops at the first failure
static cudaError_t queued_cam_alloc(immesh_mesh::QueuedCam& c) {
    RfDyn *rd = nullptr, *h_rd = nullptr;
    cudaError_t e = c.dev.alloc(&rd, 1);
    if (e == cudaSuccess) e = c.pinned.alloc(&h_rd, IM_SLOTS, 0);
    c.rd = rd;
    c.h_rd = h_rd;
    return e;
}
// the frame's camera source, from pinned slot s, ahead of its kernels in stream order
int queued_cam_stage(immesh_mesh* h, immesh_mesh::QueuedCam& c, int s) {
    RfDyn* r = (RfDyn*)c.h_rd + s;
    r->mode = c.mode;
    for (int i = 0; i < 9; ++i) r->R[i] = c.R[i];
    for (int i = 0; i < 3; ++i) r->t[i] = c.t[i];
    IM_CUDA(cudaMemcpyAsync(c.rd, r, sizeof(RfDyn), cudaMemcpyHostToDevice, h->stream));
    return IMMESH_OK;
}
// the camera of the frame just queued (k_rf_pose: its pose also into the result buffer), the tile counters cleared
static void queued_cam_pose_launch(const immesh_mesh* h, const immesh_mesh::QueuedCam& c, cudaStream_t st) {
    IM_LAUNCH(k_rf_pose, 1, 256, 0, st, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame, (const FrameDyn*)h->d_dyn, (const RfDyn*)c.rd, c.win, c.base,
              c.img.cam, c.img.out[0], c.img.out[1], c.img.tile_cnt, c.img.ntiles);
}
// the newest frame queued with c, once finished (the next frame writes the other result buffer: the caller's copies do not wait)
static int queued_cam_newest(immesh_mesh* h, const immesh_mesh::QueuedCam& c, const char* what, const char* stage, const char* enable, int* frame) {
    if (!c.on) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": the " + stage + " is not enabled (" + enable + ")").c_str());
    if (!c.last_frame) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": no frame has been queued since " + enable).c_str());
    *frame = c.last_frame;
    IM_CUDA(cudaEventSynchronize(h->ev_done[c.last_frame & (IM_SLOTS - 1)]));
    return IMMESH_OK;
}
// the reinforcement of the frame just queued: its camera, then its image
void mesh_reinforce_launch(immesh_mesh* h, cudaStream_t st) {
    queued_cam_pose_launch(h, h->rf, st);
    rf_image_launch(h, h->rf.img, h->d_dyn, st);
}
// the shaded image of the camera in im.cam (tile counters zeroed) with style v into out[dyn->frame & 1]: binning, the automatic z
// range when the height colour needs it, the tiles
// (the overlays' keys resolved in the tiles when v.ov is on; the wireframe in place of the faces with v.ov.wire)
static void view_image_launch(const immesh_mesh* h, const immesh_mesh::View& v, const RfImage& im, const ViewOut* out, const FrameDyn* dyn, cudaStream_t st) {
    const int wire = v.ov.on && v.ov.wire;
    const unsigned long long* ov = v.ov.on ? v.ov.key : nullptr;
    rf_bin_launch(h, im, v.pos, st, wire);
    if (v.color && v.auto_range) IM_LAUNCH(k_view_zrange, v.zr_blocks, VIEW_ZR_THREADS, 0, st, h->M, v.pos, v.zr_part, v.zr_done, v.zr);
    if (wire)
        IM_LAUNCH(k_view_wire_tile, im.ntiles, IM_RT_THREADS, 0, st, h->M, v.pos, v.color, (const float*)v.zr, (const DepthCam*)im.cam, (const int*)im.tile_off,
                  (const int*)im.bin, (const int*)im.misc, dyn, out[0], out[1], ov);
    else
        IM_LAUNCH(k_view_tile, im.ntiles, IM_RT_THREADS, 0, st, h->M, v.pos, v.color, (const float*)v.zr, (const DepthCam*)im.cam, (const int*)im.tile_off,
                  (const int*)im.bin, (const int*)im.misc, dyn, out[0], out[1], ov);
}
// the queued view of the frame just queued: its camera, then its image
void mesh_view_launch(immesh_mesh* h, cudaStream_t st) {
    auto& v = h->vw;
    queued_cam_pose_launch(h, v, st);
    if (v.ov.on) {   // the overlays' keys; the reinforced points are those of the reinforcement queued just before, while it is on
        const int g = h->n_sm * 8;
        IM_LAUNCH(k_ov_begin, g, 256, 0, st, v.ov, (const FrameDyn*)h->d_dyn, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame);
        IM_LAUNCH(k_ov_points, g, 128, 0, st, v.ov, (const DepthCam*)v.img.cam, (const FrameDyn*)h->d_dyn, h->rf.img.out[0], h->rf.img.out[1], h->rf.on);
        IM_LAUNCH(k_ov_lines, g, 128, 0, st, v.ov, (const DepthCam*)v.img.cam);
    }
    const ViewOut out[2] = {{v.rgba[0], v.img.out[0].depth}, {v.rgba[1], v.img.out[1].depth}};
    view_image_launch(h, v, v.img, out, h->d_dyn, st);
}

int immesh_mesh_render_depth(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, const double* cam_R, const double* cam_t,
                             float* depth, float* points, int32_t* point_pixel, int* n_points) {
    DepthCam C;
    if (!h || !cam_R || !cam_t || !depth || !depth_cam(&C, intrinsics, width, height, z_near, z_far, false, 0, cam_R, cam_t)) return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    const int n = width * height;
    immesh::MemSet tmp;   // h->rf is not touched: a queued frame's result stays readable
    RfImage im;
    IM_CUDA(rf_image_alloc(tmp, width, height, 1, &im));
    im.out[1] = im.out[0];   // k_rf_emit picks out[frame & 1]
    IM_CUDA(cudaMemcpyAsync(im.cam, &C, sizeof(C), cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaMemsetAsync(im.tile_cnt, 0, (size_t)im.ntiles * sizeof(int), h->stream));
    rf_image_launch(h, im, h->d_dyn, h->stream);
    IM_CUDA(cudaGetLastError());
    int np = 0;
    IM_CUDA(cudaMemcpyAsync(depth, im.out[0].depth, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(&np, im.out[0].n, 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    if (!points) np = 0;   // the count is that of the points written
    if (np > 0) {
        IM_CUDA(cudaMemcpy(points, im.out[0].pts, (size_t)np * 3 * sizeof(float), cudaMemcpyDeviceToHost));
        if (point_pixel) IM_CUDA(cudaMemcpy(point_pixel, im.out[0].pix, (size_t)np * sizeof(int), cudaMemcpyDeviceToHost));
    }
    if (n_points) *n_points = np;
    return IMMESH_OK;
}

int immesh_mesh_reinforce_enable(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, int win) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reinforce_enable: a sharded mesh handle is not supported (the reinforcement runs on a single GPU)");
    immesh_mesh::QueuedCam r;   // built in full before it replaces h->rf: after a failure the reinforcement stays disabled
    if (intrinsics && !depth_cam(&r.base, intrinsics, width, height, z_near, z_far, true, win))
        return im_fail(IMMESH_E_INVALID, "reinforce_enable: bad argument (finite intrinsics with fx, fy != 0; 1 <= width * height <= 2^26; 0 < z_near < z_far; 1 <= win <= 63)");
    IM_CUDA(im_stage_reset(h, [h] { h->rf = immesh_mesh::QueuedCam(); }));
    if (!intrinsics) return IMMESH_OK;
    r.win = win;
    cudaError_t e = rf_image_alloc(r.dev, width, height, 2, &r.img);
    if (e == cudaSuccess) e = queued_cam_alloc(r);
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = r.dev.alloc(&r.img.out[b].pose, 12);
    if (e != cudaSuccess) return im_fail_alloc(e, "reinforce_enable: allocation of the reinforcement buffers failed");
    r.on = 1;
    h->rf = std::move(r);
    return IMMESH_OK;
}
int immesh_mesh_reinforce_pose(immesh_mesh_t* h, const double* cam_R, const double* cam_t) {
    if (!h || (!cam_R) != (!cam_t)) return im_fail(IMMESH_E_INVALID, "bad argument (cam_R and cam_t both given or both NULL)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reinforce_pose: a sharded mesh handle is not supported");
    h->rf.mode = cam_R ? 1 : 0;
    for (int i = 0; i < 9; ++i) h->rf.R[i] = cam_R ? cam_R[i] : 0.0;
    for (int i = 0; i < 3; ++i) h->rf.t[i] = cam_t ? cam_t[i] : 0.0;
    return IMMESH_OK;
}
int immesh_mesh_reinforced_cloud(immesh_mesh_t* h, float* depth, float* points, int32_t* point_pixel, int cap, int* n_out, double* pose_out) {
    if (!h || !n_out || cap < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reinforced_cloud: a sharded mesh handle is not supported");
    int f = 0;
    if (const int rc = queued_cam_newest(h, h->rf, "reinforced_cloud", "reinforcement", "immesh_mesh_reinforce_enable", &f)) return rc;
    const int b = f & 1;
    int n = 0;
    double pose[12];
    const RfOut& o = h->rf.img.out[b];
    IM_CUDA(cudaMemcpy(&n, o.n, sizeof(int), cudaMemcpyDeviceToHost));
    IM_CUDA(cudaMemcpy(pose, o.pose, sizeof(pose), cudaMemcpyDeviceToHost));
    *n_out = n;
    if (n > cap) return im_fail(IMMESH_E_CAPACITY, "reinforced_cloud: more points than cap (*n_out holds the number needed; nothing was written)");
    if (depth) IM_CUDA(cudaMemcpy(depth, o.depth, (size_t)h->rf.base.w * h->rf.base.h * sizeof(float), cudaMemcpyDeviceToHost));
    if (points && n > 0) IM_CUDA(cudaMemcpy(points, o.pts, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    if (point_pixel && n > 0) IM_CUDA(cudaMemcpy(point_pixel, o.pix, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    if (pose_out) std::memcpy(pose_out, pose, sizeof(pose));
    return IMMESH_OK;
}

// the style of a view (NULL: raw positions, white); the caller's z range is checked only when the height colour is on
static int view_style_set(const immesh_view_style* style, const char* what, immesh_mesh::View& v, float* zr) {
    const immesh_view_style d = {0, 0, {NAN, NAN}}, &s = style ? *style : d;
    if ((s.positions != 0 && s.positions != 1) || (s.color_by_height != 0 && s.color_by_height != 1))
        return im_fail(IMMESH_E_INVALID, (std::string(what) + ": bad style (positions and color_by_height are 0 or 1)").c_str());
    v.pos = s.positions;
    v.color = s.color_by_height;
    v.auto_range = v.color && std::isnan(s.z_range[0]) && std::isnan(s.z_range[1]);
    if (v.color && !v.auto_range) {
        if (!std::isfinite(s.z_range[0]) || !std::isfinite(s.z_range[1]) || !(s.z_range[0] < s.z_range[1]))
            return im_fail(IMMESH_E_INVALID, (std::string(what) + ": bad z_range (finite with z_range[0] < z_range[1], or both NaN)").c_str());
        zr[0] = (float)s.z_range[0];
        zr[1] = (float)s.z_range[1];
    }
    return IMMESH_OK;
}
// the buffers of a w x h view with `nbuf` result buffers into v.dev; stops at the first failure
static cudaError_t view_alloc(immesh_mesh::View& v, int w, int h, int nbuf, int zr_blocks) {
    const size_t n = (size_t)w * h;
    cudaError_t e = rf_image_alloc(v.dev, w, h, 0, &v.img);
    auto add = [&e, &v](auto** p, size_t count) { if (e == cudaSuccess) e = v.dev.alloc(p, std::max<size_t>(count, 1)); };
    for (int b = 0; b < nbuf; ++b) { add(&v.img.out[b].depth, n); add(&v.img.out[b].pose, 12); add(&v.rgba[b], n); }
    v.zr_blocks = zr_blocks;
    add(&v.zr, 2); add(&v.zr_part, 2 * (size_t)zr_blocks); add(&v.zr_done, 1);
    return e;
}
int immesh_mesh_render_view(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, const double* cam_R, const double* cam_t,
                            const immesh_view_style* style, uint8_t* rgba, float* depth) {
    DepthCam C;
    if (!h || !cam_R || !cam_t || !rgba || !depth_cam(&C, intrinsics, width, height, z_near, z_far, false, 0, cam_R, cam_t))
        return im_fail(IMMESH_E_INVALID, "render_view: bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "render_view: a sharded mesh handle is not supported");
    immesh_mesh::View v;   // this call's buffers; h->vw is not touched, so a queued frame's result stays readable
    float zr[2] = {0.f, 0.f};
    if (const int rc = view_style_set(style, "render_view", v, zr)) return rc;
    IM_CUDA(cudaStreamSynchronize(h->stream));
    const cudaError_t e = view_alloc(v, width, height, 1, h->n_sm * 4);
    if (e != cudaSuccess) return im_fail_alloc(e, "render_view: allocation of the image buffers failed");
    const size_t n = (size_t)width * height;
    IM_CUDA(cudaMemcpyAsync(v.img.cam, &C, sizeof(C), cudaMemcpyHostToDevice, h->stream));
    IM_CUDA(cudaMemsetAsync(v.img.tile_cnt, 0, (size_t)v.img.ntiles * sizeof(int), h->stream));
    IM_CUDA(cudaMemsetAsync(v.zr_done, 0, sizeof(int), h->stream));
    IM_CUDA(cudaMemcpyAsync(v.zr, zr, sizeof(zr), cudaMemcpyHostToDevice, h->stream));
    const ViewOut out[2] = {{v.rgba[0], v.img.out[0].depth}, {v.rgba[0], v.img.out[0].depth}};   // k_view_tile picks out[frame & 1]
    view_image_launch(h, v, v.img, out, h->d_dyn, h->stream);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(rgba, v.rgba[0], n * 4, cudaMemcpyDeviceToHost, h->stream));
    if (depth) IM_CUDA(cudaMemcpyAsync(depth, v.img.out[0].depth, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    return IMMESH_OK;
}
int immesh_mesh_view_enable(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, int win, const immesh_view_style* style) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "view_enable: a sharded mesh handle is not supported (the view runs on a single GPU)");
    immesh_mesh::View v;   // built in full before it replaces h->vw: after a failure the view stays disabled
    float zr[2] = {0.f, 0.f};
    if (intrinsics) {
        if (!depth_cam(&v.base, intrinsics, width, height, z_near, z_far, true, win))
            return im_fail(IMMESH_E_INVALID, "view_enable: bad argument (finite intrinsics with fx, fy != 0; 1 <= width * height <= 2^26; 0 < z_near < z_far < inf; 1 <= win <= 63)");
        if (const int rc = view_style_set(style, "view_enable", v, zr)) return rc;
    }
    IM_CUDA(im_stage_reset(h, [h] {
        h->vw = immesh_mesh::View();
        auto& f = h->feed;   // its image ring was sized for the view that goes: image recording stops until the feed is enabled again
        f.img_mem = immesh::MemSet();
        f.rgba = nullptr; f.depth_ring = nullptr; f.max_images = 0; f.npx = 0; f.depth = 0;
    }));
    if (!intrinsics) return IMMESH_OK;
    v.win = win;
    cudaError_t e = view_alloc(v, width, height, 2, h->n_sm * 4);
    if (e == cudaSuccess) e = queued_cam_alloc(v);
    if (e == cudaSuccess) e = cudaMemsetAsync(v.zr_done, 0, sizeof(int), h->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(v.zr, zr, sizeof(zr), cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) return im_fail_alloc(e, "view_enable: allocation of the view's buffers failed");
    v.on = 1;
    h->vw = std::move(v);
    return IMMESH_OK;
}
int immesh_mesh_view_pose(immesh_mesh_t* h, const double* cam_R, const double* cam_t, int follow) {
    if (!h || (!cam_R) != (!cam_t) || (follow != 0 && follow != 1) || (!cam_R && follow))
        return im_fail(IMMESH_E_INVALID, "view_pose: bad argument (cam_R and cam_t both given or both NULL; follow 0 or 1, and 0 with NULL)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "view_pose: a sharded mesh handle is not supported");
    if (!h->vw.on) return im_fail(IMMESH_E_INVALID, "view_pose: the view is not enabled (immesh_mesh_view_enable)");
    h->vw.mode = cam_R ? (follow ? 2 : 1) : 0;
    for (int i = 0; i < 9; ++i) h->vw.R[i] = cam_R ? cam_R[i] : 0.0;
    for (int i = 0; i < 3; ++i) h->vw.t[i] = cam_t ? cam_t[i] : 0.0;
    return IMMESH_OK;
}
int immesh_mesh_view_image(immesh_mesh_t* h, uint8_t* rgba, float* depth, double* pose_out, int64_t* frame_out) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "view_image: a sharded mesh handle is not supported");
    int f = 0;
    if (const int rc = queued_cam_newest(h, h->vw, "view_image", "view", "immesh_mesh_view_enable", &f)) return rc;
    const int b = f & 1;
    const size_t n = (size_t)h->vw.base.w * h->vw.base.h;
    if (rgba) IM_CUDA(cudaMemcpy(rgba, h->vw.rgba[b], n * 4, cudaMemcpyDeviceToHost));
    if (depth) IM_CUDA(cudaMemcpy(depth, h->vw.img.out[b].depth, n * sizeof(float), cudaMemcpyDeviceToHost));
    if (pose_out) IM_CUDA(cudaMemcpy(pose_out, h->vw.img.out[b].pose, 12 * sizeof(double), cudaMemcpyDeviceToHost));
    if (frame_out) *frame_out = f;
    return IMMESH_OK;
}

int immesh_mesh_view_overlay(immesh_mesh_t* h, const immesh_view_overlay* o) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "view_overlay: a sharded mesh handle is not supported");
    if (!h->vw.on) return im_fail(IMMESH_E_INVALID, "view_overlay: the view is not enabled (immesh_mesh_view_enable)");
    if (o) {
        auto size_ok = [](int s) { return s >= 0 && s <= 64; };
        if ((o->wireframe != 0 && o->wireframe != 1) || (o->axis_and_grid != 0 && o->axis_and_grid != 1) || !size_ok(o->scan_point_size) ||
            !size_ok(o->reinforced_point_size) || !size_ok(o->path_width) || !std::isfinite(o->camera_size) || o->camera_size < 0.0 ||
            (o->path_width > 0 && (o->path_capacity < 1 || o->path_capacity > (1 << 24))))
            return im_fail(IMMESH_E_INVALID, "view_overlay: bad argument (wireframe and axis_and_grid 0 or 1; sizes and widths in [0, 64]; finite camera_size >= 0; "
                                             "1 <= path_capacity <= 2^24 with a path)");
        if (o->scan_point_size > 0 && h->max_frame_points >= (1 << OV_IDX_BITS))
            return im_fail(IMMESH_E_INVALID, "view_overlay: scan points need max_frame_points < 2^29");
    }
    auto& v = h->vw;
    IM_CUDA(im_stage_reset(h, [&v] { v.ov = ViewOverlay{}; v.ov_dev = immesh::MemSet(); }));
    if (!o || !(o->wireframe || o->scan_point_size || o->reinforced_point_size || o->axis_and_grid || o->camera_size > 0.0 || o->path_width))
        return IMMESH_OK;   // every layer off: as NULL
    ViewOverlay ov = {};
    ov.wire = o->wireframe;
    ov.scan_size = o->scan_point_size;
    ov.reinforced_size = o->reinforced_point_size;
    ov.axis_and_grid = o->axis_and_grid;
    ov.camera_size = o->camera_size;
    ov.path_width = o->path_width;
    ov.path_cap = o->path_width > 0 ? o->path_capacity : 1;
    ov.npx = v.base.w * v.base.h;
    immesh::MemSet dev;
    cudaError_t e = dev.alloc(&ov.key, (size_t)ov.npx);
    if (e == cudaSuccess) e = dev.alloc(&ov.path, (size_t)ov.path_cap);
    if (e == cudaSuccess) e = dev.alloc(&ov.path_n, 1, 0);
    if (e == cudaSuccess) e = dev.alloc(&ov.frustum, 11);
    if (e == cudaSuccess) e = dev.alloc(&ov.frustum_on, 1, 0);
    if (e != cudaSuccess) return im_fail_alloc(e, "view_overlay: allocation of the overlay's buffers failed");
    ov.on = 1;
    v.ov = ov;
    v.ov_dev = std::move(dev);
    return IMMESH_OK;
}

