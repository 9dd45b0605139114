// immesh_b200 -- CUDA kernels (sm_90a) and C-ABI host orchestration of the voxel-wise incremental mesher.
// Kernel bodies live in mesh_core.cuh / mesh_voxel.cuh.  No CPU path.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"
#include "nccl_api.hpp"

using namespace immesh;

// ------------------------------------------------------------------ kernels
__global__ void k_frame_begin(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (unsigned int i = tid; i <= F.cmask; i += nt) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    for (unsigned int i = tid; i <= F.fset_mask; i += nt) F.fset[i] = -1;
    if (tid == 0) {
        for (int k = 5; k <= 10; ++k) M.cnt[k] = 0;
        for (int k = 17; k <= 26; ++k) M.cnt[k] = 0;
        M.cnt[28] = 0;
        M.cnt[29] = 0;
        M.cnt[30] = 0; M.cnt[31] = 0; M.cnt[32] = 0;
    }
}
__global__ void __launch_bounds__(128) k_cand_init(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_init(M, P, F, c);
}
__global__ void __launch_bounds__(128) k_cand_conflicts(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_conflicts(M, P, F, c);
}
// Priority polling: candidate c waits only on candidates with a smaller index.  Blocks take tickets so that the
// block holding the smallest undecided candidate is always resident; a poll cap turns a (never observed) livelock
// into an error flag instead of a hang.
__global__ void __launch_bounds__(128) k_cand_resolve(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ int s_ticket;
    const int nblocks = (F.m + blockDim.x - 1) / blockDim.x;
    while (true) {
        if (threadIdx.x == 0) s_ticket = atomicAdd(&M.cnt[18], 1);
        __syncthreads();
        const int b = s_ticket;
        __syncthreads();
        if (b >= nblocks) break;
        const int c = b * blockDim.x + threadIdx.x;
        if (c < F.m && F.cand_status[c] == CAND_UNDECIDED) {
            int polls = 0;
            while (!cand_poll(M, P, F, c)) {
                if (++polls > (1 << 22)) { atomicOr(&M.cnt[3], IM_MERR_LIST_CAP); atomicAdd(&M.cnt[9], 1); break; }
                __nanosleep(64);
            }
            __threadfence();
        }
    }
}
// exclusive scan of the accept flags by one block in ONE pass: thread t owns a contiguous chunk of ceil(m/1024) candidates
__global__ void __launch_bounds__(1024) k_cand_scan(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ int s_warp[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int per = (F.m + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(lo + per, F.m);
    int mine = 0;
    for (int c = lo; c < hi; ++c) mine += (F.cand_status[c] == CAND_ACCEPT) ? 1 : 0;
    int v = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) s_warp[warp] = v;
    __syncthreads();
    if (warp == 0) {
        int wv = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, wv, o);
            if (lane >= o) wv += u;
        }
        s_warp[lane] = wv;
    }
    __syncthreads();
    int run = (warp ? s_warp[warp - 1] : 0) + v - mine;
    for (int c = lo; c < hi; ++c) {
        F.cand_scan[c] = run;
        run += (F.cand_status[c] == CAND_ACCEPT) ? 1 : 0;
    }
}
__global__ void __launch_bounds__(128) k_cand_commit(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[0];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_commit(M, P, F, c, base);
}
__global__ void __launch_bounds__(128) k_cand_place(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[0];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_place(M, F, c, base);
}
__global__ void __launch_bounds__(128) k_voxel_select(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int na = min(M.cnt[5], F.max_act);
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < na; a += gridDim.x * blockDim.x) voxel_select(M, F, a);
}
// stage A: dilation (exact 20-NN of the in-voxel vertices + smoothing); one block per (voxel, group of <= 8 queries)
__global__ void __launch_bounds__(128) k_voxel_dilate(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ DilateSmem S;
    __shared__ int s_item;
    const int ni = min(M.cnt[29], F.max_ditem);
    while (true) {
        if (threadIdx.x == 0) s_item = atomicAdd(&M.cnt[24], 1);
        __syncthreads();
        const int i = s_item;
        __syncthreads();
        if (i >= ni) break;
        voxel_dilate(M, P, F, F.ditem[i], &S, threadIdx.x, blockDim.x);
        __syncthreads();
    }
}
// stage B, small dilated sets: one warp per voxel (four independent voxels per block), voxels claimed dynamically
#define IM_WARP_NMAX 96
__global__ void __launch_bounds__(128) k_voxel_tri_warp(MeshDev M, MeshParams P, FrameBuf F_, int n_max) {
    const FrameBuf F = frame_load_dyn(F_);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    MeshWarpSmem<128>* S = reinterpret_cast<MeshWarpSmem<128>*>(smem_raw) + warp;
    const int nw = work_total(M, F);
    IM_STAMP(30, nw);
    int n_done = 0;
    while (true) {
        int i = 0;
        if (lane == 0) i = atomicAdd(&M.cnt[19], 1);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= nw) break;
        voxel_mesh_warp<128>(M, P, F, work_slot(M, F, i), S, lane, 32, n_max);
        __syncwarp();
        ++n_done;
    }
    IM_STAMP(31, n_done);
    IM_STAMP_IF(blockIdx.x == 0 && threadIdx.x == 0 && (immesh_stamp_store(41, n_done), true), 42, nw);
}
// stage C (flat): after every voxel's smoothing is final
__global__ void __launch_bounds__(128) k_commit_faces(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int nf = min(M.cnt[25], F.max_list);
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += gridDim.x * blockDim.x) commit_face(M, P, F, f);
}
__global__ void __launch_bounds__(128) k_pull_vertices(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int nr = min(M.cnt[26], F.max_vref);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) pull_vertex(M, P, F, r);
}
__global__ void __launch_bounds__(128) k_pull_check(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int ne = min(M.cnt[28], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < ne; e += gridDim.x * blockDim.x) pull_check(M, F, e);
}
template <int MAXD>
__global__ void __launch_bounds__(128) k_voxel_mesh(MeshDev M, MeshParams P, FrameBuf F_, int lo, int store_only) {
    const FrameBuf F = frame_load_dyn(F_);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MeshSmem<MAXD>* S = reinterpret_cast<MeshSmem<MAXD>*>(smem_raw);
    const int nw = work_total(M, F);
    for (int i = blockIdx.x; i < nw; i += gridDim.x) {
        const int w = work_slot(M, F, i);
        const int n = F.work_n_ids[w];
        const int na = n < 0 ? -n : n;
        if ((n < 0 && !store_only) || (n > 0 && na > lo && na <= MAXD)) voxel_mesh<MAXD>(M, P, F, w, S, threadIdx.x, blockDim.x, store_only);
        __syncthreads();
    }
}
__global__ void __launch_bounds__(128) k_push_remove(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[8], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) tri_remove(M, F.rem_tri[e]);
}
__global__ void __launch_bounds__(128) k_push_add(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[7], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x)
        tri_add(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
}
__global__ void k_frame_end(MeshDev M) {
    M.cnt[0] += M.cnt[10];
}
// snapshot: compact live triangles
__global__ void __launch_bounds__(128) k_snapshot(MeshDev M, int n_alloc, int* out_tri, int* out_flip, int* out_n) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        const int k = atomicAdd(out_n, 1);
        out_tri[(size_t)k * 3 + 0] = r.x; out_tri[(size_t)k * 3 + 1] = r.y; out_tri[(size_t)k * 3 + 2] = r.z;
        out_flip[k] = (int)(M.tri_flip[t] & 1ull);
    }
}

// exact kNN over the mesh vertices for arbitrary queries (KD_TREE::Nearest_Search): one warp per query, ring
// expansion over the mesh-voxel hash, per-lane sorted top-k lists merged with warp shuffles.
#define KNN_KMAX 32
__global__ void __launch_bounds__(128) k_knn(MeshDev M, MeshParams P, const float* q, int qstride, int nq, int k, double max_dist, int* out_idx, float* out_d2) {
    const int lane = threadIdx.x & 31;
    const int wglobal = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    const double max_d2 = max_dist * max_dist;
    for (int qi = wglobal; qi < nq; qi += nw) {
        const float qx = q[(size_t)qi * qstride + 0], qy = q[(size_t)qi * qstride + 1], qz = q[(size_t)qi * qstride + 2];
        const int cx = round_key(qx, P.res), cy = round_key(qy, P.res), cz = round_key(qz, P.res);
        float ld[KNN_KMAX];
        int lid[KNN_KMAX];
        int ln = 0;
        int far = 0;
        if (M.cnt[4] > 0) {
            far = max(far, max(abs(cx - M.cnt[11]), abs(cx - M.cnt[14])));
            far = max(far, max(abs(cy - M.cnt[12]), abs(cy - M.cnt[15])));
            far = max(far, max(abs(cz - M.cnt[13]), abs(cz - M.cnt[16])));
        } else {
            far = -1;
        }
        float kth = INFINITY;
        int total = 0;
        for (int ring = 0; ring <= far; ++ring) {
            if (ring >= 1) {
                const double lb = (double)(ring - 1) * P.res;
                if (lb > max_dist) break;
                if (total >= k && (double)kth < lb * lb * 0.999999) break;
            }
            const int side = 2 * ring + 1;
            for (int c = lane; c < side * side * side; c += 32) {
                const int dx = c / (side * side) - ring, dy = (c / side) % side - ring, dz = c % side - ring;
                if (max(abs(dx), max(abs(dy), abs(dz))) != ring) continue;
                if (!ikey_ok(cx + dx, cy + dy, cz + dz)) continue;
                const int s = table_find(M.vkeys, M.vmask, pack_ikey(cx + dx, cy + dy, cz + dz));
                if (s < 0) continue;
                int cntv = M.vox_count[s];
                if (cntv > IM_VCHUNKS * 16) cntv = IM_VCHUNKS * 16;
                for (int kk = 0; kk < cntv; ++kk) {
                    const float4 p = M.vchunk_pts[(size_t)M.vox_chunk[(size_t)s * IM_VCHUNKS + (kk >> 4)] * 16 + (kk & 15)];
                    const int v = __float_as_int(p.w);
                    const float d2 = dist2f(qx, qy, qz, p.x, p.y, p.z);
                    if (!((double)d2 <= max_d2)) continue;
                    // insert (d2, v) into this lane's ascending list, keeping at most k
                    if (ln == k && !(d2 < ld[ln - 1] || (d2 == ld[ln - 1] && v < lid[ln - 1]))) continue;
                    int pos = ln < k ? ln : k - 1;
                    while (pos > 0 && (d2 < ld[pos - 1] || (d2 == ld[pos - 1] && v < lid[pos - 1]))) {
                        ld[pos] = ld[pos - 1]; lid[pos] = lid[pos - 1];
                        --pos;
                    }
                    ld[pos] = d2; lid[pos] = v;
                    if (ln < k) ++ln;
                }
            }
            // k-th smallest over the warp: merge the lane lists (non-destructively)
            int cur = 0;
            total = 0;
            kth = INFINITY;
            for (int r = 0; r < k; ++r) {
                float bd = cur < ln ? ld[cur] : INFINITY;
                int bid = cur < ln ? lid[cur] : 0x7fffffff;
                int who = lane;
                warp_min_pair(&bd, &bid, &who);
                if (bid == 0x7fffffff) break;
                if (who == lane) ++cur;
                kth = bd;
                ++total;
            }
        }
        int cur = 0;
        for (int r = 0; r < k; ++r) {
            float bd = cur < ln ? ld[cur] : INFINITY;
            int bid = cur < ln ? lid[cur] : 0x7fffffff;
            int who = lane;
            warp_min_pair(&bd, &bid, &who);
            if (bid != 0x7fffffff && who == lane) ++cur;
            if (lane == 0) {
                out_idx[(size_t)qi * k + r] = bid == 0x7fffffff ? -1 : bid;
                out_d2[(size_t)qi * k + r] = bid == 0x7fffffff ? INFINITY : bd;
            }
        }
    }
}

// Global_map::smooth_pts (pointcloud_rgbd.cpp:932-958) on every vertex = smooth_all_pts (mesh_rec_geometry.cpp:60-69): from the
// vertex's knn nearest vertices (k_knn, ascending; the first is the vertex itself and is skipped) those with sqrt(d2) < max_dis
// are averaged, smoothed = p (1 - f) + sum f / valid; stored as the smoothed position (set_smooth_pos) and written to out.
__global__ void __launch_bounds__(128) k_smooth_all(MeshDev M, int nv, int k, const int* __restrict__ idx, const float* __restrict__ d2, double sf, double max_dis, double* out) {
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += gridDim.x * blockDim.x) {
        const float4 p = M.vpos[v];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, valid = 0.0;
        for (int j = 1; j < k; ++j) {
            const int id = idx[(size_t)v * k + j];
            if (id < 0) break;
            if ((double)sqrtf(d2[(size_t)v * k + j]) < max_dis) {
                const float4 q = M.vpos[id];
                s0 = s0 + (double)q.x; s1 = s1 + (double)q.y; s2 = s2 + (double)q.z;
                valid += 1.0;
            }
        }
        const double r0 = (double)p.x * (1.0 - sf) + s0 * sf / valid, r1 = (double)p.y * (1.0 - sf) + s1 * sf / valid, r2 = (double)p.z * (1.0 - sf) + s2 * sf / valid;
        M.vsmooth[(size_t)v * 3 + 0] = r0; M.vsmooth[(size_t)v * 3 + 1] = r1; M.vsmooth[(size_t)v * 3 + 2] = r2;
        if (out) { out[(size_t)v * 3 + 0] = r0; out[(size_t)v * 3 + 1] = r1; out[(size_t)v * 3 + 2] = r2; }
    }
}
// Triangle_manager::insert_triangle_to_list (triangle.cpp:35-53): region = round(centre / region_size) of every live triangle
__global__ void __launch_bounds__(128) k_region_keys(MeshDev M, int n_alloc, double region_size, int* out_tri, int* out_key, int* out_n) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        const float4 a = M.vpos[r.x], b = M.vpos[r.y], c = M.vpos[r.z];
        const int e = atomicAdd(out_n, 1);
        out_tri[(size_t)e * 3 + 0] = r.x; out_tri[(size_t)e * 3 + 1] = r.y; out_tri[(size_t)e * 3 + 2] = r.z;
        out_key[(size_t)e * 3 + 0] = (int)round((((double)a.x + (double)b.x) + (double)c.x) / 3.0 / region_size);
        out_key[(size_t)e * 3 + 1] = (int)round((((double)a.y + (double)b.y) + (double)c.y) / 3.0 / region_size);
        out_key[(size_t)e * 3 + 2] = (int)round((((double)a.z + (double)b.z) + (double)c.z) / 3.0 / region_size);
    }
}

// ---- depth rasterisation of the live mesh ("LiDAR point-cloud reinforcement", src/ImMesh_node.cpp:305-329: draw_triangle into a depth
// camera, Cam_view::read_depth, convert_depth_buffer_to_truth_depth + unproject_point, src/tools/openGL_libs/openGL_camera_view.cpp:316-
// 418).  The reference lets OpenGL rasterise; here a CUDA rasteriser with a defined sampling rule produces the metric depth directly:
// camera frame x right / y down / z forward (the frame unproject_point inverts: world = R diag(1,-1,-1) p + t), pixel (u, v) =
// (fx x / z + cx, fy y / z + cy), samples at integer pixel coordinates, a sample is covered when the three edge functions have one
// sign (zero included), depth interpolated perspective-correctly (1/z is affine in the image), nearest surface wins (atomicMin on the
// float bits).  Triangles with a vertex outside (z_near, z_far) are skipped (GL would clip them).
struct DepthCam { double fx, fy, cx, cy, z_near, z_far; double R[9], t[3]; int w, h; };
__device__ __forceinline__ void depth_project(const DepthCam& C, const float4& p, double* u, double* v, double* z) {
    const double d[3] = {(double)p.x - C.t[0], (double)p.y - C.t[1], (double)p.z - C.t[2]};
    const double xc = (C.R[0] * d[0] + C.R[3] * d[1]) + C.R[6] * d[2];     // R^T d
    const double yc = -((C.R[1] * d[0] + C.R[4] * d[1]) + C.R[7] * d[2]);
    const double zc = -((C.R[2] * d[0] + C.R[5] * d[1]) + C.R[8] * d[2]);
    *z = zc;
    *u = C.fx * xc / zc + C.cx;
    *v = C.fy * yc / zc + C.cy;
}
__global__ void __launch_bounds__(128) k_depth_clear(unsigned int* depth, int n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) depth[i] = 0x7f800000u;   // +inf
}
__global__ void __launch_bounds__(128) k_depth_raster(MeshDev M, int n_alloc, DepthCam C, unsigned int* depth) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        const int4 r = M.tri[t];
        if (!r.w) continue;
        double u0, v0, z0, u1, v1, z1, u2, v2, z2;
        depth_project(C, M.vpos[r.x], &u0, &v0, &z0);
        depth_project(C, M.vpos[r.y], &u1, &v1, &z1);
        depth_project(C, M.vpos[r.z], &u2, &v2, &z2);
        if (!(z0 > C.z_near && z0 < C.z_far && z1 > C.z_near && z1 < C.z_far && z2 > C.z_near && z2 < C.z_far)) continue;
        const double area = (u1 - u0) * (v2 - v0) - (v1 - v0) * (u2 - u0);
        if (area == 0.0) continue;
        const int x_lo = max(0, (int)ceil(fmin(u0, fmin(u1, u2)))), x_hi = min(C.w - 1, (int)floor(fmax(u0, fmax(u1, u2))));
        const int y_lo = max(0, (int)ceil(fmin(v0, fmin(v1, v2)))), y_hi = min(C.h - 1, (int)floor(fmax(v0, fmax(v1, v2))));
        const double iz0 = 1.0 / z0, iz1 = 1.0 / z1, iz2 = 1.0 / z2;
        for (int y = y_lo; y <= y_hi; ++y)
            for (int x = x_lo; x <= x_hi; ++x) {
                const double px = (double)x, py = (double)y;
                const double e0 = (u2 - u1) * (py - v1) - (v2 - v1) * (px - u1);   // weight of vertex 0
                const double e1 = (u0 - u2) * (py - v2) - (v0 - v2) * (px - u2);
                const double e2 = (u1 - u0) * (py - v0) - (v1 - v0) * (px - u0);
                if (!((e0 >= 0 && e1 >= 0 && e2 >= 0) || (e0 <= 0 && e1 <= 0 && e2 <= 0))) continue;
                const double iz = ((e0 * iz0 + e1 * iz1) + e2 * iz2) / area;
                const float zf = (float)(1.0 / iz);
                if (zf > 0.f) atomicMin(&depth[(size_t)y * C.w + x], __float_as_uint(zf));
            }
    }
}
// convert_depth_buffer_to_truth_depth's validity rule (val < 0.99 z_far, else -1) + unproject_point (openGL_camera_view.cpp:407-414)
__global__ void __launch_bounds__(128) k_depth_finish(DepthCam C, const unsigned int* depth, float* out_depth, float* out_pts, int* n_pts) {
    const int n = C.w * C.h;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float val = __uint_as_float(depth[i]);
        const bool ok = (double)val < C.z_far * 0.99;
        out_depth[i] = ok ? val : -1.0f;
        if (ok && out_pts) {
            const int x = i % C.w, y = i / C.w;
            // m_camera_intrinsic_inv * (x, y, 1), scaled to depth val, GL camera axes (x, -y, -z), then R p + t
            const double sx = ((double)x - C.cx) / C.fx, sy = ((double)y - C.cy) / C.fy;
            const double g[3] = {sx * (double)val, -(sy * (double)val), -(double)val};
            const int k = atomicAdd(n_pts, 1);
            for (int a = 0; a < 3; ++a) out_pts[(size_t)k * 4 + a] = (float)(((C.R[a * 3 + 0] * g[0] + C.R[a * 3 + 1] * g[1]) + C.R[a * 3 + 2] * g[2]) + C.t[a]);
            out_pts[(size_t)k * 4 + 3] = __int_as_float(i);   // the pixel the point came from (the order of the list is arbitrary)
        }
    }
}

// ------------------------------------------------------------------ host side

template <class T>
static cudaError_t mdev_alloc(immesh_mesh* h, T** p, size_t count, int memset_byte = -1) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T));
    if (e != cudaSuccess) return e;
    h->allocs.push_back(q);
    *p = (T*)q;
    if (memset_byte >= 0) e = cudaMemset(q, memset_byte, count * sizeof(T));
    return e;
}
static size_t pow2_at_least(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

#if defined(IM_DEBUG_STAMPS)
extern "C" int immesh_debug_stamps_mesh(long long* out64) {   // debug variant only (tools/debug/build_stamps.sh); not declared in include/
    return cudaMemcpyFromSymbol(out64, immesh::g_stamps, 64 * sizeof(long long)) == cudaSuccess ? 0 : -1;
}
#endif

extern "C" {

int immesh_mesh_destroy(immesh_mesh_t* h);
int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    if (!cfg || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    if (!(cfg->points_minimum_scale > 0) || !(cfg->voxel_resolution > 0) || cfg->number_of_pts_append_to_map < 1) return im_fail(IMMESH_E_INVALID, "bad mesh configuration");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path");
    immesh_mesh* h = new immesh_mesh();
    // every failure below releases what has been created so far (immesh_mesh_destroy copes with a partially built handle)
#define IM_CREATE_M(expr)                                                                   \
    do {                                                                                    \
        cudaError_t im_e_ = (expr);                                                         \
        if (im_e_ != cudaSuccess) { immesh_mesh_destroy(h); return immesh::im_fail_cuda(im_e_, __FILE__, __LINE__); } \
    } while (0)
    h->F.shard_rank = 0; h->F.shard_n = 1; h->F.x_cap = 0;
    h->bps = std::getenv("IMMESH_MESH_BPS") ? std::atoi(std::getenv("IMMESH_MESH_BPS")) : 3;
    h->dilate_bps = std::getenv("IMMESH_DILATE_BPS") ? std::atoi(std::getenv("IMMESH_DILATE_BPS")) : h->bps;
    // dilated sets up to warp_nmax vertices are triangulated by one warp each (side stream), larger ones by a thread block each
    // (main stream, concurrently): the split balances the two kernels' longest serial insertion chains
    h->warp_nmax = std::getenv("IMMESH_WARP_NMAX") ? std::atoi(std::getenv("IMMESH_WARP_NMAX")) : IM_WARP_NMAX;
    if (h->warp_nmax < 3) h->warp_nmax = 3;
    if (h->warp_nmax > 128) h->warp_nmax = 128;
    h->use_graph = std::getenv("IMMESH_GRAPH") ? std::atoi(std::getenv("IMMESH_GRAPH")) : 1;
    MeshParams& P = h->P;
    P.xi = cfg->points_minimum_scale;
    P.res = cfg->voxel_resolution;
    P.accept = cfg->voxel_resolution * 1.25;
    P.knn_max = P.accept * 2 * 1.000001;
    P.inv_q = 4194304.0 / cfg->voxel_resolution;
    P.append_target = cfg->number_of_pts_append_to_map;
    const int max_v = cfg->max_vertices ? cfg->max_vertices : (8 << 20);
    const int max_t = cfg->max_triangles ? cfg->max_triangles : (32 << 20);
    const int max_vox = cfg->max_voxels ? cfg->max_voxels : (2 << 20);
    h->max_frame_points = cfg->max_frame_points ? cfg->max_frame_points : (2 << 20);
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    IM_CREATE_M(cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, im_stream_priority("IMMESH_MESH_PRIO")));
    for (auto& e : h->ev) IM_CREATE_M(cudaEventCreate(&e));
    MeshDev& M = h->M;
    M.max_v = max_v;
    M.max_t = max_t;
    IM_CREATE_M(mdev_alloc(h, &M.vpos, (size_t)max_v));
    IM_CREATE_M(mdev_alloc(h, &M.vsmooth, (size_t)max_v * 3));
    IM_CREATE_M(mdev_alloc(h, &M.v_tri_head, (size_t)max_v, 0xFF));
    const size_t gcap = pow2_at_least((size_t)max_v * 2);
    IM_CREATE_M(mdev_alloc(h, &M.gkeys, gcap, 0xFF));
    IM_CREATE_M(mdev_alloc(h, &M.gval, gcap, 0xFF));
    M.gmask = (unsigned)(gcap - 1);
    const size_t vcap = pow2_at_least((size_t)max_vox * 2);
    IM_CREATE_M(mdev_alloc(h, &M.vkeys, vcap, 0xFF));
    M.vmask = (unsigned)(vcap - 1);
    IM_CREATE_M(mdev_alloc(h, &M.vox_chunk, vcap * IM_VCHUNKS, 0xFF));
    M.max_vchunks = max_v / 4 + 1024;
    IM_CREATE_M(mdev_alloc(h, &M.vchunk_pts, (size_t)M.max_vchunks * 16));
    IM_CREATE_M(mdev_alloc(h, &M.vox_count, vcap, 0));
    IM_CREATE_M(mdev_alloc(h, &M.vox_meshing_times, vcap, 0));
    IM_CREATE_M(mdev_alloc(h, &M.vox_new_added, vcap, 0));
    IM_CREATE_M(mdev_alloc(h, &M.vox_frame, vcap, 0xFF));
    M.vox_short_axis = nullptr;
    IM_CREATE_M(mdev_alloc(h, &M.tri, (size_t)max_t));
    IM_CREATE_M(mdev_alloc(h, &M.tri_next, (size_t)max_t * 3));
    IM_CREATE_M(mdev_alloc(h, &M.tri_flip, (size_t)max_t));
    const size_t tcap = pow2_at_least((size_t)max_t * 2);
    IM_CREATE_M(mdev_alloc(h, &M.thash, tcap, 0xFF));
    M.tmask = (unsigned)(tcap - 1);
    IM_CREATE_M(mdev_alloc(h, &M.cnt, 64, 0));
    {
        int init[32];
        std::memset(init, 0, sizeof(init));
        init[11] = init[12] = init[13] = 0x7fffffff;
        init[14] = init[15] = init[16] = -0x7fffffff;
        IM_CREATE_M(cudaMemcpy(M.cnt, init, sizeof(init), cudaMemcpyHostToDevice));
    }
    FrameBuf& F = h->F;
    const size_t mc = (size_t)h->max_frame_points;  // candidates <= points
    F.max_cand = (int)mc;
    F.max_work = max_vox < (1 << 16) ? max_vox : std::min(std::max(max_vox / 16, 1 << 16), 1 << 18);   // voxels (re)meshed per frame; 4 KB of id list each
    F.max_act = (int)std::min<size_t>((size_t)max_vox, mc);
    F.max_list = 4 << 20;
    IM_CREATE_M(mdev_alloc(h, &h->d_pts, IM_SLOTS * mc * 3));
    IM_CREATE_M(mdev_alloc(h, &h->d_body, IM_SLOTS * mc * 3));   // staging of body-frame scans handed over by the localization handle (not allocated lazily: a cudaMalloc inside a frame stalls the pipeline)
    F.pts = h->d_pts;
    IM_CREATE_M(mdev_alloc(h, &h->d_fp, IM_SLOTS));
    for (int i = 0; i < IM_SLOTS; ++i) { IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming)); IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming)); }
    IM_CREATE_M(mdev_alloc(h, &F.cand_gkey, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_vslot, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_status, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_scan, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_conf, mc * IM_CONF_K));
    IM_CREATE_M(mdev_alloc(h, &F.cand_nconf, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_next, mc));
    IM_CREATE_M(mdev_alloc(h, &F.cand_pos, mc));
    h->ccap = pow2_at_least(mc * 2);
    IM_CREATE_M(mdev_alloc(h, &F.ckeys, h->ccap));
    IM_CREATE_M(mdev_alloc(h, &F.chead, h->ccap));
    F.scan_block = nullptr;
    IM_CREATE_M(mdev_alloc(h, &F.act, (size_t)F.max_act));
    IM_CREATE_M(mdev_alloc(h, &F.work, (size_t)F.max_work));
    IM_CREATE_M(mdev_alloc(h, &F.work_n_ids, (size_t)F.max_work));
    IM_CREATE_M(mdev_alloc(h, &F.work_ids, (size_t)F.max_work * IM_MAXD));
    IM_CREATE_M(mdev_alloc(h, &F.work_nfaces, (size_t)F.max_work));
    IM_CREATE_M(mdev_alloc(h, &F.work_bits, (size_t)F.max_work * (IM_MAXG / 32), 0));
    IM_CREATE_M(mdev_alloc(h, &F.work_ring, (size_t)F.max_work, 0));
    IM_CREATE_M(mdev_alloc(h, &F.work_done, (size_t)F.max_work, 0));
    F.max_ditem = F.max_work * 4;
    IM_CREATE_M(mdev_alloc(h, &F.ditem, (size_t)F.max_ditem));
    F.max_vref = 8 << 20;
    IM_CREATE_M(mdev_alloc(h, &F.all_faces, (size_t)F.max_list));
    IM_CREATE_M(mdev_alloc(h, &F.all_vref, (size_t)F.max_vref));
    IM_CREATE_M(mdev_alloc(h, &F.pulled, (size_t)F.max_list * 2));
    F.fset_mask = (1u << 21) - 1;
    IM_CREATE_M(mdev_alloc(h, &F.fset, (size_t)F.fset_mask + 1, 0xFF));
    IM_CREATE_M(mdev_alloc(h, &F.work_axes, (size_t)F.max_work * 9));
    IM_CREATE_M(mdev_alloc(h, &F.add_tri, (size_t)F.max_list * 3));
    IM_CREATE_M(mdev_alloc(h, &F.add_flip, (size_t)F.max_list));
    IM_CREATE_M(mdev_alloc(h, &F.rem_tri, (size_t)F.max_list));
    IM_CREATE_M(cudaMallocHost((void**)&h->h_pts, IM_SLOTS * mc * 3 * sizeof(float)));
    IM_CREATE_M(cudaMallocHost((void**)&h->h_cnt, IM_SLOTS * 32 * sizeof(int)));
    IM_CREATE_M(cudaMallocHost((void**)&h->h_fp, IM_SLOTS * sizeof(FramePose)));
    IM_CREATE_M(cudaMallocHost((void**)&h->h_dyn, IM_SLOTS * sizeof(FrameDyn)));
    IM_CREATE_M(mdev_alloc(h, &h->d_dyn, 1, 0));
    F.dyn = h->d_dyn;
    F.epoch = 0;
    IM_CREATE_M(cudaFuncSetAttribute(k_voxel_mesh<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<1024>)));
    IM_CREATE_M(cudaFuncSetAttribute(k_voxel_tri_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(4 * sizeof(MeshWarpSmem<128>))));
    IM_CREATE_M(cudaFuncSetAttribute(k_voxel_mesh<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<256>)));
    IM_CREATE_M(cudaStreamCreateWithPriority(&h->stream2, cudaStreamNonBlocking, im_stream_priority("IMMESH_MESH_PRIO")));
    IM_CREATE_M(cudaStreamCreateWithPriority(&h->stream3, cudaStreamNonBlocking, im_stream_priority("IMMESH_MESH_PRIO")));
    IM_CREATE_M(cudaStreamCreateWithFlags(&h->stream_up, cudaStreamNonBlocking));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_up[i], cudaEventDisableTiming));
    IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    IM_CREATE_M(cudaEventCreateWithFlags(&h->ev_join3, cudaEventDisableTiming));
    std::memset(h->last_cnt, 0, sizeof(h->last_cnt));
    IM_CREATE_M(cudaDeviceSynchronize());
#undef IM_CREATE_M
    *out = h;
    return IMMESH_OK;
}

int immesh_mesh_destroy(immesh_mesh_t* h) {
    if (!h) return IMMESH_OK;
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->graph.destroy();
    if (h->win.local) immesh::peer_window_close(h->win);
    if (h->nccl_comm && immesh::nccl().CommDestroy) immesh::nccl().CommDestroy(h->nccl_comm);
    for (void* p : h->allocs) cudaFree(p);
    if (h->h_pts) cudaFreeHost(h->h_pts);
    if (h->h_cnt) cudaFreeHost(h->h_cnt);
    if (h->h_fp) cudaFreeHost(h->h_fp);
    if (h->h_dyn) cudaFreeHost(h->h_dyn);
    for (int i = 0; i < IM_SLOTS; ++i) { if (h->ev_in[i]) cudaEventDestroy(h->ev_in[i]); if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]); }
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    if (h->stream) cudaStreamDestroy(h->stream);
    if (h->stream2) cudaStreamDestroy(h->stream2);
    if (h->stream3) cudaStreamDestroy(h->stream3);
    if (h->stream_up) cudaStreamDestroy(h->stream_up);
    for (int i = 0; i < IM_SLOTS; ++i) if (h->ev_up[i]) cudaEventDestroy(h->ev_up[i]);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    if (h->ev_join3) cudaEventDestroy(h->ev_join3);
    delete h;
    return IMMESH_OK;
}

static int mesh_grid(const immesh_mesh* h, int n, int threads, int waves = 8) {
    int g = (n + threads - 1) / threads;
    if (g > h->n_sm * waves) g = h->n_sm * waves;
    return g < 1 ? 1 : g;
}

// transformLidar of the full-resolution scan with the converged state (ImMesh_mesh_reconstruction.cpp:413 ->
// voxel_mapping_common.cpp:709-726): p_w = (float)( R (R_ext p + t_ext) + t ).  First kernel of a frame handed over by the
// localization handle: the pose is the one that scan converged to (LioCtrl::pose_ring, written by the last kernel of the
// scan's sequence; the localization stream may already be working on later scans).  Block 0 also derives the frame's sensor
// position + the origin of the flip-priority rank.
__global__ void __launch_bounds__(128) k_transform_full(LioParams P, const LioCtrl* ctrl, FrameBuf F_, double res) {
    __shared__ double s[12];
    const FrameDyn d = *F_.dyn;
    if (threadIdx.x < 12) s[threadIdx.x] = ctrl->pose_ring[d.pose_idx][threadIdx.x];
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < 3) {
        const double t = s[9 + threadIdx.x];
        d.fp->pose_t[threadIdx.x] = t;
        d.fp->prio_origin[threadIdx.x] = (long long)floor(t / res) - 1024;
    }
    const float* body = d.body;
    float* world = const_cast<float*>(d.pts);
    const int n = d.n;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double pb[3] = {(double)body[(size_t)i * 3 + 0], (double)body[(size_t)i * 3 + 1], (double)body[(size_t)i * 3 + 2]};
        double pw[3];
        body_to_world(P, s, s + 9, pb, pw);
        world[(size_t)i * 3 + 0] = (float)pw[0]; world[(size_t)i * 3 + 1] = (float)pw[1]; world[(size_t)i * 3 + 2] = (float)pw[2];
    }
}
// blocking localization calls (immesh_lio_estimate, set_state, ...) do not publish a pose: done on request, on the localization stream
__global__ void k_pose_publish(LioCtrl* ctrl, int idx) {
    if (threadIdx.x < 12) ctrl->pose_ring[idx][threadIdx.x] = ctrl->state[threadIdx.x];
}

// ---- multi-GPU exchange of the per-voxel stage (sharded mesher).  A segment = [16-B header: counts][entries, x_cap each].
struct XHeader { int n_smooth, n_face, n_rem, pad; };
__global__ void k_xhdr(MeshDev M, FrameBuf F_, XHeader* hdr) {
    const FrameBuf F = frame_load_dyn(F_);
    if (threadIdx.x == 0) {
        hdr->n_smooth = min(M.cnt[32], F.x_cap);
        hdr->n_face = min(M.cnt[30], F.x_cap);
        hdr->n_rem = min(M.cnt[31], F.x_cap);
        hdr->pad = 0;
    }
}
// ---- the same exchange over peer windows (peer_win.cuh): k_xpush stores the USED part of this rank's segment straight into
// slot `rank` of every rank's receive area (its own included) and the last block raises the epoch flag; the apply kernels
// wait on the flags of their peers.  Window: flag[2][8] u64 | pad to 256 | recv1[n][seg1_bytes] | recv2[n][seg2_bytes].
struct MeshPeers {
    unsigned char* w[IM_MAX_RANKS];
    int rank, n;          // n == 0: NCCL transport (no waiting inside the apply kernels)
    unsigned long long recv_off[2], seg_bytes[2];
};
__device__ __forceinline__ unsigned long long* meshwin_flag(unsigned char* w, int which, int src) { return (unsigned long long*)w + which * IM_MAX_RANKS + src; }
__device__ __forceinline__ void copy16(unsigned char* dst, const unsigned char* src, size_t n16, int tid, int nt) {
    for (size_t i = tid; i < n16; i += nt) ((uint4*)dst)[i] = ((const uint4*)src)[i];
}
__global__ void __launch_bounds__(256) k_xpush(MeshDev M, FrameBuf F_, const unsigned char* seg, int which, MeshPeers pe, int* done) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    __shared__ int s_last;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    const int n_smooth = min(M.cnt[32], F.x_cap), n_face = min(M.cnt[30], F.x_cap), n_rem = min(M.cnt[31], F.x_cap);
    for (int r = 0; r < pe.n; ++r) {
        unsigned char* dst = pe.w[r] + pe.recv_off[which] + (size_t)pe.rank * pe.seg_bytes[which];
        if (tid == 0) *(int4*)dst = make_int4(n_smooth, n_face, n_rem, 0);
        if (which == 0) {
            copy16(dst + 16, seg + 16, (size_t)n_smooth * 2, tid, nt);
        } else {
            copy16(dst + 16, seg + 16, (size_t)n_face, tid, nt);
            const size_t woff = 16 + (size_t)F.x_cap * 16, roff = 16 + (size_t)F.x_cap * 24;
            copy16(dst + woff, seg + woff, ((size_t)n_face + 1) / 2, tid, nt);
            copy16(dst + roff, seg + roff, (size_t)n_rem, tid, nt);
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(done, 1) == (int)gridDim.x - 1);
    __syncthreads();
    if (s_last) {
        if (threadIdx.x == 0) *done = 0;
        __threadfence_system();
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) immesh::st_release_sys(meshwin_flag(pe.w[threadIdx.x], which, pe.rank), epoch);
    }
}
__device__ __forceinline__ void mesh_wait_peers(const MeshPeers& pe, int which, unsigned long long epoch, int* err) {
    if (pe.n > 0) {
        if (threadIdx.x < pe.n && threadIdx.x != pe.rank) {
            immesh::wait_epoch(meshwin_flag(pe.w[pe.rank], which, threadIdx.x), epoch, err, IM_MERR_PEER_TIMEOUT);
        }
        __syncthreads();
    }
}
// smoothed positions written by the other ranks' dilations -> this rank's replica
__global__ void __launch_bounds__(256) k_apply_smooth(MeshDev M, FrameBuf F_, const unsigned char* recv, size_t seg_bytes, MeshPeers pe) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    mesh_wait_peers(pe, 0, epoch, &M.cnt[3]);
    for (int r = 0; r < F.shard_n; ++r) {
        if (r == F.shard_rank) continue;
        const unsigned char* seg = recv + (size_t)r * seg_bytes;
        const int n = __ldcg((const int*)seg);
        const double2* e = (const double2*)(seg + 16);
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            const double2 a = __ldcg(e + 2 * (size_t)i), b = __ldcg(e + 2 * (size_t)i + 1);   // {id|pad, x}, {y, z}
            const int id = (int)(__double_as_longlong(a.x) & 0xffffffffLL);
            M.vsmooth[(size_t)id * 3 + 0] = a.y; M.vsmooth[(size_t)id * 3 + 1] = b.x; M.vsmooth[(size_t)id * 3 + 2] = b.y;
        }
    }
}
// facets / removals of ALL ranks (own segment included) -> add / remove lists of this rank's replica
__global__ void __launch_bounds__(256) k_apply_lists(MeshDev M, FrameBuf F_, const unsigned char* recv, size_t seg_bytes, MeshPeers pe) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    mesh_wait_peers(pe, 1, epoch, &M.cnt[3]);
    for (int r = 0; r < F.shard_n; ++r) {
        const unsigned char* seg = recv + (size_t)r * seg_bytes;
        const int4 h = __ldcg((const int4*)seg);   // n_smooth, n_face, n_rem, -
        const int4* face = (const int4*)(seg + 16);
        const unsigned long long* word = (const unsigned long long*)(seg + 16 + (size_t)F.x_cap * 16);
        const int4* rem = (const int4*)(seg + 16 + (size_t)F.x_cap * 24);
        const int nf = h.y, nr = h.z;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nf + nr; i += gridDim.x * blockDim.x) {
            if (i < nf) { const int4 f = __ldcg(face + i); apply_face(M, F, f.x, f.y, f.z, __ldcg(word + i)); }
            else { const int4 t = __ldcg(rem + (i - nf)); apply_remove(M, F, t.x, t.y, t.z); }
        }
    }
}

static int mesh_status(int err) {
    if (err & (IM_MERR_VERT_POOL | IM_MERR_TRI_POOL | IM_MERR_HASH_FULL | IM_MERR_LIST_CAP | IM_MERR_VOXEL_CAP)) {
        // name every flag that fired: the caller can tell a full pool from a per-voxel working set over its cap
        std::string m = "mesh pool / per-voxel working-set overflow (flags:";
        if (err & IM_MERR_VERT_POOL) m += " VERT_POOL";
        if (err & IM_MERR_TRI_POOL) m += " TRI_POOL";
        if (err & IM_MERR_HASH_FULL) m += " HASH_FULL";
        if (err & IM_MERR_LIST_CAP) m += " LIST_CAP";
        if (err & IM_MERR_VOXEL_CAP) m += " VOXEL_CAP";
        m += ")";
        return im_fail(IMMESH_E_CAPACITY, m.c_str());
    }
    if (err & (IM_MERR_KEY_RANGE | IM_MERR_PRIO_RANGE)) return im_fail(IMMESH_E_RANGE, "mesh key out of range");
    if (err & IM_MERR_PEER_TIMEOUT) return im_fail(IMMESH_E_CUDA, "sharded mesher: a peer rank did not publish its segment in time (peer window epoch flag)");
    return IMMESH_OK;
}
// wait for the frame queued in slot s and take over its counters
static int mesh_harvest(immesh_mesh* h, int s) {
    if (!h->inflight[s]) return IMMESH_OK;
    if (cudaEventQuery(h->ev_done[s]) != cudaSuccess) {
        cudaGetLastError();
        const auto t0 = std::chrono::steady_clock::now();
        IM_CUDA(cudaEventSynchronize(h->ev_done[s]));
        h->host_wait_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    }
    h->inflight[s] = 0;
    std::memcpy(h->last_cnt, h->h_cnt + 32 * s, 32 * sizeof(int));
    const int rc = mesh_status(h->last_cnt[3]);
    if (rc && !h->pending_rc) h->pending_rc = rc;
    return rc;
}

static bool mesh_host_ptr_is_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}
static int mesh_grid_fixed(const immesh_mesh* h, long long n_cap, int threads, int waves = 8) {
    long long g = (n_cap + threads - 1) / threads;
    if (g > (long long)h->n_sm * waves) g = (long long)h->n_sm * waves;
    return g < 1 ? 1 : (int)g;
}
// src_mode: 0 host world points, 1 device world points, 2 host body points + lio state, 3 device body points + lio state.
// Queues one frame (no host synchronisation except when both staging slots are still busy).  Host work per frame in the
// pipelined form: (memcpy into the pinned slot unless the caller's buffer is pinned) + H2D scan + H2D FrameDyn + one stream
// wait + ONE cudaGraphLaunch (no node is touched: every per-frame value is read from the FrameDyn) + one D2H of the counters.
static int mesh_enqueue(immesh_mesh_t* h, const float* xyz, int n, const double* pose_t, int src_mode, immesh_lio* lio, bool allow_graph = false) {
    if (!h || (!xyz && n > 0) || n < 0 || (src_mode < 2 && !pose_t)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_frame_points) return im_fail(IMMESH_E_CAPACITY, "frame larger than max_frame_points");
    FrameBuf& F = h->F;
    const MeshParams& P = h->P;
    // append_point_step = max(1, round(N / appending_pts_frame)), integer division first (ImMesh_mesh_reconstruction.cpp:111)
    const int step = std::max(1, (int)std::lround((double)(n / P.append_target)));
    F.n = n;
    F.step = step;
    F.m = n > 0 ? (n + step - 1) / step : 0;
    F.frame = ++h->frame_counter;
    const int s = F.frame & (IM_SLOTS - 1);
    int rc = mesh_harvest(h, s);  // the frame IM_SLOTS calls ago used this slot
    (void)rc;
    const size_t slot_pts = (size_t)h->max_frame_points * 3;
    float* d_pts = h->d_pts + s * slot_pts;
    float* h_pts = h->h_pts + s * slot_pts;
    FramePose* d_fp = h->d_fp + s;
    F.fp = d_fp;
    F.cmask = (unsigned)(pow2_at_least((size_t)std::max(F.m, 1) * 2) - 1);
    cudaStream_t st = h->stream;
    const bool graphed = allow_graph && h->use_graph && !profiler().enabled && (F.shard_n <= 1 || h->win.ok);
    if (!graphed) IM_CUDA(cudaEventRecord(h->ev[0], st));
    F.pts = d_pts;
    const float* d_body = nullptr;
    int pose_idx = 0;
    if (src_mode < 2) {
        FramePose* hp = h->h_fp + s;
        for (int j = 0; j < 3; ++j) { hp->pose_t[j] = pose_t[j]; hp->prio_origin[j] = (long long)std::floor(pose_t[j] / P.res) - 1024; }
        IM_CUDA(cudaMemcpyAsync(d_fp, hp, sizeof(FramePose), cudaMemcpyHostToDevice, st));
        if (n > 0) {
            if (src_mode == 0) {
                const float* src = xyz;
                if (!mesh_host_ptr_is_pinned(xyz)) { std::memcpy(h_pts, xyz, (size_t)n * 3 * sizeof(float)); src = h_pts; }
                IM_CUDA(cudaMemcpyAsync(d_pts, src, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream_up));
                IM_CUDA(cudaEventRecord(h->ev_up[s], h->stream_up));
                IM_CUDA(cudaStreamWaitEvent(st, h->ev_up[s], 0));
            } else {
                F.pts = xyz;
            }
        }
    } else {
        // the body-frame scan does not depend on the localization: it is uploaded on the mesh stream right away
        d_body = xyz;
        if (src_mode == 2 && n > 0) {
            if (!h->d_body) IM_CUDA(mdev_alloc(h, &h->d_body, IM_SLOTS * slot_pts));
            const float* src = xyz;
            if (!mesh_host_ptr_is_pinned(xyz)) { std::memcpy(h_pts, xyz, (size_t)n * 3 * sizeof(float)); src = h_pts; }
            // upload stream: overlaps the kernels of the frame before (slot s was released by mesh_harvest above)
            IM_CUDA(cudaMemcpyAsync(h->d_body + s * slot_pts, src, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream_up));
            IM_CUDA(cudaEventRecord(h->ev_up[s], h->stream_up));
            IM_CUDA(cudaStreamWaitEvent(st, h->ev_up[s], 0));
            d_body = h->d_body + s * slot_pts;
        }
        // the pose: published by the last kernel of the scan's sequence (step entry points), else on request
        if (lio->pose_pub_idx < 0) {
            lio->pose_pub_idx = ++lio->scan_counter;
            IM_LAUNCH(k_pose_publish, 1, 32, 0, lio->stream, lio->d_ctrl, lio->pose_pub_idx & (IM_POSE_RING - 1));
        }
        pose_idx = lio->pose_pub_idx & (IM_POSE_RING - 1);
        IM_CUDA(cudaEventRecord(lio->ev_pose, lio->stream));
        IM_CUDA(cudaStreamWaitEvent(st, lio->ev_pose, 0));
    }
    MeshPeers pe;
    std::memset(&pe, 0, sizeof(pe));
    unsigned long long epoch = 0;
    if (F.shard_n > 1 && h->win.ok) {   // one epoch per frame; the two exchanges have separate flag rows
        for (int r = 0; r < IM_MAX_RANKS; ++r) pe.w[r] = h->win.peer[r];
        pe.rank = h->win.rank; pe.n = h->win.n;
        pe.recv_off[0] = 256; pe.recv_off[1] = 256 + (unsigned long long)h->seg1_bytes * h->win.n;
        pe.seg_bytes[0] = h->seg1_bytes; pe.seg_bytes[1] = h->seg2_bytes;
        epoch = ++h->win.epoch;
    }
    F.epoch = epoch;
    {   // the frame's device-resident inputs
        FrameDyn& d = h->h_dyn[s];
        d.pts = F.pts; d.body = d_body; d.fp = d_fp;
        d.n = F.n; d.step = F.step; d.m = F.m; d.frame = F.frame; d.cmask = F.cmask; d.pose_idx = pose_idx; d.epoch = epoch;
        IM_CUDA(cudaMemcpyAsync(h->d_dyn, &d, sizeof(FrameDyn), cudaMemcpyHostToDevice, st));
    }
    // the frame's launch sequence (fixed grids: grid-stride loops over the counts the kernels read on the device)
    bool nccl_failed = false;
    const int g_pts = mesh_grid_fixed(h, h->max_frame_points, 128);
    const int g_cand = mesh_grid_fixed(h, std::min<long long>(h->max_frame_points, 2LL * P.append_target), 128);
    auto launch_frame = [&](bool timing) {
        if (src_mode >= 2) IM_LAUNCH(k_transform_full, g_pts, 128, 0, st, lio->P, (const LioCtrl*)lio->d_ctrl, F, P.res);
        IM_LAUNCH(k_frame_begin, h->n_sm * 8, 256, 0, st, h->M, F);
        if (timing) cudaEventRecord(h->ev[1], st);
        IM_LAUNCH(k_cand_init, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_cand_conflicts, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_cand_resolve, h->n_sm * 4, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_cand_scan, 1, 1024, 0, st, h->M, F);
        IM_LAUNCH(k_cand_commit, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_cand_place, g_cand, 128, 0, st, h->M, F);
        IM_LAUNCH(k_voxel_select, g_cand, 128, 0, st, h->M, F);
        if (timing) cudaEventRecord(h->ev[2], st);
        IM_LAUNCH(k_voxel_dilate, h->n_sm * h->dilate_bps, 128, 0, st, h->M, P, F);
        if (F.shard_n > 1 && h->win.ok) {   // smoothed positions of the other ranks' voxels, pushed into their windows
            IM_LAUNCH(k_xpush, h->n_sm, 256, 0, st, h->M, F, (const unsigned char*)h->d_seg1, 0, pe, h->d_xdone);
            IM_LAUNCH(k_apply_smooth, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv1, h->seg1_bytes, pe);
        } else if (F.shard_n > 1) {   // NCCL transport
            IM_LAUNCH(k_xhdr, 1, 32, 0, st, h->M, F, (XHeader*)h->d_seg1);
            if (immesh::nccl().AllGather(h->d_seg1, h->d_recv1, h->seg1_bytes, immesh::kNcclUint8, h->nccl_comm, st)) nccl_failed = true;
            IM_LAUNCH(k_apply_smooth, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv1, h->seg1_bytes, pe);
        }
        // triangulation: small dilated sets warp-level on the side stream, mid-size ones block-level on the main stream,
        // concurrently; then the rare large / handed-over ones (monolithic: triangulate + commit in shared memory)
        cudaEventRecord(h->ev_fork, st);
        cudaStreamWaitEvent(h->stream2, h->ev_fork, 0);
        cudaStreamWaitEvent(h->stream3, h->ev_fork, 0);
        IM_LAUNCH(k_voxel_tri_warp, h->n_sm * h->bps, 128, 4 * sizeof(MeshWarpSmem<128>), h->stream2, h->M, P, F, h->warp_nmax);
        cudaEventRecord(h->ev_join, h->stream2);
        IM_LAUNCH(k_pull_vertices, h->n_sm * 8, 128, 0, h->stream3, h->M, P, F);   // incidence-list walk: only needs the dilation
        cudaEventRecord(h->ev_join3, h->stream3);
        IM_LAUNCH((k_voxel_mesh<256>), h->n_sm * h->bps, 128, sizeof(MeshSmem<256>), st, h->M, P, F, h->warp_nmax, 1);
        cudaStreamWaitEvent(st, h->ev_join, 0);
        cudaStreamWaitEvent(st, h->ev_join3, 0);
        IM_LAUNCH((k_voxel_mesh<1024>), h->n_sm * 2, 128, sizeof(MeshSmem<1024>), st, h->M, P, F, 256, 0);
        IM_LAUNCH(k_commit_faces, h->n_sm * 8, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_pull_check, h->n_sm * 8, 128, 0, st, h->M, F);
        if (F.shard_n > 1 && h->win.ok) {   // every rank applies the facets / removals of all ranks to its replica of the store
            IM_LAUNCH(k_xpush, h->n_sm, 256, 0, st, h->M, F, (const unsigned char*)h->d_seg2, 1, pe, h->d_xdone + 1);
            IM_LAUNCH(k_apply_lists, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv2, h->seg2_bytes, pe);
        } else if (F.shard_n > 1) {
            IM_LAUNCH(k_xhdr, 1, 32, 0, st, h->M, F, (XHeader*)h->d_seg2);
            if (immesh::nccl().AllGather(h->d_seg2, h->d_recv2, h->seg2_bytes, immesh::kNcclUint8, h->nccl_comm, st)) nccl_failed = true;
            IM_LAUNCH(k_apply_lists, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv2, h->seg2_bytes, pe);
        }
        if (timing) cudaEventRecord(h->ev[3], st);
        IM_LAUNCH(k_push_remove, h->n_sm * 2, 128, 0, st, h->M, F);
        IM_LAUNCH(k_push_add, h->n_sm * 2, 128, 0, st, h->M, F);
        IM_LAUNCH(k_frame_end, 1, 1, 0, st, h->M);
    };
    bool queued = false;
    if (graphed) {
        // signature: everything that changes the sequence or its (static) arguments
        const unsigned long long lp = (unsigned long long)(uintptr_t)lio;
        const unsigned sig = (h->win.ok ? 2u : 0u) | 1u | ((unsigned)src_mode << 2) | ((unsigned)F.shard_n << 5) | ((unsigned)((lp >> 4) ^ (lp >> 36)) << 9);
        queued = immesh::run_graphed_static(h->graph, sig, st, [&] { launch_frame(false); }) == cudaSuccess;
        if (!queued) { h->use_graph = 0; IM_CUDA(cudaEventRecord(h->ev[0], st)); }
    }
    if (!queued) launch_frame(true);
    if (nccl_failed) return im_fail(IMMESH_E_CUDA, "ncclAllGather failed");
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(h->h_cnt + 32 * s, h->M.cnt, 32 * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!queued) IM_CUDA(cudaEventRecord(h->ev[4], st));
    IM_CUDA(cudaEventRecord(h->ev_done[s], st));
    h->inflight[s] = 1;
    h->timed_last = queued ? 0 : 1;
    return IMMESH_OK;
}
// drain the queue; returns the status of the frames harvested since the last call
static int mesh_wait_impl(immesh_mesh_t* h, bool timings) {
    for (int i = 1; i <= IM_SLOTS; ++i) mesh_harvest(h, (h->frame_counter + i) & (IM_SLOTS - 1));   // oldest frame first: last_cnt ends as the newest frame's
    if (profiler().enabled) {
        cudaStreamSynchronize(h->stream);
        profiler().collect();
    }
    if (timings && h->timed_last) {
        float a = 0, b = 0, c = 0, d = 0;
        cudaEventElapsedTime(&a, h->ev[0], h->ev[4]);
        cudaEventElapsedTime(&b, h->ev[1], h->ev[2]);
        cudaEventElapsedTime(&c, h->ev[2], h->ev[3]);
        cudaEventElapsedTime(&d, h->ev[3], h->ev[4]);
        h->last_ms[0] = a; h->last_ms[1] = b; h->last_ms[2] = c; h->last_ms[3] = d;
    }
    const int rc = h->pending_rc;
    h->pending_rc = 0;
    return rc;
}

int immesh_mesh_push_frame(immesh_mesh_t* h, const float* world_xyz, int n, const double* pose_t, int frame_idx) {
    (void)frame_idx;
    int rc = mesh_enqueue(h, world_xyz, n, pose_t, 0, nullptr);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_dev(immesh_mesh_t* h, const float* d_world_xyz, int n, const double* pose_t, int frame_idx) {
    (void)frame_idx;
    int rc = mesh_enqueue(h, d_world_xyz, n, pose_t, 1, nullptr);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_from_lio(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    int rc = mesh_enqueue(h, body_xyz, n, nullptr, on_device ? 3 : 2, lio);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_from_lio_async(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    return mesh_enqueue(h, body_xyz, n, nullptr, on_device ? 3 : 2, lio, true);
}
// device-side timing of a pipelined batch: begin mark on the localization stream, end mark behind BOTH streams
int immesh_pipeline_mark_begin(immesh_lio_t* lio) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null handle");
    if (!lio->ev_mark) IM_CUDA(cudaEventCreate(&lio->ev_mark));
    IM_CUDA(cudaEventRecord(lio->ev_mark, lio->stream));
    return IMMESH_OK;
}
int immesh_pipeline_mark_end(immesh_lio_t* lio, immesh_mesh_t* h, double* ms) {
    if (!lio || !h || !ms || !lio->ev_mark) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!h->ev_mark) { IM_CUDA(cudaEventCreate(&h->ev_mark)); IM_CUDA(cudaEventCreateWithFlags(&h->ev_sync, cudaEventDisableTiming)); }
    IM_CUDA(cudaEventRecord(h->ev_sync, lio->stream));
    IM_CUDA(cudaStreamWaitEvent(h->stream, h->ev_sync, 0));
    IM_CUDA(cudaEventRecord(h->ev_mark, h->stream));
    IM_CUDA(cudaEventSynchronize(h->ev_mark));
    float t = 0.f;
    IM_CUDA(cudaEventElapsedTime(&t, lio->ev_mark, h->ev_mark));
    *ms = t;
    return IMMESH_OK;
}
int immesh_mesh_shard(immesh_mesh_t* h, int rank, int nranks, const char* unique_id128) {
    if (!h || !unique_id128 || nranks < 1 || rank < 0 || rank >= nranks) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (nranks == 1) { h->F.shard_rank = 0; h->F.shard_n = 1; return IMMESH_OK; }
    if (!immesh::nccl().load()) return im_fail(IMMESH_E_CUDA, "libnccl.so.2 not found");
    immesh::nccl_uid_t id;
    std::memcpy(id.internal, unique_id128, 128);
    immesh::nccl_comm_t comm = nullptr;
    const int rc = immesh::nccl().CommInitRank(&comm, nranks, id, rank);
    if (rc) return im_fail(IMMESH_E_CUDA, immesh::nccl().GetErrorString ? immesh::nccl().GetErrorString(rc) : "ncclCommInitRank failed");
    h->nccl_comm = comm;
    FrameBuf& F = h->F;
    F.shard_rank = rank;
    F.shard_n = nranks;
    F.x_cap = 1 << 16;
    // segment 1: header + smoothed positions; segment 2: header + facets + words + removals
    h->seg1_bytes = 16 + (size_t)F.x_cap * sizeof(immesh::XSmooth);
    h->seg2_bytes = 16 + (size_t)F.x_cap * (16 + 8 + 16);
    unsigned char *s1 = nullptr, *s2 = nullptr;
    IM_CUDA(mdev_alloc(h, &s1, h->seg1_bytes, 0));
    IM_CUDA(mdev_alloc(h, &s2, h->seg2_bytes, 0));
    // receive areas: inside a peer window (other ranks store into it over NVLink) or, with NCCL transport, private buffers
    const char* force_nccl = std::getenv("IMMESH_SHARD_NCCL");
    if (!(force_nccl && force_nccl[0] == '1')) {
        const cudaError_t e = immesh::peer_window_open(h->win, 256 + (h->seg1_bytes + h->seg2_bytes) * (size_t)nranks, rank, nranks, comm, h->stream);
        if (e != cudaSuccess) {
            std::fprintf(stderr, "[immesh_b200] rank %d: peer window unavailable (%s); sharded mesher falls back to NCCL all-gathers\n", rank, cudaGetErrorString(e));
            cudaGetLastError();
        }
    }
    if (h->win.ok) {
        h->d_recv1 = h->win.local + 256;
        h->d_recv2 = h->win.local + 256 + h->seg1_bytes * (size_t)nranks;
        IM_CUDA(mdev_alloc(h, &h->d_xdone, 2, 0));
    } else {
        IM_CUDA(mdev_alloc(h, &h->d_recv1, h->seg1_bytes * nranks, 0));
        IM_CUDA(mdev_alloc(h, &h->d_recv2, h->seg2_bytes * nranks, 0));
    }
    h->d_seg1 = s1; h->d_seg2 = s2;
    F.x_smooth = (immesh::XSmooth*)(s1 + 16);
    F.x_face = (int4*)(s2 + 16);
    F.x_word = (unsigned long long*)(s2 + 16 + (size_t)F.x_cap * 16);
    F.x_rem = (int4*)(s2 + 16 + (size_t)F.x_cap * 24);
    return IMMESH_OK;
}
int immesh_mesh_shard_transport(immesh_mesh_t* h) {
    if (!h || h->F.shard_n <= 1) return 0;
    return h->win.ok ? 2 : 1;
}
int immesh_graph_stats(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 6; ++i) out[i] = 0;
    if (lio) { out[0] = lio->graph.captures; out[1] = lio->graph.replays; out[2] = lio->graph.failures; }
    if (mesh) { out[3] = mesh->graph.captures; out[4] = mesh->graph.replays; out[5] = mesh->graph.failures; }
    return IMMESH_OK;
}
// host time (ms) the enqueue calls spent blocked on busy staging slots since the last call of this function: [lio, mesh].
// Queueing a scan costs (wall time of the call) - (this): the rest is back-pressure from the device.
int immesh_host_wait_ms(immesh_lio_t* lio, immesh_mesh_t* mesh, double* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    out[0] = lio ? lio->host_wait_ms : 0.0;
    out[1] = mesh ? mesh->host_wait_ms : 0.0;
    if (lio) lio->host_wait_ms = 0;
    if (mesh) mesh->host_wait_ms = 0;
    return IMMESH_OK;
}
int immesh_mesh_wait(immesh_mesh_t* h) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    return mesh_wait_impl(h, false);
}

int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    out[0] = c[0]; out[1] = c[2]; out[2] = c[10]; out[3] = c[6] + c[17]; out[4] = c[7]; out[5] = c[8]; out[6] = c[4]; out[7] = c[5];
    return IMMESH_OK;
}

int immesh_mesh_work_stats(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    out[0] = h->F.m; out[1] = c[20]; out[2] = c[21]; out[3] = c[22]; out[4] = c[23]; out[5] = c[6] + c[17]; out[6] = c[7]; out[7] = c[8];
    return IMMESH_OK;
}

int immesh_mesh_snapshot(immesh_mesh_t* h, float* vertices, int32_t* triangles, int32_t* flips) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    int cnt[32];
    IM_CUDA(cudaMemcpy(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    const int nv = cnt[0], nalloc = std::min(cnt[1], h->M.max_t), nlive = cnt[2];
    if (vertices && nv > 0) {
        std::vector<float4> v(nv);
        IM_CUDA(cudaMemcpy(v.data(), h->M.vpos, (size_t)nv * sizeof(float4), cudaMemcpyDeviceToHost));
        for (int i = 0; i < nv; ++i) { vertices[i * 3] = v[i].x; vertices[i * 3 + 1] = v[i].y; vertices[i * 3 + 2] = v[i].z; }
    }
    if ((triangles || flips) && nlive > 0) {
        int *d_tri = nullptr, *d_flip = nullptr, *d_n = nullptr;
        IM_CUDA(cudaMalloc(&d_tri, (size_t)nlive * 3 * sizeof(int)));
        IM_CUDA(cudaMalloc(&d_flip, (size_t)nlive * sizeof(int)));
        IM_CUDA(cudaMalloc(&d_n, sizeof(int)));
        IM_CUDA(cudaMemset(d_n, 0, sizeof(int)));
        IM_LAUNCH(k_snapshot, mesh_grid(h, nalloc, 128), 128, 0, h->stream, h->M, nalloc, d_tri, d_flip, d_n);
        std::vector<int> t((size_t)nlive * 3), f(nlive);
        IM_CUDA(cudaMemcpyAsync(t.data(), d_tri, (size_t)nlive * 3 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        IM_CUDA(cudaMemcpyAsync(f.data(), d_flip, (size_t)nlive * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        IM_CUDA(cudaStreamSynchronize(h->stream));
        cudaFree(d_tri); cudaFree(d_flip); cudaFree(d_n);
        std::vector<int> order(nlive);
        for (int i = 0; i < nlive; ++i) order[i] = i;
        std::sort(order.begin(), order.end(), [&](int a, int b) {
            for (int j = 0; j < 3; ++j)
                if (t[(size_t)a * 3 + j] != t[(size_t)b * 3 + j]) return t[(size_t)a * 3 + j] < t[(size_t)b * 3 + j];
            return false;
        });
        for (int i = 0; i < nlive; ++i) {
            if (triangles)
                for (int j = 0; j < 3; ++j) triangles[(size_t)i * 3 + j] = t[(size_t)order[i] * 3 + j];
            if (flips) flips[i] = f[order[i]];
        }
    }
    return IMMESH_OK;
}

int immesh_knn(immesh_mesh_t* h, const float* query_xyz, int nq, int k, double max_dist, int32_t* idx, float* d2) {
    if (!h || !query_xyz || !idx || !d2 || nq < 0 || k < 1 || k > KNN_KMAX) return im_fail(IMMESH_E_INVALID, "bad argument (k must be in [1,32])");
    if (nq == 0) return IMMESH_OK;
    float* dq = nullptr;
    int* di = nullptr;
    float* dd = nullptr;
    IM_CUDA(cudaMalloc(&dq, (size_t)nq * 3 * sizeof(float)));
    IM_CUDA(cudaMalloc(&di, (size_t)nq * k * sizeof(int)));
    IM_CUDA(cudaMalloc(&dd, (size_t)nq * k * sizeof(float)));
    IM_CUDA(cudaMemcpyAsync(dq, query_xyz, (size_t)nq * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    IM_LAUNCH(k_knn, mesh_grid(h, nq * 32, 128), 128, 0, h->stream, h->M, h->P, (const float*)dq, 3, nq, k, max_dist, di, dd);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(idx, di, (size_t)nq * k * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(d2, dd, (size_t)nq * k * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(dq); cudaFree(di); cudaFree(dd);
    return IMMESH_OK;
}

int immesh_mesh_smooth_all(immesh_mesh_t* h, double smooth_factor, int knn, double* smoothed) {
    if (!h || knn < 1 || knn > KNN_KMAX) return im_fail(IMMESH_E_INVALID, "bad argument (knn must be in [1,32])");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int cnt[32];
    IM_CUDA(cudaMemcpy(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    const int nv = cnt[0];
    if (nv == 0) return IMMESH_OK;
    int* di = nullptr;
    float* dd = nullptr;
    double* dout = nullptr;
    IM_CUDA(cudaMalloc(&di, (size_t)nv * knn * sizeof(int)));
    IM_CUDA(cudaMalloc(&dd, (size_t)nv * knn * sizeof(float)));
    if (smoothed) IM_CUDA(cudaMalloc(&dout, (size_t)nv * 3 * sizeof(double)));
    IM_LAUNCH(k_knn, mesh_grid(h, nv, 4), 128, 0, h->stream, h->M, h->P, (const float*)h->M.vpos, 4, nv, knn, (double)INFINITY, di, dd);
    IM_LAUNCH(k_smooth_all, mesh_grid(h, nv, 128), 128, 0, h->stream, h->M, nv, knn, (const int*)di, (const float*)dd, smooth_factor, h->P.accept, dout);
    IM_CUDA(cudaGetLastError());
    if (smoothed) IM_CUDA(cudaMemcpyAsync(smoothed, dout, (size_t)nv * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(di); cudaFree(dd); if (dout) cudaFree(dout);
    return IMMESH_OK;
}

int immesh_mesh_region_stream(immesh_mesh_t* h, double region_size, int32_t* region_keys, int32_t* region_offsets, int cap_regions, int32_t* triangles, int* n_regions) {
    if (!h || !(region_size > 0) || !n_regions) return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int cnt[32];
    IM_CUDA(cudaMemcpy(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    const int nalloc = std::min(cnt[1], h->M.max_t), nlive = cnt[2];
    *n_regions = 0;
    if (nlive == 0) { if (region_offsets && cap_regions >= 0) region_offsets[0] = 0; return IMMESH_OK; }
    int *d_tri = nullptr, *d_key = nullptr, *d_n = nullptr;
    IM_CUDA(cudaMalloc(&d_tri, (size_t)nlive * 3 * sizeof(int)));
    IM_CUDA(cudaMalloc(&d_key, (size_t)nlive * 3 * sizeof(int)));
    IM_CUDA(cudaMalloc(&d_n, sizeof(int)));
    IM_CUDA(cudaMemset(d_n, 0, sizeof(int)));
    IM_LAUNCH(k_region_keys, mesh_grid(h, nalloc, 128), 128, 0, h->stream, h->M, nalloc, region_size, d_tri, d_key, d_n);
    std::vector<int> t((size_t)nlive * 3), kx((size_t)nlive * 3);
    IM_CUDA(cudaMemcpyAsync(t.data(), d_tri, t.size() * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(kx.data(), d_key, kx.size() * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    cudaFree(d_tri); cudaFree(d_key); cudaFree(d_n);
    std::vector<int> order(nlive);
    for (int i = 0; i < nlive; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) {   // regions by ascending key, triangles by ascending triple inside a region
        for (int j = 0; j < 3; ++j)
            if (kx[(size_t)a * 3 + j] != kx[(size_t)b * 3 + j]) return kx[(size_t)a * 3 + j] < kx[(size_t)b * 3 + j];
        for (int j = 0; j < 3; ++j)
            if (t[(size_t)a * 3 + j] != t[(size_t)b * 3 + j]) return t[(size_t)a * 3 + j] < t[(size_t)b * 3 + j];
        return false;
    });
    int nr = 0;
    for (int i = 0; i < nlive; ++i) {
        const int o = order[i];
        const bool first = (i == 0) || kx[(size_t)o * 3] != kx[(size_t)order[i - 1] * 3] || kx[(size_t)o * 3 + 1] != kx[(size_t)order[i - 1] * 3 + 1] ||
                           kx[(size_t)o * 3 + 2] != kx[(size_t)order[i - 1] * 3 + 2];
        if (first) {
            if (nr < cap_regions) {
                if (region_keys) for (int j = 0; j < 3; ++j) region_keys[(size_t)nr * 3 + j] = kx[(size_t)o * 3 + j];
                if (region_offsets) region_offsets[nr] = i;
            }
            ++nr;
        }
        if (triangles) for (int j = 0; j < 3; ++j) triangles[(size_t)i * 3 + j] = t[(size_t)o * 3 + j];
    }
    if (region_offsets && nr <= cap_regions) region_offsets[nr] = nlive;
    *n_regions = nr;
    return nr <= cap_regions ? IMMESH_OK : im_fail(IMMESH_E_CAPACITY, "more regions than cap_regions");
}

// reconstruct_mesh_from_pointcloud (src/ImMesh_mesh_reconstruction.cpp:328-345, the offline entry of config/offline_pointcloud.yaml):
// the whole cloud is down-sampled by a pcl::VoxelGrid with leaf = minimum_pts_distance and meshed as ONE frame with the identity pose
// (Eigen::Quaterniond::Identity(), vec_3::Zero(), frame 0).  Both steps run on the device; the down-sampled cloud never leaves it.
int immesh_mesh_reconstruct_from_pointcloud(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int n, int on_device, double minimum_pts_distance, int* n_downsampled) {
    if (!h || !vg || (!xyz && n > 0) || n < 0 || !(minimum_pts_distance > 0)) return im_fail(IMMESH_E_INVALID, "bad argument");
    int m = 0, small = 0;
    int rc = immesh_voxelgrid_filter(vg, xyz, n, on_device, (float)minimum_pts_distance, nullptr, &m, &small);
    if (rc) return rc;
    if (n_downsampled) *n_downsampled = m;
    const double zero[3] = {0.0, 0.0, 0.0};
    return immesh_mesh_push_frame_dev(h, immesh_voxelgrid_device_points(vg), m, zero, 0);
}

int immesh_mesh_render_depth(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, const double* cam_R, const double* cam_t,
                             float* depth, float* points, int32_t* point_pixel, int* n_points) {
    if (!h || !intrinsics || !cam_R || !cam_t || !depth || width < 1 || height < 1 || (long long)width * height > (1 << 26) || !(z_near > 0) || !(z_far > z_near))
        return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int cnt[32];
    IM_CUDA(cudaMemcpy(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    const int nalloc = std::min(cnt[1], h->M.max_t);
    DepthCam C;
    C.fx = intrinsics[0]; C.fy = intrinsics[1]; C.cx = intrinsics[2]; C.cy = intrinsics[3]; C.z_near = z_near; C.z_far = z_far;
    for (int i = 0; i < 9; ++i) C.R[i] = cam_R[i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam_t[i];
    C.w = width; C.h = height;
    const int n = width * height;
    unsigned int* d_depth = nullptr;
    float *d_out = nullptr, *d_pts = nullptr;
    int* d_n = nullptr;
    IM_CUDA(cudaMalloc(&d_depth, (size_t)n * 4));
    IM_CUDA(cudaMalloc(&d_out, (size_t)n * 4));
    if (points) IM_CUDA(cudaMalloc(&d_pts, (size_t)n * 16));
    IM_CUDA(cudaMalloc(&d_n, 4));
    IM_CUDA(cudaMemsetAsync(d_n, 0, 4, h->stream));
    IM_LAUNCH(k_depth_clear, mesh_grid(h, n, 128), 128, 0, h->stream, d_depth, n);
    if (nalloc > 0) IM_LAUNCH(k_depth_raster, mesh_grid(h, nalloc, 128), 128, 0, h->stream, h->M, nalloc, C, d_depth);
    IM_LAUNCH(k_depth_finish, mesh_grid(h, n, 128), 128, 0, h->stream, C, (const unsigned int*)d_depth, d_out, d_pts, d_n);
    IM_CUDA(cudaGetLastError());
    int np = 0;
    IM_CUDA(cudaMemcpyAsync(depth, d_out, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(&np, d_n, 4, cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    if (points && np > 0) {
        std::vector<float> tmp((size_t)np * 4);
        IM_CUDA(cudaMemcpy(tmp.data(), d_pts, (size_t)np * 16, cudaMemcpyDeviceToHost));
        // deterministic order: ascending pixel index (the image scan order of convert_depth_buffer_to_truth_depth)
        std::vector<int> order(np);
        for (int i = 0; i < np; ++i) order[i] = i;
        std::sort(order.begin(), order.end(), [&](int a, int b) {
            int pa, pb;
            std::memcpy(&pa, &tmp[(size_t)a * 4 + 3], 4); std::memcpy(&pb, &tmp[(size_t)b * 4 + 3], 4);
            return pa < pb;
        });
        for (int i = 0; i < np; ++i) {
            const float* q = &tmp[(size_t)order[i] * 4];
            points[(size_t)i * 3] = q[0]; points[(size_t)i * 3 + 1] = q[1]; points[(size_t)i * 3 + 2] = q[2];
            if (point_pixel) std::memcpy(&point_pixel[i], &q[3], 4);
        }
    }
    if (n_points) *n_points = np;
    cudaFree(d_depth); cudaFree(d_out); if (d_pts) cudaFree(d_pts); cudaFree(d_n);
    return IMMESH_OK;
}

int immesh_mesh_last_timing(immesh_mesh_t* h, double* ms) {
    if (!h || !ms) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 4; ++i) ms[i] = h->last_ms[i];
    return IMMESH_OK;
}

}  // extern "C"
