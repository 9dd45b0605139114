// immesh_b200 -- CUDA kernels (sm_90a) and C-ABI host orchestration of the voxel-wise incremental mesher.
// Kernel bodies live in mesh_core.cuh / mesh_voxel.cuh.  No CPU path.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"
#include "pool_growth.cuh"
#include "nccl_api.hpp"
#include "reinforce.cuh"
#include "view_overlay.cuh"
#include "pdl.cuh"

using namespace immesh;
namespace {
#include "radix_sort.cuh"
}

// ------------------------------------------------------------------ kernels
__global__ void k_frame_begin(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (unsigned int i = tid; i <= F.cmask; i += nt) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    for (unsigned int i = tid; i <= F.fset_mask; i += nt) F.fset[i] = -1;
    if (tid == 0) mesh_cnt_frame_begin(M);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_init(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_init(M, P, F, c);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_conflicts(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_conflicts(M, P, F, c);
    pdl_trigger();
}
// Priority polling: candidate c waits only on candidates with a smaller index.  Blocks take tickets so that the
// block holding the smallest undecided candidate is always resident; a poll cap turns a (never observed) livelock
// into an error flag instead of a hang.
__global__ void __launch_bounds__(128) k_cand_resolve(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ int s_ticket;
    const int nblocks = (F.m + blockDim.x - 1) / blockDim.x;
    while (true) {
        if (threadIdx.x == 0) s_ticket = atomicAdd(&M.cnt[IM_MC_RESOLVE_TICKET], 1);
        __syncthreads();
        const int b = s_ticket;
        __syncthreads();
        if (b >= nblocks) break;
        const int c = b * blockDim.x + threadIdx.x;
        if (c < F.m && F.cand_status[c] == CAND_UNDECIDED) {
            int polls = 0;
            while (!cand_poll(M, P, F, c)) {
                if (++polls > (1 << 22)) { atomicOr(&M.cnt[IM_MC_ERR], IM_MERR_LIST_CAP); atomicAdd(&M.cnt[IM_MC_UNDECIDED], 1); break; }
                __nanosleep(64);
            }
            __threadfence();
        }
    }
    pdl_trigger();
}
// exclusive scan of n items by one block of 1024 threads in ONE pass: thread t owns a contiguous chunk of ceil(n/1024) items.
// count(c) is item c's value; emit(c, run) stores item c's offset run and returns its value.  Returns the offset after the thread's
// chunk (thread 1023: the total).
template <class Count, class Emit>
__device__ __forceinline__ int chunk_scan_1024(int n, Count count, Emit emit) {
    const int per = (n + 1023) / 1024;
    const int lo = threadIdx.x * per, hi = min(lo + per, n);
    int mine = 0;
    for (int c = lo; c < hi; ++c) mine += count(c);
    int run = block_scan_1024(mine);
    for (int c = lo; c < hi; ++c) run += emit(c, run);
    return run;
}
// the accept flags into the candidates' output ranks
__global__ void __launch_bounds__(1024) k_cand_scan(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    chunk_scan_1024(F.m, [&](int c) { return F.cand_status[c] == CAND_ACCEPT ? 1 : 0; },
                    [&](int c, int run) { F.cand_scan[c] = run; return F.cand_status[c] == CAND_ACCEPT ? 1 : 0; });
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_commit(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[IM_MC_VERTICES];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_commit(M, P, F, c, base);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_cand_place(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int base = M.cnt[IM_MC_VERTICES];
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < F.m; c += gridDim.x * blockDim.x) cand_place(M, F, c, base);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_voxel_select(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int na = min(M.cnt[IM_MC_ACT], F.max_act);
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < na; a += gridDim.x * blockDim.x) voxel_select(M, F, a);
    pdl_trigger();
}
// stage A: dilation (exact 20-NN of the in-voxel vertices + smoothing); one block per (voxel, group of <= 8 queries)
__global__ void __launch_bounds__(128) k_voxel_dilate(MeshDev M, MeshParams P, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    __shared__ DilateSmem S;
    __shared__ int s_item;
    const int ni = min(M.cnt[IM_MC_DITEMS], F.max_ditem);
    while (true) {
        if (threadIdx.x == 0) s_item = atomicAdd(&M.cnt[IM_MC_DILATE_TICKET], 1);
        __syncthreads();
        const int i = s_item;
        __syncthreads();
        if (i >= ni) break;
        voxel_dilate(M, P, F, F.ditem[i], &S, threadIdx.x, blockDim.x);
        __syncthreads();
    }
    pdl_trigger();
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
        if (lane == 0) i = atomicAdd(&M.cnt[IM_MC_TRI_TICKET], 1);
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
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int nf = min(M.cnt[IM_MC_FACES], F.max_list);
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < nf; f += gridDim.x * blockDim.x) commit_face(M, P, F, f);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_pull_vertices(MeshDev M, MeshParams P, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int nr = min(M.cnt[IM_MC_VREFS], F.max_vref);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < nr; r += gridDim.x * blockDim.x) pull_vertex(M, P, F, r);
}
__global__ void __launch_bounds__(128) k_pull_check(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int ne = min(M.cnt[IM_MC_PULLED], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < ne; e += gridDim.x * blockDim.x) pull_check(M, F, e);
    pdl_trigger();
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
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[IM_MC_REMOVE], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) tri_remove(M, F.rem_tri[e]);
    pdl_trigger();
}
__global__ void __launch_bounds__(128) k_push_add(MeshDev M, FrameBuf F_) {
    pdl_wait();
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x)
        tri_add(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
    pdl_trigger();
}
__global__ void k_frame_end(MeshDev M) {
    pdl_wait();
    mesh_cnt_frame_end(M);
}
// ---- the change feed (mesh_changes.cuh), queued after the push when enabled.  full: the frame lists its slots by the sweep (batched)
__global__ void __launch_bounds__(128) k_chg_gather(MeshDev M, FrameBuf F_) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = chg_gather_count(M, F);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) chg_gather(M, F, e);
}
__global__ void __launch_bounds__(128) k_chg_sweep(MeshDev M, FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    if (!chg_sweeping(F, full)) return;
    const int n = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) chg_sweep_slot(M, F, C, t);
}
__global__ void __launch_bounds__(128) k_chg_mark(MeshDev M, FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(chg_listed(F, full), F.chg_cap);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) chg_row_mark(M, F, C, i);
}
__global__ void __launch_bounds__(1024) k_chg_rows(FrameBuf F_, ChgDev C, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    const int n = min(chg_listed(F, full), F.chg_cap);
    const int total = chunk_scan_1024(n, [&](int i) { return chg_row_count(C, i); }, [&](int i, int run) { return chg_row_emit(C, i, run); });
    if (threadIdx.x == 1023) F.chg_cnt[IM_CH_ROWS] = total;
}
__global__ void __launch_bounds__(128) k_chg_word(const int* cnt, ChgDev C, int w, const unsigned int* vin, unsigned int* kout, unsigned int* vout) {
    const int n = cnt[IM_CH_ROWS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vin ? vin[i] : (unsigned int)i;
        kout[i] = chg_word(C, w, (int)v);
        vout[i] = v;
    }
}
__global__ void __launch_bounds__(128) k_chg_emit(FrameBuf F_, ChgDev C, const unsigned int* order, int full) {
    const FrameBuf F = frame_load_dyn(F_);
    if (chg_lost(F, C, full)) return;
    const int n = F.chg_cnt[IM_CH_ROWS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) chg_append(C, order, i);
}
__global__ void k_chg_end(MeshDev M, FrameBuf F_, ChgDev C, int full, int v_after) { chg_frame_end(M, frame_load_dyn(F_), C, full, v_after); }
// enable: the published bytes of the allocated slots from the store as it is
__global__ void __launch_bounds__(128) k_chg_init(MeshDev M, unsigned char* pub, int n_alloc) {
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) pub[t] = chg_state(M, t);
}
// ---- the live triangles in order (mesh_tri_order).  k_tri_gather compacts the live records of the slots [0, n_alloc) into rec[0, cap),
// w = the slot, and counts every kept one in misc[0].  With a region size it keys them (tri_region_key): all regions (qkeys null) keep
// the key in reg[3 e ..]; requested regions keep only the triangles of a region in the table, with the caller's index in reg[e].  The
// minimum and maximum of each region word go to misc[2..7], reduced once per warp.  A key outside ikey_ok sets misc[1].
__global__ void __launch_bounds__(128) k_tri_gather(MeshDev M, int n_alloc, int cap, double region_size, const unsigned long long* qkeys, const int* qval,
                                                    unsigned int qmask, int4* rec, int* reg, int* misc) {
    const int nreg = region_size > 0 ? (qkeys ? 1 : 3) : 0;
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_alloc; t += gridDim.x * blockDim.x) {
        int4 r = M.tri[t];
        if (!r.w) continue;
        int k[3] = {0, 0, 0};
        if (region_size > 0) {
            tri_region_key(M, r, region_size, k);
            if (!ikey_ok(k[0], k[1], k[2])) atomicOr(&misc[1], 1);
            if (qkeys) {
                const int s = table_find(qkeys, qmask, pack_ikey(k[0], k[1], k[2]));
                if (s < 0) continue;
                k[0] = qval[s];
            }
            for (int c = 0; c < 3; ++c) { lo[c] = min(lo[c], k[c]); hi[c] = max(hi[c], k[c]); }
        }
        const int e = atomicAdd(&misc[0], 1);
        if (e >= cap) continue;
        r.w = t;
        rec[e] = r;
        for (int c = 0; c < nreg; ++c) reg[(size_t)e * nreg + c] = k[c];
    }
    for (int c = 0; c < nreg; ++c) {
        const int a = __reduce_min_sync(0xffffffffu, lo[c]), b = __reduce_max_sync(0xffffffffu, hi[c]);
        if ((threadIdx.x & 31) == 0 && a <= b) { atomicMin(&misc[2 + c], a); atomicMax(&misc[5 + c], b); }
    }
}
// sort word w of the records in the order vin (null: as gathered): 0..2 = c, b, a of the triple; 3 + j = region word j less its minimum
__global__ void __launch_bounds__(128) k_tri_word(const int4* rec, const int* reg, int nreg, int n, int w, unsigned int base, const unsigned int* vin,
                                                  unsigned int* kout, unsigned int* vout) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vin ? vin[i] : (unsigned int)i;
        unsigned int x;
        if (w < 3) { const int4 r = rec[v]; x = (unsigned int)(w == 0 ? r.z : w == 1 ? r.y : r.x); }
        else x = (unsigned int)reg[(size_t)v * nreg + (w - 3)] - base;
        kout[i] = x;
        vout[i] = v;
    }
}
// snapshot and region stream: the records in order, their triples and (flip not null) the orientation flags of their slots
__global__ void __launch_bounds__(128) k_tri_emit(MeshDev M, const int4* rec, const unsigned int* order, int n, int* tri, int* flip) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 r = rec[order[i]];
        tri[(size_t)i * 3 + 0] = r.x; tri[(size_t)i * 3 + 1] = r.y; tri[(size_t)i * 3 + 2] = r.z;
        if (flip) flip[i] = (int)(M.tri_flip[r.w] & 1ull);
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
        if (M.cnt[IM_MC_VOXELS] > 0) {
            far = max(far, max(abs(cx - M.cnt[IM_MC_BBOX_MIN_X]), abs(cx - M.cnt[IM_MC_BBOX_MAX_X])));
            far = max(far, max(abs(cy - M.cnt[IM_MC_BBOX_MIN_Y]), abs(cy - M.cnt[IM_MC_BBOX_MAX_Y])));
            far = max(far, max(abs(cz - M.cnt[IM_MC_BBOX_MIN_Z]), abs(cz - M.cnt[IM_MC_BBOX_MAX_Z])));
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
                    const float4 p = M.vchunk_pts[(size_t)im_chunk_or0(M.vox_chunk[(size_t)s * IM_VCHUNKS + (kk >> 4)]) * 16 + (kk & 15)];
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
        double r[3];
        smooth_vertex(M, v, k, idx + (size_t)v * k, d2 + (size_t)v * k, sf, max_dis, r);
        store_smooth(M, v, r[0], r[1], r[2]);
        if (out) { out[(size_t)v * 3 + 0] = r[0]; out[(size_t)v * 3 + 1] = r[1]; out[(size_t)v * 3 + 2] = r[2]; }
    }
}

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

// ---- depth-camera frames (immesh_mesh_push_depth): the kernels of depth_kernels.cuh without a filter; block 0 of k_depth_emit sets the
// frame's n, step, m and cmask in its FrameDyn, and the kernels after it read the device count.  Grids cover max_frame_points samples.
namespace {
#include "depth_kernels.cuh"
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

// ---- the region segments of records in region order (mesh_tri_order with a region size): the region stream and the viewer's region
// buffers (immesh_mesh_region_buffers, mesh_rec_display.cpp:78-137 + :220-258).  For the buffers, the vertices of the kept triangles
// whose m_smoothed is clear are claimed once (bitmap), compacted, searched with k_knn and smoothed from raw positions; k_rb_emit
// gathers vsmooth into the float rows and reduces the axis box per block.
#define RB_THREADS 128
__device__ __forceinline__ bool rb_same_region(const int* reg, unsigned int a, unsigned int b) {   // all regions: three key words per record
    return reg[(size_t)a * 3] == reg[(size_t)b * 3] && reg[(size_t)a * 3 + 1] == reg[(size_t)b * 3 + 1] && reg[(size_t)a * 3 + 2] == reg[(size_t)b * 3 + 2];
}
__global__ void __launch_bounds__(RB_THREADS) k_rb_starts(int n, const unsigned int* order, const int* reg, int* flag) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) flag[i] = (i == 0 || !rb_same_region(reg, order[i], order[i - 1])) ? 1 : 0;
}
// all regions: the first row of every region writes its key and offset (scan: exclusive region number of each row)
__global__ void __launch_bounds__(RB_THREADS) k_rb_regions(int n, const unsigned int* order, const int* reg, const int* scan, int* keys, int* off) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (i > 0 && rb_same_region(reg, order[i], order[i - 1])) continue;
        const int r = scan[i];
        for (int c = 0; c < 3; ++c) keys[(size_t)r * 3 + c] = reg[(size_t)order[i] * 3 + c];
        off[r] = i;
    }
}
// requested regions (n >= 1 rows): offsets of nk segments, empty ones included
__global__ void __launch_bounds__(RB_THREADS) k_rb_offsets(int n, int nk, const unsigned int* order, const int* reg, int* off) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int cur = reg[order[i]], prev = i > 0 ? reg[order[i - 1]] : -1;
        for (int r = prev + 1; r <= cur; ++r) off[r] = i;
        if (i == n - 1) for (int r = cur + 1; r <= nk; ++r) off[r] = n;
    }
}
// vertices of the kept triangles with m_smoothed clear, each claimed once, compacted with its position as a k_knn query
__global__ void __launch_bounds__(RB_THREADS) k_rb_claim(MeshDev M, int n, const int4* rec, unsigned int* bits, int* claimed, int* list, float4* q) {
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < 3 * n; e += gridDim.x * blockDim.x) {
        const int4 r = rec[e / 3];
        const int v = e % 3 == 0 ? r.x : e % 3 == 1 ? r.y : r.z;
        if (M.vsmoothed[v]) continue;
        const unsigned int bit = 1u << (v & 31);
        if (atomicOr(&bits[v >> 5], bit) & bit) continue;
        const int k = atomicAdd(claimed, 1);
        list[k] = v;
        q[k] = M.vpos[v];
    }
}
__global__ void __launch_bounds__(RB_THREADS) k_rb_smooth(MeshDev M, int nq, int k, const int* list, const int* __restrict__ idx, const float* __restrict__ d2, double sf, double max_dis) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
        double r[3];
        smooth_vertex(M, list[i], k, idx + (size_t)i * k, d2 + (size_t)i * k, sf, max_dis, r);
        store_smooth(M, list[i], r[0], r[1], r[2]);
    }
}
__global__ void __launch_bounds__(RB_THREADS) k_rb_emit(MeshDev M, int n, const unsigned int* order, const int4* rec, float* xyz, int* ids, AxisAcc* part) {
    __shared__ AxisAcc s[RB_THREADS];
    AxisAcc a;
    axis_init(a);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 r = rec[order[i]];
        float row[9];
        region_row(M, r, row);
        for (int c = 0; c < 9; ++c) xyz[(size_t)i * 9 + c] = row[c];
        ids[(size_t)i * 3 + 0] = r.x; ids[(size_t)i * 3 + 1] = r.y; ids[(size_t)i * 3 + 2] = r.z;
        for (int j = 0; j < 3; ++j)
            for (int d = 0; d < 3; ++d) { axis_take(a, d, row[j * 3 + d], i * 3 + j); axis_take(a, d + 3, row[j * 3 + d], i * 3 + j); }
    }
    s[threadIdx.x] = a;
    __syncthreads();
    for (int h = RB_THREADS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) axis_merge(s[threadIdx.x], s[threadIdx.x + h]);
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = s[0];
}
__global__ void k_rb_axis(const AxisAcc* part, int nb, float* box) {
    AxisAcc a;
    axis_init(a);
    for (int b = 0; b < nb; ++b) axis_merge(a, part[b]);
    axis_apply(a, box);
}

// ---- the batched frame (immesh_mesh_push_frame_batched): one frame, append in chunks, per-voxel stage in batches.  The frame-level
// counters of the per-frame path are accumulated across chunks / batches in the IM_MC_BAT_* slots and written back by k_bat_frame_end.
__global__ void k_bat_chunk_begin(MeshDev M, FrameBuf F) {   // the candidate grid of one append chunk after the first
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    for (unsigned int i = tid; i <= F.cmask; i += nt) { F.ckeys[i] = IM_EMPTY_KEY; F.chead[i] = -1; }
    if (tid == 0) mesh_cnt_bat_chunk_begin(M);
}
__global__ void k_bat_chunk_end(MeshDev M) { mesh_cnt_bat_chunk_end(M); }
// activation rule over every activated voxel of the frame (after the last chunk); the meshed ones with their keys
__global__ void __launch_bounds__(128) k_bat_select(MeshDev M, FrameBuf F, int* sel, unsigned long long* key) {
    const int na = min(M.cnt[IM_MC_ACT], F.max_act);
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < na; a += gridDim.x * blockDim.x) {
        const int vs = F.act[a];
        if (!voxel_activate(M, F, vs)) continue;
        const int k = atomicAdd(&M.cnt[IM_MC_BAT_SELECTED], 1);
        sel[k] = vs;
        key[k] = M.vkeys[vs];
    }
}
// sort word of position i: half 0 / 1 = low / high 32 bits of the key (LSD order)
__global__ void __launch_bounds__(128) k_bat_word(int n, int half, const unsigned long long* key, const unsigned int* vin, unsigned int* kout, unsigned int* vout) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned int v = vin ? vin[i] : (unsigned int)i;
        kout[i] = (unsigned int)(key[v] >> (32 * half));
        vout[i] = v;
    }
}
__global__ void k_bat_reset(MeshDev M, FrameBuf F, int clear_fset) {   // the per-batch lists
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nt = gridDim.x * blockDim.x;
    if (clear_fset) for (unsigned int i = tid; i <= F.fset_mask; i += nt) F.fset[i] = -1;
    if (tid == 0) mesh_cnt_bat_reset(M);
}
// meshed voxels [lo, hi) in key order -> the batch's work list; the rank is the flip priority
__global__ void __launch_bounds__(128) k_bat_fill(MeshDev M, FrameBuf F, const int* sel, const unsigned int* order, int lo, int hi, int* rank) {
    for (int r = lo + blockIdx.x * blockDim.x + threadIdx.x; r < hi; r += gridDim.x * blockDim.x) {
        const int w = voxel_enqueue(M, F, sel[order[r]]);
        if (w >= 0) rank[w] = r;
    }
}
// the batch's additions, pushed at once; marked so that later batches' pulls and commits do not see them as pre-frame triangles
__global__ void __launch_bounds__(128) k_bat_push_add(MeshDev M, FrameBuf F) {
    const int n = min(M.cnt[IM_MC_ADD], F.max_list);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
        const int t = tri_add(M, F.add_tri[(size_t)e * 3 + 0], F.add_tri[(size_t)e * 3 + 1], F.add_tri[(size_t)e * 3 + 2], F.add_flip[e]);
        if (t >= 0) F.tri_mark[t] = IM_TRI_BORN;
    }
}
__global__ void k_bat_batch_end(MeshDev M) { mesh_cnt_bat_batch_end(M); }
// after the last batch: the deferred removals; every mark cleared for the next frame
__global__ void __launch_bounds__(128) k_bat_sweep(MeshDev M, FrameBuf F) {
    const int n = min(M.cnt[IM_MC_TRIS_ALLOC], M.max_t);
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x) {
        const unsigned char m = F.tri_mark[t];
        if (!m) continue;
        if (m == IM_TRI_REMOVE) tri_remove(M, t);
        F.tri_mark[t] = 0;
    }
}
__global__ void k_bat_frame_end(MeshDev M) { mesh_cnt_bat_frame_end(M); }

// ---- growth of the mesh pools (immesh_mesh_reserve): the three open-addressed tables rebuilt into tables of the new size
#define MGROW_THREADS 256
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_xi(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.gmask; s += gridDim.x * blockDim.x) rehash_xi_slot(from, to, s);
}
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_voxels(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.vmask; s += gridDim.x * blockDim.x) rehash_voxel_slot(from, to, s);
}
__global__ void __launch_bounds__(MGROW_THREADS) k_rehash_tris(MeshDev from, MeshDev to) {
    for (unsigned int s = blockIdx.x * blockDim.x + threadIdx.x; s <= from.tmask; s += gridDim.x * blockDim.x) rehash_tri_slot(from, to, s);
}

// ------------------------------------------------------------------ host side

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

int immesh_mesh_create(const immesh_mesh_config* cfg, immesh_mesh_t** out) {
    if (!cfg || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    if (!(cfg->points_minimum_scale > 0) || !(cfg->voxel_resolution > 0) || cfg->number_of_pts_append_to_map < 1) return im_fail(IMMESH_E_INVALID, "bad mesh configuration");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return im_fail(IMMESH_E_NO_DEVICE, "no CUDA device: immesh_b200 has no CPU path");
    immesh::Building<immesh_mesh> owner(new immesh_mesh(), immesh_mesh_destroy);   // every failure below releases what was created
    immesh_mesh* h = owner.get();
    h->F.shard_rank = 0; h->F.shard_n = 1; h->F.x_cap = 0;
    h->F.work_rank = nullptr; h->F.tri_mark = nullptr;   // the per-frame path
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
    h->max_vox = max_vox;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, dev);
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto& e : h->ev) IM_CUDA(cudaEventCreate(&e));
    MeshDev& M = h->M;
    M.max_v = max_v;
    M.max_t = max_t;
    IM_CUDA(h->dev.alloc(&M.vpos, (size_t)max_v));
    IM_CUDA(h->dev.alloc(&M.vsmooth, (size_t)max_v * 3));
    IM_CUDA(h->dev.alloc(&M.vsmoothed, (size_t)max_v, 0));
    IM_CUDA(h->dev.alloc(&M.v_tri_head, (size_t)max_v, 0xFF));
    const size_t gcap = pow2_at_least((size_t)max_v * 2);
    IM_CUDA(h->dev.alloc(&M.gkeys, gcap, 0xFF));
    IM_CUDA(h->dev.alloc(&M.gval, gcap, 0xFF));
    M.gmask = (unsigned)(gcap - 1);
    const size_t vcap = pow2_at_least((size_t)max_vox * 2);
    IM_CUDA(h->dev.alloc(&M.vkeys, vcap, 0xFF));
    M.vmask = (unsigned)(vcap - 1);
    IM_CUDA(h->dev.alloc(&M.vox_chunk, vcap * IM_VCHUNKS, 0xFF));
    M.max_vchunks = max_v / 4 + 1024;
    IM_CUDA(h->dev.alloc(&M.vchunk_pts, (size_t)M.max_vchunks * 16));
    IM_CUDA(h->dev.alloc(&M.vox_count, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_meshing_times, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_new_added, vcap, 0));
    IM_CUDA(h->dev.alloc(&M.vox_frame, vcap, 0xFF));
    M.vox_short_axis = nullptr;
    IM_CUDA(h->dev.alloc(&M.tri, (size_t)max_t));
    IM_CUDA(h->dev.alloc(&M.tri_next, (size_t)max_t * 3));
    IM_CUDA(h->dev.alloc(&M.tri_flip, (size_t)max_t));
    const size_t tcap = pow2_at_least((size_t)max_t * 2);
    IM_CUDA(h->dev.alloc(&M.thash, tcap, 0xFF));
    M.tmask = (unsigned)(tcap - 1);
    IM_CUDA(h->dev.alloc(&M.cnt, IM_MC_ALLOC, 0));
    {
        int init[IM_MC_HOST] = {};
        mesh_cnt_init(init);
        IM_CUDA(cudaMemcpy(M.cnt, init, sizeof(init), cudaMemcpyHostToDevice));
    }
    FrameBuf& F = h->F;
    const size_t mc = (size_t)h->max_frame_points;  // candidates <= points
    F.max_cand = (int)mc;
    F.max_work = max_vox < (1 << 16) ? max_vox : std::min(std::max(max_vox / 16, 1 << 16), 1 << 18);   // voxels (re)meshed per frame; 4 KB of id list each
    F.max_act = (int)std::min<size_t>((size_t)max_vox, mc);
    F.max_list = 4 << 20;
    IM_CUDA(h->dev.alloc(&h->d_pts, IM_SLOTS * mc * 3));
    IM_CUDA(h->dev.alloc(&h->d_body, IM_SLOTS * mc * 3));   // staging of body-frame scans handed over by the localization handle (not allocated lazily: an allocation inside a frame stalls the pipeline)
    F.pts = h->d_pts;
    IM_CUDA(h->dev.alloc(&h->d_fp, IM_SLOTS));
    for (int i = 0; i < IM_SLOTS; ++i) { IM_CUDA(cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming)); IM_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming)); }
    IM_CUDA(h->dev.alloc(&F.cand_gkey, mc));
    IM_CUDA(h->dev.alloc(&F.cand_vslot, mc));
    IM_CUDA(h->dev.alloc(&F.cand_status, mc));
    IM_CUDA(h->dev.alloc(&F.cand_scan, mc));
    IM_CUDA(h->dev.alloc(&F.cand_conf, mc * IM_CONF_K));
    IM_CUDA(h->dev.alloc(&F.cand_nconf, mc));
    IM_CUDA(h->dev.alloc(&F.cand_next, mc));
    IM_CUDA(h->dev.alloc(&F.cand_pos, mc));
    h->ccap = pow2_at_least(mc * 2);
    IM_CUDA(h->dev.alloc(&F.ckeys, h->ccap));
    IM_CUDA(h->dev.alloc(&F.chead, h->ccap));
    F.scan_block = nullptr;
    IM_CUDA(h->dev.alloc(&F.act, (size_t)F.max_act));
    IM_CUDA(h->dev.alloc(&F.work, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_n_ids, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_ids, (size_t)F.max_work * IM_MAXD));
    IM_CUDA(h->dev.alloc(&F.work_nfaces, (size_t)F.max_work));
    IM_CUDA(h->dev.alloc(&F.work_bits, (size_t)F.max_work * (IM_MAXG / 32), 0));
    IM_CUDA(h->dev.alloc(&F.work_ring, (size_t)F.max_work, 0));
    IM_CUDA(h->dev.alloc(&F.work_done, (size_t)F.max_work, 0));
    F.max_ditem = F.max_work * 4;
    IM_CUDA(h->dev.alloc(&F.ditem, (size_t)F.max_ditem));
    F.max_vref = 8 << 20;
    IM_CUDA(h->dev.alloc(&F.all_faces, (size_t)F.max_list));
    IM_CUDA(h->dev.alloc(&F.all_vref, (size_t)F.max_vref));
    IM_CUDA(h->dev.alloc(&F.pulled, (size_t)F.max_list * 2));
    F.fset_mask = (1u << 21) - 1;
    IM_CUDA(h->dev.alloc(&F.fset, (size_t)F.fset_mask + 1, 0xFF));
    IM_CUDA(h->dev.alloc(&F.work_axes, (size_t)F.max_work * 9));
    IM_CUDA(h->dev.alloc(&F.add_tri, (size_t)F.max_list * 3));
    IM_CUDA(h->dev.alloc(&F.add_flip, (size_t)F.max_list));
    IM_CUDA(h->dev.alloc(&F.rem_tri, (size_t)F.max_list));
    IM_CUDA(h->pinned.alloc(&h->h_pts, IM_SLOTS * mc * 3));
    IM_CUDA(h->pinned.alloc(&h->h_cnt, IM_SLOTS * IM_MC_HOST));
    IM_CUDA(h->pinned.alloc(&h->h_fp, IM_SLOTS));
    IM_CUDA(h->pinned.alloc(&h->h_dyn, IM_SLOTS));
    IM_CUDA(h->dev.alloc(&h->d_dyn, 1, 0));
    IM_CUDA(h->dev.alloc(&h->cam_ring, IM_RF_RING, 0));
    IM_CUDA(h->dev.alloc(&h->cam_ring_frame, IM_RF_RING, 0));
    F.dyn = h->d_dyn;
    F.epoch = 0;
    IM_CUDA(cudaFuncSetAttribute(k_voxel_mesh<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<1024>)));
    IM_CUDA(cudaFuncSetAttribute(k_voxel_tri_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(4 * sizeof(MeshWarpSmem<128>))));
    IM_CUDA(cudaFuncSetAttribute(k_voxel_mesh<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MeshSmem<256>)));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream3, cudaStreamNonBlocking));
    IM_CUDA(cudaStreamCreateWithFlags(&h->stream_up, cudaStreamNonBlocking));
    for (int i = 0; i < IM_SLOTS; ++i) IM_CUDA(cudaEventCreateWithFlags(&h->ev_up[i], cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));
    IM_CUDA(cudaEventCreateWithFlags(&h->ev_join3, cudaEventDisableTiming));
    std::memset(h->last_cnt, 0, sizeof(h->last_cnt));
    IM_CUDA(cudaDeviceSynchronize());
    *out = owner.release();
    return IMMESH_OK;
}

static void mesh_feed_free(immesh_mesh* h);
int immesh_mesh_destroy(immesh_mesh_t* h) {
    if (!h) return IMMESH_OK;
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->graph.destroy();
    mesh_feed_free(h);   // after the drain: no queued kernel still writes the done word
    if (h->win.local) immesh::peer_window_close(h->win);
    if (h->nccl_comm && immesh::nccl().CommDestroy) immesh::nccl().CommDestroy(h->nccl_comm);
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
// resident blocks per SM of the persistent per-voxel kernels (headroom for the kernels on the other streams)
#define MESH_TRI_BPS 3      // k_voxel_tri_warp, k_voxel_mesh<256>
#define MESH_DILATE_BPS 3   // k_voxel_dilate

// transformLidar of the full-resolution scan with the converged state (ImMesh_mesh_reconstruction.cpp:413 ->
// voxel_mapping_common.cpp:709-726): p_w = (float)( R (R_ext p + t_ext) + t ).  First kernel of a frame handed over by the
// localization handle: the pose is the one that scan converged to (LioCtrl::pose_ring, written by the last kernel of the
// scan's sequence; the localization stream may already be working on later scans).  Block 0 also derives the frame's sensor
// position + the origin of the flip-priority rank, and records the pose in the handle's camera ring (reinforce.cuh, rf_avr_pose).
// A count read on the device (FrameDyn::n_dev, immesh_mesh_push_frame_from_lio_async_dev_n): every block reads it there, and block 0 sets
// the frame's n, step, m and cmask from it (frame_append_dims) for the kernels after this one.
__global__ void __launch_bounds__(128) k_transform_full(LioParams P, const LioCtrl* ctrl, FrameBuf F_, double res, double (*cam_ring)[12], int* cam_ring_frame,
                                                        int append_target) {
    __shared__ double s[12];
    const FrameDyn d = *F_.dyn;
    const int n = d.n_dev ? *d.n_dev : d.n;
    if (d.n_dev && blockIdx.x == 0 && threadIdx.x == 0) {
        FrameDyn* w = const_cast<FrameDyn*>(F_.dyn);
        w->n = n;
        frame_append_dims(n, append_target, &w->step, &w->m, &w->cmask);
    }
    if (threadIdx.x < 12) s[threadIdx.x] = ctrl->pose_ring[d.pose_idx][threadIdx.x];
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < 3) {
        const double t = s[9 + threadIdx.x];
        d.fp->pose_t[threadIdx.x] = t;
        d.fp->prio_origin[threadIdx.x] = (long long)floor(t / res) - 1024;
    }
    if (blockIdx.x == 0 && threadIdx.x < 12) {
        cam_ring[d.frame % IM_RF_RING][threadIdx.x] = s[threadIdx.x];
        if (threadIdx.x == 0) cam_ring_frame[d.frame % IM_RF_RING] = d.frame;
    }
    const float* body = d.body;
    float* world = const_cast<float*>(d.pts);
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
        hdr->n_smooth = min(M.cnt[IM_MC_X_SMOOTHS], F.x_cap);
        hdr->n_face = min(M.cnt[IM_MC_X_FACES], F.x_cap);
        hdr->n_rem = min(M.cnt[IM_MC_X_REMS], F.x_cap);
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
    const int n_smooth = min(M.cnt[IM_MC_X_SMOOTHS], F.x_cap), n_face = min(M.cnt[IM_MC_X_FACES], F.x_cap), n_rem = min(M.cnt[IM_MC_X_REMS], F.x_cap);
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
    mesh_wait_peers(pe, 0, epoch, &M.cnt[IM_MC_ERR]);
    for (int r = 0; r < F.shard_n; ++r) {
        if (r == F.shard_rank) continue;
        const unsigned char* seg = recv + (size_t)r * seg_bytes;
        const int n = __ldcg((const int*)seg);
        const double2* e = (const double2*)(seg + 16);
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
            const double2 a = __ldcg(e + 2 * (size_t)i), b = __ldcg(e + 2 * (size_t)i + 1);   // {id|pad, x}, {y, z}
            const int id = (int)(__double_as_longlong(a.x) & 0xffffffffLL);
            store_smooth(M, id, a.y, b.x, b.y);
        }
    }
}
// facets / removals of ALL ranks (own segment included) -> add / remove lists of this rank's replica
__global__ void __launch_bounds__(256) k_apply_lists(MeshDev M, FrameBuf F_, const unsigned char* recv, size_t seg_bytes, MeshPeers pe) {
    const FrameBuf F = frame_load_dyn(F_);
    const unsigned long long epoch = F.epoch;
    mesh_wait_peers(pe, 1, epoch, &M.cnt[IM_MC_ERR]);
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
    if (err & IM_MERR_FEED_INDEX) return im_fail(IMMESH_E_CUDA, "frame feed: internal error (a record slot outside its ring; nothing was written)");
    return IMMESH_OK;
}
static void mesh_note(immesh_mesh* h, const int* c, int frame);
// the host's copy of the counters (the first IM_MC_HOST slots), blocking: the caller has drained what it needs
static cudaError_t mesh_read_counters(const immesh_mesh* h, int (&c)[IM_MC_HOST]) {
    return cudaMemcpy(c, h->M.cnt, sizeof(c), cudaMemcpyDeviceToHost);
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
    std::memcpy(h->last_cnt, h->h_cnt + IM_MC_HOST * s, sizeof(h->last_cnt));
    if (h->grow_max_bytes > 0) mesh_note(h, h->last_cnt, h->h_dyn[s].frame);
    const int rc = mesh_status(h->last_cnt[IM_MC_ERR]);
    if (rc && !h->pending_rc) h->pending_rc = rc;
    return rc;
}

// ---- growth of the mesh pools.  Device bytes per record: vertex 109 (vpos 16, vsmooth 24, m_smoothed 1, incidence head 4, its
// share of the vertex chunks 64 at max_v / 4 chunks of 16 float4), plus the xi-grid at 12 B per slot over 2 max_v rounded up to a
// power of two; triangle 36 (record 16, incidence links 12, flip word 8) plus the triple hash at 4 B per slot over 2 max_t; mesh
// voxel 88 B per slot (key 8, 16 chunk ids 64, count / meshing_times / new_added / frame 16) over 2 max_voxels.  Ids are 32-bit:
// every pool stops at 2^30 records.
#define IM_MPOOL_LIMIT (1LL << 30)
static size_t mesh_pool_bytes(const immesh_mesh* h, long long v, long long t, long long x) {
    const size_t gcap = pow2_at_least((size_t)v * 2), tcap = pow2_at_least((size_t)t * 2), vcap = pow2_at_least((size_t)x * 2);
    const size_t act = std::min<size_t>((size_t)x, (size_t)h->max_frame_points);
    return (size_t)v * 45 + gcap * 12 + ((size_t)v / 4 + 1024) * 16 * sizeof(float4) + (size_t)t * 36 + tcap * 4 + vcap * (8 + IM_VCHUNKS * 4 + 16) + act * 4;
}
// counters of frame number `frame`, finished (see note_counters of the localization handle)
static void mesh_note(immesh_mesh* h, const int* c, int frame) {
    if (frame <= h->known_frame) return;
    h->max_step_tris = std::max(h->max_step_tris, c[IM_MC_TRIS_ALLOC] - h->known[IM_MC_TRIS_ALLOC]);   // over several frames: an upper bound of one
    std::memcpy(h->known, c, sizeof(h->known));
    h->known_frame = frame;
}
// Enlarge the pools to (vertices, triangles, voxels), each >= the current one: as lio_grow (lio_capi.cu) -- drain, allocate all,
// migrate on the stream, free the old buffers, drop the captured launch sequence.  The batched frame's scratch (sized by max_voxels
// and max_triangles) is freed, and allocated again at the new sizes by the next batched frame.
static int mesh_grow(immesh_mesh* h, long long verts, long long tris, long long vox) {
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "a sharded mesh handle cannot grow (its replicas would have to grow in lockstep)");
    if (verts > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "vertex pool: more than 2^30 vertices (32-bit vertex ids)");
    if (tris > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "triangle pool: more than 2^30 triangles (32-bit triangle ids)");
    if (vox > IM_MPOOL_LIMIT) return im_fail(IMMESH_E_CAPACITY, "voxel hash: more than 2^30 mesh voxels (32-bit voxel ids)");
    MeshDev& M = h->M;
    const long long v0 = M.max_v, t0 = M.max_t, x0 = h->max_vox;
    const bool gv = verts > v0, gt = tris > t0, gx = vox > x0;
    if (!gv && !gt && !gx) return IMMESH_OK;
    verts = std::max(verts, v0); tris = std::max(tris, t0); vox = std::max(vox, x0);
    // the batched frame's scratch (h->batch) goes, so it is not part of the sum
    const size_t bytes = h->dev.bytes() - mesh_pool_bytes(h, v0, t0, x0) + mesh_pool_bytes(h, verts, tris, vox);
    if (h->grow_max_bytes > 0 && bytes > (size_t)h->grow_max_bytes) {
        const std::string pools = std::string(gv ? " vertex pool" : "") + (gt ? " triangle pool" : "") + (gx ? " voxel hash" : "");
        return im_fail(IMMESH_E_CAPACITY, ("growth of the" + pools + " to " + std::to_string(bytes) + " device bytes is above the ceiling of " +
                                           std::to_string(h->grow_max_bytes) + " (immesh_mesh_set_growth)").c_str());
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, c));
    const int nv = std::min(c[IM_MC_VERTICES], M.max_v), nt = std::min(c[IM_MC_TRIS_ALLOC], M.max_t), nch = std::min(c[IM_MC_VERT_CHUNKS], M.max_vchunks);
    MeshDev nm = M;
    FrameBuf nf = h->F;
    immesh::MemSet fresh;   // the new buffers, freed on every failure below
    const char* pool = "";
    const size_t gcap = pow2_at_least((size_t)verts * 2), tcap = pow2_at_least((size_t)tris * 2), vcap = pow2_at_least((size_t)vox * 2);
    const int vch = (int)(verts / 4 + 1024), act = (int)std::min<long long>(vox, h->max_frame_points);
    cudaError_t e = cudaSuccess;
    if (gv) {
        pool = "vertex pool";
        if ((e = fresh.alloc(&nm.vpos, verts)) == cudaSuccess && (e = fresh.alloc(&nm.vsmooth, verts * 3)) == cudaSuccess && (e = fresh.alloc(&nm.vsmoothed, verts)) == cudaSuccess &&
            (e = fresh.alloc(&nm.v_tri_head, verts)) == cudaSuccess && (e = fresh.alloc(&nm.vchunk_pts, (size_t)vch * 16)) == cudaSuccess && gcap > (size_t)M.gmask + 1 &&
            (e = fresh.alloc(&nm.gkeys, gcap)) == cudaSuccess)
            e = fresh.alloc(&nm.gval, gcap);
    }
    if (gt && e == cudaSuccess) {
        pool = "triangle pool";
        if ((e = fresh.alloc(&nm.tri, tris)) == cudaSuccess && (e = fresh.alloc(&nm.tri_next, tris * 3)) == cudaSuccess && (e = fresh.alloc(&nm.tri_flip, tris)) == cudaSuccess &&
            tcap > (size_t)M.tmask + 1)
            e = fresh.alloc(&nm.thash, tcap);
    }
    if (gx && e == cudaSuccess) {
        pool = "voxel hash";
        if (vcap > (size_t)M.vmask + 1 && (e = fresh.alloc(&nm.vkeys, vcap)) == cudaSuccess && (e = fresh.alloc(&nm.vox_chunk, vcap * IM_VCHUNKS)) == cudaSuccess &&
            (e = fresh.alloc(&nm.vox_count, vcap)) == cudaSuccess && (e = fresh.alloc(&nm.vox_meshing_times, vcap)) == cudaSuccess &&
            (e = fresh.alloc(&nm.vox_new_added, vcap)) == cudaSuccess)
            e = fresh.alloc(&nm.vox_frame, vcap);
        if (e == cudaSuccess && act > h->F.max_act) e = fresh.alloc(&nf.act, act);
    }
    // the change feed's per-triangle stamp and published byte follow the triangle pool
    immesh::MemSet cfresh;
    int* c_stamp = h->F.chg_stamp;
    unsigned char* c_pub = h->chg.C.pub;
    if (gt && h->chg.on && e == cudaSuccess) {
        pool = "triangle pool (change feed)";
        if ((e = cfresh.alloc(&c_stamp, tris)) == cudaSuccess) e = cfresh.alloc(&c_pub, tris);
    }
    auto fail = [&](cudaError_t err, const char* what) {
        cudaGetLastError();
        return im_fail(err == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA,
                       (std::string(what) + ": " + cudaGetErrorString(err) + " during the growth; the handle is unchanged").c_str());
    };
    if (e != cudaSuccess) return fail(e, pool);
    cudaStream_t st = h->stream;
    const int g = h->n_sm * 16;
    auto migrate = [&]() -> cudaError_t {
        cudaError_t r = cudaSuccess;
#define MG(x) do { if ((r = (x)) != cudaSuccess) return r; } while (0)
        if (gv) {
            MG(cudaMemsetAsync(nm.vsmoothed, 0, (size_t)verts, st));
            MG(cudaMemsetAsync(nm.v_tri_head, 0xFF, (size_t)verts * 4, st));
            if (nv > 0) {
                MG(cudaMemcpyAsync(nm.vpos, M.vpos, (size_t)nv * sizeof(float4), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.vsmooth, M.vsmooth, (size_t)nv * 3 * sizeof(double), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.vsmoothed, M.vsmoothed, (size_t)nv, cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.v_tri_head, M.v_tri_head, (size_t)nv * 4, cudaMemcpyDeviceToDevice, st));
            }
            if (nch > 0) MG(cudaMemcpyAsync(nm.vchunk_pts, M.vchunk_pts, (size_t)nch * 16 * sizeof(float4), cudaMemcpyDeviceToDevice, st));
            nm.max_v = (int)verts;
            nm.max_vchunks = vch;
            if (nm.gkeys != M.gkeys) {
                MG(cudaMemsetAsync(nm.gkeys, 0xFF, gcap * 8, st));
                MG(cudaMemsetAsync(nm.gval, 0xFF, gcap * 4, st));
                nm.gmask = (unsigned)(gcap - 1);
                IM_LAUNCH(k_rehash_xi, g, MGROW_THREADS, 0, st, M, nm);
            }
        }
        if (gt) {
            if (nt > 0) {
                MG(cudaMemcpyAsync(nm.tri, M.tri, (size_t)nt * sizeof(int4), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.tri_next, M.tri_next, (size_t)nt * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
                MG(cudaMemcpyAsync(nm.tri_flip, M.tri_flip, (size_t)nt * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
            }
            if (c_pub != h->chg.C.pub) {
                MG(cudaMemsetAsync(c_stamp, 0xFF, (size_t)tris * 4, st));
                MG(cudaMemsetAsync(c_pub, 0, (size_t)tris, st));
                if (nt > 0) {
                    MG(cudaMemcpyAsync(c_stamp, h->F.chg_stamp, (size_t)nt * 4, cudaMemcpyDeviceToDevice, st));
                    MG(cudaMemcpyAsync(c_pub, h->chg.C.pub, (size_t)nt, cudaMemcpyDeviceToDevice, st));
                }
            }
            nm.max_t = (int)tris;
            if (nm.thash != M.thash) {
                MG(cudaMemsetAsync(nm.thash, 0xFF, tcap * 4, st));
                nm.tmask = (unsigned)(tcap - 1);
                IM_LAUNCH(k_rehash_tris, g, MGROW_THREADS, 0, st, M, nm);
            }
        }
        if (gx && nm.vkeys != M.vkeys) {
            MG(cudaMemsetAsync(nm.vkeys, 0xFF, vcap * 8, st));
            MG(cudaMemsetAsync(nm.vox_chunk, 0xFF, vcap * IM_VCHUNKS * 4, st));
            for (int* q : {nm.vox_count, nm.vox_meshing_times, nm.vox_new_added}) MG(cudaMemsetAsync(q, 0, vcap * 4, st));
            MG(cudaMemsetAsync(nm.vox_frame, 0xFF, vcap * 4, st));
            nm.vmask = (unsigned)(vcap - 1);
            IM_LAUNCH(k_rehash_voxels, g, MGROW_THREADS, 0, st, M, nm);
        }
        MG(cudaGetLastError());
        MG(cudaStreamSynchronize(st));
#undef MG
        return r;
    };
    e = migrate();
    if (e != cudaSuccess) return fail(e, "mesh migration");   // the old buffers were only read: the handle is as it was
    // the replaced buffers go; the new ones join the handle's device memory
    const std::pair<const void*, const void*> replaced[] = {   // (old, new)
        {M.vpos, nm.vpos}, {M.vsmooth, nm.vsmooth}, {M.vsmoothed, nm.vsmoothed}, {M.v_tri_head, nm.v_tri_head}, {M.vchunk_pts, nm.vchunk_pts},
        {M.gkeys, nm.gkeys}, {M.gval, nm.gval}, {M.tri, nm.tri}, {M.tri_next, nm.tri_next}, {M.tri_flip, nm.tri_flip}, {M.thash, nm.thash},
        {M.vkeys, nm.vkeys}, {M.vox_chunk, nm.vox_chunk}, {M.vox_count, nm.vox_count}, {M.vox_meshing_times, nm.vox_meshing_times},
        {M.vox_new_added, nm.vox_new_added}, {M.vox_frame, nm.vox_frame}, {h->F.act, nf.act}};
    for (const auto& r : replaced)
        if (r.first != r.second) h->dev.free(r.first);
    h->dev.take(std::move(fresh));
    if (c_pub != h->chg.C.pub) {
        h->chg.dev.free(h->F.chg_stamp);
        h->chg.dev.free(h->chg.C.pub);
        h->chg.dev.take(std::move(cfresh));
        h->F.chg_stamp = c_stamp;
        h->chg.C.pub = c_pub;
    }
    if (h->b_fp) {   // batched-frame scratch: allocated again at the new sizes by the next batched frame
        h->batch = immesh::MemSet();
        h->b_act = h->b_sel = h->b_rank = h->b_hist = h->b_fset = nullptr;
        h->b_key = nullptr; h->b_ku = h->b_vu = nullptr; h->b_mark = nullptr; h->b_fp = nullptr;
    }
    nf.max_act = std::max(h->F.max_act, act);
    M = nm;
    h->F.act = nf.act;
    h->F.max_act = nf.max_act;
    h->max_vox = (int)vox;
    h->growths++;
    h->graph.destroy();
    IM_CUDA(cudaGetLastError());
    return IMMESH_OK;
}
// Automatic growth (immesh_mesh_set_growth) before a frame of m candidates: mesh_growth_targets (pool_growth.cuh) on the counters of
// the last frame known to have finished; the handle is drained only when a pool is short.
static int mesh_growth_check(immesh_mesh* h, long long m) {
    if (h->grow_max_bytes <= 0) return IMMESH_OK;
    long long steps = 1, m_max = m;
    for (int i = 1; i <= IM_SLOTS; ++i) {   // oldest frame first: consecutive frames give one frame's use each
        const int s = (h->frame_counter + i) & (IM_SLOTS - 1);
        if (!h->inflight[s]) continue;
        if (cudaEventQuery(h->ev_done[s]) == cudaSuccess) {
            mesh_note(h, h->h_cnt + IM_MC_HOST * s, h->h_dyn[s].frame);
        } else {
            ++steps;
            m_max = std::max<long long>(m_max, h->h_dyn[s].m);
        }
    }
    cudaGetLastError();   // cudaErrorNotReady of the queries
    for (int pass = 0; pass < 2; ++pass) {
        long long v = h->M.max_v, t = h->M.max_t, x = h->max_vox;
        mesh_growth_targets(h->known, steps, m_max, h->max_step_tris, &v, &t, &x);
        if (v == h->M.max_v && t == h->M.max_t && x == h->max_vox) return IMMESH_OK;
        if (pass == 1) return mesh_grow(h, v, t, x);
        IM_CUDA(cudaStreamSynchronize(h->stream));
        for (int i = 1; i <= IM_SLOTS; ++i) {
            const int s = (h->frame_counter + i) & (IM_SLOTS - 1);
            if (h->inflight[s]) mesh_note(h, h->h_cnt + IM_MC_HOST * s, h->h_dyn[s].frame);
        }
        steps = 1;
        m_max = m;
    }
    return IMMESH_OK;
}

static int mesh_grid_fixed(const immesh_mesh* h, long long n_cap, int threads, int waves = 8) {
    long long g = (n_cap + threads - 1) / threads;
    if (g > (long long)h->n_sm * waves) g = (long long)h->n_sm * waves;
    return g < 1 ? 1 : (int)g;
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
// the image of the camera in im.cam, with the tile counters zeroed, into result buffer (dyn->frame & 1) (fixed grids: every
// per-image value is read on the device)
// the binning passes of an image: the triangles at positions pos_mode (view_vertex) into the tiles' bins
static void rf_bin_launch(const immesh_mesh* h, const RfImage& im, int pos_mode, cudaStream_t st, int wire = 0) {
    const int g = h->n_sm * 8;
    IM_LAUNCH(k_rf_count, g, 128, 0, st, h->M, pos_mode, wire, (const DepthCam*)im.cam, im.tile_cnt);
    IM_LAUNCH(k_rf_scan, 1, 1024, 0, st, (const int*)im.tile_cnt, im.ntiles, im.tile_off, im.tile_cnt, im.bin_cap, im.misc);
    IM_LAUNCH(k_rf_fill, g, 128, 0, st, h->M, pos_mode, wire, (const DepthCam*)im.cam, im.tile_cnt, im.bin, (const int*)im.misc);
}
static void rf_image_launch(const immesh_mesh* h, const RfImage& im, const FrameDyn* dyn, cudaStream_t st) {
    const DepthCam* cam = im.cam;
    rf_bin_launch(h, im, 0, st);
    IM_LAUNCH(k_rf_tile, im.ntiles, IM_RT_THREADS, 0, st, h->M, cam, (const int*)im.tile_off, (const int*)im.bin, (const int*)im.misc, im.depth_bits);
    IM_LAUNCH(k_rf_fcount, im.nb, RF_FIN, 0, st, cam, (const unsigned int*)im.depth_bits, im.blk);
    IM_LAUNCH(k_rf_scan, 1, 1024, 0, st, (const int*)im.blk, im.nb, im.blk_off, (int*)nullptr, 0, (int*)nullptr);
    IM_LAUNCH(k_rf_emit, im.nb, RF_FIN, 0, st, cam, dyn, (const unsigned int*)im.depth_bits, (const int*)im.blk_off, im.nb, im.out[0], im.out[1]);
}
// the reinforcement of the frame just queued: its camera, then its image
static void mesh_reinforce_launch(immesh_mesh* h, cudaStream_t st) {
    auto& r = h->rf;
    IM_LAUNCH(k_rf_pose, 1, 256, 0, st, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame, (const FrameDyn*)h->d_dyn, (const RfDyn*)r.rd, r.win, r.base,
              r.img.cam, r.img.out[0], r.img.out[1], r.img.tile_cnt, r.img.ntiles);
    rf_image_launch(h, r.img, h->d_dyn, st);
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
// the queued view of the frame just queued: its camera (k_rf_pose, pose into the result buffer), then its image
static void mesh_view_launch(immesh_mesh* h, cudaStream_t st) {
    auto& v = h->vw;
    IM_LAUNCH(k_rf_pose, 1, 256, 0, st, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame, (const FrameDyn*)h->d_dyn, (const RfDyn*)v.rd, v.win, v.base,
              v.img.cam, v.img.out[0], v.img.out[1], v.img.tile_cnt, v.img.ntiles);
    if (v.ov.on) {   // the overlays' keys; the reinforced points are those of the reinforcement queued just before, while it is on
        const int g = h->n_sm * 8;
        IM_LAUNCH(k_ov_begin, g, 256, 0, st, v.ov, (const FrameDyn*)h->d_dyn, (const double (*)[12])h->cam_ring, (const int*)h->cam_ring_frame);
        IM_LAUNCH(k_ov_points, g, 128, 0, st, v.ov, (const DepthCam*)v.img.cam, (const FrameDyn*)h->d_dyn, h->rf.img.out[0], h->rf.img.out[1], h->rf.on);
        IM_LAUNCH(k_ov_lines, g, 128, 0, st, v.ov, (const DepthCam*)v.img.cam);
    }
    const ViewOut out[2] = {{v.rgba[0], v.img.out[0].depth}, {v.rgba[1], v.img.out[1].depth}};
    view_image_launch(h, v, v.img, out, h->d_dyn, st);
}

// ---- the frame feed (immesh_mesh_feed_enable, mesh_feed.cuh).  k_mfeed_begin stamps the start of the frame's launch sequence; behind
// the frame's last kernel (k_frame_end / k_chg_end, the reinforcement, the view) k_mfeed_head writes the header, the poses and the
// cursors (mfeed_head), k_mfeed_points and k_mfeed_image copy the reinforced points and the view image into their rings at the cursors,
// and k_mfeed_done stamps the end and publishes the frame's number to the host word the reader polls.  Fixed grids: every count is
// read on the device.  A slot outside its ring sets IM_MERR_FEED_INDEX and nothing is written.
__device__ __forceinline__ long long mfeed_clock() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__global__ void k_mfeed_begin(MeshFeedDev* fd) {
    pdl_wait();
    if (threadIdx.x == 0) fd->t_begin = mfeed_clock();
}
#define MFEED_THREADS 64
#define MFEED_COPY_THREADS 256
static_assert(IMMESH_MESH_FEED_POSE <= MFEED_THREADS, "one thread per pose value");
__global__ void __launch_bounds__(MFEED_THREADS) k_mfeed_head(MeshFeedDev* fd, int* cnt, long long* hdr, double* poses, long long max_frames, long long max_rows,
                                                              long long max_images, const double (*cam_ring)[12], RfOut rf0, RfOut rf1, const double* vw_pose0,
                                                              const double* vw_pose1, const FrameDyn* dyn) {
    pdl_wait();
    __shared__ long long s_slot, s_img;
    const long long frame = fd->dyn.frame;
    const int b = (int)(frame & 1);
    if (threadIdx.x == 0) {
        if (fd->dyn.n < 0) { fd->dyn.n = dyn->n; fd->dyn.step = dyn->step; }   // a depth frame: counted on the device
        const long long c[8] = {cnt[IM_MC_VERTICES], cnt[IM_MC_TRIS_LIVE], cnt[IM_MC_NEW_VERTICES], (long long)cnt[IM_MC_WORK_FRONT] + cnt[IM_MC_WORK_BACK],
                                cnt[IM_MC_ADD], cnt[IM_MC_REMOVE], cnt[IM_MC_VOXELS], cnt[IM_MC_ACT]};
        const int* nrf = b ? rf1.n : rf0.n;
        const long long slot = mfeed_head(*fd, c, cnt[IM_MC_ERR], (fd->dyn.rf && nrf) ? *nrf : 0, max_frames, max_rows, max_images, hdr);
        if (slot < 0) im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX);
        s_slot = slot;
        s_img = fd->img_slot;
    }
    __syncthreads();
    const long long slot = s_slot;
    if (slot < 0 || threadIdx.x >= IMMESH_MESH_FEED_POSE) return;
    // the frame pose, the reinforcement camera, the view camera: 12 doubles each (row-major R, then t)
    const int i = threadIdx.x, part = i / 12, k = i % 12;
    double v = 0.0;
    if (part == 0) {
        if (fd->dyn.has_rot) v = cam_ring[frame % IM_RF_RING][k];
        else if (k >= 9) v = fd->dyn.pose_t[k - 9];
    } else if (part == 1) {
        const double* p = b ? rf1.pose : rf0.pose;
        if (fd->dyn.rf && p) v = p[k];
    } else {
        const double* p = b ? vw_pose1 : vw_pose0;
        if (s_img >= 0 && p) v = p[k];
    }
    poses[slot * IMMESH_MESH_FEED_POSE + i] = v;
}
__global__ void __launch_bounds__(MFEED_COPY_THREADS) k_mfeed_points(const MeshFeedDev* fd, int* cnt, RfOut rf0, RfOut rf1, float* pts, int* pix, long long max_rows) {
    pdl_wait();
    const long long n = fd->nrows, base = fd->row_base;
    if (fd->hdr_slot < 0 || n <= 0) return;
    const RfOut o = (fd->dyn.frame & 1) ? rf1 : rf0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long s = mfeed_row_slot(base, i, max_rows);
        if (s < 0) { im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX); continue; }
        pts[s * 3 + 0] = o.pts[i * 3 + 0];
        pts[s * 3 + 1] = o.pts[i * 3 + 1];
        pts[s * 3 + 2] = o.pts[i * 3 + 2];
        pix[s] = o.pix[i];
    }
}
__global__ void __launch_bounds__(MFEED_COPY_THREADS) k_mfeed_image(const MeshFeedDev* fd, int* cnt, const uchar4* rgba0, const uchar4* rgba1, const float* depth0,
                                                                    const float* depth1, uchar4* ring, float* depth_ring, long long npx, long long max_images) {
    pdl_wait();
    const long long s = fd->img_slot;
    if (s < 0) return;   // no image for this frame
    if (!mfeed_slot_ok(s, max_images)) {
        if (blockIdx.x == 0 && threadIdx.x == 0) im_atomic_or(&cnt[IM_MC_ERR], IM_MERR_FEED_INDEX);
        return;
    }
    const int b = (int)(fd->dyn.frame & 1);
    const uchar4* src = b ? rgba1 : rgba0;
    const float* dsrc = b ? depth1 : depth0;
    uchar4* dst = ring + s * npx;
    float* ddst = depth_ring ? depth_ring + s * npx : nullptr;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
        dst[i] = src[i];
        if (ddst) ddst[i] = dsrc[i];
    }
}
__global__ void k_mfeed_done(const MeshFeedDev* fd, long long* hdr, long long* done) {
    pdl_wait();
    if (threadIdx.x == 0) {
        const long long slot = fd->hdr_slot;   // checked by k_mfeed_head (-1: refused)
        if (slot >= 0) hdr[slot * IMMESH_MESH_FEED_HDR + IMMESH_MFEED_T_END_NS] = mfeed_clock();
        __threadfence_system();
        *(volatile long long*)done = fd->dyn.frame;
    }
}
// the frame's feed inputs, from pinned slot s (released with the frame that last used it), ahead of its kernels in stream order
static int mesh_feed_stage(immesh_mesh* h, int s, long long frame, long long n, int step, int kind, const double* pose_t, bool rf, bool img) {
    auto& f = h->feed;
    MeshFeedDyn& d = f.h_dyn[s];
    d.frame = frame;
    d.n = n;
    d.step = step;
    d.kind = kind;
    d.has_rot = pose_t ? 0 : 1;
    d.rf = rf ? 1 : 0;
    d.img = img ? 1 : 0;
    d.pad_ = 0;
    for (int j = 0; j < 3; ++j) d.pose_t[j] = pose_t ? pose_t[j] : 0.0;
    IM_CUDA(cudaMemcpyAsync(&f.dev->dyn, &d, sizeof(MeshFeedDyn), cudaMemcpyHostToDevice, h->stream));
    return IMMESH_OK;
}
// the record behind the frame's last kernel; rf / img: the frame ran the reinforcement / its image is recorded (grids fixed)
static void mesh_feed_launch(immesh_mesh* h, cudaStream_t st, bool rf, bool img) {
    auto& f = h->feed;
    const RfOut none = {};
    const RfOut r0 = rf ? h->rf.img.out[0] : none, r1 = rf ? h->rf.img.out[1] : none;
    IM_LAUNCH(k_mfeed_head, 1, MFEED_THREADS, 0, st, f.dev, h->M.cnt, f.hdr, f.poses, f.max_frames, f.max_rows, f.max_images, (const double (*)[12])h->cam_ring, r0, r1,
              img ? (const double*)h->vw.img.out[0].pose : (const double*)nullptr, img ? (const double*)h->vw.img.out[1].pose : (const double*)nullptr,
              (const FrameDyn*)h->d_dyn);
    if (rf && f.max_rows > 0)
        IM_LAUNCH(k_mfeed_points, h->n_sm * 2, MFEED_COPY_THREADS, 0, st, (const MeshFeedDev*)f.dev, h->M.cnt, r0, r1, f.pts, f.pix, f.max_rows);
    if (img)
        IM_LAUNCH(k_mfeed_image, h->n_sm * 4, MFEED_COPY_THREADS, 0, st, (const MeshFeedDev*)f.dev, h->M.cnt, (const uchar4*)h->vw.rgba[0], (const uchar4*)h->vw.rgba[1],
                  (const float*)h->vw.img.out[0].depth, (const float*)h->vw.img.out[1].depth, f.rgba, f.depth_ring, f.npx, f.max_images);
    IM_LAUNCH(k_mfeed_done, 1, 32, 0, st, (const MeshFeedDev*)f.dev, f.hdr, f.d_done);
}
static int mesh_feed_commit(immesh_mesh* h, long long frame) {
    h->feed.queued = frame;
    IM_CUDA(cudaEventRecord(h->feed.ev, h->stream));
    return IMMESH_OK;
}
// drops the feed's buffers, stream and event; the caller has drained the stream and dropped the graph
static void mesh_feed_free(immesh_mesh* h) {
    auto& f = h->feed;
    if (f.ev) cudaEventDestroy(f.ev);
    if (f.stream) cudaStreamDestroy(f.stream);
    h->feed = immesh_mesh::Feed();
}

static int rb_passes(unsigned long long max_value) {   // 8-bit radix passes that cover max_value
    int b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return std::max(1, (b + 7) / 8);
}

// TriOrder (handles.hpp): the gather, one read-back of its counters, then the LSD passes over c, b, a and the region words from the last,
// each over the bits it can hold: the vertex ids below cnt[IM_MC_VERTICES], or the word's range (less its minimum)
extern "C++" int mesh_tri_order(immesh_mesh* h, const int* cnt, double region_size, TriOrder& o) {
    cudaStream_t st = h->stream;
    const int nalloc = std::min(cnt[IM_MC_TRIS_ALLOC], h->M.max_t), nv = cnt[IM_MC_VERTICES];
    const int nreg = region_size > 0 ? (o.qkeys ? 1 : 3) : 0;
    int m[8] = {0, 0, INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    IM_CUDA(cudaMemcpyAsync(o.misc, m, sizeof(m), cudaMemcpyHostToDevice, st));
    IM_LAUNCH(k_tri_gather, mesh_grid(h, nalloc, 128), 128, 0, st, h->M, nalloc, o.cap, region_size, o.qkeys, o.qval, o.qmask, o.rec, o.reg, o.misc);
    IM_CUDA(cudaMemcpyAsync(m, o.misc, sizeof(m), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (m[0] > o.cap) return im_fail(IMMESH_E_CUDA, "more live triangles than the mesh's counters hold (internal error)");
    o.n = m[0];
    o.range = m[1];
    int cur = 0;
    for (int w = 0; o.n > 0 && w < 3 + nreg; ++w) {
        const int c = w < 3 ? 0 : nreg - 1 - (w - 3);   // the region word of this pass
        const unsigned int base = w < 3 ? 0u : (unsigned int)m[2 + c];
        const unsigned long long top = w < 3 ? (unsigned long long)std::max(nv - 1, 0) : (unsigned long long)((unsigned int)m[5 + c] - base);
        IM_LAUNCH(k_tri_word, mesh_grid(h, o.n, 128), 128, 0, st, (const int4*)o.rec, (const int*)o.reg, nreg, o.n, w < 3 ? w : 3 + c, base,
                  w == 0 ? (const unsigned int*)nullptr : (const unsigned int*)o.v[cur], o.k[cur ^ 1], o.v[cur ^ 1]);
        cur = rs_sort_passes(st, o.k, o.v, cur ^ 1, o.n, rb_passes(top), o.hist);
    }
    IM_CUDA(cudaGetLastError());
    o.order = o.v[cur];
    return IMMESH_OK;
}
// mesh_tri_order's buffers for cap records with nreg region words each, placed in one block of 4-byte words: the records, the sort's
// keys and values, misc, hist, the region words.  Returns the block's words; a null base only counts them.
static size_t tri_order_carve(unsigned int* base, int cap, int nreg, TriOrder& o) {
    const size_t c = (size_t)std::max(cap, 1), nh = 256 * ((c + VG_TILE - 1) / VG_TILE);
    if (base) {
        o.cap = cap;
        o.rec = (int4*)base;
        o.k[0] = base + 4 * c; o.k[1] = o.k[0] + c;
        o.v[0] = o.k[1] + c; o.v[1] = o.v[0] + c;
        o.misc = (int*)(o.v[1] + c);
        o.hist = o.misc + 8;
        o.reg = o.hist + nh;
    }
    return 8 * c + 8 + nh + (size_t)nreg * c;
}

// the change feed of the frame whose push was just queued (F: its FrameBuf; batched: a batched frame, after k_bat_frame_end): the
// touched set (the sweep when batched or overflowed), the rows against the published bytes (marked per slot, then compacted), their LSD sort by (a, b, c) over words
// of the bits of max_v - 1, the ring append and the header.  Fixed grids: every count is read on the device.
static void mesh_changes_launch(immesh_mesh* h, const FrameBuf& F, cudaStream_t st, bool batched) {
    auto& c = h->chg;
    const int full = batched ? 1 : 0, cap = F.chg_cap;
    if (!batched) IM_LAUNCH(k_chg_gather, h->n_sm * 2, 128, 0, st, h->M, F);
    IM_LAUNCH(k_chg_sweep, h->n_sm * 8, 128, 0, st, h->M, F, c.C, full);
    unsigned int* ku[2] = {c.ku, c.ku + cap};
    unsigned int* vu[2] = {c.vu, c.vu + cap};
    const int g = mesh_grid_fixed(h, cap, 128), passes = rb_passes((unsigned long long)std::max(h->M.max_v - 1, 0));
    IM_LAUNCH(k_chg_mark, g, 128, 0, st, h->M, F, c.C, full);
    IM_LAUNCH(k_chg_rows, 1, 1024, 0, st, F, c.C, full);
    int cur = 0;
    for (int w = 0; w < 3; ++w) {
        IM_LAUNCH(k_chg_word, g, 128, 0, st, (const int*)F.chg_cnt, c.C, w, w == 0 ? (const unsigned int*)nullptr : (const unsigned int*)vu[cur], ku[cur ^ 1], vu[cur ^ 1]);
        cur = rs_sort_passes(st, ku, vu, cur ^ 1, cap, passes, c.hist, F.chg_cnt + IM_CH_ROWS);
    }
    IM_LAUNCH(k_chg_emit, g, 128, 0, st, F, c.C, (const unsigned int*)vu[cur], full);
    IM_LAUNCH(k_chg_end, 1, 1, 0, st, h->M, F, c.C, full, full);
}

// A depth frame's source (src_mode 4): the kernels' DepthFrame, and the host image to stage (null: df.img is the caller's device image)
struct DepthSrc {
    DepthFrame df;
    const unsigned char* host_img;
    long long pitch;
    int bpp;
};

// src_mode: 0 host world points, 1 device world points, 2 host body points + lio state, 3 device body points + lio state (n_dev: their
// count is read on the device, n its upper bound), 4 a depth image (dsrc; n is the sampled pixels, the upper bound of the count its
// kernels set on the device).
// Queues one frame (no host synchronisation except when both staging slots are still busy).  Host work per frame in the
// pipelined form: (memcpy into the pinned slot unless the caller's buffer is pinned) + H2D scan + H2D FrameDyn + one stream
// wait + ONE cudaGraphLaunch (no node is touched: every per-frame value is read from the FrameDyn) + one D2H of the counters.
static int mesh_enqueue(immesh_mesh_t* h, const float* xyz, int n, const double* pose_t, int src_mode, immesh_lio* lio, int kind, bool allow_graph = false,
                        const DepthSrc* dsrc = nullptr, const int* n_dev = nullptr) {
    const bool from_lio = src_mode == 2 || src_mode == 3, depth = src_mode == 4;
    const bool dev_dims = depth || n_dev;   // n, step, m and cmask are set on the device
    if (!h || (!xyz && n > 0 && !depth) || n < 0 || (!from_lio && !pose_t) || (depth && !dsrc)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (n > h->max_frame_points) return im_fail(IMMESH_E_CAPACITY, "frame larger than max_frame_points");
    FrameBuf& F = h->F;
    const MeshParams& P = h->P;
    // a depth frame's n, step, m and cmask are set by its kernels from the valid count, a device-count hand-off's by k_transform_full:
    // the host holds n = the upper bound and the most candidates it can give, for the growth check and for the grids, which cover
    // max_frame_points anyway
    int step, m;
    unsigned int cmask;
    frame_append_dims(n, P.append_target, &step, &m, &cmask);
    if (dev_dims) m = frame_append_max_m(n, P.append_target);
    const int grc = mesh_growth_check(h, m);
    if (grc) return grc;
    F.n = n;
    F.step = step;
    F.m = m;
    F.frame = ++h->frame_counter;
    const int s = F.frame & (IM_SLOTS - 1);
    int rc = mesh_harvest(h, s);  // the frame IM_SLOTS calls ago used this slot
    (void)rc;
    const size_t slot_pts = (size_t)h->max_frame_points * 3;
    float* d_pts = h->d_pts + s * slot_pts;
    float* h_pts = h->h_pts + s * slot_pts;
    FramePose* d_fp = h->d_fp + s;
    F.fp = d_fp;
    F.cmask = cmask;
    cudaStream_t st = h->stream;
    const bool graphed = allow_graph && h->use_graph && !profiler().enabled && (F.shard_n <= 1 || h->win.ok);
    if (!graphed) IM_CUDA(cudaEventRecord(h->ev[0], st));
    F.pts = d_pts;
    const float* d_body = nullptr;
    int pose_idx = 0;
    if (!from_lio) {
        FramePose* hp = h->h_fp + s;
        for (int j = 0; j < 3; ++j) { hp->pose_t[j] = pose_t[j]; hp->prio_origin[j] = (long long)std::floor(pose_t[j] / P.res) - 1024; }
        IM_CUDA(cudaMemcpyAsync(d_fp, hp, sizeof(FramePose), cudaMemcpyHostToDevice, st));
        if (depth) {
            F.pts = h->dep.pts;
            DepthFrame* hd = h->dep.h_df + s;
            *hd = dsrc->df;
            if (dsrc->host_img) {   // the sampled grid, tight, through the pinned slot (sw * sh * bpp <= 4 max_frame_points bytes)
                unsigned char* hb = reinterpret_cast<unsigned char*>(h_pts);
                const size_t rowb = (size_t)hd->sw * dsrc->bpp;
                depth_stage_grid(*hd, dsrc->host_img, dsrc->pitch, dsrc->bpp, hb);
                unsigned char* db = reinterpret_cast<unsigned char*>(h->d_body + s * slot_pts);
                IM_CUDA(cudaMemcpyAsync(db, hb, rowb * hd->sh, cudaMemcpyHostToDevice, h->stream_up));
                IM_CUDA(cudaEventRecord(h->ev_up[s], h->stream_up));
                IM_CUDA(cudaStreamWaitEvent(st, h->ev_up[s], 0));
                hd->img = db;
                hd->row_bytes = (long long)rowb;
                hd->col_bytes = dsrc->bpp;
            }
            IM_CUDA(cudaMemcpyAsync(h->dep.d_df, hd, sizeof(DepthFrame), cudaMemcpyHostToDevice, st));
        } else if (n > 0) {
            if (src_mode == 0) {
                const float* src = xyz;
                if (!immesh::host_ptr_is_pinned(xyz)) { std::memcpy(h_pts, xyz, (size_t)n * 3 * sizeof(float)); src = h_pts; }
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
            const float* src = xyz;
            if (!immesh::host_ptr_is_pinned(xyz)) { std::memcpy(h_pts, xyz, (size_t)n * 3 * sizeof(float)); src = h_pts; }
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
        d.n = F.n; d.step = F.step; d.m = F.m; d.frame = F.frame; d.cmask = F.cmask; d.pose_idx = pose_idx; d.epoch = epoch; d.n_dev = n_dev;
        IM_CUDA(cudaMemcpyAsync(h->d_dyn, &d, sizeof(FrameDyn), cudaMemcpyHostToDevice, st));
    }
    const bool rf_on = h->rf.on != 0, chg_on = h->chg.on != 0;
    if (rf_on) {   // the camera source of this frame
        RfDyn* r = (RfDyn*)h->rf.h_rd + s;
        r->mode = h->rf.explicit_pose;
        for (int i = 0; i < 9; ++i) r->R[i] = h->rf.R[i];
        for (int i = 0; i < 3; ++i) r->t[i] = h->rf.t[i];
        IM_CUDA(cudaMemcpyAsync(h->rf.rd, r, sizeof(RfDyn), cudaMemcpyHostToDevice, st));
    }
    const bool vw_on = h->vw.on != 0;
    const bool fd_on = h->feed.on != 0, fd_img = fd_on && vw_on && h->feed.max_images > 0;
    if (fd_on) {
        rc = mesh_feed_stage(h, s, F.frame, dev_dims ? -1 : F.n, F.step, kind, from_lio ? nullptr : pose_t, rf_on, fd_img);
        if (rc) return rc;
    }
    if (vw_on) {   // the view's camera source of this frame
        RfDyn* r = (RfDyn*)h->vw.h_rd + s;
        r->mode = h->vw.mode;
        for (int i = 0; i < 9; ++i) r->R[i] = h->vw.R[i];
        for (int i = 0; i < 3; ++i) r->t[i] = h->vw.t[i];
        IM_CUDA(cudaMemcpyAsync(h->vw.rd, r, sizeof(RfDyn), cudaMemcpyHostToDevice, st));
    }
    // the frame's launch sequence (fixed grids: grid-stride loops over the counts the kernels read on the device)
    bool nccl_failed = false;
    const int g_pts = mesh_grid_fixed(h, h->max_frame_points, 128);
    const int g_cand = mesh_grid_fixed(h, std::min<long long>(h->max_frame_points, 2LL * P.append_target), 128);
    // Graph-replayed and not sharded: a kernel that directly follows another kernel on `st` is a programmatic dependent launch.  The
    // first kernel after a copy, an event wait or the triangulation's join keeps an ordinary edge, as do the change feed's kernels.
    const bool pdl_frame = F.shard_n <= 1;
    auto launch_frame = [&](bool timing) {
        const bool pdl = pdl_frame && !timing;
        if (fd_on) IM_LAUNCH(k_mfeed_begin, 1, 32, 0, st, h->feed.dev);
        if (from_lio) IM_LAUNCH(k_transform_full, g_pts, 128, 0, st, lio->P, (const LioCtrl*)lio->d_ctrl, F, P.res, h->cam_ring, h->cam_ring_frame, P.append_target);
        if (depth) {
            auto& D = h->dep;
            IM_LAUNCH(k_depth_count, D.nb, DF_BLOCK, 0, st, (const DepthFrame*)D.d_df, D.blk);
            IM_LAUNCH(k_rf_scan, 1, 1024, 0, st, (const int*)D.blk, D.nb, D.blk_off, (int*)nullptr, 0, (int*)nullptr);
            IM_LAUNCH(k_depth_emit, D.nb, DF_BLOCK, 0, st, (const DepthFrame*)D.d_df, (const int*)D.blk_off, (const int*)D.blk_off, D.nb, 1, 0.0, P.append_target,
                      h->d_dyn, D.pts, D.n);
        }
        IM_LAUNCH_PDL(pdl && src_mode >= 2, k_frame_begin, h->n_sm * 8, 256, 0, st, h->M, F);
        if (timing) cudaEventRecord(h->ev[1], st);
        IM_LAUNCH_PDL(pdl, k_cand_init, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH_PDL(pdl, k_cand_conflicts, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH_PDL(pdl, k_cand_resolve, h->n_sm * 4, 128, 0, st, h->M, P, F);
        IM_LAUNCH_PDL(pdl, k_cand_scan, 1, 1024, 0, st, h->M, F);
        IM_LAUNCH_PDL(pdl, k_cand_commit, g_cand, 128, 0, st, h->M, P, F);
        IM_LAUNCH_PDL(pdl, k_cand_place, g_cand, 128, 0, st, h->M, F);
        IM_LAUNCH_PDL(pdl, k_voxel_select, g_cand, 128, 0, st, h->M, F);
        if (timing) cudaEventRecord(h->ev[2], st);
        IM_LAUNCH_PDL(pdl, k_voxel_dilate, h->n_sm * MESH_DILATE_BPS, 128, 0, st, h->M, P, F);
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
        IM_LAUNCH(k_voxel_tri_warp, h->n_sm * MESH_TRI_BPS, 128, 4 * sizeof(MeshWarpSmem<128>), h->stream2, h->M, P, F, h->warp_nmax);
        cudaEventRecord(h->ev_join, h->stream2);
        IM_LAUNCH(k_pull_vertices, h->n_sm * 8, 128, 0, h->stream3, h->M, P, F);   // incidence-list walk: only needs the dilation
        cudaEventRecord(h->ev_join3, h->stream3);
        IM_LAUNCH((k_voxel_mesh<256>), h->n_sm * MESH_TRI_BPS, 128, sizeof(MeshSmem<256>), st, h->M, P, F, h->warp_nmax, 1);
        cudaStreamWaitEvent(st, h->ev_join, 0);
        cudaStreamWaitEvent(st, h->ev_join3, 0);
        IM_LAUNCH((k_voxel_mesh<1024>), h->n_sm * 2, 128, sizeof(MeshSmem<1024>), st, h->M, P, F, 256, 0);
        IM_LAUNCH_PDL(pdl, k_commit_faces, h->n_sm * 8, 128, 0, st, h->M, P, F);
        IM_LAUNCH_PDL(pdl, k_pull_check, h->n_sm * 8, 128, 0, st, h->M, F);
        if (F.shard_n > 1 && h->win.ok) {   // every rank applies the facets / removals of all ranks to its replica of the store
            IM_LAUNCH(k_xpush, h->n_sm, 256, 0, st, h->M, F, (const unsigned char*)h->d_seg2, 1, pe, h->d_xdone + 1);
            IM_LAUNCH(k_apply_lists, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv2, h->seg2_bytes, pe);
        } else if (F.shard_n > 1) {
            IM_LAUNCH(k_xhdr, 1, 32, 0, st, h->M, F, (XHeader*)h->d_seg2);
            if (immesh::nccl().AllGather(h->d_seg2, h->d_recv2, h->seg2_bytes, immesh::kNcclUint8, h->nccl_comm, st)) nccl_failed = true;
            IM_LAUNCH(k_apply_lists, h->n_sm * 2, 256, 0, st, h->M, F, (const unsigned char*)h->d_recv2, h->seg2_bytes, pe);
        }
        if (timing) cudaEventRecord(h->ev[3], st);
        IM_LAUNCH_PDL(pdl, k_push_remove, h->n_sm * 2, 128, 0, st, h->M, F);
        IM_LAUNCH_PDL(pdl, k_push_add, h->n_sm * 2, 128, 0, st, h->M, F);
        if (chg_on) mesh_changes_launch(h, F, st, false);
        IM_LAUNCH_PDL(pdl && !chg_on, k_frame_end, 1, 1, 0, st, h->M);
        if (rf_on) mesh_reinforce_launch(h, st);
        if (vw_on) mesh_view_launch(h, st);
        if (fd_on) mesh_feed_launch(h, st, rf_on, fd_img);
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
    IM_CUDA(cudaMemcpyAsync(h->h_cnt + IM_MC_HOST * s, h->M.cnt, IM_MC_HOST * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (!queued) IM_CUDA(cudaEventRecord(h->ev[4], st));
    IM_CUDA(cudaEventRecord(h->ev_done[s], st));
    h->inflight[s] = 1;
    h->timed_last = queued ? 0 : 1;
    if (rf_on) h->rf.last_frame = F.frame;
    if (vw_on) h->vw.last_frame = F.frame;
    if (chg_on) h->chg.last_frame = F.frame;
    if (depth) h->dep.last_frame = F.frame;
    if (dev_dims) h->dev_dims_frame = F.frame;
    if (fd_on) return mesh_feed_commit(h, F.frame);
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
    int rc = mesh_enqueue(h, world_xyz, n, pose_t, 0, nullptr, IMMESH_MFEED_KIND_PUSH);
    return rc ? rc : mesh_wait_impl(h, true);
}
static int mesh_push_dev(immesh_mesh_t* h, const float* d_world_xyz, int n, const double* pose_t, int kind) {
    int rc = mesh_enqueue(h, d_world_xyz, n, pose_t, 1, nullptr, kind);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_dev(immesh_mesh_t* h, const float* d_world_xyz, int n, const double* pose_t, int frame_idx) {
    (void)frame_idx;
    return mesh_push_dev(h, d_world_xyz, n, pose_t, IMMESH_MFEED_KIND_PUSH_DEV);
}
int immesh_mesh_push_frame_from_lio(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    int rc = mesh_enqueue(h, body_xyz, n, nullptr, on_device ? 3 : 2, lio, IMMESH_MFEED_KIND_FROM_LIO);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_frame_from_lio_async(immesh_mesh_t* h, immesh_lio_t* lio, const float* body_xyz, int n, int on_device) {
    if (!lio) return im_fail(IMMESH_E_INVALID, "null lio handle");
    return mesh_enqueue(h, body_xyz, n, nullptr, on_device ? 3 : 2, lio, IMMESH_MFEED_KIND_FROM_LIO_ASYNC, true);
}
int immesh_mesh_push_frame_from_lio_async_dev_n(immesh_mesh_t* h, immesh_lio_t* lio, const float* d_body_xyz, int n_max, const int* d_n) {
    if (!h || !lio || !d_body_xyz || !d_n || n_max < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_push_frame_from_lio_async_dev_n: the mesh handle is sharded");
    return mesh_enqueue(h, d_body_xyz, n_max, nullptr, 3, lio, IMMESH_MFEED_KIND_FROM_LIO_ASYNC_DEV_N, true, nullptr, d_n);
}

// ---- depth-camera frames (include/immesh_b200.h, immesh_depth_frame)
// the image and camera of f checked and turned into the kernels' DepthFrame; the handle's depth buffers allocated by the first frame
static int depth_source(immesh_mesh* h, const immesh_depth_frame* f, const void* img, int on_device, DepthSrc* src, int* n_sampled) {
    if (!h) return im_fail(IMMESH_E_INVALID, "depth frame: null argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "depth frame: a sharded mesh handle takes world-frame points only");
    if (const char* bad = depth_frame_setup(f, img, &src->df, &src->pitch, &src->bpp)) return im_fail(IMMESH_E_INVALID, bad);
    const int sw = src->df.sw, sh = src->df.sh;
    if ((long long)sw * sh > h->max_frame_points) return im_fail(IMMESH_E_CAPACITY, "depth frame: more sampled pixels than max_frame_points");
    auto& D = h->dep;
    if (!D.pts) {
        immesh::MemSet dev, pinned{immesh::MemSet::Pinned};
        const int nb = (h->max_frame_points + DF_BLOCK - 1) / DF_BLOCK;
        cudaError_t e = dev.alloc(&D.d_df, 1);
        if (e == cudaSuccess) e = pinned.alloc(&D.h_df, IM_SLOTS);
        if (e == cudaSuccess) e = dev.alloc(&D.pts, (size_t)h->max_frame_points * 3);
        if (e == cudaSuccess) e = dev.alloc(&D.n, 1, 0);
        if (e == cudaSuccess) e = dev.alloc(&D.blk, (size_t)nb);
        if (e == cudaSuccess) e = dev.alloc(&D.blk_off, (size_t)nb + 1);
        if (e != cudaSuccess) {
            cudaGetLastError();
            D = immesh_mesh::Depth();
            return im_fail(IMMESH_E_CAPACITY, "depth frame: out of device or pinned memory for its buffers");
        }
        D.nb = nb;
        D.dev = std::move(dev);
        D.pinned = std::move(pinned);
    }
    src->host_img = on_device ? nullptr : static_cast<const unsigned char*>(img);
    *n_sampled = sw * sh;
    return IMMESH_OK;
}
int immesh_mesh_push_depth(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device) {
    DepthSrc src;
    int n = 0, rc = depth_source(h, f, depth, on_device, &src, &n);
    if (!rc) rc = mesh_enqueue(h, nullptr, n, f->cam_t, 4, nullptr, IMMESH_MFEED_KIND_DEPTH, false, &src);
    return rc ? rc : mesh_wait_impl(h, true);
}
int immesh_mesh_push_depth_async(immesh_mesh_t* h, const immesh_depth_frame* f, const void* depth, int on_device) {
    DepthSrc src;
    int n = 0;
    const int rc = depth_source(h, f, depth, on_device, &src, &n);
    return rc ? rc : mesh_enqueue(h, nullptr, n, f->cam_t, 4, nullptr, IMMESH_MFEED_KIND_DEPTH, true, &src);
}
int immesh_mesh_depth_points(immesh_mesh_t* h, float* xyz, int cap, int* n) {
    if (!h || !n || cap < 0 || (cap > 0 && !xyz)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (!h->dep.last_frame) return im_fail(IMMESH_E_INVALID, "no depth frame was pushed");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c = 0;
    IM_CUDA(cudaMemcpy(&c, h->dep.n, sizeof(int), cudaMemcpyDeviceToHost));
    *n = c;
    if (cap == 0) return IMMESH_OK;
    if (c > cap) return im_fail(IMMESH_E_CAPACITY, "more depth points than cap");
    if (c > 0) IM_CUDA(cudaMemcpy(xyz, h->dep.pts, (size_t)c * 3 * sizeof(float), cudaMemcpyDeviceToHost));
    return IMMESH_OK;
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
    if (h->grow_max_bytes > 0) return im_fail(IMMESH_E_INVALID, "a mesh handle with automatic growth cannot be sharded (immesh_mesh_set_growth(h, 0) first)");
    if (h->rf.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the reinforcement enabled cannot be sharded (immesh_mesh_reinforce_enable(h, NULL, ...) first)");
    if (h->chg.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the change feed enabled cannot be sharded (immesh_mesh_changes_enable(h, 0, 0) first)");
    if (h->feed.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the frame feed enabled cannot be sharded (immesh_mesh_feed_enable(h, NULL) first)");
    if (h->vw.on) return im_fail(IMMESH_E_INVALID, "a mesh handle with the queued view enabled cannot be sharded (immesh_mesh_view_enable(h, NULL, ...) first)");
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
    IM_CUDA(h->dev.alloc(&s1, h->seg1_bytes, 0));
    IM_CUDA(h->dev.alloc(&s2, h->seg2_bytes, 0));
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
        IM_CUDA(h->dev.alloc(&h->d_xdone, 2, 0));
    } else {
        IM_CUDA(h->dev.alloc(&h->d_recv1, h->seg1_bytes * nranks, 0));
        IM_CUDA(h->dev.alloc(&h->d_recv2, h->seg2_bytes * nranks, 0));
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
int immesh_graph_pdl_edges(immesh_lio_t* lio, immesh_mesh_t* mesh, int64_t* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "null argument");
    out[0] = lio ? lio->graph.pdl_edges : 0;
    out[1] = mesh ? mesh->graph.pdl_edges : 0;
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

int immesh_mesh_capacity(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int c[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, c));
    out[0] = h->M.max_v; out[1] = c[IM_MC_VERTICES];
    out[2] = h->M.max_t; out[3] = c[IM_MC_TRIS_ALLOC];
    out[4] = h->max_vox; out[5] = c[IM_MC_VOXELS];
    out[6] = (int64_t)(h->dev.bytes() + h->batch.bytes()); out[7] = h->growths;
    return IMMESH_OK;
}
int immesh_mesh_reserve(immesh_mesh_t* h, int64_t vertices, int64_t triangles, int64_t voxels) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_reserve: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    const int rc = mesh_grow(h, std::max<long long>(vertices, h->M.max_v), std::max<long long>(triangles, h->M.max_t), std::max<long long>(voxels, h->max_vox));
    if (rc == IMMESH_OK) return rc;
    return im_fail(rc, (std::string("immesh_mesh_reserve: ") + immesh::last_error_storage()).c_str());
}
int immesh_mesh_set_growth(immesh_mesh_t* h, int64_t max_bytes) {
    if (!h || max_bytes < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (max_bytes > 0 && h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "immesh_mesh_set_growth: a sharded handle cannot grow (its replicas would have to grow in lockstep)");
    if (max_bytes > 0 && h->grow_max_bytes <= 0) {   // growth starts from the mesh as it is now
        IM_CUDA(cudaStreamSynchronize(h->stream));
        IM_CUDA(mesh_read_counters(h, h->known));
        h->known_frame = h->frame_counter;
    }
    h->grow_max_bytes = max_bytes;
    return IMMESH_OK;
}
int immesh_mesh_counts(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    out[0] = c[IM_MC_VERTICES]; out[1] = c[IM_MC_TRIS_LIVE]; out[2] = c[IM_MC_NEW_VERTICES]; out[3] = c[IM_MC_WORK_FRONT] + c[IM_MC_WORK_BACK];
    out[4] = c[IM_MC_ADD]; out[5] = c[IM_MC_REMOVE]; out[6] = c[IM_MC_VOXELS]; out[7] = c[IM_MC_ACT];
    return IMMESH_OK;
}

int immesh_mesh_work_stats(immesh_mesh_t* h, int64_t* out) {
    if (!h || !out) return im_fail(IMMESH_E_INVALID, "null argument");
    const int* c = h->last_cnt;
    int m = h->F.m;
    if (h->dev_dims_frame && h->dev_dims_frame == h->frame_counter) {   // the newest frame's m is set on the device
        FrameDyn d;
        IM_CUDA(cudaStreamSynchronize(h->stream));
        IM_CUDA(cudaMemcpy(&d, h->d_dyn, sizeof(d), cudaMemcpyDeviceToHost));
        m = d.m;
    }
    out[0] = m; out[1] = c[IM_MC_STAT_GATHERED]; out[2] = c[IM_MC_STAT_QUERIES]; out[3] = c[IM_MC_STAT_DILATED]; out[4] = c[IM_MC_STAT_FACETS];
    out[5] = c[IM_MC_WORK_FRONT] + c[IM_MC_WORK_BACK]; out[6] = c[IM_MC_ADD]; out[7] = c[IM_MC_REMOVE];
    return IMMESH_OK;
}

int immesh_mesh_snapshot(immesh_mesh_t* h, float* vertices, int32_t* triangles, int32_t* flips) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    int cnt[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, cnt));
    const int nv = cnt[IM_MC_VERTICES], nlive = cnt[IM_MC_TRIS_LIVE];
    if (vertices && nv > 0) {
        std::vector<float4> v(nv);
        IM_CUDA(cudaMemcpy(v.data(), h->M.vpos, (size_t)nv * sizeof(float4), cudaMemcpyDeviceToHost));
        for (int i = 0; i < nv; ++i) { vertices[i * 3] = v[i].x; vertices[i * 3 + 1] = v[i].y; vertices[i * 3 + 2] = v[i].z; }
    }
    if ((triangles || flips) && nlive > 0) {
        immesh::MemSet tmp;
        TriOrder o = {};
        unsigned int* block = nullptr;
        int* d_tri = nullptr;   // [3 nlive] triples, then [nlive] flips
        IM_CUDA(tmp.alloc(&block, tri_order_carve(nullptr, nlive, 0, o)));
        tri_order_carve(block, nlive, 0, o);
        IM_CUDA(tmp.alloc(&d_tri, (size_t)nlive * 4));
        int* d_flip = d_tri + (size_t)nlive * 3;
        if (const int rc = mesh_tri_order(h, cnt, 0.0, o)) return rc;
        if (o.n > 0) IM_LAUNCH(k_tri_emit, mesh_grid(h, o.n, 128), 128, 0, h->stream, h->M, (const int4*)o.rec, o.order, o.n, d_tri, d_flip);
        IM_CUDA(cudaGetLastError());
        if (triangles) IM_CUDA(cudaMemcpyAsync(triangles, d_tri, (size_t)o.n * 3 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        if (flips) IM_CUDA(cudaMemcpyAsync(flips, d_flip, (size_t)o.n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        IM_CUDA(cudaStreamSynchronize(h->stream));
    }
    return IMMESH_OK;
}

int immesh_knn(immesh_mesh_t* h, const float* query_xyz, int nq, int k, double max_dist, int32_t* idx, float* d2) {
    if (!h || !query_xyz || !idx || !d2 || nq < 0 || k < 1 || k > KNN_KMAX) return im_fail(IMMESH_E_INVALID, "bad argument (k must be in [1,32])");
    if (nq == 0) return IMMESH_OK;
    immesh::MemSet tmp;
    float* dq = nullptr;
    int* di = nullptr;
    float* dd = nullptr;
    IM_CUDA(tmp.alloc(&dq, (size_t)nq * 3));
    IM_CUDA(tmp.alloc(&di, (size_t)nq * k));
    IM_CUDA(tmp.alloc(&dd, (size_t)nq * k));
    IM_CUDA(cudaMemcpyAsync(dq, query_xyz, (size_t)nq * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    IM_LAUNCH(k_knn, mesh_grid(h, nq * 32, 128), 128, 0, h->stream, h->M, h->P, (const float*)dq, 3, nq, k, max_dist, di, dd);
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(idx, di, (size_t)nq * k * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaMemcpyAsync(d2, dd, (size_t)nq * k * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    return IMMESH_OK;
}

int immesh_mesh_smooth_all(immesh_mesh_t* h, double smooth_factor, int knn, double* smoothed) {
    if (!h || knn < 1 || knn > KNN_KMAX) return im_fail(IMMESH_E_INVALID, "bad argument (knn must be in [1,32])");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int cnt[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, cnt));
    const int nv = cnt[IM_MC_VERTICES];
    if (nv == 0) return IMMESH_OK;
    immesh::MemSet tmp;
    int* di = nullptr;
    float* dd = nullptr;
    double* dout = nullptr;
    IM_CUDA(tmp.alloc(&di, (size_t)nv * knn));
    IM_CUDA(tmp.alloc(&dd, (size_t)nv * knn));
    if (smoothed) IM_CUDA(tmp.alloc(&dout, (size_t)nv * 3));
    IM_LAUNCH(k_knn, mesh_grid(h, nv, 4), 128, 0, h->stream, h->M, h->P, (const float*)h->M.vpos, 4, nv, knn, (double)INFINITY, di, dd);
    IM_LAUNCH(k_smooth_all, mesh_grid(h, nv, 128), 128, 0, h->stream, h->M, nv, knn, (const int*)di, (const float*)dd, smooth_factor, h->P.accept, dout);
    IM_CUDA(cudaGetLastError());
    if (smoothed) IM_CUDA(cudaMemcpyAsync(smoothed, dout, (size_t)nv * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    IM_CUDA(cudaStreamSynchronize(h->stream));
    return IMMESH_OK;
}

int immesh_mesh_region_stream(immesh_mesh_t* h, double region_size, int32_t* region_keys, int32_t* region_offsets, int cap_regions, int32_t* triangles, int* n_regions) {
    if (!h || !(region_size > 0) || !n_regions) return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    int cnt[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, cnt));
    const int nlive = cnt[IM_MC_TRIS_LIVE];
    *n_regions = 0;
    if (nlive == 0) { if (region_offsets && cap_regions >= 0) region_offsets[0] = 0; return IMMESH_OK; }
    cudaStream_t st = h->stream;
    immesh::MemSet tmp;
    TriOrder o = {};
    unsigned int* block = nullptr;
    int* d_flag = nullptr;   // [nlive + 1] region starts, scanned; then the keys [3 nlive], offsets [nlive] and triples [3 nlive]
    IM_CUDA(tmp.alloc(&block, tri_order_carve(nullptr, nlive, 3, o)));
    tri_order_carve(block, nlive, 3, o);
    IM_CUDA(tmp.alloc(&d_flag, (size_t)nlive * 8 + 1));
    int *d_keys = d_flag + nlive + 1, *d_off = d_keys + (size_t)nlive * 3, *d_tri = d_off + nlive;
    if (const int rc = mesh_tri_order(h, cnt, region_size, o)) return rc;   // a key past +-1048000 is ordered as any other: o.range is not an error here
    const int n = o.n, g = mesh_grid(h, n, RB_THREADS);
    IM_LAUNCH(k_rb_starts, g, RB_THREADS, 0, st, n, o.order, (const int*)o.reg, d_flag);
    IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, d_flag, n, d_flag + nlive);
    IM_LAUNCH(k_rb_regions, g, RB_THREADS, 0, st, n, o.order, (const int*)o.reg, (const int*)d_flag, d_keys, d_off);
    IM_LAUNCH(k_tri_emit, g, RB_THREADS, 0, st, h->M, (const int4*)o.rec, o.order, n, d_tri, (int*)nullptr);
    IM_CUDA(cudaGetLastError());
    int nr = 0;
    IM_CUDA(cudaMemcpyAsync(&nr, d_flag + nlive, sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    const int nc = std::min(nr, std::max(cap_regions, 0));   // the regions whose keys and offsets fit
    if (region_keys && nc > 0) IM_CUDA(cudaMemcpyAsync(region_keys, d_keys, (size_t)nc * 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (region_offsets && nc > 0) IM_CUDA(cudaMemcpyAsync(region_offsets, d_off, (size_t)nc * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (triangles && n > 0) IM_CUDA(cudaMemcpyAsync(triangles, d_tri, (size_t)n * 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (region_offsets && nr <= cap_regions) region_offsets[nr] = n;
    *n_regions = nr;
    return nr <= cap_regions ? IMMESH_OK : im_fail(IMMESH_E_CAPACITY, "more regions than cap_regions");
}

int immesh_mesh_region_buffers(immesh_mesh_t* h, double region_size, const int32_t* keys, int n_keys, double smooth_factor, int knn,
                               float* tri_xyz, int32_t* tri_ids, int cap, int32_t* region_keys, int32_t* region_offsets, int cap_regions,
                               float* axis_min_max, int* n_regions, int* n_tris, int* n_smoothed) {
    if (!h || !n_regions || !n_tris || !(region_size > 0) || knn < 1 || knn > KNN_KMAX || cap < 0 || cap_regions < 0 || (keys && n_keys < 0))
        return im_fail(IMMESH_E_INVALID, "bad argument (region_size > 0, knn in [1,32], cap >= 0, cap_regions >= 0)");
    *n_regions = 0;
    *n_tris = 0;
    if (n_smoothed) *n_smoothed = 0;
    const bool use_keys = keys != nullptr;
    const int nk = use_keys ? n_keys : 0;
    // the requested keys: a repeat is an error; a key outside the mesh's key range can hold no triangle (an empty segment)
    std::vector<unsigned long long> qk;
    std::vector<int> qv;
    unsigned int qmask = 0;
    if (use_keys) {
        std::vector<std::array<int, 3>> sk((size_t)nk);
        for (int i = 0; i < nk; ++i) sk[i] = {keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]};
        std::sort(sk.begin(), sk.end());
        if (std::adjacent_find(sk.begin(), sk.end()) != sk.end()) return im_fail(IMMESH_E_INVALID, "region_buffers: a region key is repeated");
        const size_t qcap = pow2_at_least((size_t)std::max(nk, 1) * 2);
        qk.assign(qcap, IM_EMPTY_KEY);
        qv.assign(qcap, -1);
        qmask = (unsigned int)(qcap - 1);
        for (int i = 0; i < nk; ++i) {
            if (!ikey_ok(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2])) continue;
            int created = 0;
            const int s = table_insert(qk.data(), qmask, pack_ikey(keys[3 * i], keys[3 * i + 1], keys[3 * i + 2]), &created);
            qv[s] = i;
        }
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));   // everything queued on the handle, the pipelined frames included
    cudaStream_t st = h->stream;
    int cnt[IM_MC_HOST];
    IM_CUDA(mesh_read_counters(h, cnt));
    const int nv = cnt[IM_MC_VERTICES], nlive = cnt[IM_MC_TRIS_LIVE];
    const size_t nl = (size_t)std::max(nlive, 1);
    // scratch buffer i of the call, at least `bytes` long (grow-only, kept by the handle)
    auto grown = [h](int i, size_t bytes, void** out) {
        const cudaError_t e = h->scratch.regrow(&h->region_scratch[i], &h->region_scratch_cap[i], bytes, 4096);
        *out = h->region_scratch[i];
        return e;
    };
    void *p_order, *p_flag, *p_misc, *p_q;
    TriOrder o = {};
    IM_CUDA(grown(0, tri_order_carve(nullptr, (int)nl, 3, o) * sizeof(unsigned int), &p_order));
    tri_order_carve((unsigned int*)p_order, (int)nl, 3, o);
    IM_CUDA(grown(1, (nl + 1) * sizeof(int), &p_flag));
    IM_CUDA(grown(2, 8 * sizeof(int), &p_misc));
    IM_CUDA(grown(3, std::max<size_t>(qk.size(), 1) * (sizeof(unsigned long long) + sizeof(int)), &p_q));
    int* flag = (int*)p_flag;
    int* misc = (int*)p_misc;   // [0] vertices claimed, [1] regions
    unsigned long long* d_qk = (unsigned long long*)p_q;
    int* d_qv = (int*)(d_qk + std::max<size_t>(qk.size(), 1));
    if (use_keys) {
        IM_CUDA(cudaMemcpyAsync(d_qk, qk.data(), qk.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaMemcpyAsync(d_qv, qv.data(), qv.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    }
    o.qkeys = use_keys ? d_qk : nullptr;
    o.qval = d_qv;
    o.qmask = qmask;
    IM_CUDA(cudaMemsetAsync(misc, 0, 8 * sizeof(int), st));
    if (const int rc = mesh_tri_order(h, cnt, region_size, o)) return rc;
    if (o.range) return im_fail(IMMESH_E_RANGE, "region_buffers: a region key is out of range (region_size too small for the mesh's extent)");
    const int n = o.n;
    int nr = use_keys ? nk : 0;
    if (n > 0 && !use_keys) {
        IM_LAUNCH(k_rb_starts, mesh_grid(h, n, RB_THREADS), RB_THREADS, 0, st, n, o.order, (const int*)o.reg, flag);
        IM_LAUNCH(k_rs_scan, 1, 1024, 0, st, flag, n, misc + 1);
        IM_CUDA(cudaGetLastError());
        IM_CUDA(cudaMemcpyAsync(&nr, misc + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
    }
    *n_tris = n;
    *n_regions = nr;
    if (n > cap || nr > cap_regions)
        return im_fail(IMMESH_E_CAPACITY, "region_buffers: more triangles than cap or more regions than cap_regions (*n_tris / *n_regions hold the numbers needed; nothing was smoothed)");
    void *p_reg, *p_rows, *p_part, *p_box;
    IM_CUDA(grown(4, ((size_t)nr * 3 + (size_t)nr + 1) * sizeof(int), &p_reg));
    int* d_rkeys = (int*)p_reg;
    int* d_roff = d_rkeys + (size_t)nr * 3;
    int* h_off_src = nullptr;
    std::vector<int> zeros;
    if (n == 0) {
        zeros.assign((size_t)nr + 1, 0);
        h_off_src = zeros.data();
    } else if (use_keys) {
        IM_LAUNCH(k_rb_offsets, mesh_grid(h, n, RB_THREADS), RB_THREADS, 0, st, n, nk, o.order, (const int*)o.reg, d_roff);
    } else {
        IM_LAUNCH(k_rb_regions, mesh_grid(h, n, RB_THREADS), RB_THREADS, 0, st, n, o.order, (const int*)o.reg, (const int*)flag, d_rkeys, d_roff);
        IM_CUDA(cudaMemcpyAsync(d_roff + nr, &n, sizeof(int), cudaMemcpyHostToDevice, st));
    }
    // lazy smoothing of the kept triangles' vertices (unparse_triangle_set_to_vector, :88-94)
    int nq = 0;
    if (n > 0) {
        void *p_bits, *p_list, *p_qpos;
        IM_CUDA(grown(5, (((size_t)nv + 31) / 32) * sizeof(unsigned int), &p_bits));
        const size_t qmax = (size_t)std::min<long long>((long long)nv, 3LL * n);
        IM_CUDA(grown(6, qmax * sizeof(int), &p_list));
        IM_CUDA(grown(7, qmax * sizeof(float4), &p_qpos));
        IM_CUDA(cudaMemsetAsync(p_bits, 0, (((size_t)nv + 31) / 32) * sizeof(unsigned int), st));
        IM_LAUNCH(k_rb_claim, mesh_grid(h, 3 * n, RB_THREADS), RB_THREADS, 0, st, h->M, n, (const int4*)o.rec, (unsigned int*)p_bits, misc, (int*)p_list, (float4*)p_qpos);
        IM_CUDA(cudaGetLastError());
        IM_CUDA(cudaMemcpyAsync(&nq, misc, sizeof(int), cudaMemcpyDeviceToHost, st));
        IM_CUDA(cudaStreamSynchronize(st));
        if (nq > 0) {
            void *p_idx, *p_d2;
            IM_CUDA(grown(8, (size_t)nq * knn * sizeof(int), &p_idx));
            IM_CUDA(grown(9, (size_t)nq * knn * sizeof(float), &p_d2));
            IM_LAUNCH(k_knn, mesh_grid(h, nq * 32, 128), 128, 0, st, h->M, h->P, (const float*)p_qpos, 4, nq, knn, (double)INFINITY, (int*)p_idx, (float*)p_d2);
            IM_LAUNCH(k_rb_smooth, mesh_grid(h, nq, RB_THREADS), RB_THREADS, 0, st, h->M, nq, knn, (const int*)p_list, (const int*)p_idx, (const float*)p_d2, smooth_factor, h->P.accept);
        }
    }
    if (n_smoothed) *n_smoothed = nq;
    // rows + axis box
    const int ge = mesh_grid(h, std::max(n, 1), RB_THREADS);
    IM_CUDA(grown(10, std::max<size_t>((size_t)n, 1) * 12 * sizeof(float), &p_rows));
    IM_CUDA(grown(11, (size_t)ge * sizeof(AxisAcc) + 8 * sizeof(float), &p_part));
    float* d_rows = (float*)p_rows;
    int* d_ids = (int*)(d_rows + (size_t)std::max(n, 1) * 9);
    AxisAcc* part = (AxisAcc*)p_part;
    p_box = (void*)(part + ge);
    if (n > 0) {
        IM_LAUNCH(k_rb_emit, ge, RB_THREADS, 0, st, h->M, n, o.order, (const int4*)o.rec, d_rows, d_ids, part);
        if (axis_min_max) {
            IM_CUDA(cudaMemcpyAsync(p_box, axis_min_max, 6 * sizeof(float), cudaMemcpyHostToDevice, st));
            IM_LAUNCH(k_rb_axis, 1, 1, 0, st, (const AxisAcc*)part, ge, (float*)p_box);
            IM_CUDA(cudaMemcpyAsync(axis_min_max, p_box, 6 * sizeof(float), cudaMemcpyDeviceToHost, st));
        }
    }
    IM_CUDA(cudaGetLastError());
    if (n > 0 && tri_xyz) IM_CUDA(cudaMemcpyAsync(tri_xyz, d_rows, (size_t)n * 9 * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (n > 0 && tri_ids) IM_CUDA(cudaMemcpyAsync(tri_ids, d_ids, (size_t)n * 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    if (region_offsets) {
        if (h_off_src) std::memcpy(region_offsets, h_off_src, ((size_t)nr + 1) * sizeof(int));
        else IM_CUDA(cudaMemcpyAsync(region_offsets, d_roff, ((size_t)nr + 1) * sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    if (region_keys) {
        if (use_keys) std::memcpy(region_keys, keys, (size_t)nk * 3 * sizeof(int));
        else if (nr > 0) IM_CUDA(cudaMemcpyAsync(region_keys, d_rkeys, (size_t)nr * 3 * sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    IM_CUDA(cudaStreamSynchronize(st));
    return IMMESH_OK;
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
    return mesh_push_dev(h, immesh_voxelgrid_device_points(vg), m, zero, IMMESH_MFEED_KIND_RECONSTRUCT);
}

// scratch of the batched frame: sized by max_voxels, max_work, max_triangles and max_list, never by the frame
// (all or nothing: after a failure the handle has none of it)
static cudaError_t mesh_batched_scratch(immesh_mesh* h) {
    if (h->b_fp) return cudaSuccess;
    const size_t nv = (size_t)std::max(h->max_vox, 1), nb = (nv + VG_TILE - 1) / VG_TILE, fcap = pow2_at_least((size_t)h->F.max_list * 2);
    immesh::MemSet b;
    int *act, *sel, *hist, *rank, *fset;
    unsigned long long* key;
    unsigned int *ku, *vu;
    unsigned char* mark;
    FramePose* fp;
    cudaError_t e;
    if ((e = b.alloc(&act, nv)) != cudaSuccess || (e = b.alloc(&sel, nv)) != cudaSuccess || (e = b.alloc(&key, nv)) != cudaSuccess ||
        (e = b.alloc(&ku, 2 * nv)) != cudaSuccess || (e = b.alloc(&vu, 2 * nv)) != cudaSuccess || (e = b.alloc(&hist, 256 * nb)) != cudaSuccess ||
        (e = b.alloc(&rank, (size_t)h->F.max_work)) != cudaSuccess || (e = b.alloc(&mark, (size_t)h->M.max_t, 0)) != cudaSuccess ||
        (e = b.alloc(&fset, fcap, 0xFF)) != cudaSuccess || (e = b.alloc(&fp, 1)) != cudaSuccess)
        return e;
    // the initialising memsets ran on the legacy stream, which the handle's non-blocking streams do not wait for
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return e;
    h->b_act = act; h->b_sel = sel; h->b_key = key; h->b_ku = ku; h->b_vu = vu; h->b_hist = hist; h->b_rank = rank; h->b_mark = mark; h->b_fset = fset; h->b_fp = fp;
    h->b_fset_mask = (unsigned int)(fcap - 1);
    h->batch = std::move(b);
    return cudaSuccess;
}

// incremental_mesh_reconstruction (src/ImMesh_mesh_reconstruction.cpp:92-267) as ONE frame of any size: append in chunks of <= B
// candidates, then the per-voxel stage in batches of <= V meshed voxels (DESIGN.md, batched frame).  Blocking.
static int mesh_push_batched(immesh_mesh* h, const float* xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels, int64_t* stats,
                             int kind) {
    if (!h || (!xyz && n > 0) || n < 0 || !pose_t || batch_points < 0 || batch_points > h->max_frame_points || batch_voxels < 0 || batch_voxels > h->F.max_work)
        return im_fail(IMMESH_E_INVALID, "bad argument (batch_points in [0, max_frame_points], batch_voxels in [0, the frame's work capacity])");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "push_frame_batched: a sharded handle is not supported");
    const int prev = mesh_wait_impl(h, false);   // frames queued before this one
    if (prev) return prev;
    {   // growth before the frame only (m candidates at most); an overflow inside it stays IMMESH_E_CAPACITY
        const int64_t st0 = std::max<int64_t>(1, (int64_t)std::llround((double)(n / (int64_t)h->P.append_target)));
        const int grc = mesh_growth_check(h, n > 0 ? (n + st0 - 1) / st0 : 0);
        if (grc) return grc;
    }
    IM_CUDA(mesh_batched_scratch(h));
    const MeshParams& P = h->P;
    const int B = batch_points ? batch_points : h->max_frame_points, V = batch_voxels ? batch_voxels : h->F.max_work;
    // append_point_step = max(1, round(N / appending_pts_frame)), integer division first (ImMesh_mesh_reconstruction.cpp:111), 64-bit
    const int64_t step = std::max<int64_t>(1, (int64_t)std::llround((double)(n / (int64_t)P.append_target)));
    if (step > 0x7fffffff) return im_fail(IMMESH_E_INVALID, "push_frame_batched: append step out of range");
    const int64_t m_total = n > 0 ? (n + step - 1) / step : 0;
    cudaStream_t st = h->stream;
    FrameBuf F = h->F;
    F.dyn = nullptr;
    F.epoch = 0;
    F.act = h->b_act; F.max_act = h->max_vox;
    F.work_rank = h->b_rank; F.tri_mark = h->b_mark;
    F.fset = h->b_fset; F.fset_mask = h->b_fset_mask;
    F.fp = h->b_fp;
    F.frame = ++h->frame_counter;   // one frame: one frame number, one vox_frame stamp
    FramePose fp;
    for (int j = 0; j < 3; ++j) { fp.pose_t[j] = pose_t[j]; fp.prio_origin[j] = 0; }
    IM_CUDA(cudaMemcpyAsync(h->b_fp, &fp, sizeof(FramePose), cudaMemcpyHostToDevice, st));
    IM_CUDA(cudaMemsetAsync(h->M.cnt + IM_MC_BAT_VERTICES, 0, (IM_MC_BAT_SELECTED + 1 - IM_MC_BAT_VERTICES) * sizeof(int), st));
    const bool fd_on = h->feed.on != 0;   // a header and the pose: the reinforcement and the view do not follow batched frames
    if (fd_on) {
        const int rc = mesh_feed_stage(h, F.frame & (IM_SLOTS - 1), F.frame, n, (int)step, kind, pose_t, false, false);
        if (rc) return rc;
        IM_LAUNCH(k_mfeed_begin, 1, 32, 0, st, h->feed.dev);
    }
    // ---- append, chunk c = candidates [c B, (c + 1) B), candidate i = point i step.  Host input: gathered into the pinned slot c & 1
    // while the device works on the other one
    const size_t slot_pts = (size_t)h->max_frame_points * 3;
    int64_t chunks = 0;
    for (int64_t c0 = 0; c0 < m_total || chunks == 0; c0 += B, ++chunks) {
        const int m = (int)std::min<int64_t>(B, m_total - c0);
        FrameBuf Fc = F;
        Fc.m = m; Fc.n = m;
        Fc.cmask = (unsigned)(pow2_at_least((size_t)std::max(m, 1) * 2) - 1);
        const int s = (int)(chunks & 1);
        if (m > 0 && !on_device) {
            float* hs = h->h_pts + s * slot_pts;
            float* ds = h->d_pts + s * slot_pts;
            if (chunks >= 2) IM_CUDA(cudaEventSynchronize(h->ev_up[s]));   // the slot's previous upload has left the pinned buffer
            if (step == 1) std::memcpy(hs, xyz + (size_t)c0 * 3, (size_t)m * 3 * sizeof(float));
            else for (int i = 0; i < m; ++i) std::memcpy(hs + (size_t)i * 3, xyz + (size_t)(c0 + i) * step * 3, 3 * sizeof(float));
            if (chunks >= 2) IM_CUDA(cudaStreamWaitEvent(h->stream_up, h->ev_in[s], 0));   // the chunk that read the slot has finished
            IM_CUDA(cudaMemcpyAsync(ds, hs, (size_t)m * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream_up));
            IM_CUDA(cudaEventRecord(h->ev_up[s], h->stream_up));
            IM_CUDA(cudaStreamWaitEvent(st, h->ev_up[s], 0));
            Fc.pts = ds; Fc.step = 1;
        } else {
            Fc.pts = xyz ? xyz + (size_t)c0 * step * 3 : nullptr;
            Fc.step = (int)step;
        }
        if (chunks == 0) IM_LAUNCH(k_frame_begin, h->n_sm * 8, 256, 0, st, h->M, Fc);
        else IM_LAUNCH(k_bat_chunk_begin, h->n_sm * 8, 256, 0, st, h->M, Fc);
        if (m > 0) {
            const int g = mesh_grid(h, m, 128);
            IM_LAUNCH(k_cand_init, g, 128, 0, st, h->M, P, Fc);
            IM_LAUNCH(k_cand_conflicts, g, 128, 0, st, h->M, P, Fc);
            IM_LAUNCH(k_cand_resolve, h->n_sm * 4, 128, 0, st, h->M, P, Fc);
            IM_LAUNCH(k_cand_scan, 1, 1024, 0, st, h->M, Fc);
            IM_LAUNCH(k_cand_commit, g, 128, 0, st, h->M, P, Fc);
            IM_LAUNCH(k_cand_place, g, 128, 0, st, h->M, Fc);
        }
        IM_LAUNCH(k_bat_chunk_end, 1, 1, 0, st, h->M);
        if (m > 0 && !on_device) IM_CUDA(cudaEventRecord(h->ev_in[s], st));
    }
    if (m_total == 0) chunks = 0;
    // ---- the activation rule after the last chunk; the meshed voxels in ascending key order
    IM_LAUNCH(k_bat_select, mesh_grid(h, h->max_vox, 128), 128, 0, st, h->M, F, h->b_sel, h->b_key);
    int nsel = 0;
    IM_CUDA(cudaGetLastError());
    IM_CUDA(cudaMemcpyAsync(&nsel, h->M.cnt + IM_MC_BAT_SELECTED, sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    unsigned int* ku[2] = {h->b_ku, h->b_ku + h->max_vox};
    unsigned int* vu[2] = {h->b_vu, h->b_vu + h->max_vox};
    int cur = 0;
    if (nsel > 0) {
        const int g = mesh_grid(h, nsel, 128);
        for (int half = 0; half < 2; ++half) {
            IM_LAUNCH(k_bat_word, g, 128, 0, st, nsel, half, (const unsigned long long*)h->b_key, half == 0 ? (const unsigned int*)nullptr : (const unsigned int*)vu[cur],
                      ku[cur ^ 1], vu[cur ^ 1]);
            cur = rs_sort_passes(st, ku, vu, cur ^ 1, nsel, 4, h->b_hist);
        }
    }
    const unsigned int* order = vu[cur];
    const int nbat = (nsel + V - 1) / V;
    const int g_fill = mesh_grid(h, V, 128);
    // ---- pass 1: every dilation of the frame, with its smoothing store, before any orientation
    for (int b = 0; b < nbat; ++b) {
        IM_LAUNCH(k_bat_reset, 1, 32, 0, st, h->M, F, 0);
        IM_LAUNCH(k_bat_fill, g_fill, 128, 0, st, h->M, F, (const int*)h->b_sel, order, b * V, std::min(nsel, (b + 1) * V), h->b_rank);
        IM_LAUNCH(k_voxel_dilate, h->n_sm * MESH_DILATE_BPS, 128, 0, st, h->M, P, F);
    }
    // ---- pass 2: the dilation lists again (the smoothing reads raw positions: the re-store writes the same bits), triangulation,
    // pull + commit against the pre-frame store, the batch's additions pushed at once
    for (int b = 0; b < nbat; ++b) {
        IM_LAUNCH(k_bat_reset, h->n_sm * 8, 256, 0, st, h->M, F, 1);
        IM_LAUNCH(k_bat_fill, g_fill, 128, 0, st, h->M, F, (const int*)h->b_sel, order, b * V, std::min(nsel, (b + 1) * V), h->b_rank);
        IM_LAUNCH(k_voxel_dilate, h->n_sm * MESH_DILATE_BPS, 128, 0, st, h->M, P, F);
        IM_CUDA(cudaEventRecord(h->ev_fork, st));
        IM_CUDA(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
        IM_CUDA(cudaStreamWaitEvent(h->stream3, h->ev_fork, 0));
        IM_LAUNCH(k_voxel_tri_warp, h->n_sm * MESH_TRI_BPS, 128, 4 * sizeof(MeshWarpSmem<128>), h->stream2, h->M, P, F, h->warp_nmax);
        IM_CUDA(cudaEventRecord(h->ev_join, h->stream2));
        IM_LAUNCH(k_pull_vertices, h->n_sm * 8, 128, 0, h->stream3, h->M, P, F);
        IM_CUDA(cudaEventRecord(h->ev_join3, h->stream3));
        IM_LAUNCH((k_voxel_mesh<256>), h->n_sm * MESH_TRI_BPS, 128, sizeof(MeshSmem<256>), st, h->M, P, F, h->warp_nmax, 1);
        IM_CUDA(cudaStreamWaitEvent(st, h->ev_join, 0));
        IM_CUDA(cudaStreamWaitEvent(st, h->ev_join3, 0));
        IM_LAUNCH((k_voxel_mesh<1024>), h->n_sm * 2, 128, sizeof(MeshSmem<1024>), st, h->M, P, F, 256, 0);
        IM_LAUNCH(k_commit_faces, h->n_sm * 8, 128, 0, st, h->M, P, F);
        IM_LAUNCH(k_pull_check, h->n_sm * 8, 128, 0, st, h->M, F);
        IM_LAUNCH(k_bat_push_add, h->n_sm * 2, 128, 0, st, h->M, F);
        IM_LAUNCH(k_bat_batch_end, 1, 1, 0, st, h->M);
    }
    IM_LAUNCH(k_bat_sweep, h->n_sm * 8, 128, 0, st, h->M, F);
    IM_LAUNCH(k_bat_frame_end, 1, 1, 0, st, h->M);
    if (h->chg.on) {
        mesh_changes_launch(h, F, st, true);
        h->chg.last_frame = F.frame;
    }
    if (fd_on) mesh_feed_launch(h, st, false, false);
    IM_CUDA(cudaGetLastError());
    if (fd_on) {
        const int rc = mesh_feed_commit(h, F.frame);
        if (rc) return rc;
    }
    int cnt[IM_MC_HOST];
    IM_CUDA(cudaMemcpyAsync(cnt, h->M.cnt, sizeof(cnt), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    std::memcpy(h->last_cnt, cnt, sizeof(cnt));
    if (h->grow_max_bytes > 0) mesh_note(h, cnt, F.frame);
    if (stats) { stats[0] = chunks; stats[1] = nbat; stats[2] = (int64_t)h->batch.bytes(); stats[3] = cnt[IM_MC_ADD]; }
    return mesh_status(cnt[IM_MC_ERR]);
}

int immesh_mesh_push_frame_batched(immesh_mesh_t* h, const float* world_xyz, int64_t n, int on_device, const double* pose_t, int batch_points, int batch_voxels,
                                   int64_t* stats) {
    return mesh_push_batched(h, world_xyz, n, on_device, pose_t, batch_points, batch_voxels, stats, IMMESH_MFEED_KIND_BATCHED);
}

int immesh_voxelgrid_leaf_too_small(immesh_voxelgrid_t* h, const float* xyz, int64_t n, int on_device, float leaf, int* too_small);   // frontend_capi.cu

int immesh_mesh_reconstruct_from_pointcloud_batched(immesh_mesh_t* h, immesh_voxelgrid_t* vg, const float* xyz, int64_t n, int on_device, double minimum_pts_distance,
                                                    int batch_points, int batch_voxels, int64_t* n_meshed_points) {
    if (!h || !vg || (!xyz && n > 0) || n < 0 || !(minimum_pts_distance > 0)) return im_fail(IMMESH_E_INVALID, "bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reconstruct_from_pointcloud_batched: a sharded handle is not supported");
    if (batch_points < 0 || batch_points > h->max_frame_points || batch_voxels < 0 || batch_voxels > h->F.max_work)
        return im_fail(IMMESH_E_INVALID, "bad argument (batch_points in [0, max_frame_points], batch_voxels in [0, the frame's work capacity])");
    if (n_meshed_points) *n_meshed_points = 0;
    const double zero[3] = {0.0, 0.0, 0.0};
    int small = 0;
    if (n > 0) {
        const int rc = immesh_voxelgrid_leaf_too_small(vg, xyz, n, on_device, (float)minimum_pts_distance, &small);
        if (rc) return rc;
    }
    if (small || n == 0) {   // PCL passes the cloud through: every raw point goes into the frame, whatever the VoxelGrid handle holds
        if (n_meshed_points) *n_meshed_points = n;
        return mesh_push_batched(h, xyz, n, on_device, zero, batch_points, batch_voxels, nullptr, IMMESH_MFEED_KIND_RECONSTRUCT_BATCHED);
    }
    int m = 0, small2 = 0;
    const int rc = n > 0x7fffffff ? IMMESH_E_CAPACITY : immesh_voxelgrid_filter(vg, xyz, (int)n, on_device, (float)minimum_pts_distance, nullptr, &m, &small2);
    if (rc == IMMESH_E_CAPACITY)
        return im_fail(IMMESH_E_CAPACITY, "reconstruct_from_pointcloud_batched: PCL down-samples this cloud and it holds more points than the VoxelGrid handle's max_points");
    if (rc) return rc;
    if (n_meshed_points) *n_meshed_points = m;
    return mesh_push_batched(h, immesh_voxelgrid_device_points(vg), m, 1, zero, batch_points, batch_voxels, nullptr, IMMESH_MFEED_KIND_RECONSTRUCT_BATCHED);
}

int immesh_mesh_render_depth(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, const double* cam_R, const double* cam_t,
                             float* depth, float* points, int32_t* point_pixel, int* n_points) {
    if (!h || !intrinsics || !cam_R || !cam_t || !depth || width < 1 || height < 1 || (long long)width * height > (1 << 26) || !(z_near > 0) || !(z_far > z_near))
        return im_fail(IMMESH_E_INVALID, "bad argument");
    IM_CUDA(cudaStreamSynchronize(h->stream));
    DepthCam C;
    C.fx = intrinsics[0]; C.fy = intrinsics[1]; C.cx = intrinsics[2]; C.cy = intrinsics[3]; C.z_near = z_near; C.z_far = z_far;
    for (int i = 0; i < 9; ++i) C.R[i] = cam_R[i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam_t[i];
    C.w = width; C.h = height;
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
    if (intrinsics) {
        const double* K = intrinsics;
        if (width < 1 || height < 1 || (long long)width * height > (1 << 26) || !(z_near > 0) || !(z_far > z_near) || !std::isfinite(z_far) || win < 1 ||
            win > IM_RF_RING - 1 || !std::isfinite(K[0]) || !std::isfinite(K[1]) || !std::isfinite(K[2]) || !std::isfinite(K[3]) || K[0] == 0.0 || K[1] == 0.0)
            return im_fail(IMMESH_E_INVALID, "reinforce_enable: bad argument (finite intrinsics with fx, fy != 0; 1 <= width * height <= 2^26; 0 < z_near < z_far; 1 <= win <= 63)");
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));   // frames in flight use the buffers
    h->graph.destroy();                          // the captured sequence changes
    h->rf = immesh_mesh::Reinforce();            // the buffers of an earlier enable go
    if (!intrinsics) return IMMESH_OK;
    immesh_mesh::Reinforce r;   // built in full before it replaces h->rf: after a failure the reinforcement stays disabled
    DepthCam& C = r.base;
    C.fx = intrinsics[0]; C.fy = intrinsics[1]; C.cx = intrinsics[2]; C.cy = intrinsics[3]; C.z_near = z_near; C.z_far = z_far;
    C.w = width; C.h = height;
    r.win = win;
    RfDyn *rd = nullptr, *h_rd = nullptr;
    cudaError_t e = rf_image_alloc(r.dev, width, height, 2, &r.img);
    if (e == cudaSuccess) e = r.dev.alloc(&rd, 1);
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = r.dev.alloc(&r.img.out[b].pose, 12);
    if (e == cudaSuccess) e = r.pinned.alloc(&h_rd, IM_SLOTS, 0);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "reinforce_enable: allocation of the reinforcement buffers failed");
    }
    r.rd = rd;
    r.h_rd = h_rd;
    r.on = 1;
    h->rf = std::move(r);
    return IMMESH_OK;
}
int immesh_mesh_reinforce_pose(immesh_mesh_t* h, const double* cam_R, const double* cam_t) {
    if (!h || (!cam_R) != (!cam_t)) return im_fail(IMMESH_E_INVALID, "bad argument (cam_R and cam_t both given or both NULL)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reinforce_pose: a sharded mesh handle is not supported");
    h->rf.explicit_pose = cam_R ? 1 : 0;
    for (int i = 0; i < 9; ++i) h->rf.R[i] = cam_R ? cam_R[i] : 0.0;
    for (int i = 0; i < 3; ++i) h->rf.t[i] = cam_t ? cam_t[i] : 0.0;
    return IMMESH_OK;
}
int immesh_mesh_reinforced_cloud(immesh_mesh_t* h, float* depth, float* points, int32_t* point_pixel, int cap, int* n_out, double* pose_out) {
    if (!h || !n_out || cap < 0) return im_fail(IMMESH_E_INVALID, "bad argument");
    *n_out = 0;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "reinforced_cloud: a sharded mesh handle is not supported");
    if (!h->rf.on) return im_fail(IMMESH_E_INVALID, "reinforced_cloud: the reinforcement is not enabled (immesh_mesh_reinforce_enable)");
    if (!h->rf.last_frame) return im_fail(IMMESH_E_INVALID, "reinforced_cloud: no frame has been queued since immesh_mesh_reinforce_enable");
    // the newest frame's result; the next queued frame writes the other buffer, so these copies (legacy stream) do not wait for it
    const int f = h->rf.last_frame, b = f & 1;
    IM_CUDA(cudaEventSynchronize(h->ev_done[f & (IM_SLOTS - 1)]));
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
static bool view_camera(const double* K, int width, int height, double z_near, double z_far, DepthCam* C) {
    if (!K || width < 1 || height < 1 || (long long)width * height > (1 << 26) || !(z_near > 0) || !(z_far > z_near)) return false;
    C->fx = K[0]; C->fy = K[1]; C->cx = K[2]; C->cy = K[3]; C->z_near = z_near; C->z_far = z_far;
    C->w = width; C->h = height;
    return true;
}
int immesh_mesh_render_view(immesh_mesh_t* h, const double* intrinsics, int width, int height, double z_near, double z_far, const double* cam_R, const double* cam_t,
                            const immesh_view_style* style, uint8_t* rgba, float* depth) {
    DepthCam C;
    if (!h || !cam_R || !cam_t || !rgba || !view_camera(intrinsics, width, height, z_near, z_far, &C)) return im_fail(IMMESH_E_INVALID, "render_view: bad argument");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "render_view: a sharded mesh handle is not supported");
    immesh_mesh::View v;   // this call's buffers; h->vw is not touched, so a queued frame's result stays readable
    float zr[2] = {0.f, 0.f};
    if (const int rc = view_style_set(style, "render_view", v, zr)) return rc;
    for (int i = 0; i < 9; ++i) C.R[i] = cam_R[i];
    for (int i = 0; i < 3; ++i) C.t[i] = cam_t[i];
    IM_CUDA(cudaStreamSynchronize(h->stream));
    const cudaError_t e = view_alloc(v, width, height, 1, h->n_sm * 4);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "render_view: allocation of the image buffers failed");
    }
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
        const double* K = intrinsics;
        if (!view_camera(K, width, height, z_near, z_far, &v.base) || !std::isfinite(z_far) || win < 1 || win > IM_RF_RING - 1 || !std::isfinite(K[0]) ||
            !std::isfinite(K[1]) || !std::isfinite(K[2]) || !std::isfinite(K[3]) || K[0] == 0.0 || K[1] == 0.0)
            return im_fail(IMMESH_E_INVALID, "view_enable: bad argument (finite intrinsics with fx, fy != 0; 1 <= width * height <= 2^26; 0 < z_near < z_far < inf; 1 <= win <= 63)");
        if (const int rc = view_style_set(style, "view_enable", v, zr)) return rc;
    }
    IM_CUDA(cudaStreamSynchronize(h->stream));   // frames in flight use the buffers
    h->graph.destroy();                          // the captured sequence changes
    h->vw = immesh_mesh::View();                 // the buffers of an earlier enable go
    {   // the frame feed's image ring was sized for the view that goes: image recording stops until the feed is enabled again
        auto& f = h->feed;
        f.img_mem = immesh::MemSet();
        f.rgba = nullptr; f.depth_ring = nullptr;
        f.max_images = 0; f.npx = 0; f.depth = 0;
    }
    if (!intrinsics) return IMMESH_OK;
    v.win = win;
    RfDyn *rd = nullptr, *h_rd = nullptr;
    cudaError_t e = view_alloc(v, width, height, 2, h->n_sm * 4);
    if (e == cudaSuccess) e = v.dev.alloc(&rd, 1);
    if (e == cudaSuccess) e = v.pinned.alloc(&h_rd, IM_SLOTS, 0);
    if (e == cudaSuccess) e = cudaMemsetAsync(v.zr_done, 0, sizeof(int), h->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(v.zr, zr, sizeof(zr), cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "view_enable: allocation of the view's buffers failed");
    }
    v.rd = rd;
    v.h_rd = h_rd;
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
    if (!h->vw.on) return im_fail(IMMESH_E_INVALID, "view_image: the view is not enabled (immesh_mesh_view_enable)");
    if (!h->vw.last_frame) return im_fail(IMMESH_E_INVALID, "view_image: no frame has been queued since immesh_mesh_view_enable");
    // the newest frame's result; the next queued frame writes the other buffer, so these copies (legacy stream) do not wait for it
    const int f = h->vw.last_frame, b = f & 1;
    const size_t n = (size_t)h->vw.base.w * h->vw.base.h;
    IM_CUDA(cudaEventSynchronize(h->ev_done[f & (IM_SLOTS - 1)]));
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
    IM_CUDA(cudaStreamSynchronize(h->stream));   // frames in flight use the buffers
    h->graph.destroy();                          // the captured sequence changes
    auto& v = h->vw;
    v.ov = ViewOverlay{};
    v.ov_dev = immesh::MemSet();
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
    if (e != cudaSuccess) {
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "view_overlay: allocation of the overlay's buffers failed");
    }
    ov.on = 1;
    v.ov = ov;
    v.ov_dev = std::move(dev);
    return IMMESH_OK;
}

int immesh_mesh_changes_enable(immesh_mesh_t* h, int64_t max_rows, int max_frames) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (max_rows < 0 || max_rows > IM_MPOOL_LIMIT || (max_rows > 0 && (max_frames < 1 || max_frames > (1 << 20))))
        return im_fail(IMMESH_E_INVALID, "changes_enable: bad argument (0 <= max_rows <= 2^30; 1 <= max_frames <= 2^20 when max_rows > 0)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "changes_enable: a sharded mesh handle is not supported");
    IM_CUDA(cudaStreamSynchronize(h->stream));   // frames in flight use the buffers
    h->graph.destroy();                          // the captured sequence changes
    h->chg = immesh_mesh::Changes();             // the buffers of an earlier enable go
    h->F.chg_stamp = nullptr; h->F.chg_list = nullptr; h->F.chg_cnt = nullptr; h->F.chg_cap = 0;
    if (max_rows == 0) return IMMESH_OK;
    immesh_mesh::Changes c;   // built in full before it replaces h->chg: after a failure the feed stays disabled
    ChgDev& C = c.C;
    C.max_rows = max_rows;
    C.max_frames = max_frames;
    const int cap = (int)std::min<int64_t>(max_rows, 1 << 21), max_t = h->M.max_t;   // a frame's touched slots: a bounded list
    int *stamp = nullptr, *list = nullptr, *cnt = nullptr;
    cudaError_t e = c.dev.alloc(&stamp, (size_t)max_t, 0xFF);
    auto add = [&e, &c](auto** p, size_t count, int fill = -1) { if (e == cudaSuccess) e = c.dev.alloc(p, std::max<size_t>(count, 1), fill); };
    add(&C.pub, (size_t)max_t, 0); add(&list, (size_t)cap); add(&cnt, IM_CH_SIZE, 0); add(&C.marked, (size_t)cap); add(&C.rowbuf, (size_t)cap);
    add(&c.ku, 2 * (size_t)cap); add(&c.vu, 2 * (size_t)cap); add(&c.hist, 256 * (((size_t)cap + VG_TILE - 1) / VG_TILE));
    add(&C.hdr, (size_t)max_frames, 0xFF); add(&C.ring, (size_t)max_rows); add(&C.written, 1, 0);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();   // the initialising memsets ran on the legacy stream
    int cnt_host[IM_MC_HOST];
    if (e == cudaSuccess) e = mesh_read_counters(h, cnt_host);
    if (e == cudaSuccess) {
        const int nalloc = std::min(cnt_host[IM_MC_TRIS_ALLOC], max_t);
        if (nalloc > 0) IM_LAUNCH(k_chg_init, mesh_grid(h, nalloc, 128), 128, 0, h->stream, h->M, C.pub, nalloc);
        if ((e = cudaGetLastError()) == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "changes_enable: allocation of the change feed's buffers failed");
    }
    c.on = 1;
    c.enable_frame = c.last_frame = h->frame_counter;
    h->chg = std::move(c);
    h->F.chg_stamp = stamp; h->F.chg_list = list; h->F.chg_cnt = cnt; h->F.chg_cap = cap;
    return IMMESH_OK;
}
int immesh_mesh_changes(immesh_mesh_t* h, int64_t since_frame, int64_t* frames, int cap_frames, int32_t* rows, int64_t cap_rows, float* vertices,
                        int64_t cap_vertices, int64_t* counts) {
    if (!h || !counts || cap_frames < 0 || cap_rows < 0 || cap_vertices < 0 || (cap_frames > 0 && !frames) || (cap_rows > 0 && !rows) || (cap_vertices > 0 && !vertices))
        return im_fail(IMMESH_E_INVALID, "changes: bad argument");
    for (int i = 0; i < 4; ++i) counts[i] = 0;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "changes: a sharded mesh handle is not supported");
    const auto& c = h->chg;
    if (!c.on) return im_fail(IMMESH_E_INVALID, "changes: the change feed is not enabled (immesh_mesh_changes_enable)");
    const int64_t newest = c.last_frame, nf = newest - since_frame;
    counts[3] = newest;
    if (since_frame > newest) return im_fail(IMMESH_E_INVALID, "changes: since_frame is newer than the newest queued frame");
    if (since_frame < c.enable_frame) return im_fail(IMMESH_E_RANGE, "changes: since_frame is older than the enable (resync: snapshot, then read from the newest frame)");
    if (nf > c.C.max_frames) return im_fail(IMMESH_E_RANGE, "changes: the frames after since_frame are no longer held (max_frames; resync: snapshot, then read from the newest frame)");
    if (nf == 0) return IMMESH_OK;
    IM_CUDA(cudaEventSynchronize(h->ev_done[newest & (IM_SLOTS - 1)]));   // the newest frame only (a batched frame has finished already)
    std::vector<ChgHdr> hdr((size_t)c.C.max_frames);
    long long written = 0;
    IM_CUDA(cudaMemcpy(hdr.data(), c.C.hdr, hdr.size() * sizeof(ChgHdr), cudaMemcpyDeviceToHost));
    IM_CUDA(cudaMemcpy(&written, c.C.written, sizeof(written), cudaMemcpyDeviceToHost));
    for (int64_t f = since_frame + 1; f <= newest; ++f) {
        const ChgHdr& r = hdr[(size_t)(f % c.C.max_frames)];
        if (r.frame != f || r.lost || r.r_begin < written - c.C.max_rows)
            return im_fail(IMMESH_E_RANGE, ("changes: the rows of frame " + std::to_string(f) + " are not held (" + (r.frame != f ? "not recorded" : r.lost ? "lost to the feed's per-frame list or ring" : "ring wrapped") +
                                            "; resync: snapshot, then read from the newest frame)").c_str());
    }
    const ChgHdr& first = hdr[(size_t)((since_frame + 1) % c.C.max_frames)];
    const ChgHdr& last = hdr[(size_t)(newest % c.C.max_frames)];
    const int64_t nrows = last.r_end - first.r_begin, nverts = last.v_end - first.v_begin;
    counts[0] = nf; counts[1] = nrows; counts[2] = nverts;
    if (nf > cap_frames || nrows > cap_rows || nverts > cap_vertices)
        return im_fail(IMMESH_E_CAPACITY, "changes: a buffer is smaller than the counts (counts holds them; nothing was written)");
    for (int64_t f = since_frame + 1, k = 0; f <= newest; ++f, ++k) {
        const ChgHdr& r = hdr[(size_t)(f % c.C.max_frames)];
        frames[k * 4 + 0] = f; frames[k * 4 + 1] = r.v_begin; frames[k * 4 + 2] = r.v_end; frames[k * 4 + 3] = r.r_end - first.r_begin;
    }
    for (int64_t g = first.r_begin; g < last.r_end;) {   // the ring range, in at most two pieces
        const int64_t pos = g % c.C.max_rows, len = std::min(last.r_end - g, c.C.max_rows - pos);
        IM_CUDA(cudaMemcpy(rows + (g - first.r_begin) * 4, c.C.ring + pos, (size_t)len * sizeof(int4), cudaMemcpyDeviceToHost));
        g += len;
    }
    if (nverts > 0) {   // a vertex never moves after its append: the positions are read now
        std::vector<float4> v((size_t)nverts);
        IM_CUDA(cudaMemcpy(v.data(), h->M.vpos + first.v_begin, (size_t)nverts * sizeof(float4), cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < nverts; ++i) { vertices[i * 3] = v[i].x; vertices[i * 3 + 1] = v[i].y; vertices[i * 3 + 2] = v[i].z; }
    }
    return IMMESH_OK;
}

int immesh_mesh_feed_enable(immesh_mesh_t* h, const immesh_mesh_feed_config* c) {
    if (!h) return im_fail(IMMESH_E_INVALID, "null handle");
    if (c && (c->max_frames < 1 || c->max_frames > (1LL << 20) || c->max_rows < 0 || c->max_rows > (1LL << 32) || c->max_images < 0 || c->max_images > (1LL << 16) ||
              (c->depth != 0 && c->depth != 1) || (c->depth && c->max_images == 0)))
        return im_fail(IMMESH_E_INVALID, "feed_enable: bad argument (max_frames in [1, 2^20], max_rows in [0, 2^32], max_images in [0, 2^16], depth 0 or 1 and 1 only with images)");
    if (c && c->max_images > 0 && !h->vw.on) return im_fail(IMMESH_E_INVALID, "feed_enable: images need the queued view (immesh_mesh_view_enable first)");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "feed_enable: a sharded mesh handle is not supported (the frame feed runs on a single GPU)");
    IM_CUDA(cudaStreamSynchronize(h->stream));   // frames in flight write the rings and the done word
    h->graph.destroy();                          // the captured sequence changes
    mesh_feed_free(h);                           // the rings of an earlier enable go
    if (!c) return IMMESH_OK;
    auto& f = h->feed;
    f.max_frames = c->max_frames;
    f.max_rows = c->max_rows;
    f.max_images = c->max_images;
    f.depth = c->depth;
    f.npx = c->max_images > 0 ? (long long)h->vw.base.w * h->vw.base.h : 0;   // the view as it is configured now
    auto fail = [&](cudaError_t e) {
        mesh_feed_free(h);
        cudaGetLastError();
        return im_fail(e == cudaErrorMemoryAllocation ? IMMESH_E_CAPACITY : IMMESH_E_CUDA, "feed_enable: allocation of the frame feed's buffers failed");
    };
    cudaError_t e;
    if ((e = f.dev_mem.alloc(&f.dev, 1, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.hdr, (size_t)f.max_frames * IMMESH_MESH_FEED_HDR, 0)) != cudaSuccess) return fail(e);
    if ((e = f.dev_mem.alloc(&f.poses, (size_t)f.max_frames * IMMESH_MESH_FEED_POSE, 0)) != cudaSuccess) return fail(e);
    if (f.max_rows > 0) {
        if ((e = f.dev_mem.alloc(&f.pts, (size_t)f.max_rows * 3)) != cudaSuccess) return fail(e);
        if ((e = f.dev_mem.alloc(&f.pix, (size_t)f.max_rows)) != cudaSuccess) return fail(e);
    }
    if (f.max_images > 0) {
        if ((e = f.img_mem.alloc(&f.rgba, (size_t)f.max_images * (size_t)f.npx)) != cudaSuccess) return fail(e);
        if (f.depth && (e = f.img_mem.alloc(&f.depth_ring, (size_t)f.max_images * (size_t)f.npx)) != cudaSuccess) return fail(e);
    }
    if ((e = f.pinned.alloc(&f.h_dyn, IM_SLOTS, 0)) != cudaSuccess) return fail(e);
    if ((e = f.pinned.alloc(&f.h_done, 1)) != cudaSuccess) return fail(e);
    *f.h_done = h->frame_counter;
    if ((e = cudaHostGetDevicePointer((void**)&f.d_done, f.h_done, 0)) != cudaSuccess) return fail(e);
    if ((e = cudaStreamCreateWithFlags(&f.stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e);
    if ((e = cudaEventCreateWithFlags(&f.ev, cudaEventDisableTiming)) != cudaSuccess) return fail(e);
    if ((e = cudaEventRecord(f.ev, h->stream)) != cudaSuccess) return fail(e);
    if ((e = cudaDeviceSynchronize()) != cudaSuccess) return fail(e);   // the initialising memsets ran on the legacy stream
    f.enable_frame = f.queued = h->frame_counter;
    f.on = 1;
    return IMMESH_OK;
}
// the marks a read checks after its copies: the newest frame whose slot is being written and the cursor of the ring read (points or images)
static int mesh_feed_marks(immesh_mesh* h, bool images, long long* m) {
    auto& f = h->feed;
    long long b[3];
    IM_CUDA(cudaMemcpyAsync(b, &f.dev->started, sizeof(b), cudaMemcpyDeviceToHost, f.stream));
    IM_CUDA(cudaStreamSynchronize(f.stream));
    static_assert(offsetof(MeshFeedDev, rows_total) == offsetof(MeshFeedDev, started) + 8 && offsetof(MeshFeedDev, imgs_total) == offsetof(MeshFeedDev, started) + 16,
                  "the marks are read with one copy");
    m[0] = b[0];
    m[1] = images ? b[2] : b[1];
    return IMMESH_OK;
}
// the common part of the two reads: arguments, the wait, counts[2..3]; returns the newest finished frame in *fin
static int mesh_feed_begin_read(immesh_mesh* h, const char* what, int64_t since, int wait, int64_t* counts, long long* fin) {
    auto& f = h->feed;
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": a sharded mesh handle is not supported").c_str());
    if (!f.on) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": the frame feed is not enabled (immesh_mesh_feed_enable)").c_str());
    if (since > f.queued) return im_fail(IMMESH_E_INVALID, (std::string(what) + ": since_frame is newer than the newest queued frame").c_str());
    if (wait) IM_CUDA(cudaEventSynchronize(f.ev));   // the newest queued frame's record, nothing else
    *fin = *(volatile long long*)f.h_done;
    counts[2] = *fin;
    counts[3] = f.queued;
    return IMMESH_OK;
}
static int mesh_feed_end_read(int rc, const char* what) {
    if (rc == IMMESH_E_RANGE)
        return im_fail(rc, (std::string(what) + ": frames of the range predate the enable, left the rings or were overwritten while they were read; read on from counts[2]").c_str());
    if (rc == IMMESH_E_CAPACITY) return im_fail(rc, (std::string(what) + ": more frames or rows than the caps (counts holds them; nothing was written)").c_str());
    return rc;
}
int immesh_mesh_feed(immesh_mesh_t* h, int64_t since, int wait, int64_t* frames, double* poses, int cap_frames, float* points, int32_t* pixels, int64_t cap_rows,
                     int64_t* counts) {
    if (counts) for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (!h || !counts || since < 0 || cap_frames < 0 || cap_rows < 0 || (cap_frames > 0 && !frames)) return im_fail(IMMESH_E_INVALID, "feed: bad argument");
    long long fin = 0;
    int rc = mesh_feed_begin_read(h, "feed", since, wait, counts, &fin);
    if (rc) return rc;
    auto& f = h->feed;
    const FeedRings rings = mfeed_point_rings(f.max_frames, f.max_rows, f.hdr, f.poses, f.pts, f.pix);
    auto copy = [&](void* dst, const void* src, size_t bytes) {   // on the feed's stream, never the handle's
        IM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, f.stream));
        return IMMESH_OK;
    };
    auto marks = [&](long long* m) { return mesh_feed_marks(h, false, m); };
    rc = feed_read(rings, since, fin, frames, poses, cap_frames, points, pixels, cap_rows, counts, copy, marks);
    return mesh_feed_end_read(rc, "feed");
}
int immesh_mesh_feed_images(immesh_mesh_t* h, int64_t since, int wait, int64_t* frames, int cap_images, uint8_t* rgba, float* depth, int64_t* counts) {
    if (counts) for (int k = 0; k < 4; ++k) counts[k] = 0;
    if (!h || !counts || since < 0 || cap_images < 0 || (cap_images > 0 && !frames)) return im_fail(IMMESH_E_INVALID, "feed_images: bad argument");
    auto& f = h->feed;
    if (f.on && f.max_images == 0)
        return im_fail(IMMESH_E_INVALID, "feed_images: image recording is off (max_images = 0, or immesh_mesh_view_enable was called after the enable)");
    if (f.on && depth && !f.depth) return im_fail(IMMESH_E_INVALID, "feed_images: depth requested but the feed was enabled without depth");
    long long fin = 0;
    int rc = mesh_feed_begin_read(h, "feed_images", since, wait, counts, &fin);
    if (rc) return rc;
    FeedRings rings = mfeed_image_rings(f.max_frames, f.max_images, f.npx, f.hdr, f.rgba, f.depth_ring);
    void* rows = rgba;
    void* second = depth;
    if (!rgba && depth) {   // the depth images alone: they are the rows
        rings.rows = f.depth_ring;
        rings.idx = nullptr;
        rows = depth;
        second = nullptr;
    }
    auto copy = [&](void* dst, const void* src, size_t bytes) {
        IM_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, f.stream));
        return IMMESH_OK;
    };
    auto marks = [&](long long* m) { return mesh_feed_marks(h, true, m); };
    rc = feed_read(rings, since, fin, frames, nullptr, cap_images, rows, second, cap_images, counts, copy, marks);
    return mesh_feed_end_read(rc, "feed_images");
}

int immesh_mesh_last_timing(immesh_mesh_t* h, double* ms) {
    if (!h || !ms) return im_fail(IMMESH_E_INVALID, "null argument");
    for (int i = 0; i < 4; ++i) ms[i] = h->last_ms[i];
    return IMMESH_OK;
}

}  // extern "C"
