// immesh_b200 -- the mesher's queries: the live triangles in order (mesh_tri_order), the snapshot, kNN, smooth_all, the region
// stream and the viewer's region buffers.  CUDA kernels (sm_90a) and their C-ABI host orchestration.
#include <array>
#include <climits>
#include <cmath>

#include "handles.hpp"

using namespace immesh;
namespace {
#include "radix_sort.cuh"
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

int mesh_sort_passes(cudaStream_t st, unsigned int* const k[2], unsigned int* const v[2], int cur, int n, int passes, int* hist, const int* n_dev) {
    return rs_sort_passes(st, k, v, cur, n, passes, hist, n_dev);
}
size_t mesh_sort_hist_ints(size_t n) { return 256 * ((n + VG_TILE - 1) / VG_TILE); }

// TriOrder (handles.hpp): the gather, one read-back of its counters, then the LSD passes over c, b, a and the region words from the last,
// each over the bits it can hold: the vertex ids below cnt[IM_MC_VERTICES], or the word's range (less its minimum)
int mesh_tri_order(immesh_mesh* h, const int* cnt, double region_size, TriOrder& o) {
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

