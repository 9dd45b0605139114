// immesh_b200 -- immesh_mesh_evaluate: the fairness and correctness metrics of the paper's Experiment-3 (ImMesh, section VIII-C,
// Tables V and VI, Fig. 8 and 9) for the device-resident mesh against a ground-truth cloud.  The per-element bodies are in
// mesh_eval.cuh; the rules are stated in include/immesh_b200.h.
//
// Shape of the call (every step on the device, the host only plans tiles and reads a few counts):
//   1. live triangles compacted and sorted by (a, b, c) (mesh_tri_order, as immesh_mesh_snapshot orders them); per triangle the float32 corner positions,
//      the fairness terms and the subdivision count n.
//   2. space is split into tiles (bisection of the bounding box of the mesh and the ground truth) until the scratch one tile needs
//      fits the budget.  A query (sample or down-sampled ground-truth point) is answered in the tile that holds it, against the
//      targets of the tile and a halo of max_dist around it, so that nothing depends on the tiling.
//   3. per tile: the samples of every triangle whose box touches the halo are generated (k_eval_samples); the ground-truth points are
//      gathered, sorted into input order and by leaf, and one thread per leaf sums the leaf in input order (k_eval_leaf_points); a
//      hashed uniform grid is built over each target set and each query runs a ring search for its exact nearest target
//      (k_eval_query).  Counts, quantised distance sums and per-facet counts are integer atomics, so they do not depend on order.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/immesh_b200.h"
#include "common_host.hpp"
#include "handles.hpp"
#include "mesh_eval.cuh"

using namespace immesh;
namespace {
#include "radix_sort.cuh"
}

namespace {

// device accumulators of one call (unsigned long long each)
enum : int {
    EA_DEGENERATE = 0, EA_SUM_N2, EA_N_MAX, EA_UNSMOOTHED, EA_N_RANGE,
    EA_BOX_MIN,                     // 3 slots: ordered-float minimum of every mesh and ground-truth coordinate
    EA_BOX_MAX = EA_BOX_MIN + 3,    // 3 slots: maximum
    EA_NONFINITE = EA_BOX_MAX + 3,  // non-finite ground-truth points
    EA_PLAN_S, EA_PLAN_G,           // tile planning: samples / ground-truth points a tile gathers (upper bound / exact)
    EA_SAMPLES, EA_GT, EA_S_WITHIN, EA_G_WITHIN, EA_S_FAR, EA_G_FAR, EA_S_Q, EA_G_Q, EA_INCORRECT, EA_OVERFLOW,
    EA_SIZE
};
constexpr int EVAL_KEY_BITS = 21;   // bits per axis of a packed cell / leaf key inside a tile's halo
constexpr long long EVAL_KEY_SPAN = (1LL << EVAL_KEY_BITS) - 4;

struct EvalBox { double lo[3], hi[3]; };
// what a tile gathers: targets inside `halo` (leaf == 0), or the whole leaves whose keys lie in [klo, khi] (leaf > 0)
struct EvalGather {
    EvalBox halo;
    double leaf;
    long long klo[3], khi[3];
};
struct EvalGrid {
    const unsigned long long* keys;
    const int* cnt;
    const int* end;       // one past the cell's last point in pts
    const float4* pts;
    unsigned int mask;
    int n;
    double org[3];
    double cell;
};

__device__ __forceinline__ unsigned long long eval_ord(float f) {   // order-preserving map of a float onto an unsigned integer
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? (unsigned long long)(~u) : (unsigned long long)(u | 0x80000000u);
}
inline float eval_unord(unsigned long long o) {
    const unsigned u = (unsigned)o;
    const unsigned b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    std::memcpy(&f, &b, 4);
    return f;
}
__device__ __forceinline__ bool in_box(float x, float y, float z, const EvalBox& b) {   // half-open: every point in exactly one tile
    return (double)x >= b.lo[0] && (double)x < b.hi[0] && (double)y >= b.lo[1] && (double)y < b.hi[1] && (double)z >= b.lo[2] && (double)z < b.hi[2];
}
__device__ __forceinline__ bool in_halo(float x, float y, float z, const EvalBox& b) {
    return (double)x >= b.lo[0] && (double)x <= b.hi[0] && (double)y >= b.lo[1] && (double)y <= b.hi[1] && (double)z >= b.lo[2] && (double)z <= b.hi[2];
}
__device__ __forceinline__ bool in_gather(const float* p, const EvalGather& g) {
    if (g.leaf == 0.0) return in_halo(p[0], p[1], p[2], g.halo);
    for (int c = 0; c < 3; ++c) {
        const long long k = eval_leaf_key(p[c], g.leaf);
        if (k < g.klo[c] || k > g.khi[c]) return false;
    }
    return true;
}
__device__ __forceinline__ unsigned long long leaf_local_key(const float* p, const EvalGather& g) {
    unsigned long long key = 0;
    for (int c = 0; c < 3; ++c) key = (key << EVAL_KEY_BITS) | (unsigned long long)(eval_leaf_key(p[c], g.leaf) - g.klo[c]);
    return key;
}
__device__ __forceinline__ unsigned long long warp_sum_ull(unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void acc_add(unsigned long long* acc, int slot, unsigned long long v) {   // once per warp
    v = warp_sum_ull(v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(acc + slot, v);
}

// ---- 1. live triangles
// per sorted triangle: its triple, the float32 corners (raw or (float) of the smoothed position), fairness and subdivisions
__global__ void __launch_bounds__(128) k_eval_tri(MeshDev M, int smoothed, const int4* tri, const unsigned* perm, int n, double spacing, int4* st,
                                                   float* tp, int* nsub, double* fair, unsigned long long* acc) {
    unsigned long long deg = 0, n2 = 0, nmax = 0, unsm = 0, nrange = 0;
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 t = tri[perm[i]];
        st[i] = t;
        float p[9];
        const int v[3] = {t.x, t.y, t.z};
        for (int q = 0; q < 3; ++q) {
            for (int c = 0; c < 3; ++c) {
                p[q * 3 + c] = smoothed ? (float)M.vsmooth[(size_t)v[q] * 3 + c] : (c == 0 ? M.vpos[v[q]].x : c == 1 ? M.vpos[v[q]].y : M.vpos[v[q]].z);
                mn[c] = fminf(mn[c], p[q * 3 + c]);
                mx[c] = fmaxf(mx[c], p[q * 3 + c]);
            }
            if (smoothed && !(M.vsmoothed && M.vsmoothed[v[q]])) ++unsm;
        }
        for (int k = 0; k < 9; ++k) tp[(size_t)i * 9 + k] = p[k];
        const EvalTri e = eval_triangle(p, p + 3, p + 6);
        int ns = 0;
        if (e.degenerate) {
            ++deg;
        } else {
            ns = eval_subdivisions(e.longest, spacing);
            if (ns == 0) ++nrange;
            n2 += (unsigned long long)ns * ns;
            nmax = max(nmax, (unsigned long long)ns);
        }
        nsub[i] = ns;
        fair[2 * (size_t)i] = e.degenerate ? 0.0 : e.maxmin;
        fair[2 * (size_t)i + 1] = e.degenerate ? 0.0 : e.c2se;
    }
    acc_add(acc, EA_DEGENERATE, deg);
    acc_add(acc, EA_SUM_N2, n2);
    acc_add(acc, EA_UNSMOOTHED, unsm);
    acc_add(acc, EA_N_RANGE, nrange);
    if (nmax) atomicMax(acc + EA_N_MAX, nmax);
    for (int c = 0; c < 3; ++c) {
        if (mn[c] <= mx[c]) { atomicMin(acc + EA_BOX_MIN + c, eval_ord(mn[c])); atomicMax(acc + EA_BOX_MAX + c, eval_ord(mx[c])); }
    }
}
// the two fairness sums in a fixed order (one block of 1024 threads: strided partial sums, then a fixed tree)
__global__ void __launch_bounds__(1024) k_eval_fair_sum(const double* fair, int n, double* out) {
    __shared__ double s[2][1024];
    double a = 0, b = 0;
    for (int i = threadIdx.x; i < n; i += 1024) { a += fair[2 * (size_t)i]; b += fair[2 * (size_t)i + 1]; }
    s[0][threadIdx.x] = a;
    s[1][threadIdx.x] = b;
    __syncthreads();
    for (int w = 512; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) { s[0][threadIdx.x] += s[0][threadIdx.x + w]; s[1][threadIdx.x] += s[1][threadIdx.x + w]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out[0] = s[0][0]; out[1] = s[1][0]; }
}
// ground truth: non-finite points and the bounding box
__global__ void __launch_bounds__(128) k_eval_gt_scan(const float* gt, long long n, unsigned long long* acc) {
    unsigned long long bad = 0;
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float* p = gt + i * 3;
        if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) { ++bad; continue; }
        for (int c = 0; c < 3; ++c) { mn[c] = fminf(mn[c], p[c]); mx[c] = fmaxf(mx[c], p[c]); }
    }
    acc_add(acc, EA_NONFINITE, bad);
    for (int c = 0; c < 3; ++c) {
        if (mn[c] <= mx[c]) { atomicMin(acc + EA_BOX_MIN + c, eval_ord(mn[c])); atomicMax(acc + EA_BOX_MAX + c, eval_ord(mx[c])); }
    }
}

__device__ __forceinline__ bool tri_touches(const float* p, const EvalBox& b) {
    for (int c = 0; c < 3; ++c) {
        const double lo = fminf(p[c], fminf(p[3 + c], p[6 + c])), hi = fmaxf(p[c], fmaxf(p[3 + c], p[6 + c]));
        if (hi < b.lo[c] || lo > b.hi[c]) return false;
    }
    return true;
}

// ---- 2. tile planning: samples of the triangles that touch the halo (n^2 each, an upper bound) and ground-truth points gathered
__global__ void __launch_bounds__(128) k_eval_plan(EvalGather g, const float* tp, const int* nsub, int nt, const float* gt, long long ngt, unsigned long long* acc) {
    unsigned long long s = 0, q = 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nt; i += stride) {
        const int ns = nsub[i];
        if (ns > 0 && tri_touches(tp + i * 9, g.halo)) s += (unsigned long long)ns * ns;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ngt; i += stride) q += in_gather(gt + i * 3, g);
    acc_add(acc, EA_PLAN_S, s);
    acc_add(acc, EA_PLAN_G, q);
}

// ---- 3. one tile
// one warp per triangle: its samples inside the halo, w = the triangle's sorted index when the sample lies in the tile (a query), else -1
__global__ void __launch_bounds__(128) k_eval_samples(const float* tp, const int* nsub, int nt, EvalBox tile, EvalBox halo, float4* out, int* out_n, int cap,
                                                       unsigned long long* acc) {
    const int lane = threadIdx.x & 31;
    const int w0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (int t = w0; t < nt; t += nw) {
        const int ns = nsub[t];
        if (ns == 0) continue;
        float p[9];
        for (int k = 0; k < 9; ++k) p[k] = tp[(size_t)t * 9 + k];
        if (!tri_touches(p, halo)) continue;
        const long long total = (long long)ns * ns;
        for (long long base = 0; base < total; base += 32) {
            const long long k = base + lane;
            float s[3] = {0, 0, 0};
            bool keep = false;
            if (k < total) {
                eval_sample(p, p + 3, p + 6, ns, k, s);
                keep = in_halo(s[0], s[1], s[2], halo);
            }
            const unsigned ballot = __ballot_sync(0xffffffffu, keep);
            if (!ballot) continue;
            int pos = 0;
            if (lane == 0) pos = atomicAdd(out_n, __popc(ballot));
            pos = __shfl_sync(0xffffffffu, pos, 0) + __popc(ballot & ((1u << lane) - 1u));
            if (keep) {
                if (pos < cap) out[pos] = make_float4(s[0], s[1], s[2], __int_as_float(in_box(s[0], s[1], s[2], tile) ? t : -1));
                else atomicAdd(acc + EA_OVERFLOW, 1ull);
            }
        }
    }
}
// ground truth as given (leaf == 0): the points inside the halo, w = 1 when in the tile (a query)
__global__ void __launch_bounds__(128) k_eval_gt_points(const float* gt, long long n, EvalGather g, EvalBox tile, float4* out, int* out_n, int cap, unsigned long long* acc) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float* p = gt + i * 3;
        if (!in_gather(p, g)) continue;
        const int pos = atomicAdd(out_n, 1);
        if (pos < cap) out[pos] = make_float4(p[0], p[1], p[2], __int_as_float(in_box(p[0], p[1], p[2], tile) ? 1 : 0));
        else atomicAdd(acc + EA_OVERFLOW, 1ull);
    }
}
// ground truth to down-sample (leaf > 0): the input indices of the points of the gathered leaves (key and value, to be sorted into input order)
__global__ void __launch_bounds__(128) k_eval_gt_idx(const float* gt, long long n, EvalGather g, unsigned* key, unsigned* val, int* out_n, int cap, unsigned long long* acc) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        if (!in_gather(gt + i * 3, g)) continue;
        const int pos = atomicAdd(out_n, 1);
        if (pos < cap) { key[pos] = (unsigned)i; val[pos] = (unsigned)i; }
        else atomicAdd(acc + EA_OVERFLOW, 1ull);
    }
}
// sort key of the leaf passes: the low (hi = 0) or high 32 bits of the packed leaf key of point sidx[perm[i]]; the value is perm[i]
__global__ void __launch_bounds__(128) k_eval_leaf_key(const float* gt, const unsigned* sidx, const unsigned* perm, int n, EvalGather g, int hi, unsigned* key, unsigned* val) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned s = perm ? perm[i] : (unsigned)i;
        const unsigned long long k = leaf_local_key(gt + (size_t)sidx[s] * 3, g);
        key[i] = hi ? (unsigned)(k >> 32) : (unsigned)k;
        val[i] = s;
    }
}
// one thread per leaf (the first of its run in leaf order): the sum of its points in input order, (float)(sum / count); w as k_eval_gt_points
__global__ void __launch_bounds__(128) k_eval_leaf_points(const float* gt, const unsigned* sidx, const unsigned* perm, int n, EvalGather g, EvalBox tile,
                                                           float4* out, int* out_n) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const unsigned long long k = leaf_local_key(gt + (size_t)sidx[perm[i]] * 3, g);
        if (i > 0 && leaf_local_key(gt + (size_t)sidx[perm[i - 1]] * 3, g) == k) continue;
        double s[3] = {0, 0, 0};
        int c = 0;
        for (int j = i; j < n; ++j) {
            const float* p = gt + (size_t)sidx[perm[j]] * 3;
            if (j > i && leaf_local_key(p, g) != k) break;
            s[0] += (double)p[0]; s[1] += (double)p[1]; s[2] += (double)p[2];
            ++c;
        }
        const float x = (float)(s[0] / c), y = (float)(s[1] / c), z = (float)(s[2] / c);
        out[atomicAdd(out_n, 1)] = make_float4(x, y, z, __int_as_float(in_box(x, y, z, tile) ? 1 : 0));
    }
}

// hashed uniform grid over a target set: cell key -> slot (count, end); points bucketed by slot
__device__ __forceinline__ unsigned long long grid_key(long long x, long long y, long long z) {
    return ((unsigned long long)x << (2 * EVAL_KEY_BITS)) | ((unsigned long long)y << EVAL_KEY_BITS) | (unsigned long long)z;
}
__device__ __forceinline__ long long grid_cell(float p, double org, double cell) { return (long long)floor(((double)p - org) / cell); }
__global__ void __launch_bounds__(128) k_eval_grid_insert(const float4* pts, int n, EvalGrid g, unsigned long long* keys, int* cnt, int* slot) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = pts[i];
        int created = 0;
        const int s = table_insert(keys, g.mask, grid_key(grid_cell(p.x, g.org[0], g.cell), grid_cell(p.y, g.org[1], g.cell), grid_cell(p.z, g.org[2], g.cell)), &created);
        slot[i] = s;
        atomicAdd(cnt + s, 1);
    }
}
__global__ void __launch_bounds__(128) k_eval_grid_start(const int* cnt, int cap, int* end, int* total) {
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += gridDim.x * blockDim.x)
        if (cnt[s] > 0) end[s] = atomicAdd(total, cnt[s]);
}
__global__ void __launch_bounds__(128) k_eval_grid_fill(const float4* pts, int n, const int* slot, int* end, float4* out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[atomicAdd(end + slot[i], 1)] = pts[i];
}
// exact nearest target within max_dist (ring search over the grid's cells; ring r >= 1 lies at least (r - 1) cell from the query,
// less 1 um for the rounding of the cell assignment); INFINITY when there is none
__device__ __forceinline__ double grid_nearest(const EvalGrid& g, float x, float y, float z, double max_dist) {
    double best = INFINITY;
    if (g.n == 0) return best;
    const long long cx = grid_cell(x, g.org[0], g.cell), cy = grid_cell(y, g.org[1], g.cell), cz = grid_cell(z, g.org[2], g.cell);
    const int rmax = (int)ceil(max_dist / g.cell) + 2;
    for (int r = 0; r <= rmax; ++r) {
        if (r >= 1) {
            const double lb = (double)(r - 1) * g.cell - 1e-6;
            if (best <= lb || lb > max_dist) break;
        }
        for (int dx = -r; dx <= r; ++dx) {
            const long long ix = cx + dx;
            if (ix < 0 || ix >= (1LL << EVAL_KEY_BITS)) continue;
            for (int dy = -r; dy <= r; ++dy) {
                const long long iy = cy + dy;
                if (iy < 0 || iy >= (1LL << EVAL_KEY_BITS)) continue;
                const bool shell = dx == -r || dx == r || dy == -r || dy == r;
                const int step = (shell || r == 0) ? 1 : 2 * r;
                for (int dz = -r; dz <= r; dz += step) {
                    const long long iz = cz + dz;
                    if (iz < 0 || iz >= (1LL << EVAL_KEY_BITS)) continue;
                    const int s = table_find(g.keys, g.mask, grid_key(ix, iy, iz));
                    if (s < 0) continue;
                    const int e = g.end[s];
                    for (int j = e - g.cnt[s]; j < e; ++j) {
                        const float4 p = g.pts[j];
                        const double d = eval_dist(x, y, z, p.x, p.y, p.z);
                        if (d < best) best = d;
                    }
                }
            }
        }
    }
    return best <= max_dist ? best : INFINITY;
}
// the queries of the tile (samples: w >= 0, the facet; ground truth: w == 1) against the other set's grid
__global__ void __launch_bounds__(128) k_eval_query(EvalGrid g, const float4* q, int nq, int samples, double threshold, double max_dist,
                                                     int* f_samples, int* f_far, unsigned long long* acc) {
    unsigned long long n = 0, within = 0, far = 0, qs = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += gridDim.x * blockDim.x) {
        const float4 p = q[i];
        const int w = __float_as_int(p.w);
        if (samples ? w < 0 : w != 1) continue;
        double d = grid_nearest(g, p.x, p.y, p.z, max_dist);
        if (d == INFINITY) { d = max_dist; ++far; }
        const bool in = d < threshold;
        ++n;
        within += in;
        qs += (unsigned long long)eval_quant(d);
        if (samples) {
            atomicAdd(f_samples + w, 1);
            if (!in) atomicAdd(f_far + w, 1);
        }
    }
    acc_add(acc, samples ? EA_SAMPLES : EA_GT, n);
    acc_add(acc, samples ? EA_S_WITHIN : EA_G_WITHIN, within);
    acc_add(acc, samples ? EA_S_FAR : EA_G_FAR, far);
    acc_add(acc, samples ? EA_S_Q : EA_G_Q, qs);
}
// ---- 4. facets: incorrect when n_far >= ratio n_samples (facets with samples), and the rows a b c n_samples n_far
__global__ void __launch_bounds__(128) k_eval_facets(const int4* st, const int* f_samples, const int* f_far, int n, double ratio, int* rows, unsigned long long* acc) {
    unsigned long long bad = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int ns = f_samples[i], nf = f_far[i];
        bad += ns > 0 && (double)nf >= ratio * (double)ns;
        if (rows) {
            const int4 t = st[i];
            int* r = rows + (size_t)i * 5;
            r[0] = t.x; r[1] = t.y; r[2] = t.z; r[3] = ns; r[4] = nf;
        }
    }
    acc_add(acc, EA_INCORRECT, bad);
}

// ---- host
struct Tile { EvalBox box; long long s, g; };

size_t pow2_ge(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}
size_t hist_ints(long long n) { return 256 * (size_t)std::max<long long>(1, (n + VG_TILE - 1) / VG_TILE); }
int eval_grid_dim(int n_sm, long long n, int threads) {
    const long long b = (n + threads - 1) / threads;
    return (int)std::max<long long>(1, std::min<long long>(b, (long long)n_sm * 8));
}

// buffers carved from one block at 256-byte alignment; a null base only counts the bytes (the same code sizes and places them)
struct Carve {
    char* base = nullptr;
    size_t off = 0;
    template <class T>
    void take(T*& p, size_t n) {
        off = (off + 255) & ~(size_t)255;
        if (base) p = reinterpret_cast<T*>(base + off);
        off += n * sizeof(T);
    }
};
// the per-call table: accumulators, counters, and per live triangle its record (mesh_tri_order's buffers), its triple in order,
// corners, subdivisions, fairness, per-facet counts and the rows
struct Table {
    unsigned long long* acc; int* d_n; double* fsum;
    TriOrder ord; int4* stri; float* tp; int* nsub; double* fair; int *f_s, *f_f; int* rows;
};
size_t table_carve(Carve& c, long long nt, bool rows, Table& T) {
    const size_t n1 = (size_t)std::max<long long>(nt, 1);
    c.take(T.acc, EA_SIZE); c.take(T.d_n, 8); c.take(T.fsum, 2);
    c.take(T.ord.rec, n1); c.take(T.stri, n1); c.take(T.tp, n1 * 9); c.take(T.nsub, n1); c.take(T.fair, n1 * 2); c.take(T.f_s, n1); c.take(T.f_f, n1);
    for (int b = 0; b < 2; ++b) { c.take(T.ord.k[b], n1); c.take(T.ord.v[b], n1); }
    c.take(T.ord.hist, hist_ints(nt));
    T.rows = nullptr;
    if (rows) c.take(T.rows, n1 * 5);
    return c.off;
}
// the scratch of one tile that gathers s samples and g ground-truth points: raw, bucketed and slot arrays and the hashed grid of each set,
// and with leaves the index / key sort of the gathered points
struct Scratch {
    float4* s_raw; float4* s_pts; int* s_slot; unsigned long long* s_keys; int* s_cnt; int* s_end;
    float4* g_raw; float4* g_pts; int* g_slot; unsigned long long* g_keys; int* g_cnt; int* g_end;
    unsigned *k[2], *v[2], *sidx; int* hist;
    size_t ms, mg, cs, cg;   // capacities: samples, points, grid slots of each set
};
size_t tile_carve(Carve& c, long long s, long long g, bool leaf, Scratch& S) {
    S.ms = (size_t)std::max<long long>(s, 1);
    S.mg = (size_t)std::max<long long>(g, 1);
    S.cs = pow2_ge(S.ms * 2);
    S.cg = pow2_ge(S.mg * 2);
    c.take(S.s_raw, S.ms); c.take(S.s_pts, S.ms); c.take(S.s_slot, S.ms); c.take(S.s_keys, S.cs); c.take(S.s_cnt, S.cs); c.take(S.s_end, S.cs);
    c.take(S.g_raw, S.mg); c.take(S.g_pts, S.mg); c.take(S.g_slot, S.mg); c.take(S.g_keys, S.cg); c.take(S.g_cnt, S.cg); c.take(S.g_end, S.cg);
    if (leaf) {
        for (int b = 0; b < 2; ++b) { c.take(S.k[b], S.mg); c.take(S.v[b], S.mg); }
        c.take(S.sidx, S.mg);
        c.take(S.hist, hist_ints(g));
    }
    return c.off;
}
size_t tile_bytes(long long s, long long g, bool leaf) {
    Carve c;
    Scratch S;
    return tile_carve(c, s, g, leaf, S);
}

// what the last immesh_mesh_evaluate of this thread did (immesh_mesh_evaluate_stats)
thread_local int64_t eval_stats[4] = {0, 0, 0, 0};

}  // namespace

int immesh_mesh_evaluate(immesh_mesh_t* h, const float* gt_xyz, int64_t n_gt, int on_device, const immesh_eval_config* cfg, int64_t* counts,
                         double* metrics, int32_t* facet_rows, int64_t cap_rows, int64_t* n_rows) {
    if (!h || !cfg || !counts || !metrics) return im_fail(IMMESH_E_INVALID, "evaluate: null handle, cfg, counts or metrics");
    const double spacing = cfg->sample_spacing, leaf = cfg->gt_leaf, thr = cfg->threshold, md = cfg->max_dist, ratio = cfg->incorrect_ratio;
    if (!(spacing > 0) || !std::isfinite(spacing)) return im_fail(IMMESH_E_INVALID, "evaluate: sample_spacing must be finite and > 0");
    if (!(leaf >= 0) || !std::isfinite(leaf)) return im_fail(IMMESH_E_INVALID, "evaluate: gt_leaf must be finite and >= 0");
    if (!(thr > 0) || !(md >= thr) || !(md <= 1024)) return im_fail(IMMESH_E_INVALID, "evaluate: need 0 < threshold <= max_dist <= 1024");
    if (!(ratio > 0) || !(ratio <= 1)) return im_fail(IMMESH_E_INVALID, "evaluate: incorrect_ratio must be in (0, 1]");
    if (cfg->positions != 0 && cfg->positions != 1) return im_fail(IMMESH_E_INVALID, "evaluate: positions must be 0 (raw) or 1 (smoothed)");
    if (cfg->max_batch_bytes < 0) return im_fail(IMMESH_E_INVALID, "evaluate: max_batch_bytes must be >= 0");
    if (n_gt < 0 || (n_gt > 0 && !gt_xyz) || (on_device != 0 && on_device != 1) || cap_rows < 0)
        return im_fail(IMMESH_E_INVALID, "evaluate: bad ground-truth arguments or cap_rows");
    if (n_gt > 0x7fffffffLL) return im_fail(IMMESH_E_RANGE, "evaluate: more than 2^31 - 1 ground-truth points in one call");
    if (h->F.shard_n > 1) return im_fail(IMMESH_E_INVALID, "evaluate: a sharded handle");
    for (int64_t& v : eval_stats) v = 0;

    IM_CUDA(cudaStreamSynchronize(h->stream));   // everything queued on the handle, the pipelined frames included
    cudaStream_t st = h->stream;
    int mc[IM_MC_HOST];
    IM_CUDA(cudaMemcpy(mc, h->M.cnt, sizeof(mc), cudaMemcpyDeviceToHost));
    const int nt = mc[IM_MC_TRIS_LIVE];
    if (n_rows) *n_rows = nt;
    if (facet_rows && cap_rows < nt) return im_fail(IMMESH_E_CAPACITY, "evaluate: cap_rows is below the live triangle count (*n_rows)");

    const size_t budget = cfg->max_batch_bytes ? (size_t)cfg->max_batch_bytes : ((size_t)2 << 30);
    Table T = {};
    Carve tc;
    const size_t tb = table_carve(tc, nt, facet_rows != nullptr, T);
    if (tb > budget)
        return im_fail(IMMESH_E_CAPACITY, ("evaluate: the table of the " + std::to_string(nt) + " live triangles needs " + std::to_string(tb) +
                                           " bytes, above max_batch_bytes").c_str());
    eval_stats[3] = (int64_t)tb;
    const int nsm = h->n_sm;
    MemSet mem;
    tc.off = 0;
    IM_CUDA(mem.alloc(&tc.base, tb));
    table_carve(tc, nt, facet_rows != nullptr, T);
    unsigned long long* acc = T.acc;
    int* d_n = T.d_n;
    {   // every fill on the call's stream, ordered before the kernels that use the buffers
        std::vector<unsigned long long> a0(EA_SIZE, 0);
        for (int c = 0; c < 3; ++c) a0[EA_BOX_MIN + c] = ~0ull;
        IM_CUDA(cudaMemcpyAsync(acc, a0.data(), EA_SIZE * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
        IM_CUDA(cudaMemsetAsync(d_n, 0, 8 * sizeof(int), st));
        IM_CUDA(cudaMemsetAsync(T.fsum, 0, 2 * sizeof(double), st));
        IM_CUDA(cudaMemsetAsync(T.f_s, 0, (size_t)std::max(nt, 1) * sizeof(int), st));
        IM_CUDA(cudaMemsetAsync(T.f_f, 0, (size_t)std::max(nt, 1) * sizeof(int), st));
    }

    // 1. live triangles in triple order (mesh_tri_order, with the table's buffers)
    if (nt > 0) {
        T.ord.cap = nt;
        T.ord.misc = d_n;
        if (const int rc = mesh_tri_order(h, mc, 0.0, T.ord)) return rc;
        IM_LAUNCH(k_eval_tri, eval_grid_dim(nsm, nt, 128), 128, 0, st, h->M, cfg->positions, (const int4*)T.ord.rec, T.ord.order, nt, spacing, T.stri,
                  T.tp, T.nsub, T.fair, acc);
        IM_LAUNCH(k_eval_fair_sum, 1, 1024, 0, st, (const double*)T.fair, nt, T.fsum);
    }
    // the ground truth, read in place or copied once (outside the budget)
    const float* gt = gt_xyz;
    if (n_gt > 0 && !on_device) {
        float* d = nullptr;
        IM_CUDA(mem.alloc(&d, (size_t)n_gt * 3));
        IM_CUDA(cudaMemcpyAsync(d, gt_xyz, (size_t)n_gt * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
        gt = d;
    }
    if (n_gt > 0) IM_LAUNCH(k_eval_gt_scan, eval_grid_dim(nsm, n_gt, 128), 128, 0, st, gt, (long long)n_gt, acc);
    IM_CUDA(cudaGetLastError());
    unsigned long long a[EA_SIZE];
    IM_CUDA(cudaMemcpyAsync(a, acc, sizeof(a), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (a[EA_UNSMOOTHED]) return im_fail(IMMESH_E_INVALID, "evaluate: positions = 1 with unsmoothed vertices in live triangles: smooth first (immesh_mesh_smooth_all)");
    if (a[EA_NONFINITE]) return im_fail(IMMESH_E_INVALID, "evaluate: a ground-truth point is not finite");
    if (a[EA_N_RANGE]) return im_fail(IMMESH_E_RANGE, "evaluate: a triangle needs more than 2^15 subdivisions at this sample_spacing");
    if (a[EA_SUM_N2] > (1ull << 33)) return im_fail(IMMESH_E_RANGE, "evaluate: more than 2^33 samples");

    // 2. tiles: bisect the bounding box until a tile's scratch fits what the table leaves of the budget
    const bool use_leaf = leaf > 0;
    const double cell = std::max({thr / 2, 2 * spacing, 2 * leaf, md / 16});
    const double min_side = std::max(md / 4, 2 * cell);   // a tile is not halved below this side (its halo would dominate)
    const size_t avail = budget - tb;
    std::vector<Tile> tiles;
    size_t arena = 0;
    const bool any = nt > 0 || n_gt > 0;
    double amax = 0;
    // what the tile `b` gathers: its box grown by max_dist and a pad beyond the float rounding of a sample at this scale
    auto gather_of = [&](const EvalBox& b) {
        const double pad = 1e-3 + amax * std::ldexp(1.0, -20);
        EvalGather g;
        g.leaf = leaf;
        for (int c = 0; c < 3; ++c) {
            g.halo.lo[c] = b.lo[c] - md - pad;
            g.halo.hi[c] = b.hi[c] + md + pad;
            g.klo[c] = use_leaf ? (long long)std::floor(g.halo.lo[c] / leaf) : 0;
            g.khi[c] = use_leaf ? (long long)std::floor(g.halo.hi[c] / leaf) : 0;
        }
        return g;
    };
    // the largest extent, in cells and in leaves, that the packed keys of a tile with this box must span
    auto keys_fit = [&](double side) {
        const double ext = side + 2 * (md + 1e-3 + amax * std::ldexp(1.0, -20)) + 2 * leaf + 2 * cell;
        return ext / cell < (double)EVAL_KEY_SPAN && (!use_leaf || ext / leaf < (double)EVAL_KEY_SPAN);
    };
    if (any && a[EA_BOX_MIN] != ~0ull) {
        double bmin[3], bmax[3];
        for (int c = 0; c < 3; ++c) {
            bmin[c] = eval_unord(a[EA_BOX_MIN + c]);
            bmax[c] = eval_unord(a[EA_BOX_MAX + c]);
            amax = std::max({amax, std::fabs(bmin[c]), std::fabs(bmax[c])});
        }
        if (!keys_fit(min_side)) {
            char msg[320];
            std::snprintf(msg, sizeof(msg), "evaluate: even the smallest tile (side %.4g m, halo %.4g m, coordinates up to %.4g m) spans more than 2^21 - 4 "
                          "grid cells (%.4g m) or ground-truth leaves (%.4g m) per axis: raise gt_leaf or lower max_dist", min_side, md, amax, cell, leaf);
            return im_fail(IMMESH_E_RANGE, msg);
        }
        std::vector<EvalBox> stack(1);
        for (int c = 0; c < 3; ++c) { stack[0].lo[c] = bmin[c] - 1.0; stack[0].hi[c] = bmax[c] + 1.0; }
        while (!stack.empty()) {
            const EvalBox b = stack.back();
            stack.pop_back();
            double side = 0;
            for (int c = 0; c < 3; ++c) side = std::max(side, b.hi[c] - b.lo[c]);
            // a box above the smallest side is halved until its keys fit and it fits the budget; keys_fit(min_side) holds (checked above),
            // so every box at the smallest side is counted and either taken or refused: the bisection ends
            const bool small = side <= min_side;
            unsigned long long sg[2] = {0, 0};
            if (small || keys_fit(side)) {
                IM_CUDA(cudaMemsetAsync(acc + EA_PLAN_S, 0, 2 * sizeof(unsigned long long), st));
                IM_LAUNCH(k_eval_plan, eval_grid_dim(nsm, std::max<long long>(nt, n_gt), 128), 128, 0, st, gather_of(b), (const float*)T.tp, (const int*)T.nsub, nt, gt,
                          (long long)n_gt, acc);
                IM_CUDA(cudaMemcpyAsync(sg, acc + EA_PLAN_S, sizeof(sg), cudaMemcpyDeviceToHost, st));
                IM_CUDA(cudaStreamSynchronize(st));
                ++eval_stats[1];
                if (sg[0] == 0 && sg[1] == 0) continue;
                const size_t bytes = tile_bytes((long long)sg[0], (long long)sg[1], use_leaf);
                if (sg[0] < (1ull << 30) && sg[1] < (1ull << 30) && bytes <= avail) {
                    tiles.push_back({b, (long long)sg[0], (long long)sg[1]});
                    arena = std::max(arena, bytes);
                    continue;
                }
                if (small) {
                    char msg[320];
                    std::snprintf(msg, sizeof(msg), "evaluate: max_batch_bytes too small: a tile of side %.4g m with its %.4g m halo gathers %llu samples (upper bound) and "
                                  "%llu ground-truth points, %zu bytes (the triangle table takes %zu)", side, md, sg[0], sg[1], bytes, tb);
                    return im_fail(IMMESH_E_CAPACITY, msg);
                }
            }
            int ax = 0;
            for (int c = 1; c < 3; ++c) if (b.hi[c] - b.lo[c] > b.hi[ax] - b.lo[ax]) ax = c;
            const double mid = 0.5 * (b.lo[ax] + b.hi[ax]);
            EvalBox l = b, r = b;
            l.hi[ax] = mid;
            r.lo[ax] = mid;
            stack.push_back(r);
            stack.push_back(l);
        }
    }
    eval_stats[0] = (int64_t)tiles.size();
    eval_stats[2] = (int64_t)(tb + arena);

    // 3. the tiles, one at a time in one block of the largest tile's size (table + block <= max_batch_bytes)
    if (!tiles.empty()) {
        Carve ac;
        IM_CUDA(mem.alloc(&ac.base, arena));
        for (const Tile& t : tiles) {
            Scratch S;
            ac.off = 0;
            tile_carve(ac, t.s, t.g, use_leaf, S);
            const size_t ms = S.ms, mg = S.mg, cs = S.cs, cg = S.cg;
            const EvalGather g = gather_of(t.box);
            IM_CUDA(cudaMemsetAsync(d_n, 0, 8 * sizeof(int), st));   // 0 samples, 1 gathered indices, 2 ground-truth points, 3 / 4 grid totals
            if (t.s > 0) IM_LAUNCH(k_eval_samples, eval_grid_dim(nsm, (long long)nt * 32, 128), 128, 0, st, (const float*)T.tp, (const int*)T.nsub, nt, t.box, g.halo, S.s_raw, d_n,
                                   (int)ms, acc);
            if (t.g > 0 && !use_leaf) IM_LAUNCH(k_eval_gt_points, eval_grid_dim(nsm, n_gt, 128), 128, 0, st, gt, (long long)n_gt, g, t.box, S.g_raw, d_n + 2, (int)mg, acc);
            if (t.g > 0 && use_leaf) IM_LAUNCH(k_eval_gt_idx, eval_grid_dim(nsm, n_gt, 128), 128, 0, st, gt, (long long)n_gt, g, S.k[0], S.v[0], d_n + 1, (int)mg, acc);
            int hn[3];
            IM_CUDA(cudaMemcpyAsync(hn, d_n, sizeof(hn), cudaMemcpyDeviceToHost, st));
            IM_CUDA(cudaStreamSynchronize(st));
            const int ns = std::min(hn[0], (int)ms);
            int ng = std::min(hn[2], (int)mg);
            if (use_leaf && hn[1] > 0) {
                // input order, then leaf order (stable passes on the low and the high 32 bits of the packed key), then one thread per leaf
                const int ni = std::min(hn[1], (int)mg);
                int cur = rs_sort_passes(st, S.k, S.v, 0, ni, 4, S.hist);
                IM_CUDA(cudaMemcpyAsync(S.sidx, S.v[cur], (size_t)ni * sizeof(unsigned), cudaMemcpyDeviceToDevice, st));
                IM_LAUNCH(k_eval_leaf_key, eval_grid_dim(nsm, ni, 128), 128, 0, st, gt, (const unsigned*)S.sidx, (const unsigned*)nullptr, ni, g, 0, S.k[0], S.v[0]);
                cur = rs_sort_passes(st, S.k, S.v, 0, ni, 4, S.hist);
                IM_LAUNCH(k_eval_leaf_key, eval_grid_dim(nsm, ni, 128), 128, 0, st, gt, (const unsigned*)S.sidx, (const unsigned*)S.v[cur], ni, g, 1, S.k[cur ^ 1], S.v[cur ^ 1]);
                cur = rs_sort_passes(st, S.k, S.v, cur ^ 1, ni, 4, S.hist);
                IM_LAUNCH(k_eval_leaf_points, eval_grid_dim(nsm, ni, 128), 128, 0, st, gt, (const unsigned*)S.sidx, (const unsigned*)S.v[cur], ni, g, t.box, S.g_raw, d_n + 2);
                IM_CUDA(cudaMemcpyAsync(hn + 2, d_n + 2, sizeof(int), cudaMemcpyDeviceToHost, st));
                IM_CUDA(cudaStreamSynchronize(st));
                ng = hn[2];
            }
            // the two grids, then each set's queries against the other's grid
            EvalGrid gs = {}, gg = {};
            struct Build { EvalGrid* G; const float4* raw; float4* pts; int* slot; unsigned long long* keys; int* cnt; int* end; size_t cap; int n; int* total; };
            Build bl[2] = {{&gs, S.s_raw, S.s_pts, S.s_slot, S.s_keys, S.s_cnt, S.s_end, cs, ns, d_n + 3}, {&gg, S.g_raw, S.g_pts, S.g_slot, S.g_keys, S.g_cnt, S.g_end, cg, ng, d_n + 4}};
            for (Build& b : bl) {
                EvalGrid& G = *b.G;
                G.n = b.n;
                G.cell = cell;
                for (int c = 0; c < 3; ++c) G.org[c] = g.halo.lo[c] - leaf - cell;   // a gathered leaf's point lies at most one leaf outside the halo
                if (b.n == 0) continue;
                const size_t cap = std::min(b.cap, pow2_ge((size_t)b.n * 2));
                G.mask = (unsigned int)(cap - 1);
                G.keys = b.keys; G.cnt = b.cnt; G.end = b.end; G.pts = b.pts;
                IM_CUDA(cudaMemsetAsync(b.keys, 0xff, cap * sizeof(unsigned long long), st));
                IM_CUDA(cudaMemsetAsync(b.cnt, 0, cap * sizeof(int), st));
                IM_LAUNCH(k_eval_grid_insert, eval_grid_dim(nsm, b.n, 128), 128, 0, st, (const float4*)b.raw, b.n, G, b.keys, b.cnt, b.slot);
                IM_LAUNCH(k_eval_grid_start, eval_grid_dim(nsm, (long long)cap, 128), 128, 0, st, (const int*)b.cnt, (int)cap, b.end, b.total);
                IM_LAUNCH(k_eval_grid_fill, eval_grid_dim(nsm, b.n, 128), 128, 0, st, (const float4*)b.raw, b.n, (const int*)b.slot, b.end, b.pts);
            }
            if (ns > 0) IM_LAUNCH(k_eval_query, eval_grid_dim(nsm, ns, 128), 128, 0, st, gg, (const float4*)S.s_raw, ns, 1, thr, md, T.f_s, T.f_f, acc);
            if (ng > 0) IM_LAUNCH(k_eval_query, eval_grid_dim(nsm, ng, 128), 128, 0, st, gs, (const float4*)S.g_raw, ng, 0, thr, md, T.f_s, T.f_f, acc);
            IM_CUDA(cudaGetLastError());
        }
    }

    // 4. facets, rows and the results
    if (nt > 0) IM_LAUNCH(k_eval_facets, eval_grid_dim(nsm, nt, 128), 128, 0, st, (const int4*)T.stri, (const int*)T.f_s, (const int*)T.f_f, nt, ratio, T.rows, acc);
    IM_CUDA(cudaGetLastError());
    double fs[2] = {0, 0};
    IM_CUDA(cudaMemcpyAsync(a, acc, sizeof(a), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaMemcpyAsync(fs, T.fsum, sizeof(fs), cudaMemcpyDeviceToHost, st));
    if (facet_rows && nt > 0) IM_CUDA(cudaMemcpyAsync(facet_rows, T.rows, (size_t)nt * 5 * sizeof(int), cudaMemcpyDeviceToHost, st));
    IM_CUDA(cudaStreamSynchronize(st));
    if (a[EA_OVERFLOW]) return im_fail(IMMESH_E_CUDA, "evaluate: a tile gathered more than its plan (internal error)");
    const long long live = nt, deg = (long long)a[EA_DEGENERATE], ns = (long long)a[EA_SAMPLES], ng = (long long)a[EA_GT];
    const long long c[12] = {live, deg, ns, ng, (long long)a[EA_S_WITHIN], (long long)a[EA_G_WITHIN], (long long)a[EA_S_FAR], (long long)a[EA_G_FAR],
                             (long long)a[EA_INCORRECT], (long long)a[EA_S_Q], (long long)a[EA_G_Q], (long long)a[EA_N_MAX]};
    for (int i = 0; i < 12; ++i) counts[i] = c[i];
    eval_metrics(c, fs[0], fs[1], metrics);
    return IMMESH_OK;
}

int immesh_mesh_evaluate_stats(int64_t* out) {
    if (!out) return im_fail(IMMESH_E_INVALID, "evaluate_stats: null out");
    for (int i = 0; i < 4; ++i) out[i] = eval_stats[i];
    return IMMESH_OK;
}
