// immesh_b200 -- device-resident VoxelMap: open-addressed root-voxel hash, pooled adaptive
// octree nodes, probabilistic plane records, chunked per-node point storage, and the three
// operations of the localization path on it: point-to-plane residual selection, plane fit,
// and order-preserving incremental update.
//
// Reference semantics being reproduced (all /root/reference):
//   key rule            src/voxel_mapping.cpp:118-127 (insert, float voxel_size), :172-181 (lookup, double)
//   OctoTree / Plane    src/voxel_loc.hpp:89-177
//   init_plane          src/voxel_loc.cpp:47-139
//   init/cut/Update     src/voxel_loc.cpp:141-308
//   build_single_residual / BuildResidualListOMP   src/voxel_mapping.cpp:153-318
//
// Layout in HBM (struct-of-pools, index-linked, no pointers):
//   keys[cap] u64 + root_node[cap] i32        open addressing, linear probing, 16 B / slot pair
//   NodeRec[max_nodes]  176 B                 children, voxel centre, counters, chunk list head/tail, running point sums
//   PlaneRec[max_nodes]  256 B (2 x 128 B lines, first line = everything the residual range test reads)
//   Chunk[max_chunks]    512 B                8 points SoA: xyz f32 + symmetric covariance 6 x f64
// Work decomposition: residual selection = 1 thread / scan point (read-only map); update =
// 1 warp / touched root voxel, points applied in the reference's sorted order inside the voxel,
// plane refits parallel over the 21 covariance entries (never across a sum: bit-reproducible).
#pragma once
#include "hd_math.cuh"

#if defined(__CUDA_ARCH__)
#define IM_SYNCWARP() __syncwarp()
#define IM_BCAST_I(x) __shfl_sync(0xffffffffu, (x), 0)
#else
#define IM_SYNCWARP()
#define IM_BCAST_I(x) (x)
#endif
// Predicates of the per-node state machine are evaluated by every lane on data that only lane 0 writes, always behind a warp
// barrier.  (Taking lane 0's value through a shuffle instead was tried and changed results -- tools/debug/lio_diff.py -- so the
// per-lane evaluation, validated bit for bit against the oracle, stays.)
#define IM_UPRED(x) (x)

namespace immesh {

struct LioParams {
    double voxel_size;      // lookup rule divides by the double
    double voxel_size_ins;  // insert rule divides by (double)(float)voxel_size
    float voxel_size_f;
    int max_layer;
    int layer_init[5];
    int max_points;
    float planer_threshold;
    float dept_err;
    double dir_var, dir_var_calib;
    int calib_laser;
    int max_iter;
    double extR[9], extT[3];
    int shard_rank, shard_n;   // multi-GPU: this rank owns the root voxels with voxel_owner(key) == shard_rank (1 rank: owns all)
};

struct alignas(16) PlaneRec {
    double center[3];   //   0
    double normal[3];   //  24
    float d;            //  48
    float radius;       //  52
    float min_eig;      //  56
    int is_plane;       //  60
    double pv[21];      //  64 .. 232   upper triangle of the 6x6 plane covariance
    int points_size;    // 232
    int plane_inited;   // 236
    int pad_[4];        // 240 .. 256
};
struct alignas(16) NodeRec {
    int children[8];
    double vc[3];
    float quater;
    int layer;
    int n_pts;
    int new_points;
    int first_chunk;
    int last_chunk;
    int init_octo;
    int update_enable;
    int octo_state;
    int root_slot;
    double sum_p[3];   // running sum of the stored points, in append order (= the reference's loop order in init_plane)
    double sum_pp[6];  // running sum of p p^T, upper triangle
    double pad_;
    // Running moments of the stored points' covariances about the node's FIXED voxel centre, q = p - vc, in append order:
    //   mq[p*6+s]      = sum_i q_j q_k Sigma_i[s]   p = pair (j<=k) in the order 00 01 02 11 12 22, s = symmetric 3x3 index
    //   mq[36+j*6+s]   = sum_i q_j Sigma_i[s]
    //   mq[54+s]       = sum_i Sigma_i[s]
    // plane_var = sum_i J_i Sigma_i J_i^T with J_i linear in (p_i - c) is a fixed contraction of these 60 sums (init_plane): a
    // refit costs O(1) instead of a pass over all stored points (the reference recomputes from every stored point on each of
    // its refits, voxel_loc.cpp:76-121: O(n^2/5) per node lifetime, ~4 ms per KITTI-shape scan on this GPU before).
    double mq[60];
};
struct alignas(16) Chunk {
    float x[8], y[8], z[8];
    int next;
    int pad_[7];
    double var[6][8];
};
// What the plane-map publisher (pubPlaneMap, voxel_mapping.cpp:947-1159) reads besides the plane record, kept out of PlaneRec so
// that the record's first 128-B line stays what k_match reads.
struct alignas(16) PubRec {
    float p_center[3];   // Plane::m_p_center x y z: the centre of the last PLANAR fit (voxel_loc.cpp:111-113), zero until there is one
    float p_normal[3];   // m_p_center.normal_x/y/z, same rule (:114-116)
    int updated;         // Plane::m_is_update: set by every fit, planar or not (:118, :136), cleared when the plane is published
    int pad_;
};
static_assert(sizeof(PlaneRec) == 256, "PlaneRec must be 256 B");
static_assert(sizeof(NodeRec) == 656, "NodeRec must be 656 B");
static_assert(sizeof(Chunk) == 512, "Chunk must be 512 B");
static_assert(sizeof(PubRec) == 32, "PubRec must be 32 B");

enum : int {
    IM_ERR_KEY_RANGE = 1,
    IM_ERR_NODE_POOL = 2,
    IM_ERR_CHUNK_POOL = 4,
    IM_ERR_HASH_FULL = 8,
    IM_ERR_FX_RANGE = 16,
    IM_ERR_SEG_POOL = 32,
    IM_ERR_PEER_TIMEOUT = 64,   // sharded mode: a peer rank's epoch flag did not arrive (peer_win.cuh)
    IM_ERR_IMU_CARRY = 128,     // immesh_lio_step_async_depth_imu: carried + own IMU samples exceeded max_imu (the frame's samples dropped)
};

struct VoxelMapDev {
    unsigned long long* keys;
    int* root_node;
    unsigned int cap_mask;
    NodeRec* nodes;
    PlaneRec* planes;
    int* node_count;
    int max_nodes;
    Chunk* chunks;
    int* chunk_bump;
    int max_chunks;
    int* avail;
    int* avail_top;
    int* pending;
    int* pending_n;
    int* err;
    int* n_roots;
    int* stat;   // optional work counters of the current scan: [0] plane refits, [1] points read by them (roofline byte model); may be null
    // plane-map publication: per node PubRec; per hash slot a "pending" mark, and the list of marked slots (pub_n entries).  A root
    // is marked by the first fit under it after it left the list; the publication walk visits only the listed roots.  pub == null:
    // a map without the publisher (the library always allocates it; the host emulation of the other entry points does not).
    PubRec* pub;
    int* pub_mark;
    int* pub_list;
    int* pub_n;
    // local map (local_map.cuh): node ids freed by the eviction of root voxels, popped by alloc_node before it bumps node_count.
    // node_free == null: nothing was ever evicted from this map (alloc_node only bumps); n_tombs counts the tombstones in the table.
    int* node_free;
    int* node_free_top;
    int* n_tombs;
};

#define IM_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
// a root voxel evicted by the local map: bit 63 set (pack_key never sets it), not IM_EMPTY_KEY; never matches a key, never claimed
#define IM_TOMB_KEY 0x8000000000000000ull

// ------------------------------------------------------------------ atomics (plain ops in the host emulation)
IM_HD int im_atomic_add(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    const int o = *p; *p = o + v; return o;
#endif
}
IM_HD int im_atomic_or(int* p, int v) {
#if defined(__CUDA_ARCH__)
    return atomicOr(p, v);
#else
    const int o = *p; *p = o | v; return o;
#endif
}
IM_HD unsigned long long im_atomic_cas64(unsigned long long* p, unsigned long long cmp, unsigned long long val) {
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, cmp, val);
#else
    const unsigned long long o = *p; if (o == cmp) *p = val; return o;
#endif
}

// ------------------------------------------------------------------ keys + hash
IM_HD bool voxel_key3(const double* p, double vs, long long* k) {
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float loc = (float)(p[j] / vs);
        if (loc < 0) loc = (float)((double)loc - 1.0);
        k[j] = (long long)loc;
        if (!(loc > -1048000.0f && loc < 1048000.0f)) ok = false;
    }
    return ok;
}
IM_HD bool voxel_key3_loc(const double* p, double vs, long long* k, float* loc_out) {
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float loc = (float)(p[j] / vs);
        if (loc < 0) loc = (float)((double)loc - 1.0);
        loc_out[j] = loc;
        k[j] = (long long)loc;
        if (!(loc > -1048000.0f && loc < 1048000.0f)) ok = false;
    }
    return ok;
}
IM_HD unsigned long long pack_key(long long x, long long y, long long z) {
    return ((unsigned long long)(x + 1048576) << 42) | ((unsigned long long)(y + 1048576) << 21) | (unsigned long long)(z + 1048576);
}
IM_HD void unpack_key(unsigned long long k, long long* x, long long* y, long long* z) {
    *x = (long long)((k >> 42) & 0x1FFFFF) - 1048576;
    *y = (long long)((k >> 21) & 0x1FFFFF) - 1048576;
    *z = (long long)(k & 0x1FFFFF) - 1048576;
}
IM_HD unsigned int hash_key(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned int)k;
}
// owner rank of a root voxel when the VoxelMap is sharded over n ranks (bits independent of the table hash)
IM_HD int voxel_owner(unsigned long long key, int n) {
    return (int)((unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 40) % (unsigned int)n);
}
IM_HD int hash_find(const VoxelMapDev& m, unsigned long long key) {
    unsigned int s = hash_key(key) & m.cap_mask;
    for (unsigned int probe = 0; probe <= m.cap_mask; ++probe) {
        const unsigned long long k = m.keys[s];
        if (k == key) return (int)s;
        if (k == IM_EMPTY_KEY) return -1;
        s = (s + 1) & m.cap_mask;
    }
    return -1;
}
// returns slot; *created = 1 for the thread that claimed an empty slot
IM_HD int hash_insert(const VoxelMapDev& m, unsigned long long key, int* created) {
    unsigned int s = hash_key(key) & m.cap_mask;
    *created = 0;
    for (unsigned int probe = 0; probe <= m.cap_mask; ++probe) {
        unsigned long long k = m.keys[s];
        if (k == key) return (int)s;
        if (k == IM_EMPTY_KEY) {
            k = im_atomic_cas64(&m.keys[s], IM_EMPTY_KEY, key);
            if (k == IM_EMPTY_KEY) { *created = 1; return (int)s; }
            if (k == key) return (int)s;
        }
        s = (s + 1) & m.cap_mask;
    }
    im_atomic_or(m.err, IM_ERR_HASH_FULL);
    return -1;
}

// ------------------------------------------------------------------ pools
IM_HD int alloc_node(const VoxelMapDev& m) {
    if (m.node_free) {   // node records freed by an eviction first, as alloc_chunk takes recycled chunks first
        const int i = im_atomic_add(m.node_free_top, -1) - 1;
        if (i >= 0) return m.node_free[i];
    }
    const int id = im_atomic_add(m.node_count, 1);
    if (id >= m.max_nodes) { im_atomic_or(m.err, IM_ERR_NODE_POOL); return -1; }
    return id;
}
IM_HD int alloc_chunk(const VoxelMapDev& m) {
    const int i = im_atomic_add(m.avail_top, -1) - 1;
    if (i >= 0) return m.avail[i];
    const int id = im_atomic_add(m.chunk_bump, 1);
    if (id >= m.max_chunks) { im_atomic_or(m.err, IM_ERR_CHUNK_POOL); return -1; }
    return id;
}
IM_HD void init_node(const VoxelMapDev& m, int id, int layer, const double* vc, float quater, int root_slot) {
    NodeRec& n = m.nodes[id];
    for (int i = 0; i < 8; ++i) n.children[i] = -1;
    n.vc[0] = vc[0]; n.vc[1] = vc[1]; n.vc[2] = vc[2];
    n.quater = quater;
    n.layer = layer;
    n.n_pts = 0;
    n.new_points = 0;
    n.first_chunk = -1;
    n.last_chunk = -1;
    n.init_octo = 0;
    n.update_enable = 1;
    n.octo_state = 0;
    n.root_slot = root_slot;
    for (int i = 0; i < 3; ++i) n.sum_p[i] = 0.0;
    for (int i = 0; i < 6; ++i) n.sum_pp[i] = 0.0;
    for (int i = 0; i < 60; ++i) n.mq[i] = 0.0;
    PlaneRec& p = m.planes[id];
    p.center[0] = p.center[1] = p.center[2] = 0.0;
    p.normal[0] = p.normal[1] = p.normal[2] = 0.0;
    p.d = 0.f; p.radius = 0.f; p.min_eig = 1.f; p.is_plane = 0;
    for (int i = 0; i < 21; ++i) p.pv[i] = 0.0;
    p.points_size = 0;
    p.plane_inited = 0;
    if (m.pub) {
        PubRec& q = m.pub[id];
        for (int i = 0; i < 3; ++i) { q.p_center[i] = 0.f; q.p_normal[i] = 0.f; }
        q.updated = 0;
    }
}
// new root voxel, voxel_mapping.cpp:136-141 / :345-350
IM_HD int make_root(const VoxelMapDev& m, const LioParams& P, unsigned long long key, int slot) {
    const int id = alloc_node(m);
    if (id < 0) return -1;
    long long kx, ky, kz;
    unpack_key(key, &kx, &ky, &kz);
    const double vc[3] = {(0.5 + (double)kx) * (double)P.voxel_size_f, (0.5 + (double)ky) * (double)P.voxel_size_f, (0.5 + (double)kz) * (double)P.voxel_size_f};
    init_node(m, id, 0, vc, P.voxel_size_f / 4, slot);
    return id;
}

// one point of a node (single-lane helper; callers guard with lane == 0)
IM_HD void node_append(const VoxelMapDev& m, int nd, float x, float y, float z, const double* var6) {
    NodeRec& n = m.nodes[nd];
    const int pos = n.n_pts;
    const int slot = pos & 7;
    int ch = n.last_chunk;
    if (slot == 0) {
        const int nc = alloc_chunk(m);
        if (nc < 0) return;
        m.chunks[nc].next = -1;
        if (ch >= 0) m.chunks[ch].next = nc; else n.first_chunk = nc;
        n.last_chunk = nc;
        ch = nc;
    }
    Chunk& c = m.chunks[ch];
    c.x[slot] = x; c.y[slot] = y; c.z[slot] = z;
    for (int k = 0; k < 6; ++k) c.var[k][slot] = var6[k];
    n.n_pts = pos + 1;
    const double dx = (double)x, dy = (double)y, dz = (double)z;
    n.sum_pp[0] += dx * dx; n.sum_pp[1] += dx * dy; n.sum_pp[2] += dx * dz;
    n.sum_pp[3] += dy * dy; n.sum_pp[4] += dy * dz; n.sum_pp[5] += dz * dz;
    n.sum_p[0] += dx; n.sum_p[1] += dy; n.sum_p[2] += dz;
}
// moment update of an appended point, spread over the lanes (entry e of 60 by lane e % nlanes); call with all lanes, right
// next to the lane-0 node_append of the same point
IM_HDN inline void node_moments_add(const VoxelMapDev& m, int nd, float x, float y, float z, const double* var6, int lane, int nlanes) {
    NodeRec& n = m.nodes[nd];
    const double q[3] = {(double)x - n.vc[0], (double)y - n.vc[1], (double)z - n.vc[2]};
    for (int e = lane; e < 60; e += nlanes) {
        double w;
        int sidx;
        if (e < 36) {
            const int pr = e / 6;
            sidx = e - pr * 6;
            const int j = pr < 3 ? 0 : (pr < 5 ? 1 : 2), k = pr < 3 ? pr : (pr < 5 ? pr - 2 : 2);
            w = q[j] * q[k];
        } else if (e < 54) {
            const int j = (e - 36) / 6;
            sidx = (e - 36) - j * 6;
            w = q[j];
        } else {
            sidx = e - 54;
            w = 1.0;
        }
        n.mq[e] = n.mq[e] + w * var6[sidx];
    }
}
// std::vector<Point_with_var>().swap(m_temp_points_): chunks go to the pending-free list (recycled between scans); returns their number
IM_HD int node_free_points(const VoxelMapDev& m, int nd) {
    NodeRec& n = m.nodes[nd];
    int ch = n.first_chunk;
    int freed = 0;
    while (ch >= 0) {
        const int nx = m.chunks[ch].next;
        const int i = im_atomic_add(m.pending_n, 1);
        if (i < m.max_chunks) m.pending[i] = ch;
        ch = nx;
        ++freed;
    }
    n.first_chunk = -1;
    n.last_chunk = -1;
    n.n_pts = 0;
    for (int i = 0; i < 3; ++i) n.sum_p[i] = 0.0;
    for (int i = 0; i < 6; ++i) n.sum_pp[i] = 0.0;
    for (int i = 0; i < 60; ++i) n.mq[i] = 0.0;
    return freed;
}

// ------------------------------------------------------------------ init_plane (voxel_loc.cpp:47-139)
// Cooperative over `nlanes` lanes (32 on the GPU, 1 in the host emulation).  Every lane recomputes the centre / covariance
// and the eigen-decomposition from the node's running sums (identical bits in all lanes); lane e owns plane_var entry e of 21.
//
// plane_var = sum_i J_i Sigma_i J_i^T,  J_i = [U F_i ; I/n],  F_i[m,:] = (p_i - c)^T s_m M_m  (m != min; s_m = 1/(n (l_min - l_m)),
// M_m = u_m u_min^T + u_min u_m^T).  U F_i = sum_j d_ij G_j with d_i = p_i - c and the 27 constants
//     G_j[a][b] = U[a][m0] (s0 M0[j][b]) + U[a][m1] (s1 M1[j][b]),
// so with W_jk = sum_i d_ij d_ik Sigma_i, V_j = sum_i d_ij Sigma_i, S0 = sum_i Sigma_i:
//     top-left  = sum_jk G_j W_jk G_k^T      top-right = (sum_j G_j V_j) / n      bottom-right = S0 / n^2,
// and W, V follow from the node's moments about its voxel centre (NodeRec::mq) with e = c - vc:
//     W_jk = ((Q2_jk - e_j Q1_k) - e_k Q1_j) + (e_j e_k) S0,      V_j = Q1_j - e_j S0.
// The oracle evaluates the same expressions in the same order (orc_lio.hpp, plane_var_mode 0) and bounds the distance to the
// reference's literal per-point loop (plane_var_mode 1; tests/test_oracle_crosscheck.py).
#if defined(__CUDA_ARCH__)
#define IM_ENT_PER_LANE 1
#else
#define IM_ENT_PER_LANE 21
#endif
IM_HDN inline void init_plane(const VoxelMapDev& m, const LioParams& P, int nd, int lane, int nlanes) {
    const NodeRec& n = m.nodes[nd];
    PlaneRec& pl = m.planes[nd];
    const int np = n.n_pts;
    if (lane == 0 && m.stat) { im_atomic_add(m.stat, 1); im_atomic_add(m.stat + 1, np); }
    // centre / covariance sums are kept incrementally by node_append in append order: bit-identical to the
    // reference's loop over m_temp_points_ (voxel_loc.cpp:55-59)
    double cov[6], c[3];
    for (int i = 0; i < 6; ++i) cov[i] = n.sum_pp[i];
    for (int i = 0; i < 3; ++i) c[i] = n.sum_p[i];
    const double dn = (double)np;
    c[0] = c[0] / dn; c[1] = c[1] / dn; c[2] = c[2] / dn;
    cov[0] = cov[0] / dn - c[0] * c[0]; cov[1] = cov[1] / dn - c[0] * c[1]; cov[2] = cov[2] / dn - c[0] * c[2];
    cov[3] = cov[3] / dn - c[1] * c[1]; cov[4] = cov[4] / dn - c[1] * c[2]; cov[5] = cov[5] / dn - c[2] * c[2];
    double ev[3], U[9];
    jacobi3(cov, ev, U);
    int imin = 0, imax = 0;
    for (int i = 1; i < 3; ++i) {
        if (ev[i] < ev[imin]) imin = i;
        if (ev[i] > ev[imax]) imax = i;
    }
    const bool planar = ev[imin] < (double)P.planer_threshold;
    double acc[IM_ENT_PER_LANE];
    for (int k = 0; k < IM_ENT_PER_LANE; ++k) acc[k] = 0.0;
    if (planar) {
        const double invn = 1.0 / dn;
        const int m0 = (imin == 0) ? 1 : 0;            // the two rows of F that are not identically zero
        const int m1 = (imin == 2) ? 1 : 2;
        const double s0 = 1.0 / (dn * (ev[imin] - ev[m0])), s1 = 1.0 / (dn * (ev[imin] - ev[m1]));
        const double e3[3] = {c[0] - n.vc[0], c[1] - n.vc[1], c[2] - n.vc[2]};
        const double* mq = n.mq;
        for (int k = 0; k < IM_ENT_PER_LANE; ++k) {
            const int e = lane + k * nlanes;
            if (e >= 21) break;
            int ei = 0, base = 0;
            while (e >= base + (6 - ei)) { base += 6 - ei; ++ei; }
            const int ej = ei + (e - base);
            double r;
            if (ei >= 3) {
                r = (invn * mq[54 + s6(ei - 3, ej - 3)]) * invn;
            } else {
                // G_j[a][.] for this entry's row a = ei, and (top-left only) G_k[b][.] for b = ej
                double Ga[9], Gb[9];
                for (int j = 0; j < 3; ++j)
                    for (int x = 0; x < 3; ++x) {
                        const double M0jx = U[j * 3 + m0] * U[x * 3 + imin] + U[j * 3 + imin] * U[x * 3 + m0];
                        const double M1jx = U[j * 3 + m1] * U[x * 3 + imin] + U[j * 3 + imin] * U[x * 3 + m1];
                        Ga[j * 3 + x] = U[ei * 3 + m0] * (s0 * M0jx) + U[ei * 3 + m1] * (s1 * M1jx);
                        const int bb = ej < 3 ? ej : 0;
                        Gb[j * 3 + x] = U[bb * 3 + m0] * (s0 * M0jx) + U[bb * 3 + m1] * (s1 * M1jx);
                    }
                if (ej >= 3) {
                    // top-right (ei, 3 + l): (sum_j sum_x G_j[ei][x] V_j[x][l]) / n
                    const int l = ej - 3;
                    double a2 = 0.0;
                    for (int j = 0; j < 3; ++j)
                        for (int x = 0; x < 3; ++x) {
                            const int sx = s6(x, l);
                            const double v = mq[36 + j * 6 + sx] - e3[j] * mq[54 + sx];
                            a2 = a2 + Ga[j * 3 + x] * v;
                        }
                    r = a2 * invn;
                } else {
                    // top-left (ei, ej): sum_jk sum_xy G_j[ei][x] W_jk[x][y] G_k[ej][y]
                    double a2 = 0.0;
                    for (int j = 0; j < 3; ++j)
                        for (int k2 = 0; k2 < 3; ++k2) {
                            const int pr = s6(j, k2);
                            const double ejk = e3[j] * e3[k2];
                            for (int x = 0; x < 3; ++x)
                                for (int y = 0; y < 3; ++y) {
                                    const int sx = s6(x, y);
                                    const double w = ((mq[pr * 6 + sx] - e3[j] * mq[36 + k2 * 6 + sx]) - e3[k2] * mq[36 + j * 6 + sx]) + ejk * mq[54 + sx];
                                    a2 = a2 + (Ga[j * 3 + x] * w) * Gb[k2 * 3 + y];
                                }
                        }
                    r = a2;
                }
            }
            acc[k] = r;
        }
    }
    IM_SYNCWARP();  // all lanes have finished reading the old record
    for (int k = 0; k < IM_ENT_PER_LANE; ++k) {
        const int e = lane + k * nlanes;
        if (e < 21) pl.pv[e] = acc[k];  // zero when not planar (voxel_loc.cpp:49)
    }
    if (lane == 0) {
        pl.center[0] = c[0]; pl.center[1] = c[1]; pl.center[2] = c[2];
        pl.points_size = np;
        if (planar) {
            const double nx = U[0 * 3 + imin], ny = U[1 * 3 + imin], nz = U[2 * 3 + imin];
            pl.normal[0] = nx; pl.normal[1] = ny; pl.normal[2] = nz;
            pl.min_eig = (float)ev[imin];
            pl.radius = (float)sqrt(ev[imax]);
            pl.d = (float)(-((nx * c[0] + ny * c[1]) + nz * c[2]));
            pl.is_plane = 1;
        } else {
            pl.normal[0] = 0.0; pl.normal[1] = 0.0; pl.normal[2] = 0.0;
            pl.radius = 0.f;
            pl.is_plane = 0;
        }
        pl.plane_inited = 1;
        if (m.pub) {   // plane-map publisher state (absent from a map built without it)
            PubRec& q = m.pub[nd];
            if (planar)
                for (int i = 0; i < 3; ++i) { q.p_center[i] = (float)c[i]; q.p_normal[i] = (float)U[i * 3 + imin]; }
            q.updated = 1;
            // one warp grows a root voxel at a time, so the mark of this root is not contended
            const int rs = n.root_slot;
            if (m.pub_mark[rs] == 0) {
                m.pub_mark[rs] = 1;
                m.pub_list[im_atomic_add(m.pub_n, 1)] = rs;
            }
        }
    }
    IM_SYNCWARP();
}

// child creation, voxel_loc.cpp:186-190 / :279-283 (lane 0 allocates, id broadcast)
IM_HDN inline int make_child(const VoxelMapDev& m, int parent, int leaf, int lane) {
    int id = -1;
    if (lane == 0) {
        id = alloc_node(m);
        if (id >= 0) {
            const NodeRec& pn = m.nodes[parent];
            const int xyz[3] = {(leaf >> 2) & 1, (leaf >> 1) & 1, leaf & 1};
            double vc[3];
            for (int j = 0; j < 3; ++j) vc[j] = pn.vc[j] + (double)((float)(2 * xyz[j] - 1) * pn.quater);
            init_node(m, id, pn.layer + 1, vc, pn.quater / 2, pn.root_slot);
            m.nodes[parent].children[leaf] = id;
        }
    }
    id = IM_BCAST_I(id);
    IM_SYNCWARP();
    return id;
}
IM_HD int leaf_of(const NodeRec& n, float x, float y, float z) {
    return 4 * (((double)x > n.vc[0]) ? 1 : 0) + 2 * (((double)y > n.vc[1]) ? 1 : 0) + (((double)z > n.vc[2]) ? 1 : 0);
}

// cut_octo_tree + the init that follows, voxel_loc.cpp:141-217, recursion unrolled on an explicit stack.
// `nd` has just been fitted and found non-planar (octo_state = 1).
IM_HDN inline void cut_octo_tree(const VoxelMapDev& m, const LioParams& P, int nd0, int lane, int nlanes) {
    int st_node[8], st_child[8];
    int sp = 0;
    st_node[0] = nd0; st_child[0] = -1;
    sp = 1;
    while (sp > 0) {
        const int nd = st_node[sp - 1];
        if (st_child[sp - 1] < 0) {
            // first visit: distribute the stored points (in order) to the children
            if (m.nodes[nd].layer >= P.max_layer) {
                if (lane == 0) m.nodes[nd].octo_state = 0;
                IM_SYNCWARP();
                --sp;
                continue;
            }
            const int np = m.nodes[nd].n_pts;
            int ch = m.nodes[nd].first_chunk;
            for (int i = 0; i < np; ++i) {
                const int s = i & 7;
                if (i && s == 0) ch = m.chunks[ch].next;
                const float x = m.chunks[ch].x[s], y = m.chunks[ch].y[s], z = m.chunks[ch].z[s];
                const int leaf = leaf_of(m.nodes[nd], x, y, z);
                int child = m.nodes[nd].children[leaf];
                if (child < 0) child = make_child(m, nd, leaf, lane);
                if (child < 0) break;
                double v6[6];
                for (int k = 0; k < 6; ++k) v6[k] = m.chunks[ch].var[k][s];
                if (lane == 0) {
                    node_append(m, child, x, y, z, v6);
                    m.nodes[child].new_points += 1;
                }
                node_moments_add(m, child, x, y, z, v6, lane, nlanes);
                IM_SYNCWARP();
            }
            st_child[sp - 1] = 0;
        }
        // resume the child loop (voxel_loc.cpp:195-216)
        bool pushed = false;
        for (int i = st_child[sp - 1]; i < 8; ++i) {
            const int child = m.nodes[nd].children[i];
            if (child < 0) continue;
            if (m.nodes[child].n_pts > P.layer_init[m.nodes[child].layer]) {
                init_plane(m, P, child, lane, nlanes);
                const int planar = m.planes[child].is_plane;
                if (lane == 0) {
                    m.nodes[child].octo_state = planar ? 0 : 1;
                    m.nodes[child].init_octo = 1;
                    m.nodes[child].new_points = 0;
                }
                IM_SYNCWARP();
                if (!planar) {
                    st_child[sp - 1] = i + 1;
                    st_node[sp] = child; st_child[sp] = -1;
                    ++sp;
                    pushed = true;
                    break;
                }
            }
        }
        if (!pushed) --sp;
    }
}
// init_octo_tree, voxel_loc.cpp:141-159
IM_HDN inline void init_octo_tree(const VoxelMapDev& m, const LioParams& P, int nd, int lane, int nlanes) {
    if (m.nodes[nd].n_pts > P.layer_init[m.nodes[nd].layer]) {
        init_plane(m, P, nd, lane, nlanes);
        const int planar = m.planes[nd].is_plane;
        if (lane == 0) {
            m.nodes[nd].octo_state = planar ? 0 : 1;
            m.nodes[nd].init_octo = 1;
            m.nodes[nd].new_points = 0;
        }
        IM_SYNCWARP();
        if (!planar) cut_octo_tree(m, P, nd, lane, nlanes);
    }
}
// UpdateOctoTree, voxel_loc.cpp:219-308 (tail recursion turned into a descent loop)
IM_HDN inline void update_octo_tree(const VoxelMapDev& m, const LioParams& P, int root, float x, float y, float z, const double* var6, int lane, int nlanes) {
    int nd = root;
    for (int guard = 0; guard < 16; ++guard) {
        const NodeRec& n = m.nodes[nd];
        if (!n.init_octo) {
            if (lane == 0) {
                m.nodes[nd].new_points += 1;
                node_append(m, nd, x, y, z, var6);
            }
            node_moments_add(m, nd, x, y, z, var6, lane, nlanes);
            IM_SYNCWARP();
            if (IM_UPRED(m.nodes[nd].n_pts > P.layer_init[m.nodes[nd].layer] ? 1 : 0)) init_octo_tree(m, P, nd, lane, nlanes);
            return;
        }
        if (m.planes[nd].is_plane) {
            if (n.update_enable) {
                if (lane == 0) {
                    m.nodes[nd].new_points += 1;
                    node_append(m, nd, x, y, z, var6);
                }
                node_moments_add(m, nd, x, y, z, var6, lane, nlanes);
                IM_SYNCWARP();
                if (IM_UPRED(m.nodes[nd].new_points > 5 ? 1 : 0)) {
                    init_plane(m, P, nd, lane, nlanes);
                    if (lane == 0) m.nodes[nd].new_points = 0;
                    IM_SYNCWARP();
                }
                if (IM_UPRED(m.nodes[nd].n_pts >= P.max_points ? 1 : 0)) {
                    if (lane == 0) {
                        m.nodes[nd].update_enable = 0;
                        node_free_points(m, nd);
                        m.nodes[nd].new_points = 0;
                    }
                    IM_SYNCWARP();
                }
            }
            return;
        }
        if (n.layer < P.max_layer) {
            if (IM_UPRED(n.n_pts != 0 ? 1 : 0)) {
                if (lane == 0) node_free_points(m, nd);
                IM_SYNCWARP();
            }
            const int leaf = leaf_of(m.nodes[nd], x, y, z);
            int child = m.nodes[nd].children[leaf];
            if (child < 0) child = make_child(m, nd, leaf, lane);
            if (child < 0) return;
            nd = child;
            continue;
        }
        // non-planar node at the maximum layer (voxel_loc.cpp:287-305)
        if (n.update_enable) {
            if (lane == 0) {
                m.nodes[nd].new_points += 1;
                node_append(m, nd, x, y, z, var6);
            }
            node_moments_add(m, nd, x, y, z, var6, lane, nlanes);
            IM_SYNCWARP();
            if (IM_UPRED(m.nodes[nd].new_points > 5 ? 1 : 0)) {
                init_plane(m, P, nd, lane, nlanes);
                if (lane == 0) m.nodes[nd].new_points = 0;
                IM_SYNCWARP();
            }
            if (IM_UPRED(m.nodes[nd].n_pts > 1000 ? 1 : 0)) {  // g_max_points, voxel_loc.cpp:45
                if (lane == 0) {
                    m.nodes[nd].update_enable = 0;
                    node_free_points(m, nd);
                }
                IM_SYNCWARP();
            }
        }
        return;
    }
}

// ------------------------------------------------------------------ plane-map publication (pubPlaneMap, voxel_mapping.cpp:947-1159)
// One root voxel of the reference's walk, literally:
//   root flag set            -> publish the root (radius 1.25 r, alpha = is_plane), clear; its children are not looked at
//   else each child i        -> flag set: publish (1.25 r, alpha = is_plane), clear; its children are not looked at
//   else each grandchild j   -> octo_state == 0 and flag set: counted as a sub-sub plane; published (radius r, alpha 1) and
//                               cleared only when planar, a non-planar one keeps its flag
//   layers >= 3 are never published.
// Row (IM_PUB_COLS doubles): kx ky kz path layer id | p_center xyz, p_center normal xyz (floats) | radius (the float pubPlane is
// given) | min_eig | trace | alpha.  path: the dump's encoding (child l -> path * 9 + l + 1); id: the node record index;
// trace: (pv00 + pv11) + pv22, the order of Eigen's 3-vector sum.  rows == nullptr: nothing written, no flag cleared (a count).
// counts (may be null) += plane, sub-plane, sub-sub-plane and update counts of the reference's two log lines.
// The walk's k-th row goes to row first + k of rows[], or of a ring of `ring` rows (slot (first + k) % ring) when ring > 0.
#define IM_PUB_COLS 16
IM_HD double* plane_pub_at(double* rows, long long first, int k, long long ring) {
    const long long r = first + k;
    return rows + (size_t)(ring > 0 ? r % ring : r) * IM_PUB_COLS;
}
IM_HD void plane_pub_row(const VoxelMapDev& m, int nd, long long kx, long long ky, long long kz, long long path, int layer, bool scaled, double* row) {
    const PlaneRec& pl = m.planes[nd];
    const PubRec& q = m.pub[nd];
    row[0] = (double)kx; row[1] = (double)ky; row[2] = (double)kz;
    row[3] = (double)path; row[4] = (double)layer; row[5] = (double)nd;
    for (int i = 0; i < 3; ++i) { row[6 + i] = (double)q.p_center[i]; row[9 + i] = (double)q.p_normal[i]; }
    row[12] = scaled ? (double)(float)(1.25 * (double)pl.radius) : (double)pl.radius;
    row[13] = (double)pl.min_eig;
    row[14] = (pl.pv[0] + pl.pv[6]) + pl.pv[11];
    row[15] = scaled ? (pl.is_plane ? 1.0 : 0.0) : 1.0;
}
IM_HD int plane_pub_root(const VoxelMapDev& m, int root, unsigned long long key, double* rows, int* counts, long long first = 0, long long ring = 0) {
    long long kx, ky, kz;
    unpack_key(key, &kx, &ky, &kz);
    int c[4] = {0, 0, 0, 0};
    int nrow = 0;
    if (m.pub[root].updated) {
        if (rows) { plane_pub_row(m, root, kx, ky, kz, 0, 0, true, plane_pub_at(rows, first, 0, ring)); m.pub[root].updated = 0; }
        nrow = 1; c[0] = 1; c[3] = 1;
    } else {
        for (int i = 0; i < 8; ++i) {
            const int ch = m.nodes[root].children[i];
            if (ch < 0) continue;
            if (m.pub[ch].updated) {
                if (rows) { plane_pub_row(m, ch, kx, ky, kz, i + 1, 1, true, plane_pub_at(rows, first, nrow, ring)); m.pub[ch].updated = 0; }
                ++nrow; ++c[1]; ++c[3];
                continue;
            }
            for (int j = 0; j < 8; ++j) {
                const int g = m.nodes[ch].children[j];
                if (g < 0 || m.nodes[g].octo_state != 0 || !m.pub[g].updated) continue;
                if (m.planes[g].is_plane) {
                    if (rows) {
                        plane_pub_row(m, g, kx, ky, kz, (long long)(i + 1) * 9 + (j + 1), 2, false, plane_pub_at(rows, first, nrow, ring));
                        m.pub[g].updated = 0;
                    }
                    ++nrow; ++c[3];
                }
                ++c[2];
            }
        }
    }
    if (counts)
        for (int k = 0; k < 4; ++k) counts[k] += c[k];
    return nrow;
}
// Publish the root listed at `slot` into rows[] (room for what plane_pub_root counted) and settle its mark: the root stays pending
// while the same walk over what is left would publish something (a child held back by the root's own flag, a grandchild behind a
// child that was published), and leaves the list otherwise -- flags that can never be published (non-planar or split layer-2 nodes,
// layers >= 3) do not keep it there; the next fit under it marks it again.  Returns 1 when the root stays pending.  first, ring: as
// in plane_pub_root.
IM_HD int plane_pub_commit(const VoxelMapDev& m, int slot, double* rows, long long first = 0, long long ring = 0) {
    const int root = m.root_node[slot];
    if (root < 0) { m.pub_mark[slot] = 0; return 0; }
    plane_pub_root(m, root, m.keys[slot], rows, nullptr, first, ring);
    const int again = plane_pub_root(m, root, m.keys[slot], nullptr, nullptr) > 0 ? 1 : 0;
    if (!again) m.pub_mark[slot] = 0;
    return again;
}

// ------------------------------------------------------------------ residual selection
// sigma_l = J_nq * plane_var * J_nq^T, J_nq = [p - c, -n]  (voxel_mapping.cpp:264-267, :1523-1526)
IM_HD double plane_sigma(const double* pw, const double* center, const double* normal, const double* pv) {
    const double J[6] = {pw[0] - center[0], pw[1] - center[1], pw[2] - center[2], -normal[0], -normal[1], -normal[2]};
    double acc = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double row = 0.0;
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            const double mij = (i <= j) ? pv[u21(i, j)] : pv[u21(j, i)];
            row = row + mij * J[j];
        }
        acc = acc + J[i] * row;
    }
    return acc;
}

struct MatchResult {
    int node;   // plane node index, -1 when unmatched
    int layer;
    double prob;
};

// one plane candidate of build_single_residual (voxel_mapping.cpp:252-283): range gate, 3-sigma gate, keep the most probable plane
IM_HDN inline void match_eval_plane(const PlaneRec& pl, int nd, int layer, const double* pw, const double* var6, bool* ok, MatchResult* best) {
    const float dis_to_plane = (float)fabs(((pl.normal[0] * pw[0] + pl.normal[1] * pw[1]) + pl.normal[2] * pw[2]) + (double)pl.d);
    const float dis_to_center = (float)(((pl.center[0] - pw[0]) * (pl.center[0] - pw[0]) + (pl.center[1] - pw[1]) * (pl.center[1] - pw[1])) +
                                        (pl.center[2] - pw[2]) * (pl.center[2] - pw[2]));
    const float range_dis = sqrtf(dis_to_center - dis_to_plane * dis_to_plane);
    if ((double)range_dis <= 3.0 * (double)pl.radius) {
        double sigma_l = plane_sigma(pw, pl.center, pl.normal, pl.pv);
        sigma_l = sigma_l + quad6(pl.normal, var6);
        const double sq = sqrt(sigma_l);
        if ((double)dis_to_plane < 3.0 * sq) {  // sigma_num is the literal 3.0 (voxel_mapping.cpp:1365)
            *ok = true;
            const double dd = (double)dis_to_plane;
            const double this_prob = 1.0 / sq * im_exp(-0.5 * dd * dd / sigma_l);
            if (this_prob > best->prob) {
                best->prob = this_prob;
                best->node = nd;
                best->layer = layer;
            }
        }
    }
}

// build_single_residual below node `start` at octree layer `depth0` (voxel_mapping.cpp:247-318); recursion -> explicit stack
IM_HDN inline void match_subtree(const VoxelMapDev& m, const LioParams& P, int start, int depth0, const double* pw, const double* var6, bool* ok, MatchResult* best) {
    int st_node[8], st_child[8];
    int sp = 1;
    st_node[0] = start; st_child[0] = -1;
    while (sp > 0) {
        const int nd = st_node[sp - 1];
        if (st_child[sp - 1] < 0) {
            const PlaneRec& pl = m.planes[nd];
            if (pl.is_plane) {
                match_eval_plane(pl, nd, depth0 + sp - 1, pw, var6, ok, best);
                --sp;
                continue;
            }
            if (depth0 + sp - 1 >= P.max_layer) { --sp; continue; }
            st_child[sp - 1] = 0;
        }
        bool pushed = false;
        for (int i = st_child[sp - 1]; i < 8; ++i) {
            const int child = m.nodes[nd].children[i];
            if (child >= 0) {
                st_child[sp - 1] = i + 1;
                st_node[sp] = child; st_child[sp] = -1;
                ++sp;
                pushed = true;
                break;
            }
        }
        if (!pushed) --sp;
    }
}
IM_HDN inline void match_in_voxel(const VoxelMapDev& m, const LioParams& P, int root, const double* pw, const double* var6, bool* ok, MatchResult* best) {
    match_subtree(m, P, root, 0, pw, var6, ok, best);
}
// One lane's share of match_in_voxel when `nl` lanes (8, or 1 = the whole walk) work on the same point: the root itself (lane 0) when it
// is a plane, else the subtrees below the lane's 8/nl first-level children.  The serial walk finishes child 0's subtree before it enters
// child 1's and replaces the best plane only on a strictly larger probability, so taking, over the lanes in order, the first lane that
// holds the largest probability reproduces its choice (MatchCombine8 in lio_capi.cu; the replay over the lanes in the host emulation).
IM_HDN inline void match_in_voxel_lane(const VoxelMapDev& m, const LioParams& P, int root, int lane, int nl, const double* pw, const double* var6, bool* ok, MatchResult* best) {
    const PlaneRec& pl = m.planes[root];
    if (pl.is_plane) {
        if (lane == 0) match_eval_plane(pl, root, 0, pw, var6, ok, best);
        return;
    }
    if (0 >= P.max_layer) return;
    const int per = 8 / nl;
    for (int c = lane * per; c < (lane + 1) * per; ++c) {
        const int child = m.nodes[root].children[c];
        if (child >= 0) match_subtree(m, P, child, 1, pw, var6, ok, best);
    }
}

// neighbour voxel of the one-shot retry (voxel_mapping.cpp:192-216).  The root voxel's centre and quarter length are
// functions of its key alone (:138-141), so the neighbour key does not need the map; the voxel-unit coordinate is
// compared with metric bounds exactly as the reference does.
IM_HD void neighbour_key(const LioParams& P, const long long* k, const float* loc, long long* nk) {
    const double ql = (double)(P.voxel_size_f / 4);
    for (int j = 0; j < 3; ++j) {
        const double vc = (0.5 + (double)k[j]) * (double)P.voxel_size_f;
        nk[j] = k[j];
        if ((double)loc[j] > vc + ql) nk[j] = k[j] + 1;
        else if ((double)loc[j] < vc - ql) nk[j] = k[j] - 1;
    }
}

// BuildResidualListOMP body for one point (voxel_mapping.cpp:169-236): root voxel, then one neighbour retry
IM_HDN inline MatchResult match_point(const VoxelMapDev& m, const LioParams& P, const double* pw, const double* var6) {
    MatchResult best;
    best.node = -1; best.layer = 0; best.prob = 0.0;
    long long k[3];
    float loc[3];
    if (!voxel_key3_loc(pw, P.voxel_size, k, loc)) return best;
    const int slot = hash_find(m, pack_key(k[0], k[1], k[2]));
    if (slot < 0) return best;
    const int root = m.root_node[slot];
    if (root < 0) return best;
    bool ok = false;
    match_in_voxel(m, P, root, pw, var6, &ok, &best);
    if (!ok) {
        long long nk[3];
        neighbour_key(P, k, loc, nk);
        if (nk[0] > -1048000 && nk[0] < 1048000 && nk[1] > -1048000 && nk[1] < 1048000 && nk[2] > -1048000 && nk[2] < 1048000) {
            const int s2 = hash_find(m, pack_key(nk[0], nk[1], nk[2]));
            if (s2 >= 0 && m.root_node[s2] >= 0) match_in_voxel(m, P, m.root_node[s2], pw, var6, &ok, &best);
        }
    }
    if (!ok) best.node = -1;
    return best;
}
// The same with the walk of each root voxel split over nl lanes.  `combine(ok, best)` merges the lanes' results (in lane order, see
// match_in_voxel_lane) and hands every lane the merged pair; the lanes of a point always call it together (nl = 1: it does nothing).
template <class Combine>
IM_HDN inline MatchResult match_point_lanes(const VoxelMapDev& m, const LioParams& P, const double* pw, const double* var6, int lane, int nl, Combine combine) {
    MatchResult best;
    best.node = -1; best.layer = 0; best.prob = 0.0;
    bool ok = false;
    long long k[3] = {0, 0, 0};
    float loc[3] = {0.f, 0.f, 0.f};
    int root = -1;
    if (voxel_key3_loc(pw, P.voxel_size, k, loc)) {
        const int slot = hash_find(m, pack_key(k[0], k[1], k[2]));
        if (slot >= 0) root = m.root_node[slot];
    }
    IM_STAMP(4, root);
    if (root >= 0) match_in_voxel_lane(m, P, root, lane, nl, pw, var6, &ok, &best);
    IM_STAMP(5, best.node);
    combine(&ok, &best);
    IM_STAMP(6, best.node);
    if (root >= 0 && !ok) {   // the same decision in all 8 lanes
        long long nk[3];
        neighbour_key(P, k, loc, nk);
        int root2 = -1;
        if (nk[0] > -1048000 && nk[0] < 1048000 && nk[1] > -1048000 && nk[1] < 1048000 && nk[2] > -1048000 && nk[2] < 1048000) {
            const int s2 = hash_find(m, pack_key(nk[0], nk[1], nk[2]));
            if (s2 >= 0) root2 = m.root_node[s2];
        }
        if (root2 >= 0) match_in_voxel_lane(m, P, root2, lane, nl, pw, var6, &ok, &best);
        combine(&ok, &best);
    }
    if (!ok) best.node = -1;
    return best;
}

// ------------------------------------------------------------------ per-point geometry
// calcBodyVar, voxel_mapping.cpp:1221-1241 (pb may be modified exactly as the reference modifies it)
IM_HDN inline void calc_body_var(double* pb, float range_inc, double direction_var, double* var6) {
    if (pb[2] == 0) pb[2] = 0.0001;
    const float range = (float)sqrt((pb[0] * pb[0] + pb[1] * pb[1]) + pb[2] * pb[2]);
    const float range_var = range_inc * range_inc;
    const double nrm = sqrt((pb[0] * pb[0] + pb[1] * pb[1]) + pb[2] * pb[2]);
    const double dir[3] = {pb[0] / nrm, pb[1] / nrm, pb[2] / nrm};
    double hat[9];
    skew3(dir, hat);
    double b1[3] = {1.0, 1.0, -(dir[0] + dir[1]) / dir[2]};
    const double n1 = sqrt((b1[0] * b1[0] + b1[1] * b1[1]) + b1[2] * b1[2]);
    b1[0] = b1[0] / n1; b1[1] = b1[1] / n1; b1[2] = b1[2] / n1;
    double b2[3] = {b1[1] * dir[2] - b1[2] * dir[1], b1[2] * dir[0] - b1[0] * dir[2], b1[0] * dir[1] - b1[1] * dir[0]};
    const double n2 = sqrt((b2[0] * b2[0] + b2[1] * b2[1]) + b2[2] * b2[2]);
    b2[0] = b2[0] / n2; b2[1] = b2[1] / n2; b2[2] = b2[2] / n2;
    double A0[3], A1[3];
    const double rg = (double)range;
    for (int i = 0; i < 3; ++i) {
        const double h0 = rg * hat[i * 3 + 0], h1 = rg * hat[i * 3 + 1], h2 = rg * hat[i * 3 + 2];
        A0[i] = (h0 * b1[0] + h1 * b1[1]) + h2 * b1[2];
        A1[i] = (h0 * b2[0] + h1 * b2[1]) + h2 * b2[2];
    }
    const double rv = (double)range_var;
    for (int i = 0; i < 3; ++i)
        for (int j = i; j < 3; ++j)
            var6[s6(i, j)] = (dir[i] * rv) * dir[j] + ((A0[i] * direction_var) * A0[j] + (A1[i] * direction_var) * A1[j]);
}
// R (R_ext p + t_ext) + t   (transformLidar, voxel_mapping_common.cpp:709-726; pointBodyToWorld :121-131)
IM_HD void body_to_world(const LioParams& P, const double* R, const double* t, const double* pb, double* pw) {
    double q[3], w[3];
    m3_vec(P.extR, pb, q);
    q[0] = q[0] + P.extT[0]; q[1] = q[1] + P.extT[1]; q[2] = q[2] + P.extT[2];
    m3_vec(R, q, w);
    pw[0] = w[0] + t[0]; pw[1] = w[1] + t[1]; pw[2] = w[2] + t[2];
}

}  // namespace immesh
