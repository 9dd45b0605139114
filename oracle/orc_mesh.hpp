// ORACLE (test infrastructure, NOT product code) -- CPU restatement of ImMesh's voxel-wise
// incremental mesher: vertex append (grid de-dup + minimum-distance test), exact kNN (what the
// reference asks of ikd-Tree), in-voxel retrieval + dilation, PCA projection, 2D Delaunay,
// 150-degree facet filter, pull / commit / push on the triangle store.
// Parity status: "parity unpinned" (see orc_math.hpp header).  Citations are relative to
// /root/reference.
//
// Defined semantics where the reference is racy or library-defined (see DESIGN.md):
//   * frames are sequential (frame k fully pushed before frame k+1 appends);
//   * within a frame all dilation/smoothing (phase A) precedes all triangulation/flip work
//     (phase B); activated voxels are processed in ascending (x,y,z) key order and the last
//     voxel in that order that touches a triangle defines its m_index_flip;
//   * kNN ties on the float squared distance are broken by the lower vertex id;
//   * Delaunay predicates are exact on coordinates snapped to voxel_resolution * 2^-22
//     (the reference uses CGAL's inexact Simple_cartesian<double>; CGAL is not vendored).
#pragma once
#include <limits>
#include <algorithm>
#include <array>
#include <map>
#include <set>
#include <unordered_map>
#include <vector>

#include "orc_math.hpp"

namespace orc {

struct MeshCfg {
    double minimum_pts;       // meshing/points_minimum_scale * distance_scale (xi)
    double voxel_resolution;  // meshing/voxel_resolution * distance_scale
    int append_target;        // meshing/number_of_pts_append_to_map
    int threads;              // voxel-parallel workers for phase A/B (reference: TBB over all cores)
};

struct IKey {
    int x, y, z;
    bool operator==(const IKey& o) const { return x == o.x && y == o.y && z == o.z; }
    bool operator<(const IKey& o) const {
        if (x != o.x) return x < o.x;
        if (y != o.y) return y < o.y;
        return z < o.z;
    }
};
struct IKeyHash {  // tools_kd_hash.hpp:69-79 (HASH_PRIME 116101, MAX_N 201326611)
    size_t operator()(const IKey& s) const {
        return (size_t)(((((int64_t)s.z) * 116101LL) % 201326611LL + (int64_t)s.y) * 116101LL % 201326611LL + (int64_t)s.x);
    }
};
typedef std::array<int, 3> Tri;  // sorted ids (Triangle ctor sorts, triangle.hpp:27-33)

// ---------------------------------------------------------------- exact 2D Delaunay (Bowyer-Watson)
static const double kCosThr150 = -8.65928972248464878803e-01;  // smallest double c with !(acos(c)*57.3 > 150) under glibc

inline int sgn128(__int128 v) { return (v > 0) - (v < 0); }
inline int orient2d_i(const int64_t* a, const int64_t* b, const int64_t* c) {
    const int64_t d = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]);
    return (d > 0) - (d < 0);
}
// > 0 iff d strictly inside the circumcircle of CCW (a,b,c)
inline int incircle_i(const int64_t* a, const int64_t* b, const int64_t* c, const int64_t* d) {
    const int64_t adx = a[0] - d[0], ady = a[1] - d[1], bdx = b[0] - d[0], bdy = b[1] - d[1], cdx = c[0] - d[0], cdy = c[1] - d[1];
    const __int128 al = (__int128)(adx * adx + ady * ady), bl = (__int128)(bdx * bdx + bdy * bdy), cl = (__int128)(cdx * cdx + cdy * cdy);
    const __int128 det = al * (__int128)(bdx * cdy - bdy * cdx) + bl * (__int128)(cdx * ady - cdy * adx) + cl * (__int128)(adx * bdy - ady * bdx);
    return sgn128(det);
}

class Delaunay2D {
  public:
    struct T {
        int v[3];
        int n[3];  // n[i]: neighbour across the edge opposite v[i]
        bool alive;
    };
    static const int G = -1;  // ghost vertex
    const int64_t* P;         // snapped coordinates, 2 per point
    int np;
    std::vector<T> tris;
    std::vector<int> free_list;
    int last = -1;
    std::vector<int> stamp, cav, link_by_start;  // scratch
    // path statistics of the last run() (test instrumentation: which kernel path the same input takes on the device)
    int max_cav = 0;           // largest conflict region (triangles, ghosts included) of one insertion
    int n_dup = 0;             // insertions skipped because the point coincides with a vertex
    mutable long n_ties = 0;   // in-circle evaluations that returned exactly 0 (cocircular)

    const int64_t* pt(int i) const { return P + 2 * i; }
    bool conflict(const T& t, int p) const {
        for (int i = 0; i < 3; ++i)
            if (t.v[i] == G) {
                const int u = t.v[(i + 1) % 3], v = t.v[(i + 2) % 3];
                const int o = orient2d_i(pt(u), pt(v), pt(p));
                if (o > 0) return true;
                if (o < 0) return false;
                // collinear: strictly between u and v
                const int64_t *a = pt(u), *b = pt(v), *q = pt(p);
                const int64_t dx = b[0] - a[0], dy = b[1] - a[1];
                const int64_t t1 = (q[0] - a[0]) * dx + (q[1] - a[1]) * dy;
                const int64_t t2 = (q[0] - b[0]) * dx + (q[1] - b[1]) * dy;
                return t1 > 0 && t2 < 0;
            }
        const int ic = incircle_i(pt(t.v[0]), pt(t.v[1]), pt(t.v[2]), pt(p));
        if (ic == 0) ++n_ties;
        return ic > 0;
    }
    int new_tri(int a, int b, int c) {
        int id;
        if (!free_list.empty()) { id = free_list.back(); free_list.pop_back(); }
        else { id = (int)tris.size(); tris.push_back(T()); }
        T& t = tris[id];
        t.v[0] = a; t.v[1] = b; t.v[2] = c;
        t.n[0] = t.n[1] = t.n[2] = -1;
        t.alive = true;
        return id;
    }
    // returns false when all points are collinear / fewer than 3 distinct
    bool run(const int64_t* pts, int n) {
        P = pts; np = n;
        tris.clear(); free_list.clear();
        max_cav = 0; n_dup = 0; n_ties = 0;
        if (n < 3) return false;
        // seed: first point distinct from p0, then first non-collinear
        int i1 = -1, i2 = -1;
        for (int i = 1; i < n; ++i)
            if (pt(i)[0] != pt(0)[0] || pt(i)[1] != pt(0)[1]) { i1 = i; break; }
        if (i1 < 0) return false;
        for (int i = 1; i < n; ++i)
            if (i != i1 && orient2d_i(pt(0), pt(i1), pt(i)) != 0) { i2 = i; break; }
        if (i2 < 0) return false;
        int a = 0, b = i1, c = i2;
        if (orient2d_i(pt(a), pt(b), pt(c)) < 0) std::swap(b, c);
        const int t0 = new_tri(a, b, c);
        // ghosts: for CCW hull edge x->y the ghost triangle is (y, x, G)
        const int g0 = new_tri(c, b, G);  // across edge opposite a: (b,c)
        const int g1 = new_tri(a, c, G);  // across edge opposite b: (c,a)
        const int g2 = new_tri(b, a, G);  // across edge opposite c: (a,b)
        tris[t0].n[0] = g0; tris[t0].n[1] = g1; tris[t0].n[2] = g2;
        // ghost (y,x,G): n[2] (opposite G) = finite tri; n[0] (opposite y: edge x,G) ; n[1] (opposite x: edge G,y)
        tris[g0].n[2] = t0; tris[g1].n[2] = t0; tris[g2].n[2] = t0;
        // g0=(c,b,G): edge (b,G) shared with ghost having b as first vertex: g2=(b,a,G) edge (G,b);
        tris[g0].n[0] = g2; tris[g2].n[1] = g0;  // g0 opp c -> edge(b,G) ; g2 opp a -> edge (G,b)
        tris[g1].n[0] = g0; tris[g0].n[1] = g1;  // g1=(a,c,G): opp a -> edge (c,G) with g0=(c,b,G) opp b -> edge (G,c)
        tris[g2].n[0] = g1; tris[g1].n[1] = g2;  // g2=(b,a,G): opp b -> edge (a,G) with g1=(a,c,G) opp c -> edge (G,a)
        last = t0;
        stamp.assign(16, 0);
        link_by_start.assign(n + 1, -1);
        for (int p = 1; p < n; ++p) {
            if (p == i1 || p == i2) continue;
            insert(p);
        }
        return true;
    }
    void insert(int p) {
        // ---- locate by visibility walk
        int t = last;
        int guard = 0;
        while (true) {
            const T& tr = tris[t];
            bool ghost = (tr.v[0] == G || tr.v[1] == G || tr.v[2] == G);
            if (ghost) break;
            bool moved = false;
            for (int i = 0; i < 3; ++i) {
                const int u = tr.v[(i + 1) % 3], v = tr.v[(i + 2) % 3];
                if (orient2d_i(pt(u), pt(v), pt(p)) < 0) { t = tr.n[i]; moved = true; break; }
            }
            if (!moved) break;
            if (++guard > 4 * (int)tris.size() + 16) break;  // cannot happen on a Delaunay triangulation
        }
        if (!conflict(tris[t], p)) {
            // p coincides with a vertex of t (duplicate), or lies on the hull line without conflict: look around
            const T& tr = tris[t];
            for (int i = 0; i < 3; ++i)
                if (tr.v[i] != G && pt(tr.v[i])[0] == pt(p)[0] && pt(tr.v[i])[1] == pt(p)[1]) { ++n_dup; return; }  // duplicate point: skipped (CGAL does too)
            int found = -1;
            for (int i = 0; i < 3 && found < 0; ++i)
                if (tr.n[i] >= 0 && conflict(tris[tr.n[i]], p)) found = tr.n[i];
            if (found < 0) {
                for (size_t k = 0; k < tris.size() && found < 0; ++k)
                    if (tris[k].alive && conflict(tris[k], p)) found = (int)k;
            }
            if (found < 0) return;
            t = found;
        }
        // ---- grow the cavity
        if (stamp.size() < tris.size() + 8) stamp.resize(tris.size() * 2 + 8, 0);
        cav.clear();
        cav.push_back(t);
        stamp[t] = p + 1;
        struct BE { int a, b, out, out_slot; };
        std::vector<BE> boundary;
        for (size_t h = 0; h < cav.size(); ++h) {
            const int ct = cav[h];
            for (int i = 0; i < 3; ++i) {
                const int nb = tris[ct].n[i];
                if (stamp[nb] == p + 1) continue;
                if (conflict(tris[nb], p)) {
                    stamp[nb] = p + 1;
                    cav.push_back(nb);
                } else {
                    int slot = 0;
                    for (int k = 0; k < 3; ++k)
                        if (tris[nb].n[k] == ct) slot = k;
                    boundary.push_back(BE{tris[ct].v[(i + 1) % 3], tris[ct].v[(i + 2) % 3], nb, slot});
                }
            }
        }
        if ((int)cav.size() > max_cav) max_cav = (int)cav.size();
        for (int ct : cav) { tris[ct].alive = false; free_list.push_back(ct); }
        // ---- re-triangulate: (a,b,p) per boundary edge
        std::vector<int> created;
        for (const BE& e : boundary) {
            const int id = new_tri(e.a, e.b, p);
            if (stamp.size() < tris.size() + 8) stamp.resize(tris.size() * 2 + 8, 0);
            stamp[id] = 0;
            tris[id].n[2] = e.out;
            tris[e.out].n[e.out_slot] = id;
            link_by_start[e.a + 1] = id;
            created.push_back(id);
        }
        for (int id : created) {
            // neighbour opposite a (edge b,p) is the new triangle starting with b
            const int b = tris[id].v[1];
            const int nb = link_by_start[b + 1];
            tris[id].n[0] = nb;
            tris[nb].n[1] = id;
        }
        for (int id : created)
            if (tris[id].v[0] != G && tris[id].v[1] != G) last = id;
    }
};

// ---------------------------------------------------------------- the mesher
class MeshOracle {
  public:
    MeshCfg cfg;
    // vertices
    std::vector<std::array<float, 3>> vpos;    // kd-tree coordinates (float), = (float) m_pos
    std::vector<std::array<double, 3>> vsmooth;  // m_pos_aft_smooth
    std::unordered_map<IKey, int, IKeyHash> grid;  // m_hashmap_3d_pts (one vertex per xi-cell)
    struct Voxel {
        IKey key;
        std::vector<int> pts;  // m_pts_in_grid
        long meshing_times = 0, new_added = 0;
        double short_axis[3] = {0, 0, 0};
    };
    std::vector<Voxel> voxels;
    std::unordered_map<IKey, int, IKeyHash> voxel_map;  // m_hashmap_voxels
    std::vector<int> activated;                          // m_voxels_recent_visited (this frame)
    // kNN acceleration: vertices bucketed by the mesh-voxel key (exact search by ring expansion)
    // triangle store (live set = m_map_pt_triangle, triangle.hpp:330-395)
    std::set<Tri> live;
    std::unordered_map<int, std::set<Tri>> pt_tri;
    std::map<Tri, int> flip;  // m_index_flip of live triangles
    // per-frame outputs
    std::vector<Tri> frame_added, frame_removed;
    int frame_new_vertices = 0, frame_voxels_meshed = 0;
    long frame_added_mult = 0, frame_removed_mult = 0;  // summed over voxels (total_add_triangle / total_delete_triangle, :226-237)

    explicit MeshOracle(const MeshCfg& c) : cfg(c) {}

    static int round_key(float x, double cell) { return (int)std::round((double)x / cell); }  // pointcloud_rgbd.cpp:467-472

    // exact kNN over all vertices (KD_TREE::Nearest_Search semantics, ikd_Tree.cpp:441-476,1097-1279):
    // float coordinates, dist = ((dx*dx + dy*dy) + dz*dz) in float (ikd_Tree.cpp:1722-1727), ascending by (d2, id).
    // max_dist: only neighbours with d2 <= max_dist^2 (double compare, ikd_Tree.cpp:1101-1123).
    void knn(const float* q, int k, double max_dist, std::vector<std::pair<float, int>>& out) const {
        out.clear();
        if (vpos.empty()) return;
        const double res = cfg.voxel_resolution;
        const int cx = round_key(q[0], res), cy = round_key(q[1], res), cz = round_key(q[2], res);
        const double max_d2 = max_dist * max_dist;
        // farthest occupied cell (Chebyshev) from the query cell: no ring beyond it holds a vertex
        int far = 0;
        far = std::max(far, std::max(std::abs(cx - kmin[0]), std::abs(cx - kmax[0])));
        far = std::max(far, std::max(std::abs(cy - kmin[1]), std::abs(cy - kmax[1])));
        far = std::max(far, std::max(std::abs(cz - kmin[2]), std::abs(cz - kmax[2])));
        std::vector<std::pair<float, int>> heap;  // max-heap on (d2,id)
        auto visit = [&](int dx, int dy, int dz) {
            auto it = voxel_map.find(IKey{cx + dx, cy + dy, cz + dz});
            if (it == voxel_map.end()) return;
            for (int id : voxels[it->second].pts) {
                const float ex = q[0] - vpos[id][0], ey = q[1] - vpos[id][1], ez = q[2] - vpos[id][2];
                const float d2 = (ex * ex + ey * ey) + ez * ez;
                if (!((double)d2 <= max_d2)) continue;
                const std::pair<float, int> cand(d2, id);
                if ((int)heap.size() < k) {
                    heap.push_back(cand);
                    std::push_heap(heap.begin(), heap.end());
                } else if (cand < heap.front()) {
                    std::pop_heap(heap.begin(), heap.end());
                    heap.back() = cand;
                    std::push_heap(heap.begin(), heap.end());
                }
            }
        };
        for (int ring = 0; ring <= far; ++ring) {
            // a vertex in a cell at Chebyshev ring r is at least (r-1)*res away from the query
            if (ring >= 1) {
                const double lb = (double)(ring - 1) * res;
                if (lb > max_dist) break;
                if ((int)heap.size() >= k && (double)heap.front().first < lb * lb * 0.999999) break;
            }
            for (int dx = -ring; dx <= ring; ++dx)
                for (int dy = -ring; dy <= ring; ++dy) {
                    if (std::abs(dx) == ring || std::abs(dy) == ring) {
                        for (int dz = -ring; dz <= ring; ++dz) visit(dx, dy, dz);
                    } else {
                        visit(dx, dy, -ring);
                        if (ring > 0) visit(dx, dy, ring);
                    }
                }
        }
        std::sort(heap.begin(), heap.end());
        out = heap;
    }
    int kmin[3] = {0, 0, 0}, kmax[3] = {0, 0, 0};
    bool have_bbox = false;

    // append_points_to_global_map, pointcloud_rgbd.cpp:411-552.  pts: world-frame float xyz.
    void append_points(const float* pts, int n, int step) {
        activated.clear();  // m_recent_visited_voxel_activated_time == 0 (ImMesh_node.cpp:272)
        std::set<int> act_set;
        frame_new_vertices = 0;
        std::vector<std::pair<float, int>> nn;
        for (long i = 0; i < n; i += step) {
            const float* p = pts + 3 * i;
            const IKey g{round_key(p[0], cfg.minimum_pts), round_key(p[1], cfg.minimum_pts), round_key(p[2], cfg.minimum_pts)};
            const IKey b{round_key(p[0], cfg.voxel_resolution), round_key(p[1], cfg.voxel_resolution), round_key(p[2], cfg.voxel_resolution)};
            const bool occupied = grid.find(g) != grid.end();
            int vi;
            auto itv = voxel_map.find(b);
            if (itv == voxel_map.end()) {
                vi = (int)voxels.size();
                Voxel v;
                v.key = b;
                voxels.push_back(v);
                voxel_map[b] = vi;
                const int bk[3] = {b.x, b.y, b.z};
                for (int j = 0; j < 3; ++j) {
                    if (!have_bbox || bk[j] < kmin[j]) kmin[j] = bk[j];
                    if (!have_bbox || bk[j] > kmax[j]) kmax[j] = bk[j];
                }
                have_bbox = true;
            } else {
                vi = itv->second;
            }
            if (act_set.insert(vi).second) activated.push_back(vi);
            if (occupied) continue;
            if (!vpos.empty()) {
                // reference: 1-NN, reject if sqrt(d2) < xi (:507-517).  Searching within xi*(1+1e-6) is equivalent.
                knn(p, 1, cfg.minimum_pts * 1.000001, nn);
                if (!nn.empty() && (double)std::sqrt(nn[0].first) < cfg.minimum_pts) continue;
            }
            const int id = (int)vpos.size();
            vpos.push_back({p[0], p[1], p[2]});
            vsmooth.push_back({(double)p[0], (double)p[1], (double)p[2]});
            grid[g] = id;
            voxels[vi].pts.push_back(id);
            voxels[vi].new_added++;
            voxels[vi].meshing_times = 0;
            frame_new_vertices++;
        }
    }

    // smooth_all_pts (mesh_rec_geometry.cpp:60-69) = Global_map::smooth_pts on every vertex (pointcloud_rgbd.cpp:932-958) with
    // maximum_smooth_dis = g_kd_tree_accept_pt_dis = 1.25 * res (mesh_rec_geometry.cpp:343): knn nearest vertices (the first one is
    // the vertex itself and is skipped), those with sqrt(d2) < the limit are averaged (double sums in neighbour order),
    //   smoothed = p (1 - f) + sum f / valid        (valid == 0 divides by zero exactly like the reference)
    // The result is stored as the vertex's smoothed position (set_smooth_pos) and returned.
    void smooth_all(double smooth_factor, int knn_k, std::vector<std::array<double, 3>>& out) {
        const double maxdis = cfg.voxel_resolution * 1.25;
        const int nv = (int)vpos.size();
        out.assign(nv, {0, 0, 0});
        std::vector<std::pair<float, int>> nn;
        for (int v = 0; v < nv; ++v) {
            const float q[3] = {vpos[v][0], vpos[v][1], vpos[v][2]};
            knn(q, knn_k, std::numeric_limits<double>::infinity(), nn);
            double sv[3] = {0, 0, 0}, valid = 0.0;
            for (size_t k = 1; k < nn.size(); ++k) {
                if ((double)std::sqrt(nn[k].first) < maxdis) {
                    for (int j = 0; j < 3; ++j) sv[j] = sv[j] + (double)vpos[nn[k].second][j];
                    valid += 1.0;
                }
            }
            for (int j = 0; j < 3; ++j) out[v][j] = (double)vpos[v][j] * (1.0 - smooth_factor) + sv[j] * smooth_factor / valid;
            vsmooth[v] = out[v];
        }
    }
    // Triangle_manager::insert_triangle_to_list (triangle.cpp:35-53): every live triangle belongs to the region
    // round(centre / region_size), centre = mean of its three vertex positions (Triangle_manager::get_triangle_center)
    void region_keys(double region_size, std::vector<std::array<int, 3>>& out) const {
        out.clear();
        for (const Tri& t : live) {
            std::array<int, 3> k;
            for (int j = 0; j < 3; ++j) {
                const double c = (((double)vpos[t[0]][j] + (double)vpos[t[1]][j]) + (double)vpos[t[2]][j]) / 3.0;
                k[j] = (int)std::round(c / region_size);
            }
            out.push_back(k);
        }
    }

    // Depth image of the live mesh from a camera (ImMesh_node.cpp:305-329 + openGL_camera_view.cpp:316-418; the sampling rule that the
    // reference leaves to OpenGL is the one stated in include/immesh_b200.h: immesh_mesh_render_depth).  depth[h*w]: -1 where empty.
    void render_depth(const double* K4, int w, int h, double z_near, double z_far, const double* R, const double* t, std::vector<float>& depth,
                      std::vector<std::array<float, 3>>& pts, std::vector<int>& pix) const {
        std::vector<float> zb((size_t)w * h, INFINITY);
        auto project = [&](const std::array<float, 3>& p, double* u, double* v, double* z) {
            const double d[3] = {(double)p[0] - t[0], (double)p[1] - t[1], (double)p[2] - t[2]};
            const double xc = (R[0] * d[0] + R[3] * d[1]) + R[6] * d[2];
            const double yc = -((R[1] * d[0] + R[4] * d[1]) + R[7] * d[2]);
            const double zc = -((R[2] * d[0] + R[5] * d[1]) + R[8] * d[2]);
            *z = zc;
            *u = K4[0] * xc / zc + K4[2];
            *v = K4[1] * yc / zc + K4[3];
        };
        for (const Tri& tr : live) {
            double u0, v0, z0, u1, v1, z1, u2, v2, z2;
            project(vpos[tr[0]], &u0, &v0, &z0);
            project(vpos[tr[1]], &u1, &v1, &z1);
            project(vpos[tr[2]], &u2, &v2, &z2);
            if (!(z0 > z_near && z0 < z_far && z1 > z_near && z1 < z_far && z2 > z_near && z2 < z_far)) continue;
            const double area = (u1 - u0) * (v2 - v0) - (v1 - v0) * (u2 - u0);
            if (area == 0.0) continue;
            const int x_lo = std::max(0, (int)std::ceil(std::fmin(u0, std::fmin(u1, u2)))), x_hi = std::min(w - 1, (int)std::floor(std::fmax(u0, std::fmax(u1, u2))));
            const int y_lo = std::max(0, (int)std::ceil(std::fmin(v0, std::fmin(v1, v2)))), y_hi = std::min(h - 1, (int)std::floor(std::fmax(v0, std::fmax(v1, v2))));
            const double iz0 = 1.0 / z0, iz1 = 1.0 / z1, iz2 = 1.0 / z2;
            for (int y = y_lo; y <= y_hi; ++y)
                for (int x = x_lo; x <= x_hi; ++x) {
                    const double px = (double)x, py = (double)y;
                    const double e0 = (u2 - u1) * (py - v1) - (v2 - v1) * (px - u1);
                    const double e1 = (u0 - u2) * (py - v2) - (v0 - v2) * (px - u2);
                    const double e2 = (u1 - u0) * (py - v0) - (v1 - v0) * (px - u0);
                    if (!((e0 >= 0 && e1 >= 0 && e2 >= 0) || (e0 <= 0 && e1 <= 0 && e2 <= 0))) continue;
                    const double iz = ((e0 * iz0 + e1 * iz1) + e2 * iz2) / area;
                    const float zf = (float)(1.0 / iz);
                    if (zf > 0.f && zf < zb[(size_t)y * w + x]) zb[(size_t)y * w + x] = zf;
                }
        }
        depth.assign((size_t)w * h, -1.0f);
        pts.clear();
        pix.clear();
        for (int i = 0; i < w * h; ++i) {
            const float val = zb[i];
            if (!((double)val < z_far * 0.99)) continue;
            depth[i] = val;
            const int x = i % w, y = i / w;
            const double sx = ((double)x - K4[2]) / K4[0], sy = ((double)y - K4[3]) / K4[1];
            const double g[3] = {sx * (double)val, -(sy * (double)val), -(double)val};
            std::array<float, 3> p;
            for (int a = 0; a < 3; ++a) p[a] = (float)(((R[a * 3 + 0] * g[0] + R[a * 3 + 1] * g[1]) + R[a * 3 + 2] * g[2]) + t[a]);
            pts.push_back(p);
            pix.push_back(i);
        }
    }

    // retrieve_neighbor_pts_kdtree, mesh_rec_geometry.cpp:336-377
    void dilate(const std::vector<int>& in_voxel, std::set<long>& out_ids, std::vector<std::pair<int, std::array<double, 3>>>& smooth_out) const {
        const double accept = cfg.voxel_resolution * 1.25;
        std::vector<std::pair<float, int>> nn;
        for (int v : in_voxel) {
            const float q[3] = {vpos[v][0], vpos[v][1], vpos[v][2]};
            // k = 20; neighbours beyond 2*accept are ignored by both filters below, so the search may stop there
            knn(q, 20, accept * 2 * 1.000001, nn);
            double sv[3] = {0, 0, 0};
            int cnt = 0;
            for (auto& pr : nn) {
                const float sd = std::sqrt(pr.first);
                if ((double)sd < accept) out_ids.insert(pr.second);
                if ((double)sd < accept * 2) {
                    cnt++;
                    for (int j = 0; j < 3; ++j) sv[j] = sv[j] + (double)vpos[pr.second][j];
                }
            }
            std::array<double, 3> s;
            for (int j = 0; j < 3; ++j) {
                const double m = sv[j] / (double)cnt;
                s[j] = m * (double)1.0f + (double)vpos[v][j] * (double)(1 - 1.0f);  // smooth_factor = 1.0f (:334,:368)
            }
            smooth_out.push_back({v, s});
        }
    }

    // per meshed voxel of the last frame: key, dilated-set size, largest Bowyer-Watson cavity, seed found, exact in-circle ties,
    // duplicate (same snapped point) skips.  Test instrumentation: from n and the cavity a test can tell which kernel path ran.
    struct VoxStat { int key[3] = {0, 0, 0}; int n = 0, max_cav = 0, seeded = 0, n_dup = 0; long n_ties = 0; };
    std::vector<VoxStat> frame_stats;

    // delaunay_triangulation, mesh_rec_geometry.cpp:174-295 (+ is_face_is_ok :31-57)
    void triangulate(const std::vector<long>& ids, double* short_axis, std::vector<Tri>& faces, VoxStat* st = nullptr) const {
        faces.clear();
        const int n = (int)ids.size();
        if (st) st->n = n;
        if (n < 3) return;
        double c[3] = {0, 0, 0};
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < 3; ++j) c[j] = c[j] + (double)vpos[ids[i]][j];
        for (int j = 0; j < 3; ++j) c[j] = c[j] / (double)n;
        double cov[6] = {0, 0, 0, 0, 0, 0};
        for (int i = 0; i < n; ++i) {
            const double d[3] = {(double)vpos[ids[i]][0] - c[0], (double)vpos[ids[i]][1] - c[1], (double)vpos[ids[i]][2] - c[2]};
            cov[0] += d[0] * d[0]; cov[1] += d[0] * d[1]; cov[2] += d[0] * d[2];
            cov[3] += d[1] * d[1]; cov[4] += d[1] * d[2]; cov[5] += d[2] * d[2];
        }
        for (double& v : cov) v = v / (double)n;
        double ev[3], U[9];
        jacobi_eig3(cov, ev, U);
        int order[3] = {0, 1, 2};  // ascending eigenvalues (SelfAdjointEigenSolver order)
        for (int a = 0; a < 2; ++a)
            for (int b = 0; b < 2 - a; ++b)
                if (ev[order[b + 1]] < ev[order[b]]) std::swap(order[b], order[b + 1]);
        double s[3], m[3], l[3];
        for (int j = 0; j < 3; ++j) { s[j] = U[j * 3 + order[0]]; m[j] = U[j * 3 + order[1]]; }
        const double d0[3] = {(double)vpos[ids[0]][0] - c[0], (double)vpos[ids[0]][1] - c[1], (double)vpos[ids[0]][2] - c[2]};
        const double d1[3] = {(double)vpos[ids[1]][0] - c[0], (double)vpos[ids[1]][1] - c[1], (double)vpos[ids[1]][2] - c[2]};
        if (dot3(d0, s) < 0) for (int j = 0; j < 3; ++j) s[j] = -s[j];
        if (dot3(d1, m) < 0) for (int j = 0; j < 3; ++j) m[j] = -m[j];
        l[0] = s[1] * m[2] - s[2] * m[1];
        l[1] = s[2] * m[0] - s[0] * m[2];
        l[2] = s[0] * m[1] - s[1] * m[0];
        for (int j = 0; j < 3; ++j) short_axis[j] = s[j];
        std::vector<double> uv(2 * (size_t)n);
        std::vector<int64_t> snapped(2 * (size_t)n);
        const double inv_q = 4194304.0 / cfg.voxel_resolution;
        for (int i = 0; i < n; ++i) {
            const double d[3] = {(double)vpos[ids[i]][0] - c[0], (double)vpos[ids[i]][1] - c[1], (double)vpos[ids[i]][2] - c[2]};
            uv[2 * i] = dot3(d, l);
            uv[2 * i + 1] = dot3(d, m);
            snapped[2 * i] = std::llrint(uv[2 * i] * inv_q);
            snapped[2 * i + 1] = std::llrint(uv[2 * i + 1] * inv_q);
        }
        Delaunay2D dt;
        const bool seeded = dt.run(snapped.data(), n);
        if (st) { st->seeded = seeded; st->max_cav = dt.max_cav; st->n_ties = dt.n_ties; st->n_dup = dt.n_dup; }
        if (!seeded) return;
        for (const auto& t : dt.tris) {
            if (!t.alive || t.v[0] < 0 || t.v[1] < 0 || t.v[2] < 0) continue;
            bool ok = true;
            for (int a = 0; a < 3 && ok; ++a) {
                const int ia = t.v[a], ib = t.v[(a + 1) % 3], ic = t.v[(a + 2) % 3];
                const double abx = uv[2 * ib] - uv[2 * ia], aby = uv[2 * ib + 1] - uv[2 * ia + 1];
                const double acx = uv[2 * ic] - uv[2 * ia], acy = uv[2 * ic + 1] - uv[2 * ia + 1];
                const double cosv = (abx * acx + aby * acy) / (std::sqrt(abx * abx + aby * aby) * std::sqrt(acx * acx + acy * acy));
                if (cosv < kCosThr150 && cosv >= -1.0) ok = false;
            }
            if (!ok) continue;
            Tri f = {(int)ids[t.v[0]], (int)ids[t.v[1]], (int)ids[t.v[2]]};
            std::sort(f.begin(), f.end());
            faces.push_back(f);
        }
        std::sort(faces.begin(), faces.end());
    }

    // correct_triangle_index, mesh_rec_geometry.cpp:399-433
    int compute_flip(const Tri& t, const double* cam, const double* short_axis_in) const {
        const double* a = vsmooth[t[0]].data();
        const double* b = vsmooth[t[1]].data();
        const double* c = vsmooth[t[2]].data();
        const double ab[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]};
        const double ac[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
        const double tc[3] = {cam[0] - a[0], cam[1] - a[1], cam[2] - a[2]};
        double nrm[3] = {ab[1] * ac[2] - ab[2] * ac[1], ab[2] * ac[0] - ab[0] * ac[2], ab[0] * ac[1] - ab[1] * ac[0]};
        const double nn = norm3(nrm);
        if (nn != 0) { nrm[0] = nrm[0] / nn; nrm[1] = nrm[1] / nn; nrm[2] = nrm[2] / nn; }
        else { nrm[0] = 0; nrm[1] = 0; nrm[2] = 1; }
        double sa[3] = {short_axis_in[0], short_axis_in[1], short_axis_in[2]};
        if (dot3(sa, tc) < 0) { sa[0] = -sa[0]; sa[1] = -sa[1]; sa[2] = -sa[2]; }
        return (dot3(sa, nrm) < 0) ? 0 : 1;
    }

    // incremental_mesh_reconstruction, ImMesh_mesh_reconstruction.cpp:92-267
    void push_frame(const float* pts_world, int n, const double* pose_t) {
        const int step = std::max(1, (int)std::round((double)(n / cfg.append_target)));  // integer division first (:111)
        append_points(pts_world, n, step);
        frame_added.clear();
        frame_removed.clear();
        frame_voxels_meshed = 0;
        std::vector<int> order(activated);
        std::sort(order.begin(), order.end(), [&](int a, int b) { return voxels[a].key < voxels[b].key; });
        // ---- phase A: activation test, retrieval, dilation, smoothing
        struct Work { int vi; std::vector<long> ids; };
        std::vector<Work> work;
        for (int vi : order) {
            Voxel& vx = voxels[vi];
            if (vx.meshing_times >= 1 || vx.new_added < 0) continue;
            vx.meshing_times++;
            vx.new_added = 0;
            if (vx.pts.size() < 3) continue;
            work.push_back(Work{vi, {}});
        }
        std::vector<std::vector<std::pair<int, std::array<double, 3>>>> smooth(work.size());
        const int nthr = cfg.threads > 0 ? cfg.threads : 1;
#pragma omp parallel for num_threads(nthr) schedule(dynamic, 8)
        for (int w = 0; w < (int)work.size(); ++w) {
            std::set<long> ids;
            dilate(voxels[work[w].vi].pts, ids, smooth[w]);
            work[w].ids.assign(ids.begin(), ids.end());
        }
        for (auto& sv : smooth)
            for (auto& pr : sv) vsmooth[pr.first] = pr.second;
        // ---- phase B: triangulate, pull, commit, orient
        struct Res { std::vector<Tri> to_add, to_remove, existing; std::vector<int> flip_add, flip_exist; };
        std::vector<Res> res(work.size());
        frame_stats.assign(work.size(), VoxStat());
#pragma omp parallel for num_threads(nthr) schedule(dynamic, 8)
        for (int w = 0; w < (int)work.size(); ++w) {
            Voxel& vx = voxels[work[w].vi];
            std::vector<Tri> faces;
            frame_stats[w].key[0] = vx.key.x; frame_stats[w].key[1] = vx.key.y; frame_stats[w].key[2] = vx.key.z;
            triangulate(work[w].ids, vx.short_axis, faces, &frame_stats[w]);
            // pull: find_relative_triangulation_combination, triangle.hpp:223-246
            std::set<Tri> pulled;
            const std::vector<long>& ids = work[w].ids;
            for (long v : ids) {
                auto it = pt_tri.find((int)v);
                if (it == pt_tri.end()) continue;
                for (const Tri& t : it->second) {
                    if (std::binary_search(ids.begin(), ids.end(), (long)t[0]) && std::binary_search(ids.begin(), ids.end(), (long)t[1]) &&
                        std::binary_search(ids.begin(), ids.end(), (long)t[2]))
                        pulled.insert(t);
                }
            }
            // commit: triangle_compare, mesh_rec_geometry.cpp:137-172
            std::set<Tri> fset(faces.begin(), faces.end());
            Res& r = res[w];
            for (const Tri& t : fset) {
                if (pulled.count(t)) r.existing.push_back(t);
                else r.to_add.push_back(t);
            }
            for (const Tri& t : pulled)
                if (!fset.count(t)) r.to_remove.push_back(t);
            for (const Tri& t : r.to_add) r.flip_add.push_back(compute_flip(t, pose_t, vx.short_axis));
            for (const Tri& t : r.existing) r.flip_exist.push_back(compute_flip(t, pose_t, vx.short_axis));
        }
        frame_voxels_meshed = (int)work.size();
        frame_added_mult = 0;
        frame_removed_mult = 0;
        for (auto& r : res) { frame_added_mult += (long)r.to_add.size(); frame_removed_mult += (long)r.to_remove.size(); }
        for (auto& r : res)
            for (size_t i = 0; i < r.existing.size(); ++i) flip[r.existing[i]] = r.flip_exist[i];
        // ---- push: all removals, then all insertions (:228-244)
        std::set<Tri> rem_set, add_set;
        for (auto& r : res)
            for (const Tri& t : r.to_remove) {
                if (live.erase(t)) {
                    for (int k = 0; k < 3; ++k) pt_tri[t[k]].erase(t);
                    flip.erase(t);
                }
                rem_set.insert(t);
            }
        for (auto& r : res)
            for (size_t i = 0; i < r.to_add.size(); ++i) {
                const Tri& t = r.to_add[i];
                if (live.insert(t).second)
                    for (int k = 0; k < 3; ++k) pt_tri[t[k]].insert(t);
                flip[t] = r.flip_add[i];
                add_set.insert(t);
            }
        frame_added.assign(add_set.begin(), add_set.end());
        frame_removed.assign(rem_set.begin(), rem_set.end());
    }
};

}  // namespace orc
