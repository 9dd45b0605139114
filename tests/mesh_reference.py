"""Independent numpy/scipy restatement of one incremental_mesh_reconstruction frame (src/ImMesh_mesh_reconstruction.cpp:92-267),
written from the reference's code and sharing nothing with the kernels, the host emulation or the oracle.  Citations are relative to
the reference's tree.

Float types: world points and vertex positions are float (pcl::PointXYZI, ikd-Tree's float points); kd-tree distances are float
((dx*dx + dy*dy) + dz*dz, ikd_Tree.cpp:1722-1727); everything else is float64.

Two rules are the project's, not the reference's, because the reference leaves them open (DESIGN section 3):
* every dilation and smoothing of a frame precedes every triangulation and orientation (the reference runs voxels in a TBB
  parallel_for_each, so a voxel may orient from a neighbour's smoothed position before or after that neighbour smooths it);
* where several voxels of a frame set the orientation flag of one triangle, the voxel with the largest (x, y, z) key wins (in the
  reference this is a race on m_index_flip);
* kNN ties go to the lower vertex id.

One correction to a common reading: RGB_pts::set_pos writes m_pos_aft_smooth as well as m_pos (pointcloud_rgbd.cpp:59-66), so a
vertex that was never smoothed orients its facets from its raw position, not from the zero its member initialiser gives it
(pointcloud_rgbd.hpp:91).
"""
import math

import numpy as np
from scipy.spatial import Delaunay, cKDTree
from scipy.spatial._qhull import QhullError

F32 = np.float32


def std_round(x):
    """std::round: half away from zero (np.round rounds half to even)"""
    x = np.asarray(x, np.float64)
    t = np.trunc(x)
    return (t + np.sign(x) * (np.abs(x - t) >= 0.5)).astype(np.int64)


def keys(p, cell):
    """(int)std::round(x / cell) per axis of float points (pointcloud_rgbd.cpp:464-469)"""
    return std_round(np.asarray(p, np.float32).astype(np.float64) / cell)


def kd_dist(a, b):
    """KD_TREE::calc_dist in float: (dx*dx + dy*dy) + dz*dz"""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    d = a - b
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def sqrt_f(d):
    """sqrt of a float distance: float, then widened for the comparison with a double"""
    return np.sqrt(np.asarray(d, F32)).astype(np.float64)


def is_face_ok(uv):
    """is_face_is_ok (mesh_rec_geometry.cpp:31-57): the argument is overwritten with 150, so every face -- hull faces included --
    is dropped when an apex angle acos(cos) * 57.3 exceeds 150 (compute_angle :22-29).  Returns (ok, the three cosines)."""
    cs = []
    for a, b, c in ((0, 1, 2), (1, 0, 2), (2, 0, 1)):
        ab, ac = uv[b] - uv[a], uv[c] - uv[a]
        cs.append((ab[0] * ac[0] + ab[1] * ac[1]) / (math.sqrt(ab[0] ** 2 + ab[1] ** 2) * math.sqrt(ac[0] ** 2 + ac[1] ** 2)))
    ok = True
    for c in cs:
        if -1.0 <= c <= 1.0 and math.acos(c) * 57.3 > 150:
            ok = False
    return ok, cs


def pca_axes(P):
    """delaunay_triangulation's frame (mesh_rec_geometry.cpp:190-213): centre, covariance / n, eigenvectors of the two smallest
    eigenvalues, signs from the first two rows, long = short x mid"""
    P = np.asarray(P, np.float64)
    c = P.mean(axis=0)
    D = P - c
    C = (D.T @ D) / float(len(P))
    w, U = np.linalg.eigh(C)
    s, m = U[:, 0].copy(), U[:, 1].copy()
    if D[0] @ s < 0:
        s = -s
    if D[1] @ m < 0:
        m = -m
    return c, D, C, w, s, m, np.cross(s, m)


def triangulate(P, ids):
    """delaunay_triangulation on the dilated set (ids ascending, P their raw positions): projected points (d.l, d.m), their Delaunay
    triangulation (scipy/Qhull), the 150-degree filter.  Returns a dict with the kept faces as sorted id triples, the frame, the
    projected points, the Qhull result and the faces' cosines (for the exclusion bounds of the checks)."""
    c, D, C, w, s, m, l = pca_axes(P)
    uv = np.stack([D @ l, D @ m], 1)
    out = dict(centre=c, D=D, C=C, ev=w, short=s, uv=uv, faces=set(), simplices=None, coplanar=False, dropped_hull=0, dropped_inner=0)
    try:
        tri = Delaunay(uv)
    except QhullError:
        out["coplanar"] = True
        return out
    out["simplices"] = tri.simplices
    out["coplanar"] = len(tri.coplanar) > 0
    hull = set(np.unique(tri.convex_hull).tolist())
    for f in tri.simplices:
        ok, _ = is_face_ok(uv[f])
        if not ok:
            if any(int(i) in hull for i in f):
                out["dropped_hull"] += 1
            else:
                out["dropped_inner"] += 1
            continue
        out["faces"].add(tuple(sorted(int(ids[i]) for i in f)))
    return out


def orientation(sm, tri, cam, short):
    """correct_triangle_index (mesh_rec_geometry.cpp:399-433) on the smoothed positions sm of the sorted triple: n = ab x ac
    (normalised; (0, 0, 1) when zero), the short axis re-signed toward the camera, flip = !(s.n < 0).  Returns (flip, s.n, s.(cam - a))"""
    a, b, c = (np.asarray(sm[i], np.float64) for i in tri)
    n = np.cross(b - a, c - a)
    nn = math.sqrt(n @ n)
    n = n / nn if nn != 0 else np.array([0.0, 0.0, 1.0])
    s = np.asarray(short, np.float64).copy()
    sc = s @ (np.asarray(cam, np.float64) - a)
    if sc < 0:
        s = -s
    sn = s @ n
    return int(not (sn < 0)), sn, sc


class MeshReference:
    """The mesher's own state that numpy carries across frames: the voxels (key -> [meshing_times, new_added_pts_count]) and the
    smoothed positions.  Everything else -- the vertices, the xi-cell occupancy, each voxel's points and the live triangles -- is
    read from the implementation's store before every frame (predict)."""

    def __init__(self, xi, res, append_target):
        self.xi, self.res, self.target = float(xi), float(res), int(append_target)
        self.vox = {}
        self.smooth = np.zeros((0, 3))
        self.smoothed = np.zeros(0, bool)

    # ------------------------------------------------------------------ 1. append (pointcloud_rgbd.cpp:411-552)
    def append(self, V, pts, stats):
        """the greedy insertion of the examined points of one frame into the store V (float[nv][3]).  Returns (new positions,
        examined voxel keys, per-examined-point decision: 0 cell rejected, 1 distance rejected, 2 appended)."""
        n = len(pts)
        step = max(1, int(n // self.target))      # std::round of an integer division (ImMesh_mesh_reconstruction.cpp:111)
        ex = np.asarray(pts, F32)[::step]
        gk, vk = keys(ex, self.xi), keys(ex, self.res)
        nv = len(V)
        occupied = {tuple(k) for k in keys(V, self.xi).tolist()} if nv else set()
        # candidates against the vertices of earlier frames: every vertex whose float distance could be below xi
        near_old = [[] for _ in range(len(ex))]
        if nv:
            tree = cKDTree(np.asarray(V, np.float64))
            for i, js in enumerate(tree.query_ball_point(ex.astype(np.float64), self.xi * (1 + 1e-5) + 1e-9)):
                near_old[i] = js
        acc_by_cell = {}           # xi-cell -> accepted in-frame position, for the in-frame nearest test
        new_pos, decision = [], np.zeros(len(ex), np.int8)
        min_margin = np.inf
        for i in range(len(ex)):
            g = tuple(gk[i].tolist())
            if g in occupied:
                decision[i] = 0
                continue
            # nearest vertex closer than xi (:507-517): the kd-tree holds the earlier frames' vertices and this frame's appends
            close = False
            cand = [V[j] for j in near_old[i]]
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    for dz in (-1, 0, 1):
                        q = acc_by_cell.get((g[0] + dx, g[1] + dy, g[2] + dz))
                        if q is not None:
                            cand.append(q)
            if cand:
                d = sqrt_f(kd_dist(ex[i], np.asarray(cand, F32)))
                min_margin = min(min_margin, float(np.abs(d - self.xi).min()))
                close = bool((d < self.xi).any())
            if close:
                decision[i] = 1
                continue
            decision[i] = 2
            occupied.add(g)
            acc_by_cell[g] = ex[i]
            new_pos.append(ex[i])
        stats["xi_margin"] = min(stats.get("xi_margin", np.inf), min_margin)
        return np.asarray(new_pos, F32).reshape(-1, 3), vk, decision

    # ------------------------------------------------------------------ the frame
    def predict(self, V, T, flips, pts, cam, stats):
        """One frame from the implementation's pre-frame store: V float[nv][3], T int[nt][3] sorted live triples, flips int[nt].
        Returns a dict: new vertex positions, the counts, the meshed voxels, the post-frame triangle set with flips and, per
        meshed voxel, its dilated set and triangulation (for the exclusions of the checks)."""
        V = np.asarray(V, F32)
        nv0 = len(V)
        new, vk, decision = self.append(V, pts, stats)
        stats["cell_reject"] = stats.get("cell_reject", 0) + int((decision == 0).sum())
        stats["dist_reject"] = stats.get("dist_reject", 0) + int((decision == 1).sum())
        Vn = np.concatenate([V, new]) if len(new) else V
        nv = len(Vn)
        # the voxels: created for every examined point, accepted or not (:482-495); an append resets meshing_times (:537-541)
        vk_list = [tuple(k) for k in vk.tolist()]
        new_vk = [vk_list[i] for i in np.nonzero(decision == 2)[0]]
        for k in vk_list:
            self.vox.setdefault(k, [0, 0])
        for k in new_vk:
            self.vox[k][1] += 1
            self.vox[k][0] = 0
        # each voxel's points (m_pts_in_grid, append order = id order)
        allk = keys(Vn, self.res)
        members = {}
        for i, k in enumerate(map(tuple, allk.tolist())):
            members.setdefault(k, []).append(i)
        # smoothed positions: set_pos writes the raw position (pointcloud_rgbd.cpp:59-66)
        sm = np.zeros((nv, 3))
        sm[:len(self.smooth)] = self.smooth
        sm[len(self.smooth):] = Vn[len(self.smooth):].astype(np.float64)
        smoothed = np.zeros(nv, bool)
        smoothed[:len(self.smoothed)] = self.smoothed
        # 2. activation (ImMesh_mesh_reconstruction.cpp:129-151; the recently visited set holds this frame's voxels only,
        #    m_recent_visited_voxel_activated_time = 0, ImMesh_node.cpp:272)
        visited = sorted(set(vk_list))
        meshed = []
        for k in visited:
            r = self.vox[k]
            if r[0] >= 1 or r[1] < 0:
                stats["visited_not_meshed"] = stats.get("visited_not_meshed", 0) + 1
                continue
            r[0] += 1                                  # incremented before the points test
            r[1] = 0
            if len(members.get(k, ())) < 3:
                stats["few_points_marked"] = stats.get("few_points_marked", 0) + 1
                continue
            meshed.append(k)
        # 3. dilation and smoothing (mesh_rec_geometry.cpp:336-377) of every meshed voxel, before any triangulation
        tree = cKDTree(Vn.astype(np.float64)) if nv else None
        accept = self.res * 1.25
        per_vox = {}
        for k in meshed:
            q = members[k]
            idx, dd = self._knn20(tree, Vn, q)
            dist = sqrt_f(dd)
            S = set()
            for r, v in enumerate(q):
                ok = idx[r] >= 0
                S.update(idx[r][ok & (dist[r] < accept)].tolist())
                near = ok & (dist[r] < accept * 2)
                sm[v] = Vn[idx[r][near]].astype(np.float64).sum(axis=0) / float(near.sum())
                smoothed[v] = True
            ids = np.array(sorted(S), np.int64)
            reach = any(tuple(kk) != k for kk in allk[ids].tolist())
            stats["dilation_reaches_neighbour"] = stats.get("dilation_reaches_neighbour", 0) + int(reach)
            per_vox[k] = dict(ids=ids, knn_d=dist[idx >= 0])
        # 4. triangulation, 5. pull / commit, 6. orientation
        T = np.asarray(T, np.int64).reshape(-1, 3)
        live = {tuple(t): i for i, t in enumerate(T.tolist())}
        inc = {}
        for i, t in enumerate(T.tolist()):
            for v in t:
                inc.setdefault(v, []).append(i)
        removed, flip_set = set(), {}
        for k in meshed:
            pv = per_vox[k]
            ids = pv["ids"]
            n = len(ids)
            cls = "warp" if n <= 96 else ("block256" if n <= 256 else ("block1024" if n <= 1024 else "cap"))
            stats.setdefault("size_class", {}).setdefault(cls, 0)
            stats["size_class"][cls] += 1
            tri = triangulate(Vn[ids], ids)
            stats["drop_hull"] = stats.get("drop_hull", 0) + tri["dropped_hull"]
            stats["drop_inner"] = stats.get("drop_inner", 0) + tri["dropped_inner"]
            pv["tri"] = tri
            Sset = set(ids.tolist())
            # find_relative_triangulation_combination (triangle.hpp:224-246): live triangles with all three ids in S
            pulled = set()
            for v in ids.tolist():
                for t in inc.get(v, ()):
                    tt = tuple(T[t].tolist())
                    if tt[0] in Sset and tt[1] in Sset and tt[2] in Sset:
                        pulled.add(tt)
            # triangle_compare (mesh_rec_geometry.cpp:137-172)
            faces = tri["faces"]
            add, keep, rem = faces - pulled, faces & pulled, pulled - faces
            pv.update(add=add, keep=keep, rem=rem)
            removed |= rem
            for t in sorted(add | keep):
                f, sn, sc = orientation(sm, t, cam, tri["short"])
                flip_set.setdefault(t, []).append((k, f, sn, sc))
        # 7. push (ImMesh_mesh_reconstruction.cpp:227-244): every removal, then every insertion; a kept triangle is re-flipped in place
        out_tris = {}
        for t, i in live.items():
            if t not in removed:
                out_tris[t] = int(flips[i])
        pre_flip = {t: int(flips[i]) for t, i in live.items()}
        claims = {}
        for t, lst in flip_set.items():
            if t in removed:
                continue                    # kept by one voxel, removed by another: removed
            k, f, sn, sc = max(lst, key=lambda e: e[0])
            out_tris[t] = f
            claims[t] = lst
            if len(lst) > 1:
                stats["claimed_twice"] = stats.get("claimed_twice", 0) + 1
            if t in pre_flip and pre_flip[t] != f:
                stats["kept_flip_changed"] = stats.get("kept_flip_changed", 0) + 1
            if any(not smoothed[v] for v in t):
                stats["flip_from_unsmoothed"] = stats.get("flip_from_unsmoothed", 0) + 1
        stats["removed_pre_frame"] = stats.get("removed_pre_frame", 0) + len(removed)
        for k in meshed:      # a voxel that had been meshed with >= 3 points, meshed again because a point was appended to it
            before = sum(v < nv0 for v in members[k])
            stats["remeshed_after_new_point"] = stats.get("remeshed_after_new_point", 0) + int(3 <= before < len(members[k]))
        self.smooth, self.smoothed = sm, smoothed
        return dict(new=new, nv=nv, n_voxels=len(self.vox), n_activated=len(visited), meshed=meshed, tris=out_tris, claims=claims,
                    per_vox=per_vox, removed=removed, smooth=sm, smoothed=smoothed, V=Vn)

    @staticmethod
    def _knn20(tree, V, q, k=20):
        """KD_TREE::Nearest_Search(pt, 20): the 20 nearest vertices by the float metric, ties to the lower id.  Candidates come
        from scipy's kd-tree (float64 distances) with a margin, and are re-ranked by the exact float metric."""
        nv = len(V)
        kk = min(nv, k + 12)
        while True:
            d64, cand = tree.query(V[q].astype(np.float64), k=kk)
            cand = np.asarray(cand).reshape(len(q), kk)
            d64 = np.asarray(d64).reshape(len(q), kk)
            df = kd_dist(V[q][:, None, :], V[cand])
            order = np.lexsort((cand, df), axis=1)
            cs = np.take_along_axis(cand, order, 1)[:, :k]
            ds = np.take_along_axis(df, order, 1)[:, :k]
            if kk == nv or bool((np.sqrt(ds[:, -1].astype(np.float64)) * (1 + 1e-5) < d64[:, -1]).all()):
                break
            kk = min(nv, kk * 2)
        if cs.shape[1] < k:
            cs = np.concatenate([cs, -np.ones((len(q), k - cs.shape[1]), np.int64)], 1)
            ds = np.concatenate([ds, np.full((len(q), k - ds.shape[1]), np.inf, F32)], 1)
        return cs, ds
