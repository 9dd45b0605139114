"""Shared driver of tests/test_mesh_reference_{emu,gpu}.py: mesher frames of an implementation under test (the CUDA library through
the C ABI, or the host emulation of its kernel bodies) against tests/mesh_reference.py, the independent numpy restatement.

One-step form: before every frame numpy reads the implementation's store (vertices, live triangles, flips) and predicts the frame
from it with its own voxel counters and its own smoothed positions, so a decision excluded in one frame cannot carry into the next.

Compared after every frame:
* the vertices (positions and ids): exact;
* the counts of immesh_mesh_counts (mesh_capi.cu), exact: n_vertices (vertex counter, IM_MC_VERTICES), frame_new_vertices (this
  frame's appends, IM_MC_NEW_VERTICES), n_voxels (mesh voxels ever created, IM_MC_VOXELS: a voxel is created by every examined point,
  appended or not), n_activated (distinct voxels of this frame's examined points, IM_MC_ACT), frame_voxels_meshed (work-list length
  IM_MC_WORK_FRONT + IM_MC_WORK_BACK: activated voxels that passed the meshing-times test and hold at least 3 points);
* the set of meshed voxels (where the implementation exposes it: the emulation's work list): exact;
* the live facet set and the flips: exact outside the exclusions below.

Exclusions (a voxel's triangulation, or one flip, whose decision is closer to its threshold than the rounding between the two sides
can move it):
* kNN and append decisions need none: both sides take them on the same float distance ((dx*dx + dy*dy) + dz*dz, then sqrtf),
  so they are compared exactly (and numpy reports the smallest |sqrtf(d) - xi| it met, which must exceed one float ulp of xi);
* a voxel's projected points may differ by delta = the snap unit res 2^-22 + |D|max tau_s + 64 eps |centre|, where tau_s =
  64 eps (||C|| + |centre| |D|max) / (lambda_1 - lambda_0) bounds the short axis's error (Davis-Kahan on the covariance C of
  the dilated set about its centre).  The voxel is excluded when Qhull reports coplanar points or fails, when a face's doubled area
  is below 4 delta times its perimeter, when an interior edge's Delaunay margin pi - (alpha + beta) is below
  2 delta (1/l1 + 1/l2 + 1/l3 + 1/l4) over the four edges of its two triangles (an apex angle moves by at most
  2 delta (1/la + 1/lb) when each of its three points moves by delta), when a point lies within 4 delta of a hull edge's
  line next to the edge, or when an apex angle acos(cos) 57.3 lies within 2 57.3 delta (1/l1 + 1/l2) of 150;
  it removes from the comparison the triangles with all three vertices in its dilated set, in that frame only;
* one flip is excluded when |s.n| <= tau_s + e (|ab| + |ac| + |bc|) 4 / |ab x ac| or |s.(cam - a)| <= tau_s |cam - a| + 4 e, with
  e = 64 eps max|x| the tolerance carried on the smoothed positions (their summation order is not pinned).
"""
import ctypes as C

import numpy as np

import mesh_reference as ref
from immesh_b200 import api

EPS = np.finfo(np.float64).eps
MAX_EXCLUDED = 5e-3


def f32_ulp(x):
    return float(np.spacing(np.float32(abs(x))))


def voxel_bounds(tri, res):
    """(delta, tau_s) of one voxel's triangulation (module docstring)"""
    D, C, ev, c = tri["D"], tri["C"], tri["ev"], tri["centre"]
    dmax = float(np.sqrt((D * D).sum(1)).max())
    cmag = float(np.abs(c).max())
    gap = float(ev[1] - ev[0])
    tau = 64 * EPS * (np.linalg.norm(C) + cmag * dmax) / gap if gap > 0 else np.inf
    delta = res * 2.0 ** -22 + dmax * tau + 64 * EPS * cmag
    return delta, tau


def voxel_excluded(tri, res):
    """True when the voxel's triangulation could differ between the two sides (module docstring)"""
    if tri["coplanar"] or tri["simplices"] is None:
        return True
    delta, tau = voxel_bounds(tri, res)
    if not np.isfinite(delta):
        return True
    uv, S = tri["uv"], tri["simplices"]
    edges = {}
    for fi, f in enumerate(S):
        p = uv[f]
        L = [np.linalg.norm(p[(j + 2) % 3] - p[(j + 1) % 3]) for j in range(3)]     # L[j]: edge opposite vertex j
        area2 = abs((p[1, 0] - p[0, 0]) * (p[2, 1] - p[0, 1]) - (p[1, 1] - p[0, 1]) * (p[2, 0] - p[0, 0]))
        if area2 <= 4 * delta * sum(L):
            return True
        for j in range(3):
            a, b = p[(j + 1) % 3] - p[j], p[(j + 2) % 3] - p[j]
            la, lb = np.linalg.norm(a), np.linalg.norm(b)
            cosv = float(np.clip(a @ b / (la * lb), -1, 1))
            ang = np.arccos(cosv)
            if abs(ang * 57.3 - 150) <= 2 * 57.3 * delta * (1 / la + 1 / lb) * 2:
                return True
            e = tuple(sorted((int(f[(j + 1) % 3]), int(f[(j + 2) % 3]))))
            edges.setdefault(e, []).append((ang, 1 / la + 1 / lb))
    for e, lst in edges.items():
        if len(lst) == 2:
            margin = np.pi - (lst[0][0] + lst[1][0])
            if margin <= 2 * delta * (lst[0][1] + lst[1][1]):
                return True
        else:   # hull edge: no other point may lie near its line beside the edge
            a, b = uv[e[0]], uv[e[1]]
            ab = b - a
            L2 = ab @ ab
            t = (uv - a) @ ab / L2
            dist = np.abs((uv[:, 0] - a[0]) * ab[1] - (uv[:, 1] - a[1]) * ab[0]) / np.sqrt(L2)
            near = (t > -0.1) & (t < 1.1) & (dist <= 4 * delta)
            near[list(e)] = False
            if near.any():
                return True
    return False


def flip_excluded(V, sm, t, cam, tau, sn, sc):
    p = np.asarray(sm, np.float64)[list(t)]
    e = 64 * EPS * max(float(np.abs(p).max()), 1.0)
    ab, ac, bc = p[1] - p[0], p[2] - p[0], p[2] - p[1]
    cr = np.linalg.norm(np.cross(ab, ac))
    if cr == 0:
        return True
    bn = tau + e * (np.linalg.norm(ab) + np.linalg.norm(ac) + np.linalg.norm(bc)) * 4 / cr
    bc_ = tau * np.linalg.norm(np.asarray(cam, np.float64) - p[0]) + 4 * e
    return abs(sn) <= bn or abs(sc) <= bc_


def _tri_dict(T, Fl):
    return {tuple(int(x) for x in t): int(f) for t, f in zip(np.asarray(T).reshape(-1, 3), np.asarray(Fl))}


def frame_voxels(lib, h):
    """the emulation's meshed voxels of the last frame"""
    n = lib.emu_mesh_frame_voxels(h._h, None)
    k = np.zeros((max(n, 1), 3), np.int32)
    lib.emu_mesh_frame_voxels(h._h, k.ctypes.data_as(C.c_void_p))
    return {tuple(r) for r in k[:n].tolist()}


def smooth_state(lib, h):
    nv = h.counts()["n_vertices"]
    f = np.zeros(nv, np.uint8)
    s = np.zeros((nv, 3))
    lib.emu_mesh_smooth_state(h._h, f.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p))
    return f.astype(bool), s


def check_stream(lib, frames, cfg, emu=False, push=None, xi_ties=False):
    """frames: list of (float32[n][3] world points, camera position).  push(h, pts, cam, k): how a frame enters the
    implementation (default push_frame).  xi_ties: the stream is built with append distances of exactly xi (no margin
    assertion).  Returns the statistics (branches reached, excluded and compared counts, the numpy
    reference and the handle)."""
    h = api.Mesh(cfg, lib=lib)
    R = ref.MeshReference(cfg.points_minimum_scale, cfg.voxel_resolution, cfg.number_of_pts_append_to_map)
    st = dict(meshed=0, excluded=0, flips_compared=0, flips_excluded=0, tris_compared=0)
    for k, (pts, cam) in enumerate(frames):
        V, T, Fl = h.snapshot()
        pred = R.predict(V, T, Fl, pts, cam, st)
        (push or (lambda hh, p, c, i: hh.push_frame(p, c, i)))(h, pts, cam, k)
        cg = h.counts()
        want = dict(n_vertices=pred["nv"], frame_new_vertices=len(pred["new"]), n_voxels=pred["n_voxels"],
                    n_activated=pred["n_activated"], frame_voxels_meshed=len(pred["meshed"]))
        got = {kk: cg[kk] for kk in want}
        assert got == want, f"frame {k}: counts {got} vs numpy {want}"
        V2, T2, F2 = h.snapshot()
        assert np.array_equal(V2[:len(V)], V) and np.array_equal(V2[len(V):], pred["new"]), f"frame {k}: vertices"
        if emu:
            assert frame_voxels(lib, h) == set(pred["meshed"]), f"frame {k}: meshed voxels"
            fl, sv = smooth_state(lib, h)
            assert np.array_equal(fl, pred["smoothed"]), f"frame {k}: smoothed flags"
            s = pred["smoothed"]
            tol = 16 * EPS * np.maximum(np.abs(pred["smooth"][s]), 1.0)
            assert (np.abs(sv[s] - pred["smooth"][s]) <= tol).all(), f"frame {k}: smoothed positions"
        # exclusions
        res = cfg.voxel_resolution
        skip_sets, tau_of = [], {}
        for vk in pred["meshed"]:
            pv = pred["per_vox"][vk]
            st["meshed"] += 1
            tau_of[vk] = voxel_bounds(pv["tri"], res)[1] if pv["tri"]["simplices"] is not None else np.inf
            if voxel_excluded(pv["tri"], res):
                st["excluded"] += 1
                skip_sets.append(set(pv["ids"].tolist()))

        def skipped(t):
            return any(t[0] in s and t[1] in s and t[2] in s for s in skip_sets)

        got_t = {t: f for t, f in _tri_dict(T2, F2).items() if not skipped(t)}
        want_t = {t: f for t, f in pred["tris"].items() if not skipped(t)}
        missing, extra = set(want_t) - set(got_t), set(got_t) - set(want_t)
        assert not missing and not extra, f"frame {k}: facet set: {len(missing)} missing {sorted(missing)[:5]}, {len(extra)} extra {sorted(extra)[:5]}"
        st["tris_compared"] += len(got_t)
        for t, f in want_t.items():
            if t in pred["claims"]:
                vk, _, sn, sc = max(pred["claims"][t], key=lambda e: e[0])
                if flip_excluded(pred["V"], pred["smooth"], t, cam, tau_of[vk], sn, sc):
                    st["flips_excluded"] += 1
                    continue
            st["flips_compared"] += 1
            assert got_t[t] == f, f"frame {k}: flip of {t}: {got_t[t]} vs numpy {f}"
    if not xi_ties:
        assert st["xi_margin"] > f32_ulp(cfg.points_minimum_scale), st["xi_margin"]
    assert st["excluded"] <= MAX_EXCLUDED * st["meshed"], (st["excluded"], st["meshed"])
    st["ref"], st["handle"] = R, h
    return st


def end_smooth_check(h, R):
    """GPU: the smoothed positions at the end of a stream, through one all-regions region_buffers call (it smooths only vertices whose
    flag is clear, which numpy's flags name): rows whose three vertices numpy has smoothed equal (float) of numpy's value to 1 ulp."""
    xyz, ids, _, _, _ = h.region_buffers()
    s = R.smoothed
    rows = s[ids].all(1)
    want = R.smooth[ids[rows]].reshape(-1, 9).astype(np.float32)
    got = xyz[rows]
    assert (np.abs(got.astype(np.float64) - want) <= np.spacing(np.abs(want)).astype(np.float64)).all()
    return int(rows.sum())


def stream(kind, n_frames, seed, n_points=None, offset=(0.0, 0.0, 0.0)):
    """world-frame frames with the sensor position as the camera; offset translates points and camera"""
    from mesh_common import world_scans
    off = np.asarray(offset, np.float64)
    return [((w.astype(np.float64) + off).astype(np.float32), np.asarray(t, np.float64) + off) for w, t in world_scans(kind, n_frames, seed, n_points)]


def scene_frames(scene):
    pose = scene.centre + np.array([0.3, -0.2, 1.5])
    return [(p, pose) for p in scene.frames]


BRANCHES = ("cell_reject", "dist_reject", "visited_not_meshed", "remeshed_after_new_point", "few_points_marked",
            "dilation_reaches_neighbour", "drop_hull", "drop_inner", "removed_pre_frame", "kept_flip_changed", "claimed_twice",
            "flip_from_unsmoothed")


def merge(tot, st):
    for b in BRANCHES:
        tot[b] = tot.get(b, 0) + st.get(b, 0)
    for c, v in st.get("size_class", {}).items():
        tot.setdefault("size_class", {})[c] = tot.get("size_class", {}).get(c, 0) + v
    for c in ("meshed", "excluded", "flips_compared", "flips_excluded", "tris_compared"):
        tot[c] = tot.get(c, 0) + st[c]
    return tot
