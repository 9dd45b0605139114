"""Independent numpy restatement of the texturing queued behind every frame (immesh_mesh_texture_enable / _rows) as
include/immesh_b200.h states it: per frame with a camera, texture_reference.py's rule (visibility, won and covered pixels, the "seen"
test) on that frame's live mesh at that frame's camera; the state keyed by the vertex triple, kept for triples that are not live, and
replaced only by a strictly nearer camera; the rig composed with the sensor pose element by element in Python floats.  TEST
INFRASTRUCTURE."""
import numpy as np

from texture_reference import coverage, raster_R
from view_reference import _project


def compose(rig_R, rig_t, R_f, t_f):
    """(R, t) = (R_f R_rig, R_f t_rig + t_f), every entry summed left to right in Python floats"""
    A = [[float(x) for x in row] for row in np.asarray(R_f, np.float64).reshape(3, 3)]
    B = [[float(x) for x in row] for row in np.asarray(rig_R, np.float64).reshape(3, 3)]
    tr = [float(x) for x in np.asarray(rig_t, np.float64).reshape(3)]
    tf = [float(x) for x in np.asarray(t_f, np.float64).reshape(3)]
    R = [[(A[r][0] * B[0][c] + A[r][1] * B[1][c]) + A[r][2] * B[2][c] for c in range(3)] for r in range(3)]
    t = [((A[r][0] * tr[0] + A[r][1] * tr[1]) + A[r][2] * tr[2]) + tf[r] for r in range(3)]
    return np.array(R, np.float64), np.array(t, np.float64)


def frame_camera(rig, frame):
    """(R, t) of a frame dict (caller=(R, t): that camera; pose=(R_f, t_f): the rig on it; neither: None)"""
    if frame.get("caller") is not None:
        R, t = frame["caller"]
        return np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)
    if frame.get("pose") is not None:
        return compose(rig["R"], rig["t"], *frame["pose"])
    return None


def _seen(K, w, h, R, t, Q, won, cov, min_cos, permille, two_sided):
    """(seen bool [n], e2 float64 [n]) of facets with face-order corners Q [n, 3, 3]"""
    n = len(Q)
    u, v, _ = _project(K, raster_R(R), t, Q.reshape(-1, 3))
    u, v = u.reshape(n, 3), v.reshape(n, 3)
    in_img = ((u >= 0.0) & (u <= w - 1.0) & (v >= 0.0) & (v <= h - 1.0)).all(axis=1)
    g = ((Q[:, 0] + Q[:, 1]) + Q[:, 2]) / 3.0
    e = t - g
    a, b = Q[:, 1] - Q[:, 0], Q[:, 2] - Q[:, 0]
    nrm = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)
    s = (nrm[:, 0] * e[:, 0] + nrm[:, 1] * e[:, 1]) + nrm[:, 2] * e[:, 2]
    nn = (nrm[:, 0] * nrm[:, 0] + nrm[:, 1] * nrm[:, 1]) + nrm[:, 2] * nrm[:, 2]
    ee = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
    side = (s != 0.0) if two_sided else (s > 0.0)
    with np.errstate(over="ignore", invalid="ignore"):
        angle = s * s >= (min_cos * min_cos) * (nn * ee)
    return in_img & (won >= 1) & (1000 * won >= permille * cov) & side & angle, ee


def fold(rig, frames, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False):
    """The state after a sequence of frames: dict triple -> (frame, e2, won, covered, uv float32 [6] in stored order), and the pixels
    rasterised.  rig: dict(width, height, K, R, t); frames: dicts of number, verts float32 [nv, 3], tris [n, 3] (the live triples
    at the frame's end, ascending ids), flips [n], and caller / pose as frame_camera reads them."""
    state, pixels = {}, 0
    w, h, K = rig["width"], rig["height"], rig["K"]
    for fr in frames:
        cam = frame_camera(rig, fr)
        tris = np.asarray(fr["tris"], np.int64).reshape(-1, 3)
        if cam is None:
            continue
        pixels += w * h
        if len(tris) == 0:
            continue
        R, t = cam
        verts = np.asarray(fr["verts"], np.float32)
        flips = np.asarray(fr["flips"]).reshape(-1) != 0
        won, cov = coverage(K, w, h, z_near, z_far, raster_R(R), t, verts, tris)
        P = verts[tris].astype(np.float64)                      # stored order
        Q = np.where(flips[:, None, None], P, P[:, [0, 2, 1]])  # face order
        seen, ee = _seen(K, w, h, R, t, Q, won, cov, min_cos, min_visible_permille, two_sided)
        u, v, _ = _project(K, raster_R(R), t, P.reshape(-1, 3))
        uv = np.stack([u.reshape(-1, 3), v.reshape(-1, 3)], axis=2).reshape(-1, 6).astype(np.float32)
        for i in np.nonzero(seen)[0]:
            key = tuple(int(x) for x in tris[i])
            if key not in state or ee[i] < state[key][1]:
                state[key] = (int(fr["number"]), float(ee[i]), int(won[i]), int(cov[i]), uv[i].copy())
    return state, pixels


def rows(state, pixels, tris, flips):
    """texture_rows of the live triples tris [n, 3] (snapshot order) with their current flips: dict(cam, uv (NaN where -1), px,
    counts [4], frames)"""
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    flips = np.asarray(flips).reshape(-1) != 0
    n = len(tris)
    cam = np.full(n, -1, np.int32)
    uv = np.full((n, 6), np.nan, np.float32)
    px = np.zeros((n, 2), np.int32)
    for i in range(n):
        s = state.get(tuple(int(x) for x in tris[i]))
        if s is None:
            continue
        cam[i], px[i] = s[0], (s[2], s[3])
        c = [0, 1, 2] if flips[i] else [0, 2, 1]
        uv[i] = s[4].reshape(3, 2)[c].reshape(6)
    textured = int((cam >= 0).sum())
    counts = np.array([textured, n - textured, len(np.unique(cam[cam >= 0])), pixels], np.int64)
    frames = np.array(sorted({s[0] for s in state.values()}), np.int32)
    return dict(cam=cam, uv=uv, px=px, counts=counts, frames=frames)
