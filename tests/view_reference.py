"""Independent numpy restatement of the shaded view's image rule as include/immesh_b200.h states it for immesh_mesh_render_view: the
depth image's sampling rule pixel by pixel, the nearest sample with the lower (a, b, c) triple on equal depth bits, the facet shading
from the camera position and the height colour's five-stop ramp; and the queued view's camera sources with scipy.  Float64 in the
order the rule writes it, so the bytes and floats agree.  TEST INFRASTRUCTURE."""
import numpy as np

from reinforce_reference import avr_pose

# the height colour's stops: blue, cyan, green, yellow, red
STOPS = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 1.0], [0.0, 1.0, 0.0], [1.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
INF_BITS = np.uint32(0x7F800000)


def heat(z, lo, hi):
    """uint8 [n, 3]: t = (z - lo) / (hi - lo) in float32 (0 when hi == lo), s = clamp(1 - t, 0, 1), the stops floor(4 s) and
    ceil(4 s) mixed linearly, each channel truncated to a byte"""
    z = np.asarray(z, np.float32).reshape(-1)
    lo, hi = np.float32(lo), np.float32(hi)
    val = np.zeros_like(z) if hi == lo else (z - lo) / (hi - lo)
    s = np.clip(1.0 - val.astype(np.float64), 0.0, 1.0)
    a = s * 4.0
    f = a - np.floor(a)
    c = (1.0 - f)[:, None] * STOPS[np.floor(a).astype(int)] + f[:, None] * STOPS[np.ceil(a).astype(int)]
    return np.floor(c * 255.0).astype(np.uint8)


def positions(raw, smooth=None, flags=None, mode=0):
    """the drawn vertex positions (float32): mode 1 takes the smoothed position (as float) where the flag is set"""
    raw = np.asarray(raw, np.float32)
    if mode == 0 or smooth is None:
        return raw.copy()
    sm = np.asarray(smooth, np.float64).astype(np.float32)
    return np.where(np.asarray(flags, bool)[:, None], sm, raw)


def z_range_of(verts, tris):
    """the automatic range: min / max z over the vertices of the triangles"""
    if len(tris) == 0:
        return np.float32(0), np.float32(0)
    z = np.asarray(verts, np.float32)[np.asarray(tris).reshape(-1), 2]
    return z.min(), z.max()


def _project(K, R, t, P):
    fx, fy, cx, cy = K
    d = P.astype(np.float64) - t
    xc = (R[0, 0] * d[:, 0] + R[1, 0] * d[:, 1]) + R[2, 0] * d[:, 2]
    yc = -((R[0, 1] * d[:, 0] + R[1, 1] * d[:, 1]) + R[2, 1] * d[:, 2])
    zc = -((R[0, 2] * d[:, 0] + R[1, 2] * d[:, 1]) + R[2, 2] * d[:, 2])
    return fx * xc / zc + cx, fy * yc / zc + cy, zc


def _edges(u, v, px, py):
    e0 = (u[2] - u[1]) * (py - v[1]) - (v[2] - v[1]) * (px - u[1])
    e1 = (u[0] - u[2]) * (py - v[2]) - (v[0] - v[2]) * (px - u[2])
    e2 = (u[1] - u[0]) * (py - v[0]) - (v[1] - v[0]) * (px - u[0])
    return e0, e1, e2


def _byte(c):
    return np.floor(np.where(c > 0.0, np.where(c < 1.0, c, 1.0), 0.0) * 255.0 + 0.5).astype(np.uint8)


def render(K, w, h, z_near, z_far, R, t, verts, tris, color=False, z_range=None):
    """(rgba uint8 [h, w, 4], depth float32 [h, w]) of the triangles tris (ascending triples) over the drawn positions verts"""
    R = np.asarray(R, np.float64)
    t = np.asarray(t, np.float64)
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    best = np.full((h, w), INF_BITS, np.uint32)
    ba = np.full((h, w), np.iinfo(np.int64).max, np.int64)
    bb, bc = ba.copy(), ba.copy()
    win = np.full((h, w), -1, np.int64)
    if len(tris) == 0:
        cand = []
    else:   # only triangles with every vertex inside (z_near, z_far) can be drawn: the others are skipped below anyway
        _, _, zv = _project(K, R, t, verts)
        inside = (zv > z_near) & (zv < z_far)
        cand = np.nonzero(inside[tris].all(axis=1))[0]
    for k in cand:
        tri = tris[k]
        u, v, zc = _project(K, R, t, verts[tri])
        if not np.all((zc > z_near) & (zc < z_far)):
            continue
        area = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0])
        if area == 0.0:
            continue
        x0, x1 = max(0, int(np.ceil(u.min()))), min(w - 1, int(np.floor(u.max())))
        y0, y1 = max(0, int(np.ceil(v.min()))), min(h - 1, int(np.floor(v.max())))
        if x0 > x1 or y0 > y1:
            continue
        py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.float64)
        e0, e1, e2 = _edges(u, v, px, py)
        cov = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            iz = ((e0 * (1.0 / zc[0]) + e1 * (1.0 / zc[1])) + e2 * (1.0 / zc[2])) / area
            zf = (1.0 / iz).astype(np.float32)
        cov &= zf > 0
        bits = zf.view(np.uint32)
        sl = (slice(y0, y1 + 1), slice(x0, x1 + 1))
        a, b, c = tri
        tie = (a < ba[sl]) | ((a == ba[sl]) & ((b < bb[sl]) | ((b == bb[sl]) & (c < bc[sl]))))
        better = cov & (bits < INF_BITS) & ((bits < best[sl]) | ((bits == best[sl]) & tie))
        best[sl] = np.where(better, bits, best[sl])
        ba[sl] = np.where(better, a, ba[sl])
        bb[sl] = np.where(better, b, bb[sl])
        bc[sl] = np.where(better, c, bc[sl])
        win[sl] = np.where(better, k, win[sl])
    val = best.view(np.float32)
    depth = np.where(val.astype(np.float64) < z_far * 0.99, val, np.float32(-1.0))
    rgba = np.zeros((h, w, 4), np.uint8)
    rgba[..., 3] = 255
    if color:
        lo, hi = z_range_of(verts, tris) if z_range is None else (np.float32(z_range[0]), np.float32(z_range[1]))
    for k in np.unique(win[win >= 0]):
        ys, xs = np.nonzero(win == k)
        P = verts[tris[k]].astype(np.float64)
        u, v, zc = _project(K, R, t, verts[tris[k]])
        e0, e1, e2 = _edges(u, v, xs.astype(np.float64), ys.astype(np.float64))
        w0, w1, w2 = e0 * (1.0 / zc[0]), e1 * (1.0 / zc[1]), e2 * (1.0 / zc[2])
        ws = (w0 + w1) + w2
        ea, eb = P[1] - P[0], P[2] - P[0]
        n = np.array([ea[1] * eb[2] - ea[2] * eb[1], ea[2] * eb[0] - ea[0] * eb[2], ea[0] * eb[1] - ea[1] * eb[0]])
        col = heat(P[:, 2].astype(np.float32), lo, hi).astype(np.float64) / 255.0 if color else np.ones((3, 3))
        l = [t[j] - ((w0 * P[0, j] + w1 * P[1, j]) + w2 * P[2, j]) / ws for j in range(3)]
        cc = [((w0 * col[0, j] + w1 * col[1, j]) + w2 * col[2, j]) / ws for j in range(3)]
        nn = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
        ln = np.sqrt((l[0] * l[0] + l[1] * l[1]) + l[2] * l[2])
        d = ((n[0] / nn) * (l[0] / ln) + (n[1] / nn) * (l[1] / ln)) + (n[2] / nn) * (l[2] / ln)
        s = 0.2 + 0.5 * np.abs(d)
        for j in range(3):
            rgba[ys, xs, j] = _byte(s * cc[j])
    return rgba, depth


def frame_pose(poses, frame, win, mode=0, R_in=None, t_in=None):
    """the queued view's camera of frame `frame`: 0 sensor-bound (avr_pose), 1 fixed (R_in, t_in), 2 follow (R_in at the window's mean
    translation plus t_in; an empty window's translation is zero)"""
    if mode == 1:
        return np.asarray(R_in, np.float64), np.asarray(t_in, np.float64)
    R, t = avr_pose(poses, frame, win)
    if mode == 2:
        return np.asarray(R_in, np.float64), t + np.asarray(t_in, np.float64)
    return R, t
