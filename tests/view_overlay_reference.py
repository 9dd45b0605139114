"""Independent numpy restatement of the queued view's overlay rule as include/immesh_b200.h states it for immesh_mesh_view_overlay:
points of size s, segments clipped in camera space and widened as GL's non-antialiased lines, the wireframe's edges in the vertex
colours, the frustum, axis, grid and trajectory geometry, and the layered visibility (depth bits, then draw order, then index)
against the faces of view_reference.render.  Float64 in the order the rule writes it, so the bytes agree.  TEST INFRASTRUCTURE."""
import numpy as np

from view_reference import INF_BITS, _edges, _project, heat, render, z_range_of

SCAN, REINFORCED, AXIS, GRID, MESH, CAMERA, PATH = range(7)
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
FRUSTUM_K = (704.504153913163, 703.6790228113778, 708.8501128392297, 562.7041625276061)   # fx, fy, cx, cy of the reference's frustum


def _cam(R, t, P):
    """camera-frame coordinates (x right, y down, z forward) of world points P [n, 3]"""
    d = np.asarray(P, np.float64).reshape(-1, 3) - t
    xc = (R[0, 0] * d[:, 0] + R[1, 0] * d[:, 1]) + R[2, 0] * d[:, 2]
    yc = -((R[0, 1] * d[:, 0] + R[1, 1] * d[:, 1]) + R[2, 1] * d[:, 2])
    zc = -((R[0, 2] * d[:, 0] + R[1, 2] * d[:, 1]) + R[2, 2] * d[:, 2])
    return np.stack([xc, yc, zc], axis=1)


def key_of(zf, layer, idx):
    bits = np.asarray(zf, np.float32).view(np.uint32).astype(np.uint64)
    return (bits << np.uint64(32)) | (np.uint64(layer) << np.uint64(29)) | np.asarray(idx, np.uint64)


def points(K, w, h, zn, zf, R, t, P, size):
    """fragments (x, y, zf, idx) of points P [n, 3] of size `size`"""
    fx, fy, cx, cy = K
    c = _cam(R, t, P)
    idx = np.nonzero((c[:, 2] > zn) & (c[:, 2] < zf))[0]
    c = c[idx]
    u = fx * c[:, 0] / c[:, 2] + cx
    v = fy * c[:, 1] / c[:, 2] + cy
    hs = size * 0.5
    out = []
    for oy in range(size + 2):
        y = np.ceil(v - hs) + oy
        for ox in range(size + 2):
            x = np.ceil(u - hs) + ox
            ok = (x < u + hs) & (y < v + hs) & (x >= 0) & (y >= 0) & (x < w) & (y < h)
            out.append((x[ok].astype(np.int64), y[ok].astype(np.int64), c[ok, 2].astype(np.float32), idx[ok]))
    return [np.concatenate(a) for a in zip(*out)] if out else [np.zeros(0, np.int64)] * 4


def clip(K, zn, zf, R, t, p0, p1):
    """the segment p0 -> p1 clipped to [zn, zf] in camera space and projected: (u0, v0, iz0, u1, v1, iz1), or None"""
    a, b = _cam(R, t, np.array([p0, p1], np.float64))
    a, b = a.copy(), b.copy()
    if not (a[2] >= zn or b[2] >= zn) or not (a[2] <= zf or b[2] <= zf):
        return None

    def move(p, q, zp):
        s = (zp - p[2]) / (q[2] - p[2])
        p[0] = p[0] + s * (q[0] - p[0])
        p[1] = p[1] + s * (q[1] - p[1])
        p[2] = zp
    if a[2] < zn:
        move(a, b, zn)
    elif b[2] < zn:
        move(b, a, zn)
    if a[2] > zf:
        move(a, b, zf)
    elif b[2] > zf:
        move(b, a, zf)
    fx, fy, cx, cy = K
    return (fx * a[0] / a[2] + cx, fy * a[1] / a[2] + cy, 1.0 / a[2], fx * b[0] / b[2] + cx, fy * b[1] / b[2] + cy, 1.0 / b[2])


def line(seg, width, w, h):
    """fragments (x, y, zf, t) of a projected segment of width `width` (GL's non-antialiased wide line)"""
    u0, v0, iz0, u1, v1, iz1 = seg
    xm = abs(u1 - u0) >= abs(v1 - v0)
    m0, m1, n0, n1 = (u0, u1, v0, v1) if xm else (v0, v1, u0, u1)
    mlim, nlim = (w, h) if xm else (h, w)
    lo, hi = min(m0, m1), max(m0, m1)
    start = max(np.ceil(lo), 0.0)
    end = min(hi, float(mlim))
    if not start < end:
        return [np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0)]
    m = np.arange(start, end, 1.0)
    m = m[m < end]
    tt = (m - m0) / (m1 - m0)
    n = n0 + tt * (n1 - n0)
    z = (1.0 / (iz0 + tt * (iz1 - iz0))).astype(np.float32)
    hw = width * 0.5
    xs, ys, zs, ts = [], [], [], []
    for o in range(width + 2):
        k = np.maximum(np.ceil(n - hw), 0.0) + o
        ok = (k < n + hw) & (k < nlim)
        a, b = m[ok].astype(np.int64), k[ok].astype(np.int64)
        xs.append(a if xm else b)
        ys.append(b if xm else a)
        zs.append(z[ok])
        ts.append(tt[ok])
    return [np.concatenate(v) for v in (xs, ys, zs, ts)]


def axis_segments():
    return [(np.zeros(3), np.eye(3)[k]) for k in range(3)]


def grid_segments():
    out = []
    for i in range(21):
        c = 10.0 * (i - 10)
        out.append((np.array([c, -100.0, 0.0]), np.array([c, 100.0, 0.0])))
        out.append((np.array([-100.0, c, 0.0]), np.array([100.0, c, 0.0])))
    return out


def frustum(R, t, cs):
    """[11, 3] world vertices of the camera frustum of rot_end R, pos_end t at camera size cs"""
    fx, fy, cx, cy = FRUSTUM_K
    s = 1.5
    fu, u0, fv, v0 = 1.0 / fx, -cx / fx, 1.0 / fy, -cy / fy
    xl, xh, yl, yh = s * u0, s * (1440.0 * fu + u0), s * v0, s * (1080.0 * fv + v0)
    loc = [(xl, yl, s), (xh, yl, s), (xh, yh, s), (xl, yh, s), (xl, yl, s), (0, 0, 0), (xh, yl, s), (0, 0, 0), (xl, yh, s), (0, 0, 0), (xh, yh, s)]
    R = np.asarray(R, np.float64)
    out = np.zeros((11, 3))
    for i, (x, y, z) in enumerate(loc):
        for k in range(3):
            out[i, k] = t[k] + cs * ((-R[k, 1] * x + -R[k, 2] * y) + R[k, 0] * z)
    return out


def face_bits(K, w, h, zn, zf, R, t, verts, tris):
    """the faces' winning depth bits per pixel (INF_BITS: none), the visibility of view_reference.render"""
    best = np.full((h, w), INF_BITS, np.uint32)
    verts = np.asarray(verts, np.float32)
    for tri in np.asarray(tris, np.int64).reshape(-1, 3):
        u, v, zc = _project(K, R, t, verts[tri])
        if not np.all((zc > zn) & (zc < zf)):
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
            z = (1.0 / iz).astype(np.float32)
        cov &= (z > 0) & (z.view(np.uint32) < INF_BITS)
        sl = (slice(y0, y1 + 1), slice(x0, x1 + 1))
        best[sl] = np.where(cov, np.minimum(best[sl], z.view(np.uint32)), best[sl])
    return best


def wireframe(K, w, h, zn, zf, R, t, verts, tris, color=False, z_range=None):
    """(rgb uint8 [h, w, 3], best bits [h, w]) of the live triangles' edges"""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    big = np.iinfo(np.int64).max
    best = np.full((h, w), INF_BITS, np.uint32)
    rank = np.full((h, w, 4), big, np.int64)   # a, b, c, edge
    rgb = np.zeros((h, w, 3), np.uint8)
    if color:
        lo, hi = z_range_of(verts, tris) if z_range is None else (np.float32(z_range[0]), np.float32(z_range[1]))
    _, _, zv = _project(K, R, t, verts) if len(verts) else (None, None, np.zeros(0))
    for tri in tris:
        if not np.all((zv[tri] > zn) & (zv[tri] < zf)):
            continue
        u, v, zc = _project(K, R, t, verts[tri])
        col = heat(verts[tri, 2], lo, hi).astype(np.float64) / 255.0 if color else np.ones((3, 3))
        for e, (i, j) in enumerate(((0, 1), (1, 2), (0, 2))):
            x, y, z, tt = line((u[i], v[i], 1.0 / zc[i], u[j], v[j], 1.0 / zc[j]), 1, w, h)
            bits = z.view(np.uint32)
            r = np.array([tri[0], tri[1], tri[2], e])
            cur, cr = best[y, x], rank[y, x]
            tie = np.zeros(len(x), bool)
            decided = np.zeros(len(x), bool)
            for q in range(4):
                lt, ne = r[q] < cr[:, q], r[q] != cr[:, q]
                tie |= ~decided & lt
                decided |= ne
            better = (bits < INF_BITS) & ((bits < cur) | ((bits == cur) & tie))
            x, y, bits, tt = x[better], y[better], bits[better], tt[better]
            best[y, x] = bits
            rank[y, x] = r
            w0, w1 = (1.0 - tt) * (1.0 / zc[i]), tt * (1.0 / zc[j])
            for k in range(3):
                c = (w0 * col[i, k] + w1 * col[j, k]) / (w0 + w1)
                rgb[y, x, k] = np.floor(np.where(c > 0.0, np.where(c < 1.0, c, 1.0), 0.0) * 255.0 + 0.5).astype(np.uint8)
    return rgb, best


def overlay_keys(K, w, h, zn, zf, R, t, scan=None, scan_size=0, rf=None, rf_size=0, axis_and_grid=False, frustum_pose=None, camera_size=0.0,
                 path=(), path_width=0):
    """[h, w] uint64: the minimum key over every overlay fragment (NONE: none).  path: the kept positions, oldest first."""
    keys = np.full(h * w, NONE, np.uint64)

    def put(x, y, z, layer, idx):
        if len(x):
            np.minimum.at(keys, y * w + x, key_of(z, layer, idx))
    for P, size, layer in ((scan, scan_size, SCAN), (rf, rf_size, REINFORCED)):
        if P is not None and size > 0 and len(P):
            x, y, z, idx = points(K, w, h, zn, zf, R, t, P, size)
            put(x, y, z, layer, idx)
    segs = []
    if axis_and_grid:
        segs += [(AXIS, k, 10, a, b) for k, (a, b) in enumerate(axis_segments())]
        segs += [(GRID, k, 1, a, b) for k, (a, b) in enumerate(grid_segments())]
    if frustum_pose is not None and camera_size > 0:
        F = frustum(frustum_pose[0], frustum_pose[1], camera_size)
        segs += [(CAMERA, k, 5, F[k], F[k + 1]) for k in range(10)]
    if path_width > 0:
        segs += [(PATH, k, path_width, np.asarray(path[k], np.float64), np.asarray(path[k + 1], np.float64)) for k in range(len(path) - 1)]
    for layer, idx, width, a, b in segs:
        s = clip(K, zn, zf, R, t, a, b)
        if s is None:
            continue
        x, y, z, _ = line(s, width, w, h)
        put(x, y, z, layer, np.full(len(x), idx))
    return keys.reshape(h, w)


def key_colors(keys):
    """rgb uint8 [h, w, 3] of the overlay keys' layers"""
    layer = ((keys >> np.uint64(29)) & np.uint64(7)).astype(np.int64)
    idx = (keys & np.uint64((1 << 29) - 1)).astype(np.int64)
    rgb = np.full(keys.shape + (3,), 255, np.uint8)
    rgb[layer == REINFORCED] = (255, 0, 255)
    for k in range(3):
        sel = (layer == AXIS) & (idx == k)
        rgb[sel] = 0
        rgb[sel, k] = 255
    rgb[layer == GRID] = 115
    return rgb


def render_overlay(K, w, h, zn, zf, R, t, verts, tris, color=False, z_range=None, wire=False, **ov):
    """(rgba, depth) of the queued view with overlays: the faces (view_reference.render) or the wireframe, and the overlay keys"""
    R = np.asarray(R, np.float64)
    t = np.asarray(t, np.float64)
    rgba, depth = render(K, w, h, zn, zf, R, t, verts, tris, color, z_range)
    if wire:
        rgb, mesh_bits = wireframe(K, w, h, zn, zf, R, t, verts, tris, color, z_range)
        rgba[..., :3] = rgb
    else:
        mesh_bits = face_bits(K, w, h, zn, zf, R, t, verts, tris)
    keys = overlay_keys(K, w, h, zn, zf, R, t, **ov)
    kb = (keys >> np.uint64(32)).astype(np.uint32)
    kl = ((keys >> np.uint64(29)) & np.uint64(7)).astype(np.int64)
    over = (keys != NONE) & ((kb < mesh_bits) | ((kb == mesh_bits) & (kl < MESH)))
    rgba[over, :3] = key_colors(keys)[over]
    return rgba, depth
