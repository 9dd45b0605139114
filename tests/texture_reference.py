"""Independent numpy restatement of immesh_mesh_texture_select's selection rule as include/immesh_b200.h states it: the OpenCV camera
as the rasteriser's (columns 1 and 2 of cam_R negated), immesh_mesh_render_view's visibility per pixel (integer samples, the
edge-function cover, affine 1/z, the (z_near, z_far) skip, the nearest depth bits then the lower (a, b, c) triple), the covered and
won pixels per facet, the "seen" test, the nearest camera (smallest |e|^2, the lower index on a tie) and the texture coordinates.
Float64 in the order the rule writes it.  Also a reader of immesh_write_obj_textured's OBJ / MTL pair.  TEST INFRASTRUCTURE."""
import numpy as np

from view_reference import _edges, _project

INF_BITS = np.uint32(0x7F800000)


def raster_R(cam_R):
    """the rasteriser's rotation (world = R diag(1,-1,-1) p + t) of an OpenCV camera-to-world rotation"""
    R = np.asarray(cam_R, np.float64).reshape(3, 3).copy()
    R[:, 1] = -R[:, 1]
    R[:, 2] = -R[:, 2]
    return R


def corners(verts, tris, flips):
    """float32 [nt, 3, 3]: q0 q1 q2 of every facet in immesh_write_ply's face order (flip != 0: p0 p1 p2, else p0 p2 p1)"""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    f = np.asarray(flips).reshape(-1) != 0
    order = np.where(f[:, None], tris, tris[:, [0, 2, 1]])
    return verts[order]


def coverage(K, w, h, z_near, z_far, R, t, verts, tris):
    """(won, covered) int64 [nt]: the pixels each facet wins and the pixels where it has a sample"""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    nt = len(tris)
    covered = np.zeros(nt, np.int64)
    best = np.full((h, w), INF_BITS, np.uint32)
    ba = np.full((h, w), np.iinfo(np.int64).max, np.int64)
    bb, bc = ba.copy(), ba.copy()
    win = np.full((h, w), -1, np.int64)
    if nt == 0:
        return np.zeros(0, np.int64), covered
    _, _, zv = _project(K, R, t, verts)
    inside = (zv > z_near) & (zv < z_far)
    for k in np.nonzero(inside[tris].all(axis=1))[0]:
        tri = tris[k]
        u, v, zc = _project(K, R, t, verts[tri])
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
        bits = zf.view(np.uint32)
        cov &= (zf > 0) & (bits < INF_BITS)
        covered[k] = int(cov.sum())
        sl = (slice(y0, y1 + 1), slice(x0, x1 + 1))
        a, b, c = tri
        tie = (a < ba[sl]) | ((a == ba[sl]) & ((b < bb[sl]) | ((b == bb[sl]) & (c < bc[sl]))))
        better = cov & ((bits < best[sl]) | ((bits == best[sl]) & tie))
        best[sl] = np.where(better, bits, best[sl])
        ba[sl] = np.where(better, a, ba[sl])
        bb[sl] = np.where(better, b, bb[sl])
        bc[sl] = np.where(better, c, bc[sl])
        win[sl] = np.where(better, k, win[sl])
    won = np.bincount(win[win >= 0], minlength=nt).astype(np.int64)
    return won, covered


def camera(width, height, K, cam_R, cam_t):
    return dict(width=int(width), height=int(height), K=tuple(float(k) for k in K), R=np.asarray(cam_R, np.float64).reshape(3, 3),
                t=np.asarray(cam_t, np.float64).reshape(3))


def select(cams, verts, tris, flips, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False):
    """dict(cam int32 [nt], uv float32 [nt, 6] (NaN where untextured), px int32 [nt, 2], counts int64 [4]) over the drawn float32
    positions verts; cams: camera(...) dicts"""
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    nt = len(tris)
    Q = corners(verts, tris, flips).astype(np.float64)   # [nt, 3 corners, 3]
    best_e2 = np.full(nt, np.inf)
    best = np.full(nt, -1, np.int64)
    px = np.zeros((nt, 2), np.int64)
    for k, c in enumerate(cams):
        R, t, w, h = raster_R(c["R"]), c["t"], c["width"], c["height"]
        won, cov = coverage(c["K"], w, h, z_near, z_far, R, t, verts, tris)
        if nt == 0:
            continue
        u, v, _ = _project(c["K"], R, t, Q.reshape(-1, 3))
        u, v = u.reshape(nt, 3), v.reshape(nt, 3)
        in_img = ((u >= 0.0) & (u <= w - 1.0) & (v >= 0.0) & (v <= h - 1.0)).all(axis=1)
        g = ((Q[:, 0] + Q[:, 1]) + Q[:, 2]) / 3.0
        e = t - g
        a, b = Q[:, 1] - Q[:, 0], Q[:, 2] - Q[:, 0]
        n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2], a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)
        s = (n[:, 0] * e[:, 0] + n[:, 1] * e[:, 1]) + n[:, 2] * e[:, 2]
        nn = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
        ee = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
        side = (s != 0.0) if two_sided else (s > 0.0)
        with np.errstate(over="ignore", invalid="ignore"):
            angle = s * s >= (min_cos * min_cos) * (nn * ee)
        seen = in_img & (won >= 1) & (1000 * won >= min_visible_permille * cov) & side & angle
        take = seen & (ee < best_e2)
        best_e2[take] = ee[take]
        best[take] = k
        px[take, 0] = won[take]
        px[take, 1] = cov[take]
    uv = np.full((nt, 6), np.nan, np.float32)
    for k in np.unique(best[best >= 0]):
        c = cams[k]
        rows = np.nonzero(best == k)[0]
        u, v, _ = _project(c["K"], raster_R(c["R"]), c["t"], Q[rows].reshape(-1, 3))
        uv[rows, 0::2] = u.reshape(-1, 3).astype(np.float32)
        uv[rows, 1::2] = v.reshape(-1, 3).astype(np.float32)
    textured = int((best >= 0).sum())
    pixels = sum(c["width"] * c["height"] for c in cams)
    counts = np.array([textured, nt - textured, len(np.unique(best[best >= 0])), pixels], np.int64)
    return dict(cam=best.astype(np.int32), uv=uv, px=px.astype(np.int32), counts=counts)


def read_obj(obj_path, mtl_path):
    """(v float64 [nv, 3], vt float64 [m, 2], groups: list of (material, faces int64 [f, 3] 0-based, tex int64 [f, 3] 0-based or None),
    mtllib name, materials: dict name -> map_Kd or None) of an OBJ / MTL pair"""
    v, vt, groups, mtllib = [], [], [], None
    for line in open(obj_path):
        p = line.split()
        if not p or p[0] == "#":
            continue
        if p[0] == "mtllib":
            mtllib = p[1]
        elif p[0] == "v":
            v.append([float(x) for x in p[1:4]])
        elif p[0] == "vt":
            vt.append([float(x) for x in p[1:3]])
        elif p[0] == "usemtl":
            groups.append([p[1], [], []])
        elif p[0] == "f":
            idx = [x.split("/") for x in p[1:]]
            groups[-1][1].append([int(x[0]) - 1 for x in idx])
            groups[-1][2].append([int(x[1]) - 1 for x in idx] if len(idx[0]) > 1 else None)
    out = []
    for name, faces, tex in groups:
        out.append((name, np.array(faces, np.int64).reshape(-1, 3), None if tex[0] is None else np.array(tex, np.int64).reshape(-1, 3)))
    mats, cur = {}, None
    for line in open(mtl_path):
        p = line.split()
        if not p:
            continue
        if p[0] == "newmtl":
            cur = p[1]
            mats[cur] = None
        elif p[0] == "map_Kd":
            mats[cur] = line.strip()[len("map_Kd "):]
    return np.array(v, np.float64).reshape(-1, 3), np.array(vt, np.float64).reshape(-1, 2), out, mtllib, mats
