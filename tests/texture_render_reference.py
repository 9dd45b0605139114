"""Independent numpy restatement of immesh_mesh_render_textured's pixel rule and counts as include/immesh_b200.h states it: the OpenCV view
as the rasteriser's camera, immesh_mesh_render_view's visibility (integer samples, the edge-function cover, affine 1/z, the (z_near,
z_far) skip, the nearest depth bits then the lower (a, b, c) triple), the winner's weights e_i / z_i in stored order permuted into its
row's face order, the row's uv scaled to its image by the bake's rule 1, the perspective-correct source point, the bake's clamp-to-edge
bilinear sample, and the integer score against a truth image.  Float64 in the order the rule writes it.  TEST INFRASTRUCTURE."""
import numpy as np

from texture_bake_reference import scaled
from texture_reference import raster_R
from view_reference import INF_BITS, _edges, _project


def visibility(K, w, h, z_near, z_far, R, t, verts, tris):
    """(depth bits uint32 [h, w], winner int64 [h, w], -1 where no triangle has a sample) over the drawn float32 positions verts"""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    best = np.full((h, w), INF_BITS, np.uint32)
    ba = np.full((h, w), np.iinfo(np.int64).max, np.int64)
    bb, bc = ba.copy(), ba.copy()
    win = np.full((h, w), -1, np.int64)
    if len(tris) == 0:
        return best, win
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
        sl = (slice(y0, y1 + 1), slice(x0, x1 + 1))
        a, b, c = tri
        tie = (a < ba[sl]) | ((a == ba[sl]) & ((b < bb[sl]) | ((b == bb[sl]) & (c < bc[sl]))))
        better = cov & ((bits < best[sl]) | ((bits == best[sl]) & tie))
        best[sl] = np.where(better, bits, best[sl])
        ba[sl] = np.where(better, a, ba[sl])
        bb[sl] = np.where(better, b, bb[sl])
        bc[sl] = np.where(better, c, bc[sl])
        win[sl] = np.where(better, k, win[sl])
    return best, win


def bilinear(img, x, y):
    """uint8 [n, 3]: the bake's rule 6 sample of img [H, W, 3] at float64 points (x, y), clamped to the image"""
    img = np.asarray(img)
    H, W = img.shape[:2]
    x = np.clip(x, 0.0, float(W - 1))
    y = np.clip(y, 0.0, float(H - 1))
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    I = img.astype(np.float64)
    top = (1.0 - fx) * I[y0, x0] + fx * I[y0, x1]
    bot = (1.0 - fx) * I[y1, x0] + fx * I[y1, x1]
    return np.floor(((1.0 - fy) * top + fy * bot) + 0.5).astype(np.uint8)


def render_textured(view, sel_wh, images, facet_cam, facet_uv, verts, tris, flips, z_near=0.1, z_far=1000.0, truth=None,
                    untextured=(128, 128, 128), background=(0, 0, 0)):
    """view: texture_reference.camera(...); sel_wh [n_cams, 2] the cameras' sizes; images [n_cams] uint8 [H, W, 3] or None (None as a
    whole: the query); rows facet_cam [nt], facet_uv [nt, 6] in snapshot order over tris / flips and the drawn positions verts.
    Returns dict(rgb uint8 [h, w, 3] (None for the query), depth float32 [h, w], facet int32 [h, w], needed uint8 [n_cams],
    counts int64 [8])"""
    K, w, h = view["K"], view["width"], view["height"]
    R, t = raster_R(view["R"]), view["t"]
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    cam = np.asarray(facet_cam, np.int64).reshape(-1)
    uv = np.asarray(facet_uv, np.float32).reshape(-1, 6)
    flips = np.asarray(flips).reshape(-1) != 0
    n_cams = len(sel_wh)
    best, win = visibility(K, w, h, z_near, z_far, R, t, verts, tris)
    val = best.view(np.float32)
    depth = np.where(val.astype(np.float64) < z_far * 0.99, val, np.float32(-1.0))
    k_of = np.where(win >= 0, cam[np.maximum(win, 0)] if len(cam) else -1, -1)
    tex = k_of >= 0
    needed = np.zeros(n_cams, np.uint8)
    needed[np.unique(k_of[tex])] = 1
    counts = np.zeros(8, np.int64)
    counts[0], counts[1], counts[2], counts[3] = tex.sum(), ((win >= 0) & ~tex).sum(), (win < 0).sum(), needed.sum()
    out = dict(rgb=None, depth=depth, facet=win.astype(np.int32), needed=needed, counts=counts)
    if images is None:
        return out
    rgb = np.zeros((h, w, 3), np.uint8)
    rgb[win < 0] = np.asarray(background, np.uint8)
    rgb[(win >= 0) & ~tex] = np.asarray(untextured, np.uint8)
    ys, xs = np.nonzero(tex)
    if len(ys):
        rows = win[ys, xs]
        ks = k_of[ys, xs]
        u, v, zc = _project(K, R, t, verts[tris[rows]].reshape(-1, 3))
        u, v, zc = u.reshape(-1, 3), v.reshape(-1, 3), zc.reshape(-1, 3)
        e0, e1, e2 = _edges(u.T, v.T, xs.astype(np.float64), ys.astype(np.float64))
        w0, w1, w2 = e0 * (1.0 / zc[:, 0]), e1 * (1.0 / zc[:, 1]), e2 * (1.0 / zc[:, 2])
        f = flips[rows]
        o0, o1, o2 = w0, np.where(f, w1, w2), np.where(f, w2, w1)
        img_wh = np.array([(1, 1) if im is None else (im.shape[1], im.shape[0]) for im in images], np.int64)
        p = scaled(uv[rows], img_wh[ks], np.asarray(sel_wh, np.int64).reshape(-1, 2)[ks])
        s = (o0 + o1) + o2
        x = ((o0 * p[:, 0] + o1 * p[:, 2]) + o2 * p[:, 4]) / s
        y = ((o0 * p[:, 1] + o1 * p[:, 3]) + o2 * p[:, 5]) / s
        for k in np.unique(ks):
            m = ks == k
            rgb[ys[m], xs[m]] = bilinear(images[k], x[m], y[m])
    out["rgb"] = rgb
    if truth is not None:
        d = rgb[tex].astype(np.int64) - np.asarray(truth)[tex].astype(np.int64)
        counts[4:7] = (d * d).sum(axis=0)
        counts[7] = np.abs(d).sum()
    return out
