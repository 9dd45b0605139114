"""Independent numpy restatement of immesh_mesh_texture_bake's atlas rule as include/immesh_b200.h states it: the corners scaled to each
image, the cell class from the longest edge, the stable (class descending, camera ascending) order with two rows per cell, the Morton
placement of 8 x 8-texel units on pages, and each owned texel's clamped barycentrics and bilinear sample, float64 in the order the rule
writes it.  Also the slot geometry the property checks use.  TEST INFRASTRUCTURE."""
import functools

import numpy as np

MIN_CLASS, MAX_CLASS = 3, 13


def scaled(uv, img_wh, sel_wh):
    """float64 [n, 6]: rule 1, uv [n, 6] in the selection camera's pixels to image pixels; img_wh / sel_wh [n, 2]"""
    p = np.asarray(uv, np.float32).astype(np.float64).reshape(-1, 6).copy()
    W, H = img_wh[:, 0:1].astype(np.float64), img_wh[:, 1:2].astype(np.float64)
    Ws, Hs = sel_wh[:, 0:1].astype(np.float64), sel_wh[:, 1:2].astype(np.float64)
    p[:, 0::2] = ((p[:, 0::2] + 0.5) * W) / Ws - 0.5
    p[:, 1::2] = ((p[:, 1::2] + 0.5) * H) / Hs - 0.5
    return p


def cell_class(p, max_cell):
    """int [n]: rule 2, log2 of the smallest power of two >= 8 and >= ceil(L) + 4, capped at max_cell"""
    L = np.zeros(len(p))
    for k in range(3):
        e = (k + 1) % 3
        du, dv = p[:, 2 * e] - p[:, 2 * k], p[:, 2 * e + 1] - p[:, 2 * k + 1]
        L = np.maximum(L, np.sqrt(du * du + dv * dv))
    need = np.ceil(L) + 4.0
    cls = np.full(len(p), MIN_CLASS, np.int64)
    for c in range(MIN_CLASS + 1, MAX_CLASS + 1):
        s = float(1 << (c - 1))
        cls = np.where((cls == c - 1) & (s < need) & (s < max_cell), c, cls)
    return cls


def slot_triangle(S, slot):
    """the slot's triangle corners [(x, y)] * 3 in a cell of side S (rule 4)"""
    if slot == 0:
        return [(0, 0), (S - 4, 0), (0, S - 4)]
    return [(S - 2, S - 2), (2, S - 2), (S - 2, 2)]


@functools.lru_cache(maxsize=None)
def owner(S):
    """int [S, S] indexed [j, i]: the slot that owns each texel of a cell (read-only)"""
    j, i = np.mgrid[0:S, 0:S]
    o = np.where(i + j <= S - 2, 0, 1)
    o.flags.writeable = False
    return o


def morton(off):
    """(x, y) of unit offsets: the even bits and the odd bits"""
    off = np.asarray(off, np.int64)
    x, y = np.zeros_like(off), np.zeros_like(off)
    for b in range(MAX_CLASS):
        x |= ((off >> (2 * b)) & 1) << b
        y |= ((off >> (2 * b + 1)) & 1) << b
    return x, y


def layout(sel_wh, img_wh, facet_cam, facet_uv, page_size, max_cell):
    """rules 1-5.  Returns dict(page int32[n] (-1 untextured), uv float32[n, 6] (NaN untextured), slots: list of (row, page, ox, oy, S,
    slot, cam) in sorted order, n_pages, counts [textured, untextured, cells, texels], p: the scaled corners [n, 6])"""
    cam = np.asarray(facet_cam, np.int64).reshape(-1)
    n = len(cam)
    rows = np.nonzero(cam >= 0)[0]
    sel_wh, img_wh = np.asarray(sel_wh, np.int64).reshape(-1, 2), np.asarray(img_wh, np.int64).reshape(-1, 2)
    p = np.full((n, 6), np.nan)
    page = np.full(n, -1, np.int32)
    auv = np.full((n, 6), np.nan, np.float32)
    if len(rows) == 0:
        return dict(page=page, uv=auv, slots=[], n_pages=0, counts=np.array([0, n, 0, 0], np.int64), p=p)
    p[rows] = scaled(np.asarray(facet_uv, np.float32).reshape(-1, 6)[rows], img_wh[cam[rows]], sel_wh[cam[rows]])
    cls = cell_class(p[rows], max_cell)
    key = ((MAX_CLASS - cls) << 27) | cam[rows]
    order = rows[np.argsort(key, kind="stable")]
    cls_of = dict(zip(rows.tolist(), cls.tolist()))
    U = (page_size // 8) ** 2
    slots, off, cells, texels = [], 0, 0, 0
    by_class = {c: [] for c in range(MIN_CLASS, MAX_CLASS + 1)}
    for r in order.tolist():
        by_class[cls_of[r]].append(r)
    for c in range(MAX_CLASS, MIN_CLASS - 1, -1):
        members = by_class[c]
        S, area = 1 << c, (1 << (c - MIN_CLASS)) ** 2
        for q, r in enumerate(members):
            o = off + (q // 2) * area
            x, y = morton(o % U)
            slots.append((r, o // U, 8 * int(x), 8 * int(y), S, q % 2, int(cam[r])))
            texels += int((owner(S) == q % 2).sum())
        m = (len(members) + 1) // 2
        off += m * area
        cells += m
    for r, pg, ox, oy, S, slot, _ in slots:
        page[r] = pg
        auv[r] = np.array([v for xy in slot_triangle(S, slot) for v in (ox + xy[0], oy + xy[1])], np.float32)
    return dict(page=page, uv=auv, slots=slots, n_pages=-(-off // U), counts=np.array([len(rows), n - len(rows), cells, texels], np.int64), p=p)


def texels(img, p, S, slot):
    """uint8 [S, S, 3] of one slot (rule 6) from image img [H, W, 3] and scaled corners p [6]; texels of the other slot are 0"""
    img = np.asarray(img)
    H, W = img.shape[:2]
    j, i = np.mgrid[0:S, 0:S]
    T = float(S - 4)
    if slot == 0:
        w1, w2 = i.astype(np.float64) / T, j.astype(np.float64) / T
    else:
        w1, w2 = (S - 2 - i).astype(np.float64) / T, (S - 2 - j).astype(np.float64) / T
    a, b = np.maximum(w1, 0.0), np.maximum(w2, 0.0)
    s = a + b
    over = s > 1.0
    a = np.where(over, a / np.where(over, s, 1.0), a)
    b = np.where(over, b / np.where(over, s, 1.0), b)
    w0 = (1.0 - a) - b
    x = (w0 * p[0] + a * p[2]) + b * p[4]
    y = (w0 * p[1] + a * p[3]) + b * p[5]
    x = np.clip(x, 0.0, float(W - 1))
    y = np.clip(y, 0.0, float(H - 1))
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    fx, fy = (x - x0)[..., None], (y - y0)[..., None]
    I = img.astype(np.float64)
    top = (1.0 - fx) * I[y0, x0] + fx * I[y0, x1]
    bot = (1.0 - fx) * I[y1, x0] + fx * I[y1, x1]
    v = (1.0 - fy) * top + fy * bot
    out = np.floor(v + 0.5).astype(np.uint8)
    out[owner(S) != slot] = 0
    return out


def bake(sel_wh, images, facet_cam, facet_uv, page_size=4096, max_cell=64):
    """the whole call: images [n_cams] of uint8 [H, W, 3] (None where unused).  layout()'s dict plus pages uint8 [n_pages, P, P, 3]"""
    img_wh = [(1, 1) if im is None else (im.shape[1], im.shape[0]) for im in images]
    out = layout(sel_wh, img_wh, facet_cam, facet_uv, page_size, max_cell)
    P = page_size
    pages = np.zeros((out["n_pages"], P, P, 3), np.uint8)
    for r, pg, ox, oy, S, slot, k in out["slots"]:
        t = texels(images[k], out["p"][r], S, slot)
        mine = owner(S) == slot
        cell = pages[pg, oy:oy + S, ox:ox + S]
        cell[mine] = t[mine]
    out["pages"] = pages
    return out
