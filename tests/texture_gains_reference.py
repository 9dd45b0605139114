"""Independent numpy restatement of immesh_mesh_texture_gains' rule as include/immesh_b200.h states it: the 10 barycentric sample points
in the row's face order, the nearest-pixel samples of the chosen side (the row's uv scaled by the bake's rule 1) and of every observer
that sees the facet by texture_select's steps 1-3 (tests/texture_reference.py's visibility and the "seen" test restated here), the
clipping of 0 and 255, the exact int64 pair sums in ascending (k, c), the per-channel normal equations, solved directly with
scipy.sparse.linalg.spsolve (independent of the call's conjugate gradients), and immesh_texture_apply_gains' rounding.  Float64 in the
order the rule writes it.  TEST INFRASTRUCTURE."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.linalg import spsolve

from texture_bake_reference import scaled
from texture_reference import corners, coverage, raster_R
from view_reference import _project

POINTS = [(i, j, 6 - i - j) for i in range(1, 5) for j in range(1, 6 - i)]


def samples(img, p):
    """uint8 [m, 10, 3]: the nearest-pixel samples of img [H, W, 3] at the 10 points of scaled corners p [m, 6]"""
    img = np.asarray(img)
    H, W = img.shape[:2]
    out = np.zeros((len(p), len(POINTS), 3), np.uint8)
    for s, (i, j, l) in enumerate(POINTS):
        b0, b1, b2 = i / 6.0, j / 6.0, l / 6.0
        x = np.floor(((b0 * p[:, 0] + b1 * p[:, 2]) + b2 * p[:, 4]) + 0.5)
        y = np.floor(((b0 * p[:, 1] + b1 * p[:, 3]) + b2 * p[:, 5]) + 0.5)
        x = np.clip(x, 0.0, W - 1.0).astype(np.int64)
        y = np.clip(y, 0.0, H - 1.0).astype(np.int64)
        out[:, s] = img[y, x]
    return out


def seen(cam, verts, tris, flips, z_near, z_far, min_cos, min_visible_permille, two_sided):
    """bool [nt]: texture_select's steps 1-3 for one camera (texture_reference.camera dict), and uv float32 [nt, 6] of the corners"""
    R, t, w, h = raster_R(cam["R"]), cam["t"], cam["width"], cam["height"]
    tris = np.asarray(tris, np.int64).reshape(-1, 3)
    nt = len(tris)
    won, cov = coverage(cam["K"], w, h, z_near, z_far, R, t, verts, tris)
    Q = corners(verts, tris, flips).astype(np.float64)
    u, v, _ = _project(cam["K"], R, t, Q.reshape(-1, 3))
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
    ok = in_img & (won >= 1) & (1000 * won >= min_visible_permille * cov) & side & angle
    uv = np.zeros((nt, 6), np.float32)
    uv[:, 0::2] = u.astype(np.float32)
    uv[:, 1::2] = v.astype(np.float32)
    return ok, uv


def pairs(cams, images, facet_cam, facet_uv, verts, tris, flips, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False):
    """(pair_cam int32 [m, 2], pair_sums int64 [m, 7], used, clipped): cams texture_reference.camera dicts, images [n_cams] uint8 or None,
    rows in snapshot order over tris / flips and the drawn positions verts"""
    cam = np.asarray(facet_cam, np.int64).reshape(-1)
    uv = np.asarray(facet_uv, np.float32).reshape(-1, 6)
    n_cams = len(cams)
    wh = lambda k: (np.array([[images[k].shape[1], images[k].shape[0]]]), np.array([[cams[k]["width"], cams[k]["height"]]]))
    chosen = np.zeros((len(cam), len(POINTS), 3), np.uint8)
    for c in np.unique(cam[cam >= 0]):
        rows = np.nonzero(cam == c)[0]
        iw, sw = wh(c)
        chosen[rows] = samples(images[c], scaled(uv[rows], np.repeat(iw, len(rows), 0), np.repeat(sw, len(rows), 0)))
    pc, ps, used, clipped = [], [], 0, 0
    for k in range(n_cams):
        if images[k] is None or len(cam) == 0:
            continue
        ok, ouv = seen(cams[k], verts, tris, flips, z_near, z_far, min_cos, min_visible_permille, two_sided)
        rows = np.nonzero(ok & (cam >= 0) & (cam != k))[0]
        iw, sw = wh(k)
        obs = samples(images[k], scaled(ouv[rows], np.repeat(iw, len(rows), 0), np.repeat(sw, len(rows), 0))) if len(rows) else np.zeros((0, 10, 3), np.uint8)
        ch = chosen[rows]
        bad = ((obs == 0) | (obs == 255) | (ch == 0) | (ch == 255)).any(axis=2)   # [m, 10]
        clipped += int(bad.sum())
        used += int((~bad).sum())
        for c in range(n_cams):
            m = cam[rows] == c
            keep = ~bad[m]
            n = int(keep.sum())
            if n == 0:
                continue
            Sk = obs[m].astype(np.int64)[keep].sum(axis=0)
            Sc = ch[m].astype(np.int64)[keep].sum(axis=0)
            pc.append((k, c))
            ps.append([n, *Sk, *Sc])
    return np.array(pc, np.int32).reshape(-1, 2), np.array(ps, np.int64).reshape(-1, 7), used, clipped


def solve(n_cams, pair_cam, pair_sums, sigma_n=10.0, sigma_g=0.1):
    """float64 [n_cams, 3]: the normal equations of every channel solved directly (a camera in no pair: g = 1)"""
    sn2, sg2 = sigma_n * sigma_n, sigma_g * sigma_g
    g = np.ones((n_cams, 3))
    inp = np.zeros(n_cams, bool)
    inp[np.asarray(pair_cam, np.int64).reshape(-1)] = True
    for ch in range(3):
        rows, cols, vals = [], [], []
        rhs = np.where(inp, 0.0, 1.0)
        for k in np.nonzero(~inp)[0]:
            rows.append(k); cols.append(k); vals.append(1.0)
        for (a, b), s in zip(np.asarray(pair_cam).reshape(-1, 2), np.asarray(pair_sums).reshape(-1, 7)):
            n, Sa, Sb = float(s[0]), float(s[1 + ch]), float(s[4 + ch])
            rows += [a, b, a, b]
            cols += [a, b, b, a]
            off = -((Sa * Sb / n) / sn2)
            vals += [(Sa * Sa / n) / sn2 + n / sg2, (Sb * Sb / n) / sn2 + n / sg2, off, off]
            rhs[a] += n / sg2
            rhs[b] += n / sg2
        A = coo_matrix((vals, (rows, cols)), shape=(n_cams, n_cams)).tocsc()
        g[:, ch] = np.atleast_1d(spsolve(A, rhs))
    return g


def apply_gains(img, g):
    """uint8 [H, W, 3]: min(255, floor(v g + 0.5)) per channel"""
    return np.minimum(255.0, np.floor(np.asarray(img, np.float64) * np.asarray(g, np.float64).reshape(1, 1, 3) + 0.5)).astype(np.uint8)
