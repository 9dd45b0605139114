"""Independent numpy / scipy restatement of immesh_mesh_evaluate (include/immesh_b200.h): the paper's Experiment-3 fairness and
correctness metrics of a mesh against a ground-truth cloud.  The sub-triangle lattice is enumerated literally, each leaf is summed
in input order (not np.mean, whose pairwise summation differs), and the nearest neighbour is a cKDTree query for a few candidates,
rechecked with the defined distance so that a near-tie cannot pick a different value."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

QSCALE = 2.0 ** 20
MAX_N = 1 << 15


def fairness(A, B, C):
    """(maxmin deg, c2se, longest, degenerate) per triangle, float64 from float32 corners [m,3]."""
    A, B, C = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (A, B, C))

    def norm(v):
        return np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])

    def cross(u, v):
        return np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2], u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], axis=1)

    def angle(u, v):
        dot = (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]
        return np.degrees(np.arctan2(norm(cross(u, v)), dot))

    ab, ac, bc = B - A, C - A, C - B
    lab, lac, lbc = norm(ab), norm(ac), norm(bc)
    cr = norm(cross(ab, ac))
    deg = cr == 0.0
    a = np.stack([angle(ab, ac), angle(bc, -ab), angle(-ac, -bc)], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        c2se = ((lbc * lac) * lab) / (2.0 * cr) / np.minimum(lab, np.minimum(lac, lbc))
    return a.max(axis=1) - a.min(axis=1), c2se, np.maximum(lab, np.maximum(lac, lbc)), deg


def subdivisions(longest, spacing):
    n = np.ceil(np.asarray(longest) / spacing)
    if np.any(n > MAX_N):
        raise OverflowError("a triangle needs more than 2^15 subdivisions")
    return np.maximum(n, 1).astype(np.int64)


def lattice(n):
    """barycentrics (u, v) float64[n^2] of the n-subdivision's centroids: "up" (i, j < n - i), then "down" (j < n - i - 1), row by row"""
    ij_up = [(i, j) for i in range(n) for j in range(n - i)]
    ij_dn = [(i, j) for i in range(n) for j in range(n - i - 1)]
    i = np.array([p[0] for p in ij_up] + [p[0] for p in ij_dn], dtype=np.float64)
    j = np.array([p[1] for p in ij_up] + [p[1] for p in ij_dn], dtype=np.float64)
    off = np.array([1.0] * len(ij_up) + [2.0] * len(ij_dn))
    return (3.0 * i + off) / (3.0 * n), (3.0 * j + off) / (3.0 * n)


def triangle_samples(A, B, C, n):
    """the n^2 sub-triangle centroids of m triangles with the same n (corners [m,3]), float32[m,n^2,3]"""
    u, v = lattice(n)
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64).reshape(-1, 1, 3) for x in (A, B, C))
    return (a + (u[None, :, None] * (b - a) + v[None, :, None] * (c - a))).astype(np.float32)


def downsample(gt, leaf):
    """one point per occupied leaf, (float)(sum in input order / count); leaves in ascending key order"""
    gt = np.asarray(gt, dtype=np.float32).reshape(-1, 3)
    if leaf == 0 or gt.shape[0] == 0:
        return gt.copy()
    key = np.floor(gt.astype(np.float64) / leaf).astype(np.int64)
    order = np.lexsort((np.arange(gt.shape[0]), key[:, 2], key[:, 1], key[:, 0]))   # by key, then input order
    ks = key[order]
    start = np.ones(len(order), dtype=bool)
    start[1:] = np.any(ks[1:] != ks[:-1], axis=1)
    leaf_id = np.cumsum(start) - 1
    rank = np.arange(len(order)) - np.flatnonzero(start)[leaf_id]
    nl = int(leaf_id[-1]) + 1
    s = np.zeros((nl, 3))
    cnt = np.bincount(leaf_id, minlength=nl)
    p = gt[order].astype(np.float64)
    for r in range(int(rank.max()) + 1):   # the r-th point of every leaf: a sequential sum per leaf
        m = rank == r
        s[leaf_id[m]] += p[m]
    return (s / cnt[:, None]).astype(np.float32)


def dist(q, t):
    q = q.astype(np.float64)
    t = t.astype(np.float64)
    d = q - t
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def nearest(q, t, max_dist, k=4):
    """(d float64[m], far bool[m]): the defined distance to the nearest of t within max_dist, max_dist when none"""
    q = np.asarray(q, dtype=np.float32).reshape(-1, 3)
    t = np.asarray(t, dtype=np.float32).reshape(-1, 3)
    if q.shape[0] == 0:
        return np.zeros(0), np.zeros(0, dtype=bool)
    if t.shape[0] == 0:
        return np.full(q.shape[0], float(max_dist)), np.ones(q.shape[0], dtype=bool)
    k = min(k, t.shape[0])
    tree = cKDTree(t.astype(np.float64))
    _, idx = tree.query(q.astype(np.float64), k=k, distance_upper_bound=max_dist * (1 + 1e-9) + 1e-9)
    idx = np.asarray(idx).reshape(q.shape[0], k)
    valid = idx < t.shape[0]
    tt = t[np.where(valid, idx, 0)]
    d = np.where(valid, dist(q[:, None, :], tt), np.inf).min(axis=1)
    far = ~(d <= max_dist)
    return np.where(far, float(max_dist), d), far


def evaluate(verts, tris, gt, spacing=0.01, gt_leaf=0.01, threshold=0.05, max_dist=1.0, incorrect_ratio=0.8):
    """verts float32[nv,3]; tris int[nt,3] live triangles as ascending triples in ascending order (snapshot()).  Returns
    dict(counts int64[12], metrics float64[8], rows int32[nt,5], samples float32[ns,3], sample_facet int[ns], gt float32[ng,3])."""
    verts = np.asarray(verts, dtype=np.float32).reshape(-1, 3)
    tris = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
    nt = tris.shape[0]
    A, B, C = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    mm, c2, longest, deg = fairness(A, B, C)
    ok = ~deg
    n = np.zeros(nt, dtype=np.int64)
    n[ok] = subdivisions(longest[ok], spacing)
    parts, facet = [], []
    for nn in np.unique(n[ok]):
        ts = np.flatnonzero(ok & (n == nn))
        parts.append(triangle_samples(A[ts], B[ts], C[ts], int(nn)).reshape(-1, 3))
        facet.append(np.repeat(ts, int(nn) ** 2))
    s = np.concatenate(parts) if parts else np.zeros((0, 3), dtype=np.float32)
    sf = np.concatenate(facet) if facet else np.zeros(0, dtype=np.int64)
    order = np.argsort(sf, kind="stable")   # triangle order, each triangle's lattice in order
    s, sf = s[order], sf[order]
    g = downsample(gt, gt_leaf)
    ds, far_s = nearest(s, g, max_dist)
    dg, far_g = nearest(g, s, max_dist)
    ins, ing = ds < threshold, dg < threshold
    f_s = np.bincount(sf, minlength=nt).astype(np.int64)
    f_f = np.bincount(sf[~ins], minlength=nt).astype(np.int64)
    incorrect = int(np.sum((f_s > 0) & (f_f.astype(np.float64) >= incorrect_ratio * f_s.astype(np.float64))))
    counts = np.array([nt, int(deg.sum()), len(s), len(g), int(ins.sum()), int(ing.sum()), int(far_s.sum()), int(far_g.sum()), incorrect,
                       int(np.rint(ds * QSCALE).astype(np.int64).sum()), int(np.rint(dg * QSCALE).astype(np.int64).sum()),
                       int(n.max()) if nt else 0], dtype=np.int64)
    nf = nt - int(deg.sum())
    m = np.full(8, np.nan)
    if nf:
        m[0] = mm[ok].sum() / nf
        m[1] = c2[ok].sum() / nf
    p = counts[4] / counts[2] if counts[2] else np.nan
    r = counts[5] / counts[3] if counts[3] else np.nan
    if counts[2]:
        m[2] = counts[9] / QSCALE / counts[2]
    if counts[3]:
        m[3] = counts[10] / QSCALE / counts[3]
    m[4], m[5] = p, r
    if counts[2] and counts[3]:
        m[6] = 2 * p * r / (p + r) if p + r > 0 else 0.0
    m[7] = 0.0
    rows = np.concatenate([tris, f_s[:, None], f_f[:, None]], axis=1).astype(np.int32) if nt else np.zeros((0, 5), dtype=np.int32)
    return dict(counts=counts, metrics=m, rows=rows, samples=s, sample_facet=sf, gt=g)
