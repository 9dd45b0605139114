"""CPU tier: the oracle against independent implementations (numpy / scipy / brute force).  The reference ships no
golden vectors (parity unpinned, DESIGN.md 2), so these checks are what keeps oracle bugs from being baked in."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial import Delaunay

import oracle_api as oa
from immesh_b200 import api, synth


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_deterministic_libm_subset():
    L = oa.lib()
    x = np.concatenate([np.linspace(-3.1, 3.1, 2001), np.linspace(-1e-3, 1e-3, 101), [0.0, 1.0, -1.0, 0.5, -0.5]])
    s, c, e, ac = (np.zeros_like(x) for _ in range(4))
    L.orc_math_probe(_p(x), C.c_int(x.size), _p(s), _p(c), _p(e), _p(ac))
    assert np.max(np.abs(s - np.sin(x))) < 4e-16
    assert np.max(np.abs(c - np.cos(x))) < 4e-16
    assert np.max(np.abs(e / np.exp(-np.abs(x)) - 1)) < 1e-15
    xc = np.clip(x, -1, 1)
    assert np.max(np.abs(ac - np.arccos(xc))) < 1e-15 * np.pi + 5e-16


def test_jacobi_matches_eigh():
    L = oa.lib()
    rng = np.random.default_rng(0)
    for _ in range(300):
        A = rng.normal(size=(3, 3)) * rng.uniform(1e-3, 10)
        S = A @ A.T
        if rng.random() < 0.3:
            S = S * np.array([1.0, 1e-3, 1e-6])[:, None] * np.array([1.0, 1e-3, 1e-6])[None, :]
        a6 = np.array([S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]])
        d, V = np.zeros(3), np.zeros(9)
        L.orc_jacobi_eig3(_p(a6), _p(d), _p(V))
        V = V.reshape(3, 3)
        w = np.linalg.eigvalsh(S)
        assert np.allclose(np.sort(d), w, rtol=1e-12, atol=1e-14 * abs(w).max())
        assert np.allclose(V @ np.diag(d) @ V.T, S, rtol=1e-12, atol=1e-14 * abs(S).max())
        assert np.allclose(V.T @ V, np.eye(3), atol=1e-14)


def test_lu_inverse18_matches_numpy():
    L = oa.lib()
    rng = np.random.default_rng(1)
    for _ in range(20):
        B = rng.normal(size=(18, 18))
        A = B @ B.T + np.diag(rng.uniform(1e-6, 1e3, 18))
        out = np.zeros((18, 18))
        L.orc_lu_inverse18(_p(np.ascontiguousarray(A)), _p(out))
        assert np.allclose(out @ A, np.eye(18), atol=1e-8)
        assert np.allclose(out, np.linalg.inv(A), rtol=1e-7, atol=1e-10)


def test_voxel_key_rule():
    L = oa.lib()
    # truncation toward zero after the -1.0f shift; exact negative multiples land one cell lower than floor (SURVEY App. C.2)
    cases = [((0.24, 0.26, 0.74), 0.5, (0, 0, 1)), ((-0.01, -0.5, -0.51), 0.5, (-1, -2, -2)), ((-1.0, 1.0, 0.0), 0.5, (-3, 2, 0)), ((3.9999, -3.0, 2.99), 3.0, (1, -2, 0))]
    for p, vs, want in cases:
        out = np.zeros(3, dtype=np.int64)
        L.orc_voxel_key(_p(np.array(p, dtype=np.float64)), C.c_double(vs), _p(out))
        assert tuple(out) == want, (p, vs, tuple(out))


def test_calc_body_var_matches_formula():
    L = oa.lib()
    rng = np.random.default_rng(2)
    for _ in range(100):
        p = rng.normal(size=3) * rng.uniform(1, 50)
        out = np.zeros(6)
        L.orc_calc_body_var(_p(p), 0.02, 0.05, _p(out))
        V = np.array([[out[0], out[1], out[2]], [out[1], out[3], out[4]], [out[2], out[4], out[5]]])
        r = np.float32(np.linalg.norm(p))
        d = p / np.linalg.norm(p)
        hat = np.array([[0, -d[2], d[1]], [d[2], 0, -d[0]], [-d[1], d[0], 0]])
        b1 = np.array([1, 1, -(d[0] + d[1]) / d[2]]); b1 /= np.linalg.norm(b1)
        b2 = np.cross(b1, d); b2 /= np.linalg.norm(b2)
        N = np.stack([b1, b2], 1)
        A = float(r) * hat @ N
        dv = np.sin(float(np.float32(0.05)) * 0.017453293) ** 2
        ref = np.outer(d, d) * float(np.float32(0.02) ** 2) + A @ (np.eye(2) * dv) @ A.T
        assert np.allclose(V, ref, rtol=1e-10, atol=1e-18)


def test_delaunay_matches_qhull():
    rng = np.random.default_rng(3)
    for trial in range(40):
        n = int(rng.integers(3, 300))
        pts = rng.integers(-(1 << 22), 1 << 22, size=(n, 2))
        if trial % 5 == 0:                       # clustered + collinear runs
            pts[: n // 3, 1] = pts[0, 1]
        pts = np.unique(pts, axis=0)
        if len(pts) < 3:
            continue
        rng.shuffle(pts)
        mine = oa.delaunay2d_int(pts)
        try:
            ref = Delaunay(pts.astype(np.float64)).simplices
        except Exception:
            continue
        a = {tuple(sorted(t)) for t in mine.tolist()}
        b = {tuple(sorted(t)) for t in ref.tolist()}
        if a != b:
            # differences can only be co-circular flips or zero-area hull slivers Qhull merges; check the empty-circle property
            P = pts.astype(object)
            for t in a ^ b:
                x = [P[i] for i in t]
                area2 = (x[1][0] - x[0][0]) * (x[2][1] - x[0][1]) - (x[1][1] - x[0][1]) * (x[2][0] - x[0][0])
                assert area2 != 0 or t in b
        for t in mine:                            # every face is counter-clockwise and has an empty circumcircle
            A, B, Cc = (pts[i].astype(object) for i in t)
            assert (B[0] - A[0]) * (Cc[1] - A[1]) - (B[1] - A[1]) * (Cc[0] - A[0]) > 0
        idx = rng.integers(0, len(mine), size=min(30, len(mine)))
        for f in idx:
            A, B, Cc = (pts[i].astype(object) for i in mine[f])
            for q in rng.integers(0, len(pts), size=20):
                D = pts[q].astype(object)
                adx, ady, bdx, bdy, cdx, cdy = A[0] - D[0], A[1] - D[1], B[0] - D[0], B[1] - D[1], Cc[0] - D[0], Cc[1] - D[1]
                det = (adx * adx + ady * ady) * (bdx * cdy - bdy * cdx) + (bdx * bdx + bdy * bdy) * (cdx * ady - cdy * adx) + (cdx * cdx + cdy * cdy) * (adx * bdy - ady * bdx)
                assert det <= 0


def _greedy_append_bruteforce(frames, xi, res, target):
    verts, grid = [], {}
    for pts in frames:
        step = max(1, round(len(pts) // target))
        for i in range(0, len(pts), step):
            p = pts[i]
            g = tuple(int(np.round(np.float64(p[j]) / xi)) for j in range(3))
            if g in grid:
                continue
            if verts:
                V = np.asarray(verts, dtype=np.float32)
                d = V - p
                d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
                if np.sqrt(d2.min()) < xi:
                    continue
            grid[g] = len(verts)
            verts.append(p.copy())
    return np.asarray(verts, dtype=np.float32)


def test_vertex_append_and_knn_match_bruteforce():
    sensor, scans = synth.make_stream("avia", 3, seed=11, n_points=6000)
    frames = [(s["body_full"].astype(np.float64) @ s["R_true"].T + s["t_true"]).astype(np.float32) for s in scans]
    cfg = api.MeshConfig()
    o = oa.OracleMesh(cfg)
    for k, f in enumerate(frames):
        o.push_frame(f, scans[k]["t_true"], k)
    v, tris, flips = o.snapshot()
    ref = _greedy_append_bruteforce(frames, cfg.points_minimum_scale, cfg.voxel_resolution, cfg.number_of_pts_append_to_map)
    assert v.shape == ref.shape and np.array_equal(v, ref)
    # exact kNN, float metric, ties by id
    rng = np.random.default_rng(5)
    q = (v[rng.integers(0, len(v), 64)] + rng.normal(0, 0.1, (64, 3))).astype(np.float32)
    idx, d2 = o.knn(q, 20)
    for i in range(len(q)):
        d = v - q[i]
        dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        order = np.lexsort((np.arange(len(v)), dd))[:20]
        assert np.array_equal(idx[i], order)
        assert np.array_equal(d2[i], dd[order])
    # every live facet has its three vertices within the dilation reach and is stored sorted
    assert np.all(tris[:, 0] < tris[:, 1]) and np.all(tris[:, 1] < tris[:, 2])
    e = np.linalg.norm(v[tris[:, 0]] - v[tris[:, 1]], axis=1)
    assert e.max() < 2 * (1.25 * cfg.voxel_resolution) + cfg.voxel_resolution * 3 ** 0.5 + 1e-3


def test_fixed_point_sums_close_to_serial_double():
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 4, seed=9, ext_T=cfg.ext_T)
    a, b = oa.OracleLio(cfg, sum_mode=0), oa.OracleLio(cfg, sum_mode=1)
    for h in (a, b):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        h.voxel_map_init(scans[0]["body_full"])
    for k in (1, 2, 3):
        for h in (a, b):
            h.lio_state_estimation(scans[k]["body_ds"])
            h.map_incremental_grow(scans[k]["body_ds"])
        ia, ib = a.iter_stats(0), b.iter_stats(0)
        assert np.allclose(ia["HTH"], ib["HTH"], rtol=1e-9, atol=1e-4)
        assert np.allclose(a.get_state()[:12], b.get_state()[:12], rtol=1e-9, atol=1e-10)


def test_ieskf_gain_6x6_form_equals_reference_form():
    """The IESKF update is evaluated through the matrix inversion lemma, K1[:, :6] = P[:, :6] (I + A P11)^-1 (solve_mode 0: what the
    CUDA product computes), instead of the reference's two 18x18 inverses (voxel_mapping.cpp:1588-1592, solve_mode 1).  Same
    stream through both forms: identical iteration counts / match sets, state and covariance within 1e-9 relative; plus the
    solution of one iteration against numpy's literal  (H^T R^-1 H (+) 0 + P^-1)^-1."""
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 6, seed=21, ext_T=cfg.ext_T)
    a, b = oa.OracleLio(cfg, sum_mode=0, solve_mode=0), oa.OracleLio(cfg, sum_mode=0, solve_mode=1)
    for h in (a, b):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        s = h.get_state()
        s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
        h.set_state(s)
        h.voxel_map_init(scans[0]["body_full"])
    for k in range(1, 6):
        for h in (a, b):
            h.predict(scans[k]["dt"])
        prop = a.get_state()
        ia, ib = a.lio_state_estimation(scans[k]["body_ds"]), b.lio_state_estimation(scans[k]["body_ds"])
        assert ia == ib
        assert np.array_equal(a.matches(), b.matches())
        sa, sb = a.get_state(), b.get_state()
        assert np.allclose(sa[:24], sb[:24], rtol=1e-9, atol=1e-12), np.abs(sa[:24] - sb[:24]).max()
        Pa, Pb = sa[24:].reshape(18, 18), sb[24:].reshape(18, 18)
        assert np.abs(Pa - Pb).max() <= 1e-9 * np.abs(Pb).max()
        # first iteration against numpy: state == propagated state there, so v = 0 and solution = K1[:, :6] H^T z
        st = a.iter_stats(0)
        P = prop[24:].reshape(18, 18)
        M = np.linalg.inv(P)
        M[:6, :6] += st["HTH"]
        sol = np.linalg.inv(M)[:, :6] @ st["HTz"]
        assert np.allclose(st["solution"], sol, rtol=1e-7, atol=1e-12)
        for h in (a, b):
            h.map_incremental_grow(scans[k]["body_ds"])
    assert a.dump_map().shape == b.dump_map().shape


def test_plane_covariance_from_moments_equals_per_point_loop():
    """plane_var = sum_i J_i Sigma_i J_i^T is evaluated from 60 running moments of the stored points (plane_var_mode 0: what the
    CUDA product computes, O(1) per refit) instead of the reference's loop over every stored point (voxel_loc.cpp:76-121,
    plane_var_mode 1).  Same streams through both: identical octree shape and match sets, plane covariances within 1e-9
    (relative to the largest entry of the matrix), states within 1e-9."""
    for kind, cfg, n_pts in (("avia", api.AVIA, None), ("hdl64", api.VELODYNE, 32768)):
        sensor, scans = synth.make_stream(kind, 5, seed=23, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_pts)
        a, b = oa.OracleLio(cfg, plane_var_mode=0), oa.OracleLio(cfg, plane_var_mode=1)
        for h in (a, b):
            h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
            h.voxel_map_init(scans[0]["body_full"])
        for k in range(1, 5):
            for h in (a, b):
                h.predict(scans[k]["dt"])
            ia, ib = a.lio_state_estimation(scans[k]["body_ds"]), b.lio_state_estimation(scans[k]["body_ds"])
            assert ia == ib
            assert np.array_equal(a.matches(), b.matches())
            assert np.allclose(a.get_state()[:24], b.get_state()[:24], rtol=1e-9, atol=1e-12)
            for h in (a, b):
                h.map_incremental_grow(scans[k]["body_ds"])
            da, db = a.dump_map(), b.dump_map()
            assert da.shape == db.shape
            assert np.array_equal(da[:, :24], db[:, :24])          # keys, octree shape, centres, normals, d, radius, eigenvalue, counts
            pa, pb = da[:, 24:], db[:, 24:]
            scale = np.abs(pb).max(axis=1, keepdims=True) + 1e-300
            assert (np.abs(pa - pb) / scale).max() < 1e-9
        assert (da[:, 6] == 1).sum() > 50


def test_kitti_calib_oracle_vs_numpy():
    """orc_frontend.hpp: kitti_calib (voxel_mapping.cpp:1844-1859) against the same formulas through numpy / glibc: the arithmetic-only
    asin / atan2 / sin / cos agree to a few ulp, so the float outputs may differ in the last bit only."""
    rng = np.random.default_rng(5)
    d = rng.normal(size=(20000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = (d * rng.uniform(2.0, 120.0, (20000, 1))).astype(np.float32)
    got = oa.kitti_calib(pts)
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    rng_f = np.sqrt((x * x + y * y) + z * z).astype(np.float64)          # float32 arithmetic, float sqrt
    va = np.arcsin(z.astype(np.float64) / rng_f) + 0.15 * 3.14159265358 / 180.0
    ha = np.arctan2(y, x).astype(np.float32).astype(np.float64)            # atan2f
    ref = np.stack([rng_f * np.cos(va) * np.cos(ha), rng_f * np.cos(va) * np.sin(ha), rng_f * np.sin(va)], axis=1)
    err = np.abs(got.astype(np.float64) - ref)
    # the horizon angle goes through float (atan2f): its last bit (2.4e-7 rad near pi) moves x / y by that times the range
    assert np.all(err <= 3.0e-7 * rng_f[:, None] + 4e-6)
    assert (got == ref.astype(np.float32)).mean() > 0.7
    # the calibration raises every elevation angle by 0.15 degrees and keeps the range
    el0 = np.degrees(np.arcsin(z.astype(np.float64) / rng_f))
    el1 = np.degrees(np.arcsin(got[:, 2].astype(np.float64) / np.linalg.norm(got.astype(np.float64), axis=1)))
    assert np.allclose(el1 - el0, 0.15, atol=2e-4)


def test_voxel_grid_oracle_vs_numpy_restatement():
    """orc_frontend.hpp (pcl::VoxelGrid restatement) against an independent numpy statement of the same published algorithm:
    float32 inverse leaf / box / cell index, leaves in ascending index, float32 sums in scan order."""
    rng = np.random.default_rng(2)
    for pts, leaf in ((synth.make_stream("avia", 1, seed=1)[1][0]["body_full"], 0.4),
                      (rng.normal(0, 5, (20000, 3)).astype(np.float32), 0.5),
                      ((rng.integers(-30, 30, (5000, 3)) * 0.25).astype(np.float32), 0.25)):
        out, small, (min_b, div_b) = oa.voxel_grid(pts, leaf)
        assert not small
        inv = np.float32(1.0) / np.float32(leaf)
        mb = np.floor(pts.min(axis=0) * inv).astype(np.int32)
        assert np.array_equal(mb, min_b)
        ijk = (np.floor(pts * inv) - mb.astype(np.float32)).astype(np.int32)
        idx = ijk[:, 0] + ijk[:, 1] * div_b[0] + ijk[:, 2] * div_b[0] * div_b[1]
        order = np.argsort(idx, kind="stable")
        uniq, start = np.unique(idx[order], return_index=True)
        assert len(uniq) == len(out)
        ends = list(start[1:]) + [len(order)]
        for r in rng.integers(0, len(uniq), 300):
            run = pts[order[start[r]:ends[r]]]
            s = np.zeros(3, np.float32)
            for p in run:
                s = (s + p).astype(np.float32)
            assert np.array_equal(out[r], s / np.float32(len(run)))


def test_imu_oracle_vs_numpy_propagation():
    """orc_imu.hpp against an independent numpy/scipy statement of the same equations (IMU_Processing.cpp:809-896, 930-950):
    matrix exponential from scipy, dense F P F^T + Q, closed-form compensation -- agreement to rounding."""
    from scipy.linalg import expm

    def skew(v):
        return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0.0]])

    rng = np.random.default_rng(5)
    cfg = dict(cov_gyr=[0.1, 0.12, 0.09], cov_acc=[0.4, 0.5, 0.45], cov_bias_gyr=[1e-4, 1e-4, 2e-4], cov_bias_acc=[1e-3, 2e-3, 1e-3],
               mean_acc_norm=9.78, lid_R=np.eye(3), lid_T=[0.04, 0.02, -0.03])
    o = oa.OracleImu(cfg)
    t0 = 50.0
    last = np.array([t0 - 0.004, 0.02, -0.01, 0.03, 0.1, 0.2, 9.7])
    o.reset(last, t0 - 0.001, 0.0, None, None)
    st = np.zeros(348)
    st[0:9] = np.eye(3).reshape(9)
    st[12:15] = [1.0, 0.2, -0.1]
    st[15:18] = [0.001, 0.002, -0.001]
    st[18:21] = [0.02, -0.01, 0.03]
    st[21:24] = [0, 0, -9.81]
    P0 = rng.normal(size=(18, 18))
    P0 = P0 @ P0.T * 1e-4
    st[24:] = P0.reshape(-1)
    tt = t0 + 0.005 * np.arange(1, 21)
    imu = np.concatenate([tt[:, None], rng.normal(0, 0.2, (20, 3)), np.array([0.1, -0.2, 9.78]) + rng.normal(0, 0.3, (20, 3))], axis=1)
    n = 500
    pts = np.concatenate([rng.normal(0, 5, (n, 3)), rng.uniform(0, 100.0, (n, 1))], axis=1).astype(np.float32)
    st1, out, poses = o.undistort(st, imu, pts, t0)
    # numpy restatement
    R, p, v, bg, ba, g = np.eye(3), st[9:12].copy(), st[12:15].copy(), st[15:18], st[18:21], st[21:24]
    P = P0.copy()
    v_imu = np.vstack([last, imu])
    lle = t0 - 0.001
    ref_poses = [(0.0, np.zeros(3), np.zeros(3), v.copy(), p.copy(), R.copy())]
    for k in range(len(v_imu) - 1):
        head, tail = v_imu[k], v_imu[k + 1]
        if tail[0] < lle:
            continue
        w = 0.5 * (head[1:4] + tail[1:4]) - bg
        a = 0.5 * (head[4:7] + tail[4:7]) * 9.81 / 9.78 - ba
        dt = tail[0] - lle if head[0] < lle else tail[0] - head[0]
        F = np.eye(18)
        F[0:3, 0:3] = expm(skew(w) * (-dt))
        F[0:3, 9:12] = -np.eye(3) * dt
        F[3:6, 6:9] = np.eye(3) * dt
        F[6:9, 0:3] = -R @ skew(a) * dt
        F[6:9, 12:15] = -R * dt
        F[6:9, 15:18] = np.eye(3) * dt
        Q = np.zeros((18, 18))
        Q[0:3, 0:3] = np.diag(cfg["cov_gyr"]) * dt * dt
        Q[6:9, 6:9] = R @ np.diag(cfg["cov_acc"]) @ R.T * dt * dt
        Q[9:12, 9:12] = np.diag(cfg["cov_bias_gyr"]) * dt * dt
        Q[12:15, 12:15] = np.diag(cfg["cov_bias_acc"]) * dt * dt
        P = F @ P @ F.T + Q
        R = R @ expm(skew(w) * dt)
        acc = R @ a + g
        p = p + v * dt + 0.5 * acc * dt * dt
        v = v + acc * dt
        ref_poses.append((tail[0] - t0, acc.copy(), w.copy(), v.copy(), p.copy(), R.copy()))
    pcl_end = t0 + float(pts[-1, 3]) / 1000.0
    imu_end = v_imu[-1, 0]
    note = 1.0 if pcl_end > imu_end else -1.0
    dte = note * (pcl_end - imu_end)
    v_end = v + note * acc * dte
    R_end = R @ expm(skew(note * w) * dte)
    p_end = p + note * v * dte + note * 0.5 * acc * dte * dte
    assert len(poses) == len(ref_poses)
    assert np.allclose(st1[24:].reshape(18, 18), P, rtol=1e-9, atol=1e-15)
    assert np.allclose(st1[0:9].reshape(3, 3), R_end, atol=1e-12) and np.allclose(st1[9:12], p_end, atol=1e-12) and np.allclose(st1[12:15], v_end, atol=1e-12)
    # compensation of a few interior points
    order = np.argsort(pts[:, 3], kind="stable")
    offs = np.array([q[0] for q in ref_poses])
    lT = np.asarray(cfg["lid_T"])
    for s in rng.integers(1, n, 40):
        x = pts[order[s]].astype(np.float64)
        t = x[3] / 1000.0
        j = np.max(np.nonzero(offs[:-1] < t)[0])
        _, a_h, w_h, v_h, p_h, R_h = ref_poses[j]
        dt = t - offs[j]
        R_i = R_h @ expm(skew(w_h) * dt)
        T_ei = p_h + v_h * dt + 0.5 * a_h * dt * dt - p_end
        ref = R_end.T @ (R_i @ (x[:3] + lT) + T_ei) - lT
        assert np.allclose(out[s, :3], ref, atol=2e-5), (s, out[s, :3], ref)


# ---------------------------------------------------------------- the mesher's per-voxel triangulation without the oracle's Delaunay
IM_COS150 = -8.65928972248464878803e-01


def _scene_facets(scene):
    from mesh_common import SMALL
    o = oa.OracleMesh(api.MeshConfig(**{**SMALL, **scene.cfg_kw}))
    for pts in scene.frames:
        o.push_frame(pts, scene.centre + np.array([0.3, -0.2, 1.5]))
    v, t, _ = o.snapshot()
    return v.astype(np.float64), t, o


def _pca_uv(v):
    """mesh_rec_geometry.cpp:193-213 restated: centroid, covariance / n, ascending eigen-pairs, the sign rule on d0.s and d1.m,
    l = s x m, projection (d.l, d.m)"""
    c = v.mean(0)
    d = v - c
    w, U = np.linalg.eigh(d.T @ d / len(v))
    s, m = U[:, 0].copy(), U[:, 1].copy()
    if d[0] @ s < 0:
        s = -s
    if d[1] @ m < 0:
        m = -m
    return np.stack([d @ np.cross(s, m), d @ m], 1)


def _apex_cos(uv, t):
    out = []
    for a, b, c in ((0, 1, 2), (1, 2, 0), (2, 0, 1)):
        u, w = uv[t[:, b]] - uv[t[:, a]], uv[t[:, c]] - uv[t[:, a]]
        out.append((u * w).sum(1) / (np.linalg.norm(u, axis=1) * np.linalg.norm(w, axis=1)))
    return np.stack(out, 1)


@pytest.mark.parametrize("n,seed", [(40, 10), (96, 3), (97, 4), (256, 5)])
def test_voxel_triangulation_matches_numpy_qhull(n, seed):
    """general-position single-voxel scenes (jitter 3 mm >> the snap unit res * 2^-22 = 0.1 um): the oracle's facet set equals
    numpy PCA + scipy Delaunay + the 150-degree filter"""
    import mesh_scenes as ms
    scene = ms.jittered_patch(n, seed=seed)
    v, t_orc, _ = _scene_facets(scene)
    uv = _pca_uv(v)
    tri = np.sort(Delaunay(uv).simplices, axis=1)
    cos = _apex_cos(uv, tri)
    near = (np.abs(cos - IM_COS150) < 1e-9).any(1)
    keep = ~((cos < IM_COS150) & (cos >= -1.0)).any(1)
    ref = {tuple(f) for f in tri[keep & ~near]}
    got = {tuple(f) for f in t_orc} - {tuple(f) for f in tri[near]}
    assert (~keep).sum() > 0 or n < 90          # the filter is exercised by the larger patches
    assert got == ref


def _invariants(scene, tol_units=8):
    import scipy.spatial
    v, t, o = _scene_facets(scene)
    res = scene.cfg_kw["voxel_resolution"]
    key = np.round(scene.centre / res)
    inside = np.where((np.round(v / res) == key).all(1))[0]
    uv = _pca_uv(v[inside])
    pos = np.full(len(v), -1)
    pos[inside] = np.arange(len(inside))
    t = t[(pos[t] >= 0).all(1)]
    assert len(t) > 0
    a, b, c = uv[pos[t[:, 0]]], uv[pos[t[:, 1]]], uv[pos[t[:, 2]]]
    area2 = (b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0])
    assert (np.abs(area2) > 0).all()
    hull = scipy.spatial.ConvexHull(uv)
    assert np.abs(area2).sum() / 2 <= hull.volume * (1 + 1e-9)
    # empty circumcircles (float64 from the world coordinates): no vertex inside by more than a few snap units
    unit = res * 2.0 ** -22
    bx, by, cx, cy = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1], c[:, 0] - a[:, 0], c[:, 1] - a[:, 1]
    d = 2 * (bx * cy - by * cx)
    ux = (cy * (bx ** 2 + by ** 2) - by * (cx ** 2 + cy ** 2)) / d
    uy = (bx * (cx ** 2 + cy ** 2) - cx * (bx ** 2 + by ** 2)) / d
    cen = a + np.stack([ux, uy], 1)
    r = np.hypot(ux, uy)
    dist = np.sqrt(((uv[None, :, :] - cen[:, None, :]) ** 2).sum(-1))
    assert (dist >= r[:, None] - tol_units * unit).all()
    return o


@pytest.mark.parametrize("name", ["lattice8x8", "lattice16x8", "stacked6x6", "stacked8x8", "ring30", "ring100", "ring250"])
def test_degenerate_voxel_triangulation_invariants(name):
    """exact ties, duplicate projections, cocircular rings: non-zero projected areas, no overlap beyond the hull, empty
    circumcircles up to the snap unit; and the oracle's path statistics see the degeneracy"""
    import mesh_scenes as ms
    scene = {s.name: s for s, _ in ms.path_scenes()}[name]
    o = _invariants(scene)
    st = ms.centre_stats(o.frame_voxel_stats(), scene, scene.cfg_kw["voxel_resolution"])
    if name.startswith("lattice"):
        assert st["ties"] > 0
    if name.startswith("stacked"):
        assert st["dups"] == scene.n_points // 2
    if name.startswith("ring"):
        n_ring = int(name[4:])
        assert st["max_cav"] == n_ring - 2 and np.array_equal(o.snapshot()[1], ms.ring_fan(n_ring))


def test_collinear_voxel_has_no_seed():
    import mesh_scenes as ms
    scene = ms.collinear()
    v, t, o = _scene_facets(scene)
    st = ms.centre_stats(o.frame_voxel_stats(), scene, 0.4)
    assert len(t) == 0 and not st["seeded"] and st["n"] == 12
