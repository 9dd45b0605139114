"""Shared driver for the localization parity tests: runs the same scan stream through an implementation
under test (CUDA library or host emulation of the kernels) and the oracle, comparing after every stage."""
import numpy as np

from immesh_b200 import api, synth
from oracle_api import OracleLio

SHAPE_COLS = slice(0, 11)  # key, path, layer, flags, point counters: the integer part of the canonical dump


def init_velocity(h, sensor, scans):
    """Start the constant-velocity filter at the true velocity (as a converged filter would be)."""
    s = h.get_state()
    s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
    h.set_state(s)


def run_stream_parity(lib, kind, cfg, n_scans, seed, exact_state=True, n_points=None, body_len=None):
    """body_len: optional {scan index: length} -- those down-sampled scans are truncated to their first `length` points"""
    sensor, scans = synth.make_stream(kind, n_scans, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    for k, m in (body_len or {}).items():
        assert scans[k]["body_ds"].shape[0] >= m
        scans[k]["body_ds"] = scans[k]["body_ds"][:m]
    g = api.Lio(cfg, lib=lib)
    o = OracleLio(cfg, sum_mode=0)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    dg, do = g.dump_map(), o.dump_map()
    assert dg.shape == do.shape
    assert np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), "octree shape after buildVoxelMap"
    assert np.array_equal(dg, do), "plane parameters after buildVoxelMap"
    stats = []
    for k in range(1, n_scans):
        body = scans[k]["body_ds"]
        g.predict(scans[k]["dt"])
        o.predict(scans[k]["dt"])
        assert np.array_equal(g.get_state(), o.get_state()), f"scan {k}: prediction"
        ig = g.lio_state_estimation(body)
        io = o.lio_state_estimation(body)
        assert ig == io, f"scan {k}: iteration count {ig} vs {io}"
        assert np.array_equal(g.matches(), o.matches()), f"scan {k}: matched point set / layers"
        for it in range(io):
            a, b = g.iter_stats(it), o.iter_stats(it)
            assert a["n_match"] == b["n_match"]
            assert np.array_equal(a["HTH"], b["HTH"]) and np.array_equal(a["HTz"], b["HTz"]), f"scan {k} iter {it}: normal equations"
        sg, so = g.get_state(), o.get_state()
        if exact_state:
            assert np.array_equal(sg, so), f"scan {k}: state max diff {np.abs(sg - so).max()}"
        else:
            assert np.allclose(sg, so, rtol=1e-9, atol=1e-12)
        g.map_incremental_grow()
        o.map_incremental_grow(body)
        dg, do = g.dump_map(), o.dump_map()
        assert dg.shape == do.shape, f"scan {k}: node count {dg.shape[0]} vs {do.shape[0]}"
        assert np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), f"scan {k}: octree shape"
        assert np.array_equal(dg, do), f"scan {k}: plane parameters"
        stats.append(dict(n=body.shape[0], n_match=g.iter_stats(0)["n_match"], iters=ig,
                          pos_err=float(np.linalg.norm(sg[9:12] - scans[k]["t_true"]))))
    assert g.counts()["err"] == 0
    return stats


def degenerate_root_voxels():
    """Body-frame points (identity pose, zero extrinsic translation, root voxel 0.5 m, child borders at the voxel centres) of five
    kinds of root voxel, with what the reference's init_plane (voxel_loc.cpp:76-121) computes there:
      pole      collinear points along z: the covariance has one non-zero entry, two eigenvalues are exactly 0, evalsMin <
                threshold makes it a plane, and the variance term divides by evalsReal[evalsMin] - evalsReal[evalsMid] = 0 and
                multiplies the resulting inf by 0 -> NaN entries in the plane variance
      repeated  one point repeated: the covariance is exactly 0, every eigenvalue 0, (p - c) / 0 = 0 / 0 -> NaN plane variance
      plane     an exact axis-aligned plane at binary-exact coordinates on the z = -0.5 root border: min eigenvalue exactly 0,
                finite plane; the reference's key rule (p / size, minus 1 when negative, truncated) puts z = -0.5 in voxel -2
      borders   a tilted plane whose points lie on root borders at negative coordinates (x = -3, -2.5, -2, y = -2, -1.5, -1)
      cube      a 3-D lattice with spacing 0.125 m filling the negative root voxel (-3, -3, -3) and its lower borders: not a plane
                (isotropic, every eigenvalue 0.0195 > 0.01), so it is cut; points at x = -1.25 etc. lie exactly on the child
                borders (voxel centre: the reference sends them to the lower child, strict >); the eight 2 x 2 x 2 children
                have three equal eigenvalues 0.0039 < 0.01, so they are planes whose variance term divides by 0 -> NaN
    Returns (points float32[n,3], {case: root key})."""
    out, keys = [], {}
    z = np.arange(12) * 0.03125 - 0.96875
    out.append(np.stack([np.full(12, -1.25), np.full(12, 2.25), z], 1))
    keys["pole"] = (-3, 4, -2)
    out.append(np.tile([[3.125, -2.1875, 0.6875]], (10, 1)))
    keys["repeated"] = (6, -5, 1)
    gx, gy = np.meshgrid(np.arange(8) * 0.0625 + 1.0, np.arange(8) * 0.0625 + 1.0)
    out.append(np.stack([gx.ravel(), gy.ravel(), np.full(64, -0.5)], 1))
    keys["plane"] = (2, 2, -2)
    gx, gy = np.meshgrid(np.arange(-8, 1) * 0.125 - 2.0, np.arange(-8, 1) * 0.125 - 1.0)
    out.append(np.stack([gx.ravel(), gy.ravel(), gx.ravel() * 0.25 - 3.0], 1))
    keys["borders"] = (-7, -5, -8)
    g = np.arange(5) * 0.125 - 1.5
    cx, cy, cz = np.meshgrid(g, g, g, indexing="ij")
    out.append(np.stack([cx.ravel(), cy.ravel(), cz.ravel()], 1))
    keys["cube"] = (-3, -3, -3)
    pts = np.concatenate(out)
    assert np.array_equal(pts.astype(np.float32).astype(np.float64), pts)
    return pts.astype(np.float32), keys


def run_degenerate_map_parity(lib):
    """degenerate_root_voxels() through buildVoxelMap and one state estimation, implementation under test against the oracle,
    NaN-aware; asserts that every case reached what degenerate_root_voxels() says it does"""
    import dataclasses
    cfg = dataclasses.replace(api.AVIA, ext_T=(0.0, 0.0, 0.0))   # the body points are the world points: the borders stay exact
    body, keys = degenerate_root_voxels()
    g, o = api.Lio(cfg, lib=lib), OracleLio(cfg)
    for h in (g, o):
        h.set_pose(np.eye(3), np.zeros(3))
        h.voxel_map_init(body)
    pw, _ = o.pv_lists(body, mode=0)
    assert np.array_equal(pw, body.astype(np.float64)), "the world points must be the body points"
    on_root = (np.fmod(pw, 0.5) == 0) & (pw < 0)
    on_child = (np.fmod(pw + 0.25, 0.5) == 0) & (pw < 0)
    assert on_root.any(1).sum() > 100 and on_child.any(1).sum() > 50
    dg, do = g.dump_map(), o.dump_map()
    assert dg.shape == do.shape and np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), "octree shape"
    assert np.array_equal(dg, do, equal_nan=True), "plane parameters (NaN-aware)"
    rows = {c: do[(do[:, 0:3] == k).all(1)] for c, k in keys.items()}
    for c in ("pole", "repeated"):
        r = rows[c]
        assert len(r) == 1 and r[0, 6] == 1 and r[0, 19] == 0 and np.isnan(r[0, 24:]).any(), c
    assert len(rows["plane"]) == 1 and rows["plane"][0, 6] == 1 and rows["plane"][0, 19] == 0 and np.isfinite(rows["plane"][0]).all()
    assert len(rows["borders"]) == 1 and rows["borders"][0, 8] == 1          # x = -3 -> key -7: the lower neighbour takes the border
    cube = rows["cube"]
    assert cube[0, 6] == 0 and len(cube) == 9 and (cube[1:, 4] == 1).all() and (cube[1:, 6] == 1).all() and np.isnan(cube[1:, 24:]).any(1).all()
    rng = np.random.default_rng(0)
    scan = (body + rng.normal(0, 0.002, body.shape)).astype(np.float32)
    ig, io = g.lio_state_estimation(scan), o.lio_state_estimation(scan)
    assert ig == io
    assert np.array_equal(g.matches(), o.matches())
    for it in range(io):
        a, b = g.iter_stats(it), o.iter_stats(it)
        assert a["n_match"] == b["n_match"]
        assert np.array_equal(a["HTH"], b["HTH"], equal_nan=True) and np.array_equal(a["HTz"], b["HTz"], equal_nan=True)
    assert np.array_equal(g.get_state(), o.get_state(), equal_nan=True)
    return dg
