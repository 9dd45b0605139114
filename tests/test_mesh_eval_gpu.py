"""GPU tier of the mesh evaluation (immesh_mesh_evaluate): meshes built from synthetic Avia-shaped and KITTI-shaped (hdl64) streams,
evaluated against synth.make_gt_cloud, equal the numpy restatement (tests/mesh_eval_reference.py) exactly in every count, both
quantised distance sums and every facet row, with raw and smoothed positions, for any batch budget and either ground-truth location;
the call changes nothing on the handle; and the error contract."""
import ctypes as C

import numpy as np
import pytest
import torch

import mesh_eval_reference as ref
from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans

pytestmark = pytest.mark.gpu
E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5
CFG = dict(spacing=0.04, gt_leaf=0.03, threshold=0.05, max_dist=0.5, incorrect_ratio=0.8)
STREAMS = {"avia": dict(n=5, n_points=None), "hdl64": dict(n=3, n_points=32768)}


def build_mesh(lib, kind, seed=5):
    s = STREAMS[kind]
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    for k, (w, t) in enumerate(world_scans(kind, s["n"], seed=seed, n_points=s["n_points"])):
        mesh.push_frame(w, t, k)
    gt = synth.make_gt_cloud(kind, s["n"], seed=seed, n_points=s["n_points"])
    return mesh, gt


def positions(mesh, smoothed):
    v, t, _ = mesh.snapshot()
    if smoothed:
        v = mesh.smooth_all(0.5, 20).astype(np.float32)
    return v, t


def check(res, r, what):
    c = np.array([res["counts"][k] for k in api.EVAL_COUNT_KEYS], dtype=np.int64)
    assert np.array_equal(c, r["counts"]), (what, c, r["counts"])
    m = np.array([res["metrics"][k] for k in api.EVAL_METRIC_KEYS])
    assert np.allclose(m[:2], r["metrics"][:2], rtol=1e-12, atol=0), what
    assert np.array_equal(m[2:], r["metrics"][2:7], equal_nan=True), what
    assert np.array_equal(res["rows"], r["rows"]), what


@pytest.fixture(scope="module", params=sorted(STREAMS))
def stream(request, cuda_lib):
    mesh, gt = build_mesh(cuda_lib, request.param)
    yield request.param, mesh, gt
    mesh.close()


def test_against_reference_raw_then_smoothed(stream):
    kind, mesh, gt = stream
    v, t = positions(mesh, False)
    r = ref.evaluate(v, t, gt, **CFG)
    assert r["counts"][2] > 10000 and r["counts"][3] > 10000
    res = mesh.evaluate(gt, **CFG, facets=True)
    check(res, r, f"{kind} raw")
    again = mesh.evaluate(gt, **CFG, facets=True)
    assert again["counts"] == res["counts"] and np.array_equal(again["rows"], res["rows"])
    assert [again["metrics"][k] for k in api.EVAL_METRIC_KEYS[:2]] == [res["metrics"][k] for k in api.EVAL_METRIC_KEYS[:2]]
    # many small tiles, and the ground truth read in place on the device: bit-identical
    small = mesh.evaluate(gt, **CFG, facets=True, max_batch_bytes=24 << 20)
    assert small["stats"]["tiles"] > 4 and small["stats"]["scratch_bytes"] <= 24 << 20, small["stats"]
    assert res["stats"]["scratch_bytes"] <= 2 << 30 and res["stats"]["tiles"] < small["stats"]["tiles"], res["stats"]
    assert small["counts"] == res["counts"] and np.array_equal(small["rows"], res["rows"]) and small["metrics"] == res["metrics"]
    d = torch.from_numpy(gt).cuda()
    dev = mesh.evaluate((d.data_ptr(), d.shape[0]), **CFG, facets=True, on_device=True)
    assert dev["counts"] == res["counts"] and np.array_equal(dev["rows"], res["rows"]) and dev["metrics"] == res["metrics"]
    # smoothed positions: refused before smooth_all, then equal to the reference on the smoothed floats
    with pytest.raises(RuntimeError, match="smooth first"):
        mesh.evaluate(gt, **CFG, smoothed=True)
    vs, _ = positions(mesh, True)
    rs = ref.evaluate(vs, t, gt, **CFG)
    check(mesh.evaluate(gt, **CFG, smoothed=True, facets=True), rs, f"{kind} smoothed")
    check(mesh.evaluate(gt, **CFG, smoothed=True, facets=True, max_batch_bytes=24 << 20), rs, f"{kind} smoothed, small tiles")


def test_gt_as_given_and_finer_sampling(cuda_lib):
    mesh, gt = build_mesh(cuda_lib, "avia", seed=9)
    v, t = positions(mesh, False)
    cfg = dict(CFG, gt_leaf=0.0)
    check(mesh.evaluate(gt, **cfg, facets=True), ref.evaluate(v, t, gt, **cfg), "gt_leaf 0")
    cfg = dict(spacing=0.02, gt_leaf=0.01, threshold=0.05, max_dist=0.2, incorrect_ratio=0.8)
    sub = gt[:20000]
    check(mesh.evaluate(sub, **cfg, facets=True), ref.evaluate(v, t, sub, **cfg), "finer sampling")


def test_handle_unchanged_by_evaluation(cuda_lib):
    """further frames after an evaluation give the same snapshot and change-feed rows as a twin that was never evaluated"""
    scans = world_scans("avia", 6, seed=21)
    a, b = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib), api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    gt = synth.make_gt_cloud("avia", 3, seed=21)
    for m in (a, b):
        for k in range(3):
            m.push_frame(*scans[k], k)
        m.changes_enable(1 << 20, 64)
    a.smooth_all(0.5, 20)
    b.smooth_all(0.5, 20)
    a.evaluate(gt, **CFG, facets=True)
    a.evaluate(gt, **CFG, smoothed=True)
    for k in range(3, 6):
        for m in (a, b):
            m.push_frame(*scans[k], k)
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    ca, cb = a.changes(3), b.changes(3)   # the frames after the enable (frame 3)
    assert np.array_equal(ca["rows"], cb["rows"]) and np.array_equal(ca["frames"], cb["frames"])


def test_evaluation_drains_queued_frames(cuda_lib):
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 6, seed=3, ext_T=cfg.ext_T)
    gt = synth.make_gt_cloud("avia", 6, seed=3, ext_T=cfg.ext_T)
    res = []
    for early in (True, False):
        lio, mesh = api.Lio(cfg, lib=cuda_lib), api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
        lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(lio, sensor, scans)
        lio.voxel_map_init(scans[0]["body_full"])
        for k in range(1, 6):
            lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
            mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if not early:
            mesh.wait()
        res.append(mesh.evaluate(gt, **CFG, facets=True))
        assert res[-1]["counts"]["live_triangles"] > 0
    assert res[0]["counts"] == res[1]["counts"] and np.array_equal(res[0]["rows"], res[1]["rows"])


def test_error_contract(cuda_lib):
    L = cuda_lib
    mesh, gt = build_mesh(L, "avia", seed=13)
    nt = mesh.counts()["n_triangles"]
    counts, metrics = np.zeros(12, np.int64), np.zeros(8)
    rows = np.zeros((nt, 5), np.int32)
    nr = C.c_int64(-1)
    g = np.ascontiguousarray(gt)
    i64, i32, dp = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_double)

    def call(cfg, pts=g, rows_p=None, cap=0, cfg_ptr=True):
        return L.immesh_mesh_evaluate(mesh._h, pts.ctypes.data_as(C.c_void_p), len(pts), 0, C.byref(cfg) if cfg_ptr else None, counts.ctypes.data_as(i64),
                                      metrics.ctypes.data_as(dp), rows_p, cap, C.byref(nr))

    def cfg(**kw):
        d = dict(sample_spacing=0.04, gt_leaf=0.03, threshold=0.05, max_dist=0.5, incorrect_ratio=0.8, positions=0, pad=0, max_batch_bytes=0)
        d.update(kw)
        return api._EvalCfg(*d.values())

    for bad in (dict(sample_spacing=0.0), dict(sample_spacing=float("nan")), dict(gt_leaf=-0.01), dict(threshold=0.0), dict(max_dist=0.04),
                dict(max_dist=2000.0), dict(incorrect_ratio=0.0), dict(incorrect_ratio=1.5), dict(positions=2), dict(max_batch_bytes=-1)):
        assert call(cfg(**bad)) == E_INVALID, bad
    assert call(cfg(), cfg_ptr=False) == E_INVALID
    assert call(cfg(positions=1)) == E_INVALID                 # no vertex smoothed yet
    assert b"smooth first" in L.immesh_last_error()
    # a count query: nothing computed, counts untouched
    counts[:] = -7
    assert call(cfg(), rows_p=rows.ctypes.data_as(i32), cap=0) == E_CAPACITY and nr.value == nt and np.all(counts == -7)
    assert call(cfg(), rows_p=rows.ctypes.data_as(i32), cap=nt - 1) == E_CAPACITY and np.all(counts == -7)
    bad = g.copy()
    bad[len(bad) // 2, 1] = np.nan
    assert call(cfg(), pts=bad) == E_INVALID
    assert call(cfg(sample_spacing=1e-6)) == E_RANGE           # a triangle would need more than 2^15 subdivisions
    assert call(cfg(max_batch_bytes=4096)) == E_CAPACITY       # below the triangle table
    assert b"triangle" in L.immesh_last_error()
    assert call(cfg(), rows_p=rows.ctypes.data_as(i32), cap=nt) == 0 and counts[0] == nt


def test_points_on_tile_boundaries_and_tile_limits(cuda_lib):
    """two far ground-truth points make the root box symmetric about x = 0, so the first bisection (x is the longest axis) lies at
    x = 0 exactly; ground-truth points moved onto x = 0 and onto the later split planes x = +-(A + 1) / 2 must each be answered once"""
    mesh, gt = build_mesh(cuda_lib, "avia", seed=17)
    v, t = positions(mesh, False)
    A = 400.0
    near0 = gt[np.abs(gt[:, 0]) < 0.3].copy()
    near0[:, 0] = 0.0
    extra = np.array([[-A, 0, 0], [A, 0, 0], [(A + 1) / 2, 1, 1], [-(A + 1) / 2, 1, 1]], np.float32)
    g = np.concatenate([gt, near0, extra]).astype(np.float32)
    assert g[:, 0].min() == -A and g[:, 0].max() == A and len(near0) > 100
    for leaf in (0.03, 0.0):
        cfg = dict(CFG, gt_leaf=leaf)
        r = ref.evaluate(v, t, g, **cfg)
        small = mesh.evaluate(g, **cfg, facets=True, max_batch_bytes=16 << 20)
        assert small["stats"]["tiles"] > 2 and small["stats"]["scratch_bytes"] <= 16 << 20
        check(small, r, f"tile boundaries, gt_leaf {leaf}")
        check(mesh.evaluate(g, **cfg, facets=True), r, f"tile boundaries, default budget, gt_leaf {leaf}")
    # a budget that holds the table but no tile at the smallest side: the tile's capacity error, after the table's
    table = mesh.evaluate(gt, **CFG)["stats"]["table_bytes"]
    with pytest.raises(RuntimeError, match="code -3.*a tile of side"):
        mesh.evaluate(gt, **CFG, max_batch_bytes=table + 4096)
    with pytest.raises(RuntimeError, match="code -3.*table"):
        mesh.evaluate(gt, **CFG, max_batch_bytes=table - 1)
    # leaves too small for the search radius: refused before any tile (the smallest tile's keys would not fit 21 bits)
    for leaf, md in ((1e-7, 0.5), (0.0005, 1024.0)):
        with pytest.raises(RuntimeError, match="code -5.*smallest tile"):
            mesh.evaluate(gt, **dict(CFG, gt_leaf=leaf, max_dist=md))
