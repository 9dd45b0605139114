"""GPU tier: the overlays of the queued mesh view (immesh_mesh_view_overlay).  Every queued image with every layer on equals the numpy
restatement of the rule (tests/view_overlay_reference.py) byte for byte, its depth bit for bit, from the frame's mesh
(immesh_mesh_snapshot), reinforced cloud (immesh_mesh_reinforced_cloud) and localization states: world-frame pushes of an Avia and
an HDL-64 stream (the scan layer from the pushed world points) in the fixed and follow modes, and the graph-replayed localization
chain in the sensor-bound, fixed and follow modes (the frustum, the trajectory and the reinforced points; the scan layer is checked
on the world-frame pushes, whose world points the caller holds), with faces and wireframe, white and height colour.  A NULL overlay
and on-then-off give the images and launches of a twin that never called it; nothing else changes; the error contract."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans
from view_overlay_reference import render_overlay

pytestmark = pytest.mark.gpu

ZN, ZF = 0.1, 1500.0
W, H = 320, 240
K = api.reinforce_intrinsics(W, H, 200.0)
DEFAULTS = dict(scan_point_size=2, reinforced_point_size=2, axis_and_grid=True, camera_size=1.0, path_width=4)
R_FIX = np.array([[0.0, 0.0, -1.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])   # looking along +x


def same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check(frame, image, verts, tris, color, wire, **ov):
    rgba, depth, R, t, _ = image
    rn, dn = render_overlay(K, W, H, ZN, ZF, R, t, verts, tris, color, None, wire, **ov)
    assert same(depth, dn), f"frame {frame}: depth differs from the restatement"
    bad = np.argwhere((rgba != rn).any(axis=2))
    assert len(bad) == 0, (frame, len(bad), bad[:5], rgba[tuple(bad[0])], rn[tuple(bad[0])])
    return rgba


@pytest.mark.parametrize("kind,wire,color", [("avia", False, False), ("hdl64", True, True), ("avia", True, False), ("hdl64", False, True)])
def test_world_pushes_against_restatement(cuda_lib, kind, wire, color):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.reinforce_enable()
    mesh.view_enable(K, W, H, ZN, ZF, color_by_height=color)
    mesh.view_overlay(wireframe=wire, path_capacity=3, **DEFAULTS)
    scans = world_scans(kind, 5, 5)
    drawn = {}
    for k, (wld, t) in enumerate(scans):
        f = k + 1
        if f % 2:
            mesh.view_pose(R_FIX, t + np.array([-14.0, 1.0, 6.0]))
        else:
            mesh.view_pose(R_FIX, np.array([-10.0, -2.0, 5.0]), follow=True)
        mesh.push_frame(wld, t, k)
        mesh.wait()
        v, tri, _ = mesh.snapshot()
        img = mesh.view_image()
        assert img[4] == f
        rf = mesh.reinforced_cloud()[1]
        path = [scans[j][1] for j in range(max(0, k - 2), k + 1)]
        rgba = check(f, img, v, tri, color, wire, scan=wld if f >= 2 else None, scan_size=2, rf=rf, rf_size=2, axis_and_grid=True,
                     frustum_pose=None, camera_size=1.0, path=path, path_width=4)
        drawn[f] = rgba
    # the overlays drew something: the white scan and the grey grid
    last = drawn[max(drawn)]
    assert (last[..., :3] == 115).all(axis=2).sum() > 50 and (last[..., :3] == 255).all(axis=2).sum() > 200


def lio_stream(lib, n_scans=8, seed=3, overlay=None, wire=False, color=False, modes=None, each=None, reinforce=True, feed=False, view=True):
    """the graph-replayed chain (step_async + push_frame_from_lio_async) with the queued view; each(k, mesh, states) after every frame"""
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    if reinforce:
        mesh.reinforce_enable()
    if feed:
        mesh.changes_enable(1 << 20, 64)
    if view:
        mesh.view_enable(K, W, H, ZN, ZF, win=2, color_by_height=color)
        if overlay is not None:
            mesh.view_overlay(wireframe=wire, **overlay)
    states = {}
    for k in range(1, n_scans):
        if modes:
            mesh.view_pose(*modes(k))
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        s = lio.get_state()
        states[k] = (s[0:9].reshape(3, 3).copy(), s[9:12].copy())
        if each:
            each(k, mesh, states)
    lio.wait()
    mesh.wait()
    return lio, mesh, states


def modes(k):
    if k <= 2:
        return (None, None, False)
    if k <= 4:
        return (R_FIX, np.array([-5.0, 0.0, 3.0]), False)
    return (R_FIX, np.array([-8.0, 0.5, 4.0]), True)


@pytest.mark.parametrize("wire,color", [(False, True), (True, False)])
def test_localization_chain_against_restatement(cuda_lib, wire, color):
    ov = dict(DEFAULTS, scan_point_size=0, path_capacity=4)
    seen = []

    def each(k, mesh, states):
        mesh.wait()
        v, tri, _ = mesh.snapshot()
        img = mesh.view_image()
        assert img[4] == k
        rf = mesh.reinforced_cloud()[1]
        path = [states[j][1] for j in range(max(1, k - 3), k + 1)]
        rgba = check(k, img, v, tri, color, wire, rf=rf, rf_size=2, axis_and_grid=True, frustum_pose=states[k], camera_size=1.0, path=path,
                     path_width=4)
        seen.append((rgba[..., :3] == (255, 0, 255)).all(axis=2).sum())
    lio, mesh, _ = lio_stream(cuda_lib, overlay=ov, wire=wire, color=color, modes=modes, each=each)
    st = api.graph_stats(None, mesh)
    assert st["mesh_captures"] == 1 and st["mesh_replays"] >= 5, st
    assert max(seen) > 100   # the reinforced points are drawn


def test_null_and_on_then_off_equal_never(cuda_lib, monkeypatch):
    monkeypatch.setenv("IMMESH_GRAPH", "0")   # every frame launches its kernels
    scans = world_scans("avia", 4, 4)

    def run(setup):
        mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
        mesh.view_enable(K, W, H, ZN, ZF, color_by_height=True)
        setup(mesh)
        out, imgs = [], []
        for k, (wld, t) in enumerate(scans):
            mesh.view_pose(R_FIX, t + np.array([-12.0, 0.0, 5.0]))
            n0 = api.launch_count(cuda_lib)
            mesh.push_frame(wld, t, k)
            out.append(api.launch_count(cuda_lib) - n0)
            imgs.append(mesh.view_image())
        return out, imgs

    def on_off(m):
        m.view_overlay(wireframe=True, **DEFAULTS)
        m.view_overlay_off()
    la, ia = run(lambda m: None)
    lb, ib = run(lambda m: m.view_overlay_off())
    lc, ic = run(on_off)
    ld, id_ = run(lambda m: m.view_overlay(wireframe=False, scan_point_size=0, reinforced_point_size=0, axis_and_grid=False, camera_size=0.0,
                                           path_width=0))
    le, ie = run(lambda m: m.view_overlay(**DEFAULTS))
    assert la == lb == lc == ld, (la, lb, lc, ld)
    assert all(x > y for x, y in zip(le, la))
    for other in (ib, ic, id_):
        for a, b in zip(ia, other):
            assert np.array_equal(a[0], b[0]) and same(a[1], b[1]) and np.array_equal(a[2], b[2]) and a[4] == b[4]
    assert any(not np.array_equal(a[0], e[0]) for a, e in zip(ia, ie))
    # disabling the view clears the overlay: enabled again, it draws none
    m = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    m.view_enable(K, W, H, ZN, ZF, color_by_height=True)
    m.view_overlay(**DEFAULTS)
    m.view_disable()
    m.view_enable(K, W, H, ZN, ZF, color_by_height=True)
    m.view_pose(R_FIX, scans[0][1] + np.array([-12.0, 0.0, 5.0]))
    n0 = api.launch_count(cuda_lib)
    m.push_frame(*scans[0])
    assert api.launch_count(cuda_lib) - n0 == la[0]


def test_nothing_else_changes(cuda_lib):
    keep = {}

    def each(k, mesh, states):
        keep.setdefault(id(mesh), []).append((mesh.reinforced_cloud(), mesh.view_image()))
    a_lio, a_mesh, _ = lio_stream(cuda_lib, overlay=dict(DEFAULTS, path_capacity=8), wire=True, color=True, modes=modes, each=each, feed=True)
    b_lio, b_mesh, _ = lio_stream(cuda_lib, color=True, modes=modes, each=each, feed=True)
    assert a_mesh.counts() == b_mesh.counts()
    for x, y in zip(a_mesh.snapshot(), b_mesh.snapshot()):
        assert np.array_equal(x, y)
    assert np.array_equal(a_lio.get_state(), b_lio.get_state())
    ca, cb = a_mesh.changes(0), b_mesh.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key
    ra, rb = keep[id(a_mesh)], keep[id(b_mesh)]
    assert len(ra) == len(rb) == 7
    for (cla, ima), (clb, imb) in zip(ra, rb):
        for u, v in zip(cla, clb):
            assert same(u, v) if u.dtype == np.float32 else np.array_equal(u, v)
        assert same(ima[1], imb[1]) and np.array_equal(ima[2], imb[2]) and np.array_equal(ima[3], imb[3])   # depth and camera
    assert any(not np.array_equal(ima[0], imb[0]) for (_, ima), (_, imb) in zip(ra, rb))


def test_error_contract(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)

    def ov(**kw):
        d = dict(wireframe=0, scan_point_size=2, reinforced_point_size=2, axis_and_grid=1, camera_size=1.0, path_width=4, path_capacity=16)
        d.update(kw)
        return L.immesh_mesh_view_overlay(mesh._h, C.byref(api._ViewOverlay(**d)))
    assert ov() == -1                                              # the view is not enabled
    assert L.immesh_mesh_view_overlay(mesh._h, None) == -1
    mesh.view_enable(K, W, H, ZN, ZF)
    assert ov() == 0 and L.immesh_mesh_view_overlay(mesh._h, None) == 0
    for bad in (dict(wireframe=2), dict(axis_and_grid=-1), dict(scan_point_size=-1), dict(scan_point_size=65), dict(reinforced_point_size=65),
                dict(path_width=65), dict(path_width=-1), dict(camera_size=-0.5), dict(camera_size=float("nan")), dict(camera_size=float("inf")),
                dict(path_capacity=0), dict(path_capacity=(1 << 24) + 1)):
        assert ov(**bad) == -1, bad
    assert ov(path_width=0, path_capacity=0) == 0                  # the capacity is read only with a path
    assert ov(scan_point_size=64, reinforced_point_size=0, path_width=64, path_capacity=1 << 24) == 0
    mesh.push_frame(np.zeros((0, 3), np.float32), np.array([1.0, 2.0, 3.0]))
    rgba, depth, R, t, f = mesh.view_image()
    assert f == 1 and (depth == -1).all()
    uid = C.create_string_buffer(128)
    assert L.immesh_mesh_shard(mesh._h, 0, 2, uid) == -1          # the view is on
    mesh.view_disable()
    assert ov() == -1
