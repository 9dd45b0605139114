"""GPU tier: the mesh viewer's shaded image on the device (immesh_mesh_render_view, immesh_mesh_view_enable / _pose / _image).
render_view on meshes of Avia and HDL-64 streams against the numpy restatement of the image rule on immesh_mesh_snapshot (raw
positions, and the smoothed positions of smooth_all cast to float), byte for byte and depth bit for bit; its positions-0 depth equal
to render_depth's; every queued frame's image equal to render_view at that frame's camera on a twin handle, in the sensor-bound,
fixed and follow modes, graph-replayed; nothing else changes; enable then disable launches what never enabling launches; the empty
mesh is black; the error contract."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans
from view_reference import frame_pose, render

pytestmark = pytest.mark.gpu

K0 = api.reinforce_intrinsics(640, 480)
ZN, ZF = 0.1, 1500.0


def same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def look_at(eye, target):
    """camera rotation (world = R diag(1,-1,-1) p + t) looking from eye at target, image up towards world +z"""
    f = np.asarray(target, np.float64) - eye
    f /= np.linalg.norm(f)
    x = np.cross(f, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    y = np.cross(x, f)
    return np.stack([x, y, -f], axis=1)


def world_mesh(lib, kind, n_frames=3, seed=5):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    scans = world_scans(kind, n_frames, seed)
    for k, (wld, t) in enumerate(scans):
        mesh.push_frame(wld, t, k)
    return mesh, scans[-1][1]


def check_view(mesh, K, w, h, R, t, verts, tris, **style):
    rgba, depth = mesh.render_view(K, w, h, ZN, ZF, R, t, **style)
    rn, dn = render(K, w, h, ZN, ZF, R, t, verts, tris, style.get("color_by_height", False), style.get("z_range"))
    assert same(depth, dn), "depth differs from the restatement"
    bad = np.argwhere((rgba != rn).any(axis=2))
    assert len(bad) == 0, (len(bad), bad[:5], rgba[tuple(bad[0])], rn[tuple(bad[0])])
    return rgba, depth


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_render_view_against_restatement(cuda_lib, kind):
    mesh, pos = world_mesh(cuda_lib, kind)
    v, tri, _ = mesh.snapshot()
    assert len(tri) > 1000
    K, w, h = (160.0, 160.0, 160.0, 120.0), 320, 240
    eye = pos + np.array([-12.0, -9.0, 10.0])
    R = look_at(eye, pos)
    for style in (dict(), dict(color_by_height=True), dict(color_by_height=True, z_range=(-1.0, 4.0))):
        rgba, depth = check_view(mesh, K, w, h, R, eye, v, tri, **style)
        assert (depth > 0).sum() > 2000
        d_ref, _, _ = mesh.render_depth(K, w, h, ZN, ZF, R, eye)
        assert same(depth, d_ref), "positions-0 depth differs from render_depth"
    # the smoothed positions (every vertex smoothed by smooth_all), drawn as floats
    sm = mesh.smooth_all()
    vs = sm.astype(np.float32)
    for style in (dict(positions=1), dict(positions=1, color_by_height=True)):
        check_view(mesh, K, w, h, R, eye, vs, tri, **style)
    raw, _ = mesh.render_view(K, w, h, ZN, ZF, R, eye)
    smoothed, _ = mesh.render_view(K, w, h, ZN, ZF, R, eye, positions=1)
    assert not np.array_equal(raw, smoothed)
    # the view wrote nothing: the raw positions and the snapshot are as they were
    v2, tri2, _ = mesh.snapshot()
    assert np.array_equal(v, v2) and np.array_equal(tri, tri2)


def lio_stream(lib, n_scans=8, seed=3, view=None, poses_for=None, twin=None, reinforce=False, feed=False):
    """the graph-replayed chain (localization step + push_frame_from_lio_async) with the queued view; view = dict of view_enable
    arguments; poses_for(k) -> view_pose arguments for scan k; twin: called with (k, mesh, image) after each frame"""
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
    if view is not None:
        mesh.view_enable(**view)
    images, clouds, states = [], [], {}
    for k in range(1, n_scans):
        if view is not None and poses_for:
            mesh.view_pose(*poses_for(k))
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if reinforce:
            clouds.append(mesh.reinforced_cloud())
        if view is not None:
            images.append(mesh.view_image())
        s = lio.get_state()
        states[k] = (s[0:9].reshape(3, 3).copy(), s[9:12].copy())
        if twin:
            twin(k, mesh, images[-1] if images else None)
    lio.wait()
    mesh.wait()
    return lio, mesh, images, clouds, states


R_FIX = np.array([[0.0, 0.0, -1.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])   # looking along the sensor's +x


def modes(k):
    if k <= 2:
        return (None, None, False)
    if k <= 4:
        return (R_FIX, np.array([-5.0, 0.0, 3.0]), False)
    return (R_FIX, np.array([-8.0, 0.5, 4.0]), True)


@pytest.mark.parametrize("style", [dict(), dict(color_by_height=True, positions=1)])
def test_queued_view_equals_render_view_on_a_twin(cuda_lib, style):
    K, w, h = K0, 640, 480
    lio, mesh, images, _, states = lio_stream(cuda_lib, view=dict(style, win=2), poses_for=modes)
    st = api.graph_stats(None, mesh)
    assert st["mesh_captures"] == 1 and st["mesh_replays"] == len(images) - 1, st
    frames = [im[4] for im in images]
    assert frames == list(range(1, len(images) + 1)), frames
    cams = {f: (im[2], im[3]) for f, im in zip(frames, images)}
    seen = {}

    def render_twin(k, m, _):   # the twin: the same stream without the view, rendered at each frame's camera once the frame is done
        m.wait()
        R, t = cams[k]
        seen[k] = m.render_view(K, w, h, ZN, ZF, R, t, **style)
    lio_stream(cuda_lib, twin=render_twin)
    for (rgba, depth, R, t, f), k in zip(images, range(1, len(images) + 1)):
        rr, dr = seen[k]
        assert np.array_equal(rgba, rr) and same(depth, dr), f"frame {k}: the queued image differs from render_view"
        Rn, tn = frame_pose(states, k, 2, {1: 0, 2: 0, 3: 1, 4: 1}.get(k, 2), modes(k)[0], modes(k)[1])
        assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12, (k, R, Rn, t, tn)
    assert max((im[1] > 0).sum() for im in images) > 20000


def test_nothing_else_changes(cuda_lib):
    a_lio, a_mesh, imgs, a_clouds, _ = lio_stream(cuda_lib, view=dict(color_by_height=True), reinforce=True, feed=True)
    b_lio, b_mesh, _, b_clouds, _ = lio_stream(cuda_lib, reinforce=True, feed=True)
    assert len(imgs) == len(a_clouds)
    assert a_mesh.counts() == b_mesh.counts()
    for x, y in zip(a_mesh.snapshot(), b_mesh.snapshot()):
        assert np.array_equal(x, y)
    assert np.array_equal(a_lio.get_state(), b_lio.get_state())
    ca, cb = a_mesh.changes(0), b_mesh.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key
    for x, y in zip(a_clouds, b_clouds):
        for u, v in zip(x, y):
            assert same(u, v) if u.dtype == np.float32 else np.array_equal(u, v)


def test_enable_then_disable_launches_as_never_enabled(cuda_lib, monkeypatch):
    monkeypatch.setenv("IMMESH_GRAPH", "0")   # every frame launches its kernels
    scans = world_scans("avia", 3, 4)

    def per_frame(mesh):
        out = []
        for k, (wld, t) in enumerate(scans):
            n0 = api.launch_count(cuda_lib)
            mesh.push_frame(wld, t, k)
            out.append(api.launch_count(cuda_lib) - n0)
        return out
    a = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    b = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    b.view_enable(color_by_height=True)
    b.view_disable()
    la, lb = per_frame(a), per_frame(b)
    assert la == lb, (la, lb)
    c = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    c.view_enable(color_by_height=True)
    assert all(x > y for x, y in zip(per_frame(c), la))
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)


def test_empty_mesh(cuda_lib):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    rgba, depth = mesh.render_view(K0, 640, 480, ZN, ZF, np.eye(3), np.zeros(3), color_by_height=True)
    assert (rgba == [0, 0, 0, 255]).all() and (depth == -1).all()
    mesh.view_enable(color_by_height=True)
    mesh.push_frame(np.zeros((0, 3), np.float32), np.zeros(3))
    rgba, depth, R, t, f = mesh.view_image()
    assert (rgba == [0, 0, 0, 255]).all() and (depth == -1).all() and np.array_equal(R, np.eye(3)) and f == 1


def test_error_contract(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    dp, u8, fp = C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.POINTER(C.c_float)
    K = np.array(K0, np.float64)
    R, t = np.eye(3).reshape(9).copy(), np.zeros(3)
    img = np.zeros((480, 640, 4), np.uint8)

    def rv(w=640, h=480, zn=ZN, zf=ZF, style=None, rgba=img, Kd=K):
        return L.immesh_mesh_render_view(mesh._h, None if Kd is None else Kd.ctypes.data_as(dp), w, h, zn, zf, R.ctypes.data_as(dp), t.ctypes.data_as(dp),
                                         None if style is None else C.byref(style), None if rgba is None else rgba.ctypes.data_as(u8), None)
    assert rv() == 0
    for bad in (dict(w=0), dict(zn=0.0), dict(zn=2.0, zf=1.0), dict(rgba=None), dict(Kd=None)):
        assert rv(**bad) == -1, bad
    nan2 = (C.c_double * 2)(float("nan"), float("nan"))
    for style in (api._ViewStyle(2, 0, nan2), api._ViewStyle(0, 2, nan2), api._view_style(0, True, (1.0, 1.0)), api._view_style(0, True, (2.0, 1.0)),
                  api._view_style(0, True, (float("nan"), 1.0)), api._view_style(0, True, (0.0, float("inf")))):
        assert rv(style=style) == -1
    assert rv(style=api._view_style(0, False, (2.0, 1.0))) == 0   # the range is read only with the height colour
    frame = C.c_int64(0)
    assert L.immesh_mesh_view_image(mesh._h, None, None, None, C.byref(frame)) == -1       # not enabled
    assert L.immesh_mesh_view_pose(mesh._h, None, None, 0) == -1                              # not enabled
    for Kb, w, h, zn, zf, win in (((0.0, 400.0, 320.0, 240.0), 640, 480, ZN, ZF, 1), ((400.0, float("nan"), 320.0, 240.0), 640, 480, ZN, ZF, 1),
                                  (K0, 0, 480, ZN, ZF, 1), (K0, 640, 480, 0.0, ZF, 1), (K0, 640, 480, ZN, float("inf"), 1), (K0, 640, 480, ZN, ZF, 0),
                                  (K0, 640, 480, ZN, ZF, 64)):
        Kd = np.array(Kb, np.float64)
        assert L.immesh_mesh_view_enable(mesh._h, Kd.ctypes.data_as(dp), w, h, zn, zf, win, None) == -1, (Kb, w, h, zn, zf, win)
    assert L.immesh_mesh_view_enable(mesh._h, K.ctypes.data_as(dp), 640, 480, ZN, ZF, 1, C.byref(api._view_style(0, True, (3.0, 3.0)))) == -1
    mesh.view_enable()
    assert L.immesh_mesh_view_image(mesh._h, None, None, None, C.byref(frame)) == -1       # no frame yet
    assert L.immesh_mesh_view_pose(mesh._h, R.ctypes.data_as(dp), None, 0) == -1            # mismatched
    assert L.immesh_mesh_view_pose(mesh._h, None, None, 1) == -1                            # follow without a pose
    assert L.immesh_mesh_view_pose(mesh._h, R.ctypes.data_as(dp), t.ctypes.data_as(dp), 2) == -1
    assert L.immesh_mesh_view_pose(mesh._h, R.ctypes.data_as(dp), t.ctypes.data_as(dp), 1) == 0
    mesh.push_frame(np.zeros((0, 3), np.float32), np.array([1.0, 2.0, 3.0]))
    assert L.immesh_mesh_view_image(mesh._h, None, None, None, C.byref(frame)) == 0 and frame.value == 1
    # a handle with the view on refuses to be sharded (the view runs on a single GPU)
    uid = C.create_string_buffer(128)
    assert L.immesh_mesh_shard(mesh._h, 0, 2, uid) == -1
    mesh.view_disable()
    assert L.immesh_mesh_view_image(mesh._h, None, None, None, C.byref(frame)) == -1
