"""GPU tier of the texturing queued behind every frame (immesh_mesh_texture_enable / _pose / _rows):
- frames that add nothing, each at a caller camera, give exactly immesh_mesh_texture_select's rows over those cameras (camera k <->
  frame f0 + k), the mesh unchanged;
- Avia-shaped localization hand-offs and depth frames in rig mode equal the numpy fold (tests/texture_online_reference.py) over each
  frame's mesh, rows and frames list bit for bit;
- a handle with the texturing on meshes exactly as a twin without it; rows read behind queued frames equal rows read after wait();
- a handle that grows its triangle pool mid-run gives the rows of one created at the larger capacity;
- rows -> texture_bake -> write_obj_textured with the cameras indexed by frame number and None images for unused frames;
- disable, re-enable and the error contract."""
import ctypes as C
import os

import numpy as np
import pytest

import depth_reference as dr
from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans
from texture_online_reference import fold, rows

pytestmark = pytest.mark.gpu

E_INVALID, E_CAPACITY = -1, -3
# the colour camera in the localization body frame: OpenCV axes with z along the body's +x; 10 cm ahead, 5 cm up
R_EXT = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
T_EXT = np.array([0.1, 0.0, 0.05])
W, H = 320, 240
K = (160.0, 160.0, 159.5, 119.5)
RIG = (W, H, K, R_EXT, T_EXT)


def yaw(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def same_uv(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def same_rows(got, ref):
    assert np.array_equal(got["cam"], ref["cam"]), int((got["cam"] != ref["cam"]).sum())
    assert np.array_equal(got["px"], ref["px"]), "won / covered differ"
    assert same_uv(got["uv"], ref["uv"]), "texture coordinates differ"
    assert [got["counts"][k] for k in api.TEXTURE_COUNT_KEYS] == list(ref["counts"]), (got["counts"], ref["counts"])
    assert np.array_equal(got["frames"], ref["frames"]), (got["frames"], ref["frames"])


def test_static_frames_equal_texture_select(cuda_lib):
    sensor, scans = synth.make_stream("avia", 4, seed=5)
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    for k, (wld, t) in enumerate(world_scans("avia", 4, 5)):
        mesh.push_frame(wld, t, k)
    v, tri, fl = mesh.snapshot()
    assert len(tri) > 1000
    cams = []
    for s in scans[1:]:
        for a in (0.0, np.radians(70.0)):
            cams.append((W, H, K, s["R_true"] @ yaw(a) @ R_EXT, s["t_true"] + s["R_true"] @ T_EXT))
    mesh.texture_enable(RIG, min_visible_permille=100)
    f0 = 5   # frames 1..4 built the mesh
    for k, (_, _, _, R, t) in enumerate(cams):
        mesh.texture_pose(R, t)
        mesh.push_frame(np.zeros((0, 3), np.float32), t, 4 + k)
    got = mesh.texture_rows()
    for x, y in zip((v, tri, fl), mesh.snapshot()):
        assert np.array_equal(x, y)
    sel = mesh.texture_select(cams, min_visible_permille=100, vertices=False)
    expect = np.where(sel["cam"] >= 0, sel["cam"] + f0, -1).astype(np.int32)
    assert np.array_equal(got["cam"], expect)
    assert np.array_equal(got["px"], sel["px"]) and same_uv(got["uv"], sel["uv"])
    assert got["counts"] == sel["counts"], (got["counts"], sel["counts"])
    assert np.array_equal(got["frames"], np.unique(expect[expect >= 0]))
    assert got["counts"]["textured"] > 200 and got["counts"]["cameras_used"] >= 3


def lio_run(lib, n_scans, tex=True, cfg_kw=None, per_frame=None, growth=0):
    """localization steps and push_frame_from_lio_async with the change feed; per_frame(k, mesh, lio) after queueing scan k"""
    from lio_common import init_velocity
    sensor, scans = synth.make_stream("avia", n_scans, seed=3, ext_T=api.AVIA.ext_T)
    lio, mesh = api.Lio(api.AVIA, lib=lib), api.Mesh(api.MeshConfig(**{**SMALL, **(cfg_kw or {})}), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    mesh.changes_enable(1 << 20, 64)
    if growth:
        mesh.set_growth(growth)
    if tex:
        mesh.texture_enable(RIG)
    for k in range(1, n_scans):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if per_frame:
            per_frame(k, mesh, lio)
    lio.wait()
    mesh.wait()
    return mesh


def test_lio_frames_against_fold(cuda_lib):
    frames = []

    def record(k, mesh, lio):
        lio.wait()
        mesh.wait()
        s = lio.get_state()
        v, tri, fl = mesh.snapshot()
        frames.append(dict(number=k, verts=v, tris=tri, flips=fl, pose=(s[:9].reshape(3, 3), s[9:12])))

    mesh = lio_run(cuda_lib, 8, per_frame=record)
    got = mesh.texture_rows()
    state, pixels = fold(dict(width=W, height=H, K=K, R=R_EXT, t=T_EXT), frames)
    _, tri, fl = mesh.snapshot()
    same_rows(got, rows(state, pixels, tri, fl))
    assert got["counts"]["textured"] > 100 and len(got["frames"]) >= 3


def test_depth_frames_against_fold(cuda_lib):
    cam = dr.camera()
    mesh = api.Mesh(api.MeshConfig(**dict(SMALL, number_of_pts_append_to_map=4000)), lib=cuda_lib)
    rig_R, rig_t = yaw(0.05) @ np.eye(3), np.array([0.03, -0.01, 0.0])
    rig = (160, 120, (cam.fx, cam.fy, cam.cx, cam.cy), rig_R, rig_t)
    mesh.texture_enable(rig)
    frames = []
    rng = np.random.default_rng(0)
    for k in range(6):
        R, t = dr.camera_pose(k)
        img = dr.inject_edges(dr.render(cam, 160, 120, R, t), cam, rng)
        mesh.push_depth_async(img, cam, R, t)
        mesh.wait()
        v, tri, fl = mesh.snapshot()
        frames.append(dict(number=k + 1, verts=v, tris=tri, flips=fl, pose=(R, t)))
    got = mesh.texture_rows()
    state, pixels = fold(dict(width=160, height=120, K=rig[2], R=rig_R, t=rig_t), frames)
    _, tri, fl = mesh.snapshot()
    same_rows(got, rows(state, pixels, tri, fl))
    assert got["counts"]["textured"] > 50


def test_twin_and_queued_rows(cuda_lib):
    seen = {}

    def read(k, mesh, lio):
        if k == 6:
            queued = mesh.texture_rows(vertices=False)   # behind the frames still queued
            mesh.wait()
            after = mesh.texture_rows()
            for key in ("cam", "px", "frames"):
                assert np.array_equal(queued[key], after[key]), key
            assert same_uv(queued["uv"], after["uv"]) and queued["counts"] == after["counts"]
            seen[k] = after["counts"]

    a = lio_run(cuda_lib, 10, per_frame=read)
    b = lio_run(cuda_lib, 10, tex=False)
    assert seen[6]["textured"] > 0
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    assert a.counts() == b.counts()
    ca, cb = a.changes(0), b.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key


def test_growth_mid_run(cuda_lib):
    small = lio_run(cuda_lib, 8, cfg_kw=dict(max_triangles=1 << 12), growth=1 << 40)
    big = lio_run(cuda_lib, 8)
    assert small.capacity()["growths"] > 0 and small.capacity()["triangles_cap"] > 1 << 12
    a, b = small.texture_rows(), big.texture_rows()
    for key in ("cam", "px", "frames"):
        assert np.array_equal(a[key], b[key]), key
    assert same_uv(a["uv"], b["uv"]) and a["counts"] == b["counts"]


def test_bake_and_export(cuda_lib, tmp_path):
    mesh = lio_run(cuda_lib, 6)
    r = mesh.texture_rows()
    n_cams = int(r["frames"][-1]) + 1
    cams = [RIG] * n_cams   # indexed by frame number: width and height
    rng = np.random.default_rng(1)
    images = [rng.integers(0, 256, (H, W, 3), np.uint8) if f in set(r["frames"].tolist()) else None for f in range(n_cams)]
    bake = mesh.texture_bake(r, cams, images, page_size=1024)
    assert bake["counts"]["textured"] == r["counts"]["textured"] and len(bake["pages"]) >= 1
    v, tri, fl = mesh.snapshot()
    files = [f"frame_{f:06d}.png" for f in range(n_cams)]
    api.write_obj_textured(str(tmp_path / "m.obj"), str(tmp_path / "m.mtl"), v, tri, fl, r["cam"], r["uv"], [(W, H)] * n_cams, files, lib=cuda_lib)
    mtl = open(tmp_path / "m.mtl").read()
    for f in r["frames"]:
        if f in set(r["cam"].tolist()):
            assert f"map_Kd frame_{int(f):06d}.png" in mtl
    pages = [str(tmp_path / f"p{i}.png") for i in range(len(bake["pages"]))]
    api.write_obj_textured(str(tmp_path / "a.obj"), str(tmp_path / "a.mtl"), v, tri, fl, bake["page"], bake["uv"], [(1024, 1024)] * len(pages), pages,
                           lib=cuda_lib)
    assert os.path.getsize(tmp_path / "a.obj") > 0


def test_disable_reenable_and_errors(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    h = mesh._h
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    nf, nfr = C.c_int64(0), C.c_int64(0)
    assert L.immesh_mesh_texture_rows(h, None, None, None, 0, C.byref(nf), None, None, 0, None) == E_INVALID   # off
    assert L.immesh_mesh_texture_pose(h, None, None) == E_INVALID
    arr, _ = api.texture_cameras([RIG])
    for cfg in (api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 1, 0), api._TexCfg(0.0, 1000.0, 0.0, 0, 0, 0, 0), api._TexCfg(0.1, 1000.0, 0.0, 1001, 0, 0, 0)):
        assert L.immesh_mesh_texture_enable(h, arr, C.byref(cfg)) == E_INVALID
    bad, _ = api.texture_cameras([(0, H, K, R_EXT, T_EXT)])
    good = api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 0, 0)
    assert L.immesh_mesh_texture_enable(h, bad, C.byref(good)) == E_INVALID
    assert L.immesh_mesh_texture_enable(h, arr, None) == E_INVALID
    mesh.texture_enable(RIG)
    R = np.ascontiguousarray(np.eye(3)).reshape(9)
    assert L.immesh_mesh_texture_pose(h, R.ctypes.data_as(C.POINTER(C.c_double)), None) == E_INVALID   # mismatched NULLs
    assert L.immesh_mesh_texture_rows(h, None, None, None, -1, C.byref(nf), None, None, 0, None) == E_INVALID
    assert L.immesh_mesh_texture_rows(h, None, None, None, 0, None, None, None, 0, None) == E_INVALID
    fr = np.zeros(4, np.int32)
    assert L.immesh_mesh_texture_rows(h, None, None, None, 0, C.byref(nf), None, fr.ctypes.data_as(i32), 4, None) == E_INVALID
    # world-frame pushes have no camera: nothing observed until a caller camera is set
    scans = world_scans("avia", 3, 5)
    for k, (wld, t) in enumerate(scans[:2]):
        mesh.push_frame(wld, t, k)
    r = mesh.texture_rows()
    assert r["counts"]["textured"] == 0 and r["counts"]["pixels"] == 0 and len(r["frames"]) == 0 and len(r["cam"]) > 0
    s1 = synth.make_stream("avia", 3, seed=5)[1][1]
    mesh.texture_pose(s1["R_true"] @ R_EXT, s1["t_true"] + s1["R_true"] @ T_EXT)
    mesh.push_frame(np.zeros((0, 3), np.float32), scans[1][1], 2)
    r = mesh.texture_rows()
    assert r["counts"]["pixels"] == W * H and list(r["frames"]) == [3] and r["counts"]["textured"] > 0
    n = len(r["cam"])
    cam = np.full(n, 7, np.int32)
    counts = np.zeros(4, np.int64)
    # a short cap or cap_frames: the counts, nothing written
    assert L.immesh_mesh_texture_rows(h, cam.ctypes.data_as(i32), None, None, n - 1, C.byref(nf), counts.ctypes.data_as(i64), None, 0, C.byref(nfr)) == E_CAPACITY
    assert nf.value == n and nfr.value == 1 and (cam == 7).all() and counts[0] == r["counts"]["textured"]
    assert L.immesh_mesh_texture_rows(h, cam.ctypes.data_as(i32), None, None, n, C.byref(nf), None, fr.ctypes.data_as(i32), 0, C.byref(nfr)) == E_CAPACITY
    assert (cam == 7).all()
    assert L.immesh_mesh_texture_rows(h, cam.ctypes.data_as(i32), None, None, n, C.byref(nf), None, fr.ctypes.data_as(i32), 4, C.byref(nfr)) == 0
    assert np.array_equal(cam, r["cam"]) and fr[0] == 3
    # disable: off again; enable again: every record starts unobserved
    mesh.texture_enable(None)
    assert L.immesh_mesh_texture_rows(h, None, None, None, 0, C.byref(nf), None, None, 0, None) == E_INVALID
    mesh.texture_enable(RIG)
    r = mesh.texture_rows()
    assert r["counts"] == dict(textured=0, untextured=n, cameras_used=0, pixels=0) and len(r["frames"]) == 0
    mesh.texture_pose(None, None)
    mesh.push_frame(scans[2][0], scans[2][1], 3)
    assert mesh.texture_rows()["counts"]["pixels"] == 0
