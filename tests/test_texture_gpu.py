"""GPU tier of the textured mesh (immesh_mesh_texture_select): meshes of Avia-shaped and HDL-64 synthetic streams with 6 cameras along
the trajectory, posed from the frames' poses and a fixed extrinsic, at 320 x 240 and at half that resolution (scaled intrinsics),
positions 0 and 1, against the numpy restatement of the selection rule (tests/texture_reference.py) on immesh_mesh_snapshot: the
chosen camera, won and covered pixels exactly, the texture coordinates bit for bit.  A call issued behind queued
push_frame_from_lio_async frames equals one made after wait(); a handle that textured computes the same later frames and change-feed
rows as a twin that never did; the error contract."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans
from texture_reference import camera, select

pytestmark = pytest.mark.gpu

# the camera in the sensor frame: OpenCV axes with z along the sensor's +x, x along -y, y along -z; 10 cm ahead, 5 cm up
R_EXT = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
T_EXT = np.array([0.1, 0.0, 0.05])
W, H = 320, 240
K = (160.0, 160.0, 159.5, 119.5)


def yaw(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def trajectory_cameras(poses, scale=1.0):
    """two cameras per pose (ahead, and turned 70 degrees left): cam_R = R yaw R_EXT, cam_t = t + R T_EXT; intrinsics scaled"""
    w, h = int(W * scale), int(H * scale)
    Ks = (K[0] * scale, K[1] * scale, (K[2] + 0.5) * scale - 0.5, (K[3] + 0.5) * scale - 0.5)
    cams = []
    for R, t in poses:
        for a in (0.0, np.radians(70.0)):
            cams.append(camera(w, h, Ks, R @ yaw(a) @ R_EXT, t + R @ T_EXT))
    return cams


def as_tuples(cams):
    return [(c["width"], c["height"], c["K"], c["R"], c["t"]) for c in cams]


def world_mesh(lib, kind, n_frames=4, seed=5):
    sensor, scans = synth.make_stream(kind, n_frames, seed=seed)
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    for k, (wld, t) in enumerate(world_scans(kind, n_frames, seed)):
        mesh.push_frame(wld, t, k)
    return mesh, [(s["R_true"], s["t_true"]) for s in scans[1:]]


def same_uv(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check(mesh, cams, verts, tris, flips, **kw):
    got = mesh.texture_select(as_tuples(cams), **kw)
    ref = select(cams, verts, tris, flips, **{k: v for k, v in kw.items() if k != "positions"})
    assert np.array_equal(got["cam"], ref["cam"]), int((got["cam"] != ref["cam"]).sum())
    assert np.array_equal(got["px"], ref["px"]), "won / covered differ"
    assert same_uv(got["uv"], ref["uv"]), "texture coordinates differ"
    assert [got["counts"][k] for k in api.TEXTURE_COUNT_KEYS] == ref["counts"].tolist()
    assert same_uv(got["vertices"], np.asarray(verts, np.float32)), "positions differ"
    return got


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_texture_select_against_restatement(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    v, tri, fl = mesh.snapshot()
    assert len(tri) > 1000
    cams = trajectory_cameras(poses)
    assert len(cams) == 6
    full = check(mesh, cams, v, tri, fl)
    assert full["counts"]["textured"] > 200 and full["counts"]["cameras_used"] >= 3, full["counts"]
    check(mesh, cams, v, tri, fl, min_cos=0.2, min_visible_permille=500)
    half = check(mesh, trajectory_cameras(poses, 0.5), v, tri, fl, two_sided=True)
    assert half["counts"]["textured"] > 0
    # the smoothed positions (every vertex smoothed by smooth_all), as floats
    vs = mesh.smooth_all(1.0, 20).astype(np.float32)
    sm = check(mesh, cams, vs, tri, fl, positions=1)
    check(mesh, trajectory_cameras(poses, 0.5), vs, tri, fl, positions=1, min_cos=0.1)
    assert not np.array_equal(sm["uv"], full["uv"], equal_nan=True)
    # the call wrote nothing on the handle
    v2, tri2, fl2 = mesh.snapshot()
    assert np.array_equal(v, v2) and np.array_equal(tri, tri2) and np.array_equal(fl, fl2)


def lio_chain(lib, n_scans, between=None, feed=True):
    """the queued chain (localization step + push_frame_from_lio_async) with the change feed; between(k, mesh, scans) after queueing scan k"""
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=3, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    if feed:
        mesh.changes_enable(1 << 20, 64)
    for k in range(1, n_scans):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if between:
            between(k, mesh, scans)
    lio.wait()
    mesh.wait()
    return lio, mesh, scans


def test_queued_frames_and_twin(cuda_lib):
    seen = {}

    def texture(k, mesh, scans):
        if k in (4, 6):
            cams = as_tuples(trajectory_cameras([(s["R_true"], s["t_true"]) for s in scans[k - 2:k + 1]]))
            queued = mesh.texture_select(cams, vertices=False)   # behind the frames still queued
            mesh.wait()
            after = mesh.texture_select(cams)
            for key in ("cam", "px"):
                assert np.array_equal(queued[key], after[key]), key
            assert same_uv(queued["uv"], after["uv"]) and queued["counts"] == after["counts"]
            seen[k] = after["counts"]

    _, a, _ = lio_chain(cuda_lib, 10, between=texture)
    _, b, _ = lio_chain(cuda_lib, 10)
    assert seen[6]["textured"] > 0
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    assert a.counts() == b.counts()
    ca, cb = a.changes(0), b.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key


def test_empty_mesh_and_error_contract(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    cams = trajectory_cameras([(np.eye(3), np.zeros(3))])
    r = mesh.texture_select(as_tuples(cams))
    assert len(r["cam"]) == 0 and r["counts"] == dict(textured=0, untextured=0, cameras_used=0, pixels=2 * W * H)
    for k, (wld, t) in enumerate(world_scans("avia", 2, 5)):
        mesh.push_frame(wld, t, k)
    n_live = mesh.counts()["n_triangles"]
    arr, n = api.texture_cameras(as_tuples(cams))
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    nf, counts = C.c_int64(0), np.zeros(4, np.int64)
    cam = np.full(n_live, 7, np.int32)

    def ts(cfg=None, cams_arr=arr, n_cams=n, cap=n_live, out=cam):
        cfg = cfg or api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 0, 0)
        return L.immesh_mesh_texture_select(mesh._h, cams_arr, n_cams, C.byref(cfg), None if out is None else out.ctypes.data_as(i32), None, None, None, cap,
                                            C.byref(nf), counts.ctypes.data_as(i64))
    assert ts() == 0 and nf.value == n_live and (cam >= -1).all() and (cam < 2).all()
    cam[:] = 7
    assert ts(cap=n_live - 1) == -3 and nf.value == n_live and (cam == 7).all()   # a short cap: the count, nothing written
    assert ts(cap=0, out=None) == -3 and nf.value == n_live                        # a count query
    for cfg in (api._TexCfg(0.0, 1000.0, 0.0, 0, 0, 0, 0), api._TexCfg(2.0, 1.0, 0.0, 0, 0, 0, 0), api._TexCfg(0.1, float("inf"), 0.0, 0, 0, 0, 0),
                api._TexCfg(0.1, 1000.0, -0.1, 0, 0, 0, 0), api._TexCfg(0.1, 1000.0, 1.5, 0, 0, 0, 0), api._TexCfg(0.1, 1000.0, 0.0, -1, 0, 0, 0),
                api._TexCfg(0.1, 1000.0, 0.0, 1001, 0, 0, 0), api._TexCfg(0.1, 1000.0, 0.0, 0, 2, 0, 0), api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 2, 0)):
        assert ts(cfg=cfg) == -1
    assert ts(n_cams=0) == -1 and ts(cap=-1) == -1
    assert L.immesh_mesh_texture_select(mesh._h, None, 1, C.byref(api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 0, 0)), None, None, None, None, 0, C.byref(nf), None) == -1
    good = as_tuples(cams)[0]
    for bad in ((0, H, K, good[3], good[4]), (W, H, (0.0, 160.0, 1.0, 1.0), good[3], good[4]), (W, H, (160.0, float("nan"), 1.0, 1.0), good[3], good[4]),
                (1 << 14, 1 << 13, K, good[3], good[4]), (W, H, K, np.full((3, 3), np.inf), good[4])):
        barr, bn = api.texture_cameras([good, bad])
        assert ts(cams_arr=barr, n_cams=bn) == -1, bad[:3]
    # positions = 1 with no vertex smoothed by the caller reads the raw position where m_smoothed is clear: a valid call
    assert ts(cfg=api._TexCfg(0.1, 1000.0, 0.0, 0, 0, 1, 0)) == 0
