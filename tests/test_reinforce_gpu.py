"""GPU tier: the LiDAR point-cloud reinforcement queued behind every mesh frame (immesh_mesh_reinforce_enable / _pose /
immesh_mesh_reinforced_cloud).  Every frame's result against the blocking immesh_mesh_render_depth at the pose the frame used, bit
for bit (both run the same kernels: this checks the pose, the double buffer and the graph); the newest frame of a stream, a facet
that fills the image and the empty mesh also against the numpy restatement of the sampling rule on the mesh's snapshot, bit for bit;
the pose against the numpy restatement of get_last_avr_pose; nothing else changes; the frames are graph-replayed; the error paths."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL
from reinforce_reference import avr_pose, raster

pytestmark = pytest.mark.gpu

K0 = api.reinforce_intrinsics(640, 480)
ZN, ZF = 0.1, 1500.0


def same(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check_frame(mesh, K=K0, w=640, h=480, zn=ZN, zf=ZF, restated=False):
    """the newest frame's queued result against render_depth at the pose it reports and, with restated, against the numpy
    rasteriser on the mesh's snapshot; returns (points, pose)"""
    d, p, x, R, t = mesh.reinforced_cloud()
    dr, pr, xr = mesh.render_depth(K, w, h, zn, zf, R, t)
    assert same(d, dr), "depth image differs from render_depth"
    assert np.array_equal(x, xr) and same(p, pr), "points / pixels differ from render_depth"
    if restated:
        mesh.wait()   # snapshot() sizes its arrays by counts(), which a queued frame updates when it is drained
        v, tri, _ = mesh.snapshot()
        dn, pn, xn = raster(K, w, h, zn, zf, R, t, v, tri)
        assert same(d, dn), "depth image differs from the numpy restatement"
        assert np.array_equal(x, xn) and same(p, pn), "points / pixels differ from the numpy restatement"
    return p, (R, t)


def run_stream(lib, win=1, reinforce=True, n_scans=8, seed=3, read=True):
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    if reinforce:
        mesh.reinforce_enable(win=win)
    poses, out = {}, []
    for k in range(1, n_scans):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if reinforce and read:
            pts, (R, t) = check_frame(mesh, restated=k == n_scans - 1)
            s = lio.get_state()
            poses[k] = (s[0:9].reshape(3, 3).copy(), s[9:12].copy())   # the pose frame k was transformed with
            Rn, tn = avr_pose(poses, k, win)
            assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12, (k, R, Rn, t, tn)
            out.append(len(pts))
    lio.wait()
    mesh.wait()
    return lio, mesh, out


@pytest.mark.parametrize("win", [1, 3])
def test_avia_stream_against_render_depth(cuda_lib, win):
    lio, mesh, n = run_stream(cuda_lib, win=win)
    assert n[0] >= 0 and max(n) > 5000, n
    st = api.graph_stats(None, mesh)
    assert st["mesh_captures"] == 1 and st["mesh_replays"] == len(n) - 1, st


def test_nothing_else_changes(cuda_lib):
    a_lio, a_mesh, _ = run_stream(cuda_lib, reinforce=True, read=False)
    b_lio, b_mesh, _ = run_stream(cuda_lib, reinforce=False)
    assert a_mesh.counts() == b_mesh.counts()
    for x, y in zip(a_mesh.snapshot(), b_mesh.snapshot()):
        assert np.array_equal(x, y)
    assert np.array_equal(a_lio.get_state(), b_lio.get_state())
    assert np.array_equal(a_lio.dump_map(), b_lio.dump_map())
    check_frame(a_mesh)   # the newest frame, read after the stream drained


def test_large_triangle_and_explicit_pose(cuda_lib):
    """a camera a few centimetres in front of one facet, looking at it: that facet covers every tile of the image"""
    lio, mesh, _ = run_stream(cuda_lib, read=False, n_scans=4)
    v, tri, _ = mesh.snapshot()
    P = v[tri].astype(np.float64)
    n = np.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0])
    area = np.linalg.norm(n, axis=1)
    i = int(np.argmax(area))
    c, nz = P[i].mean(axis=0), n[i] / area[i]
    ax = np.cross(nz, [0.0, 0.0, 1.0] if abs(nz[2]) < 0.9 else [1.0, 0.0, 0.0])
    ax /= np.linalg.norm(ax)
    ay = np.cross(nz, ax)
    cam_t = c + 0.02 * nz
    R = np.stack([ax, -ay, nz], axis=1)   # camera forward (world = R diag(1,-1,-1) p): -R[:, 2] = -nz, towards the facet
    K = (400.0, 400.0, 320.0, 240.0)
    mesh.reinforce_enable(K, 640, 480, 0.005, 100.0, 1)
    mesh.reinforce_pose(R, cam_t)
    mesh.push_frame(np.zeros((0, 3), np.float32), cam_t)
    d, p, x, Rr, tr = mesh.reinforced_cloud()
    assert np.array_equal(Rr, R) and np.array_equal(tr, cam_t)
    check_frame(mesh, K, 640, 480, 0.005, 100.0, restated=True)
    assert (d > 0).mean() > 0.9
    # back to the sensor-bound pose: a frame with world points records none, so the window is empty -> identity
    mesh.reinforce_pose(None)
    mesh.push_frame(np.zeros((0, 3), np.float32), cam_t)
    _, _, _, Ri, ti = mesh.reinforced_cloud()
    assert np.array_equal(Ri, np.eye(3)) and np.array_equal(ti, np.zeros(3))


def test_empty_mesh(cuda_lib):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.reinforce_enable()
    mesh.push_frame(np.zeros((0, 3), np.float32), np.zeros(3))
    d, p, x, R, t = mesh.reinforced_cloud()
    assert (d == -1).all() and len(p) == 0 and np.array_equal(R, np.eye(3))
    check_frame(mesh, restated=True)


def test_error_paths(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    n = C.c_int(0)
    assert L.immesh_mesh_reinforced_cloud(mesh._h, None, None, None, 0, C.byref(n), None) == -1      # not enabled
    for K, w, h, zn, zf, win in (((0.0, 400.0, 320.0, 240.0), 640, 480, ZN, ZF, 1), ((400.0, float("nan"), 320.0, 240.0), 640, 480, ZN, ZF, 1),
                                 (K0, 0, 480, ZN, ZF, 1), (K0, 640, 480, 0.0, ZF, 1), (K0, 640, 480, 2.0, 1.0, 1), (K0, 640, 480, ZN, ZF, 0),
                                 (K0, 640, 480, ZN, ZF, 64)):
        Kd = np.array(K, np.float64)
        assert L.immesh_mesh_reinforce_enable(mesh._h, Kd.ctypes.data_as(C.POINTER(C.c_double)), w, h, zn, zf, win) == -1, (K, w, h, zn, zf, win)
    mesh.reinforce_enable()
    assert L.immesh_mesh_reinforced_cloud(mesh._h, None, None, None, 0, C.byref(n), None) == -1      # no frame yet
    from mesh_common import world_scans
    for k, (wld, t) in enumerate(world_scans("avia", 3, 4)):
        mesh.reinforce_pose(*avr_pose({1: (np.eye(3), t)}, 2, 1))
        mesh.push_frame(wld, t, k)
    d, p, x, R, t = mesh.reinforced_cloud()
    assert len(p) > 100
    pts = np.zeros((len(p) - 1, 3), np.float32)
    assert L.immesh_mesh_reinforced_cloud(mesh._h, None, pts.ctypes.data_as(C.POINTER(C.c_float)), None, len(p) - 1, C.byref(n), None) == -3
    assert n.value == len(p) and not pts.any()
    # a handle with the reinforcement on refuses to be sharded (the reinforcement runs on a single GPU)
    uid = C.create_string_buffer(128)
    assert L.immesh_mesh_shard(mesh._h, 0, 2, uid) == -1
    mesh.reinforce_disable()
    assert L.immesh_mesh_reinforced_cloud(mesh._h, None, None, None, 0, C.byref(n), None) == -1
