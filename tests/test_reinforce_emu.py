"""CPU tier: the reinforcement's device bodies (immesh_b200/csrc/reinforce.cuh) run by the host emulation (tests/reinforce/
emu_reinforce.cpp) against independent numpy restatements: get_last_avr_pose (ImMesh_node.cpp:169-206) with scipy's Rotation, and the
documented sampling rule pixel by pixel against the tiled rasteriser's count / scan / fill / tile passes and the compaction."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from reinforce_reference import L2C, avr_pose, raster


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_reinforce())
    L.emu_rf_pose.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_rf_raster.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_pose(lib, poses, n_frames, frame, win):
    arr = np.zeros((n_frames, 12))
    has = np.zeros(n_frames, np.int32)
    for f, (R, t) in poses.items():
        arr[f - 1, :9], arr[f - 1, 9:], has[f - 1] = R.reshape(9), t, 1
    R, t = np.zeros(9), np.zeros(3)
    lib.emu_rf_pose(_p(arr), _p(has), n_frames, frame, win, _p(R), _p(t))
    return R.reshape(3, 3), t


def random_poses(n, seed):
    rng = np.random.default_rng(seed)
    rots = Rotation.random(n, random_state=seed)
    ts = np.cumsum(rng.normal(size=(n, 3)), axis=0) * 3.0
    return {f + 1: (rots[f].as_matrix(), ts[f]) for f in range(n)}


@pytest.mark.parametrize("win", [1, 3])
def test_pose_against_scipy(lib, win):
    poses = random_poses(12, seed=win)
    for frame in range(1, 13):
        R, t = emu_pose(lib, poses, 12, frame, win)
        Rn, tn = avr_pose(poses, frame, win)
        assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12, frame
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12 and np.linalg.det(R) > 0


def test_pose_rules(lib):
    poses = random_poses(6, seed=9)
    # the first frame (the reference's cur < 1): the identity, without the camera axes
    R, t = emu_pose(lib, poses, 6, 1, 1)
    assert np.array_equal(R, np.eye(3)) and np.array_equal(t, np.zeros(3))
    # win 1: the previous frame's rotation times lidar_frame_to_camera_frame, its position
    R, t = emu_pose(lib, poses, 6, 4, 1)
    assert np.abs(R - poses[3][0] @ L2C).max() < 1e-14 and np.array_equal(t, poses[3][1])
    # the identity sensor pose gives the camera axes themselves: camera forward (-R[:, 2]) is the sensor's +x
    R, _ = emu_pose(lib, {1: (np.eye(3), np.zeros(3))}, 1, 2, 1)
    assert np.abs(R - L2C).max() < 1e-15 and np.array_equal(-R[:, 2], [1.0, 0.0, 0.0])
    # frames without a pose are skipped; a window with none gives the identity
    part = {f: p for f, p in poses.items() if f != 4}
    R, t = emu_pose(lib, part, 6, 6, 3)
    Rn, tn = avr_pose(part, 6, 3)
    assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12
    R, t = emu_pose(lib, {}, 6, 5, 3)
    assert np.array_equal(R, np.eye(3)) and np.array_equal(t, np.zeros(3))
    # rotations near pi apart inside the window (the log's |w| < eps branch side) still agree
    half = {1: (np.eye(3), np.zeros(3)), 2: (Rotation.from_rotvec([0.0, 0.0, np.pi - 1e-3]).as_matrix(), np.ones(3))}
    R, t = emu_pose(lib, half, 2, 3, 2)
    Rn, tn = avr_pose(half, 3, 2)
    assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12


def emu_raster(lib, K, w, h, zn, zf, R, t, verts, tris):
    cam = np.concatenate([K, [zn, zf], np.asarray(R, np.float64).reshape(9), t]).astype(np.float64)
    v = np.ascontiguousarray(verts, np.float32)
    tr = np.ascontiguousarray(tris, np.int32)
    depth = np.zeros((h, w), np.float32)
    pts = np.zeros((w * h, 3), np.float32)
    pix = np.zeros(w * h, np.int32)
    bins = C.c_longlong(0)
    n = lib.emu_rf_raster(_p(cam), w, h, _p(v), _p(tr), len(tr), _p(depth), _p(pts), _p(pix), C.byref(bins))
    return depth, pts[:n], pix[:n], bins.value


def check_scene(lib, K, w, h, zn, zf, R, t, verts, tris):
    d, p, x, bins = emu_raster(lib, K, w, h, zn, zf, R, t, verts, tris)
    dn, pn, xn = raster(K, w, h, zn, zf, R, t, verts, tris)
    assert np.array_equal(d.view(np.uint32), dn.view(np.uint32))
    assert np.array_equal(x, xn) and np.array_equal(p.view(np.uint32), pn.view(np.uint32))
    return d, bins


# camera at the origin looking down world -z (world = R diag(1,-1,-1) p + t with R = I)
R0, T0 = np.eye(3), np.zeros(3)


def test_large_triangle_covers_many_tiles(lib):
    K, w, h = (40.0, 40.0, 30.0, 20.0), 61, 45
    verts = np.array([[-50.0, -50.0, -2.0], [50.0, -50.0, -2.5], [0.0, 60.0, -3.0]])
    d, bins = check_scene(lib, K, w, h, 0.1, 100.0, R0, T0, verts, [[0, 1, 2]])
    assert (d > 0).all() and bins == 4 * 3   # one triangle, every tile of the 61 x 45 image


def test_samples_exactly_on_edges(lib):
    # vertices on integer pixel coordinates at constant depth: the shared edge of two triangles passes through pixel centres
    K, w, h, z = (10.0, 10.0, 0.0, 0.0), 40, 40, 10.0   # world coordinates = pixel coordinates, exactly
    def at(u, v):
        return [u * z / 10.0, -(v * z / 10.0), -z]
    verts = np.array([at(2, 2), at(30, 2), at(2, 30), at(30, 30), at(10, 10), at(20, 20)], np.float32)
    tris = [[0, 1, 2], [1, 3, 2], [4, 5, 1]]
    d, _ = check_scene(lib, K, w, h, 0.1, 100.0, R0, T0, verts, tris)
    assert d[2, 2] > 0 and d[30, 30] > 0 and d[16, 16] > 0 and d[31, 31] == -1


def test_vertex_behind_z_near_is_skipped(lib):
    K, w, h = (20.0, 20.0, 16.0, 16.0), 33, 33
    verts = np.array([[-1.0, -1.0, -2.0], [1.0, -1.0, -2.0], [0.0, 1.0, -0.05],     # one vertex nearer than z_near: skipped
                      [-1.0, -1.0, -3.0], [1.0, -1.0, -3.0], [0.0, 1.0, -3.0]])
    d, _ = check_scene(lib, K, w, h, 0.1, 100.0, R0, T0, verts, [[0, 1, 2], [3, 4, 5]])
    assert d.max() == np.float32(3.0)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_scenes(lib, seed):
    """random triangles in front of a rotated, moved camera, some beyond the image, z_far and z_near; many overlapping"""
    rng = np.random.default_rng(seed)
    K, w, h = (60.0, 55.0, 37.5, 24.0), 75, 50
    R = Rotation.random(random_state=seed).as_matrix()
    t = rng.normal(size=3)
    pc = np.stack([rng.uniform(-6, 6, 300), rng.uniform(-4, 4, 300), rng.uniform(0.05, 30, 300)], axis=1)   # camera frame, z forward
    verts = ((pc @ np.diag([1.0, -1.0, -1.0]).T) @ R.T + t).astype(np.float32)
    tris = np.array([rng.choice(300, 3, replace=False) for _ in range(400)])
    d, bins = check_scene(lib, K, w, h, 0.2, 25.0, R, t, verts, tris)
    assert (d > 0).sum() > 500 and bins > 400
