"""CPU tier: the queued view's overlays (immesh_b200/csrc/view_overlay.cuh) run by the host emulation
(tests/view_overlay/emu_view_overlay.cpp) in the device chain's orchestration, against the numpy restatement of the rule
(tests/view_overlay_reference.py), byte for byte and depth bit for bit: each layer alone and all together, segments crossing the
near and far planes or wholly behind the camera, lines over many tiles, wide lines and large points at image and tile borders,
equal-depth ties between and inside layers, shared wireframe edges, bin overflow, a trajectory ring that wraps, and the frustum's
vertices against scipy rotations."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from view_overlay_reference import CAMERA, NONE, PATH, SCAN, frustum, key_of, overlay_keys, render_overlay

W, H = 96, 80
K = (60.0, 60.0, 47.5, 39.5)


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_view_overlay())
    vp, i = C.c_void_p, C.c_int
    L.emu_ov_render.argtypes = [vp, i, i, vp, i, vp, i, i, vp, C.c_longlong, i, vp, i, i, vp, i, i, i, vp, vp, vp, i, i, C.c_double, i, i,
                                vp, vp, vp, vp, vp]
    L.emu_ov_frustum.argtypes = [vp, vp, C.c_double, vp]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def look_at(eye, target):
    f = np.asarray(target, np.float64) - eye
    f /= np.linalg.norm(f)
    x = np.cross(f, [0.0, 0.0, 1.0])
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(x, f), -f], axis=1)


class Frames:
    """frames 1..n: rot_end / pos_end (has = 0: a world-frame push with pose_t only)"""

    def __init__(self, n, seed=0, has=None, center=(0.0, 0.0, 0.0), spread=3.0):
        rng = np.random.default_rng(seed)
        self.R = Rotation.random(n, random_state=seed).as_matrix().reshape(n, 3, 3)
        self.t = np.asarray(center) + rng.normal(scale=spread, size=(n, 3))
        self.has = np.ones(n, np.int32) if has is None else np.asarray(has, np.int32)

    def poses(self):
        return np.concatenate([self.R.reshape(-1, 9), self.t], axis=1)


def both(lib, R, t, verts=None, tris=None, zn=0.1, zf=1500.0, color=False, z_range=None, wire=False, scan=None, scan_size=0, rf=None, rf_size=0,
         axis_and_grid=False, frames=None, path_from=1, camera_size=0.0, path_width=0, path_cap=16, bin_cap=1 << 30, w=W, h=H):
    """(emulated rgba, depth, keys, overflow) after checking them against the restatement"""
    verts = np.zeros((0, 3), np.float32) if verts is None else np.ascontiguousarray(verts, np.float32)
    tris = np.zeros((0, 3), np.int32) if tris is None else np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    frames = frames or Frames(1)
    nf = len(frames.t)
    cam = np.concatenate([K, [zn, zf], np.asarray(R, np.float64).reshape(9), t]).astype(np.float64)
    zr = np.array([np.nan, np.nan] if z_range is None else z_range, np.float64)
    sc = np.zeros((0, 3), np.float32) if scan is None else np.ascontiguousarray(scan, np.float32)
    rp = np.zeros((0, 3), np.float32) if rf is None else np.ascontiguousarray(rf, np.float32)
    poses, pos = np.ascontiguousarray(frames.poses()), np.ascontiguousarray(frames.t)
    rgba = np.zeros((h, w, 4), np.uint8)
    depth = np.zeros((h, w), np.float32)
    keys = np.zeros((h, w), np.uint64)
    bins, over = C.c_longlong(0), C.c_int(0)
    lib.emu_ov_render(_p(cam), w, h, _p(verts), len(verts), _p(tris), len(tris), int(color), _p(zr), bin_cap, int(wire), _p(sc), len(sc), scan_size,
                      _p(rp), len(rp), rf_size, int(axis_and_grid), _p(poses), _p(frames.has), _p(pos), nf, path_from, camera_size, path_width,
                      path_cap, _p(rgba), _p(depth), _p(keys), C.byref(bins), C.byref(over))
    path = [frames.t[f - 1] for f in range(path_from, nf + 1)][-path_cap:] if path_width > 0 else []
    fp = (frames.R[-1], frames.t[-1]) if frames.has[-1] else None
    ov = dict(scan=sc if nf >= 2 else None, scan_size=scan_size, rf=rp, rf_size=rf_size, axis_and_grid=axis_and_grid, frustum_pose=fp,
              camera_size=camera_size, path=path, path_width=path_width)
    kn = overlay_keys(K, w, h, zn, zf, np.asarray(R, np.float64), np.asarray(t, np.float64), **ov)
    assert np.array_equal(keys, kn), f"overlay keys differ at {np.argwhere(keys != kn)[:5]}"
    rn, dn = render_overlay(K, w, h, zn, zf, R, t, verts, tris, color, z_range, wire, **ov)
    assert np.array_equal(depth.view(np.uint32), dn.view(np.uint32)), "depth differs from the restatement"
    bad = np.argwhere((rgba != rn).any(axis=2))
    assert len(bad) == 0, (len(bad), bad[:5], rgba[tuple(bad[0])], rn[tuple(bad[0])])
    return rgba, depth, keys, over.value


def scene(seed, n_verts=120, n_tris=150):
    """a camera 30 m above the grid looking down at a random mesh near the origin, with scan points over it"""
    rng = np.random.default_rng(seed)
    eye = np.array([-20.0, -14.0, 18.0]) + rng.normal(size=3)
    R = look_at(eye, np.zeros(3))
    verts = rng.uniform([-6, -6, -1], [6, 6, 4], size=(n_verts, 3)).astype(np.float32)
    tris = np.sort(np.array([rng.choice(n_verts, 3, replace=False) for _ in range(n_tris)]), axis=1)
    scan = rng.uniform([-15, -15, -1], [15, 15, 5], size=(400, 3)).astype(np.float32)
    rf = rng.uniform([-8, -8, 0], [8, 8, 3], size=(300, 3)).astype(np.float32)
    return R, eye, verts, tris, scan, rf


ALL = dict(scan_size=2, rf_size=2, axis_and_grid=True, camera_size=1.0, path_width=4)


@pytest.mark.parametrize("layer", ["scan", "rf", "axis_and_grid", "camera", "path", "all"])
@pytest.mark.parametrize("wire", [False, True])
def test_each_layer_and_all(lib, layer, wire):
    R, eye, verts, tris, scan, rf = scene(1)
    fr = Frames(12, seed=2, spread=4.0)
    on = {"scan": dict(scan_size=2), "rf": dict(rf_size=2), "axis_and_grid": dict(axis_and_grid=True), "camera": dict(camera_size=1.0),
          "path": dict(path_width=4), "all": ALL}[layer]
    rgba, _, keys, _ = both(lib, R, eye, verts, tris, wire=wire, scan=scan, rf=rf, frames=fr, **on)
    assert (keys != NONE).sum() > 30
    both(lib, R, eye, verts, tris, color=True, wire=wire, scan=scan, rf=rf, frames=fr, **on)


@pytest.mark.parametrize("seed", range(4))
def test_random_scenes_everything_on(lib, seed):
    R, eye, verts, tris, scan, rf = scene(10 + seed, 200, 300)
    fr = Frames(30, seed=seed, spread=6.0, has=np.random.default_rng(seed).integers(0, 2, 30))
    for wire in (False, True):
        for color, zr in ((False, None), (True, None), (True, (-1.0, 3.0))):
            both(lib, R, eye, verts, tris, color=color, z_range=zr, wire=wire, scan=scan, rf=rf, frames=fr, path_cap=20, **ALL)


def test_segments_cross_near_and_far_and_behind(lib):
    # a camera 1.6 m above the grid looking along +x: the grid lines run behind the camera (near plane) and beyond z_far = 60
    eye = np.array([3.0, 2.0, 1.6])
    R = look_at(eye, eye + np.array([1.0, 0.2, -0.05]))
    fr = Frames(40, seed=3, center=eye, spread=40.0)   # trajectory segments across both planes and wholly behind
    _, _, keys, _ = both(lib, R, eye, zn=0.5, zf=60.0, axis_and_grid=True, camera_size=2.0, path_width=3, path_cap=64, frames=fr)
    assert (keys != NONE).sum() > 200
    # a segment wholly behind the camera draws nothing
    back = Frames(2, seed=4)
    back.t[:] = [eye + 5 * R[:, 2], eye + 9 * R[:, 2]]   # camera z = -5, -9
    _, _, keys, _ = both(lib, R, eye, path_width=4, frames=back)
    assert (keys == NONE).all()
    # the grid from a follow camera close to the ground, with a small z_near
    for zn in (0.1, 1e-3):
        both(lib, R, eye, zn=zn, zf=1500.0, axis_and_grid=True)


def test_wide_lines_and_large_points_at_borders(lib):
    R = np.eye(3)
    t = np.zeros(3)
    # points near the image corners and tile borders (camera looks down -z): sizes up to 64
    uv = np.array([[0.2, 0.3], [95.6, 79.4], [15.5, 15.5], [16.0, 31.99], [47.5, 39.5], [-3.0, 40.0], [99.0, 2.0]])
    z = np.array([5.0, 6.0, 7.0, 8.0, 9.0, 10.0, 11.0])
    pts = np.stack([(uv[:, 0] - K[2]) / K[0] * z, -(uv[:, 1] - K[3]) / K[1] * z, -z], axis=1).astype(np.float32)
    fr = Frames(6, seed=5, center=(0.0, 0.0, -20.0), spread=8.0)
    for size in (1, 2, 3, 17, 64):
        both(lib, R, t, scan=pts, scan_size=size, rf=pts[::-1].copy(), rf_size=max(size // 2, 1), frames=Frames(2, seed=1), w=W, h=H)
        both(lib, R, t, frames=fr, path_width=size, path_cap=6)
    # a line over many tiles at a large image
    both(lib, R, t, frames=fr, path_width=9, path_cap=6, w=300, h=200)


def test_equal_depth_ties(lib):
    R = np.eye(3)
    t = np.zeros(3)
    p = np.array([[0.5, 0.2, -10.0], [0.5, 0.2, -10.0], [-1.0, 0.4, -12.0]], np.float32)
    fr = Frames(2, seed=6)
    _, _, keys, _ = both(lib, R, t, scan=p, scan_size=4, rf=p, rf_size=4, frames=fr)
    # the scan layer wins over the reinforced one at equal depth, and its lower index over its higher
    drawn = keys[keys != NONE]
    layers = (drawn >> np.uint64(29)) & np.uint64(7)
    assert (layers == SCAN).all() and ((drawn & np.uint64(0x1FFFFFFF)) != 1).all()
    # a trajectory along the x axis: the axis (drawn before) wins where the depths are equal; the frustum over the trajectory
    eye = np.array([0.5, -3.0, 2.0])
    Rl = look_at(eye, np.array([0.5, 0.0, 0.0]))
    fr = Frames(3, seed=7)
    fr.t[:] = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
    fr.R[:] = np.eye(3)
    _, _, keys, _ = both(lib, Rl, eye, axis_and_grid=True, path_width=10, camera_size=1.0, frames=fr)
    ref = overlay_keys(K, W, H, 0.1, 1500.0, Rl, eye, path=list(fr.t), path_width=10)
    same = (ref != NONE) & ((ref >> np.uint64(32)) == (keys >> np.uint64(32)))
    assert same.sum() > 20 and (((keys[same] >> np.uint64(29)) & np.uint64(7)) != PATH).any()


def test_shared_wireframe_edges_any_slot_order(lib):
    # a height field: every inner edge shared by two triangles
    n = 9
    g = np.stack(np.meshgrid(np.arange(n) - 4.0, np.arange(n) - 4.0), axis=-1).reshape(-1, 2)
    verts = np.concatenate([g, np.sin(g[:, :1]) * 0.7 + 0.1 * g[:, 1:]], axis=1).astype(np.float32)
    tris = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, i * n + j + 1, (i + 1) * n + j, (i + 1) * n + j + 1
            tris += [sorted((a, b, d)), sorted((a, d, c))]
    tris = np.array(tris)
    eye = np.array([-7.0, -9.0, 8.0])
    R = look_at(eye, np.zeros(3))
    ref = None
    for seed in range(3):
        order = np.random.default_rng(seed).permutation(len(tris))
        for color in (False, True):
            rgba, depth, _, _ = both(lib, R, eye, verts, tris[order], color=color, wire=True)
            if not color:
                ref = rgba if ref is None else ref
                assert np.array_equal(rgba, ref)
    assert (ref[..., :3] != 0).any(axis=2).sum() > 300


@pytest.mark.parametrize("wire", [False, True])
def test_bin_overflow_same_image(lib, wire):
    R, eye, verts, tris, scan, rf = scene(4, 150, 250)
    fr = Frames(8, seed=8)
    a, da, _, oa = both(lib, R, eye, verts, tris, wire=wire, scan=scan, frames=fr, **ALL)
    b, db, _, ob = both(lib, R, eye, verts, tris, wire=wire, scan=scan, frames=fr, bin_cap=3, **ALL)
    assert oa == 0 and ob == 1
    assert np.array_equal(a, b) and np.array_equal(da.view(np.uint32), db.view(np.uint32))


def test_trajectory_ring_wraps(lib):
    R = look_at(np.array([0.0, -30.0, 25.0]), np.zeros(3))
    eye = np.array([0.0, -30.0, 25.0])
    fr = Frames(50, seed=9, spread=8.0)
    for cap, start in ((7, 1), (7, 20), (49, 3), (50, 1), (64, 1), (1, 1)):
        _, _, keys, _ = both(lib, R, eye, frames=fr, path_width=2, path_cap=cap, path_from=start)
        assert (keys != NONE).any() == (min(cap, 51 - start) > 1)


def test_frustum_against_scipy(lib):
    fx, fy, cx, cy = 704.504153913163, 703.6790228113778, 708.8501128392297, 562.7041625276061
    L = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
    for seed in range(5):
        rot = Rotation.random(random_state=seed)
        R = rot.as_matrix()
        t = np.random.default_rng(seed).normal(size=3) * 10
        cs = [1.0, 0.5, 2.25, 1.0, 3.0][seed]
        out = np.zeros((11, 3))
        lib.emu_ov_frustum(_p(np.ascontiguousarray(R.reshape(9))), _p(t), cs, _p(out))
        assert np.array_equal(out, frustum(R, t, cs))
        # the corners are the image corners of K at 1.5 m in the camera frame R L, scaled by cs, at t
        cam = (Rotation.from_matrix(R) * Rotation.from_matrix(L)).inv().apply(out - t) / cs
        corners = np.array([[0, 0], [1440, 0], [1440, 1080], [0, 1080], [0, 0]], np.float64)
        expect = np.stack([(corners[:, 0] - cx) / fx * 1.5, (corners[:, 1] - cy) / fy * 1.5, np.full(5, 1.5)], axis=1)
        assert np.abs(cam[:5] - expect).max() < 1e-9
        assert np.abs(out[[5, 7, 9]] - t).max() < 1e-12
        assert np.array_equal(out[[6, 8, 10]], out[[1, 3, 2]])


def test_key_order():
    # depth bits first, then the layer in draw order, then the index
    assert key_of(1.0, PATH, 0) < key_of(np.nextafter(np.float32(1.0), np.float32(2.0)), SCAN, 0)
    assert key_of(1.0, SCAN, 5) < key_of(1.0, CAMERA, 0) < key_of(1.0, PATH, 0)
    assert key_of(1.0, SCAN, 5) > key_of(1.0, SCAN, 4)
