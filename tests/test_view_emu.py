"""CPU tier: the shaded view's device bodies (immesh_b200/csrc/reinforce.cuh) run by the host emulation (tests/view/emu_view.cpp) in the
tiled rasteriser's orchestration, against the numpy restatement of the image rule (tests/view_reference.py), byte for byte and depth
bit for bit.  The rule, as include/immesh_b200.h states it: the depth image's sampling rule at the drawn positions; the nearest
sample wins, the lower (a, b, c) triple on equal depth bits; the winner shaded in float64 with its face normal, perspective-correct
weights e_i (1 / z_i), light at the camera position, (0.2 + 0.5 |n . l|) times the interpolated vertex colour, rounded to bytes;
undrawn pixels opaque black; the height colour t = (z - lo) / (hi - lo) in float32, s = clamp(1 - t), the stops blue, cyan, green,
yellow, red at 4 s, bytes truncated.  Also the queued view's fixed and follow cameras against scipy."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from view_reference import frame_pose, heat, positions, render


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_view())
    vp = C.c_void_p
    L.emu_view_render.argtypes = [vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, C.c_longlong, vp, vp, vp, vp]
    L.emu_view_heat.argtypes = [vp, C.c_int, C.c_float, C.c_float, vp]
    L.emu_view_pose.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def emu_render(lib, K, w, h, zn, zf, R, t, verts, tris, smooth=None, flags=None, mode=0, color=False, z_range=None, bin_cap=1 << 30):
    cam = np.concatenate([K, [zn, zf], np.asarray(R, np.float64).reshape(9), t]).astype(np.float64)
    v = np.ascontiguousarray(verts, np.float32)
    sm = None if smooth is None else np.ascontiguousarray(smooth, np.float64)
    fl = None if flags is None else np.ascontiguousarray(flags, np.uint8)
    tr = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    zr = np.array([np.nan, np.nan] if z_range is None else z_range, np.float64)
    rgba = np.zeros((h, w, 4), np.uint8)
    depth = np.zeros((h, w), np.float32)
    bins, over = C.c_longlong(0), C.c_int(0)
    lib.emu_view_render(_p(cam), w, h, _p(v), _p(sm), _p(fl), len(v), _p(tr), len(tr), mode, 1 if color else 0, _p(zr), bin_cap, _p(rgba), _p(depth),
                        C.byref(bins), C.byref(over))
    return rgba, depth, bins.value, over.value


def check(lib, K, w, h, zn, zf, R, t, verts, tris, smooth=None, flags=None, mode=0, color=False, z_range=None, bin_cap=1 << 30):
    rgba, depth, bins, over = emu_render(lib, K, w, h, zn, zf, R, t, verts, tris, smooth, flags, mode, color, z_range, bin_cap)
    rn, dn = render(K, w, h, zn, zf, R, t, positions(verts, smooth, flags, mode), tris, color, z_range)
    assert np.array_equal(depth.view(np.uint32), dn.view(np.uint32)), "depth differs from the restatement"
    bad = np.argwhere((rgba != rn).any(axis=2))
    assert len(bad) == 0, (len(bad), bad[:5], rgba[tuple(bad[0])], rn[tuple(bad[0])])
    return rgba, depth, bins, over


R0, T0 = np.eye(3), np.zeros(3)   # camera at the origin looking down world -z


def random_scene(seed, n_verts=300, n_tris=400):
    rng = np.random.default_rng(seed)
    R = Rotation.random(random_state=seed).as_matrix()
    t = rng.normal(size=3)
    pc = np.stack([rng.uniform(-6, 6, n_verts), rng.uniform(-4, 4, n_verts), rng.uniform(0.05, 30, n_verts)], axis=1)
    verts = ((pc @ np.diag([1.0, -1.0, -1.0]).T) @ R.T + t).astype(np.float32)
    tris = np.sort(np.array([rng.choice(n_verts, 3, replace=False) for _ in range(n_tris)]), axis=1)
    return R, t, verts, tris


# ---- the height colour ramp
def test_heat_stops_midpoints_clamp_and_flat(lib):
    lo, hi = np.float32(-2.0), np.float32(6.0)
    z = np.array([6.0, 4.0, 2.0, 0.0, -2.0, 5.0, 3.0, 1.0, -1.0, 100.0, -100.0, 0.3, 5.9], np.float32)
    out = np.zeros((len(z), 3), np.uint8)
    lib.emu_view_heat(_p(z), len(z), lo, hi, _p(out))
    assert np.array_equal(out, heat(z, lo, hi))
    # top of the range is blue, bottom red, the stops between cyan, green, yellow
    assert out[:5].tolist() == [[0, 0, 255], [0, 255, 255], [0, 255, 0], [255, 255, 0], [255, 0, 0]]
    # midpoints: 0.5 * 255 = 127.5 truncated to 127
    assert out[5].tolist() == [0, 127, 255] and out[6].tolist() == [0, 255, 127] and out[7].tolist() == [127, 255, 0] and out[8].tolist() == [255, 127, 0]
    # beyond the range: clamped to the ends
    assert out[9].tolist() == [0, 0, 255] and out[10].tolist() == [255, 0, 0]
    # a flat range: t = 0, the bottom's red
    flat = np.zeros((3, 3), np.uint8)
    lib.emu_view_heat(_p(z[:3]), 3, np.float32(1.5), np.float32(1.5), _p(flat))
    assert (flat == [255, 0, 0]).all() and np.array_equal(flat, heat(z[:3], 1.5, 1.5))
    # a dense sweep: truncation agrees everywhere
    zs = np.linspace(-3.0, 7.0, 20001, dtype=np.float32)
    o = np.zeros((len(zs), 3), np.uint8)
    lib.emu_view_heat(_p(zs), len(zs), lo, hi, _p(o))
    assert np.array_equal(o, heat(zs, lo, hi))


# ---- images
@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("color,z_range", [(False, None), (True, None), (True, (-5.0, 3.0))])
def test_random_scenes(lib, seed, color, z_range):
    """random triangles in front of a rotated, moved camera, some beyond the image, z_far and z_near; many overlapping"""
    R, t, verts, tris = random_scene(seed)
    K, w, h = (60.0, 55.0, 37.5, 24.0), 75, 50
    rgba, depth, bins, over = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, color=color, z_range=z_range)
    drawn = (rgba[..., :3] != 0).any(axis=2)
    assert drawn.sum() > 500 and bins > 400 and not over
    assert (rgba[..., 3] == 255).all()
    # slot order does not matter
    perm = np.random.default_rng(seed + 10).permutation(len(tris))
    rgba2, depth2, _, _ = emu_render(lib, K, w, h, 0.2, 25.0, R, t, verts, tris[perm], color=color, z_range=z_range)
    assert np.array_equal(rgba, rgba2) and np.array_equal(depth.view(np.uint32), depth2.view(np.uint32))


def test_bin_overflow_walks_every_slot(lib):
    R, t, verts, tris = random_scene(5)
    K, w, h = (60.0, 55.0, 37.5, 24.0), 75, 50
    a = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, color=True)
    b = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, color=True, bin_cap=100)
    assert not a[3] and b[3] and a[2] > 100
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_large_triangle_covers_many_tiles(lib):
    K, w, h = (40.0, 40.0, 30.0, 20.0), 61, 45
    verts = np.array([[-50.0, -50.0, -2.0], [50.0, -50.0, -2.5], [0.0, 60.0, -3.0]], np.float32)
    rgba, depth, bins, _ = check(lib, K, w, h, 0.1, 100.0, R0, T0, verts, [[0, 1, 2]], color=True)
    assert (depth > 0).all() and bins == 4 * 3 and (rgba[..., :3] != 0).any(axis=2).all()


def test_shared_edges_and_coplanar_duplicates(lib):
    """vertices on integer pixel coordinates at one depth: shared edges pass through pixel centres; coplanar duplicates with other
    vertex ids and other colours cover the same pixels at equal depth bits, so only the triple decides"""
    K, w, h, z = (10.0, 10.0, 0.0, 0.0), 40, 40, 10.0

    def at(u, v, zz=z):
        return [u * zz / 10.0, -(v * zz / 10.0), -zz]
    base = [at(2, 2), at(30, 2), at(2, 30), at(30, 30), at(10, 10), at(20, 20)]
    verts = np.array(base + base, np.float32)           # ids 6..11 repeat 0..5
    verts[6:, 2] = verts[:6, 2]
    tris = np.array([[6, 7, 8], [0, 1, 2], [7, 8, 9], [1, 2, 3], [4, 5, 7], [1, 4, 5]])
    for color, zr in ((False, None), (True, (-10.5, -9.5))):
        rgba, depth, _, _ = check(lib, K, w, h, 0.1, 100.0, R0, T0, verts, tris, color=color, z_range=zr)
        rgba2, _, _, _ = emu_render(lib, K, w, h, 0.1, 100.0, R0, T0, verts, tris[::-1], color=color, z_range=zr)
        assert np.array_equal(rgba, rgba2)
    # different coplanar triangles overlapping at one camera depth, seen by a tilted camera so that world z (and with it the height
    # colour, interpolated differently by each triangle) varies across them: where the depth bits are equal the lower triple is drawn,
    # so the image is the same in any slot order and changes when the ids are swapped
    Rt = Rotation.from_rotvec([0.5, 0.2, 0.0]).as_matrix()
    cam = [at(2, 2), at(36, 3), at(3, 37), at(5, 4), at(38, 8), at(8, 38)]
    verts = ((np.array(cam) @ np.diag([1.0, -1.0, -1.0]).T) @ np.diag([1.0, -1.0, -1.0]).T @ Rt.T).astype(np.float32)
    tris = np.array([[0, 1, 2], [3, 4, 5]])
    rgba, depth, _, _ = check(lib, K, w, h, 0.1, 100.0, Rt, T0, verts, tris, color=True)
    rgba2, _, _, _ = emu_render(lib, K, w, h, 0.1, 100.0, Rt, T0, verts, tris[::-1], color=True)
    assert np.array_equal(rgba, rgba2)
    swapped = verts[[3, 4, 5, 0, 1, 2]]
    rgba3, depth3, _, _ = check(lib, K, w, h, 0.1, 100.0, Rt, T0, swapped, tris, color=True)
    assert np.array_equal(depth.view(np.uint32), depth3.view(np.uint32)) and not np.array_equal(rgba, rgba3)


def test_vertex_behind_z_near_is_skipped_and_undrawn_is_black(lib):
    K, w, h = (20.0, 20.0, 16.0, 16.0), 33, 33
    verts = np.array([[-1.0, -1.0, -2.0], [1.0, -1.0, -2.0], [0.0, 1.0, -0.05], [-1.0, -1.0, -3.0], [1.0, -1.0, -3.0], [0.0, 1.0, -3.0]], np.float32)
    rgba, depth, _, _ = check(lib, K, w, h, 0.1, 100.0, R0, T0, verts, [[0, 1, 2], [3, 4, 5]])
    assert depth.max() == np.float32(3.0)
    assert (rgba[depth == -1] == [0, 0, 0, 255]).all()
    # the facet faces the camera at the image centre: d = 1, so white * 0.7 -> 179
    assert rgba[16, 16].tolist() == [179, 179, 179, 255]
    # the empty scene: all black
    rgba, depth, _, _ = check(lib, K, w, h, 0.1, 100.0, R0, T0, verts, np.zeros((0, 3), int))
    assert (rgba == [0, 0, 0, 255]).all() and (depth == -1).all()


@pytest.mark.parametrize("color", [False, True])
def test_mixed_smoothed_and_raw_positions(lib, color):
    """positions 1: the smoothed position where the flag is set, the raw one elsewhere (flags chosen here)"""
    R, t, verts, tris = random_scene(7, n_verts=200, n_tris=250)
    rng = np.random.default_rng(7)
    smooth = verts.astype(np.float64) + rng.normal(scale=0.05, size=verts.shape)
    flags = (rng.random(len(verts)) < 0.5).astype(np.uint8)
    K, w, h = (60.0, 55.0, 37.5, 24.0), 75, 50
    a = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, smooth, flags, mode=1, color=color)
    b = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, smooth, flags, mode=0, color=color)
    assert not np.array_equal(a[0], b[0])
    # positions 0 ignores the smoothed positions; all flags clear is the raw image
    c = check(lib, K, w, h, 0.2, 25.0, R, t, verts, tris, smooth, np.zeros_like(flags), mode=1, color=color)
    assert np.array_equal(c[0], b[0]) and np.array_equal(c[1].view(np.uint32), b[1].view(np.uint32))


# ---- the queued view's cameras
def emu_pose(lib, poses, n_frames, frame, win, mode, R_in, t_in):
    arr = np.zeros((n_frames, 12))
    has = np.zeros(n_frames, np.int32)
    for f, (R, t) in poses.items():
        arr[f - 1, :9], arr[f - 1, 9:], has[f - 1] = R.reshape(9), t, 1
    Ri = np.ascontiguousarray(R_in, np.float64).reshape(9)
    ti = np.ascontiguousarray(t_in, np.float64)
    R, t = np.zeros(9), np.zeros(3)
    lib.emu_view_pose(_p(arr), _p(has), n_frames, frame, win, mode, _p(Ri), _p(ti), _p(R), _p(t))
    return R.reshape(3, 3), t


@pytest.mark.parametrize("win", [1, 3])
def test_follow_and_fixed_poses_against_scipy(lib, win):
    rng = np.random.default_rng(win)
    rots = Rotation.random(12, random_state=win)
    ts = np.cumsum(rng.normal(size=(12, 3)), axis=0) * 3.0
    poses = {f + 1: (rots[f].as_matrix(), ts[f]) for f in range(12) if f != 5}   # frame 6 recorded no pose
    R_in, t_in = Rotation.random(random_state=99).as_matrix(), np.array([-4.0, 0.5, 2.0])
    for frame in range(1, 13):
        for mode in (0, 1, 2):
            R, t = emu_pose(lib, poses, 12, frame, win, mode, R_in, t_in)
            Rn, tn = frame_pose(poses, frame, win, mode, R_in, t_in)
            assert np.abs(R - Rn).max() < 1e-12 and np.abs(t - tn).max() < 1e-12, (frame, mode)
            if mode:
                assert np.array_equal(R, R_in)
            if mode == 1:
                assert np.array_equal(t, t_in)
    # a window without a pose: the follow camera sits at the offset itself
    R, t = emu_pose(lib, {}, 4, 3, win, 2, R_in, t_in)
    assert np.array_equal(R, R_in) and np.array_equal(t, t_in)
