"""GPU tier: depth-camera frames (immesh_mesh_push_depth, _async, immesh_mesh_depth_points).  Depth images are ray-cast from the synth
scene with a pinhole camera along synth.trajectory_pose (tests/depth_reference.py), with misses as holes and the edge values injected.
The device's points equal the numpy restatement bit for bit, and every depth frame leaves the mesh exactly as immesh_mesh_push_frame of
those points at cam_t leaves a twin handle: snapshot, counts, change feed and frame feed (KIND aside), with host or device images,
blocking or queued, with growth, and for an image without a valid pixel.  Also the error contract."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from immesh_b200 import api
from mesh_common import SMALL
import depth_reference as dr

pytestmark = pytest.mark.gpu

E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5
W, H = 160, 120
APPEND = 4000   # 160 x 120 frames give step 2 .. 4
H_KEYS = {k: i for i, k in enumerate(api.MESH_FEED_HDR_KEYS)}


def mesh(append=APPEND, **kw):
    cfg = dict(SMALL, number_of_pts_append_to_map=append)
    cfg.update(kw)
    return api.Mesh(api.MeshConfig(**cfg))


def frames(n, cam, fmt="f32", kind="planar", seed=0, w=W, h=H):
    rng = np.random.default_rng(seed)
    for k in range(n):
        R, t = dr.camera_pose(k)
        img = dr.inject_edges(dr.render(cam, w, h, R, t, kind=kind, fmt=fmt), cam, rng)
        yield img, R, t


def same_state(a, b):
    assert a.counts() == b.counts()
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert x.shape == y.shape and x.tobytes() == y.tobytes()


def expect_rc(fn, code):
    with pytest.raises(RuntimeError, match=f"code {code}:"):
        fn()


@pytest.mark.parametrize("fmt,kind,stride,pad", [("f32", "range", 1, 0), ("u16", "planar", 2, 16), ("f32", "planar", 3, 8)])
def test_points_bit_exact(fmt, kind, stride, pad):
    w, h = 640, 480
    cam = dr.camera(w, h, kind=kind, stride=stride, z_min=0.5, z_max=40.0, depth_scale=0.001)
    m = mesh(max_frame_points=w * h)
    for img, R, t in frames(2, cam, fmt, kind, seed=stride, w=w, h=h):
        ref, _ = dr.unproject(img, cam, R, t)
        m.push_depth(img, cam, R, t)
        got = m.depth_points()
        assert got.shape == ref.shape and got.tobytes() == ref.tobytes()
        # the same image on the device with padded rows
        dev = torch.zeros((h, w + pad // img.itemsize), dtype=torch.float32 if fmt == "f32" else torch.int16, device="cuda")
        dev[:, :w] = torch.from_numpy(img.view(np.float32 if fmt == "f32" else np.int16)).cuda()
        m.push_depth(dev.data_ptr(), cam, R, t, on_device=True, shape=(h, w), fmt=fmt, pitch_bytes=dev.stride(0) * dev.element_size())
        got = m.depth_points()
        assert got.tobytes() == ref.tobytes()


def test_sequence_equals_push_frame():
    """>= 30 frames: after every frame the same snapshot and counts as push_frame of the numpy points at cam_t (every third frame at
    stride 2, so that append_point_step changes along the sequence)"""
    cam = dr.camera(W, H, kind="range", z_min=0.5, z_max=40.0)
    a, b = mesh(), mesh()
    steps = set()
    for k, (img, R, t) in enumerate(frames(32, cam, kind="range")):
        if k % 3 == 2:
            cam = dataclasses.replace(cam, stride=2)
        else:
            cam = dataclasses.replace(cam, stride=1)
        pts, _ = dr.unproject(img, cam, R, t)
        a.push_depth(img, cam, R, t)
        b.push_frame(pts, t)
        steps.add(dr.append_dims(pts.shape[0], APPEND)[0])
        same_state(a, b)
        assert a.work_stats() == b.work_stats()
    assert len(steps) > 1 and a.counts()["n_triangles"] > 1000


def test_host_device_sync_async():
    """host or device images, blocking or queued: the same mesh and the same points"""
    cam = dr.camera(W, H, stride=1, z_min=0.5, z_max=40.0, depth_scale=0.002)
    ms = [mesh() for _ in range(4)]
    keep = []
    for img, R, t in frames(12, cam, fmt="u16", seed=4):
        dev = torch.from_numpy(img.view(np.int16)).cuda()
        keep.append(dev)   # a queued frame reads the device image when it runs
        ms[0].push_depth(img, cam, R, t)
        ms[1].push_depth(dev.data_ptr(), cam, R, t, on_device=True, shape=img.shape, fmt="u16")
        ms[2].push_depth_async(img, cam, R, t)
        ms[3].push_depth_async(dev.data_ptr(), cam, R, t, on_device=True, shape=img.shape, fmt="u16")
    for m in ms[2:]:
        m.wait()
    ref = ms[0].depth_points()
    for m in ms[1:]:
        same_state(ms[0], m)
        assert m.depth_points().tobytes() == ref.tobytes()


def test_feeds_equal_push_frame_twin():
    """change feed and frame feed: the rows of the push_frame twin; only KIND (and the time stamps) differ, N_POINTS / STEP are the
    valid count and the rule"""
    cam = dr.camera(W, H, z_min=0.5, z_max=40.0)
    a, b = mesh(), mesh()
    for m in (a, b):
        m.changes_enable()
        m.feed_enable(max_frames=64, max_rows=0)
    counts = []
    for i, (img, R, t) in enumerate(frames(10, cam, seed=7)):
        pts, _ = dr.unproject(img, cam, R, t)
        counts.append(pts.shape[0])
        if i % 2:
            a.push_depth_async(img, cam, R, t)
        else:
            a.push_depth(img, cam, R, t)
        b.push_frame(pts, t)
    a.wait()
    ca, cb = a.changes(0), b.changes(0)
    for k in ("frames", "rows", "vertices"):
        assert ca[k].tobytes() == cb[k].tobytes(), k
    fa, fb = a.feed(0, wait=True), b.feed(0, wait=True)
    ha, hb = fa["frames"].copy(), fb["frames"].copy()
    assert len(ha) == 10 and np.all(ha[:, H_KEYS["kind"]] == api.MESH_FEED_KINDS.index("depth"))
    assert np.all(hb[:, H_KEYS["kind"]] == api.MESH_FEED_KINDS.index("push"))
    np.testing.assert_array_equal(ha[:, H_KEYS["n_points"]], counts)
    np.testing.assert_array_equal(ha[:, H_KEYS["step"]], [dr.append_dims(n, APPEND)[0] for n in counts])
    for h in (ha, hb):
        h[:, [H_KEYS["kind"], H_KEYS["t_begin_ns"], H_KEYS["t_end_ns"]]] = 0
    np.testing.assert_array_equal(ha, hb)
    assert fa["poses"].tobytes() == fb["poses"].tobytes()


def test_all_invalid_image():
    cam = dr.camera(W, H, z_min=0.5, z_max=40.0)
    a, b = mesh(), mesh()
    for m in (a, b):
        m.feed_enable(max_frames=8, max_rows=0)
    img, R, t = next(frames(1, cam))
    a.push_depth(img, cam, R, t)
    b.push_frame(dr.unproject(img, cam, R, t)[0], t)
    a.push_depth(np.full((H, W), np.nan, np.float32), cam, R, t)
    b.push_frame(np.zeros((0, 3), np.float32), t)
    same_state(a, b)
    assert a.depth_points().shape == (0, 3)
    ha, hb = a.feed(0, wait=True)["frames"], b.feed(0, wait=True)["frames"]
    assert ha[1, H_KEYS["n_points"]] == 0 and ha[1, H_KEYS["step"]] == 1
    cols = [H_KEYS[k] for k in ("n_points", "step", "n_vertices", "n_triangles", "new_vertices", "n_activated", "err")]
    np.testing.assert_array_equal(ha[:, cols], hb[:, cols])


def test_growth_equals_presized():
    cam = dr.camera(W, H, z_min=0.5, z_max=40.0)
    grown = mesh(max_vertices=4096, max_triangles=8192, max_voxels=1024)
    grown.set_growth(1 << 31)
    sized = mesh()
    for img, R, t in frames(16, cam, seed=2):
        grown.push_depth_async(img, cam, R, t)
        sized.push_depth(img, cam, R, t)
    grown.wait()
    assert grown.capacity()["growths"] > 0
    same_state(grown, sized)


def test_errors():
    cam = dr.camera(W, H, z_min=0.5, z_max=40.0)
    m = mesh(max_frame_points=W * H - 1)
    img, R, t = next(frames(1, cam))
    expect_rc(lambda: m.depth_points(), E_INVALID)   # no depth frame yet
    expect_rc(lambda: m.push_depth(img, cam, R, t), E_CAPACITY)   # more sampled pixels than max_frame_points
    ok = dataclasses.replace(cam, stride=2)
    m.push_depth(img, ok, R, t)
    bad_cams = [dataclasses.replace(ok, fx=0.0), dataclasses.replace(ok, fy=np.inf), dataclasses.replace(ok, fx=np.nan), dataclasses.replace(ok, cx=np.nan),
                dataclasses.replace(ok, stride=0), dataclasses.replace(ok, z_min=-0.1), dataclasses.replace(ok, z_min=5.0, z_max=5.0),
                dataclasses.replace(ok, z_max=np.inf), dataclasses.replace(ok, z_min=np.nan)]
    for c in bad_cams:
        expect_rc(lambda: m.push_depth(img, c, R, t), E_INVALID)
        expect_rc(lambda: m.push_depth_async(img, c, R, t), E_INVALID)
    u16 = np.zeros((H, W), np.uint16)
    for scale in (0.0, -1.0, np.inf):
        expect_rc(lambda: m.push_depth(u16, dataclasses.replace(ok, depth_scale=scale), R, t), E_INVALID)
    expect_rc(lambda: m.push_depth(img, ok, R * np.nan, t), E_INVALID)
    dev = torch.zeros((H, W + 1), dtype=torch.float32, device="cuda")
    args = dict(on_device=True, shape=(H, W))
    expect_rc(lambda: m.push_depth(dev.data_ptr(), ok, R, t, pitch_bytes=W * 4 - 4, **args), E_INVALID)   # pitch below a row
    expect_rc(lambda: m.push_depth(dev.data_ptr(), ok, R, t, pitch_bytes=W * 4 + 2, **args), E_INVALID)   # pitch not a pixel multiple
    expect_rc(lambda: m.push_depth(dev.data_ptr() + 2, ok, R, t, **args), E_INVALID)                     # misaligned image
    expect_rc(lambda: m.push_depth(dev.data_ptr(), ok, R, t, on_device=True, shape=(0, W)), E_INVALID)
    expect_rc(lambda: m.push_depth(dev.data_ptr(), ok, R, t, on_device=True, shape=(H, -3)), E_INVALID)
    f, ptr, _keep = api.Mesh._depth_args(ok, R, t, img, None, "f32", 0, False)
    lib = m.lib
    for field, val in (("format", 2), ("kind", 5)):
        g = api._DepthFrame.from_buffer_copy(f)
        setattr(g, field, val)
        assert lib.immesh_mesh_push_depth(m._h, g, ptr, 0) == E_INVALID
    assert lib.immesh_mesh_push_depth(m._h, f, None, 0) == E_INVALID
    # far from cam_t: the codes of push_frame
    far = np.full((H, W), 30.0, np.float32)
    tf = np.array([6.0e5, 0.0, 0.0])
    b, c = mesh(), mesh()
    expect_rc(lambda: b.push_depth(far, ok, R, tf), E_RANGE)
    expect_rc(lambda: c.push_frame(dr.unproject(far, ok, R, tf)[0], tf), E_RANGE)
    # the count query and the capacity of the read
    n = m.depth_points().shape[0]
    out = np.zeros((n, 3), np.float32)
    got = C.c_int(0)
    assert m.lib.immesh_mesh_depth_points(m._h, out.ctypes.data_as(C.POINTER(C.c_float)), n - 1, C.byref(got)) == E_CAPACITY and got.value == n
