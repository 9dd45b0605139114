"""GPU tier: the mesh frame feed (immesh_mesh_feed_enable / immesh_mesh_feed / immesh_mesh_feed_images).  A handle queues frames with
the feed on and never waits between them; a twin runs the same frames blocking and reads immesh_mesh_counts,
immesh_mesh_reinforced_cloud and immesh_mesh_view_image after each one.  Every header field but the two stamps, every pose, point,
pixel, rgba byte and depth float of the records equals what the twin read, bit for bit: on the localization chain, for every entry
point kind (batched frames included), with images at a small size and at 640 x 480.  Also: the stamps, non-blocking reads while
frames are queued, off means off, the lifetime rules (view and reinforcement re-enabled mid-stream, pool growth, a second enable,
destroy with frames in flight), point losses, and the error contract.  The sharded-handle rejection needs a multi-rank communicator
and is not tested here."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_common import SMALL, world_scans

pytestmark = pytest.mark.gpu

H = {k: i for i, k in enumerate(api.MESH_FEED_HDR_KEYS)}
STAMPS = (H["t_begin_ns"], H["t_end_ns"])
E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5
SMALL_VIEW = dict(width=160, height=120)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8)


def same(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


class Expect:
    """the records a frame feed must hold, built from a blocking twin's reads right after each frame"""

    def __init__(self):
        self.hdr, self.poses, self.points, self.pixels, self.images = {}, {}, {}, {}, {}

    def add(self, f, mesh, kind, n, pose=None, pose_t=None, rf=False, view=False, batched=False, img=False):
        c = mesh.counts()
        step = max(1, n // mesh.cfg.number_of_pts_append_to_map)
        h = np.zeros(api.MESH_FEED_HDR, np.int64)
        h[H["frame"]], h[H["kind"]], h[H["n_points"]], h[H["step"]] = f, api.MESH_FEED_KINDS.index(kind), n, step
        h[H["n_vertices"]:H["n_vertices"] + 8] = list(c.values())
        h[H["has_rotation"]] = 1 if pose is not None else 0
        p = np.zeros((3, 12))
        if pose is not None:
            p[0, :9], p[0, 9:] = pose[0].reshape(9), pose[1]
        else:
            p[0, 9:] = pose_t
        self.points[f] = np.zeros((0, 3), np.float32)
        self.pixels[f] = np.zeros(0, np.int32)
        if rf and not batched:
            _, pts, pix, R, t = mesh.reinforced_cloud()
            self.points[f], self.pixels[f] = pts, pix
            p[1, :9], p[1, 9:] = R.reshape(9), t
            h[H["rf"]] = 1
        if view and img and not batched:
            rgba, depth, R, t, vf = mesh.view_image()
            assert vf == f
            self.images[f] = (rgba, depth)
            p[2, :9], p[2, 9:] = R.reshape(9), t
        self.hdr[f], self.poses[f] = h, p

    def check(self, out, frames, points=True, max_rows=None):
        hdr, poses = out["frames"], out["poses"]
        assert hdr[:, H["frame"]].tolist() == list(frames)
        r0 = hdr[0, H["row_begin"]] if len(hdr) else 0
        for i, f in enumerate(frames):
            h, e = hdr[i].copy(), self.hdr[f].copy()
            lost = max_rows is not None and len(self.points[f]) > max_rows
            assert h[H["rows_lost"]] == int(lost), (f, h)
            n = 0 if lost else len(self.points[f])
            assert h[H["row_end"]] - h[H["row_begin"]] == n, (f, h, n)
            assert (h[H["img_end"]] - h[H["img_begin"]]) == (1 if f in self.images else 0), (f, h)
            for k in STAMPS + (H["row_begin"], H["row_end"], H["rows_lost"], H["img_begin"], H["img_end"]):
                h[k] = e[k] = 0
            assert np.array_equal(h, e), (f, dict(zip(api.MESH_FEED_HDR_KEYS, hdr[i])), dict(zip(api.MESH_FEED_HDR_KEYS, self.hdr[f])))
            assert same(poses[i], self.poses[f]), (f, poses[i], self.poses[f])
            if points and n:
                a, b = hdr[i, H["row_begin"]] - r0, hdr[i, H["row_end"]] - r0
                assert same(out["points"][a:b], self.points[f]) and np.array_equal(out["pixels"][a:b], self.pixels[f]), f

    def check_images(self, out, frames):
        assert out["frames"][:, H["frame"]].tolist() == list(frames)
        want = [f for f in frames if f in self.images]
        assert len(out["rgba"]) == len(want)
        for k, f in enumerate(want):
            assert np.array_equal(out["rgba"][k], self.images[f][0]), f
            if out["depth"] is not None:
                assert same(out["depth"][k], self.images[f][1]), f


def check_stamps(hdr):
    tb, te = hdr[:, STAMPS[0]], hdr[:, STAMPS[1]]
    assert (tb > 0).all() and (te >= tb).all(), hdr[:, STAMPS]
    assert (np.diff(tb) >= 0).all() and (np.diff(te) >= 0).all(), hdr[:, STAMPS]


def lio_setup(lib, n_scans, seed, mesh_cfg=None):
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(mesh_cfg or api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    return lio, mesh, scans


def lio_chain(lib, n_scans=7, seed=3, rf=True, view=None, feed=None, twin=None, actions=None, reads=None, mesh_cfg=None, growth=0):
    """The localization chain feeding the queued mesher.  feed: feed_enable arguments (the handle never waits between frames);
    twin: an Expect filled after every frame (the handle waits for each one).  actions: {k: fn(mesh, twin)} run before scan k on
    both; reads(k, mesh): called after each queued frame of the feed handle."""
    lio, mesh, scans = lio_setup(lib, n_scans, seed, mesh_cfg)
    if growth:
        mesh.set_growth(growth)
    state = dict(rf=rf, view=view is not None, img=feed is not None and feed.get("max_images", 0) > 0)
    if rf:
        mesh.reinforce_enable()
    if view is not None:
        mesh.view_enable(**view)
    if feed is not None:
        mesh.feed_enable(**feed)
    for k in range(1, n_scans):
        if actions and k in actions:
            actions[k](mesh, state)
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if twin is not None:
            mesh.wait()
            s = lio.get_state()
            twin.add(k, mesh, "from_lio_async", len(scans[k]["body_full"]), pose=(s[0:9].reshape(3, 3), s[9:12]), rf=state["rf"], view=state["view"],
                     img=state.get("twin_img", state["view"]))
        elif reads:
            reads(k, mesh)
    return lio, mesh


@pytest.mark.parametrize("size", [(160, 120), (640, 480)])
def test_twin_parity_on_the_localization_chain(cuda_lib, size):
    view = dict(width=size[0], height=size[1], color_by_height=True)
    tw = Expect()
    lio_chain(cuda_lib, rf=True, view=view, twin=tw)
    seen = []

    def reads(k, mesh):   # wait = 0 while frames are queued: a growing prefix
        out = mesh.feed(0, wait=False)
        assert out["newest_finished"] <= out["newest_queued"] == k
        assert out["frames"][:, H["frame"]].tolist() == list(range(1, out["newest_finished"] + 1))
        seen.append(out["newest_finished"])
    _, mesh = lio_chain(cuda_lib, rf=True, view=view, feed=dict(max_frames=64, max_rows=1 << 22, max_images=8, depth=True), reads=reads)
    assert seen == sorted(seen)
    st = api.graph_stats(None, mesh)
    assert st["mesh_captures"] == 1, st
    out = mesh.feed(0, wait=True)
    assert out["newest_finished"] == out["newest_queued"] == 6
    tw.check(out, range(1, 7))
    check_stamps(out["frames"])
    assert sum(len(p) for p in tw.points.values()) > 1000
    imgs = mesh.feed_images(0, wait=True)
    tw.check_images(imgs, range(1, 7))
    assert max((d > 0).sum() for d in imgs["depth"]) > 100


def test_entry_point_kinds(cuda_lib):
    """push_frame, push_frame_dev (by reconstruct_from_pointcloud), push_frame_batched, reconstruct_from_pointcloud_batched, and
    from_lio / from_lio_async, on one handle"""
    scans = world_scans("avia", 6, 11)
    lio, _, lscans = lio_setup(cuda_lib, 3, 3)
    vg = api.VoxelGrid(1 << 18, lib=cuda_lib)
    tw = Expect()
    mesh_a = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh_b = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    for m in (mesh_a, mesh_b):
        m.reinforce_enable(width=320, height=240)
        m.view_enable(**SMALL_VIEW)
    mesh_a.feed_enable(max_frames=32, max_rows=1 << 20, max_images=16)
    lio_b = api.Lio(api.AVIA, lib=cuda_lib)
    lio_b.set_state(lio.get_state())
    calls = [
        ("push", lambda m, l: m.push_frame(scans[0][0], scans[0][1], 0), len(scans[0][0]), scans[0][1]),
        ("batched", lambda m, l: m.push_frame_batched(scans[1][0], scans[1][1], batch_points=4096, batch_voxels=256), len(scans[1][0]), scans[1][1]),
        ("push", lambda m, l: m.push_frame(scans[2][0], scans[2][1], 2), len(scans[2][0]), scans[2][1]),
        ("reconstruct", lambda m, l: m.reconstruct_from_pointcloud(vg, scans[3][0], 0.1), None, np.zeros(3)),
        ("reconstruct_batched", lambda m, l: m.reconstruct_from_pointcloud_batched(vg, scans[4][0], 0.1, batch_points=4096), None, np.zeros(3)),
        ("from_lio", lambda m, l: m.push_frame_from_lio(l, lscans[1]["body_full"]), len(lscans[1]["body_full"]), None),
    ]
    for f, (kind, call, n, pose_t) in enumerate(calls, start=1):
        call(mesh_a, lio)
        ret = call(mesh_b, lio_b)
        if n is None:
            n = ret
        pose = None
        if pose_t is None:
            s = lio_b.get_state()
            pose = (s[0:9].reshape(3, 3), s[9:12])
        batched = "batched" in kind
        tw.add(f, mesh_b, kind, n, pose=pose, pose_t=pose_t, rf=True, view=True, img=not batched, batched=batched)
    out = mesh_a.feed(0, wait=True)
    tw.check(out, range(1, 7))
    check_stamps(out["frames"])
    tw.check_images(mesh_a.feed_images(0, wait=True), range(1, 7))


def per_frame_launches(lib, mesh, scans):
    out = []
    for k, (wld, t) in enumerate(scans):
        n0 = api.launch_count(lib)
        mesh.push_frame(wld, t, k)
        out.append(api.launch_count(lib) - n0)
    return out


def test_off_means_off(cuda_lib):
    scans = world_scans("avia", 3, 4)
    a = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    b = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    b.feed_enable(max_frames=8, max_rows=1 << 16)
    b.feed_disable()
    la, lb = per_frame_launches(cuda_lib, a, scans), per_frame_launches(cuda_lib, b, scans)
    assert la == lb, (la, lb)
    c = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    c.feed_enable(max_frames=8, max_rows=1 << 16)
    assert all(x > y for x, y in zip(per_frame_launches(cuda_lib, c, scans), la))
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    # the queued chain: graphs, PDL edges, snapshot, change rows and view image as without the feed
    res = []
    for mode in ("never", "on_off", "on"):
        def act(mesh, state, mode=mode):
            mesh.changes_enable(1 << 20, 64)
            if mode != "never":
                mesh.feed_enable(max_frames=16, max_rows=1 << 20, max_images=4)
            if mode == "on_off":
                mesh.feed_disable()
        lio, mesh = lio_chain(cuda_lib, n_scans=5, view=dict(SMALL_VIEW), actions={1: act})
        lio.wait()
        mesh.wait()
        res.append((api.graph_stats(lio, mesh), mesh.snapshot(), mesh.changes(0), mesh.view_image()))
    (g0, s0, c0, v0), (g1, s1, c1, v1), (g2, s2, c2, v2) = res
    assert g0 == g1, (g0, g1)
    for x, y, z in zip(s0, s1, s2):
        assert np.array_equal(x, y) and np.array_equal(x, z)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(c0[key], c1[key]) and np.array_equal(c0[key], c2[key]), key
    for x, y, z in zip(v0, v1, v2):
        assert np.array_equal(np.asarray(x), np.asarray(y)) and np.array_equal(np.asarray(x), np.asarray(z))


def test_lifetime_rules(cuda_lib):
    """view_enable at another size, reinforce_enable at another size and off / on, pool growth and a second feed_enable, each with
    frames in flight; the records on either side match the twin; destroy with the feed on and frames queued"""
    small = api.MeshConfig(max_vertices=1 << 13, max_triangles=1 << 14, max_voxels=1 << 11, max_frame_points=1 << 18)

    def view_resize(mesh, st):
        mesh.view_enable(width=96, height=64)
        st["twin_img"] = False   # the feed records no image from here on

    def rf_resize(mesh, st):
        mesh.reinforce_enable(width=200, height=150)

    def rf_off(mesh, st):
        mesh.reinforce_disable()
        st["rf"] = False

    def rf_on(mesh, st):
        mesh.reinforce_enable(width=256, height=128)
        st["rf"] = True

    def refeed(mesh, st):
        if st.get("feed"):
            mesh.feed_enable(max_frames=32, max_rows=1 << 20)

    acts = {3: view_resize, 4: rf_resize, 5: rf_off, 6: rf_on, 8: refeed}
    tw = Expect()
    _, twin_mesh = lio_chain(cuda_lib, n_scans=11, rf=True, view=dict(SMALL_VIEW), twin=tw, actions=acts, mesh_cfg=small, growth=4 << 30)
    st = {}

    def refeed_check(mesh, s):
        s["feed"] = True
        before = mesh.feed(0, wait=True)   # the records of the first enable, read before the second one drops them
        st["before"] = before
        st["images_after_resize"] = mesh.lib.immesh_mesh_feed_images(mesh._h, 0, 0, None, 0, None, None, np.zeros(4, np.int64).ctypes.data_as(C.POINTER(C.c_int64)))
        refeed(mesh, s)

    acts_feed = dict(acts)
    acts_feed[8] = refeed_check
    lio, mesh = lio_chain(cuda_lib, n_scans=11, rf=True, view=dict(SMALL_VIEW), feed=dict(max_frames=64, max_rows=1 << 20, max_images=4, depth=True),
                          actions=acts_feed, mesh_cfg=small, growth=4 << 30)
    tw.check(st["before"], range(1, 8))
    assert st["images_after_resize"] == E_INVALID
    out = mesh.feed(7, wait=True)
    tw.check(out, range(8, 11))
    with pytest.raises(api.FeedLost):
        mesh.feed(5)
    assert mesh.capacity()["growths"] > 0 and twin_mesh.capacity()["growths"] > 0   # the pools grew during the stream
    mesh.wait()   # snapshot sizes its buffers from the counts of the last harvested frame
    for x, y in zip(mesh.snapshot(), twin_mesh.snapshot()):
        assert np.array_equal(x, y)
    # destroy with the feed on and frames in flight
    lio2, m2 = lio_chain(cuda_lib, n_scans=4, rf=True, feed=dict(max_frames=8, max_rows=1 << 20))
    m2.close()
    lio2.wait()


def test_losses(cuda_lib):
    tw = Expect()
    _, twin_mesh = lio_chain(cuda_lib, rf=True, twin=tw)
    sizes = sorted(len(p) for p in tw.points.values())
    max_rows = sizes[len(sizes) // 2]
    assert sizes[0] < sizes[-1]
    outs = []

    def reads(k, mesh):   # the ring holds one frame's points at most: read each frame as soon as it is recorded
        outs.append(mesh.feed(k - 1, wait=True))
    _, mesh = lio_chain(cuda_lib, rf=True, feed=dict(max_frames=64, max_rows=max_rows), reads=reads)
    lost = []
    for k, out in enumerate(outs, start=1):
        tw.check(out, [k], max_rows=max_rows)
        lost.append(int(out["frames"][0, H["rows_lost"]]))
    assert 0 < sum(lost) < len(lost), lost
    mesh.wait()   # snapshot sizes its buffers from the counts of the last harvested frame
    for x, y in zip(mesh.snapshot(), twin_mesh.snapshot()):
        assert np.array_equal(x, y)


def test_error_contract(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=L)
    counts = np.zeros(4, np.int64)
    cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
    cfg = api._MeshFeedCfg

    def enable(*a):
        return L.immesh_mesh_feed_enable(mesh._h, C.byref(cfg(*a)))
    assert L.immesh_mesh_feed_enable(None, None) == E_INVALID
    for bad in ((0, 0, 0, 0, 0), ((1 << 20) + 1, 0, 0, 0, 0), (8, -1, 0, 0, 0), (8, (1 << 32) + 1, 0, 0, 0), (8, 0, -1, 0, 0),
                (8, 0, (1 << 16) + 1, 0, 0), (8, 0, 0, 2, 0), (8, 0, 0, 1, 0), (8, 0, 4, 0, 0)):   # the last two: depth without images, images without the view
        assert enable(*bad) == E_INVALID, bad
    # the feed off
    assert L.immesh_mesh_feed(mesh._h, 0, 0, None, None, 0, None, None, 0, cp) == E_INVALID
    assert L.immesh_mesh_feed_images(mesh._h, 0, 0, None, 0, None, None, cp) == E_INVALID
    scans = world_scans("avia", 4, 2)
    mesh.push_frame(scans[0][0], scans[0][1], 0)   # frame 1, before the enable
    assert enable(8, 1 << 20, 0, 0, 0) == 0
    for k in (1, 2, 3):
        mesh.push_frame(scans[k][0], scans[k][1], k)
    assert L.immesh_mesh_feed(mesh._h, 0, 0, None, None, 0, None, None, 0, cp) == E_RANGE and counts[2] == 4 and counts[3] == 4
    assert L.immesh_mesh_feed(mesh._h, 1, 0, None, None, 0, None, None, 0, cp) == 0 and counts.tolist()[0] == 3
    assert L.immesh_mesh_feed(mesh._h, 5, 0, None, None, 0, None, None, 0, cp) == E_INVALID   # newer than the newest queued
    assert L.immesh_mesh_feed(mesh._h, -1, 0, None, None, 0, None, None, 0, cp) == E_INVALID
    assert L.immesh_mesh_feed(mesh._h, 1, 0, None, None, -1, None, None, 0, cp) == E_INVALID
    assert L.immesh_mesh_feed(mesh._h, 1, 0, None, None, 1, None, None, 0, cp) == E_INVALID   # frames NULL with cap > 0
    assert L.immesh_mesh_feed(mesh._h, 1, 0, None, None, 0, None, None, 0, None) == E_INVALID
    hdr = np.zeros((2, api.MESH_FEED_HDR), np.int64)
    assert L.immesh_mesh_feed(mesh._h, 1, 0, hdr.ctypes.data_as(C.POINTER(C.c_int64)), None, 2, None, None, 0, cp) == E_CAPACITY
    assert counts[0] == 3 and not hdr.any()
    assert L.immesh_mesh_feed_images(mesh._h, 1, 0, None, 0, None, None, cp) == E_INVALID   # no image recording
    # a view enabled after the feed does not start image recording; its re-enable keeps it off
    mesh.view_enable(**SMALL_VIEW)
    assert L.immesh_mesh_feed_images(mesh._h, 1, 0, None, 0, None, None, cp) == E_INVALID
    assert enable(8, 0, 2, 0, 0) == 0
    mesh.push_frame(scans[0][0], scans[0][1], 4)
    dep = np.zeros((1, 120, 160), np.float32)
    assert L.immesh_mesh_feed_images(mesh._h, 4, 1, hdr.ctypes.data_as(C.POINTER(C.c_int64)), 1, None, dep.ctypes.data_as(C.POINTER(C.c_float)), cp) == E_INVALID
    assert L.immesh_mesh_feed_images(mesh._h, 4, 1, None, 0, None, None, cp) == 0 and counts.tolist() == [1, 1, 5, 5]
    mesh.view_enable(width=64, height=48)
    assert L.immesh_mesh_feed_images(mesh._h, 4, 1, None, 0, None, None, cp) == E_INVALID
    mesh.push_frame(scans[1][0], scans[1][1], 5)
    out = mesh.feed(4, wait=True)
    assert out["frames"][1, H["img_begin"]] == out["frames"][1, H["img_end"]] == 1
    assert L.immesh_mesh_feed_enable(mesh._h, None) == 0
    assert L.immesh_mesh_feed(mesh._h, 0, 0, None, None, 0, None, None, 0, cp) == E_INVALID
