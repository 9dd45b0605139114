"""GPU tier: the IMU-enabled loop on depth frames (immesh_lio_step_async_depth_imu), whose drop rule and branch are decided on the device.
The bar is bit-exact equality with the host-decided path it replaces, run on a second set of handles: immesh_frontend_prepare_depth for
the cloud, the host applying sync_packages' <= 1 drop and carrying the IMU samples, then immesh_lio_step_async_imu on x y z t records
with t = 0 and the mesher hand-off in branch 3.  Over a stream with dropped frames in the initialisation, right after it and after the
map, and an immesh_imu_init_begin mid-stream (Reset()): state, map, scan-feed records and rows, plane-marker records, the mesh and the
non-empty mesh frames.  The same stream queued without any wait between frames gives the same results (one input-ring and one pose-ring
slot per call), the graph-replayed step and the direct launches agree, and a 200-frame queued run waits on the host only where
immesh_host_wait_ms counts it.  Also the carry overflow, the mixing rule and the counters."""
import time

import numpy as np
import pytest

from immesh_b200 import api
import depth_lio_reference as dlr
import depth_reference as dr
from plane_markers_common import NOT_ID

pytestmark = pytest.mark.gpu

E_INVALID, E_CAPACITY = -1, -3
W, H = 640, 480
LEAF, PFN, BLIND, MAX_INI = 0.2, 2, 0.5, 3
F_SCAN, F_KIND, F_BRANCH, F_ERR = 0, 1, 2, 6   # IMMESH_FEED_SCAN, _KIND, _BRANCH, _ERR
T0, DT = 500.0, 0.1


def cam():
    return dr.camera(W, H, kind="range", z_min=0.3, z_max=40.0, stride=1)


def image(k, valid=None):
    """frame k of the synthetic depth stream; valid = 0 / 1: an image with no / exactly one valid pixel (a cloud sync_packages drops)"""
    R, t = dr.camera_pose(k)
    img = dr.render(cam(), W, H, R, t, kind="range")
    if valid is None:
        return img
    out = np.full_like(img, np.nan)
    if valid:
        ys, xs = np.nonzero(np.isfinite(img) & (img > 2.0))
        out[ys[0], xs[0]] = img[ys[0], xs[0]]
    return out


def imu_batch(k, m, seed=0):
    """m samples of a near-static IMU over frame k: stamp, gyro, specific force (gravity along the camera's -y, seeded noise)"""
    rng = np.random.default_rng([seed, k])
    t = T0 + DT * k + (np.arange(m) + 1) * (DT / max(m, 1)) - DT
    gyr = rng.normal(0.0, 0.002, (m, 3))
    acc = np.array([0.0, -9.81, 0.0]) + rng.normal(0.0, 0.02, (m, 3))
    return np.concatenate([t[:, None], gyr, acc], axis=1)


def imu_cfg():
    return dict(cov_gyr=[0.1] * 3, cov_acc=[0.1] * 3, cov_bias_gyr=[1e-4] * 3, cov_bias_acc=[1e-4] * 3, mean_acc_norm=9.81, lid_R=np.eye(3), lid_T=[0.0] * 3)


# (frame image index, valid: None full / 0 / 1, IMU samples): dropped frames during the initialisation (counts 0 and 1), right after it,
# and after the map; an empty IMU batch; two drops in a row
# and "begin": immesh_imu_init_begin on both IMU handles mid-stream (the loop's reset), with samples still carried
STREAM = [(0, None, 2), (1, 0, 3), (1, None, 2), (2, 1, 4), (2, None, 0), (3, None, 5), (4, 0, 6), (4, 1, 5), (4, None, 5), (5, None, 10),
          (6, None, 10), (7, 0, 10), (7, None, 10), (8, None, 10), (9, None, 10), (10, 1, 10), (10, None, 10), (11, None, 10), (12, 0, 4),
          "begin", (12, None, 2), (13, 1, 1), (13, None, 1), (14, None, 10), (15, None, 10), (16, None, 10)]
N_DROPPED = 8
MAX_MARKER_ROWS = 1 << 20


class Handles:
    def __init__(self, max_imu=64):
        self.lio = api.Lio(api.LioConfig(ext_T=(0.0, 0.0, 0.0)))
        self.vg = api.VoxelGrid(W * H)
        self.imu = api.Imu(imu_cfg(), max_points=W * H, max_imu=max_imu)
        self.mesh = api.Mesh(api.MeshConfig(max_frame_points=W * H))
        self.lio.feed_enable(max_scans=256, max_rows=1 << 22, effect=True, registered=2)
        self.lio.feed_markers_enable(MAX_MARKER_ROWS)
        self.mesh.feed_enable(max_frames=256)
        self.imu.init_begin(MAX_INI)


def queued_frame(hd, k, valid, batch):
    ns = hd.vg.step_async_depth_imu(hd.lio, hd.imu, batch, image(k, valid), cam(), T0 + DT * k, LEAF, point_filter_num=PFN, blind=BLIND,
                                    cam_R=dlr.SENSOR_FROM_CAM)
    hd.mesh.push_frame_from_lio_async_dev_n(hd.lio, hd.vg.input_points(), ns, hd.vg.input_count())


class HostPath:
    """the round trip the queued chain replaces: the cloud read back, sync_packages' drop and carry on the host, t = 0 records"""

    def __init__(self):
        self.hd = Handles()
        self.carry = np.zeros((0, 7))
        self.branches = []

    def begin(self):
        self.hd.imu.init_begin(MAX_INI)
        self.carry = np.zeros((0, 7))

    def frame(self, k, valid, batch):
        cloud = self.hd.vg.prepare_depth(image(k, valid), cam(), dlr.SENSOR_FROM_CAM, point_filter_num=PFN, blind=BLIND)
        if cloud.shape[0] <= 1:
            self.carry = np.concatenate([self.carry, batch])
            return None
        pts = np.concatenate([cloud, np.zeros((cloud.shape[0], 1), np.float32)], axis=1)
        br = self.hd.vg.step_async_imu(self.hd.lio, self.hd.imu, np.concatenate([self.carry, batch]), pts, T0 + DT * k, LEAF)
        self.carry = np.zeros((0, 7))
        if br == 3:
            self.hd.mesh.push_frame_from_lio_async(self.hd.lio, self.hd.vg.input_points(), cloud.shape[0], on_device=True)
        self.branches.append(br)
        return br


def same(a, b, tag):
    sa, sb = a.lio.get_state(), b.lio.get_state()
    assert sa.tobytes() == sb.tobytes(), f"{tag}: state, max diff {np.abs(sa - sb).max()}"
    assert a.lio.dump_map().tobytes() == b.lio.dump_map().tobytes(), f"{tag}: map"
    a.mesh.wait()
    b.mesh.wait()
    for x, y in zip(a.mesh.snapshot(), b.mesh.snapshot()):
        assert x.tobytes() == y.tobytes(), f"{tag}: mesh snapshot"


def queue_stream(dev, wait_each=None):
    """the stream through the queued chain; wait_each(i): called after frame i (None: everything queued before one wait)"""
    i = 0
    for s in STREAM:
        if s == "begin":
            dev.imu.init_begin(MAX_INI)
            continue
        k, valid, m = s
        queued_frame(dev, k, valid, imu_batch(k, m, seed=i))
        if wait_each:
            wait_each(i)
        i += 1
    dev.lio.wait()
    dev.mesh.wait()


def host_stream():
    host = HostPath()
    expect = []
    i = 0
    for s in STREAM:
        if s == "begin":
            host.begin()
            continue
        k, valid, m = s
        br = host.frame(k, valid, imu_batch(k, m, seed=i))
        expect.append(api.FEED_BRANCH_DROPPED if br is None else br)
        i += 1
    host.hd.lio.wait()
    host.hd.mesh.wait()
    return host, expect


def n_frames():
    return sum(1 for s in STREAM if s != "begin")


def same_feeds(dev, host, expect):
    """the scan feed (one record per call; the kept frames' records are the host path's apart from the scan number and the kind), the
    plane-marker records, and the mesh frame feed (a frame per call; the non-empty ones are the host path's branch-3 frames)"""
    fa, fb = dev.lio.feed(0, wait=True), host.lio.feed(0, wait=True)
    ha, hb = fa["scans"], fb["scans"]
    assert len(ha) == n_frames() and len(hb) == n_frames() - N_DROPPED
    assert list(ha[:, F_BRANCH]) == expect
    assert np.all(ha[:, F_KIND] == api.FEED_KINDS.index("depth_imu")) and np.all(hb[:, F_KIND] == api.FEED_KINDS.index("imu"))
    kept = np.array([b != api.FEED_BRANCH_DROPPED for b in expect])
    x, y = ha[kept].copy(), hb.copy()
    x[:, [F_SCAN, F_KIND]] = y[:, [F_SCAN, F_KIND]] = 0
    np.testing.assert_array_equal(x, y)
    assert fa["states"][kept].tobytes() == fb["states"].tobytes()
    assert fa["rows"].tobytes() == fb["rows"].tobytes() and np.array_equal(fa["row_index"], fb["row_index"])
    for i in np.nonzero(~kept)[0]:   # a dropped frame leaves the state as it was
        if i > 0:
            assert fa["states"][i].tobytes() == fa["states"][i - 1].tobytes()
    qa, qb = dev.lio.feed_markers(0, wait=True), host.lio.feed_markers(0, wait=True)
    mk = {k: i for i, k in enumerate(api.MARKER_HDR_KEYS)}
    x, y = qa["scans"][kept].copy(), qb["scans"].copy()
    assert len(qa["scans"]) == n_frames() and np.all(qa["scans"][~kept][:, mk["row_end"]] == qa["scans"][~kept][:, mk["row_begin"]])
    x[:, mk["scan"]] = y[:, mk["scan"]] = 0
    np.testing.assert_array_equal(x, y)
    # the rows apart from the id column (the node's record index, which follows the device's allocation order; as in the marker tests)
    assert len(qa["rows"]) > 0 and np.array_equal(qa["rows"][:, NOT_ID], qb["rows"][:, NOT_ID])
    ma, mb = dev.mesh.feed(0, wait=True), host.mesh.feed(0, wait=True)
    keys = {k: i for i, k in enumerate(api.MESH_FEED_HDR_KEYS)}
    fra, frb = ma["frames"].copy(), mb["frames"].copy()
    assert len(fra) == n_frames() and len(frb) == expect.count(3)
    nz = fra[:, keys["n_points"]] > 0
    assert list(np.nonzero(nz)[0]) == [i for i, b in enumerate(expect) if b == 3]
    assert np.all(fra[:, keys["kind"]] == api.MESH_FEED_KINDS.index("from_lio_async_dev_n"))
    for h in (fra, frb):
        h[:, [keys["frame"], keys["kind"], keys["t_begin_ns"], keys["t_end_ns"]]] = 0
    np.testing.assert_array_equal(fra[nz], frb)
    assert ma["poses"][nz].tobytes() == mb["poses"].tobytes()


def test_stream_equals_host_decided_path():
    dev, ref = Handles(), HostPath()   # compared after every frame
    expect = []
    i = 0
    for s in STREAM:
        if s == "begin":
            dev.imu.init_begin(MAX_INI)
            ref.begin()
            continue
        k, valid, m = s
        batch = imu_batch(k, m, seed=i)
        queued_frame(dev, k, valid, batch)
        br = ref.frame(k, valid, batch)
        expect.append(api.FEED_BRANCH_DROPPED if br is None else br)
        dev.lio.wait()
        ref.hd.lio.wait()
        same(dev, ref.hd, f"frame {i}")
        i += 1
    assert expect.count(1) >= 3 and expect.count(2) == 1 and expect.count(3) >= 8 and expect.count(api.FEED_BRANCH_DROPPED) == N_DROPPED, expect
    st = dev.imu.depth_chain_state()
    assert st == dict(calls=n_frames(), dropped=N_DROPPED, branch1=expect.count(1), branch2=1, branch3=expect.count(3), carried=0,
                      carry_overflows=0, init_finished=1), st
    same_feeds(dev, ref.hd, expect)


def test_pipelined_stream_equals_host_decided_path():
    """no wait between frames: each frame's cloud, count and pose must stay in its ring slots until the mesher has read them"""
    dev = Handles()
    queue_stream(dev)
    host, expect = host_stream()
    same(dev, host.hd, "pipelined")
    same_feeds(dev, host.hd, expect)


def test_direct_launches_equal_graph_replay():
    """the localization step replays its captured launch sequence; with the profiler on it launches directly: the same results"""
    runs = []
    for direct in (False, True):
        api.profile_enable(direct)
        try:
            hd = Handles()
            queue_stream(hd)
            runs.append((hd, api.graph_stats(hd.lio, None)))
        finally:
            api.profile_enable(False)
    (g, gs), (d, ds) = runs
    assert gs["lio_replays"] > 0 and ds["lio_replays"] == 0, (gs, ds)
    same(g, d, "direct vs graph")
    fa, fb = g.lio.feed(0, wait=True), d.lio.feed(0, wait=True)
    for key in ("scans", "states", "rows", "row_index"):
        assert np.array_equal(fa[key], fb[key]), key


def test_queued_run_waits_only_on_staging():
    """200 frames queued with device images: every host wait inside the calls is staging back-pressure, counted by
    immesh_host_wait_ms.  A large memset queued on the localization stream ahead of every frame makes each frame take several ms of
    device time, so that a hidden synchronisation would block the host for about that long per frame without being counted."""
    import torch
    hd = Handles()
    hd.lio.feed_disable()
    imgs = [torch.from_numpy(image(k)).cuda() for k in range(8)]
    load = torch.empty(1 << 32, dtype=torch.uint8, device="cuda")   # 4 GiB: over 1 ms of memset per frame
    torch.cuda.synchronize()
    frames = 200
    api.host_wait_ms(hd.lio, hd.mesh)   # reset the counters
    t0 = time.perf_counter()
    for i in range(frames):
        k = i % 8
        hd.lio.enqueue_memset(load.data_ptr(), load.numel())
        ns = hd.vg.step_async_depth_imu(hd.lio, hd.imu, imu_batch(i, 10), imgs[k].data_ptr(), cam(), T0 + DT * i, LEAF, point_filter_num=PFN,
                                        blind=BLIND, cam_R=dlr.SENSOR_FROM_CAM, on_device=True, shape=(H, W))
        hd.mesh.push_frame_from_lio_async_dev_n(hd.lio, hd.vg.input_points(), ns, hd.vg.input_count())
    enqueue_ms = (time.perf_counter() - t0) * 1e3
    waited = sum(api.host_wait_ms(hd.lio, hd.mesh))
    t1 = time.perf_counter()
    hd.lio.wait()
    hd.mesh.wait()
    drain_ms = (time.perf_counter() - t1) * 1e3
    device_ms_per_frame = (enqueue_ms + drain_ms) / frames
    uncounted_ms_per_frame = (enqueue_ms - waited) / frames
    print(f"enqueue {enqueue_ms:.1f} ms, counted waits {waited:.1f} ms, drain {drain_ms:.1f} ms over {frames} frames")
    assert hd.imu.depth_chain_state()["calls"] == frames
    assert device_ms_per_frame > 1.0   # the load is there
    assert uncounted_ms_per_frame < 0.5 * device_ms_per_frame, (uncounted_ms_per_frame, device_ms_per_frame)

    # the scan feed: one record per call; the kept frames' records are the host path's, apart from the scan number and the kind


def test_carry_overflow_is_reported():
    hd = Handles(max_imu=8)
    queued_frame(hd, 0, None, imu_batch(0, 2))
    queued_frame(hd, 1, 0, imu_batch(1, 5))   # dropped, 5 carried
    queued_frame(hd, 1, None, imu_batch(1, 5, seed=1))   # 5 + 5 > 8: dropped, its own samples discarded
    with pytest.raises(RuntimeError, match=f"code {E_CAPACITY}"):
        hd.lio.wait()
    st = hd.imu.depth_chain_state()
    assert st["carry_overflows"] == 1 and st["carried"] == 5 and st["dropped"] == 2, st
    f = hd.lio.feed(0, wait=True)["scans"]
    assert list(f[:, F_BRANCH]) == [1, api.FEED_BRANCH_DROPPED, api.FEED_BRANCH_DROPPED]
    assert f[2, F_ERR] & 128 and not f[1, F_ERR] & 128


def test_mixing_entry_points_is_refused():
    a, b = Handles(), Handles()
    queued_frame(a, 0, None, imu_batch(0, 2))
    cloud = b.vg.prepare_depth(image(0), cam(), dlr.SENSOR_FROM_CAM, point_filter_num=PFN, blind=BLIND)
    pts = np.concatenate([cloud, np.zeros((cloud.shape[0], 1), np.float32)], axis=1)
    with pytest.raises(RuntimeError, match=f"code {E_INVALID}"):
        a.vg.step_async_imu(a.lio, a.imu, imu_batch(1, 2), pts, T0 + DT, LEAF)
    b.vg.step_async_imu(b.lio, b.imu, imu_batch(0, 2), pts, T0, LEAF)
    with pytest.raises(RuntimeError, match=f"code {E_INVALID}"):
        queued_frame(b, 1, None, imu_batch(1, 2))
    with pytest.raises(RuntimeError, match=f"code {E_CAPACITY}"):
        queued_frame(a, 1, None, imu_batch(1, 65))
    a.lio.wait()
    b.lio.wait()
    assert a.imu.depth_chain_state()["calls"] == 1
