"""GPU tier: the scan feed (immesh_lio_feed_enable / immesh_lio_feed).  Every chain -- step_async, _raw, _raw_i, _imu, _imu_i -- runs
with the feed on and no wait between scans; a twin handle runs the same scans and, after each one, waits and calls the blocking
publishers.  Every recorded header field, state and row must equal the twin's bit for bit.  Also: the direct and the graph-replayed
step agree; reads without draining return a growing prefix; the feed off leaves the launch sequence, the graphs and the outputs as
they were; losses, capacity and count queries; the error contract."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from frontend_intensity_common import intensities, records
from imu_stream_common import imu_cfg, make_imu_stream, true_velocity

pytestmark = pytest.mark.gpu

N_SCANS = 7
MAX_INI = 30          # 20 IMU samples per scan: branch 1 twice, then branch 2, then branch 3
KINDS = {"step_async": 2, "raw": 4, "raw_i": 5, "imu": 6, "imu_i": 7}   # IMMESH_FEED_KIND_*
H = {k: i for i, k in enumerate(api.FEED_HDR_KEYS)}


# ---- fixtures: the streams, built in this file
def _lio_stream(kind, seed):
    n_points = 32768 if kind == "hdl64" else None
    _, scans = synth.make_stream(kind, N_SCANS, seed=seed, ext_T=api.AVIA.ext_T, n_points=n_points)
    return scans


def _imu_stream(kind, seed):
    n_points = 32768 if kind == "hdl64" else None
    sensor, scans = make_imu_stream(N_SCANS, seed=seed, kind=kind, n_points=n_points)
    s0 = np.zeros(348)
    s0[0:9] = np.eye(3).reshape(9)
    s0[12:15] = true_velocity(sensor, scans[0]["beg"])
    for i in range(18):
        s0[24 + i * 18 + i] = 1e-7
    return s0, scans


class Chain:
    """one handle set (localization, VoxelGrid, IMU) running one chain over a stream"""

    def __init__(self, lib, chain, kind, seed=3):
        self.chain, self.lib = chain, lib
        self.g = api.Lio(api.AVIA, lib=lib)
        self.vg = api.VoxelGrid(1 << 17, lib=lib)
        self.leaf = api.AVIA.filter_size_surf
        if chain.startswith("imu"):
            s0, self.scans = _imu_stream(kind, seed)
            self.g.set_state(s0)
            self.imu = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32, lib=lib)
            self.imu.init_begin(MAX_INI)
        else:
            self.scans = _lio_stream(kind, seed)
            self.g.set_pose(self.scans[0]["R_true"], self.scans[0]["t_true"])
            self.g.voxel_map_init(self.scans[0]["body_full"])
            self.scans = self.scans[1:]

    def n(self, k):
        sc = self.scans[k]
        return (sc["pts"] if "pts" in sc else sc["body_full"]).shape[0]

    def step(self, k):
        """queue scan k; returns its IMU branch (0: LiDAR-only)"""
        sc, g, vg = self.scans[k], self.g, self.vg
        if self.chain == "step_async":
            g.step_async(sc["body_ds"])
        elif self.chain == "raw":
            vg.step_async_raw(g, sc["body_full"], self.leaf)
        elif self.chain == "raw_i":
            xyz = sc["body_full"]
            vg.step_async_raw_i(g, records(xyz, intensities(xyz.shape[0], k), 5, 4), self.leaf, 4)
        elif self.chain == "imu":
            return vg.step_async_imu(g, self.imu, sc["imu"], sc["pts"], sc["beg"], self.leaf)
        else:
            p = sc["pts"]
            rec = records(p[:, :3], intensities(p.shape[0], k), 5, 4, stamps=p[:, 3], time_col=3)
            return vg.step_async_imu_i(g, self.imu, sc["imu"], rec, sc["beg"], self.leaf, 3, 4)
        return 0

    def blocking_record(self, k, branch, effect, registered, skip):
        """what the blocking calls give right after scan k: (header, state, rows, row_index)"""
        g = self.g
        state, iters = g.wait()
        lio = branch in (0, 3)
        if not lio:
            state, iters = g.get_state(), 0
        st = g.iter_stats(iters - 1) if iters > 0 else dict(n_match=0, converged=0)
        rows, idx = [np.zeros((0, 4), np.float32)], [np.zeros(0, np.int32)]
        src = 0
        if lio and effect:
            r, i = g.effect_cloud()
            rows.append(r)
            idx.append(i)
        if lio and registered:
            if registered == 2 and self.chain in ("raw", "imu"):
                r, src = g.registered_cloud(self.vg.input_points(), point_skip=skip, on_device=True, n=self.n(k), stride=3), 2
            elif registered == 2 and self.chain in ("raw_i", "imu_i"):
                r, src = g.frontend_cloud(self.vg, True, point_skip=skip), 2
            else:
                r, src = g.registered_cloud(None, point_skip=skip), 1
            rows.append(r)
            idx.append(np.full(r.shape[0], -1, np.int32))
        hdr = dict(kind=KINDS[self.chain], branch=branch, iters=iters, matches=int(st["n_match"]), converged=int(st["converged"]),
                   err=g.counts()["err"], source=src, rows_lost=0)
        return hdr, state, np.concatenate(rows), np.concatenate(idx)

    def close(self):
        self.g.close()


def _check_records(feed, expected, first=1):
    scans, states, rows, ridx = feed["scans"], feed["states"], feed["rows"], feed["row_index"]
    assert scans.shape[0] == len(expected)
    r0 = scans[0, H["row_begin"]] if len(expected) else 0
    for i, (hdr, state, erows, eidx) in enumerate(expected):
        h = scans[i]
        assert h[H["scan"]] == first + i
        for key, v in hdr.items():
            assert h[H[key]] == v, (i, key, h[H[key]], v)
        assert np.array_equal(states[i], state), (i, np.abs(states[i] - state).max())
        a, e, b = h[H["row_begin"]] - r0, h[H["row_effect_end"]] - r0, h[H["row_end"]] - r0
        assert b - a == erows.shape[0], (i, b - a, erows.shape[0])
        assert np.array_equal(rows[a:b], erows), i
        assert np.array_equal(ridx[a:b], eidx), i
        assert e - a == int((eidx >= 0).sum())


def _run_pair(lib, chain, kind, effect, registered, skip):
    a, b = Chain(lib, chain, kind), Chain(lib, chain, kind)
    a.g.feed_enable(max_scans=64, max_rows=1 << 22, effect=effect, registered=registered, point_skip=skip)
    expected, branches = [], []
    for k in range(len(a.scans)):
        branches.append(a.step(k))                     # nothing waited between scans
        br = b.step(k)
        assert br == branches[-1]
        expected.append(b.blocking_record(k, br, effect, registered, skip))
    feed = a.g.feed(0, wait=True)
    assert feed["newest_finished"] == feed["newest_queued"] == len(a.scans)
    _check_records(feed, expected)
    a.g.wait()
    # the feed changes nothing the chain computes
    assert np.array_equal(a.g.get_state(), b.g.get_state())
    assert np.array_equal(a.g.dump_map(), b.g.dump_map())
    return a, b, branches, feed


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
@pytest.mark.parametrize("chain", list(KINDS))
@pytest.mark.parametrize("skip", [1, 5])
def test_feed_equals_blocking_twin(cuda_lib, chain, kind, skip):
    registered = 2 if chain != "step_async" else 1
    a, b, branches, feed = _run_pair(cuda_lib, chain, kind, True, registered, skip)
    if chain.startswith("imu"):
        assert branches[:3] == [1, 1, 2] and set(branches[3:]) == {3}
        s = feed["scans"]
        assert (s[:3, H["row_end"]] == s[:3, H["row_begin"]]).all() and (s[:3, H["iters"]] == 0).all()
    assert (feed["scans"][:, H["rows_lost"]] == 0).all()
    a.close(); b.close()


@pytest.mark.parametrize("registered", [0, 1, 2])
def test_feed_sources_without_effect(cuda_lib, registered):
    """effect off and each registered source: registered = 2 on a plain step falls back to the down-sampled scan and says so"""
    _run_pair(cuda_lib, "raw", "avia", False, registered, 3)
    a, b, _, feed = _run_pair(cuda_lib, "step_async", "avia", False, registered, 3)
    assert (feed["scans"][:, H["source"]] == (1 if registered else 0)).all()


def test_direct_and_graphed_paths_agree(cuda_lib):
    scans = _lio_stream("avia", 5)
    hs = []
    for blocking in (True, False):
        g = api.Lio(api.AVIA, lib=cuda_lib)
        g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        g.voxel_map_init(scans[0]["body_full"])
        g.feed_enable(max_scans=16, effect=True, registered=1, point_skip=2)
        for sc in scans[1:]:
            g.step(sc["body_ds"]) if blocking else g.step_async(sc["body_ds"])
        hs.append(g.feed(0, wait=True))
    d, q = hs
    assert (d["scans"][:, H["kind"]] == 0).all() and (q["scans"][:, H["kind"]] == 2).all()
    d["scans"][:, H["kind"]] = 2
    for key in ("scans", "states", "rows", "row_index"):
        assert np.array_equal(d[key], q[key]), key


def test_read_without_draining(cuda_lib):
    a, b = Chain(cuda_lib, "raw", "avia"), Chain(cuda_lib, "raw", "avia")
    a.g.feed_enable(max_scans=64, effect=True, registered=2, point_skip=1)
    seen, reads = 0, []
    for k in range(len(a.scans)):
        a.step(k)
        b.step(k)
        f = a.g.feed(0, wait=False)
        m = f["scans"].shape[0]
        assert seen <= m == f["newest_finished"] <= f["newest_queued"] == k + 1
        seen = m
        reads.append(f)
    full = a.g.feed(0, wait=True)
    assert full["scans"].shape[0] == len(a.scans)
    for f in reads:   # every early read is a prefix of the final one, bit for bit
        m, r = f["scans"].shape[0], f["rows"].shape[0]
        assert np.array_equal(f["scans"], full["scans"][:m]) and np.array_equal(f["states"], full["states"][:m])
        assert np.array_equal(f["rows"], full["rows"][:r]) and np.array_equal(f["row_index"], full["row_index"][:r])
    # incremental reads from the last scan seen
    part = a.g.feed(3, wait=False)
    assert np.array_equal(part["scans"], full["scans"][3:])
    b.g.wait()
    assert np.array_equal(a.g.get_state(), b.g.get_state()) and np.array_equal(a.g.dump_map(), b.g.dump_map())


def test_nothing_changes_while_off(cuda_lib):
    def run(mode):
        c = Chain(cuda_lib, "raw", "avia")
        if mode == "on_off":
            c.g.feed_enable(max_scans=8, effect=True, registered=2)
            c.g.feed_disable()
        n0 = api.launch_count(cuda_lib)
        for k in range(len(c.scans)):
            c.step(k)
        c.g.wait()
        n1 = api.launch_count(cuda_lib)
        return c, n1 - n0, api.graph_stats(c.g, None)
    never, n_never, gs_never = run("never")
    onoff, n_onoff, gs_onoff = run("on_off")
    assert n_never == n_onoff
    assert gs_never == gs_onoff
    assert np.array_equal(never.g.get_state(), onoff.g.get_state()) and np.array_equal(never.g.dump_map(), onoff.g.dump_map())
    # the feed on adds its kernels to the captured graph, and nothing else changes
    on = Chain(cuda_lib, "raw", "avia")
    on.g.feed_enable(max_scans=8, effect=True, registered=2)
    for k in range(len(on.scans)):
        on.step(k)
    on.g.wait()
    gs_on = api.graph_stats(on.g, None)
    assert gs_on["lio_pdl_edges"] > gs_never["lio_pdl_edges"]
    assert np.array_equal(never.g.get_state(), on.g.get_state()) and np.array_equal(never.g.dump_map(), on.g.dump_map())
    with pytest.raises(RuntimeError, match="code -1"):
        onoff.g.feed(0)


def test_ring_losses_and_resync(cuda_lib):
    a = Chain(cuda_lib, "step_async", "avia")
    a.g.feed_enable(max_scans=3, max_rows=1 << 20, effect=True, registered=1)
    for k in range(len(a.scans)):
        a.step(k)
    with pytest.raises(api.FeedLost) as e:
        a.g.feed(0, wait=True)
    last = e.value.newest_finished
    assert last == len(a.scans)
    assert a.g.feed(last)["scans"].shape[0] == 0
    tail = a.g.feed(last - 3)
    assert tail["scans"][:, H["scan"]].tolist() == [last - 2, last - 1, last]
    # rows overwritten in a small row ring: headers and states stay, reading an old scan gives the loss
    b = Chain(cuda_lib, "step_async", "avia")
    b.g.feed_enable(max_scans=64, max_rows=40000, effect=False, registered=1)
    for k in range(len(b.scans)):
        b.step(k)
    with pytest.raises(api.FeedLost):
        b.g.feed(0, wait=True)
    assert b.g.feed(len(b.scans) - 1)["scans"].shape[0] == 1


def test_oversized_cloud_keeps_state(cuda_lib):
    a, b = Chain(cuda_lib, "raw", "avia"), Chain(cuda_lib, "raw", "avia")
    a.g.feed_enable(max_scans=16, max_rows=100, effect=True, registered=2)
    for k in range(len(a.scans)):
        a.step(k)
        b.step(k)
        b.g.wait()
    f = a.g.feed(0, wait=True)
    s = f["scans"]
    assert (s[:, H["rows_lost"]] == 1).all() and (s[:, H["row_end"]] == s[:, H["row_begin"]]).all() and f["rows"].shape[0] == 0
    assert np.array_equal(f["states"][-1], b.g.get_state())
    assert np.array_equal(a.g.get_state(), b.g.get_state()) and np.array_equal(a.g.dump_map(), b.g.dump_map())


def _raw_feed(g, since, cap_scans, cap_rows, rows=True, wait=1):
    counts = np.zeros(4, np.int64)
    hdr = np.zeros((max(cap_scans, 1), api.FEED_HDR), np.int64)
    r = np.zeros((max(cap_rows, 1), 4), np.float32)
    rc = g.lib.immesh_lio_feed(g._h, since, wait, hdr.ctypes.data_as(C.POINTER(C.c_int64)), None, cap_scans,
                               r.ctypes.data_as(C.POINTER(C.c_float)) if rows else None, None, cap_rows, counts.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc, counts, hdr


def test_capacity_and_count_query(cuda_lib):
    a = Chain(cuda_lib, "step_async", "avia")
    a.g.feed_enable(max_scans=16, effect=True, registered=1)
    for k in range(4):
        a.step(k)
    rc, counts, _ = _raw_feed(a.g, 0, 0, 0)
    assert rc == 0 and counts[0] == 4 and counts[1] > 0 and counts[2] == counts[3] == 4
    rc, c2, hdr = _raw_feed(a.g, 0, 3, 1 << 20)
    assert rc == -3 and np.array_equal(c2, counts) and not hdr.any()
    rc, c3, hdr = _raw_feed(a.g, 0, 4, int(counts[1]) - 1)
    assert rc == -3 and not hdr.any()
    rc, c4, hdr = _raw_feed(a.g, 1, 3, 0, rows=False)   # no rows asked: the row cap does not apply
    assert rc == 0 and c4[0] == 3 and hdr[:, 0].tolist() == [2, 3, 4]


def test_error_contract(cuda_lib):
    g = api.Lio(api.AVIA, lib=cuda_lib)
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed(0)
    for bad in (dict(max_scans=0), dict(max_rows=0), dict(registered=3), dict(point_skip=0), dict(effect=2)):
        args = dict(max_scans=4, max_rows=16, effect=True, registered=1, point_skip=1)
        args.update(bad)
        c = api._FeedCfg(args["max_scans"], args["max_rows"], int(args["effect"]), args["registered"], args["point_skip"], 0)
        assert g.lib.immesh_lio_feed_enable(g._h, C.byref(c)) == -1, bad
    g.feed_enable(max_scans=4, max_rows=0, effect=False, registered=0)   # headers and states only
    assert g.lib.immesh_lio_feed(g._h, 1, 0, None, None, 0, None, None, 0, (C.c_int64 * 4)()) == -1   # beyond the newest queued scan
    assert g.lib.immesh_lio_feed(g._h, -1, 0, None, None, 0, None, None, 0, (C.c_int64 * 4)()) == -1
    assert g.lib.immesh_lio_feed(g._h, 0, 0, None, None, 0, None, None, 0, None) == -1
    assert g.lib.immesh_lio_shard(g._h, 0, 2, b"\0" * 128) == -1   # sharding is refused while the feed is on
    g.feed_disable()
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed(0)


@pytest.mark.parametrize("chain,max_rows", [("step_async", 17011), ("raw_i", 37003), ("imu", 33013)])
def test_rows_wrap_the_ring_bit_for_bit(cuda_lib, chain, max_rows):
    """a row ring a scan's rows straddle: each scan read right after it and compared with the blocking twin, rows and row_index"""
    registered = 1 if chain == "step_async" else 2
    a, b = Chain(cuda_lib, chain, "avia"), Chain(cuda_lib, chain, "avia")
    a.g.feed_enable(max_scans=4, max_rows=max_rows, effect=True, registered=registered, point_skip=1)
    straddled, records, last = 0, [], []
    for k in range(len(a.scans)):
        br = a.step(k)
        assert b.step(k) == br
        records.append(b.blocking_record(k, br, True, registered, 1))
        f = a.g.feed(k, wait=True)
        _check_records(f, records[-1:], first=k + 1)
        h = f["scans"][0]
        straddled += h[H["row_begin"]] % max_rows + (h[H["row_end"]] - h[H["row_begin"]]) > max_rows
        assert h[H["rows_lost"]] == 0
        last.append(h)
    assert straddled >= 1
    # two scans in one read where both still fit the ring: a read across the wrap; where they do not, the older one's rows are gone
    n = len(a.scans)
    if last[-1][H["row_end"]] - last[-2][H["row_begin"]] <= max_rows:
        _check_records(a.g.feed(n - 2), records[-2:], first=n - 1)
    else:
        with pytest.raises(api.FeedLost):
            a.g.feed(n - 2)


def test_mesh_and_change_feed_unchanged(cuda_lib):
    """the mesh fed from the localization handle, and its change feed, are the same with the scan feed never on, on then off, and on"""
    def run(mode):
        c = Chain(cuda_lib, "raw", "avia")
        gm = api.Mesh(api.MeshConfig(max_vertices=1 << 19, max_triangles=1 << 20, max_voxels=1 << 17, max_frame_points=1 << 17), lib=cuda_lib)
        gm.changes_enable(1 << 20, 64)
        if mode != "never":
            c.g.feed_enable(max_scans=8, effect=True, registered=2)
        if mode == "on_off":
            c.g.feed_disable()
        for k in range(len(c.scans)):
            c.step(k)
            gm.push_frame_from_lio_async(c.g, c.vg.input_points(), c.n(k), on_device=True)
        c.g.wait()
        gm.wait()
        return gm.snapshot(), gm.changes(0)
    (sv, st, sf), ch = run("never")
    assert st.shape[0] > 0 and ch["rows"].shape[0] > 0
    for mode in ("on_off", "on"):
        (v, t, fl), c2 = run(mode)
        assert np.array_equal(v, sv) and np.array_equal(t, st) and np.array_equal(fl, sf), mode
        for key in ("frames", "rows", "vertices"):
            assert np.array_equal(c2[key], ch[key]), (mode, key)
