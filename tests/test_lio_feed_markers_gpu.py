"""GPU tier: the scan feed's plane-map markers (immesh_lio_feed_markers_enable / immesh_lio_feed_markers).  Every entry point that
records a feed scan runs with the feed and the markers on and no wait between scans; a twin handle runs the same scans and calls the
blocking immesh_voxelmap_plane_markers after each one.  Headers and rows must equal the twin's bit for bit except the id column (the
node record index), whose values must be unique within a scan and stable per node.  Also: the blocking and the staged chains against
the oracle's full walk; the IMU chain's branches; lost scans; blocking calls between queued scans; the local map and a rehash; direct
launches; reads without draining; nothing changes while the markers are off; the error contract."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from immesh_b200 import api, synth
from lio_common import init_velocity
from plane_markers_common import NOT_ID, ID, PubOracle
from test_lio_feed_gpu import Chain

pytestmark = pytest.mark.gpu

M = {k: i for i, k in enumerate(api.MARKER_HDR_KEYS)}
CHAINS = ("step", "step_dev", "step_async", "step_async_dev_n", "raw", "raw_i", "imu", "imu_i")


class MarkChain(Chain):
    """Chain with the blocking and device-pointer entry points as well"""

    def step(self, k):
        import torch
        sc, g = self.scans[k], self.g
        if self.chain == "step":
            g.step(sc["body_ds"])
        elif self.chain == "step_dev":
            t = torch.from_numpy(np.ascontiguousarray(sc["body_ds"], np.float32)).cuda()
            g.step_dev(t.data_ptr(), t.shape[0])
        elif self.chain == "step_async_dev_n":
            t = torch.from_numpy(np.ascontiguousarray(sc["body_ds"], np.float32)).cuda()
            n = torch.tensor([t.shape[0]], dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            self.keep = (t, n)   # the queued step reads both at execution time
            assert g.lib.immesh_lio_step_async_dev_n(g._h, C.c_void_p(t.data_ptr()), t.shape[0], C.c_void_p(n.data_ptr()), 0.0, 0.1, 0.1) == 0
        else:
            return super().step(k)
        return 0


def blocking(g):
    """the twin's record: header fields and rows of a blocking call right after the scan"""
    g.wait()
    rows, c = g.plane_markers()
    hdr = dict(rows_needed=rows.shape[0], lost=0, roots_walked=c["roots_walked"], plane=c["plane"], sub_plane=c["sub_plane"],
               sub_sub_plane=c["sub_sub_plane"], update=c["update"])
    return hdr, rows


def check_records(feed, expected, first=1, ids=None, stable_ids=True):
    """feed records against the twin's: every header field, the rows except the id column; ids unique per scan, and stable per node
    unless nodes may be freed and made again (stable_ids False: the local map evicts roots)"""
    scans, rows = feed["scans"], feed["rows"]
    assert scans.shape[0] == len(expected)
    r0 = scans[0, M["row_begin"]] if len(expected) else 0
    ids = {} if ids is None else ids
    for i, (hdr, erows) in enumerate(expected):
        h = scans[i]
        assert h[M["scan"]] == first + i
        for key, v in hdr.items():
            assert h[M[key]] == v, (i, key, h[M[key]], v)
        a, b = h[M["row_begin"]] - r0, h[M["row_end"]] - r0
        got = rows[a:b]
        assert got.shape == erows.shape, (i, got.shape, erows.shape)
        assert np.array_equal(got[:, NOT_ID], erows[:, NOT_ID]), i
        assert np.unique(got[:, ID]).size == got.shape[0]
        for r in got if stable_ids else ():
            kp = tuple(int(v) for v in r[:4])
            assert ids.setdefault(kp, int(r[ID])) == int(r[ID]), kp
    return ids


def _pair(lib, chain, kind, max_rows=1 << 20):
    a, b = MarkChain(lib, chain, kind), MarkChain(lib, chain, kind)
    a.g.feed_enable(max_scans=64, effect=False, registered=0)
    a.g.feed_markers_enable(max_rows)
    if chain not in ("imu", "imu_i"):   # the first message after immesh_voxelmap_build: one blocking call on each before queuing
        ra, _ = a.g.plane_markers()
        rb, _ = b.g.plane_markers()
        assert np.array_equal(ra[:, NOT_ID], rb[:, NOT_ID])
    return a, b


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
@pytest.mark.parametrize("chain", CHAINS)
def test_markers_equal_blocking_twin(cuda_lib, chain, kind):
    a, b = _pair(cuda_lib, chain, kind)
    expected, branches = [], []
    for k in range(len(a.scans)):
        branches.append(a.step(k))
        assert b.step(k) == branches[-1]
        expected.append(blocking(b.g))
    f = a.g.feed_markers(0, wait=True)
    assert f["newest_finished"] == f["newest_queued"] == len(a.scans)
    check_records(f, expected)
    assert f["rows"].shape[0] > 0
    if chain.startswith("imu"):
        assert branches[:3] == [1, 1, 2]
        s = f["scans"]
        assert (s[:2, M["roots_walked"]] == 0).all() and (s[:2, M["rows_needed"]] == 0).all()
        assert s[2, M["rows_needed"]] > 0            # voxel_map_init is published
    a.g.wait()
    assert np.array_equal(a.g.get_state(), b.g.get_state()) and np.array_equal(a.g.dump_map(), b.g.dump_map())
    a.close(); b.close()


@pytest.mark.parametrize("chain", ["step", "staged"])
def test_chain_against_oracle(cuda_lib, chain):
    """against the oracle's walk over the whole map after each scan.  step: immesh_lio_step records every scan.  staged: the staged
    calls (predict, estimate, update) record nothing, and a blocking call after each of them publishes what the oracle does; the
    queued steps that follow are recorded and equal the oracle too"""
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 10, seed=6, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T)
    g, o = api.Lio(cfg, lib=cuda_lib), PubOracle(cfg)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    g.feed_enable(max_scans=16, effect=False, registered=0)
    g.feed_markers_enable(1 << 18)
    rg, _ = g.plane_markers()
    ro, _ = o.plane_markers()
    assert np.array_equal(rg[:, NOT_ID], ro[:, NOT_ID])
    expected, n_staged = [], 4 if chain == "staged" else 0
    for k in range(1, len(scans)):
        body, dt = scans[k]["body_ds"], scans[k]["dt"]
        o.predict(dt)
        o.lio_state_estimation(body)
        o.map_incremental_grow(body)
        ro, co = o.plane_markers()
        if k <= n_staged:
            g.predict(dt)
            g.lio_state_estimation(body)
            g.map_incremental_grow()
            rg, cg = g.plane_markers()
            assert np.array_equal(rg[:, NOT_ID], ro[:, NOT_ID]) and [cg["plane"], cg["sub_plane"], cg["update"]] == [co[0], co[1], co[3]]
            assert g.feed_markers(0, wait=True)["scans"].shape[0] == 0
            continue
        if chain == "step":
            g.step(body, dt=dt)
        else:
            g.step_async(body, dt=dt)
        expected.append((dict(rows_needed=ro.shape[0], plane=int(co[0]), sub_plane=int(co[1]), update=int(co[3])), ro))
    f = g.feed_markers(0, wait=True)
    check_records(f, expected)
    assert f["rows"].shape[0] > 0


def test_losses_consume_nothing(cuda_lib):
    """a ring smaller than some scans' rows: lost scans report ROWS_NEEDED and no rows; later scans equal a twin that skipped the
    blocking call at the lost scans; state, map and mesh equal a run with the markers off"""
    ref = MarkChain(cuda_lib, "raw", "hdl64")
    ref.g.feed_enable(max_scans=64, effect=False, registered=0)
    need = []
    ref.g.plane_markers()
    for k in range(len(ref.scans)):
        ref.step(k)
        need.append(blocking(ref.g)[1].shape[0])
    max_rows = int(np.median(need))
    assert min(need) <= max_rows < max(need)
    a, b = _pair(cuda_lib, "raw", "hdl64", max_rows=max_rows)
    off = MarkChain(cuda_lib, "raw", "hdl64")
    off.g.feed_enable(max_scans=64, effect=False, registered=0)
    off.g.plane_markers()
    gm = [api.Mesh(api.MeshConfig(max_vertices=1 << 19, max_triangles=1 << 20, max_voxels=1 << 17, max_frame_points=1 << 17), lib=cuda_lib) for _ in range(2)]
    lost, ids, recs = 0, {}, []
    for k in range(len(a.scans)):
        a.step(k)
        b.step(k)
        off.step(k)
        gm[0].push_frame_from_lio_async(a.g, a.vg.input_points(), a.n(k), on_device=True)
        gm[1].push_frame_from_lio_async(off.g, off.vg.input_points(), off.n(k), on_device=True)
        b.g.wait()
        n, c = C.c_int(0), np.zeros(5, np.int64)
        rc = cuda_lib.immesh_voxelmap_plane_markers(b.g._h, None, 0, C.byref(n), c.ctypes.data_as(C.POINTER(C.c_int64)))
        if n.value > max_rows:   # the twin skips pubPlaneMap where the ring loses the scan
            assert rc == -3
            lost += 1
            expected = (dict(rows_needed=n.value, lost=1, roots_walked=int(c[4]), plane=int(c[0]), update=int(c[3])), np.zeros((0, 16)))
        else:
            expected = blocking(b.g)
        f = a.g.feed_markers(k, wait=True)   # each scan on its own: the small ring holds about one scan's rows
        check_records(f, [expected], first=k + 1, ids=ids)
        recs.append(f["scans"][0])
    assert lost > 0
    recs = np.array(recs)
    lost_rows = recs[recs[:, M["lost"]] == 1]
    assert (lost_rows[:, M["row_begin"]] == lost_rows[:, M["row_end"]]).all()
    for h in (a.g, off.g):
        h.wait()
    for m in gm:
        m.wait()
    assert np.array_equal(a.g.get_state(), off.g.get_state()) and np.array_equal(a.g.dump_map(), off.g.dump_map())
    for x, y in zip(gm[0].snapshot(), gm[1].snapshot()):
        assert np.array_equal(x, y)


def test_blocking_call_between_queued_scans(cuda_lib):
    """a blocking call after a queued scan drains behind that scan's record and takes what the record held back: the next scan's
    record has none of it, on both handles alike"""
    a, b = _pair(cuda_lib, "step_async", "avia")
    expected = []
    for k in range(len(a.scans)):
        a.step(k)
        b.step(k)
        expected.append(blocking(b.g))
        if k % 2 == 1:
            ra, ca = a.g.plane_markers()
            rb, cb = b.g.plane_markers()
            assert np.array_equal(ra[:, NOT_ID], rb[:, NOT_ID]) and ca == cb
    check_records(a.g.feed_markers(0, wait=True), expected)


def test_local_map_and_rehash(cuda_lib):
    """a small local-map cube that evicts roots, and a reserve that rehashes the root table mid-run"""
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=14)
    sensor, scans = synth.make_stream("hdl64loop", 24, seed=4, leaf=cfg.filter_size_surf, n_points=32768)
    hs = []
    for _ in range(2):
        g = api.Lio(cfg, lib=cuda_lib)
        g.local_map(40.0, 10.0, 1.5)
        g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(g, sensor, scans)
        g.voxel_map_init(scans[0]["body_full"])
        g.plane_markers()
        hs.append(g)
    a, b = hs
    a.feed_enable(max_scans=64, effect=False, registered=0)
    a.feed_markers_enable(1 << 18)
    expected = []
    for k in range(1, len(scans)):
        if k == 12:
            for g in (a, b):
                g.reserve(root_slots=1 << 16)
        a.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        b.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        expected.append(blocking(b))
    check_records(a.feed_markers(0, wait=True), expected, stable_ids=False)
    _, st = a.local_map_state()
    assert st["roots_evicted"] > 0 and a.capacity()["root_slots"] == 1 << 16


def test_direct_launches_agree_with_graph(cuda_lib, monkeypatch):
    out = []
    for graph in ("1", "0"):
        monkeypatch.setenv("IMMESH_GRAPH", graph)
        a, _ = _pair(cuda_lib, "raw", "avia")
        for k in range(len(a.scans)):
            a.step(k)
        out.append(a.g.feed_markers(0, wait=True))
    assert out[0]["rows"].shape[0] > 0
    assert np.array_equal(out[0]["scans"], out[1]["scans"])
    assert np.array_equal(out[0]["rows"][:, NOT_ID], out[1]["rows"][:, NOT_ID])


def test_read_without_draining(cuda_lib):
    """a 4 GB write queued on the handle's stream ahead of each scan keeps the scan unfinished for about a millisecond: a read with
    wait = 0 right after the enqueue must return without it (a read that synchronised the stream would see every scan finished)"""
    import torch
    a, _ = _pair(cuda_lib, "raw", "avia")
    slow = torch.empty(1 << 30, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    seen, reads, behind = 0, [], 0
    for k in range(len(a.scans)):
        a.g.enqueue_memset(slow.data_ptr(), slow.numel() * 4)
        a.step(k)
        f = a.g.feed_markers(0, wait=False)
        m = f["scans"].shape[0]
        assert seen <= m == f["newest_finished"] <= f["newest_queued"] == k + 1
        behind += f["newest_finished"] < f["newest_queued"]
        seen = m
        reads.append(f)
    assert behind > 0
    full = a.g.feed_markers(0, wait=True)
    for f in reads:
        m, r = f["scans"].shape[0], f["rows"].shape[0]
        assert np.array_equal(f["scans"], full["scans"][:m]) and np.array_equal(f["rows"], full["rows"][:r])
    part = a.g.feed_markers(3)
    assert np.array_equal(part["scans"], full["scans"][3:])


def test_off_means_off(cuda_lib):
    def run(mode):
        c = MarkChain(cuda_lib, "raw", "avia")
        c.g.feed_enable(max_scans=16, effect=True, registered=2)
        if mode != "never":
            c.g.feed_markers_enable(1 << 16)
        if mode == "on_off":
            c.g.feed_markers_enable(0)
        n0 = api.launch_count(cuda_lib)
        for k in range(len(c.scans)):
            c.step(k)
        c.g.wait()
        n1 = api.launch_count(cuda_lib)
        return c, n1 - n0, api.graph_stats(c.g, None), c.g.feed(0, wait=True)
    never, n_never, gs_never, f_never = run("never")
    onoff, n_onoff, gs_onoff, f_onoff = run("on_off")
    on, _, gs_on, f_on = run("on")
    assert n_never == n_onoff and gs_never == gs_onoff
    assert gs_on["lio_pdl_edges"] > gs_never["lio_pdl_edges"]
    for f in (f_onoff, f_on):   # the scan feed's own records do not change
        for key in ("scans", "states", "rows", "row_index"):
            assert np.array_equal(f[key], f_never[key]), key
    for c in (onoff, on):
        assert np.array_equal(c.g.get_state(), never.g.get_state()) and np.array_equal(c.g.dump_map(), never.g.dump_map())
    with pytest.raises(RuntimeError, match="code -1"):
        onoff.g.feed_markers(0)


def test_error_contract(cuda_lib):
    g = api.Lio(api.AVIA, lib=cuda_lib)
    assert cuda_lib.immesh_lio_feed_markers_enable(g._h, 16) == -1          # the feed is off
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed_markers(0)
    g.feed_enable(max_scans=4, max_rows=0, effect=False, registered=0)
    assert cuda_lib.immesh_lio_feed_markers_enable(g._h, -1) == -1
    for big in ((1 << 32) + 1, 1 << 59, (1 << 63) - 1):   # beyond 2^32 rows: refused, never a wrapped allocation size
        assert cuda_lib.immesh_lio_feed_markers_enable(g._h, big) == -1
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed_markers(0)                                                       # the markers are off
    g.feed_markers_enable(64)
    cnt = (C.c_int64 * 4)()
    assert cuda_lib.immesh_lio_feed_markers(g._h, 1, 0, None, 0, None, 0, cnt) == -1    # beyond the newest queued scan
    assert cuda_lib.immesh_lio_feed_markers(g._h, -1, 0, None, 0, None, 0, cnt) == -1
    assert cuda_lib.immesh_lio_feed_markers(g._h, 0, 0, None, 0, None, 0, None) == -1
    assert cuda_lib.immesh_lio_feed_markers(g._h, 0, 0, None, -1, None, 0, cnt) == -1
    assert cuda_lib.immesh_lio_feed_markers(g._h, 0, 0, None, 0, None, 0, cnt) == 0
    g.feed_enable(max_scans=4, max_rows=0, effect=False, registered=0)      # re-enabling the feed turns the markers off
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed_markers(0)
    g.feed_markers_enable(64)
    g.feed_disable()
    with pytest.raises(RuntimeError, match="code -1"):
        g.feed_markers(0)
