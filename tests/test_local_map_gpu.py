"""GPU tier: the local map of the device VoxelMap (immesh_lio_local_map / immesh_voxelmap_evict_boxes) against the oracle extended by
laser_map_fov_segment and the deletion of the boxes it leaves behind (tests/local_map/orc_local_map.cpp).  A small cube on an
hdl64loop stream moves the box, evicts and re-creates root voxels many times; state, match set and canonical dump must equal the
oracle's after every scan."""
import dataclasses

import numpy as np
import pytest

from immesh_b200 import api, synth
from lio_common import init_velocity
from local_map_common import SHAPE_COLS, OracleLocalMap, f32, in_boxes, root_centres

pytestmark = pytest.mark.gpu

CUBE, DET, MOV = 40.0, 10.0, 1.5


def _crop(body, max_range):
    return body if max_range is None else body[np.linalg.norm(body.astype(np.float64), axis=1) < max_range]


def _run(cfg, n_scans, pipelined, growth=0, seed=4, n_points=32768, max_range=None, cube=(CUBE, DET, MOV), markers_at=()):
    """pipelined: True (immesh_lio_step_async + wait), False (immesh_lio_step) or "estimate" (immesh_lio_predict, immesh_lio_estimate,
    immesh_voxelmap_update); scans cropped to max_range metres when given; plane markers read after the scans in markers_at"""
    sensor, scans = synth.make_stream("hdl64loop", n_scans, seed=seed, leaf=cfg.filter_size_surf, n_points=n_points)
    for sc in scans:
        sc["body_full"], sc["body_ds"] = _crop(sc["body_full"], max_range), _crop(sc["body_ds"], max_range)
    g, o = api.Lio(cfg), OracleLocalMap(cfg)
    if growth:
        g.set_growth(growth)
    g.local_map(*cube)
    o.local_map(*cube)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
    o.segment()                      # the building scan's pose places the box
    g.voxel_map_init(scans[0]["body_full"])
    o.voxel_map_init(scans[0]["body_full"])
    assert np.array_equal(g.dump_map(), o.dump_map())
    evicted = 0
    for k in range(1, n_scans):
        body = scans[k]["body_ds"]
        o.predict(scans[k]["dt"])
        box_o, rm, ev = o.segment()
        evicted += ev
        io = o.lio_state_estimation(body)
        o.map_incremental_grow(body)
        if pipelined == "estimate":
            g.predict(scans[k]["dt"])
            ig = g.lio_state_estimation(body)
            g.map_incremental_grow()
            sg = g.get_state()
        elif pipelined:
            g.step_async(body, dt=scans[k]["dt"])
            sg, ig = g.wait()
        else:
            sg, ig = g.step(body, dt=scans[k]["dt"])
        assert ig == io, f"scan {k}: iterations"
        assert np.array_equal(g.matches(), o.matches()), f"scan {k}: matches"
        assert np.array_equal(sg, o.get_state()), f"scan {k}: state"
        box_g, st = g.local_map_state()
        assert np.array_equal(box_g.view(np.uint32), box_o.view(np.uint32)), f"scan {k}: box"
        assert st["roots_evicted"] == evicted, f"scan {k}: roots evicted"
        dg, do = g.dump_map(), o.dump_map()
        assert np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), f"scan {k}: octree shape"
        assert np.array_equal(dg, do), f"scan {k}: dump"
        if k in markers_at:
            _check_markers(g, dg)
    c = g.counts()
    assert c["err"] == 0 and c["roots"] == o.num_roots()
    return g, st


def _check_markers(g, dump):
    """the pending plane markers: every row belongs to a live root (entries of evicted roots were dropped)"""
    rows, cnt = g.plane_markers()
    live = set(map(tuple, root_centres(dump)[0].tolist()))
    assert all(tuple(int(v) for v in r[0:3]) in live for r in rows)
    return rows, cnt


@pytest.mark.parametrize("pipelined,graph", [(True, "1"), (True, "0"), (False, "1"), ("estimate", "1")], ids=["graph", "graph_off", "blocking", "estimate"])
def test_local_map_matches_oracle(monkeypatch, pipelined, graph):
    monkeypatch.setenv("IMMESH_GRAPH", graph)
    g, st = _run(api.VELODYNE, 40, pipelined)
    assert st["placed"] == 1 and st["moves"] >= 4 and st["roots_evicted"] > 0
    assert st["nodes_freed"] >= st["roots_evicted"] and st["chunks_freed"] > 0
    assert st["tombstones"] == st["roots_evicted"] and st["rebuilds"] == 0


def test_local_map_purge_matches_oracle():
    """growth off and a 2^11-slot root hash: the scans (cropped to 15 m, so that the live roots fit) leave more than 256 tombstones
    several times, and each time the next step rebuilds the table at its size.  The plane-marker list is left pending across the
    first rebuilds (its entries of evicted roots are dropped by the rebuild) and read afterwards; the oracle is matched after every
    scan, rebuilds included"""
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=11, max_nodes=1 << 15, max_chunks=1 << 16)
    g, st = _run(cfg, 70, True, max_range=15.0, cube=(30.0, 10.0, 1.5), markers_at=(45, 69))
    cap = g.capacity()
    assert st["rebuilds"] >= 2 and cap["growths"] == 0 and cap["root_slots"] == 1 << 11


def test_local_map_purge_and_growth():
    """a 2^10-slot root hash with automatic growth: tombstones are dropped by the growths' rebuilds, and the results do not move"""
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=10, max_nodes=1 << 14, max_chunks=1 << 15)
    g, st = _run(cfg, 40, True, growth=4 << 30)
    cap = g.capacity()
    assert st["rebuilds"] + cap["growths"] > 0 and st["tombstones"] < cap["root_slots"] // 8 + 1
    assert st["roots_evicted"] > 0 and st["free_nodes"] >= 0


def test_evict_boxes_hand_placed():
    cfg = api.VELODYNE
    sensor, scans = synth.make_stream("hdl64loop", 3, seed=2, leaf=cfg.filter_size_surf, n_points=32768)
    g, o = api.Lio(cfg), OracleLocalMap(cfg)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        h.voxel_map_init(scans[0]["body_full"])
    keys, ctr = root_centres(o.dump_map())
    a, b = ctr[0], ctr[-1]
    boxes = np.array([[a[0], a[1], a[2], a[0] + 7, a[1] + 7, a[2] + 7],      # a on the min edge: evicted
                      [b[0] - 7, b[1] - 7, b[2] - 7, b[0], b[1], b[2]],       # b on the max edge: kept
                      [-1e4, -1e4, -1e4, scans[0]["t_true"][0] - 20.0, 1e4, 1e4]], f32)
    hit = in_boxes(ctr, boxes)
    assert hit[0] and not in_boxes(b[None], boxes[1:2])[0]
    n0 = g.counts()
    g.evict_boxes(boxes)
    assert o.evict_boxes(boxes) == hit.sum()
    _, st = g.local_map_state()
    assert st["roots_evicted"] == hit.sum() == st["tombstones"] and st["placed"] == 0
    assert g.counts()["roots"] == n0["roots"] - hit.sum()
    assert np.array_equal(g.dump_map(), o.dump_map())
    # the map keeps working on: node records and chunks are reused
    for k in (1, 2):
        body = scans[k]["body_ds"]
        g.predict(scans[k]["dt"])
        o.predict(scans[k]["dt"])
        assert g.lio_state_estimation(body) == o.lio_state_estimation(body)
        assert np.array_equal(g.matches(), o.matches())
        g.map_incremental_grow()
        o.map_incremental_grow(body)
        assert np.array_equal(g.dump_map(), o.dump_map())
    _, st2 = g.local_map_state()
    assert st2["free_nodes"] < st["free_nodes"], "no node record was taken from the free stack"


def test_local_map_error_contract():
    g = api.Lio(api.AVIA)
    for args in ((-1.0, 300.0, 1.5), (1000.0, 0.0, 1.5), (1000.0, 300.0, -1.0), (float("inf"), 300.0, 1.5), (float("nan"), 300.0, 1.5),
                 (1000.0, float("nan"), 1.5)):
        with pytest.raises(RuntimeError):
            g.local_map(*args)
    with pytest.raises(RuntimeError):
        g.evict_boxes(np.array([[0, 0, 0, np.nan, 1, 1]], f32))
    g.local_map(100.0, 300.0, 1.5)   # cube_len <= 2 mov det is allowed
    g.local_map(0.0)
    box, st = g.local_map_state()
    assert st == dict(placed=0, moves=0, roots_evicted=0, nodes_freed=0, chunks_freed=0, tombstones=0, rebuilds=0, free_nodes=0)
    g.evict_boxes(np.zeros((0, 6), f32))


def test_local_map_invariance():
    """a straight drive with the scans cropped to 40 m and a 100 m cube: the slabs the box gives up lie at least 52 m behind the
    sensor, so no point or neighbour retry reaches an evicted root.  The state is then bit-identical to a run without the local map,
    and the dump is that run's dump minus the roots in the removed boxes (reconstructed from the box after every scan)"""
    cfg = api.VELODYNE
    sensor, scans = synth.make_stream("hdl64", 45, seed=6, leaf=cfg.filter_size_surf, n_points=32768)
    a, b = api.Lio(cfg), api.Lio(cfg)
    b.local_map(100.0, 20.0, 1.5)
    for h in (a, b):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(_crop(scans[0]["body_full"], 40.0))
    removed = []
    box, _ = b.local_map_state()
    for k in range(1, len(scans)):
        body = _crop(scans[k]["body_ds"], 40.0)
        for h in (a, b):
            h.step_async(body, dt=scans[k]["dt"])
        sa, _ = a.wait()
        sb, _ = b.wait()
        assert np.array_equal(sa, sb), f"scan {k}: state"
        nb, _ = b.local_map_state()
        for i in range(3):    # the slab given up on each axis that moved: the old box with that axis narrowed
            if nb[i] != box[i]:
                r = box.copy()
                if nb[i] < box[i]:
                    r[i] = nb[3 + i]
                else:
                    r[3 + i] = nb[i]
                removed.append(r)
        box = nb
    _, st = b.local_map_state()
    assert len(removed) >= st["moves"] >= 1 and st["roots_evicted"] > 0
    da, db = a.dump_map(), b.dump_map()
    keys, ctr = root_centres(da)
    gone = set(map(tuple, keys[in_boxes(ctr, removed)].tolist()))
    assert len(gone) == st["roots_evicted"]
    keep = np.array([tuple(int(v) for v in r[0:3]) not in gone for r in da])
    assert np.array_equal(da[keep], db)


def _oracle_raw(o, body_full, leaf):
    import oracle_api as oa
    return oa.voxel_grid(body_full, leaf)[0]


def test_local_map_raw_chain_matches_oracle():
    """the device front-end chain (immesh_lio_step_async_raw: VoxelGrid -> predict -> box rule -> IESKF -> update) with the local map"""
    cfg = api.VELODYNE
    sensor, scans = synth.make_stream("hdl64loop", 30, seed=8, leaf=cfg.filter_size_surf, n_points=32768)
    g, o = api.Lio(cfg), OracleLocalMap(cfg)
    vg = api.VoxelGrid(1 << 17)
    for h in (g, o):
        h.local_map(CUBE, DET, MOV)
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
    o.segment()
    for h in (g, o):
        h.voxel_map_init(scans[0]["body_full"])
    for k in range(1, len(scans)):
        ds = _oracle_raw(o, scans[k]["body_full"], cfg.filter_size_surf)
        o.predict(scans[k]["dt"])
        o.segment()
        o.lio_state_estimation(ds)
        o.map_incremental_grow(ds)
        vg.step_async_raw(g, scans[k]["body_full"], cfg.filter_size_surf, dt=scans[k]["dt"])
        sg, _ = g.wait()
        assert np.array_equal(sg, o.get_state()), f"scan {k}: state"
        assert np.array_equal(g.dump_map(), o.dump_map()), f"scan {k}: dump"
    _, st = g.local_map_state()
    assert st["moves"] > 0 and st["roots_evicted"] > 0


def test_local_map_imu_chain_matches_oracle():
    """the IMU chain (immesh_lio_step_async_imu): the box placed by the first map build (branch 2), then evaluated after UndistortPcl
    on every steady scan; the oracle chain evaluates laser_map_fov_segment at the same points (after its state is set)"""
    from imu_stream_common import OracleChain, imu_cfg, make_imu_stream, true_velocity
    n_scans, max_ini, lm = 11, 30, (2.0, 1.0, 1.5)   # cube_len < 2 mov det: the box moves on every steady scan

    class LocalMapLio(OracleLocalMap):
        def set_state(self, s):       # OracleChain sets the state right after UndistortPcl, before the build or the IESKF
            super().set_state(s)
            self.segment()

    sensor, scans = make_imu_stream(n_scans, seed=3, empty_batch=1)
    s0 = np.zeros(348)
    s0[0:9] = np.eye(3).reshape(9)
    s0[12:15] = true_velocity(sensor, scans[0]["beg"])
    for i in range(18):
        s0[24 + i * 18 + i] = 1e-7
    o = OracleChain(api.AVIA, imu_cfg(), None, max_ini, s0, api.AVIA.filter_size_surf)
    o.lio = LocalMapLio(api.AVIA)
    o.lio.local_map(*lm)
    br_o = [o.step(sc["imu"], sc["pts"], sc["beg"]) for sc in scans]
    g = api.Lio(api.AVIA)
    g.set_state(s0)
    g.local_map(*lm)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32)
    vg = api.VoxelGrid(1 << 17)
    imu_h.init_begin(max_ini)
    br_g = [vg.step_async_imu(g, imu_h, sc["imu"], sc["pts"], sc["beg"], api.AVIA.filter_size_surf) for sc in scans]
    g.wait()
    assert br_g == br_o and 2 in br_o and 3 in br_o
    assert np.array_equal(g.get_state(), o.lio.get_state())
    assert np.array_equal(g.dump_map(), o.lio.dump_map())
    box_g, st = g.local_map_state()
    assert st["placed"] == 1 and st["moves"] == br_o.count(3)
