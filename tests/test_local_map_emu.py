"""CPU tier: the local map's device bodies (immesh_b200/csrc/local_map.cuh) on the host emulation (tests/local_map/emu_local_map.cpp)
-- the box rule against a numpy float32 restatement of laser_map_fov_segment and against the extended oracle, and the eviction sweep
and the purge against the oracle's deletion from feat_map along a scan stream."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from immesh_b200 import api, build, synth
from lio_common import init_velocity
from local_map_common import SHAPE_COLS, OracleLocalMap, f32, fov_segment, in_boxes, oracle_rule, root_centres

IM_LC_NODES, IM_LC_CHUNK_BUMP, IM_LC_AVAIL_TOP, IM_LC_ROOTS, IM_LC_NODE_FREE, IM_LC_TOMBS = 0, 1, 2, 5, 13, 14


@pytest.fixture(scope="module")
def lib():
    L = api.load_library(build.build_local_map()[0])
    L.emu_lm_rule.argtypes = [C.c_double, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_lm_evict.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.emu_lm_enable.argtypes = [C.c_void_p]
    L.emu_lm_purge.argtypes = [C.c_void_p]
    L.emu_lm_table.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_lm_table.restype = C.c_longlong
    L.emu_lm_find.argtypes = [C.c_void_p, C.c_uint64]
    L.emu_lm_counter.argtypes = [C.c_void_p, C.c_int]
    L.emu_lm_root_slots.argtypes = [C.c_void_p, C.c_void_p]
    L.emu_lm_set_order.argtypes = [C.c_uint]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_rule(lib, cube_len, det, mov, placed, box, pos):
    pl = C.c_int(1 if placed else 0)
    b = np.array(box, dtype=f32)
    p = np.asarray(pos, dtype=np.float64)
    rm = np.zeros((3, 6), f32)
    k = lib.emu_lm_rule(cube_len, det, mov, C.byref(pl), _p(b), _p(p), _p(rm))
    return bool(pl.value), b, rm[:k].copy()


def _same(a, b):
    return a[0] == b[0] and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)) and np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))


def _rule_cases():
    """(cube_len, det, mov, placed, box, pos) cases: edges at exactly mov * det, both sides of one axis, several axes at once,
    cube_len <= 2 mov det, negative coordinates, and a random walk"""
    cases = []
    box = np.array([-500, -500, -500, 500, 500, 500], f32)
    thr = float(f32(1.5) * f32(300.0))
    cases.append((1000.0, 300.0, 1.5, False, np.zeros(6, f32), [1.25, -2.5, 0.75]))
    for d in (thr, np.nextafter(thr, 0), np.nextafter(thr, 1e9)):
        cases.append((1000.0, 300.0, 1.5, True, box, [500 - d, 0.0, 0.0]))     # max side of x
        cases.append((1000.0, 300.0, 1.5, True, box, [-500 + d, 0.0, 0.0]))    # min side of x
    cases.append((1000.0, 300.0, 1.5, True, box, [-60.0, 80.0, 70.0]))        # both sides in reach on every axis (min side wins)
    cases.append((1000.0, 300.0, 1.5, True, box, [460.0, -460.0, 470.0]))     # three axes at once
    cases.append((800.0, 300.0, 1.5, True, np.array([-400, -400, -400, 400, 400, 400], f32), [10.0, 0.0, 0.0]))   # cube <= 2 mov det
    cases.append((40.0, 10.0, 1.5, True, np.array([-1020.5, -35.25, -20, -980.5, 4.75, 20], f32), [-1012.3, -20.1, -7.7]))  # negative
    rng = np.random.default_rng(3)
    for _ in range(200):
        c = float(rng.choice([30.0, 60.0, 1000.0]))
        det, mov = float(rng.choice([10.0, 20.0, 300.0])), float(rng.choice([1.5, 1.2, 2.0]))
        ctr = rng.uniform(-2000, 2000, 3)
        b = np.concatenate([ctr - c / 2, ctr + c / 2]).astype(f32)
        cases.append((c, det, mov, True, b, ctr + rng.uniform(-c, c, 3)))
    return cases


def test_box_rule_matches_restatement_and_oracle(lib):
    for (c, det, mov, placed, box, pos) in _rule_cases():
        want = fov_segment(c, det, mov, placed, box, pos)
        assert _same(emu_rule(lib, c, det, mov, placed, box, pos), want), (c, det, mov, box, pos)
        assert _same(oracle_rule(c, det, mov, placed, box, pos), want), (c, det, mov, box, pos)


def test_box_rule_walk(lib):
    """a long walk that moves the box many times, state carried from evaluation to evaluation"""
    st_e = st_n = (False, np.zeros(6, f32))
    moves = 0
    for k in range(3000):
        pos = [-30.0 + 0.7 * k, 25.0 * np.sin(0.01 * k), -3.0 - 0.02 * k]
        e = emu_rule(lib, 60.0, 20.0, 1.5, st_e[0], st_e[1], pos)
        n = fov_segment(60.0, 20.0, 1.5, st_n[0], st_n[1], pos)
        assert _same(e, n), k
        moves += n[2].shape[0] > 0
        st_e, st_n = e[:2], n[:2]
    assert moves > 50


def _stream(lib, cfg, n_scans, evict_at, seed=5, purge_at=()):
    """hdl64loop stream through the emulation and the oracle; at the scans in evict_at, boxes chosen from the map (one with a root
    centre exactly on its min edge, one with a root centre exactly on its max edge) are evicted in both; dumps compared every scan"""
    sensor, scans = synth.make_stream("hdl64loop", n_scans, seed=seed, leaf=cfg.filter_size_surf, n_points=16384)
    g, o = api.Lio(cfg, lib=lib), OracleLocalMap(cfg)
    lib.emu_lm_enable(g._h)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    stats = np.zeros(3, dtype=np.int64)
    seen = dict(evicted=0, reused_nodes=False, edge_min=0, edge_max=0, layers=0)
    for k in range(1, n_scans):
        if k in evict_at:
            keys, ctr = root_centres(o.dump_map())
            t = scans[k]["t_true"]
            far = np.argsort(-np.linalg.norm(ctr - t, axis=1))
            a, b = ctr[far[0]], ctr[far[1]]
            boxes = np.array([[a[0], a[1], a[2], a[0] + 6, a[1] + 6, a[2] + 6],     # a on the min edge: evicted
                              [b[0] - 6, b[1] - 6, b[2] - 6, b[0], b[1], b[2]]],    # b on the max edge: kept (unless in the first box)
                             dtype=f32)
            if k == min(evict_at):   # and a large slab behind the sensor: whole multi-layer octrees
                boxes = np.vstack([boxes, np.array([[-1e4, -1e4, -1e4, t[0] - 15.0, 1e4, 1e4]], f32)])
            assert np.all(boxes[0, :3].astype(np.float64) == a) and np.all(boxes[1, 3:].astype(np.float64) == b)
            hit = in_boxes(ctr, boxes)
            seen["edge_min"] += int(hit[far[0]])
            seen["edge_max"] += int(not in_boxes(b[None], boxes[1:])[0])
            d0 = o.dump_map()
            ev_keys = set(map(tuple, keys[hit].tolist()))
            rows = [r for r in d0 if tuple(int(v) for v in r[0:3]) in ev_keys]
            seen["layers"] = max([seen["layers"]] + [int(r[4]) for r in rows])
            ev_o = o.evict_boxes(boxes)
            lib.emu_lm_evict(g._h, _p(boxes), boxes.shape[0], _p(stats))
            assert stats[0] == ev_o == hit.sum(), (k, stats, ev_o)
            seen["evicted"] += int(ev_o)
            assert lib.emu_lm_counter(g._h, IM_LC_ROOTS) == o.num_roots()
            assert np.array_equal(g.dump_map(), o.dump_map()), f"scan {k}: dump after the eviction"
        if k in purge_at:
            d = g.dump_map()
            lib.emu_lm_purge(g._h)
            assert lib.emu_lm_counter(g._h, IM_LC_TOMBS) == 0
            assert np.array_equal(g.dump_map(), d), "purge changed the map"
        free_before = max(lib.emu_lm_counter(g._h, IM_LC_NODE_FREE), 0)
        body = scans[k]["body_ds"]
        g.predict(scans[k]["dt"])
        o.predict(scans[k]["dt"])
        assert g.lio_state_estimation(body) == o.lio_state_estimation(body), k
        assert np.array_equal(g.matches(), o.matches()), f"scan {k}: matches"
        assert np.array_equal(g.get_state(), o.get_state()), f"scan {k}: state"
        g.map_incremental_grow()
        o.map_incremental_grow(body)
        if free_before > 0 and lib.emu_lm_counter(g._h, IM_LC_NODE_FREE) < free_before:
            seen["reused_nodes"] = True
        dg, do = g.dump_map(), o.dump_map()
        assert np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), f"scan {k}: octree shape"
        assert np.array_equal(dg, do), f"scan {k}: dump"
    assert lib.emu_lm_counter(g._h, 4) == 0   # no error flag
    return g, o, seen


def test_eviction_stream_matches_oracle(lib):
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=12, max_nodes=1 << 17, max_chunks=1 << 17)
    lib.emu_lm_set_order(11)
    g, o, seen = _stream(lib, cfg, 16, evict_at={3, 5, 8, 11, 13}, purge_at={12})
    assert seen["evicted"] > 0 and seen["edge_min"] > 0 and seen["edge_max"] > 0
    assert seen["reused_nodes"], "no node record was taken from the free stack"
    assert seen["layers"] >= 1, "no multi-layer octree was evicted"
    # the chunks freed went back through the pending list into the free stack, and were taken again
    assert lib.emu_lm_counter(g._h, IM_LC_CHUNK_BUMP) > 0


def test_tombstones_survive_lookups_and_inserts(lib):
    """a tiny table with long probe chains: after evictions every live key is still found, an evicted key is not, and re-creating it
    takes a fresh slot past the tombstones; the purge then leaves exactly the live keys, each found, and no tombstone"""
    cfg = dataclasses.replace(api.VELODYNE, hash_capacity_log2=10, max_nodes=1 << 16, max_chunks=1 << 17)
    sensor, scans = synth.make_stream("hdl64loop", 4, seed=9, leaf=cfg.filter_size_surf, n_points=8192)
    g = api.Lio(cfg, lib=lib)
    lib.emu_lm_enable(g._h)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    cap = lib.emu_lm_table(g._h, None, None)
    keys, roots = np.zeros(cap, np.uint64), np.zeros(cap, np.int32)
    lib.emu_lm_table(g._h, _p(keys), _p(roots))
    live = keys[keys != np.uint64(0xFFFFFFFFFFFFFFFF)]
    assert live.size > cap // 4
    _, ctr = root_centres(g.dump_map())
    box = np.array([[ctr[:, 0].min(), -1e4, -1e4, np.median(ctr[:, 0]), 1e4, 1e4]], f32)
    stats = np.zeros(3, dtype=np.int64)
    lib.emu_lm_evict(g._h, _p(box), 1, _p(stats))
    lib.emu_lm_table(g._h, _p(keys), _p(roots))
    tomb = keys == np.uint64(1 << 63)
    assert tomb.sum() == stats[0] == lib.emu_lm_counter(g._h, IM_LC_TOMBS) > 0
    assert np.all(roots[tomb] == -1)
    kept = keys[(keys >> np.uint64(63)) == 0]
    gone = np.setdiff1d(live, kept)
    assert gone.size == stats[0]
    for k in kept:
        s = lib.emu_lm_find(g._h, int(k))
        assert s >= 0 and keys[s] == k
    for k in gone:
        assert lib.emu_lm_find(g._h, int(k)) == -1
    # re-create the evicted roots: the same scan again
    g.voxel_map_init(scans[0]["body_full"])
    lib.emu_lm_table(g._h, _p(keys), _p(roots))
    assert (keys == np.uint64(1 << 63)).sum() == tomb.sum(), "a tombstone was claimed"
    for k in gone:
        s = lib.emu_lm_find(g._h, int(k))
        assert s >= 0 and not tomb[s]
    # purge = a fresh insert of the live keys at the same capacity
    d = g.dump_map()
    lib.emu_lm_purge(g._h)
    k2, r2 = np.zeros(cap, np.uint64), np.zeros(cap, np.int32)
    lib.emu_lm_table(g._h, _p(k2), _p(r2))
    occupied = keys[(keys >> np.uint64(63)) == 0]
    assert np.array_equal(np.sort(k2[k2 != np.uint64(0xFFFFFFFFFFFFFFFF)]), np.sort(occupied))
    assert not (k2 == np.uint64(1 << 63)).any()
    for k in occupied:
        s = lib.emu_lm_find(g._h, int(k))
        assert s >= 0 and k2[s] == k and r2[s] == roots[np.nonzero(keys == k)[0][0]]
    assert np.array_equal(g.dump_map(), d, equal_nan=True)
    rs = np.zeros(1 << 16, np.int32)
    n = lib.emu_lm_root_slots(g._h, _p(rs))
    live_nodes = set(r2[r2 >= 0].tolist())
    for s in range(cap):
        if r2[s] >= 0:
            assert rs[r2[s]] == s, "root back-pointer after the purge"
    assert n > 0 and live_nodes
