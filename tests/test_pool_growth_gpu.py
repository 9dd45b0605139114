"""GPU tier: growth of the localization and mesh pools on the device (immesh_lio_* / immesh_mesh_* reserve, set_growth).  Handles
created just above what the first scan or frame needs run whole streams against the oracle, or side by side with handles of fixed
capacities."""
import os
import subprocess
import sys

import numpy as np
import pytest

from immesh_b200 import api
from oracle_api import OracleLio, OracleMesh
from parity_gate import pipeline_parity
from plane_markers_common import NOT_ID
from pool_growth_common import (MESH_SMALL, check_mesh, doublings, first_frame_use, first_scan_use, make_scans, mesh_doublings,
                                run_growth_parity, run_pipelined_pair, start, tiny_config, tiny_mesh_config, world_frames)

pytestmark = pytest.mark.gpu

SLOT_B, NODE_B, CHUNK_B = 32, 944, 520   # device bytes per root slot, node record, chunk (INTEGRATION.md, "Long runs")


def pool_bytes(c):
    return c["root_slots"] * SLOT_B + c["nodes_cap"] * NODE_B + c["chunks_cap"] * CHUNK_B


def test_avia_stream_from_tiny_handle(cuda_lib):
    r = run_growth_parity(cuda_lib, "avia", api.AVIA, n_scans=12, seed=0)
    d = doublings(r["first"], r["last"])
    assert all(v >= 3 for v in d.values()), d
    assert r["last"]["device_bytes"] - r["first"]["device_bytes"] == pool_bytes(r["last"]) - pool_bytes(r["first"])
    assert r["last"]["growths"] >= 3
    r["handle"].close()


def test_hdl64_stream_from_tiny_handle(cuda_lib):
    r = run_growth_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768)
    d = doublings(r["first"], r["last"])
    assert all(v >= 3 for v in d.values()), d
    r["handle"].close()


def gate_from_tiny_handles(lib, monkeypatch, n_scans=12, seed=3):
    """tests/parity_gate.py's pipelined run (step_async + push_frame_from_lio_async, graph-replayed) on handles created just above
    the first scan's use with automatic growth on; returns (report, [(class, capacity(), graph_stats) of each handle at its close])"""
    cfg = api.AVIA
    sensor, scans = make_scans("avia", cfg, n_scans + 1, seed)
    lcfg = tiny_config(cfg, first_scan_use(lib, cfg, sensor, scans))
    mcfg = tiny_mesh_config(first_frame_use(lib, world_frames(scans[:1])))
    caps = []
    Lio, Mesh = api.Lio, api.Mesh

    class GrowingLio(Lio):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.set_growth(1 << 40)

        def close(self):
            if self._h:
                caps.append(("lio", self.capacity(), api.graph_stats(self, None)))
            super().close()

    class GrowingMesh(Mesh):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.set_growth(1 << 40)

        def close(self):
            if self._h:
                caps.append(("mesh", self.capacity(), api.graph_stats(None, self)))
            super().close()
    monkeypatch.setattr(api, "Lio", GrowingLio)
    monkeypatch.setattr(api, "Mesh", GrowingMesh)
    try:
        rep = pipeline_parity(lib, lcfg, mcfg, scans, n_scans)
    finally:
        monkeypatch.undo()
    return rep, caps


def test_pipelined_from_tiny_handles(cuda_lib, monkeypatch):
    rep, caps = gate_from_tiny_handles(cuda_lib, monkeypatch)
    assert rep["ok"], rep
    (_, lc, lg), (_, mc, mg) = caps
    assert lc["growths"] >= 2 and mc["growths"] >= 2, caps
    assert lg["lio_captures"] >= 2 and mg["mesh_captures"] >= 2, caps   # every growth drops the captured sequence: captured again


_NO_GRAPH = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import pytest
from immesh_b200 import api
from test_pool_growth_gpu import gate_from_tiny_handles
rep, caps = gate_from_tiny_handles(api.load_library(), pytest.MonkeyPatch(), n_scans=10, seed=4)
assert rep["ok"], rep
assert caps[0][1]["growths"] >= 2 and caps[1][1]["growths"] >= 2, caps
assert caps[0][2]["lio_captures"] == 0 and caps[1][2]["mesh_captures"] == 0, caps
print("ok")
"""


def test_pipelined_from_tiny_handles_without_graphs():
    tests = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, IMMESH_GRAPH="0")
    p = subprocess.run([sys.executable, "-c", _NO_GRAPH.format(root=os.path.dirname(tests), tests=tests)], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stdout + p.stderr


def test_lio_pipeline_against_default_handle(cuda_lib):
    g, d = run_pipelined_pair(cuda_lib, "avia", api.AVIA, n_scans=16, seed=3)
    assert g.capacity()["growths"] >= 2
    g.close(); d.close()


def test_explicit_reserve_between_scans(cuda_lib):
    def before(g, k):
        c = g.capacity()
        f = (4, 0, 1)[k % 3]   # x4, a no-op request, +1 record, in turn
        if f == 0:
            g.reserve(c["root_slots"], c["nodes_cap"], c["chunks_cap"])
        elif f == 1:
            g.reserve(c["root_slots"] + 1, c["nodes_cap"] + 1, c["chunks_cap"] + 1)
        else:
            g.reserve(c["root_slots"] * 4, c["nodes_cap"] * 4, c["chunks_cap"] * 4)
    r = run_growth_parity(cuda_lib, "avia", api.AVIA, n_scans=9, seed=2, growth=0, before_scan=before)
    r["handle"].close()


def test_growth_off_keeps_todays_overflow(cuda_lib):
    cfg = api.AVIA
    sensor, scans = make_scans("avia", cfg, 12, 0)
    g = api.Lio(tiny_config(cfg, first_scan_use(cuda_lib, cfg, sensor, scans)), lib=cuda_lib)
    first = g.capacity()
    start(g, sensor, scans)
    g.voxel_map_init(scans[0]["body_full"])
    with pytest.raises(RuntimeError) as e:
        for k in range(1, 12):
            g.step(scans[k]["body_ds"], dt=scans[k]["dt"])
    assert "code -3" in str(e.value) and "device pool overflow (raise the capacities in immesh_lio_config)" in str(e.value)
    last = g.capacity()
    assert all(last[k] == first[k] for k in ("root_slots", "nodes_cap", "chunks_cap", "device_bytes", "growths"))
    g.close()


def test_ceiling_refuses_and_leaves_the_handle(cuda_lib):
    cfg = api.AVIA
    sensor, scans = make_scans("avia", cfg, 6, 0)
    g = api.Lio(tiny_config(cfg, first_scan_use(cuda_lib, cfg, sensor, scans)), lib=cuda_lib)
    start(g, sensor, scans)
    g.set_growth(g.capacity()["device_bytes"] + 1)
    before = g.capacity()
    with pytest.raises(RuntimeError) as e:
        g.voxel_map_init(scans[0]["body_full"])
    msg = str(e.value)
    assert "code -3" in msg and "ceiling" in msg and ("root hash" in msg or "node pool" in msg or "chunk pool" in msg), msg
    assert g.capacity() == before
    assert g.counts() == dict(roots=0, nodes=0, chunks=0, err=0)
    g.close()


def test_impossible_reserve_is_refused(cuda_lib):
    def before(g, k):
        if k == 3:
            c = g.capacity()
            for args, pool in (((1 << 31, 0, 0), "root hash"), ((0, 1 << 31, 0), "node pool"), ((0, 0, 1 << 31), "chunk pool")):
                with pytest.raises(RuntimeError) as e:
                    g.reserve(*args)
                assert "code -3" in str(e.value) and pool in str(e.value)
            assert g.capacity() == c
    r = run_growth_parity(cuda_lib, "avia", api.AVIA, n_scans=6, seed=5, before_scan=before)
    r["handle"].close()


def test_growth_and_sharding_exclude_each_other(cuda_lib):
    g = api.Lio(api.AVIA, lib=cuda_lib)
    g.set_growth(1 << 40)
    with pytest.raises(RuntimeError) as e:
        g.shard(0, 2, b"\0" * 128)
    assert "code -1" in str(e.value)
    g.close()


def test_publishers_read_the_migrated_map(cuda_lib):
    # plane markers and the two scan publishers of a grown handle equal those of a default-sized handle fed the same scans
    cfg = api.AVIA
    sensor, scans = make_scans("avia", cfg, 10, 6)
    g = api.Lio(tiny_config(cfg, first_scan_use(cuda_lib, cfg, sensor, scans)), lib=cuda_lib)
    d = api.Lio(cfg, lib=cuda_lib)
    g.set_growth(1 << 40)
    for h in (g, d):
        start(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    for k in range(1, 10):
        for h in (g, d):
            h.step(scans[k]["body_ds"], dt=scans[k]["dt"])
        (rg, cg), (rd, cd) = g.plane_markers(), d.plane_markers()
        assert np.array_equal(rg[:, NOT_ID], rd[:, NOT_ID]) and cg == cd, f"scan {k}: plane markers"
        (eg, ig), (ed, idd) = g.effect_cloud(), d.effect_cloud()
        assert np.array_equal(eg, ed) and np.array_equal(ig, idd), f"scan {k}: effect cloud"
        assert np.array_equal(g.registered_cloud(), d.registered_cloud()), f"scan {k}: registered cloud"
    assert g.capacity()["growths"] >= 2
    g.close(); d.close()


def test_long_stream_side_by_side(cuda_lib):
    # hdl64loop at reduced points per scan: a growing handle pair (localization + mesh) and a default-sized pair agree after every
    # scan; the first 20 scans are also checked against the oracle
    cfg = api.VELODYNE
    n = 200
    sensor, scans = make_scans("hdl64loop", cfg, n, 8, n_points=16384)
    g = api.Lio(tiny_config(cfg, first_scan_use(cuda_lib, cfg, sensor, scans)), lib=cuda_lib)
    d = api.Lio(cfg, lib=cuda_lib)
    gm = api.Mesh(tiny_mesh_config(first_frame_use(cuda_lib, world_frames(scans[:1]))), lib=cuda_lib)
    dm = api.Mesh(api.MeshConfig(**{**MESH_SMALL, "max_vertices": 1 << 22, "max_triangles": 1 << 24, "max_voxels": 1 << 20}), lib=cuda_lib)
    o = OracleLio(cfg, sum_mode=0)
    g.set_growth(1 << 40)
    gm.set_growth(1 << 40)
    for h in (g, d, o):
        start(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    growths, mgrowths = 0, 0
    for k in range(1, n):
        (sg, ig), (sd, idd) = (h.step(scans[k]["body_ds"], dt=scans[k]["dt"]) for h in (g, d))
        assert ig == idd and np.array_equal(sg, sd), f"scan {k}: state"
        if k <= 20:
            o.predict(scans[k]["dt"])
            io = o.lio_state_estimation(scans[k]["body_ds"])
            o.map_incremental_grow(scans[k]["body_ds"])
            assert ig == io and np.array_equal(sg, o.get_state()), f"scan {k}: state against the oracle"
            if k == 20:
                assert np.array_equal(g.dump_map(), o.dump_map()), "map dump against the oracle"
        for m, h in ((gm, g), (dm, d)):
            m.push_frame_from_lio(h, scans[k]["body_full"])
        c = g.capacity()
        if c["growths"] != growths:
            growths = c["growths"]
            assert c["roots"] * 2 <= c["root_slots"], f"scan {k}: load factor {c['roots'] / c['root_slots']}"
        mgrowths = gm.capacity()["growths"]
        if k % 50 == 0 or k == n - 1:
            assert np.array_equal(g.dump_map(), d.dump_map()), f"scan {k}: map dump"
            check_mesh(gm, dm, f"scan {k}: mesh")
    assert growths >= 3 and mgrowths >= 3 and g.counts()["err"] == 0
    for h in (g, d, gm, dm):
        h.close()


def test_no_device_memory_left_behind(cuda_lib):
    import torch
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    r = run_growth_parity(cuda_lib, "avia", api.AVIA, n_scans=6, seed=7)
    assert r["last"]["growths"] >= 2
    r["handle"].close()
    del r
    assert torch.cuda.mem_get_info()[0] == free0


# ---- the mesh handle
@pytest.mark.parametrize("kind,n_frames,n_points", [("avia", 8, None), ("hdl64", 4, 32768)])
def test_mesh_stream_from_tiny_handle(cuda_lib, kind, n_frames, n_points):
    sensor, scans = make_scans(kind, api.AVIA, n_frames, 0, n_points)
    frames = world_frames(scans)
    g = api.Mesh(tiny_mesh_config(first_frame_use(cuda_lib, frames)), lib=cuda_lib)
    o = OracleMesh(api.MeshConfig(**MESH_SMALL))
    g.set_growth(1 << 40)
    first = g.capacity()
    for k, (w, t) in enumerate(frames):
        g.push_frame(w, t, k)
        o.push_frame(w, t, k)
        check_mesh(g, o, f"frame {k}")
    last = g.capacity()
    d = mesh_doublings(first, last)
    assert last["growths"] >= 3 and all(v >= 1 for v in d.values()), d
    g.close()


def grown_and_presized(lib, n_frames=8, seed=5):
    sensor, scans = make_scans("avia", api.AVIA, n_frames, seed)
    frames = world_frames(scans)
    g = api.Mesh(tiny_mesh_config(first_frame_use(lib, frames)), lib=lib)
    d = api.Mesh(api.MeshConfig(**MESH_SMALL), lib=lib)
    g.set_growth(1 << 40)
    for k, (w, t) in enumerate(frames):
        for h in (g, d):
            h.push_frame(w, t, k)
    assert g.capacity()["growths"] >= 3
    check_mesh(g, d, "after the frames")
    return g, d, frames


def test_mesh_outputs_after_growth(cuda_lib):
    # the calls that read the migrated store return what a pre-sized handle fed the same frames returns
    g, d, frames = grown_and_presized(cuda_lib)
    q = frames[-1][0][::97]
    ig, dg = g.knn(q, 8)
    idd, dd = d.knn(q, 8)
    assert np.array_equal(ig, idd) and np.array_equal(dg, dd), "knn"
    rg, rd = g.region_buffers(region_size=5.0), d.region_buffers(region_size=5.0)
    assert all(np.array_equal(a, b) for a, b in zip(rg, rd)), "region buffers"
    # a vertex without a neighbour inside the limit divides by zero on both sides (NaN, the reference's value)
    assert np.array_equal(g.smooth_all(0.5, 10), d.smooth_all(0.5, 10), equal_nan=True), "smooth_all"
    rs = [h.region_stream(region_size=5.0) for h in (g, d)]
    assert all(np.array_equal(a, b) for a, b in zip(*rs)), "region stream"
    g.close(); d.close()


def test_mesh_batched_frame_after_growth(cuda_lib):
    # a batched offline frame of a whole cloud on a small handle with growth on (grown before the frame) equals the same frame on a
    # pre-sized handle; a second batched frame then runs on the scratch allocated again at the grown sizes
    sensor, scans = make_scans("avia", api.AVIA, 4, 6)
    frames = world_frames(scans)
    cloud = np.concatenate([w for w, _ in frames])
    pose = frames[-1][1]
    g = api.Mesh(tiny_mesh_config(first_frame_use(cuda_lib, frames)), lib=cuda_lib)
    d = api.Mesh(api.MeshConfig(**MESH_SMALL), lib=cuda_lib)
    g.set_growth(1 << 40)
    for h in (g, d):
        h.push_frame_batched(frames[0][0], frames[0][1], batch_points=1 << 13, batch_voxels=1 << 9)
        h.push_frame_batched(cloud, pose, batch_points=1 << 15, batch_voxels=1 << 10)
    assert g.capacity()["growths"] >= 1
    check_mesh(g, d, "batched frames")
    g.close(); d.close()


def test_mesh_growth_off_ceiling_and_limits(cuda_lib):
    sensor, scans = make_scans("avia", api.AVIA, 6, 0)
    frames = world_frames(scans)
    tiny = tiny_mesh_config(first_frame_use(cuda_lib, frames))
    g = api.Mesh(tiny, lib=cuda_lib)   # growth off: today's overflow
    first = g.capacity()
    with pytest.raises(RuntimeError) as e:
        for k, (w, t) in enumerate(frames):
            g.push_frame(w, t, k)
    assert "code -3" in str(e.value) and "mesh pool / per-voxel working-set overflow" in str(e.value)
    assert all(g.capacity()[k] == first[k] for k in ("vertices_cap", "triangles_cap", "voxels_cap", "device_bytes", "growths"))
    g.close()
    h = api.Mesh(tiny, lib=cuda_lib)
    h.push_frame(frames[0][0], frames[0][1], 0)
    h.set_growth(h.capacity()["device_bytes"] + 1)   # the ceiling
    before = h.capacity()
    with pytest.raises(RuntimeError) as e:
        h.push_frame(frames[1][0], frames[1][1], 1)
    msg = str(e.value)
    assert "code -3" in msg and "ceiling" in msg and ("vertex pool" in msg or "triangle pool" in msg or "voxel hash" in msg), msg
    assert h.capacity() == before
    for args, pool in (((1 << 31, 0, 0), "vertex pool"), ((0, 1 << 31, 0), "triangle pool"), ((0, 0, 1 << 31), "voxel hash")):
        with pytest.raises(RuntimeError) as e:
            h.reserve(*args)
        assert "code -3" in str(e.value) and pool in str(e.value)
    assert h.capacity() == before
    h.set_growth(1 << 40)   # and the handle carries on, equal to the oracle
    o = OracleMesh(api.MeshConfig(**MESH_SMALL))
    o.push_frame(frames[0][0], frames[0][1], 0)
    for k in (1, 2):
        h.push_frame(frames[k][0], frames[k][1], k)
        o.push_frame(frames[k][0], frames[k][1], k)
        check_mesh(h, o, f"frame {k}")
    with pytest.raises(RuntimeError) as e:
        h.shard(0, 2, b"\0" * 128)
    assert "code -1" in str(e.value)
    h.close()


def test_mesh_explicit_reserve_between_frames(cuda_lib):
    sensor, scans = make_scans("avia", api.AVIA, 8, 2)
    frames = world_frames(scans)
    g = api.Mesh(tiny_mesh_config(first_frame_use(cuda_lib, frames)), lib=cuda_lib)
    o = OracleMesh(api.MeshConfig(**MESH_SMALL))
    keys = ("vertices_cap", "triangles_cap", "voxels_cap")
    for k, (w, t) in enumerate(frames):
        c = g.capacity()
        f = (4, 0, 1)[k % 3]   # x4, a no-op request, +1 record, in turn
        g.reserve(*[c[x] * 4 if f == 4 else c[x] + f for x in keys])
        g.push_frame(w, t, k)
        o.push_frame(w, t, k)
        check_mesh(g, o, f"frame {k}")
    g.close()


def test_mesh_no_device_memory_left_behind(cuda_lib):
    import torch
    torch.cuda.init()
    free0 = torch.cuda.mem_get_info()[0]
    g, d, _ = grown_and_presized(cuda_lib, n_frames=5, seed=7)
    c = g.capacity()
    g.close(); d.close()
    del g, d
    assert c["growths"] >= 3
    assert torch.cuda.mem_get_info()[0] == free0
