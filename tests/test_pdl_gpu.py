"""GPU tier: the graph-replayed scan and mesh-frame sequences, whose kernel boundaries are programmatic dependent launches, give
bit for bit what the same sequences give launched kernel by kernel without the attribute (IMMESH_GRAPH=0): the state, the VoxelMap
dump and the mesh snapshot along a 100k-point Avia-shape stream, a closed-loop HDL-64 stream and the raw front-end chain."""
import numpy as np
import pytest

import bench
from immesh_b200 import api

pytestmark = pytest.mark.gpu

_STREAMS = {}


def stream(config, n):
    if (config, n) not in _STREAMS:
        _STREAMS[(config, n)] = bench.get_stream(bench.workloads()[config], n)
    return _STREAMS[(config, n)]


def run_pipelined(lib, config, n_scans, raw=False):
    """n_scans pipelined scans (queued without a wait, read back every 10); returns the states read, the map, the mesh, graph stats"""
    wl = bench.workloads()[config]
    scans = stream(config, n_scans + 1)
    lio, mesh = api.Lio(wl["lio"], lib=lib), api.Mesh(wl["mesh"], lib=lib)
    vg = api.VoxelGrid(max(s["body_full"].shape[0] for s in scans) + 1024, lib=lib) if raw else None
    lio.set_state(bench.init_state_vec(scans))
    lio.voxel_map_init(scans[0]["body_full"])
    states = []
    for k in range(1, n_scans + 1):
        sc = scans[k]
        if raw:
            vg.step_async_raw(lio, sc["body_full"], wl["lio"].filter_size_surf, dt=sc["dt"], calib_laser=bool(wl["lio"].calib_laser))
            mesh.push_frame_from_lio_async(lio, vg.input_points(), sc["body_full"].shape[0], on_device=True)
        else:
            lio.step_async(sc["body_ds"], dt=sc["dt"])
            mesh.push_frame_from_lio_async(lio, sc["body_full"])
        if k % 10 == 0 or k == n_scans:
            s, it = lio.wait()
            mesh.wait()
            states.append((s.copy(), it))
    out = dict(states=states, map=lio.dump_map(), mesh=mesh.snapshot(), stats=api.graph_stats(lio, mesh))
    if vg is not None:
        vg.close()
    lio.close()
    mesh.close()
    return out


def assert_same(a, b):
    assert len(a["states"]) == len(b["states"])
    for (sa, ia), (sb, ib) in zip(a["states"], b["states"]):
        assert ia == ib and np.array_equal(sa, sb)
    assert np.array_equal(a["map"], b["map"])
    for x, y in zip(a["mesh"], b["mesh"]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("config,n_scans,raw", [("C100k", 60, False), ("C4", 20, False), ("C100k", 20, True)],
                         ids=["avia100k", "hdl64loop", "avia100k_raw"])
def test_programmatic_launches_equal_direct_launches(cuda_lib, monkeypatch, config, n_scans, raw):
    pdl = run_pipelined(cuda_lib, config, n_scans, raw)
    st = pdl["stats"]
    assert st["lio_replays"] > 0 and st["mesh_replays"] > 0 and st["lio_failures"] == 0 and st["mesh_failures"] == 0, st
    assert st["lio_pdl_edges"] > 0 and st["mesh_pdl_edges"] > 0, st
    monkeypatch.setenv("IMMESH_GRAPH", "0")    # read when a handle is created
    direct = run_pipelined(cuda_lib, config, n_scans, raw)
    assert direct["stats"]["lio_captures"] == 0 and direct["stats"]["lio_pdl_edges"] == 0, direct["stats"]
    assert_same(pdl, direct)


def test_graph_pdl_edges_count(cuda_lib):
    """one scan: every kernel after k_predict (16 edges at 4 IESKF iterations); one frame: the 14 kernels of the non-sharded frame
    that follow a kernel on the same stream, outside the triangulation's fork and join"""
    st = run_pipelined(cuda_lib, "C100k", 3)["stats"]
    assert st["lio_pdl_edges"] == 2 + 2 * bench.workloads()["C100k"]["lio"].max_iteration + 6, st
    assert st["mesh_pdl_edges"] == 14, st
