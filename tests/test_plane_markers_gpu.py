"""GPU tier: immesh_voxelmap_plane_markers (pubPlaneMap on the device-resident VoxelMap) through the C ABI against the oracle's
full walk, on the staged calls, the pipelined graph-replayed step and direct launches; the capacity contract; the empty map;
the roots walked per call."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from plane_markers_common import BRANCHES, ID, NOT_ID, run_markers_parity

pytestmark = pytest.mark.gpu


def test_avia_staged(cuda_lib):
    r = run_markers_parity(cuda_lib, "avia", api.AVIA, n_scans=12, seed=0)
    assert all(w <= b for w, b in zip(r["walked"], r["pending_bound"]))
    # on a steady stream the call visits far fewer roots than the map holds
    assert all(w < 0.5 * n for w, n in zip(r["walked"][3:], r["roots"][3:]))


def test_hdl64_staged_and_every_third(cuda_lib):
    reached = set()
    reached |= run_markers_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=5, seed=1, n_points=32768)["reached"]
    reached |= run_markers_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=7, seed=2, n_points=16384, every=3, repeat=2)["reached"]
    reached |= run_markers_parity(cuda_lib, "avia", api.AVIA, n_scans=13, seed=4, every=3, repeat=2)["reached"]
    reached |= run_markers_parity(cuda_lib, "avia", api.AVIA, n_scans=12, seed=0)["reached"]
    missing = [b for b in BRANCHES if b not in reached]
    assert not missing, missing


def test_pipelined_graph_path(cuda_lib):
    run_markers_parity(cuda_lib, "avia", api.AVIA, n_scans=10, seed=6, mode="async", oracle_checks=False)
    run_markers_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=5, seed=1, n_points=32768, mode="async", every=2, oracle_checks=False)


def test_pipelined_direct_launches(cuda_lib, monkeypatch):
    monkeypatch.setenv("IMMESH_GRAPH", "0")    # read when a handle is created
    run_markers_parity(cuda_lib, "avia", api.AVIA, n_scans=8, seed=7, mode="async", oracle_checks=False)


def test_capacity_contract_and_empty_map(cuda_lib):
    g = api.Lio(api.AVIA, lib=cuda_lib)
    rows, c = g.plane_markers()
    assert rows.shape == (0, api.PLANE_MARKER_COLS) and c["roots_walked"] == 0
    _, scans = synth.make_stream("avia", 2, seed=5, ext_T=api.AVIA.ext_T)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    n = C.c_int(0)
    cnt = np.zeros(5, dtype=np.int64)
    small = np.zeros((4, api.PLANE_MARKER_COLS))
    for cap, buf in ((0, None), (4, small.ctypes.data_as(C.POINTER(C.c_double)))):
        rc = cuda_lib.immesh_voxelmap_plane_markers(g._h, buf, cap, C.byref(n), cnt.ctypes.data_as(C.POINTER(C.c_int64)))
        assert rc == -3 and n.value > 4
    need = n.value
    a, ca = g.plane_markers(cap=need)          # nothing was consumed by the refused calls
    assert a.shape[0] == need and ca["update"] == need
    assert np.unique(a[:, ID]).size == need
    b, cb = g.plane_markers()
    assert b.shape[0] == 0 and cb["roots_walked"] == 0
    # the same rows as a handle that never saw a refused call
    h = api.Lio(api.AVIA, lib=cuda_lib)
    h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    h.voxel_map_init(scans[0]["body_full"])
    r2, _ = h.plane_markers()
    assert np.array_equal(a[:, NOT_ID], r2[:, NOT_ID])
