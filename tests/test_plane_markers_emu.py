"""CPU tier: the plane-marker walk (pubPlaneMap) and its pending-root bookkeeping, executed by the host emulation of the device
code, against the oracle's literal full walk; plus the oracle's rows against numpy."""
import numpy as np
import pytest

from immesh_b200 import api
from plane_markers_common import BRANCHES, emu_pub_lib, run_markers_parity


@pytest.fixture(scope="module")
def emu_lib():
    """the host emulation with the publisher's device state (tests/pubmap/emu_pub.cpp)"""
    return emu_pub_lib()


def test_avia_every_scan(emu_lib):
    r = run_markers_parity(emu_lib, "avia", api.AVIA, n_scans=12, seed=0)
    assert r["calls"] == 12
    assert all(w <= b for w, b in zip(r["walked"], r["pending_bound"]))


def test_hdl64_every_scan(emu_lib):
    r = run_markers_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=5, seed=1, n_points=32768)
    assert all(w <= b for w, b in zip(r["walked"], r["pending_bound"]))


def test_every_third_scan(emu_lib):
    # a marker call every third scan: flags accumulate between calls and children wait behind their roots' flags
    a = run_markers_parity(emu_lib, "avia", api.AVIA, n_scans=13, seed=4, every=3, repeat=2)
    b = run_markers_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=7, seed=2, n_points=16384, every=3, repeat=2)
    assert "child_held_back" in a["reached"] | b["reached"]


def test_branch_coverage(emu_lib):
    reached = set()
    reached |= run_markers_parity(emu_lib, "avia", api.AVIA, n_scans=12, seed=0)["reached"]
    reached |= run_markers_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=5, seed=1, n_points=32768)["reached"]
    reached |= run_markers_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=7, seed=2, n_points=16384, every=3, repeat=2)["reached"]
    missing = [b for b in BRANCHES if b not in reached]
    assert not missing, missing


def test_empty_map_and_count_query(emu_lib):
    import ctypes as C
    g = api.Lio(api.AVIA, lib=emu_lib)
    rows, c = g.plane_markers()
    assert rows.shape == (0, api.PLANE_MARKER_COLS) and c["roots_walked"] == 0 and c["update"] == 0
    from immesh_b200 import synth
    _, scans = synth.make_stream("avia", 2, seed=5, ext_T=api.AVIA.ext_T)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    n = C.c_int(0)
    cnt = np.zeros(5, dtype=np.int64)
    rc = emu_lib.immesh_voxelmap_plane_markers(g._h, None, 0, C.byref(n), cnt.ctypes.data_as(C.POINTER(C.c_int64)))
    # only the roots with a fit are listed (a root that has not reached its init size has never been fitted)
    assert rc == -3 and n.value > 0 and 0 < cnt[4] < g.counts()["roots"]
    rows, c = g.plane_markers()             # nothing was consumed by the count query
    assert rows.shape[0] == n.value and c["update"] == n.value
    rows, c = g.plane_markers()
    assert rows.shape[0] == 0 and c["roots_walked"] == 0
