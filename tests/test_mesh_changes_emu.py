"""CPU tier: the mesh's change feed (immesh_mesh_changes) with its shipped bodies (mesh_changes.cuh, chg_touch in apply_face) run in
the device's order on the mesher emulation (tests/changes/emu_changes.cpp).  A mirror fed only the rows equals the oracle's live set,
flips and vertices after every frame; the branches (a pre-frame triangle removed, a kept one re-oriented, a triple revived) are
reached; ring, header and per-frame-list losses follow their arithmetic; a batched frame gives the single frame's rows."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api
from mesh_changes_common import Mirror, code_of
from mesh_common import SMALL, world_scans
from offline_batched_common import avia_cloud, new_config
from oracle_api import OracleMesh

E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    return api.load_library(build.build_changes())


def stream(lib, kind, n, seed, max_rows=1 << 20, max_frames=64):
    cfg = api.MeshConfig(**SMALL)
    g, o = api.Mesh(cfg, lib=lib), OracleMesh(cfg)
    g.changes_enable(max_rows, max_frames)
    return g, o, Mirror(g), world_scans(kind, n, seed)


@pytest.mark.parametrize("kind,n", [("avia", 8), ("hdl64", 5)])
def test_mirror_equals_the_oracle(lib, kind, n):
    g, o, m, scans = stream(lib, kind, n, seed=3)
    seen, removed_before = set(), set()
    revived = pre_removed = 0
    for k, (w, t) in enumerate(scans):
        before = set(m.tri)
        g.push_frame(w, t, k)
        o.push_frame(w, t, k)
        ch = g.changes(m.newest)
        for a, b, c, code in ch["rows"].tolist():
            key = (a, b, c)
            if code == 0:
                pre_removed += key in before
                removed_before.add(key)
            elif code in (2, 3) and key in removed_before:
                revived += 1
        m.apply(ch)
        m.check_state(*o.snapshot(), f"{kind} frame {k}")
        seen |= set(m.tri)
    assert pre_removed > 0, "no pre-frame triangle was removed"
    assert m.codes[4] + m.codes[5] > 0, "no kept triangle was re-oriented"
    if kind == "avia":
        assert revived > 0, "no removed triple was made live again"


def test_empty_frame(lib):
    g, o, m, scans = stream(lib, "avia", 1, seed=5)
    g.push_frame(*scans[0], 0)
    g.push_frame(np.zeros((0, 3), np.float32), scans[0][1], 1)
    ch = g.changes(0)
    assert ch["frames"].tolist()[1][1:] == [ch["frames"][0, 2], ch["frames"][0, 2], len(ch["rows"])]
    m.apply(ch)
    m.check(g)


def test_touched_list_overflow_falls_back_to_the_sweep_and_ring_losses(lib):
    """max_rows below a frame's touched triangles: that frame is lost (its per-frame list overflowed; the sweep keeps the published
    bytes right), the push succeeds and the mesh is untouched; a resync reads the next frames exactly; two frames that fit alone
    but not together overwrite the older one's rows; max_frames wraps"""
    probe, o, pm, scans = stream(lib, "avia", 6, seed=7)
    sizes = []
    for k, (w, t) in enumerate(scans):
        probe.push_frame(w, t, k)
        sizes.append(len(probe.changes(k)["rows"]))
    ring = sizes[2]
    assert sizes[1] + sizes[2] > ring and max(sizes[3:]) > ring, sizes
    g, _, m, _ = stream(lib, "avia", 0, seed=7, max_rows=ring, max_frames=3)
    g.push_frame(*scans[0], 0)
    m.sync(g)
    m.check(g, "frame 0")
    g.push_frame(*scans[1], 1)
    g.push_frame(*scans[2], 2)
    with pytest.raises(RuntimeError) as e:   # frame 3's rows overwrote those of frame 2
        g.changes(1)
    assert code_of(e) == E_RANGE
    m = Mirror(g)
    lost = 0
    for k in (3, 4, 5):
        g.push_frame(*scans[k], k)
        if sizes[k] > ring:   # more touched triangles than the per-frame list holds: the sweep, the frame lost
            with pytest.raises(RuntimeError) as e:
                g.changes(m.newest)
            assert code_of(e) == E_RANGE
            m = Mirror(g)
            lost += 1
        else:
            m.sync(g)
            m.check(g, f"frame {k}")
    assert lost
    with pytest.raises(RuntimeError) as e:   # four frames back: beyond max_frames = 3
        g.changes(2)
    assert code_of(e) == E_RANGE
    assert g.counts() == probe.counts()
    for a, b in zip(g.snapshot(), probe.snapshot()):
        assert np.array_equal(a, b)


def test_count_query_and_contract(lib):
    g, _, m, scans = stream(lib, "avia", 3, seed=9)
    counts = np.zeros(4, np.int64)
    cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
    assert lib.immesh_mesh_changes(g._h, 0, None, 0, None, 0, None, 0, cp) == 0 and counts.tolist() == [0, 0, 0, 0]
    assert lib.immesh_mesh_changes(g._h, 1, None, 0, None, 0, None, 0, cp) == E_INVALID
    g.push_frame(*scans[0], 0)
    assert lib.immesh_mesh_changes(g._h, 0, None, 0, None, 0, None, 0, cp) == E_CAPACITY
    assert counts[0] == 1 and counts[1] > 0 and counts[2] > 0 and counts[3] == 1
    assert lib.immesh_mesh_changes(g._h, -1, None, 0, None, 0, None, 0, cp) == E_RANGE and counts[3] == 1
    assert lib.immesh_mesh_changes_enable(g._h, 8, 0) == E_INVALID
    g.changes_disable()
    assert lib.immesh_mesh_changes(g._h, 1, None, 0, None, 0, None, 0, cp) == E_INVALID


def test_batched_rows_equal_the_single_frame(lib):
    """the batched scenes: the same cloud after two frames as one push_frame and as push_frame_batched in many chunks / batches"""
    cfg = new_config()
    scans = world_scans("avia", 2, seed=11, n_points=30000)
    cloud = avia_cloud(3)
    rows = []
    for batched in (False, True):
        g = api.Mesh(cfg, lib=lib)
        g.changes_enable(1 << 21, 16)
        m = Mirror(g)
        for k, (w, _) in enumerate(scans):
            g.push_frame(w, np.zeros(3), k)
        if batched:
            st = g.push_frame_batched(cloud, np.zeros(3), len(cloud) // 9, 150)
            assert st["append_chunks"] >= 9 and st["voxel_batches"] >= 2, st
        else:
            g.push_frame(cloud, np.zeros(3), 2)
        m.sync(g)
        m.check(g, "batched" if batched else "single frame")
        rows.append(m.rows)
    assert rows[0].keys() == rows[1].keys()
    for f in rows[0]:
        assert np.array_equal(rows[0][f], rows[1][f]), f"frame {f}"
    assert len(rows[0][3]) > 1000
