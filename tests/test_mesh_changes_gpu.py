"""GPU tier: the mesh's change feed (immesh_mesh_changes_enable / immesh_mesh_changes).  A mirror built from snapshot() at enable and
fed only the rows must equal snapshot() after every frame -- the sorted triples, the flips and the vertex floats bit for bit -- on the
per-frame, graph-replayed, graph-off, batched and offline paths, through pool growth, beside the reinforcement, across ring and header
wraps with the resync, and after disable / re-enable; the feed never changes what the mesher computes."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api, synth
from mesh_changes_common import Mirror, code_of
from mesh_common import SMALL, world_scans
from offline_batched_common import avia_cloud, new_config

pytestmark = pytest.mark.gpu
E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5


def lio_stream(lib, n_scans=8, seed=3, feed=True, read_every=1, reinforce=False):
    """the graph-replayed chain: localization step + push_frame_from_lio_async; the mirror read every read_every frames"""
    from lio_common import init_velocity
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", n_scans, seed=seed, ext_T=cfg.ext_T)
    lio, mesh = api.Lio(cfg, lib=lib), api.Mesh(api.MeshConfig(**SMALL), lib=lib)
    lio.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(lio, sensor, scans)
    lio.voxel_map_init(scans[0]["body_full"])
    if reinforce:
        mesh.reinforce_enable()
    m = None
    if feed:
        mesh.changes_enable(1 << 20, 64)
        m = Mirror(mesh)
    clouds = []
    for k in range(1, n_scans):
        lio.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        mesh.push_frame_from_lio_async(lio, scans[k]["body_full"])
        if reinforce:
            d, p, x, R, t = mesh.reinforced_cloud()
            clouds.append((d, p, x, R, t))
        if feed and (k % read_every == 0 or k == n_scans - 1):
            m.sync(mesh)
            m.check(mesh, f"scan {k}")
    lio.wait()
    mesh.wait()
    return lio, mesh, m, clouds


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_push_frame_stream(cuda_lib, kind):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.changes_enable(1 << 20, 64)
    m = Mirror(mesh)
    for k, (w, t) in enumerate(world_scans(kind, 6, seed=5)):
        mesh.push_frame(w, t, k)
        m.sync(mesh)
        m.check(mesh, f"{kind} frame {k}")
    assert m.codes[0] > 0 and m.codes[2] + m.codes[3] > 0, m.codes


def test_graph_replayed_chain_and_graph_off(cuda_lib, monkeypatch):
    """read after every frame and after three queued frames, with graphs and with IMMESH_GRAPH=0: the same rows"""
    _, mesh, m1, _ = lio_stream(cuda_lib)
    stats = np.zeros(6, np.int64)
    cuda_lib.immesh_graph_stats(None, mesh._h, stats.ctypes.data_as(C.POINTER(C.c_int64)))
    assert stats[4] > 0, "the frames were not graph-replayed"
    _, _, m3, _ = lio_stream(cuda_lib, read_every=3)
    monkeypatch.setenv("IMMESH_GRAPH", "0")
    _, _, m0, _ = lio_stream(cuda_lib)
    for m in (m3, m0):
        assert m1.rows.keys() == m.rows.keys()
        for f in m1.rows:
            assert np.array_equal(m1.rows[f], m.rows[f]), f"frame {f}"


def test_enable_on_a_non_empty_mesh_disable_and_reenable(cuda_lib):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    scans = world_scans("avia", 9, seed=7)
    for k, (w, t) in enumerate(scans[:3]):
        mesh.push_frame(w, t, k)
    mesh.changes_enable(1 << 20, 64)
    m = Mirror(mesh)
    assert len(m.tri) > 0
    for k, (w, t) in enumerate(scans[3:6]):
        mesh.push_frame(w, t, 3 + k)
        m.sync(mesh)
        m.check(mesh, f"frame {3 + k}")
    mesh.changes_disable()
    with pytest.raises(RuntimeError) as e:
        mesh.changes(m.newest)
    assert code_of(e) == E_INVALID
    mesh.push_frame(*scans[6], 6)
    mesh.changes_enable(1 << 18, 8)
    m = Mirror(mesh)
    for k, (w, t) in enumerate(scans[7:]):
        mesh.push_frame(w, t, 7 + k)
        m.sync(mesh)
        m.check(mesh, f"re-enabled, frame {7 + k}")


def test_batched_and_offline_rows_equal_push_frame(cuda_lib):
    """the same points as one push_frame, one push_frame_batched in many chunks / batches and one reconstruct_from_pointcloud_batched
    (passed through: every raw point goes into the frame), after two ordinary frames: the same rows"""
    cfg = new_config()
    scans = world_scans("avia", 2, seed=9, n_points=30000)
    cloud = avia_cloud(3)
    assert len(cloud) <= cfg.max_frame_points
    out = []
    for mode in ("frame", "batched", "offline"):
        mesh = api.Mesh(cfg, lib=cuda_lib)
        mesh.changes_enable(1 << 21, 16)
        m = Mirror(mesh)
        for k, (w, _) in enumerate(scans):
            mesh.push_frame(w, np.zeros(3), k)
        if mode == "frame":
            mesh.push_frame(cloud, np.zeros(3), 2)
        elif mode == "batched":
            st = mesh.push_frame_batched(cloud, np.zeros(3), len(cloud) // 7, 200)
            assert st["append_chunks"] >= 7 and st["voxel_batches"] >= 2, st
        else:
            vg = api.VoxelGrid(lib=cuda_lib)
            assert mesh.reconstruct_from_pointcloud_batched(vg, cloud, 0.01, len(cloud) // 5, 300) == len(cloud)
        m.sync(mesh)
        m.check(mesh, mode)
        out.append(m.rows)
    for rows in out[1:]:
        assert rows.keys() == out[0].keys()
        for f in rows:
            assert np.array_equal(rows[f], out[0][f]), f"frame {f}"
    assert len(out[0][3]) > 1000


def test_pool_growth_and_reserve(cuda_lib):
    cfg = api.MeshConfig(**{**SMALL, "max_vertices": 4096, "max_triangles": 4096, "max_voxels": 2048})
    mesh = api.Mesh(cfg, lib=cuda_lib)
    mesh.set_growth(8 << 30)
    mesh.changes_enable(1 << 20, 64)
    m = Mirror(mesh)
    for k, (w, t) in enumerate(world_scans("avia", 6, seed=11)):
        if k == 3:
            cap = mesh.capacity()
            mesh.reserve(cap["vertices_cap"] * 2, cap["triangles_cap"] * 2, cap["voxels_cap"] * 2)
        mesh.push_frame(w, t, k)
        m.sync(mesh)
        m.check(mesh, f"frame {k}")
    assert mesh.capacity()["growths"] >= 2


def test_with_the_reinforcement_and_outputs_unchanged(cuda_lib):
    """feed on beside the reinforcement: the mirror holds, and the state, mesh and reinforced clouds equal those of a run without it"""
    lio1, mesh1, m, c1 = lio_stream(cuda_lib, reinforce=True)
    lio0, mesh0, _, c0 = lio_stream(cuda_lib, reinforce=True, feed=False)
    assert np.array_equal(lio1.get_state(), lio0.get_state())
    assert mesh1.counts() == mesh0.counts()
    for a, b in zip(mesh1.snapshot(), mesh0.snapshot()):
        assert np.array_equal(a, b)
    for x, y in zip(c1, c0):
        for a, b in zip(x, y):
            assert np.array_equal(a, b)


def test_ring_too_small_then_resync(cuda_lib):
    """a ring below some frames' rows: those frames are lost (IMMESH_E_RANGE, the pushes succeed), two frames that do not fit together
    overwrite the older one's rows; after each loss the resync (snapshot + the newest frame) mirrors the later frames exactly"""
    scans = world_scans("avia", 10, seed=13)
    probe = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    probe.changes_enable(1 << 20, 64)
    sizes = []
    for k, (w, t) in enumerate(scans):
        probe.push_frame(w, t, k)
        sizes.append(len(probe.changes(k)["rows"]))
    ring = int(np.median(sizes))
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.changes_enable(ring, 64)
    m = Mirror(mesh)
    lost = kept = wrapped = 0
    k = 0
    while k < len(scans):
        pair = k + 1 < len(scans) and sizes[k] <= ring and sizes[k + 1] <= ring and sizes[k] + sizes[k + 1] > ring and not wrapped
        for j in range(k, k + (2 if pair else 1)):
            mesh.push_frame(*scans[j], j)
        try:
            m.sync(mesh)
            m.check(mesh, f"frame {k}")
            assert not pair and sizes[k] <= ring
            kept += 1
        except RuntimeError as e:
            assert "code -5" in str(e), e
            assert pair or sizes[k] > ring
            lost += 1
            wrapped += pair
            m = Mirror(mesh)
        k += 2 if pair else 1
    assert probe.counts() == mesh.counts()
    assert kept and lost and wrapped, (sizes, ring, kept, lost, wrapped)


def test_max_frames_wrap(cuda_lib):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.changes_enable(1 << 20, 2)
    m = Mirror(mesh)
    scans = world_scans("avia", 5, seed=17)
    for k in range(3):
        mesh.push_frame(*scans[k], k)
    with pytest.raises(RuntimeError) as e:
        mesh.changes(m.newest)
    assert code_of(e) == E_RANGE
    ch = mesh.changes(mesh.changes_newest() - 2)
    assert ch["frames"][:, 0].tolist() == [2, 3]


def test_count_query_and_error_contract(cuda_lib):
    L = cuda_lib
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=L)
    counts = np.zeros(4, np.int64)
    cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
    call = lambda since, *a: L.immesh_mesh_changes(mesh._h, since, *a, cp)  # noqa: E731
    assert call(0, None, 0, None, 0, None, 0) == E_INVALID                        # not enabled
    assert L.immesh_mesh_changes_enable(mesh._h, -1, 4) == E_INVALID
    assert L.immesh_mesh_changes_enable(mesh._h, 16, 0) == E_INVALID
    assert L.immesh_mesh_changes_enable(mesh._h, (1 << 30) + 1, 4) == E_INVALID
    scans = world_scans("avia", 3, seed=19)
    mesh.push_frame(*scans[0], 0)
    mesh.changes_enable(1 << 20, 8)
    assert call(1, None, 0, None, 0, None, 0) == 0 and counts.tolist() == [0, 0, 0, 1]   # nothing after enable yet
    assert call(0, None, 0, None, 0, None, 0) == E_RANGE and counts[3] == 1           # before the enable
    assert call(2, None, 0, None, 0, None, 0) == E_INVALID                            # newer than the newest
    assert call(1, None, -1, None, 0, None, 0) == E_INVALID
    assert call(1, None, 1, None, 0, None, 0) == E_INVALID                            # a cap without its buffer
    mesh.push_frame(*scans[1], 1)
    mesh.push_frame(*scans[2], 2)
    assert call(1, None, 0, None, 0, None, 0) == E_CAPACITY
    nf, nr, nv, newest = counts.tolist()
    assert nf == 2 and nr > 0 and nv > 0 and newest == 3
    fr = np.zeros((nf, 4), np.int64)
    rows = np.zeros((nr, 4), np.int32)
    v = np.zeros((nv, 3), np.float32)
    args = (fr.ctypes.data_as(C.POINTER(C.c_int64)), nf, rows.ctypes.data_as(C.POINTER(C.c_int32)), nr, v.ctypes.data_as(C.POINTER(C.c_float)))
    assert call(1, *args, nv - 1) == E_CAPACITY and not v.any() and not rows.any()   # one short: nothing written
    assert call(1, *args, nv) == 0
    assert fr[:, 0].tolist() == [2, 3] and fr[-1, 3] == nr and fr[-1, 2] - fr[0, 1] == nv
    assert np.array_equal(mesh.changes(1)["rows"], rows)
    mesh.push_frame_batched(scans[0][0], scans[0][1])
    assert mesh.changes_newest() == 4 and len(mesh.changes(3)["frames"]) == 1
    assert L.immesh_mesh_changes_enable(mesh._h, 0, 0) == 0                            # off
    assert call(3, None, 0, None, 0, None, 0) == E_INVALID


def test_empty_frame(cuda_lib):
    mesh = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    mesh.changes_enable(1 << 16, 8)
    m = Mirror(mesh)
    w, t = world_scans("avia", 1, seed=21)[0]
    mesh.push_frame(w, t, 0)
    mesh.push_frame(np.zeros((0, 3), np.float32), t, 1)
    m.sync(mesh)
    m.check(mesh, "empty frame")
    fr = m.rows
    assert len(fr[2]) == 0
