"""GPU tier: immesh_mesh_push_frame_batched and immesh_mesh_reconstruct_from_pointcloud_batched through the C ABI, bit-exact against the
oracle's single frame (the smoothed positions and m_smoothed flags through the viewer's region buffers, which emit the stored smoothed
positions and smooth exactly the unflagged vertices), against the unbatched frame where one fits, and on one cloud beyond every
one-frame limit of a default-capacity frame."""
import numpy as np
import pytest

from immesh_b200 import api
from mesh_common import SMALL, world_scans
from offline_batched_common import (E_CAPACITY, E_INVALID, assert_same_state, avia_cloud, batch_sizes, new_config, oracle_frame, oracle_state,
                                    split_clusters)
from oracle_api import OracleMesh, voxel_grid
from region_buffers_common import compare_call

pytestmark = pytest.mark.gpu


def gpu_state(g):
    v, t, f = g.snapshot()
    return dict(counts=g.counts(), v=v, t=t, f=f)


def check(g, o, what):
    assert_same_state(gpu_state(g), oracle_state(o), what)
    compare_call(g, o, 10.0)   # smoothed positions + m_smoothed flags (and the write-back stays identical on both sides)


def test_offline_size_frame_bit_exact(cuda_lib):
    cloud = avia_cloud(3)
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    bp, bv = batch_sizes(len(cloud), o.counts()["frame_voxels_meshed"], 12, 12)
    g = api.Mesh(new_config(), lib=cuda_lib)
    st = g.push_frame_batched(cloud, np.zeros(3), bp, bv)
    assert st["append_chunks"] >= 10 and st["voxel_batches"] >= 10, st
    check(g, o, "offline cloud")


def test_batch_size_invariance_and_device_input(cuda_lib):
    import torch
    cloud = avia_cloud(3)
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    ref = oracle_state(o)
    n_meshed = ref["counts"]["frame_voxels_meshed"]
    d = torch.from_numpy(cloud).cuda()
    for bp, bv, dev in ((0, 0, False), (len(cloud) // 17, n_meshed // 5, False), (len(cloud) // 3, 7, True), (len(cloud) // 11, n_meshed // 13, True)):
        g = api.Mesh(new_config(), lib=cuda_lib)
        if dev:
            g.push_frame_batched(d.data_ptr(), np.zeros(3), bp, bv, n=len(cloud), on_device=True)
        else:
            g.push_frame_batched(cloud, np.zeros(3), bp, bv)
        assert_same_state(gpu_state(g), ref, f"batches {bp} / {bv}, device input {dev}")


def test_batched_frame_on_a_non_empty_mesh(cuda_lib):
    cfg = api.MeshConfig(**SMALL)
    scans = world_scans("avia", 6, seed=3)
    big = np.concatenate([w for w, _ in scans[3:]], axis=0)
    o = oracle_frame(cfg, scans[:3])
    g = api.Mesh(cfg, lib=cuda_lib)
    for k, (w, t) in enumerate(scans[:3]):
        g.push_frame(w, t, k)
    o.push_frame(big, scans[5][1], 3)
    st = g.push_frame_batched(big, scans[5][1], 1000, max(1, o.counts()["frame_voxels_meshed"] // 10))
    assert st["append_chunks"] >= 10 and st["voxel_batches"] >= 10, st
    assert o.counts()["frame_removed"] > 0
    check(g, o, "batched frame after three frames")
    # the mesh goes on: a normal frame on top
    w, t = world_scans("avia", 7, seed=3)[6]
    g.push_frame(w, t, 4)
    o.push_frame(w, t, 4)
    check(g, o, "normal frame after the batched one")


def test_range_beyond_the_flip_priority_field(cuda_lib):
    cloud = split_clusters()
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    g = api.Mesh(new_config(), lib=cuda_lib)
    g.push_frame_batched(cloud, np.zeros(3), 0, max(1, o.counts()["frame_voxels_meshed"] // 4))
    check(g, o, "1 km apart")
    with pytest.raises(RuntimeError, match="code -5"):
        api.Mesh(new_config(), lib=cuda_lib).push_frame(cloud, np.zeros(3))


def test_batched_equals_unbatched(cuda_lib):
    """where one frame fits, the batched frame is the unbatched one, frame after frame"""
    cfg = api.MeshConfig(**SMALL)
    a, b = api.Mesh(cfg, lib=cuda_lib), api.Mesh(cfg, lib=cuda_lib)
    for k, (w, t) in enumerate(world_scans("avia", 5, seed=21)):
        a.push_frame(w, t, k)
        b.push_frame_batched(w, t, 777, 97)
        sa, sb = gpu_state(a), gpu_state(b)
        assert_same_state(sb, sa, f"frame {k}")


def test_offline_entry_both_branches(cuda_lib):
    # pass-through: a 1 cm leaf on a cloud wider than 13 m; the VoxelGrid handle is far too small for the cloud and does not matter
    cloud = avia_cloud(2)
    ds, small, _ = voxel_grid(cloud, 0.01)
    assert small and np.ptp(cloud, axis=0).max() > 13.0
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    g = api.Mesh(new_config(), lib=cuda_lib)
    m = g.reconstruct_from_pointcloud_batched(api.VoxelGrid(1024, lib=cuda_lib), cloud, 0.01, 20000, 300)
    assert m == len(cloud)
    check(g, o, "pass-through")
    # filtered: a small cloud, leaf 0.1 m
    ds, small, _ = voxel_grid(cloud, 0.1)
    assert not small
    o = oracle_frame(new_config(), [(ds, np.zeros(3))])
    g = api.Mesh(new_config(), lib=cuda_lib)
    m = g.reconstruct_from_pointcloud_batched(api.VoxelGrid(1 << 18, lib=cuda_lib), cloud, 0.1, 5000, 200)
    assert m == len(ds)
    check(g, o, "filtered")
    # filtered, but larger than the VoxelGrid handle
    with pytest.raises(RuntimeError, match=f"code {E_CAPACITY}"):
        api.Mesh(new_config(), lib=cuda_lib).reconstruct_from_pointcloud_batched(api.VoxelGrid(1024, lib=cuda_lib), cloud, 0.1)


def test_argument_contract(cuda_lib):
    import ctypes as C
    cfg = new_config()
    g = api.Mesh(cfg, lib=cuda_lib)
    a = np.ascontiguousarray(avia_cloud(1, n_points=2000), np.float32)
    z = np.zeros(3)
    dp = C.POINTER(C.c_double)
    call = lambda bp, bv, n=len(a): cuda_lib.immesh_mesh_push_frame_batched(g._h, a.ctypes.data_as(C.c_void_p), n, 0, z.ctypes.data_as(dp), bp, bv, None)  # noqa: E731
    for bp, bv, n in ((cfg.max_frame_points + 1, 0, len(a)), (-1, 0, len(a)), (0, -1, len(a)), (0, 1 << 20, len(a)), (0, 0, -1)):
        assert call(bp, bv, n) == E_INVALID
    assert g.counts()["n_vertices"] == 0
    assert call(0, 0, 0) == 0
    o = OracleMesh(cfg)
    o.push_frame(np.zeros((0, 3), np.float32), z)
    assert g.counts() == o.counts()


def tiled_cloud(tile, k):
    """k translated copies of `tile` on a grid with gaps of at least 10 m"""
    ext = np.ptp(tile, axis=0) + 10.0
    side = int(np.ceil(np.sqrt(k)))
    offs = [np.array([(i % side) * ext[0], (i // side) * ext[1], 0.0], np.float32) for i in range(k)]
    return [tile + o for o in offs]


def test_cloud_beyond_every_one_frame_limit(cuda_lib):
    """~14 M points, > 262 144 meshed voxels, > 4 Mi facets, > 409.6 m wide, one batched frame on a default-capacity frame: tiles far apart
    mesh independently with contiguous vertex ids, so the first, a middle and the last tile equal the oracle on that tile alone"""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip(f"needs 24 GB of free device memory, {free >> 30} GB free")
    tile = avia_cloud(3, seed=15, n_points=50000)
    K = 112
    tiles = tiled_cloud(tile, K)
    cloud = np.concatenate(tiles, axis=0)
    assert len(cloud) > 13_000_000 and np.ptp(cloud[:, :2], axis=0).max() > 409.6
    cfg = api.MeshConfig(points_minimum_scale=0.1, voxel_resolution=0.4, number_of_pts_append_to_map=1 << 30, max_vertices=1 << 24,
                         max_triangles=1 << 25, max_voxels=1 << 22, max_frame_points=0)   # frame capacities at their defaults
    g = api.Mesh(cfg, lib=cuda_lib)
    st = g.push_frame_batched(cloud, np.zeros(3), 0, 1 << 16)   # 2 Mi-candidate chunks; 65536 voxels keep a batch's facets under 4 Mi
    c = g.counts()
    assert c["frame_voxels_meshed"] > 262_144 and st["facets_added"] > 4 << 20, (c, st)
    v, t, f = g.snapshot()
    tid = np.full(len(v), -1)
    for i, tl in enumerate(tiles):
        inside = np.all((v >= tl.min(axis=0)) & (v <= tl.max(axis=0)), axis=1)
        tid[inside] = i
    assert (tid >= 0).all() and np.all(np.diff(tid) >= 0), "vertex ids are not contiguous per tile"
    start = np.searchsorted(tid, np.arange(K + 1))
    for i in (0, K // 2, K - 1):
        o = OracleMesh(cfg)
        o.push_frame(tiles[i], np.zeros(3))
        vo, to, fo = o.snapshot()
        sel = (t[:, 0] >= start[i]) & (t[:, 0] < start[i + 1])
        assert np.array_equal(v[start[i]:start[i + 1]], vo), f"tile {i}: vertices"
        assert np.array_equal(t[sel] - start[i], to) and np.array_equal(f[sel], fo), f"tile {i}: facets / flips"
    g2 = api.Mesh(cfg, lib=cuda_lib)
    st2 = g2.push_frame_batched(cloud, np.zeros(3), 1 << 20, 50_000)
    assert st2["append_chunks"] > st["append_chunks"] and st2["voxel_batches"] > st["voxel_batches"]
    v2, t2, f2 = g2.snapshot()
    assert g2.counts() == c and np.array_equal(v2, v) and np.array_equal(t2, t) and np.array_equal(f2, f)
    del g2
    st4 = g.push_frame_batched(np.concatenate(tiles[: K // 4]), np.zeros(3), 0, 1 << 16)
    assert st4["scratch_bytes"] == st["scratch_bytes"]
    w, pose = world_scans("avia", 1, seed=4)[0]
    g.push_frame(w, pose)
    xyz, ids, keys, offs, _ = g.region_buffers(50.0)
    assert len(xyz) == g.counts()["n_triangles"] and len(keys) > K
