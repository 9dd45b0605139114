"""CPU tier: the batched frame (immesh_mesh_push_frame_batched) run by the host emulation on the device's __host__ __device__ bodies
with the device's orchestration (append chunks, the activation rule after the last chunk, pass 1 = every dilation's smoothing, pass 2 =
dilation lists again + triangulation + pull / commit + the batch's additions, removals after the last batch, rank flip priority),
bit-exact against the oracle's single frame.  The offline entry's VoxelGrid branch runs on the device only (test_offline_batched_gpu.py)."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api
from mesh_common import SMALL, world_scans
from offline_batched_common import (E_CAPACITY, E_INVALID, assert_same_state, avia_cloud, batch_sizes, emu_state, new_config,
                                    oracle_frame, oracle_state, split_clusters, voxel_batch_of)


@pytest.fixture(scope="module")
def emu_lib():
    """the host emulation with the m_smoothed flags and the batched frame (tests/batched/emu_batched.cpp)"""
    from immesh_b200 import build
    return api.load_library(build.build_batched())


@pytest.fixture(scope="module")
def offline_cloud():
    cloud = avia_cloud(3)
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    return cloud, oracle_state(o)


def test_offline_size_frame_bit_exact(emu_lib, offline_cloud):
    """a 126 k-point offline cloud in >= 10 append chunks and >= 10 voxel batches equals the oracle's single frame"""
    cloud, ref = offline_cloud
    assert 100_000 <= len(cloud) <= 200_000
    bp, bv = batch_sizes(len(cloud), ref["counts"]["frame_voxels_meshed"], 12, 12)
    g = api.Mesh(new_config(), lib=emu_lib)
    st = g.push_frame_batched(cloud, np.zeros(3), bp, bv)
    assert st["append_chunks"] >= 10 and st["voxel_batches"] >= 10, st
    assert st["facets_added"] == ref["counts"]["frame_added"] > 50_000
    assert_same_state(emu_state(emu_lib, g), ref, "offline cloud")


def test_batch_size_invariance(emu_lib, offline_cloud):
    """three batch settings, one chunk / one batch included, give the same state (and the oracle's)"""
    cloud, ref = offline_cloud
    n_meshed = ref["counts"]["frame_voxels_meshed"]
    states = []
    for bp, bv in ((0, 0), (len(cloud) // 17, n_meshed // 5), (len(cloud) // 3, 7)):
        g = api.Mesh(new_config(), lib=emu_lib)
        g.push_frame_batched(cloud, np.zeros(3), bp, bv)
        states.append(emu_state(emu_lib, g))
    for s in states:
        assert_same_state(s, ref, "batch invariance")
        assert_same_state(s, states[0], "batch invariance")


def test_batched_frame_on_a_non_empty_mesh(emu_lib):
    """three normal Avia frames, then a three-scan batched frame (append step > 1): it removes pre-frame triangles, raises the flip words
    of pre-frame facets from voxels of different batches and pulls pre-frame triangles next to facets an earlier batch added -- and
    equals the oracle"""
    cfg = api.MeshConfig(**SMALL)
    scans = world_scans("avia", 6, seed=3)
    big = np.concatenate([w for w, _ in scans[3:]], axis=0)
    pose = scans[5][1]
    o = oracle_frame(cfg, scans[:3])
    g = api.Mesh(cfg, lib=emu_lib)
    for k, (w, t) in enumerate(scans[:3]):
        g.push_frame(w, t, k)
    v0, t0, _ = g.snapshot()
    o.push_frame(big, pose, 3)
    ref = oracle_state(o)
    bp, bv = batch_sizes(len(big) // max(1, len(big) // cfg.number_of_pts_append_to_map), ref["counts"]["frame_voxels_meshed"], 10, 10)
    st = g.push_frame_batched(big, pose, bp, bv)
    assert st["append_chunks"] >= 10 and st["voxel_batches"] >= 10, st
    got = emu_state(emu_lib, g)
    assert_same_state(got, ref, "batched frame after three frames")
    assert ref["counts"]["frame_removed"] > 0
    # which batch meshes the voxel each vertex lies in (ascending key order of the meshed voxels, batch_voxels each)
    vb = voxel_batch_of(o.frame_voxel_stats(), bv, cfg.voxel_resolution, got["v"])
    before = {tuple(r) for r in t0}
    after = {tuple(r) for r in got["t"]}
    kept = [r for r in after & before if len({vb[i] for i in r} - {-1}) >= 2]
    assert kept, "no pre-frame facet spans voxels of two batches"
    born = after - before
    removed = before - after
    edge_batch = {}
    for r in born:
        b = max(vb[i] for i in r)
        for e in ((r[0], r[1]), (r[0], r[2]), (r[1], r[2])):
            edge_batch[e] = min(edge_batch.get(e, 1 << 30), b)
    late = [r for r in removed if max(vb[i] for i in r) > min(edge_batch.get(e, 1 << 30) for e in ((r[0], r[1]), (r[0], r[2]), (r[1], r[2])))]
    assert late, "no pre-frame triangle was pulled in a later batch than a neighbouring new facet"


def test_range_beyond_the_flip_priority_field(emu_lib):
    """two clusters 1 km apart (2500 voxels at 0.4 m from the pose): the per-frame path's 11-bit priority field is out of range
    (IM_MERR_PRIO_RANGE), the batched frame's rank is not, and it equals the oracle, which has no limit"""
    cloud = split_clusters()
    o = oracle_frame(new_config(), [(cloud, np.zeros(3))])
    ref = oracle_state(o)
    g = api.Mesh(new_config(), lib=emu_lib)
    g.push_frame_batched(cloud, np.zeros(3), 0, max(1, ref["counts"]["frame_voxels_meshed"] // 4))
    assert_same_state(emu_state(emu_lib, g), ref, "1 km apart")
    plain = api.Mesh(new_config(), lib=emu_lib)
    with pytest.raises(RuntimeError):
        plain.push_frame(cloud, np.zeros(3))
    assert emu_lib.emu_mesh_error_word(plain._h) == 64   # IM_MERR_PRIO_RANGE alone


def test_bounded_facet_set_probe(emu_lib):
    """a facet set too small for the batch's facets: the commit sets IM_MERR_LIST_CAP and the call returns IMMESH_E_CAPACITY"""
    cloud = avia_cloud(1)
    g = api.Mesh(new_config(), lib=emu_lib)
    emu_lib.emu_mesh_set_batch_fset_bits(g._h, 4)
    with pytest.raises(RuntimeError, match=f"code {E_CAPACITY}"):
        g.push_frame_batched(cloud, np.zeros(3))
    assert emu_lib.emu_mesh_error_word(g._h) & 16


def test_argument_contract(emu_lib):
    cloud = avia_cloud(1, n_points=2000)
    cfg = new_config()
    g = api.Mesh(cfg, lib=emu_lib)
    dp = C.POINTER(C.c_double)
    z = np.zeros(3)
    a = np.ascontiguousarray(cloud, np.float32)
    call = lambda bp, bv, n=len(a): emu_lib.immesh_mesh_push_frame_batched(g._h, a.ctypes.data_as(C.c_void_p), n, 0, z.ctypes.data_as(dp), bp, bv, None)  # noqa: E731
    assert call(cfg.max_frame_points + 1, 0) == E_INVALID
    assert call(-1, 0) == E_INVALID
    assert call(0, -1) == E_INVALID
    assert call(0, 1 << 20) == E_INVALID          # more than the frame's work capacity
    assert call(0, 0, -1) == E_INVALID
    assert g.counts()["n_vertices"] == 0          # nothing ran
    assert call(0, 0, 0) == 0                     # an empty frame
    o = oracle_frame(cfg, [(np.zeros((0, 3), np.float32), z)])
    assert g.counts() == o.counts()
    sh = api.Mesh(cfg, lib=emu_lib)
    emu_lib.emu_mesh_set_shard(sh._h, 0, 2)
    assert emu_lib.immesh_mesh_push_frame_batched(sh._h, a.ctypes.data_as(C.c_void_p), len(a), 0, z.ctypes.data_as(dp), 0, 0, None) == E_INVALID
