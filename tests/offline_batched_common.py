"""Shared scenes and checks of the batched frame (immesh_mesh_push_frame_batched) and the batched offline entry
(immesh_mesh_reconstruct_from_pointcloud_batched): one incremental_mesh_reconstruction frame run in bounded append chunks and voxel
batches must leave the mesh bit-identical to the oracle's single frame on the same points -- counts, vertices and ids, facets and
orientation flags, and the smoothed positions with their m_smoothed flags (the oracle side keeps them: tests/pubmap/orc_region_buf.cpp)."""
import ctypes as C

import numpy as np

from immesh_b200 import api
from mesh_common import SMALL, world_scans
from oracle_api import _p
from region_buffers_common import RegionOracle

# offline_pointcloud.yaml: every point of the cloud is an append candidate
OFFLINE = {**SMALL, "number_of_pts_append_to_map": 1 << 30}
E_INVALID, E_CAPACITY, E_RANGE = -1, -3, -5
# The region-buffer oracle keeps its m_smoothed flags in a table keyed by the handle's address and never drops an entry, so a
# new oracle allocated where a destroyed one lived would start with that one's flags: every oracle made here stays alive.
_ALIVE = []


def avia_cloud(n_scans=3, seed=15, n_points=50000):
    """world-frame Avia scans concatenated into one offline cloud (about 42 k points per scan)"""
    return np.concatenate([w for w, _ in world_scans("avia", n_scans, seed, n_points)], axis=0)


def split_clusters(seed=15):
    """two copies of an Avia scan 1 km apart: most meshed voxels are more than 2048 voxels from the pose at the origin"""
    a = avia_cloud(1, seed)
    return np.concatenate([a, a + np.array([1000.0, 0.0, 0.0], np.float32)], axis=0)


def oracle_state(o):
    """counts, vertices, facets, flips, smoothed positions and m_smoothed flags of a RegionOracle"""
    c = o.counts()
    v = np.zeros((c["n_vertices"], 3), np.float32)
    s = np.zeros((c["n_vertices"], 3))
    o.L.orc_mesh_get_vertices(o.h, _p(v), _p(s))
    _, t, f = o.snapshot()
    return dict(counts=c, v=v, t=t, f=f, smooth=s, flags=o.flags())


def emu_state(lib, g):
    """the same fields from the host emulation with the m_smoothed flags (tests/batched/emu_batched.cpp)"""
    c = g.counts()
    v, t, f = g.snapshot()
    fl = np.zeros(c["n_vertices"], np.uint8)
    s = np.zeros((c["n_vertices"], 3))
    lib.emu_mesh_smooth_state(g._h, fl.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p))
    return dict(counts=c, v=v, t=t, f=f, smooth=s, flags=fl)


def assert_same_state(a, b, what):
    assert a["counts"] == b["counts"], f"{what}: counts {a['counts']} vs {b['counts']}"
    assert np.array_equal(a["v"], b["v"]), f"{what}: vertices / ids"
    assert a["t"].shape == b["t"].shape and np.array_equal(a["t"], b["t"]), f"{what}: facet set"
    assert np.array_equal(a["f"], b["f"]), f"{what}: orientation flags"
    for k in ("smooth", "flags"):
        if k in a and k in b:
            x, y = a[k], b[k]
            same = (x == y) | (np.isnan(x) & np.isnan(y)) if x.dtype.kind == "f" else x == y
            assert x.shape == y.shape and same.all(), f"{what}: {k}"


def batch_sizes(n_points, n_meshed, chunks, batches):
    """batch_points / batch_voxels that split a frame into at least `chunks` append chunks and `batches` voxel batches"""
    return max(1, n_points // chunks), max(1, n_meshed // batches)


def voxel_batch_of(o_stats, batch_voxels, res, pts):
    """batch index of the voxel each point lies in, for the voxels the last frame meshed (ascending key = the batched frame's rank
    order), -1 elsewhere"""
    keys = o_stats["key"].astype(np.int64)
    k = np.round(pts.astype(np.float64) / res).astype(np.int64)
    lut = {tuple(r): i // batch_voxels for i, r in enumerate(keys)}
    return np.array([lut.get(tuple(r), -1) for r in k])


def new_config(**kw):
    return api.MeshConfig(**{**OFFLINE, **kw})


def oracle_frame(cfg, frames, pose=np.zeros(3)):
    """RegionOracle after the given (pts, pose) frames"""
    o = RegionOracle(cfg)
    _ALIVE.append(o)
    for k, (pts, t) in enumerate(frames):
        o.push_frame(pts, t, k)
    return o
