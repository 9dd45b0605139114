"""Shared driver of the viewer region-buffer tests (synchronize_triangle_list_for_disp -> unparse_triangle_set_to_vector +
get_axis_min_max, mesh_rec_display.cpp:78-137, :220-258): the same frame stream through an implementation under test (CUDA library or
host emulation) and the oracle, the same region-buffer calls between frames, rows / ids / regions / smoothed counts / axis box compared
bit for bit, and the mesh of later frames compared too (the smoothed positions a call stores are read by correct_triangle_index).

The oracle side is tests/pubmap/liborc_regionbuf.so (the oracle with m_smoothed kept beside it and the viewer's walk,
orc_region_buf.cpp); the emulation side is tests/pubmap/libimmesh_emu_regionbuf.so (emu_region_buf.cpp)."""
import ctypes as C

import numpy as np

from immesh_b200 import api
from mesh_common import SMALL, world_scans
from oracle_api import OracleMesh, _p

BOX0 = np.array([1e8, 1e8, 1e8, -1e8, -1e8, -1e8], dtype=np.float32)   # g_axis_min_max at service start (mesh_rec_display.cpp:264)
_lib = None


def emu_regionbuf_lib():
    from immesh_b200 import build
    return api.load_library(build.build_regionbuf()[0])


def _orc():
    global _lib
    if _lib is None:
        from immesh_b200 import build
        L = C.CDLL(build.build_regionbuf()[1])
        L.orc_mesh_create.restype = C.c_void_p
        L.orc_mesh_create.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
        L.orc_mesh_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
        L.orc_view_smooth_all.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_void_p]
        L.orc_view_region_buffers.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_double, C.c_int] + [C.c_void_p] * 7
        _lib = L
    return _lib


class RegionOracle(OracleMesh):
    """The oracle with m_smoothed kept and the viewer's walk (orc_region_buf.cpp)."""

    def __init__(self, cfg):
        self.L = _orc()
        self.h = C.c_void_p(self.L.orc_mesh_create(cfg.points_minimum_scale, cfg.voxel_resolution, cfg.number_of_pts_append_to_map, 1))

    def push_frame(self, pts, pose_t, frame_idx=0):
        a = np.ascontiguousarray(pts, dtype=np.float32)
        t = np.ascontiguousarray(pose_t, dtype=np.float64)
        self.L.orc_view_push_frame(self.h, _p(a), C.c_int(a.shape[0]), _p(t))

    def smooth_all(self, smooth_factor=0.1, knn=20):
        out = np.zeros((self.counts()["n_vertices"], 3))
        self.L.orc_view_smooth_all(self.h, smooth_factor, knn, _p(out))
        return out

    def flags(self):
        f = np.zeros(self.counts()["n_vertices"], dtype=np.uint8)
        self.L.orc_view_flags(self.h, _p(f))
        return f

    def region_buffers(self, region_size=10.0, keys=None, smooth_factor=1.0, knn=20, axis_min_max=None):
        nt = self.counts()["n_triangles"]
        k = None if keys is None else np.ascontiguousarray(keys, dtype=np.int32).reshape(-1, 3)
        nk = 0 if k is None else k.shape[0]
        xyz = np.zeros((max(nt, 1), 9), dtype=np.float32)
        ids = np.zeros((max(nt, 1), 3), dtype=np.int32)
        rkeys = np.zeros((nk + nt + 1, 3), dtype=np.int32)
        roff = np.zeros(nk + nt + 2, dtype=np.int32)
        nr, ns = C.c_int(0), C.c_int(0)
        n = self.L.orc_view_region_buffers(self.h, region_size, None if k is None else _p(k), nk, smooth_factor, knn, _p(xyz), _p(ids), _p(rkeys), _p(roff),
                                           None if axis_min_max is None else _p(axis_min_max), C.byref(nr), C.byref(ns))
        return xyz[:n].copy(), ids[:n].copy(), rkeys[:nr.value].copy(), roff[:nr.value + 1].copy(), ns.value


def same_bits(a, b):
    """bit-identical float arrays, except that a NaN equals a NaN (a vertex without a neighbour inside the limit divides by zero)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def compare_call(g, o, region_size, keys=None, knn=20, smooth_factor=1.0, box=None):
    """one region-buffer call on both sides; returns the implementation's result and the oracle's"""
    bg = BOX0.copy() if box is None else box[0]
    bo = BOX0.copy() if box is None else box[1]
    rg = g.region_buffers(region_size, keys, smooth_factor, knn, bg)
    ro = o.region_buffers(region_size, keys, smooth_factor, knn, bo)
    what = f"region_size {region_size}, keys {None if keys is None else len(keys)}, knn {knn}"
    assert same_bits(rg[0], ro[0]), f"{what}: rows"
    assert np.array_equal(rg[1], ro[1]), f"{what}: ids"
    assert np.array_equal(rg[2], ro[2]) and np.array_equal(rg[3], ro[3]), f"{what}: regions"
    assert rg[4] == ro[4], f"{what}: smoothed {rg[4]} vs {ro[4]}"
    assert np.array_equal(bg.view(np.uint32), bo.view(np.uint32)), f"{what}: axis box {bg} vs {bo}"
    return rg, ro


def subset_keys(o, region_size, every=3):
    """every `every`-th non-empty region in descending key order, plus one region that holds no triangle"""
    k = np.unique(o.region_keys(region_size), axis=0)[::-1][::every]
    return np.concatenate([k, np.array([[1000, -1000, 999]], dtype=np.int32)]).astype(np.int32)


def check_mesh(g, o, what):
    vg, tg, fg = g.snapshot()
    vo, to, fo = o.snapshot()
    assert np.array_equal(vg, vo), f"{what}: vertices"
    assert tg.shape == to.shape and np.array_equal(tg, to), f"{what}: facet set"
    assert np.array_equal(fg, fo), f"{what}: orientation flags"


def run_region_parity(lib, kind, n_frames, seed, call_after=(1, 3, 5), region_size=2.0, n_points=None, push=None, wait=None, cfg_kw=None):
    """frames through the implementation (push(g, k, world, t); wait(g) before a call) and the oracle; after the frames in call_after a
    key-subset call, then an all-regions call, on both sides.  Returns (g, o, [(n_rows, n_smoothed) of every call])."""
    cfg = api.MeshConfig(**{**SMALL, **(cfg_kw or {})})
    g, o = api.Mesh(cfg, lib=lib), RegionOracle(cfg)
    push = push or (lambda m, k, w, t: m.push_frame(w, t, k))
    stats = []
    for k, (world, t) in enumerate(world_scans(kind, n_frames, seed, n_points)):
        push(g, k, world, t)
        o.push_frame(world, t, k)
        if k in call_after:
            if wait:
                wait(g)
            check_mesh(g, o, f"frame {k}")
            for keys in (subset_keys(o, region_size), None):
                rg, _ = compare_call(g, o, region_size, keys)
                stats.append((len(rg[0]), rg[4]))
    if wait:
        wait(g)
    check_mesh(g, o, "end")
    return g, o, stats
