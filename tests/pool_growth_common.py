"""Shared driver of the pool-growth tests: a localization handle created far below what a stream needs, grown on the way
(automatically, or by explicit reserve calls at scan boundaries), against the oracle with every per-scan assertion of
lio_common.run_stream_parity, or against a handle created at the default capacities."""
import dataclasses
import math

import numpy as np

from immesh_b200 import api, synth
from lio_common import SHAPE_COLS, init_velocity
from oracle_api import OracleLio

CAP_KEYS = ("root_slots", "nodes_cap", "chunks_cap")


def make_scans(kind, cfg, n_scans, seed, n_points=None):
    return synth.make_stream(kind, n_scans, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)


def start(h, sensor, scans):
    h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(h, sensor, scans)


def first_scan_use(lib, cfg, sensor, scans):
    """what the map of the first scan (buildVoxelMap) uses on a handle of the default capacities"""
    h = api.Lio(cfg, lib=lib)
    start(h, sensor, scans)
    h.voxel_map_init(scans[0]["body_full"])
    c = h.capacity()
    h.close()
    return c


def tiny_config(cfg, use):
    """capacities just above what the first scan uses"""
    return dataclasses.replace(cfg, hash_capacity_log2=max(10, math.ceil(math.log2(use["roots"] + 1))),
                               max_nodes=use["nodes"] + 1, max_chunks=use["chunks"] + 1)


def check_scan(g, o, k, ig, io):
    assert ig == io, f"scan {k}: iteration count {ig} vs {io}"
    assert np.array_equal(g.matches(), o.matches()), f"scan {k}: matched point set / layers"
    for it in range(io):
        a, b = g.iter_stats(it), o.iter_stats(it)
        assert a["n_match"] == b["n_match"]
        assert np.array_equal(a["HTH"], b["HTH"]) and np.array_equal(a["HTz"], b["HTz"]), f"scan {k} iter {it}: normal equations"
    sg, so = g.get_state(), o.get_state()
    assert np.array_equal(sg, so), f"scan {k}: state max diff {np.abs(sg - so).max()}"


def check_map(g, o, what):
    dg, do = g.dump_map(), o.dump_map()
    assert dg.shape == do.shape, f"{what}: node count {dg.shape[0]} vs {do.shape[0]}"
    assert np.array_equal(dg[:, SHAPE_COLS], do[:, SHAPE_COLS]), f"{what}: octree shape"
    assert np.array_equal(dg, do), f"{what}: plane parameters"


def run_growth_parity(lib, kind, cfg, n_scans, seed, n_points=None, growth=1 << 40, before_scan=None, stream=None):
    """A tiny handle (tiny_config) with automatic growth up to `growth` bytes (0: off), against the oracle after every stage
    (prediction, iteration count, matches, normal equations, state, map dump).  before_scan(g, k): called before scan k.
    stream: (sensor, scans) of make_scans.  Returns dict(first=capacity at create, last=capacity at the end, caps=[capacity after
    every scan], handle=the grown handle)."""
    sensor, scans = stream or make_scans(kind, cfg, n_scans, seed, n_points)
    small = tiny_config(cfg, first_scan_use(lib, cfg, sensor, scans))
    g = api.Lio(small, lib=lib)
    if growth:
        g.set_growth(growth)
    o = OracleLio(cfg, sum_mode=0)
    first = g.capacity()
    for h in (g, o):
        start(h, sensor, scans)
    if before_scan:
        before_scan(g, 0)
    g.voxel_map_init(scans[0]["body_full"])
    o.voxel_map_init(scans[0]["body_full"])
    check_map(g, o, "buildVoxelMap")
    caps = [g.capacity()]
    for k in range(1, n_scans):
        body, dt = scans[k]["body_ds"], scans[k]["dt"]
        if before_scan:
            before_scan(g, k)
        g.predict(dt)
        o.predict(dt)
        assert np.array_equal(g.get_state(), o.get_state()), f"scan {k}: prediction"
        ig = g.lio_state_estimation(body)
        io = o.lio_state_estimation(body)
        check_scan(g, o, k, ig, io)
        g.map_incremental_grow()
        o.map_incremental_grow(body)
        check_map(g, o, f"scan {k}")
        caps.append(g.capacity())
    assert g.counts()["err"] == 0
    return dict(first=first, last=g.capacity(), caps=caps, handle=g)


def doublings(first, last):
    """how many times each pool doubled between two capacity() results"""
    return {k: int(round(math.log2(last[k] / first[k]))) for k in CAP_KEYS}


def run_pipelined_pair(lib, kind, cfg, n_scans, seed, n_points=None, growth=1 << 40):
    """The graph-replayed pipeline (immesh_lio_step_async) on a tiny growing handle and on a default-sized one, side by side:
    the state after every scan and the map dump at the end must be bit-identical.  Returns (grown handle, default handle)."""
    sensor, scans = make_scans(kind, cfg, n_scans, seed, n_points)
    small = tiny_config(cfg, first_scan_use(lib, cfg, sensor, scans))
    g, d = api.Lio(small, lib=lib), api.Lio(cfg, lib=lib)
    g.set_growth(growth)
    for h in (g, d):
        start(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    for k in range(1, n_scans):
        for h in (g, d):
            h.step_async(scans[k]["body_ds"], dt=scans[k]["dt"])
        if k % 3 == 0 or k == n_scans - 1:   # let several steps queue between the checks
            (sg, ig), (sd, idd) = g.wait(), d.wait()
            assert ig == idd and np.array_equal(sg, sd), f"scan {k}: state"
    assert np.array_equal(g.dump_map(), d.dump_map())
    assert g.counts()["err"] == 0
    return g, d


# ---- the mesh handle
MESH_CAP_KEYS = ("vertices_cap", "triangles_cap", "voxels_cap")
MESH_SMALL = dict(max_vertices=1 << 19, max_triangles=1 << 21, max_voxels=1 << 17, max_frame_points=1 << 18)


def world_frames(scans):
    return [((s["body_full"].astype(np.float64) @ s["R_true"].T + s["t_true"]).astype(np.float32), s["t_true"]) for s in scans]


def first_frame_use(lib, frames):
    """what the first frame uses on a mesh handle of MESH_SMALL capacities"""
    h = api.Mesh(api.MeshConfig(**MESH_SMALL), lib=lib)
    h.push_frame(frames[0][0], frames[0][1], 0)
    c = h.capacity()
    h.close()
    return c


def tiny_mesh_config(use):
    """mesh capacities just above what the first frame uses (the per-frame capacities of MESH_SMALL).  The vertex chunks come with
    the vertices (max_vertices / 4 + 1024 of them) and a voxel holds at most count / 16 + 1: the vertex capacity is raised so that
    the first frame's chunks fit too."""
    return api.MeshConfig(max_vertices=use["vertices"] + 1 + 4 * use["voxels"], max_triangles=use["triangles"] + 1, max_voxels=use["voxels"] + 1,
                          max_frame_points=MESH_SMALL["max_frame_points"])


def mesh_doublings(first, last):
    return {k: int(round(math.log2(last[k] / first[k]))) for k in MESH_CAP_KEYS}


def check_mesh(g, o, what):
    cg, co = g.counts(), o.counts()
    assert cg == co, f"{what}: counts {cg} vs {co}"
    (vg, tg, fg), (vo, to, fo) = g.snapshot(), o.snapshot()
    assert np.array_equal(vg, vo), f"{what}: vertex positions / ids"
    assert tg.shape == to.shape and np.array_equal(tg, to), f"{what}: facet set"
    assert np.array_equal(fg, fo), f"{what}: orientation flags"
