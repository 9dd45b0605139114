"""GPU tier: the mesher's size- and geometry-dependent kernel paths on the device, bit-exact against the oracle (the scenes and
the path table are in tests/mesh_scenes.py and test_mesh_paths_emu.py; on the device the warp kernel's one_pass boundary search
runs for every insertion whose cavity has at most 10 triangles), the capacity errors, the run-time knobs that select other code
(INTEGRATION.md), and immesh_knn at its largest k."""
import os
import subprocess
import sys

import numpy as np
import pytest

import mesh_scenes as ms
from immesh_b200 import api
from mesh_common import SMALL, run_mesh_parity, run_scene_parity
from oracle_api import OracleMesh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENES = ms.path_scenes()


@pytest.mark.parametrize("scene,path", SCENES, ids=[s.name for s, _ in SCENES])
def test_scene_path_bit_exact(cuda_lib, scene, path):
    g, o, stats = run_scene_parity(cuda_lib, scene)
    assert ms.path_of(ms.centre_stats(stats, scene, scene.cfg_kw["voxel_resolution"])) == path


@pytest.mark.parametrize("n_ring", [67, 250])
def test_ring_late_centre_is_the_fan(cuda_lib, n_ring):
    g, o, stats = run_scene_parity(cuda_lib, ms.ring(n_ring))
    assert np.array_equal(g.snapshot()[1], ms.ring_fan(n_ring))


@pytest.mark.parametrize("scene", ms.cap_scenes(), ids=lambda s: s.name)
def test_caps_raise_capacity(cuda_lib, scene):
    """IMMESH_E_CAPACITY with the per-voxel flag alone: no pool or list overflowed on the way"""
    g = api.Mesh(api.MeshConfig(**{**SMALL, **scene.cfg_kw}), lib=cuda_lib)
    with pytest.raises(RuntimeError, match=r"code -3: .*\(flags: VOXEL_CAP\)$"):
        for k, pts in enumerate(scene.frames):
            g.push_frame(pts, scene.centre, k)


# ---------------------------------------------------------------- run-time knobs (read when the handle is created)
@pytest.mark.parametrize("nmax", ["3", "64"])
def test_knob_warp_nmax(cuda_lib, monkeypatch, nmax):
    """IMMESH_WARP_NMAX (the product clamps it to [3, 128]): 3 sends every set above 3 vertices, one_pass voxels included, to the
    block variants; 64 splits the warp scenes (lattice8x8 stays warp, patch96 / stacked6x6 / ring67 / ring95 go block-level)"""
    monkeypatch.setenv("IMMESH_WARP_NMAX", nmax)
    for scene, path in SCENES:
        if path.startswith("warp") or path == "handover":
            run_scene_parity(cuda_lib, scene)
    run_mesh_parity(cuda_lib, "avia", 3, seed=0)


def test_knob_graph_off(cuda_lib, monkeypatch):
    """IMMESH_GRAPH=0: the pipelined entry points launch kernel by kernel instead of replaying a CUDA graph"""
    import test_mesh_gpu
    monkeypatch.setenv("IMMESH_GRAPH", "0")
    test_mesh_gpu.test_pipelined_equals_sequential(cuda_lib)


def test_knob_voxelgrid_block_centroid(cuda_lib, monkeypatch):
    """IMMESH_VG_WARP_CENTROID=0: the VoxelGrid centroids are summed by the block-level code"""
    import test_frontend_gpu
    monkeypatch.setenv("IMMESH_VG_WARP_CENTROID", "0")
    test_frontend_gpu.test_edge_cases(cuda_lib)


def test_knob_lio_split_off():
    """IMMESH_LIO_SPLIT=0 (read once per process): the fused k_residual instead of k_match + k_terms, in a fresh process"""
    code = ("import sys; sys.path[:0] = [%r, %r]\n"
            "from immesh_b200 import api\n"
            "from lio_common import run_stream_parity\n"
            "s = run_stream_parity(api.load_library(), 'avia', api.AVIA, n_scans=4, seed=3)\n"
            "print('split0 ok', s[-1]['n_match'])\n") % (ROOT, os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env={**os.environ, "IMMESH_LIO_SPLIT": "0"}, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "split0 ok" in r.stdout, (r.stdout + r.stderr)[-3000:]


# ---------------------------------------------------------------- kNN at KNN_KMAX
def test_knn_k32_on_vertices_and_ties(cuda_lib):
    """k = 32 fills the per-lane lists; queries exactly on vertices (distance 0) and on exact distance ties (lattice midpoints,
    where 2 or 4 vertices are equally near and the lower id must win) against the oracle and the live ikd-Tree"""
    import ref_ikd
    scene = ms.lattice(16, 8, dx=0.015625, xi=0.005)
    cfg = api.MeshConfig(**{**SMALL, **scene.cfg_kw})
    g, o = api.Mesh(cfg, lib=cuda_lib), OracleMesh(cfg)
    for m in (g, o):
        m.push_frame(scene.frames[0], scene.centre, 0)
    v = g.snapshot()[0]
    assert np.array_equal(v, o.snapshot()[0])
    mid = ((v[:-1] + v[1:]) / 2).astype(np.float32)
    q = np.concatenate([v, mid]).astype(np.float32)
    for k, md in ((32, np.inf), (32, 0.05), (31, np.inf)):
        ig, dg = g.knn(q, k, md)
        io, do = o.knn(q, k, md)
        assert np.array_equal(ig, io) and np.array_equal(dg, do), (k, md)
        if np.isinf(md):
            assert (dg[: len(v), 0] == 0).all() and (ig[: len(v), 0] == np.arange(len(v))).all()
            assert (dg[:, 1:] == dg[:, :-1]).any()   # the lattice produces exact ties inside the lists
    if ref_ikd.available():
        # the ikd-Tree orders a tie group by its tree shape; when the k-th slot cuts a tie group, which of its members make the
        # list differs too.  So: the distances identical, every complete tie group the same set, the cut group a subset of the
        # vertices at exactly that float distance ((dx*dx + dy*dy) + dz*dz in float, as both compute it).
        t = ref_ikd.RefIkdTree()
        t.add(v)
        ig, dg = g.knn(q, 32)
        ir, dr, _ = t.knn(q, 32, np.inf)
        assert np.array_equal(dg, dr)
        for r in range(len(q)):
            e = q[r] - v
            d2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
            for val in np.unique(dg[r]):
                m = dg[r] == val
                if val == dg[r, -1]:
                    at = set(np.where(d2 == val)[0].tolist())
                    assert set(ig[r][m].tolist()) <= at and set(ir[r][m].tolist()) <= at, r
                else:
                    assert sorted(ig[r][m].tolist()) == sorted(ir[r][m].tolist()), r
