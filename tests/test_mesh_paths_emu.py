"""CPU tier: the scenes of tests/mesh_scenes.py through the host emulation of the mesher kernels, bit-exact against the oracle,
each asserting (from the oracle's frame_voxel_stats) that its voxel reaches the path it is there for.  The emulation runs the
device's split (warp kernel up to 96 vertices with the hand-over, the 256 store-only variant, the 1024 monolithic variant) but
compiles the warp kernel's looped boundary search instead of one_pass; the GPU tier (test_mesh_paths_gpu.py) runs the same
scenes on the device.

    path (mesh_scenes.path_of)         scenes
    warp, one_pass                     patch96, lattice8x8, stacked6x6
    warp, looped boundary search       ring30
    warp, seed triangle only           patch3 (no insertion after the seed)
    warp hand-over -> 1024 variant     ring67, ring95
    k_voxel_mesh<256> (store only)     patch97, patch256, ring100, ring250, lattice16x8, stacked8x8
    k_voxel_mesh<1024> direct          patch256+1 (257), shell_c3 (1008)
    no seed triangle                   collinear12
    IMMESH_E_CAPACITY                  patch300 (> 256 in a voxel), ring300, shell_c4 (dilated set 1260 > 1024)
"""
import numpy as np
import pytest

import mesh_scenes as ms
from immesh_b200 import api
from mesh_common import SMALL, run_scene_parity
from oracle_api import OracleMesh

SCENES = ms.path_scenes()


@pytest.mark.parametrize("scene,path", SCENES, ids=[s.name for s, _ in SCENES])
def test_scene_path_bit_exact(emu_lib, scene, path):
    g, o, stats = run_scene_parity(emu_lib, scene)
    st = ms.centre_stats(stats, scene, scene.cfg_kw["voxel_resolution"])
    assert ms.path_of(st) == path, (scene, st)
    if scene.name.startswith("lattice"):
        assert st["ties"] > 0
    if scene.name.startswith("stacked"):
        assert st["dups"] == scene.n_points // 2
    if path == "noseed":
        assert g.counts()["n_triangles"] == 0


@pytest.mark.parametrize("n_ring", [30, 67, 95, 100, 250])
def test_ring_late_centre_is_the_fan(emu_lib, n_ring):
    """closed form, no oracle: after the centre is appended the live facets are exactly the fan (centre, r_i, r_i+1); no fan
    triangle comes near the 150-degree filter (largest angle 90 - 180/N degrees at the ring)"""
    scene = ms.ring(n_ring)
    g, o, stats = run_scene_parity(emu_lib, scene)
    st = ms.centre_stats(stats, scene, 0.4)
    assert st["n"] == n_ring + 1 and st["max_cav"] == n_ring - 2
    v, t, f = g.snapshot()
    assert np.array_equal(t, ms.ring_fan(n_ring))
    p = v.astype(np.float64)
    for a, b, c in ((t[:, 0], t[:, 1], t[:, 2]), (t[:, 1], t[:, 2], t[:, 0]), (t[:, 2], t[:, 0], t[:, 1])):
        u, w = p[b] - p[a], p[c] - p[a]
        cosv = (u * w).sum(1) / np.linalg.norm(u, axis=1) / np.linalg.norm(w, axis=1)
        assert np.degrees(np.arccos(cosv)).max() < 150 - 45


@pytest.mark.parametrize("scene", ms.cap_scenes(), ids=lambda s: s.name)
def test_caps_raise_capacity(emu_lib, scene):
    """over a per-voxel cap the product refuses the frame (IMMESH_E_CAPACITY) instead of returning a different mesh"""
    cfg = api.MeshConfig(**{**SMALL, **scene.cfg_kw})
    o = OracleMesh(cfg)
    for pts in scene.frames:
        o.push_frame(pts, scene.centre, 0)
    st = ms.centre_stats(o.frame_voxel_stats(), scene, cfg.voxel_resolution)
    in_voxel = o.voxels()[:, 3]
    assert in_voxel.max() > 256 or st["n"] > 1024, st      # the scene is over a cap ...
    if st["n"] > 1024:
        assert in_voxel.max() <= 256                       # ... and the dilation one is not the in-voxel one
    g = api.Mesh(cfg, lib=emu_lib)
    with pytest.raises(RuntimeError, match="code -3"):
        for k, pts in enumerate(scene.frames):
            g.push_frame(pts, scene.centre, k)
    assert emu_lib.emu_mesh_error_word(g._h) == 8   # IM_MERR_VOXEL_CAP alone: no pool or list overflowed
