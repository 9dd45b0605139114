"""CPU tier: the __host__ __device__ bodies of the mesher, executed by the host emulation (tests/pubmap/emu_region_buf.cpp: the
mesher emulation with the smoothed-position flags), against tests/mesh_reference.py -- a numpy restatement of one
incremental_mesh_reconstruction frame that shares nothing with the kernels or the oracle.  Every frame is compared one step at a time
(tests/mesh_reference_checks.py): vertices, counts and the meshed voxels exactly, facets and flips outside the stated exclusions, and
the smoothed positions and their flags after every frame."""
import dataclasses

import pytest

import mesh_reference_checks as K
import mesh_scenes
from immesh_b200 import api
from mesh_common import SMALL
from region_buffers_common import emu_regionbuf_lib

CFG = api.MeshConfig(**SMALL)


@pytest.fixture(scope="module")
def emu_lib():
    return emu_regionbuf_lib()


def streams():
    """(name, frames, config): the Avia stream (append step 2), with a smaller append target (step 5), the HDL-64 stream at 65 536
    points, voxel resolutions 0.2 and 0.8 m, the Avia stream translated by (4000, -3000, 50) m"""
    return [
        ("avia", K.stream("avia", 6, 0), CFG),
        ("avia_step5", K.stream("avia", 3, 1), dataclasses.replace(CFG, number_of_pts_append_to_map=4000)),
        ("hdl64", K.stream("hdl64", 2, 2, n_points=65536), CFG),
        ("avia_res0.2", K.stream("avia", 2, 3), dataclasses.replace(CFG, voxel_resolution=0.2)),
        ("avia_res0.8", K.stream("avia", 3, 4), dataclasses.replace(CFG, voxel_resolution=0.8)),
        ("avia_far", K.stream("avia", 3, 0, offset=(4000.0, -3000.0, 50.0)), CFG),
    ]


def test_streams_match_numpy(emu_lib):
    tot = {}
    for name, frames, cfg in streams():
        st = K.check_stream(emu_lib, frames, cfg, emu=True)
        print(f"{name}: {st['excluded']} of {st['meshed']} meshed voxels excluded, {st['flips_excluded']} of "
              f"{st['flips_excluded'] + st['flips_compared']} flips excluded, {st['tris_compared']} facets compared")
        K.merge(tot, st)
    missing = [b for b in K.BRANCHES if b not in ("claimed_twice",) and tot[b] == 0]
    assert not missing, missing
    assert tot["claimed_twice"] > 0
    # the dilated-set sizes of real streams stay in the warp class; the block classes come from the scenes below
    assert tot["size_class"].get("warp", 0) > 0


def test_path_scenes_match_numpy(emu_lib):
    """general-position scenes of tests/mesh_scenes.py: jittered patches of 96 / 97 / 256 / 256 + 1 points, dilated sets in all
    three kernel size classes (<= 96 warp, 97-256 k_voxel_mesh<256>, 257-1024 k_voxel_mesh<1024>).  The shell scene is left out: its
    dilated sets are pieces of a cube's surface, whose covariance has no usable gap between its two smallest eigenvalues, so every
    one of its voxels is excluded by the normal bound."""
    tot = {}
    for sc in (mesh_scenes.jittered_patch(96, seed=3), mesh_scenes.jittered_patch(97, seed=4), mesh_scenes.jittered_patch(256, seed=5),
               mesh_scenes.jittered_patch(256, seed=6, extra_outside=True)):
        cfg = api.MeshConfig(**{**SMALL, **sc.cfg_kw})
        st = K.check_stream(emu_lib, K.scene_frames(sc), cfg, emu=True)
        K.merge(tot, st)
    assert {"warp", "block256", "block1024"} <= set(tot["size_class"]), tot["size_class"]


def test_append_ties_at_xi(emu_lib):
    """points exactly xi apart are appended, in the frame and against the map (the reference's test is sqrt(d) < xi)"""
    sc = mesh_scenes.xi_tie()
    st = K.check_stream(emu_lib, K.scene_frames(sc), api.MeshConfig(**{**SMALL, **sc.cfg_kw}), emu=True, xi_ties=True)
    assert st["xi_margin"] == 0.0 and st["handle"].counts()["n_vertices"] == 3
