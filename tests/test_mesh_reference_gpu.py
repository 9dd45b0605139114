"""GPU tier: the CUDA mesher through the C ABI against tests/mesh_reference.py, the numpy restatement of one
incremental_mesh_reconstruction frame that shares nothing with the kernels or the oracle (the streams of
tests/test_mesh_reference_emu.py, one step at a time, by push_frame and by push_frame_batched in small batches).  The device does not
expose its work list, so the meshed voxels are compared through their number; the smoothed positions are compared at the end of each
stream through one all-regions region_buffers call."""
import dataclasses

import pytest

import mesh_reference_checks as K
import mesh_scenes
from immesh_b200 import api
from mesh_common import SMALL

pytestmark = pytest.mark.gpu

CFG = api.MeshConfig(**SMALL)


def streams():
    return [
        ("avia", K.stream("avia", 6, 0), CFG),
        ("avia_step5", K.stream("avia", 3, 1), dataclasses.replace(CFG, number_of_pts_append_to_map=4000)),
        ("hdl64", K.stream("hdl64", 4, 2, n_points=65536), CFG),
        ("avia_res0.2", K.stream("avia", 3, 3), dataclasses.replace(CFG, voxel_resolution=0.2)),
        ("avia_res0.8", K.stream("avia", 3, 4), dataclasses.replace(CFG, voxel_resolution=0.8)),
        ("avia_far", K.stream("avia", 4, 0, offset=(4000.0, -3000.0, 50.0)), CFG),
    ]


def _batched(h, pts, cam, k):
    # a few hundred voxels per batch and 4096 candidates per append chunk: several batches and chunks per frame
    h.push_frame_batched(pts, cam, batch_points=4096, batch_voxels=256)


@pytest.mark.parametrize("mode", ["push_frame", "batched"])
def test_streams_match_numpy(cuda_lib, mode):
    tot = {}
    for name, frames, cfg in streams():
        st = K.check_stream(cuda_lib, frames, cfg, push=_batched if mode == "batched" else None)
        rows = K.end_smooth_check(st["handle"], st["ref"])
        print(f"{name} ({mode}): {st['excluded']} of {st['meshed']} meshed voxels excluded, {st['flips_excluded']} of "
              f"{st['flips_excluded'] + st['flips_compared']} flips excluded, {rows} smoothed rows compared")
        assert rows > 0
        K.merge(tot, st)
    assert all(tot[b] > 0 for b in K.BRANCHES), {b: tot[b] for b in K.BRANCHES}


def test_path_scenes_match_numpy(cuda_lib):
    tot = {}
    for sc in (mesh_scenes.jittered_patch(96, seed=3), mesh_scenes.jittered_patch(97, seed=4), mesh_scenes.jittered_patch(256, seed=5),
               mesh_scenes.jittered_patch(256, seed=6, extra_outside=True)):
        cfg = api.MeshConfig(**{**SMALL, **sc.cfg_kw})
        st = K.check_stream(cuda_lib, K.scene_frames(sc), cfg)
        K.end_smooth_check(st["handle"], st["ref"])
        K.merge(tot, st)
    assert {"warp", "block256", "block1024"} <= set(tot["size_class"]), tot["size_class"]


def test_append_ties_at_xi(cuda_lib):
    """points exactly xi apart are appended, in the frame and against the map (the reference's test is sqrt(d) < xi)"""
    sc = mesh_scenes.xi_tie()
    st = K.check_stream(cuda_lib, K.scene_frames(sc), api.MeshConfig(**{**SMALL, **sc.cfg_kw}), xi_ties=True)
    assert st["xi_margin"] == 0.0 and st["handle"].counts()["n_vertices"] == 3
