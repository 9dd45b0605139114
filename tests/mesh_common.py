"""Shared driver for the mesher parity tests: the same world-frame scan stream through an implementation under
test and the oracle; vertex ids/positions, voxel activation counts, the live facet set and its orientation flags
must be identical after every frame."""
import numpy as np

from immesh_b200 import api, synth
from oracle_api import OracleMesh

SMALL = dict(max_vertices=1 << 19, max_triangles=1 << 21, max_voxels=1 << 17, max_frame_points=1 << 18)


def world_scans(kind, n_frames, seed, n_points=None):
    sensor, scans = synth.make_stream(kind, n_frames, seed=seed, n_points=n_points)
    out = []
    for s in scans:
        R, t = s["R_true"], s["t_true"]
        out.append(((s["body_full"].astype(np.float64) @ R.T + t).astype(np.float32), t))
    return out


def run_scene_parity(lib, scene):
    """A tests/mesh_scenes.py scene through the implementation under test and the oracle, frame by frame, bit-exact as in
    run_mesh_parity.  Returns (impl, oracle, the oracle's frame_voxel_stats of the last frame)."""
    cfg = api.MeshConfig(**{**SMALL, **scene.cfg_kw})
    g, o = api.Mesh(cfg, lib=lib), OracleMesh(cfg)
    pose = scene.centre + np.array([0.3, -0.2, 1.5])   # the camera: above the scene, as the orientation flags need one
    for k, pts in enumerate(scene.frames):
        g.push_frame(pts, pose, k)
        o.push_frame(pts, pose, k)
        cg, co = g.counts(), o.counts()
        assert cg == co, f"{scene} frame {k}: counts {cg} vs {co}"
        vg, tg, fg = g.snapshot()
        vo, to, fo = o.snapshot()
        assert np.array_equal(vg, vo), f"{scene} frame {k}: vertex positions / ids"
        assert tg.shape == to.shape and np.array_equal(tg, to), f"{scene} frame {k}: facet set"
        assert np.array_equal(fg, fo), f"{scene} frame {k}: orientation flags"
    assert g.counts()["n_vertices"] == scene.n_points, f"{scene}: every point must become a vertex"
    return g, o, o.frame_voxel_stats()


def run_mesh_parity(lib, kind, n_frames, seed, cfg_kw=None, n_points=None, check_every=1):
    cfg = api.MeshConfig(**{**SMALL, **(cfg_kw or {})})
    g, o = api.Mesh(cfg, lib=lib), OracleMesh(cfg)
    stats = []
    for k, (world, t) in enumerate(world_scans(kind, n_frames, seed, n_points)):
        g.push_frame(world, t, k)
        o.push_frame(world, t, k)
        cg, co = g.counts(), o.counts()
        assert cg == co, f"frame {k}: counts {cg} vs {co}"
        if k % check_every == 0 or k == n_frames - 1:
            vg, tg, fg = g.snapshot()
            vo, to, fo = o.snapshot()
            assert np.array_equal(vg, vo), f"frame {k}: vertex positions / ids"
            assert tg.shape == to.shape and np.array_equal(tg, to), f"frame {k}: facet set"
            assert np.array_equal(fg, fo), f"frame {k}: orientation flags"
        stats.append(cg)
    return g, o, stats
