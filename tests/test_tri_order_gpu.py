"""GPU tier: the order in which immesh_mesh_snapshot, immesh_mesh_region_stream, immesh_mesh_region_buffers and immesh_mesh_evaluate
return the live triangles, in the cases the other tests do not reach: region keys past +-1048000, an empty mesh, and vertex ids past
2^16 (three 8-bit digits per vertex id)."""
import numpy as np
import pytest

from immesh_b200 import api
from mesh_common import run_mesh_parity, world_scans, SMALL

pytestmark = pytest.mark.gpu


def region_keys(v, t, region_size):
    """tri_region_key in float64: round(((a + b) + c) / 3 / region_size) per axis, halves away from zero as C's round()."""
    v = v.astype(np.float64)
    x = ((v[t[:, 0]] + v[t[:, 1]]) + v[t[:, 2]]) / 3.0 / region_size
    a = np.abs(x)
    r = np.floor(a)
    r += (a - r) >= 0.5
    return (np.sign(x) * r).astype(np.int64)


def check_region_stream(mesh, region_size):
    """region_stream against the snapshot: regions by ascending key, triangles by ascending triple inside a region."""
    v, t, _ = mesh.snapshot()
    k = region_keys(v, t, region_size)
    order = np.lexsort((t[:, 2], t[:, 1], t[:, 0], k[:, 2], k[:, 1], k[:, 0]))
    ref_keys, first = np.unique(k[order], axis=0, return_index=True)
    keys, offs, tris = mesh.region_stream(region_size, cap=len(t) + 1)
    assert np.array_equal(tris, t[order])
    assert np.array_equal(keys, ref_keys) and np.array_equal(offs[:-1], np.sort(first)) and offs[-1] == len(t)
    return k


def test_region_stream_beyond_packed_key_range(cuda_lib):
    """A mesh far from the origin and a region size whose keys pass +-1048000 on two axes, with both signs: region_stream orders the
    triangles by the exact int keys; region_buffers, whose keys are packed in 21 bits per axis, refuses the size."""
    offset = np.array([3000.0, -2500.0, 40.0])
    g = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    for k, (world, t) in enumerate(world_scans("avia", 2, seed=21)):
        g.push_frame((world.astype(np.float64) + offset).astype(np.float32), t + offset, k)
    assert g.counts()["n_triangles"] > 1000
    keys = check_region_stream(g, 0.002)
    assert (keys[:, 0] > 1048000).all() and (keys[:, 1] < -1048000).all()
    check_region_stream(g, 10.0)
    with pytest.raises(RuntimeError, match="code -5"):
        g.region_buffers(0.002)


def test_empty_mesh(cuda_lib):
    """No triangle: snapshot, region_stream, region_buffers and evaluate return empty results."""
    g = api.Mesh(api.MeshConfig(**SMALL), lib=cuda_lib)
    v, t, f = g.snapshot()
    assert v.shape == (0, 3) and t.shape == (0, 3) and f.shape == (0,)
    keys, offs, tris = g.region_stream(10.0)
    assert keys.shape == (0, 3) and np.array_equal(offs, [0]) and tris.shape == (0, 3)
    xyz, ids, rkeys, roff, ns = g.region_buffers(10.0)
    assert xyz.shape == (0, 9) and ids.shape == (0, 3) and rkeys.shape == (0, 3) and np.array_equal(roff, [0]) and ns == 0
    gt = np.array([[0.0, 0.0, 1.0], [1.0, 2.0, 3.0]], dtype=np.float32)
    r = g.evaluate(gt, facets=True)
    assert r["counts"]["live_triangles"] == 0 and r["rows"].shape == (0, 5)


def test_vertex_ids_past_two_to_the_sixteen(cuda_lib):
    """More than 2^16 vertices, so each vertex word of the triple sort takes three passes: the snapshot against the oracle, the region
    stream against its restatement, the evaluation's facet rows in the snapshot's order."""
    g, _, _ = run_mesh_parity(cuda_lib, "hdl64", 3, seed=3, cfg_kw={"number_of_pts_append_to_map": 100000})
    _, t, _ = g.snapshot()
    assert g.counts()["n_vertices"] > 1 << 16 and t.max() >= 1 << 16
    check_region_stream(g, 10.0)
    check_region_stream(g, 1.0)
    xyz, ids, _, roff, _ = g.region_buffers(10.0)
    keys, offs, tris = g.region_stream(10.0, cap=len(t) + 1)
    assert np.array_equal(ids, tris) and np.array_equal(roff, offs)
    r = g.evaluate(np.zeros((1, 3), dtype=np.float32), spacing=0.5, gt_leaf=0.0, facets=True)
    assert np.array_equal(r["rows"][:, :3], t)
