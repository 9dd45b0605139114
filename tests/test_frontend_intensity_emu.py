"""CPU tier: the numpy restatement of the VoxelGrid intensity rule (tests/frontend_intensity_common.py) against the oracle's
orc::voxel_grid_filter -- same leaves, same order, same x y z bit for bit; an intensity equal to a coordinate averages to that
coordinate's centroid; the leaf-too-small and non-finite cases; a plain loop on a small cloud."""
import numpy as np
import pytest

import oracle_api as oa
from frontend_intensity_common import intensities, voxel_grid_i
from immesh_b200 import synth


def _check(xyz, leaf, seed=0):
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    inten = intensities(xyz.shape[0], seed)
    rows, small = voxel_grid_i(xyz, inten, leaf)
    ref, ref_small, _ = oa.voxel_grid(xyz, leaf)
    assert small == bool(ref_small)
    assert rows.shape == (ref.shape[0], 4)
    assert np.array_equal(rows[:, :3].view(np.uint32), ref.view(np.uint32))
    # the intensity takes the x y z sums' path: fed the x coordinate, it is the oracle's x centroid
    if xyz.shape[0]:
        as_x, _ = voxel_grid_i(xyz, xyz[:, 0], leaf)
        assert np.array_equal(as_x[:, 3].view(np.uint32), ref[:, 0].view(np.uint32))
    return rows, small


@pytest.mark.parametrize("kind,leaf", [("avia", 0.1), ("avia", 0.4), ("avia", 0.5), ("hdl64", 0.1), ("hdl64", 0.4), ("hdl64", 0.5)])
def test_scan_shapes_match_the_oracle(kind, leaf):
    _, scans = synth.make_stream(kind, 1, seed=4, n_points=20000)
    rows, small = _check(scans[0]["body_full"], leaf, seed=1)
    assert not small and 0 < rows.shape[0] < scans[0]["body_full"].shape[0]


def test_edge_cases():
    rng = np.random.default_rng(2)
    assert voxel_grid_i(np.zeros((0, 3)), np.zeros(0), 0.4)[0].shape == (0, 4)
    one = np.array([[1.5, -2.25, 0.75]], np.float32)
    rows, _ = _check(one, 0.4)
    assert rows[0, 3] == intensities(1, 0)[0]
    same = (rng.uniform(0.01, 0.39, (5000, 3)) + np.array([0.4, -0.8, 1.2])).astype(np.float32)
    assert _check(same, 0.4)[0].shape[0] == 1
    p = rng.normal(0, 3, (30000, 3)).astype(np.float32)
    p[::7] = np.nan
    p[5::11, 1] = np.inf
    _check(p, 0.25)                                                   # non-finite points are dropped with their intensity
    assert voxel_grid_i(np.full((10, 3), np.nan, np.float32), np.ones(10), 0.4)[0].shape == (0, 4)
    wide = rng.uniform(-3000, 3000, (2000, 3)).astype(np.float32)
    wide[3] = np.nan
    inten = intensities(2000, 5)
    rows, small = voxel_grid_i(wide, inten, 0.01)                     # leaf too small: output = input, intensity included
    assert small and np.array_equal(rows[:, :3], wide, equal_nan=True) and np.array_equal(rows[:, 3], inten)
    _check(wide, 0.01, seed=5)


def test_against_a_plain_loop():
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-2, 2, (3000, 3)).astype(np.float32)
    inten = intensities(3000, 9)
    rows, _ = voxel_grid_i(xyz, inten, 0.7)
    inv = np.float32(1) / np.float32(0.7)
    mn, mx = xyz.min(0), xyz.max(0)
    min_b = np.floor(mn * inv).astype(np.int32)
    div_b = np.floor(mx * inv).astype(np.int32) - min_b + 1
    leaves = {}
    for i in range(xyz.shape[0]):
        ijk = [int(np.floor(xyz[i, a] * inv) - np.float32(min_b[a])) for a in range(3)]
        leaves.setdefault(ijk[0] + ijk[1] * int(div_b[0]) + ijk[2] * int(div_b[0] * div_b[1]), []).append(i)
    assert rows.shape[0] == len(leaves)
    for r, key in zip(rows, sorted(leaves)):
        s = np.float32(0)
        for i in leaves[key]:
            s = np.float32(s + inten[i])
        assert r[3] == np.float32(s / np.float32(len(leaves[key])))
