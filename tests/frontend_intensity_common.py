"""Intensity through the front-end: an independent numpy restatement of what PCL's VoxelGrid does with a point's intensity, and the
point records the intensity-carrying (_i) entry points take.  TEST INFRASTRUCTURE.

voxel_grid_i restates pcl::VoxelGrid<PointXYZINormal>::applyFilter with downsample_all_data_ = true (filters/impl/voxel_grid.hpp;
src/voxel_mapping.cpp:1888-1889): the leaf of every finite point from the float box (as oracle/orc_frontend.hpp restates it), the
points grouped by leaf index in ascending order, ascending scan index inside a leaf (the project's defined order), and per leaf
CentroidPoint: x, y, z and intensity (AccumulatorIntensity) summed in float32, one point after the other, divided by (float)count.
It shares no code with the oracle or the CUDA path; tests/test_frontend_intensity_emu.py checks its x y z against
orc::voxel_grid_filter."""
import numpy as np

INT_MAX = 2 ** 31 - 1


def voxel_grid_i(xyz, inten, leaf):
    """(rows float32[m, 4] = x y z intensity, leaf_too_small)"""
    p = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    it = np.ascontiguousarray(inten, dtype=np.float32).reshape(-1)
    fin = np.isfinite(p).all(axis=1)
    if not fin.any():
        return np.zeros((0, 4), np.float32), False
    inv = np.float32(1.0) / np.float32(leaf)
    q, qi = p[fin], it[fin]
    mn, mx = q.min(axis=0), q.max(axis=0)
    d = ((mx - mn) * inv).astype(np.int64) + 1
    if int(d[0]) * int(d[1]) * int(d[2]) > INT_MAX:               # PCL: leaf too small -> output = input
        return np.concatenate([p, it[:, None]], axis=1), True
    min_b = np.floor(mn * inv).astype(np.int32)
    div_b = np.floor(mx * inv).astype(np.int32) - min_b + 1
    ijk = (np.floor(q * inv) - min_b.astype(np.float32)).astype(np.int64)
    idx = ijk[:, 0] + ijk[:, 1] * int(div_b[0]) + ijk[:, 2] * int(div_b[0]) * int(div_b[1])
    order = np.argsort(idx, kind="stable")
    vals = np.concatenate([q, qi[:, None]], axis=1)[order]
    sidx = idx[order]
    starts = np.flatnonzero(np.r_[True, sidx[1:] != sidx[:-1]])
    counts = np.diff(np.r_[starts, sidx.shape[0]])
    acc = np.zeros((starts.shape[0], 4), np.float32)
    for k in range(int(counts.max())):                            # float32 sums, one run position after the other
        sel = counts > k
        acc[sel] += vals[starts[sel] + k]
    return acc / counts.astype(np.float32)[:, None], False


def records(xyz, inten, stride, intensity_col, stamps=None, time_col=None, seed=0):
    """point records of `stride` floats: x y z in 0..2, intensity and stamps in their columns, seeded filler elsewhere"""
    xyz = np.asarray(xyz, dtype=np.float32)
    n = xyz.shape[0]
    r = np.random.default_rng([seed, stride, intensity_col]).normal(size=(n, stride)).astype(np.float32)
    r[:, :3] = xyz
    r[:, intensity_col] = inten
    if stamps is not None:
        r[:, time_col] = stamps
    return r


def intensities(n, seed):
    """a LiDAR-like intensity per point (0..255, not integer-valued, so that the float averages round)"""
    return np.random.default_rng([seed, 7]).uniform(0.0, 255.0, n).astype(np.float32)


LAYOUTS = ((4, 3), (5, 4), (12, 8))   # (stride, intensity_col): x y z i; x y z pad i; pcl::PointXYZINormal


def check_filter_i(vg, xyz, inten, leaf, stride, intensity_col, on_device):
    """immesh_voxelgrid_filter_i on records against voxel_grid_i, and its x y z against immesh_voxelgrid_filter on the same points"""
    rec = records(xyz, inten, stride, intensity_col)
    if on_device:
        import torch
        d = torch.from_numpy(rec).cuda()
        got = vg.filter_i(d.data_ptr(), leaf, intensity_col, n=rec.shape[0], stride=stride, on_device=True)
    else:
        got = vg.filter_i(rec, leaf, intensity_col)
    small = vg.leaf_too_small
    ref, ref_small = voxel_grid_i(xyz, inten, leaf)
    assert small == ref_small
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    plain = vg.filter(xyz, leaf)
    assert np.array_equal(got[:, :3].view(np.uint32), plain.view(np.uint32))
    return got


def run_filter_i_cases(lib):
    """the scan shapes and edge cases of the GPU tier, in whatever centroid mode the process runs"""
    from immesh_b200 import api, synth
    vg = api.VoxelGrid(1 << 17, lib=lib)
    rng = np.random.default_rng(8)
    for kind in ("avia", "hdl64"):
        _, scans = synth.make_stream(kind, 1, seed=6, n_points=60000)
        xyz = scans[0]["body_full"]
        for leaf, (stride, col), dev in ((0.1, LAYOUTS[2], False), (0.4, LAYOUTS[1], True), (0.5, LAYOUTS[0], False)):
            check_filter_i(vg, xyz, intensities(xyz.shape[0], 3), leaf, stride, col, dev)
    same = (rng.uniform(0.01, 0.39, (5000, 3)) + np.array([0.4, -0.8, 1.2])).astype(np.float32)
    assert check_filter_i(vg, same, intensities(5000, 4), 0.4, 12, 8, False).shape[0] == 1
    p = rng.normal(0, 3, (30000, 3)).astype(np.float32)
    p[::7] = np.nan
    p[5::11, 1] = np.inf
    check_filter_i(vg, p, intensities(30000, 5), 0.25, 5, 4, True)
    wide = rng.uniform(-3000, 3000, (2000, 3)).astype(np.float32)
    check_filter_i(vg, wide, intensities(2000, 6), 0.01, 12, 8, False)
    assert vg.leaf_too_small
    vg.close()
