"""CPU tier of the mesh evaluation (immesh_mesh_evaluate): the shipped per-element bodies (immesh_b200/csrc/mesh_eval.cuh) run on the
host by tests/eval/emu_eval.cpp, against the independent numpy restatement (tests/mesh_eval_reference.py) and known answers."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import mesh_eval_reference as ref  # noqa: E402
from immesh_b200 import build  # noqa: E402

CFG = dict(spacing=0.01, gt_leaf=0.01, threshold=0.05, max_dist=1.0, incorrect_ratio=0.8)


@pytest.fixture(scope="module")
def lib():
    lib = C.CDLL(build.build_eval())
    lib.emu_evaluate.restype = C.c_int
    lib.emu_evaluate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_longlong] + [C.c_double] * 5 + [C.c_void_p] * 4 + [C.c_longlong, C.c_void_p, C.c_longlong]
    return lib


def emu(lib, verts, tris, gt, spacing=0.01, gt_leaf=0.01, threshold=0.05, max_dist=1.0, incorrect_ratio=0.8):
    v = np.ascontiguousarray(verts, dtype=np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(tris, dtype=np.int32).reshape(-1, 3)
    g = np.ascontiguousarray(gt, dtype=np.float32).reshape(-1, 3)
    counts, metrics = np.zeros(12, dtype=np.int64), np.zeros(8)
    rows = np.zeros((max(len(t), 1), 5), dtype=np.int32)
    cap = 1 << 20
    samples, gout = np.zeros((cap, 4), dtype=np.float32), np.zeros((max(len(g), 1), 3), dtype=np.float32)
    rc = lib.emu_evaluate(v.ctypes.data, t.ctypes.data, len(t), g.ctypes.data, len(g), spacing, gt_leaf, threshold, max_dist, incorrect_ratio,
                          counts.ctypes.data, metrics.ctypes.data, rows.ctypes.data, samples.ctypes.data, cap, gout.ctypes.data, len(gout))
    if rc:
        return rc
    return dict(counts=counts, metrics=metrics, rows=rows[:len(t)], samples=samples[:counts[2]], gt=gout[:counts[3]])


def check_same(e, r):
    assert np.array_equal(e["counts"], r["counts"]), (e["counts"], r["counts"])
    assert np.array_equal(e["rows"], r["rows"])
    assert np.allclose(e["metrics"][:2], r["metrics"][:2], rtol=1e-12, atol=0, equal_nan=True)
    assert np.array_equal(e["metrics"][2:], r["metrics"][2:], equal_nan=True)
    assert np.array_equal(e["samples"][:, :3], r["samples"])
    assert np.array_equal(e["samples"][:, 3].astype(np.int64), r["sample_facet"])
    assert np.array_equal(np.unique(e["gt"], axis=0), np.unique(r["gt"], axis=0))


def unit_square():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], dtype=np.float32)
    t = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    return v, t


def test_unit_square_offset_within(lib):
    v, t = unit_square()
    s = ref.evaluate(v, t, np.zeros((0, 3)), spacing=0.05, gt_leaf=0)["samples"]
    gt = s + np.array([0, 0, 0.02], dtype=np.float32)
    e = emu(lib, v, t, gt, spacing=0.05, gt_leaf=0)
    check_same(e, ref.evaluate(v, t, gt, spacing=0.05, gt_leaf=0))
    tol = 2.0 ** -20 + 1e-8
    assert abs(e["metrics"][2] - 0.02) <= tol and abs(e["metrics"][3] - 0.02) <= tol
    assert e["metrics"][4] == 1 and e["metrics"][5] == 1 and e["metrics"][6] == 1
    assert e["counts"][8] == 0 and e["counts"][6] == 0 and e["counts"][7] == 0


def test_unit_square_offset_beyond(lib):
    v, t = unit_square()
    s = ref.evaluate(v, t, np.zeros((0, 3)), spacing=0.05, gt_leaf=0)["samples"]
    gt = s + np.array([0, 0, 0.06], dtype=np.float32)
    e = emu(lib, v, t, gt, spacing=0.05, gt_leaf=0)
    check_same(e, ref.evaluate(v, t, gt, spacing=0.05, gt_leaf=0))
    assert e["metrics"][4] == 0 and e["metrics"][5] == 0 and e["metrics"][6] == 0
    assert e["counts"][8] == 2   # every facet incorrect


def test_equilateral(lib):
    h = np.float32(np.sqrt(3.0) / 2)
    v = np.array([[0, 0, 0], [1, 0, 0], [0.5, h, 0]], dtype=np.float32)
    e = emu(lib, v, [[0, 1, 2]], v, spacing=0.1)
    assert abs(e["metrics"][0]) < 1e-5
    assert abs(e["metrics"][1] - 1 / np.sqrt(3)) < 1e-6
    check_same(e, ref.evaluate(v, [[0, 1, 2]], v, spacing=0.1))


def test_degenerate_sliver_and_single_subdivision(lib):
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0],            # collinear: degenerate
                  [0, 1, 0], [1, 1, 0.001], [0.5, 1.0001, 0],   # sliver
                  [5, 5, 5], [5.004, 5, 5], [5, 5.004, 5],      # n = 1
                  [3, 3, 3]], dtype=np.float32)
    t = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [6, 8, 9]], dtype=np.int32)
    rng = np.random.default_rng(3)
    gt = np.concatenate([v + rng.normal(0, 0.02, v.shape), rng.uniform(-1, 6, (300, 3))]).astype(np.float32)
    e = emu(lib, v, t, gt)
    check_same(e, ref.evaluate(v, t, gt))
    assert e["counts"][1] == 1 and e["rows"][0, 3] == 0
    assert e["rows"][2, 3] == 1   # n = 1: one sample, the centroid


def test_negative_coordinates_and_leaf_boundaries(lib):
    v = np.array([[-1.0, -1.0, -0.5], [-0.5, -1.0, -0.5], [-1.0, -0.5, -0.25]], dtype=np.float32)
    # points exactly on leaf boundaries (multiples of the power-of-two leaf) and just below them: floor, not truncation
    base = np.array([[-0.75, -0.875, -0.5], [-0.5, -1.0, -0.375], [-1.0, -0.5, -0.25], [0.0, -0.0, 0.125]], dtype=np.float32)
    below = np.nextafter(base, np.float32(-np.inf))
    gt = np.concatenate([base, below, base]).astype(np.float32)
    for leaf in (0.125, 0.0625, 0.0):
        e = emu(lib, v, [[0, 1, 2]], gt, spacing=0.05, gt_leaf=leaf)
        r = ref.evaluate(v, [[0, 1, 2]], gt, spacing=0.05, gt_leaf=leaf)
        check_same(e, r)
    # floor(-2.0) = floor(-1.04) = -2: one leaf (truncation would give -2 and -1)
    assert ref.downsample(np.array([[-0.5, 0, 0], [-0.26, 0, 0]], np.float32), 0.25).shape[0] == 1
    e = emu(lib, v, [[0, 1, 2]], np.array([[-0.5, 0, 0], [-0.26, 0, 0]], np.float32), spacing=0.05, gt_leaf=0.25)
    assert e["counts"][3] == 1


def test_distance_equal_to_threshold_and_beyond_max_dist(lib):
    # one triangle with n = 1: its only sample is the centroid; ground truth exactly threshold above it, and one beyond max_dist
    v = np.array([[0, 0, 0], [0.0078125, 0, 0], [0, 0.0078125, 0]], dtype=np.float32)
    c = ref.evaluate(v, [[0, 1, 2]], np.zeros((0, 3)), spacing=0.01, gt_leaf=0)["samples"][0]
    gt = np.array([c + np.float32([0, 0, 0.25]), c + np.float32([0, 0, 3.0])], dtype=np.float32)
    assert ref.dist(gt[0][None], c[None])[0] == 0.25
    e = emu(lib, v, [[0, 1, 2]], gt, spacing=0.01, gt_leaf=0, threshold=0.25, max_dist=1.0)
    check_same(e, ref.evaluate(v, [[0, 1, 2]], gt, spacing=0.01, gt_leaf=0, threshold=0.25, max_dist=1.0))
    assert e["counts"][4] == 0 and e["counts"][5] == 0   # d == threshold is not within
    assert e["counts"][7] == 1 and e["counts"][6] == 0    # the far point takes max_dist
    assert e["counts"][10] == 2 ** 18 + 2 ** 20


def test_empty_mesh_and_empty_ground_truth(lib):
    v, t = unit_square()
    gt = np.array([[0.5, 0.5, 0.01], [2, 2, 2]], dtype=np.float32)
    e = emu(lib, v, np.zeros((0, 3)), gt)
    check_same(e, ref.evaluate(v, np.zeros((0, 3)), gt))
    assert e["counts"][2] == 0 and e["counts"][7] == 2 and np.isnan(e["metrics"][0]) and np.isnan(e["metrics"][2])
    e = emu(lib, v, t, np.zeros((0, 3)), spacing=0.1)
    check_same(e, ref.evaluate(v, t, np.zeros((0, 3)), spacing=0.1))
    assert e["counts"][6] == e["counts"][2] == 2 * 15 * 15 and np.isnan(e["metrics"][3]) and np.isnan(e["metrics"][6])


def test_random_meshes_against_reference(lib):
    rng = np.random.default_rng(11)
    for trial in range(4):
        v = rng.uniform(-2, 2, (30, 3)).astype(np.float32)
        t = np.sort(rng.choice(30, (12, 3), replace=True), axis=1)
        t = t[(t[:, 0] < t[:, 1]) & (t[:, 1] < t[:, 2])]
        t = np.unique(t, axis=0).astype(np.int32)
        gt = (v[rng.integers(0, 30, 2000)] + rng.normal(0, 0.3, (2000, 3))).astype(np.float32)
        cfg = dict(spacing=0.15, gt_leaf=(0.05, 0.0, 0.2, 0.1)[trial], threshold=0.1, max_dist=0.4, incorrect_ratio=0.5)
        check_same(emu(lib, v, t, gt, **cfg), ref.evaluate(v, t, gt, **cfg))


def test_subdivision_range_and_sample_enumeration(lib):
    v = np.array([[0, 0, 0], [400, 0, 0], [0, 1, 0]], dtype=np.float32)
    assert emu(lib, v, [[0, 1, 2]], np.zeros((0, 3)), spacing=0.01) == -5   # n = 40000 > 2^15
    v = np.array([[0, 0, 0], [1, 0.1, 0], [0.2, 1, 0.3]], dtype=np.float32)
    e = emu(lib, v, [[0, 1, 2]], np.zeros((0, 3)), spacing=0.013)
    n = e["counts"][11]
    assert e["counts"][2] == n * n and len(np.unique(e["samples"][:, :3], axis=0)) == n * n
