"""GPU tier: the CUDA localization path through the C ABI against tests/lio_reference.py, the numpy restatement of the reference's
equations that shares nothing with the kernels or the oracle (the same checks as tests/test_lio_reference_emu.py, plus the C-ABI
calls the emulation does not have)."""
import dataclasses

import pytest

from immesh_b200 import api
import lio_reference_checks as L

pytestmark = pytest.mark.gpu


def test_prediction_matches_numpy(cuda_lib):
    L.check_prediction(cuda_lib)


def test_plane_map_matches_numpy(cuda_lib):
    stats = {}
    for kind, cfg, n, off in (("avia", api.AVIA, None, (0.0, 0.0, 0.0)), ("avia", api.AVIA, None, (4000.0, -3000.0, 50.0)),
                              ("avia", api.AVIA, None, (2.0e5, -1.5e5, 30.0)), ("hdl64", api.VELODYNE, 32768, (0.0, 0.0, 0.0))):
        vm, out = L.check_plane_map(cuda_lib, kind, cfg, n, off)
        for k, v in vm.stats.items():
            stats[k] = stats.get(k, 0) + v
    assert stats["planar_to_nonplanar"] > 0 and stats["max_points_freeze"] > 0


def test_residual_selection_matches_numpy(cuda_lib):
    # immesh_residual_build (the one-thread walk of k_residual) on down-sampled Avia scans (7 k and 19 k points) and the HDL-64 scan
    # with max_layer 4 (8.7 k points); k_match is compared through the estimation test below
    tot = {}
    for kind, cfg, n, seed in (("avia", api.AVIA, None, 5), ("avia", api.AVIA, 100_000, 6), ("hdl64", api.VELODYNE, 131072, 7)):
        out = L.check_residual_build(cuda_lib, kind, cfg, n, seed)
        assert out["excluded"] < L.MAX_EXCLUDED * out["n"]
        for k, v in out.items():
            tot[k] = (tot.get(k, set()) | v) if isinstance(v, set) else tot.get(k, 0) + v
    assert tot["range_reject"] > 0 and tot["sigma_reject"] > 0 and tot["retry_success"] > 0 and tot["non_first_argmax"] > 0
    assert {0, 1, 2, 3} <= tot["layers"], tot["layers"]


def test_normal_equations_and_ieskf_iterations_match_numpy(cuda_lib):
    layers, iters = set(), {}
    seen = dict(rematch_stop=0, last_iter_stop=0, exp_identity=0, multi=0, weights=0)
    runs = [(dataclasses.replace(api.AVIA, max_iteration=1), 3, True), (dataclasses.replace(api.AVIA, max_iteration=1, calib_laser=1), 3, True),
            # started at rest, scan 1 of this stream needs 6 iterations: the limit of 4 stops it without convergence, 8 does not
            (dataclasses.replace(api.AVIA, max_iteration=4), 11, False), (dataclasses.replace(api.AVIA, max_iteration=8), 11, False)]
    for cfg, seed, init_vel in runs:
        out = _ieskf(cuda_lib, "avia", cfg, 4, seed, init_vel=init_vel)
        layers |= out["layers"]
        iters[cfg.max_iteration] = max(iters.get(cfg.max_iteration, 0), max(out["iters"]))
        for k in seen:
            seen[k] += out[k] if k != "multi" else sum(i > 1 for i in out["iters"])
    assert iters[4] == 4 and iters[8] > 4, iters
    # full-resolution Avia scans of more than 2 SMs 1024 / 8 points (33 792 on 132 SMs): k_match's one-lane mode; the down-sampled
    # scans above (7 k points) run its 8-lane mode
    out = _ieskf(cuda_lib, "avia", api.AVIA, 3, 6, n_points=100_000, full=True)
    assert min(out["scan_points"]) > 2 * 132 * 1024 // 8, out["scan_points"]
    layers |= out["layers"]
    # the HDL-64 stream at 131 072 points per scan (down-sampled to 8.7 k), velodyne.yaml's 3 m voxels and 4 layers: layers 0 to 3
    out = _ieskf(cuda_lib, "hdl64", api.VELODYNE, 3, 7, n_points=131072)
    layers |= out["layers"]
    assert all(v > 0 for v in seen.values()), seen
    assert {0, 1, 2, 3} <= layers, layers


def _ieskf(lib, *args, **kw):
    out = L.check_ieskf(lib, *args, **kw)
    assert out["excluded"] < L.MAX_EXCLUDED * out["n"]
    assert out["compared"] == sum(out["iters"])          # every iteration's normal equations compared
    return out


def test_fixed_point_sums_of_a_dense_wall(cuda_lib):
    L.check_fixed_point_range(cuda_lib)


def test_pv_lists_store_float_world_points(cuda_lib):
    L.check_pv_float_rounding(cuda_lib)


def test_residual_build_pv_keeps_double_world_points(cuda_lib):
    L.check_residual_build_pv(cuda_lib)
