"""CPU tier: the __host__ __device__ bodies of the localization kernels, executed by the host emulation harness (tests/emu), against
tests/lio_reference.py -- a numpy restatement of the reference's equations that shares nothing with the kernels or the oracle."""
import dataclasses

from immesh_b200 import api
import lio_reference_checks as L


def test_prediction_matches_numpy(emu_lib):
    L.check_prediction(emu_lib)


def test_plane_map_matches_numpy(emu_lib):
    stats = {}
    for kind, cfg, n, off in (("avia", api.AVIA, None, (0.0, 0.0, 0.0)), ("avia", api.AVIA, None, (4000.0, -3000.0, 50.0)),
                              ("avia", api.AVIA, None, (2.0e5, -1.5e5, 30.0)), ("hdl64", api.VELODYNE, 32768, (0.0, 0.0, 0.0))):
        vm, out = L.check_plane_map(emu_lib, kind, cfg, n, off)
        for k, v in vm.stats.items():
            stats[k] = stats.get(k, 0) + v
    assert stats["planar_to_nonplanar"] > 0 and stats["max_points_freeze"] > 0


def test_normal_equations_and_ieskf_iterations_match_numpy(emu_lib):
    layers, iters = set(), {}
    seen = dict(rematch_stop=0, last_iter_stop=0, exp_identity=0, multi=0)
    runs = [(dataclasses.replace(api.AVIA, max_iteration=1), 3, True), (dataclasses.replace(api.AVIA, max_iteration=1, calib_laser=1), 3, True),
            # started at rest, scan 1 of this stream needs 6 iterations: the limit of 4 stops it without convergence, 8 does not
            (dataclasses.replace(api.AVIA, max_iteration=4), 11, False), (dataclasses.replace(api.AVIA, max_iteration=8), 11, False)]
    for cfg, seed, init_vel in runs:
        out = _ieskf(emu_lib, "avia", cfg, 4, seed, init_vel=init_vel)
        layers |= out["layers"]
        iters[cfg.max_iteration] = max(iters.get(cfg.max_iteration, 0), max(out["iters"]))
        for k in seen:
            seen[k] += out[k] if k != "multi" else sum(i > 1 for i in out["iters"])
    assert iters[4] == 4 and iters[8] > 4, iters
    # the one-lane body of k_match (its mode for scans of more than 2 SMs 1024 / 8 points) and the one-step k_residual body
    try:
        for mode in (2, 0):
            emu_lib.emu_lio_set_split(mode)
            _ieskf(emu_lib, "avia", dataclasses.replace(api.AVIA, max_iteration=4), 4, 11, init_vel=False)
    finally:
        emu_lib.emu_lio_set_split(1)
    # the HDL-64 stream at 131 072 points per scan (down-sampled to 8.7 k), velodyne.yaml's 3 m voxels and 4 layers: layers 0 to 3
    out = _ieskf(emu_lib, "hdl64", api.VELODYNE, 3, 7, n_points=131072)
    layers |= out["layers"]
    assert all(v > 0 for v in seen.values()), seen
    assert {0, 1, 2, 3} <= layers, layers


def _ieskf(lib, *args, **kw):
    out = L.check_ieskf(lib, *args, **kw)
    assert out["excluded"] < L.MAX_EXCLUDED * out["n"]
    assert out["compared"] == sum(out["iters"])          # every iteration's normal equations compared
    return out
