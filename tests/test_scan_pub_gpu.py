"""GPU tier: immesh_lio_effect_cloud / immesh_lio_registered_cloud (publish_effect_world / publish_frame_world) through the C ABI
against the oracle on every path that forms the IESKF weights: the staged calls, the fused step, the pipelined graph-replayed step
and its direct launches, k_match at 8 and at 1 lane per point, the raw device chain; the dense cloud from the device (the
calibrated input of the raw chain, the IMU chain's [n][4] output); the capacity contract, the validity rules and an empty scan."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oracle_api as oa
from immesh_b200 import api, synth
from lio_common import init_velocity
from scan_pub_common import ScanPubOracle, run_scan_pub_parity

pytestmark = pytest.mark.gpu
E_INVALID, E_CAPACITY = -1, -3


def test_staged_calls(cuda_lib):
    assert min(run_scan_pub_parity(cuda_lib, "avia", api.AVIA, n_scans=8, seed=0)) > 100
    assert min(run_scan_pub_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768)) > 100


def test_fused_step(cuda_lib):
    run_scan_pub_parity(cuda_lib, "avia", api.AVIA, n_scans=6, seed=2, mode="step", oracle_checks=False)


def test_pipelined_graph_path(cuda_lib):
    run_scan_pub_parity(cuda_lib, "avia", api.AVIA, n_scans=8, seed=6, mode="async", oracle_checks=False)
    run_scan_pub_parity(cuda_lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768, mode="async", oracle_checks=False)


def test_pipelined_direct_launches(cuda_lib, monkeypatch):
    monkeypatch.setenv("IMMESH_GRAPH", "0")    # read when a handle is created
    run_scan_pub_parity(cuda_lib, "avia", api.AVIA, n_scans=6, seed=7, mode="async", oracle_checks=False)


def test_k_match_both_lane_modes(cuda_lib):
    """scan 1 above 256 * SMs points (k_match with 1 lane per point), scan 2 truncated to exactly that (8 lanes), scan 3 to one more"""
    import torch
    thr = 256 * torch.cuda.get_device_properties(0).multi_processor_count
    cfg = api.LioConfig(filter_size_surf=0.1)
    _, scans = synth.make_stream("avia100k", 2, seed=0, leaf=0.1, ext_T=cfg.ext_T)
    assert scans[1]["body_ds"].shape[0] > thr + 1
    counts = run_scan_pub_parity(cuda_lib, "avia100k", cfg, n_scans=4, seed=0, body_len={2: thr, 3: thr + 1}, oracle_checks=False)
    assert min(counts) > 1000


def test_raw_device_chain_and_its_dense_cloud(cuda_lib):
    """immesh_lio_step_async_raw (calibration -> VoxelGrid -> localization, the count device resident): effect rows and the
    down-sampled cloud against the oracle, and the dense cloud read from immesh_voxelgrid_input_points (the calibrated full scan)"""
    cfg = dataclasses.replace(api.VELODYNE, calib_laser=1)
    sensor, scans = synth.make_stream("hdl64", 4, seed=12, leaf=cfg.filter_size_surf, n_points=65536)
    g, o = api.Lio(cfg, lib=cuda_lib), ScanPubOracle(cfg)
    vg = api.VoxelGrid(1 << 17, lib=cuda_lib)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(oa.kitti_calib(scans[0]["body_full"]))
    for k in (1, 2, 3):
        raw = scans[k]["body_full"]
        vg.step_async_raw(g, raw, cfg.filter_size_surf, dt=scans[k]["dt"], calib_laser=True)
        full = oa.kitti_calib(raw)
        ds, _, _ = oa.voxel_grid(full, cfg.filter_size_surf)
        o.predict(scans[k]["dt"])
        o.lio_state_estimation(ds)
        o.map_incremental_grow(ds)
        rg, ig = g.effect_cloud()
        ro, io = o.effect_cloud()
        assert rg.shape[0] > 100 and np.array_equal(ig, io) and np.array_equal(rg.view(np.uint32), ro.view(np.uint32)), k
        for skip in (1, 3):
            assert np.array_equal(g.registered_cloud(None, point_skip=skip), o.frame_world(ds, skip)), k
            dense = g.registered_cloud(vg.input_points(), point_skip=skip, on_device=True, n=raw.shape[0], stride=3)
            assert np.array_equal(dense, o.frame_world(full, skip)), k
    g.wait()
    assert np.array_equal(g.get_state(), o.get_state())


def test_imu_chain_output_as_dense_cloud(cuda_lib):
    """the IMU front-end's undistorted [n][4] output (x y z t) in device memory, stride 4, no intensity"""
    from test_imu_emu import _imu_cfg, _make_scan
    rng = np.random.default_rng(11)
    icfg = _imu_cfg(rng)
    lio = api.Lio(api.AVIA, lib=cuda_lib)
    s0 = lio.get_state()
    s0[12:15] = [0.5, -0.2, 0.05]
    s0[21:24] = [0.0, 0.0, -9.81]
    lio.set_state(s0)
    g, oi = api.Imu(icfg, lib=cuda_lib), oa.OracleImu(icfg)
    t0 = 100.0
    last = np.array([t0 - 0.002, 0.01, 0.0, 0.02, 0.1, 0.0, 9.8])
    for h in (g, oi):
        h.reset(last, t0 - 0.001, 0.0, [0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    beg, imu, pts = _make_scan(rng, 0, 20000, t0)
    out_g = g.undistort(lio, imu, pts, beg)
    st_o, out_o, _ = oi.undistort(s0.copy(), imu, pts, beg)
    assert np.array_equal(out_g, out_o) and np.array_equal(lio.get_state(), st_o)
    o = ScanPubOracle(api.AVIA)
    o.set_state(st_o)
    dptr = cuda_lib.immesh_imu_device_points(g._h)
    for skip in (1, 7):
        a = lio.registered_cloud(dptr, point_skip=skip, on_device=True, n=out_o.shape[0], stride=4)
        assert a.shape[0] == (out_o.shape[0] - 1) // skip + 1
        assert np.array_equal(a, o.frame_world(out_o, skip))


def _rc_effect(lib, g, cap, buf=None):
    n = C.c_int(-7)
    rc = lib.immesh_lio_effect_cloud(g._h, None if buf is None else buf.ctypes.data_as(C.POINTER(C.c_float)), None, cap, C.byref(n))
    return rc, n.value


def _rc_registered(lib, g, pts=None, n=0, stride=3, col=-1, skip=1, cap=0, buf=None):
    nout = C.c_int(-7)
    p = None if pts is None else pts.ctypes.data_as(C.c_void_p)
    rc = lib.immesh_lio_registered_cloud(g._h, p, n, stride, col, 0, skip, None if buf is None else buf.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(nout))
    return rc, nout.value


def test_capacity_validity_and_empty_scan(cuda_lib):
    L = cuda_lib
    cfg = api.AVIA
    _, scans = synth.make_stream("avia", 3, seed=5, ext_T=cfg.ext_T)
    g = api.Lio(cfg, lib=L)
    # a fresh handle: no effect rows, no localised scan
    assert _rc_effect(L, g, 0) == (0, 0)
    assert _rc_registered(L, g)[0] == E_INVALID
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    assert _rc_effect(L, g, 0) == (0, 0)                 # after the map build the reference publishes nothing either
    assert _rc_registered(L, g)[0] == E_INVALID
    body = scans[1]["body_ds"]
    g.lio_state_estimation(body)
    rows, idx = g.effect_cloud()
    m = rows.shape[0]
    assert m > 100
    # capacity: a count query and a too-small buffer report the rows needed
    small = np.zeros((4, 4), dtype=np.float32)
    assert _rc_effect(L, g, 0) == (E_CAPACITY, m)
    assert _rc_effect(L, g, 4, small) == (E_CAPACITY, m)
    exact = np.zeros((m, 4), dtype=np.float32)
    assert _rc_effect(L, g, m, exact) == (0, m) and np.array_equal(exact, rows)
    nreg = (body.shape[0] - 1) // 2 + 1
    assert _rc_registered(L, g, skip=2) == (E_CAPACITY, nreg)
    dense = np.ascontiguousarray(scans[1]["body_full"], dtype=np.float32)
    assert _rc_registered(L, g, dense, dense.shape[0], 3, -1, 5, 4, small) == (E_CAPACITY, (dense.shape[0] - 1) // 5 + 1)
    # bad arguments
    assert _rc_registered(L, g, skip=0)[0] == E_INVALID
    assert _rc_registered(L, g, dense, dense.shape[0], 2, -1, 1)[0] == E_INVALID
    assert _rc_registered(L, g, dense, dense.shape[0], 3, 3, 1)[0] == E_INVALID
    # the map update leaves the rows as they are (the parity tests compare them before and after); residual_build overwrites them
    g.map_incremental_grow()
    assert np.array_equal(g.effect_cloud()[0], rows)
    g.residual_build(scans[2]["body_ds"])
    for rc in (_rc_effect(L, g, 0)[0], _rc_registered(L, g)[0]):
        assert rc == E_INVALID
        assert "immesh_residual_build" in L.immesh_last_error().decode()
    assert _rc_registered(L, g, dense, dense.shape[0], 3, -1, 1)[0] == E_CAPACITY   # a caller's cloud is still published
    g.lio_state_estimation(scans[2]["body_ds"])          # the next run makes the rows valid again
    assert g.effect_cloud()[0].shape[0] > 100
    pw, var9 = np.zeros((3, 3)), np.tile(np.eye(3).ravel() * 1e-4, (3, 1))
    g.voxelmap_update_pv(pw + scans[2]["t_true"], var9)
    assert _rc_effect(L, g, 0)[0] == E_INVALID and "immesh_voxelmap_update_pv" in L.immesh_last_error().decode()
    # an empty scan
    g.lio_state_estimation(np.zeros((0, 3), dtype=np.float32))
    assert _rc_effect(L, g, 0) == (0, 0) and _rc_registered(L, g) == (0, 0)
