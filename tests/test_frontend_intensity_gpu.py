"""GPU tier: point intensity through the device front-end, all comparisons bit-exact.  immesh_voxelgrid_filter_i against the numpy
restatement of PCL's intensity average (tests/frontend_intensity_common.py) and against immesh_voxelgrid_filter's x y z; the raw and
IMU chains on point records (immesh_lio_step_async_raw_i / _imu_i) against the plain chains fed the same x y z (and stamps) --
state, map, effect rows, mesh; immesh_lio_frontend_cloud against the oracle's publish_frame_world with the restated intensities;
the validity, capacity and argument rules."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oracle_api as oa
from frontend_intensity_common import LAYOUTS, check_filter_i, intensities, records, run_filter_i_cases, voxel_grid_i
from immesh_b200 import api, synth
from imu_stream_common import OracleChain, imu_cfg, make_imu_stream
from lio_common import init_velocity
from scan_pub_common import ScanPubOracle

pytestmark = pytest.mark.gpu
E_INVALID, E_CAPACITY = -1, -3
MESH_CFG = api.MeshConfig(max_vertices=1 << 19, max_triangles=1 << 20, max_voxels=1 << 17, max_frame_points=1 << 17)
RAW_CFG = dataclasses.replace(api.VELODYNE, calib_laser=1)


def _xyzi(xyz, inten):
    return np.concatenate([np.asarray(xyz, np.float32), np.asarray(inten, np.float32)[:, None]], axis=1)


def _rc_frontend(lib, g, vg, dense=0, skip=1, cap=0, buf=None):
    n = C.c_int(-7)
    rc = lib.immesh_lio_frontend_cloud(g._h, vg._h, dense, skip, None if buf is None else buf.ctypes.data_as(C.POINTER(C.c_float)), cap, C.byref(n))
    return rc, n.value


# ---- immesh_voxelgrid_filter_i

@pytest.mark.parametrize("kind", ["avia", "hdl64"])
@pytest.mark.parametrize("leaf", [0.1, 0.4, 0.5])
def test_filter_i_scan_shapes(cuda_lib, kind, leaf):
    vg = api.VoxelGrid(1 << 18, lib=cuda_lib)
    _, scans = synth.make_stream(kind, 1, seed=5)
    xyz = scans[0]["body_full"]
    for stride, col in LAYOUTS:
        for dev in (False, True):
            out = check_filter_i(vg, xyz, intensities(xyz.shape[0], stride), leaf, stride, col, dev)
            assert 0 < out.shape[0] < xyz.shape[0]


def test_filter_i_edge_cases(cuda_lib):
    vg = api.VoxelGrid(1 << 16, lib=cuda_lib)
    assert vg.filter_i(np.zeros((0, 12), np.float32), 0.4, 8).shape == (0, 4)
    check_filter_i(vg, np.array([[1.5, -2.25, 0.75]], np.float32), np.array([17.25], np.float32), 0.4, 4, 3, False)
    check_filter_i(vg, np.full((10, 3), np.nan, np.float32), intensities(10, 1), 0.4, 12, 8, True)      # nothing finite -> empty
    rng = np.random.default_rng(0)
    wide = rng.uniform(-3000, 3000, (2000, 3)).astype(np.float32)
    wide[::97] = np.nan
    inten = intensities(2000, 2)
    out = check_filter_i(vg, wide, inten, 0.01, 5, 4, True)                   # leaf too small: output = input, intensity included
    assert vg.leaf_too_small and np.array_equal(out[:, 3], inten)
    run_filter_i_cases(cuda_lib)


# ---- the raw chain (velodyne.yaml with calib_laser, HDL-64 stream)

@pytest.fixture(scope="module")
def raw_stream():
    sensor, scans = synth.make_stream("hdl64", 5, seed=12, leaf=RAW_CFG.filter_size_surf, n_points=65536)
    for k, sc in enumerate(scans):
        sc["inten"] = intensities(sc["body_full"].shape[0], 40 + k)
    return sensor, scans


def _run_raw(lib, sensor, scans, with_i, after_scan=None):
    g, vg, gm = api.Lio(RAW_CFG, lib=lib), api.VoxelGrid(1 << 17, lib=lib), api.Mesh(MESH_CFG, lib=lib)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(g, sensor, scans)
    g.voxel_map_init(oa.kitti_calib(scans[0]["body_full"]))
    leaf = RAW_CFG.filter_size_surf
    for k in range(1, len(scans)):
        raw, n = scans[k]["body_full"], scans[k]["body_full"].shape[0]
        if with_i:
            vg.step_async_raw_i(g, records(raw, scans[k]["inten"], 12, 8, seed=k), leaf, 8, dt=scans[k]["dt"], calib_laser=True)
        else:
            vg.step_async_raw(g, raw, leaf, dt=scans[k]["dt"], calib_laser=True)
        gm.push_frame_from_lio_async(g, vg.input_points(), n, on_device=True)
        if after_scan:
            after_scan(k, g, vg)
    g.wait()
    gm.wait()
    return g, vg, gm


def _raw_oracle(sensor, scans, upto):
    o = ScanPubOracle(RAW_CFG)
    o.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(o, sensor, scans)
    o.voxel_map_init(oa.kitti_calib(scans[0]["body_full"]))
    for k in range(1, upto + 1):
        full = oa.kitti_calib(scans[k]["body_full"])
        ds, _, _ = oa.voxel_grid(full, RAW_CFG.filter_size_surf)
        o.predict(scans[k]["dt"])
        o.lio_state_estimation(ds)
        o.map_incremental_grow(ds)
    return o, full, ds


def _check_frontend_against_oracle(g, vg, o, full, ds, inten):
    ds_i, _ = voxel_grid_i(full, inten, RAW_CFG.filter_size_surf)
    assert np.array_equal(ds_i[:, :3], ds)
    for skip in (1, 3):
        assert np.array_equal(g.frontend_cloud(vg, True, skip), o.frame_world(_xyzi(full, inten), skip, intensity_col=3))
        sparse = g.frontend_cloud(vg, False, skip)
        assert np.array_equal(sparse, o.frame_world(ds_i, skip, intensity_col=3))
        assert np.array_equal(sparse[:, :3], g.registered_cloud(None, point_skip=skip)[:, :3])


def _compare_runs(a, b):
    (ga, _, ma), (gb, _, mb) = a, b
    assert np.array_equal(ga.get_state(), gb.get_state())
    assert np.array_equal(ga.dump_map(), gb.dump_map())
    (va, ta, fa), (vb, tb, fb) = ma.snapshot(), mb.snapshot()
    assert va.shape == vb.shape and np.array_equal(va, vb)
    assert ta.shape == tb.shape and np.array_equal(ta, tb) and ta.shape[0] > 0
    assert np.array_equal(fa, fb)


def test_raw_chain_i_equals_plain_chain_and_oracle(cuda_lib, raw_stream):
    sensor, scans = raw_stream
    eff = {True: [], False: []}
    checked = []

    def after(with_i):
        def f(k, g, vg):
            eff[with_i].append(g.effect_cloud())
            if with_i:
                o, full, ds = _raw_oracle(sensor, scans, k)
                assert np.array_equal(g.get_state(), o.get_state())
                _check_frontend_against_oracle(g, vg, o, full, ds, scans[k]["inten"])
                checked.append(k)
        return f
    plain = _run_raw(cuda_lib, sensor, scans, False, after(False))
    with_i = _run_raw(cuda_lib, sensor, scans, True, after(True))
    _compare_runs(plain, with_i)
    assert checked == [1, 2, 3, 4]
    for (ra, ia), (rb, ib) in zip(eff[False], eff[True]):
        assert ra.shape[0] > 100 and np.array_equal(ia, ib) and np.array_equal(ra.view(np.uint32), rb.view(np.uint32))


@pytest.mark.parametrize("graph", ["1", "0"])
def test_raw_chain_i_queued_scans(cuda_lib, raw_stream, monkeypatch, graph):
    """several scans queued without a wait, then frontend_cloud publishes the last one; IMMESH_GRAPH=0: direct launches"""
    monkeypatch.setenv("IMMESH_GRAPH", graph)    # read when a handle is created
    sensor, scans = raw_stream
    g, vg, _ = _run_raw(cuda_lib, sensor, scans, True)
    o, full, ds = _raw_oracle(sensor, scans, len(scans) - 1)
    assert np.array_equal(g.get_state(), o.get_state())
    _check_frontend_against_oracle(g, vg, o, full, ds, scans[-1]["inten"])


# ---- the IMU chain (the 11-scan stream of test_imu_chain_gpu.py as stride-12 PointXYZINormal records)

MAX_INI, N_SCANS = 30, 11


@pytest.fixture(scope="module")
def imu_stream():
    from test_imu_chain_gpu import _state0
    sensor, scans = make_imu_stream(N_SCANS, seed=3, empty_batch=1)
    for k, sc in enumerate(scans):
        sc["inten"] = intensities(sc["pts"].shape[0], 70 + k)
        sc["rec"] = records(sc["pts"][:, :3], sc["inten"], 12, 8, stamps=sc["pts"][:, 3], time_col=9, seed=k)
    return sensor, scans, _state0(sensor, scans)


@pytest.mark.parametrize("on_device,calib", [(False, False), (True, True)])
def test_imu_chain_i(cuda_lib, imu_stream, monkeypatch, on_device, calib):
    import torch
    from test_imu_chain_gpu import _run
    sensor, scans, s0 = imu_stream
    leaf = api.AVIA.filter_size_surf
    br_p, gp, mp, _, _ = _run(cuda_lib, scans, s0, on_device, calib)
    # the oracle chain, with the calibrated undistorted scan it down-samples kept for the intensity check
    fulls = []
    real_vg = oa.voxel_grid
    monkeypatch.setattr(oa, "voxel_grid", lambda pts, lf: (fulls.append(np.array(pts)), real_vg(pts, lf))[1])
    o = OracleChain(api.AVIA, imu_cfg(), None, MAX_INI, s0, leaf, calib=calib)
    g, vg, gm = api.Lio(api.AVIA, lib=cuda_lib), api.VoxelGrid(1 << 17, lib=cuda_lib), api.Mesh(MESH_CFG, lib=cuda_lib)
    g.set_state(s0)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32, lib=cuda_lib)
    imu_h.init_begin(MAX_INI)
    branches, keep = [], []
    for k, sc in enumerate(scans):
        n = sc["rec"].shape[0]
        if on_device:
            d = torch.from_numpy(sc["rec"]).cuda()
            keep.append(d)
            br = vg.step_async_imu_i(g, imu_h, sc["imu"], d.data_ptr(), sc["beg"], leaf, 9, 8, calib_laser=calib, n=n, stride=12, on_device=True)
        else:
            br = vg.step_async_imu_i(g, imu_h, sc["imu"], sc["rec"], sc["beg"], leaf, 9, 8, calib_laser=calib)
        assert br == o.step(sc["imu"], sc["pts"], sc["beg"])
        branches.append(br)
        if br != 3:      # branches 1 and 2 publish nothing
            assert _rc_frontend(cuda_lib, g, vg)[0] == E_INVALID
            assert _rc_frontend(cuda_lib, g, vg, dense=1)[0] == E_INVALID
            continue
        gm.push_frame_from_lio_async(g, vg.input_points(), n, on_device=True)
        order = np.argsort(sc["pts"][:, 3], kind="stable")           # time_list: stable sort of the float32 stamps
        dense = g.frontend_cloud(vg, True)
        assert np.array_equal(dense[:, 3], sc["inten"][order])
        assert np.array_equal(dense[:, :3], g.registered_cloud(vg.input_points(), on_device=True, n=n, stride=3)[:, :3])
        ds_i, _ = voxel_grid_i(fulls[-1], sc["inten"][order], leaf)
        sparse = g.frontend_cloud(vg, False, 3)
        assert np.array_equal(sparse[:, 3], ds_i[::3, 3])
        assert np.array_equal(sparse[:, :3], g.registered_cloud(None, point_skip=3)[:, :3])
        assert np.array_equal(g.get_state(), o.lio.get_state())
    g.wait()
    gm.wait()
    assert branches == br_p == [1, 1, 1, 2] + [3] * (N_SCANS - 4)
    _compare_runs((gp, None, mp), (g, None, gm))


# ---- contract

def test_validity_capacity_and_arguments(cuda_lib, raw_stream):
    L = cuda_lib
    sensor, scans = raw_stream
    leaf = RAW_CFG.filter_size_surf
    g, vg, vg2 = api.Lio(RAW_CFG, lib=L), api.VoxelGrid(1 << 17, lib=L), api.VoxelGrid(1 << 17, lib=L)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    init_velocity(g, sensor, scans)
    g.voxel_map_init(oa.kitti_calib(scans[0]["body_full"]))
    assert _rc_frontend(L, g, vg)[0] == E_INVALID                       # no step yet
    raw, n = scans[1]["body_full"], scans[1]["body_full"].shape[0]

    def step_i(k=1):
        vg.step_async_raw_i(g, records(scans[k]["body_full"], scans[k]["inten"], 12, 8), leaf, 8, dt=scans[k]["dt"], calib_laser=True)
    step_i(1)
    # capacity: a count query and a too-small buffer report the rows needed; an exact buffer takes them
    assert _rc_frontend(L, g, vg, 1, 1) == (E_CAPACITY, n)
    assert _rc_frontend(L, g, vg, 1, 4) == (E_CAPACITY, (n - 1) // 4 + 1)
    small = np.zeros((4, 4), np.float32)
    assert _rc_frontend(L, g, vg, 1, 1, 4, small) == (E_CAPACITY, n)
    m = g.frontend_cloud(vg, False).shape[0]
    assert _rc_frontend(L, g, vg, 0, 1) == (E_CAPACITY, m)
    exact = np.zeros((m, 4), np.float32)
    assert _rc_frontend(L, g, vg, 0, 1, m, exact) == (0, m) and np.array_equal(exact, g.frontend_cloud(vg, False))
    assert _rc_frontend(L, g, vg, 0, 0)[0] == E_INVALID                 # point_skip <= 0
    assert _rc_frontend(L, g, vg2)[0] == E_INVALID                      # another VoxelGrid handle
    g.registered_cloud(None)                                            # publishers leave it valid
    g.effect_cloud()
    assert _rc_frontend(L, g, vg, 0, 1)[0] == E_CAPACITY
    # after a plain step, and after another call on vg
    vg.step_async_raw(g, scans[2]["body_full"], leaf, dt=scans[2]["dt"], calib_laser=True)
    assert _rc_frontend(L, g, vg)[0] == E_INVALID
    step_i(3)
    assert _rc_frontend(L, g, vg)[0] == E_CAPACITY
    vg.filter(raw, leaf)
    assert _rc_frontend(L, g, vg)[0] == E_INVALID
    step_i(4)
    assert _rc_frontend(L, g, vg)[0] == E_CAPACITY
    g.lio_state_estimation(scans[4]["body_ds"])                         # another scan in the localization handle
    assert _rc_frontend(L, g, vg)[0] == E_INVALID
    # bad records
    for stride, col in ((17, 8), (12, 2), (12, 12), (3, 2), (4, -1)):
        bad = np.zeros((8, max(stride, 3)), np.float32)
        with pytest.raises(RuntimeError, match="code -1"):
            vg.filter_i(bad, leaf, col)
        with pytest.raises(RuntimeError, match="code -1"):
            vg.step_async_raw_i(g, bad, leaf, col)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32, lib=L)
    for stride, tcol, icol in ((12, 8, 8), (12, 2, 8), (12, 9, 12), (17, 9, 8), (12, -1, 8)):
        bad = np.zeros((8, stride), np.float32)
        with pytest.raises(RuntimeError, match="code -1"):
            vg.step_async_imu_i(g, imu_h, np.zeros((0, 7)), bad, 0.0, leaf, tcol, icol)
    g.wait()
