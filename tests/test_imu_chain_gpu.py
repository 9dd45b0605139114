"""GPU tier: the IMU-enabled scan loop (immesh_lio_step_async_imu: IMU initialisation, first map, steady scans meshed through
push_frame_from_lio_async) queued with no wait between scans, against the oracle chain of tests/imu_stream_common.py -- branch sequence,
filter state, VoxelMap dump, mesh vertices, facets and flips bit-exact; the same stream through today's separate calls; the errors."""
import numpy as np
import pytest

import oracle_api as oa
from immesh_b200 import api
from imu_stream_common import InitRef, OracleChain, imu_cfg, make_imu_stream, true_velocity

pytestmark = pytest.mark.gpu

MAX_INI = 30          # 20 samples per scan: initialisation spans two scans with samples (and an empty batch between)
N_SCANS = 11
MESH_CFG = api.MeshConfig(max_vertices=1 << 19, max_triangles=1 << 20, max_voxels=1 << 17, max_frame_points=1 << 17)


def _state0(sensor, scans):
    s = np.zeros(348)
    s[0:9] = np.eye(3).reshape(9)
    s[12:15] = true_velocity(sensor, scans[0]["beg"])
    for i in range(18):
        s[24 + i * 18 + i] = 1e-7
    return s


def _run(lib, scans, s0, on_device, calib, resets=(), errors=False, lio_cfg=api.AVIA, mesh=True):
    """the stream through the queued call; returns (branches, lio, mesh, graph stats)"""
    import torch
    leaf = lio_cfg.filter_size_surf
    g = api.Lio(lio_cfg, lib=lib)
    g.set_state(s0)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32, lib=lib)
    vg = api.VoxelGrid(1 << 17, lib=lib)
    gm = api.Mesh(MESH_CFG, lib=lib) if mesh else None
    imu_h.init_begin(MAX_INI)
    branches, keep = [], []
    for k, sc in enumerate(scans):
        if k in resets:
            imu_h.init_begin(MAX_INI)
        if errors:
            _error_calls(lib, g, imu_h, vg, sc, leaf)
        if on_device:
            d = torch.from_numpy(sc["pts"]).cuda()
            keep.append(d)                      # read when the queued work runs
            br = vg.step_async_imu(g, imu_h, sc["imu"], d.data_ptr(), sc["beg"], leaf, calib_laser=calib, n=d.shape[0], on_device=True)
        else:
            br = vg.step_async_imu(g, imu_h, sc["imu"], sc["pts"], sc["beg"], leaf, calib_laser=calib)
        if br == 3 and gm is not None:
            gm.push_frame_from_lio_async(g, vg.input_points(), sc["pts"].shape[0], on_device=True)
        branches.append(br)
    g.wait()
    if gm is not None:
        gm.wait()
    return branches, g, gm, api.graph_stats(g, None), (imu_h, vg)


def _error_calls(lib, g, imu_h, vg, sc, leaf):
    """each capacity error returns IMMESH_E_CAPACITY before anything is queued"""
    big_batch = np.repeat(sc["imu"][:1], 40, axis=0) if sc["imu"].shape[0] else np.zeros((40, 7))
    with pytest.raises(RuntimeError, match="code -3"):
        vg.step_async_imu(g, imu_h, big_batch, sc["pts"], sc["beg"], leaf)
    big_scan = np.concatenate([sc["pts"]] * 7)                                   # > max_points of the IMU / VoxelGrid handles
    with pytest.raises(RuntimeError, match="code -3"):
        vg.step_async_imu(g, imu_h, sc["imu"], big_scan, sc["beg"], leaf)


def _oracle(scans, s0, calib, resets=(), mesh=True):
    o = OracleChain(api.AVIA, imu_cfg(), MESH_CFG if mesh else None, MAX_INI, s0, api.AVIA.filter_size_surf, calib=calib)
    branches = []
    for k, sc in enumerate(scans):
        if k in resets:
            o.init_begin()
        branches.append(o.step(sc["imu"], sc["pts"], sc["beg"]))
    return branches, o


def _compare(g, gm, o):
    assert np.array_equal(g.get_state(), o.lio.get_state()), np.abs(g.get_state() - o.lio.get_state()).max()
    dg, do = g.dump_map(), o.lio.dump_map()
    assert dg.shape == do.shape and np.array_equal(dg, do)
    if gm is not None:
        (vv, tt, ff), (ov, ot, of) = gm.snapshot(), o.mesh.snapshot()
        assert vv.shape == ov.shape and np.array_equal(vv, ov)
        assert tt.shape == ot.shape and np.array_equal(tt, ot)
        assert np.array_equal(ff, of)
        assert tt.shape[0] > 0


@pytest.fixture(scope="module")
def stream():
    sensor, scans = make_imu_stream(N_SCANS, seed=3, empty_batch=1)
    return sensor, scans, _state0(sensor, scans)


@pytest.mark.parametrize("on_device,calib", [(False, False), (True, True)])
def test_imu_chain_bit_exact(cuda_lib, stream, on_device, calib):
    sensor, scans, s0 = stream
    br_o, o = _oracle(scans, s0, calib)
    assert br_o == [1, 1, 1, 2] + [3] * (N_SCANS - 4), br_o        # init over scans 0-2 (empty batch at 1), map at 3, steady after
    br_g, g, gm, gs, _ = _run(cuda_lib, scans, s0, on_device, calib)
    assert br_g == br_o
    _compare(g, gm, o)
    assert gs["lio_replays"] > 0, gs
    assert g.counts()["err"] == 0


def test_imu_chain_reset_reinitialises(cuda_lib, stream):
    """a reset in the middle of the stream: Reset() (means from (0, 0, -1), b_first_frame_ kept false), re-initialisation, and the map
    kept (m_init_map survives): steady scans follow without a second map build"""
    sensor, scans, s0 = stream
    resets = (6,)
    br_o, o = _oracle(scans, s0, False, resets=resets)
    assert br_o[6:9] == [1, 1, 3], br_o
    br_g, g, gm, gs, _ = _run(cuda_lib, scans, s0, False, False, resets=resets)
    assert br_g == br_o
    _compare(g, gm, o)


def test_imu_chain_errors_leave_results_unchanged(cuda_lib, stream):
    """capacity errors before every scan (initialising and steady) change nothing: the stream still equals the oracle"""
    sensor, scans, s0 = stream
    br_o, o = _oracle(scans[:7], s0, False, mesh=False)
    br_g, g, _, _, _ = _run(cuda_lib, scans[:7], s0, False, False, errors=True, mesh=False)
    assert br_g == br_o
    _compare(g, None, o)
    # a scan above the localization handle's max_scan_points (but within the IMU / VoxelGrid capacities)
    import dataclasses
    small = dataclasses.replace(api.AVIA, max_scan_points=scans[0]["pts"].shape[0] // 2)
    g2 = api.Lio(small, lib=cuda_lib)
    imu_h = api.Imu(imu_cfg(), max_points=1 << 17, max_imu=32, lib=cuda_lib)
    vg = api.VoxelGrid(1 << 17, lib=cuda_lib)
    imu_h.init_begin(MAX_INI)
    with pytest.raises(RuntimeError, match="code -3"):
        vg.step_async_imu(g2, imu_h, scans[0]["imu"], scans[0]["pts"], scans[0]["beg"], small.filter_size_surf)


def test_imu_chain_equals_separate_calls(cuda_lib, stream):
    """the same stream through today's calls -- immesh_imu_undistort + immesh_voxelmap_build / immesh_lio_step_async_raw, the IMU
    handle created with the oracle's |mean_acc| -- gives the chain's state and map"""
    sensor, scans, s0 = stream
    br_g, g, _, _, _ = _run(cuda_lib, scans, s0, False, False, mesh=False)
    init = InitRef()
    st = s0.copy()
    for sc in scans[:3]:
        if sc["imu"].shape[0]:
            norm, grav = init.batch(sc["imu"])
            last_imu = sc["imu"][-1]
    st[0:9] = np.eye(3).reshape(9); st[15:18] = 0.0; st[21:24] = grav
    cfg = imu_cfg()
    cfg["mean_acc_norm"] = norm
    l2 = api.Lio(api.AVIA, lib=cuda_lib)
    l2.set_state(st)
    im2 = api.Imu(cfg, max_points=1 << 17, max_imu=32, lib=cuda_lib)
    vg2 = api.VoxelGrid(1 << 17, lib=cuda_lib)
    end2 = scans[2]["beg"] + float(scans[2]["pts"][-1, 3]) / 1000.0
    im2.reset(last_imu, 0.0, end2, [0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    for k, sc in enumerate(scans[3:]):
        out = im2.undistort(l2, sc["imu"], sc["pts"], sc["beg"])
        if k == 0:
            l2.voxel_map_init(out[:, :3])
        else:
            vg2.step_async_raw(l2, out, api.AVIA.filter_size_surf, stride=4)
            l2.wait()
    assert np.array_equal(g.get_state(), l2.get_state())
    assert np.array_equal(g.dump_map(), l2.dump_map())
