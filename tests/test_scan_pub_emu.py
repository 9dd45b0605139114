"""CPU tier: the two scan publishers (publish_effect_world / publish_frame_world) executed by the host emulation of the device code
against the oracle, and the oracle's effect rows against its own record of the last IESKF iteration."""
import numpy as np
import pytest

from immesh_b200 import api, synth
from scan_pub_common import ScanPubOracle, check_weights_against_normal_equations, emu_scanpub_lib, run_scan_pub_parity

E_INVALID, E_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def emu_lib():
    """the host emulation with ScanBuf::wsqrt and the two calls (tests/pubmap/emu_scan_pub.cpp)"""
    return emu_scanpub_lib()


@pytest.mark.parametrize("split", [1, 0])
def test_avia_every_scan(emu_lib, split):
    emu_lib.emu_lio_set_split(split)   # 1: k_match + k_terms bodies, 0: the k_residual body
    try:
        counts = run_scan_pub_parity(emu_lib, "avia", api.AVIA, n_scans=8, seed=0)
    finally:
        emu_lib.emu_lio_set_split(1)
    assert min(counts) > 100


def test_hdl64_every_scan(emu_lib):
    counts = run_scan_pub_parity(emu_lib, "hdl64", api.VELODYNE, n_scans=4, seed=1, n_points=32768)
    assert min(counts) > 100


def test_fresh_handle_empty_scan_and_capacity(emu_lib):
    import ctypes as C
    g = api.Lio(api.AVIA, lib=emu_lib)
    rows, idx = g.effect_cloud()
    assert rows.shape == (0, 4) and idx.shape == (0,)
    n = C.c_int(0)
    assert emu_lib.immesh_lio_registered_cloud(g._h, None, 0, 3, -1, 0, 1, None, 0, C.byref(n)) == E_INVALID
    _, scans = synth.make_stream("avia", 2, seed=5, ext_T=api.AVIA.ext_T)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    g.lio_state_estimation(scans[1]["body_ds"])
    rows, idx = g.effect_cloud()
    assert rows.shape[0] > 10
    buf = np.zeros((4, 4), dtype=np.float32)
    fp = buf.ctypes.data_as(C.POINTER(C.c_float))
    assert emu_lib.immesh_lio_effect_cloud(g._h, fp, None, 4, C.byref(n)) == E_CAPACITY and n.value == rows.shape[0]
    assert emu_lib.immesh_lio_registered_cloud(g._h, None, 0, 3, -1, 0, 0, fp, 4, C.byref(n)) == E_INVALID   # point_skip 0
    g.lio_state_estimation(np.zeros((0, 3), dtype=np.float32))
    rows, idx = g.effect_cloud()
    assert rows.shape == (0, 4) and g.registered_cloud().shape == (0, 4)


def test_oracle_weights_reproduce_the_normal_equations():
    """independent of any implementation under test: the oracle's rows are its last iteration's matches, and their weights give
    that iteration's H^T R^-1 H translation block"""
    cfg = api.AVIA
    sensor, scans = synth.make_stream("hdl64", 4, seed=3, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=16384)
    o = ScanPubOracle(cfg)
    o.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    o.voxel_map_init(scans[0]["body_full"])
    for k in range(1, 4):
        o.predict(scans[k]["dt"])
        it = o.lio_state_estimation(scans[k]["body_ds"])
        assert it >= 2     # the weights come from a state that differs from the start state and from the final one
        check_weights_against_normal_equations(o, it)
        o.map_incremental_grow(scans[k]["body_ds"])
