"""GPU tier: the IMU front-end (immesh_imu_*, SURVEY 8f-2) through the C ABI against the oracle restatement of
ImuProcess::UndistortPcl.  Same scenario as tests/test_imu_emu.py (which runs the same device bodies on the CPU, bit-exact)."""
import numpy as np
import pytest

import oracle_api as oa
from immesh_b200 import api
from test_imu_emu import _imu_cfg, _make_scan

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n_pts,dup", [(3000, False), (50000, True), (1, False)])
def test_undistort_stream_bit_exact_gpu(cuda_lib, n_pts, dup):
    rng = np.random.default_rng(11)
    cfg = _imu_cfg(rng)
    lio = api.Lio(api.AVIA, lib=cuda_lib)
    s0 = lio.get_state()
    s0[12:15] = [0.5, -0.2, 0.05]
    s0[21:24] = [0.0, 0.0, -9.81]
    s0[15:18] = [0.001, -0.002, 0.0005]
    s0[18:21] = [0.01, 0.02, -0.01]
    lio.set_state(s0)
    g, o = api.Imu(cfg, lib=cuda_lib), oa.OracleImu(cfg)
    t0 = 100.0
    last = np.array([t0 - 0.002, 0.01, 0.0, 0.02, 0.1, 0.0, 9.8])
    for h in (g, o):
        h.reset(last, t0 - 0.001, 0.0, [0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    st_o = s0.copy()
    for k in range(3):
        beg, imu, pts = _make_scan(rng, k, n_pts, t0, dup_stamps=dup)
        out_g = g.undistort(lio, imu, pts, beg)
        st_o, out_o, poses_o = o.undistort(st_o, imu, pts, beg)
        assert np.array_equal(g.poses(), poses_o)
        assert np.array_equal(lio.get_state(), st_o)
        assert np.array_equal(out_g, out_o)
