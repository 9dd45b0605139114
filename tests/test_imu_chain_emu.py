"""CPU tier: the two bodies of the IMU-enabled scan loop that do not run on the GPU tier's arithmetic alone, built for the host
(tests/imu_chain/emu_imu_chain.cpp):
  * imu_plan, the interval plan k_imu_forward works out on the device from the staged samples, against the host loop immesh_imu_undistort
    used before the plan moved to the device (restated below) -- random batches with stamps before, at and after last_lidar_end_time,
    equal stamps, a single sample, an empty batch, and the members carried over several scans;
  * imu_init_batch / imu_init_reset (IMU_init and Reset() on the host) against the numpy restatement in tests/imu_stream_common.py,
    the first-frame seeding and the loop's reset path included."""
import ctypes as C

import numpy as np
import pytest

from imu_stream_common import InitRef


@pytest.fixture(scope="module")
def emu(built):
    from immesh_b200 import build
    L = C.CDLL(build.build_imu_chain())
    L.emu_imu_plan.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_void_p, C.c_void_p]
    L.emu_imu_plan.restype = C.c_int
    L.emu_imu_init.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    L.emu_imu_init.restype = C.c_double
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_plan(tm, imu, last_curv, lidar_beg_time):
    """the host loop of immesh_imu_undistort before the plan moved to the device (v_imu = last_imu_ + meas.imu, :759-787, :810-836,
    :881-896); tm = dict(last_imu, last_lidar_end_time, last_update_time), updated in place"""
    v = [tm["last_imu"]] + [imu[i] for i in range(imu.shape[0])]
    imu_end_time = v[-1][0]
    pcl_beg_time = max(lidar_beg_time, tm["last_update_time"])
    pcl_end_time = lidar_beg_time + float(np.float32(last_curv)) / 1000.0
    tm["last_update_time"] = pcl_end_time
    steps = []
    for k in range(len(v) - 1):
        head, tail = v[k], v[k + 1]
        if tail[0] < tm["last_lidar_end_time"]:
            continue
        s = [0.5 * (head[1 + i] + tail[1 + i]) for i in range(3)] + [0.5 * (head[4 + i] + tail[4 + i]) for i in range(3)]
        s.append(tail[0] - tm["last_lidar_end_time"] if head[0] < tm["last_lidar_end_time"] else tail[0] - head[0])
        s.append(tail[0] - pcl_beg_time)
        steps.append(s)
    if imu_end_time > pcl_beg_time:
        note = 1.0 if pcl_end_time > imu_end_time else -1.0
        dt = note * (pcl_end_time - imu_end_time)
    else:
        note = 1.0 if pcl_end_time > pcl_beg_time else -1.0
        dt = note * (pcl_end_time - pcl_beg_time)
    tm["last_imu"] = np.array(v[-1], dtype=np.float64)
    tm["last_lidar_end_time"] = pcl_end_time
    return np.array(steps).reshape(-1, 8), note, dt


def _batch(rng, t0, m, dup=False):
    t = np.sort(t0 + rng.uniform(0.0, 0.1, m))
    if dup and m > 2:
        t[1] = t[0]
        t[-1] = t[-2]
    return np.concatenate([t[:, None], rng.normal(0, 0.3, (m, 3)), rng.normal(0, 1, (m, 3)) + [0, 0, 9.8]], axis=1)


def _check_stream(emu, batches, rng, tm_start):
    dev = np.zeros(11)
    dev[0:7], dev[7], dev[8], dev[9] = tm_start["last_imu"], tm_start["last_lidar_end_time"], tm_start["last_update_time"], 0.0
    ref = {k: (np.array(v) if k == "last_imu" else v) for k, v in tm_start.items()}
    for beg, imu, curv in batches:
        imu = np.ascontiguousarray(imu, dtype=np.float64).reshape(-1, 7)
        steps = np.zeros((max(imu.shape[0], 1), 8))
        out = np.zeros(2)
        m = emu.emu_imu_plan(_p(dev), _p(imu), imu.shape[0], C.c_float(curv), beg, _p(steps), _p(out))
        rs, note, dt = host_plan(ref, imu, curv, beg)
        assert m == rs.shape[0]
        assert np.array_equal(steps[:m], rs)
        assert out[0] == note and out[1] == dt
        assert np.array_equal(dev[0:7], ref["last_imu"])
        assert dev[7] == ref["last_lidar_end_time"]
        assert dev[8] + float(dev[9]) / 1000.0 == ref["last_update_time"]
        assert dev[10] == m + 1


def test_plan_matches_host_loop(emu):
    rng = np.random.default_rng(5)
    for trial in range(40):
        t0 = 100.0 + trial
        batches = []
        for k in range(4):
            beg = t0 + 0.1 * k
            m = int(rng.choice([0, 1, 2, 5, 20]))
            imu = _batch(rng, beg - 0.02, m, dup=bool(trial % 3 == 0))
            if m and k == 1:
                imu[0, 0] = batches[-1][0] + float(np.float32(batches[-1][2])) / 1000.0   # a stamp exactly AT last_lidar_end_time
            batches.append((beg, imu, float(np.float32(rng.choice([99.0, 99.5, 100.0, 37.25])))))
        if trial % 4 == 1:   # a stream whose first stamps lie BEFORE last_lidar_end_time
            tm = dict(last_imu=np.array([t0 - 0.5, 0, 0, 0, 0, 0, 9.8]), last_lidar_end_time=t0 + 0.05, last_update_time=t0 - 0.1)
        else:
            tm = dict(last_imu=np.array([t0 - 0.003, 0.01, 0, 0.02, 0.1, 0, 9.8]), last_lidar_end_time=t0 - 0.001, last_update_time=0.0)
        _check_stream(emu, batches, rng, tm)


def test_plan_single_sample_and_fresh_handle(emu):
    rng = np.random.default_rng(6)
    fresh = dict(last_imu=np.zeros(7), last_lidar_end_time=0.0, last_update_time=0.0)     # last_lidar_end_time_ = 0.0 (the header's choice)
    _check_stream(emu, [(50.0, _batch(rng, 50.0, 1), 99.0), (50.1, _batch(rng, 50.1, 1), 99.0), (50.2, np.zeros((0, 7)), 98.0)], rng, fresh)


def _emu_init(emu, st, reset, imu):
    imu = np.ascontiguousarray(imu, dtype=np.float64).reshape(-1, 7)
    g = np.zeros(3)
    norm = emu.emu_imu_init(_p(st), int(reset), _p(imu), imu.shape[0], _p(g))
    return norm, g


def test_imu_init_matches_numpy_restatement(emu):
    rng = np.random.default_rng(7)
    for trial in range(10):
        st = np.array([0.0, 0.0, -1.0, 0, 0, 0, 1, 1], dtype=np.float64)   # a fresh ImuProcess: b_first_frame_
        ref = InitRef()
        for k in range(6):
            if k == 3:   # the loop's reset: Reset() with b_first_frame_ already false
                ref.reset()
                _emu_init(emu, st, True, np.zeros((0, 7)))
                assert np.array_equal(st[0:3], [0.0, 0.0, -1.0]) and st[6] == 1 and st[7] == 0
            imu = _batch(rng, 10.0 + 0.1 * k, int(rng.integers(1, 25)))
            norm, g = _emu_init(emu, st, False, imu)
            rn, rg = ref.batch(imu)
            assert norm == rn and np.array_equal(g, rg)
            assert np.array_equal(st[0:3], ref.mean_acc) and np.array_equal(st[3:6], ref.mean_gyr) and st[6] == ref.N
    # the seeded first frame and the reset path differ: the reset path starts from (0, 0, -1) with N = 1
    imu = _batch(rng, 20.0, 7)
    a = np.array([0.0, 0.0, -1.0, 0, 0, 0, 1, 1])
    b = np.array([0.0, 0.0, -1.0, 0, 0, 0, 1, 0])
    _emu_init(emu, a, False, imu)
    _emu_init(emu, b, False, imu)
    assert a[6] == 8 and b[6] == 8
    assert np.allclose(a[0:3], b[0:3], rtol=1e-12, atol=1e-12)
