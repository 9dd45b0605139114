"""CPU tier: the decision the depth IMU chain (immesh_lio_step_async_depth_imu) takes on the device -- sync_packages' drop rule and
carry, the branch of Process2 / service_LiDAR_update, and IMU_init with its init-end test -- run by the host emulation
(tests/depth_imu/emu_depth_imu.cpp, the same imu_core.cuh code the kernels run) against a Python restatement of the reference, bit for
bit: over scripted and seeded sequences with clouds of 0, 1 and 2 points during the initialisation, right after it and after the map,
empty IMU batches, repeated drops, carry overflows and immesh_imu_init_begin mid-stream.  IMU_init's means are also checked against
the host chain's imu_init_batch (tests/imu_chain)."""
import ctypes as C

import numpy as np
import pytest

from imu_stream_common import InitRef

STATE_DOUBLES = 348


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_depth_imu())
    vp, dp = C.c_void_p, C.POINTER(C.c_double)
    L.emu_dimu_setup.argtypes = [vp, C.c_double, C.c_int, C.c_int, C.c_int]
    L.emu_dimu_begin.argtypes = [vp, C.c_int, C.c_int]
    L.emu_dimu_frame.argtypes = [vp, C.c_int, dp, C.c_int, dp, C.c_int, dp, dp, C.c_double, C.POINTER(C.c_int)]
    L.emu_dimu_frame.restype = C.c_int
    L.emu_dimu_read.argtypes = [vp, dp, C.POINTER(C.c_longlong)]
    return L


@pytest.fixture(scope="module")
def chain_lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_imu_chain())
    dp = C.POINTER(C.c_double)
    L.emu_imu_init.argtypes = [dp, C.c_int, dp, C.c_int, dp]
    L.emu_imu_init.restype = C.c_double
    return L


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class Ref:
    """sync_packages (src/voxel_mapping_common.cpp:393-400) + Process2's branches (src/IMU_Processing.cpp:960-1006) + m_init_map
    (src/voxel_mapping.cpp:1894-1905), restated: the host-decided loop the device replaces"""

    def __init__(self, max_ini, max_imu, norm0=9.81):
        self.init = InitRef()
        self.max_ini, self.max_imu, self.norm = max_ini, max_imu, norm0
        self.init_phase, self.map_built = True, False
        self.carry = np.zeros((0, 7))
        self.state = np.zeros(STATE_DOUBLES)
        self.last_imu, self.upd_beg = np.zeros(7), 0.0
        self.cnt = [0] * 7

    def begin(self):   # immesh_imu_init_begin mid-stream: Reset() of IMU_init's members; the buffered samples go with the reset
        self.init.reset()
        self.init_phase = True
        self.carry = np.zeros((0, 7))

    def frame(self, n, own, t):
        self.cnt[0] += 1
        if self.carry.shape[0] + own.shape[0] > self.max_imu:
            self.cnt[1] += 1
            self.cnt[6] += 1
            return 4, True
        if n <= 1:
            self.carry = np.concatenate([self.carry, own])
            self.cnt[1] += 1
            return 4, False
        batch = np.concatenate([self.carry, own])
        self.carry = np.zeros((0, 7))
        if self.init_phase:
            br = 1
            self.upd_beg = t
            if batch.shape[0]:
                norm, grav = self.init.batch(batch)
                self.state[0:9] = np.eye(3).reshape(-1)
                self.state[15:18] = 0.0
                self.state[21:24] = grav
                self.last_imu = batch[-1].copy()
                if self.init.N > self.max_ini:
                    self.init_phase = False
                    self.norm = norm
        elif not self.map_built:
            br = 2
            self.map_built = True
        else:
            br = 3
        self.cnt[1 + br] += 1
        return br, False


class Emu:
    def __init__(self, lib, max_ini, max_imu, norm0=9.81):
        self.lib, self.max_imu = lib, max_imu
        self.buf = C.create_string_buffer(lib.emu_dimu_size())
        lib.emu_dimu_setup(self.buf, norm0, 1, max_ini, 1)
        self.batch = np.zeros((max_imu, 7))
        self.state = np.zeros(STATE_DOUBLES)
        self.tm = np.zeros(9)

    def frame(self, n, own, t):
        own = np.ascontiguousarray(own, dtype=np.float64).reshape(-1, 7)
        ov = C.c_int(0)
        br = self.lib.emu_dimu_frame(self.buf, n, _d(own), own.shape[0], _d(self.batch), self.max_imu, _d(self.state), _d(self.tm), t, C.byref(ov))
        return br, bool(ov.value)

    def read(self):
        out, cnt = np.zeros(16), (C.c_longlong * 8)()
        self.lib.emu_dimu_read(self.buf, _d(out), cnt)
        return out, list(cnt)


def check(ref, emu, tag):
    out, cnt = emu.read()
    assert out[0:3].tobytes() == ref.init.mean_acc.tobytes() and out[3:6].tobytes() == ref.init.mean_gyr.tobytes(), tag
    assert int(out[6]) == ref.init.N and out[8] == ref.norm and bool(out[9]) == ref.init_phase and bool(out[10]) == ref.map_built, tag
    assert int(out[11]) == ref.carry.shape[0], tag
    assert cnt[:5] == ref.cnt[:5] and cnt[5] == ref.carry.shape[0] and cnt[6] == ref.cnt[6], (tag, cnt, ref.cnt)
    assert emu.state.tobytes() == ref.state.tobytes(), tag
    assert emu.tm[:7].tobytes() == ref.last_imu.tobytes() and emu.tm[7] == ref.upd_beg, tag


def samples(rng, m, t0):
    t = t0 + np.sort(rng.uniform(0.0, 0.1, m))
    gyr = rng.normal(0.0, 0.01, (m, 3))
    acc = np.array([0.1, -9.7, 0.3]) + rng.normal(0.0, 0.05, (m, 3))
    return np.concatenate([t[:, None], gyr, acc], axis=1)


def run(lib, script, max_ini=3, max_imu=16, seed=0):
    """script: (n, samples) per frame, or "begin" for immesh_imu_init_begin; every count is the device's: 0 and 1 drop the frame"""
    rng = np.random.default_rng(seed)
    ref, emu = Ref(max_ini, max_imu), Emu(lib, max_ini, max_imu)
    branches = []
    for i, step in enumerate(script):
        if step == "begin":
            ref.begin()
            lib.emu_dimu_begin(emu.buf, 0, max_ini)
            check(ref, emu, f"begin at {i}")
            continue
        n, m = step
        own = samples(rng, m, 100.0 + 0.1 * i)
        a, b = ref.frame(n, own, 100.0 + 0.1 * i), emu.frame(n, own, 100.0 + 0.1 * i)
        assert a == b, (i, a, b)
        out, _ = emu.read()
        assert int(out[13]) == (n if a[0] in (2, 3) else 0) and int(out[14]) == (n if a[0] == 2 else 0) and int(out[15]) == (n if a[0] == 3 else 0)
        check(ref, emu, f"frame {i}")
        branches.append(a[0])
    return branches


def test_scripted_sequence(lib):
    script = [(0, 1), (1, 2), (2, 1),            # drops during the initialisation (counts 0, 1), then a 2-point cloud: N = 5 > 3
              (1, 3), (0, 0), (2, 2),            # drops right after it, an empty batch, then the map (branch 2)
              (5000, 12), (1, 4), (0, 4), (300, 6), (2, 0),   # branch 3, repeated drops, the carried samples consumed, an empty batch
              (1, 10), (1, 10), (100, 1),        # 10 + 10 > 16: the second drop overflows and loses its samples
              "begin", (0, 2), (1, 1), (7, 0), (9, 1), (9, 3)]   # reset mid-stream: the carry discarded, the means restart from
    br = run(lib, script)                                          # N = 1 (3 samples: N = 4 > 3), the map stays built
    assert br == [4, 4, 1, 4, 4, 2, 3, 4, 4, 3, 3, 4, 4, 3, 4, 4, 1, 3, 3], br


def test_empty_batches_keep_initialising(lib):
    br = run(lib, [(10, 0), (10, 0), (0, 3), (10, 0), (10, 2), (10, 1)], max_ini=4)
    assert br == [1, 1, 4, 1, 1, 2], br   # 3 carried + 0 own: N = 4, not > 4; 2 more: N = 6 ends the phase in that branch-1 frame


@pytest.mark.parametrize("seed", range(6))
def test_seeded_sequences(lib, seed):
    rng = np.random.default_rng([seed, 7])
    script = []
    for _ in range(120):
        u = rng.uniform()
        if u < 0.03:
            script.append("begin")
        else:
            n = int(rng.choice([0, 1, 2, 3, 50000], p=[0.2, 0.2, 0.2, 0.2, 0.2]))
            script.append((n, int(rng.integers(0, 9))))
    run(lib, script, max_ini=int(rng.integers(0, 30)), max_imu=int(rng.integers(8, 24)), seed=seed)


def test_init_equals_host_chain(lib, chain_lib):
    """the device IMU_init (dimu_init) equals the host chain's imu_init_batch, batch by batch"""
    rng = np.random.default_rng(5)
    emu = Emu(lib, 10 ** 6, 64)
    st = np.array([0.0, 0.0, -1.0, 0.0, 0.0, 0.0, 1.0, 1.0])
    for i in range(12):
        own = samples(rng, int(rng.integers(0, 9)), float(i))
        emu.frame(100, own, float(i))
        grav = np.zeros(3)
        if own.shape[0]:
            norm = chain_lib.emu_imu_init(_d(st), 0, _d(np.ascontiguousarray(own)), own.shape[0], _d(grav))
            assert emu.state[21:24].tobytes() == grav.tobytes()
            assert norm == np.sqrt((st[0] * st[0] + st[1] * st[1]) + st[2] * st[2])
        out, _ = emu.read()
        assert out[0:6].tobytes() == st[0:6].tobytes() and out[6] == st[6]
