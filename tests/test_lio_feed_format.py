"""CPU tier: the scan feed's host-side formatters against numpy / scipy -- immesh_odometry_pose (RotMtoEuler, both branches, then tf's
setRPY quaternion) and immesh_lio_state_line (Log of so3_math.h in its three cases, byte for byte against a "%f " restatement)."""
import math

import numpy as np
from scipy.spatial.transform import Rotation

from immesh_b200 import api


def _state(R, rng):
    s = np.zeros(348)
    s[0:9] = np.asarray(R, dtype=np.float64).reshape(9)
    s[9:24] = rng.normal(0, 5, 15)
    return s


def _rot_m_to_euler(R):
    """include/so3_math.h RotMtoEuler, restated"""
    sy = math.sqrt(R[0, 0] * R[0, 0] + R[1, 0] * R[1, 0])
    if not sy < 1e-6:
        return math.atan2(R[2, 1], R[2, 2]), math.atan2(-R[2, 0], sy), math.atan2(R[1, 0], R[0, 0])
    return math.atan2(-R[1, 2], R[1, 1]), math.atan2(-R[2, 0], sy), 0.0


def _set_rpy(r, p, y):
    """tf::Quaternion::setRPY, restated: x y z w"""
    cy, sy, cp, sp, cr, sr = math.cos(y * 0.5), math.sin(y * 0.5), math.cos(p * 0.5), math.sin(p * 0.5), math.cos(r * 0.5), math.sin(r * 0.5)
    return (sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy)


def _log(R):
    """include/so3_math.h Log, restated"""
    tr = (R[0, 0] + R[1, 1]) + R[2, 2]
    theta = 0.0 if tr > 3.0 - 1e-6 else math.acos(0.5 * (tr - 1))
    K = (R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1])
    f = 0.5 if abs(theta) < 0.001 else 0.5 * theta / math.sin(theta)
    return [k * f for k in K]


def _line(s, t):
    R = s[0:9].reshape(3, 3)
    vals = [t, *_log(R), *s[9:12], 0.0, 0.0, 0.0, *s[12:15], 0.0, 0.0, 0.0, *s[15:18], *s[18:21], *s[21:24]]
    return "".join("%f " % v for v in vals) + "\r\n"


def _rotations(rng):
    Rs = list(Rotation.random(64, random_state=7).as_matrix())
    Rs.append(np.eye(3))
    Rs += [Rotation.from_euler("xyz", [a, s * math.pi / 2, c]).as_matrix() for a, c in ((0.3, -1.2), (2.0, 0.7)) for s in (1, -1)]  # gimbal lock: sy ~ 0
    Rs += [Rotation.from_rotvec(v).as_matrix() for v in rng.normal(0, 4e-4, (6, 3))]     # near the identity: Log sets theta to 0
    Rs += [Rotation.from_rotvec(v).as_matrix() for v in rng.normal(0, 1e-7, (3, 3))]     # trace above 3 - 1e-6
    Rs.append(Rotation.from_rotvec([0, 0, math.pi - 1e-9]).as_matrix())
    return Rs


def test_odometry_pose_matches_restatement_and_scipy():
    lib = api.load_library()
    rng = np.random.default_rng(3)
    singular = 0
    for R in _rotations(rng):
        s = _state(R, rng)
        got = api.odometry_pose(s, lib=lib)
        assert np.array_equal(got[:3], s[9:12])
        r, p, y = _rot_m_to_euler(R)
        singular += math.sqrt(R[0, 0] ** 2 + R[1, 0] ** 2) < 1e-6
        assert np.array_equal(got[3:], np.array(_set_rpy(r, p, y))), (got[3:], _set_rpy(r, p, y))
        # the quaternion is a unit quaternion of rot_end, up to sign, away from the singular branch (which drops the yaw)
        q = Rotation.from_quat(got[3:]).as_matrix()
        if math.sqrt(R[0, 0] ** 2 + R[1, 0] ** 2) >= 1e-6:
            assert np.allclose(q, R, atol=1e-9)
        assert abs(np.linalg.norm(got[3:]) - 1) < 1e-12
    assert singular >= 2


def test_odometry_pose_singular_branch():
    lib = api.load_library()
    R = Rotation.from_euler("ZYX", [0.9, math.pi / 2, 0.2]).as_matrix()   # pitch +90 degrees: r00 = r10 = 0
    R[0, 0] = R[1, 0] = 0.0
    s = _state(R, np.random.default_rng(1))
    got = api.odometry_pose(s, lib=lib)
    r, p, y = math.atan2(-R[1, 2], R[1, 1]), math.atan2(-R[2, 0], 0.0), 0.0
    assert np.array_equal(got[3:], np.array(_set_rpy(r, p, y)))


def test_state_line_bytes():
    lib = api.load_library()
    rng = np.random.default_rng(5)
    cases = {"identity": 0, "small": 0, "general": 0}
    for R in _rotations(rng):
        s = _state(R, rng)
        t = float(rng.uniform(0, 1000))
        line = api.lio_state_line(s, t, lib=lib)
        assert line == _line(s, t)
        assert line.endswith(" \r\n") and len(line.split()) == 25
        # Log's K / 2 branch: theta is set to 0 when the trace is above 3 - 1e-6 (acos never returns below 0.001 otherwise); the
        # identity, and rotations near it whose K is not zero
        tr = (R[0, 0] + R[1, 1]) + R[2, 2]
        theta = 0.0 if tr > 3.0 - 1e-6 else math.acos(0.5 * (tr - 1))
        cases["identity" if np.array_equal(R, np.eye(3)) else "small" if abs(theta) < 0.001 else "general"] += 1
        # Log agrees with scipy's rotation vector away from the small-angle approximation
        if abs(theta) >= 0.001 and theta < math.pi - 1e-6:
            assert np.allclose(_log(R), Rotation.from_matrix(R).as_rotvec(), atol=1e-9)
    assert all(v > 0 for v in cases.values()), cases


def test_state_line_capacity():
    import ctypes as C
    lib = api.load_library()
    s = np.zeros(348)
    s[0] = s[4] = s[8] = 1.0
    buf = C.create_string_buffer(16)
    assert lib.immesh_lio_state_line(s.ctypes.data_as(C.POINTER(C.c_double)), 1.0, buf, 16) == -3
    assert lib.immesh_odometry_pose(None, None) == -1
