"""Synthetic IMU-driven streams for the IMU-enabled scan loop (immesh_lio_step_async_imu) and their oracle chain.  TEST INFRASTRUCTURE.

make_imu_stream: an Avia-shaped scan stream (synth.make_scan, the LiDAR at 10 Hz) with the 200 Hz IMU samples of the same trajectory --
gyro from the relative rotation, specific force R^T (a - g), seeded noise and biases -- and per-point curvature stamps over the 0.1 s
scan.  OracleChain runs ImuProcess::Process2 + the rest of service_LiDAR_update on the CPU: IMU_init restated here in numpy in the
reference's order, OracleImu.undistort, oa.kitti_calib, oa.voxel_grid, OracleLio and OracleMesh, the state carried between them."""
import dataclasses
import math

import numpy as np

import oracle_api as oa
from immesh_b200 import api, synth

G = np.array([0.0, 0.0, -9.81])
IMU_HZ = 200.0
SCAN_DT = 0.1
T0 = 1000.0


def imu_cfg():
    return dict(cov_gyr=[0.1, 0.1, 0.1], cov_acc=[0.1, 0.1, 0.1], cov_bias_gyr=[1e-4, 1e-4, 1e-4], cov_bias_acc=[1e-4, 1e-4, 1e-4],
                mean_acc_norm=9.81, lid_R=np.eye(3), lid_T=list(api.AVIA.ext_T))


def _log_so3(R):
    c = max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0))
    th = math.acos(c)
    w = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return 0.5 * w if th < 1e-9 else th / (2.0 * math.sin(th)) * w


def make_imu_stream(n_scans, seed=0, n_points=None, kind="avia", empty_batch=None, speed=1.0):
    """scans[k] = dict(beg, imu float64[m,7], pts float32[n,4]); scan k covers [T0 + 0.1 k, T0 + 0.1 (k + 1)] and its points are cast
    from the pose at the scan end.  empty_batch: index of a scan whose IMU batch is empty (its samples are lost)."""
    sensor = dataclasses.replace(synth.make_sensor(kind, n_points), hz=1.0 / SCAN_DT, speed=speed)
    rng = np.random.default_rng([seed, 99])
    pose = lambda t: synth.trajectory_pose(sensor, (t - T0) / SCAN_DT)   # noqa: E731
    b_g, b_a = np.array([0.002, -0.001, 0.0015]), np.array([0.03, -0.02, 0.05])
    h = 1e-3
    scans = []
    for k in range(n_scans):
        beg = T0 + SCAN_DT * k
        body, _, _ = synth.make_scan(sensor, k + 1, seed, ext_T=np.asarray(api.AVIA.ext_T))
        n = body.shape[0]
        curv = rng.uniform(0.0, 100.0, n).astype(np.float32)
        curv[-1] = np.float32(99.9)                              # the scan's end stamp (UndistortPcl reads the LAST point's)
        pts = np.concatenate([body, curv[:, None]], axis=1).astype(np.float32)
        j0, j1 = int(round((beg - T0) * IMU_HZ)), int(round((beg + SCAN_DT - T0) * IMU_HZ))
        rows = []
        for j in range(j0, j1):
            t = T0 + (j + 1) / IMU_HZ - 0.5 / IMU_HZ
            R0, p0 = pose(t - h)
            R1, p1 = pose(t)
            R2, p2 = pose(t + h)
            gyr = _log_so3(R0.T @ R2) / (2 * h) + b_g + rng.normal(0, 0.002, 3)
            acc = (p2 - 2 * p1 + p0) / (h * h)
            f = R1.T @ (acc - G) + b_a + rng.normal(0, 0.02, 3)
            rows.append([t, *gyr, *f])
        imu = np.array(rows, dtype=np.float64).reshape(-1, 7)
        if k == empty_batch:
            imu = imu[:0]
        scans.append(dict(beg=beg, imu=imu, pts=pts))
    return sensor, scans


def true_velocity(sensor, t):
    """world-frame velocity of the trajectory at time t (finite difference)"""
    h = 1e-3
    _, p0 = synth.trajectory_pose(sensor, (t - h - T0) / SCAN_DT)
    _, p1 = synth.trajectory_pose(sensor, (t + h - T0) / SCAN_DT)
    return (p1 - p0) / (2 * h)


class InitRef:
    """IMU_init, StatesGroup version (IMU_Processing.cpp:188-232), with ImuProcess::Reset() (:73-86), in the reference's order."""

    def __init__(self):
        self.first = True
        self.reset()

    def reset(self):
        self.mean_acc = np.array([0.0, 0.0, -1.0])
        self.mean_gyr = np.zeros(3)
        self.N = 1

    def batch(self, imu):
        if self.first:
            self.reset()
            self.first = False
            self.mean_acc = imu[0, 4:7].copy()
            self.mean_gyr = imu[0, 1:4].copy()
        for row in imu:
            N = float(self.N)
            self.mean_acc = self.mean_acc + (row[4:7] - self.mean_acc) / N
            self.mean_gyr = self.mean_gyr + (row[1:4] - self.mean_gyr) / N
            self.N += 1
        m = self.mean_acc
        norm = math.sqrt((m[0] * m[0] + m[1] * m[1]) + m[2] * m[2])
        return norm, -m / norm * 9.81


class OracleChain:
    """The reference's imu_en loop on the CPU oracle; step() returns the branch (1 initialising, 2 map built, 3 localised + meshed)."""

    def __init__(self, cfg, icfg, mesh_cfg, max_ini, state0, leaf, calib=False):
        self.cfg, self.icfg, self.max_ini, self.leaf, self.calib = cfg, icfg, max_ini, leaf, calib
        self.lio = oa.OracleLio(cfg, sum_mode=0)
        self.mesh = oa.OracleMesh(mesh_cfg) if mesh_cfg is not None else None
        self.st = np.array(state0, dtype=np.float64)
        self.init = InitRef()
        self._imus = {}
        self.map_built = False
        self.frames = 0
        self.init_begin(first=True)

    def init_begin(self, first=False):
        """immesh_imu_init_begin: a fresh ImuProcess (first) or Reset()"""
        self.init_phase = True
        self.init.reset()
        self.last_imu = np.zeros(7)
        self.angvel_last = np.zeros(3)
        if first:
            self.acc_s_last = np.zeros(3)
            self.last_lidar_end_time = 0.0
            self.last_update_time = 0.0

    def _imu(self, norm):
        if norm not in self._imus:
            c = dict(self.icfg)
            c["mean_acc_norm"] = norm
            self._imus[norm] = oa.OracleImu(c)
        return self._imus[norm]

    def step(self, imu, pts, beg):
        end = beg + float(pts[-1, 3]) / 1000.0
        if self.init_phase:
            self.last_update_time = end
            if imu.shape[0] == 0:
                return 1
            norm, grav = self.init.batch(imu)
            self.st[0:9] = np.eye(3).reshape(9)
            self.st[15:18] = 0.0
            self.st[21:24] = grav
            self.last_imu = imu[-1].copy()
            if self.init.N > self.max_ini:
                self.init_phase = False
                self.norm = norm
            return 1
        o = self._imu(self.norm)
        o.reset(self.last_imu, self.last_lidar_end_time, self.last_update_time, self.acc_s_last, self.angvel_last)
        self.st, und, poses = o.undistort(self.st, imu, pts, beg)
        self.last_update_time = self.last_lidar_end_time = end
        if imu.shape[0]:
            self.last_imu = imu[-1].copy()
        self.acc_s_last, self.angvel_last = poses[-1, 1:4].copy(), poses[-1, 4:7].copy()
        full = und[:, :3].copy()
        if self.calib:
            full = oa.kitti_calib(full)
        self.lio.set_state(self.st)
        if not self.map_built:
            self.lio.voxel_map_init(full)
            self.map_built = True
            br = 2
        else:
            ds, _, _ = oa.voxel_grid(full, self.leaf)
            self.lio.lio_state_estimation(ds)
            self.lio.map_incremental_grow(ds)
            if self.mesh is not None:
                self.mesh.push_frame(self.lio.transform_full(full), self.lio.get_state()[9:12], self.frames)
                self.frames += 1
            br = 3
        self.st = self.lio.get_state()
        return br
