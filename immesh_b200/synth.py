"""Deterministic synthetic LiDAR scans for parity tests and benchmarks (SURVEY.md section 8d).

A closed piecewise-planar scene (ground, perimeter walls, boxes) with a few curved bodies
(spheres) so that non-planar voxels and octree splits occur, ray-cast from a sensor moving on a
smooth trajectory, with per-point range noise (sigma = dept_err) and bearing noise (sigma =
beam_err degrees).  Scans are body-frame float32 xyz exactly like pcl::PointXYZI; the
down-sampled cloud is a centroid voxel grid (what pcl::VoxelGrid produces at
src/voxel_mapping.cpp:1888-1889 of the reference -- the step *before* the hot path).
"""
from __future__ import annotations

import dataclasses
import numpy as np

# ----------------------------------------------------------------------------- scene
_BOXES = np.array(
    [
        # xmin, ymin, zmin, xmax, ymax, zmax
        [-8.0, 6.0, 0.0, -2.0, 12.0, 6.0],
        [4.0, 7.0, 0.0, 14.0, 14.0, 9.0],
        [20.0, 5.0, 0.0, 30.0, 11.0, 5.0],
        [-6.0, -13.0, 0.0, 2.0, -6.5, 7.0],
        [8.0, -12.0, 0.0, 18.0, -7.0, 4.0],
        [24.0, -14.0, 0.0, 34.0, -6.0, 8.0],
        [-20.0, 6.5, 0.0, -12.0, 13.0, 4.5],
        [-22.0, -12.0, 0.0, -11.0, -7.0, 6.0],
        [10.0, -2.0, 0.0, 11.0, -1.0, 2.5],   # a pole-like box
        [-3.0, 2.5, 0.0, -2.2, 3.3, 1.6],
        [38.0, -3.0, 0.0, 44.0, 3.0, 5.0],
    ],
    dtype=np.float64,
)
_ROOM = np.array([-60.0, -30.0, 0.0, 60.0, 30.0, 40.0])  # rays hit its inside faces (ground + perimeter walls); no ceiling return
_SPHERES = np.array(
    [
        # cx, cy, cz, r
        [2.0, 3.5, 0.4, 1.2],
        [16.0, -3.5, 0.2, 1.5],
        [-9.0, -3.0, 0.9, 0.9],
        [30.0, 2.0, 1.0, 2.0],
    ],
    dtype=np.float64,
)


def _raycast(origin: np.ndarray, dirs: np.ndarray, max_range: float) -> np.ndarray:
    """Nearest hit distance along unit rays (inf when nothing within max_range)."""
    n = dirs.shape[0]
    best = np.full(n, np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
        # outside boxes: slab test
        for b in _BOXES:
            t1 = (b[:3] - origin) * inv
            t2 = (b[3:] - origin) * inv
            tmin = np.nanmax(np.minimum(t1, t2), axis=1)
            tmax = np.nanmin(np.maximum(t1, t2), axis=1)
            hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 1e-6)
            best = np.where(hit & (tmin < best), tmin, best)
        # room: we are inside, take the exit distance, drop ceiling hits
        t1 = (_ROOM[:3] - origin) * inv
        t2 = (_ROOM[3:] - origin) * inv
        tfar = np.maximum(t1, t2)
        texit = np.nanmin(tfar, axis=1)
        axis = np.nanargmin(tfar, axis=1)
        ceiling = (axis == 2) & (dirs[:, 2] > 0)
        ok = (~ceiling) & (texit > 1e-6)
        best = np.where(ok & (texit < best), texit, best)
        for s in _SPHERES:
            oc = origin - s[:3]
            bq = dirs @ oc
            cq = oc @ oc - s[3] * s[3]
            disc = bq * bq - cq
            t = -bq - np.sqrt(np.where(disc > 0, disc, np.nan))
            hit = (disc > 0) & (t > 1e-6)
            best = np.where(hit & (t < best), t, best)
    best[best > max_range] = np.inf
    return best


# open-ended scene: the boxes and spheres above repeated along x every _OPEN_PERIOD metres, the ground and the two long side walls of
# the room, no end walls -- a straight drive through it keeps reaching new ground for as long as it lasts
_OPEN_PERIOD = 80.0


def _raycast_open(origin: np.ndarray, dirs: np.ndarray, max_range: float) -> np.ndarray:
    """Nearest hit distance along unit rays in the open-ended scene (inf when nothing within max_range)."""
    n = dirs.shape[0]
    best = np.full(n, np.inf)
    lo, hi = origin[0] - max_range - _BOXES[:, 3].max(), origin[0] + max_range - _BOXES[:, 0].min()
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
        for k in range(int(np.floor(lo / _OPEN_PERIOD)), int(np.ceil(hi / _OPEN_PERIOD)) + 1):
            shift = np.array([k * _OPEN_PERIOD, 0.0, 0.0])
            for b in _BOXES:
                t1 = (b[:3] + shift - origin) * inv
                t2 = (b[3:] + shift - origin) * inv
                tmin = np.nanmax(np.minimum(t1, t2), axis=1)
                tmax = np.nanmin(np.maximum(t1, t2), axis=1)
                hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 1e-6)
                best = np.where(hit & (tmin < best), tmin, best)
            for sp in _SPHERES:
                oc = origin - (sp[:3] + shift)
                bq = dirs @ oc
                cq = oc @ oc - sp[3] * sp[3]
                disc = bq * bq - cq
                t = -bq - np.sqrt(np.where(disc > 0, disc, np.nan))
                hit = (disc > 0) & (t > 1e-6)
                best = np.where(hit & (t < best), t, best)
        tg = np.where(dirs[:, 2] < 0, (_ROOM[2] - origin[2]) * inv[:, 2], np.inf)            # ground
        tw = np.where(dirs[:, 1] > 0, (_ROOM[4] - origin[1]) * inv[:, 1],
                      np.where(dirs[:, 1] < 0, (_ROOM[1] - origin[1]) * inv[:, 1], np.inf))  # side walls
        for t in (tg, tw):
            best = np.where((t > 1e-6) & (t < best), t, best)
    best[best > max_range] = np.inf
    return best


def _rot_z(a: float) -> np.ndarray:
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _rot_y(a: float) -> np.ndarray:
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


@dataclasses.dataclass
class SensorModel:
    name: str
    n_points: int
    blind: float
    max_range: float
    dept_err: float   # metres
    beam_err: float   # degrees
    hz: float
    speed: float      # m/s along the trajectory

    def directions(self, rng: np.random.Generator) -> np.ndarray:
        raise NotImplementedError


class Avia(SensorModel):
    """Livox Avia shape: 70.4 x 77.2 deg forward FoV, non-repetitive (uniform random) pattern."""

    def directions(self, rng):
        n = self.n_points
        az = np.deg2rad(rng.uniform(-35.2, 35.2, n))
        el = np.deg2rad(rng.uniform(-38.6, 38.6, n))
        return np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], axis=1)


class Spinning(SensorModel):
    """Ring LiDAR shape (HDL-64: 64 rings +2 .. -24.8 deg; Ouster-128: 128 rings +-22.5 deg)."""

    rings: int = 64
    el_hi: float = 2.0
    el_lo: float = -24.8

    def directions(self, rng):
        rings = self.rings
        cols = self.n_points // rings
        el = np.deg2rad(np.linspace(self.el_hi, self.el_lo, rings))
        az = np.linspace(-np.pi, np.pi, cols, endpoint=False) + rng.uniform(0, 2 * np.pi / cols)
        azg, elg = np.meshgrid(az, el, indexing="xy")  # ring-major like a packet stream
        azg = azg.T.reshape(-1)
        elg = elg.T.reshape(-1)
        return np.stack([np.cos(elg) * np.cos(azg), np.cos(elg) * np.sin(azg), np.sin(elg)], axis=1)


def make_sensor(kind: str, n_points: int | None = None) -> SensorModel:
    if kind == "avia":
        return Avia("avia", n_points or 24000, 1.0, 300.0, 0.02, 0.05, 100.0, 1.0)
    if kind == "avia100k":
        return Avia("avia100k", n_points or 100000, 1.0, 300.0, 0.02, 0.05, 10.0, 1.0)
    if kind == "hdl64":
        s = Spinning("hdl64", n_points or 131072, 2.0, 120.0, 0.04, 0.1, 10.0, 10.0)
        s.rings, s.el_hi, s.el_lo = 64, 2.0, -24.8
        return s
    if kind == "hdl64loop":
        s = Spinning("hdl64loop", n_points or 131072, 2.0, 120.0, 0.04, 0.1, 10.0, 10.0)
        s.rings, s.el_hi, s.el_lo = 64, 2.0, -24.8
        return s
    if kind == "hdl64open":
        # the HDL-64 shape on a straight drive through the open-ended scene (trajectory_pose's weave along +x, 1 m per scan)
        s = Spinning("hdl64open", n_points or 131072, 2.0, 120.0, 0.04, 0.1, 10.0, 10.0)
        s.rings, s.el_hi, s.el_lo = 64, 2.0, -24.8
        return s
    if kind == "ouster1m":
        s = Spinning("ouster1m", n_points or 1048576, 0.5, 120.0, 0.02, 0.05, 10.0, 2.0)
        s.rings, s.el_hi, s.el_lo = 128, 22.5, -22.5
        return s
    raise ValueError(kind)


def _loop_pose(s: float) -> tuple[np.ndarray, np.ndarray]:
    """Closed race-track loop inside the scene (two 58 m straights at y = -5 / +5 joined by half circles): the KITTI-seq-00-shape
    stream (BASELINE config C4, 4541 scans) revisits its own map lap after lap."""
    L, r = 58.0, 5.0
    per = 2 * L + 2 * np.pi * r
    u = s % per
    if u < L:                       # lower straight, heading +x
        x, y, yaw = -26.0 + u, -r, 0.0
    elif u < L + np.pi * r:         # right turn-around
        a = (u - L) / r
        x, y, yaw = 32.0 + r * np.sin(a), -r * np.cos(a), a
    elif u < 2 * L + np.pi * r:     # upper straight, heading -x
        x, y, yaw = 32.0 - (u - L - np.pi * r), r, np.pi
    else:
        a = (u - 2 * L - np.pi * r) / r
        x, y, yaw = -26.0 - r * np.sin(a), r * np.cos(a), np.pi + a
    z = 1.73 + 0.03 * np.sin(0.5 * s)
    return _rot_z(yaw) @ _rot_y(0.008 * np.sin(0.3 * s)), np.array([x, y, z])


def trajectory_pose(sensor: SensorModel, k: int) -> tuple[np.ndarray, np.ndarray]:
    """Ground-truth IMU/body pose of scan k (R, t): smooth forward motion with a gentle weave."""
    dt = 1.0 / sensor.hz
    s = sensor.speed * dt * k
    if sensor.name.endswith("loop"):
        return _loop_pose(s)
    x = -30.0 + s
    y = 1.2 * np.sin(0.15 * s)
    z = 1.6 + 0.05 * np.sin(0.4 * s)
    yaw = 0.18 * np.cos(0.15 * s) * 1.2 * 0.15 + 0.05 * np.sin(0.07 * s)
    pitch = 0.01 * np.sin(0.3 * s)
    return _rot_z(yaw) @ _rot_y(pitch), np.array([x, y, z])


def voxel_grid_downsample(pts: np.ndarray, leaf: float) -> np.ndarray:
    """Centroid per occupied leaf (pcl::VoxelGrid semantics), float32 in/out, leaves in index order."""
    if pts.shape[0] == 0:
        return pts.astype(np.float32)
    p = pts.astype(np.float64)
    mn = np.floor(p.min(axis=0) / leaf)
    ijk = (np.floor(p / leaf) - mn).astype(np.int64)
    dims = ijk.max(axis=0) + 1
    key = ijk[:, 0] + dims[0] * (ijk[:, 1] + dims[1] * ijk[:, 2])
    uniq, inv = np.unique(key, return_inverse=True)
    cnt = np.bincount(inv).astype(np.float64)
    out = np.stack([np.bincount(inv, weights=p[:, j]) / cnt for j in range(3)], axis=1)
    return out.astype(np.float32)


def make_scan(sensor: SensorModel, k: int, seed: int, ext_R: np.ndarray | None = None, ext_T: np.ndarray | None = None):
    """Scan k of the stream: (body_full float32[N,3], R_true, t_true).  Points are in the LiDAR frame;
    ext_R/ext_T (LiDAR -> IMU/body) default to identity / zero."""
    rng = np.random.default_rng([seed, k])
    R, t = trajectory_pose(sensor, k)
    eR = np.eye(3) if ext_R is None else np.asarray(ext_R, dtype=np.float64).reshape(3, 3)
    eT = np.zeros(3) if ext_T is None else np.asarray(ext_T, dtype=np.float64)
    d_l = sensor.directions(rng)                  # LiDAR frame
    RL = R @ eR                                   # LiDAR -> world rotation
    oL = R @ eT + t                               # LiDAR origin in world
    d_w = d_l @ RL.T
    rng_true = (_raycast_open if sensor.name.endswith("open") else _raycast)(oL, d_w, sensor.max_range)
    ok = np.isfinite(rng_true) & (rng_true > sensor.blind)
    d_l = d_l[ok]
    r = rng_true[ok] + rng.normal(0.0, sensor.dept_err, ok.sum())
    # bearing noise: small random rotation of the direction
    sig = np.deg2rad(sensor.beam_err)
    pert = rng.normal(0.0, sig, (d_l.shape[0], 3))
    d_n = d_l + np.cross(pert, d_l)
    d_n /= np.linalg.norm(d_n, axis=1, keepdims=True)
    body = (d_n * r[:, None]).astype(np.float32)
    return body, R, t


def make_gt_cloud(kind: str, n_scans: int, seed: int = 0, n_points: int | None = None, ext_R=None, ext_T=None) -> np.ndarray:
    """The noise-free world-frame hits of exactly the rays make_scan draws for scans 0 .. n_scans - 1 (the ground truth of
    make_stream with the same arguments), float32[N,3] in scan order.  make_scan's random stream is replayed, not changed."""
    sensor = make_sensor(kind, n_points)
    eR = np.eye(3) if ext_R is None else np.asarray(ext_R, dtype=np.float64).reshape(3, 3)
    eT = np.zeros(3) if ext_T is None else np.asarray(ext_T, dtype=np.float64)
    out = []
    for k in range(n_scans):
        rng = np.random.default_rng([seed, k])
        R, t = trajectory_pose(sensor, k)
        d_w = sensor.directions(rng) @ (R @ eR).T
        oL = R @ eT + t
        rng_true = _raycast(oL, d_w, sensor.max_range)
        ok = np.isfinite(rng_true) & (rng_true > sensor.blind)
        out.append((oL + d_w[ok] * rng_true[ok, None]).astype(np.float32))
    return np.concatenate(out) if out else np.zeros((0, 3), dtype=np.float32)


def make_stream(kind: str, n_scans: int, seed: int = 0, leaf: float = 0.4, n_points: int | None = None,
                ext_R=None, ext_T=None):
    """List of dicts with body_full, body_ds (voxel-grid down-sampled), R_true, t_true, dt."""
    sensor = make_sensor(kind, n_points)
    out = []
    for k in range(n_scans):
        body, R, t = make_scan(sensor, k, seed, ext_R, ext_T)
        out.append(dict(body_full=body, body_ds=voxel_grid_downsample(body, leaf), R_true=R, t_true=t, dt=1.0 / sensor.hz))
    return sensor, out
