"""Depth-camera frames for the tests: synthetic depth images ray-cast from the synth scenes with a pinhole camera along
synth.trajectory_pose, and an independent numpy restatement of the unprojection documented in include/immesh_b200.h
(immesh_depth_frame): float64 in the written order, so that it equals the device's points bit for bit."""
import numpy as np

from immesh_b200 import synth
from immesh_b200.api import DEPTH_FORMATS, DEPTH_KINDS, DepthCamera

# body (x forward, y left, z up) -> OpenCV camera (x right, y down, z forward): the camera's axes in body coordinates, as columns
BODY_FROM_CAM = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])


def camera(width=160, height=120, fov_deg=70.0, **kw):
    f = 0.5 * width / np.tan(np.deg2rad(fov_deg) / 2)
    return DepthCamera(fx=f, fy=f, cx=(width - 1) / 2, cy=(height - 1) / 2, **kw)


def camera_pose(k, speed=0.25):
    """camera to world of frame k: the synth trajectory (a sensor at 10 Hz moving `speed` m per frame), camera looking forward"""
    sensor = synth.make_sensor("avia")
    sensor.hz, sensor.speed = 10.0, speed * 10.0
    R, t = synth.trajectory_pose(sensor, k)
    return R @ BODY_FROM_CAM, np.asarray(t, dtype=np.float64)


def render(cam: DepthCamera, width, height, R, t, kind="planar", fmt="f32", max_range=60.0):
    """the depth image of the synth scene seen by cam at (R, t): misses are NaN (f32) or 0 (u16)"""
    v, u = np.mgrid[0:height, 0:width].astype(np.float64)
    dc = np.stack([(u - cam.cx) / cam.fx, (v - cam.cy) / cam.fy, np.ones_like(u)], axis=-1).reshape(-1, 3)
    norm = np.linalg.norm(dc, axis=1)
    rng = synth._raycast(t, (dc / norm[:, None]) @ R.T, max_range)
    d = rng / norm if kind == "planar" else rng
    d = d.reshape(height, width)
    if fmt == "f32":
        return np.where(np.isfinite(d), d, np.nan).astype(np.float32)
    q = np.where(np.isfinite(d), np.round(d / cam.depth_scale), 0)
    return np.clip(q, 0, 65535).astype(np.uint16)


def inject_edges(img, cam: DepthCamera, rng):
    """the edge values on scattered pixels: NaN, +-inf, 0, 65535 and depths exactly at z_min / z_max (planar) -- in place"""
    flat = img.reshape(-1)
    idx = rng.permutation(flat.size)
    n = max(flat.size // 50, 8)
    if img.dtype == np.float32:
        vals = [np.nan, np.inf, -np.inf, 0.0, -1.0, np.float32(cam.z_min), np.float32(cam.z_max), 65535.0]
    else:
        vals = [0, 65535, int(round(cam.z_min / cam.depth_scale)), int(cam.z_max / cam.depth_scale)]
    for i, val in enumerate(vals):
        flat[idx[i * n:(i + 1) * n]] = val
    return img


def unproject(img, cam: DepthCamera, R, t):
    """the valid sampled pixels' world points float32[n][3] in ascending pixel order, and their pixel indices"""
    h, w = img.shape
    s = cam.stride
    v, u = np.mgrid[0:h:s, 0:w:s]
    raw = img[::s, ::s]
    if img.dtype == np.uint16:
        ok = raw != 0
        d = raw.astype(np.float64) * cam.depth_scale
    else:
        ok = np.isfinite(raw)
        d = raw.astype(np.float64)
    a = (u.astype(np.float64) - cam.cx) / cam.fx
    b = (v.astype(np.float64) - cam.cy) / cam.fy
    with np.errstate(invalid="ignore"):
        z = d / np.sqrt((a * a + b * b) + 1.0) if cam.kind == "range" else d
        ok &= (cam.z_min <= z) & (z <= cam.z_max)
    a, b, z = a[ok], b[ok], z[ok]
    x, y = a * z, b * z
    R = np.asarray(R, dtype=np.float64)
    t = np.asarray(t, dtype=np.float64)
    pts = np.stack([((R[i, 0] * x + R[i, 1] * y) + R[i, 2] * z) + t[i] for i in range(3)], axis=1).astype(np.float32)
    return pts, (v * w + u)[ok].astype(np.int32)


def append_dims(n, append_target):
    """append_point_step = max(1, round(n // appending_pts_frame)) and m = ceil(n / step) (ImMesh_mesh_reconstruction.cpp:111)"""
    step = max(1, int(round(float(n // append_target))))
    return step, -(-n // step)


def cam_array(cam: DepthCamera, R, t):
    """fx fy cx cy z_min z_max depth_scale R[9] t[3] (the host emulation's layout)"""
    return np.concatenate([[cam.fx, cam.fy, cam.cx, cam.cy, cam.z_min, cam.z_max, cam.depth_scale], np.asarray(R, np.float64).reshape(9),
                           np.asarray(t, np.float64)]).astype(np.float64)


FORMATS, KINDS = DEPTH_FORMATS, DEPTH_KINDS
