"""Depth images through the localization, for the tests: an independent numpy restatement of the sensor-frame cloud documented in
include/immesh_b200.h (immesh_lio_step_async_depth) -- depth_reference.unproject with the camera-to-sensor mount, then the reference's
Preprocess::l515_handler filter (src/preprocess.cpp:250-256): every point_filter_num-th valid sample in pixel order, and the points
closer than blind dropped with the float32 squared range widened to float64."""
import numpy as np

import depth_reference as dr

# the x-forward, z-up sensor frame of an L515 mounted looking forward: camera -> sensor is BODY_FROM_CAM
SENSOR_FROM_CAM = dr.BODY_FROM_CAM


def filter_cloud(pts, pix, point_filter_num=1, blind=0.0):
    """the valid samples' points (ascending pixel order) -> the kept ones, and their pixel indices"""
    i = np.arange(pts.shape[0])
    keep = i % point_filter_num == 0
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    with np.errstate(over="ignore"):
        r = (x * x + y * y) + z * z          # float32, no FMA
    keep &= ~(r.astype(np.float64) < np.float64(blind) * np.float64(blind))
    return pts[keep], pix[keep]


def sensor_cloud(img, cam, mount_R=np.eye(3), mount_t=np.zeros(3), point_filter_num=1, blind=0.0):
    """the localization's cloud of one image: float32[n][3] in the sensor frame and the pixel index of each point"""
    pts, pix = dr.unproject(img, cam, mount_R, mount_t)
    return filter_cloud(pts, pix, point_filter_num, blind)


def sensor_pose(k, speed=0.25):
    """sensor (x forward, z up) to world of stream frame k: depth_reference.camera_pose with the mount taken off"""
    R, t = dr.camera_pose(k, speed)
    return R @ SENSOR_FROM_CAM.T, t


def state_from_pose(state, R, t):
    """a 348-double state with its rotation (row-major, slots 0..8) and position (9..11) set to (R, t)"""
    s = np.array(state, dtype=np.float64, copy=True)
    s[0:9] = np.asarray(R, dtype=np.float64).reshape(9)
    s[9:12] = t
    return s
