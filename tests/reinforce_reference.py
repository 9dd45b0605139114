"""Independent numpy restatements for the LiDAR point-cloud reinforcement (ImMesh_node.cpp:302-329): get_last_avr_pose (:169-206) with
scipy's Rotation, and a per-pixel rasteriser that follows the sampling rule documented for immesh_mesh_render_depth.  TEST INFRASTRUCTURE."""
import numpy as np
from scipy.spatial.transform import Rotation

# lidar_frame_to_camera_frame (ImMesh_node.cpp:172-174)
L2C = np.array([[0.0, 0.0, -1.0], [-1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])


def avr_pose(poses, frame, win):
    """Camera pose of frame `frame` (frames counted from 1; the reference's current frame is frame - 1).  poses: {frame: (R, t)} of
    the frames that recorded one.  Frames [max(1, frame - win), frame): R_first exp(mean log(R_first^T R_i)) L2C and the mean t;
    the identity when the window holds no pose (the reference's cur < 1)."""
    window = [poses[f] for f in range(max(1, frame - win), frame) if f in poses]
    if not window:
        return np.eye(3), np.zeros(3)
    r_first = Rotation.from_matrix(window[0][0])
    logs = np.array([(r_first.inv() * Rotation.from_matrix(R)).as_rotvec() for R, _ in window])
    t = np.sum([t for _, t in window], axis=0) / len(window)
    R = (r_first * Rotation.from_rotvec(logs.mean(axis=0))).as_matrix() @ L2C
    return R, t


def raster(K, w, h, z_near, z_far, R, t, verts, tris):
    """The documented sampling rule, pixel by pixel: samples at integer pixel coordinates, covered when the three edge functions share a
    sign (zero included), 1/z interpolated affinely, nearest sample wins, triangles with a vertex outside (z_near, z_far) skipped; valid
    where depth < 0.99 z_far; points unprojected (world = R diag(1,-1,-1) p + t) in ascending pixel order.  Float64 throughout, the
    same expression order as the device code, so the floats agree."""
    fx, fy, cx, cy = K
    R = np.asarray(R, np.float64)
    depth = np.full((h, w), np.inf, np.float32)
    for tri in tris:
        P = verts[tri].astype(np.float64) - t
        xc = (R[0, 0] * P[:, 0] + R[1, 0] * P[:, 1]) + R[2, 0] * P[:, 2]
        yc = -((R[0, 1] * P[:, 0] + R[1, 1] * P[:, 1]) + R[2, 1] * P[:, 2])
        zc = -((R[0, 2] * P[:, 0] + R[1, 2] * P[:, 1]) + R[2, 2] * P[:, 2])
        if not np.all((zc > z_near) & (zc < z_far)):
            continue
        u = fx * xc / zc + cx
        v = fy * yc / zc + cy
        area = (u[1] - u[0]) * (v[2] - v[0]) - (v[1] - v[0]) * (u[2] - u[0])
        if area == 0.0:
            continue
        x0, x1 = max(0, int(np.ceil(u.min()))), min(w - 1, int(np.floor(u.max())))
        y0, y1 = max(0, int(np.ceil(v.min()))), min(h - 1, int(np.floor(v.max())))
        if x0 > x1 or y0 > y1:
            continue
        py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1].astype(np.float64)
        e0 = (u[2] - u[1]) * (py - v[1]) - (v[2] - v[1]) * (px - u[1])
        e1 = (u[0] - u[2]) * (py - v[2]) - (v[0] - v[2]) * (px - u[2])
        e2 = (u[1] - u[0]) * (py - v[0]) - (v[1] - v[0]) * (px - u[0])
        cov = ((e0 >= 0) & (e1 >= 0) & (e2 >= 0)) | ((e0 <= 0) & (e1 <= 0) & (e2 <= 0))
        with np.errstate(divide="ignore", invalid="ignore"):
            iz = ((e0 * (1.0 / zc[0]) + e1 * (1.0 / zc[1])) + e2 * (1.0 / zc[2])) / area
            zf = (1.0 / iz).astype(np.float32)
        cov &= zf > 0
        sub = depth[y0:y1 + 1, x0:x1 + 1]
        depth[y0:y1 + 1, x0:x1 + 1] = np.where(cov, np.minimum(sub, zf), sub)
    valid = depth.astype(np.float64) < z_far * 0.99
    pix = np.nonzero(valid.reshape(-1))[0].astype(np.int32)
    val = depth.reshape(-1)[pix].astype(np.float64)
    x, y = (pix % w).astype(np.float64), (pix // w).astype(np.float64)
    g = np.stack([((x - cx) / fx) * val, -(((y - cy) / fy) * val), -val], axis=1)
    pts = ((((R[:, 0][None] * g[:, 0:1]) + (R[:, 1][None] * g[:, 1:2])) + (R[:, 2][None] * g[:, 2:3])) + t).astype(np.float32)
    return np.where(valid, depth, np.float32(-1.0)), pts, pix
