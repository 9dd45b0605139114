"""ctypes harness of the CPU oracle (oracle/liborc.so).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_ORC = os.path.join(_ROOT, "oracle", "liborc.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_ORC):
            subprocess.check_call(["make", "-C", os.path.join(_ROOT, "oracle")])
        L = C.CDLL(_ORC)
        L.orc_lio_create.restype = C.c_void_p
        L.orc_mesh_create.restype = C.c_void_p
        L.orc_mesh_create.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
        L.orc_lio_dump_map.restype = C.c_long
        L.orc_lio_num_root_voxels.restype = C.c_long
        L.orc_mesh_get_voxels.restype = C.c_long
        L.orc_lio_predict.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        L.orc_mesh_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
        L.orc_voxel_triangulate.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
        L.orc_calc_body_var.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p]
        L.orc_voxel_key.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class OracleLio:
    def __init__(self, cfg, sum_mode=0, omp_threads=1, solve_mode=0, plane_var_mode=0):
        L = lib()
        cd = np.array([cfg.voxel_size, cfg.min_eigen_value, cfg.dept_err, cfg.beam_err, *cfg.ext_R, *cfg.ext_T], dtype=np.float64)
        ci = np.array([cfg.max_layer, *cfg.layer_init_size, cfg.max_points_size, cfg.max_iteration, cfg.calib_laser, sum_mode, omp_threads, solve_mode, plane_var_mode], dtype=np.int32)
        self.h = C.c_void_p(L.orc_lio_create(_p(cd), _p(ci)))
        self.L = L

    def __del__(self):
        try:
            self.L.orc_lio_destroy(self.h)
        except Exception:
            pass

    def get_state(self):
        s = np.zeros(348)
        self.L.orc_lio_get_state(self.h, _p(s))
        return s

    def set_state(self, s):
        s = np.ascontiguousarray(s, dtype=np.float64)
        self.L.orc_lio_set_state(self.h, _p(s))

    def set_pose(self, R, t):
        s = self.get_state()
        s[0:9] = np.asarray(R, dtype=np.float64).reshape(9)
        s[9:12] = t
        self.set_state(s)

    def predict(self, dt, cov_gyr=0.1, cov_acc=0.1):
        self.L.orc_lio_predict(self.h, dt, cov_gyr, cov_acc)

    def voxel_map_init(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        self.L.orc_lio_map_init(self.h, _p(a), C.c_int(a.shape[0]))

    def lio_state_estimation(self, body, state_prop=None):
        a = np.ascontiguousarray(body, dtype=np.float32)
        sp = self.get_state() if state_prop is None else np.ascontiguousarray(state_prop, dtype=np.float64)
        self._n = a.shape[0]
        return self.L.orc_lio_estimate(self.h, _p(a), C.c_int(a.shape[0]), _p(sp))

    def map_incremental_grow(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        self.L.orc_lio_map_grow(self.h, _p(a), C.c_int(a.shape[0]))

    def iter_stats(self, it):
        o = np.zeros(63)
        self.L.orc_lio_iter_stats(self.h, C.c_int(it), _p(o))
        return dict(HTH=o[:36].reshape(6, 6).copy(), HTz=o[36:42].copy(), n_match=int(o[42]), total_residual=o[43], solution=o[44:62].copy(), converged=int(o[62]))

    def matches(self):
        idx = np.zeros(self._n, dtype=np.int32)
        lay = np.zeros(self._n, dtype=np.int32)
        m = self.L.orc_lio_last_matches(self.h, _p(idx), _p(lay), C.c_int(self._n))
        out = np.full(self._n, -1, dtype=np.int32)
        out[idx[:m]] = lay[:m]
        return out

    def residual_list(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        n = a.shape[0]
        il = np.zeros((n, 2), dtype=np.int32)
        vals = np.zeros((n, 31))
        m = self.L.orc_lio_residual_list(self.h, _p(a), C.c_int(n), _p(il), _p(vals), C.c_int(n))
        return il[:m], vals[:m]

    def transform_full(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        out = np.zeros_like(a)
        self.L.orc_lio_transform_full(self.h, _p(a), C.c_int(a.shape[0]), _p(out))
        return out

    def pv_lists(self, body, mode=0):
        """(pts_world f64[n,3], var f64[n,9]) as the reference builds its Point_with_var lists (mode 0: map growth, 1: matching)."""
        a = np.ascontiguousarray(body, dtype=np.float32)
        pw, v9 = np.zeros((a.shape[0], 3)), np.zeros((a.shape[0], 9))
        self.L.orc_lio_pv_lists(self.h, _p(a), C.c_int(a.shape[0]), C.c_int(mode), _p(pw), _p(v9))
        return pw, v9

    def build_pv(self, pts_world, var9):
        pw, v9 = np.ascontiguousarray(pts_world, dtype=np.float64), np.ascontiguousarray(var9, dtype=np.float64)
        self.L.orc_lio_build_pv(self.h, _p(pw), _p(v9), C.c_int(pw.shape[0]))

    def update_pv(self, pts_world, var9):
        pw, v9 = np.ascontiguousarray(pts_world, dtype=np.float64), np.ascontiguousarray(var9, dtype=np.float64)
        self.L.orc_lio_update_pv(self.h, _p(pw), _p(v9), C.c_int(pw.shape[0]))

    def residual_pv(self, pts_body, pts_world, var9):
        pb, pw, v9 = (np.ascontiguousarray(x, dtype=np.float64) for x in (pts_body, pts_world, var9))
        n = pb.shape[0]
        il, vals = np.zeros((n, 2), dtype=np.int32), np.zeros((n, 31))
        m = self.L.orc_lio_residual_pv(self.h, _p(pb), _p(pw), _p(v9), C.c_int(n), _p(il), _p(vals), C.c_int(n))
        return il[:m], vals[:m]

    def dump_map(self):
        rows = self.L.orc_lio_dump_map(self.h, None, C.c_long(0))
        out = np.zeros((rows, 45))
        self.L.orc_lio_dump_map(self.h, _p(out), C.c_long(rows))
        return out


class OracleMesh:
    def __init__(self, cfg, threads=1):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_mesh_create(cfg.points_minimum_scale, cfg.voxel_resolution, cfg.number_of_pts_append_to_map, threads))

    def __del__(self):
        try:
            self.L.orc_mesh_destroy(self.h)
        except Exception:
            pass

    def push_frame(self, pts, pose_t, frame_idx=0):
        a = np.ascontiguousarray(pts, dtype=np.float32)
        t = np.ascontiguousarray(pose_t, dtype=np.float64)
        self.L.orc_mesh_push_frame(self.h, _p(a), C.c_int(a.shape[0]), _p(t))

    def counts(self):
        o = np.zeros(8, dtype=np.int64)
        self.L.orc_mesh_counts(self.h, _p(o))
        keys = ["n_vertices", "n_triangles", "frame_new_vertices", "frame_voxels_meshed", "frame_added", "frame_removed", "n_voxels", "n_activated"]
        return dict(zip(keys, (int(v) for v in o)))

    def render_depth(self, intrinsics, width, height, z_near, z_far, cam_R, cam_t):
        K = np.ascontiguousarray(intrinsics, dtype=np.float64)
        R = np.ascontiguousarray(cam_R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(cam_t, dtype=np.float64)
        depth = np.zeros((height, width), dtype=np.float32)
        pts = np.zeros((height * width, 3), dtype=np.float32)
        pix = np.zeros(height * width, dtype=np.int32)
        self.L.orc_mesh_render_depth.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self.L.orc_mesh_render_depth.restype = C.c_long
        n = self.L.orc_mesh_render_depth(self.h, _p(K), width, height, z_near, z_far, _p(R), _p(t), _p(depth), _p(pts), _p(pix))
        return depth, pts[:n].copy(), pix[:n].copy()

    def smooth_all(self, smooth_factor=0.1, knn=20):
        out = np.zeros((self.counts()["n_vertices"], 3))
        self.L.orc_mesh_smooth_all.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_void_p]
        self.L.orc_mesh_smooth_all(self.h, smooth_factor, knn, _p(out))
        return out

    def region_keys(self, region_size=10.0):
        """region key of every live triangle, in the snapshot's (ascending triple) order"""
        self.L.orc_mesh_region_keys.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
        self.L.orc_mesh_region_keys.restype = C.c_long
        n = self.L.orc_mesh_region_keys(self.h, region_size, None)
        out = np.zeros((n, 3), dtype=np.int32)
        self.L.orc_mesh_region_keys(self.h, region_size, _p(out))
        return out

    def snapshot(self):
        c = self.counts()
        v = np.zeros((c["n_vertices"], 3), dtype=np.float32)
        s = np.zeros((c["n_vertices"], 3), dtype=np.float64)
        t = np.zeros((c["n_triangles"], 3), dtype=np.int32)
        f = np.zeros(c["n_triangles"], dtype=np.int32)
        self.L.orc_mesh_get_vertices(self.h, _p(v), _p(s))
        self.L.orc_mesh_get_tris(self.h, _p(t), _p(f))
        return v, t, f

    def frame_delta(self):
        c = self.counts()
        a = np.zeros((c["frame_added"], 3), dtype=np.int32)      # upper bounds (unique sets are smaller)
        r = np.zeros((c["frame_removed"], 3), dtype=np.int32)
        self.L.orc_mesh_get_frame_delta(self.h, _p(a), _p(r))
        return a, r

    def frame_voxel_stats(self):
        """One row per voxel meshed in the last frame, ascending key: dict of arrays key[m,3], n (dilated-set size), max_cav (largest
        Bowyer-Watson conflict region, ghost triangles included), seeded, ties (in-circle evaluations == 0), dups (same snapped point)."""
        self.L.orc_mesh_frame_voxel_stats.restype = C.c_long
        n = self.L.orc_mesh_frame_voxel_stats(self.h, None, C.c_long(0))
        o = np.zeros((n, 8), dtype=np.int64)
        self.L.orc_mesh_frame_voxel_stats(self.h, _p(o), C.c_long(n))
        return dict(key=o[:, 0:3].astype(np.int32), n=o[:, 3], max_cav=o[:, 4], seeded=o[:, 5].astype(bool), ties=o[:, 6], dups=o[:, 7])

    def voxels(self):
        n = self.L.orc_mesh_get_voxels(self.h, None, C.c_long(0))
        o = np.zeros((n, 4), dtype=np.int32)
        self.L.orc_mesh_get_voxels(self.h, _p(o), C.c_long(n))
        return o

    def knn(self, q, k, max_dist=float("inf")):
        a = np.ascontiguousarray(q, dtype=np.float32)
        idx = np.zeros((a.shape[0], k), dtype=np.int32)
        d2 = np.zeros((a.shape[0], k), dtype=np.float32)
        self.L.orc_mesh_knn(self.h, _p(a), a.shape[0], k, max_dist, _p(idx), _p(d2))
        return idx, d2


class OracleImu:
    """orc_imu.hpp: ImuProcess::UndistortPcl restatement."""

    def __init__(self, cfg: dict):
        self.L = lib()
        v = np.zeros(25)
        v[0:3], v[3:6], v[6:9], v[9:12] = cfg["cov_gyr"], cfg["cov_acc"], cfg["cov_bias_gyr"], cfg["cov_bias_acc"]
        v[12] = cfg["mean_acc_norm"]
        v[13:22] = np.asarray(cfg["lid_R"]).reshape(9)
        v[22:25] = cfg["lid_T"]
        self.L.orc_imu_create.restype = C.c_void_p
        self.L.orc_imu_create.argtypes = [C.c_void_p]
        self.L.orc_imu_destroy.argtypes = [C.c_void_p]
        self.L.orc_imu_reset.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_void_p]
        self.L.orc_imu_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int]
        self.h = C.c_void_p(self.L.orc_imu_create(_p(v)))

    def __del__(self):
        try:
            self.L.orc_imu_destroy(self.h)
        except Exception:
            pass

    def reset(self, last_imu7, last_lidar_end_time, last_update_time=0.0, acc_s_last=None, angvel_last=None):
        a = np.ascontiguousarray(last_imu7, dtype=np.float64)
        f = lambda x: None if x is None else _p(np.ascontiguousarray(x, dtype=np.float64))  # noqa: E731
        self.L.orc_imu_reset(self.h, _p(a), last_lidar_end_time, last_update_time, f(acc_s_last), f(angvel_last))

    def undistort(self, state348, imu, pts_xyzt, lidar_beg_time):
        """Returns (state348 after, sorted + compensated cloud, IMUpose[m,22])."""
        st = np.ascontiguousarray(state348, dtype=np.float64).copy()
        im = np.ascontiguousarray(imu, dtype=np.float64).reshape(-1, 7)
        p = np.ascontiguousarray(pts_xyzt, dtype=np.float32).reshape(-1, 4).copy()
        poses = np.zeros((im.shape[0] + 2, 22))
        m = self.L.orc_imu_undistort(self.h, _p(st), _p(im), im.shape[0], _p(p), p.shape[0], lidar_beg_time, _p(poses), poses.shape[0])
        return st, p, poses[:m].copy()


def voxel_grid(pts, leaf):
    """pcl::VoxelGrid restatement: returns (out float32[m,3], leaf_too_small, (min_b, div_b))."""
    L = lib()
    a = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
    out = np.zeros((max(a.shape[0], 1), 3), dtype=np.float32)
    grid = np.zeros(6, dtype=np.int32)
    L.orc_voxel_grid.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int, C.c_void_p]
    m = L.orc_voxel_grid(_p(a), a.shape[0], C.c_float(leaf), _p(out), out.shape[0], _p(grid))
    small = m < 0
    if small:
        m = -m - 1
    return out[:m].copy(), small, (grid[:3].copy(), grid[3:].copy())


def delaunay2d_int(pts):
    L = lib()
    a = np.ascontiguousarray(pts, dtype=np.int64)
    out = np.zeros((4 * a.shape[0] + 8, 3), dtype=np.int32)
    n = L.orc_delaunay2d_int(_p(a), C.c_int(a.shape[0]), _p(out), C.c_int(out.shape[0]))
    return out[:n]


def voxel_triangulate(pts, voxel_res=0.4):
    L = lib()
    a = np.ascontiguousarray(pts, dtype=np.float32)
    out = np.zeros((4 * a.shape[0] + 8, 3), dtype=np.int32)
    sa = np.zeros(3)
    n = L.orc_voxel_triangulate(_p(a), a.shape[0], voxel_res, _p(out), out.shape[0], _p(sa))
    return out[:n], sa


def kitti_calib(pts):
    """KITTI laser calibration (voxel_mapping.cpp:1844-1859) of a packed float32[n,3] cloud; returns a new array."""
    a = np.ascontiguousarray(pts, dtype=np.float32).copy()
    lib().orc_kitti_calib(_p(a), C.c_int(a.shape[0]))
    return a
