"""ctypes binding of include/immesh_b200.h (test / bench harness; no compute happens in Python)."""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libimmesh_b200.so")
_lib_cache: dict[str, C.CDLL] = {}

STATE_DOUBLES = 348
PLANE_MARKER_COLS = 16  # IMMESH_PLANE_MARKER_COLS
SCAN_PUB_COLS = 4       # IMMESH_SCAN_PUB_COLS: x y z intensity


class _LioCfg(C.Structure):
    _fields_ = [
        ("voxel_size", C.c_double), ("max_layer", C.c_int), ("layer_init_size", C.c_int * 5), ("max_points_size", C.c_int),
        ("min_eigen_value", C.c_double), ("dept_err", C.c_double), ("beam_err", C.c_double),
        ("ext_R", C.c_double * 9), ("ext_T", C.c_double * 3), ("max_iteration", C.c_int), ("calib_laser", C.c_int),
        ("hash_capacity_log2", C.c_int), ("max_nodes", C.c_int), ("max_chunks", C.c_int), ("max_scan_points", C.c_int),
    ]


class _MeshCfg(C.Structure):
    _fields_ = [
        ("points_minimum_scale", C.c_double), ("voxel_resolution", C.c_double), ("number_of_pts_append_to_map", C.c_int),
        ("max_vertices", C.c_int), ("max_triangles", C.c_int), ("max_voxels", C.c_int), ("max_frame_points", C.c_int),
    ]


class _EvalCfg(C.Structure):
    _fields_ = [("sample_spacing", C.c_double), ("gt_leaf", C.c_double), ("threshold", C.c_double), ("max_dist", C.c_double),
                ("incorrect_ratio", C.c_double), ("positions", C.c_int), ("pad", C.c_int), ("max_batch_bytes", C.c_int64)]


EVAL_COUNT_KEYS = ("live_triangles", "degenerate", "samples", "gt_points", "samples_within", "gt_within", "samples_far", "gt_far",
                   "incorrect_facets", "sum_q_samples", "sum_q_gt", "max_subdivisions")
EVAL_METRIC_KEYS = ("maxmin_deg", "c2se", "accuracy", "completeness", "precision", "recall", "fscore")


class _TexCamera(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("cam_R", C.c_double * 9), ("cam_t", C.c_double * 3)]


class _TexCfg(C.Structure):
    _fields_ = [("z_near", C.c_double), ("z_far", C.c_double), ("min_cos", C.c_double), ("min_visible_permille", C.c_int), ("two_sided", C.c_int),
                ("positions", C.c_int), ("pad", C.c_int)]


TEXTURE_COUNT_KEYS = ("textured", "untextured", "cameras_used", "pixels")


class _TexImage(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("pitch", C.c_int64)]


class _AtlasCfg(C.Structure):
    _fields_ = [("page_size", C.c_int), ("max_cell", C.c_int), ("max_image_bytes", C.c_int64)]


BAKE_COUNT_KEYS = ("textured", "untextured", "cells", "texels")


class _TexViewCfg(C.Structure):
    _fields_ = [("z_near", C.c_double), ("z_far", C.c_double), ("positions", C.c_int), ("untextured", C.c_uint8 * 3), ("background", C.c_uint8 * 3),
                ("max_image_bytes", C.c_int64)]


# Mesh.render_textured's counts: pixels won by a textured / an untextured row, pixels without a sample, cameras sampled; with a truth
# image the sums over the textured pixels of the squared difference per channel and of the absolute difference over all channels
TEXTURE_VIEW_COUNT_KEYS = ("textured", "untextured", "empty", "cameras_sampled", "sse_0", "sse_1", "sse_2", "sad")


class _TexGainsCfg(C.Structure):
    _fields_ = [("sel", _TexCfg), ("sigma_n", C.c_double), ("sigma_g", C.c_double), ("max_pairs", C.c_int64), ("max_image_bytes", C.c_int64)]


# Mesh.texture_gains' counts: pairs (k, c), sample pairs used, sample pairs clipped (a channel at 0 or 255), observer cameras rasterised,
# cameras left at gain 1 (in no pair), CG iterations (the most over the channels), pixels rasterised, spare
TEXTURE_GAINS_COUNT_KEYS = ("pairs", "samples", "clipped", "observers", "unpaired", "cg_iterations", "pixels", "spare")


def texture_images(images):
    """(ctypes array of immesh_texture_image, on_device, keep-alive list) from HxWx3 uint8 numpy arrays or CUDA torch tensors (all one
    kind; None for a camera no facet uses).  Rows may be padded; pixels must be 3 contiguous bytes."""
    images = list(images)
    arr = (_TexImage * max(len(images), 1))()
    kinds = {type(im).__module__.split(".")[0] for im in images if im is not None}
    if len(kinds) > 1:
        raise ValueError("texture images: all numpy arrays or all CUDA torch tensors")
    on_device = kinds == {"torch"}
    keep = []
    for i, im in enumerate(images):
        if im is None:
            continue
        if on_device:
            if not im.is_cuda or im.dtype.itemsize != 1 or im.dim() != 3 or im.shape[2] != 3 or im.stride(2) != 1 or im.stride(1) != 3:
                raise ValueError(f"texture image {i}: a CUDA uint8 tensor [H, W, 3] with contiguous pixels")
            arr[i] = _TexImage(im.data_ptr(), int(im.shape[1]), int(im.shape[0]), int(im.stride(0)))
        else:
            a = np.asarray(im)
            if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.strides[2] != 1 or a.strides[1] != 3:
                a = np.ascontiguousarray(a, dtype=np.uint8)
                if a.ndim != 3 or a.shape[2] != 3:
                    raise ValueError(f"texture image {i}: uint8 [H, W, 3]")
            keep.append(a)
            arr[i] = _TexImage(a.ctypes.data, int(a.shape[1]), int(a.shape[0]), int(a.strides[0]))
        keep.append(im)
    return arr, int(on_device), keep


def texture_cameras(cameras):
    """ctypes array of immesh_texture_camera from (width, height, (fx, fy, cx, cy), cam_R [3, 3], cam_t [3]) tuples: OpenCV axes
    (x right, y down, z forward), camera to world"""
    cameras = list(cameras)
    arr = (_TexCamera * max(len(cameras), 1))()
    for i, (w, h, K, R, t) in enumerate(cameras):
        fx, fy, cx, cy = (float(k) for k in K)
        arr[i] = _TexCamera(int(w), int(h), fx, fy, cx, cy, (C.c_double * 9)(*np.asarray(R, np.float64).reshape(9)), (C.c_double * 3)(*np.asarray(t, np.float64).reshape(3)))
    return arr, len(cameras)


class _ViewStyle(C.Structure):
    _fields_ = [("positions", C.c_int), ("color_by_height", C.c_int), ("z_range", C.c_double * 2)]


def _view_style(positions, color_by_height, z_range):
    lo, hi = (float("nan"), float("nan")) if z_range is None else (float(z_range[0]), float(z_range[1]))
    return _ViewStyle(int(positions), 1 if color_by_height else 0, (C.c_double * 2)(lo, hi))


class _ViewOverlay(C.Structure):
    _fields_ = [("wireframe", C.c_int), ("scan_point_size", C.c_int), ("reinforced_point_size", C.c_int), ("axis_and_grid", C.c_int),
                ("camera_size", C.c_double), ("path_width", C.c_int), ("path_capacity", C.c_int)]


class _FeedCfg(C.Structure):
    _fields_ = [("max_scans", C.c_int64), ("max_rows", C.c_int64), ("effect", C.c_int), ("registered", C.c_int), ("point_skip", C.c_int), ("pad", C.c_int)]


FEED_HDR = 12   # IMMESH_LIO_FEED_HDR: the header columns of a recorded scan, in this order
FEED_HDR_KEYS = ("scan", "kind", "branch", "iters", "matches", "converged", "err", "row_begin", "row_effect_end", "row_end", "source", "rows_lost")
FEED_KINDS = ("step", "step_dev", "step_async", "step_async_dev_n", "raw", "raw_i", "imu", "imu_i", "depth", "depth_imu")   # IMMESH_FEED_KIND_*
FEED_BRANCH_DROPPED = 4   # IMMESH_FEED_BRANCH_DROPPED: a step_async_depth_imu frame that sync_packages dropped


MARKER_HDR = 10   # IMMESH_LIO_FEED_MARKER_HDR: the header columns of a scan's plane-marker record, in this order
MARKER_HDR_KEYS = ("scan", "row_begin", "row_end", "rows_needed", "lost", "roots_walked", "plane", "sub_plane", "sub_sub_plane", "update")


class _MeshFeedCfg(C.Structure):
    _fields_ = [("max_frames", C.c_int64), ("max_rows", C.c_int64), ("max_images", C.c_int64), ("depth", C.c_int), ("pad", C.c_int)]


MESH_FEED_HDR = 22    # IMMESH_MESH_FEED_HDR: the header columns of a recorded mesh frame, in this order
MESH_FEED_HDR_KEYS = ("frame", "kind", "n_points", "step", "n_vertices", "n_triangles", "new_vertices", "voxels_meshed", "n_add", "n_remove", "n_voxels",
                      "n_activated", "err", "has_rotation", "t_begin_ns", "t_end_ns", "row_begin", "row_end", "rows_lost", "rf", "img_begin", "img_end")
MESH_FEED_POSE = 36   # IMMESH_MESH_FEED_POSE: frame pose, reinforcement camera, view camera; each a row-major R then t
MESH_FEED_KINDS = ("push", "push_dev", "from_lio", "from_lio_async", "reconstruct", "batched", "reconstruct_batched", "depth",
                   "from_lio_async_dev_n")   # IMMESH_MFEED_KIND_*


class _DepthFrame(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("pitch_bytes", C.c_int64), ("format", C.c_int), ("kind", C.c_int), ("depth_scale", C.c_double),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double), ("z_min", C.c_double), ("z_max", C.c_double),
                ("stride", C.c_int), ("pad", C.c_int), ("cam_R", C.c_double * 9), ("cam_t", C.c_double * 3)]


def _sampled(f: "_DepthFrame") -> int:
    """the sampled pixels of a depth frame: ceil(width / stride) * ceil(height / stride)"""
    s = max(f.stride, 1)   # (stride < 1 is refused by the call)
    return -(-f.width // s) * -(-f.height // s)


DEPTH_FORMATS = {"f32": 0, "u16": 1}        # IMMESH_DEPTH_F32, IMMESH_DEPTH_U16
DEPTH_KINDS = {"planar": 0, "range": 1}     # IMMESH_DEPTH_PLANAR, IMMESH_DEPTH_RANGE


@dataclasses.dataclass
class DepthCamera:
    """The pinhole camera of a depth stream (immesh_depth_frame): intrinsics in pixels, the depth kind ("planar": z along the optical
    axis, AirSim DepthPlanar; "range": distance along the ray, AirSim DepthPerspective), the valid z range in metres, the pixel stride
    and the metres per count of a uint16 image.  Poses are camera to world with OpenCV axes (x right, y down, z forward)."""
    fx: float
    fy: float
    cx: float
    cy: float
    kind: str = "planar"
    z_min: float = 0.1
    z_max: float = 100.0
    stride: int = 1
    depth_scale: float = 0.001


class FeedLost(RuntimeError):
    """immesh_lio_feed returned IMMESH_E_RANGE: scans of the range left the rings.  Read on from newest_finished."""

    def __init__(self, msg, newest_finished):
        super().__init__(msg)
        self.newest_finished = newest_finished


class _ImuCfg(C.Structure):
    _fields_ = [("cov_gyr", C.c_double * 3), ("cov_acc", C.c_double * 3), ("cov_bias_gyr", C.c_double * 3), ("cov_bias_acc", C.c_double * 3),
                ("mean_acc_norm", C.c_double), ("lid_R", C.c_double * 9), ("lid_T", C.c_double * 3), ("max_points", C.c_int), ("max_imu", C.c_int)]


@dataclasses.dataclass
class LioConfig:
    """Hot-path parameters of Voxel_mapping (config/*.yaml of the reference)."""
    voxel_size: float = 0.5
    max_layer: int = 2
    layer_init_size: tuple = (5, 5, 5, 5, 5)
    max_points_size: int = 100
    min_eigen_value: float = 0.01
    dept_err: float = 0.02
    beam_err: float = 0.05
    ext_R: tuple = (1, 0, 0, 0, 1, 0, 0, 0, 1)
    ext_T: tuple = (0.04165, 0.02326, -0.0284)
    max_iteration: int = 4
    calib_laser: int = 0
    filter_size_surf: float = 0.4   # leaf of the down-sampling step before the path
    hash_capacity_log2: int = 0
    max_nodes: int = 0
    max_chunks: int = 0
    max_scan_points: int = 0


@dataclasses.dataclass
class MeshConfig:
    points_minimum_scale: float = 0.1
    voxel_resolution: float = 0.4
    number_of_pts_append_to_map: int = 10000
    max_vertices: int = 0
    max_triangles: int = 0
    max_voxels: int = 0
    max_frame_points: int = 0


AVIA = LioConfig()  # config/avia.yaml
VELODYNE = LioConfig(voxel_size=3.0, max_layer=4, max_points_size=1000, dept_err=0.04, beam_err=0.1, ext_T=(0, 0, 0),
                     max_iteration=3, calib_laser=0, filter_size_surf=0.5)  # config/velodyne.yaml (calib_laser applied upstream)


def load_library(path: Optional[str] = None) -> C.CDLL:
    """Load the C-ABI shared library.  There is no fallback: a missing CUDA build is an error."""
    path = path or _LIB_PATH
    if path in _lib_cache:
        return _lib_cache[path]
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()')")
    lib = C.CDLL(path)
    vp, ip, dp, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_float)
    lib.immesh_lio_create.argtypes = [C.POINTER(_LioCfg), C.POINTER(vp)]
    lib.immesh_lio_destroy.argtypes = [vp]
    lib.immesh_lio_set_state.argtypes = [vp, dp]
    lib.immesh_lio_get_state.argtypes = [vp, dp]
    lib.immesh_lio_predict.argtypes = [vp, C.c_double, C.c_double, C.c_double]
    lib.immesh_voxelmap_build.argtypes = [vp, fp, C.c_int]
    lib.immesh_lio_estimate.argtypes = [vp, fp, C.c_int, ip]
    lib.immesh_voxelmap_update.argtypes = [vp]
    lib.immesh_lio_iter_stats.argtypes = [vp, C.c_int, dp]
    lib.immesh_lio_matches.argtypes = [vp, ip, C.c_int]
    lib.immesh_voxelmap_dump.argtypes = [vp, dp, C.c_int64]
    lib.immesh_voxelmap_dump.restype = C.c_int64
    lib.immesh_voxelmap_counts.argtypes = [vp, C.POINTER(C.c_int64)]
    for name, args in (
        ("immesh_lio_step", [vp, fp, C.c_int, C.c_double, C.c_double, C.c_double, dp, ip]),
        ("immesh_lio_step_dev", [vp, vp, C.c_int, C.c_double, C.c_double, C.c_double, dp, ip]),
        ("immesh_residual_build", [vp, fp, C.c_int, ip, dp, C.c_int, ip]),
        ("immesh_mesh_push_frame_dev", [vp, vp, C.c_int, dp, C.c_int]),
        ("immesh_mesh_push_frame_from_lio", [vp, vp, vp, C.c_int, C.c_int]),
        ("immesh_lio_match_nodes", [vp, ip, C.c_int]),
        ("immesh_voxelmap_plane_markers", [vp, dp, C.c_int, ip, C.POINTER(C.c_int64)]),
        ("immesh_lio_effect_cloud", [vp, fp, ip, C.c_int, ip]),
        ("immesh_lio_registered_cloud", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, fp, C.c_int, ip]),
        ("immesh_voxelmap_build_pv", [vp, dp, dp, C.c_int]),
        ("immesh_voxelmap_update_pv", [vp, dp, dp, C.c_int]),
        ("immesh_residual_build_pv", [vp, dp, dp, dp, C.c_int, ip, dp, C.c_int, ip]),
        ("immesh_comm_unique_id", [C.c_char_p]),
        ("immesh_lio_shard", [vp, C.c_int, C.c_int, C.c_char_p]),
        ("immesh_mesh_shard", [vp, C.c_int, C.c_int, C.c_char_p]),
        ("immesh_lio_shard_transport", [vp]),
        ("immesh_mesh_shard_transport", [vp]),
        ("immesh_lio_step_async", [vp, vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double]),
        ("immesh_lio_wait", [vp, dp, ip]),
        ("immesh_lio_enqueue_memset", [vp, vp, C.c_size_t]),
        ("immesh_mesh_push_frame_from_lio_async", [vp, vp, vp, C.c_int, C.c_int]),
        ("immesh_mesh_wait", [vp]),
        ("immesh_mesh_push_depth", [vp, C.POINTER(_DepthFrame), vp, C.c_int]),
        ("immesh_mesh_push_depth_async", [vp, C.POINTER(_DepthFrame), vp, C.c_int]),
        ("immesh_mesh_depth_points", [vp, fp, C.c_int, ip]),
        ("immesh_mesh_push_frame_from_lio_async_dev_n", [vp, vp, vp, C.c_int, vp]),
        ("immesh_pipeline_mark_begin", [vp]),
        ("immesh_pipeline_mark_end", [vp, vp, dp]),
        ("immesh_mesh_work_stats", [vp, C.POINTER(C.c_int64)]),
        ("immesh_host_wait_ms", [vp, vp, dp]),
        ("immesh_lio_work_stats", [vp, C.POINTER(C.c_int64)]),
        ("immesh_profile_enable", [C.c_int]),
        ("immesh_profile_reset", []),
        ("immesh_profile_report", [C.c_char_p, C.c_int]),
        ("immesh_profile_timeline", [C.c_char_p, C.c_int]),
        ("immesh_launch_count", []),
        ("immesh_graph_stats", [vp, vp, C.POINTER(C.c_int64)]),
        ("immesh_graph_pdl_edges", [vp, vp, C.POINTER(C.c_int64)]),
        ("immesh_lio_last_timing", [vp, dp]),
        ("immesh_lio_capacity", [vp, C.POINTER(C.c_int64)]),
        ("immesh_lio_reserve", [vp, C.c_int64, C.c_int64, C.c_int64]),
        ("immesh_lio_set_growth", [vp, C.c_int64]),
        ("immesh_lio_local_map", [vp, C.c_double, C.c_float, C.c_float]),
        ("immesh_voxelmap_evict_boxes", [vp, fp, C.c_int]),
        ("immesh_lio_local_map_state", [vp, fp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_capacity", [vp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_reserve", [vp, C.c_int64, C.c_int64, C.c_int64]),
        ("immesh_mesh_set_growth", [vp, C.c_int64]),
        ("immesh_mesh_create", [C.POINTER(_MeshCfg), C.POINTER(vp)]),
        ("immesh_mesh_destroy", [vp]),
        ("immesh_mesh_push_frame", [vp, fp, C.c_int, dp, C.c_int]),
        ("immesh_mesh_counts", [vp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_snapshot", [vp, fp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
        ("immesh_knn", [vp, fp, C.c_int, C.c_int, C.c_double, C.POINTER(C.c_int32), fp]),
        ("immesh_mesh_last_timing", [vp, dp]),
        ("immesh_write_ply", [C.c_char_p, fp, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int]),
        ("immesh_write_pcd", [C.c_char_p, fp, C.c_int]),
        ("immesh_mesh_render_depth", [vp, dp, C.c_int, C.c_int, C.c_double, C.c_double, dp, dp, fp, fp, C.POINTER(C.c_int32), ip]),
        ("immesh_mesh_reinforce_enable", [vp, dp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int]),
        ("immesh_mesh_reinforce_pose", [vp, dp, dp]),
        ("immesh_mesh_reinforced_cloud", [vp, fp, fp, C.POINTER(C.c_int32), C.c_int, ip, dp]),
        ("immesh_mesh_render_view", [vp, dp, C.c_int, C.c_int, C.c_double, C.c_double, dp, dp, C.POINTER(_ViewStyle), C.POINTER(C.c_uint8), fp]),
        ("immesh_mesh_view_enable", [vp, dp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.POINTER(_ViewStyle)]),
        ("immesh_mesh_view_pose", [vp, dp, dp, C.c_int]),
        ("immesh_mesh_view_image", [vp, C.POINTER(C.c_uint8), fp, dp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_view_overlay", [vp, C.POINTER(_ViewOverlay)]),
        ("immesh_mesh_changes_enable", [vp, C.c_int64, C.c_int]),
        ("immesh_mesh_changes", [vp, C.c_int64, C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_int32), C.c_int64, fp, C.c_int64, C.POINTER(C.c_int64)]),
        ("immesh_mesh_reconstruct_from_pointcloud", [vp, vp, vp, C.c_int, C.c_int, C.c_double, ip]),
        ("immesh_mesh_feed_enable", [vp, C.POINTER(_MeshFeedCfg)]),
        ("immesh_mesh_feed", [vp, C.c_int64, C.c_int, C.POINTER(C.c_int64), dp, C.c_int, fp, C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64)]),
        ("immesh_mesh_feed_images", [vp, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_uint8), fp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_push_frame_batched", [vp, vp, C.c_int64, C.c_int, dp, C.c_int, C.c_int, C.POINTER(C.c_int64)]),
        ("immesh_mesh_reconstruct_from_pointcloud_batched", [vp, vp, vp, C.c_int64, C.c_int, C.c_double, C.c_int, C.c_int, C.POINTER(C.c_int64)]),
        ("immesh_mesh_smooth_all", [vp, C.c_double, C.c_int, dp]),
        ("immesh_mesh_evaluate", [vp, vp, C.c_int64, C.c_int, C.POINTER(_EvalCfg), C.POINTER(C.c_int64), dp, C.POINTER(C.c_int32), C.c_int64,
                                  C.POINTER(C.c_int64)]),
        ("immesh_mesh_evaluate_stats", [C.POINTER(C.c_int64)]),
        ("immesh_mesh_texture_select", [vp, C.POINTER(_TexCamera), C.c_int, C.POINTER(_TexCfg), C.POINTER(C.c_int32), fp, C.POINTER(C.c_int32), fp, C.c_int64,
                                        C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
        ("immesh_mesh_texture_enable", [vp, C.POINTER(_TexCamera), C.POINTER(_TexCfg)]),
        ("immesh_mesh_texture_pose", [vp, dp, dp]),
        ("immesh_mesh_texture_rows", [vp, C.POINTER(C.c_int32), fp, C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                      C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64)]),
        ("immesh_mesh_texture_bake", [vp, C.POINTER(_TexCamera), C.c_int, C.POINTER(_TexImage), C.c_int, C.POINTER(C.c_int32), fp, C.c_int64,
                                      C.POINTER(_AtlasCfg), vp, C.c_int, C.POINTER(C.c_int32), fp, ip, C.POINTER(C.c_int64)]),
        ("immesh_mesh_render_textured", [vp, C.POINTER(_TexCamera), C.POINTER(_TexViewCfg), C.POINTER(_TexCamera), C.c_int, C.POINTER(_TexImage), C.c_int,
                                         C.POINTER(C.c_int32), fp, C.c_int64, C.POINTER(_TexImage), vp, fp, C.POINTER(C.c_int32), vp, C.POINTER(C.c_int64)]),
        ("immesh_mesh_render_textured_stats", [dp]),
        ("immesh_mesh_texture_gains", [vp, C.POINTER(_TexCamera), C.c_int, C.POINTER(_TexImage), C.c_int, C.POINTER(C.c_int32), fp, C.c_int64,
                                       C.POINTER(_TexGainsCfg), dp, C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
        ("immesh_mesh_texture_gains_stats", [dp]),
        ("immesh_texture_apply_gains", [vp, C.POINTER(_TexImage), C.POINTER(_TexImage), C.c_int, C.c_int, dp]),
        ("immesh_write_png", [C.c_char_p, vp, C.c_int, C.c_int]),
        ("immesh_write_obj_textured", [C.c_char_p, C.c_char_p, fp, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32), fp, C.c_int,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_char_p), C.c_int]),
        ("immesh_mesh_region_stream", [vp, C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_int32), ip]),
        ("immesh_mesh_region_buffers", [vp, C.c_double, C.POINTER(C.c_int32), C.c_int, C.c_double, C.c_int, fp, C.POINTER(C.c_int32), C.c_int,
                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int, fp, ip, ip, ip]),
        ("immesh_kitti_pose_line", [dp, C.c_double, C.c_char_p, C.c_int]),
        ("immesh_voxelgrid_create", [C.c_int, C.POINTER(vp)]),
        ("immesh_voxelgrid_destroy", [vp]),
        ("immesh_voxelgrid_filter", [vp, vp, C.c_int, C.c_int, C.c_float, vp, ip, ip]),
        ("immesh_voxelgrid_device_points", [vp]),
        ("immesh_frontend_prepare", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
        ("immesh_voxelgrid_input_points", [vp]),
        ("immesh_lio_step_async_raw", [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double, C.c_double]),
        ("immesh_lio_step_async_dev_n", [vp, vp, C.c_int, vp, C.c_double, C.c_double, C.c_double]),
        ("immesh_frontend_prepare_depth", [vp, C.POINTER(_DepthFrame), vp, C.c_int, C.c_int, C.c_double, fp, C.c_int, ip]),
        ("immesh_lio_step_async_depth", [vp, vp, C.POINTER(_DepthFrame), vp, C.c_int, C.c_int, C.c_double, C.c_float, C.c_double, C.c_double, C.c_double]),
        ("immesh_voxelgrid_input_count", [vp]),
        ("immesh_imu_create", [C.POINTER(_ImuCfg), C.POINTER(vp)]),
        ("immesh_imu_destroy", [vp]),
        ("immesh_imu_reset", [vp, dp, C.c_double, C.c_double, dp, dp]),
        ("immesh_imu_undistort", [vp, vp, dp, C.c_int, vp, C.c_int, C.c_int, C.c_double, vp]),
        ("immesh_imu_device_points", [vp]),
        ("immesh_imu_get_poses", [vp, dp, C.c_int]),
        ("immesh_imu_init_begin", [vp, C.c_int]),
        ("immesh_lio_step_async_depth_imu", [vp, vp, vp, dp, C.c_int, C.POINTER(_DepthFrame), vp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_float]),
        ("immesh_imu_depth_chain_state", [vp, C.POINTER(C.c_int64)]),
        ("immesh_lio_step_async_imu", [vp, vp, vp, dp, C.c_int, vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_float, ip]),
        ("immesh_voxelgrid_filter_i", [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, vp, ip, ip]),
        ("immesh_lio_step_async_raw_i", [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double, C.c_double]),
        ("immesh_lio_step_async_imu_i", [vp, vp, vp, dp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_float, ip]),
        ("immesh_lio_frontend_cloud", [vp, vp, C.c_int, C.c_int, fp, C.c_int, ip]),
        ("immesh_lio_feed_enable", [vp, C.POINTER(_FeedCfg)]),
        ("immesh_lio_feed", [vp, C.c_int64, C.c_int, C.POINTER(C.c_int64), dp, C.c_int, fp, C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_int64)]),
        ("immesh_lio_feed_markers_enable", [vp, C.c_int64]),
        ("immesh_lio_feed_markers", [vp, C.c_int64, C.c_int, C.POINTER(C.c_int64), C.c_int, dp, C.c_int64, C.POINTER(C.c_int64)]),
        ("immesh_odometry_pose", [dp, dp]),
        ("immesh_lio_state_line", [dp, C.c_double, C.c_char_p, C.c_int]),
    ):
        if hasattr(lib, name):
            getattr(lib, name).argtypes = args
    if hasattr(lib, "immesh_imu_device_points"):
        lib.immesh_imu_device_points.restype = C.c_void_p
    if hasattr(lib, "immesh_voxelgrid_device_points"):
        lib.immesh_voxelgrid_device_points.restype = C.c_void_p
    if hasattr(lib, "immesh_voxelgrid_input_points"):
        lib.immesh_voxelgrid_input_points.restype = C.c_void_p
    if hasattr(lib, "immesh_voxelgrid_input_count"):
        lib.immesh_voxelgrid_input_count.restype = C.c_void_p
    if hasattr(lib, "immesh_launch_count"):
        lib.immesh_launch_count.restype = C.c_longlong
    if hasattr(lib, "immesh_last_error"):
        lib.immesh_last_error.restype = C.c_char_p
    if hasattr(lib, "immesh_version"):
        lib.immesh_version.restype = C.c_char_p
    _lib_cache[path] = lib
    return lib


def reinforce_intrinsics(width=640, height=480, focus=400.0):
    """Cam_view::set_gl_projection (openGL_camera_view.cpp:83-101): the width rounded up to a multiple of 4, then
    m_camera_intrinsic = [focus 0 w/2; 0 focus h/2] with integer halves; focus 400 for the reinforcement camera (ImMesh_node.cpp:291)."""
    w = width + (4 - width % 4) % 4
    return (float(focus), float(focus), float(w // 2), float(height // 2))


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(C.POINTER(C.c_float))


def _check(lib, rc, what):
    if rc != 0:
        msg = lib.immesh_last_error().decode() if hasattr(lib, "immesh_last_error") else ""
        raise RuntimeError(f"{what} failed with code {rc}: {msg}")


class Lio:
    """Mirror of the reference's Voxel_mapping hot-path methods (voxel_map_init / lio_state_estimation /
    map_incremental_grow) on the device-resident VoxelMap."""

    def __init__(self, cfg: LioConfig = AVIA, lib: Optional[C.CDLL] = None):
        self.lib = lib or load_library()
        self.cfg = cfg
        c = _LioCfg()
        c.voxel_size = cfg.voxel_size
        c.max_layer = cfg.max_layer
        for i in range(5):
            c.layer_init_size[i] = cfg.layer_init_size[i]
        c.max_points_size = cfg.max_points_size
        c.min_eigen_value = cfg.min_eigen_value
        c.dept_err, c.beam_err = cfg.dept_err, cfg.beam_err
        for i in range(9):
            c.ext_R[i] = cfg.ext_R[i]
        for i in range(3):
            c.ext_T[i] = cfg.ext_T[i]
        c.max_iteration, c.calib_laser = cfg.max_iteration, cfg.calib_laser
        c.hash_capacity_log2, c.max_nodes, c.max_chunks, c.max_scan_points = cfg.hash_capacity_log2, cfg.max_nodes, cfg.max_chunks, cfg.max_scan_points
        self._h = C.c_void_p()
        _check(self.lib, self.lib.immesh_lio_create(C.byref(c), C.byref(self._h)), "immesh_lio_create")

    def close(self):
        if self._h:
            self.lib.immesh_lio_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- state
    def get_state(self) -> np.ndarray:
        s = np.zeros(STATE_DOUBLES)
        _check(self.lib, self.lib.immesh_lio_get_state(self._h, s.ctypes.data_as(C.POINTER(C.c_double))), "get_state")
        return s

    def set_state(self, s):
        s = np.ascontiguousarray(s, dtype=np.float64)
        assert s.size == STATE_DOUBLES
        _check(self.lib, self.lib.immesh_lio_set_state(self._h, s.ctypes.data_as(C.POINTER(C.c_double))), "set_state")

    def set_pose(self, R, t):
        s = self.get_state()
        s[0:9] = np.asarray(R, dtype=np.float64).reshape(9)
        s[9:12] = t
        self.set_state(s)

    # --- reference-named operations
    def predict(self, dt, cov_gyr=0.1, cov_acc=0.1):
        _check(self.lib, self.lib.immesh_lio_predict(self._h, dt, cov_gyr, cov_acc), "predict")

    def voxel_map_init(self, body_full):
        a, p = _f32(body_full)
        _check(self.lib, self.lib.immesh_voxelmap_build(self._h, p, a.shape[0]), "voxelmap_build")

    def lio_state_estimation(self, body_ds) -> int:
        a, p = _f32(body_ds)
        it = C.c_int(0)
        _check(self.lib, self.lib.immesh_lio_estimate(self._h, p, a.shape[0], C.byref(it)), "lio_estimate")
        self._last_n = a.shape[0]
        return it.value

    def map_incremental_grow(self):
        _check(self.lib, self.lib.immesh_voxelmap_update(self._h), "voxelmap_update")

    def step(self, body_ds, dt=0.0, cov_gyr=0.1, cov_acc=0.1):
        a, p = _f32(body_ds)
        it = C.c_int(0)
        s = np.zeros(STATE_DOUBLES)
        _check(self.lib, self.lib.immesh_lio_step(self._h, p, a.shape[0], dt, cov_gyr, cov_acc, s.ctypes.data_as(C.POINTER(C.c_double)), C.byref(it)), "lio_step")
        self._last_n = a.shape[0]
        return s, it.value

    def step_dev(self, dev_ptr, n, dt=0.0, cov_gyr=0.1, cov_acc=0.1):
        """Same as step() with the scan already in device memory (dev_ptr: integer CUDA address of float32[n][3])."""
        it = C.c_int(0)
        s = np.zeros(STATE_DOUBLES)
        _check(self.lib, self.lib.immesh_lio_step_dev(self._h, C.c_void_p(dev_ptr), n, dt, cov_gyr, cov_acc, s.ctypes.data_as(C.POINTER(C.c_double)), C.byref(it)), "lio_step_dev")
        self._last_n = n
        return s, it.value

    def step_async(self, body, n=None, dt=0.0, cov_gyr=0.1, cov_acc=0.1, on_device=False):
        """Queue one scan (predict + estimate + map update) without waiting; body: float32[n][3] host array or CUDA address."""
        if on_device:
            ptr = C.c_void_p(body)
        else:
            a, p = _f32(body)
            n = a.shape[0]
            ptr = C.cast(p, C.c_void_p)
        _check(self.lib, self.lib.immesh_lio_step_async(self._h, ptr, n, 1 if on_device else 0, dt, cov_gyr, cov_acc), "lio_step_async")
        self._last_n = n

    def wait(self):
        it = C.c_int(0)
        s = np.zeros(STATE_DOUBLES)
        _check(self.lib, self.lib.immesh_lio_wait(self._h, s.ctypes.data_as(C.POINTER(C.c_double)), C.byref(it)), "lio_wait")
        return s, it.value

    def enqueue_memset(self, dev_ptr, nbytes):
        _check(self.lib, self.lib.immesh_lio_enqueue_memset(self._h, C.c_void_p(dev_ptr), nbytes), "enqueue_memset")

    def shard(self, rank: int, nranks: int, unique_id: bytes):
        """Shard the VoxelMap over nranks processes (NCCL); unique_id: 128 bytes from comm_unique_id() of rank 0."""
        _check(self.lib, self.lib.immesh_lio_shard(self._h, rank, nranks, unique_id), "lio_shard")

    def shard_transport(self) -> str:
        return ("none", "nccl", "peer-window")[self.lib.immesh_lio_shard_transport(self._h)]

    def residual_build(self, body_ds):
        a, p = _f32(body_ds)
        n = a.shape[0]
        il = np.zeros((n, 2), dtype=np.int32)
        vals = np.zeros((n, 31))
        m = C.c_int(0)
        _check(self.lib, self.lib.immesh_residual_build(self._h, p, n, il.ctypes.data_as(C.POINTER(C.c_int)), vals.ctypes.data_as(C.POINTER(C.c_double)), n, C.byref(m)), "residual_build")
        return il[: m.value], vals[: m.value]

    # --- the three free functions of src/voxel_mapping.hpp:80-105 on caller-built Point_with_var lists
    @staticmethod
    def _f64(a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        return a, a.ctypes.data_as(C.POINTER(C.c_double))

    def voxelmap_build_pv(self, pts_world, var9):
        (pw, ppw), (v9, pv9) = self._f64(pts_world), self._f64(var9)
        _check(self.lib, self.lib.immesh_voxelmap_build_pv(self._h, ppw, pv9, pw.shape[0]), "voxelmap_build_pv")

    def voxelmap_update_pv(self, pts_world, var9):
        (pw, ppw), (v9, pv9) = self._f64(pts_world), self._f64(var9)
        _check(self.lib, self.lib.immesh_voxelmap_update_pv(self._h, ppw, pv9, pw.shape[0]), "voxelmap_update_pv")

    def residual_build_pv(self, pts_body, pts_world, var9):
        (pb, ppb), (pw, ppw), (v9, pv9) = self._f64(pts_body), self._f64(pts_world), self._f64(var9)
        n = pb.shape[0]
        il = np.zeros((max(n, 1), 2), dtype=np.int32)
        vals = np.zeros((max(n, 1), 31))
        m = C.c_int(0)
        _check(self.lib, self.lib.immesh_residual_build_pv(self._h, ppb, ppw, pv9, n, il.ctypes.data_as(C.POINTER(C.c_int)), vals.ctypes.data_as(C.POINTER(C.c_double)), n, C.byref(m)), "residual_build_pv")
        return il[: m.value], vals[: m.value]

    # --- diagnostics
    def iter_stats(self, it):
        o = np.zeros(63)
        _check(self.lib, self.lib.immesh_lio_iter_stats(self._h, it, o.ctypes.data_as(C.POINTER(C.c_double))), "iter_stats")
        return dict(HTH=o[:36].reshape(6, 6).copy(), HTz=o[36:42].copy(), n_match=int(o[42]), total_residual=o[43], solution=o[44:62].copy(), converged=int(o[62]))

    def matches(self, n=None):
        n = n or self._last_n
        o = np.zeros(n, dtype=np.int32)
        _check(self.lib, self.lib.immesh_lio_matches(self._h, o.ctypes.data_as(C.POINTER(C.c_int)), n), "matches")
        return o

    def match_nodes(self, n=None):
        n = n or self._last_n
        o = np.zeros(n, dtype=np.int32)
        _check(self.lib, self.lib.immesh_lio_match_nodes(self._h, o.ctypes.data_as(C.POINTER(C.c_int)), n), "match_nodes")
        return o

    def dump_map(self) -> np.ndarray:
        rows = self.lib.immesh_voxelmap_dump(self._h, None, 0)
        out = np.zeros((rows, 45))
        r2 = self.lib.immesh_voxelmap_dump(self._h, out.ctypes.data_as(C.POINTER(C.c_double)), rows)
        assert r2 == rows
        return out

    def counts(self):
        o = np.zeros(4, dtype=np.int64)
        self.lib.immesh_voxelmap_counts(self._h, o.ctypes.data_as(C.POINTER(C.c_int64)))
        return dict(roots=int(o[0]), nodes=int(o[1]), chunks=int(o[2]), err=int(o[3]))

    def plane_markers(self, cap=None):
        """pubPlaneMap: the markers of the planes refitted since the last call, float64[m, PLANE_MARKER_COLS] rows
        (kx ky kz path layer id | px py pz nx ny nz | radius min_eig trace alpha), and the counters
        dict(plane, sub_plane, sub_sub_plane, update, roots_walked).  cap=None sizes the buffer with a count query first; with a
        cap that is too small the call raises and nothing is consumed."""
        n = C.c_int(0)
        cnt = np.zeros(5, dtype=np.int64)
        pc = cnt.ctypes.data_as(C.POINTER(C.c_int64))
        if cap is None:
            rc = self.lib.immesh_voxelmap_plane_markers(self._h, None, 0, C.byref(n), pc)
            if rc not in (0, -3):
                _check(self.lib, rc, "voxelmap_plane_markers")
            cap = n.value
        rows = np.zeros((max(cap, 1), PLANE_MARKER_COLS))
        _check(self.lib, self.lib.immesh_voxelmap_plane_markers(self._h, rows.ctypes.data_as(C.POINTER(C.c_double)), cap, C.byref(n), pc),
               "voxelmap_plane_markers")
        keys = ("plane", "sub_plane", "sub_sub_plane", "update", "roots_walked")
        return rows[: n.value], dict(zip(keys, (int(v) for v in cnt)))

    def effect_cloud(self):
        """publish_effect_world: the points matched in the last IESKF iteration as float32[m, SCAN_PUB_COLS] rows x y z intensity
        (world frame, current state; intensity = sqrt(R_inv), the point's IESKF weight) and their scan indices int32[m], ascending."""
        n = C.c_int(0)
        rc = self.lib.immesh_lio_effect_cloud(self._h, None, None, 0, C.byref(n))
        if rc not in (0, -3):
            _check(self.lib, rc, "lio_effect_cloud")
        rows = np.zeros((max(n.value, 1), SCAN_PUB_COLS), dtype=np.float32)
        idx = np.zeros(max(n.value, 1), dtype=np.int32)
        _check(self.lib, self.lib.immesh_lio_effect_cloud(self._h, rows.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int)),
                                                          n.value, C.byref(n)), "lio_effect_cloud")
        return rows[: n.value], idx[: n.value]

    def registered_cloud(self, pts=None, point_skip=1, intensity_col=-1, on_device=False, n=None, stride=3):
        """publish_frame_world: points 0, point_skip, 2 point_skip, ... in the world frame of the current state, float32[m, 4] rows
        x y z intensity (intensity = pts[:, intensity_col], 0 when intensity_col < 0).  pts: float32[n, stride] host array, or with
        on_device a CUDA address of n rows of `stride` floats; None: the down-sampled scan the handle last localised."""
        if pts is None:
            ptr, n, stride, dev = None, 0, 3, 0
        elif on_device:
            ptr, dev = C.c_void_p(pts), 1
        else:
            a = np.ascontiguousarray(pts, dtype=np.float32)
            a = a.reshape(a.shape[0], -1)
            ptr, n, stride, dev = a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1], 0
        n_out = C.c_int(0)

        def call(rows, cap):
            return self.lib.immesh_lio_registered_cloud(self._h, ptr, n, stride, intensity_col, dev, point_skip, rows, cap, C.byref(n_out))
        rc = call(None, 0)
        if rc not in (0, -3):
            _check(self.lib, rc, "lio_registered_cloud")
        rows = np.zeros((max(n_out.value, 1), SCAN_PUB_COLS), dtype=np.float32)
        _check(self.lib, call(rows.ctypes.data_as(C.POINTER(C.c_float)), n_out.value), "lio_registered_cloud")
        return rows[: n_out.value]

    def feed_enable(self, max_scans=1024, max_rows=1 << 22, effect=True, registered=1, point_skip=1):
        """Record every queued scan's header, state and published clouds on the device (immesh_lio_feed_enable).  registered: 0 none,
        1 the down-sampled scan, 2 the full scan where the chain has one."""
        c = _FeedCfg(max_scans, max_rows, 1 if effect else 0, registered, point_skip, 0)
        _check(self.lib, self.lib.immesh_lio_feed_enable(self._h, C.byref(c)), "lio_feed_enable")

    def feed_disable(self):
        _check(self.lib, self.lib.immesh_lio_feed_enable(self._h, None), "lio_feed_enable")

    def feed(self, since: int, wait: bool = False):
        """The scans (since, newest finished] of the scan feed: dict(scans=int64[m, FEED_HDR], states=float64[m, 348],
        rows=float32[r, 4], row_index=int32[r] (-1 on registered rows), newest_finished, newest_queued).  wait=False never blocks on
        unfinished work.  Raises FeedLost when scans of the range left the rings."""
        counts = np.zeros(4, dtype=np.int64)
        cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
        for _ in range(8):   # scans may finish between the count query and the read
            rc = self.lib.immesh_lio_feed(self._h, since, 1 if wait else 0, None, None, 0, None, None, 0, cp)
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, "lio_feed")
            ns, nr = int(counts[0]), int(counts[1])
            scans = np.zeros((max(ns, 1), FEED_HDR), dtype=np.int64)
            states = np.zeros((max(ns, 1), STATE_DOUBLES))
            rows = np.zeros((max(nr, 1), SCAN_PUB_COLS), dtype=np.float32)
            idx = np.zeros(max(nr, 1), dtype=np.int32)
            if ns == 0:
                break
            rc = self.lib.immesh_lio_feed(self._h, since, 0, scans.ctypes.data_as(C.POINTER(C.c_int64)), states.ctypes.data_as(C.POINTER(C.c_double)), ns,
                                          rows.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int32)), nr, cp)
            if rc == -3:
                continue
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, "lio_feed")
            ns, nr = int(counts[0]), int(counts[1])
            break
        else:
            raise RuntimeError("lio_feed: the scans kept finishing faster than they were read")
        return dict(scans=scans[:ns], states=states[:ns], rows=rows[:nr], row_index=idx[:nr], newest_finished=int(counts[2]), newest_queued=int(counts[3]))

    def feed_markers_enable(self, max_rows: int):
        """Record each fed scan's plane-map markers (pubPlaneMap) in a ring of max_rows rows (immesh_lio_feed_markers_enable); 0 turns
        the recording off.  Needs the feed on; feed_enable and feed_disable turn it off."""
        _check(self.lib, self.lib.immesh_lio_feed_markers_enable(self._h, int(max_rows)), "lio_feed_markers_enable")

    def feed_markers(self, since: int, wait: bool = False):
        """The plane-marker records of the scans (since, newest finished]: dict(scans=int64[m, MARKER_HDR] (MARKER_HDR_KEYS),
        rows=float64[r, PLANE_MARKER_COLS] as plane_markers() gives them, newest_finished, newest_queued).  wait=False never blocks on
        unfinished work.  Raises FeedLost when records of the range left the rings."""
        counts = np.zeros(4, dtype=np.int64)
        cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
        for _ in range(8):   # scans may finish between the count query and the read
            rc = self.lib.immesh_lio_feed_markers(self._h, since, 1 if wait else 0, None, 0, None, 0, cp)
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, "lio_feed_markers")
            ns, nr = int(counts[0]), int(counts[1])
            scans = np.zeros((max(ns, 1), MARKER_HDR), dtype=np.int64)
            rows = np.zeros((max(nr, 1), PLANE_MARKER_COLS))
            if ns == 0:
                break
            rc = self.lib.immesh_lio_feed_markers(self._h, since, 0, scans.ctypes.data_as(C.POINTER(C.c_int64)), ns, rows.ctypes.data_as(C.POINTER(C.c_double)),
                                                  nr, cp)
            if rc == -3:
                continue
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, "lio_feed_markers")
            ns, nr = int(counts[0]), int(counts[1])
            break
        else:
            raise RuntimeError("lio_feed_markers: the scans kept finishing faster than they were read")
        return dict(scans=scans[:ns], rows=rows[:nr], newest_finished=int(counts[2]), newest_queued=int(counts[3]))

    def frontend_cloud(self, vg: "VoxelGrid", dense: bool, point_skip=1):
        """publish_frame_world from the front-end clouds of the last _i step through vg (immesh_lio_frontend_cloud): float32[m, 4] rows
        world x y z intensity of the calibrated full scan (dense) or of the down-sampled scan the step localised."""
        n_out = C.c_int(0)

        def call(rows, cap):
            return self.lib.immesh_lio_frontend_cloud(self._h, vg._h, 1 if dense else 0, point_skip, rows, cap, C.byref(n_out))
        rc = call(None, 0)
        if rc not in (0, -3):
            _check(self.lib, rc, "lio_frontend_cloud")
        rows = np.zeros((max(n_out.value, 1), SCAN_PUB_COLS), dtype=np.float32)
        _check(self.lib, call(rows.ctypes.data_as(C.POINTER(C.c_float)), n_out.value), "lio_frontend_cloud")
        return rows[: n_out.value]

    def work_stats(self):
        o = np.zeros(4, dtype=np.int64)
        _check(self.lib, self.lib.immesh_lio_work_stats(self._h, o.ctypes.data_as(C.POINTER(C.c_int64))), "lio_work_stats")
        return dict(n=int(o[0]), roots=int(o[1]), refits=int(o[2]), refit_points=int(o[3]))

    def last_timing(self):
        o = np.zeros(3)
        self.lib.immesh_lio_last_timing(self._h, o.ctypes.data_as(C.POINTER(C.c_double)))
        return o

    # --- long runs: capacities and growth of the map pools
    def capacity(self):
        """dict(root_slots, roots, nodes_cap, nodes, chunks_cap, chunks, device_bytes, growths)"""
        o = np.zeros(8, dtype=np.int64)
        _check(self.lib, self.lib.immesh_lio_capacity(self._h, o.ctypes.data_as(C.POINTER(C.c_int64))), "lio_capacity")
        keys = ("root_slots", "roots", "nodes_cap", "nodes", "chunks_cap", "chunks", "device_bytes", "growths")
        return dict(zip(keys, (int(v) for v in o)))

    def reserve(self, root_slots=0, nodes=0, chunks=0):
        """Grow the pools to at least these capacities (0: keep); never shrinks."""
        _check(self.lib, self.lib.immesh_lio_reserve(self._h, root_slots, nodes, chunks), "lio_reserve")

    def set_growth(self, max_bytes):
        """Automatic growth before every step, up to max_bytes of device memory for the handle (0: off)."""
        _check(self.lib, self.lib.immesh_lio_set_growth(self._h, max_bytes), "lio_set_growth")

    # --- long runs: the local map (a cube that follows the sensor; root voxels it leaves behind are evicted)
    def local_map(self, cube_len, det_range=300.0, mov_threshold=1.5):
        """Turn the automatic local map on (cube_len: the reference's cube_side_length) or off (cube_len = 0).  Drains the handle;
        the box is placed at the next evaluation (once per scan, before its IESKF)."""
        _check(self.lib, self.lib.immesh_lio_local_map(self._h, float(cube_len), float(det_range), float(mov_threshold)), "lio_local_map")

    def evict_boxes(self, boxes):
        """Evict the root voxels whose centre lies in one of the boxes, float32[n, 6] rows min xyz, max xyz (half-open
        min <= c < max); queued behind the steps already queued."""
        a = np.ascontiguousarray(np.asarray(boxes, dtype=np.float32).reshape(-1, 6))
        _check(self.lib, self.lib.immesh_voxelmap_evict_boxes(self._h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0]), "voxelmap_evict_boxes")

    def local_map_state(self):
        """(box float32[6] min xyz, max xyz, dict(placed, moves, roots_evicted, nodes_freed, chunks_freed, tombstones, rebuilds,
        free_nodes)); blocking."""
        box = np.zeros(6, dtype=np.float32)
        o = np.zeros(8, dtype=np.int64)
        _check(self.lib, self.lib.immesh_lio_local_map_state(self._h, box.ctypes.data_as(C.POINTER(C.c_float)), o.ctypes.data_as(C.POINTER(C.c_int64))),
               "lio_local_map_state")
        keys = ("placed", "moves", "roots_evicted", "nodes_freed", "chunks_freed", "tombstones", "rebuilds", "free_nodes")
        return box, dict(zip(keys, (int(v) for v in o)))


class Mesh:
    """Mirror of incremental_mesh_reconstruction + Global_map/Triangle_manager snapshot + KD_TREE::Nearest_Search."""

    def __init__(self, cfg: MeshConfig = MeshConfig(), lib: Optional[C.CDLL] = None):
        self.lib = lib or load_library()
        self.cfg = cfg
        c = _MeshCfg(cfg.points_minimum_scale, cfg.voxel_resolution, cfg.number_of_pts_append_to_map, cfg.max_vertices, cfg.max_triangles,
                     cfg.max_voxels, cfg.max_frame_points)
        self._h = C.c_void_p()
        _check(self.lib, self.lib.immesh_mesh_create(C.byref(c), C.byref(self._h)), "immesh_mesh_create")

    def close(self):
        if self._h:
            self.lib.immesh_mesh_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push_frame(self, world_xyz, pose_t, frame_idx=0):
        a, p = _f32(world_xyz)
        t = np.ascontiguousarray(pose_t, dtype=np.float64)
        _check(self.lib, self.lib.immesh_mesh_push_frame(self._h, p, a.shape[0], t.ctypes.data_as(C.POINTER(C.c_double)), frame_idx), "mesh_push_frame")

    def push_frame_dev(self, dev_ptr, n, pose_t, frame_idx=0):
        t = np.ascontiguousarray(pose_t, dtype=np.float64)
        _check(self.lib, self.lib.immesh_mesh_push_frame_dev(self._h, C.c_void_p(dev_ptr), n, t.ctypes.data_as(C.POINTER(C.c_double)), frame_idx), "mesh_push_frame_dev")

    def push_frame_from_lio(self, lio: "Lio", body_full, n=None, on_device=False):
        """map_incremental_grow's hand-off: transform the full-resolution body scan with lio's converged state on the
        device and mesh it.  body_full: float32[n][3] host array, or an integer CUDA address when on_device."""
        if on_device:
            ptr = C.c_void_p(body_full)
        else:
            a, p = _f32(body_full)
            n = a.shape[0]
            ptr = C.cast(p, C.c_void_p)
        _check(self.lib, self.lib.immesh_mesh_push_frame_from_lio(self._h, lio._h, ptr, n, 1 if on_device else 0), "mesh_push_frame_from_lio")

    def push_frame_from_lio_async(self, lio: "Lio", body_full, n=None, on_device=False):
        if on_device:
            ptr = C.c_void_p(body_full)
        else:
            a, p = _f32(body_full)
            n = a.shape[0]
            ptr = C.cast(p, C.c_void_p)
        _check(self.lib, self.lib.immesh_mesh_push_frame_from_lio_async(self._h, lio._h, ptr, n, 1 if on_device else 0), "mesh_push_frame_from_lio_async")

    def push_frame_from_lio_async_dev_n(self, lio: "Lio", d_body, n_max: int, d_n: int):
        """push_frame_from_lio_async of a device cloud whose count is device resident (int CUDA address d_n, *d_n <= n_max): e.g.
        input_points() / input_count() of a VoxelGrid after step_async_depth, with n_max its sampled pixels"""
        _check(self.lib, self.lib.immesh_mesh_push_frame_from_lio_async_dev_n(self._h, lio._h, C.c_void_p(int(d_body)), int(n_max), C.c_void_p(int(d_n))),
               "mesh_push_frame_from_lio_async_dev_n")

    def wait(self):
        _check(self.lib, self.lib.immesh_mesh_wait(self._h), "mesh_wait")

    @staticmethod
    def _depth_args(cam: DepthCamera, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device):
        """the immesh_depth_frame of one image: a 2-D float32 / uint16 numpy array (rows may be padded), or a CUDA address with
        shape = (height, width), fmt ("f32" / "u16") and pitch_bytes (0: tight)"""
        if on_device:
            height, width = shape
            ptr, keep = C.c_void_p(int(depth)), None
        else:
            keep = np.asarray(depth)
            if keep.ndim != 2 or keep.dtype not in (np.float32, np.uint16):
                raise ValueError("depth: a 2-D float32 or uint16 array")
            if keep.strides[1] != keep.itemsize or keep.strides[0] < keep.shape[1] * keep.itemsize:
                keep = np.ascontiguousarray(keep)
            height, width = keep.shape
            fmt, pitch_bytes = ("f32" if keep.dtype == np.float32 else "u16"), keep.strides[0]
            ptr = C.c_void_p(keep.ctypes.data)
        f = _DepthFrame(int(width), int(height), int(pitch_bytes), DEPTH_FORMATS[fmt], DEPTH_KINDS[cam.kind], float(cam.depth_scale), float(cam.fx),
                        float(cam.fy), float(cam.cx), float(cam.cy), float(cam.z_min), float(cam.z_max), int(cam.stride), 0,
                        (C.c_double * 9)(*np.asarray(cam_R, dtype=np.float64).reshape(9)), (C.c_double * 3)(*np.asarray(cam_t, dtype=np.float64).reshape(3)))
        return f, ptr, keep

    def push_depth(self, depth, cam: DepthCamera, cam_R, cam_t, on_device=False, shape=None, fmt="f32", pitch_bytes=0):
        """One mesh frame from a depth image, unprojected on the device (immesh_mesh_push_depth): the valid samples' world points,
        meshed at pose_t = cam_t.  cam_R, cam_t: camera to world, OpenCV axes."""
        f, ptr, _keep = self._depth_args(cam, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device)
        _check(self.lib, self.lib.immesh_mesh_push_depth(self._h, C.byref(f), ptr, 1 if on_device else 0), "mesh_push_depth")

    def push_depth_async(self, depth, cam: DepthCamera, cam_R, cam_t, on_device=False, shape=None, fmt="f32", pitch_bytes=0):
        """queued push_depth; wait() drains.  A host image is staged before the call returns; a device image must stay unchanged
        until the frame has run."""
        f, ptr, _keep = self._depth_args(cam, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device)
        _check(self.lib, self.lib.immesh_mesh_push_depth_async(self._h, C.byref(f), ptr, 1 if on_device else 0), "mesh_push_depth_async")

    def depth_points(self):
        """the newest depth frame's world points, float32[n][3] in ascending pixel order (immesh_mesh_depth_points; blocking)"""
        n = C.c_int(0)
        _check(self.lib, self.lib.immesh_mesh_depth_points(self._h, None, 0, C.byref(n)), "mesh_depth_points")
        out = np.zeros((n.value, 3), dtype=np.float32)
        if n.value:
            _check(self.lib, self.lib.immesh_mesh_depth_points(self._h, out.ctypes.data_as(C.POINTER(C.c_float)), n.value, C.byref(n)), "mesh_depth_points")
        return out

    def counts(self):
        o = np.zeros(8, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_counts(self._h, o.ctypes.data_as(C.POINTER(C.c_int64))), "mesh_counts")
        keys = ["n_vertices", "n_triangles", "frame_new_vertices", "frame_voxels_meshed", "frame_added", "frame_removed", "n_voxels", "n_activated"]
        return dict(zip(keys, (int(v) for v in o)))

    def shard(self, rank: int, nranks: int, unique_id: bytes):
        """Shard the per-voxel meshing stage over nranks processes (NCCL, own communicator: pass a second unique id)."""
        _check(self.lib, self.lib.immesh_mesh_shard(self._h, rank, nranks, unique_id), "mesh_shard")

    def shard_transport(self) -> str:
        return ("none", "nccl", "peer-window")[self.lib.immesh_mesh_shard_transport(self._h)]

    def work_stats(self):
        o = np.zeros(8, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_work_stats(self._h, o.ctypes.data_as(C.POINTER(C.c_int64))), "mesh_work_stats")
        keys = ["candidates", "gathered", "queries", "dilated", "faces", "voxels_meshed", "add_entries", "remove_entries"]
        return dict(zip(keys, (int(v) for v in o)))

    def snapshot(self):
        c = self.counts()
        v = np.zeros((c["n_vertices"], 3), dtype=np.float32)
        t = np.zeros((c["n_triangles"], 3), dtype=np.int32)
        f = np.zeros(c["n_triangles"], dtype=np.int32)
        _check(self.lib, self.lib.immesh_mesh_snapshot(self._h, v.ctypes.data_as(C.POINTER(C.c_float)), t.ctypes.data_as(C.POINTER(C.c_int32)),
                                                     f.ctypes.data_as(C.POINTER(C.c_int32))), "mesh_snapshot")
        return v, t, f

    def knn(self, q, k, max_dist=float("inf")):
        a, p = _f32(q)
        nq = a.shape[0]
        idx = np.zeros((nq, k), dtype=np.int32)
        d2 = np.zeros((nq, k), dtype=np.float32)
        _check(self.lib, self.lib.immesh_knn(self._h, p, nq, k, max_dist, idx.ctypes.data_as(C.POINTER(C.c_int32)), d2.ctypes.data_as(C.POINTER(C.c_float))), "knn")
        return idx, d2

    def reconstruct_from_pointcloud(self, vg: "VoxelGrid", pts, minimum_pts_distance: float) -> int:
        """reconstruct_mesh_from_pointcloud: VoxelGrid(leaf = minimum_pts_distance) + one frame with the identity pose; returns the down-sampled size."""
        a, p = _f32(pts)
        m = C.c_int(0)
        _check(self.lib, self.lib.immesh_mesh_reconstruct_from_pointcloud(self._h, vg._h, C.cast(p, C.c_void_p), a.shape[0], 0, minimum_pts_distance, C.byref(m)), "mesh_reconstruct_from_pointcloud")
        return m.value

    def push_frame_batched(self, world_xyz, pose_t, batch_points=0, batch_voxels=0, n=None, on_device=False):
        """One incremental_mesh_reconstruction frame of any size, run in bounded batches (the same mesh as one push_frame).
        world_xyz: float32[n][3] host array, or an integer CUDA address with n when on_device.  batch_points / batch_voxels: append
        candidates per chunk / activated voxels per batch (0: the handle's capacities).  Returns the frame's stats dict."""
        if on_device:
            ptr = C.c_void_p(world_xyz)
        else:
            a, p = _f32(world_xyz)
            n = a.shape[0]
            ptr = C.cast(p, C.c_void_p)
        t = np.ascontiguousarray(pose_t, dtype=np.float64)
        st = np.zeros(4, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_push_frame_batched(self._h, ptr, n, 1 if on_device else 0, t.ctypes.data_as(C.POINTER(C.c_double)), batch_points, batch_voxels,
                                                               st.ctypes.data_as(C.POINTER(C.c_int64))), "mesh_push_frame_batched")
        return dict(zip(["append_chunks", "voxel_batches", "scratch_bytes", "facets_added"], (int(v) for v in st)))

    def reconstruct_from_pointcloud_batched(self, vg: "VoxelGrid", pts, minimum_pts_distance: float, batch_points=0, batch_voxels=0) -> int:
        """reconstruct_mesh_from_pointcloud on a cloud of any size: PCL's VoxelGrid decision on the whole cloud, then one batched frame with
        the identity pose; returns the number of points meshed (the cloud's size when PCL passes it through)."""
        a, p = _f32(pts)
        m = C.c_int64(0)
        _check(self.lib, self.lib.immesh_mesh_reconstruct_from_pointcloud_batched(self._h, vg._h, C.cast(p, C.c_void_p), a.shape[0], 0, minimum_pts_distance, batch_points,
                                                                                batch_voxels, C.byref(m)), "mesh_reconstruct_from_pointcloud_batched")
        return m.value

    def render_depth(self, intrinsics, width, height, z_near, z_far, cam_R, cam_t):
        """(depth float32[h,w] (-1 = empty), points float32[n,3], pixel int32[n]) -- depth rasterisation of the live mesh."""
        K = np.ascontiguousarray(intrinsics, dtype=np.float64)
        R = np.ascontiguousarray(cam_R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(cam_t, dtype=np.float64)
        depth = np.zeros((height, width), dtype=np.float32)
        pts = np.zeros((height * width, 3), dtype=np.float32)
        pix = np.zeros(height * width, dtype=np.int32)
        n = C.c_int(0)
        dp = C.POINTER(C.c_double)
        _check(self.lib, self.lib.immesh_mesh_render_depth(self._h, K.ctypes.data_as(dp), width, height, z_near, z_far, R.ctypes.data_as(dp), t.ctypes.data_as(dp),
                                                           depth.ctypes.data_as(C.POINTER(C.c_float)), pts.ctypes.data_as(C.POINTER(C.c_float)),
                                                           pix.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n)), "mesh_render_depth")
        return depth, pts[:n.value].copy(), pix[:n.value].copy()

    def reinforce_enable(self, intrinsics=None, width=640, height=480, z_near=0.1, z_far=1500.0, win=1):
        """Queue the LiDAR point-cloud reinforcement behind every frame (intrinsics None: the reference's camera, reinforce_intrinsics)."""
        if intrinsics is None:
            intrinsics = reinforce_intrinsics(width, height)
        K = np.ascontiguousarray(intrinsics, dtype=np.float64)
        self._rf_shape = (height, width)
        _check(self.lib, self.lib.immesh_mesh_reinforce_enable(self._h, K.ctypes.data_as(C.POINTER(C.c_double)), width, height, z_near, z_far, win), "mesh_reinforce_enable")

    def reinforce_disable(self):
        _check(self.lib, self.lib.immesh_mesh_reinforce_enable(self._h, None, 0, 0, 0.0, 0.0, 0), "mesh_reinforce_enable")

    def reinforce_pose(self, cam_R=None, cam_t=None):
        """The caller's camera pose from the next frame on (None: back to the pose bound to the sensor)."""
        if cam_R is None:
            _check(self.lib, self.lib.immesh_mesh_reinforce_pose(self._h, None, None), "mesh_reinforce_pose")
            return
        R = np.ascontiguousarray(cam_R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(cam_t, dtype=np.float64).reshape(3)
        dp = C.POINTER(C.c_double)
        _check(self.lib, self.lib.immesh_mesh_reinforce_pose(self._h, R.ctypes.data_as(dp), t.ctypes.data_as(dp)), "mesh_reinforce_pose")

    def reinforced_cloud(self):
        """(depth float32[h,w], points float32[n,3], pixel int32[n], cam_R float64[3,3], cam_t float64[3]) of the newest queued frame."""
        n = C.c_int(0)
        pose = np.zeros(12)
        dp = C.POINTER(C.c_double)
        rc = self.lib.immesh_mesh_reinforced_cloud(self._h, None, None, None, 0, C.byref(n), pose.ctypes.data_as(dp))
        if rc not in (0, -3):
            _check(self.lib, rc, "mesh_reinforced_cloud")
        depth = np.zeros(self._rf_shape, dtype=np.float32)
        pts = np.zeros((max(n.value, 1), 3), dtype=np.float32)
        pix = np.zeros(max(n.value, 1), dtype=np.int32)
        _check(self.lib, self.lib.immesh_mesh_reinforced_cloud(self._h, depth.ctypes.data_as(C.POINTER(C.c_float)), pts.ctypes.data_as(C.POINTER(C.c_float)),
                                                               pix.ctypes.data_as(C.POINTER(C.c_int32)), n.value, C.byref(n), pose.ctypes.data_as(dp)), "mesh_reinforced_cloud")
        return depth, pts[:n.value].copy(), pix[:n.value].copy(), pose[:9].reshape(3, 3).copy(), pose[9:].copy()

    def render_view(self, intrinsics, width, height, z_near, z_far, cam_R, cam_t, positions=0, color_by_height=False, z_range=None):
        """(rgba uint8[h,w,4], depth float32[h,w]) -- the viewer's shaded image of the live mesh at the caller's camera (positions 0: raw,
        1: smoothed where the vertex is smoothed; z_range None: the height colour's range from the mesh)."""
        K = np.ascontiguousarray(intrinsics, dtype=np.float64)
        R = np.ascontiguousarray(cam_R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(cam_t, dtype=np.float64).reshape(3)
        rgba = np.zeros((height, width, 4), dtype=np.uint8)
        depth = np.zeros((height, width), dtype=np.float32)
        st = _view_style(positions, color_by_height, z_range)
        dp = C.POINTER(C.c_double)
        _check(self.lib, self.lib.immesh_mesh_render_view(self._h, K.ctypes.data_as(dp), width, height, z_near, z_far, R.ctypes.data_as(dp), t.ctypes.data_as(dp),
                                                          C.byref(st), rgba.ctypes.data_as(C.POINTER(C.c_uint8)), depth.ctypes.data_as(C.POINTER(C.c_float))),
               "mesh_render_view")
        return rgba, depth

    def view_enable(self, intrinsics=None, width=640, height=480, z_near=0.1, z_far=1500.0, win=1, positions=0, color_by_height=False, z_range=None):
        """Queue the shaded view behind every frame (intrinsics None: the reference's camera, reinforce_intrinsics), sensor-bound."""
        if intrinsics is None:
            intrinsics = reinforce_intrinsics(width, height)
        K = np.ascontiguousarray(intrinsics, dtype=np.float64)
        st = _view_style(positions, color_by_height, z_range)
        _check(self.lib, self.lib.immesh_mesh_view_enable(self._h, K.ctypes.data_as(C.POINTER(C.c_double)), width, height, z_near, z_far, win, C.byref(st)),
               "mesh_view_enable")
        self._vw_shape = (height, width)
        self._feed_img = None   # every view_enable turns the frame feed's images off

    def view_disable(self):
        _check(self.lib, self.lib.immesh_mesh_view_enable(self._h, None, 0, 0, 0.0, 0.0, 0, None), "mesh_view_enable")
        self._feed_img = None

    def view_pose(self, cam_R=None, cam_t=None, follow=False):
        """The queued view's camera from the next frame on: None the sensor-bound pose; (cam_R, cam_t) a fixed camera; with follow, the
        rotation cam_R at the sensor window's mean position plus the offset cam_t."""
        dp = C.POINTER(C.c_double)
        if cam_R is None:
            _check(self.lib, self.lib.immesh_mesh_view_pose(self._h, None, None, 0), "mesh_view_pose")
            return
        R = np.ascontiguousarray(cam_R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(cam_t, dtype=np.float64).reshape(3)
        _check(self.lib, self.lib.immesh_mesh_view_pose(self._h, R.ctypes.data_as(dp), t.ctypes.data_as(dp), 1 if follow else 0), "mesh_view_pose")

    def view_overlay(self, wireframe=False, scan_point_size=2, reinforced_point_size=2, axis_and_grid=True, camera_size=1.0, path_width=4,
                     path_capacity=1 << 16):
        """Draw the rest of the viewer's window into the queued view from the next frame on (defaults: the reference's): the current
        scan, the reinforced points, the axis and ground grid, the sensor's camera frustum and the trajectory of the frames queued
        from now on (the newest path_capacity positions); wireframe draws the live triangles' edges instead of the faces.  Sizes and
        widths in pixels, 0: off."""
        o = _ViewOverlay(1 if wireframe else 0, int(scan_point_size), int(reinforced_point_size), 1 if axis_and_grid else 0, float(camera_size),
                         int(path_width), int(path_capacity))
        _check(self.lib, self.lib.immesh_mesh_view_overlay(self._h, C.byref(o)), "mesh_view_overlay")

    def view_overlay_off(self):
        _check(self.lib, self.lib.immesh_mesh_view_overlay(self._h, None), "mesh_view_overlay")

    def view_image(self):
        """(rgba uint8[h,w,4], depth float32[h,w], cam_R float64[3,3], cam_t float64[3], frame) of the newest queued frame."""
        rgba = np.zeros(self._vw_shape + (4,), dtype=np.uint8)
        depth = np.zeros(self._vw_shape, dtype=np.float32)
        pose = np.zeros(12)
        frame = C.c_int64(0)
        _check(self.lib, self.lib.immesh_mesh_view_image(self._h, rgba.ctypes.data_as(C.POINTER(C.c_uint8)), depth.ctypes.data_as(C.POINTER(C.c_float)),
                                                         pose.ctypes.data_as(C.POINTER(C.c_double)), C.byref(frame)), "mesh_view_image")
        return rgba, depth, pose[:9].reshape(3, 3).copy(), pose[9:].copy(), frame.value

    def changes_enable(self, max_rows=1 << 20, max_frames=256):
        """Record every later frame's triangle changes on the device: a ring of max_rows rows, the headers of the last max_frames frames.
        The published state starts as the mesh is now (snapshot())."""
        _check(self.lib, self.lib.immesh_mesh_changes_enable(self._h, max_rows, max_frames), "mesh_changes_enable")

    def changes_disable(self):
        _check(self.lib, self.lib.immesh_mesh_changes_enable(self._h, 0, 0), "mesh_changes_enable")

    def changes_newest(self) -> int:
        """the newest frame queued with the change feed on (where a mirror resynchronised by snapshot() reads on from)"""
        counts = np.zeros(4, dtype=np.int64)
        rc = self.lib.immesh_mesh_changes(self._h, -1, None, 0, None, 0, None, 0, counts.ctypes.data_as(C.POINTER(C.c_int64)))
        if rc != -5:   # before the enable: IMMESH_E_RANGE with counts[3] = newest
            _check(self.lib, rc, "mesh_changes")
        return int(counts[3])

    def changes(self, since: int):
        """The frames (since, newest] of the change feed: dict(frames int64[n][4] = frame, v_begin, v_end, rows_end; rows int32[m][4] =
        a, b, c, code (0 removed, 2 | flip added, 4 | flip re-oriented), ascending triples inside a frame; vertices float32[k][3] of the
        ids [frames[0, 1], frames[-1, 2]); newest).  RuntimeError with code -5 (IMMESH_E_RANGE) when a frame is no longer held."""
        counts = np.zeros(4, dtype=np.int64)
        cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
        rc = self.lib.immesh_mesh_changes(self._h, since, None, 0, None, 0, None, 0, cp)
        if rc not in (0, -3):
            _check(self.lib, rc, "mesh_changes")
        fr = np.zeros((int(counts[0]), 4), dtype=np.int64)
        rows = np.zeros((int(counts[1]), 4), dtype=np.int32)
        v = np.zeros((int(counts[2]), 3), dtype=np.float32)
        if rc:
            _check(self.lib, self.lib.immesh_mesh_changes(self._h, since, fr.ctypes.data_as(C.POINTER(C.c_int64)), len(fr), rows.ctypes.data_as(C.POINTER(C.c_int32)),
                                                          len(rows), v.ctypes.data_as(C.POINTER(C.c_float)), len(v), cp), "mesh_changes")
        return dict(frames=fr, rows=rows, vertices=v, newest=int(counts[3]))

    def feed_enable(self, max_frames=1024, max_rows=1 << 22, max_images=0, depth=False):
        """Record every later frame's header, poses, reinforced points and (max_images > 0, the queued view on) viewer image on the
        device (immesh_mesh_feed_enable).  The image ring is sized for the view as it is now; view_enable turns the images off."""
        c = _MeshFeedCfg(int(max_frames), int(max_rows), int(max_images), 1 if depth else 0, 0)
        _check(self.lib, self.lib.immesh_mesh_feed_enable(self._h, C.byref(c)), "mesh_feed_enable")
        self._feed_img = (getattr(self, "_vw_shape", None), bool(depth)) if max_images > 0 else None

    def feed_disable(self):
        _check(self.lib, self.lib.immesh_mesh_feed_enable(self._h, None), "mesh_feed_enable")
        self._feed_img = None

    def _feed_read(self, call, alloc, what):
        """count query, then the read; frames may finish between the two"""
        counts = np.zeros(4, dtype=np.int64)
        cp = counts.ctypes.data_as(C.POINTER(C.c_int64))
        for first in (True,) + (False,) * 8:
            rc = call(None, counts, cp, first)
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, what)
            bufs = alloc(int(counts[0]), int(counts[1]))
            if counts[0] == 0:
                return bufs, counts
            rc = call(bufs, counts, cp, False)
            if rc == -3:
                continue
            if rc == -5:
                raise FeedLost(self.lib.immesh_last_error().decode(), int(counts[2]))
            _check(self.lib, rc, what)
            return bufs, counts
        raise RuntimeError(f"{what}: the frames kept finishing faster than they were read")

    def feed(self, since: int, wait: bool = False):
        """The frames (since, newest finished] of the frame feed: dict(frames=int64[m, MESH_FEED_HDR] (MESH_FEED_HDR_KEYS),
        poses=float64[m, 3, 12] (frame pose, reinforcement camera, view camera; R row-major then t), points=float32[r, 3],
        pixels=int32[r], newest_finished, newest_queued).  wait=False never blocks on unfinished work.  Raises FeedLost when frames of
        the range predate the enable or left the rings."""
        i64, f32, i32, dp = C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_double)

        def alloc(nf, nr):
            return (np.zeros((max(nf, 1), MESH_FEED_HDR), np.int64), np.zeros((max(nf, 1), MESH_FEED_POSE)), np.zeros((max(nr, 1), 3), np.float32),
                    np.zeros(max(nr, 1), np.int32), nf, nr)

        def call(b, counts, cp, first):
            if b is None:
                return self.lib.immesh_mesh_feed(self._h, since, 1 if (wait and first) else 0, None, None, 0, None, None, 0, cp)
            return self.lib.immesh_mesh_feed(self._h, since, 0, b[0].ctypes.data_as(i64), b[1].ctypes.data_as(dp), b[4], b[2].ctypes.data_as(f32),
                                             b[3].ctypes.data_as(i32), b[5], cp)
        b, counts = self._feed_read(call, alloc, "mesh_feed")
        nf, nr = int(counts[0]), int(counts[1])
        return dict(frames=b[0][:nf], poses=b[1][:nf].reshape(nf, 3, 12), points=b[2][:nr], pixels=b[3][:nr], newest_finished=int(counts[2]),
                    newest_queued=int(counts[3]))

    def feed_images(self, since: int, wait: bool = False):
        """The frames (since, newest finished] and the view images they hold: dict(frames=int64[m, MESH_FEED_HDR], rgba=uint8[k, h, w, 4],
        depth=float32[k, h, w] (feed enabled with depth) or None, newest_finished, newest_queued).  Raises FeedLost when an image of the
        range left the ring, even while its header is held."""
        (hh, ww), with_depth = getattr(self, "_feed_img", None) or ((1, 1), False)
        i64 = C.POINTER(C.c_int64)

        def alloc(nf, ni):
            return (np.zeros((max(nf, 1), MESH_FEED_HDR), np.int64), np.zeros((max(ni, 1), hh, ww, 4), np.uint8),
                    np.zeros((max(ni, 1), hh, ww), np.float32) if with_depth else None, nf, ni)

        def call(b, counts, cp, first):
            if b is None:
                return self.lib.immesh_mesh_feed_images(self._h, since, 1 if (wait and first) else 0, None, 0, None, None, cp)
            return self.lib.immesh_mesh_feed_images(self._h, since, 0, b[0].ctypes.data_as(i64), b[3], b[1].ctypes.data_as(C.POINTER(C.c_uint8)),
                                                    b[2].ctypes.data_as(C.POINTER(C.c_float)) if b[2] is not None else None, cp)
        b, counts = self._feed_read(call, alloc, "mesh_feed_images")
        nf, ni = int(counts[0]), int(counts[1])
        return dict(frames=b[0][:nf], rgba=b[1][:ni], depth=b[2][:ni] if b[2] is not None else None, newest_finished=int(counts[2]),
                    newest_queued=int(counts[3]))

    def smooth_all(self, smooth_factor=0.1, knn=20):
        """smooth_all_pts: returns the smoothed positions float64[nv,3] (and stores them as the vertices' smoothed positions)."""
        nv = self.counts()["n_vertices"]
        out = np.zeros((nv, 3))
        _check(self.lib, self.lib.immesh_mesh_smooth_all(self._h, smooth_factor, knn, out.ctypes.data_as(C.POINTER(C.c_double))), "mesh_smooth_all")
        return out

    def evaluate(self, gt, *, spacing=0.01, gt_leaf=0.01, threshold=0.05, max_dist=1.0, incorrect_ratio=0.8, smoothed=False, facets=False,
                 max_batch_bytes=0, on_device=False):
        """The paper's Experiment-3 metrics of the mesh against the ground-truth cloud gt (float32[n,3] host array, or (CUDA address, n)
        when on_device).  Returns dict(counts={EVAL_COUNT_KEYS: int}, metrics={EVAL_METRIC_KEYS: float}) and, with facets, rows
        int32[live][5] = a b c n_samples n_far in ascending triple order.  smoothed: evaluate the smoothed positions (smooth_all first)."""
        if on_device:
            ptr, n = C.c_void_p(gt[0]), int(gt[1])
        else:
            a, p = _f32(np.asarray(gt).reshape(-1, 3))
            ptr, n = C.cast(p, C.c_void_p), a.shape[0]
        cfg = _EvalCfg(spacing, gt_leaf, threshold, max_dist, incorrect_ratio, 1 if smoothed else 0, 0, max_batch_bytes)
        counts = np.zeros(12, dtype=np.int64)
        metrics = np.zeros(8)
        nr = C.c_int64(0)
        i64 = C.POINTER(C.c_int64)
        rows = None
        if facets:   # a count query (cap_rows = 0) sizes the rows
            dummy = np.zeros(5, dtype=np.int32)
            rc = self.lib.immesh_mesh_evaluate(self._h, ptr, n, 1 if on_device else 0, C.byref(cfg), counts.ctypes.data_as(i64), metrics.ctypes.data_as(C.POINTER(C.c_double)),
                                               dummy.ctypes.data_as(C.POINTER(C.c_int32)), 0, C.byref(nr))
            if rc not in (0, -3):
                _check(self.lib, rc, "mesh_evaluate")
            rows = np.zeros((max(nr.value, 1), 5), dtype=np.int32)
        _check(self.lib, self.lib.immesh_mesh_evaluate(self._h, ptr, n, 1 if on_device else 0, C.byref(cfg), counts.ctypes.data_as(i64),
                                                       metrics.ctypes.data_as(C.POINTER(C.c_double)),
                                                       rows.ctypes.data_as(C.POINTER(C.c_int32)) if facets else None, len(rows) if facets else 0,
                                                       C.byref(nr)), "mesh_evaluate")
        out = dict(counts=dict(zip(EVAL_COUNT_KEYS, (int(v) for v in counts))), metrics=dict(zip(EVAL_METRIC_KEYS, (float(v) for v in metrics[:7]))))
        if facets:
            out["rows"] = rows[:nr.value].copy()
        st = np.zeros(4, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_evaluate_stats(st.ctypes.data_as(i64)), "mesh_evaluate_stats")
        out["stats"] = dict(zip(("tiles", "plan_boxes", "scratch_bytes", "table_bytes"), (int(v) for v in st)))
        return out

    def texture_select(self, cameras, *, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False, positions=0, vertices=True):
        """The paper's textured mesh (Application-2): per live triangle, in snapshot order, the nearest camera that sees it and its
        corners' pixel coordinates there.  cameras: (width, height, (fx, fy, cx, cy), cam_R, cam_t) tuples, OpenCV axes, camera to world.
        positions 1: the smoothed positions where the vertex is smoothed (smooth_all first to match the smoothed PLY).  Returns
        dict(cam int32[nt] (-1: none), uv float32[nt,6] (u0 v0 u1 v1 u2 v2 of the corners in face order; NaN where cam = -1),
        px int32[nt,2] (won, covered pixels in the chosen camera), vertices float32[nv,3] (the positions used; with vertices, which
        first waits for the queued frames so that nv is known; else None), counts {TEXTURE_COUNT_KEYS: int})."""
        arr, n_cams = texture_cameras(cameras)
        cfg = _TexCfg(float(z_near), float(z_far), float(min_cos), int(min_visible_permille), 1 if two_sided else 0, int(positions), 0)
        i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
        nf = C.c_int64(0)
        counts = np.zeros(4, dtype=np.int64)
        rc = self.lib.immesh_mesh_texture_select(self._h, arr, n_cams, C.byref(cfg), None, None, None, None, 0, C.byref(nf), None)   # a count query
        if rc not in (0, -3):
            _check(self.lib, rc, "mesh_texture_select")
        if vertices:
            self.wait()
        n, nv = nf.value, self.counts()["n_vertices"] if vertices else 0
        cam = np.zeros(max(n, 1), dtype=np.int32)
        uv = np.full((max(n, 1), 6), np.nan, dtype=np.float32)
        px = np.zeros((max(n, 1), 2), dtype=np.int32)
        verts = np.zeros((max(nv, 1), 3), dtype=np.float32)
        _check(self.lib, self.lib.immesh_mesh_texture_select(self._h, arr, n_cams, C.byref(cfg), cam.ctypes.data_as(i32), uv.ctypes.data_as(C.POINTER(C.c_float)),
                                                             px.ctypes.data_as(i32), verts.ctypes.data_as(C.POINTER(C.c_float)) if vertices else None, n, C.byref(nf),
                                                             counts.ctypes.data_as(i64)), "mesh_texture_select")
        return dict(cam=cam[:n].copy(), uv=uv[:n].copy(), px=px[:n].copy(), vertices=verts[:nv].copy() if vertices else None,
                    counts=dict(zip(TEXTURE_COUNT_KEYS, (int(v) for v in counts))))

    def texture_enable(self, rig, *, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False, positions=0):
        """Texture the mesh behind every queued frame: each triangle record keeps the nearest frame whose camera sees it (texture_select's
        rule at raw positions).  rig: (width, height, (fx, fy, cx, cy), cam_R, cam_t), the colour camera in the frame's sensor frame
        (the localization body frame, or the depth camera), OpenCV axes; None turns the texturing off.  Every record starts unobserved."""
        if rig is None:
            _check(self.lib, self.lib.immesh_mesh_texture_enable(self._h, None, None), "mesh_texture_enable")
            return
        arr, _ = texture_cameras([rig])
        cfg = _TexCfg(float(z_near), float(z_far), float(min_cos), int(min_visible_permille), 1 if two_sided else 0, int(positions), 0)
        _check(self.lib, self.lib.immesh_mesh_texture_enable(self._h, arr, C.byref(cfg)), "mesh_texture_enable")

    def texture_pose(self, R=None, t=None):
        """From the next queued frame on: (R, t) a fixed caller camera (camera to world, OpenCV axes) for every frame; None, None the rig."""
        dp = C.POINTER(C.c_double)
        if R is None and t is None:
            _check(self.lib, self.lib.immesh_mesh_texture_pose(self._h, None, None), "mesh_texture_pose")
            return
        R = np.ascontiguousarray(R, dtype=np.float64).reshape(9)
        t = np.ascontiguousarray(t, dtype=np.float64).reshape(3)
        _check(self.lib, self.lib.immesh_mesh_texture_pose(self._h, R.ctypes.data_as(dp), t.ctypes.data_as(dp)), "mesh_texture_pose")

    def texture_rows(self, vertices=True):
        """The queued texturing's rows, ordered behind the queued frames, in texture_select's layout: dict(cam int32[nt] (the frame
        number, -1: none), uv float32[nt,6] (NaN where cam = -1), px int32[nt,2], vertices float32[nv,3] (the snapshot's raw
        positions, or None), counts {TEXTURE_COUNT_KEYS: int} (cameras_used: distinct frames
        of the live rows), frames int32[nf] (ascending frames any record still uses: keep these images, delete the others)).  With the
        cameras indexed by frame number (None images for the other frames) it goes to texture_bake and write_obj_textured."""
        i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
        nf, nfr = C.c_int64(0), C.c_int64(0)
        rc = self.lib.immesh_mesh_texture_rows(self._h, None, None, None, 0, C.byref(nf), None, None, 0, C.byref(nfr))   # a count query
        if rc not in (0, -3):
            _check(self.lib, rc, "mesh_texture_rows")
        n, m = nf.value, nfr.value
        cam = np.zeros(max(n, 1), dtype=np.int32)
        uv = np.full((max(n, 1), 6), np.nan, dtype=np.float32)
        px = np.zeros((max(n, 1), 2), dtype=np.int32)
        frames = np.zeros(max(m, 1), dtype=np.int32)
        counts = np.zeros(4, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_texture_rows(self._h, cam.ctypes.data_as(i32), uv.ctypes.data_as(C.POINTER(C.c_float)), px.ctypes.data_as(i32), n,
                                                           C.byref(nf), counts.ctypes.data_as(i64), frames.ctypes.data_as(i32), m, C.byref(nfr)),
               "mesh_texture_rows")
        verts = self.snapshot()[0] if vertices else None
        return dict(cam=cam[:n].copy(), uv=uv[:n].copy(), px=px[:n].copy(), vertices=verts, counts=dict(zip(TEXTURE_COUNT_KEYS, (int(v) for v in counts))),
                    frames=frames[:m].copy())

    def texture_bake(self, sel, cameras, images, *, page_size=4096, max_cell=64, max_image_bytes=0):
        """The texture atlas of a selection: every textured facet's pixels resampled out of its chosen image into square pages.
        sel: texture_select's result (cam, uv); cameras: the selection's camera tuples (their width and height rescale uv to each
        image); images: per camera an HxWx3 uint8 numpy array or CUDA torch tensor (all one kind), None for a camera no facet uses.
        Blocking, ordered behind the queued frames; writes nothing on the handle.  Returns dict(pages uint8[n_pages, P, P, 3],
        page int32[nt] (-1: untextured), uv float32[nt,6] (the corners in page texels; NaN where page = -1),
        counts {BAKE_COUNT_KEYS: int}).  Export: write_obj_textured(..., page, uv, [(P, P)] * n_pages, png_files) after write_png."""
        arr, n_cams = texture_cameras(cameras)
        imgs, on_device, keep = texture_images(images)
        cam = np.ascontiguousarray(sel["cam"], dtype=np.int32).reshape(-1)
        uv = np.ascontiguousarray(sel["uv"], dtype=np.float32).reshape(-1, 6)
        n = len(cam)
        cfg = _AtlasCfg(int(page_size), int(max_cell), int(max_image_bytes))
        i32 = C.POINTER(C.c_int32)
        np_ = C.c_int(0)
        page = np.full(max(n, 1), -1, np.int32)
        auv = np.full((max(n, 1), 6), np.nan, np.float32)
        counts = np.zeros(4, np.int64)
        rc = self.lib.immesh_mesh_texture_bake(self._h, arr, n_cams, imgs, on_device, cam.ctypes.data_as(i32), uv.ctypes.data_as(C.POINTER(C.c_float)), n,
                                               C.byref(cfg), None, 0, None, None, C.byref(np_), None)   # a count query
        _check(self.lib, rc, "mesh_texture_bake")
        P = int(page_size)
        pages = np.zeros((np_.value, P, P, 3), np.uint8)
        _check(self.lib, self.lib.immesh_mesh_texture_bake(self._h, arr, n_cams, imgs, on_device, cam.ctypes.data_as(i32), uv.ctypes.data_as(C.POINTER(C.c_float)), n,
                                                           C.byref(cfg), pages.ctypes.data_as(C.c_void_p), pages.shape[0], page.ctypes.data_as(i32),
                                                           auv.ctypes.data_as(C.POINTER(C.c_float)), C.byref(np_), counts.ctypes.data_as(C.POINTER(C.c_int64))),
               "mesh_texture_bake")
        del keep
        return dict(pages=pages, page=page[:n].copy(), uv=auv[:n].copy(), counts=dict(zip(BAKE_COUNT_KEYS, (int(v) for v in counts))))

    def render_textured(self, view, sel, cameras, images=None, *, truth=None, z_near=0.1, z_far=1000.0, positions=0, untextured=(128, 128, 128),
                        background=(0, 0, 0), max_image_bytes=0):
        """The textured mesh rendered at camera view ((width, height, (fx, fy, cx, cy), cam_R, cam_t), OpenCV axes, camera to world), and
        scored against truth, a photo taken there.  sel: rows of texture_select or texture_rows (cam, uv), or of texture_bake (page, uv);
        cameras: the rows' camera tuples (only the sizes are read: (P, P) per page for the bake's rows); images: per camera an HxWx3 uint8
        numpy array or CUDA torch tensor (all one kind, truth too), None for a camera the view does not sample.  images None: the query
        (depth, facet, needed and the first four counts).  positions: the rows' own setting.  Blocking, ordered behind the queued frames;
        writes nothing on the handle.  Returns dict(rgb uint8[h,w,3] (None for the query), depth float32[h,w] (render_view's), facet
        int32[h,w] (the winning snapshot row, -1: no sample), needed uint8[n_cams] (1: the view samples that camera), counts
        {TEXTURE_VIEW_COUNT_KEYS: int}); with truth also mse = sum sse / (3 n), psnr = 10 log10(255^2 / mse) (inf when mse = 0), mae =
        sad / (3 n) and coverage = n / (w h), n the textured pixels (mse, psnr and mae NaN when n = 0).  Report coverage beside psnr:
        texturing fewer pixels can raise psnr."""
        vw, _ = texture_cameras([view])
        arr, n_cams = texture_cameras(cameras)
        keep = []
        imgs, on_device = None, 0
        if images is not None:
            imgs, on_device, keep = texture_images(images)
        tr = None
        if truth is not None:
            if images is None:
                raise ValueError("render_textured: truth needs images")
            tr, t_dev, tk = texture_images([truth])
            if t_dev != on_device and any(im is not None for im in images):
                raise ValueError("render_textured: truth and images must be the same kind")
            on_device = t_dev if all(im is None for im in images) else on_device
            keep += tk
        cam = np.ascontiguousarray(sel["cam"] if "cam" in sel else sel["page"], dtype=np.int32).reshape(-1)
        uv = np.ascontiguousarray(sel["uv"], dtype=np.float32).reshape(-1, 6)
        cfg = _TexViewCfg(float(z_near), float(z_far), int(positions), (C.c_uint8 * 3)(*untextured), (C.c_uint8 * 3)(*background), int(max_image_bytes))
        w, h = int(view[0]), int(view[1])
        rgb = np.zeros((h, w, 3), np.uint8) if images is not None else None
        depth = np.zeros((h, w), np.float32)
        facet = np.zeros((h, w), np.int32)
        needed = np.zeros(max(n_cams, 1), np.uint8)
        counts = np.zeros(8, np.int64)
        i32 = C.POINTER(C.c_int32)
        _check(self.lib, self.lib.immesh_mesh_render_textured(self._h, vw, C.byref(cfg), arr, n_cams, imgs, on_device, cam.ctypes.data_as(i32),
                                                              uv.ctypes.data_as(C.POINTER(C.c_float)), len(cam), tr,
                                                              None if rgb is None else rgb.ctypes.data_as(C.c_void_p), depth.ctypes.data_as(C.POINTER(C.c_float)),
                                                              facet.ctypes.data_as(i32), needed.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.POINTER(C.c_int64))),
               "mesh_render_textured")
        del keep
        out = dict(rgb=rgb, depth=depth, facet=facet, needed=needed[:n_cams].copy(), counts=dict(zip(TEXTURE_VIEW_COUNT_KEYS, (int(v) for v in counts))))
        if truth is not None:
            n = int(counts[0])
            sse, sad = int(counts[4] + counts[5] + counts[6]), int(counts[7])
            mse = sse / (3.0 * n) if n else float("nan")
            out.update(mse=mse, psnr=(float("inf") if mse == 0 else 10.0 * np.log10(255.0 ** 2 / mse)) if n else float("nan"),
                       mae=sad / (3.0 * n) if n else float("nan"), coverage=n / float(w * h))
        return out

    def render_textured_stats(self):
        """the phases of this thread's last render_textured in ms, from CUDA events: dict(pass_a, pass_b (host images: with the uploads
        it waits for), score)"""
        ms = np.zeros(3, np.float64)
        _check(self.lib, self.lib.immesh_mesh_render_textured_stats(ms.ctypes.data_as(C.POINTER(C.c_double))), "mesh_render_textured_stats")
        return dict(zip(("pass_a", "pass_b", "score"), (float(v) for v in ms)))

    def texture_gains(self, rows, cameras, images, *, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False, positions=0,
                      sigma_n=10.0, sigma_g=0.1, max_pairs=1 << 20, max_image_bytes=0, pairs=False):
        """Colour equalisation between cameras (Brown & Lowe gain compensation): one gain per camera and channel so that cameras agree
        on the facets several of them see.  rows: texture_select's or texture_rows' result (cam, uv), before any bake; cameras: full
        camera tuples indexed as the rows index them (by frame number for texture_rows); images: per camera an HxWx3 uint8 numpy array
        or CUDA torch tensor (all one kind), None for a camera that takes no part (every camera that textures a row needs one).  The
        select keywords decide whether an observer sees a facet: pass the rows' own.  Blocking, ordered behind the queued frames; writes
        nothing on the handle.  Returns dict(gains float64[n_cams, 3], counts {TEXTURE_GAINS_COUNT_KEYS: int}) and with pairs=True also
        pair_cam int32[n_pairs, 2] (observer k, chosen c) and pair_sums int64[n_pairs, 7] (n, S_k[3], S_c[3]).  Correct the images with
        apply_gains, then bake, render or export them."""
        arr, n_cams = texture_cameras(cameras)
        imgs, on_device, keep = texture_images(images)
        cam = np.ascontiguousarray(rows["cam"], dtype=np.int32).reshape(-1)
        uv = np.ascontiguousarray(rows["uv"], dtype=np.float32).reshape(-1, 6)
        sel = _TexCfg(float(z_near), float(z_far), float(min_cos), int(min_visible_permille), 1 if two_sided else 0, int(positions), 0)
        cfg = _TexGainsCfg(sel, float(sigma_n), float(sigma_g), int(max_pairs), int(max_image_bytes))
        gains = np.zeros((max(n_cams, 1), 3), np.float64)
        cap = int(max_pairs) if pairs else 0
        pc = np.zeros((max(cap, 1), 2), np.int32)
        ps = np.zeros((max(cap, 1), 7), np.int64)
        npairs = C.c_int64(0)
        counts = np.zeros(8, np.int64)
        i64 = C.POINTER(C.c_int64)
        _check(self.lib, self.lib.immesh_mesh_texture_gains(self._h, arr, n_cams, imgs, on_device, cam.ctypes.data_as(C.POINTER(C.c_int32)),
                                                            uv.ctypes.data_as(C.POINTER(C.c_float)), len(cam), C.byref(cfg),
                                                            gains.ctypes.data_as(C.POINTER(C.c_double)),
                                                            pc.ctypes.data_as(C.POINTER(C.c_int32)) if pairs else None, ps.ctypes.data_as(i64) if pairs else None,
                                                            C.byref(npairs), counts.ctypes.data_as(i64)), "mesh_texture_gains")
        del keep
        out = dict(gains=gains[:n_cams].copy(), counts=dict(zip(TEXTURE_GAINS_COUNT_KEYS, (int(v) for v in counts))))
        if pairs:
            out.update(pair_cam=pc[:npairs.value].copy(), pair_sums=ps[:npairs.value].copy())
        return out

    def texture_gains_stats(self):
        """the phases of this thread's last texture_gains in ms: dict(chosen, observers (CUDA events; host images: with the uploads they
        wait for), solve (host clock, read-back included))"""
        ms = np.zeros(3, np.float64)
        _check(self.lib, self.lib.immesh_mesh_texture_gains_stats(ms.ctypes.data_as(C.POINTER(C.c_double))), "mesh_texture_gains_stats")
        return dict(zip(("chosen", "observers", "solve"), (float(v) for v in ms)))

    def apply_gains(self, images, gains):
        """The corrected images: each channel min(255, floor(v g + 0.5)) with g = gains[k][ch].  images: HxWx3 uint8 numpy arrays or
        CUDA torch tensors (all one kind; None stays None); returns new images of the same kind (device images: one kernel on the mesh
        stream)."""
        images = list(images)
        g = np.ascontiguousarray(gains, dtype=np.float64).reshape(-1, 3)
        if len(g) < len(images):
            raise ValueError("apply_gains: one gain row per image")
        outs = []
        for im in images:
            if im is None:
                outs.append(None)
            elif type(im).__module__.split(".")[0] == "torch":
                outs.append(im.new_empty(im.shape).contiguous())
            else:
                outs.append(np.empty(np.asarray(im).shape, np.uint8))
        ia, on_device, keep = texture_images(images)
        oa, _, okeep = texture_images(outs)
        _check(self.lib, self.lib.immesh_texture_apply_gains(self._h, ia, oa, len(images), on_device, g.ctypes.data_as(C.POINTER(C.c_double))),
               "texture_apply_gains")
        del keep, okeep
        return outs

    def region_stream(self, region_size=10.0, cap=1 << 16):
        """(region_keys int32[nr,3], region_offsets int32[nr+1], triangles int32[nt,3]) -- the viewer's region-bucketed triangle sets."""
        nt = self.counts()["n_triangles"]
        keys, offs = np.zeros((cap, 3), dtype=np.int32), np.zeros(cap + 1, dtype=np.int32)
        tri = np.zeros((max(nt, 1), 3), dtype=np.int32)
        nr = C.c_int(0)
        i32 = C.POINTER(C.c_int32)
        _check(self.lib, self.lib.immesh_mesh_region_stream(self._h, region_size, keys.ctypes.data_as(i32), offs.ctypes.data_as(i32), cap, tri.ctypes.data_as(i32), C.byref(nr)), "mesh_region_stream")
        return keys[:nr.value].copy(), offs[:nr.value + 1].copy(), tri[:nt].copy()

    def region_buffers(self, region_size=10.0, keys=None, smooth_factor=1.0, knn=20, axis_min_max=None):
        """The viewer's triangle buffers (synchronize_triangle_list_for_disp -> unparse_triangle_set_to_vector + get_axis_min_max):
        (tri_xyz float32[n,9], tri_ids int32[n,3], region_keys int32[nr,3], region_offsets int32[nr+1], n_smoothed).  keys: int[k,3]
        regions in the order wanted, or None for every non-empty region.  axis_min_max: float32[6] (min xyz, max xyz), updated in place.
        A count query sizes the buffers first; vertices of the returned triangles whose smoothed flag is clear are smoothed."""
        i32, f32p = C.POINTER(C.c_int32), C.POINTER(C.c_float)
        kp, nk = None, 0
        if keys is not None:
            k = np.ascontiguousarray(keys, dtype=np.int32).reshape(-1, 3)
            kp, nk = k.ctypes.data_as(i32), k.shape[0]
        box = None
        if axis_min_max is not None:
            assert isinstance(axis_min_max, np.ndarray) and axis_min_max.dtype == np.float32 and axis_min_max.shape == (6,) and axis_min_max.flags.c_contiguous
            box = axis_min_max.ctypes.data_as(f32p)
        nr, nt, ns = C.c_int(0), C.c_int(0), C.c_int(0)
        rc = self.lib.immesh_mesh_region_buffers(self._h, region_size, kp, nk, smooth_factor, knn, None, None, 0, None, None, 0, None,
                                                 C.byref(nr), C.byref(nt), C.byref(ns))
        if rc not in (0, -3):
            _check(self.lib, rc, "mesh_region_buffers")
        xyz = np.zeros((nt.value, 9), dtype=np.float32)
        ids = np.zeros((nt.value, 3), dtype=np.int32)
        rkeys = np.zeros((nr.value, 3), dtype=np.int32)
        roff = np.zeros(nr.value + 1, dtype=np.int32)
        _check(self.lib, self.lib.immesh_mesh_region_buffers(self._h, region_size, kp, nk, smooth_factor, knn, xyz.ctypes.data_as(f32p), ids.ctypes.data_as(i32),
                                                             nt.value, rkeys.ctypes.data_as(i32), roff.ctypes.data_as(i32), nr.value, box,
                                                             C.byref(nr), C.byref(nt), C.byref(ns)), "mesh_region_buffers")
        return xyz, ids, rkeys, roff, ns.value

    # --- long runs: capacities and growth of the mesh pools
    def capacity(self):
        """dict(vertices_cap, vertices, triangles_cap, triangles, voxels_cap, voxels, device_bytes, growths)"""
        o = np.zeros(8, dtype=np.int64)
        _check(self.lib, self.lib.immesh_mesh_capacity(self._h, o.ctypes.data_as(C.POINTER(C.c_int64))), "mesh_capacity")
        keys = ("vertices_cap", "vertices", "triangles_cap", "triangles", "voxels_cap", "voxels", "device_bytes", "growths")
        return dict(zip(keys, (int(v) for v in o)))

    def reserve(self, vertices=0, triangles=0, voxels=0):
        """Grow the pools to at least these capacities (0: keep); never shrinks."""
        _check(self.lib, self.lib.immesh_mesh_reserve(self._h, vertices, triangles, voxels), "mesh_reserve")

    def set_growth(self, max_bytes):
        """Automatic growth before every frame, up to max_bytes of device memory for the handle (0: off)."""
        _check(self.lib, self.lib.immesh_mesh_set_growth(self._h, max_bytes), "mesh_set_growth")

    def last_timing(self):
        o = np.zeros(4)
        self.lib.immesh_mesh_last_timing(self._h, o.ctypes.data_as(C.POINTER(C.c_double)))
        return o


class VoxelGrid:
    """pcl::VoxelGrid front-end on the device (immesh_voxelgrid_*): filter(points, leaf) -> centroids, leaves in PCL index order."""

    def __init__(self, max_points: int = 1 << 20, lib: Optional[C.CDLL] = None):
        self.lib = lib or load_library()
        self._h = C.c_void_p()
        _check(self.lib, self.lib.immesh_voxelgrid_create(max_points, C.byref(self._h)), "voxelgrid_create")
        self.leaf_too_small = False
        self.m = 0

    def close(self):
        if self._h:
            self.lib.immesh_voxelgrid_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def filter(self, pts, leaf: float, n=None, on_device=False, fetch=True):
        """pts: float32[n,3] host array, or a device pointer (int) with n and on_device=True.  Returns float32[m,3] (or m if not fetch)."""
        if on_device:
            ptr, cnt = C.c_void_p(int(pts)), int(n)
        else:
            a = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 3)
            ptr, cnt = a.ctypes.data_as(C.c_void_p), a.shape[0]
        out = np.zeros((max(cnt, 1), 3), dtype=np.float32) if fetch else None
        m, small = C.c_int(0), C.c_int(0)
        _check(self.lib, self.lib.immesh_voxelgrid_filter(self._h, ptr, cnt, 1 if on_device else 0, C.c_float(leaf),
                                                          out.ctypes.data_as(C.c_void_p) if fetch else None, C.byref(m), C.byref(small)), "voxelgrid_filter")
        self.m, self.leaf_too_small = m.value, bool(small.value)
        return out[:m.value].copy() if fetch else m.value

    def device_points(self) -> int:
        return int(self.lib.immesh_voxelgrid_device_points(self._h) or 0)

    @staticmethod
    def _records(pts, n, stride, on_device):
        """(pointer, n, stride) of point records: a float32[n, stride] host array, or an integer CUDA address with n and stride"""
        if on_device:
            return C.c_void_p(int(pts)), int(n), int(stride)
        a = np.ascontiguousarray(pts, dtype=np.float32)
        if a.ndim != 2:
            a = a.reshape(a.shape[0], -1)
        return a, a.shape[0], a.shape[1]

    def filter_i(self, pts, leaf: float, intensity_col: int, n=None, stride=None, on_device=False):
        """filter() on point records of `stride` floats (x y z, intensity in column intensity_col): float32[m, 4] x y z intensity"""
        a, cnt, stride = self._records(pts, n, stride, on_device)
        ptr = a if on_device else a.ctypes.data_as(C.c_void_p)
        out = np.zeros((max(cnt, 1), 4), dtype=np.float32)
        m, small = C.c_int(0), C.c_int(0)
        _check(self.lib, self.lib.immesh_voxelgrid_filter_i(self._h, ptr, cnt, stride, intensity_col, 1 if on_device else 0, C.c_float(leaf),
                                                            out.ctypes.data_as(C.c_void_p), C.byref(m), C.byref(small)), "voxelgrid_filter_i")
        self.m, self.leaf_too_small = m.value, bool(small.value)
        return out[:m.value].copy()

    def prepare(self, pts, calib_laser=False, fetch=True):
        """KITTI laser calibration (optional) + repack of a float32[n,3] or [n,4] cloud; the packed cloud stays on the device
        (input_points()).  Returns it as float32[n,3] when fetch."""
        a = np.ascontiguousarray(pts, dtype=np.float32)
        n, stride = a.shape[0], a.shape[1]
        out = np.zeros((n, 3), dtype=np.float32) if fetch else None
        _check(self.lib, self.lib.immesh_frontend_prepare(self._h, a.ctypes.data_as(C.c_void_p), n, stride, 0, 1 if calib_laser else 0,
                                                          out.ctypes.data_as(C.c_void_p) if fetch else None), "frontend_prepare")
        return out

    def input_points(self) -> int:
        return int(self.lib.immesh_voxelgrid_input_points(self._h) or 0)

    def input_count(self) -> int:
        """CUDA address of the device count of input_points() after a depth entry point (0 otherwise)"""
        return int(self.lib.immesh_voxelgrid_input_count(self._h) or 0)

    def prepare_depth(self, depth, cam: DepthCamera, cam_R=np.eye(3), cam_t=np.zeros(3), point_filter_num=1, blind=0.0, on_device=False, shape=None,
                      fmt="f32", pitch_bytes=0):
        """The localization's sensor-frame cloud of one depth image (immesh_frontend_prepare_depth; blocking): unprojected with the
        camera-to-sensor mount cam_R / cam_t, every point_filter_num-th valid sample kept, points closer than blind dropped.  It stays on
        the device (input_points(), input_count()); returned as float32[n][3] in ascending pixel order."""
        f, ptr, _keep = Mesh._depth_args(cam, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device)
        out = np.zeros((_sampled(f), 3), dtype=np.float32)   # the sampled pixels bound the count
        n = C.c_int(0)
        _check(self.lib, self.lib.immesh_frontend_prepare_depth(self._h, C.byref(f), ptr, 1 if on_device else 0, int(point_filter_num), float(blind),
                                                                out.ctypes.data_as(C.POINTER(C.c_float)), out.shape[0], C.byref(n)), "frontend_prepare_depth")
        return out[:n.value].copy()

    def step_async_depth(self, lio: "Lio", depth, cam: DepthCamera, leaf: float, cam_R=np.eye(3), cam_t=np.zeros(3), point_filter_num=1, blind=0.0,
                         dt=0.0, cov_gyr=0.1, cov_acc=0.1, on_device=False, shape=None, fmt="f32", pitch_bytes=0) -> int:
        """The queued depth chain (immesh_lio_step_async_depth): the image's filtered cloud -> VoxelGrid(leaf) -> lio.step_async, every
        count on the device.  Returns the sampled pixels, the n_max of Mesh.push_frame_from_lio_async_dev_n(lio, input_points(),
        n_max, input_count())."""
        f, ptr, _keep = Mesh._depth_args(cam, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device)
        _check(self.lib, self.lib.immesh_lio_step_async_depth(lio._h, self._h, C.byref(f), ptr, 1 if on_device else 0, int(point_filter_num), float(blind),
                                                              C.c_float(leaf), dt, cov_gyr, cov_acc), "lio_step_async_depth")
        lio._last_n = _sampled(f)
        return lio._last_n

    def step_async_raw(self, lio: "Lio", pts, leaf: float, dt=0.0, calib_laser=False, cov_gyr=0.1, cov_acc=0.1, n=None, stride=3, on_device=False):
        """The device-resident front-end chain: [calibration] -> VoxelGrid -> lio.step_async, no host round trip in between."""
        if on_device:
            ptr, cnt = C.c_void_p(int(pts)), int(n)
        else:
            a = np.ascontiguousarray(pts, dtype=np.float32)
            ptr, cnt, stride = a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1]
        _check(self.lib, self.lib.immesh_lio_step_async_raw(lio._h, self._h, ptr, cnt, stride, 1 if on_device else 0, 1 if calib_laser else 0, C.c_float(leaf),
                                                            dt, cov_gyr, cov_acc), "lio_step_async_raw")
        lio._last_n = cnt

    def step_async_raw_i(self, lio: "Lio", pts, leaf: float, intensity_col: int, dt=0.0, calib_laser=False, cov_gyr=0.1, cov_acc=0.1, n=None, stride=None,
                         on_device=False):
        """step_async_raw on point records of `stride` floats, the intensity (column intensity_col) kept for lio.frontend_cloud(self, ...)"""
        a, cnt, stride = self._records(pts, n, stride, on_device)
        ptr = a if on_device else a.ctypes.data_as(C.c_void_p)
        _check(self.lib, self.lib.immesh_lio_step_async_raw_i(lio._h, self._h, ptr, cnt, stride, intensity_col, 1 if on_device else 0, 1 if calib_laser else 0,
                                                              C.c_float(leaf), dt, cov_gyr, cov_acc), "lio_step_async_raw_i")
        lio._last_n = cnt

    def step_async_imu_i(self, lio: "Lio", imu_h: "Imu", batch, pts, lidar_beg_time: float, leaf: float, time_col: int, intensity_col: int,
                         calib_laser=False, n=None, stride=None, on_device=False) -> int:
        """step_async_imu on point records of `stride` floats (time stamp in time_col, intensity in intensity_col; pcl::PointXYZINormal:
        stride 12, time 9, intensity 8).  Returns the branch; after branch 3, lio.frontend_cloud(self, ...) publishes with intensity."""
        im = np.ascontiguousarray(batch, dtype=np.float64).reshape(-1, 7)
        a, cnt, stride = self._records(pts, n, stride, on_device)
        ptr = a if on_device else a.ctypes.data_as(C.c_void_p)
        br = C.c_int(0)
        _check(self.lib, self.lib.immesh_lio_step_async_imu_i(lio._h, imu_h._h, self._h, im.ctypes.data_as(C.POINTER(C.c_double)), im.shape[0], ptr, cnt,
                                                              stride, time_col, intensity_col, 1 if on_device else 0, lidar_beg_time, 1 if calib_laser else 0,
                                                              C.c_float(leaf), C.byref(br)), "lio_step_async_imu_i")
        lio._last_n = cnt
        return br.value

    def step_async_depth_imu(self, lio: "Lio", imu_h: "Imu", batch, depth, cam: DepthCamera, frame_time: float, leaf: float, point_filter_num=1, blind=0.0,
                             cam_R=np.eye(3), cam_t=np.zeros(3), on_device=False, shape=None, fmt="f32", pitch_bytes=0) -> int:
        """The IMU-enabled loop on one depth frame (immesh_lio_step_async_depth_imu): batch float64[n_imu,7] (stamp, gyr, acc), the image's
        cloud of prepare_depth with t = 0 at frame_time.  The drop rule and the branch are decided on the device; nothing is returned
        about them (Imu.depth_chain_state, the scan feed).  Returns the sampled pixels, the n_max of
        Mesh.push_frame_from_lio_async_dev_n(lio, input_points(), n_max, input_count())."""
        im = np.ascontiguousarray(batch, dtype=np.float64).reshape(-1, 7)
        f, ptr, _keep = Mesh._depth_args(cam, cam_R, cam_t, depth, shape, fmt, pitch_bytes, on_device)
        _check(self.lib, self.lib.immesh_lio_step_async_depth_imu(lio._h, imu_h._h, self._h, im.ctypes.data_as(C.POINTER(C.c_double)), im.shape[0], C.byref(f), ptr,
                                                                  1 if on_device else 0, int(point_filter_num), float(blind), float(frame_time), C.c_float(leaf)),
               "lio_step_async_depth_imu")
        lio._last_n = _sampled(f)
        return lio._last_n

    def step_async_imu(self, lio: "Lio", imu_h: "Imu", batch, pts, lidar_beg_time: float, leaf: float, calib_laser=False, n=None, on_device=False) -> int:
        """The IMU-enabled scan loop, one queued call per scan (immesh_lio_step_async_imu): batch float64[n_imu,7] (stamp, gyr, acc);
        pts float32[n,4] (x, y, z, curvature ms) host array, or an integer CUDA address with n when on_device.  Returns the branch taken:
        1 initialising, 2 map built, 3 localised and grown (then hand the frame to the mesher: input_points(), n, on_device)."""
        im = np.ascontiguousarray(batch, dtype=np.float64).reshape(-1, 7)
        if on_device:
            ptr, cnt = C.c_void_p(int(pts)), int(n)
        else:
            a = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 4)
            ptr, cnt = a.ctypes.data_as(C.c_void_p), a.shape[0]
        br = C.c_int(0)
        _check(self.lib, self.lib.immesh_lio_step_async_imu(lio._h, imu_h._h, self._h, im.ctypes.data_as(C.POINTER(C.c_double)), im.shape[0], ptr, cnt,
                                                            1 if on_device else 0, lidar_beg_time, 1 if calib_laser else 0, C.c_float(leaf), C.byref(br)),
               "lio_step_async_imu")
        lio._last_n = cnt
        return br.value


class Imu:
    """ImuProcess::UndistortPcl on the device (immesh_imu_*): forward propagation of the localization handle's state over the IMU
    samples of a scan + per-point motion compensation.  cfg: dict with cov_gyr, cov_acc, cov_bias_gyr, cov_bias_acc, mean_acc_norm,
    lid_R (3x3), lid_T."""

    def __init__(self, cfg: dict, max_points: int = 1 << 18, max_imu: int = 128, lib: Optional[C.CDLL] = None):
        self.lib = lib or load_library()
        c = _ImuCfg()
        for k in ("cov_gyr", "cov_acc", "cov_bias_gyr", "cov_bias_acc", "lid_T"):
            for i in range(3):
                getattr(c, k)[i] = float(np.asarray(cfg[k]).reshape(-1)[i])
        for i in range(9):
            c.lid_R[i] = float(np.asarray(cfg["lid_R"]).reshape(-1)[i])
        c.mean_acc_norm = float(cfg["mean_acc_norm"])
        c.max_points, c.max_imu = max_points, max_imu
        self._h = C.c_void_p()
        _check(self.lib, self.lib.immesh_imu_create(C.byref(c), C.byref(self._h)), "imu_create")

    def close(self):
        if self._h:
            self.lib.immesh_imu_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, last_imu7, last_lidar_end_time, last_update_time=0.0, acc_s_last=None, angvel_last=None):
        a = np.ascontiguousarray(last_imu7, dtype=np.float64)
        dp = C.POINTER(C.c_double)
        f = lambda v: None if v is None else np.ascontiguousarray(v, dtype=np.float64).ctypes.data_as(dp)  # noqa: E731
        _check(self.lib, self.lib.immesh_imu_reset(self._h, a.ctypes.data_as(dp), last_lidar_end_time, last_update_time, f(acc_s_last), f(angvel_last)), "imu_reset")

    def init_begin(self, max_ini_count: int = 3):
        """Enter the IMU initialisation phase of step_async_imu (first call: a fresh ImuProcess; later calls: the loop's reset)."""
        _check(self.lib, self.lib.immesh_imu_init_begin(self._h, max_ini_count), "imu_init_begin")

    def depth_chain_state(self) -> dict:
        """VoxelGrid.step_async_depth_imu's counters (immesh_imu_depth_chain_state; blocking)"""
        out = (C.c_int64 * 8)()
        _check(self.lib, self.lib.immesh_imu_depth_chain_state(self._h, out), "imu_depth_chain_state")
        keys = ("calls", "dropped", "branch1", "branch2", "branch3", "carried", "carry_overflows", "init_finished")
        return dict(zip(keys, (int(v) for v in out)))

    def undistort(self, lio: "Lio", imu, pts_xyzt, lidar_beg_time):
        """imu: float64[n_imu,7] (stamp, gyr, acc); pts_xyzt: float32[n,4] (x, y, z, curvature ms).  Returns the time-sorted, compensated cloud."""
        im = np.ascontiguousarray(imu, dtype=np.float64).reshape(-1, 7)
        p = np.ascontiguousarray(pts_xyzt, dtype=np.float32).reshape(-1, 4)
        out = np.zeros_like(p)
        _check(self.lib, self.lib.immesh_imu_undistort(self._h, lio._h, im.ctypes.data_as(C.POINTER(C.c_double)), im.shape[0], p.ctypes.data_as(C.c_void_p), p.shape[0], 0,
                                                       lidar_beg_time, out.ctypes.data_as(C.c_void_p)), "imu_undistort")
        return out

    def poses(self, cap=300):
        o = np.zeros((cap, 22))
        m = self.lib.immesh_imu_get_poses(self._h, o.ctypes.data_as(C.POINTER(C.c_double)), cap)
        return o[:m].copy()


def write_ply(path: str, vertices, triangles, flips=None, lib: Optional[C.CDLL] = None):
    """save_to_ply_file layout for a snapshot (vertices float32[nv,3], triangles int32[nt,3], flips int32[nt])."""
    lib = lib or load_library()
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(triangles, dtype=np.int32).reshape(-1, 3)
    fl = None if flips is None else np.ascontiguousarray(flips, dtype=np.int32)
    _check(lib, lib.immesh_write_ply(path.encode(), v.ctypes.data_as(C.POINTER(C.c_float)), v.shape[0], t.ctypes.data_as(C.POINTER(C.c_int32)),
                                     None if fl is None else fl.ctypes.data_as(C.POINTER(C.c_int32)), t.shape[0]), "write_ply")


def write_obj_textured(obj_path: str, mtl_path: str, vertices, triangles, flips, facet_cam, facet_uv, cam_wh, image_files, lib: Optional[C.CDLL] = None):
    """Wavefront OBJ + MTL of a texture selection: vertices float32[nv,3], triangles int32[nt,3] and flips int32[nt] (a snapshot),
    facet_cam / facet_uv (Mesh.texture_select's cam / uv), cam_wh int32[n_cams,2] the cameras' image sizes, image_files their paths
    as the MTL names them (map_Kd).  Texture coordinates are normalised: the images may be larger than the ones selected at."""
    lib = lib or load_library()
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(triangles, dtype=np.int32).reshape(-1, 3)
    fl = None if flips is None else np.ascontiguousarray(flips, dtype=np.int32).reshape(-1)
    fc = np.ascontiguousarray(facet_cam, dtype=np.int32).reshape(-1)
    uv = np.ascontiguousarray(facet_uv, dtype=np.float32).reshape(-1, 6)
    wh = np.ascontiguousarray(cam_wh, dtype=np.int32).reshape(-1, 2)
    files = (C.c_char_p * max(len(image_files), 1))(*[str(f).encode() for f in image_files])
    i32 = C.POINTER(C.c_int32)
    _check(lib, lib.immesh_write_obj_textured(obj_path.encode(), mtl_path.encode(), v.ctypes.data_as(C.POINTER(C.c_float)), v.shape[0], t.ctypes.data_as(i32),
                                              None if fl is None else fl.ctypes.data_as(i32), fc.ctypes.data_as(i32), uv.ctypes.data_as(C.POINTER(C.c_float)),
                                              t.shape[0], wh.ctypes.data_as(i32), files, len(image_files)), "write_obj_textured")


def write_png(path: str, rgb, lib: Optional[C.CDLL] = None):
    """an uncompressed 8-bit RGB PNG of rgb uint8[H, W, 3] (rows top to bottom), e.g. a page of Mesh.texture_bake"""
    lib = lib or load_library()
    a = np.ascontiguousarray(rgb, dtype=np.uint8)
    if a.ndim != 3 or a.shape[2] != 3:
        raise ValueError("write_png: rgb must be uint8 [H, W, 3]")
    _check(lib, lib.immesh_write_png(str(path).encode(), a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0]), "write_png")


def write_pcd(path: str, vertices, lib: Optional[C.CDLL] = None):
    lib = lib or load_library()
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    _check(lib, lib.immesh_write_pcd(path.encode(), v.ctypes.data_as(C.POINTER(C.c_float)), v.shape[0]), "write_pcd")


def kitti_pose_line(state, stamp: float, lib: Optional[C.CDLL] = None) -> str:
    lib = lib or load_library()
    s = np.ascontiguousarray(state, dtype=np.float64)
    buf = C.create_string_buffer(512)
    _check(lib, lib.immesh_kitti_pose_line(s.ctypes.data_as(C.POINTER(C.c_double)), stamp, buf, 512), "kitti_pose_line")
    return buf.value.decode()


def odometry_pose(state, lib: Optional[C.CDLL] = None) -> np.ndarray:
    """publish_odometry's pose of a state: float64[7] pos_end, then the quaternion x y z w of tf's setRPY(RotMtoEuler(rot_end))."""
    lib = lib or load_library()
    s = np.ascontiguousarray(state, dtype=np.float64)
    out = np.zeros(7)
    _check(lib, lib.immesh_odometry_pose(s.ctypes.data_as(C.POINTER(C.c_double)), out.ctypes.data_as(C.POINTER(C.c_double))), "odometry_pose")
    return out


def lio_state_line(state, t: float, lib: Optional[C.CDLL] = None) -> str:
    """dump_lio_state_to_log's line of a state at time t (ending in \\r\\n)."""
    lib = lib or load_library()
    s = np.ascontiguousarray(state, dtype=np.float64)
    buf = C.create_string_buffer(4096)
    _check(lib, lib.immesh_lio_state_line(s.ctypes.data_as(C.POINTER(C.c_double)), t, buf, 4096), "lio_state_line")
    return buf.value.decode()


def profile_enable(on: bool, lib: Optional[C.CDLL] = None):
    lib = lib or load_library()
    lib.immesh_profile_enable(int(on))   # 0 off, 1 per-kernel totals, 2 totals + launch timeline


def profile_reset(lib: Optional[C.CDLL] = None):
    (lib or load_library()).immesh_profile_reset()


def profile_report(lib: Optional[C.CDLL] = None) -> dict:
    """{kernel: (total_ms, launches)} measured with CUDA events on the launching stream."""
    lib = lib or load_library()
    n = lib.immesh_profile_report(None, 0)
    buf = C.create_string_buffer(n + 16)
    lib.immesh_profile_report(buf, n + 16)
    out = {}
    for line in buf.value.decode().splitlines():
        name, ms, cnt = line.rsplit(" ", 2)
        out[name.strip("()")] = (float(ms), int(cnt))
    return out


def profile_timeline(lib: Optional[C.CDLL] = None):
    """[(kernel, t0_ms, t1_ms)] of every launch since profile_enable(2)."""
    lib = lib or load_library()
    need = lib.immesh_profile_timeline(None, 0)
    buf = C.create_string_buffer(need + 16)
    lib.immesh_profile_timeline(buf, need + 16)
    out = []
    for line in buf.value.decode().splitlines():
        name, t0, t1 = line.rsplit(" ", 2)
        out.append((name.strip("()"), float(t0), float(t1)))
    return out


def launch_count(lib: Optional[C.CDLL] = None) -> int:
    return int((lib or load_library()).immesh_launch_count())


def graph_stats(lio: Optional["Lio"], mesh: Optional["Mesh"]) -> dict:
    """CUDA-graph replay accounting of the pipelined entry points, and the programmatic dependent-launch edges of each captured graph."""
    lib = (lio or mesh).lib
    h_lio, h_mesh = lio._h if lio else None, mesh._h if mesh else None
    out = (C.c_int64 * 6)()
    _check(lib, lib.immesh_graph_stats(h_lio, h_mesh, out), "graph_stats")
    keys = ("lio_captures", "lio_replays", "lio_failures", "mesh_captures", "mesh_replays", "mesh_failures")
    res = dict(zip(keys, [int(v) for v in out]))
    pdl = (C.c_int64 * 2)()
    _check(lib, lib.immesh_graph_pdl_edges(h_lio, h_mesh, pdl), "graph_pdl_edges")
    res["lio_pdl_edges"], res["mesh_pdl_edges"] = int(pdl[0]), int(pdl[1])
    return res


def host_wait_ms(lio: Optional["Lio"], mesh: Optional["Mesh"]):
    """Host milliseconds the enqueue calls spent blocked on busy staging slots since the last call: (lio, mesh)."""
    lib = (lio or mesh).lib
    out = (C.c_double * 2)()
    _check(lib, lib.immesh_host_wait_ms(lio._h if lio else None, mesh._h if mesh else None, out), "host_wait_ms")
    return float(out[0]), float(out[1])


def pipeline_mark_begin(lio: Lio):
    _check(lio.lib, lio.lib.immesh_pipeline_mark_begin(lio._h), "pipeline_mark_begin")


def pipeline_mark_end(lio: Lio, mesh: Mesh) -> float:
    ms = C.c_double(0)
    _check(lio.lib, lio.lib.immesh_pipeline_mark_end(lio._h, mesh._h, C.byref(ms)), "pipeline_mark_end")
    return ms.value


def comm_unique_id(lib: Optional[C.CDLL] = None) -> bytes:
    lib = lib or load_library()
    buf = C.create_string_buffer(128)
    _check(lib, lib.immesh_comm_unique_id(buf), "comm_unique_id")
    return buf.raw
