"""Shared pieces of the local-map tests: a numpy float32 restatement of laser_map_fov_segment (src/voxel_mapping_common.cpp:214-288),
the oracle extended by the local map (tests/local_map/orc_local_map.cpp), and a stream driver that runs the library (or its host
emulation) and the oracle side by side with the same eviction."""
import ctypes as C

import numpy as np

from immesh_b200 import build
from oracle_api import OracleLio

SHAPE_COLS = slice(0, 11)
f32 = np.float32


def fov_segment(cube_len, det, mov, placed, box, pos):
    """The reference's rule in its own types: returns (placed, new box float32[6], removal boxes float32[k, 6])."""
    pos = np.asarray(pos, dtype=np.float64)
    det, mov = f32(det), f32(mov)
    box = np.array(box, dtype=f32)
    if not placed:
        return True, np.concatenate([(pos - cube_len / 2.0).astype(f32), (pos + cube_len / 2.0).astype(f32)]), np.zeros((0, 6), f32)
    thr = f32(mov * det)
    d0 = np.abs(pos - box[:3].astype(np.float64)).astype(f32)
    d1 = np.abs(pos - box[3:].astype(np.float64)).astype(f32)
    if not ((d0 <= thr) | (d1 <= thr)).any():
        return True, box, np.zeros((0, 6), f32)
    a = (cube_len - 2.0 * float(mov) * float(det)) * 0.5 * 0.9
    b = float(f32(det * f32(mov - f32(1))))
    md = f32(max(a, b))
    new, rm = box.copy(), []
    for i in range(3):
        tmp = box.copy()
        if d0[i] <= thr:
            new[3 + i] = f32(new[3 + i] - md)
            new[i] = f32(new[i] - md)
            tmp[i] = f32(box[3 + i] - md)
            rm.append(tmp)
        elif d1[i] <= thr:
            new[3 + i] = f32(new[3 + i] + md)
            new[i] = f32(new[i] + md)
            tmp[3 + i] = f32(box[i] + md)
            rm.append(tmp)
    return True, new, np.array(rm, dtype=f32).reshape(-1, 6)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


_orc = None


def oracle_lib():
    global _orc
    if _orc is None:
        L = C.CDLL(build.build_local_map()[1])
        L.orc_lio_create.restype = C.c_void_p
        L.orc_lio_dump_map.restype = C.c_long
        L.orc_lio_num_root_voxels.restype = C.c_long
        L.orc_lio_predict.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        L.orc_lm_set.argtypes = [C.c_void_p, C.c_double, C.c_float, C.c_float]
        L.orc_lm_segment.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_lio_evict_boxes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.orc_lio_evict_boxes.restype = C.c_long
        L.orc_lm_rule.argtypes = [C.c_double, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _orc = L
    return _orc


class OracleLocalMap(OracleLio):
    """OracleLio on the extended oracle: the same tree, plus laser_map_fov_segment and the deletion of its boxes."""

    def __init__(self, cfg):
        L = oracle_lib()
        cd = np.array([cfg.voxel_size, cfg.min_eigen_value, cfg.dept_err, cfg.beam_err, *cfg.ext_R, *cfg.ext_T], dtype=np.float64)
        ci = np.array([cfg.max_layer, *cfg.layer_init_size, cfg.max_points_size, cfg.max_iteration, cfg.calib_laser, 0, 1, 0, 0], dtype=np.int32)
        self.h = C.c_void_p(L.orc_lio_create(_p(cd), _p(ci)))
        self.L = L

    def local_map(self, cube_len, det_range=300.0, mov_threshold=1.5):
        self.L.orc_lm_set(self.h, cube_len, det_range, mov_threshold)

    def segment(self):
        """the rule at the current pos_end and the deletion: (box, removal boxes, roots evicted)"""
        box, rm, ev = np.zeros(6, f32), np.zeros((3, 6), f32), C.c_long(0)
        k = self.L.orc_lm_segment(self.h, _p(box), _p(rm), C.byref(ev))
        return box, rm[:k].copy(), ev.value

    def evict_boxes(self, boxes):
        a = np.ascontiguousarray(np.asarray(boxes, dtype=f32).reshape(-1, 6))
        return self.L.orc_lio_evict_boxes(self.h, _p(a), a.shape[0])

    def num_roots(self):
        return self.L.orc_lio_num_root_voxels(self.h)


def oracle_rule(cube_len, det, mov, placed, box, pos):
    L = oracle_lib()
    pl = C.c_int(1 if placed else 0)
    b = np.array(box, dtype=f32)
    p = np.asarray(pos, dtype=np.float64)
    rm = np.zeros((3, 6), f32)
    k = L.orc_lm_rule(cube_len, det, mov, C.byref(pl), _p(b), _p(p), _p(rm))
    return bool(pl.value), b, rm[:k].copy()


def root_centres(dump):
    """(key xyz int64[m, 3], centre float64[m, 3]) of the root rows of a canonical dump (path 0)"""
    roots = dump[dump[:, 3] == 0]
    return roots[:, 0:3].astype(np.int64), roots[:, 21:24]


def in_boxes(c, boxes):
    boxes = np.asarray(boxes, dtype=f32).reshape(-1, 6).astype(np.float64)
    hit = np.zeros(c.shape[0], dtype=bool)
    for b in boxes:
        hit |= np.all((b[:3] <= c) & (b[3:] > c), axis=1)
    return hit
