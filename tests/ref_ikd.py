"""ctypes wrapper over oracle/_ref/libref_ikd.so -- the REFERENCE's own ikd-Tree (include/ikd-Tree/ikd_Tree.{h,cpp}) compiled
unmodified by oracle/Makefile.ref.  Test infrastructure only.  The library is (re)built where the reference checkout is
present (immesh_b200.build.build_ref); elsewhere a library built earlier is used.  `available()` is False when neither exists
(tests then skip and the committed fixtures under tests/golden/ carry the pin)."""
import ctypes as C
import os

import numpy as np

from immesh_b200 import build as _build

_SO = _build.REF_IKD
_lib = None


def build():
    _build.build_ref()
    return os.path.exists(_SO)


def available():
    try:
        return build()
    except Exception:
        return os.path.exists(_SO)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libref_ikd.so is not built")
        L = C.CDLL(_SO)
        L.ref_ikd_create.restype = C.c_void_p
        L.ref_ikd_destroy.argtypes = [C.c_void_p]
        L.ref_ikd_add.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int64]
        L.ref_ikd_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_ikd_size.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class RefIkdTree:
    """KD_TREE<ikdTree_PointType> driven like Global_map does: Add_Point one vertex at a time, Nearest_Search."""

    def __init__(self):
        self.L = lib()
        self.h = C.c_void_p(self.L.ref_ikd_create())
        self.n = 0

    def __del__(self):
        try:
            self.L.ref_ikd_destroy(self.h)
        except Exception:
            pass

    def add(self, xyz):
        a = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        self.L.ref_ikd_add(self.h, a.ctypes.data_as(C.c_void_p), a.shape[0], self.n)
        self.n += a.shape[0]

    def knn(self, q, k, max_dist=float("inf")):
        a = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 3)
        idx = np.zeros((a.shape[0], k), dtype=np.int64)
        d2 = np.zeros((a.shape[0], k), dtype=np.float32)
        cnt = np.zeros(a.shape[0], dtype=np.int32)
        self.L.ref_ikd_knn(self.h, a.ctypes.data_as(C.c_void_p), a.shape[0], k, max_dist, idx.ctypes.data_as(C.c_void_p),
                           d2.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p))
        return idx, d2, cnt


def same_knn(idx_a, d2_a, idx_b, d2_b):
    """kNN equality up to the order inside groups of EXACTLY equal float distances (tie order in the ikd-Tree depends on the
    tree shape, ikd_Tree.cpp:1123; ours is defined as lower id first)."""
    if not np.array_equal(d2_a, d2_b):
        return False
    for r in range(idx_a.shape[0]):
        if np.array_equal(idx_a[r], idx_b[r]):
            continue
        d = d2_a[r]
        for v in np.unique(d):
            m = d == v
            if sorted(idx_a[r][m].tolist()) != sorted(idx_b[r][m].tolist()):
                return False
    return True
