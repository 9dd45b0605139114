"""CPU tier: the localization's depth filter (immesh_b200/csrc/depth_frame.cuh: depth_point, depth_keep), run by the host emulation
(tests/depth_lio/emu_depth_lio.cpp) with the front-end kernels' multi-pass block compaction, against the numpy restatement of
tests/depth_lio_reference.py, bit for bit: both formats, both kinds, strides 1 and 3, point_filter_num 1 / 3 / 10, blind 0 / 0.5 / 1.0,
the edge values, a point exactly at blind, and blocks that split a decimation period."""
import ctypes as C

import numpy as np
import pytest

import depth_lio_reference as dlr
import depth_reference as dr

DF_BLOCK = 1024   # depth_kernels.cuh


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_depth_lio())
    L.emu_depth_lio.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_int,
                                C.c_void_p, C.c_void_p]
    L.emu_depth_lio.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_cloud(lib, img, cam, R, t, point_filter_num, blind, block=DF_BLOCK):
    h, w = img.shape
    img = np.ascontiguousarray(img)
    ns = -(-h // cam.stride) * -(-w // cam.stride)
    pts = np.zeros((ns, 3), dtype=np.float32)
    pix = np.zeros(ns, dtype=np.int32)
    n = lib.emu_depth_lio(_p(img), w * img.itemsize, w, h, dr.FORMATS["u16" if img.dtype == np.uint16 else "f32"], dr.KINDS[cam.kind], cam.stride,
                          _p(dr.cam_array(cam, R, t)), point_filter_num, blind, block, _p(pts), _p(pix))
    return pts[:n], pix[:n]


@pytest.mark.parametrize("fmt", ["f32", "u16"])
@pytest.mark.parametrize("kind", ["planar", "range"])
@pytest.mark.parametrize("stride", [1, 3])
@pytest.mark.parametrize("point_filter_num", [1, 3, 10])
@pytest.mark.parametrize("blind", [0.0, 0.5, 1.0])
def test_cloud_bit_exact(lib, fmt, kind, stride, point_filter_num, blind):
    w, h = 131, 97   # more than one block of sampled pixels at stride 1; 1024 is not a multiple of 3 or 10
    cam = dr.camera(w, h, kind=kind, stride=stride, z_min=0.2, z_max=40.0, depth_scale=0.001)
    rng = np.random.default_rng(stride * 100 + point_filter_num * 10 + int(blind * 2))
    for k, (R, t) in enumerate([(np.eye(3), np.zeros(3)), (dlr.SENSOR_FROM_CAM, np.array([0.05, -0.02, 0.1]))]):
        Rw, tw = dr.camera_pose(7 * k)
        img = dr.inject_edges(dr.render(cam, w, h, Rw, tw, kind=kind, fmt=fmt), cam, rng)
        if k == 0:   # some returns inside blind (walls are metres away in the synth scene)
            img.reshape(-1)[rng.permutation(img.size)[:img.size // 8]] = np.float32(0.6) if fmt == "f32" else 600
        ref, rpix = dlr.sensor_cloud(img, cam, R, t, point_filter_num, blind)
        for block in (DF_BLOCK, 7):   # 7: blocks end inside decimation periods everywhere
            pts, pix = emu_cloud(lib, img, cam, R, t, point_filter_num, blind, block)
            assert pts.shape[0] > 10
            np.testing.assert_array_equal(pix, rpix)
            assert pts.tobytes() == ref.tobytes()
        if point_filter_num == 1 and blind == 0.0:   # no filter: the cloud of every valid sample
            assert ref.shape[0] == dr.unproject(img, cam, R, t)[0].shape[0]


def test_point_at_blind_is_kept(lib):
    w, h = 33, 21   # the principal point (16, 10) is a pixel: its planar depth d gives the point (0, 0, d), r = d * d exactly
    cam = dr.camera(w, h, kind="planar", z_min=0.1, z_max=10.0)
    img = np.full((h, w), 5.0, dtype=np.float32)
    img[10, 16] = 2.0
    centre = 10 * w + 16
    for blind, kept in ((2.0, True), (np.nextafter(2.0, 3.0), False), (np.nextafter(2.0, 1.0), True)):
        ref, rpix = dlr.sensor_cloud(img, cam, point_filter_num=1, blind=blind)
        pts, pix = emu_cloud(lib, img, cam, np.eye(3), np.zeros(3), 1, blind)
        assert pts.tobytes() == ref.tobytes() and np.array_equal(pix, rpix)
        assert (centre in pix) == kept
        assert pts.shape[0] == (w * h - 1) + (1 if kept else 0)


def test_decimation_counts_valid_samples_only(lib):
    """i numbers the valid samples, not the pixels: invalid pixels between them do not shift the decimation"""
    w, h = 50, 40
    cam = dr.camera(w, h, kind="planar", z_min=0.1, z_max=10.0)
    img = np.full((h, w), 3.0, dtype=np.float32)
    img.reshape(-1)[::4] = np.nan
    pts, pix = emu_cloud(lib, img, cam, np.eye(3), np.zeros(3), 3, 0.0, block=5)
    valid = np.flatnonzero(np.isfinite(img.reshape(-1)))
    np.testing.assert_array_equal(pix, valid[::3])
