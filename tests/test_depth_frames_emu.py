"""CPU tier: the depth frame's unprojection and append-step bodies (immesh_b200/csrc/depth_frame.cuh), run by the host emulation
(tests/depth_frame/emu_depth_frame.cpp) with the kernels' block compaction, against the numpy restatement of tests/depth_reference.py:
both formats, both kinds, strides 1 / 2 / 3, a padded pitch and the edge values, bit for bit; and the device's step / m rule against
the host rule of immesh_mesh_push_frame around multiples of appending_pts_frame."""
import ctypes as C

import numpy as np
import pytest

import depth_reference as dr


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_depth_frame())
    L.emu_depth_frame.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p]
    L.emu_depth_frame.restype = C.c_int
    L.emu_append_dims.argtypes = [C.c_int, C.c_int, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_points(lib, img, cam, R, t, append_target=10000, pad=0):
    """the emulation on img, its rows `pad` bytes longer than the pixels"""
    h, w = img.shape
    rowb = w * img.itemsize + pad
    buf = np.zeros(h * rowb, dtype=np.uint8)
    for v in range(h):
        buf[v * rowb:v * rowb + w * img.itemsize] = np.frombuffer(img[v].tobytes(), dtype=np.uint8)
    ns = -(-h // cam.stride) * -(-w // cam.stride)
    pts = np.zeros((max(ns, 1), 3), dtype=np.float32)
    pix = np.zeros(max(ns, 1), dtype=np.int32)
    dims = np.zeros(4, dtype=np.int64)
    n = lib.emu_depth_frame(_p(buf), rowb, w, h, dr.FORMATS["u16" if img.dtype == np.uint16 else "f32"], dr.KINDS[cam.kind], cam.stride,
                            _p(dr.cam_array(cam, R, t)), append_target, _p(pts), _p(pix), _p(dims))
    return pts[:n], pix[:n], dims


@pytest.mark.parametrize("fmt", ["f32", "u16"])
@pytest.mark.parametrize("kind", ["planar", "range"])
@pytest.mark.parametrize("stride,pad", [(1, 0), (2, 0), (3, 0), (1, 12), (3, 36)])
def test_points_bit_exact(lib, fmt, kind, stride, pad):
    w, h = 97, 61   # neither a multiple of the strides nor of a warp
    cam = dr.camera(w, h, kind=kind, stride=stride, z_min=0.5, z_max=40.0, depth_scale=0.001)
    rng = np.random.default_rng(stride * 10 + pad)
    for k in (0, 17):
        R, t = dr.camera_pose(k)
        img = dr.inject_edges(dr.render(cam, w, h, R, t, kind=kind, fmt=fmt), cam, rng)
        pts, pix, dims = emu_points(lib, img, cam, R, t, pad=pad)
        ref, rpix = dr.unproject(img, cam, R, t)
        assert pts.shape[0] > 100 and pts.shape[0] < img.size
        np.testing.assert_array_equal(pix, rpix)
        assert pts.tobytes() == ref.tobytes()
        assert dims[0] == ref.shape[0]


def test_edge_values(lib):
    """each edge value on its own: which raw values are samples, with the z range closed at both ends"""
    cam = dr.camera(4, 1, z_min=0.5, z_max=40.0, depth_scale=0.25)
    R, t = np.eye(3), np.zeros(3)
    f32 = np.array([[np.nan, np.inf, -np.inf, 0.0]], dtype=np.float32)
    assert emu_points(lib, f32, cam, R, t)[0].shape[0] == 0
    f32 = np.array([[0.5, 40.0, np.nextafter(np.float32(0.5), 0, dtype=np.float32), np.nextafter(np.float32(40.0), 100, dtype=np.float32)]],
                   dtype=np.float32)
    _, pix, _ = emu_points(lib, f32, cam, R, t)
    np.testing.assert_array_equal(pix, [0, 1])
    u16 = np.array([[0, 2, 160, 65535]], dtype=np.uint16)   # 0: invalid; 0.5 m and 40 m: the range's ends; 16383.75 m: beyond it
    pts, pix, _ = emu_points(lib, u16, cam, R, t)
    np.testing.assert_array_equal(pix, [1, 2])
    ref, _ = dr.unproject(u16, cam, R, t)
    assert pts.tobytes() == ref.tobytes()


def test_pixel_order_across_blocks(lib):
    """more than one DF_BLOCK of samples: the points stay in ascending pixel order across the blocks' offsets"""
    w, h = 320, 240
    cam = dr.camera(w, h, z_min=0.5, z_max=40.0)
    R, t = dr.camera_pose(5)
    img = dr.inject_edges(dr.render(cam, w, h, R, t), cam, np.random.default_rng(3))
    pts, pix, _ = emu_points(lib, img, cam, R, t)
    ref, rpix = dr.unproject(img, cam, R, t)
    assert np.all(np.diff(pix) > 0) and pts.shape[0] > 4 * 1024
    np.testing.assert_array_equal(pix, rpix)
    assert pts.tobytes() == ref.tobytes()


@pytest.mark.parametrize("append_target", [1, 7, 1000, 10000])
def test_append_rule(lib, append_target):
    A = append_target
    ns = {0, 1, 2, 3}
    for j in range(0, 8):
        for d in (-2, -1, 0, 1, 2):
            n = j * A + d
            ns.update({n, n + A // 2, n + (A + 1) // 2})
    out = np.zeros(4, dtype=np.int64)
    for n in sorted(x for x in ns if x >= 0):
        lib.emu_append_dims(n, A, _p(out))
        step, m = dr.append_dims(n, A)
        assert (out[0], out[1]) == (step, m), n
        assert out[2] + 1 >= 2 * max(m, 1) and (out[2] + 1) & out[2] == 0 and (out[2] + 1) // 2 < 2 * max(m, 1), n
        # the host's bound of a depth frame's candidates covers every count up to the sampled pixels
        assert out[3] >= max(dr.append_dims(k, A)[1] for k in range(0, n + 1, max(1, n // 200))), n
        assert out[3] >= m
