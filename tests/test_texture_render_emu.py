"""CPU tier of the textured render (immesh_mesh_render_textured): the device bodies and argument check (immesh_b200/csrc/
texture_render_core.cuh) run by the host emulation (tests/texture_render/emu_texture_render.cpp) in the device call's orchestration,
byte-equal to the numpy restatement (tests/texture_render_reference.py): one facet, both flips, untextured winners and empty pixels,
shared edges and equal-depth ties, images larger and smaller than the selection camera, uv beyond the image border, several host-image
batches (one image per batch among them), NULL images for cameras the view does not sample, the query, a truth image with zero and
non-zero error, overflowing bins, and random meshes and rows; then the error contract."""
import ctypes as C

import numpy as np
import pytest

from texture_reference import camera
from texture_render_reference import render_textured as ref_render

W, H = 48, 40
K = (40.0, 40.0, 23.5, 19.5)


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_texture_render())
    L.emu_texture_render_error.restype = C.c_char_p
    vp = C.c_void_p
    L.emu_texture_render.argtypes = [vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, C.c_int64, vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_longlong, C.c_int,
                                     vp, vp, vp, vp, vp, vp]
    return L


def view_cam(w=W, h=H, k=K):
    return camera(w, h, k, np.eye(3), np.zeros(3))   # OpenCV axes: the world's z is forward, x right, y down


def emu(lib, view, sel_wh, images, cam, uv, verts, tris, flips, truth=None, max_image_bytes=0, on_device=0, bin_cap=1 << 40, shard_n=1, n_facets=None,
        z_near=0.1, z_far=1000.0, untextured=(128, 128, 128), background=(0, 0, 0), positions=0, rgb=True):
    """(rc, dict(rgb, depth, facet, needed, counts, batches)) of the emulation; images None: the query"""
    from immesh_b200 import api
    vw, _ = api.texture_cameras([(view["width"], view["height"], view["K"], view["R"], view["t"])])
    arr, n_cams = api.texture_cameras([(w, h, K, np.eye(3), np.zeros(3)) for w, h in sel_wh])
    keep = []
    imgs = None
    if images is not None:
        imgs, _, keep = api.texture_images(images)
    tr = None
    if truth is not None:
        t_arr, _, tk = api.texture_images([truth])
        keep += tk
        tr = C.cast(t_arr, C.c_void_p)
    cfg = api._TexViewCfg(z_near, z_far, positions, (C.c_uint8 * 3)(*untextured), (C.c_uint8 * 3)(*background), max_image_bytes)
    cam = np.ascontiguousarray(cam, np.int32).reshape(-1)
    uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 6)
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    flips = np.ascontiguousarray(flips, np.int32).reshape(-1)
    h, w = view["height"], view["width"]
    out = dict(rgb=np.full((h, w, 3), 77, np.uint8) if rgb else None, depth=np.full((h, w), 7.0, np.float32), facet=np.full((h, w), 9, np.int32),
               needed=np.full(n_cams, 5, np.uint8), counts=np.full(8, -3, np.int64))
    nb = C.c_int(-1)
    rc = lib.emu_texture_render(C.cast(vw, C.c_void_p), C.addressof(cfg), C.cast(arr, C.c_void_p), n_cams, None if imgs is None else C.cast(imgs, C.c_void_p),
                                on_device, cam.ctypes.data, uv.ctypes.data, len(cam) if n_facets is None else n_facets, tr, verts.ctypes.data, None, None,
                                len(verts), tris.ctypes.data, flips.ctypes.data, len(tris), bin_cap, shard_n,
                                None if out["rgb"] is None else out["rgb"].ctypes.data, out["depth"].ctypes.data, out["facet"].ctypes.data,
                                out["needed"].ctypes.data, out["counts"].ctypes.data, C.addressof(nb))
    del keep
    out["batches"] = nb.value
    return rc, out


def check(lib, view, sel_wh, images, cam, uv, verts, tris, flips, truth=None, **kw):
    """the emulation equals the restatement byte for byte; returns the emulation's result"""
    kw.setdefault("rgb", images is not None)
    rc, got = emu(lib, view, sel_wh, images, cam, uv, verts, tris, flips, truth=truth, **kw)
    assert rc == 0, lib.emu_texture_render_error()
    keys = {k: kw[k] for k in ("z_near", "z_far", "untextured", "background") if k in kw}
    ref = ref_render(view, sel_wh, images, cam, uv, verts, tris, flips, truth=truth, **keys)
    assert np.array_equal(got["depth"].view(np.uint32), ref["depth"].view(np.uint32))
    assert np.array_equal(got["facet"], ref["facet"])
    assert np.array_equal(got["needed"], ref["needed"])
    assert got["counts"].tolist() == ref["counts"].tolist(), (got["counts"], ref["counts"])
    if images is not None:
        assert np.array_equal(got["rgb"], ref["rgb"]), int((got["rgb"] != ref["rgb"]).any(axis=-1).sum())
    return got


def ramp(w, h, k=0):
    img = np.zeros((h, w, 3), np.uint8)
    img[..., 0] = np.round(np.arange(w) * 255.0 / max(w - 1, 1))[None, :]
    img[..., 1] = np.round(np.arange(h) * 255.0 / max(h - 1, 1))[:, None]
    img[..., 2] = (40 * k + 20) % 256
    return img


def project(verts, tri, wh=(W, H), k=K):
    """uv [6] of a triangle's corners in a camera at the origin looking down +z"""
    p = np.asarray(verts, np.float64)[list(tri)]
    return np.stack([k[0] * p[:, 0] / p[:, 2] + k[2], k[1] * p[:, 1] / p[:, 2] + k[3]], axis=1).reshape(-1).astype(np.float32)


def face_uv(verts, tri, flip):
    a, b, c = tri
    return project(verts, (a, b, c) if flip else (a, c, b))


QUAD = np.array([[-1.0, -1.0, 4.0], [1.0, -1.0, 4.5], [1.0, 1.0, 5.0], [-1.0, 1.0, 4.5]], np.float32)


def test_one_facet_both_flips(lib):
    rng = np.random.default_rng(1)
    tri = (0, 1, 2)
    for flip in (0, 1):
        uv = face_uv(QUAD, tri, flip)
        img = rng.integers(0, 256, (H, W, 3), np.uint8)
        g = check(lib, view_cam(), [(W, H)], [img], [0], [uv], QUAD, [tri], [flip])
        assert g["counts"][0] > 100 and g["counts"][3] == 1
        # a facet facing the camera (constant depth) textured from a ramp taken at the view itself: the render is the ramp within the
        # rounding (on tilted facets the perspective-correct rule legitimately departs from the projective mapping)
        flat = QUAD.copy()
        flat[:, 2] = 4.5
        g = check(lib, view_cam(), [(W, H)], [ramp(W, H)], [0], [face_uv(flat, tri, flip)], flat, [tri], [flip])
        m = g["facet"] == 0
        assert np.abs(g["rgb"][m].astype(int) - ramp(W, H)[m].astype(int)).max() <= 1
    # swapping the flip without permuting the uv gives another image: the weights follow the face order
    uv = face_uv(QUAD, tri, 1)
    a = check(lib, view_cam(), [(W, H)], [ramp(W, H)], [0], [uv], QUAD, [tri], [1])
    b = check(lib, view_cam(), [(W, H)], [ramp(W, H)], [0], [uv], QUAD, [tri], [0])
    assert not np.array_equal(a["rgb"], b["rgb"])


def test_untextured_empty_shared_edges_and_ties(lib):
    verts = np.concatenate([QUAD, QUAD[[0, 1, 2]]])   # vertices 4, 5, 6 repeat 0, 1, 2: an exact tie with triangle (0, 1, 2)
    tris = [(0, 1, 2), (0, 2, 3), (4, 5, 6)]
    flips = [1, 0, 1]
    uv = [face_uv(verts, t, f) for t, f in zip(tris, flips)]
    for cams in ([0, -1, 1], [-1, 0, 0], [1, 1, -1]):
        g = check(lib, view_cam(), [(W, H), (W, H)], [ramp(W, H, 0), ramp(W, H, 1)], cams, uv, verts, tris, flips, untextured=(1, 2, 3), background=(9, 8, 7))
        assert (g["facet"] != 2).all(), "the lower triple wins an exact tie"
        assert g["counts"][2] > 0 and g["counts"][0] + g["counts"][1] + g["counts"][2] == W * H


def test_image_sizes_and_border(lib):
    rng = np.random.default_rng(2)
    tris, flips = [(0, 1, 2), (0, 2, 3)], [1, 1]
    uv = np.stack([face_uv(QUAD, t, f) for t, f in zip(tris, flips)])
    for scale in (0.5, 1.0, 2.0, 3.0):
        w, h = max(1, int(W * scale)), max(1, int(H * scale))
        imgs = [rng.integers(0, 256, (h, w, 3), np.uint8), ramp(w, h)]
        check(lib, view_cam(), [(W, H), (W, H)], imgs, [0, 1], uv, QUAD, tris, flips)
    # uv far beyond the image on every side: the clamp to the edge
    wild = uv.copy()
    wild[0] = [-50.0, -40.0, 300.0, -10.0, 20.0, 500.0]
    wild[1] = [-1e6, 1e6, 1e6, -1e6, 0.0, 0.0]
    check(lib, view_cam(), [(W, H)], [rng.integers(0, 256, (H, W, 3), np.uint8)], [0, 0], wild, QUAD, tris, flips)
    # a 1 x 1 image
    check(lib, view_cam(), [(W, H)], [np.full((1, 1, 3), 200, np.uint8)], [0, 0], uv, QUAD, tris, flips)


def strip(n_cams, seed):
    """a strip of 2 n_cams columns of two facets across the view, two neighbouring columns per camera in camera order"""
    rng = np.random.default_rng(seed)
    n = 2 * n_cams
    xs = np.linspace(-1.2, 1.2, n + 1)
    verts = np.array([[x, y, 5.0 + 0.1 * rng.random()] for x in xs for y in (-1.0, 1.0)], np.float32)
    tris, flips, cam = [], [], []
    for i in range(n):
        a, b, c, d = 2 * i, 2 * i + 1, 2 * i + 2, 2 * i + 3
        for t in ((a, b, c), (b, c, d)):
            f = int(rng.integers(0, 2))
            tris.append(t)
            flips.append(f)
            cam.append(i * n_cams // n)
    uv = np.stack([face_uv(verts, t, f) for t, f in zip(tris, flips)])
    return verts, tris, flips, cam, uv


def test_batches_and_null_images(lib):
    rng = np.random.default_rng(3)
    n_cams = 6
    verts, tris, flips, cam, uv = strip(n_cams, 3)
    sizes = [(W + 2 * k, H + k) for k in range(n_cams)]   # no two images fit in the largest one's bytes
    imgs = [rng.integers(0, 256, (h, w, 3), np.uint8) for w, h in sizes]
    sel = [(W, H)] * n_cams
    one = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips)
    assert one["batches"] == 1 and one["counts"][3] == n_cams
    big = max(im.nbytes for im in imgs)
    each = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, max_image_bytes=big)
    assert each["batches"] == n_cams, "one image per batch"
    some = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, max_image_bytes=2 * big + 1)
    assert 1 < some["batches"] < n_cams
    dev = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, on_device=1)
    assert dev["batches"] == 0
    for g in (each, some, dev):
        assert np.array_equal(g["rgb"], one["rgb"])
    # padded rows give the same bytes
    padded = []
    for im in imgs:
        buf = np.zeros((im.shape[0], im.shape[1] + 3, 3), np.uint8)
        buf[:, :im.shape[1]] = im
        padded.append(buf[:, :im.shape[1]])
    assert np.array_equal(check(lib, view_cam(), sel, padded, cam, uv, verts, tris, flips, max_image_bytes=big)["rgb"], one["rgb"])
    # cameras used by rows but not sampled by a narrower view may be NULL; their rows are untouched
    narrow = camera(W, H, (200.0, 200.0, 23.5, 19.5), np.eye(3), np.zeros(3))
    q = check(lib, narrow, sel, None, cam, uv, verts, tris, flips)
    assert 0 < q["needed"].sum() < n_cams
    only = [im if q["needed"][k] else None for k, im in enumerate(imgs)]
    g = check(lib, narrow, sel, only, cam, uv, verts, tris, flips, max_image_bytes=big)
    assert g["batches"] == int(q["needed"].sum())
    # a NULL image for a camera the view samples is refused, nothing written
    k = int(np.nonzero(q["needed"])[0][0])
    bad = list(only)
    bad[k] = None
    rc, out = emu(lib, narrow, sel, bad, cam, uv, verts, tris, flips)
    assert rc == -1 and b"sampled by the view" in lib.emu_texture_render_error()
    assert (out["rgb"] == 77).all() and (out["depth"] == 7.0).all() and (out["facet"] == 9).all() and (out["needed"] == 5).all() and (out["counts"] == -3).all()


def test_query_and_truth(lib):
    rng = np.random.default_rng(4)
    verts, tris, flips, cam, uv = strip(3, 4)
    cam[1] = -1
    sel = [(W, H)] * 3
    imgs = [rng.integers(0, 256, (H, W, 3), np.uint8) for _ in range(3)]
    full = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips)
    q = check(lib, view_cam(), sel, None, cam, uv, verts, tris, flips)
    for key in ("depth", "facet", "needed"):
        assert np.array_equal(q[key], full[key])
    assert q["counts"].tolist() == full["counts"].tolist()
    # truth = the render itself: zero error; another image: the restatement's exact sums
    z = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, truth=full["rgb"].copy())
    assert z["counts"][4:].tolist() == [0, 0, 0, 0]
    other = rng.integers(0, 256, (H, W, 3), np.uint8)
    nz = check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, truth=other)
    assert nz["counts"][4:].min() > 0
    check(lib, view_cam(), sel, imgs, cam, uv, verts, tris, flips, truth=other, on_device=1, max_image_bytes=1)


@pytest.mark.parametrize("seed", range(6))
def test_random_meshes_and_rows(lib, seed):
    rng = np.random.default_rng(100 + seed)
    nv, nt, n_cams = 60, 120, 4
    verts = np.stack([rng.uniform(-2, 2, nv), rng.uniform(-1.5, 1.5, nv), rng.uniform(3, 8, nv)], axis=1).astype(np.float32)
    tris = np.sort(np.stack([rng.choice(nv, 3, replace=False) for _ in range(nt)]), axis=1)
    flips = rng.integers(0, 2, nt)
    cam = rng.integers(-1, n_cams, nt)
    sizes = [(int(rng.integers(8, 90)), int(rng.integers(8, 90))) for _ in range(n_cams)]
    sel = [(int(rng.integers(10, 60)), int(rng.integers(10, 60))) for _ in range(n_cams)]
    uv = rng.uniform(-10, 70, (nt, 6)).astype(np.float32)
    imgs = [rng.integers(0, 256, (h, w, 3), np.uint8) for w, h in sizes]
    vw, vh = int(rng.integers(17, 70)), int(rng.integers(17, 70))
    view = camera(vw, vh, (vw * 0.8, vw * 0.8, (vw - 1) / 2, (vh - 1) / 2), np.eye(3), np.zeros(3))
    truth = rng.integers(0, 256, (vh, vw, 3), np.uint8)
    big = max(im.nbytes for im in imgs)
    a = check(lib, view, sel, imgs, cam, uv, verts, tris, flips, truth=truth, z_far=7.0, max_image_bytes=big)
    assert a["counts"][0] > 0
    b = check(lib, view, sel, imgs, cam, uv, verts, tris, flips, truth=truth, z_far=7.0, bin_cap=seed, on_device=1)   # bins overflowing
    assert np.array_equal(a["rgb"], b["rgb"]) and a["counts"].tolist() == b["counts"].tolist()


def test_error_contract(lib):
    verts, tris, flips, cam, uv = strip(2, 5)
    sel = [(W, H)] * 2
    imgs = [ramp(W, H, 0), ramp(W, H, 1)]

    def rc(**kw):
        args = dict(view=view_cam(), sel_wh=sel, images=imgs, cam=cam, uv=uv, verts=verts, tris=tris, flips=flips)
        args.update(kw)
        return emu(lib, **args)[0]
    assert rc() == 0
    assert rc(n_facets=len(cam) - 1) == -1 and b"live triangle count" in lib.emu_texture_render_error()
    assert rc(shard_n=2) == -1 and b"sharded" in lib.emu_texture_render_error()
    for kw in (dict(z_near=0.0), dict(z_near=2.0, z_far=1.0), dict(z_far=float("inf")), dict(positions=2), dict(max_image_bytes=-1), dict(on_device=2)):
        assert rc(**kw) == -1, kw
    for v in (camera(0, H, K, np.eye(3), np.zeros(3)), camera(W, H, (0.0, 40.0, 1.0, 1.0), np.eye(3), np.zeros(3)),
              camera(1 << 14, 1 << 13, K, np.eye(3), np.zeros(3)), camera(W, H, K, np.full((3, 3), np.nan), np.zeros(3))):
        assert rc(view=v) == -1
    bad = np.array(cam)
    bad[0] = 2
    assert rc(cam=bad) == -1
    bad[0] = -2
    assert rc(cam=bad) == -1
    bu = np.array(uv)
    bu[0, 3] = np.nan
    assert rc(uv=bu) == -1
    assert rc(max_image_bytes=W * H * 3 - 1) == -1, "a host image larger than an arena"
    assert rc(max_image_bytes=W * H * 3 - 1, on_device=1) == 0
    assert rc(sel_wh=[(0, H), (W, H)]) == -1, "a used camera of size 0"
    assert emu(lib, view_cam(), sel, None, cam, uv, verts, tris, flips)[0] == -1, "rgb with the query"
    assert emu(lib, view_cam(), sel, None, cam, uv, verts, tris, flips, rgb=False)[0] == 0
    assert emu(lib, view_cam(), sel, None, cam, uv, verts, tris, flips, rgb=False, truth=ramp(W, H))[0] == -1, "truth with the query"
    assert rc(truth=ramp(W + 1, H)) == -1, "truth of another size"
    assert rc(truth=ramp(W, H)) == 0
