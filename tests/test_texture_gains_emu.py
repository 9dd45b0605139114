"""CPU tier of the colour equalisation (immesh_mesh_texture_gains, immesh_texture_apply_gains): the device bodies, argument check and
host solve (immesh_b200/csrc/texture_gains_core.cuh) run by the host emulation (tests/texture_gains/emu_texture_gains.cpp) in the device
call's orchestration.  The pair list and sums equal the numpy restatement (tests/texture_gains_reference.py) byte for byte, and the gains
are within 1e-8 relative of a direct sparse solve of the same equations: two cameras on a wall with constant colours (the 2 x 2 closed
form), an occluder, clipped samples, a NULL observer image, a camera in no pair (gain 1), images larger and smaller than the cameras,
several upload batches (one and two sweeps), max_pairs overflow, and random meshes and rows.  apply_gains' rounding byte for byte; the
error contract."""
import ctypes as C

import numpy as np
import pytest

from texture_gains_reference import apply_gains as ref_apply
from texture_gains_reference import pairs as ref_pairs
from texture_gains_reference import solve as ref_solve
from texture_reference import camera, select

W, H = 48, 40
K = (40.0, 40.0, 23.5, 19.5)


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_texture_gains())
    L.emu_texture_gains_error.restype = C.c_char_p
    vp = C.c_void_p
    L.emu_texture_gains.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int64, vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_longlong, C.c_int,
                                    vp, vp, vp, vp, vp, vp]
    L.emu_apply_gains.argtypes = [vp, vp, C.c_int, C.c_int, vp]
    return L


def cam_at(x, y=0.0, w=W, h=H, k=K):
    return camera(w, h, k, np.eye(3), np.array([x, y, 0.0]))   # OpenCV axes: the world's z is forward


def gains_cfg(sigma_n=10.0, sigma_g=0.1, max_pairs=1 << 20, max_image_bytes=0, two_sided=1, min_cos=0.0, permille=0, z_near=0.1, z_far=1000.0, positions=0):
    from immesh_b200 import api
    return api._TexGainsCfg(api._TexCfg(z_near, z_far, min_cos, permille, two_sided, positions, 0), sigma_n, sigma_g, max_pairs, max_image_bytes)


def emu(lib, cams, images, cam, uv, verts, tris, flips, cfg=None, on_device=0, bin_cap=1 << 40, shard_n=1, n_facets=None, n_cams=None):
    """(rc, dict(gains, pair_cam, pair_sums, n_pairs, counts, batches)) of the emulation"""
    from immesh_b200 import api
    cfg = cfg or gains_cfg()
    arr, nc = api.texture_cameras([(c["width"], c["height"], c["K"], c["R"], c["t"]) for c in cams])
    imgs, _, keep = api.texture_images(images)
    cam = np.ascontiguousarray(cam, np.int32).reshape(-1)
    uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 6)
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    flips = np.ascontiguousarray(flips, np.int32).reshape(-1)
    cap = max(int(cfg.max_pairs), 1)
    out = dict(gains=np.full((max(nc, 1), 3), -7.0), pair_cam=np.full((min(cap, 4096), 2), -5, np.int32), pair_sums=np.full((min(cap, 4096), 7), -5, np.int64),
               counts=np.full(8, -3, np.int64))
    npairs, nb = C.c_int64(-1), C.c_int(-1)
    rc = lib.emu_texture_gains(C.cast(arr, C.c_void_p), nc if n_cams is None else n_cams, C.cast(imgs, C.c_void_p), on_device, cam.ctypes.data, uv.ctypes.data,
                               len(cam) if n_facets is None else n_facets, C.addressof(cfg), verts.ctypes.data, None, None, len(verts), tris.ctypes.data,
                               flips.ctypes.data, len(tris), bin_cap, shard_n, out["gains"].ctypes.data, out["pair_cam"].ctypes.data,
                               out["pair_sums"].ctypes.data, C.addressof(npairs), out["counts"].ctypes.data, C.addressof(nb))
    del keep
    out["n_pairs"], out["batches"] = npairs.value, nb.value
    return rc, out


def check(lib, cams, images, cam, uv, verts, tris, flips, cfg=None, **kw):
    """the emulation equals the restatement: pairs and sums byte for byte, gains within 1e-8 of spsolve"""
    cfg = cfg or gains_cfg()
    rc, got = emu(lib, cams, images, cam, uv, verts, tris, flips, cfg=cfg, **kw)
    assert rc == 0, lib.emu_texture_gains_error()
    sel = dict(z_near=cfg.sel.z_near, z_far=cfg.sel.z_far, min_cos=cfg.sel.min_cos, min_visible_permille=cfg.sel.min_visible_permille,
               two_sided=bool(cfg.sel.two_sided))
    pc, ps, used, clipped = ref_pairs(cams, images, cam, uv, verts, tris, flips, **sel)
    n = got["n_pairs"]
    assert n == len(pc)
    assert np.array_equal(got["pair_cam"][:n], pc) and np.array_equal(got["pair_sums"][:n], ps)
    c = got["counts"]
    assert (c[0], c[1], c[2]) == (len(pc), used, clipped)
    assert c[3] == sum(im is not None for im in images) and c[6] == sum(cm["width"] * cm["height"] for cm, im in zip(cams, images) if im is not None)
    ref = ref_solve(len(cams), pc, ps, cfg.sigma_n, cfg.sigma_g)
    g = got["gains"][:len(cams)]
    assert np.allclose(g, ref, rtol=1e-8, atol=0), np.abs(g / ref - 1).max()
    assert (g > 0).all()
    paired = np.zeros(len(cams), bool)
    paired[pc.reshape(-1)] = True
    assert c[4] == (~paired).sum() and (g[~paired] == 1.0).all()
    return got


def wall(n=8, z=5.0, half=1.5, seed=0):
    """a grid wall at depth z facing the cameras: verts, ascending triples, random flips"""
    xs = np.linspace(-half, half, n + 1)
    X, Y = np.meshgrid(xs, xs * 0.8)
    verts = np.stack([X.reshape(-1), Y.reshape(-1), np.full(X.size, z)], axis=1).astype(np.float32)
    tris = []
    for j in range(n):
        for i in range(n):
            a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i, (j + 1) * (n + 1) + i + 1
            tris += [sorted((a, b, d)), sorted((a, d, c))]
    tris = np.array(tris, np.int32)
    flips = np.random.default_rng(seed).integers(0, 2, len(tris)).astype(np.int32)
    return verts, tris, flips


def rows_of(cams, verts, tris, flips):
    s = select(cams, verts, tris, flips, two_sided=True)
    return s["cam"], np.nan_to_num(s["uv"])


def flat(colour, w=W, h=H):
    return np.broadcast_to(np.asarray(colour, np.uint8), (h, w, 3)).copy()


def test_two_cameras_constant_colours_closed_form(lib):
    verts, tris, flips = wall()
    cams = [cam_at(-0.3), cam_at(0.3)]
    cam, uv = rows_of(cams, verts, tris, flips)
    assert (cam == 0).any() and (cam == 1).any()
    I = np.array([[100, 120, 140], [150, 130, 110]], np.float64)
    imgs = [flat(I[0]), flat(I[1])]
    for sn, sg in ((10.0, 0.1), (5.0, 1.0)):
        got = check(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(sigma_n=sn, sigma_g=sg))
        N = got["pair_sums"][:got["n_pairs"], 0].sum()
        assert got["n_pairs"] == 2 and N == got["counts"][1] > 100
        for ch in range(3):
            a00 = N * I[0, ch] ** 2 / sn ** 2 + N / sg ** 2
            a11 = N * I[1, ch] ** 2 / sn ** 2 + N / sg ** 2
            a01 = -N * I[0, ch] * I[1, ch] / sn ** 2
            b = N / sg ** 2
            det = a00 * a11 - a01 * a01
            g0, g1 = (b * a11 - a01 * b) / det, (a00 * b - a01 * b) / det
            assert np.allclose(got["gains"][:2, ch], (g0, g1), rtol=1e-9)
    # a loose prior pulls the corrected colours together
    got = check(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(sigma_n=10.0, sigma_g=100.0))
    corrected = got["gains"][:2] * I
    assert (np.abs(corrected[0] - corrected[1]) < 0.05 * np.abs(I[0] - I[1])).all()


def test_occluder_clipping_null_observer_and_unpaired(lib):
    rng = np.random.default_rng(3)
    verts, tris, flips = wall(n=10)
    occ = np.array([[-0.4, -0.3, 3.0], [0.4, -0.3, 3.0], [0.4, 0.3, 3.0], [-0.4, 0.3, 3.0]], np.float32)
    v = np.concatenate([verts, occ])
    b = len(verts)
    t = np.concatenate([tris, [[b, b + 1, b + 2], [b, b + 2, b + 3]]]).astype(np.int32)
    f = np.concatenate([flips, [0, 1]]).astype(np.int32)
    cams = [cam_at(-0.5), cam_at(0.0, 0.2), cam_at(0.5), cam_at(40.0)]   # camera 3 looks past the wall
    cam, uv = rows_of(cams[:3], v, t, f)
    imgs = [rng.integers(1, 255, (H, W, 3), np.uint8) for _ in cams]
    got = check(lib, cams, imgs, cam, uv, v, t, f)
    assert got["counts"][0] >= 4 and got["counts"][2] == 0 and got["counts"][4] == 1 and (got["gains"][3] == 1.0).all()
    # clipped samples: saturated and black patches
    clip = [im.copy() for im in imgs]
    clip[0][:, :20] = 255
    clip[1][10:30, :, 1] = 0
    got = check(lib, cams, clip, cam, uv, v, t, f)
    assert got["counts"][2] > 0
    # a NULL observer image: camera 1 textures nothing here and takes no part
    cam2, uv2 = rows_of([cams[0], cams[2]], v, t, f)
    cam2 = np.where(cam2 == 1, 2, cam2)
    none = [imgs[0], None, imgs[2], imgs[3]]
    got = check(lib, cams, none, cam2, uv2, v, t, f)
    assert got["counts"][3] == 3 and (got["gains"][1] == 1.0).all()
    assert 1 not in got["pair_cam"][:got["n_pairs"]]


def test_image_sizes_batches_and_device(lib):
    rng = np.random.default_rng(5)
    verts, tris, flips = wall(n=9)
    cams = [cam_at(x) for x in (-0.6, -0.2, 0.2, 0.6)]
    cam, uv = rows_of(cams, verts, tris, flips)
    sizes = [(W, H), (2 * W, 2 * H), (W // 2, H // 2), (W + 7, H - 5)]
    imgs = [rng.integers(1, 255, (h, w, 3), np.uint8) for w, h in sizes]
    one = check(lib, cams, imgs, cam, uv, verts, tris, flips)
    assert one["batches"] == 1 and one["n_pairs"] >= 6
    dev = check(lib, cams, imgs, cam, uv, verts, tris, flips, on_device=1)
    assert dev["batches"] == 0
    for mib in (max(im.nbytes for im in imgs), imgs[0].nbytes + imgs[1].nbytes + 100):
        got = check(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(max_image_bytes=mib))
        assert got["batches"] > 1
        for k in ("gains", "pair_cam", "pair_sums", "counts"):
            assert np.array_equal(got[k], one[k]), k
    # overflowing bins walk every slot
    got = check(lib, cams, imgs, cam, uv, verts, tris, flips, bin_cap=10)
    assert np.array_equal(got["pair_sums"], one["pair_sums"])
    # max_pairs overflow: the count, no gain or pair written
    rc, over = emu(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(max_pairs=one["n_pairs"] - 1))
    assert rc == -3 and over["n_pairs"] == one["n_pairs"] and over["counts"][0] == one["n_pairs"]
    assert (over["gains"] == -7.0).all() and (over["pair_cam"] == -5).all()
    rc, ok = emu(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(max_pairs=one["n_pairs"]))
    assert rc == 0 and np.array_equal(ok["gains"], one["gains"])


@pytest.mark.parametrize("seed", range(4))
def test_random_meshes_and_rows(lib, seed):
    rng = np.random.default_rng(100 + seed)
    nv, nt, n_cams = 40, 60, 5
    verts = np.stack([rng.uniform(-2, 2, nv), rng.uniform(-1.6, 1.6, nv), rng.uniform(3.5, 7, nv)], axis=1).astype(np.float32)
    tris = np.sort(np.stack([rng.choice(nv, 3, replace=False) for _ in range(nt)]), axis=1).astype(np.int32)
    flips = rng.integers(0, 2, nt).astype(np.int32)
    cams = [cam_at(rng.uniform(-0.8, 0.8), rng.uniform(-0.4, 0.4)) for _ in range(n_cams)]
    cam = rng.integers(-1, n_cams, nt).astype(np.int32)
    uv = np.stack([rng.uniform(-5, W + 5, (nt, 3)), rng.uniform(-5, H + 5, (nt, 3))], axis=2).reshape(nt, 6).astype(np.float32)
    imgs = [rng.integers(0, 256, (H + 3 * k, W - 2 * k, 3), np.uint8) for k in range(n_cams)]
    a = check(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(two_sided=seed % 2, permille=100 * seed))
    b = check(lib, cams, imgs, cam, uv, verts, tris, flips, cfg=gains_cfg(two_sided=seed % 2, permille=100 * seed, max_image_bytes=max(i.nbytes for i in imgs)))
    assert np.array_equal(a["pair_sums"], b["pair_sums"]) and np.array_equal(a["gains"], b["gains"])
    if seed == 0:
        assert a["n_pairs"] > 0 and a["counts"][2] > 0


def apply(lib, images, outs, gains, on_device=0, n=None):
    from immesh_b200 import api
    ia, _, k1 = api.texture_images(images)
    oa, _, k2 = api.texture_images(outs)
    g = np.ascontiguousarray(gains, np.float64).reshape(-1, 3)
    return lib.emu_apply_gains(C.cast(ia, C.c_void_p), C.cast(oa, C.c_void_p), len(images) if n is None else n, on_device, g.ctypes.data)


def test_apply_gains_rounding_and_contract(lib):
    rng = np.random.default_rng(9)
    imgs = [rng.integers(0, 256, (7, 9, 3), np.uint8), None, np.arange(256, dtype=np.uint8).repeat(3).reshape(16, 16, 3)]
    gains = np.array([[0.7, 1.0, 1.3], [5.0, 5.0, 5.0], [0.5, 1.5, 2.0 / 3.0]])
    outs = [np.full_like(imgs[0], 7), None, np.full_like(imgs[2], 7)]
    assert apply(lib, imgs, outs, gains) == 0
    for k in (0, 2):
        assert np.array_equal(outs[k], ref_apply(imgs[k], gains[k]))
    # half-way values round up; the top clamps
    x = np.array([[[1, 3, 255]]], np.uint8)
    o = np.zeros_like(x)
    assert apply(lib, [x], [o], [[0.5, 0.5, 1.01]]) == 0 and o.tolist() == [[[1, 2, 255]]]
    # in place
    y = imgs[0].copy()
    assert apply(lib, [y], [y], gains[:1]) == 0 and np.array_equal(y, outs[0])
    # refusals, nothing written
    z = np.full_like(imgs[0], 7)
    for g in ([[np.nan, 1, 1]], [[-0.1, 1, 1]], [[np.inf, 1, 1]]):
        assert apply(lib, [imgs[0]], [z], g) == -1
    assert apply(lib, [imgs[0]], [np.zeros((7, 8, 3), np.uint8)], [[1, 1, 1]]) == -1
    assert apply(lib, [imgs[0]], [None], [[1, 1, 1]]) == -1
    assert apply(lib, [imgs[0]], [z], [[1, 1, 1]], on_device=2) == -1
    assert apply(lib, [imgs[0]], [z], [[1, 1, 1]], n=-1) == -1
    assert (z == 7).all()


def test_error_contract(lib):
    rng = np.random.default_rng(2)
    verts, tris, flips = wall(n=4)
    cams = [cam_at(-0.3), cam_at(0.3)]
    cam, uv = rows_of(cams, verts, tris, flips)
    imgs = [rng.integers(1, 255, (H, W, 3), np.uint8) for _ in cams]

    def refused(**kw):
        rc, got = emu(lib, kw.pop("cams", cams), kw.pop("images", imgs), kw.pop("cam", cam), kw.pop("uv", uv), verts, tris, flips, **kw)
        assert rc == -1 and (got["gains"] == -7.0).all() and (got["counts"] == -3).all(), lib.emu_texture_gains_error()
        return lib.emu_texture_gains_error().decode()

    assert emu(lib, cams, imgs, cam, uv, verts, tris, flips)[0] == 0
    refused(n_facets=len(cam) - 1)
    refused(n_cams=0)
    refused(on_device=2)
    refused(shard_n=2)
    bad = cam.copy()
    bad[0] = 2
    refused(cam=bad)
    bu = uv.copy()
    bu[np.nonzero(cam >= 0)[0][0], 3] = np.inf
    refused(uv=bu)
    assert "needs an image" in refused(images=[imgs[0], None] if (cam == 1).any() else [None, imgs[1]])
    refused(images=[imgs[0], imgs[1][:, :1].copy()], cfg=gains_cfg(max_image_bytes=100))
    refused(cams=[cams[0], camera(W, H, (0.0, 40.0, 23.5, 19.5), np.eye(3), np.zeros(3))])
    for cfg in (gains_cfg(sigma_n=0.0), gains_cfg(sigma_g=-1.0), gains_cfg(sigma_n=np.nan), gains_cfg(sigma_g=np.inf), gains_cfg(max_pairs=0),
                gains_cfg(max_image_bytes=-1), gains_cfg(z_near=0.0), gains_cfg(min_cos=2.0), gains_cfg(permille=1001), gains_cfg(positions=2)):
        refused(cfg=cfg)
