"""GPU tier of the texture atlas (immesh_mesh_texture_bake): selections of the Avia-shaped and HDL-64 meshes with trajectory cameras
(tests/test_texture_gpu.py's), baked from ramp and random images at full and half the selection's resolution, byte-equal to the numpy
restatement (tests/texture_bake_reference.py): pages, facet_page and atlas_uv.  Host and device images give the same result, and so
do arenas that hold one image (every camera its own batch) and the default.  A bake issued behind queued push_frame_from_lio_async
frames equals one made after wait(); a handle that baked computes the same later frames and change-feed rows as a twin that never
did; the error contract."""
import ctypes as C

import numpy as np
import pytest
import torch

from immesh_b200 import api
from test_texture_gpu import as_tuples, lio_chain, trajectory_cameras, world_mesh
from texture_bake_reference import bake as ref_bake

pytestmark = pytest.mark.gpu


def ramp(w, h, k):
    img = np.zeros((h, w, 3), np.uint8)
    img[..., 0] = np.round(np.arange(w) * 255.0 / (w - 1))[None, :]
    img[..., 1] = np.round(np.arange(h) * 255.0 / (h - 1))[:, None]
    img[..., 2] = (40 * k + 20) % 256
    return img


def images_for(cams, sel, scale, kind, seed=0):
    rng = np.random.default_rng(seed)
    used = set(sel["cam"][sel["cam"] >= 0].tolist())
    out = []
    for k, c in enumerate(cams):
        w, h = max(1, int(c["width"] * scale)), max(1, int(c["height"] * scale))
        img = ramp(w, h, k) if kind == "ramp" else rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        out.append(img if k in used else None)
    return out


def same(a, b):
    assert a["counts"] == b["counts"]
    assert np.array_equal(a["page"], b["page"])
    assert np.array_equal(a["uv"].view(np.uint32), b["uv"].view(np.uint32))
    assert np.array_equal(a["pages"], b["pages"])


def check(mesh, sel, cams, images, page_size=1024, max_cell=64, **kw):
    got = mesh.texture_bake(sel, as_tuples(cams), images, page_size=page_size, max_cell=max_cell, **kw)
    ref = ref_bake([(c["width"], c["height"]) for c in cams], [None if im is None else np.asarray(im.cpu() if torch.is_tensor(im) else im) for im in images],
                   sel["cam"], sel["uv"], page_size=page_size, max_cell=max_cell)
    assert got["pages"].shape[0] == ref["n_pages"]
    assert np.array_equal(got["page"], ref["page"])
    t = sel["cam"] >= 0
    assert np.array_equal(got["uv"][t].view(np.uint32), ref["uv"][t].view(np.uint32))
    assert np.isnan(got["uv"][~t]).all()
    assert [got["counts"][k] for k in api.BAKE_COUNT_KEYS] == ref["counts"].tolist()
    assert np.array_equal(got["pages"], ref["pages"]), int((got["pages"] != ref["pages"]).any(axis=-1).sum())
    return got


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_texture_bake_against_restatement(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    assert sel["counts"]["textured"] > 200
    for scale, img_kind in ((1.0, "ramp"), (0.5, "random"), (2.0, "random")):
        imgs = images_for(cams, sel, scale, img_kind, seed=int(scale * 10))
        host = check(mesh, sel, cams, imgs)
        dev = mesh.texture_bake(sel, as_tuples(cams), [None if im is None else torch.from_numpy(im).cuda() for im in imgs], page_size=1024)
        same(host, dev)
        one = max(im.nbytes for im in imgs if im is not None)
        same(host, mesh.texture_bake(sel, as_tuples(cams), imgs, page_size=1024, max_image_bytes=one))
    # several pages and a selection made at half resolution
    half = trajectory_cameras(poses, 0.5)
    sel_h = mesh.texture_select(as_tuples(half), vertices=False)
    g = check(mesh, sel_h, half, images_for(half, sel_h, 2.0, "ramp"), page_size=256, max_cell=32)
    assert g["pages"].shape[0] >= 1 and g["counts"]["textured"] > 0
    # padded rows of device images
    imgs = images_for(cams, sel, 1.0, "random", seed=3)
    padded = []
    for im in imgs:
        if im is None:
            padded.append(None)
            continue
        buf = torch.zeros((im.shape[0], im.shape[1] + 5, 3), dtype=torch.uint8, device="cuda")
        buf[:, :im.shape[1]] = torch.from_numpy(im).cuda()
        padded.append(buf[:, :im.shape[1]])
    same(check(mesh, sel, cams, imgs), mesh.texture_bake(sel, as_tuples(cams), padded, page_size=1024))


def test_queued_frames_and_twin(cuda_lib):
    seen = {}

    def bake(k, mesh, scans):
        if k in (4, 6):
            cams = trajectory_cameras([(s["R_true"], s["t_true"]) for s in scans[k - 2:k + 1]])
            mesh.wait()
            sel = mesh.texture_select(as_tuples(cams), vertices=False)
            imgs = images_for(cams, sel, 1.0, "random", seed=k)
            seen[k] = (cams, sel, imgs)

    def replay(k, mesh, scans):
        if k in (5, 7):
            cams, sel, imgs = seen[k - 1]
            queued = mesh.texture_bake(sel, as_tuples(cams), imgs, page_size=512)   # behind the frames still queued
            mesh.wait()
            same(queued, mesh.texture_bake(sel, as_tuples(cams), imgs, page_size=512))
            seen[("n", k)] = queued["counts"]["textured"]

    _, a, _ = lio_chain(cuda_lib, 10, between=lambda k, m, s: (bake(k, m, s), replay(k, m, s)))
    _, b, _ = lio_chain(cuda_lib, 10, between=lambda k, m, s: bake(k, m, s))
    assert seen[("n", 7)] > 0
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    assert a.counts() == b.counts()
    ca, cb = a.changes(0), b.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key


def test_error_contract(cuda_lib):
    L = cuda_lib
    mesh, poses = world_mesh(cuda_lib, "avia")
    cams = trajectory_cameras(poses[:1])
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    assert sel["counts"]["textured"] > 0
    imgs = images_for(cams, sel, 1.0, "random")
    arr, n = api.texture_cameras(as_tuples(cams))
    ia, on_dev, keep = api.texture_images(imgs)
    cam = np.ascontiguousarray(sel["cam"], np.int32)
    uv = np.ascontiguousarray(sel["uv"], np.float32)
    nf = len(cam)
    i32, f32 = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    npg = C.c_int(0)

    def tb(cfg=None, c=cam, u=uv, images=ia, on_device=0, pages=None, cap=0, page=None, auv=None):
        cfg = cfg or api._AtlasCfg(256, 64, 0)
        return L.immesh_mesh_texture_bake(mesh._h, arr, n, images, on_device, c.ctypes.data_as(i32), u.ctypes.data_as(f32), len(c), C.byref(cfg),
                                          None if pages is None else pages.ctypes.data_as(C.c_void_p), cap,
                                          None if page is None else page.ctypes.data_as(i32), None if auv is None else auv.ctypes.data_as(f32),
                                          C.byref(npg), None)
    page = np.full(nf, 9, np.int32)
    assert tb(page=page) == 0 and npg.value >= 1 and (page[cam >= 0] >= 0).all() and (page[cam < 0] == -1).all()   # a count query
    need = npg.value
    pages = np.full((need, 256, 256, 3), 77, np.uint8)
    page[:] = 9
    auv = np.full((nf, 6), np.nan, np.float32)
    assert tb(pages=pages, cap=need - 1, page=page, auv=auv) == -3 and npg.value == need
    assert (pages == 77).all() and (page == 9).all() and np.isnan(auv).all(), "nothing written"
    assert tb(pages=pages, cap=need, page=page, auv=auv) == 0 and not (pages == 77).all()
    for cfg in (api._AtlasCfg(128, 8, 0), api._AtlasCfg(300, 8, 0), api._AtlasCfg(256, 4, 0), api._AtlasCfg(256, 512, 0), api._AtlasCfg(256, 64, -1),
                api._AtlasCfg(256, 64, 100)):
        assert tb(cfg=cfg) == -1, (cfg.page_size, cfg.max_cell, cfg.max_image_bytes)
    bad = cam.copy()
    bad[0] = n
    assert tb(c=bad) == -1
    bu = uv.copy()
    bu[np.nonzero(cam >= 0)[0][0], 2] = np.inf
    assert tb(u=bu) == -1
    assert tb(on_device=2) == -1
    none, _, _ = api.texture_images([None] * len(cams))
    assert tb(images=none) == -1
    assert L.immesh_mesh_texture_bake(mesh._h, arr, n, ia, 0, cam.ctypes.data_as(i32), uv.ctypes.data_as(f32), nf, None, None, 0, None, None, C.byref(npg), None) == -1
    del keep
    # the handle still meshes after the refused calls
    r = mesh.texture_select(as_tuples(cams), vertices=False)
    assert np.array_equal(r["cam"], sel["cam"])
