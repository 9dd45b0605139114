"""GPU tier of the textured render (immesh_mesh_render_textured): on the Avia- and HDL-64-shaped meshes with trajectory cameras
(tests/test_texture_gpu.py's), texture_select's rows rendered from ramp and random images at 0.5x, 1x and 2x the selection's size at
a selection camera and at a camera between two of them: rgb, depth, facet, needed and every count equal the numpy restatement
(tests/texture_render_reference.py) byte for byte, and depth equals render_view's at the converted camera bit for bit.  Host images,
device images (also with padded rows), one-image arenas and needed-only image lists agree.  Self-checks that need no restatement: a
planar wall facing an axis-aligned camera reproduces that camera's image within 1 on the pixels its own facets win; the bake's pages
and rows render like the source ramp images within the bound derived below.  texture_rows' rows render with frame-indexed cameras;
held-out views score better with the right images than with shifted ones; a render behind queued frames equals one after wait(), and
a handle that rendered meshes like a twin that never did; the error contract (a sharded handle needs two GPUs: its refusal is checked
by the CPU tier through the shared argument check)."""
import ctypes as C

import numpy as np
import pytest
import torch

from immesh_b200 import api
from test_texture_bake_gpu import images_for, ramp
from test_texture_gpu import as_tuples, lio_chain, trajectory_cameras, world_mesh
from texture_reference import camera, raster_R
from texture_render_reference import render_textured as ref_render

pytestmark = pytest.mark.gpu


def tup(c):
    return (c["width"], c["height"], c["K"], c["R"], c["t"])


def between(a, b):
    """a camera halfway between two cameras' positions, with a's orientation and intrinsics"""
    return camera(a["width"], a["height"], a["K"], a["R"], (a["t"] + b["t"]) / 2.0)


def same(a, b, rgb=True):
    for k in ("depth", "facet", "needed"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    assert a["counts"] == b["counts"]
    if rgb:
        assert np.array_equal(a["rgb"], b["rgb"])


def check(mesh, view, sel, cams, images, verts, tris, flips, truth=None, **kw):
    got = mesh.render_textured(tup(view), sel, as_tuples(cams), images, truth=truth, **kw)
    host = [None if im is None else np.asarray(im.cpu() if torch.is_tensor(im) else im) for im in images]
    ref = ref_render(view, [(c["width"], c["height"]) for c in cams], host, sel["cam"], sel["uv"], verts, tris, flips, truth=truth)
    assert np.array_equal(got["depth"].view(np.uint32), ref["depth"].view(np.uint32))
    assert np.array_equal(got["facet"], ref["facet"]), int((got["facet"] != ref["facet"]).sum())
    assert np.array_equal(got["needed"], ref["needed"])
    assert [got["counts"][k] for k in api.TEXTURE_VIEW_COUNT_KEYS] == ref["counts"].tolist(), (got["counts"], ref["counts"])
    assert np.array_equal(got["rgb"], ref["rgb"]), int((got["rgb"] != ref["rgb"]).any(axis=-1).sum())
    # the visibility is render_view's at the converted camera
    _, depth = mesh.render_view(view["K"], view["width"], view["height"], 0.1, 1000.0, raster_R(view["R"]), view["t"])
    assert np.array_equal(got["depth"].view(np.uint32), depth.view(np.uint32))
    return got


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_against_restatement_and_image_sources(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    v, tri, fl = mesh.snapshot()
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    assert sel["counts"]["textured"] > 200
    views = (cams[2], between(cams[0], cams[2]))
    for scale, img_kind in ((1.0, "ramp"), (0.5, "random"), (2.0, "random")):
        imgs = images_for(cams, sel, scale, img_kind, seed=int(scale * 10))
        for view in views:
            truth = np.random.default_rng(7).integers(0, 256, (view["height"], view["width"], 3), np.uint8)
            host = check(mesh, view, sel, cams, imgs, v, tri, fl, truth=truth)
            assert host["counts"]["textured"] > 1000 and host["counts"]["sse_0"] > 0
            dev = mesh.render_textured(tup(view), sel, as_tuples(cams), [None if im is None else torch.from_numpy(im).cuda() for im in imgs],
                                       truth=torch.from_numpy(truth).cuda())
            same(host, dev)
            one = max(im.nbytes for im in imgs if im is not None)
            same(host, mesh.render_textured(tup(view), sel, as_tuples(cams), imgs, truth=truth, max_image_bytes=one))
            only = [im if host["needed"][k] else None for k, im in enumerate(imgs)]
            same(host, mesh.render_textured(tup(view), sel, as_tuples(cams), only, truth=truth))
            q = mesh.render_textured(tup(view), sel, as_tuples(cams))
            assert q["rgb"] is None
            same(dict(host, counts={k: (host["counts"][k] if i < 4 else 0) for i, k in enumerate(api.TEXTURE_VIEW_COUNT_KEYS)}), q, rgb=False)
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
    same(check(mesh, cams[1], sel, cams, imgs, v, tri, fl), mesh.render_textured(tup(cams[1]), sel, as_tuples(cams), padded))
    # the call wrote nothing on the handle
    for x, y in zip((v, tri, fl), mesh.snapshot()):
        assert np.array_equal(x, y)


def test_wall_reproduces_its_camera(cuda_lib):
    """A planar wall x = 5 seen by cameras whose rotation is an exact axis permutation: every facet has constant depth there, so the
    perspective-correct source point is the projective one and a render at a selection camera samples its own image at the pixel
    centres (up to the float rounding of the uv): within 1 per channel on every pixel its own facets win."""
    rng = np.random.default_rng(11)
    g = np.arange(-2.0, 2.0, 0.04)
    yy, zz = np.meshgrid(g, g[:75] - 1.5)
    mesh = api.Mesh(api.MeshConfig(max_vertices=1 << 19, max_triangles=1 << 21, max_voxels=1 << 17, max_frame_points=1 << 18), lib=cuda_lib)
    for f in range(2):
        pts = np.stack([np.full(yy.size, 5.0), yy.reshape(-1) + rng.uniform(-0.01, 0.01, yy.size), zz.reshape(-1) + rng.uniform(-0.01, 0.01, yy.size)], axis=1)
        mesh.push_frame(pts.astype(np.float32), np.zeros(3), f)
    v, tri, fl = mesh.snapshot()
    assert len(tri) > 500
    R = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])   # OpenCV z along world +x, x along -y, y along -z
    cams = [camera(320, 240, (160.0, 160.0, 159.5, 119.5), R, np.array([0.0, dy, 0.0])) for dy in (-0.6, 0.0, 0.6)]
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    imgs = [np.random.default_rng(k).integers(0, 256, (240, 320, 3), np.uint8) for k in range(3)]
    for k in range(3):
        r = check(mesh, cams[k], sel, cams, imgs, v, tri, fl)
        own = (r["facet"] >= 0) & (sel["cam"][np.maximum(r["facet"], 0)] == k)
        assert own.sum() > 1000
        assert np.abs(r["rgb"][own].astype(int) - imgs[k][own].astype(int)).max() <= 1


def test_atlas_round_trip(cuda_lib):
    """Rendering from the bake's pages and rows against rendering from the source ramp images (channel c linear in the pixel: L_c with
    slope g <= 255 / 239 per pixel, each stored value rounded, so a bilinear sample of the image is L_c + e with |e| <= 0.5).  Direct:
    D = round(L(s) + e) within 1 of L(s).  Atlas: each texel is round(L(s_t) + e) within 1 of L at its source point; the render's
    bilinear weights reproduce L(s) from the texels' source points where the cell map is affine (|error| <= 1 from the texels, 0.5 from
    the final rounding), and texels just outside the slot's triangle take clamped barycentrics, which moves their source point by at
    most one source pixel along each axis (a cell side is at least the longest edge plus 4): at most g sqrt(2) < 1.6 more.  So
    |A - D| <= 1 + 1.5 + 1.6 < 5, i.e. at most 4, on pixels whose facet's cell is not capped at max_cell (a capped cell shrinks the
    facet and the bound does not hold)."""
    mesh, poses = world_mesh(cuda_lib, "avia")
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    imgs = [ramp(c["width"], c["height"], k) for k, c in enumerate(cams)]
    P, max_cell = 2048, 64
    bake = mesh.texture_bake(sel, as_tuples(cams), imgs, page_size=P, max_cell=max_cell)
    pcams = [(P, P, (1.0, 1.0, 0.0, 0.0), np.eye(3), np.zeros(3))] * len(bake["pages"])
    from texture_bake_reference import scaled
    p = scaled(np.nan_to_num(sel["uv"]), np.array([(c["width"], c["height"]) for c in cams])[np.maximum(sel["cam"], 0)],
               np.array([(c["width"], c["height"]) for c in cams])[np.maximum(sel["cam"], 0)])
    L = np.zeros(len(p))
    for k in range(3):
        e = (k + 1) % 3
        L = np.maximum(L, np.hypot(p[:, 2 * e] - p[:, 2 * k], p[:, 2 * e + 1] - p[:, 2 * k + 1]))
    capped = np.ceil(L) + 4.0 > max_cell
    for view in (cams[0], between(cams[0], cams[2])):
        d = mesh.render_textured(tup(view), sel, as_tuples(cams), imgs)
        a = mesh.render_textured(tup(view), bake, pcams, list(bake["pages"]))
        assert np.array_equal(a["facet"], d["facet"]) and np.array_equal(a["depth"].view(np.uint32), d["depth"].view(np.uint32))
        f = d["facet"]
        ok = (f >= 0) & (sel["cam"][np.maximum(f, 0)] >= 0) & ~capped[np.maximum(f, 0)]
        assert ok.sum() > 1000
        diff = np.abs(a["rgb"].astype(int) - d["rgb"].astype(int))[ok]
        assert diff.max() <= 4, np.bincount(diff.reshape(-1))


def test_online_rows_render(cuda_lib):
    """texture_rows' rows with frame-indexed cameras render exactly like texture_select's rows over the same cameras"""
    mesh, poses = world_mesh(cuda_lib, "avia")
    cams = trajectory_cameras(poses)
    rig = (cams[0]["width"], cams[0]["height"], cams[0]["K"], np.eye(3), np.zeros(3))
    mesh.texture_enable(rig)
    f0 = 5
    for k, c in enumerate(cams):
        mesh.texture_pose(c["R"], c["t"])
        mesh.push_frame(np.zeros((0, 3), np.float32), c["t"], 4 + k)
    rows = mesh.texture_rows(vertices=False)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    assert np.array_equal(rows["cam"], np.where(sel["cam"] >= 0, sel["cam"] + f0, -1))
    imgs = images_for(cams, sel, 1.0, "random", seed=5)
    by_frame = [cams[0]] * f0 + cams
    fimgs = [None] * f0 + imgs
    view = between(cams[1], cams[3])
    a = mesh.render_textured(tup(view), rows, as_tuples(by_frame), fimgs)
    b = mesh.render_textured(tup(view), sel, as_tuples(cams), imgs)
    assert np.array_equal(a["rgb"], b["rgb"]) and np.array_equal(a["facet"], b["facet"]) and a["counts"] == b["counts"]
    assert np.array_equal(np.nonzero(a["needed"])[0], np.nonzero(b["needed"])[0] + f0)
    # the query names the frames whose images a node has to load
    q = mesh.render_textured(tup(view), rows, as_tuples(by_frame))
    assert np.array_equal(q["needed"], a["needed"])


def painted(mesh, cams, seed=0):
    """per camera the image of a smooth seeded pattern painted on the world: render_view's depth unprojected, coloured by the point"""
    rng = np.random.default_rng(seed)
    f = rng.uniform(0.5, 2.0, (3, 3))
    ph = rng.uniform(0, 2 * np.pi, 3)
    out = []
    for c in cams:
        w, h = c["width"], c["height"]
        _, depth = mesh.render_view(c["K"], w, h, 0.1, 1000.0, raster_R(c["R"]), c["t"])
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
        fx, fy, cx, cy = c["K"]
        pc = np.stack([(xs - cx) / fx * depth, (ys - cy) / fy * depth, depth.astype(np.float64)], axis=-1)
        pw = pc @ c["R"].T + c["t"]
        img = np.zeros((h, w, 3), np.uint8)
        for ch in range(3):
            img[..., ch] = np.clip(127.5 + 127.5 * np.sin(pw @ f[ch] + ph[ch]), 0, 255).astype(np.uint8)
        img[depth < 0] = 0
        out.append(img)
    return out


def test_held_out_score(cuda_lib):
    mesh, poses = world_mesh(cuda_lib, "avia")
    cams = trajectory_cameras(poses)
    imgs = painted(mesh, cams)
    held = 2   # the middle pose's forward camera; its neighbours' forward cameras see most of what it sees
    train = [k for k in range(len(cams)) if k != held]
    sel = mesh.texture_select(as_tuples([cams[k] for k in train]), vertices=False)
    right = [imgs[k] for k in train]
    shifted = right[1:] + right[:1]
    a = mesh.render_textured(tup(cams[held]), sel, as_tuples([cams[j] for j in train]), right, truth=imgs[held])
    b = mesh.render_textured(tup(cams[held]), sel, as_tuples([cams[j] for j in train]), shifted, truth=imgs[held])
    assert a["coverage"] == b["coverage"] and a["coverage"] > 0.05, a["coverage"]
    assert a["psnr"] > b["psnr"] + 3.0, (a["psnr"], b["psnr"])


def test_queued_frames_and_twin(cuda_lib):
    """The twin b (never renders) selects the rows of the mesh after frame k; handle a, fed the same stream, renders those rows while
    frame k is still queued, then again after wait(): both equal.  a then meshes exactly like b."""
    seen = {}

    def select(k, mesh, scans):
        if k in (5, 7):
            cams = trajectory_cameras([(s["R_true"], s["t_true"]) for s in scans[k - 2:k + 1]])
            mesh.wait()
            sel = mesh.texture_select(as_tuples(cams), vertices=False)
            seen[k] = (cams, sel, images_for(cams, sel, 1.0, "random", seed=k))

    def render(k, mesh, scans):
        if k in (5, 7):
            cams, sel, imgs = seen[k]
            queued = mesh.render_textured(tup(cams[1]), sel, as_tuples(cams), imgs)   # behind frame k, still queued
            mesh.wait()
            same(queued, mesh.render_textured(tup(cams[1]), sel, as_tuples(cams), imgs))
            seen[("n", k)] = queued["counts"]["textured"]

    _, b, _ = lio_chain(cuda_lib, 10, between=select)
    _, a, _ = lio_chain(cuda_lib, 10, between=render)
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
    imgs = images_for(cams, sel, 1.0, "random")
    view = cams[0]
    vw, _ = api.texture_cameras([tup(view)])
    arr, n = api.texture_cameras(as_tuples(cams))
    ia, _, keep = api.texture_images(imgs)
    cam = np.ascontiguousarray(sel["cam"], np.int32)
    uv = np.ascontiguousarray(sel["uv"], np.float32)
    w, h = view["width"], view["height"]
    rgb = np.full((h, w, 3), 77, np.uint8)
    counts = np.full(8, -3, np.int64)
    i32, f32 = C.POINTER(C.c_int32), C.POINTER(C.c_float)

    def rt(cfg=None, v=vw, c=cam, u=uv, nf=None, images=ia, on_device=0, truth=None, out=rgb):
        cfg = cfg or api._TexViewCfg(0.1, 1000.0, 0, (C.c_uint8 * 3)(128, 128, 128), (C.c_uint8 * 3)(0, 0, 0), 0)
        return L.immesh_mesh_render_textured(mesh._h, v, C.byref(cfg), arr, n, images, on_device, c.ctypes.data_as(i32), u.ctypes.data_as(f32),
                                             len(c) if nf is None else nf, truth, None if out is None else out.ctypes.data_as(C.c_void_p), None, None, None,
                                             counts.ctypes.data_as(C.POINTER(C.c_int64)))
    for cfg in (api._TexViewCfg(0.0, 1000.0, 0, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), 0), api._TexViewCfg(2.0, 1.0, 0, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), 0),
                api._TexViewCfg(0.1, float("inf"), 0, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), 0), api._TexViewCfg(0.1, 1000.0, 2, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), 0),
                api._TexViewCfg(0.1, 1000.0, 0, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), -1), api._TexViewCfg(0.1, 1000.0, 0, (C.c_uint8 * 3)(), (C.c_uint8 * 3)(), 100)):
        assert rt(cfg=cfg) == -1
    bv, _ = api.texture_cameras([(0, h, view["K"], view["R"], view["t"])])
    assert rt(v=bv) == -1
    assert rt(nf=len(cam) - 1) == -1, "rows of another mesh state"
    bad = cam.copy()
    bad[0] = n
    assert rt(c=bad) == -1
    bu = uv.copy()
    bu[np.nonzero(cam >= 0)[0][0], 2] = np.nan
    assert rt(u=bu) == -1
    assert rt(on_device=2) == -1
    assert rt(images=None) == -1, "rgb with the query"
    assert rt(images=None, out=None) == 0 and counts[0] > 0
    tb, _, tk = api.texture_images([np.zeros((h, w + 1, 3), np.uint8)])
    assert rt(truth=tb) == -1, "truth of another size"
    none, _, _ = api.texture_images([None] * len(cams))
    assert rt(images=none) == -1, "a NULL image for a needed camera"
    assert (rgb == 77).all() and (counts[4:] == 0).all(), "nothing written by the refused calls"
    assert L.immesh_mesh_render_textured(mesh._h, vw, None, arr, n, ia, 0, cam.ctypes.data_as(i32), uv.ctypes.data_as(f32), len(cam), None, None, None, None,
                                         None, None) == -1
    assert rt() == 0 and not (rgb == 77).all()
    del keep, tk
    # the handle still meshes after the refused calls
    r = mesh.texture_select(as_tuples(cams), vertices=False)
    assert np.array_equal(r["cam"], sel["cam"])
