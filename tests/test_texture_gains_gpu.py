"""GPU tier of the colour equalisation (immesh_mesh_texture_gains, immesh_texture_apply_gains): on the Avia- and HDL-64-shaped meshes with
trajectory cameras (tests/test_texture_gpu.py's), the pair list and sums equal the numpy restatement (tests/texture_gains_reference.py)
bit for bit with host images in one and in several batches and with device images, and the gains are within 1e-8 of a direct sparse
solve.  Recovery: images painted with a world pattern and multiplied by seeded per-camera gains t are equalised so that g_k t_k / (g_c
t_c) is near 1 on every well-sampled pair.  Score: the even cameras texture, the odd ones render against the unscaled painting, and the
equalised images score higher at equal coverage; with t = 1 the gains stay near 1 and the score does not drop.  A call behind queued
frames equals one after wait(), and a handle that equalised meshes like a twin that did not; apply_gains on the device equals numpy; the
error contract (a sharded handle needs two GPUs: its refusal is checked by the CPU tier through the shared argument check)."""
import ctypes as C

import numpy as np
import pytest
import torch

from immesh_b200 import api
from test_texture_gpu import as_tuples, lio_chain, trajectory_cameras, world_mesh
from texture_gains_reference import apply_gains as ref_apply
from texture_gains_reference import pairs as ref_pairs
from texture_gains_reference import solve as ref_solve
from texture_reference import raster_R

pytestmark = pytest.mark.gpu


def tup(c):
    return (c["width"], c["height"], c["K"], c["R"], c["t"])


def painted(mesh, cams, gains=None, seed=0):
    """per camera the image of a smooth seeded pattern painted on the world (render_view's depth unprojected, coloured by the point),
    each channel multiplied by gains [k][ch], rounded and clipped to 255"""
    rng = np.random.default_rng(seed)
    f = rng.uniform(0.5, 2.0, (3, 3))
    ph = rng.uniform(0, 2 * np.pi, 3)
    out = []
    for k, c in enumerate(cams):
        w, h = c["width"], c["height"]
        _, depth = mesh.render_view(c["K"], w, h, 0.1, 1000.0, raster_R(c["R"]), c["t"])
        ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
        fx, fy, cx, cy = c["K"]
        pc = np.stack([(xs - cx) / fx * depth, (ys - cy) / fy * depth, depth.astype(np.float64)], axis=-1)
        pw = pc @ c["R"].T + c["t"]
        img = np.zeros((h, w, 3), np.uint8)
        for ch in range(3):
            v = np.floor(np.clip(127.5 + 127.5 * np.sin(pw @ f[ch] + ph[ch]), 0, 255))
            g = 1.0 if gains is None else gains[k][ch]
            img[..., ch] = np.clip(np.floor(v * g + 0.5), 0, 255).astype(np.uint8)
        img[depth < 0] = 0
        out.append(img)
    return out


def same(a, b):
    assert np.array_equal(a["gains"], b["gains"])
    assert a["counts"] == b["counts"]
    assert np.array_equal(a["pair_cam"], b["pair_cam"]) and np.array_equal(a["pair_sums"], b["pair_sums"])


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_against_restatement_and_image_sources(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    v, tri, fl = mesh.snapshot()
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    t = np.random.default_rng(1).uniform(0.7, 1.3, (len(cams), 3))
    imgs = painted(mesh, cams, t)
    # images larger and smaller than the cameras, and one camera without an image that textures nothing
    imgs[1] = np.repeat(np.repeat(imgs[1], 2, axis=0), 2, axis=1)
    imgs[4] = imgs[4][::2, ::2].copy()
    rows = dict(cam=np.where(sel["cam"] == 5, -1, sel["cam"]), uv=sel["uv"])
    imgs[5] = None
    host = mesh.texture_gains(rows, as_tuples(cams), imgs, pairs=True)
    c = host["counts"]
    assert c["pairs"] >= 4 and c["samples"] > 1000 and c["observers"] == 5 and c["clipped"] > 0, c
    pc, ps, used, clipped = ref_pairs(cams, imgs, rows["cam"], np.nan_to_num(rows["uv"]), v, tri, fl)
    assert np.array_equal(host["pair_cam"], pc) and np.array_equal(host["pair_sums"], ps)
    assert (c["pairs"], c["samples"], c["clipped"]) == (len(pc), used, clipped)
    ref = ref_solve(len(cams), pc, ps)
    assert np.allclose(host["gains"], ref, rtol=1e-8, atol=0) and (host["gains"] > 0).all()
    assert (host["gains"][5] == 1.0).all() and c["unpaired"] >= 1
    one = max(im.nbytes for im in imgs if im is not None)
    same(host, mesh.texture_gains(rows, as_tuples(cams), imgs, pairs=True, max_image_bytes=one))
    same(host, mesh.texture_gains(rows, as_tuples(cams), [None if im is None else torch.from_numpy(im).cuda() for im in imgs], pairs=True))
    # max_pairs overflow
    with pytest.raises(RuntimeError, match="code -3"):
        mesh.texture_gains(rows, as_tuples(cams), imgs, max_pairs=len(pc) - 1)
    # the call wrote nothing on the handle
    for x, y in zip((v, tri, fl), mesh.snapshot()):
        assert np.array_equal(x, y)


# The largest |g_k t_k / (g_c t_c) - 1| over the pairs with >= 1000 samples, sigma_g = 10 (a weak prior, so that the data decides):
# measured 0.0030 (Avia) and 0.0040 (HDL-64) on an NVIDIA H100 80GB HBM3 (700 W); the bound leaves 2.5x margin over the larger for
# the nearest-pixel sampling of a smooth pattern from different views.
RECOVERY_TOL = 0.01


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_recovery_of_seeded_gains(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    t = np.random.default_rng(2).uniform(0.7, 1.3, (len(cams), 3))
    r = mesh.texture_gains(sel, as_tuples(cams), painted(mesh, cams, t), sigma_g=10.0, pairs=True)
    big = r["pair_sums"][:, 0] >= 1000
    assert big.sum() >= 3, r["pair_sums"][:, 0]
    gt = r["gains"] * t
    k, c = r["pair_cam"][big, 0], r["pair_cam"][big, 1]
    dev = np.abs(gt[k] / gt[c] - 1.0).max()
    raw = np.abs(t[k] / t[c] - 1.0).max()
    print(f"recovery {kind}: max |g_k t_k / (g_c t_c) - 1| = {dev:.4f} (unequalised {raw:.4f})")
    assert dev <= RECOVERY_TOL and raw > 4 * RECOVERY_TOL


def loo_scores(mesh, cams, t, **kw):
    """texture with the even cameras from images scaled by t, equalise, render at the odd cameras against the unscaled painting:
    (mean psnr raw, mean psnr equalised, coverages raw, coverages equalised, gains)"""
    truth = painted(mesh, cams)
    scaled = painted(mesh, cams, t)
    even, odd = list(range(0, len(cams), 2)), list(range(1, len(cams), 2))
    train = as_tuples([cams[k] for k in even])
    sel = mesh.texture_select(train, vertices=False)
    raw = [scaled[k] for k in even]
    g = mesh.texture_gains(sel, train, raw, **kw)["gains"]
    eq = mesh.apply_gains(raw, g)
    a, b = [], []
    for k in odd:
        ra = mesh.render_textured(tup(cams[k]), sel, train, raw, truth=truth[k])
        rb = mesh.render_textured(tup(cams[k]), sel, train, eq, truth=truth[k])
        if ra["counts"]["textured"]:
            a.append(ra)
            b.append(rb)
    assert len(a) >= 2
    return (float(np.mean([x["psnr"] for x in a])), float(np.mean([x["psnr"] for x in b])), [x["coverage"] for x in a], [x["coverage"] for x in b], g)


# The mean held-out PSNR gain of the equalised texture over the raw one (default sigmas): measured 2.2 dB (Avia, 24.1 -> 26.3) and
# 5.5 dB (HDL-64, 24.4 -> 29.8) on an NVIDIA H100 80GB HBM3 (700 W); the bound sits below the smaller.  With t = 1 both scores were
# equal to 0.01 dB and the gains within 2e-4 of 1.
SCORE_MARGIN_DB = 1.5


@pytest.mark.parametrize("kind", ["avia", "hdl64"])
def test_held_out_score(cuda_lib, kind):
    mesh, poses = world_mesh(cuda_lib, kind)
    cams = trajectory_cameras(poses)
    # Equalisation recovers the cameras' relative gains; their common level is not observable and the prior keeps it near the mean
    # gain of 1.  So the seeded gains are scaled to a mean of 1 per channel over the training (even) cameras: otherwise the score
    # would measure how far the seed's mean lies from the unscaled truth, not the equalisation.
    t = np.random.default_rng(3).uniform(0.7, 1.3, (len(cams), 3))
    t = t / t[0::2].mean(axis=0)
    raw, eq, cov_a, cov_b, _ = loo_scores(mesh, cams, t)
    print(f"score {kind}: psnr raw {raw:.2f} dB, equalised {eq:.2f} dB")
    assert cov_a == cov_b and min(cov_a) > 0.01
    assert eq >= raw + SCORE_MARGIN_DB, (raw, eq)
    # t = 1: gains near 1, no loss
    raw1, eq1, _, _, g1 = loo_scores(mesh, cams, np.ones((len(cams), 3)))
    print(f"score {kind} t = 1: psnr raw {raw1:.2f} dB, equalised {eq1:.2f} dB, gains in [{g1.min():.4f}, {g1.max():.4f}]")
    assert np.abs(g1 - 1.0).max() < 0.05 and eq1 >= raw1 - 0.1


def test_queued_frames_and_twin(cuda_lib):
    """The twin b (never equalises) selects the rows of the mesh after frame k; handle a, fed the same stream, computes the gains while
    frame k is still queued, then again after wait(): both equal.  a then meshes exactly like b."""
    seen = {}

    def select(k, mesh, scans):
        if k in (5, 7):
            cams = trajectory_cameras([(s["R_true"], s["t_true"]) for s in scans[k - 2:k + 1]])
            mesh.wait()
            sel = mesh.texture_select(as_tuples(cams), vertices=False)
            rng = np.random.default_rng(k)
            seen[k] = (cams, sel, [rng.integers(0, 256, (c["height"], c["width"], 3), np.uint8) for c in cams])

    def gains(k, mesh, scans):
        if k in (5, 7):
            cams, sel, imgs = seen[k]
            queued = mesh.texture_gains(sel, as_tuples(cams), imgs, pairs=True)   # behind frame k, still queued
            mesh.wait()
            same(queued, mesh.texture_gains(sel, as_tuples(cams), imgs, pairs=True))
            seen[("n", k)] = queued["counts"]["pairs"]

    _, b, _ = lio_chain(cuda_lib, 10, between=select)
    _, a, _ = lio_chain(cuda_lib, 10, between=gains)
    assert seen[("n", 7)] > 0
    for x, y in zip(a.snapshot(), b.snapshot()):
        assert np.array_equal(x, y)
    assert a.counts() == b.counts()
    ca, cb = a.changes(0), b.changes(0)
    for key in ("frames", "rows", "vertices"):
        assert np.array_equal(ca[key], cb[key]), key


def test_apply_gains_device_and_error_contract(cuda_lib):
    mesh, poses = world_mesh(cuda_lib, "avia")
    rng = np.random.default_rng(4)
    imgs = [rng.integers(0, 256, (37, 53, 3), np.uint8), None, rng.integers(0, 256, (300, 200, 3), np.uint8)]
    g = np.array([[0.7, 1.0, 1.3], [2.0, 2.0, 2.0], [0.5, 1.5, 0.999]])
    host = mesh.apply_gains(imgs, g)
    dev = mesh.apply_gains([None if im is None else torch.from_numpy(im).cuda() for im in imgs], g)
    for k in (0, 2):
        assert np.array_equal(host[k], ref_apply(imgs[k], g[k])) and np.array_equal(dev[k].cpu().numpy(), host[k])
    assert host[1] is None and dev[1] is None
    # in place on the device, with padded rows
    buf = torch.zeros((37, 60, 3), dtype=torch.uint8, device="cuda")
    view = buf[:, :53]
    view.copy_(torch.from_numpy(imgs[0]).cuda())
    ia, on_dev, keep = api.texture_images([view])
    dp = C.POINTER(C.c_double)
    g0 = np.ascontiguousarray(g[:1])
    assert cuda_lib.immesh_texture_apply_gains(mesh._h, ia, ia, 1, on_dev, g0.ctypes.data_as(dp)) == 0
    assert np.array_equal(view.cpu().numpy(), host[0]) and (buf[:, 53:] == 0).all()
    for bad in ([[np.nan, 1, 1]], [[-1.0, 1, 1]]):
        b = np.ascontiguousarray(bad, np.float64)
        assert cuda_lib.immesh_texture_apply_gains(mesh._h, ia, ia, 1, on_dev, b.ctypes.data_as(dp)) == -1
    assert np.array_equal(view.cpu().numpy(), host[0])
    del keep
    # texture_gains' refusals
    cams = trajectory_cameras(poses)
    sel = mesh.texture_select(as_tuples(cams), vertices=False)
    imgs = painted(mesh, cams)
    for kw in (dict(sigma_n=0.0), dict(sigma_g=float("nan")), dict(max_pairs=0), dict(min_cos=2.0), dict(max_image_bytes=10)):
        with pytest.raises(RuntimeError, match="code -1"):
            mesh.texture_gains(sel, as_tuples(cams), imgs, **kw)
    with pytest.raises(RuntimeError, match="code -1"):
        mesh.texture_gains(dict(cam=sel["cam"][:-1], uv=sel["uv"][:-1]), as_tuples(cams), imgs)
    used = int(sel["cam"][sel["cam"] >= 0][0])
    with pytest.raises(RuntimeError, match="code -1"):
        mesh.texture_gains(sel, as_tuples(cams), [None if k == used else im for k, im in enumerate(imgs)])
    # the handle still works after the refused calls
    r = mesh.texture_gains(sel, as_tuples(cams), imgs)
    assert r["counts"]["pairs"] > 0
