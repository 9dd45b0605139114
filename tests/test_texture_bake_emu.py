"""CPU tier of the texture atlas (immesh_mesh_texture_bake): the device bodies and argument check (immesh_b200/csrc/texture_bake_core.cuh)
run by the host emulation (tests/texture_bake/emu_texture_bake.cpp) in the device call's orchestration, byte-equal to the numpy
restatement (tests/texture_bake_reference.py) on hand-made and random rows; property checks that do not depend on the restatement
(slot ownership and bilinear footprints, cells that do not overlap, ramp images sampled at the mapped point); the count query,
IMMESH_E_CAPACITY and the error cases; immesh_write_png read back with zlib; the OBJ export of a bake through immesh_write_obj_textured."""
import ctypes as C
import struct
import zlib

import numpy as np
import pytest

from texture_bake_reference import bake as ref_bake, owner, slot_triangle


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    L = C.CDLL(build.build_texture_bake())
    L.emu_texture_bake_error.restype = C.c_char_p
    return L


def cams_of(sizes):
    from immesh_b200 import api
    return api.texture_cameras([(w, h, (100.0, 100.0, (w - 1) / 2, (h - 1) / 2), np.eye(3), np.zeros(3)) for w, h in sizes])


def emu_bake(lib, sel_wh, images, cam, uv, page_size=256, max_cell=64, max_image_bytes=0, cap_pages=None, on_device=0, query=False):
    """(rc, dict(pages, page, uv, n_pages, counts)) of the emulation; cap_pages None: exactly the pages needed"""
    from immesh_b200.api import _AtlasCfg, texture_images
    arr, n_cams = cams_of(sel_wh)
    imgs, _, keep = texture_images(images)
    cam = np.ascontiguousarray(cam, np.int32).reshape(-1)
    uv = np.ascontiguousarray(uv, np.float32).reshape(-1, 6)
    n = len(cam)
    cfg = _AtlasCfg(page_size, max_cell, max_image_bytes)
    vp = C.c_void_p
    lib.emu_texture_bake.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int64, vp, vp, C.c_int, vp, vp, vp, vp]
    npg = C.c_int(-7)
    page = np.full(max(n, 1), -5, np.int32)
    auv = np.full((max(n, 1), 6), np.nan, np.float32)
    counts = np.zeros(4, np.int64)

    def call(pages, cap):
        return lib.emu_texture_bake(C.cast(arr, vp), n_cams, C.cast(imgs, vp), on_device, cam.ctypes.data, uv.ctypes.data, n, C.addressof(cfg),
                                    None if pages is None else pages.ctypes.data, cap, page.ctypes.data, auv.ctypes.data, C.addressof(npg),
                                    counts.ctypes.data)
    rc = call(None, 0)
    if rc != 0 or query:
        return rc, dict(page=page[:n], uv=auv[:n], n_pages=npg.value, counts=counts)
    cap = npg.value if cap_pages is None else cap_pages
    pages = np.full((max(cap, 1), page_size, page_size, 3), 77, np.uint8)
    page[:] = -5
    auv[:] = np.nan
    rc = call(pages, cap)
    del keep
    return rc, dict(pages=pages[:npg.value], page=page[:n], uv=auv[:n], n_pages=npg.value, counts=counts)


def check(lib, sel_wh, images, cam, uv, **kw):
    """the emulation equals the restatement byte for byte; returns the result"""
    rc, got = emu_bake(lib, sel_wh, images, cam, uv, **kw)
    assert rc == 0, lib.emu_texture_bake_error()
    ref = ref_bake(sel_wh, images, cam, uv, page_size=kw.get("page_size", 256), max_cell=kw.get("max_cell", 64))
    assert got["n_pages"] == ref["n_pages"], (got["n_pages"], ref["n_pages"])
    assert np.array_equal(got["page"], ref["page"])
    t = np.asarray(cam) >= 0
    assert np.array_equal(got["uv"][t].view(np.uint32), ref["uv"][t].view(np.uint32))
    assert np.isnan(got["uv"][~t]).all(), "untextured rows keep the caller's atlas_uv"
    assert np.array_equal(got["counts"], ref["counts"]), (got["counts"], ref["counts"])
    assert np.array_equal(got["pages"], ref["pages"]), int((got["pages"] != ref["pages"]).any(axis=-1).sum())
    return got


def random_image(rng, w, h):
    return rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)


def ramp_image(w, h, k):
    """R grows with x, G with y, B the camera's constant"""
    x = np.arange(w, dtype=np.float64)
    y = np.arange(h, dtype=np.float64)
    img = np.zeros((h, w, 3), np.uint8)
    img[..., 0] = np.round(x * 255.0 / max(w - 1, 1))[None, :]
    img[..., 1] = np.round(y * 255.0 / max(h - 1, 1))[:, None]
    img[..., 2] = (40 * k + 20) % 256
    return img


def tri(cx, cy, r, a=0.3):
    """a triangle of circumradius r around (cx, cy)"""
    ang = a + np.array([0.0, 2.1, 4.2])
    return np.stack([cx + r * np.cos(ang), cy + r * np.sin(ang)], axis=1).reshape(6).astype(np.float32)


def random_rows(rng, sel_wh, n, untextured=0.2, big=0.1):
    cam = rng.integers(0, len(sel_wh), n).astype(np.int32)
    cam[rng.random(n) < untextured] = -1
    uv = np.zeros((n, 6), np.float32)
    for r in range(n):
        w, h = sel_wh[max(cam[r], 0)]
        rad = rng.uniform(20, 90) if rng.random() < big else rng.uniform(0.0, 12.0)
        uv[r] = tri(rng.uniform(0, w - 1), rng.uniform(0, h - 1), rad, rng.uniform(0, 6.3))
    uv[cam < 0] = np.nan
    return cam, uv


# ---- hand-made rows against the restatement

def test_one_facet(lib):
    rng = np.random.default_rng(1)
    g = check(lib, [(64, 48)], [random_image(rng, 64, 48)], [0], [tri(30, 20, 5)])
    assert g["n_pages"] == 1 and g["counts"].tolist() == [1, 0, 1, 15 * 16 // 2]   # edges of 8.7 px: a 16-texel cell, slot 0


def test_odd_class_and_every_class(lib):
    rng = np.random.default_rng(2)
    # radii giving cells of 8, 16, 32, 64; an odd count in each class leaves one slot empty
    rows = [tri(100, 100, r) for r in (1.0, 1.5, 4.0, 5.0, 5.5, 10.0, 20.0, 25.0, 30.0)]
    img = random_image(rng, 256, 200)
    g = check(lib, [(256, 200)], [img], np.zeros(len(rows), np.int32), np.array(rows), max_cell=64)
    assert g["counts"][2] >= 5
    check(lib, [(256, 200)], [img], np.zeros(len(rows), np.int32), np.array(rows), max_cell=16)   # facets capped at max_cell
    check(lib, [(256, 200)], [img], np.zeros(len(rows), np.int32), np.array(rows), max_cell=8)
    big = [tri(100, 100, r) for r in (60.0, 90.0, 120.0)]
    check(lib, [(256, 200)], [img], np.zeros(3, np.int32), np.array(big), page_size=512, max_cell=256)


def test_degenerate_and_border_uv(lib):
    rng = np.random.default_rng(3)
    img = random_image(rng, 40, 30)
    rows = np.array([[5, 5, 5, 5, 5, 5], [0, 0, 10, 0, 20, 0], [0, 0, 39, 0, 0, 29], [39, 29, 39, 0, 0, 29],
                     [-0.5, -0.5, 39.5, -0.5, -0.5, 29.5], [-3, -2, 45, 10, 20, 35]], np.float32)
    check(lib, [(40, 30)], [img], np.zeros(len(rows), np.int32), rows)


def test_images_larger_and_smaller_than_the_selection(lib):
    rng = np.random.default_rng(4)
    cam, uv = random_rows(rng, [(80, 60), (80, 60), (50, 40)], 60)
    imgs = [random_image(rng, 160, 120), random_image(rng, 40, 30), random_image(rng, 77, 33)]
    check(lib, [(80, 60), (80, 60), (50, 40)], imgs, cam, uv)


def test_untextured_rows_several_pages_and_nothing_textured(lib):
    rng = np.random.default_rng(5)
    sel = [(120, 90), (120, 90)]
    cam, uv = random_rows(rng, sel, 400, untextured=0.3, big=0.5)
    g = check(lib, sel, [random_image(rng, 120, 90), random_image(rng, 120, 90)], cam, uv, page_size=256, max_cell=64)
    assert g["n_pages"] >= 3 and (g["page"] == -1).sum() == (cam < 0).sum()
    none = check(lib, sel, [None, None], np.full(5, -1, np.int32), np.full((5, 6), np.nan, np.float32))
    assert none["n_pages"] == 0 and none["counts"].tolist() == [0, 5, 0, 0]
    empty = check(lib, sel, [None, None], np.zeros(0, np.int32), np.zeros((0, 6), np.float32))
    assert empty["n_pages"] == 0


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_random_rows(lib, seed):
    rng = np.random.default_rng(seed)
    sel = [(int(rng.integers(40, 200)), int(rng.integers(30, 150))) for _ in range(4)]
    cam, uv = random_rows(rng, sel, 300)
    scale = rng.choice([0.5, 1.0, 2.0])
    imgs = [random_image(rng, max(1, int(w * scale)), max(1, int(h * scale))) for w, h in sel]
    imgs[3] = None
    cam[cam == 3] = -1
    check(lib, sel, imgs, cam, uv, page_size=256, max_cell=int(rng.choice([16, 32, 64])))


# ---- properties that do not depend on the restatement

@pytest.mark.parametrize("S", [8, 16, 32, 64, 128])
def test_slot_ownership_and_bilinear_footprints(S):
    own = owner(S)
    assert (own == 0).sum() == (S - 1) * S // 2 and (own == 1).sum() == S * (S + 1) // 2
    rng = np.random.default_rng(S)
    for slot in (0, 1):
        c = np.array(slot_triangle(S, slot), np.float64)
        w = rng.dirichlet((1, 1, 1), size=4000)
        w = np.concatenate([w, np.eye(3), [[0.5, 0.5, 0], [0, 0.5, 0.5], [0.5, 0, 0.5]]])
        pts = w @ c
        x0, y0 = np.floor(pts[:, 0]).astype(int), np.floor(pts[:, 1]).astype(int)
        for dx in (0, 1):
            for dy in (0, 1):
                xs, ys = x0 + dx, y0 + dy
                wx = np.where(dx, pts[:, 0] - x0, 1 - (pts[:, 0] - x0))
                wy = np.where(dy, pts[:, 1] - y0, 1 - (pts[:, 1] - y0))
                touched = wx * wy > 0
                assert ((xs[touched] >= 0) & (xs[touched] < S) & (ys[touched] >= 0) & (ys[touched] < S)).all()
                assert (own[ys[touched], xs[touched]] == slot).all()


def test_cells_do_not_overlap(lib):
    rng = np.random.default_rng(7)
    sel = [(200, 150)] * 3
    cam, uv = random_rows(rng, sel, 700, untextured=0.1, big=0.3)
    rc, g = emu_bake(lib, sel, [random_image(rng, 200, 150) for _ in sel], cam, uv, page_size=256, max_cell=64)
    assert rc == 0
    P = 256
    cover = np.zeros((g["n_pages"], P, P), np.int32)
    cells = {}
    for r in np.nonzero(cam >= 0)[0]:
        u, v = g["uv"][r, 0::2], g["uv"][r, 1::2]
        lo = np.array([u.min(), v.min()])
        S = int(max(u.max() - u.min(), v.max() - v.min())) + 4
        ox, oy = int(lo[0]) // 8 * 8, int(lo[1]) // 8 * 8
        if u[0] > u[1]:   # slot 1: corner 0 is (S - 2, S - 2)
            ox, oy = int(u[0]) + 2 - S, int(v[0]) + 2 - S
        cells.setdefault((g["page"][r], ox, oy), S)
        assert cells[(g["page"][r], ox, oy)] == S
        assert ox % 8 == 0 and oy % 8 == 0 and 0 <= ox and ox + S <= P and 0 <= oy and oy + S <= P
    for (pg, ox, oy), S in cells.items():
        cover[pg, oy:oy + S, ox:ox + S] += 1
    assert cover.max() == 1, "two cells overlap"
    assert len(cells) == g["counts"][2]
    assert all(((cover[p] > 0).sum() <= P * P) for p in range(g["n_pages"]))


def test_ramp_images_hold_the_mapped_point(lib):
    """every texel strictly inside a slot triangle holds the ramp at the source point its barycentrics map to, within 1"""
    rng = np.random.default_rng(8)
    sel = [(160, 120), (160, 120)]
    sizes = [(320, 240), (97, 61)]
    imgs = [ramp_image(w, h, k) for k, (w, h) in enumerate(sizes)]
    cam, uv = random_rows(rng, sel, 200, untextured=0.0, big=0.3)
    rc, g = emu_bake(lib, sel, imgs, cam, uv, page_size=512, max_cell=64)
    assert rc == 0
    checked = 0
    for r in range(len(cam)):
        k = cam[r]
        W, H = sizes[k]
        src = np.array(uv[r], np.float64).reshape(3, 2)
        src[:, 0] = (src[:, 0] + 0.5) * W / sel[k][0] - 0.5
        src[:, 1] = (src[:, 1] + 0.5) * H / sel[k][1] - 0.5
        dst = np.array(g["uv"][r], np.float64).reshape(3, 2)
        M = np.array([dst[1] - dst[0], dst[2] - dst[0]]).T
        x0, x1 = int(dst[:, 0].min()), int(dst[:, 0].max())
        y0, y1 = int(dst[:, 1].min()), int(dst[:, 1].max())
        for ty in range(y0, y1 + 1):
            for tx in range(x0, x1 + 1):
                ab = np.linalg.solve(M, np.array([tx, ty], np.float64) - dst[0])
                if not (ab[0] > 1e-9 and ab[1] > 1e-9 and ab.sum() < 1 - 1e-9):
                    continue
                p = src[0] + ab[0] * (src[1] - src[0]) + ab[1] * (src[2] - src[0])
                px, py = np.clip(p[0], 0, W - 1), np.clip(p[1], 0, H - 1)
                want = np.array([px * 255.0 / (W - 1), py * 255.0 / (H - 1)])
                got = g["pages"][g["page"][r], ty, tx].astype(np.float64)
                assert np.abs(got[:2] - want).max() <= 1.0 + 1e-9, (r, tx, ty, got, want)
                assert got[2] == (40 * k + 20) % 256
                checked += 1
    assert checked > 2000


# ---- the contract

def test_count_query_and_capacity(lib):
    rng = np.random.default_rng(9)
    sel = [(120, 90)]
    cam, uv = random_rows(rng, sel, 300, untextured=0.0, big=0.6)
    imgs = [random_image(rng, 120, 90)]
    rc, q = emu_bake(lib, sel, imgs, cam, uv, query=True)
    assert rc == 0 and q["n_pages"] >= 2
    assert (q["page"] >= 0).all() and not np.isnan(q["uv"]).any()
    rc, full = emu_bake(lib, sel, imgs, cam, uv)
    assert np.array_equal(q["page"], full["page"]) and np.array_equal(q["uv"], full["uv"])
    rc, short = emu_bake(lib, sel, imgs, cam, uv, cap_pages=q["n_pages"] - 1)
    assert rc == -3 and short["n_pages"] == q["n_pages"]
    assert (short["page"] == -5).all() and np.isnan(short["uv"]).all() and (short["pages"] == 77).all(), "nothing written"


def test_error_cases(lib):
    rng = np.random.default_rng(10)
    sel = [(64, 48), (64, 48)]
    img = random_image(rng, 64, 48)
    cam = np.array([0, 1, -1], np.int32)
    uv = np.array([tri(30, 20, 5)] * 3)

    def rc(**kw):
        args = dict(sel_wh=sel, images=[img, img], cam=cam, uv=uv)
        args.update(kw)
        return emu_bake(lib, args.pop("sel_wh"), args.pop("images"), args.pop("cam"), args.pop("uv"), **args)[0]
    assert rc() == 0
    for ps, mc in ((128, 8), (300, 8), (16384, 64), (256, 4), (256, 12), (256, 512)):
        assert rc(page_size=ps, max_cell=mc) == -1, (ps, mc)
    assert rc(max_image_bytes=-1) == -1
    assert rc(on_device=2) == -1
    assert rc(cam=np.array([0, 2, -1], np.int32)) == -1 and rc(cam=np.array([0, -2, -1], np.int32)) == -1
    bad = uv.copy()
    bad[1, 3] = np.inf
    assert rc(uv=bad) == -1
    bad[1, 3] = np.nan
    assert rc(uv=bad) == -1
    bad = uv.copy()
    bad[2] = np.nan   # an untextured row's uv is not read
    assert rc(uv=bad) == 0
    assert rc(images=[img, None]) == -1 and rc(images=[None, img]) == -1
    assert rc(images=[img, img], max_image_bytes=64 * 48 * 3 - 1) == -1 and rc(max_image_bytes=64 * 48 * 3) == 0
    assert rc(images=[img, np.zeros((0, 5, 3), np.uint8)]) == -1
    assert rc(sel_wh=[(64, 48), (0, 48)]) == -1


def test_short_pitch_is_refused(lib):
    from immesh_b200.api import _AtlasCfg, _TexImage
    arr, n_cams = cams_of([(64, 48)])
    img = np.zeros((48, 64, 3), np.uint8)
    imgs = (_TexImage * 1)(_TexImage(img.ctypes.data, 64, 48, 3 * 64 - 1))
    cam, uv = np.zeros(1, np.int32), tri(30, 20, 5)
    cfg = _AtlasCfg(256, 64, 0)
    npg = C.c_int(0)
    vp = C.c_void_p
    lib.emu_texture_bake.argtypes = [vp, C.c_int, vp, C.c_int, vp, vp, C.c_int64, vp, vp, C.c_int, vp, vp, vp, vp]
    assert lib.emu_texture_bake(C.cast(arr, vp), n_cams, C.cast(imgs, vp), 0, cam.ctypes.data, uv.ctypes.data, 1, C.addressof(cfg), None, 0, None, None,
                                C.addressof(npg), None) == -1


# ---- PNG and OBJ export

def read_png(path):
    """(width, height, rgb) of an 8-bit RGB PNG with filter-0 rows; every chunk's CRC checked"""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, ihdr, types = 8, b"", None, []
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        typ, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert zlib.crc32(typ + body) == crc, typ
        types.append(typ)
        if typ == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif typ == b"IDAT":
            idat += body
        pos += 12 + n
    assert types[0] == b"IHDR" and types[-1] == b"IEND"
    w, h, depth, color, comp, filt, inter = ihdr
    assert (depth, color, comp, filt, inter) == (8, 2, 0, 0, 0)
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    return w, h, raw[:, 1:].reshape(h, w, 3)


@pytest.mark.parametrize("w,h", [(1, 1), (7, 5), (300, 200), (40000, 1)])
def test_png_round_trip(tmp_path, w, h):
    from immesh_b200 import api
    rgb = np.random.default_rng(w).integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    path = str(tmp_path / "p.png")
    api.write_png(path, rgb)
    rw, rh, back = read_png(path)
    assert (rw, rh) == (w, h) and np.array_equal(back, rgb)
    lib = api.load_library()
    assert lib.immesh_write_png(path.encode(), rgb.ctypes.data_as(C.c_void_p), 0, h) == -1
    assert lib.immesh_write_png(path.encode(), None, w, h) == -1
    assert lib.immesh_write_png(str(tmp_path / "no" / "p.png").encode(), rgb.ctypes.data_as(C.c_void_p), w, h) == -1


def test_obj_export_of_a_bake(lib, tmp_path):
    from immesh_b200 import api
    from texture_reference import read_obj
    rng = np.random.default_rng(12)
    sel = [(120, 90), (120, 90)]
    cam, uv = random_rows(rng, sel, 120, untextured=0.2, big=0.5)
    rc, g = emu_bake(lib, sel, [random_image(rng, 120, 90) for _ in sel], cam, uv, page_size=256, max_cell=64)
    assert rc == 0 and g["n_pages"] >= 2
    n = len(cam)
    v = rng.normal(size=(n + 2, 3)).astype(np.float32)
    t = np.stack([np.arange(n), np.arange(n) + 1, np.arange(n) + 2], axis=1).astype(np.int32)
    fl = np.ones(n, np.int32)
    files = []
    for p in range(g["n_pages"]):
        files.append(f"atlas_{p}.png")
        api.write_png(str(tmp_path / files[-1]), g["pages"][p])
    P = 256
    obj, mtl = str(tmp_path / "m.obj"), str(tmp_path / "m.mtl")
    api.write_obj_textured(obj, mtl, v, t, fl, g["page"], g["uv"], [(P, P)] * g["n_pages"], files)
    rv, rvt, groups, _, mats = read_obj(obj, mtl)
    assert [gr[0] for gr in groups] == [f"tex_{p}" for p in range(g["n_pages"])] + ["untextured"]
    assert mats == {**{f"tex_{p}": files[p] for p in range(g["n_pages"])}, "untextured": None}
    rows = np.concatenate([np.nonzero(g["page"] == p)[0] for p in range(g["n_pages"])])
    vt = np.asarray(rvt, np.float64)
    assert np.array_equal(vt[:, 0] * P - 0.5, g["uv"][rows][:, 0::2].reshape(-1).astype(np.float64))
    assert np.array_equal((1.0 - vt[:, 1]) * P - 0.5, g["uv"][rows][:, 1::2].reshape(-1).astype(np.float64))
    for p in range(g["n_pages"]):
        assert np.array_equal(read_png(str(tmp_path / files[p]))[2], g["pages"][p])
