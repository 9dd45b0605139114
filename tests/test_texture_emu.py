"""CPU tier of the textured mesh (immesh_mesh_texture_select): the device bodies (immesh_b200/csrc/texture_core.cuh with the rasteriser
of reinforce.cuh) run by the host emulation (tests/texture/emu_texture.cpp) in the device chain's orchestration, against the numpy
restatement of the selection rule (tests/texture_reference.py) on hand-built scenes with known answers: the nearer of two cameras,
an occluder, a facet partly outside the image, a grazing view, a back-facing camera, equal distances, a degenerate facet, the
min_visible_permille boundary and an empty mesh.  Also immesh_write_obj_textured, read back: counts, winding, texture coordinates and
material groups."""
import ctypes as C
import os

import numpy as np
import pytest

from texture_reference import camera, coverage, raster_R, read_obj, select


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    return C.CDLL(build.build_texture())


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def emu_select(lib, cams, verts, tris, flips, z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False, positions=0,
               smooth=None, flags=None, bin_cap=1 << 30):
    from immesh_b200.api import _TexCfg, texture_cameras
    arr, n = texture_cameras([(c["width"], c["height"], c["K"], c["R"], c["t"]) for c in cams])
    cfg = _TexCfg(z_near, z_far, min_cos, min_visible_permille, 1 if two_sided else 0, positions, 0)
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    tr = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
    fl = np.ascontiguousarray(flips, np.int32).reshape(-1)
    sm = None if smooth is None else np.ascontiguousarray(smooth, np.float64)
    fg = None if flags is None else np.ascontiguousarray(flags, np.uint8)
    nt = len(tr)
    cam = np.zeros(max(nt, 1), np.int32)
    uv = np.full((max(nt, 1), 6), np.nan, np.float32)
    px = np.zeros((max(nt, 1), 2), np.int32)
    counts = np.zeros(4, np.int64)
    over = np.zeros(max(n, 1), np.int32)
    vp = C.c_void_p
    lib.emu_texture_select.argtypes = [vp, C.c_int, vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_longlong, vp, vp, vp, vp, vp]
    lib.emu_texture_select(C.cast(arr, vp), n, C.cast(C.pointer(cfg), vp), _p(v), _p(sm), _p(fg), len(v), _p(tr), _p(fl), nt, bin_cap, _p(cam), _p(uv), _p(px),
                           _p(counts), _p(over))
    return dict(cam=cam[:nt], uv=uv[:nt], px=px[:nt], counts=counts, overflow=over[:n])


def check(lib, cams, verts, tris, flips, **kw):
    """the emulation equals the restatement bit for bit; returns the result"""
    bin_cap = kw.pop("bin_cap", 1 << 30)
    got = emu_select(lib, cams, verts, tris, flips, bin_cap=bin_cap, **kw)
    ref = select(cams, verts, tris, flips, **kw)
    assert np.array_equal(got["cam"], ref["cam"]), (got["cam"], ref["cam"])
    assert np.array_equal(got["px"], ref["px"]), (got["px"], ref["px"])
    assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32)), "texture coordinates differ"
    assert np.array_equal(got["counts"], ref["counts"]), (got["counts"], ref["counts"])
    return got


def look(eye, target, up=(0.0, 0.0, 1.0)):
    """OpenCV camera-to-world rotation at eye looking at target (x right, y down, z forward)"""
    f = np.asarray(target, np.float64) - np.asarray(eye, np.float64)
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(f, r), f], axis=1)


def cam_at(eye, target, w=64, h=48, f=40.0):
    return camera(w, h, (f, f, (w - 1) / 2.0, (h - 1) / 2.0), look(eye, target), eye)


def orient(verts, tris, toward):
    """flips that turn each facet's face-order normal towards the point `toward`"""
    v = np.asarray(verts, np.float64)
    t = np.asarray(tris)
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    g = v[t].mean(axis=1)
    return (np.einsum("ij,ij->i", n, np.asarray(toward) - g) > 0).astype(np.int32)


def wall(x=10.0, half=2.0, n=4):
    """a square grid in the plane x = const, 2 n^2 facets with ascending triples, facing -x"""
    ys = np.linspace(-half, half, n + 1)
    v = np.array([[x, y, z] for z in ys for y in ys], np.float32)
    tris = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1
            tris += [sorted((a, b, c)), sorted((b, d, c))]
    tris = np.array(tris, np.int32)
    return v, tris, orient(v, tris, (x - 100.0, 0.0, 0.0))


def test_nearer_camera_wins(lib):
    v, t, fl = wall()
    cams = [cam_at((2.0, 0.0, 0.0), (10.0, 0.0, 0.0)), cam_at((5.0, 0.0, 0.0), (10.0, 0.0, 0.0), w=96, h=96)]
    r = check(lib, cams, v, t, fl)
    assert (r["cam"] == 1).all(), r["cam"]
    assert r["counts"].tolist() == [len(t), 0, 1, 64 * 48 + 96 * 96]
    assert (r["px"][:, 0] >= 1).all() and (r["px"][:, 0] <= r["px"][:, 1]).all()


def test_occluder_hands_facets_to_the_farther_camera(lib):
    v, t, fl = wall()
    near, far = cam_at((5.0, 0.0, 0.0), (10.0, 0.0, 0.0), w=96, h=96), cam_at((2.0, 0.0, 0.0), (10.0, 0.0, 0.0))
    base = check(lib, [far, near], v, t, fl)
    assert (base["cam"] == 1).all()
    # a square just in front of the nearer camera, hiding the middle of the wall from it
    ov, ot, _ = wall(x=6.0, half=0.5, n=1)
    verts = np.concatenate([v, ov])
    tris = np.concatenate([t, ot + len(v)])
    flips = np.concatenate([fl, orient(ov, ot, (0.0, 0.0, 0.0))])
    r = check(lib, [far, near], verts, tris, flips)
    wall_rows = np.arange(len(t))
    assert (r["cam"][wall_rows] == 0).any(), "no wall facet went to the farther camera"
    assert (r["cam"][len(t):] == 1).all(), "the occluder is textured by the nearer camera"


def test_facet_partly_outside_the_image(lib):
    v, t, fl = wall(half=4.0, n=8)
    cams = [cam_at((6.0, 0.0, 0.0), (10.0, 0.0, 0.0))]
    r = check(lib, cams, v, t, fl)
    won, _ = coverage(cams[0]["K"], 64, 48, 0.1, 1000.0, raster_R(cams[0]["R"]), cams[0]["t"], v, t)
    assert ((won > 0) & (r["cam"] < 0)).any(), "a facet with pixels but a corner outside the image must stay untextured"
    assert (r["cam"] == 0).any()


def test_grazing_view_below_min_cos(lib):
    v, t, fl = wall()
    eye = np.array([10.0 - 8.0 * np.cos(np.radians(80.0)), -8.0 * np.sin(np.radians(80.0)), 0.0])   # 80 degrees off the normal
    cams = [cam_at(eye, (10.0, 0.0, 0.0), w=160, h=120, f=60.0)]
    low = check(lib, cams, v, t, fl, min_cos=0.1)
    high = check(lib, cams, v, t, fl, min_cos=0.5)
    assert (low["cam"] == 0).sum() > 0
    assert (high["cam"] == -1).all()


def test_back_facing_camera(lib):
    v, t, fl = wall()
    cams = [cam_at((16.0, 0.0, 0.0), (10.0, 0.0, 0.0))]
    one = check(lib, cams, v, t, fl)
    two = check(lib, cams, v, t, fl, two_sided=True)
    assert (one["cam"] == -1).all()
    assert (two["cam"] == 0).all()


def test_equal_distances_lower_index_wins(lib):
    v = np.array([[10.0, -1.0, -1.0], [10.0, 1.0, -1.0], [10.0, 0.0, 2.0]], np.float32)   # centroid (10, 0, 0) exactly
    t = np.array([[0, 1, 2]], np.int32)
    fl = orient(v, t, (0.0, 0.0, 0.0))
    a, b = cam_at((4.0, 3.0, 0.0), (10.0, 0.0, 0.0)), cam_at((4.0, -3.0, 0.0), (10.0, 0.0, 0.0))
    assert check(lib, [a, b], v, t, fl)["cam"].tolist() == [0]
    assert check(lib, [b, a], v, t, fl)["cam"].tolist() == [0]
    assert check(lib, [cam_at((3.0, 0.0, 0.0), (10.0, 0.0, 0.0)), b, a], v, t, fl)["cam"].tolist() == [1]


def test_degenerate_facet(lib):
    v, t, fl = wall()
    extra = np.array([[10.0, -1.5, 0.0], [10.0, 0.0, 0.0], [10.0, 1.5, 0.0]], np.float32)   # collinear, in the wall
    verts = np.concatenate([v, extra])
    tris = np.concatenate([t, [[len(v), len(v) + 1, len(v) + 2]]])
    r = check(lib, [cam_at((5.0, 0.0, 0.0), (10.0, 0.0, 0.0), w=96, h=96)], verts, tris, np.concatenate([fl, [1]]))
    assert r["cam"][-1] == -1 and (r["cam"][:-1] == 0).all()


def test_min_visible_permille_boundary(lib):
    v, t, fl = wall(n=2)
    ov, ot, _ = wall(x=8.0, half=0.7, n=1)   # hides part of several wall facets
    verts = np.concatenate([v, ov + np.float32([0.0, 0.6, 0.3])])
    tris = np.concatenate([t, ot + len(v)])
    flips = np.concatenate([fl, orient(ov, ot, (0.0, 0.0, 0.0))])
    c = cam_at((3.0, 0.0, 0.0), (10.0, 0.0, 0.0), w=96, h=96)
    won, cov = coverage(c["K"], 96, 96, 0.1, 1000.0, raster_R(c["R"]), c["t"], verts, tris)
    part = np.nonzero((won > 0) & (won < cov))[0]
    assert len(part) > 0
    f = part[0]
    p = int(1000 * won[f] // cov[f])   # the largest share the facet passes: 1000 won >= p covered
    at = check(lib, [c], verts, tris, flips, min_visible_permille=p)
    above = check(lib, [c], verts, tris, flips, min_visible_permille=p + 1)
    assert at["cam"][f] == 0 and above["cam"][f] == -1
    assert at["px"][f].tolist() == [won[f], cov[f]]


def test_empty_mesh(lib):
    r = check(lib, [cam_at((0.0, 0.0, 0.0), (1.0, 0.0, 0.0))], np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), np.zeros(0, np.int32))
    assert r["counts"].tolist() == [0, 0, 0, 64 * 48]


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_scenes_and_bin_overflow(lib, seed):
    """random triangles around a ring of cameras, smoothed positions on a random half of the vertices, bins normal and overflowing"""
    rng = np.random.default_rng(seed)
    nv, nt = 240, 320
    v = (rng.normal(size=(nv, 3)) * [4.0, 4.0, 1.5]).astype(np.float32)
    t = np.sort(np.stack([rng.choice(nv, 3, replace=False) for _ in range(nt)]), axis=1).astype(np.int32)
    t = np.unique(t, axis=0)
    fl = rng.integers(0, 2, len(t)).astype(np.int32)
    sm = v.astype(np.float64) + rng.normal(scale=0.05, size=(nv, 3))
    flags = rng.integers(0, 2, nv).astype(np.uint8)
    cams = [cam_at((12.0 * np.cos(a), 12.0 * np.sin(a), 2.0), (0.0, 0.0, 0.0), w=80, h=60, f=50.0) for a in np.linspace(0, 2 * np.pi, 7)[:-1]]
    drawn = np.where(flags[:, None] != 0, sm.astype(np.float32), v)
    textured = []
    for kw in (dict(), dict(min_cos=0.3, min_visible_permille=250), dict(two_sided=True, min_visible_permille=600)):
        got = emu_select(lib, cams, v, t, fl, positions=1, smooth=sm, flags=flags, **kw)
        ref = select(cams, drawn, t, fl, **kw)
        for key in ("cam", "px", "counts"):
            assert np.array_equal(got[key], ref[key]), key
        assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32))
        small = emu_select(lib, cams, v, t, fl, positions=1, smooth=sm, flags=flags, bin_cap=8, **kw)
        assert small["overflow"].all()
        for key in ("cam", "px", "counts"):
            assert np.array_equal(small[key], got[key]), key
        assert np.array_equal(small["uv"].view(np.uint32), got["uv"].view(np.uint32))
        textured.append(got["cam"][got["cam"] >= 0])
    assert len(textured[0]) > 20 and len(np.unique(textured[0])) > 2


def test_write_obj_textured(tmp_path):
    from immesh_b200 import api
    lib = api.load_library()
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 0, 0.5]], np.float32)
    t = np.array([[0, 1, 2], [1, 2, 3], [1, 3, 4], [0, 2, 4]], np.int32)
    fl = np.array([1, 0, 1, 0], np.int32)
    cam = np.array([2, -1, 0, 2], np.int32)
    uv = np.full((4, 6), np.nan, np.float32)
    uv[0] = [10.5, 3.0, 20.0, 4.25, 15.0, 30.0]
    uv[2] = [0.0, 0.0, 99.0, 0.0, 50.0, 49.0]
    uv[3] = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]
    wh = np.array([[100, 50], [7, 7], [640, 480]], np.int32)
    files = ["img/a 0.png", "img/b.png", "img/c.jpg"]
    obj, mtl = str(tmp_path / "mesh.obj"), str(tmp_path / "mesh.mtl")
    api.write_obj_textured(obj, mtl, v, t, fl, cam, uv, wh, files, lib=lib)
    rv, rvt, groups, mtllib, mats = read_obj(obj, mtl)
    assert mtllib == "mesh.mtl"
    assert np.array_equal(rv.astype(np.float32), v)
    assert [g[0] for g in groups] == ["tex_0", "tex_2", "untextured"]
    assert mats == {"tex_0": "img/a 0.png", "tex_2": "img/c.jpg", "untextured": None}
    order = [2, 0, 3, 1]   # camera 0, then camera 2 in row order, then the untextured
    faces = np.concatenate([g[1] for g in groups])
    face_order = np.where(fl[:, None] != 0, t, t[:, [0, 2, 1]])
    assert np.array_equal(faces, face_order[order])
    assert groups[2][2] is None
    tex = np.concatenate([groups[0][2], groups[1][2]])
    assert np.array_equal(tex, np.arange(9).reshape(3, 3)) and len(rvt) == 9
    for j, row in enumerate(order[:3]):
        W, H = wh[cam[row]]
        u, vv = uv[row, 0::2].astype(np.float64), uv[row, 1::2].astype(np.float64)
        assert np.array_equal(rvt[3 * j:3 * j + 3, 0], (u + 0.5) / W)
        assert np.array_equal(rvt[3 * j:3 * j + 3, 1], 1.0 - (vv + 0.5) / H)
    # errors: a vertex outside the array, a camera index outside [-1, n_cams)
    with pytest.raises(RuntimeError):
        api.write_obj_textured(obj, mtl, v[:3], t, fl, cam, uv, wh, files, lib=lib)
    with pytest.raises(RuntimeError):
        api.write_obj_textured(obj, mtl, v, t, fl, np.array([3, -1, 0, 2], np.int32), uv, wh, files, lib=lib)
    assert os.path.getsize(obj) > 0
