"""CPU tier of the texturing queued behind every frame (immesh_mesh_texture_enable / _rows): the device bodies
(immesh_b200/csrc/texture_core.cuh with the rasteriser of reinforce.cuh) run by the host emulation (tests/texture_online/
emu_texture_online.cpp) in the device stage's orchestration, against the numpy restatement of the fold
(tests/texture_online_reference.py), byte for byte, on hand-made sequences: a nearer later camera, an equal distance, a facet that dies
and comes back, a flip that changes between frames, a frame without a camera, a slot allocated but never live, and the state grown in
the middle of a run; and on random sequences."""
import ctypes as C

import numpy as np
import pytest

from texture_online_reference import compose, fold, rows

W, H, FOC = 64, 48, 40.0
K = (FOC, FOC, (W - 1) / 2.0, (H - 1) / 2.0)


@pytest.fixture(scope="module")
def lib():
    from immesh_b200 import build
    return C.CDLL(build.build_texture_online())


def look(eye, target, up=(0.0, 1.0, 0.0)):
    """OpenCV camera-to-world rotation at eye looking at target (x right, y down, z forward)"""
    f = np.asarray(target, np.float64) - np.asarray(eye, np.float64)
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    return np.stack([r, np.cross(f, r), f], axis=1)


# the rig: the colour camera turned and shifted in the sensor frame
RIG_R = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]) @ look((0, 0, 0), (0.05, 0.02, 1.0))
RIG_T = np.array([0.11, -0.07, 0.03])
RIG = dict(width=W, height=H, K=K, R=RIG_R, t=RIG_T)


def sensor_pose(eye, target):
    """the sensor pose whose rig camera sits (nearly) at eye looking at target"""
    Rc = look(eye, target)
    R_f = Rc @ RIG_R.T
    return R_f, np.asarray(eye, np.float64) - R_f @ RIG_T


def grid(n=4, size=4.0, z=0.0, bump=0.0, seed=0):
    """vertices of an n x n grid on the plane z (plus a random bump) and its triangles, ascending triples"""
    rng = np.random.default_rng(seed)
    xs = np.linspace(-size / 2, size / 2, n)
    v = np.array([[x, y, z + bump * rng.standard_normal()] for y in xs for x in xs], np.float32)
    t = []
    for j in range(n - 1):
        for i in range(n - 1):
            a, b, c, d = j * n + i, j * n + i + 1, (j + 1) * n + i, (j + 1) * n + i + 1
            t += [sorted((a, b, d)), sorted((a, d, c))]
    return v, np.array(t, np.int64)


def up_flips(v, t):
    """flips that turn every face-order normal to +z"""
    n = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    return (n[:, 2] > 0).astype(np.int32)   # flip 1: p0 p1 p2 is the face order


def run(lib, verts, frames, n_alloc, row_slots, tris_of_slot, flip_now, cfg=None):
    """emulation and restatement of one sequence; frames: dicts of number, kind (0 none, 1 rig pose, 2 caller), pose (R, t), cap,
    live: list of (slot, flip).  Returns (emulated, restated) rows"""
    from immesh_b200.api import _TexCfg, texture_cameras
    cfg = {**dict(z_near=0.1, z_far=1000.0, min_cos=0.0, min_visible_permille=0, two_sided=False), **(cfg or {})}
    arr, _ = texture_cameras([(W, H, K, RIG_R, RIG_T)])
    ccfg = _TexCfg(cfg["z_near"], cfg["z_far"], cfg["min_cos"], cfg["min_visible_permille"], 1 if cfg["two_sided"] else 0, 0, 0)
    nf = len(frames)
    number = np.array([f["number"] for f in frames], np.int32)
    kind = np.array([f["kind"] for f in frames], np.int32)
    pose = np.zeros((max(nf, 1), 12), np.float64)
    for i, f in enumerate(frames):
        if f["kind"]:
            pose[i, :9] = np.asarray(f["pose"][0], np.float64).reshape(9)
            pose[i, 9:] = f["pose"][1]
    cap = np.array([f["cap"] for f in frames], np.int32)
    off = np.zeros(nf + 1, np.int32)
    slot, abc, flip = [], [], []
    for i, f in enumerate(frames):
        for s, fl in f["live"]:
            slot.append(s)
            abc.append(tris_of_slot[s])
            flip.append(fl)
        off[i + 1] = len(slot)
    slot = np.array(slot + [0], np.int32)
    abc = np.array(abc + [[0, 0, 0]], np.int32)
    flip = np.array(flip + [0], np.int32)
    rs = np.array(list(row_slots) + [0], np.int32)
    nr = len(row_slots)
    cam = np.zeros(max(nr, 1), np.int32)
    uv = np.full((max(nr, 1), 6), np.nan, np.float32)
    px = np.zeros((max(nr, 1), 2), np.int32)
    counts = np.zeros(4, np.int64)
    fr = np.zeros(max(n_alloc, 1), np.int32)
    nfo = C.c_int(0)
    v = np.ascontiguousarray(verts, np.float32)
    vp = C.c_void_p
    p = lambda a: a.ctypes.data_as(vp)
    lib.emu_texture_online.argtypes = [vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.emu_texture_online(C.cast(arr, vp), C.cast(C.pointer(ccfg), vp), p(v), len(v), nf, p(number), p(kind), p(pose), p(cap), p(off), p(slot), p(abc), p(flip),
                           n_alloc, p(rs), nr, p(cam), p(uv), p(px), p(counts), p(fr), C.cast(C.byref(nfo), vp))
    got = dict(cam=cam[:nr], uv=uv[:nr], px=px[:nr], counts=counts, frames=fr[:nfo.value])
    ref_frames = []
    for f in frames:
        tris = np.array([tris_of_slot[s] for s, _ in f["live"]], np.int64).reshape(-1, 3)
        fls = np.array([fl for _, fl in f["live"]], np.int32)
        d = dict(number=f["number"], verts=v, tris=tris, flips=fls)
        if f["kind"] == 1:
            d["pose"] = f["pose"]
        elif f["kind"] == 2:
            d["caller"] = f["pose"]
        ref_frames.append(d)
    state, pixels = fold(RIG, ref_frames, **cfg)
    ref = rows(state, pixels, np.array([tris_of_slot[s] for s in row_slots], np.int64).reshape(-1, 3), [flip_now[s] for s in row_slots])
    return got, ref


def same(got, ref):
    assert np.array_equal(got["cam"], ref["cam"]), (got["cam"], ref["cam"])
    assert np.array_equal(got["px"], ref["px"]), (got["px"], ref["px"])
    assert np.array_equal(got["uv"].view(np.uint32), ref["uv"].view(np.uint32)), "texture coordinates differ"
    assert np.array_equal(got["counts"], ref["counts"]), (got["counts"], ref["counts"])
    assert np.array_equal(got["frames"], ref["frames"]), (got["frames"], ref["frames"])


def scene():
    v, t = grid()
    fl = up_flips(v.astype(np.float64), t)
    return v, [tuple(int(x) for x in tri) for tri in t], fl


def all_live(tris, fl):
    return [(s, int(fl[s])) for s in range(len(tris))]


def test_compose_matches_written_order():
    R_f, t_f = sensor_pose((0.3, -0.2, 6.0), (0.1, 0.0, 0.0))
    R, t = compose(RIG_R, RIG_T, R_f, t_f)
    assert np.allclose(R, R_f @ RIG_R) and np.allclose(t, R_f @ RIG_T + t_f)


def test_nearer_later_camera_takes_over(lib):
    v, tris, fl = scene()
    live = all_live(tris, fl)
    frames = [dict(number=3, kind=1, pose=sensor_pose((0.2, 0.1, 9.0), (0, 0, 0)), cap=64, live=live),
              dict(number=4, kind=1, pose=sensor_pose((0.1, 0.0, 6.0), (0, 0, 0)), cap=64, live=live)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, fl)
    same(got, ref)
    assert (got["cam"] == 4).sum() > 0 and list(got["frames"]) == sorted(set(got["cam"][got["cam"] >= 0]))


def test_equal_distance_keeps_earlier_frame(lib):
    v, tris, fl = scene()
    live = all_live(tris, fl)
    R, t = look((0.0, 0.0, 8.0), (0, 0, 0)), np.array([0.0, 0.0, 8.0])
    frames = [dict(number=1, kind=2, pose=(R, t), cap=32, live=live), dict(number=2, kind=2, pose=(R, t), cap=32, live=live)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, fl)
    same(got, ref)
    assert set(got["cam"]) == {1}


def test_dead_facet_returns_with_its_choice(lib):
    v, tris, fl = scene()
    live = all_live(tris, fl)
    part = [e for e in live if e[0] % 3 != 0]
    frames = [dict(number=1, kind=1, pose=sensor_pose((0.0, 0.3, 9.0), (0, 0, 0)), cap=32, live=live),
              dict(number=2, kind=1, pose=sensor_pose((0.0, 0.1, 5.0), (0, 0, 0)), cap=32, live=part),
              dict(number=3, kind=1, pose=sensor_pose((0.0, 0.0, 20.0), (0, 0, 0)), cap=32, live=live)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, fl)
    same(got, ref)
    back = np.arange(len(tris)) % 3 == 0
    assert (got["cam"][back] == 1).all() and (got["cam"][~back] == 2).all()
    # read while the facets are dead: their frame stays in the frames list
    got, ref = run(lib, v, frames[:2], len(tris), [s for s, _ in part], tris, fl)
    same(got, ref)
    assert list(got["frames"]) == [1, 2] and set(got["cam"]) == {2}


def test_flip_change_permutes_uv_and_turns_the_front(lib):
    v, tris, fl = scene()
    flipped = 1 - fl
    live, live_f = all_live(tris, fl), all_live(tris, flipped)
    above = sensor_pose((0.2, 0.1, 8.0), (0, 0, 0))
    # textured from above, then the flip changes: the rows' uv follow the new face order
    frames = [dict(number=1, kind=1, pose=above, cap=32, live=live), dict(number=2, kind=0, cap=32, live=live_f)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, flipped)
    same(got, ref)
    assert (got["cam"] == 1).any()
    # the flipped facets face down: a nearer camera above no longer sees them (front-side test), a two-sided rule does
    nearer = sensor_pose((0.1, 0.0, 5.0), (0, 0, 0))
    frames = [dict(number=1, kind=1, pose=above, cap=32, live=live), dict(number=2, kind=1, pose=nearer, cap=32, live=live_f)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, flipped)
    same(got, ref)
    assert not (got["cam"] == 2).any()
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, flipped, cfg=dict(two_sided=True))
    same(got, ref)
    assert (got["cam"] == 2).any()


def test_frame_without_camera_changes_nothing(lib):
    v, tris, fl = scene()
    live = all_live(tris, fl)
    frames = [dict(number=1, kind=0, cap=32, live=live), dict(number=2, kind=1, pose=sensor_pose((0.0, 0.0, 7.0), (0, 0, 0)), cap=32, live=live),
              dict(number=3, kind=0, cap=32, live=live)]
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, fl)
    same(got, ref)
    assert got["counts"][3] == W * H and set(got["frames"]) <= {2}


def test_slot_allocated_never_live(lib):
    v, tris, fl = scene()
    live = [e for e in all_live(tris, fl) if e[0] != 5]
    frames = [dict(number=1, kind=1, pose=sensor_pose((0.0, 0.0, 7.0), (0, 0, 0)), cap=32, live=live)]
    got, ref = run(lib, v, frames, len(tris), [s for s, _ in live], tris, fl)
    same(got, ref)
    # the never-live slot comes alive later: it starts unobserved
    frames.append(dict(number=2, kind=0, cap=32, live=all_live(tris, fl)))
    got, ref = run(lib, v, frames, len(tris), range(len(tris)), tris, fl)
    same(got, ref)
    assert got["cam"][5] == -1


def test_growth_mid_run(lib):
    v, tris, fl = scene()
    live = all_live(tris, fl)
    cams = [sensor_pose((0.4, 0.2, 9.0), (0, 0, 0)), sensor_pose((-0.3, 0.1, 7.0), (0, 0, 0)), sensor_pose((0.0, -0.2, 6.5), (0, 0, 0))]
    small = [dict(number=i + 1, kind=1, pose=c, cap=[10, 20, 40][i], live=live[:[10, 20, 18][i]]) for i, c in enumerate(cams)]
    big = [dict(f, cap=40) for f in small]
    rows_ = range(18)
    got_s, ref = run(lib, v, small, 20, rows_, tris, fl)
    same(got_s, ref)
    got_b, _ = run(lib, v, big, 20, rows_, tris, fl)
    same(got_b, ref)


@pytest.mark.parametrize("seed", range(4))
def test_random_sequences(lib, seed):
    rng = np.random.default_rng(seed)
    v, t = grid(n=6, size=6.0, bump=0.15, seed=seed)
    tris = [tuple(int(x) for x in tri) for tri in t]
    fl = up_flips(v.astype(np.float64), t)
    frames, flips_now, cap = [], fl.copy(), 16
    for f in range(8):
        alive = rng.random(len(tris)) < 0.8
        if rng.random() < 0.3:   # some facets change their flip
            ch = rng.random(len(tris)) < 0.2
            flips_now = np.where(ch, 1 - flips_now, flips_now)
        cap = max(cap, len(tris)) if f >= 3 else cap
        kind = int(rng.choice([0, 1, 1, 2]))
        eye = (rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5), rng.uniform(3.0, 10.0))
        pose = sensor_pose(eye, (0, 0, 0)) if kind == 1 else (look(eye, (0, 0, 0)), np.array(eye))
        n_now = len(tris) if f >= 3 else 16
        live = [(s, int(flips_now[s])) for s in range(n_now) if alive[s]]
        frames.append(dict(number=2 * f + 1, kind=kind, pose=pose if kind else None, cap=cap, live=live))
    last = [s for s, _ in frames[-1]["live"]]
    got, ref = run(lib, v, frames, len(tris), last, tris, flips_now, cfg=dict(min_visible_permille=int(rng.integers(0, 500))))
    same(got, ref)
