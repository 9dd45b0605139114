"""CPU tier: the viewer's region buffers (immesh_mesh_region_buffers) executed by the host emulation of the device code against the
oracle's literal walk, the m_smoothed flag rules, the call's contract, and the smoothed rows against a numpy restatement of smooth_pts."""
import ctypes as C

import numpy as np
import pytest

from immesh_b200 import api
from mesh_common import SMALL, world_scans
from region_buffers_common import BOX0, compare_call, emu_regionbuf_lib, run_region_parity, subset_keys

E_INVALID, E_CAPACITY = -1, -3


@pytest.fixture(scope="module")
def emu_lib():
    """the host emulation with the m_smoothed flags and the call (tests/pubmap/emu_region_buf.cpp)"""
    return emu_regionbuf_lib()


def smooth_state(lib, g):
    nv = g.counts()["n_vertices"]
    f = np.zeros(nv, np.uint8)
    s = np.zeros((nv, 3))
    lib.emu_mesh_smooth_state(g._h, f.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p))
    return f, s


@pytest.mark.parametrize("kind,seed", [("avia", 0), ("hdl64", 2)])
def test_streams_bit_exact_and_the_write_back_matters(emu_lib, kind, seed):
    """calls after frames 1, 3 and 5 (a key subset, then every region), rows / ids / regions / smoothed counts / axis box bit-identical;
    later frames' facets and flags equal those of the oracle that made the same calls -- and differ from a run without the calls"""
    g, o, stats = run_region_parity(emu_lib, kind, 7, seed)
    assert all(n > 0 for n, _ in stats) and sum(s for _, s in stats) > 100
    plain = api.Mesh(api.MeshConfig(**SMALL), lib=emu_lib)
    for k, (w, t) in enumerate(world_scans(kind, 7, seed)):
        plain.push_frame(w, t, k)
    (_, tg, fg), (_, tp, fp) = g.snapshot(), plain.snapshot()
    assert tg.shape == tp.shape and np.array_equal(tg, tp)    # the calls change orientations, not the facet set
    assert not np.array_equal(fg, fp), "no flag depends on the viewer's write-back: the comparison of later frames is vacuous"


def test_oracle_flags_follow_the_dilation(emu_lib):
    """the oracle's m_smoothed bookkeeping (orc_region_buf.cpp) and the device flags agree after every frame"""
    from region_buffers_common import RegionOracle
    cfg = api.MeshConfig(**SMALL)
    g, o = api.Mesh(cfg, lib=emu_lib), RegionOracle(cfg)
    for k, (w, t) in enumerate(world_scans("avia", 4, 1)):
        g.push_frame(w, t, k)
        o.push_frame(w, t, k)
        f, _ = smooth_state(emu_lib, g)
        assert np.array_equal(f, o.flags()), k
        assert 0 < f.sum() < len(f)


def _knn_brute(v, q_ids, k):
    """k nearest vertices of vertices q_ids by the float distance ((dx*dx + dy*dy) + dz*dz), ties to the lower id"""
    idx, d2 = [], []
    for i in q_ids:
        d = v - v[i]
        dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        o = np.lexsort((np.arange(len(v)), dd))[:k]
        idx.append(o)
        d2.append(dd[o])
    return np.array(idx), np.array(d2, dtype=np.float32)


def test_smoothed_rows_against_numpy(emu_lib):
    """the vertices a call smoothed, recomputed in numpy from the raw snapshot positions (brute-force kNN, the limit 1.25 res,
    p (1 - f) + mean f), must be the rows' floats; the rows grouped by region as region_stream's keys say"""
    g, o, _ = run_region_parity(emu_lib, "avia", 4, seed=14, call_after=())
    f0, _ = smooth_state(emu_lib, g)
    xyz, ids, keys, offs, n = g.region_buffers(2.0, None, 0.7, 12)
    f1, s1 = smooth_state(emu_lib, g)
    new = np.nonzero(f1 & ~f0)[0]
    assert len(new) == n > 50
    v, tri, _ = g.snapshot()
    lim = 1.25 * api.MeshConfig(**SMALL).voxel_resolution
    sample = new[:: max(1, len(new) // 200)]
    idx, d2 = _knn_brute(v, sample, 12)
    vd = v.astype(np.float64)
    for r, i in enumerate(sample):
        s, valid = np.zeros(3), 0.0
        for j in range(1, 12):
            if np.float64(np.sqrt(d2[r, j])) < lim:
                s = s + vd[idx[r, j]]
                valid += 1.0
        with np.errstate(divide="ignore", invalid="ignore"):
            exp = vd[i] * (1.0 - 0.7) + s * 0.7 / valid
        assert np.array_equal(s1[i], exp) or (np.isnan(exp).all() and np.isnan(s1[i]).all()), i
        rows = xyz.reshape(-1, 3, 3)[ids == i]
        assert len(rows) and all(np.array_equal(x, exp.astype(np.float32)) or np.isnan(exp).all() for x in rows)
    # grouping: the same triangles as region_stream's keys, region by region, ascending triples inside
    ko = o.region_keys(2.0)
    _, to, _ = o.snapshot()
    order = np.lexsort((to[:, 2], to[:, 1], to[:, 0], ko[:, 2], ko[:, 1], ko[:, 0]))
    assert np.array_equal(ids, to[order]) and np.array_equal(tri, to)
    ref_keys, first = np.unique(ko[order], axis=0, return_index=True)
    assert np.array_equal(keys, ref_keys) and np.array_equal(offs[:-1], np.sort(first)) and offs[-1] == len(to)


def test_flag_rules(emu_lib):
    g, o, _ = run_region_parity(emu_lib, "avia", 4, seed=3, call_after=())
    ks = subset_keys(o, 2.0, every=4)
    f0, _ = smooth_state(emu_lib, g)
    sub = compare_call(g, o, 2.0, ks)[0]
    f1, _ = smooth_state(emu_lib, g)
    touched = np.unique(sub[1])
    assert sub[4] > 0 and np.array_equal(np.nonzero(f1 & ~f0)[0], touched[f0[touched] == 0])
    # a repeated call smooths nothing and returns the same rows
    again = compare_call(g, o, 2.0, ks)[0]
    assert again[4] == 0 and np.array_equal(again[0].view(np.uint32), sub[0].view(np.uint32))
    # vertices reached only through unselected regions stayed clear: the all-regions call smooths exactly them
    full = compare_call(g, o, 2.0, None)[0]
    allv = np.unique(full[1])
    assert full[4] == int((f1[allv] == 0).sum()) > 0
    f2, _ = smooth_state(emu_lib, g)
    assert f2[allv].all()
    # after smooth_all_pts nothing is left to smooth
    h, o2, _ = run_region_parity(emu_lib, "avia", 3, seed=4, call_after=())
    h.smooth_all(0.1, 20)
    o2.smooth_all(0.1, 20)
    r = compare_call(h, o2, 2.0, None)[0]
    assert r[4] == 0 and len(r[0]) > 1000


def test_contract(emu_lib):
    g, o, _ = run_region_parity(emu_lib, "avia", 3, seed=5, call_after=())
    L = emu_lib
    i32, f32 = C.POINTER(C.c_int32), C.POINTER(C.c_float)
    nr, nt, ns = C.c_int(0), C.c_int(0), C.c_int(0)
    f0, s0 = smooth_state(L, g)
    n_live = g.counts()["n_triangles"]
    rows = np.zeros((8, 9), np.float32)
    box = BOX0.copy()
    # too small a cap, or too few regions: the counts needed, nothing written, nothing smoothed
    assert L.immesh_mesh_region_buffers(g._h, 2.0, None, 0, 1.0, 20, rows.ctypes.data_as(f32), None, 8, None, None, 1 << 20, box.ctypes.data_as(f32),
                                        C.byref(nr), C.byref(nt), C.byref(ns)) == E_CAPACITY
    assert nt.value == n_live and nr.value > 2 and ns.value == 0 and not rows.any() and np.array_equal(box, BOX0)
    need_r = nr.value
    assert L.immesh_mesh_region_buffers(g._h, 2.0, None, 0, 1.0, 20, None, None, n_live, None, None, need_r - 1, None, C.byref(nr), C.byref(nt), C.byref(ns)) == E_CAPACITY
    assert nr.value == need_r and nt.value == n_live
    f1, s1 = smooth_state(L, g)
    assert np.array_equal(f0, f1) and np.array_equal(s0.view(np.uint64), s1.view(np.uint64))
    # arguments
    rep = np.array([[0, 0, 0], [1, 1, 1], [0, 0, 0]], np.int32)
    assert L.immesh_mesh_region_buffers(g._h, 2.0, rep.ctypes.data_as(i32), 3, 1.0, 20, None, None, 0, None, None, 0, None, C.byref(nr), C.byref(nt), C.byref(ns)) == E_INVALID
    for rs, knn in ((0.0, 20), (-1.0, 20), (2.0, 0), (2.0, 33)):
        assert L.immesh_mesh_region_buffers(g._h, rs, None, 0, 1.0, knn, None, None, 0, None, None, 0, None, C.byref(nr), C.byref(nt), C.byref(ns)) == E_INVALID
    # an absent key: an empty segment in the caller's place
    ks = subset_keys(o, 2.0, every=5)
    ks = np.concatenate([ks[:1], np.array([[77, 77, 77]], np.int32), ks[1:]])
    r = compare_call(g, o, 2.0, ks)[0]
    assert r[3][1] == r[3][2] and np.array_equal(r[2], ks)
    # knn 1 (no neighbour: NaN), 8, 20, 32 on fresh meshes
    for knn in (1, 8, 20, 32):
        h, oh, _ = run_region_parity(emu_lib, "avia", 2, seed=6, call_after=())
        r = compare_call(h, oh, 2.0, None, knn=knn, smooth_factor=0.25)[0]
        assert np.isnan(r[0]).any() == (knn == 1)
    # an empty mesh
    e = api.Mesh(api.MeshConfig(**SMALL), lib=emu_lib)
    xyz, ids, keys, offs, n = e.region_buffers(2.0)
    assert xyz.shape == (0, 9) and keys.shape == (0, 3) and offs.tolist() == [0] and n == 0
    xyz, ids, keys, offs, n = e.region_buffers(2.0, np.array([[1, 2, 3], [4, 5, 6]], np.int32))
    assert offs.tolist() == [0, 0, 0]
