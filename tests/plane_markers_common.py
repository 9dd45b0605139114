"""Shared driver of the plane-marker tests (pubPlaneMap, voxel_mapping.cpp:947-1159): the same scan stream through an
implementation under test (CUDA library or host emulation) and the oracle, the markers taken after the build and then at a
cadence, rows compared bit for bit except the id column.  The oracle walks the whole map every call; the implementation under
test walks only its pending roots, so equal rows check the pending-set bookkeeping against the plain rule.

Every call is also classified from the oracle's state before it (map dump + per-node flag dump), so that a test can assert which
branches of the walk the stream reached.

The oracle side is tests/pubmap/liborc_pub.so (the oracle with pubPlaneMap's state kept beside its tree, orc_pub.cpp); the
emulation side is tests/pubmap/libimmesh_emu_pub.so (the host emulation with the publisher's device state, emu_pub.cpp)."""
import ctypes as C

import numpy as np

from immesh_b200 import api, synth
from lio_common import init_velocity
from oracle_api import OracleLio, _p

_pub_lib = None


def emu_pub_lib():
    from immesh_b200 import build
    return api.load_library(build.build_pubmap()[0])


def _orc_pub():
    global _pub_lib
    if _pub_lib is None:
        from immesh_b200 import build
        L = C.CDLL(build.build_pubmap()[1])
        L.orc_lio_create.restype = C.c_void_p
        L.orc_lio_dump_map.restype = C.c_long
        L.orc_lio_predict.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        L.orc_pub_plane_markers.restype = C.c_long
        L.orc_pub_dump.restype = C.c_long
        _pub_lib = L
    return _pub_lib


class PubOracle(OracleLio):
    """The oracle with pubPlaneMap: map growth observed point by point (orc_pub.cpp), the full walk over the map."""

    def __init__(self, cfg):
        L = _orc_pub()
        cd = np.array([cfg.voxel_size, cfg.min_eigen_value, cfg.dept_err, cfg.beam_err, *cfg.ext_R, *cfg.ext_T], dtype=np.float64)
        ci = np.array([cfg.max_layer, *cfg.layer_init_size, cfg.max_points_size, cfg.max_iteration, cfg.calib_laser, 0, 1, 0, 0], dtype=np.int32)
        self.h = C.c_void_p(L.orc_lio_create(_p(cd), _p(ci)))
        self.L = L

    def __del__(self):
        try:
            self.L.orc_pub_forget(self.h)
            self.L.orc_lio_destroy(self.h)
        except Exception:
            pass

    def voxel_map_init(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        self.L.orc_pub_map_init(self.h, _p(a), C.c_int(a.shape[0]))

    def map_incremental_grow(self, body):
        a = np.ascontiguousarray(body, dtype=np.float32)
        self.L.orc_pub_map_grow(self.h, _p(a), C.c_int(a.shape[0]))

    def plane_markers(self):
        """(rows f64[m,16], counts [plane, sub-plane, sub-sub-plane, update]); clears the published flags.  Column 5 holds the
        reference's m_id (g_plane_id), not the library's record index."""
        counts = np.zeros(4, dtype=np.int64)
        m = self.L.orc_pub_plane_markers(self.h, _p(counts))
        out = np.zeros((m, 16))
        if m:
            self.L.orc_pub_rows(self.h, _p(out))
        return out, counts

    def dump_pub(self):
        """per node in dump_map()'s order: is_update, octo_state, m_p_center (x y z normal_x normal_y normal_z)"""
        rows = self.L.orc_pub_dump(self.h, None, C.c_long(0))
        out = np.zeros((rows, 8))
        self.L.orc_pub_dump(self.h, _p(out), C.c_long(rows))
        return out

ID = 5
NOT_ID = [c for c in range(api.PLANE_MARKER_COLS) if c != ID]
BRANCHES = ("root_planar", "root_never_planar", "root_planar_then_not", "layer1", "child_held_back", "layer2_planar",
            "layer2_nonplanar_kept", "layer2_octo1_skipped", "deep_flag_never")


def _index(dump):
    return {(int(r[0]), int(r[1]), int(r[2]), int(r[3])): i for i, r in enumerate(dump)}


def check_oracle_rows(rows, dump, pub):
    """The oracle's rows against numpy on its own map dump taken before the call (the call changes no plane): trace, radius,
    min_eig, alpha; and m_p_center against the float centre / normal of every planar node."""
    idx = _index(dump)
    planar = dump[:, 6] == 1
    assert np.array_equal(pub[planar, 2:5], dump[planar, 11:14].astype(np.float32).astype(np.float64))
    assert np.array_equal(pub[planar, 5:8], dump[planar, 14:17].astype(np.float32).astype(np.float64))
    for r in rows:
        i = idx[(int(r[0]), int(r[1]), int(r[2]), int(r[3]))]
        d = dump[i]
        assert r[4] == d[4]
        pv = d[24:45]
        assert r[14] == (pv[0] + pv[6]) + pv[11]
        assert np.array_equal(r[6:12], pub[i, 2:8])
        if d[6] == 1:
            assert r[13] == np.float32(d[19])
        radius = np.float64(np.float32(1.25 * d[18])) if d[4] < 2 else d[18]
        assert r[12] == radius and r[15] == (1.0 if d[4] == 2 else d[6])


def classify(rows, dump, pub, pub_after):
    """Branches of the walk taken by one call, from the oracle's state before it (dump, pub) and the flags after it."""
    got = set()
    for r in rows[rows[:, 4] == 0]:
        if r[15] == 1:
            got.add("root_planar")
        elif not r[6:12].any():
            got.add("root_never_planar")
        else:
            got.add("root_planar_then_not")
    if (rows[:, 4] == 1).any():
        got.add("layer1")
    held = set()
    kept = 0
    idx = _index(dump)
    flag = pub[:, 0] == 1
    for i, d in enumerate(dump):
        key, path, layer = (int(d[0]), int(d[1]), int(d[2])), int(d[3]), int(d[4])
        if layer >= 3 and flag[i]:
            assert pub_after[i, 0] == 1
            got.add("deep_flag_never")
        if layer == 1 and flag[i] and flag[idx[key + (0,)]]:
            held.add(key + (path,))
        if layer == 2 and flag[i]:
            root, child = idx[key + (0,)], idx[key + (path // 9,)]
            if flag[root] or flag[child]:
                continue
            if pub[i, 1] != 0:
                assert pub_after[i, 0] == 1
                got.add("layer2_octo1_skipped")
            elif d[6] == 0:
                assert pub_after[i, 0] == 1
                got.add("layer2_nonplanar_kept")
                kept += 1
            else:
                got.add("layer2_planar")
    if "layer2_planar" in got:
        assert ((rows[:, 4] == 2) & (rows[:, 15] == 1)).any()
    return got, held, kept


def run_markers_parity(lib, kind, cfg, n_scans, seed, every=1, n_points=None, mode="staged", oracle_checks=True, repeat=1):
    """mode 'staged': predict / lio_state_estimation / map_incremental_grow calls; 'async': immesh_lio_step_async (the pipelined,
    graph-replayed path), the markers call then waits for it.  Markers after the build and after every `every`-th scan, `repeat`
    calls in a row each time (a second call with no fit in between publishes exactly what the first one held back).
    Returns dict(reached=set of BRANCHES, walked=[roots walked per call], pending_bound=[roots holding a set flag before the
    call], roots=[map roots at the call], calls=n)."""
    sensor, scans = synth.make_stream(kind, n_scans, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    g = api.Lio(cfg, lib=lib)
    o = PubOracle(cfg)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    ids, owner = {}, {}
    out = dict(reached=set(), walked=[], pending_bound=[], roots=[], calls=0)
    held_prev = set()

    def call():
        nonlocal held_prev
        dump, pub = o.dump_map(), o.dump_pub()
        ro, co = o.plane_markers()
        rg, cg = g.plane_markers()
        assert rg.shape == ro.shape, f"call {out['calls']}: {rg.shape[0]} rows vs the oracle's {ro.shape[0]}"
        assert np.array_equal(rg[:, NOT_ID], ro[:, NOT_ID]), f"call {out['calls']}: rows differ"
        assert [cg[k] for k in ("plane", "sub_plane", "update")] == [co[0], co[1], co[3]]
        for r in rg:
            kp, i = (int(r[0]), int(r[1]), int(r[2]), int(r[3])), int(r[ID])
            assert ids.setdefault(kp, i) == i, f"{kp}: id changed"
            assert owner.setdefault(i, kp) == kp, f"id {i} shared by {owner[i]} and {kp}"
        pub_after = o.dump_pub()
        if oracle_checks:
            check_oracle_rows(ro, dump, pub)
        got, held, kept = classify(ro, dump, pub, pub_after)
        # the reference counts a kept non-planar layer-2 flag again on every call; the library only while its root is pending
        assert co[2] - kept <= cg["sub_sub_plane"] <= co[2]
        emitted = {(int(r[0]), int(r[1]), int(r[2]), int(r[3])) for r in ro}
        if held_prev & emitted:
            got.add("child_held_back")
        held_prev = held
        out["reached"] |= got
        # the pending list holds the roots fitted under since the last call plus those held back: all of them hold a set flag
        keys = {(int(d[0]), int(d[1]), int(d[2])) for d, f in zip(dump, pub[:, 0]) if f == 1}
        out["walked"].append(cg["roots_walked"])
        out["pending_bound"].append(len(keys))
        out["roots"].append(g.counts()["roots"])
        out["calls"] += 1

    for _ in range(repeat):
        call()
    for k in range(1, n_scans):
        body, dt = scans[k]["body_ds"], scans[k]["dt"]
        if mode == "async":
            g.step_async(body, dt=dt)
        else:
            g.predict(dt)
            g.lio_state_estimation(body)
            g.map_incremental_grow()
        o.predict(dt)
        o.lio_state_estimation(body)
        o.map_incremental_grow(body)
        if k % every == 0:
            for _ in range(repeat):
                call()
    if mode == "async":
        g.wait()
    assert np.array_equal(g.get_state(), o.get_state())
    assert np.array_equal(g.dump_map(), o.dump_map())
    assert g.counts()["err"] == 0
    g.close()
    return out
