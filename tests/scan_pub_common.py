"""Shared driver of the scan-publisher tests (publish_effect_world / publish_frame_world, voxel_mapping_common.cpp:535-547,
:595-614): the same scan stream through an implementation under test (CUDA library or host emulation) and the oracle, both clouds
taken after every scan and compared bit for bit.

The oracle side is tests/pubmap/liborc_scanpub.so (the oracle with the last iteration's weights rebuilt beside it,
orc_scan_pub.cpp); the emulation side is tests/pubmap/libimmesh_emu_scanpub.so (the host emulation with ScanBuf::wsqrt and the two
calls, emu_scan_pub.cpp)."""
import ctypes as C

import numpy as np

from immesh_b200 import api, synth
from lio_common import init_velocity
from oracle_api import OracleLio, _p

_lib = None


def emu_scanpub_lib():
    from immesh_b200 import build
    return api.load_library(build.build_scanpub()[0])


def _orc():
    global _lib
    if _lib is None:
        from immesh_b200 import build
        L = C.CDLL(build.build_scanpub()[1])
        L.orc_lio_create.restype = C.c_void_p
        L.orc_lio_dump_map.restype = C.c_long
        L.orc_lio_predict.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_double]
        _lib = L
    return _lib


class ScanPubOracle(OracleLio):
    """The oracle with publish_effect_world / publish_frame_world (orc_scan_pub.cpp)."""

    def __init__(self, cfg):
        L = _orc()
        cd = np.array([cfg.voxel_size, cfg.min_eigen_value, cfg.dept_err, cfg.beam_err, *cfg.ext_R, *cfg.ext_T], dtype=np.float64)
        ci = np.array([cfg.max_layer, *cfg.layer_init_size, cfg.max_points_size, cfg.max_iteration, cfg.calib_laser, 0, 1, 0, 0], dtype=np.int32)
        self.h = C.c_void_p(L.orc_lio_create(_p(cd), _p(ci)))
        self.L = L

    def __del__(self):
        try:
            self.L.orc_eff_forget(self.h)
            self.L.orc_lio_destroy(self.h)
        except Exception:
            pass

    def lio_state_estimation(self, body, state_prop=None):
        a = np.ascontiguousarray(body, dtype=np.float32)
        sp = self.get_state() if state_prop is None else np.ascontiguousarray(state_prop, dtype=np.float64)
        self._n = a.shape[0]
        return self.L.orc_eff_estimate(self.h, _p(a), C.c_int(a.shape[0]), _p(sp))

    def replay_ok(self):
        return bool(self.L.orc_eff_replay_ok(self.h))

    def effect_cloud(self, details=False):
        """(rows float32[m, 4], scan indices int32[m]); details=True adds R_inv f64[m] and the matched normals f64[m, 3]"""
        m = self.L.orc_eff_cloud(self.h, None, None, None, None)
        rows, idx = np.zeros((m, 4), dtype=np.float32), np.zeros(m, dtype=np.int32)
        r_inv, nrm = np.zeros(m), np.zeros((m, 3))
        self.L.orc_eff_cloud(self.h, _p(rows), _p(idx), _p(r_inv), _p(nrm))
        return (rows, idx, r_inv, nrm) if details else (rows, idx)

    def last_scan(self):
        n = self.L.orc_eff_scan(self.h, None)
        out = np.zeros((n, 3), dtype=np.float32)
        self.L.orc_eff_scan(self.h, _p(out))
        return out

    def frame_world(self, pts, point_skip=1, intensity_col=-1):
        a = np.ascontiguousarray(pts, dtype=np.float32)
        out = np.zeros((a.shape[0] + 1, 4), dtype=np.float32)
        m = self.L.orc_frame_world(self.h, _p(a), C.c_int(a.shape[0]), C.c_int(a.shape[1]), C.c_int(intensity_col), C.c_int(point_skip), _p(out))
        return out[:m]


def check_oracle_effect(o):
    """The oracle's effect rows against the oracle's own record of the last iteration: the rebuilt match set is its
    last_match_idx, the row count and indices are its n_match / matches(), and sum(intensity^2 n n^T) over the rows -- n the float
    normals the loop used -- is the translation block of that iteration's H^T R^-1 H."""
    rows, idx, r_inv, nrm = o.effect_cloud(details=True)
    assert o.replay_ok(), "the rebuilt last residual list differs from the oracle's"
    m = o.matches()
    assert np.array_equal(idx, np.nonzero(m >= 0)[0].astype(np.int32))
    return rows, idx, r_inv, nrm


def check_weights_against_normal_equations(o, iters):
    rows, idx, r_inv, nrm = check_oracle_effect(o)
    st = o.iter_stats(iters - 1)
    assert rows.shape[0] == st["n_match"]
    if rows.shape[0] == 0:
        return
    w = rows[:, 3].astype(np.float64) ** 2
    block = np.einsum("k,ki,kj->ij", w, nrm, nrm)
    ref = st["HTH"][3:6, 3:6]
    assert np.allclose(block, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max()), (block, ref)
    assert np.array_equal(rows[:, 3], np.sqrt(r_inv).astype(np.float32))


def _intensity_cloud(body_full, seed):
    """the full-resolution scan as [n][5] rows x y z pad intensity, intensity drawn per point (column 4)"""
    rng = np.random.default_rng(seed)
    n = body_full.shape[0]
    return np.concatenate([body_full, rng.normal(size=(n, 1)), rng.uniform(0, 255, (n, 1))], 1).astype(np.float32)


def compare_clouds(g, o, body_ds, dense, tag):
    """both publishers of g against the oracle o at the current state"""
    rg, ig = g.effect_cloud()
    ro, io = o.effect_cloud()
    assert rg.shape == ro.shape, f"{tag}: {rg.shape[0]} effect rows vs the oracle's {ro.shape[0]}"
    assert np.array_equal(ig, io), f"{tag}: effect scan indices"
    assert np.array_equal(rg.view(np.uint32), ro.view(np.uint32)), f"{tag}: effect rows differ"
    n = body_ds.shape[0]
    for skip in (1, 3, n + 1):
        a = g.registered_cloud(None, point_skip=skip)
        b = o.frame_world(body_ds, skip)
        assert a.shape == b.shape and np.array_equal(a, b), f"{tag}: registered rows of the localised scan, skip {skip}"
    for skip in (1, 3, dense.shape[0] + 1):
        a = g.registered_cloud(dense, point_skip=skip, intensity_col=4)
        b = o.frame_world(dense, skip, intensity_col=4)
        assert a.shape == b.shape and np.array_equal(a, b), f"{tag}: registered rows of the dense cloud, skip {skip}"
    return rg, ig


def run_scan_pub_parity(lib, kind, cfg, n_scans, seed, mode="staged", n_points=None, body_len=None, oracle_checks=True):
    """mode 'staged': predict / lio_state_estimation / map_incremental_grow, both clouds before and after the map update (they must
    not change); 'step': the fused immesh_lio_step; 'async': immesh_lio_step_async (the pipelined, graph-replayed path; each call
    waits for it).  body_len: {scan index: length} truncates those down-sampled scans.  Returns the effect row counts per scan."""
    sensor, scans = synth.make_stream(kind, n_scans, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    for k, m in (body_len or {}).items():
        scans[k]["body_ds"] = scans[k]["body_ds"][:m]
    g = api.Lio(cfg, lib=lib)
    o = ScanPubOracle(cfg)
    for h in (g, o):
        h.set_pose(scans[0]["R_true"], scans[0]["t_true"])
        init_velocity(h, sensor, scans)
        h.voxel_map_init(scans[0]["body_full"])
    rows, idx = g.effect_cloud()
    assert rows.shape == (0, 4) and idx.shape == (0,), "no effect cloud before the first IESKF run"
    counts = []
    for k in range(1, n_scans):
        body, dt = scans[k]["body_ds"], scans[k]["dt"]
        dense = _intensity_cloud(scans[k]["body_full"], seed * 100 + k)
        if mode == "staged":
            g.predict(dt)
            ig = g.lio_state_estimation(body)
        elif mode == "step":
            _, ig = g.step(body, dt=dt)
        else:
            g.step_async(body, dt=dt)
        o.predict(dt)
        io = o.lio_state_estimation(body)
        if mode != "async":
            assert ig == io, f"scan {k}: iteration count {ig} vs {io}"
        if oracle_checks:
            check_weights_against_normal_equations(o, io)
        if mode == "staged":
            before = compare_clouds(g, o, body, dense, f"scan {k}, before the map update")
            g.map_incremental_grow()
        o.map_incremental_grow(body)
        after = compare_clouds(g, o, body, dense, f"scan {k}")
        if mode == "staged":
            assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]), f"scan {k}: the map update changed the effect rows"
        counts.append(after[0].shape[0])
    if mode == "async":
        g.wait()
    assert np.array_equal(g.get_state(), o.get_state())
    assert g.counts()["err"] == 0
    g.close()
    return counts
