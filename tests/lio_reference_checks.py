"""Shared driver of tests/test_lio_reference_{emu,gpu}.py: the localization path of an implementation under test (the CUDA library
through the C ABI, or the host emulation of its kernel bodies) against tests/lio_reference.py, the independent numpy restatement.

Equality is asserted where both sides take the same discrete decision from the same float inputs; a decision whose margin is
below the rounding bound stated next to it is excluded (with everything that depends on it), and every check asserts that the
excluded share is below 0.1 %."""
import dataclasses

import numpy as np

import lio_reference as ref
from immesh_b200 import api, synth

EPS = np.finfo(np.float64).eps
MAX_EXCLUDED = 1e-3


def f32_ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


# ------------------------------------------------------------------ A. Forward_without_imu
def check_prediction(lib):
    """Random states with |b_g| above and below 1e-7 and dt in {0.01, 0.1, 1}.  The device's sin / cos are polynomials within a few
    ulp of libm, everything else is the same product in a different order: 1e-13 relative."""
    rng = np.random.default_rng(7)
    h = api.Lio(api.AVIA, lib=lib)
    small_bg = 0
    for trial in range(12):
        s = np.zeros(api.STATE_DOUBLES)
        A = rng.normal(size=(3, 3))
        Q, _ = np.linalg.qr(A)
        s[0:9] = (Q * np.sign(np.linalg.det(Q))).reshape(9)
        s[9:24] = rng.normal(size=15)
        s[15:18] *= (1e-9 if trial % 3 == 0 else 0.3)
        small_bg += int(np.linalg.norm(s[15:18]) <= 1e-7)
        B = rng.normal(size=(18, 18))
        s[24:] = (B @ B.T * 1e-3).reshape(-1)
        for dt in (0.01, 0.1, 1.0):
            h.set_state(s)
            h.predict(dt, 0.1, 0.2)
            got = h.get_state()
            want = ref.forward_without_imu(s, dt, 0.1, 0.2)
            assert np.abs(got[0:24] - want[0:24]).max() <= 1e-13 * np.abs(want[0:24]).max(), (trial, dt)
            assert np.abs(got[24:] - want[24:]).max() <= 1e-13 * np.abs(want[24:]).max(), (trial, dt)
    assert small_bg >= 4          # the identity branch of Exp(b_g, dt)


# ------------------------------------------------------------------ B. the plane map
def eig_bound(C):
    """Absolute eigenvalue error allowed between the device's cyclic Jacobi and LAPACK on the same 3x3 covariance C: both are
    backward stable with a backward error below 8 eps ||C||_F, so by Weyl's theorem each eigenvalue of either lies within
    8 eps ||C||_F of the exact one, and the two within 16 eps ||C||_F of each other."""
    return 16.0 * EPS * np.linalg.norm(C)


def prep_state(R, t, P=None):
    s = np.zeros(api.STATE_DOUBLES)
    s[0:9] = np.asarray(R, dtype=np.float64).reshape(9)
    s[9:12] = t
    s[24:] = (np.eye(18) * 1e-4 if P is None else P).reshape(-1)
    return s


def build_lists(cfg, s, body):
    """buildVoxelMap's Point_with_var list of voxel_map_init (voxel_mapping.cpp:1249-1265): world point through float, variance
    R calcBodyVar(p) R^T + (-[p]x) S_rot (-[p]x)^T + S_t at the body point, input order"""
    pb = np.asarray(body, dtype=np.float64)
    return ref.transform_lidar(s, pb, cfg), ref.world_cov(ref.rot(s), ref.calc_body_var(pb, cfg.dept_err, cfg.beam_err), pb, ref.cov(s))


def update_lists(cfg, s, body):
    """map_incremental_grow's list (ImMesh_mesh_reconstruction.cpp:387-408): world point through float, variance with
    rot_end * ext_R and the IMU-frame point, sorted by var_contrast (stable)"""
    bc, p_imu = ref.body_prep(body, cfg)
    extR = np.asarray(cfg.ext_R, dtype=np.float64).reshape(3, 3)
    pw = ref.transform_lidar(s, body, cfg)
    var = ref.world_cov(ref.rot(s) @ extR, bc, p_imu, ref.cov(s))
    order = np.argsort(ref.var_contrast(var), kind="stable")
    return pw[order], var[order]


def compare_map(dump, vm):
    """the device dump against the numpy octree: exact shape, counters, centres and point counts; normal up to its sign, d and the
    normal-centre block flipping with it; eigenvalue-derived floats and the plane covariance within the eigen-solver bound.
    Root voxels with a planar decision within eig_bound of the threshold are excluded.  Returns (rows compared, excluded share)."""
    nodes = vm.nodes()
    assert len(nodes) == len(dump), f"node count {len(dump)} vs {len(nodes)}"
    amb_roots = {k for k, _, nd in nodes if nd.ambiguous}
    compared = 0
    for r, (k, path, nd) in enumerate(nodes):
        row = dump[r]
        assert tuple(row[0:3].astype(np.int64)) == k and row[3] == path, (r, row[0:4], k, path)
        if k in amb_roots:
            continue
        compared += 1
        pl = nd.plane
        want = [nd.layer, int(nd.init_octo), int(bool(pl and pl["is_plane"])), int(nd.update_enable), len(nd.pts), nd.new_points]
        assert list(row[4:10].astype(np.int64)) == want, (r, k, path, row[4:10], want)
        assert np.array_equal(row[21:24], nd.vc), (r, row[21:24], nd.vc)
        if pl is None:
            assert row[20] == 0
            continue
        assert row[20] == pl["n"] and np.array_equal(row[11:14], pl["center"]), (r, row[11:14], pl["center"])
        if not pl["is_plane"]:
            continue
        C, ev = pl["C"], pl["ev"]
        eb = eig_bound(C)
        gap = ev[1] - ev[0]
        tol_u = eb / gap + 4 * EPS                   # Davis-Kahan: eigenvector error <= eigenvalue error / gap
        n_dev = row[14:17]
        sg = 1.0 if n_dev @ pl["normal"] >= 0 else -1.0
        assert np.abs(n_dev - sg * pl["normal"]).max() <= tol_u, (r, n_dev, pl["normal"], tol_u)
        cn = np.abs(pl["center"]).sum()
        assert abs(row[17] - sg * float(pl["d"])) <= tol_u * cn + 2 * f32_ulp(pl["d"]) + 2 * f32_ulp(cn * tol_u), (r, row[17], pl["d"])
        assert abs(row[19] - float(pl["min_eig"])) <= eb + f32_ulp(pl["min_eig"]), (r, row[19], pl["min_eig"])
        rad = float(pl["radius"])
        assert abs(row[18] - rad) <= eb / (2 * max(rad, 1e-30)) + f32_ulp(rad), (r, row[18], rad)
        M = np.zeros((6, 6))
        M[ref.IU] = row[24:45]
        M = M + np.triu(M, 1).T
        W = pl["pv"].copy()
        W[0:3, 3:6] *= sg
        W[3:6, 0:3] *= sg
        # pv is linear in the F rows, each scaled by 1/(l_min - l_m) and built from two eigenvectors: a relative error of
        # 2 (tol_u + eb / gap) from the eigen-decomposition; the device's 60-moment contraction agrees with the per-point loop to
        # 1e-9 of the largest entry (DESIGN.md 2)
        scale = np.abs(W).max()
        assert np.abs(M - W).max() <= (2 * (tol_u + eb / gap) + 1e-9) * scale, (r, np.abs(M - W).max() / scale)
    share = 1.0 - compared / len(nodes)
    assert share < MAX_EXCLUDED, share
    return compared, share


def _map_stream(kind, cfg, n_points, offset, seed):
    sensor, scans = synth.make_stream(kind, 4, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    return scans, np.asarray(offset, dtype=np.float64)


def check_plane_map(lib, kind, cfg, n_points, offset=(0.0, 0.0, 0.0), seed=31):
    """voxel_map_init on the full first scan and three map updates on the down-sampled scans, every list built by numpy at the state
    the implementation holds (its own pose), the octree grown by lio_reference.VoxelMap, compared after every step"""
    scans, off = _map_stream(kind, cfg, n_points, offset, seed)
    g = api.Lio(cfg, lib=lib)
    vm = ref.VoxelMap(cfg, eig_bound)
    s = prep_state(scans[0]["R_true"], scans[0]["t_true"] + off)
    g.set_state(s)
    g.voxel_map_init(scans[0]["body_full"])
    vm.build(*build_lists(cfg, s, scans[0]["body_full"]))
    out = [compare_map(g.dump_map(), vm)]
    for k in (1, 2, 3):
        sk = prep_state(scans[k]["R_true"], scans[k]["t_true"] + off, np.diag(np.r_[np.full(3, 1e-5), np.full(3, 1e-4), np.full(12, 1e-3)]))
        # the map update reads the scan of the last estimation and the state it finds: estimate, then put sk back
        g.set_state(sk)
        g.lio_state_estimation(scans[k]["body_ds"])
        g.set_state(sk)
        g.map_incremental_grow()
        vm.update(*update_lists(cfg, sk, scans[k]["body_ds"]))
        out.append(compare_map(g.dump_map(), vm))
    assert g.counts()["err"] == 0
    return vm, out


# ------------------------------------------------------------------ C. residual selection
FLOAT_DECISION = 2.0 * 2.0 ** -23    # two float ulps, relative: a float distance that rounds the other way across the gate
PROB_DECISION = 4e-6                 # the probability through exp(-dis^2 / 2 sigma): dis^2 / sigma <= 9 times two float ulps
WORLD_TIE = 1e-8                     # a double world point within a few double ulps of a float rounding midpoint


def match_at(cfg, s, body, dump, P=None):
    """numpy's residual list of `body` at state s on the map `dump`: (dump row per point or -1, ambiguous mask, branch stats)"""
    planes = ref.DumpPlanes(dump)
    bc, p_imu = ref.body_prep(body, cfg)
    pwd = ref.world_double(s, body, cfg)
    pw = pwd.astype(np.float32).astype(np.float64)
    var = ref.world_cov(ref.rot(s), bc, p_imu, ref.cov(s) if P is None else P)
    best, m, st = ref.match_points(planes, pw, var, cfg.voxel_size, cfg.voxel_size)
    ulp = f32_ulp(pw)
    tie = (np.abs(np.abs(pwd - pw) / np.where(ulp > 0, ulp, 1.0) - 0.5) < WORLD_TIE).any(1)
    amb = tie | (m["range"] < FLOAT_DECISION) | (m["sigma"] < FLOAT_DECISION) | (m["prob"] < PROB_DECISION) | (m["loc"] < 1e-7)
    return best, amb, st


def compare_matches(lib_layers, best, amb, dump):
    want = np.where(best >= 0, dump[np.maximum(best, 0), 4].astype(np.int64), -1)
    ok = ~amb
    assert np.array_equal(lib_layers[ok], want[ok]), np.nonzero((lib_layers != want) & ok)[0][:10]
    assert amb.mean() < MAX_EXCLUDED, amb.mean()
    return want


def check_residual_build(lib, kind, cfg, n_points, seed, perturb=((0, 0), (0.05, 0.0), (0.0, 0.5), (-0.05, -0.5))):
    """immesh_residual_build (k_residual: the one-thread walk match_point, not k_match) at the converged state of a short stream and
    at states moved by +-5 cm / +-0.5 deg: the match set, layer and chosen node (its ptpl payload equal to that node's dump row)
    against numpy's walk over the same dump"""
    sensor, scans = synth.make_stream(kind, 3, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    g = api.Lio(cfg, lib=lib)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    g.lio_state_estimation(scans[1]["body_ds"])
    g.map_incremental_grow()
    dump = g.dump_map()
    body = scans[2]["body_ds"] if n_points is None or len(scans[2]["body_ds"]) >= 1000 else scans[2]["body_full"]
    g.set_pose(scans[2]["R_true"], scans[2]["t_true"])
    s0 = g.get_state()
    tot = dict(range_reject=0, sigma_reject=0, retry_success=0, non_first_argmax=0, layers=set(), n=0, excluded=0)
    for dt_m, da_deg in perturb:
        s = s0.copy()
        s[9:12] += dt_m
        s[0:9] = (ref.rot(s0) @ ref.exp_v(np.deg2rad([0.0, 0.0, da_deg]))).reshape(9)
        g.set_state(s)
        il, vals = g.residual_build(body)
        best, amb, st = match_at(cfg, s, body, dump)
        layers = np.full(len(body), -1)
        layers[il[:, 0]] = il[:, 1]
        compare_matches(layers, best, amb, dump)
        sel = ~amb[il[:, 0]]
        rows = best[il[sel, 0]]
        assert (rows >= 0).all()
        d = dump[rows]
        payload = np.concatenate([d[:, 14:17], d[:, 11:14], d[:, 17:18], d[:, 24:45]], 1)
        assert np.array_equal(vals[sel, 3:31], payload)
        assert np.array_equal(vals[:, 0:3], body[il[:, 0]].astype(np.float64))
        for k in ("range_reject", "sigma_reject", "retry_success", "non_first_argmax"):
            tot[k] += st[k]
        tot["layers"] |= set(np.unique(il[:, 1]).tolist())
        tot["n"] += len(body)
        tot["excluded"] += int(amb.sum())
    return tot


def check_residual_build_pv(lib, seed=9):
    """immesh_residual_build_pv on numpy-built Point_with_var lists whose world points are NOT float-representable: the lookup keeps
    them in double, so the match set, layer and payload equal numpy's walk on the unrounded points"""
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 3, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T)
    g = api.Lio(cfg, lib=lib)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    g.voxel_map_init(scans[0]["body_full"])
    g.lio_state_estimation(scans[1]["body_ds"])
    g.map_incremental_grow()
    dump = g.dump_map()
    body = scans[2]["body_ds"]
    s = prep_state(scans[2]["R_true"], scans[2]["t_true"] + np.array([0.013, -0.007, 0.004]), np.eye(18) * 1e-5)
    bc, p_imu = ref.body_prep(body, cfg)
    pwd = ref.world_double(s, body, cfg)
    assert (pwd != pwd.astype(np.float32)).mean() > 0.99
    var = ref.world_cov(ref.rot(s), bc, p_imu, ref.cov(s))
    il, vals = g.residual_build_pv(body.astype(np.float64), pwd, var.reshape(-1, 9))
    best, m, st = ref.match_points(ref.DumpPlanes(dump), pwd, var, cfg.voxel_size, cfg.voxel_size)
    amb = (m["range"] < FLOAT_DECISION) | (m["sigma"] < FLOAT_DECISION) | (m["prob"] < PROB_DECISION) | (m["loc"] < 1e-7)
    layers = np.full(len(body), -1)
    layers[il[:, 0]] = il[:, 1]
    compare_matches(layers, best, amb, dump)
    sel = ~amb[il[:, 0]]
    d = dump[best[il[sel, 0]]]
    assert np.array_equal(vals[sel, 3:31], np.concatenate([d[:, 14:17], d[:, 11:14], d[:, 17:18], d[:, 24:45]], 1))
    assert np.array_equal(vals[:, 0:3], body[il[:, 0]].astype(np.float64))
    assert len(il) > 300          # 0.57 k of the scan's 7.2 k points lie on planes of the two-scan map
    return int(amb.sum()), len(body)


def candidate_bound(cfg, s, pb, dump):
    """For points whose match is ambiguous: the largest |term| each could add to HTH (6x6), HTz (6) and sum|r| under any plane it
    could be matched to (the planes of its root voxel and of its retry neighbour).  A device that decides such a point the other way
    moves the sums by at most twice that (the term numpy counted taken out, another one put in)."""
    planes = ref.DumpPlanes(dump)
    pw = ref.transform_lidar(s, pb, cfg)
    loc = ref.voxel_loc(pw, cfg.voxel_size)
    key = np.trunc(loc).astype(np.int64)
    nkey, _ = ref.neighbour_key(key, loc, cfg.voxel_size)
    bHTH, bHTz, bres = np.zeros((6, 6)), np.zeros(6), 0.0
    for i in range(len(pb)):
        rows = np.concatenate([planes.by_root.get(tuple(key[i]), np.zeros(0, np.int64)), planes.by_root.get(tuple(nkey[i]), np.zeros(0, np.int64))])
        if len(rows) == 0:
            continue
        ne = ref.normal_equations(s, np.repeat(pb[i:i + 1], len(rows), 0), rows, dump, cfg)
        H, w, z = ne["H"], ne["R_inv"], ne["z"]
        bHTH += np.abs(H[:, :, None] * w[:, None, None] * H[:, None, :]).max(0)
        bHTz += np.abs(H * (w * z)[:, None]).max(0)
        bres += np.abs(z).max()
    return 2 * bHTH, 2 * bHTz, 2 * bres


# ------------------------------------------------------------------ D + E. weights, normal equations, IESKF iterations
def check_ieskf(lib, kind, cfg, n_scans, seed, n_points=None, full=False, init_vel=True):
    """A stream through predict + lio_state_estimation; for every iteration k the start state s_k is rebuilt in numpy from the
    propagated state and the implementation's solutions, and checked: numpy's match set at s_k (n_match), HTH / HTz / sum|r| from
    numpy's rows (1e-9 relative plus the fixed-point quantum n_match 2^-21, plus candidate_bound of the points whose match is
    ambiguous), the solution by the literal 18x18 form on the implementation's own HTH / HTz (1e-7 relative), the converged flag, the
    iteration count by the rematch rule, and the final state and covariance (I - G) P.  full: localise the full-resolution scans
    instead of the down-sampled ones (more than 2 SMs 1024 / 8 points: k_match's one-lane mode).  init_vel=False starts the filter at
    rest, so that the first scans need more iterations.  Returns branch statistics."""
    sensor, scans = synth.make_stream(kind, n_scans, seed=seed, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T, n_points=n_points)
    g = api.Lio(cfg, lib=lib)
    g.set_pose(scans[0]["R_true"], scans[0]["t_true"])
    if init_vel:
        s = g.get_state()
        s[12:15] = (scans[1]["t_true"] - scans[0]["t_true"]) / scans[0]["dt"]
        g.set_state(s)
    g.voxel_map_init(scans[0]["body_full"])
    out = dict(layers=set(), iters=[], rematch_stop=0, last_iter_stop=0, n=0, excluded=0, exp_identity=0, weights=0, compared=0,
               compared_with_bound=0, scan_points=[])
    for k in range(1, n_scans):
        body = scans[k]["body_full" if full else "body_ds"]
        out["scan_points"].append(len(body))
        g.predict(scans[k]["dt"])
        s_prop = g.get_state()
        dump = g.dump_map()
        iters = g.lio_state_estimation(body)
        layers = g.matches()
        sk, rematch = s_prop.copy(), 0
        for it in range(iters):
            st = g.iter_stats(it)
            best, amb, _ = match_at(cfg, sk, body, dump)
            out["n"] += len(body)
            out["excluded"] += int(amb.sum())
            assert amb.mean() < MAX_EXCLUDED
            rows = best[best >= 0]
            ne = ref.normal_equations(sk, body[best >= 0], rows, dump, cfg)
            n = int((best >= 0).sum())
            bHTH, bHTz, bres = candidate_bound(cfg, sk, body[amb], dump) if amb.any() else (0.0, 0.0, 0.0)
            assert abs(st["n_match"] - n) <= int(amb.sum()), (k, it, st["n_match"], n)
            q = n * 2.0 ** -21
            assert np.all(np.abs(st["HTH"] - ne["HTH"]) <= 1e-9 * np.abs(ne["HTH"]).max() + q + bHTH), (k, it)
            assert np.all(np.abs(st["HTz"] - ne["HTz"]) <= 1e-9 * np.abs(ne["HTz"]).max() + q + bHTz), (k, it)
            assert abs(st["total_residual"] - ne["total_residual"]) <= 1e-9 * ne["total_residual"] + q + bres
            out["compared"] += 1
            out["compared_with_bound"] += int(amb.any())
            sol, G = ref.ieskf_solution(st["HTH"], st["HTz"], sk, s_prop)
            assert np.abs(st["solution"] - sol).max() <= 1e-7 * np.abs(sol).max() + 1e-15, (k, it, np.abs(st["solution"] - sol).max())
            conv = ref.converged(st["solution"])
            assert st["converged"] == int(conv), (k, it)
            rematch, stop = ref.ieskf_flags(conv, rematch, it, cfg.max_iteration)
            out["exp_identity"] += int(np.linalg.norm(st["solution"][0:3]) <= 1e-5)
            nxt = ref.state_plus(sk, st["solution"])
            if stop:
                assert it == iters - 1, (k, it, iters)
                nxt[24:] = ((np.eye(18) - G) @ ref.cov(sk)).reshape(-1)
                out["rematch_stop" if rematch >= 2 else "last_iter_stop"] += 1
            sk = nxt
        assert rematch >= 2 or iters == cfg.max_iteration
        # the last iteration's match set and layers (immesh_lio_matches) are numpy's walk at the last start state
        best, amb, _ = match_at(cfg, _last_start(g, s_prop, iters), body, dump)
        out["layers"] |= set(compare_matches(layers, best, amb, dump).tolist()) - {-1}
        got = g.get_state()
        assert np.abs(got[0:24] - sk[0:24]).max() <= 1e-12 * max(1.0, np.abs(sk[0:24]).max()), (k, np.abs(got[0:24] - sk[0:24]).max())
        assert np.abs(got[24:] - sk[24:]).max() <= 1e-7 * np.abs(sk[24:]).max(), k
        # the weights of the last iteration's matches (the effect cloud; the host emulation does not have the call)
        if hasattr(g.lib, "immesh_lio_effect_cloud"):
            rows_e, idx_e = g.effect_cloud()
            ne = ref.normal_equations(_last_start(g, s_prop, iters), body[idx_e], best[idx_e], dump, cfg)
            want = np.sqrt(ne["R_inv"]).astype(np.float32)
            keep = ~amb[idx_e]
            assert np.all(np.abs(rows_e[keep, 3].astype(np.float64) - want[keep]) <= 2 * f32_ulp(want[keep])), k
            out["weights"] += int(keep.sum())
        out["iters"].append(iters)
        g.map_incremental_grow()
    return out


def _last_start(g, s_prop, iters):
    s = s_prop.copy()
    for it in range(iters - 1):
        s = ref.state_plus(s, g.iter_stats(it)["solution"])
    return s


# ------------------------------------------------------------------ F. the fixed-point range edge
WALL_CFG = dataclasses.replace(api.AVIA, ext_T=(0.0, 0.0, 0.0), dept_err=1.5e-5, beam_err=1e-6, max_iteration=1, max_scan_points=1 << 21)


def dense_wall(side):
    """a side x side grid on the plane x = 1.1 m, |y|, |z| < 0.5 m, in the body frame at the identity pose.  At 1.1 m the weight is
    R_inv ~ 1 / (dept_err^2 cos^2) = 4.4e9 .. 5.3e9 and the largest term |A|^2 R_inv <= 0.5 R_inv, so every term is below the
    per-term limit 1e10, while HTH[3][3] adds R_inv ~ 5e9 per point: 2^-20 fixed point holds 2^63 / 2^20 = 8.8e12 in one int64,
    i.e. about 1700 such points -- a block of 128 threads sums 3.9 k points of a 2 Mi-point scan on an H100's grid."""
    y = (np.arange(side) + 0.5) / side - 0.5
    Y, Z = np.meshgrid(y, y)
    return np.stack([np.full(Y.size, 1.1), Y.ravel(), Z.ravel()], 1).astype(np.float32)


def check_fixed_point_range(lib, side=1448):
    """one iteration on a 2 Mi-point dense wall: the call returns IMMESH_E_RANGE or HTH / HTz equal to numpy's float64 sums"""
    cfg = WALL_CFG
    g = api.Lio(cfg, lib=lib)
    s = prep_state(np.eye(3), np.zeros(3), np.zeros((18, 18)))
    g.set_state(s)
    g.voxel_map_init(dense_wall(100))
    dump = g.dump_map()
    assert (dump[:, 6] == 1).all()
    body = dense_wall(side)
    try:
        g.lio_state_estimation(body)
    except RuntimeError as e:
        assert "code -5" in str(e), e
        return None
    st = g.iter_stats(0)
    best, amb, _ = match_at(cfg, s, body, dump, P=np.zeros((18, 18)))
    assert not amb.any() and (best >= 0).all()
    ne = ref.normal_equations(s, body, best, dump, cfg)
    terms = ne["H"][:, :, None] * ne["R_inv"][:, None, None] * ne["H"][:, None, :]
    assert np.abs(terms).max() < 1e10 and ne["R_inv"].mean() * 128 * 31 * 2.0 ** 20 > 2.0 ** 63   # a block's sum would wrap int64
    n = len(body)
    assert st["n_match"] == n
    assert np.all(np.abs(st["HTH"] - ne["HTH"]) <= 1e-9 * np.abs(ne["HTH"]).max() + n * 2.0 ** -21), (st["HTH"][3, 3], ne["HTH"][3, 3])
    assert np.all(np.abs(st["HTz"] - ne["HTz"]) <= 1e-9 * np.abs(ne["HTH"]).max() + n * 2.0 ** -21)
    return st["HTH"]


# ------------------------------------------------------------------ G. the _pv insert contract
def check_pv_float_rounding(lib):
    """immesh_voxelmap_build_pv / _update_pv store float world points (pcl::PointXYZI m_point): a map built from doubles equals the map
    built from their float roundings"""
    cfg = api.AVIA
    sensor, scans = synth.make_stream("avia", 2, seed=41, leaf=cfg.filter_size_surf, ext_T=cfg.ext_T)
    s = prep_state(scans[0]["R_true"], scans[0]["t_true"])
    pw0 = ref.world_double(s, scans[0]["body_full"], cfg)
    _, var0 = build_lists(cfg, s, scans[0]["body_full"])
    pw1 = ref.world_double(s, scans[1]["body_ds"], cfg)
    _, var1 = update_lists(cfg, s, scans[1]["body_ds"])
    assert (pw0 != pw0.astype(np.float32)).mean() > 0.9
    dumps = []
    for rnd in (lambda a: a, lambda a: a.astype(np.float32).astype(np.float64)):
        g = api.Lio(cfg, lib=lib)
        g.voxelmap_build_pv(rnd(pw0), var0.reshape(-1, 9))
        g.voxelmap_update_pv(rnd(pw1), var1.reshape(-1, 9))
        dumps.append(g.dump_map())
    assert np.array_equal(dumps[0], dumps[1])
    # and the octree is the numpy one on the float points
    vm = ref.VoxelMap(cfg, eig_bound)
    vm.build(pw0.astype(np.float32).astype(np.float64), var0)
    vm.update(pw1.astype(np.float32).astype(np.float64), var1)
    compare_map(dumps[0], vm)
