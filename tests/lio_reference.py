"""Plain numpy restatement of the localization arithmetic, written from the reference's equations (paths relative to the
reference repository, hku-mars/ImMesh).  It shares no code with the CUDA kernels or with the C++ restatement under oracle/:
it is the independent side of tests/lio_reference_checks.py.

Float types follow the reference (DESIGN.md 3): world points through pcl::PointXYZI, dis_to_plane / dis_to_center /
range_dis, Plane::m_radius / m_d / m_min_eigen_value and m_planer_threshold_ are float; everything else is float64.
State vectors use the C ABI's 348-double layout: rot_end[9] (row-major) pos vel bias_g bias_a gravity cov[18*18]."""
import math

import numpy as np

f32 = np.float32
I3 = np.eye(3)
UPDATE_SIZE_THRESHOLD = 5   # OctoTree::m_update_size_threshold_ (src/voxel_loc.hpp)
G_MAX_POINTS = 1000         # g_max_points, src/voxel_loc.cpp:45
CALIB_ANGLE_COV = 0.01      # include/common_lib.h:41


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


# ------------------------------------------------------------------ SO(3), include/so3_math.h
def exp_v(v):
    """Exp(v1, v2, v3) (so3_math.h:54-72): identity at |v| <= 1e-5."""
    n = math.sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2])
    if not n > 0.00001:
        return I3.copy()
    K = skew(np.asarray(v) / n)
    return I3 + math.sin(n) * K + (1.0 - math.cos(n)) * (K @ K)


def exp_dt(w, dt):
    """Exp(ang_vel, dt) (so3_math.h:31-51): identity at |w| <= 1e-7."""
    n = math.sqrt(float(np.dot(w, w)))
    if not n > 0.0000001:
        return I3.copy()
    K = skew(np.asarray(w) / n)
    a = n * dt
    return I3 + math.sin(a) * K + (1.0 - math.cos(a)) * (K @ K)


def log_so3(R):
    """Log(R) (so3_math.h:76-81): theta = 0 when trace > 3 - 1e-6, the first-order form when |theta| < 0.001."""
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    theta = 0.0 if tr > 3.0 - 1e-6 else math.acos(0.5 * (tr - 1.0))
    K = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return 0.5 * K if abs(theta) < 0.001 else 0.5 * theta / math.sin(theta) * K


# ------------------------------------------------------------------ StatesGroup, include/common_lib.h:238-271
def rot(s):
    return s[0:9].reshape(3, 3)


def cov(s):
    return s[24:].reshape(18, 18)


def state_minus(a, b):
    """a - b (common_lib.h:260-271): Log(b.rot^T a.rot), then the plain differences."""
    out = np.zeros(18)
    out[0:3] = log_so3(rot(b).T @ rot(a))
    out[3:18] = a[9:24] - b[9:24]
    return out


def state_plus(s, d):
    """s += d (common_lib.h:249-258): rot <- rot Exp(d[0:3]), the rest added."""
    o = s.copy()
    o[0:9] = (rot(s) @ exp_v(d[0:3])).reshape(9)
    o[9:24] = s[9:24] + d[3:18]
    return o


# ------------------------------------------------------------------ Forward_without_imu, src/IMU_Processing.cpp:486-553
def forward_without_imu(s, dt, cov_gyr, cov_acc):
    F = np.eye(18)
    F[0:3, 0:3] = exp_dt(s[15:18], -dt)
    F[0:3, 9:12] = I3 * dt
    F[3:6, 6:9] = I3 * dt
    Q = np.zeros((18, 18))
    Q[9:12, 9:12] = I3 * (cov_gyr * dt * dt)
    Q[6:9, 6:9] = I3 * (cov_acc * dt * dt)
    o = s.copy()
    o[24:] = (F @ cov(s) @ F.T + Q).reshape(-1)
    o[0:9] = (rot(s) @ exp_dt(s[15:18], dt)).reshape(9)
    o[9:12] = s[9:12] + s[12:15] * dt
    return o


# ------------------------------------------------------------------ per-point geometry
def direction_var(beam_err_deg):
    """sin(DEG2RAD(degree_inc))^2 of calcBodyVar; degree_inc is a float parameter, PCL's DEG2RAD(x) is x * 0.017453293"""
    return math.sin(float(f32(beam_err_deg)) * 0.017453293) ** 2


def calc_body_var(pb, dept_err, beam_err_deg):
    """calcBodyVar (src/voxel_mapping.cpp:1221-1241) for points pb [n,3] (float64), vectorised: z == 0 -> 0.0001 inside the function;
    range through float, range_var = range_inc^2 in float.  Returns [n,3,3]."""
    p = np.array(pb, dtype=np.float64).reshape(-1, 3)
    p[p[:, 2] == 0, 2] = 0.0001
    nrm = np.sqrt((p * p).sum(1))
    rng = nrm.astype(f32).astype(np.float64)
    rv = float(f32(dept_err) * f32(dept_err))
    d = p / nrm[:, None]
    b1 = np.stack([np.ones(len(p)), np.ones(len(p)), -(d[:, 0] + d[:, 1]) / d[:, 2]], 1)
    b1 /= np.linalg.norm(b1, axis=1)[:, None]
    b2 = np.cross(b1, d)
    b2 /= np.linalg.norm(b2, axis=1)[:, None]
    hat = np.zeros((len(p), 3, 3))
    hat[:, 0, 1], hat[:, 0, 2], hat[:, 1, 0] = -d[:, 2], d[:, 1], d[:, 2]
    hat[:, 1, 2], hat[:, 2, 0], hat[:, 2, 1] = -d[:, 0], -d[:, 1], d[:, 0]
    N = np.stack([b1, b2], 2)
    A = rng[:, None, None] * (hat @ N)
    dv = direction_var(beam_err_deg)
    return d[:, :, None] * rv * d[:, None, :] + dv * (A @ A.transpose(0, 2, 1))


def body_prep(pb, cfg):
    """m_body_cov_list / m_cross_mat_list (voxel_mapping.cpp:1302-1316): z == 0 -> 0.001 first, calcBodyVar at the body point,
    the IMU-frame point R_ext p + t_ext of the modified point.  Returns (body covariances [n,3,3], IMU-frame points [n,3])."""
    p = np.array(pb, dtype=np.float64).reshape(-1, 3)
    p[p[:, 2] == 0, 2] = 0.001
    extR, extT = np.asarray(cfg.ext_R, dtype=np.float64).reshape(3, 3), np.asarray(cfg.ext_T, dtype=np.float64)
    return calc_body_var(p, cfg.dept_err, cfg.beam_err), p @ extR.T + extT


def transform_lidar(s, pb, cfg):
    """transformLidar (voxel_mapping_common.cpp:709-726): R (R_ext p + t_ext) + t in double, stored as float.  Returns float64 values
    of the float world points [n,3]."""
    return world_double(s, pb, cfg).astype(f32).astype(np.float64)


def world_double(s, pb, cfg):
    extR, extT = np.asarray(cfg.ext_R, dtype=np.float64).reshape(3, 3), np.asarray(cfg.ext_T, dtype=np.float64)
    q = np.asarray(pb, dtype=np.float64).reshape(-1, 3) @ extR.T + extT
    return q @ rot(s).T + s[9:12]


def world_cov(Rm, body_cov, p_imu, P):
    """R S R^T + (-[p]x) S_rot (-[p]x)^T + S_t (voxel_mapping.cpp:1353-1356).  Rm: the 3x3 that rotates the body covariance
    (state.rot_end for matching, rot_end * ext_R for the map update), p_imu [n,3], P the 18x18 state covariance."""
    C = np.zeros((len(p_imu), 3, 3))
    C[:, 0, 1], C[:, 0, 2], C[:, 1, 0] = -p_imu[:, 2], p_imu[:, 1], p_imu[:, 2]
    C[:, 1, 2], C[:, 2, 0], C[:, 2, 1] = -p_imu[:, 0], -p_imu[:, 1], p_imu[:, 0]
    return Rm @ body_cov @ Rm.T + (-C) @ P[0:3, 0:3] @ (-C).transpose(0, 2, 1) + P[3:6, 3:6]


def voxel_loc(pw, voxel_size):
    """loc_xyz of voxel_mapping.cpp:118-127 / :173-181: float(p / voxel_size), minus 1.0 (in double, stored as float) when negative.
    voxel_size: the double the caller divides by (lookup: the double parameter; insert: the float parameter as double)."""
    loc = (np.asarray(pw, dtype=np.float64) / voxel_size).astype(f32)
    neg = loc < 0
    loc[neg] = (loc[neg].astype(np.float64) - 1.0).astype(f32)
    return loc


def voxel_key(pw, voxel_size):
    """VOXEL_LOC((int64_t) loc): truncation toward zero of the shifted float"""
    return np.trunc(voxel_loc(pw, voxel_size)).astype(np.int64)


def neighbour_key(key, loc, voxel_size_f):
    """the one-shot retry of BuildResidualListOMP (voxel_mapping.cpp:192-216): the voxel-unit loc compared with the METRIC centre
    +- quarter length of the root voxel, (0.5 + k) * voxel_size and voxel_size / 4 in float (:138-141).  Also returns the margin of
    each comparison (distance of loc to the nearer bound)."""
    vsf = float(f32(voxel_size_f))
    vc = (0.5 + key.astype(np.float64)) * vsf
    ql = float(f32(vsf) / f32(4))
    lo = loc.astype(np.float64)
    nk = key.copy()
    nk[lo > vc + ql] += 1
    nk[(lo < vc - ql) & ~(lo > vc + ql)] -= 1
    margin = np.minimum(np.abs(lo - (vc + ql)), np.abs(lo - (vc - ql))).min(1)
    return nk, margin


# ------------------------------------------------------------------ init_plane, src/voxel_loc.cpp:47-139
def plane_fit(P, V, planer_threshold):
    """OctoTree::init_plane on the ordered points P [n,3] (float64 values of floats) with covariances V [n,3,3].  Centre and
    covariance are summed sequentially in point order (voxel_loc.cpp:55-59); the 6x6 plane covariance is the literal per-point
    sum of J Sigma J^T (:76-101).  Returns a dict with the fields of Plane plus the eigen-decomposition."""
    n = len(P)
    S = np.cumsum(P[:, :, None] * P[:, None, :], axis=0)[-1]
    c = np.cumsum(P, axis=0)[-1] / n
    C = S / n - c[:, None] * c[None, :]
    ev, U = np.linalg.eigh(C)                      # ascending: 0 = min, 2 = max, 1 = mid
    thr = float(f32(planer_threshold))
    out = dict(n=n, center=c, C=C, ev=ev, U=U, is_plane=bool(ev[0] < thr), margin=ev[0] - thr)
    if out["is_plane"]:
        umin = U[:, 0]
        F = np.zeros((n, 3, 3))
        for m in (1, 2):
            Mm = np.outer(U[:, m], umin) + np.outer(umin, U[:, m])
            F[:, m, :] = ((P - c) / (n * (ev[0] - ev[m]))) @ Mm
        J = np.zeros((n, 6, 3))
        J[:, 0:3, :] = U @ F
        J[:, 3:6, :] = I3 / n
        out["pv"] = (J @ V @ J.transpose(0, 2, 1)).sum(0)
        out["normal"] = umin.copy()
        out["min_eig"] = f32(ev[0])
        out["radius"] = f32(math.sqrt(ev[2]))
        out["d"] = f32(-(umin[0] * c[0] + umin[1] * c[1] + umin[2] * c[2]))
    return out


# ------------------------------------------------------------------ OctoTree state machine, src/voxel_loc.cpp:141-308
class Node:
    __slots__ = ("layer", "vc", "quater", "pts", "new_points", "init_octo", "update_enable", "leaves", "plane", "fit_points", "ambiguous",
                 "octo_state", "freeze")

    def __init__(self, layer, vc, quater):
        self.layer, self.vc, self.quater = layer, vc, quater
        self.pts = []                  # indices into the map's point arrays, in m_temp_points_ order
        self.new_points = 0
        self.init_octo = False
        self.update_enable = True
        self.leaves = [None] * 8
        self.plane = None              # last init_plane result (None: never fitted)
        self.fit_points = None         # the ordered point list of the last init_plane
        self.ambiguous = False         # some planar decision here was within the eigen-solver bound of the threshold
        self.octo_state = 0
        self.freeze = None             # "max_points" / "g_max_points" once update_enable turned false


class VoxelMap:
    """buildVoxelMap / updateVoxelMap (src/voxel_mapping.cpp:110-151, :320-354) on Point_with_var lists (world point, 3x3 variance).
    eig_bound(C) gives the absolute eigenvalue error to allow in the planar decision (nodes closer to the threshold are marked)."""

    def __init__(self, cfg, eig_bound):
        self.cfg = cfg
        self.vs_f = f32(cfg.voxel_size)
        self.thr = f32(cfg.min_eigen_value)
        self.eig_bound = eig_bound
        self.roots = {}
        self.P = np.zeros((0, 3))
        self.V = np.zeros((0, 3, 3))
        self.stats = dict(planar_to_nonplanar=0, max_points_freeze=0, g_max_points_freeze=0)

    def _add(self, pw, var):
        base = len(self.P)
        self.P = np.concatenate([self.P, np.asarray(pw, dtype=np.float64)])
        self.V = np.concatenate([self.V, np.asarray(var, dtype=np.float64)])
        return base

    def _root(self, k):
        vsf = float(self.vs_f)
        vc = np.array([(0.5 + float(k[0])) * vsf, (0.5 + float(k[1])) * vsf, (0.5 + float(k[2])) * vsf])
        return Node(0, vc, f32(self.vs_f / f32(4)))

    def _init_plane(self, nd):
        pl = plane_fit(self.P[nd.pts], self.V[nd.pts], self.thr)
        if abs(pl["margin"]) <= self.eig_bound(pl["C"]):
            nd.ambiguous = True
        if nd.plane is not None and nd.plane["is_plane"] and not pl["is_plane"]:
            self.stats["planar_to_nonplanar"] += 1
        nd.plane = pl
        nd.fit_points = list(nd.pts)

    def _child(self, nd, leaf):
        xyz = ((leaf >> 2) & 1, (leaf >> 1) & 1, leaf & 1)
        vc = np.array([nd.vc[j] + float(f32(2 * xyz[j] - 1) * nd.quater) for j in range(3)])
        c = Node(nd.layer + 1, vc, f32(nd.quater / f32(2)))
        nd.leaves[leaf] = c
        return c

    def _leaf(self, nd, i):
        p = self.P[i]
        return 4 * int(p[0] > nd.vc[0]) + 2 * int(p[1] > nd.vc[1]) + int(p[2] > nd.vc[2])

    def _init_octo_tree(self, nd):
        if len(nd.pts) > self.cfg.layer_init_size[nd.layer]:
            self._init_plane(nd)
            if nd.plane["is_plane"]:
                nd.octo_state = 0
            else:
                nd.octo_state = 1
                self._cut(nd)
            nd.init_octo = True
            nd.new_points = 0

    def _cut(self, nd):
        if nd.layer >= self.cfg.max_layer:
            nd.octo_state = 0
            return
        for i in nd.pts:
            leaf = self._leaf(nd, i)
            c = nd.leaves[leaf] or self._child(nd, leaf)
            c.pts.append(i)
            c.new_points += 1
        for c in nd.leaves:
            if c is not None and len(c.pts) > self.cfg.layer_init_size[c.layer]:
                self._init_plane(c)
                if c.plane["is_plane"]:
                    c.octo_state = 0
                else:
                    c.octo_state = 1
                    self._cut(c)
                c.init_octo = True
                c.new_points = 0

    def _update(self, nd, i):
        cfg = self.cfg
        while True:
            if not nd.init_octo:
                nd.new_points += 1
                nd.pts.append(i)
                if len(nd.pts) > cfg.layer_init_size[nd.layer]:
                    self._init_octo_tree(nd)
                return
            if nd.plane["is_plane"]:
                if nd.update_enable:
                    nd.new_points += 1
                    nd.pts.append(i)
                    if nd.new_points > UPDATE_SIZE_THRESHOLD:
                        self._init_plane(nd)
                        nd.new_points = 0
                    if len(nd.pts) >= cfg.max_points_size:
                        nd.update_enable = False
                        nd.pts = []
                        nd.new_points = 0
                        nd.freeze = "max_points"
                        self.stats["max_points_freeze"] += 1
                return
            if nd.layer < cfg.max_layer:
                if len(nd.pts) != 0:
                    nd.pts = []
                leaf = self._leaf(nd, i)
                nd = nd.leaves[leaf] or self._child(nd, leaf)
                continue
            if nd.update_enable:
                nd.new_points += 1
                nd.pts.append(i)
                if nd.new_points > UPDATE_SIZE_THRESHOLD:
                    self._init_plane(nd)
                    nd.new_points = 0
                if len(nd.pts) > G_MAX_POINTS:
                    nd.update_enable = False
                    nd.pts = []
                    nd.freeze = "g_max_points"
                    self.stats["g_max_points_freeze"] += 1
            return

    def build(self, pw, var):
        base = self._add(pw, var)
        keys = voxel_key(pw, float(self.vs_f))
        for j, k in enumerate(map(tuple, keys)):
            nd = self.roots.get(k)
            if nd is None:
                nd = self.roots[k] = self._root(k)
            nd.pts.append(base + j)
            nd.new_points += 1
        for k in self.roots:
            self._init_octo_tree(self.roots[k])

    def update(self, pw, var):
        base = self._add(pw, var)
        keys = voxel_key(pw, float(self.vs_f))
        for j, k in enumerate(map(tuple, keys)):
            nd = self.roots.get(k)
            if nd is None:
                nd = self.roots[k] = self._root(k)
            self._update(nd, base + j)

    def nodes(self):
        """(key, path, node) in the canonical dump order: roots by ascending key, nodes in pre-order (child l -> path * 9 + l + 1)"""
        out = []

        def rec(k, nd, path):
            out.append((k, path, nd))
            for l, c in enumerate(nd.leaves):
                if c is not None:
                    rec(k, c, path * 9 + l + 1)
        for k in sorted(self.roots):
            rec(k, self.roots[k], 0)
        return out


def var_contrast(var):
    """the sort key of the map update's Point_with_var list (voxel_mapping.cpp:49): |diag(var)|"""
    d = np.stack([var[:, 0, 0], var[:, 1, 1], var[:, 2, 2]], 1)
    return np.sqrt((d * d).sum(1))


# ------------------------------------------------------------------ residual selection on a map dump, voxel_mapping.cpp:153-318
DUMP_KEY, DUMP_PATH, DUMP_LAYER, DUMP_PLANE = slice(0, 3), 3, 4, 6
DUMP_CENTER, DUMP_NORMAL, DUMP_D, DUMP_RADIUS = slice(11, 14), slice(14, 17), 17, 18
DUMP_PV = slice(24, 45)
IU = np.triu_indices(6)


def pv_full(row):
    M = np.zeros((6, 6))
    M[IU] = row[DUMP_PV]
    return M + np.triu(M, 1).T


class DumpPlanes:
    """The plane records of a canonical map dump (immesh_voxelmap_dump), indexed by root key.  build_single_residual's walk below a
    root visits child 0..7 depth first and evaluates every planar node it reaches; a planar node has no children that the walk
    enters, and nothing lies deeper than max_layer, so the candidates of a root are its planar rows in dump order."""

    def __init__(self, dump):
        self.dump = dump
        self.by_root = {}
        keys = dump[:, DUMP_KEY].astype(np.int64)
        start = 0
        for r in range(1, len(dump) + 1):
            if r == len(dump) or not np.array_equal(keys[r], keys[start]) or dump[r, DUMP_PATH] == 0:
                rows = np.arange(start, r)
                self.by_root[tuple(keys[start])] = rows[self._walk(rows)]
                start = r

    def _walk(self, rows):
        """rows reached by the walk and planar, in walk order"""
        d = self.dump
        keep = []
        blocked = set()
        for j, r in enumerate(rows):
            path = int(d[r, DUMP_PATH])
            par, anc = path, []
            while par:
                par //= 9
                anc.append(par)
            if any(a in blocked for a in anc):
                continue
            if d[r, DUMP_PLANE] == 1:
                keep.append(j)
                blocked.add(path)
        return np.asarray(keep, dtype=np.int64)


def match_points(planes, pw, var, voxel_size, voxel_size_f, sigma_num=3.0):
    """BuildResidualListOMP + build_single_residual for world points pw [n,3] (float64; float values for the float PointXYZI path)
    with variances var [n,3,3]: the root voxel by the lookup rule (double voxel_size), its planes in walk order, the one retry in
    the neighbour voxel when nothing passed both gates.  Vectorised per root voxel.  Returns per point the chosen dump row (-1: no
    match), and the margins of every decision taken (a dict of arrays, NaN where the decision was not taken)."""
    n = len(pw)
    loc = voxel_loc(pw, voxel_size)
    key = np.trunc(loc).astype(np.int64)
    nkey, nmargin = neighbour_key(key, loc, voxel_size_f)
    best = np.full(n, -1, dtype=np.int64)
    marg = dict(range=np.full(n, np.inf), sigma=np.full(n, np.inf), prob=np.full(n, np.inf), loc=np.full(n, np.inf))
    stats = dict(range_reject=0, sigma_reject=0, retry_success=0, non_first_argmax=0)
    frac = np.abs(loc.astype(np.float64) - np.round(loc.astype(np.float64))).min(1)
    marg["loc"] = frac

    def evaluate(idx, rows):
        """the walk over `rows` for the points idx; returns (ok, best row, best prob, best candidate position, second prob)"""
        d = planes.dump
        m = len(idx)
        ok = np.zeros(m, bool)
        prob = np.zeros(m)
        second = np.zeros(m)
        brow = np.full(m, -1, dtype=np.int64)
        bpos = np.full(m, -1, dtype=np.int64)
        p = pw[idx]
        for pos, r in enumerate(rows):
            nrm, c, dd, rad = d[r, DUMP_NORMAL], d[r, DUMP_CENTER], float(d[r, DUMP_D]), float(d[r, DUMP_RADIUS])
            dis_plane = np.abs(p @ nrm + dd).astype(f32)
            dis_center = (((c - p) ** 2).sum(1)).astype(f32)
            range_dis = np.sqrt(dis_center - dis_plane * dis_plane)
            g1 = range_dis.astype(np.float64) <= 3.0 * rad
            rel1 = np.abs(range_dis.astype(np.float64) - 3.0 * rad) / np.maximum(3.0 * rad, 1e-30)
            J = np.concatenate([p - c, np.broadcast_to(-nrm, p.shape)], 1)
            sigma = np.einsum("ni,ij,nj->n", J, pv_full(d[r]), J) + np.einsum("i,nij,j->n", nrm, var[idx], nrm)
            sq = np.sqrt(sigma)
            g2 = dis_plane.astype(np.float64) < sigma_num * sq
            rel2 = np.abs(dis_plane.astype(np.float64) - sigma_num * sq) / np.maximum(sigma_num * sq, 1e-30)
            stats["range_reject"] += int((~g1).sum())
            stats["sigma_reject"] += int((g1 & ~g2).sum())
            marg["range"][idx] = np.minimum(marg["range"][idx], rel1)
            marg["sigma"][idx] = np.minimum(marg["sigma"][idx], np.where(g1, rel2, np.inf))
            acc = g1 & g2
            ok |= acc
            pr = np.where(acc, 1.0 / sq * np.exp(-0.5 * dis_plane.astype(np.float64) ** 2 / sigma), 0.0)
            better = acc & (pr > prob)
            second = np.where(better, prob, np.maximum(second, np.where(acc, pr, 0.0)))
            prob = np.where(better, pr, prob)
            brow = np.where(better, r, brow)
            bpos = np.where(better, pos, bpos)
        return ok, brow, prob, bpos, second

    groups = {}
    for i, k in enumerate(map(tuple, key)):
        groups.setdefault(k, []).append(i)
    retry = {}
    for k, idx in groups.items():
        if k not in planes.by_root:
            continue
        idx = np.asarray(idx)
        ok, brow, prob, bpos, second = evaluate(idx, planes.by_root[k])
        best[idx[ok]] = brow[ok]
        stats["non_first_argmax"] += int((ok & (bpos > 0)).sum())
        pg = np.where(ok & (second > 0), (prob - second) / np.maximum(prob, 1e-300), np.inf)
        marg["prob"][idx] = pg
        for i in idx[~ok]:
            retry.setdefault(tuple(nkey[i]), []).append(i)
            marg["loc"][i] = min(marg["loc"][i], nmargin[i] / max(abs(float(loc[i].max())), 1.0))
    for k, idx in retry.items():
        if k not in planes.by_root:
            continue
        idx = np.asarray(idx)
        ok, brow, prob, bpos, second = evaluate(idx, planes.by_root[k])
        best[idx[ok]] = brow[ok]
        stats["retry_success"] += int(ok.sum())
        stats["non_first_argmax"] += int((ok & (bpos > 0)).sum())
        marg["prob"][idx] = np.where(ok & (second > 0), (prob - second) / np.maximum(prob, 1e-300), np.inf)
    return best, marg, stats


# ------------------------------------------------------------------ normal equations, voxel_mapping.cpp:1372-1392, :1493-1586
def normal_equations(s, pb, rows, dump, cfg):
    """HTH (6x6), HTz (6), sum|dis| and R_inv per point for the matched body points pb [m,3] (float values) against the dump rows
    `rows` at state s.  Normal and residual through the float PCL structs; R_inv with calcBodyVar at the IMU-frame point of the
    raw point (CALIB_ANGLE_COV when calib_laser); A = [p_imu]x R^T n_f; the sums over points in float64 by math.fsum."""
    R, t = rot(s), s[9:12]
    extR, extT = np.asarray(cfg.ext_R, dtype=np.float64).reshape(3, 3), np.asarray(cfg.ext_T, dtype=np.float64)
    d = dump[rows]
    nd = d[:, DUMP_NORMAL]
    nf = nd.astype(f32).astype(np.float64)
    pwd = world_double(s, pb, cfg)
    dis = ((pwd * nf).sum(1) + d[:, DUMP_D]).astype(f32).astype(np.float64)
    p_imu = np.asarray(pb, dtype=np.float64) @ extR.T + extT
    bv = calc_body_var(p_imu, cfg.dept_err, CALIB_ANGLE_COV if cfg.calib_laser else cfg.beam_err)
    RRe = R @ extR
    var = RRe @ bv @ RRe.T
    pw2 = p_imu @ R.T + t
    J = np.concatenate([pw2 - d[:, DUMP_CENTER], -nd], 1)
    PV = np.stack([pv_full(r) for r in d]) if len(d) else np.zeros((0, 6, 6))
    sigma_l = np.einsum("ni,nij,nj->n", J, PV, J)
    R_inv = 1.0 / (sigma_l + np.einsum("ni,nij,nj->n", nf, var, nf))
    A = np.cross(p_imu, nf @ R)                    # [p]x R^T n
    H = np.concatenate([A, nf], 1)
    z = -dis
    HTH = np.array([[math.fsum(H[:, a] * R_inv * H[:, b]) for b in range(6)] for a in range(6)])
    HTz = np.array([math.fsum(H[:, a] * R_inv * z) for a in range(6)])
    return dict(HTH=HTH, HTz=HTz, total_residual=math.fsum(np.abs(dis)), R_inv=R_inv, H=H, z=z)


# ------------------------------------------------------------------ IESKF update, voxel_mapping.cpp:1586-1650
def ieskf_solution(HTH6, HTz, s, s_prop):
    """the literal form: K1 = (H^T R^-1 H (+) 0_12 + P^-1)^-1 with two general inverses, G = K1[:, :6] HTH, v = s_prop - s,
    solution = K1[:, :6] HTz + v - G[:, :6] v[:6].  Returns (solution, G[18,18])."""
    P = cov(s)
    M = np.linalg.inv(P)
    M[:6, :6] += HTH6
    K1 = np.linalg.inv(M)
    G = np.zeros((18, 18))
    G[:, :6] = K1[:, :6] @ HTH6
    v = state_minus(s_prop, s)
    return K1[:, :6] @ HTz + v - G[:, :6] @ v[:6], G


def converged(sol):
    """(rot_add.norm() * 57.3 < 0.01) && (t_add.norm() * 100 < 0.015)  (:1621-1624)"""
    return bool(np.linalg.norm(sol[0:3]) * 57.3 < 0.01 and np.linalg.norm(sol[3:6]) * 100 < 0.015)


def ieskf_flags(conv, rematch_num, it, max_iter):
    """rematch judgement and the stop / covariance-update rule (:1627-1650): returns (rematch_num, stop)"""
    if conv or (rematch_num == 0 and it == max_iter - 2):
        rematch_num += 1
    return rematch_num, (rematch_num >= 2 or it == max_iter - 1)
