"""Pure-numpy scene generator for the mesher's size- and geometry-dependent paths (TEST INFRASTRUCTURE ONLY).

Every scene is a list of frames (float32[m,3] world points, pose) plus the MeshConfig overrides it needs.  Unless a scene says
otherwise its points lie inside one mesh voxel, clear of the voxel's borders, and at least 2 * points_minimum_scale
apart, so that every point becomes a vertex and the voxel's dilated set is exactly its own vertices.  The points of a frame are
appended in array order, so the array order is the vertex-id order, which is the Bowyer-Watson insertion order.

Which device path a voxel takes follows from its dilated-set size n and the largest conflict region of its insertions (the
oracle's OracleMesh.frame_voxel_stats; the kernels insert in the same order with the same exact predicates):
    n <= 96 (IM_WARP_NMAX), every cavity <= 64 and <= 192 prefiltered triangles   k_voxel_tri_warp
        one insertion with cavity * 3 <= 32                                            its one_pass boundary search
    n <= 96, a cavity > 64                                                             warp hand-over to k_voxel_mesh<1024>
    97 <= n <= 256                                                                     k_voxel_mesh<256> + k_commit_faces
    257 <= n <= 1024                                                                   k_voxel_mesh<1024> (commit in shared memory)
    > 256 vertices in one voxel, n > 1024, a cavity > 256 in the 1024 variant          IMMESH_E_CAPACITY
"""
import numpy as np

class Scene:
    def __init__(self, name, frames, cfg_kw, centre):
        self.name, self.frames, self.cfg_kw, self.centre = name, frames, cfg_kw, np.asarray(centre, np.float64)

    @property
    def n_points(self):
        return sum(len(f) for f in self.frames)

    def __repr__(self):
        return f"Scene({self.name})"


def voxel_centre(key, res):
    return np.asarray(key, np.float64) * res


def _f32(p):
    return np.ascontiguousarray(p, dtype=np.float32)


def min_distance(p):
    p = np.asarray(p, np.float64)
    d = np.sqrt(((p[:, None, :] - p[None, :, :]) ** 2).sum(-1))
    d[np.arange(len(p)), np.arange(len(p))] = np.inf
    return d.min()


def _plane_basis(tilt):
    """orthonormal in-plane axes (e1 = x, e2 = y tilted by `tilt` radians about x) and the normal"""
    c, s = np.cos(tilt), np.sin(tilt)
    return np.array([1.0, 0, 0]), np.array([0, c, s]), np.array([0, -s, c])


def jittered_patch(n, key=(3, -2, 5), res=0.4, xi=0.004, seed=0, extent=(0.18, 0.12), grid=(16, 16), tilt=0.3, jitter=0.003, extra_outside=False):
    """n points of a jittered 16 x 16 grid on a tilted plane through the voxel's centre, in a random order (the first n of a
    random permutation).  extra_outside: one more point, appended last, just across the voxel's +x border next to the patch's
    edge column: it is in the 20-NN of the patch's edge vertices, so the voxel's dilated set is n + 1."""
    rng = np.random.default_rng(seed)
    c = voxel_centre(key, res)
    e1, e2, _ = _plane_basis(tilt)
    gx, gy = np.meshgrid(np.linspace(-extent[0], extent[0], grid[0]), np.linspace(-extent[1], extent[1], grid[1]), indexing="ij")
    uv = np.stack([gx.ravel(), gy.ravel()], 1) + rng.uniform(-jitter, jitter, (grid[0] * grid[1], 2))
    uv = uv[rng.permutation(len(uv))[:n]]
    pts = c + uv[:, :1] * e1 + uv[:, 1:] * e2
    if extra_outside:
        edge = uv[np.argmax(uv[:, 0])]
        pts = np.concatenate([pts, (c + (res / 2 + 0.015) * e1 + edge[1] * e2)[None]])
    pts = _f32(pts)
    assert min_distance(pts) >= 2 * xi
    name = f"patch{n}" + ("+1" if extra_outside else "")
    return Scene(name, [pts], dict(points_minimum_scale=xi, voxel_resolution=res), c)


def ring(n_ring, key=(3, -2, 5), res=0.4, xi=0.001, radius=0.15, tilt=0.3, with_centre=True):
    """N points equally spaced on a circle (frame 0, angular order), then the circle's centre (frame 1).  Appending the centre
    re-meshes the voxel with the centre inserted last: its conflict region is every one of the N - 2 triangles of the ring.
    The in-plane covariance is isotropic, so the projection axes come from the eigen-solver's tie-breaking."""
    c = voxel_centre(key, res)
    e1, e2, _ = _plane_basis(tilt)
    a = 2 * np.pi * np.arange(n_ring) / n_ring
    pts = _f32(c + radius * (np.cos(a)[:, None] * e1 + np.sin(a)[:, None] * e2))
    assert min_distance(pts) >= 2 * xi
    frames = [pts] + ([_f32(c[None])] if with_centre else [])
    return Scene(f"ring{n_ring}", frames, dict(points_minimum_scale=xi, voxel_resolution=res), c)


def ring_fan(n_ring):
    """the closed-form live facet set after ring(n_ring)'s second frame: the fan (centre, r_i, r_i+1), sorted id triples"""
    cen = n_ring
    t = np.array([sorted((i, (i + 1) % n_ring, cen)) for i in range(n_ring)], dtype=np.int32)
    return t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]


def lattice(nx=8, ny=8, dx=0.03125, dy=0.046875, key=(2, -3, 2), res=0.5, xi=0.01, seed=1):
    """a rectangular lattice with two different binary-exact spacings in the axis-aligned plane z = const, all coordinates
    binary-exact: res = 0.5 makes the snap unit a power of two and a power-of-two point count makes the centroid exact, so the
    snapped coordinates are an exact rectangular lattice and every lattice rectangle is cocircular (in-circle == 0).  Points
    in a random order."""
    rng = np.random.default_rng(seed)
    c = voxel_centre(key, res) + np.array([0.0625, -0.03125, 0.09375])
    gx, gy = np.meshgrid((np.arange(nx) - (nx - 1) / 2) * dx, (np.arange(ny) - (ny - 1) / 2) * dy, indexing="ij")
    pts = np.stack([c[0] + gx.ravel(), c[1] + gy.ravel(), np.full(nx * ny, c[2])], 1)
    pts = pts[rng.permutation(len(pts))]
    assert np.array_equal(pts.astype(np.float32).astype(np.float64), pts)
    return Scene(f"lattice{nx}x{ny}", [_f32(pts)], dict(points_minimum_scale=xi, voxel_resolution=res), c)


def stacked(nx=6, ny=6, key=(3, -2, 5), res=0.4, xi=0.01, seed=2, spacing=0.04):
    """two copies of a jittered grid, 1.5 xi apart along the normal of the axis-aligned plane: distinct xi-cells (both become
    vertices) that project onto the same snapped points, so every second-layer insertion is a duplicate skip"""
    rng = np.random.default_rng(seed)
    c = voxel_centre(key, res)
    gx, gy = np.meshgrid((np.arange(nx) - (nx - 1) / 2) * spacing, (np.arange(ny) - (ny - 1) / 2) * spacing, indexing="ij")
    xy = np.stack([gx.ravel(), gy.ravel()], 1) + rng.uniform(-0.004, 0.004, (nx * ny, 2))
    z0 = c[2] + 0.0125
    lo = np.concatenate([c[:2] + xy, np.full((nx * ny, 1), z0)], 1)
    hi = lo.copy()
    hi[:, 2] = z0 + 1.5 * xi
    pts = _f32(np.concatenate([lo, hi]))
    return Scene(f"stacked{nx}x{ny}", [pts], dict(points_minimum_scale=xi, voxel_resolution=res), c)


def collinear(n=12, key=(3, -2, 5), res=0.4, xi=0.004, spacing=0.025):
    """every point on one axis-parallel line (exact in float): no seed triangle, no facets"""
    c = voxel_centre(key, res)
    pts = np.tile(c + np.array([0.0, 0.03, -0.02]), (n, 1))
    pts[:, 0] += (np.arange(n) - (n - 1) / 2) * spacing
    return Scene(f"collinear{n}", [_f32(pts)], dict(points_minimum_scale=xi, voxel_resolution=res), c)


def shell(per_face=(7, 6), cluster=3, key=(3, -2, 5), res=0.4, xi=0.001, spacing=0.04, gap=0.003, rho=0.004):
    """Large dilated sets without breaking the per-voxel vertex cap: 6 * 42 vertices just inside the six faces of one voxel, each
    with a private cluster of `cluster` vertices just across the face (in the face neighbour), nearer to it than anything
    else.  The centre voxel's dilated set is then 42 * 6 * (1 + cluster) (1008 for cluster = 3, 1260 for 4), every voxel holds
    at most 256 vertices and the gathered neighbourhood stays below IM_MAXG.  Not a single-voxel scene."""
    c = voxel_centre(key, res)
    offs = np.array([[0, 0], [rho, 0], [-rho, 0], [0, rho], [0, -rho]])[:cluster]
    gu, gv = np.meshgrid((np.arange(per_face[0]) - (per_face[0] - 1) / 2) * spacing, (np.arange(per_face[1]) - (per_face[1] - 1) / 2) * spacing, indexing="ij")
    uv = np.stack([gu.ravel(), gv.ravel()], 1)
    inner, outer = [], []
    for axis in range(3):
        a1, a2 = [k for k in range(3) if k != axis]
        for sgn in (-1.0, 1.0):
            for u, v in uv:
                p = c.copy()
                p[a1] += u
                p[a2] += v
                q = p.copy()
                p[axis] += sgn * (res / 2 - gap)
                inner.append(p)
                for du, dv in offs:
                    o = q.copy()
                    o[axis] += sgn * (res / 2 + gap)
                    o[a1] += du
                    o[a2] += dv
                    outer.append(o)
    pts = _f32(np.concatenate([np.array(inner), np.array(outer)]))
    assert min_distance(pts) >= 2 * xi
    return Scene(f"shell_c{cluster}", [pts], dict(points_minimum_scale=xi, voxel_resolution=res), c)


def xi_tie(xi=0.125, res=0.4):
    """points exactly xi apart in float (xi and every coordinate binary-exact), in different xi-cells: frame 0 holds two of them
    (the in-frame test), frame 1 one more at distance xi from the first vertex (the test against the map).  sqrtf(d) == xi, so
    every one of them is appended: the reference rejects only points strictly closer than xi.  The first point's x / res is 2.5,
    where std::round (half away from zero) and round-half-to-even disagree."""
    a = np.array([1.0, 2.0, 0.5])
    frames = [_f32([a, a + [0.0, xi, 0.0]]), _f32([a + [xi, 0.0, 0.0]])]
    return Scene("xi_tie", frames, dict(points_minimum_scale=xi, voxel_resolution=res), a)


def voxel_key(p, res):
    return np.round(np.asarray(p, np.float64) / res).astype(np.int64)


def centre_stats(stats, scene, res):
    """the frame_voxel_stats row of the scene's own voxel"""
    k = voxel_key(scene.centre, res)
    rows = np.where((stats["key"] == k).all(1))[0]
    assert len(rows) == 1, (scene, k, stats["key"])
    return {f: v[rows[0]] for f, v in stats.items()}


# ---------------------------------------------------------------- the scene list shared by the emulation and GPU tiers
def path_scenes():
    """(scene, expected path of its voxel in the last frame)"""
    return [
        (jittered_patch(3), "warp"),
        (jittered_patch(96, seed=3), "warp_one_pass"),
        (jittered_patch(97, seed=4), "block256"),
        (jittered_patch(256, seed=5), "block256"),
        (jittered_patch(256, seed=6, extra_outside=True), "block1024"),
        (shell(cluster=3), "block1024"),
        (ring(30), "warp"),
        (ring(67), "handover"),
        (ring(95), "handover"),
        (ring(100), "block256"),
        (ring(250), "block256"),
        (lattice(), "warp_one_pass"),
        (lattice(16, 8, dx=0.015625, xi=0.005), "block256"),
        (stacked(), "warp_one_pass"),
        (stacked(8, 8), "block256"),
        (collinear(), "noseed"),
    ]


def path_of(st):
    """the device path a voxel with these oracle stats takes (module docstring)"""
    n, cav = int(st["n"]), int(st["max_cav"])
    if not st["seeded"]:
        return "noseed"
    if n <= 96:   # warp_one_pass: there were insertions and every one of them took the one_pass boundary search
        return "handover" if cav > 64 else ("warp_one_pass" if n > 3 and cav * 3 <= 32 else "warp")
    if n <= 256:
        return "block256"
    return "block1024" if n <= 1024 else "cap"


def cap_scenes():
    """scenes the product must refuse with IMMESH_E_CAPACITY: > 256 vertices in one voxel (a patch, a ring), a dilated set > 1024"""
    return [
        jittered_patch(300, grid=(20, 15), extent=(0.17, 0.12), xi=0.002, jitter=0.002, seed=7),
        ring(300, with_centre=False),
        shell(cluster=4),
    ]
