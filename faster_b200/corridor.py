"""Synthetic corridor problems shaped like the inputs Faster::replan() feeds SolverGurobi.

Input generator for tests and bench.py only (JPS3D and the ellipsoid decomposition stay host-side input
generators, SURVEY.md section 2); the conventions follow SURVEY.md Appendix B:
  * one polytope per polyline segment (jps_manager.cpp:113), rows A x <= b with outward unit normals,
    sign-normalised w.r.t. the segment midpoint (polyhedron.h:131-152);
  * face order: obstacle-derived half-spaces (inflated by drone_radius, line_segment.h:178-190), then the six
    local-bbox faces +-dir_h (half width 2), +dir beyond p2 / -dir behind p1 (2), +-dir_v (1)
    (line_segment.h:57-98, jps_manager.cpp:100), then the ground face -z <= -z_ground (jps_manager.cpp:118-122);
  * whole: x0 = committed plan state, xf = rest at the last vertex (faster.cpp:402-407);
    safe: same model with forceFinalConstraint=false (faster.cpp:521-524).
"""
import itertools
import numpy as np

UAV = dict(lim=(5.0, 5.0, 8.0), z_ground=0.0, drone_radius=0.42, bbox=(2.0, 2.0, 1.0), seg=(1.0, 1.5),
           z=(0.5, 1.5), turn=60.0, v0=(0.0, 2.0))           # faster.yaml:7,14,18,23-25,39
GROUND = dict(lim=(1.4, 1.4, 5.0), z_ground=-0.2, drone_radius=0.5, bbox=(2.0, 0.8, 0.4), seg=(0.5, 0.9),
              z=(0.2, 0.2), turn=45.0, v0=(0.0, 0.8))        # Readme.md:112-124


def monotone_sigmas(N, P):
    """All non-decreasing interval->polytope assignments: C(N+P-1, P-1) rows of length N (uint8)."""
    out = []
    for cuts in itertools.combinations_with_replacement(range(N + 1), P - 1):
        s = np.zeros(N, np.uint8)
        for c in cuts:
            s[c:] += 1
        out.append(s)
    return np.array(sorted(map(tuple, out)), np.uint8).reshape(-1, N)


def sample_monotone_sigmas(N, P, n, rng):
    """n distinct-ish monotone assignments for large (N,P) where the full list is too long."""
    cuts = np.sort(rng.integers(0, N + 1, size=(n, P - 1)), axis=1)
    s = np.zeros((n, N), np.uint8)
    for k in range(P - 1):
        s += (np.arange(N)[None, :] >= cuts[:, k:k + 1]).astype(np.uint8)
    return s


def _segment_polytope(p1, p2, rng, prof, n_cut):
    d = p2 - p1
    dirv = d / np.linalg.norm(d)
    dir_h = np.array([dirv[1], -dirv[0], 0.0])
    if np.linalg.norm(dir_h) == 0:
        dir_h = np.array([-1.0, 0.0, 0.0])
    dir_h /= np.linalg.norm(dir_h)
    dir_v = np.cross(dirv, dir_h)
    planes = []                                              # (point, outward normal)
    r = prof["drone_radius"]
    for _ in range(n_cut):
        s = rng.uniform(0.0, 1.0)
        c = p1 + s * d
        ang = rng.uniform(0, 2 * np.pi)
        n = np.cos(ang) * dir_h + np.sin(ang) * dir_v + rng.uniform(-0.3, 0.3) * dirv
        n /= np.linalg.norm(n)
        dist = rng.uniform(r + 0.12, r + 1.2)                # obstacle point at c + dist*n, inflated by r
        planes.append((c + (dist - r) * n, n))
    bb = prof["bbox"]
    planes += [(p1 + dir_h * bb[1], dir_h), (p1 - dir_h * bb[1], -dir_h),
               (p2 + dirv * bb[0], dirv), (p1 - dirv * bb[0], -dirv),
               (p1 + dir_v * bb[2], dir_v), (p1 - dir_v * bb[2], -dir_v)]
    mid = 0.5 * (p1 + p2)
    A, b = [], []
    for pt, n in planes:
        c = float(pt @ n)
        if n @ mid - c > 0:
            n, c = -n, -c
        A.append(n)
        b.append(c)
    A.append(np.array([0.0, 0.0, -1.0]))
    b.append(-prof["z_ground"])
    return np.array(A), np.array(b)


def make_corridor(seed, P, N, profile="uav", force_final=True, DC=0.01):
    """One corridor problem: dict(N, P, x0[9], xf[9], lim[3], polys[(A,b)], force_final, DC, verts)."""
    prof = UAV if profile == "uav" else GROUND
    rng = np.random.default_rng(seed)
    verts = [np.array([rng.uniform(-5, 5), rng.uniform(-5, 5), rng.uniform(*prof["z"])])]
    yaw = rng.uniform(-np.pi, np.pi)
    for _ in range(P):
        yaw += np.deg2rad(rng.uniform(-prof["turn"], prof["turn"]))
        L = rng.uniform(*prof["seg"])
        z = rng.uniform(*prof["z"])
        nxt = verts[-1] + np.array([L * np.cos(yaw), L * np.sin(yaw), 0.0])
        nxt[2] = z
        verts.append(nxt)
    polys = [_segment_polytope(verts[i], verts[i + 1], rng, prof, int(rng.integers(1, 7))) for i in range(P)]
    d0 = verts[1] - verts[0]
    d0 /= np.linalg.norm(d0)
    x0 = np.zeros(9)
    x0[:3] = verts[0]
    x0[3:6] = d0 * rng.uniform(*prof["v0"])
    x0[6:9] = rng.uniform(-0.3, 0.3, 3) * (0.0 if profile != "uav" else 1.0)
    xf = np.zeros(9)
    xf[:3] = verts[-1]
    return dict(N=N, P=P, x0=x0, xf=xf, lim=np.array(prof["lim"]), polys=polys, force_final=bool(force_final),
                DC=DC, verts=np.array(verts), seed=seed, profile=profile)


# ------------------------------------------------------------------------------------------------------------------
# Random-forest corridors (BASELINE config 4): obstacle point cloud -> polyline -> convex decomposition -> polytopes.
# The polyline stands in for the JPS3D path (out of scope, SURVEY section 2); the decomposition is the product's
# host-side restatement of JPS_Manager::cvxEllipsoidDecomp (faster_b200/csrc/fq_decomp.cpp).
# ------------------------------------------------------------------------------------------------------------------
def make_forest(seed, n_trees=60, area=16.0, height=3.0, res=0.15):
    """Vertical cylinders (radius U[0.1,0.3], density ~ launch/ground_robot.launch 'density01') sampled on their
    surface at `res` metres, like a voxelised map.  -> (points [n,3], centres [n_trees,2], radii [n_trees])."""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-area / 2, area / 2, (n_trees, 2))
    radii = rng.uniform(0.1, 0.3, n_trees)
    pts = []
    for c, r in zip(centres, radii):
        th = np.arange(0, 2 * np.pi, res / r)
        zs = np.arange(0.0, height, res)
        ring = np.stack([c[0] + r * np.cos(th), c[1] + r * np.sin(th)], axis=1)
        pts.append(np.concatenate([np.hstack([ring, np.full((len(ring), 1), z)]) for z in zs]))
    return np.concatenate(pts), centres, radii


def _seg_point_dist_xy(a, b, c):
    ab = b - a
    t = np.clip(((c - a) @ ab) / max(ab @ ab, 1e-12), 0.0, 1.0)
    return np.linalg.norm(a + t * ab - c)


def forest_path(seed, centres, radii, n_seg, clearance, seg_len=(1.0, 1.5), z=(0.8, 1.4), area=16.0, tries=4000):
    """Polyline of n_seg segments whose every segment keeps `clearance` from every tree (xy distance to the axis minus
    the radius).  Rejection sampling; raises if the forest is too dense."""
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        p = np.array([rng.uniform(-area / 2 + 2, area / 2 - 2), rng.uniform(-area / 2 + 2, area / 2 - 2), rng.uniform(*z)])
        yaw = rng.uniform(-np.pi, np.pi)
        verts, ok = [p], True
        for _s in range(n_seg):
            yaw += np.deg2rad(rng.uniform(-50, 50))
            L = rng.uniform(*seg_len)
            q = verts[-1] + np.array([L * np.cos(yaw), L * np.sin(yaw), 0.0])
            q[2] = rng.uniform(*z)
            if any(_seg_point_dist_xy(verts[-1][:2], q[:2], c) - r < clearance for c, r in zip(centres, radii)):
                ok = False
                break
            verts.append(q)
        if ok:
            return np.array(verts)
    raise RuntimeError("no collision-free polyline found")


def make_forest_corridor(seed, P, N, force_final=True, decomp=None, DC=0.01, n_trees=60):
    """Corridor problem whose polytopes come from the convex decomposition of a random forest around a polyline.
    decomp(path, obs, bbox, inflate, z_ground) -> [(A,b)...]; default = the product's fq_ellipsoid_decomp."""
    if decomp is None:
        from . import capi
        decomp = capi.ellipsoid_decomp
    prof = UAV
    obs, centres, radii = make_forest(seed, n_trees=n_trees)
    verts = forest_path(seed + 1, centres, radii, P, clearance=prof["drone_radius"] * 1.45 + 0.05)
    polys = decomp(verts, obs, prof["bbox"], prof["drone_radius"], prof["z_ground"])
    rng = np.random.default_rng(seed + 2)
    d0 = verts[1] - verts[0]
    d0 /= np.linalg.norm(d0)
    x0 = np.zeros(9)
    x0[:3] = verts[0]
    x0[3:6] = d0 * rng.uniform(*prof["v0"])
    xf = np.zeros(9)
    xf[:3] = verts[-1]
    return dict(N=N, P=P, x0=x0, xf=xf, lim=np.array(prof["lim"]), polys=polys, force_final=bool(force_final), DC=DC,
                verts=verts, obs=obs, seed=seed, profile="uav")


# ------------------------------------------------------------------------------------------------------------------
# The whole input side on the host, as Faster::replan() chains it (faster.cpp:361-398): voxel map -> JPS3D path ->
# vertices at most dist_max_vertexes apart, at most max_poly segments -> convex decomposition -> polytopes.
# ------------------------------------------------------------------------------------------------------------------
def voxelise_forest(centres, radii, area=16.0, height=3.0, res=0.15, inflation=0.0):
    """Occupancy grid [zd,yd,xd] (int8: 0 free, 100 occupied) of vertical cylinders, origin at (-area/2,-area/2,0)."""
    n = int(round(area / res))
    zd = int(round(height / res))
    xs = (np.arange(n) + 0.5) * res - area / 2
    X, Y = np.meshgrid(xs, xs)
    occ = np.zeros((n, n), bool)
    for c, r in zip(centres, radii):
        occ |= (X - c[0]) ** 2 + (Y - c[1]) ** 2 <= (r + inflation) ** 2
    g = np.zeros((zd, n, n), np.int8)
    g[:, occ] = 100
    return g, np.array([-area / 2, -area / 2, 0.0]), res


def split_long_segments(path, max_len):
    """createMoreVertexes (faster.cpp:80-97): subdivide segments longer than max_len evenly."""
    out = [path[0]]
    for a, b in zip(path[:-1], path[1:]):
        k = int(np.ceil(np.linalg.norm(b - a) / max_len))
        for i in range(1, k + 1):
            out.append(a + (b - a) * (i / k))
    return np.array(out)


def make_jps_forest_corridor(seed, P, N, force_final=True, DC=0.01, n_trees=60):
    """Corridor problem produced by the product's own host pipeline: fq_jps3d_plan_world on the voxelised forest (obstacles
    inflated by inflation_jps = 0.47, faster.yaml:20), vertices <= 1.5 m apart (dist_max_vertexes), first P segments,
    fq_ellipsoid_decomp against the occupied cell centres (the reference decomposes against its occupied cloud)."""
    from . import capi
    prof = UAV
    rng = np.random.default_rng(seed)
    _, centres, radii = make_forest(seed, n_trees=n_trees)
    grid_jps, origin, res = voxelise_forest(centres, radii, inflation=0.47)
    grid, _, _ = voxelise_forest(centres, radii)
    zd, yd, xd = grid.shape
    for _ in range(200):
        s = np.array([rng.uniform(-6, 6), rng.uniform(-6, 6), rng.uniform(0.8, 1.4)])
        t = s + rng.uniform(3.5, 5.0) * np.array([np.cos(a := rng.uniform(-np.pi, np.pi)), np.sin(a), 0.0])
        t[2] = rng.uniform(0.8, 1.4)
        if np.abs(t[:2]).max() > 7.5:
            continue
        path, _ = capi.jps3d_plan_world(grid_jps, origin, res, s, t, True)
        if len(path) >= 2:
            break
    else:
        raise RuntimeError("no path found")
    verts = split_long_segments(path, 1.5)[:P + 1]
    if len(verts) < P + 1:
        raise RuntimeError("path too short for %d polytopes" % P)
    occ = np.argwhere(grid > 0)[:, ::-1]                       # (x, y, z) cells
    obs = (occ + 0.5) * res + origin
    polys = capi.ellipsoid_decomp(verts, obs, prof["bbox"], prof["drone_radius"], prof["z_ground"], cap_rows=8192)
    d0 = verts[1] - verts[0]
    d0 /= np.linalg.norm(d0)
    x0 = np.zeros(9)
    x0[:3] = verts[0]
    x0[3:6] = d0 * rng.uniform(*prof["v0"])
    xf = np.zeros(9)
    xf[:3] = verts[-1]
    return dict(N=N, P=P, x0=x0, xf=xf, lim=np.array(prof["lim"]), polys=polys, force_final=bool(force_final), DC=DC,
                verts=verts, obs=obs, seed=seed, profile="uav", jps_path=path)


# ------------------------------------------------------------------------------------------------------------------
# BASELINE config 4: one replan() = a whole problem and the safe problem that branches off it (faster.cpp:406-430,
# :474-475, :485-499, :521-524).  The safe corridor depends on R, a sample of the whole SOLUTION, so it is built in two
# steps: make_forest_pair_whole -> (solve the whole sweep, read R) -> make_forest_pair_safe.
# ------------------------------------------------------------------------------------------------------------------
def make_forest_pair_whole(seed, N=10, P_whole=3, n_trees=60, query=(5.5, 7.0), DC=0.01):
    """Whole problem of one replan in a random forest: JPS path (product host code) of `query` metres, vertices at most
    1.5 m apart (createMoreVertexes), the first P_whole segments decomposed against the occupied cells.  Keeps the whole
    vertex list and the obstacle cloud for the safe step."""
    from . import capi
    prof = UAV
    rng = np.random.default_rng(seed)
    _, centres, radii = make_forest(seed, n_trees=n_trees)
    grid_jps, origin, res = voxelise_forest(centres, radii, inflation=0.47)
    grid, _, _ = voxelise_forest(centres, radii)
    for _ in range(400):
        s = np.array([rng.uniform(-6, 6), rng.uniform(-6, 6), rng.uniform(0.8, 1.4)])
        ang = rng.uniform(-np.pi, np.pi)
        t = s + rng.uniform(*query) * np.array([np.cos(ang), np.sin(ang), 0.0])
        t[2] = rng.uniform(0.8, 1.4)
        if np.abs(t[:2]).max() > 7.5:
            continue
        path, _ = capi.jps3d_plan_world(grid_jps, origin, res, s, t, True)
        if len(path) < 2:
            continue
        verts_all = split_long_segments(path, 1.5)
        if len(verts_all) >= P_whole + 2:
            break
    else:
        raise RuntimeError("no path found")
    verts = verts_all[:P_whole + 1]
    obs = (np.argwhere(grid > 0)[:, ::-1] + 0.5) * res + origin
    polys = capi.ellipsoid_decomp(verts, obs, prof["bbox"], prof["drone_radius"], prof["z_ground"], cap_rows=8192)
    d0 = verts[1] - verts[0]
    d0 /= np.linalg.norm(d0)
    x0 = np.zeros(9)
    x0[:3] = verts[0]
    x0[3:6] = d0 * rng.uniform(*prof["v0"])
    xf = np.zeros(9)
    xf[:3] = verts[-1]
    return dict(N=N, P=P_whole, x0=x0, xf=xf, lim=np.array(prof["lim"]), polys=polys, force_final=True, DC=DC, verts=verts,
                verts_all=verts_all, obs=obs, seed=seed, profile="uav")


def make_forest_pair_safe(whole, R, N=10, P_safe=4):
    """Safe problem of the replan whose whole problem is `whole`, branching off at the state R (9: pos vel accel):
    JPS_safe = the path ahead of R with its first vertex replaced by R.pos (faster.cpp:485), exactly P_safe segments
    (deleteVertexes, faster.cpp:495, or an extra vertex on the longest segment when the path is short), decomposed
    against the same cloud (no unknown space in the synthetic forest, faster.cpp:499); x0 = R, xf = M = the last vertex
    at rest, final position free (faster.cpp:521-524)."""
    from . import capi
    prof = UAV
    R = np.asarray(R, float)
    va = whole["verts_all"]
    best, bi = np.inf, 0
    for i in range(len(va) - 1):                               # segment of the path closest to R
        ab = va[i + 1] - va[i]
        t = np.clip(((R[:3] - va[i]) @ ab) / max(ab @ ab, 1e-12), 0.0, 1.0)
        d = np.linalg.norm(va[i] + t * ab - R[:3])
        if d < best:
            best, bi = d, i
    path = [R[:3].copy()] + [v for v in va[bi + 1:]]
    if len(path) >= 3 and np.linalg.norm(path[1] - path[0]) < 0.3:
        del path[1]
    path = path[:P_safe + 1]
    while len(path) < P_safe + 1:
        k = int(np.argmax([np.linalg.norm(path[i + 1] - path[i]) for i in range(len(path) - 1)]))
        path.insert(k + 1, 0.5 * (path[k] + path[k + 1]))
    path = np.array(path)
    polys = capi.ellipsoid_decomp(path, whole["obs"], prof["bbox"], prof["drone_radius"], prof["z_ground"], cap_rows=8192)
    xf = np.zeros(9)
    xf[:3] = path[-1]
    return dict(N=N, P=P_safe, x0=R[:9].copy(), xf=xf, lim=whole["lim"].copy(), polys=polys, force_final=False, DC=whole["DC"],
                verts=path, seed=whole["seed"], profile="uav")


def clip_path_to_sphere(path, centre, Ra):
    """The path up to where it first leaves the sphere of radius Ra around `centre`, ending ON the sphere (the reference
    clips its JPS path at Ra before trimming it, faster.cpp:361-393)."""
    out = [np.asarray(path[0], float)]
    for a, b in zip(path[:-1], path[1:]):
        if np.linalg.norm(b - centre) <= Ra:
            out.append(np.asarray(b, float))
            continue
        d = b - a                                      # |a + t d - centre| = Ra, t in [0, 1]
        f = a - centre
        qa, qb, qc = d @ d, 2 * (f @ d), f @ f - Ra * Ra
        t = (-qb + np.sqrt(max(qb * qb - 4 * qa * qc, 0.0))) / (2 * qa) if qa > 0 else 0.0
        out.append(a + np.clip(t, 0.0, 1.0) * d)
        break
    return np.array(out)


def make_forest_pair_mixed(seed, N=10, max_poly_whole=3, max_poly_safe=4, Ra=4.0, r_fraction=0.6, n_trees=60, query=(0.6, 7.0),
                           DC=0.01):
    """One replan's (whole, safe) corridors in a random forest, with polytope counts as Faster::replan produces them: the JPS
    path (product host code) to a goal `query` metres away, clipped at Ra, vertices at most 1.5 m apart (createMoreVertexes),
    then deleteVertexes (utils.cpp:1117-1124: at most max_poly + 1 vertices), one polytope per segment.  So
    P_whole = min(segments within Ra, max_poly_whole): a goal close by gives 1 or 2 polytopes.  The safe corridor starts at an
    estimate of R -- the point r_fraction along the whole path (the device computes the true R from the whole winner) --
    and follows the rest of the path, clipped at Ra around it and trimmed to max_poly_safe segments: near the goal it has
    fewer too.  Nothing is padded.  -> (whole, safe) dicts as make_forest_pair_whole / make_forest_pair_safe."""
    from . import capi
    prof = UAV
    p = forest_pair_paths(seed, N, max_poly_whole, max_poly_safe, Ra, r_fraction, n_trees, query, DC)
    verts, spath, obs = p["path_whole"], p["path_safe"], p["obs"]
    polys_w = capi.ellipsoid_decomp(verts, obs, prof["bbox"], prof["drone_radius"], prof["z_ground"], cap_rows=8192)
    whole = dict(N=N, P=len(polys_w), x0=p["x0"], xf=p["xf_whole"], lim=p["lim"], polys=polys_w, force_final=True, DC=DC, verts=verts,
                 verts_all=p["path_all"], obs=obs, seed=seed, profile="uav")
    polys_s = capi.ellipsoid_decomp(spath, obs, prof["bbox"], prof["drone_radius"], prof["z_ground"], cap_rows=8192)
    safe = dict(N=N, P=len(polys_s), x0=p["R_estimate"], xf=p["xf_safe"], lim=p["lim"].copy(), polys=polys_s, force_final=False, DC=DC,
                verts=spath, seed=seed, profile="uav")
    return whole, safe


def forest_pair_paths(seed, N=10, max_poly_whole=3, max_poly_safe=4, Ra=4.0, r_fraction=0.6, n_trees=60, query=(0.6, 7.0), DC=0.01):
    """The inputs of one replan of make_forest_pair_mixed before any decomposition, for the chain that decomposes on the
    device (fq_replan_pairs_decomp*): the whole and safe paths, already trimmed by deleteVertexes; the occupied cells' centres
    (one cloud serves both sweeps: the synthetic forest has no unknown space); the goal G (the JPS query's end); x0 and lim.
    Vertex 0 of path_safe is the estimate of R that make_forest_pair_mixed cuts the safe corridor around (R_estimate, 9
    doubles); the device replaces it with its own R.  xf_whole / xf_safe put E and M at the paths' last vertices, as
    make_forest_pair_mixed does.  -> dict."""
    prof = UAV
    rng = np.random.default_rng(seed)
    path, _, t, grid, origin, res = _forest_query(rng, seed, n_trees, query)
    path_all = split_long_segments(path, 1.5)
    verts = split_long_segments(clip_path_to_sphere(path, path[0], Ra), 1.5)[:max_poly_whole + 1]
    obs = (np.argwhere(grid > 0)[:, ::-1] + 0.5) * res + origin
    d0 = verts[1] - verts[0]
    d0 /= np.linalg.norm(d0)
    x0 = np.zeros(9)
    x0[:3] = verts[0]
    x0[3:6] = d0 * rng.uniform(*prof["v0"])
    xf = np.zeros(9)
    xf[:3] = verts[-1]
    lim = np.array(prof["lim"])
    # R estimate: r_fraction of the whole path's length; the safe path continues along the full path from there
    seg = np.linalg.norm(np.diff(verts, axis=0), axis=1)
    at = r_fraction * seg.sum()
    k = min(int(np.searchsorted(np.cumsum(seg), at)), len(seg) - 1)
    u = (at - (np.cumsum(seg)[k] - seg[k])) / max(seg[k], 1e-12)
    R = verts[k] + np.clip(u, 0.0, 1.0) * (verts[k + 1] - verts[k])
    i = int(np.argmin([np.linalg.norm(v - verts[k + 1]) for v in path_all]))          # verts[k+1] in the full path
    rest = [R] + [v for v in path_all[i:] if np.linalg.norm(v - R) > 0.3]
    if len(rest) < 2:
        rest = [R, verts[-1] if np.linalg.norm(verts[-1] - R) > 1e-3 else R + 0.5 * d0]
    spath = split_long_segments(clip_path_to_sphere(np.array(rest), R, Ra), 1.5)[:max_poly_safe + 1]
    R9 = np.zeros(9)
    R9[:3] = R
    xfs = np.zeros(9)
    xfs[:3] = spath[-1]
    return dict(N=N, DC=DC, path_whole=np.asarray(verts, float), path_safe=np.asarray(spath, float), path_all=path_all, obs=obs,
                goal=np.asarray(t, float), x0=x0, xf_whole=xf, xf_safe=xfs, lim=lim, R_estimate=R9, seed=seed, profile="uav")


def _forest_query(rng, seed, n_trees, query):
    """The JPS query of forest_pair_paths: a start and a goal `query` metres apart drawn from rng, and the product's JPS path
    between them on the inflated forest.  -> (path, goal, grid, origin, res) with the uninflated grid."""
    from . import capi
    _, centres, radii = make_forest(seed, n_trees=n_trees)
    grid_jps, origin, res = voxelise_forest(centres, radii, inflation=0.47)
    grid, _, _ = voxelise_forest(centres, radii)
    for _ in range(400):
        s = np.array([rng.uniform(-6, 6), rng.uniform(-6, 6), rng.uniform(0.8, 1.4)])
        ang = rng.uniform(-np.pi, np.pi)
        t = s + rng.uniform(*query) * np.array([np.cos(ang), np.sin(ang), 0.0])
        t[2] = rng.uniform(0.8, 1.4)
        if np.abs(t[:2]).max() > 7.5:
            continue
        path, _ = capi.jps3d_plan_world(grid_jps, origin, res, s, t, True)
        if len(path) >= 2 and np.linalg.norm(path[-1] - path[0]) > 0.3:
            return path, s, t, grid, origin, res
    raise RuntimeError("no path found")


def forest_jps(seed, n_trees=60, query=(0.6, 7.0)):
    """The JPS query of forest_pair_paths(seed) before anything is cut from it: the planner's path (cell centres, as
    fq_jps3d_plan_world returns it), its start and its goal.  -> dict(jps, start, goal, seed, x0) with x0 = the start."""
    rng = np.random.default_rng(seed)
    path, s, t, _, _, _ = _forest_query(rng, seed, n_trees, query)
    return dict(jps=path, start=s, goal=np.asarray(t, float), seed=seed, x0=np.concatenate([s, np.zeros(6)]))


def forest_unknown_cloud(p, seed=None, half=3.0, dz=0.6, sensing=(1.6, 4.5), n_trees=60):
    """A seeded unknown cloud for the forest replan `p` (forest_pair_paths), as kdtree_unk_ holds it: the centres of the free
    cells of the local window |x - A.x|, |y - A.y| <= half, |z - A.z| <= dz around A = p["x0"] that A has not seen -- out
    of a sensing range drawn from `sensing` (U[lo, hi], seeded), or shadowed in xy by a trunk between A and the cell.
    With the defaults a corridor holds a few thousand points, and about half the corridors of a batch have a whole
    trajectory that comes within drone_radius of one (need a safe path).  -> [m, 3] float64."""
    rng = np.random.default_rng(p["seed"] + 7919 if seed is None else seed)
    _, centres, radii = make_forest(p["seed"], n_trees=n_trees)
    grid, origin, res = voxelise_forest(centres, radii)
    A = np.asarray(p["x0"][:3], float)
    reach = rng.uniform(*sensing)
    zd, yd, xd = grid.shape
    cx = (np.arange(xd) + 0.5) * res + origin[0]
    cy = (np.arange(yd) + 0.5) * res + origin[1]
    cz = (np.arange(zd) + 0.5) * res + origin[2]
    ix = np.flatnonzero(np.abs(cx - A[0]) <= half)
    iy = np.flatnonzero(np.abs(cy - A[1]) <= half)
    iz = np.flatnonzero(np.abs(cz - A[2]) <= dz)
    Y, X = np.meshgrid(cy[iy], cx[ix], indexing="ij")
    dx, dy = X - A[0], Y - A[1]
    dist = np.hypot(dx, dy)
    unseen = dist > reach
    for c, r in zip(centres, radii):                      # a trunk between A and the cell hides it
        ox, oy = c[0] - A[0], c[1] - A[1]
        t = np.clip((ox * dx + oy * dy) / np.maximum(dist * dist, 1e-12), 0.0, 1.0)
        unseen |= (np.hypot(t * dx - ox, t * dy - oy) <= r) & (t < 1.0) & (np.hypot(ox, oy) < dist)
    free = grid[np.ix_(iz, iy, ix)] == 0
    cells = free & unseen[None]
    kz, ky, kx = np.nonzero(cells)
    return np.ascontiguousarray(np.stack([cx[ix][kx], cy[iy][ky], cz[iz][kz]], axis=1))


# ------------------------------------------------------------------------------------------------------------------
# Feasibility margins (SURVEY.md section 7, "hard parts"): Gurobi decides feasibility with FeasibilityTol 1e-6 on its own
# scaled rows, this library with an absolute row tolerance (default 1e-8).  Candidates whose feasibility depends on
# which of the two is used are FLAGGED (never dropped): a benchmark or a parity claim should say how many there are.
# ------------------------------------------------------------------------------------------------------------------
def margin_flags(solver, N, force_final, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dts, sigmas, eps=1e-5):
    """For a fq_solve_multi workload: (feasible, near) with near[i] = True when candidate i's flag changes if every row
    bound (polytope offsets b and the v/a/j limits) moves by -eps versus +eps, i.e. the candidate lies within eps (m,
    m/s, m/s2, m/s3) of the feasibility boundary.  Three launches on `solver` (a faster_b200.capi.Solver)."""
    f0 = solver.solve_multi(N, force_final, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dts, sigmas)[0]
    out = []
    for s in (-eps, eps):
        A2 = np.ascontiguousarray(Ab).copy()
        A2[:, 3] += s
        out.append(solver.solve_multi(N, force_final, x0, xf, np.ascontiguousarray(lim + s), poly_ofs, face_ofs, A2, cand_ofs,
                                      dts, sigmas)[0])
    near = out[0] != out[1]
    return f0, near


def margin_report(solver, *args, eps_list=(1e-6, 1e-5, 1e-4)):
    """{'within_<eps>': count} for several eps, plus the flags at the nominal tolerance."""
    rep = {}
    f0 = None
    for e in eps_list:
        f0, near = margin_flags(solver, *args, eps=e)
        rep["within_%g" % e] = int(near.sum())
    rep["candidates"] = int(len(f0))
    rep["feasible"] = int(f0.sum())
    return rep
