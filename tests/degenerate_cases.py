"""Degenerate corridors for the dual active-set solver: several rows tight at one point, linearly dependent normals, ties in
the row ranking and in the ratio test.  Every transform takes a corridor of faster_b200.corridor.make_corridor and returns a
changed copy; every transform is deterministic.  Shared by tests/test_degenerate_gpu.py and tests/test_kernel_emu_cpu.py.

Transforms that change nothing (the answer is that of the original corridor):
  * fan: faces through polytope vertices and edges whose normals are positive combinations of the tight faces' normals;
    each contains the polytope.  A fan face can be the most violated row at an infeasible iterate while the faces it
    depends on enter later: the dependent-row branch of the solver;
  * dup / dup_scaled: every face repeated exactly, or scaled by a power of two (A and b, exact);
  * symmetry: one of the 48 signed permutations of the axes applied to the states and the columns of A;
  * vertical_slab: obstacle faces made vertical on the ground profile, plus the zero-width pair z <= h, -z <= -h at the
    height h of every vertex (the optimum without the pair already has z = h).
Degenerate transforms with no known answer (judged by the restatement and by proofs): slab (the zero-width pair on tilted
faces), near_parallel (each face paired with a copy rotated by theta), touching (consecutive polytopes that share only a
slab of given thickness), and states on the boundary (on_boundary: x0 or xf on a face, edge or vertex; at_limit: |v0| or
|a0| at its limit)."""
import itertools

import numpy as np

SIGNED_PERMUTATIONS = [(p, s) for p in itertools.permutations(range(3)) for s in itertools.product((1.0, -1.0), repeat=3)]


def _copy(pb, **kw):
    out = dict(pb, x0=np.array(pb["x0"], float), xf=np.array(pb["xf"], float), lim=np.array(pb["lim"], float),
               polys=[(np.array(A, float), np.array(b, float)) for A, b in pb["polys"]], verts=np.array(pb["verts"], float))
    out.update(kw)
    return out


def vertices(A, b, tol=1e-9):
    """Simple vertices of {x : A x <= b}: [(v, (i, j, k))] for the triples of faces that meet in one point satisfying every
    other face, exactly three faces tight there."""
    out = []
    for ijk in itertools.combinations(range(len(b)), 3):
        M = A[list(ijk)]
        if abs(np.linalg.det(M)) < 1e-6:
            continue
        v = np.linalg.solve(M, b[list(ijk)])
        s = A @ v - b
        if s.max() <= tol and int((np.abs(s) <= tol).sum()) == 3:
            out.append((v, ijk))
    return out


def _seg_dist(x, p1, p2):
    d = p2 - p1
    t = np.clip((x - p1) @ d / (d @ d), 0.0, 1.0)
    return np.linalg.norm(p1 + t * d - x)


def fan(pb, k, n_vert=6, scale=2.0):
    """k faces through each of the n_vert vertices of every polytope nearest to its segment (positive combinations of the 3
    tight normals) and k through one edge at each of them (combinations of 2), b = n.v: the polytopes are unchanged.  The
    fan rows are scaled by `scale` (A and b; a power of two is exact): the row ranking is not normalised by |a|, so a
    violated fan row is picked before the faces it depends on, and those then meet it in the active set."""
    rng = np.random.default_rng(1000 + k)
    out = _copy(pb)
    polys = []
    for p, (A, b) in enumerate(out["polys"]):
        rows, rhs = [A], [b]
        vs = sorted(vertices(A, b), key=lambda vi: _seg_dist(vi[0], out["verts"][p], out["verts"][p + 1]))
        for v, ijk in vs[:n_vert]:
            for faces in (ijk, ijk[:2]):
                w = rng.uniform(0.2, 1.0, (k, len(faces)))
                n = w @ A[list(faces)]
                n /= np.linalg.norm(n, axis=1, keepdims=True)
                rows.append(scale * n)
                rhs.append(scale * (n @ v))
        polys.append((np.vstack(rows), np.concatenate(rhs)))
    out["polys"] = polys
    return out


def dup(pb):
    """Polytope 0 (mod 3): every face next to its copy; 1: a copy of all faces appended; 2: all faces three times."""
    out = _copy(pb)
    polys = []
    for p, (A, b) in enumerate(out["polys"]):
        if p % 3 == 0:
            polys.append((np.repeat(A, 2, axis=0), np.repeat(b, 2)))
        else:
            c = 2 if p % 3 == 1 else 3
            polys.append((np.tile(A, (c, 1)), np.tile(b, c)))
    out["polys"] = polys
    return out


def dup_scaled(pb):
    """A copy of every face multiplied by 2 or 4 (alternating): the same half-space, but a copy that is not a unit row ranks
    above the original and its effective row tolerance is row_tol / c."""
    out = _copy(pb)
    polys = []
    for A, b in out["polys"]:
        c = np.where(np.arange(len(b)) % 2 == 0, 2.0, 4.0)
        polys.append((np.vstack([A, A * c[:, None]]), np.concatenate([b, b * c])))
    out["polys"] = polys
    return out


def symmetry(pb, perm, signs):
    """Axis i of the result is signs[i] * axis perm[i] of the original (states, vertices and the columns of A).  The limits
    apply to every axis alike, so the problem is the same problem."""
    perm, s = list(perm), np.asarray(signs, float)
    out = _copy(pb)
    for key in ("x0", "xf"):
        x = out[key]
        out[key] = np.concatenate([s * x[3 * j:3 * j + 3][perm] for j in range(3)])
    out["verts"] = out["verts"][:, perm] * s
    out["polys"] = [(A[:, perm] * s, b) for A, b in out["polys"]]
    return out


def unpermute_coeffs(co, perm, signs):
    """Coefficients [..., N, 12] (k = 3 * power + axis) of the permuted problem -> those of the original problem."""
    co = np.asarray(co)
    out = np.empty_like(co)
    for i, j in enumerate(perm):
        out[..., j::3] = signs[i] * co[..., i::3]
    return out


def _slab(A, b, h):
    return np.vstack([A, [[0.0, 0.0, 1.0], [0.0, 0.0, -1.0]]]), np.concatenate([b, [h, -h]])


def vertical(pb):
    """Ground-profile corridor (every vertex and both states at one height h, no vertical motion) with every tilted face made
    vertical (z component zeroed, renormalised, the face kept where it crosses z = h) and every nearly horizontal one
    horizontal (kept where it crosses the vertical line through the segment midpoint).  The z axis then decouples from x and
    y, and its optimum is z = h."""
    h = float(pb["verts"][0, 2])
    assert np.all(pb["verts"][:, 2] == h) and pb["x0"][2] == h and not pb["x0"][[5, 8]].any()
    out = _copy(pb)
    polys = []
    for p, (A, b) in enumerate(out["polys"]):
        A, b = A.copy(), b.copy()
        nxy = np.linalg.norm(A[:, :2], axis=1)
        tilt = (nxy > 0.2) & (A[:, 2] != 0)
        b[tilt] = (b[tilt] - A[tilt, 2] * h) / nxy[tilt]
        A[tilt, :2] /= nxy[tilt, None]
        A[tilt, 2] = 0.0
        flat = (nxy <= 0.2) & (nxy > 0)                      # nearly horizontal: horizontal through the point above the midpoint
        mid = 0.5 * (out["verts"][p] + out["verts"][p + 1])
        zc = (b[flat] - A[flat, :2] @ mid[:2]) / A[flat, 2]
        s = np.sign(A[flat, 2])
        A[flat] = 0.0
        A[flat, 2] = s
        b[flat] = s * zc
        polys.append((A, b))
    out["polys"] = polys
    out["slab_h"] = h
    return out


def slab(pb):
    """The zero-width pair z <= h, -z <= -h added to every polytope, h = the height of the (ground-profile) vertices."""
    h = float(pb["verts"][0, 2])
    assert np.all(pb["verts"][:, 2] == h)
    out = _copy(pb)
    out["polys"] = [_slab(A, b, h) for A, b in out["polys"]]
    return out


def vertical_slab(pb):
    return slab(vertical(pb))


def near_parallel(pb, theta):
    """Every face paired with a copy rotated by theta about a line in the face through the foot of the segment midpoint: the
    pair crosses inside the polytope, next to the path.  On one side of the line the copy cuts up to theta times the
    polytope's extent into it; within about row_tol / theta of the line both rows hold within the row tolerance."""
    out = _copy(pb)
    polys = []
    e = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    for p, (A, b) in enumerate(out["polys"]):
        mid = 0.5 * (out["verts"][p] + out["verts"][p + 1])
        rows, rhs = [], []
        for n, c in zip(A, b):
            foot = mid + (c - n @ mid) * n
            v = np.cross(n, e)
            if np.linalg.norm(v) < 0.1:
                v = np.cross(n, [1.0, 0.0, 0.0])
            v /= np.linalg.norm(v)
            n2 = np.cos(theta) * n - np.sin(theta) * v
            rows += [n, n2]
            rhs += [c, n2 @ foot]
        polys.append((np.array(rows), np.array(rhs)))
    out["polys"] = polys
    out["near_parallel"] = theta
    return out


def touching(pb, thickness):
    """Consecutive polytopes overlap only in the slab d.v <= d.x <= d.v + thickness at their shared vertex v (d = the
    direction of the earlier segment)."""
    out = _copy(pb)
    V = out["verts"]
    polys = [list(ab) for ab in out["polys"]]
    for p in range(len(polys) - 1):
        d = V[p + 1] - V[p]
        d /= np.linalg.norm(d)
        c = float(d @ V[p + 1])
        A, b = polys[p]
        polys[p] = [np.vstack([A, d]), np.append(b, c + thickness)]
        A, b = polys[p + 1]
        polys[p + 1] = [np.vstack([A, -d]), np.append(b, -c)]
    out["polys"] = [(A, b) for A, b in polys]
    return out


def on_boundary(pb, which, n_faces):
    """x0 (which = "x0") or xf ("xf") exactly on n_faces = 1, 2 or 3 faces (a face, an edge, a vertex) of every polytope that
    holds it: b = A.x.  The faces are those the motion there points away from (x0: the start velocity, or the first segment
    at rest; xf: the arrival direction), so that candidates stay feasible."""
    out = _copy(pb)
    x = out[which][:3]
    if which == "x0":
        d = -(out["x0"][3:6] if np.linalg.norm(out["x0"][3:6]) > 0 else out["verts"][1] - out["verts"][0])
    else:
        d = out["verts"][-1] - out["verts"][-2]
    for A, b in out["polys"]:
        if (A @ x - b).max() <= 0:
            picked = []
            for f in np.argsort(-(A @ d)):                    # most "behind the motion" first, independent normals only
                if np.linalg.matrix_rank(A[picked + [f]]) == len(picked) + 1:
                    picked.append(int(f))
                if len(picked) == n_faces:
                    break
            b[picked] = A[picked] @ x
    return out


def at_limit(pb, kind):
    """|v0| (kind "v") or |a0| ("a") exactly at its limit on the axis where it is largest: the limit is lowered to it."""
    out = _copy(pb)
    j = 0 if kind == "v" else 1
    comp = np.abs(out["x0"][3 + 3 * j:6 + 3 * j])
    out["lim"][j] = comp.max()
    assert out["lim"][j] > 0
    return out


def specialised_fits(N, ff, polys, warps=4):
    """Whether a batch of these polytopes fits the size-specialised kernel (fq_kernels_t.cuh's smem_bytes_t and its 227 KB
    limit, the 11-bit face index), so that a launch does not fall back to the generic kernel."""
    F = sum(len(b) for _, b in polys)
    nz = N - (3 if ff else 2)
    nw, ny = 3 * nz, 6 * N + 1
    per_warp = 8 * (nw * (nw | 1) + nw * (nw + 1) // 2 + 3 * (ny | 1) + 3 * nw + 2) + ((N * max(len(b) for _, b in polys) * 2 + 15) & ~15)
    smem = 8 * (warps * 4 * F + ny * (nz | 1) + ny) + warps * per_warp + (40 * warps + warps * 32) * 4 + 16
    return F <= 2047 and smem <= 227 * 1024
