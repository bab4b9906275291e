"""Corridors at the solver's size limits, and the shared-memory formulas that place those limits.

Every kernel keeps a problem's polytope rows in shared memory, so the faces a problem may have depend on N and on how the
faces are split among its polytopes.  `limit` mirrors the host-side size checks of the three kernels:
  * "spec": the size-specialised kernel, fqt::smem_bytes_t (faster_b200/csrc/fq_kernels_t.cuh) -- one row copy per warp plus a
    per-warp item list of N x (faces of the largest polytope) 16-bit entries.  Beyond it fq_launch_solve falls back to:
  * "generic": the size-generic kernel, fq_solve_smem_bytes (faster_b200/csrc/fq_kernels.cu) -- one row copy per CTA, no item
    list.  Beyond it the C ABI refuses with FQ_E_ARG;
  * "bnb": the branch-and-bound level kernel, fqb::launch_level (faster_b200/csrc/fq_bnb.cuh) -- smem_bytes_t with one row copy.
    Beyond it (or beyond 2047 faces, the 11-bit face field of an item) fq_gen_new_traj_exact reports exact = 0.
The tests do not trust these numbers blindly: they check with the profiler which kernel ran on each side of a limit.

The builders add faces to a corridor (tests' corridor dicts, faster_b200/corridor.py):
  * pad_loose: faces that provably never bind, so the answer must not change;
  * tangent_faces: faces tangent to a capsule around each path segment, which do bind."""
import numpy as np
from scipy.optimize import linprog

SMEM_MAX = 227 * 1024           # dynamic shared memory one block may opt into on an H100
W = 4                           # warps per CTA (FQ_WARPS_PER_CTA)
MAX_N = 16                      # FQ_MAX_N
MAX_POLY = 32                   # FQ_MAX_POLY
ITEM_FACE_CAP = 2047            # largest staged row index an item's 11-bit face field can hold, plus one


def _dims(N, ff):
    ne = 3 if ff else 2
    nz = N - ne
    nw = 3 * nz
    NY = 6 * N + 1
    return ne, nz, nw, NY


def smem_spec(N, ff, max_faces, max_poly_faces, copies=W):
    """fqt::smem_bytes_t<N, ff>(max_faces, item_cap = N * max_poly_faces, copies)."""
    ne, nz, nw, NY = _dims(N, ff)
    NYP, LD, TZLD = NY | 1, nw | 1, nz | 1
    rsz = nw * (nw + 1) // 2
    per_warp_doubles = nw * LD + rsz + 3 * NYP + 3 * nw + 2
    item_cap = N * max_poly_faces
    per_warp = per_warp_doubles * 8 + ((item_cap * 2 + 15) & ~15)
    return 8 * (copies * 4 * max_faces + NY * TZLD + NY) + W * per_warp + (40 * copies + W * 32) * 4 + 16


def smem_generic(N, ff, max_faces):
    """fq_solve_smem_bytes: the size-generic kernel."""
    ne, nz, nw, NY = _dims(N, ff)
    nzp, nwp, ld = max(nz, 1), max(nw, 1), (3 * nz) | 1
    per_warp_doubles = 2 * nwp * ld + 2 * 3 * NY + 7 * nwp + 24
    per_warp_ints = 2 * (MAX_N + 2) + 3 * MAX_N
    doubles = 4 * max_faces + NY * nzp + NY * (3 + ne) + W * per_warp_doubles
    return doubles * 8 + (36 + W * per_warp_ints) * 4


def split_counts(n_faces, split, base):
    """Faces per polytope of an n_faces corridor.  split = "even": as equal as possible (the first polytopes take the
    remainder); "dominant": every polytope but polytope `DOMINANT` keeps its `base` count, that one takes the rest."""
    P = len(base)
    if split == "even":
        return [n_faces // P + (1 if p < n_faces % P else 0) for p in range(P)]
    assert split == "dominant"
    out = list(base)
    out[DOMINANT] = n_faces - (sum(base) - base[DOMINANT])
    return out


DOMINANT = 1                    # the middle polytope of a 3-polytope corridor: segments on both sides of it use it


def fits(kind, N, ff, counts):
    mf, mp = sum(counts), max(counts)
    if kind == "spec":
        return mf <= ITEM_FACE_CAP and smem_spec(N, ff, mf, mp) <= SMEM_MAX
    if kind == "generic":
        return smem_generic(N, ff, mf) <= SMEM_MAX
    assert kind == "bnb"
    return mf <= ITEM_FACE_CAP and smem_spec(N, ff, mf, mp, copies=1) <= SMEM_MAX


def limit(kind, N, ff, split, base):
    """Largest number of faces that still fits kernel `kind` ("spec", "generic", "bnb") for a corridor whose polytopes
    start with `base` faces each and grow by `split` (see split_counts)."""
    lo, hi = sum(base), 1 << 16
    assert fits(kind, N, ff, split_counts(lo, split, base))
    while hi - lo > 1:                                  # the footprint grows with the face count
        mid = (lo + hi) // 2
        if fits(kind, N, ff, split_counts(mid, split, base)):
            lo = mid
        else:
            hi = mid
    return lo


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def support(A, b, dirs):
    """max of d . x over the polytope {A x <= b} for each row d of dirs: the polytope's vertices (the LP optimum is attained
    at one) from every triple of faces, checked against one linprog per direction on a sample."""
    A, b = np.asarray(A, float), np.asarray(b, float)
    verts = []
    F = len(b)
    for i in range(F):
        for j in range(i + 1, F):
            for k in range(j + 1, F):
                M = A[[i, j, k]]
                if abs(np.linalg.det(M)) < 1e-9:
                    continue
                x = np.linalg.solve(M, b[[i, j, k]])
                if (A @ x - b).max() <= 1e-9:
                    verts.append(x)
    V = np.array(verts)
    h = (dirs @ V.T).max(axis=1)
    for d, hv in zip(dirs[:3], h[:3]):
        r = linprog(-d, A_ub=A, b_ub=b, bounds=[(None, None)] * 3, method="highs")
        assert r.status == 0 and abs(-r.fun - hv) <= 1e-7 * max(1.0, abs(hv)), (r.status, -r.fun, hv)
    return h


def pad_loose(pb, n_faces, binding_last=True, seed=0, split="even"):
    """A copy of corridor pb with random unit-normal faces added until it has exactly n_faces rows.  Each added face is at
    least 1e-3 beyond the polytope (its maximum over the polytope is at least 1e-3 below its b), so no point of the
    polytope comes near it and the answer cannot change.  binding_last: the original faces go last in each polytope, so the
    rows that bind have the highest staged indices."""
    rng = np.random.default_rng(seed)
    base = [len(b) for _, b in pb["polys"]]
    counts = split_counts(n_faces, split, base)
    polys = []
    for (A, b), n in zip(pb["polys"], counts):
        k = n - len(b)
        assert k >= 0
        nrm = _unit(rng, k)
        bb = support(A, b, nrm) + rng.uniform(1e-3, 0.5, k) if k else np.zeros(0)
        if binding_last:
            polys.append((np.vstack([nrm, A]), np.concatenate([bb, b])))
        else:
            polys.append((np.vstack([A, nrm]), np.concatenate([b, bb])))
    out = dict(pb, polys=polys)
    assert sum(len(b) for _, b in polys) == n_faces
    return out


def tangent_faces(pb, counts, radius=0.35, seed=0):
    """A copy of corridor pb where polytope p gets counts[p] - (its faces) extra faces, each tangent to the capsule of
    `radius` around the polytope's path segment: n . x <= max(n . v0, n . v1) + radius.  They cut into the polytope and
    bind; the path (and x0, xf on it) stays inside, so easy time allocations stay feasible.  The original faces go last."""
    rng = np.random.default_rng(seed)
    verts = pb["verts"]
    polys = []
    for p, ((A, b), n) in enumerate(zip(pb["polys"], counts)):
        k = n - len(b)
        assert k >= 0
        nrm = _unit(rng, k)
        v0, v1 = verts[p], verts[p + 1]
        bb = np.maximum(nrm @ v0, nrm @ v1) + radius
        polys.append((np.vstack([nrm, A]), np.concatenate([bb, b])))
    return dict(pb, polys=polys)


def with_faces(pb, n_faces, split, seed=0, radius=0.35):
    """tangent_faces corridor with exactly n_faces rows split as split_counts does."""
    return tangent_faces(pb, split_counts(n_faces, split, [len(b) for _, b in pb["polys"]]), radius, seed)


def duplicate_polytopes(pb, copies):
    """Every polytope repeated `copies` times in a row: polytope p becomes p * copies .. p * copies + copies - 1."""
    polys = [pl for pl in pb["polys"] for _ in range(copies)]
    return dict(pb, polys=polys, P=len(polys))
