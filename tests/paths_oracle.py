"""Restatement of the reference's JPS_in and safe-path crop, written from its source lines, for tests/test_map_paths_cpu.py:
solveJPS3D's end points (jps_manager.cpp:143-144, :172-186), the clip at Ra and createMoreVertexes (faster.cpp:80-97,
:373-384), getFirstCollisionJPS with UNKNOWN_MAP and RETURN_INTERSECTION (faster.cpp:767-921), getIntersectionWithSphere,
getFirstIntersectionWithSphere and reduceJPSbyDistance (utils.cpp:690-866) and deleteVertexes (utils.cpp:1117-1124).

Where the reference computes in float, so does this file (numpy float32 scalars, each operation rounded to float); Python
floats are its doubles.  `hits` counts the branches taken, so that a test can show it reached the case it is about."""
import math

import numpy as np

f32 = np.float32
hits = {}


def _hit(k):
    hits[k] = hits.get(k, 0) + 1


def norm(a, b):
    """Eigen's (a - b).norm() for 3-vectors: sqrt((dx^2 + dy^2) + dz^2)."""
    d = [a[k] - b[k] for k in range(3)]
    return math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def _quad(x1, x2, x3, r):
    """utils.cpp:732-736 (and :754-758) with float x1.., x2.., x3..: -> (t, discrim)."""
    d = [x2[k] - x1[k] for k in range(3)]
    a = f32((float(d[0]) ** 2 + float(d[1]) ** 2) + float(d[2]) ** 2)        # pow(float, 2): double, assigned to float
    b = f32(2) * ((d[0] * (x1[0] - x3[0]) + d[1] * (x1[1] - x3[1])) + d[2] * (x1[2] - x3[2]))
    s = x3[0] * x3[0] + x3[1] * x3[1] + x3[2] * x3[2] + x1[0] * x1[0] + x1[1] * x1[1] + x1[2] * x1[2]
    m = f32(2) * ((x3[0] * x1[0] + x3[1] * x1[1]) + x3[2] * x1[2])
    c = f32(float(s - m) - r * r)                                            # `- r * r` is a double term
    disc = b * b - f32(4) * a * c
    with np.errstate(all="ignore"):
        t = (-b + np.sqrt(disc)) / (f32(2) * a)                               # the float sqrt
    return t, disc


def intersection_with_sphere(A, B, r, center):
    """getIntersectionWithSphere (utils.cpp:713-776)."""
    x1, x2, x3 = ([f32(v[k]) for k in range(3)] for v in (A, B, center))
    t, disc = _quad(x1, x2, x3, r)
    if disc <= 0:
        _hit("discriminant_fallback")
        x1, x2 = x3, x1
        t, _ = _quad(x1, x2, x3, r)
    with np.errstate(all="ignore"):
        return [float(x1[k] + (x2[k] - x1[k]) * t) for k in range(3)]


def first_intersection_with_sphere(path, r, center):
    """getFirstIntersectionWithSphere (utils.cpp:782-866) -> (intersection, last_index_inside, no_points_outside)."""
    index = next((i for i, p in enumerate(path) if norm(p, center) > r), -1)
    if index == -1:
        return intersection_with_sphere(center, path[-1], r, center), len(path) - 1, True
    if index == 0:
        _hit("first_outside")
        return list(path[0]), 1, False
    return intersection_with_sphere(path[index - 1], path[index], r, center), index - 1, False


def reduce_by_distance(path, d):
    """reduceJPSbyDistance (utils.cpp:690-710), in place."""
    so_far = 0.0
    for ii in range(len(path) - 1, 0, -1):
        v = [path[ii][k] - path[ii - 1][k] for k in range(3)]
        sq = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
        nv = math.sqrt(sq)
        so_far = so_far + nv
        if so_far > d:
            want = so_far - d
            if ii < len(path) - 1:
                _hit("reduce_several_segments")
            del path[ii:]
            u = [x / nv for x in v] if sq > 0 else v
            path.append([path[-1][k] + u[k] * want for k in range(3)])
            return


def delete_vertexes(path, max_value):
    return path[:max_value + 1]


def nearest_d2(q, unk):
    """FLANN's exact float L2 minimum ((0 + dx^2) + dy^2) + dz^2 over the cloud -> float32, or None for an empty cloud."""
    if len(unk) == 0:
        return None
    u = np.asarray(unk, np.float64).astype(np.float32)
    d = u - np.asarray(q, np.float32)
    d2 = ((f32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    return d2.min()


def first_collision(jps_in, unk, drone_radius, max_steps=4096):
    """getFirstCollisionJPS(JPS_in, UNKNOWN_MAP, RETURN_INTERSECTION) (faster.cpp:767-921) -> (path, crossed), or (None,
    None) after max_steps steps."""
    original = [list(map(float, v)) for v in jps_in]
    path = [list(v) for v in original]
    for iteration in range(max_steps):
        q = [f32(v) for v in path[0]]                                        # eigenPoint2pclPoint
        d2 = nearest_d2(q, unk)
        if d2 is None:
            _hit("empty_unknown")
            return original, False
        r = float(np.sqrt(f32(d2)))
        if r < drone_radius:
            if iteration == 0:
                _hit("collision_at_start")
                o = original[0]
                return [o, [o[0] + 0.01, o[1], o[2]]], True
            _hit("collision")
            kept = len(original) - len(path) + 1
            out = original[:kept] + [path[0]]
            reduce_by_distance(out, drone_radius)
            return out, True
        inters, last_id, no_out = first_intersection_with_sphere(path, r, path[0])
        if no_out:
            _hit("no_point_outside")
            return original, False
        path = [inters] + path[last_id + 1:]
    return None, None


def paths(jps_ins, unks, drone_radius, max_poly_whole, max_poly_safe):
    """What fq_paths_cloud returns: poly_ofs_* (int32), path_* (float64 rows), status (int32), crossed (uint8)."""
    out = {k: [] for k in ("path_whole", "path_safe", "status", "crossed")}
    ofs_w, ofs_s = [0], [0]
    for jin, unk in zip(jps_ins, unks):
        safe, crossed = first_collision(jin, unk, drone_radius)
        if safe is None:
            whole, safe, st, crossed = [[math.nan] * 3], [[math.nan] * 3], 2, False
        else:
            whole, st = delete_vertexes([list(map(float, v)) for v in jin], max_poly_whole), 0
            safe = delete_vertexes(safe, max_poly_safe)
        ofs_w.append(ofs_w[-1] + len(whole) - 1)
        ofs_s.append(ofs_s[-1] + len(safe) - 1)
        out["path_whole"] += whole
        out["path_safe"] += safe
        out["status"].append(st)
        out["crossed"].append(int(crossed))
    return dict(poly_ofs_whole=np.asarray(ofs_w, np.int32), poly_ofs_safe=np.asarray(ofs_s, np.int32),
                path_whole=np.asarray(out["path_whole"], np.float64).reshape(-1, 3),
                path_safe=np.asarray(out["path_safe"], np.float64).reshape(-1, 3),
                status=np.asarray(out["status"], np.int32), crossed=np.asarray(out["crossed"], np.uint8))


def create_more_vertexes(path, d):
    """Faster::createMoreVertexes (faster.cpp:80-97)."""
    path = [list(v) for v in path]
    j = 0
    while j < len(path) - 1:
        dist = norm(path[j + 1], path[j])
        add = math.floor(dist / d)
        v = [path[j + 1][k] - path[j][k] for k in range(3)]
        sq = (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]
        v = [x / math.sqrt(sq) for x in v] if sq > 0 else v
        if dist > d:
            for _ in range(add):
                path.insert(j + 1, [path[j][k] + v[k] * d for k in range(3)])
                j += 1
        j += 1
    return path


def jps_in(jps, start, goal, ra, dist_max):
    """faster.cpp:361-384 from a planner path: solveJPS3D's ends, the clip at ra, createMoreVertexes."""
    s = [float(start[0]), float(start[1]), max(float(start[2]), 0.0)]
    g = [float(goal[0]), float(goal[1]), max(float(goal[2]), 0.0)]
    path = [list(map(float, v)) for v in jps]
    if len(path) > 1:
        path[0], path[-1] = s, g
    else:
        _hit("one_point_path")
        path = [s, g]
    E, li, no_out = first_intersection_with_sphere(path, ra, list(path[0]))
    out = path[:li + 1]
    if not no_out:
        out.append(E)
    else:
        _hit("inside_ra")
    return np.asarray(create_more_vertexes(out, dist_max), np.float64).reshape(-1, 3)
