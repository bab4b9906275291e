"""Inputs of the convex decomposition shared by the host golden (tests/golden/decomp_host.npz, recorded by
tools/make_decomp_golden.py) and the tests that compare the device kernel with the host: forest corridors of
corridor.forest_pair_paths (whole and safe paths against the map's occupied cells) and random clouds, plus the edge
inputs of tests/test_decomp_cpu.py.  Each case is (name, path [n,3], obs [m,3], inflate)."""
import numpy as np

from faster_b200 import corridor as cr

BBOX = (2.0, 2.0, 1.0)
Z_GROUND = 0.0


def forest_cases(seeds=range(16)):
    """Two cases per seed: the whole path and the safe path (vertex 0 = the estimate of R)."""
    out = []
    for s in seeds:
        p = cr.forest_pair_paths(9000 + s)
        out.append(("forest%d_whole" % s, p["path_whole"], p["obs"], 0.42))
        out.append(("forest%d_safe" % s, p["path_safe"], p["obs"], 0.42))
    return out


def random_cases(seed=9, n=24):
    """Random 1-3 segment paths in uniform and clustered clouds of up to 600 points."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        npts = int(rng.integers(2, 5))
        path = np.cumsum(rng.uniform(-1.5, 1.5, (npts, 3)) * [1, 1, 0.3], axis=0) + [0, 0, 1.0]
        if min(np.linalg.norm(np.diff(path, axis=0), axis=1)) < 0.2:
            continue
        if len(out) % 2:
            obs = rng.uniform(-4, 4, (int(rng.integers(0, 600)), 3)) * [1, 1, 0.5] + [0, 0, 1.0]
        else:
            mid = path.mean(axis=0)
            obs = mid + rng.normal(size=(int(rng.integers(1, 400)), 3)) * rng.uniform(0.5, 2.5)
        out.append(("random%d" % len(out), path, obs, float(rng.choice([0.0, 0.2, 0.42]))))
    return out


def edge_cases():
    """No obstacles; a vertical segment; points exactly on bounding-box faces; duplicated points; a point on the axis."""
    return [
        ("empty", np.array([[0.0, 0.0, 1.0], [1.2, 0.3, 1.1]]), np.zeros((0, 3)), 0.42),
        ("vertical", np.array([[0.0, 0.0, 0.5], [0.0, 0.0, 1.6]]),
         np.array([[1.0, 0.2, 1.0], [-0.8, -0.9, 0.7], [2.0, 0.0, 1.0], [0.3, 1.1, 1.4], [5.0, 5.0, 5.0]]), 0.2),
        ("on_faces", np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 1.0]]),
         np.array([[2.5, 0.0, 1.0], [-1.5, 0.0, 1.0], [0.5, 2.0, 1.0], [0.5, -2.0, 1.0], [0.5, 0.0, 2.0]]), 0.0),
        ("duplicates", np.array([[0.0, 0.0, 1.0], [1.0, 1.0, 1.2]]), np.array([[0.4, 1.3, 1.0]] * 3 + [[1.2, -0.4, 1.1]] * 2), 0.1),
    ]


def all_cases():
    return forest_cases() + random_cases() + edge_cases()
