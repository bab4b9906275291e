"""The batch JPS rules (fq_jps_batch, include/faster_b200.h) restated over the host entries they are defined by:
capi.jps3d_plan_world (the search and its post-processing), capi.jps_in and capi.jps3d_nodes (the nodes the search
creates, which max_nodes bounds).  A plain module (no pytest).

For planner j: A = x0[j][:3] and G = goal[j], z raised to 0 for the search; ra = min(|G - P| - 0.001, Ra) with P = pos[j]
or A, the norm in Eigen's order sqrt((dx^2 + dy^2) + dz^2) (np.linalg.norm may sum in another order); the statuses and
JPS_in rows as the header states them; in_ofs the exclusive scan of the row counts."""
import math

import numpy as np

from faster_b200 import capi

OK, NO_PATH, NODES, LONG, INPUT = capi.JPS_OK, capi.JPS_NO_PATH, capi.JPS_NODES, capi.JPS_LONG, capi.JPS_INPUT
NAN_ROW = np.full((1, 3), np.nan)


def eigen_norm(v):
    """Eigen's 3-vector norm: sqrt((x^2 + y^2) + z^2) in double."""
    x, y, z = (float(c) for c in v)
    return math.sqrt((x * x + y * y) + z * z)


def ra_of(A, G, P, Ra):
    d = eigen_norm(np.asarray(G, np.float64) - np.asarray(P, np.float64)) - 0.001
    return Ra if Ra < d else d                       # std::min(d, Ra)


def _round_away(x):
    """std::round: halves away from zero."""
    a = abs(x)
    f = math.floor(a)
    r = f + 1 if a - f >= 0.5 else f
    return int(math.copysign(r, x)) if r else 0


def to_int(p, origin, res):
    """map_util.h's floatToInt: round((p - origin) / res - 0.5)."""
    return np.array([_round_away((float(p[i]) - float(origin[i])) / float(res) - 0.5) for i in range(3)], np.int32)


def _free(grid, c):
    zd, yd, xd = grid.shape
    return 0 <= c[0] < xd and 0 <= c[1] < yd and 0 <= c[2] < zd and grid[c[2], c[1], c[0]] == 0


def plan_one(grid, origin, res, A, G, P, Ra, dist_max, use_jps, max_nodes, max_in):
    """-> (status, JPS_in rows) of one planner, following the header's rules."""
    A, G, P = (np.asarray(v, np.float64) for v in (A, G, P))
    As, Gs = A.copy(), G.copy()
    As[2], Gs[2] = max(As[2], 0.0), max(Gs[2], 0.0)
    ra = ra_of(A, G, P, Ra)
    s, g = to_int(As, origin, res), to_int(Gs, origin, res)
    path = np.zeros((0, 3))
    if _free(grid, s) and _free(grid, g):
        if capi.jps3d_nodes(grid, s, g, use_jps) > max_nodes:
            return NODES, NAN_ROW
        path, _ = capi.jps3d_plan_world(grid, origin, res, As, Gs, use_jps)
    jin = capi.jps_in(path if len(path) else A[None], A, G, ra, dist_max)
    if len(jin) > max_in:
        return LONG, NAN_ROW
    return (OK if len(path) else NO_PATH), jin


def batch(grids, x0, goal, grid_index=None, pos=None, Ra=4.0, dist_max=1.5, use_jps=True, max_nodes=capi.JPS_MAX_NODES, max_in=512,
          k_end=None):
    """The batch: grids a list of (grid [zd, yd, xd] int8, origin, res).  -> dict(in_ofs, in, status, k_end) as jps_batch."""
    goal = np.asarray(goal, np.float64).reshape(-1, 3)
    n = len(goal)
    x0 = np.asarray(x0, np.float64).reshape(n, -1)
    status, rows = np.zeros(n, np.int32), []
    for j in range(n):
        gi = 0 if grid_index is None else int(grid_index[j])
        A, G = x0[j, :3], goal[j]
        P = A if pos is None else np.asarray(pos[j], np.float64)
        if not (0 <= gi < len(grids)) or not (np.isfinite(A).all() and np.isfinite(G).all() and np.isfinite(P).all()):
            status[j], r = INPUT, NAN_ROW
        else:
            grid, origin, res = grids[gi]
            status[j], r = plan_one(grid, origin, res, A, G, P, Ra, dist_max, use_jps, max_nodes, max_in)
        rows.append(np.asarray(r, np.float64).reshape(-1, 3))
    in_ofs = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    ke = None if k_end is None else np.where(status == OK, np.asarray(k_end, np.int32), -1).astype(np.int32)
    return dict(in_ofs=in_ofs, status=status, k_end=ke, **{"in": np.ascontiguousarray(np.vstack(rows))})


def assert_equal(got, want, what=""):
    """Byte equality of two batch results (NaN rows compare by their bits)."""
    for k in ("in_ofs", "status"):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), (what, k, got[k], want[k])
    n = int(want["in_ofs"][-1])
    g = np.asarray(got["in"], np.float64).reshape(-1, 3)[:n]
    assert g.tobytes() == np.asarray(want["in"], np.float64).reshape(-1, 3)[:n].tobytes(), (what, "in")
    if want.get("k_end") is not None:
        assert np.asarray(got["k_end"]).tobytes() == want["k_end"].tobytes(), (what, "k_end")
