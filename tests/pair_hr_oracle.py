"""TEST INFRASTRUCTURE ONLY -- findIndexH / findIndexR (faster/src/faster.cpp:173-251) restated in numpy, in the arithmetic
fq_replan_pairs_hr* specifies: float32 for the kd-tree query (pcl::PointXYZ holds floats, FLANN's L2 sums them in float), float64
for the braking test.  Plus the chained replan with H and R on the CPU: the host decomposition (fq_ellipsoid_decomp) and the
CPU chain of oracle/pair_oracle.py, corridor by corridor."""
import numpy as np

from faster_b200 import capi


def find_index_h(X, unk, drone_radius, delta_H):
    """X: fillX's samples (n x 12, fq_fill_x), unk: the unknown cloud (m x 3).  -> (needToComputeSafePath, indexH)."""
    n = len(X)
    P = np.asarray(unk, np.float64).reshape(-1, 3).astype(np.float32)      # the cloud's pcl::PointXYZ
    if len(P):
        for i in range(0, n, 10):                                            # :228 every 10th sample
            q = X[i, :3].astype(np.float32)                                  # :231-232 searchPoint(tmp(0), tmp(1), tmp(2))
            d = P - q
            d2 = ((np.float32(0) + d[:, 0] * d[:, 0]) + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]   # FLANN L2, float
            if float(np.sqrt(d2.min())) < drone_radius:                      # :236 sqrt(float) < par_.drone_radius
                return True, int(delta_H * i)                                # :238-241
    return False, n - 1                                                      # :226 X_temp_.size() - 1


def find_index_r(X, index_h, delta_a, a_max):
    """-> indexR: the first sample 0 .. indexH whose xy braking distance exceeds its distance to H (:173-216)."""
    H = X[index_h, :2]                                                       # :178 posHk
    den = 2 * delta_a * a_max                                                # :190 (2 * delta_a) * a_max
    for i in range(index_h + 1):                                             # :181
        v, p = X[i, 3:5], X[i, :2]                                           # :184, :187
        d = H - p
        b = np.sign(v * d) * (v * v) / den                                   # :189-190 sign(v (H - p)) v^2 / den
        if np.any(b > np.abs(d)):                                            # :195-196
            return i                                                         # :199
    return index_h                                                           # :180


def hr_of(coeffs, dt, N, DC, unk, a_max, drone_radius=0.42, delta_a=0.5, delta_H=1.0):
    """H and R of one whole winner.  -> dict(need_safe, index_H, k_safe, n, R (9 doubles, NaN without a safe path))."""
    X = capi.fill_x(N, np.asarray(coeffs, np.float64).reshape(-1), dt, DC)
    need, ih = find_index_h(X, unk, drone_radius, delta_H)
    n = len(X)
    if not need:
        return dict(need_safe=0, index_H=ih, k_safe=n - 1, n=n, R=np.full(9, np.nan))
    k = find_index_r(X, ih, delta_a, a_max)
    return dict(need_safe=1, index_H=ih, k_safe=k, n=n, R=X[k, :9].copy())


def host_corridor(path, obs, goal, N, x0, lim, bbox=(2.0, 2.0, 1.0), inflate=0.42, z_ground=0.0):
    """The host decomposition of one path (fq_ellipsoid_decomp) and its final state: the goal when the last polytope
    contains it (LinearConstraint::inside), else the last vertex.  -> problem dict of make_pair_workload."""
    polys = capi.ellipsoid_decomp(path, obs, bbox, inflate, z_ground, cap_rows=8192)
    A, b = polys[-1]
    xf = np.zeros(9)
    xf[:3] = goal if not np.any(A @ goal - b > 0) else path[-1]
    return dict(N=N, x0=np.asarray(x0, float), xf=xf, lim=np.asarray(lim, float), polys=polys)


def replan_pair_hr(p, factors, all_limit=0, drone_radius=0.42, delta_a=0.5, delta_H=1.0, threads=4, dt_base_whole=None,
                   dt_base_safe=None):
    """One forest replan (corridor.forest_pair_paths dict with "unk") through the CPU chain with H and R: the whole corridor
    from the host decomposition, the CPU whole sweep, H and R from its winner, then -- when a safe path is needed -- the safe
    corridor cut around R and the CPU safe sweep from R.  dt_base_* (optional): the time-allocation bases to use, as in
    pair_oracle.replan_pairs.  -> dict of the fq_pair_result fields plus need_safe, index_H."""
    import pair_assign_oracle as pao
    from oracle import pair_oracle
    N, DC = p["N"], p["DC"]
    whole = host_corridor(p["path_whole"], p["obs"], p["goal"], N, p["x0"], p["lim"])
    safe = host_corridor(p["path_safe"], p["obs"], p["goal"], N, p["R_estimate"], p["lim"])   # replaced below when needed
    w = capi.make_pair_workload([whole], [safe], factors, np.zeros((0, N)), factors, np.zeros((0, N)), DC=DC, r_fraction=0.0)
    db = dict(dt_base_whole=None if dt_base_whole is None else [dt_base_whole],
              dt_base_safe=None if dt_base_safe is None else [dt_base_safe])
    r = pair_oracle.replan_pairs(pao.with_own_lists(w, all_limit), threads=threads, dt_base_whole=db["dt_base_whole"])
    out = {k: r[k][0] for k in ("whole_dt_index", "whole_sigma_index", "whole_cost", "whole_dt", "whole_dt_base", "n_samples_whole")}
    if out["whole_dt_index"] < 0:
        out.update(need_safe=0, index_H=-1, k_safe=-1, R=np.full(9, np.nan), safe_dt_index=-1, safe_sigma_index=-1,
                   safe_cost=np.inf, safe_dt=np.nan)
        return out
    h = hr_of(r["coeffs_whole"][0], out["whole_dt"], N, DC, p["unk"], p["lim"][1], drone_radius, delta_a, delta_H)
    out.update(need_safe=h["need_safe"], index_H=h["index_H"], k_safe=h["k_safe"], R=h["R"])
    if not h["need_safe"]:
        out.update(safe_dt_index=-1, safe_sigma_index=-1, safe_cost=np.inf, safe_dt=np.nan)
        return out
    sp = np.asarray(p["path_safe"], float).copy()
    sp[0] = h["R"][:3]                                                       # faster.cpp:485 JPS_safe[0] = R.pos
    safe = host_corridor(sp, p["obs"], p["goal"], N, h["R"], p["lim"])
    w = capi.make_pair_workload([whole], [safe], factors, np.zeros((0, N)), factors, np.zeros((0, N)), DC=DC,
                                r_fraction=(h["k_safe"] + 0.5) / h["n"])
    r = pair_oracle.replan_pairs(pao.with_own_lists(w, all_limit), threads=threads, **db)
    assert r["k_safe"][0] == h["k_safe"] and np.allclose(r["R"][0], h["R"], rtol=0, atol=1e-12)
    out.update({k: r[k][0] for k in ("safe_dt_index", "safe_sigma_index", "safe_cost", "safe_dt")})
    return out
