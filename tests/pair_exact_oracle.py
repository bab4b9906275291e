"""TEST INFRASTRUCTURE ONLY -- the chained replan with the exact MIQP optimum of every corridor (fq_replan_pairs_exact*),
restated on the CPU one corridor at a time: each sweep takes its factors in ascending order and asks the oracle's
branch-and-bound over all P^N assignments (oracle.pyoracle.solve_miqp) at each; the first factor it solves wins.  R comes
from that winner's fillX and the safe sweep runs the same way from it.  With `ties`, the assignment is the
lexicographically smallest one within a relative 1e-9 of the optimum, found by enumerating every assignment (small N)."""
import itertools

import numpy as np

import pair_assign_oracle as pao


def polys_of(w, kind, j):
    po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
    return [(Ab[fo[p]:fo[p + 1], :3], Ab[fo[p]:fo[p + 1], 3]) for p in range(po[j], po[j + 1])]


def lexmin_tie(N, x0, xf, lim, dt, polys, ff, cost):
    """The lexicographically smallest assignment whose cost is within a relative 1e-9 of `cost` (every P^N checked)."""
    from oracle import pyoracle as po
    for sig in itertools.product(range(len(polys)), repeat=N):
        st, c, _, _ = po.solve_fixed(N, x0, xf, lim, dt, polys, np.array(sig, np.uint8), ff)
        if st == 1 and c <= cost * (1 + 1e-9):
            return np.array(sig, np.uint8)
    raise AssertionError("no assignment attains the optimum")


def exact_sweep(N, x0, xf, lim, polys, dts, ff, ties=False):
    """First time allocation (ascending) at which some assignment is feasible -> dict(dt_index, cost, sigma, coeffs);
    dt_index -1 when none is.  coeffs are a fresh fixed-assignment solve of the winning sigma."""
    from oracle import pyoracle as po
    for i, dt in enumerate(dts):
        rc, c, _, sg, _ = po.solve_miqp(N, x0, xf, lim, dt, polys, ff)
        if rc != 1:
            continue
        sg = np.asarray(sg, np.uint8)[:N]
        if ties:
            sg = lexmin_tie(N, x0, xf, lim, dt, polys, ff, c)
        st, c2, co, _ = po.solve_fixed(N, x0, xf, lim, dt, polys, sg, ff)
        assert st == 1
        return dict(dt_index=i, cost=c, sigma=sg, coeffs=co, dt=dt)
    return dict(dt_index=-1, cost=np.inf, sigma=None, coeffs=None, dt=np.nan)


def replan_pairs_exact(w, F_whole, F_safe, dt_base_whole=None, dt_base_safe=None, ties=False):
    """The exact chain over corridor j's factor lists F_whole[j], F_safe[j] -> per corridor dicts with whole / safe
    (exact_sweep's dicts), R, k_safe and n_samples.  dt_base_*: the device's bases, so that dt is the same to the bit."""
    from oracle import pyoracle as po
    out = []
    DC = w["DC"]
    for j in range(w["n_prob"]):
        dbw = dt_base_whole[j] if dt_base_whole is not None else max(po.dt_initial(w["x0"][j], w["xf_whole"][j], w["lim"][j], w["N_whole"]), 2 * DC)
        wh = exact_sweep(w["N_whole"], w["x0"][j], w["xf_whole"][j], w["lim"][j], polys_of(w, "whole", j),
                         np.asarray(F_whole[j]) * dbw, True, ties)
        rec = dict(whole=wh, safe=dict(dt_index=-1, cost=np.inf, sigma=None, coeffs=None), R=np.full(9, np.nan), k_safe=-1, n_samples=0)
        if wh["dt_index"] >= 0:
            X = po.fill_x(w["N_whole"], wh["coeffs"], wh["dt"], DC)
            k = min(len(X) - 1, int(w["r_fraction"] * len(X)))
            R = X[k, :9].copy()
            rec.update(R=R, k_safe=k, n_samples=len(X))
            dbs = dt_base_safe[j] if dt_base_safe is not None else max(po.dt_initial(R, w["xf_safe"][j], w["lim"][j], w["N_safe"]), 2 * DC)
            rec["safe"] = exact_sweep(w["N_safe"], R, w["xf_safe"][j], w["lim"][j], polys_of(w, "safe", j),
                                      np.asarray(F_safe[j]) * dbs, False, ties)
        out.append(rec)
    return out


def list_index(N, P, all_limit, sigma):
    """sigma's index in L(N, P, all_limit), or -1 when it is not in the list."""
    L = pao.assign_list(N, P, all_limit)
    hit = np.flatnonzero((L == np.asarray(sigma, np.uint8)[None, :]).all(axis=1))
    return int(hit[0]) if len(hit) else -1
