"""TEST INFRASTRUCTURE ONLY -- the chained replan with a per-corridor assignment list (fq_replan_pairs_assign*), restated on
the CPU: the lists L(N, P, all_limit) enumerated in numpy, and the chain run corridor by corridor through the CPU
restatement of oracle/pair_oracle.py (the corridors of a batch are independent, so one corridor with its own list is the
whole definition)."""
import itertools

import numpy as np

from faster_b200 import capi


def all_assignments(N, P):
    """All P^N assignments, lexicographic with segment 0 most significant (SolverGurobi::ensureAssignments' ALL order)."""
    return np.array(list(itertools.product(range(P), repeat=N)), np.uint8).reshape(-1, N)


def monotone(N, P):
    """Non-decreasing assignments in lexicographic order, enumerated here (not through the library)."""
    return np.array([c for c in itertools.combinations_with_replacement(range(P), N)], np.uint8).reshape(-1, N)


def assign_list(N, P, all_limit):
    """L(N, P, all_limit) of include/faster_b200.h."""
    if P == 0:
        return np.zeros((1, N), np.uint8)
    if P > 1 and P ** N <= all_limit:
        return all_assignments(N, P)
    return monotone(N, P)


def corridor(w, j):
    """Corridor j of a pair workload as a one-corridor workload (its sigmas_* are left to the caller)."""
    out = dict(w)
    out["n_prob"] = 1
    for k in ("x0", "xf_whole", "xf_safe", "lim"):
        out[k] = np.ascontiguousarray(w[k][j:j + 1])
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        p0, p1 = int(po[j]), int(po[j + 1])
        out["poly_ofs_" + kind] = np.array([0, p1 - p0], np.int32)
        out["face_ofs_" + kind] = np.ascontiguousarray(fo[p0:p1 + 1] - fo[p0], np.int32)
        out["Ab_" + kind] = np.ascontiguousarray(Ab[fo[p0]:fo[p1]]) if fo[p1] > fo[p0] else np.zeros((1, 4))
        faces = np.diff(out["face_ofs_" + kind])
        out["max_faces_" + kind] = max(int(faces.sum()), 1)
        out["max_poly_faces_" + kind] = int(faces.max()) if len(faces) else 0
    return out


def with_own_lists(w1, all_limit):
    """A one-corridor workload with the shared lists set to the corridor's own lists."""
    out = dict(w1)
    for kind in ("whole", "safe"):
        P = int(w1["poly_ofs_" + kind][1])
        out["sigmas_" + kind] = np.ascontiguousarray(assign_list(w1["N_" + kind], P, all_limit))
    return out


def replan_pairs_assign(w, all_limit, threads=4, dt_base_whole=None, dt_base_safe=None):
    """The CPU chain with per-corridor lists -> the fields of oracle.pair_oracle.replan_pairs, with per-candidate arrays
    concatenated in corridor order and cand_ofs_whole / cand_ofs_safe."""
    from oracle import pair_oracle
    per = []
    for j in range(w["n_prob"]):
        w1 = with_own_lists(corridor(w, j), all_limit)
        per.append(pair_oracle.replan_pairs(w1, threads=threads,
                                            dt_base_whole=None if dt_base_whole is None else dt_base_whole[j:j + 1],
                                            dt_base_safe=None if dt_base_safe is None else dt_base_safe[j:j + 1]))
    out = {}
    for k in per[0]:
        out[k] = np.concatenate([p[k] for p in per])
    for kind in ("whole", "safe"):
        out["cand_ofs_" + kind] = capi.assign_offsets(w["poly_ofs_" + kind], w["N_" + kind], len(w["factors_" + kind]), all_limit)
    return out
