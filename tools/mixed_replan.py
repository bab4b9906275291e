"""Mixed-batch chained replan: one fq_replan_pairs_assign submission versus the same corridors split into one fq_replan_pairs
submission per (P_whole, P_safe) combination, each with that combination's shared lists -- what a caller had to do before
the batch path took a list per corridor.  The corridors come from corridor.make_forest_pair_mixed (polytope counts trimmed
as Faster::replan trims them).  Both ways run through the host-pointer ABI and end in a device synchronise; the result
records of the two must be identical, byte for byte.  Prints one JSON line with replans/s of both ways, the card's name
and its power limit.

    python tools/mixed_replan.py [--corridors 64] [--N 10] [--all-limit 0] [--reps 30] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from faster_b200 import capi, corridor as cr  # noqa: E402


def assign_list(N, P, all_limit):
    """L(N, P, all_limit) of include/faster_b200.h, enumerated on the host (for the split submissions only)."""
    if P == 0:
        return np.zeros((1, N), np.uint8)
    if P > 1 and P ** N <= all_limit:
        idx = np.arange(P ** N, dtype=np.int64)[:, None]
        return ((idx // (P ** np.arange(N - 1, -1, -1, dtype=np.int64))[None, :]) % P).astype(np.uint8)
    return cr.monotone_sigmas(N, P)


def subset(w, idx):
    """Corridors idx of a pair workload as a workload of their own."""
    out = dict(w, n_prob=len(idx))
    for k in ("x0", "xf_whole", "xf_safe", "lim"):
        out[k] = np.ascontiguousarray(w[k][idx])
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        npo, nfo, rows = [0], [0], []
        for j in idx:
            for p in range(po[j], po[j + 1]):
                rows.append(Ab[fo[p]:fo[p + 1]])
                nfo.append(nfo[-1] + fo[p + 1] - fo[p])
            npo.append(npo[-1] + po[j + 1] - po[j])
        nfo, npo = np.asarray(nfo, np.int32), np.asarray(npo, np.int32)
        out["poly_ofs_" + kind], out["face_ofs_" + kind] = npo, nfo
        out["Ab_" + kind] = np.ascontiguousarray(np.vstack(rows)) if rows else np.zeros((1, 4))
        out["max_faces_" + kind] = max(int(max(nfo[npo[j + 1]] - nfo[npo[j]] for j in range(len(idx)))), 1)
        out["max_poly_faces_" + kind] = int(np.diff(nfo).max()) if len(nfo) > 1 else 0
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                                          # report what could not be read, never guess it
        return dict(gpu="unknown (%s)" % e, power_limit="unknown", max_sm_clock="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corridors", type=int, default=64)
    ap.add_argument("--N", type=int, default=10)
    ap.add_argument("--all-limit", type=int, default=0)
    ap.add_argument("--factors", type=int, default=16)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--seed", type=int, default=9000)
    args = ap.parse_args()
    N, lim = args.N, args.all_limit
    pairs = [cr.make_forest_pair_mixed(args.seed + j, N=N) for j in range(args.corridors)]
    fac = np.linspace(1.0, 3.0, args.factors)
    none = np.zeros((0, N), np.uint8)
    w = capi.make_pair_workload([p[0] for p in pairs], [p[1] for p in pairs], fac, none, fac, none, DC=0.01, r_fraction=0.6)
    pw, ps = np.diff(w["poly_ofs_whole"]), np.diff(w["poly_ofs_safe"])
    groups = {}
    for j, key in enumerate(zip(pw.tolist(), ps.tolist())):
        groups.setdefault(key, []).append(j)
    split = []
    for (a, b), idx in sorted(groups.items()):
        sw = subset(w, idx)
        sw["sigmas_whole"], sw["sigmas_safe"] = assign_list(N, a, lim), assign_list(N, b, lim)
        split.append((idx, sw))
    s = capi.Solver(0)

    def one():
        return s.replan_pairs_assign(w, all_limit=lim, want_candidates=False, want_coeffs=False)["results"]

    def many():
        rec = np.zeros(w["n_prob"], capi.PAIR_RESULT_DTYPE)
        for idx, sw in split:
            rec[idx] = s.replan_pairs(sw, want_candidates=False, want_coeffs=False)["results"]
        return rec
    a, b = one(), many()
    same = a.tobytes() == b.tobytes()
    for _ in range(args.warmup):
        one(); many()
    t_one, t_many = [], []
    for _ in range(args.reps):                                       # alternate the two ways
        t0 = time.perf_counter(); one(); t_one.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); many(); t_many.append(time.perf_counter() - t0)
    s.close()
    m1, m2 = float(np.median(t_one)), float(np.median(t_many))
    out = dict(metric="mixed_replan", corridors=args.corridors, N=N, all_limit=lim, factors=args.factors,
               candidates_whole=int(capi.assign_offsets(w["poly_ofs_whole"], N, args.factors, lim)[-1]),
               candidates_safe=int(capi.assign_offsets(w["poly_ofs_safe"], N, args.factors, lim)[-1]),
               combinations=len(split), records_identical=bool(same),
               one_submission_replans_per_s=args.corridors / m1, split_replans_per_s=args.corridors / m2,
               one_submission_ms_median=1e3 * m1, split_ms_median=1e3 * m2,
               one_submission_ms_minmax=[1e3 * min(t_one), 1e3 * max(t_one)], split_ms_minmax=[1e3 * min(t_many), 1e3 * max(t_many)],
               speedup=m2 / m1, **card())
    print(json.dumps(out))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
