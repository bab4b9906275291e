"""Price of the exact chain: one fq_replan_pairs_assign submission (the best non-decreasing assignment of every corridor)
against one fq_replan_pairs_exact submission (the MIQP optimum over all P^N assignments, by branch-and-bound on the device)
on config-4 corridors of the committed fixture, all_limit 0, factors 1..F.  Both go through the host-pointer ABI and end
in a device synchronise; the two are alternated.  Reported per batch: the median times, tree nodes per corridor (mean and
max), exact = 0 counts, and the corridors whose whole or safe winner changed.  Then the same with every corridor's
polytopes in a random order, where the non-decreasing lists miss the natural assignment.  Prints one JSON line with the
card's name and its power limit.

    python tools/exact_replan.py [--corridors 64] [--factors 16] [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
from faster_b200 import capi  # noqa: E402
from mixed_replan import card  # noqa: E402


def permuted(w, seed):
    """Every corridor's polytopes (whole and safe) in a random order."""
    rng = np.random.default_rng(seed)
    out = dict(w)
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        nfo, rows = [0], []
        for j in range(w["n_prob"]):
            for q in rng.permutation(int(po[j + 1] - po[j])):
                p = po[j] + q
                rows.append(Ab[fo[p]:fo[p + 1]])
                nfo.append(nfo[-1] + fo[p + 1] - fo[p])
        out["face_ofs_" + kind] = np.asarray(nfo, np.int32)
        out["Ab_" + kind] = np.ascontiguousarray(np.vstack(rows))
    return out


def measure(s, w, reps, warmup):
    def lst():
        return s.replan_pairs_assign(w, all_limit=0, want_candidates=False)

    def ex():
        return s.replan_pairs_exact(w, all_limit=0, want_candidates=False)
    a, e = lst(), ex()
    for _ in range(warmup):
        lst(); ex()
    t_a, t_e = [], []
    for _ in range(reps):                                            # alternate the two
        t0 = time.perf_counter(); lst(); t_a.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); ex(); t_e.append(time.perf_counter() - t0)
    ra, re_ = a["results"], e["results"]
    changed = {}
    for kind in ("whole", "safe"):
        diff = (ra[kind + "_dt_index"] != re_[kind + "_dt_index"]) | (ra[kind + "_cost"] != re_[kind + "_cost"]) | \
            (a["sigma_" + kind] != e["sigma_" + kind]).any(axis=1)
        changed[kind] = int(diff.sum())
    ma, me = float(np.median(t_a)), float(np.median(t_e))
    return dict(assign_ms_median=1e3 * ma, exact_ms_median=1e3 * me, exact_over_assign=me / ma,
                assign_ms_minmax=[1e3 * min(t_a), 1e3 * max(t_a)], exact_ms_minmax=[1e3 * min(t_e), 1e3 * max(t_e)],
                nodes_whole_mean=float(e["nodes_whole"].mean()), nodes_whole_max=int(e["nodes_whole"].max()),
                nodes_safe_mean=float(e["nodes_safe"].mean()), nodes_safe_max=int(e["nodes_safe"].max()),
                exact0_whole=int((e["exact_whole"] == 0).sum()), exact0_safe=int((e["exact_safe"] == 0).sum()),
                changed_whole=changed["whole"], changed_safe=changed["safe"],
                non_monotone_whole=int((np.diff(e["sigma_whole"].astype(int), axis=1) < 0).any(axis=1).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corridors", type=int, default=64)
    ap.add_argument("--factors", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    w = bench.load_cfg4(0, args.corridors)
    w["factors_whole"] = w["factors_safe"] = np.arange(1.0, args.factors + 1.0)
    s = capi.Solver(0)
    natural = measure(s, w, args.reps, args.warmup)
    perm = measure(s, permuted(w, args.seed), args.reps, args.warmup)
    s.close()
    out = dict(metric="exact_replan", corridors=args.corridors, N_whole=w["N_whole"], N_safe=w["N_safe"], all_limit=0,
               factors=args.factors, natural=natural, permuted=perm, **card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
