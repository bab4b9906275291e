"""What the device decomposition of the chained replan costs and changes, on 64 mixed forest corridors
(corridor.forest_pair_paths), against today's faithful route.

  decomp    one fq_replan_pairs_decomp submission: paths, clouds and G in; both corridors made on the device, the safe one
            around the device's R.
  faithful  the host decomposes the whole corridors (and the safe ones around the estimated R, which the first submission
            needs as input), runs fq_replan_pairs_assign, reads R, decomposes the safe corridors around it and runs
            fq_replan_pairs_assign again.  Its records must match decomp's (winners identical, values within 1e-12).
  host      the host decompositions of one faithful replan alone (whole + safe around R).
Also counted: safe winners that differ between corridors cut around the estimated R (today's generator, one submission) and
around the device's R.  Medians over alternated repetitions; the card's name and power limit are read in the same run.
Usage: python tools/decomp_replan.py [--n 64] [--reps 15]"""
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

UAV = cr.UAV
FAC = np.arange(1.0, 11.0)


def decompose(path, obs):
    return capi.ellipsoid_decomp(path, obs, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"], cap_rows=8192)


def corridor(p, path, polys):
    xf = np.zeros(9)
    A, b = polys[-1]
    xf[:3] = p["goal"] if not np.any(A @ p["goal"] - b > 0) else path[-1]
    return dict(N=p["N"], x0=p["x0"], xf=xf, lim=p["lim"], polys=polys)


def pair_workload(whole, safe, w):
    return capi.make_pair_workload(whole, safe, FAC, np.zeros((1, 10)), FAC, np.zeros((1, 10)), DC=w["DC"], r_fraction=w["r_fraction"])


def faithful(s, ps, w):
    t0 = time.perf_counter()
    whole = [corridor(p, p["path_whole"], decompose(p["path_whole"], p["obs"])) for p in ps]
    est = [corridor(p, p["path_safe"], decompose(p["path_safe"], p["obs"])) for p in ps]
    first = s.replan_pairs_assign(pair_workload(whole, est, w), want_candidates=False, want_coeffs=False)
    safe = []
    for j, p in enumerate(ps):
        sp = p["path_safe"].copy()
        sp[0] = first["results"]["R"][j][:3]
        safe.append(corridor(p, sp, decompose(sp, p["obs"])))
    out = s.replan_pairs_assign(pair_workload(whole, safe, w), want_candidates=False, want_coeffs=False)
    return time.perf_counter() - t0, out, first


def host_only(ps, R):
    t0 = time.perf_counter()
    for j, p in enumerate(ps):
        decompose(p["path_whole"], p["obs"])
        sp = p["path_safe"].copy()
        sp[0] = R[j][:3]
        decompose(sp, p["obs"])
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ps = [cr.forest_pair_paths(30000 + k) for k in range(args.n)]
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    s = capi.Solver(0)
    dev = s.replan_pairs_decomp(w, want_coeffs=False)           # warm-up (and the reference answer)
    _, ref, first = faithful(s, ps, w)
    rd, rf = dev["results"], ref["results"]
    same_winners = all(np.array_equal(rd[k], rf[k]) for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index",
                                                              "n_samples_whole", "k_safe"))
    rel = max(float(np.nanmax(np.abs(rd[k] - rf[k]) / np.maximum(np.abs(rf[k]), 1.0)))
              for k in ("whole_cost", "safe_cost", "whole_dt", "safe_dt", "R"))
    # today's generator: the safe corridor cut around the estimated R, one submission
    est = first["results"]
    changed = int(np.sum((est["safe_dt_index"] != rd["safe_dt_index"]) | (est["safe_sigma_index"] != rd["safe_sigma_index"])))
    t_dev, t_faith, t_host = [], [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        s.replan_pairs_decomp(w, want_coeffs=False)
        t_dev.append(time.perf_counter() - t0)
        t_faith.append(faithful(s, ps, w)[0])
        t_host.append(host_only(ps, rd["R"]))
    s.close()
    med = lambda x: float(np.median(x)) * 1e3  # noqa: E731
    print(json.dumps(dict(card=card, n_corridors=args.n, reps=args.reps, decomp_ms=med(t_dev), faithful_ms=med(t_faith),
                          host_decomp_ms=med(t_host), records_same_winners=bool(same_winners), records_max_rel_diff=rel,
                          safe_winners_changed_vs_estimated_R=changed,
                          whole_winners=int((rd["whole_dt_index"] >= 0).sum()), safe_winners=int((rd["safe_dt_index"] >= 0).sum()),
                          mean_cloud_points=float(np.mean([len(p["obs"]) for p in ps])))))


if __name__ == "__main__":
    main()
