"""What choosing H and R from the unknown clouds costs and changes, on 64 forest corridors with seeded unknown clouds
(corridor.forest_pair_paths + corridor.forest_unknown_cloud), against the r_fraction rule.

  decomp  one fq_replan_pairs_decomp submission, R at k_safe = min(n - 1, (int)(0.6 n)) on every corridor.
  hr      one fq_replan_pairs_hr submission: findIndexH / findIndexR on the device; corridors that need no safe path skip the
          safe decomposition and sweep.
Host-pointer calls timed with a host clock (each blocks until its outputs are in host memory), alternated, medians over --reps
after one warm-up of each.  Also counted: corridors that need no safe path, and corridors whose k_safe or safe winner
differs from the r_fraction rule's.  The card's name and power limit are read in the same run.
Usage: python tools/hr_replan.py [--n 64] [--reps 15]"""
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

FAC = np.arange(1.0, 11.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    ps = [cr.forest_pair_paths(30000 + k) for k in range(args.n)]
    for p in ps:
        p["unk"] = cr.forest_unknown_cloud(p)
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    w["r_fraction"] = 0.6
    s = capi.Solver(0)
    dec = s.replan_pairs_decomp(w, want_coeffs=False)          # warm-up, and the answers compared below
    hr = s.replan_pairs_hr(w, want_coeffs=False)
    rd, rh = dec["results"], hr["results"]
    won = rh["whole_dt_index"] >= 0
    t_dec, t_hr = [], []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        s.replan_pairs_decomp(w, want_coeffs=False)
        t_dec.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        s.replan_pairs_hr(w, want_coeffs=False)
        t_hr.append(time.perf_counter() - t0)
    s.close()
    med = lambda x: float(np.median(x)) * 1e3  # noqa: E731
    safe_diff = (rd["safe_dt_index"] != rh["safe_dt_index"]) | (rd["safe_sigma_index"] != rh["safe_sigma_index"])
    print(json.dumps(dict(card=card, n_corridors=args.n, reps=args.reps, decomp_ms=med(t_dec), hr_ms=med(t_hr),
                          whole_winners=int(won.sum()), no_safe_path=int((won & (hr["need_safe"] == 0)).sum()),
                          k_safe_differs=int((won & (rd["k_safe"] != rh["k_safe"])).sum()),
                          safe_winner_differs=int((won & safe_diff).sum()),
                          safe_winners_decomp=int((rd["safe_dt_index"] >= 0).sum()), safe_winners_hr=int((rh["safe_dt_index"] >= 0).sum()),
                          mean_unknown_points=float(np.mean([len(p["unk"]) for p in ps])))))


if __name__ == "__main__":
    main()
