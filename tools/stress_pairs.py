#!/usr/bin/env python
"""Large parity sweep of the chained replan (run on the GPU box): every corridor of the committed cfg4 fixture through
fq_replan_pairs against the CPU chains -- the tuned port (oracle/fq_cpu_port.c, all 512
corridors) and the literal restatement (oracle/fq_oracle.c via pair_oracle, a slice).  Prints one JSON line."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench                                    # noqa: E402
from faster_b200 import capi                    # noqa: E402
from oracle import pair_oracle, pyoracle as po  # noqa: E402

n_batches = int(sys.argv[1]) if len(sys.argv) > 1 else 8
s = capi.Solver(0)
res = {"corridors": 0, "pairs": 0, "flag_mismatches_vs_port": 0, "winner_mismatches_vs_port": 0, "max_rel_cost_err": 0.0,
       "literal_slice": {}}
t0 = time.time()
threads = os.cpu_count() or 1
for b in range(n_batches):
    w = bench.load_cfg4(64 * b, 64)
    g = s.replan_pairs(w)
    r = g["results"]
    p = po.replan_pairs_port(w, threads)
    pr = p["results"]
    for k in ("whole", "safe"):
        res["flag_mismatches_vs_port"] += int((g["feasible_" + k] != p["feasible_" + k]).sum())
        ok = g["feasible_" + k].astype(bool) & p["feasible_" + k].astype(bool)
        if ok.any():
            res["max_rel_cost_err"] = max(res["max_rel_cost_err"], float((np.abs(g["cost_" + k][ok] - p["cost_" + k][ok]) / np.maximum(1e-9, np.abs(p["cost_" + k][ok]))).max()))
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "k_safe", "n_samples_whole"):
        res["winner_mismatches_vs_port"] += int((r[f] != pr[f]).sum())
    res["corridors"] += 64
    res["pairs"] += bench.pairs_per_pass(w)
    if b == 0:
        wl = bench.load_cfg4_like(w, 16)
        gl = s.replan_pairs(wl)
        o = pair_oracle.replan_pairs(wl, threads, dt_base_whole=gl["results"]["whole_dt_base"], dt_base_safe=gl["results"]["safe_dt_base"])
        res["literal_slice"] = {"pairs": int(bench.pairs_per_pass(wl)),
                                "flag_mismatches": int((gl["feasible_whole"] != o["feasible_whole"]).sum() + (gl["feasible_safe"] != o["feasible_safe"]).sum()),
                                "winner_mismatches": int((gl["results"]["whole_dt_index"] != o["whole_dt_index"]).sum() + (gl["results"]["safe_dt_index"] != o["safe_dt_index"]).sum() +
                                                         (gl["results"]["safe_sigma_index"] != o["safe_sigma_index"]).sum())}
res["seconds"] = time.time() - t0
print(json.dumps(res))
