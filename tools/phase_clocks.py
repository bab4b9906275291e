#!/usr/bin/env python
"""Where a sweep candidate's time goes: runs the chained replan on cfg4 batch 0 (64 corridors, as one bench.py pass) with a
library built with -DFQ_PHASE_CLOCKS and prints, for the whole and the safe sweep, each phase's share of the solver warps'
clock cycles, split by outcome: "settled" candidates are decided by the iterate w = 0 (optimal with no iteration, or
infeasible at the first entering row), the others need the active-set iteration.  Candidates the early exit skips never
reach solve_candidate and are not counted; the winners' re-solve (one candidate per corridor) is.  The last line of each
table, "corridor scans", is the part of the first-scan and iteration phases spent scanning the corridor rows for the
entering row (every scan of gi_loop, up to the warp's choice): a share of the same cycles, not an eighth phase.

usage: phase_clocks.py [--build] [--reps K] [--lib NAME]   (--build compiles faster_b200/lib/NAME first, on any machine)
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["claim + input loads", "setup_rows + guards", "segment-0 check", "build_items", "first scan", "iterations", "outputs"]

ap = argparse.ArgumentParser()
ap.add_argument("--build", action="store_true")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--lib", default="libfaster_b200_phase.so")
ap.add_argument("--json", help="also write the table as JSON here")
args = ap.parse_args()
sys.path.insert(0, ROOT)
lib_path = os.path.join(ROOT, "faster_b200", "lib", args.lib)
if args.build:
    from faster_b200 import build as b
    print(b.build(extra_flags=["-DFQ_PHASE_CLOCKS"], out=lib_path))
    sys.exit(0)
os.environ["FQ_LIB"] = lib_path                 # read by faster_b200.capi at import

import numpy as np  # noqa: E402
import torch  # noqa: E402
import bench  # noqa: E402
from faster_b200 import capi  # noqa: E402

L = capi.lib()
if not hasattr(L, "fq_phase_clocks"):
    sys.exit("%s was not built with -DFQ_PHASE_CLOCKS (run with --build first)" % lib_path)
L.fq_phase_clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
buf = (C.c_ulonglong * 36)()


def read(reset):
    if L.fq_phase_clocks(buf, 1 if reset else 0) != 0:
        sys.exit("fq_phase_clocks failed")
    return np.array(buf[:], dtype=np.float64).reshape(2, 2, 9)


dev = torch.device("cuda:0")
solver = capi.Solver(0)
st = torch.cuda.Stream(device=dev)
b = bench.PairBatch(bench.load_cfg4(0, 64), dev, torch, capi)
solver.replan_pairs_dev(b.args, 0, st.cuda_stream)            # warm-up (module load, scratch allocation)
torch.cuda.synchronize()
read(True)
for _ in range(args.reps):
    solver.replan_pairs_dev(b.args, 0, st.cuda_stream)
torch.cuda.synchronize()
acc = read(True)
solver.close()

out = {}
for mi, mode in ((1, "whole"), (0, "safe")):
    cyc = acc[mi, :, :7]                      # [settled][phase]
    n = acc[mi, :, 7]
    tot = cyc.sum()
    print("%s sweep: %d candidates solved per chain, %.1f %% settled at w = 0; settled candidates take %.1f %% of the cycles"
          % (mode, n.sum() / args.reps, 100 * n[1] / max(n.sum(), 1), 100 * cyc[1].sum() / max(tot, 1)))
    print("  %-22s %9s %9s %9s   %12s %12s" % ("phase", "all %", "settled %", "other %", "settled cyc", "other cyc"))
    rows = []
    for k, name in enumerate(PHASES):
        r = dict(phase=name, share=cyc[:, k].sum() / tot, settled=cyc[1, k] / tot, other=cyc[0, k] / tot,
                 settled_cycles_per_cand=cyc[1, k] / max(n[1], 1), other_cycles_per_cand=cyc[0, k] / max(n[0], 1))
        rows.append(r)
        print("  %-22s %9.1f %9.1f %9.1f   %12.0f %12.0f" % (name, 100 * r["share"], 100 * r["settled"], 100 * r["other"],
                                                           r["settled_cycles_per_cand"], r["other_cycles_per_cand"]))
    scan = acc[mi, :, 8]
    sc = dict(share=scan.sum() / tot, settled=scan[1] / tot, other=scan[0] / tot,
              settled_cycles_per_cand=scan[1] / max(n[1], 1), other_cycles_per_cand=scan[0] / max(n[0], 1))
    print("  %-22s %9.1f %9.1f %9.1f   %12.0f %12.0f" % ("(corridor scans)", 100 * sc["share"], 100 * sc["settled"], 100 * sc["other"],
                                                       sc["settled_cycles_per_cand"], sc["other_cycles_per_cand"]))
    out[mode] = dict(candidates=float(n.sum() / args.reps), settled_fraction=float(n[1] / max(n.sum(), 1)),
                     settled_cycle_share=float(cyc[1].sum() / max(tot, 1)), phases=rows,
                     corridor_scans={k: float(v) for k, v in sc.items()})
props = torch.cuda.get_device_properties(0)
print("device:", props.name)
if args.json:
    with open(args.json, "w") as f:
        json.dump(dict(device=props.name, reps=args.reps, sweeps=out), f, indent=1)
