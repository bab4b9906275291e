#!/usr/bin/env python
"""Parity sweep over EVERY specialised kernel shape (run on the GPU box): N = 4..16, whole and safe mode, 2..8 polytopes,
UAV and ground-robot limits, monotone and arbitrary (non-monotone) assignments -- product kernel and size-generic kernel
against the CPU restatement on the same inputs.  The corridor families are tests/shape_cases.py's, which the GPU suite
runs with one corridor each (test_parity_gpu.py::test_every_solver_shape_matches_the_restatement).
usage: stress_shapes.py [corridors_per_shape]   -> one JSON line."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from faster_b200 import capi                    # noqa: E402
from oracle import pyoracle as po               # noqa: E402
from shape_cases import SHAPES, shape_batches   # noqa: E402

n_corr = int(sys.argv[1]) if len(sys.argv) > 1 else 8
solver = capi.Solver(0)
threads = os.cpu_count() or 1
res = {"corridors_per_shape": n_corr, "shapes": 0, "candidates": 0, "flag_mismatches": 0, "generic_flag_mismatches": 0,
       "max_rel_cost_err": 0.0, "max_coeff_err": 0.0, "feasible": 0, "iteration_cap_hits": 0, "per_shape": [], "mismatch_examples": []}
t0 = time.time()
for N, ff in SHAPES:
    for P, profile, c, pb, dts, sigs in shape_batches(N, ff, n_corr):
        if c == 0:
            shape = dict(N=N, P=P, ff=ff, profile=profile, candidates=0, mism=0, feasible=0)
            res["shapes"] += 1
            res["per_shape"].append(shape)
        fo, co, coo = po.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=threads)
        for generic in (0, 1):
            solver.set_option("force_generic_kernel", generic)
            fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
            bad = np.nonzero(fg != fo)[0]
            if generic:
                res["generic_flag_mismatches"] += int(bad.size)
            else:
                res["flag_mismatches"] += int(bad.size)
                shape["mism"] += int(bad.size)
                res["iteration_cap_hits"] += int((it < 0).sum())
            ok = fo.astype(bool) & fg.astype(bool)
            if ok.any():
                res["max_rel_cost_err"] = max(res["max_rel_cost_err"], float((np.abs(cg[ok] - co[ok]) / np.maximum(1e-9, np.abs(co[ok]))).max()))
                scale = np.maximum(1.0, np.abs(coo[ok]).max(axis=(1, 2), keepdims=True))
                res["max_coeff_err"] = max(res["max_coeff_err"], float((np.abs(cog[ok] - coo[ok]) / scale).max()))
            for i in bad[:2]:
                if len(res["mismatch_examples"]) < 12:
                    res["mismatch_examples"].append(dict(N=N, P=P, ff=ff, generic=generic, corridor=c, cand=int(i), gpu=int(fg[i]),
                                                         oracle=int(fo[i]), dt=float(dts[i]), gpu_cost=float(cg[i]), oracle_cost=float(co[i])))
        solver.set_option("force_generic_kernel", 0)
        shape["candidates"] += int(fo.size)
        shape["feasible"] += int(fo.sum())
        res["candidates"] += int(fo.size)
        res["feasible"] += int(fo.sum())
res["seconds"] = time.time() - t0
print(json.dumps(res))
