"""What sampling the committed plan on the device saves against sampling it on the host, on two workloads:

  assign  64 config-4 fixture corridors through the per-corridor-list chain (fq_replan_pairs_assign)
  map     the 64 forest corridors of tools/map_replan.py, one indexed map per corridor, through fq_replan_pairs_map with H/R

and two routes that give the same plan:

  plan    one fq_replan_pairs_plan submission: the family's outputs plus every corridor's plan piece, sampled on the device
  host    the family's own submission with coeffs_whole / coeffs_safe, then fq_fill_x on the host for every winner (the full
          sample count) and the pieces stitched as appendToPlan pushes them

The two routes' plans are asserted byte-identical.  Host-pointer calls timed with a host clock (each blocks until its outputs
are in host memory), alternated, medians over --reps after one warm-up of each; the host route's sampling and stitching is also
reported on its own.  Bytes copied device to host count every output of the call.  The card's name and power limit are read in
the same run.
Usage: python tools/plan_replan.py [--reps 15]"""
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


def host_plan(out, w):
    """appendToPlan on the host from the family's records and coefficients: -> (states, plan_ofs, status)."""
    res, need = out["results"], out.get("need_safe")
    pieces, status = [], np.zeros(len(res), np.int32)
    for j, r in enumerate(res):
        nd = need is None or bool(need[j])
        if r["whole_dt_index"] < 0 or (nd and r["safe_dt_index"] < 0):
            pieces.append(np.zeros((0, 12)))
            status[j] = capi.PLAN_NONE
            continue
        p = [capi.fill_x(w["N_whole"], out["coeffs_whole"][j].reshape(-1), r["whole_dt"], w["DC"])[:r["k_safe"] + 1]]
        if nd:
            p.append(capi.fill_x(w["N_safe"], out["coeffs_safe"][j].reshape(-1), r["safe_dt"], w["DC"]))
        pieces.append(np.vstack(p))
    ofs = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.int64)
    return np.vstack(pieces), ofs, status


def nbytes(out, rows=None):
    return sum(int(v[:rows].nbytes) if (k == "states" and rows is not None) else int(np.asarray(v).nbytes)
               for k, v in out.items() if not k.startswith("_"))


def run(family, w, args, kw, reps, cap=1 << 17):
    fam = getattr(s, "replan_pairs_" + family)

    def by_plan():
        return s.replan_pairs_plan(w, cap, family, *args, want_coeffs=False, **kw)

    def by_host():
        out = fam(w, *args, want_coeffs=True, **kw)
        t0 = time.perf_counter()
        hp = host_plan(out, w)
        return out, hp, time.perf_counter() - t0
    a = by_plan()
    b, hp, _ = by_host()
    total = int(a["plan_ofs"][-1])
    same = (a["plan_ofs"].tobytes() == hp[1].tobytes() and a["status"].tobytes() == hp[2].tobytes()
            and a["states"][:total].tobytes() == hp[0].tobytes() and a["results"].tobytes() == b["results"].tobytes())
    assert same, "the two routes' plans differ"
    t_plan, t_host, t_sample = [], [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        by_plan()
        t_plan.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        _, _, ts = by_host()
        t_host.append(time.perf_counter() - t0)
        t_sample.append(ts)
    med = lambda x: float(np.median(x)) * 1e3  # noqa: E731
    return dict(n_corridors=int(w["n_prob"]), plan_rows=total, ok=int((a["status"] == capi.PLAN_OK).sum()), plan_ms=med(t_plan),
                host_route_ms=med(t_host), host_sampling_ms=med(t_sample), plan_d2h_bytes=nbytes(a, total), host_d2h_bytes=nbytes(b),
                identical=bool(same))


def main():
    global s
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    s = capi.Solver(0)
    import bench
    out = dict(card=card, reps=args.reps)
    out["assign"] = run("assign", bench.load_cfg4(0, 64), (), dict(want_candidates=False), args.reps)
    ps = [cr.forest_pair_paths(30000 + k) for k in range(64)]
    for p in ps:
        p["unk"] = cr.forest_unknown_cloud(p)
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    w["r_fraction"] = 0.6
    maps = []
    for p in ps:
        m = capi.Map()
        m.update(p["obs"], p["unk"])
        maps.append(m)
    out["map"] = run("map", w, (maps, np.arange(64, dtype=np.int32)), dict(max_local=1 << 15), args.reps)
    for m in maps:
        m.close()
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
