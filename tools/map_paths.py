"""What fq_map_paths costs, and what cropping the safe paths on the device saves a replan, on 64 forest corridors.

  fixture  one map per corridor, each with its seeded unknown cloud (corridor.forest_unknown_cloud).
  mapper   the 64 corridors share one map whose U is every free cell of one forest grid (about 220 000 points).
Timed, alternated, medians over --reps after one warm-up of each:
  paths_dev    fq_map_paths_dev alone on device inputs (CUDA events around the call on one stream);
  paths_host   fq_map_paths (host pointers, blocking: uploads, kernels, copies back);
  dev_route    fq_map_paths_dev then fq_replan_pairs_map_dev (H/R, per-corridor windows) on one stream, no host round trip;
  host_route   fq_paths_cloud (the host twin over per-corridor clouds) then fq_replan_pairs_map on the host paths.
The two routes' records are checked to be byte-equal.  The card's name and power limit are read in the same run.
Usage: python tools/map_paths.py [--reps 9]"""
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

MW, MS, UAV = 3, 4, cr.UAV


def corridors(n, forest=None):
    """n replans (forest_pair_paths dicts) with their JPS_in ("jin") and unknown clouds ("unk"); forest: one shared forest"""
    orig = cr.make_forest
    if forest is not None:
        cr.make_forest = lambda seed, n_trees=60: orig(forest, n_trees=n_trees)
    try:
        out = []
        for seed in range(50000, 50400):
            try:
                fj, p = cr.forest_jps(seed), cr.forest_pair_paths(seed)
            except RuntimeError:
                continue
            p["x0"] = p["x0"].copy()
            p["x0"][:3] = fj["start"]
            p["jin"] = capi.jps_in(fj["jps"], fj["start"], fj["goal"], min(np.linalg.norm(fj["goal"] - fj["start"]) - 0.001, 4.0), 1.5)
            p["unk"] = cr.forest_unknown_cloud(p)
            out.append(p)
            if len(out) == n:
                return out
    finally:
        cr.make_forest = orig
    raise RuntimeError("not enough replans")


def run(name, ps, maps, map_index, unks, solver, torch, reps):
    n = len(ps)
    dev = torch.device("cuda", 0)
    jins = [p["jin"] for p in ps]
    ml = max(len(p["obs"]) + len(u) for p, u in zip(ps, unks))
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 8.0), init_safe=np.ones(n), final_safe=np.full(n, 8.0))
    d_ofs = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in jins])]), dtype=torch.int32, device=dev)
    d_in = torch.from_numpy(np.vstack(jins)).to(dev)
    d_idx = torch.tensor(map_index, dtype=torch.int32, device=dev)
    po = dict(poly_ofs_whole=torch.zeros(n + 1, dtype=torch.int32, device=dev), poly_ofs_safe=torch.zeros(n + 1, dtype=torch.int32, device=dev),
              path_whole=torch.zeros(n * (MW + 1) * 3, dtype=torch.float64, device=dev),
              path_safe=torch.zeros(n * (MS + 1) * 3, dtype=torch.float64, device=dev))
    args = capi.map_paths_args(n, d_ofs.data_ptr(), d_in.data_ptr(), {k: v.data_ptr() for k, v in po.items()}, maps=maps,
                               map_index=d_idx.data_ptr(), max_in=max(len(x) for x in jins), max_poly_whole=MW, max_poly_safe=MS,
                               drone_radius=UAV["drone_radius"])
    st = torch.cuda.Stream(device=dev)
    base = capi.make_decomp_workload([dict(p, path_whole=p["jin"][:2], path_safe=p["jin"][:2]) for p in ps])
    dw = {k: torch.from_numpy(np.ascontiguousarray(base[k])).to(dev) for k in ("x0", "lim", "goal")}
    win = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
    last = torch.zeros(n, dtype=torch.float64, device=dev)
    res = torch.zeros(n * 144, dtype=torch.uint8, device=dev)
    a = capi.PairArgs()
    a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, base["N_whole"], base["N_safe"], base["DC"], 0.6
    a.x0, a.lim, a.results = dw["x0"].data_ptr(), dw["lim"].data_ptr(), res.data_ptr()
    a.poly_ofs_whole, a.poly_ofs_safe = po["poly_ofs_whole"].data_ptr(), po["poly_ofs_safe"].data_ptr()
    for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
        setattr(a, k, int(base[k]))
    longest = {m: max(capi.assign_count(base["N_whole"], P) for P in range(m + 1)) for m in (MW, MS)}
    s = capi.assign_args(0, {}, MW, MS, n * 8 * longest[MW], n * 8 * longest[MS])
    wa = capi.window_args(lambda k: win[k].data_ptr(), {}, 1.0, 20.0, 8, 8)
    dc = capi.decomp_args(lambda k: None if k.startswith("obs_") else (po[k].data_ptr() if k in po else dw[k].data_ptr()), {},
                          UAV["bbox"], UAV["drone_radius"], UAV["z_ground"])
    hr = capi.hr_args(None, None, dict(last_factor_safe=last.data_ptr()))
    mp = capi.map_args(maps, d_idx.data_ptr(), ml)

    def paths_dev():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        capi.map_paths_dev(args, st.cuda_stream)
        e1.record(st)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e-3

    def paths_host():
        t = time.perf_counter()
        capi.map_paths(jins, maps, map_index, max_poly_whole=MW, max_poly_safe=MS)
        return time.perf_counter() - t

    def dev_route():
        torch.cuda.synchronize()
        t = time.perf_counter()
        capi.map_paths_dev(args, st.cuda_stream)
        solver.replan_pairs_map_dev(a, s, wa, None, dc, hr, mp, 0, st.cuda_stream)
        st.synchronize()
        return time.perf_counter() - t

    def host_route():
        t = time.perf_counter()
        hp = capi.paths_cloud(jins, unks, max_poly_whole=MW, max_poly_safe=MS)
        w = dict(base, poly_ofs_whole=hp["poly_ofs_whole"], poly_ofs_safe=hp["poly_ofs_safe"],
                 path_whole=np.ascontiguousarray(hp["path_whole"]), path_safe=np.ascontiguousarray(hp["path_safe"]))
        out = solver.replan_pairs_map(w, maps, np.asarray(map_index), max_local=ml, windows=w0)
        host_route.last = out["results"]
        return time.perf_counter() - t

    fns = dict(paths_dev=paths_dev, paths_host=paths_host, dev_route=dev_route, host_route=host_route)
    times = {k: [] for k in fns}
    for k, f in fns.items():                       # warm-up
        f()
    for _ in range(reps):
        for k, f in fns.items():
            if k == "dev_route":                   # the windows are in/out: every call starts from the same ones
                for kk, v in w0.items():
                    win[kk].copy_(torch.from_numpy(v))
            times[k].append(f())
    for kk, v in w0.items():
        win[kk].copy_(torch.from_numpy(v))
    dev_route()
    same = bytes(res.cpu().numpy()) == host_route.last.tobytes()
    out = {k: round(float(np.median(v)) * 1e3, 4) for k, v in times.items()}
    return dict(workload=name, corridors=n, unknown_points=int(sum(len(u) for u in (unks if len(maps) > 1 else unks[:1]))),
                records_equal=same, median_ms=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    import torch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    solver = capi.Solver(0)
    ps = corridors(64)
    maps = []
    for p in ps:
        m = capi.Map()
        m.update(p["obs"], p["unk"])
        maps.append(m)
    rows = [run("fixture", ps, maps, list(range(64)), [p["unk"] for p in ps], solver, torch, args.reps)]
    ps = corridors(64, forest=11)
    _, centres, radii = cr.make_forest(11, n_trees=60)
    grid, origin, res = cr.voxelise_forest(centres, radii)
    unk = np.ascontiguousarray((np.argwhere(grid == 0)[:, ::-1] + 0.5) * res + origin)
    m = capi.Map()
    m.update(ps[0]["obs"], unk)
    rows.append(run("mapper", ps, [m], [0] * 64, [unk] * 64, solver, torch, args.reps))
    for r in rows:
        r["gpu"] = gpu
        print(json.dumps(r))


if __name__ == "__main__":
    main()
