"""What an indexed map on the device saves against per-corridor clouds, on 64 forest corridors: one fq_replan_pairs_hr
submission (every corridor's O, U ++ O and U uploaded with it) against one fq_replan_pairs_map submission (the corridors read
maps uploaded and indexed beforehand), with the same answers.

  fixture  one map per corridor, each corridor in its own forest with its seeded unknown cloud (corridor.forest_unknown_cloud):
           the clouds the tests use, a few thousand unknown points per corridor.
  mapper   64 corridors in one forest sharing one map whose U is every free cell of the forest grid (16 x 16 x 3 m at
           0.15 m, about 220 000 points): the size a mapper publishes.
Host-pointer calls timed with a host clock (each blocks until its outputs are in host memory), alternated, medians over
--reps after one warm-up of each.  Map updates (fq_map_update, host clouds, blocking) are timed separately: the first
update of a new map (which also allocates the map's arrays) and, as medians over --reps, later updates with the same clouds
(the capacity already holds them: the steady cost per mapper message).  Bytes uploaded
per submission count the inputs that differ between the two entries: the clouds and offsets, or the map index.  The card's
name and power limit are read in the same run.
Usage: python tools/map_replan.py [--reps 9]"""
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


def csr(clouds):
    ofs = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    return ofs, np.ascontiguousarray(np.vstack([np.reshape(c, (-1, 3)) for c in clouds] + [np.zeros((1, 3))]), np.float64)


def same_forest(forest_seed, k):
    """k replans in the forest of `forest_seed`, each with its own start and goal."""
    orig = cr.make_forest
    cr.make_forest = lambda seed, n_trees=60: orig(forest_seed, n_trees=n_trees)
    try:
        ps = []
        for s in range(400):
            try:
                ps.append(cr.forest_pair_paths(forest_seed * 1000 + s))
            except RuntimeError:
                continue
            ps[-1]["unk"] = cr.forest_unknown_cloud(ps[-1])
            if len(ps) == k:
                return ps
    finally:
        cr.make_forest = orig
    raise RuntimeError("not enough replans")


def run(s, ps, occs, unks, shared, reps):
    n = len(ps)
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    w["r_fraction"] = 0.6
    w["obs_ofs_whole"], w["obs_whole"] = csr(occs)
    w["obs_ofs_safe"], w["obs_safe"] = csr([np.vstack([u, o]) for u, o in zip(unks, occs)])
    w["unk_ofs"], w["unk"] = csr(unks)
    t_first, t_up, maps = [], [], []
    for o, u in ([(occs[0], unks[0])] if shared else zip(occs, unks)):
        m = capi.Map()
        t0 = time.perf_counter()
        m.update(o, u)
        t_first.append(time.perf_counter() - t0)
        maps.append(m)
    for _ in range(reps):
        for m, o, u in zip(maps, occs, unks):
            t0 = time.perf_counter()
            m.update(o, u)
            t_up.append(time.perf_counter() - t0)
    idx = None if shared else np.arange(n, dtype=np.int32)
    cloud_bytes = sum(int(w[k].nbytes) for k in ("obs_ofs_whole", "obs_whole", "obs_ofs_safe", "obs_safe", "unk_ofs", "unk"))
    a = s.replan_pairs_hr(w, want_coeffs=False)
    b = s.replan_pairs_map(w, maps, idx, max_local=1 << 15, want_coeffs=False)
    def rows(o, k):                                             # of Ab_* the rows face_ofs_* fills; the rest is undefined
        return o[k][:int(o["face_ofs_" + k[3:]][-1])] if k.startswith("Ab_") else np.asarray(o[k])
    same = sorted(a) == sorted(b) and all(rows(a, k).tobytes() == rows(b, k).tobytes() for k in a)
    t_hr, t_map = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        s.replan_pairs_hr(w, want_coeffs=False)
        t_hr.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        s.replan_pairs_map(w, maps, idx, max_local=1 << 15, want_coeffs=False)
        t_map.append(time.perf_counter() - t0)
    med = lambda x: float(np.median(x)) * 1e3  # noqa: E731
    return dict(n_corridors=n, maps=len(maps), unknown_points_per_map=float(np.mean([len(u) for u in unks[:len(maps)]])),
                occupied_points_per_map=float(np.mean([len(o) for o in occs[:len(maps)]])), hr_ms=med(t_hr), map_ms=med(t_map),
                first_map_update_ms=med(t_first), map_update_ms=med(t_up), hr_cloud_bytes=cloud_bytes, map_index_bytes=0 if shared else 4 * n,
                same_outputs=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    s = capi.Solver(0)
    ps = [cr.forest_pair_paths(30000 + k) for k in range(64)]
    for p in ps:
        p["unk"] = cr.forest_unknown_cloud(p)
    out = dict(card=card, reps=args.reps)
    out["fixture"] = run(s, ps, [p["obs"] for p in ps], [p["unk"] for p in ps], False, args.reps)
    ps = same_forest(11, 64)
    _, centres, radii = cr.make_forest(11, n_trees=60)
    grid, origin, res = cr.voxelise_forest(centres, radii)
    unk = np.ascontiguousarray((np.argwhere(grid == 0)[:, ::-1] + 0.5) * res + origin)
    occ = ps[0]["obs"]
    out["mapper"] = run(s, ps, [occ] * 64, [unk] * 64, True, args.reps)
    s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
