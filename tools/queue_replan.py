"""Times the closed replan loop of a batch planner with its committed plans kept on the device against the same loop with
the plans in host deques, on one GPU, and asserts that both routes compute the same bytes.

The loop is tests/queue_loop.py's: --n forest planners on indexed maps (one map each), the _map chain with windows and
H/R.  Per cycle:
  device: fq_queue_select_dev, x0 read back, host JPS from A and fq_jps_in, JPS_in uploaded, fq_map_paths_dev,
          fq_replan_pairs_queue_dev, fq_queue_pop_dev (--ticks publications), one stream synchronise;
  host:   choosing A from Python deques, host JPS from A and fq_jps_in, fq_map_paths, the _plan host entry (x0 uploaded,
          every piece copied back), appendToPlan on the deques, the window rule gated by the append, --ticks publications.
Both routes run the same host JPS; the maps are not updated between cycles.  The two routes alternate; the medians of
the per-cycle times (host clock) are reported with the card's name and power limit, and the median time of the host JPS
and fq_jps_in step alone.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from faster_b200 import capi  # noqa: E402

import plan_queue_oracle as pqo  # noqa: E402
import queue_loop as ql  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--cycles", type=int, default=8)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--ticks", type=int, default=3)
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    solver = capi.Solver()
    pl = ql.planners(args.n)
    n = len(pl)
    st = torch.cuda.Stream(device=dev)
    dv = ql.DeviceRoute(solver, pl, np.arange(n, dtype=np.int32), torch, dev, st)
    host = ql.HostRoute(solver, pl, dv.maps)
    w0 = ql.windows0(n)
    ticks = np.full(n, args.ticks, np.int32)
    jps_t = []

    def device_run():
        times, snaps = [], []
        with torch.cuda.stream(st):
            dv.reset(w0)
            dv.ticks.copy_(torch.from_numpy(ticks))
            st.synchronize()
            for _ in range(args.cycles):
                t = time.perf_counter()
                dv.select()
                x0 = dv.read_x0()
                t1 = time.perf_counter()
                jins, ok = ql.jps_inputs(pl, x0)
                jps_t.append(time.perf_counter() - t1)
                dv.upload(jins, ok)
                dv.replan()
                dv.pop()
                st.synchronize()
                times.append(time.perf_counter() - t)
                snaps.append(dv.snap())
        return times, snaps

    def host_run():
        host.reset(w0)
        times, outs = [], []
        for _ in range(args.cycles):
            t = time.perf_counter()
            x0, k_end = host.select()
            jins, ok = ql.jps_inputs(pl, x0)
            k_end[~ok] = -1
            r = host.replan(x0, k_end, jins)
            goals = host.pop(ticks)
            times.append(time.perf_counter() - t)
            outs.append(dict(results=r["ref"]["results"], status=r["status"], plans=[np.array(p) for p in host.plans], goals=goals,
                             wins={k: v.copy() for k, v in host.wins.items()}))
        return times, outs

    device_run(), host_run()                                 # warm-up: module loads, scratch, staging
    jps_t.clear()
    dev_t, host_t = [], []
    for _ in range(args.reps):
        t, snaps = device_run()
        dev_t += t
        t, outs = host_run()
        host_t += t
    for h, o in zip(snaps, outs):                            # the last repetition of each route: identical bytes
        assert h["results"].tobytes() == o["results"].tobytes() and h["status"].tobytes() == o["status"].tobytes()
        for j in range(n):
            assert np.array(dv.plan(j, h)).tobytes() == o["plans"][j].tobytes(), j
            assert h["goals"][j, :args.ticks].tobytes() == o["goals"][j].tobytes(), j
        for k in capi.WINDOW_IN_KEYS:
            assert h["win_" + k].tobytes() == o["wins"][k].tobytes(), k
    st_all = np.concatenate([o["status"] for o in outs])
    names = {pqo.QUEUE_OK: "ok", pqo.QUEUE_NONE: "none", pqo.QUEUE_PUBLISHED: "published", pqo.QUEUE_CAPACITY: "capacity"}
    print(json.dumps(dict(card=card(), n=n, cycles=args.cycles, reps=args.reps, ticks=args.ticks,
                          device_cycle_ms=1e3 * float(np.median(dev_t)), host_cycle_ms=1e3 * float(np.median(host_t)),
                          jps_step_ms=1e3 * float(np.median(jps_t)),
                          statuses={names.get(int(s), str(s)): int((st_all == s).sum()) for s in np.unique(st_all)}, identical=True)))


if __name__ == "__main__":
    main()
