"""Times every planner's JPS step on the device (fq_jps_batch_dev) against the host JPS step it replaces, and the replan
loop without a host step against tools/queue_replan.py's device route, on one GPU; asserts identical outputs.

  kernel:  fq_jps_batch_dev alone on --n forest planners (CUDA events), per-planner grids and one shared grid;
  host:    the host JPS step as queue_replan.py runs it (queue_loop.jps_inputs, serial) and the same over a 16-thread
           pool (ctypes releases the GIL);
  loop:    per-cycle time of select_dev, jps_batch_dev, map_paths_dev, _queue_dev, pop_dev with one synchronise, eager and
           as a replayed CUDA graph, against the device route with x0 read back and host JPS.
Variants alternate; medians are reported with the card's name and power limit read in the same run.  One JSON line."""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from faster_b200 import capi  # noqa: E402

import jps_batch_oracle as jbo  # noqa: E402
import queue_loop as ql  # noqa: E402
from queue_replan import card  # noqa: E402
from test_jps_batch_gpu import DeviceJpsRoute  # noqa: E402


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
    rows = np.arange(n, dtype=np.int32)
    dj = DeviceJpsRoute(solver, pl, rows, torch, dev, st)
    dr = ql.DeviceRoute(solver, pl, rows, torch, dev, st)
    w0 = ql.windows0(n)
    ticks = np.full(n, args.ticks, np.int32)
    x0 = np.array([np.concatenate([p["start"], np.zeros(6)]) for p in pl])
    grids = [(p["grid"], p["origin"], p["res"]) for p in pl]

    # ---- the kernel alone, per-planner grids and one shared grid, against the oracle
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    kern = {}
    for name, gl, gi in (("per_planner", grids, np.arange(n, dtype=np.int32)), ("shared", grids[:1], None)):
        gd = {k: T(v) for k, v in capi.jps_grids(gl).items()}
        out = dict(in_ofs=torch.zeros(n + 1, dtype=torch.int32, device=dev), status=torch.zeros(n, dtype=torch.int32, device=dev),
                   **{"in": torch.zeros((n * ql.MAX_IN, 3), dtype=torch.float64, device=dev)})
        dx0, dgi = T(x0), None if gi is None else T(gi)      # kept alive: the struct holds their addresses only
        a = capi.jps_batch_args(n, gd, dx0, dj.G, out, dgi, None, ql.RA, ql.DIST_MAX, True, capi.JPS_MAX_NODES, ql.MAX_IN)
        kern[name] = (a, out, gd, gl, gi, dx0, dgi)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    kern_t = {k: [] for k in kern}
    for rep in range(args.reps + 1):
        for name, (a, out, *_rest) in kern.items():
            with torch.cuda.stream(st):
                ev[0].record(st)
                capi.jps_batch_dev(a, st.cuda_stream)
                ev[1].record(st)
            st.synchronize()
            if rep:
                kern_t[name].append(ev[0].elapsed_time(ev[1]))
    for name, (a, out, gd, gl, gi, *_keep) in kern.items():
        want = jbo.batch(gl, x0, np.array([p["goal"] for p in pl]), grid_index=gi, Ra=ql.RA, dist_max=ql.DIST_MAX, max_in=ql.MAX_IN)
        jbo.assert_equal({k: v.cpu().numpy() for k, v in out.items()}, want, name)

    # ---- the host JPS step, serial and over 16 threads
    pool = ThreadPoolExecutor(16)

    def host_step(threaded):
        if not threaded:
            return ql.jps_inputs(pl, x0)
        parts = list(pool.map(lambda j: ql.jps_inputs([pl[j]], x0[j:j + 1]), range(n)))
        return [p[0][0] for p in parts], np.array([p[1][0] for p in parts])
    host_t = {False: [], True: []}
    for rep in range(args.reps + 1):
        for thr in (False, True):
            t = time.perf_counter()
            jins, ok = host_step(thr)
            if rep:
                host_t[thr].append(time.perf_counter() - t)
    ref_jins, ref_ok = host_step(False)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(jins, ref_jins)) and (ok == ref_ok).all()

    # ---- the loop: device JPS eager, device JPS as a graph, host JPS (queue_replan.py's device route)
    with torch.cuda.stream(st):
        dj.reset(w0)
        dj.ticks.copy_(torch.from_numpy(ticks))
        dj.cycle()                                           # sizes the context's arenas: a capture cannot grow them
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        dj.cycle()

    def run(kind):
        times, snaps = [], []
        r = dr if kind == "host_jps" else dj
        with torch.cuda.stream(st):
            r.reset(w0)
            r.ticks.copy_(torch.from_numpy(ticks))
            st.synchronize()
            for _ in range(args.cycles):
                t = time.perf_counter()
                if kind == "host_jps":
                    r.select()
                    jins, ok = ql.jps_inputs(pl, r.read_x0())
                    r.upload(jins, ok)
                    r.replan()
                    r.pop()
                elif kind == "eager":
                    r.cycle()
                else:
                    g.replay()
                st.synchronize()
                times.append(time.perf_counter() - t)
                snaps.append(r.snap())
        return times, snaps
    loop_t = {k: [] for k in ("eager", "graph", "host_jps")}
    for rep in range(args.reps + 1):
        last = {}
        for k in loop_t:
            t, last[k] = run(k)
            if rep:
                loop_t[k] += t
    for a, b in zip(last["eager"], last["graph"]):
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
    med = lambda v: float(np.median(v))  # noqa: E731
    st_dev = last["eager"][-1]["status"]
    print(json.dumps(dict(card=card(), n=n, cycles=args.cycles, reps=args.reps, ticks=args.ticks,
                          kernel_ms={k: med(v) for k, v in kern_t.items()},
                          host_jps_serial_ms=1e3 * med(host_t[False]), host_jps_16_threads_ms=1e3 * med(host_t[True]),
                          cycle_ms={k: 1e3 * med(v) for k, v in loop_t.items()},
                          queue_status_last_cycle={str(int(s)): int((st_dev == s).sum()) for s in np.unique(st_dev)}, identical=True)))


if __name__ == "__main__":
    main()
