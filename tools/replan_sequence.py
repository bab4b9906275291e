"""Consecutive chained replans with per-corridor time-allocation windows, two ways:
  device  every step is one fq_replan_pairs_window_dev call on one stream, its next windows written over the window arrays it
          read (aliased), with no host synchronisation between the steps;
  host    every step is one fq_replan_pairs_window call; the host reads the result records back and computes the next windows
          in Python (faster.cpp:582-588 over the factors genNewTraj's loop visits).
The corridors are the config-4 forest fixture (bench_data/cfg4_forest.npz), rotated by one corridor per step, so every
corridor slot meets new corridors and the windows really differ.  The records of every step and the final windows of the two
ways must be identical, byte for byte.  Prints one JSON line with replans/s of both ways, the card's name and its power limit.

    python tools/replan_sequence.py [--corridors 64] [--steps 8] [--reps 5] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from faster_b200 import capi  # noqa: E402

KEYS = ("init_whole", "final_whole", "init_safe", "final_safe")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                                          # report what could not be read, never guess it
        return dict(gpu="unknown (%s)" % e, power_limit="unknown", max_sm_clock="unknown")


def next_windows(rec, win, inc, gamma):
    """faster.cpp:582-588 in Python: both sweeps won -> [max(f* - gamma, 1), f* + gammap], else unchanged."""
    out = {k: v.copy() for k, v in win.items()}
    for j in range(len(rec)):
        dw, ds = int(rec["whole_dt_index"][j]), int(rec["safe_dt_index"][j])
        if dw < 0 or ds < 0:
            continue
        fw = capi.window_factors(win["init_whole"][j], win["final_whole"][j], inc)[dw]
        fs = capi.window_factors(win["init_safe"][j], win["final_safe"][j], inc)[ds]
        out["init_whole"][j], out["final_whole"][j] = max(fw - gamma, 1.0), fw + gamma
        out["init_safe"][j], out["final_safe"][j] = max(fs - gamma, 1.0), fs + gamma
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corridors", type=int, default=64)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--gamma", type=float, default=20.0, help="gamma = gammap of both sweeps (faster.yaml)")
    ap.add_argument("--inc", type=float, default=1.0, help="increment of both sweeps (faster.yaml)")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    n, K, inc, gamma = args.corridors, args.steps, args.inc, args.gamma
    ws = [bench.load_cfg4(k, n) for k in range(K)]
    for w in ws:
        w["factors_whole"] = w["factors_safe"] = np.zeros(0)
    first = {k: np.full(n, 1.0 if k.startswith("init") else 10.0) for k in KEYS}      # setFactorInitialAndFinalAndIncrement(1, 10, inc)
    # capacities of the device way: the longest list of each sweep x the largest window any step can have
    mp = [(int(np.diff(w["poly_ofs_whole"]).max()), int(np.diff(w["poly_ofs_safe"]).max())) for w in ws]
    mpw, mps = max(m[0] for m in mp), max(m[1] for m in mp)
    max_fac = max(len(capi.window_factors(1.0, 10.0, inc)), len(capi.window_factors(1.0, 1.0 + 2 * gamma, inc)))
    cap_w = n * max_fac * capi.assign_count(10, mpw, 0)
    cap_s = n * max_fac * capi.assign_count(10, mps, 0)
    s = capi.Solver(0)
    d_in = [{k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith(("sigmas_", "factors_"))}
            for w in ws]
    d_res = torch.zeros((K, n * 144), dtype=torch.uint8, device=dev)
    d_win = {k: torch.zeros(n, dtype=torch.float64, device=dev) for k in KEYS}
    d_hist = torch.zeros((K, 4, n), dtype=torch.float64, device=dev)
    st = torch.cuda.Stream(device=dev)
    calls = []
    for k, w in enumerate(ws):
        a = capi.pair_args(w, lambda key, k=k: None if key.startswith(("sigmas_", "factors_")) else d_in[k][key].data_ptr(),
                           {"results": d_res[k].data_ptr()})
        a.n_sig_whole = a.n_sig_safe = a.n_fac_whole = a.n_fac_safe = 0
        sa = capi.assign_args(0, {}, mpw, mps, cap_w, cap_s)
        wa = capi.window_args(lambda key: d_win[key].data_ptr(), {"next_" + key: d_win[key].data_ptr() for key in KEYS}, inc, gamma,
                              max_fac, max_fac)
        calls.append((a, sa, wa))

    def device_way():
        for key in KEYS:
            d_win[key].copy_(torch.from_numpy(first[key]))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.cuda.stream(st):
            for k, (a, sa, wa) in enumerate(calls):
                s.replan_pairs_window_dev(a, sa, wa, 0, st.cuda_stream)
                for i, key in enumerate(KEYS):                     # the windows after each step, for the comparison only
                    d_hist[k, i].copy_(d_win[key])
        st.synchronize()
        dt = time.perf_counter() - t0
        rec = np.frombuffer(d_res.cpu().numpy().tobytes(), capi.PAIR_RESULT_DTYPE).reshape(K, n)
        return dt, rec, d_hist.cpu().numpy()

    def host_way():
        win = {k: v.copy() for k, v in first.items()}
        recs, hist = [], []
        t0 = time.perf_counter()
        for w in ws:
            r = s.replan_pairs_window(w, win, all_limit=0, inc=inc, gamma=gamma, want_candidates=False, want_coeffs=False)["results"]
            win = next_windows(r, win, inc, gamma)
            recs.append(r)
            hist.append(np.stack([win[k] for k in KEYS]))
        return time.perf_counter() - t0, np.stack(recs), np.stack(hist)
    _, rd, hd = device_way()
    _, rh, hh = host_way()
    same = rd.tobytes() == rh.tobytes() and hd.tobytes() == hh.tobytes()
    moved = int((hh[-1] != np.stack([first[k] for k in KEYS])).sum())
    for _ in range(args.warmup):
        device_way(); host_way()
    t_dev, t_host = [], []
    for _ in range(args.reps):                                       # alternate the two ways
        t_dev.append(device_way()[0])
        t_host.append(host_way()[0])
    s.close()
    m1, m2 = float(np.median(t_dev)), float(np.median(t_host))
    out = dict(metric="replan_sequence", corridors=n, steps=K, inc=inc, gamma=gamma, max_factors=max_fac, records_identical=bool(same),
               window_entries_moved=moved, whole_winners=int((rh["whole_dt_index"] >= 0).sum()), both_winners=int(((rh["whole_dt_index"] >= 0) &
               (rh["safe_dt_index"] >= 0)).sum()), device_replans_per_s=n * K / m1, host_replans_per_s=n * K / m2,
               device_ms_median=1e3 * m1, host_ms_median=1e3 * m2, device_ms_minmax=[1e3 * min(t_dev), 1e3 * max(t_dev)],
               host_ms_minmax=[1e3 * min(t_host), 1e3 * max(t_host)], speedup=m2 / m1, **card())
    print(json.dumps(out))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
