"""TEST INFRASTRUCTURE ONLY -- the chained replan with per-corridor time-allocation windows (fq_replan_pairs_window*),
restated on the CPU: genNewTraj's factor loop (solverGurobi.cpp:445-446) and the next-window rule of Faster::replan
(faster.cpp:582-588) in plain Python, and the chain run corridor by corridor through tests/pair_assign_oracle.py with the
corridor's own factors F_j (the corridors of a batch are independent, so one corridor is the whole definition)."""
import math

import numpy as np

from faster_b200 import capi

import pair_assign_oracle as pao

MAX_FACTORS = 4096
WINDOW_KEYS = ("init_whole", "final_whole", "init_safe", "final_safe")


def factors(fi, ff, inc):
    """`for (double i = fi; i <= ff; i = i + inc)`'s values, or None where the library refuses the window."""
    if not all(math.isfinite(v) for v in (fi, ff, inc)) or not fi > 0 or not inc > 0:
        return None
    out, i = [], float(fi)
    while i <= ff:
        if len(out) == MAX_FACTORS:
            return None
        out.append(i)
        if i + inc == i:
            return None
        i = i + inc
    return np.array(out, np.float64)


def next_window(both_won, f_star, gamma, gammap, init, final):
    """faster.cpp:582-588 when both sweeps won; replan() returns before it otherwise (:420-424, :529-533)."""
    if not both_won:
        return init, final
    return max(f_star - gamma, 1.0), f_star + gammap


def _pair(x):
    return (x, x) if np.isscalar(x) else tuple(x)


def _gammas(g):
    return (g,) * 4 if np.isscalar(g) else tuple(g)


def window_outputs(res, windows, Fw, Fs, gamma):
    """factor_*, trials_* and the next windows from result records and the corridors' factor lists."""
    g = _gammas(gamma)
    n = len(res["whole_dt_index"])
    out = {k: np.zeros(n) for k in ("factor_whole", "factor_safe", "next_init_whole", "next_final_whole", "next_init_safe", "next_final_safe")}
    out["trials_whole"], out["trials_safe"] = np.zeros(n, np.int32), np.zeros(n, np.int32)
    for j in range(n):
        dw, ds = int(res["whole_dt_index"][j]), int(res["safe_dt_index"][j])
        fw = Fw[j][dw] if dw >= 0 else np.nan
        fs = Fs[j][ds] if ds >= 0 else np.nan
        out["factor_whole"][j], out["factor_safe"][j] = fw, fs
        out["trials_whole"][j] = dw + 1 if dw >= 0 else len(Fw[j])
        out["trials_safe"][j] = 0 if dw < 0 else (ds + 1 if ds >= 0 else len(Fs[j]))
        both = dw >= 0 and ds >= 0
        out["next_init_whole"][j], out["next_final_whole"][j] = next_window(both, fw, g[0], g[1], windows["init_whole"][j], windows["final_whole"][j])
        out["next_init_safe"][j], out["next_final_safe"][j] = next_window(both, fs, g[2], g[3], windows["init_safe"][j], windows["final_safe"][j])
    return out


def replan_pairs_window(w, windows, all_limit, inc=1.0, gamma=20.0, threads=4, dt_base_whole=None, dt_base_safe=None):
    """The CPU chain with per-corridor lists and windows -> the fields of oracle.pair_oracle.replan_pairs (per-candidate
    arrays concatenated in corridor order), cand_ofs_*, and the window outputs of window_outputs."""
    from oracle import pair_oracle, pyoracle
    iw, is_ = _pair(inc)
    n = w["n_prob"]
    Fw = [factors(windows["init_whole"][j], windows["final_whole"][j], iw) for j in range(n)]
    Fs = [factors(windows["init_safe"][j], windows["final_safe"][j], is_) for j in range(n)]
    assert all(f is not None for f in Fw + Fs), "a window is refused"
    per = []
    for j in range(n):
        w1 = pao.with_own_lists(pao.corridor(w, j), all_limit)
        Lw, Ls = len(w1["sigmas_whole"]), len(w1["sigmas_safe"])
        dbw = None if dt_base_whole is None else dt_base_whole[j:j + 1]
        dbs = None if dt_base_safe is None else dt_base_safe[j:j + 1]
        if len(Fw[j]) == 0:                    # no whole candidate: nothing is solved in either sweep
            own = max(pyoracle.dt_initial(w1["x0"][0], w1["xf_whole"][0], w1["lim"][0], w1["N_whole"]), 2 * w1["DC"])
            o = dict(whole_dt_index=[-1], whole_sigma_index=[-1], safe_dt_index=[-1], safe_sigma_index=[-1], whole_cost=[np.inf],
                     safe_cost=[np.inf], whole_dt=[np.nan], safe_dt=[np.nan], whole_dt_base=[own if dbw is None else dbw[0]],
                     safe_dt_base=[np.nan], n_samples_whole=[0], k_safe=[-1], R=np.full((1, 9), np.nan),
                     feasible_whole=np.zeros(0, np.uint8), cost_whole=np.zeros(0), feasible_safe=np.zeros(len(Fs[j]) * Ls, np.uint8),
                     cost_safe=np.full(len(Fs[j]) * Ls, np.inf), coeffs_whole=np.zeros((1, w["N_whole"], 12)),
                     coeffs_safe=np.zeros((1, w["N_safe"], 12)), whole_dt_base_own=[own], safe_dt_base_own=[np.nan])
            o = {k: np.asarray(v) for k, v in o.items()}
        else:
            w1["factors_whole"] = Fw[j]
            w1["factors_safe"] = Fs[j] if len(Fs[j]) else np.ones(1)
            o = pair_oracle.replan_pairs(w1, threads=threads, dt_base_whole=dbw, dt_base_safe=dbs)
            if len(Fs[j]) == 0:                # no safe candidate: the stand-in factor above is dropped again
                o.update(safe_dt_index=np.array([-1], np.int32), safe_sigma_index=np.array([-1], np.int32), safe_cost=np.array([np.inf]),
                         safe_dt=np.array([np.nan]), feasible_safe=np.zeros(0, np.uint8), cost_safe=np.zeros(0),
                         coeffs_safe=np.zeros((1, w["N_safe"], 12)))
        assert len(o["feasible_whole"]) == len(Fw[j]) * Lw and len(o["feasible_safe"]) == len(Fs[j]) * Ls
        per.append(o)
    out = {k: np.concatenate([p[k] for p in per]) for k in per[0]}
    for kind, F in (("whole", Fw), ("safe", Fs)):
        counts = [len(f) for f in F]
        out["cand_ofs_" + kind] = capi.window_offsets(w["poly_ofs_" + kind], w["N_" + kind], counts, all_limit)
    res = {k: out[k] for k in ("whole_dt_index", "safe_dt_index")}
    out.update(window_outputs(res, windows, Fw, Fs, gamma))
    out["F_whole"], out["F_safe"] = Fw, Fs
    return out
