"""appendToPlan (faster.cpp:548, :606-648) restated in numpy over oracle/pyoracle.py's fillX, the restatement oracle/pair_oracle.py
uses: what one chained replan commits to the plan, from its records and its winners' coefficients.  Only tests/ import it."""
import numpy as np

from oracle import pyoracle as po

PLAN_OK, PLAN_NONE, PLAN_CAPACITY = 0, 1, 2                # FQ_PLAN_*


def piece(coeffs_w, dt_w, N_w, k_safe, coeffs_s, dt_s, N_s, DC, need_safe=True, fill_x=po.fill_x):
    """One corridor's piece: the whole winner's X_temp_[0 .. k_safe] (fillX with its full count), then the safe winner's
    whole X_temp_ (none when no safe path is needed)."""
    parts = [fill_x(N_w, coeffs_w, dt_w, DC)[:k_safe + 1]]
    if need_safe:
        parts.append(fill_x(N_s, coeffs_s, dt_s, DC))
    return np.vstack(parts)


def plan(rec, coeffs_w, coeffs_s, N_w, N_s, DC, need=None, cap=None, fill_x=po.fill_x):
    """Every corridor's piece as fq_replan_pairs_plan returns it.  rec: the result records (PAIR_RESULT_DTYPE, or a dict of
    their fields as arrays); coeffs_*: n x N x 12; need: needToComputeSafePath per corridor (None: always needed); cap:
    cap_states (None: the total).  -> (states (cap x 12, NaN where nothing is written), plan_ofs int64, status int32)."""
    n = len(rec["whole_dt_index"])
    pieces, status = [], np.full(n, PLAN_OK, np.int32)
    for j in range(n):
        nd = True if need is None else bool(need[j])
        if rec["whole_dt_index"][j] < 0 or (nd and rec["safe_dt_index"][j] < 0):
            pieces.append(np.zeros((0, 12)))
            status[j] = PLAN_NONE
            continue
        pieces.append(piece(coeffs_w[j], rec["whole_dt"][j], N_w, int(rec["k_safe"][j]), coeffs_s[j], rec["safe_dt"][j], N_s, DC, nd,
                            fill_x))
    ofs = np.concatenate([[0], np.cumsum([len(p) for p in pieces])]).astype(np.int64)
    cap = int(ofs[-1]) if cap is None else int(cap)
    states = np.full((cap, 12), np.nan)
    for j, p in enumerate(pieces):
        if len(p) and ofs[j + 1] > cap:
            status[j] = PLAN_CAPACITY
        elif len(p):
            states[ofs[j]:ofs[j + 1]] = p
    return states, ofs, status


def filled_rows(ofs, cap):
    """Rows of states that the corridors which fit fill: a prefix, up to the first FQ_PLAN_CAPACITY corridor."""
    return int(max(o for o in ofs if o <= cap))
