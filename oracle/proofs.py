"""TEST INFRASTRUCTURE ONLY -- solver-independent proofs on the LITERAL model of the reference (oracle/model_fullspace.py:
the reference's own 12N coefficient variables, every row as solverGurobi.cpp writes it).  Only tests/ and tools/ import it.

PARITY UNPINNED w.r.t. Gurobi (closed source, absent: SURVEY.md section 8c).  What these checks establish instead is that an
answer is THE answer of the reference's model, whichever solver produced it:

  * "solved" + coefficients z  ->  `prove_optimal`: z satisfies every equality and inequality row of the literal model
    (primal feasibility), and multipliers exist (mu free on the equality rows, lam >= 0 on the inequality rows that are
    tight at z) with  Q z + Aeq' mu + Ain' lam = 0  (stationarity).  For a convex QP these KKT conditions are sufficient:
    no feasible point has a smaller cost.  The multipliers are found here by a bounded least-squares fit -- they are a
    CERTIFICATE: once found, checking them needs no solver.  The cost of any feasible z' obeys
        f(z') >= f(z) - lam' slack(z) - |mu' (beq - Aeq z)| - |rho| |z' - z|,   rho = the stationarity residual,
    which is what `gap` and `resid` report.  The jerk part of the optimum is unique (the cost is strictly convex in it and
    the equality rows determine everything else), so Gurobi's GRB_OPTIMAL answer (solverGurobi.cpp:580-581) is this point
    up to its own tolerances.
  * "not solved"  ->  the Farkas certificate exported by the solver (fq_solve_batch_cert) checked on the literal rows:
    tests/test_certificates_gpu.py.
"""
import numpy as np
from scipy.optimize import lsq_linear


def prove_optimal(Q, Aeq, beq, Ain, bin_, z, active_tol=1e-7):
    """-> dict: eq (max |Aeq z - beq|), ineq (max row excess, <= 0 when strictly inside), n_active, resid (max |Q z + Aeq' mu +
    Ain' lam| relative to max(1, |Q z|_inf)), gap (lam' slack + |mu' eq residual|, relative to max(1, f)), lam_min."""
    z = np.asarray(z, float).reshape(-1)
    Qd = np.asarray(Q.todense()) if hasattr(Q, "todense") else np.asarray(Q)
    g = Qd @ z
    f = 0.5 * float(z @ g)
    req = Aeq @ z - beq
    slack = bin_ - Ain @ z
    act = np.flatnonzero(slack <= active_tol * np.maximum(1.0, np.abs(bin_)))
    M = np.hstack([Aeq.T, Ain[act].T]) if len(act) else Aeq.T
    # column scaling keeps the fit well conditioned (rows carry powers of dt); multipliers are rescaled afterwards
    cs = np.linalg.norm(M, axis=0)
    cs[cs == 0] = 1.0
    lo = np.concatenate([np.full(Aeq.shape[0], -np.inf), np.zeros(len(act))])
    sol = lsq_linear(M / cs, -g, bounds=(lo, np.full(M.shape[1], np.inf)), method="bvls", tol=1e-14, max_iter=4000)
    x = sol.x / cs
    x[Aeq.shape[0]:] = np.maximum(x[Aeq.shape[0]:], 0.0)     # the certificate's multipliers are non-negative by construction
    mu, lam = x[:Aeq.shape[0]], x[Aeq.shape[0]:]             # (the fit may leave -1e-17; the residual below is that of the clipped set)
    rho = g + M @ x
    return {
        "eq": float(np.abs(req).max()),
        "ineq": float(-slack.min()) if len(slack) else 0.0,
        "n_active": int(len(act)),
        "resid": float(np.abs(rho).max() / max(1.0, np.abs(g).max())),
        "gap": float((lam @ np.abs(slack[act]) if len(act) else 0.0) + abs(mu @ req)) / max(1.0, f),
        "lam_min": float(lam.min()) if len(lam) else 0.0,
        "lam_sum": float(lam.sum()),
        "active": act,
        "cost": f,
    }


def assert_optimal(model, z, cost=None, feas_tol=1e-7, resid_tol=1e-6, gap_tol=1e-7, active_tol=1e-7):
    """model = model_fullspace.build(...) ; z = coefficients [N,12] reported with a "solved" flag ; cost = reported cost.
    active_tol: rows with less relative slack may carry multipliers (any choice gives a valid bound; a smaller one keeps
    the fit off the slack twin of a nearly parallel tight row)."""
    Q, Aeq, beq, Ain, bin_ = model
    r = prove_optimal(Q, Aeq, beq, Ain, bin_, z, active_tol)
    assert r["eq"] <= feas_tol and r["ineq"] <= feas_tol, ("not feasible on the literal rows", r)
    assert r["lam_min"] >= 0.0
    assert r["resid"] <= resid_tol, ("no KKT multipliers: the point is not the optimum", r)
    assert r["gap"] <= gap_tol, r
    if cost is not None:
        assert abs(cost - r["cost"]) <= 1e-9 * max(1.0, abs(r["cost"])), (cost, r["cost"])
    return r


def literal_row_index(N, polys, sigma):
    """Row numbers of model_fullspace.build's inequality block for the row ids of fq_solve_batch_cert (include/faster_b200.h):
    box rows (typ, axis, t, s) and corridor rows (t, row of the packed Ab, control point k)."""
    face_ofs = np.concatenate([[0], np.cumsum([len(b) for _, b in polys])]).astype(int)
    box = {}
    r = 0
    for t in range(N):
        for ax in range(3):
            for typ in range(3):
                box[(typ, ax, t, 1)] = r
                box[(typ, ax, t, 0)] = r + 1
                r += 2
    cor = {}
    for t in range(N):
        p = int(sigma[t])
        F = len(polys[p][1])
        for k in range(4):
            for f in range(F):
                cor[(t, face_ofs[p] + f, k)] = r
                r += 1
    return box, cor, r


def assert_infeasible(model, N, polys, sigma, cert_row, resid_tol=1e-7, gap_max=-1e-9):
    """cert_row = one row of fq_solve_batch_cert's output for a candidate reported "not solved".  Checks the Farkas
    certificate on the literal rows: multipliers y >= 0 on the named inequality rows, free multipliers mu on the equality
    rows (least squares), sum y_k row_k + Aeq' mu = 0, y' bin + mu' beq < gap_max.  No point can satisfy rows that combine,
    with non-negative weights, to 0 <= negative.  gap_max = minus the row tolerance the solve ran at: a solver that refuses
    only violations beyond its tolerance leaves a gap below it.  -> the gap (negative)."""
    Q, Aeq, beq, Ain, bin_ = model
    n = int(cert_row[0])
    assert n >= 1, "infeasible candidate without certificate"
    box, cor, n_rows = literal_row_index(N, polys, sigma)
    assert n_rows == len(bin_)
    y = np.zeros(len(bin_))
    for k in range(n):
        rid, mult = int(round(cert_row[2 + 2 * k])), cert_row[3 + 2 * k]
        assert mult >= -1e-12
        if rid >= 10000000:
            rid -= 10000000
            typ, rem = divmod(rid, 10000); ax, rem = divmod(rem, 1000); t, s = divmod(rem, 10)
            y[box[(typ, ax, t, s)]] += mult
        else:
            t, rem = divmod(rid, 100000); f, kcp = divmod(rem, 10)
            y[cor[(t, f, kcp)]] += mult
    g = Ain.T @ y                                      # must vanish modulo the equality rows
    mu, *_ = np.linalg.lstsq(Aeq.T, -g, rcond=None)
    resid = np.abs(g + Aeq.T @ mu).max()
    scale = max(1.0, np.abs(g).max())
    assert resid <= resid_tol * scale, (resid, scale)
    gap = float(bin_ @ y + beq @ mu)                   # < 0: the rows cannot hold together
    assert gap < gap_max, (gap, gap_max)
    assert abs(gap + cert_row[1]) <= 1e-6 * max(1.0, abs(gap)), (gap, cert_row[1])   # = minus the violation the solver saw
    return gap
