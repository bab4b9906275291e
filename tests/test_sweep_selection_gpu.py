"""genNewTraj's selection (solverGurobi.cpp:445-472: first time allocation with a feasible assignment, then the minimum
cost, then the lowest assignment index) on its three device paths, against a numpy restatement over the full
per-candidate arrays:
  - sweep_tail_select: fq_gen_new_traj on the specialised kernel, selected by the warp that finishes the last candidate;
  - fq_select_kernel: fq_gen_new_traj_sampled, and fq_gen_new_traj with the size-generic kernel forced;
  - fq_select_multi_kernel: fq_solve_multi_sharded (and fq_replan_pairs).
And the early exit (option "sweep_early_exit"), which must leave every sweep's winner record unchanged."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

pytestmark = pytest.mark.gpu


def _select(feas, cost, n_dt, n_sigma):
    """numpy restatement -> (dt index, sigma index), (-1, -1) when nothing is feasible."""
    f = feas.reshape(n_dt, n_sigma).astype(bool)
    rows = np.flatnonzero(f.any(axis=1))
    if not len(rows):
        return -1, -1
    d = int(rows[0])
    c = np.where(f[d], cost.reshape(n_dt, n_sigma)[d], np.inf)
    return d, int(np.flatnonzero(c == c.min())[0])


def _sweep_args(pb):
    P, fo, Ab = capi.pack_polys(pb["polys"])
    return P, fo, Ab


def _sharded(solver, N, ff, pb, dts, sig):
    """One problem through fq_solve_multi_sharded (a world of one): the candidates dt-major, as the sweeps lay them out."""
    P, fo, Ab = capi.pack_polys(pb["polys"])
    n = len(dts) * len(sig)
    return solver.solve_multi_sharded(N, ff, np.ascontiguousarray([pb["x0"]]), np.ascontiguousarray([pb["xf"]]),
                                      np.ascontiguousarray([pb["lim"]]), np.array([0, P], np.int32), fo, Ab,
                                      np.array([0, n], np.int32), np.ascontiguousarray(np.repeat(dts, len(sig))),
                                      np.ascontiguousarray(np.tile(sig, (len(dts), 1))))


def _with_ties(mono, n_sigma, rng):
    """n_sigma assignment rows in which every row of the first half appears again in the second half (exact cost ties),
    second copies in shuffled order."""
    k = max(1, (n_sigma + 1) // 2)
    N, P = mono.shape[1], int(mono.max()) + 1
    even = (np.arange(N) * P // N).astype(np.uint8)               # even split over the polytopes: feasible for a loose dt
    uniq = np.vstack([even, mono[rng.choice(len(mono), k - 1, replace=len(mono) < k - 1)]])[rng.permutation(k)]
    return np.ascontiguousarray(np.vstack([uniq, uniq[rng.permutation(k)]])[:n_sigma])


@pytest.mark.parametrize("n_sigma", [1, 31, 33, 300])
def test_three_selection_paths_agree_with_the_restatement(solver, n_sigma):
    """Duplicate assignment rows give bit-identical costs: the lowest index must win.  n_sigma = 1, 31 / 33 (around a
    warp), 300 (beyond fq_select_kernel's 256-thread stride).  The winner record is bit-identical across the paths."""
    N, P, ff = 10, 4, True
    rng = np.random.default_rng(n_sigma)
    mono = cr.monotone_sigmas(N, P)
    n_win = 0
    for seed in range(3):
        pb = cr.make_corridor(64000 + seed, P, N, "uav", ff)
        sig = _with_ties(mono, n_sigma, rng)
        dts = np.array([0.6, 1.0, 1.5, 2.0, 3.0, 5.0]) * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        recs = {}
        for generic in (0, 1):
            solver.set_option("force_generic_kernel", generic)
            f, c, co, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.repeat(dts, n_sigma),
                                             np.tile(sig, (len(dts), 1)), ff, True)
            d, s = _select(f, c, len(dts), n_sigma)
            g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, ff)
            assert (g["dt_index"], g["sigma_index"]) == (d, s), (generic, seed)
            if d >= 0:
                k = d * n_sigma + s
                assert g["cost"] == c[k] and g["coeffs"].tobytes() == co[k].tobytes()
            recs[generic] = (g, f, c, co, d, s)
        solver.set_option("force_generic_kernel", 0)
        g, f, c, co, d, s = recs[0]
        h = solver.gen_new_traj_sampled(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, 0.01, ff)
        fm, cm, wi, wc = _sharded(solver, N, ff, pb, dts, sig)
        assert np.array_equal(fm, f) and cm.tobytes() == c.tobytes()
        assert (h["dt_index"], h["sigma_index"]) == (d, s)
        assert wi[0] == (d * n_sigma + s if d >= 0 else -1)
        if d < 0:
            assert np.isinf(g["cost"]) and np.isinf(h["cost"]) and np.isinf(wc[0])
            continue
        n_win += 1
        k = d * n_sigma + s
        assert h["cost"] == g["cost"] == wc[0] == c[k] and h["coeffs"].tobytes() == g["coeffs"].tobytes()
        if n_sigma > 1:
            # the winner's row has a later copy with the same cost bits: only the lowest index may win
            same = np.flatnonzero((sig == sig[s]).all(axis=1))
            assert len(same) >= 2 and s == same[0] and (c[d * n_sigma + same] == c[k]).all()
    assert n_win >= 2


def test_all_infeasible_sweep(solver):
    """No feasible candidate: index -1 and +inf cost on every path."""
    N, P = 10, 3
    pb = cr.make_corridor(64100, P, N, "uav", True)
    sig = cr.monotone_sigmas(N, P)
    dts = np.array([0.02, 0.03, 0.05])
    f, _, _, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.repeat(dts, len(sig)), np.tile(sig, (3, 1)))
    assert not f.any()
    for generic in (0, 1):
        solver.set_option("force_generic_kernel", generic)
        g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, True)
        assert not g["solved"] and g["dt_index"] == -1 and np.isinf(g["cost"])
    solver.set_option("force_generic_kernel", 0)
    h = solver.gen_new_traj_sampled(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, 0.01, True)
    assert not h["solved"] and h["dt_index"] == -1 and np.isinf(h["cost"]) and len(h["X"]) == 0
    _, _, wi, wc = _sharded(solver, N, True, pb, dts, sig)
    assert wi[0] == -1 and np.isinf(wc[0])


def _record(g):
    return (g["dt_index"], g.get("sigma_index"), np.float64(g["cost"]).tobytes(), g["coeffs"].tobytes(),
            g["sigma"].tobytes() if "sigma" in g else None, g["X"].tobytes() if "X" in g else None)


def _big_sweep(seed=64200):
    """N = 10, 6 polytopes: 3003 non-decreasing assignments plus 3000 arbitrary ones per time allocation -- far more
    candidates than the H100's resident warps (132 SMs x 4 CTAs x 4 warps)."""
    N, P = 10, 6
    pb = cr.make_corridor(seed, P, N, "uav", True)
    rng = np.random.default_rng(seed)
    sig = np.vstack([cr.monotone_sigmas(N, P), rng.integers(0, P, (3000, N)).astype(np.uint8)])
    base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
    return N, pb, sig, base


def test_early_exit_on_a_large_ascending_sweep(solver):
    """More candidates than twice the resident warps: the capped grid and the "take the rest at once" path of the early
    exit.  The in-kernel selection still runs (the host refuses a sweep that finished without it) and the winner record is
    bit-identical to the full evaluation; the chained replan's per-candidate arrays are complete up to the winner."""
    N, pb, sig, base = _big_sweep()
    facs = np.linspace(0.4, 8.0, 40)
    s2 = capi.Solver(0)
    try:
        s2.set_option("sweep_early_exit", 1)
        full = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], facs * base, sig[:600], True)
        assert 0 < full["dt_index"] < len(facs) - 1
        for _ in range(2):
            ee = s2.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], facs * base, sig[:600], True)
            assert _record(ee) == _record(full)
        w = capi.make_pair_workload([pb], [cr.make_corridor(64201, 4, N, "uav", False)], facs, sig[:600], facs[:8],
                                    cr.monotone_sigmas(N, 4)[:64], DC=0.01, r_fraction=0.3)
        a, b = solver.replan_pairs(w), s2.replan_pairs(w)
        assert a["results"].tobytes() == b["results"].tobytes()
        d = int(a["results"]["whole_dt_index"][0])
        assert d == full["dt_index"]
        upto = (d + 1) * 600
        assert np.array_equal(a["feasible_whole"][:upto], b["feasible_whole"][:upto])
        assert a["cost_whole"][:upto].tobytes() == b["cost_whole"][:upto].tobytes()
        assert b["feasible_whole"].sum() < a["feasible_whole"].sum()            # work was skipped
    finally:
        s2.close()


@pytest.mark.parametrize("order", ["descending", "shuffled"])
def test_early_exit_keeps_the_winner_of_a_non_ascending_sweep(solver, order):
    """The early exit skips a candidate whose dt exceeds the smallest dt already found feasible; the sweeps' selection
    takes the first dt INDEX with a feasible assignment.  For a dt list that is not ascending the two disagree, so the
    early exit must not change what fq_gen_new_traj, fq_gen_new_traj_sampled and fq_gen_new_traj_exact return.  The
    lowest-cost assignments of the first time allocation are put last in the list, where a skip would hit them."""
    N, pb, sig, base = _big_sweep()
    facs = np.array([8.0, 6.0, 5.0, 4.0, 3.0, 2.5, 2.0, 1.5])
    if order == "shuffled":
        facs = facs[[2, 6, 0, 7, 4, 1, 5, 3]]
    dts = facs * base
    f, c, _, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.full(len(sig), dts[0]), sig)
    assert f.sum() > 10
    c = np.where(f.astype(bool), c, np.inf)
    best = c == c.min()                          # exact ties: assignments whose corridor rows do not bind at the optimum
    sig = np.ascontiguousarray(np.vstack([sig[~best], sig[best]]))
    s2 = capi.Solver(0)
    try:
        s2.set_option("sweep_early_exit", 1)
        full = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, True)
        assert full["dt_index"] == 0 and full["sigma_index"] == len(sig) - int(best.sum())
        fs = solver.gen_new_traj_sampled(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, 0.01, True)
        assert _record(fs)[:4] == _record(full)[:4]
        for _ in range(6):
            assert _record(s2.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, True)) == _record(full)
            assert _record(s2.gen_new_traj_sampled(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, 0.01, True)) == _record(fs)
        # the exact sweep's monotone pre-sweep (3003 assignments per time allocation) sets its incumbent and search range
        xf_ = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, True)
        assert xf_["solved"] and xf_["dt_index"] == 0
        for _ in range(6):
            xe = s2.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, True)
            assert _record(xe) == _record(xf_) and xe["exact"] == xf_["exact"]
    finally:
        s2.close()
