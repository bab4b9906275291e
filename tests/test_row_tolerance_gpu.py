"""The run-time row tolerance (fq_set_option "row_tol_1e9") on every solve path, against the CPU restatement run at the same
tolerance (oracle.set_row_tol).

Ordinary corridors cannot show whether a path honours the option: their flags are the same at 1e-9 as at 1e-3.  The probes
below therefore move one row that the inputs alone fix (no rounding of the solve can change it) to a known violation
DELTA = 3e-7, above 1e-8 and below 1e-6:
  * "velocity": v_max is set DELTA below the largest |x0| velocity component (the box row at t = 0);
  * "x0_face": in every polytope that holds x0, the face the start velocity points away from is moved so that
    A.x0 - b = DELTA (control point 0 of segment 0, for every assignment);
  * "xf_face" (final position pinned): in every polytope that holds xf, the face beyond the goal is moved so that
    A.xf - b = DELTA (the last control point, for every assignment).
The probed candidates must be infeasible at 1e-9 and 1e-8 and some of them feasible at 1e-6 and 1e-3; a path that ignores
the option fails one of the two."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr
from shape_cases import SHAPES, probe, shape_batches
from test_parity_gpu import REL, _compare

pytestmark = pytest.mark.gpu

TOLS = (1, 10, 1000, 1000000)                       # row_tol_1e9: 1e-9, the default 1e-8, Gurobi's 1e-6, 1e-3
FACTORS = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])


def probe_corridors(N, ff, kind, n=2):
    """n probed corridors of 3 polytopes (UAV limits) whose start speed is large enough for the velocity probe."""
    out = []
    for seed in range(71000, 71100):
        pb = cr.make_corridor(seed, 3, N, "uav", ff)
        if np.abs(pb["x0"][3:6]).max() >= 0.6:
            out.append(probe(pb, kind))
        if len(out) == n:
            return out


def batch(pb, N):
    sig = cr.monotone_sigmas(N, 3)
    sig = sig[np.linspace(0, len(sig) - 1, min(48, len(sig))).round().astype(int)]
    base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 2 * pb["DC"])
    return FACTORS * base, np.repeat(FACTORS * base, len(sig)), np.tile(sig, (len(FACTORS), 1))


class Tol:
    """Sets the row tolerance on the solver and the restatement; restores the default on exit."""
    def __init__(self, solver, oracle, v):
        self.solver, self.oracle, self.v = solver, oracle, v

    def __enter__(self):
        self.solver.set_option("row_tol_1e9", self.v)
        self.oracle.set_row_tol(1e-9 * self.v)
        return self

    def __exit__(self, *exc):
        self.solver.set_option("row_tol_1e9", 10)
        self.oracle.set_row_tol(1e-8)


# At 1e-3 an active-set solve may stop at any point that violates rows by up to the tolerance, so two correct solvers agree
# on the flags but their costs only to the order of (multipliers x tolerance): about 1e-3 relative on these corridors (at
# 1e-6 and below they agree to 1e-14)
LOOSE_REL = 1e-2


def cost_bar(t):
    return REL if t <= 1000 else LOOSE_REL


def compare_at(t, feas_g, cost_g, co_g, feas_o, cost_o, co_o, what):
    """The suite's bar (test_parity_gpu._compare) up to 1e-6; at 1e-3 identical flags and costs within LOOSE_REL."""
    if t <= 1000:
        return _compare(feas_g, cost_g, co_g, feas_o, cost_o, co_o, what)
    assert np.array_equal(feas_g, feas_o), what + ": flags differ"
    ok = feas_o.astype(bool)
    if ok.any():
        assert (np.abs(cost_g[ok] - cost_o[ok]) / np.abs(cost_o[ok])).max() <= LOOSE_REL, what
    assert np.isinf(cost_g[~ok]).all()


def _probe_bar(counts):
    """counts[tol] = feasible probed candidates: none at 1e-9 / 1e-8, some at 1e-6 / 1e-3."""
    assert counts[1] == 0 and counts[10] == 0, counts
    assert counts[1000] > 0 and counts[1000000] > 0, counts


CASES = [(10, True, "velocity"), (10, True, "x0_face"), (10, True, "xf_face"), (10, False, "velocity"), (10, False, "x0_face"),
         (15, True, "velocity"), (15, True, "x0_face"), (15, True, "xf_face")]


@pytest.mark.parametrize("N,ff,kind", CASES)
def test_probes_through_both_kernels(solver, oracle, N, ff, kind):
    """fq_solve_batch, specialised and size-generic kernel (N = 10 whole and safe: one NW slot per lane; N = 15: two), and
    fq_solve_batch_cert (the certifying kernel), against the restatement at each tolerance."""
    counts = {t: 0 for t in TOLS}
    try:
        for pb in probe_corridors(N, ff, kind):
            _, dts, sigs = batch(pb, N)
            for t in TOLS:
                with Tol(solver, oracle, t):
                    fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
                    for generic in (0, 1):
                        solver.set_option("force_generic_kernel", generic)
                        fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
                        what = "N=%d ff=%d %s tol=%de-9 generic=%d" % (N, ff, kind, t, generic)
                        compare_at(t, fg, cg, cog, fo, co_, coo, what)
                        assert (it >= 0).all(), what + ": give-ups"
                    solver.set_option("force_generic_kernel", 0)
                    fc, cc, _ = solver.solve_batch_cert(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff)
                    assert np.array_equal(fc, fo), "N=%d %s tol=%de-9: certifying kernel" % (N, kind, t)
                    counts[t] += int(fo.sum())
    finally:
        solver.set_option("force_generic_kernel", 0)
    _probe_bar(counts)


def _first_feasible_min_cost(f, c, nf, ns):
    F = f.reshape(nf, ns).astype(bool)
    rows = np.flatnonzero(F.any(axis=1))
    if not len(rows):
        return -1, -1
    d = rows[0]
    return d, int(np.argmin(np.where(F[d], c.reshape(nf, ns)[d], np.inf)))


@pytest.mark.parametrize("N,ff,kind", [(10, True, "velocity"), (10, True, "x0_face"), (10, False, "x0_face"), (15, True, "xf_face"),
                                       (15, True, "velocity")])
def test_probes_through_the_sweep(solver, oracle, N, ff, kind):
    """fq_gen_new_traj (selection in the kernel's tail): genNewTraj's winner (first time allocation with a feasible
    assignment, then minimum cost) over the restatement's flags at the same tolerance."""
    solved = {t: 0 for t in TOLS}
    for pb in probe_corridors(N, ff, kind):
        dt_list, dts, sigs = batch(pb, N)
        sig = sigs[:len(sigs) // len(FACTORS)]
        for t in TOLS:
            with Tol(solver, oracle, t):
                fo, co_, _ = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, False, threads=8)
                g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dt_list, sig, ff)
            d, s = _first_feasible_min_cost(fo, co_, len(FACTORS), len(sig))
            assert g["dt_index"] == d and g["solved"] == (d >= 0), (kind, t, g["dt_index"], d)
            if d >= 0:
                c = co_[d * len(sig) + s]
                assert abs(g["cost"] - c) <= cost_bar(t) * max(1.0, c), (kind, t, g["cost"], c)
                if t <= 1000:                   # at 1e-3 near-equal costs may order differently
                    assert g["sigma_index"] == s, (kind, t)
                solved[t] += 1
    assert solved[1] == solved[10] == 0 and solved[1000] > 0 and solved[1000000] > 0, solved


# (seed, N, P, force_final, factor): under the x0_face probe the exact optimum of the first three is NOT a non-decreasing
# assignment at the looser tolerances, so the branch-and-bound, not the monotone pre-sweep, decides the answer; the
# fourth one's is non-decreasing
EXACT_CASES = [(5007, 10, 3, True, 5.0), (5055, 10, 4, False, 5.0), (5001, 10, 3, True, 5.0), (5004, 10, 3, True, 5.0)]


def test_probes_through_the_exact_sweep(solver, oracle):
    """fq_gen_new_traj_exact: the host presolve on the constant control points, the monotone pre-sweep and the
    branch-and-bound level kernel, against the restatement's branch-and-bound over all P^N assignments."""
    solved = {t: 0 for t in TOLS}
    n_nonmono = 0
    for seed, N, P, ff, f in EXACT_CASES:
        pb = probe(cr.make_corridor(seed, P, N, "uav", ff), "x0_face")
        dt = f * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        for t in TOLS:
            with Tol(solver, oracle, t):
                g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [dt], ff)
                rc, c, co, _, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], ff)
                what = (seed, N, t)
                assert g["exact"] and g["solved"] == (rc == 1), what
                if rc == 1:
                    solved[t] += 1
                    assert abs(g["cost"] - c) <= cost_bar(t) * max(1.0, c), (what, g["cost"], c)
                    if t <= 1000:
                        assert np.abs(g["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max()), what
                    n_nonmono += bool(np.any(np.diff(g["sigma"].astype(int)) < 0))
                # the sweep form: the same corridor over several time allocations
                dts = np.array([0.5, 1.0]) * dt
                gs = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, ff)
                first = next((k for k, d in enumerate(dts) if oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], d, pb["polys"], ff)[0] == 1), -1)
                assert gs["exact"] and gs["dt_index"] == first, (what, gs["dt_index"], first)
    assert solved[1] == solved[10] == 0 and solved[1000] >= 3 and solved[1000000] >= 3, solved
    assert n_nonmono >= 4, n_nonmono


def test_probes_through_the_chained_replan(solver, oracle):
    """fq_replan_pairs with the velocity probe on the whole side (x0 is the whole problem's start), against the CPU chain
    (oracle/pair_oracle.py) at the same tolerance."""
    from oracle import pair_oracle
    from test_pair_gpu import _check_against_oracle
    n = 8
    whole, safe = [], []
    for seed in range(71000, 71200):
        pb = cr.make_corridor(seed, 3, 10, "uav", True)
        if np.abs(pb["x0"][3:6]).max() >= 0.6:
            whole.append(probe(pb, "velocity"))
            safe.append(dict(cr.make_corridor(seed, 4, 10, "uav", False), lim=whole[-1]["lim"]))
        if len(whole) == n:
            break
    fw = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
    w = capi.make_pair_workload(whole, safe, fw, cr.monotone_sigmas(10, 3)[::3], fw, cr.monotone_sigmas(10, 4)[::12], DC=0.01,
                                r_fraction=0.3)
    won = {}
    for t in TOLS:
        with Tol(solver, oracle, t):
            g = solver.replan_pairs(w)
            r = g["results"]
            o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
        won[t] = int((o["whole_dt_index"] >= 0).sum())
        if won[t] and t <= 1000:
            _check_against_oracle(g, o, n)
        else:                                   # at 1e-3 (see LOOSE_REL) the flags and the winning time allocations
            assert np.array_equal(g["feasible_whole"], o["feasible_whole"]) and np.array_equal(r["whole_dt_index"], o["whole_dt_index"])
            ok = o["whole_dt_index"] >= 0
            assert np.allclose(r["whole_cost"][ok], o["whole_cost"][ok], rtol=LOOSE_REL)
    assert won[1] == won[10] == 0 and won[1000] > 0 and won[1000000] > 0, won


@pytest.mark.parametrize("tol", [1, 1000000])
@pytest.mark.parametrize("N,ff", SHAPES)
def test_every_solver_shape_at_the_ends_of_the_tolerance_range(solver, oracle, N, ff, tol):
    """Every compiled shape, specialised and size-generic kernel, at row tolerance 1e-9 and 1e-3: identical flags and no
    give-ups; at 1e-9 also the cost (1e-7) and coefficient (1e-6) bars of test_every_solver_shape_matches_the_restatement,
    at 1e-3 costs within LOOSE_REL."""
    try:
        with Tol(solver, oracle, tol):
            for P, profile, c, pb, dts, sigs in shape_batches(N, ff, 1, n_mono=16, n_arb=8):
                fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
                for generic in (0, 1):
                    solver.set_option("force_generic_kernel", generic)
                    fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
                    what = "N=%d ff=%d P=%d %s generic=%d tol=%de-9" % (N, ff, P, profile, generic, tol)
                    compare_at(tol, fg, cg, cog, fo, co_, coo, what)
                    assert (it >= 0).all(), what + ": iteration-cap or numeric give-ups"
    finally:
        solver.set_option("force_generic_kernel", 0)


@pytest.mark.parametrize("name,N,P,ff", [("cfg2", 10, 3, True), ("cfg3", 10, 4, False)])
def test_proofs_at_gurobis_tolerance(solver, oracle, name, N, P, ff):
    """At 1e-6 (Gurobi's default FeasibilityTol): solved flags satisfy the literal rows to 1e-6 + 1e-7 and carry KKT
    multipliers; infeasible flags carry Farkas certificates whose gap is below -1e-6, i.e. the kernel refused only
    violations beyond the tolerance."""
    from oracle import model_fullspace as mf, proofs
    from test_certificates_gpu import _candidates
    rng = np.random.default_rng(23 + N + P)
    proved = refuted = 0
    with Tol(solver, oracle, 1000):
        for seed in (6500, 6501, 6502):
            pb, dts, sigs = _candidates(N, P, ff, "uav", seed, 8, rng)
            fg, cg, cog, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, want_coeffs=True)
            fc, _, cert = solver.solve_batch_cert(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff)
            assert np.array_equal(fg, fc)
            for i in range(len(dts)):
                model = mf.build(N, pb["x0"], pb["xf"], pb["lim"], dts[i], pb["polys"], sigs[i], ff)
                if fg[i]:
                    proofs.assert_optimal(model, cog[i], cg[i], feas_tol=1e-6 + 1e-7)
                    proved += 1
                elif refuted < 16:
                    proofs.assert_infeasible(model, N, pb["polys"], sigs[i], cert[i], gap_max=-1e-6)
                    refuted += 1
    assert proved >= 10 and refuted >= 8, (proved, refuted)


def test_the_option_takes_1e9_to_1e3_only(solver):
    """0 is refused (at zero tolerance rounding keeps a just-activated row violated and the active set cycles), and so is
    anything above 1e-3; 1 (1e-9, Gurobi's lowest FeasibilityTol) and 1000000 are accepted."""
    try:
        for bad in (0, -1, 1000001):
            with pytest.raises(capi.FqError, match="1..1000000"):
                solver.set_option("row_tol_1e9", bad)
        for good in (1, 1000000):
            solver.set_option("row_tol_1e9", good)
    finally:
        solver.set_option("row_tol_1e9", 10)
