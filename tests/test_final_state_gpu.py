"""Inputs the rest of the suite holds fixed: a final state that moves (nonzero final velocity and acceleration; every other
corridor ends at rest, which multiplies the xf[3+ax]*dt and xf[6+ax]*dt^2 terms of the kernels and the literal model's
final rows by zero), and corridors far from the origin (a planner works in world coordinates; every other corridor lies
within +-5 m of it).  Each path is compared with the CPU restatement at the suite's usual bars."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr
from shape_cases import SHAPES, moving_final_state, shape_batches
from test_parity_gpu import REL, _compare

pytestmark = pytest.mark.gpu


def _moving(seed, P, N, ff, profile="uav"):
    return moving_final_state(cr.make_corridor(seed, P, N, profile, ff))


@pytest.mark.parametrize("N,ff", SHAPES)
def test_every_solver_shape_with_a_moving_final_state(solver, oracle, N, ff):
    """Every compiled (N, mode), specialised and size-generic kernel, on the families of tests/shape_cases.py with a moving
    final state, against the restatement: identical flags, cost 1e-7, coefficients 1e-6, no give-ups."""
    n_feas = n_infeas = 0
    try:
        for P, profile, c, pb, dts, sigs in shape_batches(N, ff, 1, n_mono=24, n_arb=8, final_state=moving_final_state):
            fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
            for generic in (0, 1):
                solver.set_option("force_generic_kernel", generic)
                fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
                what = "moving xf N=%d ff=%d P=%d %s generic=%d" % (N, ff, P, profile, generic)
                _compare(fg, cg, cog, fo, co_, coo, what)
                assert (it >= 0).all(), what + ": give-ups"
            ok = fo.astype(bool)
            if ok.any():                      # the solutions really end in the moving state
                x = coo[ok][:, N - 1]
                dt = dts[ok][:, None]
                vf = 3 * x[:, 0:3] * dt ** 2 + 2 * x[:, 3:6] * dt + x[:, 6:9]
                assert np.abs(vf - pb["xf"][3:6]).max() <= 1e-6
            n_feas += int(ok.sum())
            n_infeas += int((~ok).sum())
    finally:
        solver.set_option("force_generic_kernel", 0)
    assert n_feas >= 20 and n_infeas >= 20, (n_feas, n_infeas)


def test_sweeps_with_a_moving_final_state(solver, oracle):
    """fq_gen_new_traj (in-kernel selection) and fq_gen_new_traj_sampled (fillX on the device) against the restatement's
    flags, the host fq_fill_x and the oracle's fillX.  As the reference's fillX does, the last sample has its velocity,
    acceleration and jerk set to zero even though the trajectory arrives moving."""
    DC = 0.01
    n = 0
    for seed in range(4):
        for N, P, ff in ((10, 3, True), (6, 3, False)):
            pb = _moving(64000 + seed, P, N, ff)
            sig = cr.monotone_sigmas(N, P)
            dts = np.arange(1.0, 11.0) * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 2 * DC)
            fo, co_, _ = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.repeat(dts, len(sig)),
                                            np.tile(sig, (len(dts), 1)), ff, False, threads=8)
            F = fo.reshape(len(dts), len(sig)).astype(bool)
            g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, ff)
            b = solver.gen_new_traj_sampled(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sig, DC, ff)
            assert g["solved"] == b["solved"] == F.any()
            if not F.any():
                continue
            d = int(np.flatnonzero(F.any(axis=1))[0])
            s = int(np.argmin(np.where(F[d], co_.reshape(len(dts), -1)[d], np.inf)))
            assert (g["dt_index"], g["sigma_index"]) == (b["dt_index"], b["sigma_index"]) == (d, s)
            assert abs(g["cost"] - co_[d * len(sig) + s]) <= REL * max(1.0, co_[d * len(sig) + s]) and g["cost"] == b["cost"]
            Xh = capi.fill_x(N, g["coeffs"], dts[d], DC)
            Xo = oracle.fill_x(N, g["coeffs"], dts[d], DC)
            assert b["X"].shape == Xh.shape == Xo.shape
            assert np.allclose(b["X"], Xh, rtol=1e-12, atol=1e-12) and np.allclose(b["X"], Xo, rtol=1e-12, atol=1e-12)
            assert np.all(b["X"][-1, 3:] == 0)
            assert np.abs(b["X"][-2, 3:6]).max() > 0.1             # the sample before it still carries the final velocity
            if ff:
                assert np.abs(b["X"][-1, :3] - pb["xf"][:3]).max() <= 0.6 * 2 * DC + 1e-9
            n += 1
    assert n >= 4


@pytest.mark.parametrize("N,ff", [(10, True), (6, False)])
def test_exact_sweep_with_a_moving_final_state(solver, oracle, N, ff):
    """fq_gen_new_traj_exact against the restatement's branch-and-bound over all P^N assignments."""
    n_solved = n_unsolved = 0
    for seed in range(3):
        pb = _moving(64100 + seed, 3, N, ff)
        base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        for f in ((1.0, 2.0, 4.0) if ff else (0.3, 0.6, 2.0)):
            g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [f * base], ff)
            rc, c, co, _, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], f * base, pb["polys"], ff)
            assert g["exact"] and g["solved"] == (rc == 1), (seed, f)
            if rc == 1:
                n_solved += 1
                assert abs(g["cost"] - c) <= REL * max(1.0, c), (seed, f)
                assert np.abs(g["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max())
            else:
                n_unsolved += 1
    assert n_solved >= 2 and n_unsolved >= 1, (n_solved, n_unsolved)


def test_chained_replan_with_moving_final_states(solver, oracle):
    """fq_replan_pairs with moving xf_whole and xf_safe against the CPU chain (oracle/pair_oracle.py)."""
    from oracle import pair_oracle
    from test_pair_gpu import _check_against_oracle
    n = 10
    whole = [_moving(64200 + j, 3, 10, True) for j in range(n)]
    safe = [moving_final_state(cr.make_corridor(64200 + j, 4, 10, "uav", False), speed=0.4, accel=(-0.1, 0.2, 0.0)) for j in range(n)]
    fw = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
    w = capi.make_pair_workload(whole, safe, fw, cr.monotone_sigmas(10, 3)[::3], fw, cr.monotone_sigmas(10, 4)[::12], DC=0.01,
                                r_fraction=0.3)
    g = solver.replan_pairs(w)
    r = g["results"]
    o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    _check_against_oracle(g, o, n)
    assert o["feasible_safe"].any() and (o["safe_dt_index"] >= 0).any()


def test_optimality_proofs_with_a_moving_final_state(solver):
    """Every solved flag of config 2's shape with a moving final state carries a KKT proof on the literal model, whose
    final-velocity and final-acceleration rows then have nonzero right-hand sides."""
    from oracle import model_fullspace as mf, proofs
    N, P, ff = 10, 3, True
    rng = np.random.default_rng(5)
    proved = 0
    for seed in (6600, 6601, 6602):
        pb = _moving(seed, P, N, ff)
        sig = cr.monotone_sigmas(N, P)[rng.choice(66, 8, replace=False)]
        base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        dts = np.repeat(np.array([1.0, 2.0, 3.0, 5.0, 8.0]) * base, len(sig))
        sigs = np.tile(sig, (5, 1))
        fg, cg, cog, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, want_coeffs=True)
        for i in np.flatnonzero(fg):
            model = mf.build(N, pb["x0"], pb["xf"], pb["lim"], dts[i], pb["polys"], sigs[i], ff)
            assert np.abs(model[2][9:18]).max() > 0.05                  # the final rows carry the moving state
            proofs.assert_optimal(model, cog[i], cg[i])
            proved += 1
    assert proved >= 15, proved


# ---- corridors far from the origin
SHIFTS = [np.array([1e3, -7e2, 0.0]), np.array([1e4, 1e4, 1e4])]


def translate(pb, T):
    """The same corridor moved by T: positions of x0 / xf plus T, every half-space A x <= b becomes A x <= b + A.T."""
    x0, xf = pb["x0"].copy(), pb["xf"].copy()
    x0[:3] += T
    xf[:3] += T
    return dict(pb, x0=x0, xf=xf, polys=[(A, b + A @ T) for A, b in pb["polys"]], verts=pb["verts"] + T)


@pytest.mark.parametrize("N,ff", [(10, True), (10, False), (15, True)])
def test_corridors_far_from_the_origin(solver, oracle, N, ff):
    """Specialised and size-generic kernel on one family translated by (1e3, -7e2, 0) m and by 1e4 m on every axis: the
    flags of the untranslated batch and of the restatement on the translated inputs, costs within 1e-7 of both."""
    try:
        for P, profile, c, pb, dts, sigs in shape_batches(N, ff, 2, n_mono=24, n_arb=8):
            if P != 3:
                continue
            f0, c0, _, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff)
            assert f0.any() and not f0.all()
            for T in SHIFTS:
                tp = translate(pb, T)
                fo, co_, coo = oracle.solve_batch(N, tp["x0"], tp["xf"], tp["lim"], tp["polys"], dts, sigs, ff, True, threads=8)
                assert np.array_equal(fo, f0), "restatement flags move with the corridor: %s" % np.flatnonzero(fo != f0)[:8]
                for generic in (0, 1):
                    solver.set_option("force_generic_kernel", generic)
                    fg, cg, cog, it = solver.solve_batch(N, tp["x0"], tp["xf"], tp["lim"], tp["polys"], dts, sigs, ff, True, True)
                    what = "T=%s N=%d ff=%d generic=%d" % (T, N, ff, generic)
                    _compare(fg, cg, cog, fo, co_, coo, what)
                    assert (it >= 0).all(), what
                    ok = f0.astype(bool)
                    assert np.array_equal(fg, f0) and (np.abs(cg[ok] - c0[ok]) / np.abs(c0[ok])).max() <= REL, what
    finally:
        solver.set_option("force_generic_kernel", 0)


def test_exact_sweep_and_chained_replan_far_from_the_origin(solver, oracle):
    """fq_gen_new_traj_exact and fq_replan_pairs on translated corridors: the same winners and costs as at the origin."""
    from oracle import pair_oracle
    from test_pair_gpu import _check_against_oracle
    for seed in range(3):
        pb = cr.make_corridor(64300 + seed, 3, 10, "uav", True)
        dts = np.arange(1.0, 7.0) * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], 10), 0.02)
        g0 = solver.gen_new_traj_exact(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, True)
        assert g0["exact"] and g0["solved"]
        for T in SHIFTS:
            tp = translate(pb, T)
            g = solver.gen_new_traj_exact(10, tp["x0"], tp["xf"], tp["lim"], tp["polys"], dts, True)
            assert g["exact"] and g["dt_index"] == g0["dt_index"] and np.array_equal(g["sigma"], g0["sigma"]), (seed, T)
            assert abs(g["cost"] - g0["cost"]) <= REL * max(1.0, g0["cost"])
            rc, c, _, _, _ = oracle.solve_miqp(10, tp["x0"], tp["xf"], tp["lim"], dts[g["dt_index"]], tp["polys"], True)
            assert rc == 1 and abs(g["cost"] - c) <= REL * max(1.0, c)
    n = 8
    whole = [cr.make_corridor(64400 + j, 3, 10, "uav", True) for j in range(n)]
    safe = [cr.make_corridor(64400 + j, 4, 10, "uav", False) for j in range(n)]
    fw = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
    args = (fw, cr.monotone_sigmas(10, 3)[::3], fw, cr.monotone_sigmas(10, 4)[::12])
    r0 = solver.replan_pairs(capi.make_pair_workload(whole, safe, *args, DC=0.01, r_fraction=0.3))
    for T in SHIFTS:
        w = capi.make_pair_workload([translate(p, T) for p in whole], [translate(p, T) for p in safe], *args, DC=0.01, r_fraction=0.3)
        g = solver.replan_pairs(w)
        r = g["results"]
        o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
        _check_against_oracle(g, o, n)
        for k in ("feasible_whole", "feasible_safe"):
            assert np.array_equal(g[k], r0[k]), (T, k)
        for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index"):
            assert np.array_equal(r[k], r0["results"][k]), (T, k)
        ok = r["safe_dt_index"] >= 0
        assert np.allclose(r["whole_cost"], r0["results"]["whole_cost"], rtol=REL)
        assert np.allclose(r["safe_cost"][ok], r0["results"]["safe_cost"][ok], rtol=1e-6)
