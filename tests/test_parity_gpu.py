"""Parity of the CUDA path (through the C ABI) against the CPU restatement, on identical inputs.

Bar (BASELINE.json north_star): feasibility flags identical, cost and coefficients within 1e-4 relative.
The tolerance asserted here is tighter (1e-7) because both sides solve the same strictly convex QP exactly.
"""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr
from shape_cases import SHAPES, shape_batches

pytestmark = pytest.mark.gpu

REL = 1e-7


def _compare(feas_g, cost_g, co_g, feas_o, cost_o, co_o, what):
    assert np.array_equal(feas_g.astype(bool), feas_o.astype(bool)), "%s: feasibility flags differ at %s" % (
        what, np.nonzero(feas_g.astype(bool) != feas_o.astype(bool))[0][:10])
    ok = feas_o.astype(bool)
    if ok.any():
        rel = np.abs(cost_g[ok] - cost_o[ok]) / np.maximum(1e-9, np.abs(cost_o[ok]))
        assert rel.max() <= REL, "%s: cost rel err %.3e" % (what, rel.max())
        if co_g is not None:
            scale = np.maximum(1.0, np.abs(co_o[ok]).max(axis=(1, 2), keepdims=True))
            err = (np.abs(co_g[ok] - co_o[ok]) / scale).max()
            assert err <= 1e-6, "%s: coefficient err %.3e" % (what, err)
    assert np.all(np.isinf(cost_g[~ok]))


def test_demo_corridor_batch(solver, oracle, demo_corridor):
    fx = demo_corridor
    N = fx["N"]
    sig = cr.monotone_sigmas(N, 3)
    dts = np.repeat(np.array([0.5, 0.6, 0.7, 0.8, 1.0, 1.5]), len(sig))
    sigs = np.tile(sig, (6, 1))
    fg, cg, cog, it = solver.solve_batch(N, fx["x0"], fx["xf"], fx["lim"], fx["polys"], dts, sigs, True, True, True)
    fo, co_, coo = oracle.solve_batch(N, fx["x0"], fx["xf"], fx["lim"], fx["polys"], dts, sigs, True, True, threads=8)
    assert fo.sum() > 20 and (~fo.astype(bool)).sum() > 20
    _compare(fg, cg, cog, fo, co_, coo, "demo corridor")
    assert (it > 0).all()


@pytest.mark.parametrize("N,P,ff,profile", [(10, 3, True, "uav"), (10, 4, False, "uav"), (6, 3, True, "uav"),
                                            (6, 3, False, "uav"), (15, 8, True, "ground"), (4, 2, False, "uav"),
                                            (16, 5, True, "uav")])
def test_random_corridors(solver, oracle, N, P, ff, profile):
    rng = np.random.default_rng(N * 100 + P)
    sig_all = cr.monotone_sigmas(N, P) if P <= 4 else cr.sample_monotone_sigmas(N, P, 256, rng)
    for seed in range(3):
        pb = cr.make_corridor(1000 + seed, P, N, profile, ff)
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        facs = np.array([1.0, 1.5, 2.0, 3.0, 4.0, 6.0])
        sig = sig_all[rng.choice(len(sig_all), min(48, len(sig_all)), replace=False)]
        dts = np.repeat(facs * max(dti, 2 * pb["DC"]), len(sig))
        sigs = np.tile(sig, (len(facs), 1))
        fg, cg, cog, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True)
        fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
        _compare(fg, cg, cog, fo, co_, coo, "N=%d P=%d seed=%d" % (N, P, seed))


def test_no_polytopes_and_zero_dof(solver, oracle):
    """Config 1: N=3 whole has zero degrees of freedom (pure feasibility check); P=0 means no corridor rows."""
    lim = [5.0, 5.0, 8.0]
    x0 = np.zeros(9)
    for N in (3, 5):
        for scale in (0.5, 2.0, 4.0):
            xf = np.zeros(9)
            xf[:3] = scale * np.array([1.0, -0.7, 0.4])
            dti = capi.dt_initial(x0, xf, lim, N)
            dts = np.arange(1, 11) * max(dti, 0.02)
            fg, cg, cog, _ = solver.solve_batch(N, x0, xf, lim, [], dts, None, True, True)
            fo, co_, coo = oracle.solve_batch(N, x0, xf, lim, [], dts, np.zeros((len(dts), N), np.uint8), True, True)
            _compare(fg, cg, cog, fo, co_, coo, "P=0 N=%d" % N)
            assert fg.any() and not fg.all()


def test_infeasible_start_state(solver, oracle):
    """x0 outside its polytope / beyond the velocity box: every candidate must come back infeasible."""
    pb = cr.make_corridor(7, 3, 10)
    sig = cr.monotone_sigmas(10, 3)
    dts = np.full(len(sig), 0.6)
    x0 = pb["x0"].copy()
    x0[2] = -3.0                                 # below the ground face
    fg, cg, _, _ = solver.solve_batch(10, x0, pb["xf"], pb["lim"], pb["polys"], dts, sig)
    assert not fg.any() and np.all(np.isinf(cg))
    x0 = pb["x0"].copy()
    x0[3] = 9.0                                  # |v0| > v_max
    fg, cg, _, _ = solver.solve_batch(10, x0, pb["xf"], pb["lim"], pb["polys"], dts, sig)
    assert not fg.any()


def test_multi_matches_batches(solver, oracle):
    """Heterogeneous launch == the same problems solved one by one."""
    N, P = 10, 3
    sig = cr.monotone_sigmas(N, P)
    probs = [cr.make_corridor(50 + k, P, N) for k in range(5)]
    x0 = np.array([p["x0"] for p in probs]); xf = np.array([p["xf"] for p in probs])
    lim = np.array([p["lim"] for p in probs])
    poly_ofs, face_ofs, rows, cand_ofs, dts, sigs = [0], [0], [], [0], [], []
    for k, p in enumerate(probs):
        for A, b in p["polys"]:
            rows.append(np.hstack([A, b[:, None]])); face_ofs.append(face_ofs[-1] + len(b))
        poly_ofs.append(poly_ofs[-1] + P)
        dti = capi.dt_initial(p["x0"], p["xf"], p["lim"], N)
        n = 20 + 7 * k
        dts.append((1.0 + 0.25 * np.arange(n)) * dti); sigs.append(sig[np.arange(n) % len(sig)])
        cand_ofs.append(cand_ofs[-1] + n)
    Ab = np.ascontiguousarray(np.vstack(rows)); dts_all = np.concatenate(dts); sig_all = np.ascontiguousarray(np.vstack(sigs))
    fg, cg, cog, _ = solver.solve_multi(N, True, np.ascontiguousarray(x0), np.ascontiguousarray(xf),
                                        np.ascontiguousarray(lim), np.array(poly_ofs, np.int32),
                                        np.array(face_ofs, np.int32), Ab, np.array(cand_ofs, np.int32), dts_all,
                                        sig_all, want_coeffs=True)
    for k, p in enumerate(probs):
        a, b = cand_ofs[k], cand_ofs[k + 1]
        fo, co_, coo = oracle.solve_batch(N, p["x0"], p["xf"], p["lim"], p["polys"], dts[k], sigs[k], True, True)
        _compare(fg[a:b], cg[a:b], cog[a:b], fo, co_, coo, "multi prob %d" % k)


def test_gen_new_traj_matches_oracle_sweep(solver, oracle, demo_corridor):
    """First feasible dt, minimum-cost assignment: same winner as the oracle's sequential sweep with B&B over
    ALL assignments (the monotone list must contain the MIQP optimum on these corridors)."""
    cases = [(demo_corridor["N"], demo_corridor["x0"], demo_corridor["xf"], demo_corridor["lim"], demo_corridor["polys"], True)]
    for seed in range(4):
        pb = cr.make_corridor(300 + seed, 3, 10)
        cases.append((10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], True))
        pb = cr.make_corridor(400 + seed, 4, 10, force_final=False)
        cases.append((10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], False))
    for N, x0, xf, lim, polys, ff in cases:
        sig = cr.monotone_sigmas(N, len(polys))
        DC = 0.01
        dti = capi.dt_initial(x0, xf, lim, N)
        facs = np.arange(1.0, 11.0, 1.0)
        dts = facs * max(dti, 2 * DC)
        g = solver.gen_new_traj(N, x0, xf, lim, polys, dts, sig, ff)
        o = oracle.gen_new_traj(N, x0, xf, lim, polys, DC, 1.0, 10.0, 1.0, None, ff)
        assert g["solved"] == o["solved"]
        if o["solved"]:
            assert facs[g["dt_index"]] == o["factor"] and g["dt_index"] + 1 == o["trials"]
            assert abs(g["cost"] - o["cost"]) <= REL * max(1.0, o["cost"])
            assert np.abs(g["coeffs"] - o["coeffs"]).max() <= 1e-6 * max(1.0, np.abs(o["coeffs"]).max())


def test_face_ofs_start_is_free_for_sweeps_and_zero_for_batches(solver):
    """fq_gen_new_traj takes a face_ofs whose first offset is not 0 (it stages rows 0 .. face_ofs[P]-1 of Ab and starts
    the first polytope at row 0); the batch entries refuse it ("offset arrays must start at 0")."""
    import ctypes as C
    N = 10
    pb = cr.make_corridor(300, 3, N)
    P, ofs, Ab = capi.pack_polys(pb["polys"])
    ofs1 = np.ascontiguousarray(ofs + 1, np.int32)
    Ab1 = np.ascontiguousarray(np.vstack([Ab[:1], Ab]))
    sig = np.ascontiguousarray(cr.monotone_sigmas(N, P), np.uint8)
    x0, xf, lim = (np.ascontiguousarray(pb[k], np.float64) for k in ("x0", "xf", "lim"))
    dts = np.arange(1.0, 11.0) * max(capi.dt_initial(x0, xf, lim, N), 0.02)
    di, si, cost = C.c_int(-1), C.c_int(-1), C.c_double(np.inf)
    co = np.zeros((N, 12))
    rc = solver._check(solver._L.fq_gen_new_traj(solver._h, N, 1, x0.ctypes.data, xf.ctypes.data, lim.ctypes.data, P,
                                                 ofs1.ctypes.data, Ab1.ctypes.data, dts.size, dts.ctypes.data, sig.shape[0],
                                                 sig.ctypes.data, C.addressof(di), C.addressof(si), C.addressof(cost),
                                                 co.ctypes.data))
    assert rc in (0, 1)
    feas, costs = np.zeros(len(sig), np.uint8), np.zeros(len(sig))
    d = np.full(len(sig), dts[-1])
    rc = solver._L.fq_solve_batch(solver._h, N, 1, x0.ctypes.data, xf.ctypes.data, lim.ctypes.data, P, ofs1.ctypes.data,
                                  Ab1.ctypes.data, len(sig), d.ctypes.data, sig.ctypes.data, feas.ctypes.data,
                                  costs.ctypes.data, None, None)
    assert rc == -1 and solver._L.fq_last_error(solver._h).decode() == "offset arrays must start at 0"


def test_large_batch_properties(solver):
    """BASELINE config sizes (1024 whole / 8192 safe candidates): size-independent properties.
    (i) every feasible solution satisfies the model rows when re-evaluated on the host from the returned
    coefficients; (ii) cost equals sum (6a)^2; (iii) for a fixed sigma feasibility is monotone here: relaxing dt by
    large factors keeps these rest-to-rest problems feasible; (iv) identical candidates give identical bits."""
    for (N, P, ff, ndt, nsig) in ((10, 3, True, 16, 64), (10, 4, False, 32, 256)):
        pb = cr.make_corridor(2024, P, N, force_final=ff)
        sig = cr.monotone_sigmas(N, P)[:nsig]
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        dts = np.repeat(np.arange(1, ndt + 1) * max(dti, 0.02), len(sig))
        sigs = np.tile(sig, (ndt, 1))
        f1, c1, co, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True)
        f2, c2, _, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, False)
        assert np.array_equal(f1, f2) and np.array_equal(c1, c2)
        ok = f1.astype(bool)
        assert ok.any()
        a = co[ok][:, :, 0:3]
        assert np.allclose(np.sum((6 * a) ** 2, axis=(1, 2)), c1[ok], rtol=1e-9, atol=1e-12)
        lim = pb["lim"]
        for i in np.nonzero(ok)[0][::17]:
            x = co[i]; dt = dts[i]
            assert np.abs(x[:, 6:9]).max() <= lim[0] + 1e-6 and np.abs(2 * x[:, 3:6]).max() <= lim[1] + 1e-6
            assert np.abs(6 * x[:, 0:3]).max() <= lim[2] + 1e-6
            assert np.allclose(x[0, 9:12], pb["x0"][:3]) and np.allclose(x[0, 6:9], pb["x0"][3:6])
            for t in range(N):
                A, b = pb["polys"][sigs[i][t]]
                a_, b_, c_, d_ = x[t, 0:3], x[t, 3:6], x[t, 6:9], x[t, 9:12]
                cps = [d_, d_ + c_ * dt / 3, d_ + 2 * c_ * dt / 3 + b_ * dt * dt / 3,
                       a_ * dt ** 3 + b_ * dt ** 2 + c_ * dt + d_]
                for cp in cps:
                    assert (A @ cp - b).max() <= 1e-6
                if t + 1 < N:
                    assert np.allclose(cps[3], x[t + 1, 9:12], atol=1e-9)
                    assert np.allclose(3 * a_ * dt ** 2 + 2 * b_ * dt + c_, x[t + 1, 6:9], atol=1e-9)
                    assert np.allclose(6 * a_ * dt + 2 * b_, 2 * x[t + 1, 3:6], atol=1e-9)


@pytest.mark.parametrize("N,P,ff", [(10, 3, True), (10, 4, False), (6, 3, True), (15, 8, False), (16, 4, True), (4, 2, True)])
def test_generic_and_specialised_kernels_agree(built_lib, N, P, ff):
    """Two independent CUDA implementations of the same solve (size-generic / size-specialised) on the same batch."""
    rng = np.random.default_rng(N + 31 * P)
    s = capi.Solver(0)
    try:
        sig_all = cr.monotone_sigmas(N, P) if P <= 4 and N <= 10 else cr.sample_monotone_sigmas(N, P, 300, rng)
        pb = cr.make_corridor(4242 + N, P, N, "uav" if N != 15 else "ground", ff)
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        facs = np.linspace(1.0, 6.0, 11)
        sig = sig_all[rng.choice(len(sig_all), min(100, len(sig_all)), replace=False)]
        dts = np.repeat(facs * max(dti, 0.02), len(sig))
        sigs = np.tile(sig, (len(facs), 1))
        fa, ca, coa, ita = s.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
        s.set_option("force_generic_kernel", 1)
        fb, cb, cob, itb = s.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
        _compare(fa, ca, coa, fb, cb, cob, "specialised vs generic N=%d" % N)
        assert ita.max() > 0 and itb.max() > 0      # iteration counts differ: the two kernels use different pivot rules
    finally:
        s.close()


@pytest.mark.parametrize("N,ff", SHAPES)
def test_every_solver_shape_matches_the_restatement(solver, oracle, N, ff):
    """Every (N, mode) the solver is compiled for (fq_solve_kernel_t<N, WHOLE>, N = 4..16) and the size-generic kernel on the
    same batches, against the CPU restatement.  The shape sets the lane layout: NW-vector slots per lane (one up to whole
    N = 13 / safe N = 12, two from whole 14 / safe 13), Y rows per lane (1, 2, 3, 4 from N = 4, 6, 11, 16) and the
    register budget (N = 10/11, 15/16).  One corridor of each family of tests/shape_cases.py."""
    n_feas = n_infeas = 0
    try:
        for P, profile, c, pb, dts, sigs in shape_batches(N, ff, 1):
            fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
            for generic in (0, 1):
                solver.set_option("force_generic_kernel", generic)
                fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
                what = "N=%d ff=%d P=%d %s generic=%d" % (N, ff, P, profile, generic)
                _compare(fg, cg, cog, fo, co_, coo, what)
                assert (it >= 0).all(), what + ": iteration-cap or numeric give-ups"
            n_feas += int(fo.sum())
            n_infeas += int((fo == 0).sum())
    finally:
        solver.set_option("force_generic_kernel", 0)
    assert n_feas >= 20 and n_infeas >= 20, (n_feas, n_infeas)


@pytest.mark.parametrize("N,ff", [(3, True), (2, False), (3, False)])
def test_generic_only_shapes_on_corridors(solver, oracle, N, ff):
    """Shapes below the specialised range run on the size-generic kernel only: whole N = 3 and safe N = 2 have no degree
    of freedom left (a feasibility check of the one trajectory through corridor rows), safe N = 3 has one."""
    n_feas = n_infeas = 0
    for seed in range(6):
        for P in (2, 3):
            pb = cr.make_corridor(61000 + 10 * seed + P, P, N, "uav", ff)
            sig = np.vstack([cr.monotone_sigmas(N, P), np.random.default_rng(seed).integers(0, P, (4, N)).astype(np.uint8)])
            dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
            facs = np.array([0.5, 1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
            dts = np.repeat(facs * max(dti, 2 * pb["DC"]), len(sig))
            sigs = np.tile(sig, (len(facs), 1))
            fg, cg, cog, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
            fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True)
            _compare(fg, cg, cog, fo, co_, coo, "N=%d ff=%d P=%d seed=%d" % (N, ff, P, seed))
            assert (it >= 0).all()
            n_feas += int(fo.sum())
            n_infeas += int((fo == 0).sum())
    assert n_feas >= 5 and n_infeas >= 5, (n_feas, n_infeas)


@pytest.mark.parametrize("N_whole,N_safe", [(10, 2), (3, 2), (6, 3)])
def test_chained_replan_with_generic_only_shapes(solver, oracle, N_whole, N_safe):
    """fq_replan_pairs with a generic-only shape on one side (N_safe = 2 is the smallest it accepts) against the CPU chain
    (oracle/pair_oracle.py) on the device's own time-allocation bases."""
    from oracle import pair_oracle
    n = 12
    whole = [cr.make_corridor(62000 + j, 3, N_whole, "uav", True) for j in range(n)]
    safe = [cr.make_corridor(62000 + j, 2, N_safe, "uav", False) for j in range(n)]
    fw = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
    w = capi.make_pair_workload(whole, safe, fw, cr.monotone_sigmas(N_whole, 3)[:24], fw, cr.monotone_sigmas(N_safe, 2),
                                DC=0.01, r_fraction=0.3)
    g = solver.replan_pairs(w)
    r = g["results"]
    o = pair_oracle.replan_pairs(w, threads=4, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    from test_pair_gpu import _check_against_oracle
    _check_against_oracle(g, o, n)
    assert (o["safe_dt_index"] >= 0).any() and o["feasible_safe"].any() and not o["feasible_safe"].all()
    assert o["feasible_whole"].any() and not o["feasible_whole"].all()


def test_edge_cases_through_the_abi(solver, oracle):
    """Empty batch, invalid assignment, many-faced polytopes (> 32 faces: more than one pass per segment), duplicated
    polytopes, tiny and huge time allocations, ragged problems with zero candidates."""
    pb = cr.make_corridor(77, 3, 10)
    sig = cr.monotone_sigmas(10, 3)
    # empty batch
    f, c, _, _ = solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.zeros(0), np.zeros((0, 10), np.uint8))
    assert f.size == 0 and c.size == 0
    # invalid assignment entry -> argument error, not a crash
    bad = sig[:4].copy()
    bad[2, 5] = 3
    with pytest.raises(capi.FqError):
        solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.full(4, 0.5), bad)
    # N out of range
    with pytest.raises(capi.FqError):
        solver.solve_batch(2, pb["x0"], pb["xf"], pb["lim"], [], np.full(1, 0.5), None)
    # polytopes with many (redundant) faces: 45 faces each
    rng = np.random.default_rng(3)
    fat = []
    for (A, b), (v0, v1) in zip(pb["polys"], zip(pb["verts"][:-1], pb["verts"][1:])):
        mid = 0.5 * (v0 + v1)
        n = rng.normal(size=(45 - len(b), 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        fat.append((np.vstack([A, n]), np.concatenate([b, n @ mid + rng.uniform(2.5, 4.0, len(n))])))
    dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], 10)
    dts = np.repeat(np.array([1.5, 2.0, 3.0, 5.0]) * dti, len(sig))
    sigs = np.tile(sig, (4, 1))
    for polys in (fat, [pb["polys"][0], pb["polys"][0], pb["polys"][2]]):
        fg, cg, cog, _ = solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], polys, dts, sigs, True, True)
        fo, co_, coo = oracle.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], polys, dts, sigs, True, True, threads=8)
        _compare(fg, cg, cog, fo, co_, coo, "many faces / duplicate polytopes")
    # extreme time allocations: 2*DC (the floor findDT applies, solverGurobi.cpp:496) and a very slow one
    for dt in (0.02, 25.0):
        d = np.full(len(sig), dt)
        fg, cg, cog, _ = solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], d, sig, True, True)
        fo, co_, coo = oracle.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], d, sig, True, True, threads=8)
        _compare(fg, cg, cog, fo, co_, coo, "dt=%g" % dt)
    # ragged multi: a problem with zero candidates in the middle
    probs = [cr.make_corridor(90 + k, 3, 10) for k in range(3)]
    rows, face_ofs = [], [0]
    for p in probs:
        for A, b in p["polys"]:
            rows.append(np.hstack([A, b[:, None]])); face_ofs.append(face_ofs[-1] + len(b))
    cand_ofs = np.array([0, 30, 30, 66], np.int32)
    dts = np.concatenate([np.full(30, 2.5 * dti), np.full(36, 3.0 * dti)])
    sg = np.ascontiguousarray(np.vstack([sig[:30], sig[:36]]))
    fg, cg, cog, _ = solver.solve_multi(10, True, np.ascontiguousarray([p["x0"] for p in probs]),
                                        np.ascontiguousarray([p["xf"] for p in probs]),
                                        np.ascontiguousarray([p["lim"] for p in probs]), np.array([0, 3, 6, 9], np.int32),
                                        np.array(face_ofs, np.int32), np.ascontiguousarray(np.vstack(rows)), cand_ofs, dts, sg,
                                        want_coeffs=True)
    for k, (a, b) in enumerate(((0, 30), (30, 30), (30, 66))):
        if b > a:
            p = probs[k]
            fo, co_, coo = oracle.solve_batch(10, p["x0"], p["xf"], p["lim"], p["polys"], dts[a:b], sg[a:b], True, True)
            _compare(fg[a:b], cg[a:b], cog[a:b], fo, co_, coo, "ragged prob %d" % k)


def test_ground_robot_profile(solver, oracle):
    """BASELINE config 5: ground-robot limits (1.4/1.4/5.0), N=15, 8 narrow polytopes, sampled monotone assignments."""
    rng = np.random.default_rng(15)
    N, P = 15, 8
    pb = cr.make_corridor(555, P, N, "ground", True)
    sig = cr.sample_monotone_sigmas(N, P, 512, rng)
    dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
    dts = np.repeat(np.arange(1, 9) * max(dti, 0.02), 64)
    sigs = np.ascontiguousarray(sig[:512])
    fg, cg, cog, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, True, True)
    fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, True, True, threads=8)
    _compare(fg, cg, cog, fo, co_, coo, "ground robot cfg5")


def test_device_pointer_entry_matches_host_entry(solver):
    """fq_solve_multi_dev (device-resident inputs, caller's stream, no sync inside) == fq_solve_multi."""
    import torch
    N, P = 10, 4
    sig = cr.monotone_sigmas(N, P)
    probs = [cr.make_corridor(130 + k, P, N, force_final=False) for k in range(6)]
    poly_ofs, face_ofs, rows, cand_ofs, dts, sigs = [0], [0], [], [0], [], []
    for k, p in enumerate(probs):
        for A, b in p["polys"]:
            rows.append(np.hstack([A, b[:, None]])); face_ofs.append(face_ofs[-1] + len(b))
        poly_ofs.append(poly_ofs[-1] + P)
        dti = capi.dt_initial(p["x0"], p["xf"], p["lim"], N)
        n = 100 + 13 * k
        dts.append((1.0 + 0.1 * np.arange(n)) * dti); sigs.append(sig[(7 * np.arange(n)) % len(sig)])
        cand_ofs.append(cand_ofs[-1] + n)
    h = dict(x0=np.ascontiguousarray([p["x0"] for p in probs]), xf=np.ascontiguousarray([p["xf"] for p in probs]),
             lim=np.ascontiguousarray([p["lim"] for p in probs]), poly_ofs=np.array(poly_ofs, np.int32),
             face_ofs=np.array(face_ofs, np.int32), Ab=np.ascontiguousarray(np.vstack(rows)),
             cand_ofs=np.array(cand_ofs, np.int32), dt=np.concatenate(dts), sigma=np.ascontiguousarray(np.vstack(sigs)))
    fh, ch, coh, _ = solver.solve_multi(N, False, h["x0"], h["xf"], h["lim"], h["poly_ofs"], h["face_ofs"], h["Ab"],
                                        h["cand_ofs"], h["dt"], h["sigma"], want_coeffs=True)
    dev = torch.device("cuda", 0)
    d = {k: torch.from_numpy(v).to(dev) for k, v in h.items()}
    n = int(cand_ofs[-1])
    feas = torch.zeros(n, dtype=torch.uint8, device=dev)
    cost = torch.zeros(n, dtype=torch.float64, device=dev)
    coef = torch.zeros(n * N * 12, dtype=torch.float64, device=dev)
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()        # the fills above run on torch's stream; the library launches on `st`
    with torch.cuda.stream(st):
        solver.solve_multi_dev(N, False, len(probs), d["x0"].data_ptr(), d["xf"].data_ptr(), d["lim"].data_ptr(),
                               d["poly_ofs"].data_ptr(), d["face_ofs"].data_ptr(), d["Ab"].data_ptr(),
                               d["cand_ofs"].data_ptr(), int(np.diff(cand_ofs).max()),
                               int(max(face_ofs[poly_ofs[j + 1]] - face_ofs[poly_ofs[j]] for j in range(len(probs)))),
                               d["dt"].data_ptr(), d["sigma"].data_ptr(), feas.data_ptr(), cost.data_ptr(),
                               coef.data_ptr(), 0, st.cuda_stream)
    st.synchronize()
    assert np.array_equal(feas.cpu().numpy(), fh) and np.array_equal(cost.cpu().numpy(), ch)
    assert np.array_equal(coef.cpu().numpy().reshape(n, N, 12), coh)


def test_forest_paired_whole_then_safe(solver, oracle):
    """BASELINE config 4 in miniature: random-forest point cloud -> polyline -> convex decomposition (product host code)
    -> whole sweep -> the safe problem starts from a sample of the whole trajectory (faster.cpp:475) with its own
    decomposition -> safe sweep.  Every stage is compared with the oracle run on the same inputs."""
    from oracle import decomp_oracle as do
    DC, N = 0.01, 10
    done = 0
    for seed in range(200, 212):
        try:
            pb = cr.make_forest_corridor(seed, 3, N, True)
        except RuntimeError:
            continue
        polys_o = do.cvx_ellipsoid_decomp(pb["verts"], pb["obs"], (2.0, 2.0, 1.0), 0.42, 0.0)
        assert all(a.shape == b.shape for (a, _), (b, _) in zip(pb["polys"], polys_o))
        sig = cr.monotone_sigmas(N, 3)
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        facs = np.arange(1.0, 11.0)
        g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], facs * max(dti, 2 * DC), sig, True)
        o = oracle.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], DC, 1.0, 10.0, 1.0, None, True)
        assert g["solved"] == o["solved"]
        if not o["solved"]:
            continue
        assert facs[g["dt_index"]] == o["factor"] and abs(g["cost"] - o["cost"]) <= REL * max(1.0, o["cost"])
        dt = o["dt"]
        X = capi.fill_x(N, g["coeffs"], dt, DC)
        R = X[int(0.6 * len(X))]                                  # stand-in for findIndexR's choice
        j = int(np.argmin([np.linalg.norm(np.cross(R[:3] - pb["verts"][k], pb["verts"][k + 1] - pb["verts"][k]))
                           / np.linalg.norm(pb["verts"][k + 1] - pb["verts"][k]) for k in range(3)]))
        safe_path = np.vstack([R[:3], pb["verts"][j + 1:]])
        if len(safe_path) < 2 or np.linalg.norm(safe_path[1] - safe_path[0]) < 0.05:
            continue
        spolys = capi.ellipsoid_decomp(safe_path, pb["obs"], (2.0, 2.0, 1.0), 0.42, 0.0)
        Ps = len(spolys)
        x0s = np.concatenate([R[:3], R[3:6], R[6:9]])
        xfs = np.zeros(9)
        xfs[:3] = safe_path[-1]
        sigs = cr.monotone_sigmas(N, Ps)
        dtis = capi.dt_initial(x0s, xfs, pb["lim"], N)
        gs = solver.gen_new_traj(N, x0s, xfs, pb["lim"], spolys, facs * max(dtis, 2 * DC), sigs, False)
        os_ = oracle.gen_new_traj(N, x0s, xfs, pb["lim"], spolys, DC, 1.0, 10.0, 1.0, None, False)
        assert gs["solved"] == os_["solved"]
        if os_["solved"]:
            assert facs[gs["dt_index"]] == os_["factor"]
            assert abs(gs["cost"] - os_["cost"]) <= REL * max(1.0, os_["cost"])
            assert np.abs(gs["coeffs"] - os_["coeffs"]).max() <= 1e-6 * max(1.0, np.abs(os_["coeffs"]).max())
            assert np.allclose(gs["coeffs"][0, 9:12], R[:3], atol=1e-9)      # safe trajectory starts at R
            done += 1
    assert done >= 3


def test_throughput_copy_path_matches_latency_path(solver):
    """fq_solve_multi stages small inputs through one pinned buffer and DMAs large ones straight from the caller's
    arrays (> 512 KB): both paths must give identical bits."""
    N, P = 10, 3
    sig = cr.monotone_sigmas(N, P)
    probs = [cr.make_corridor(900 + k, P, N) for k in range(40)]
    poly_ofs, face_ofs, rows, cand_ofs, dts, sigs = [0], [0], [], [0], [], []
    for k, p in enumerate(probs):
        for A, b in p["polys"]:
            rows.append(np.hstack([A, b[:, None]])); face_ofs.append(face_ofs[-1] + len(b))
        poly_ofs.append(poly_ofs[-1] + P)
        dti = capi.dt_initial(p["x0"], p["xf"], p["lim"], N)
        dts.append(np.repeat(np.arange(1, 17) * dti, len(sig))); sigs.append(np.tile(sig, (16, 1)))
        cand_ofs.append(cand_ofs[-1] + 16 * len(sig))
    x0 = np.ascontiguousarray([p["x0"] for p in probs]); xf = np.ascontiguousarray([p["xf"] for p in probs])
    lim = np.ascontiguousarray([p["lim"] for p in probs]); Ab = np.ascontiguousarray(np.vstack(rows))
    po, fo, co = np.array(poly_ofs, np.int32), np.array(face_ofs, np.int32), np.array(cand_ofs, np.int32)
    dt_all, sig_all = np.concatenate(dts), np.ascontiguousarray(np.vstack(sigs))
    assert dt_all.size * (8 + N) > 512 * 1024                      # forces the throughput path
    f_big, c_big, _, _ = solver.solve_multi(N, True, x0, xf, lim, po, fo, Ab, co, dt_all, sig_all)
    for k in (0, 17, 39):                                          # the same problems one by one: latency path
        a, b = cand_ofs[k], cand_ofs[k + 1]
        f1, c1, _, _ = solver.solve_batch(N, probs[k]["x0"], probs[k]["xf"], probs[k]["lim"], probs[k]["polys"], dts[k], sigs[k])
        assert np.array_equal(f_big[a:b], f1) and np.array_equal(c_big[a:b], c1)


def test_deferred_host_batches_on_two_contexts(solver):
    """fq_solve_multi_async + fq_wait: two contexts (the reference's sg_whole_ / sg_safe_) keep a whole and a safe batch in
    flight together; results are bit-identical to the blocking call, a following call on the same context settles the
    deferred one first, and the slice count does not change any bit."""
    import bench
    second = capi.Solver(0)
    works = [bench.make_single(dict(bench.SINGLE["cfg2"], seed=4100), 32, capi.dt_initial),    # > 512 KB: throughput path
             bench.make_single(dict(bench.SINGLE["cfg2"], P=4, ff=False, seed=4200), 32, capi.dt_initial)]
    args = [(w["N"], w["ff"], w["x0"], w["xf"], w["lim"], w["poly_ofs"], w["face_ofs"], w["Ab"], w["cand_ofs"], w["dt"], w["sigma"])
            for w in works]
    ref = [solver.solve_multi(*a) for a in args]                              # blocking
    outs = []
    for sv, a in zip((solver, second), args):
        outs.append(sv.solve_multi(*a, deferred=True))
    solver.wait(); second.wait()
    for r, o in zip(ref, outs):
        assert np.array_equal(r[0], o[0]) and np.array_equal(r[1], o[1])
    assert ref[0][0].any() and not ref[0][0].all()
    # a second call on a context with a deferred batch in flight: the first batch's outputs must be complete afterwards
    o1 = solver.solve_multi(*args[0], deferred=True)
    pb = cr.make_corridor(4100, 3, 10, "uav", True)
    g = solver.gen_new_traj(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], np.arange(1, 11) * 0.3, cr.monotone_sigmas(10, 3), True)
    assert np.array_equal(o1[0], ref[0][0]) and np.array_equal(o1[1], ref[0][1]) and g["dt_index"] >= -1
    for n_slices in (1, 2, 7):
        solver.set_option("throughput_slices", n_slices)
        o = solver.solve_multi(*args[1])
        assert np.array_equal(o[0], ref[1][0]) and np.array_equal(o[1], ref[1][1])
    solver.set_option("throughput_slices", 0)


def test_non_finite_inputs_are_rejected_or_survive(solver):
    """NaN / Inf / non-positive dt: the host-pointer entries refuse them; the device-pointer entry cannot look at the
    data, so the kernels must come back (numeric failure -> infeasible) instead of faulting."""
    import torch
    pb = cr.make_corridor(31, 3, 10)
    sig = cr.monotone_sigmas(10, 3)[:8]
    for bad_dt in (np.nan, np.inf, 0.0, -0.3):
        d = np.full(8, 0.5)
        d[3] = bad_dt
        with pytest.raises(capi.FqError):
            solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], d, sig)
    x0 = pb["x0"].copy()
    x0[4] = np.nan
    with pytest.raises(capi.FqError):
        solver.solve_batch(10, x0, pb["xf"], pb["lim"], pb["polys"], np.full(8, 0.5), sig)
    with pytest.raises(capi.FqError):
        solver.gen_new_traj(10, x0, pb["xf"], pb["lim"], pb["polys"], np.arange(1, 4) * 0.3, sig)
    # device-pointer entry with poisoned data: must terminate and flag everything infeasible
    dev = torch.device("cuda", 0)
    P, fo, Ab = capi.pack_polys(pb["polys"])
    for poison in ("dt", "x0", "Ab"):
        for generic in (0, 1):
            solver.set_option("force_generic_kernel", generic)
            dts = np.full(8, 0.5)
            x0 = pb["x0"].copy()
            Abp = Ab.copy()
            if poison == "dt":
                dts[:] = [np.nan, np.inf, 0.0, -1.0, np.nan, 1e308, 1e-308, np.nan]
            elif poison == "x0":
                x0[0] = np.nan
            else:
                Abp[2, 1] = np.inf
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
            d = dict(x0=t(x0), xf=t(pb["xf"]), lim=t(pb["lim"]), po=t(np.array([0, P], np.int32)), fo=t(fo), Ab=t(Abp),
                     co=t(np.array([0, 8], np.int32)), dt=t(dts), sg=t(sig))
            feas = torch.ones(8, dtype=torch.uint8, device=dev)
            cost = torch.zeros(8, dtype=torch.float64, device=dev)
            torch.cuda.synchronize()    # torch's fills run on its own stream, the library on the context's
            solver.solve_multi_dev(10, True, 1, d["x0"].data_ptr(), d["xf"].data_ptr(), d["lim"].data_ptr(),
                                   d["po"].data_ptr(), d["fo"].data_ptr(), d["Ab"].data_ptr(), d["co"].data_ptr(), 8,
                                   int(fo[-1]), d["dt"].data_ptr(), d["sg"].data_ptr(), feas.data_ptr(), cost.data_ptr())
            torch.cuda.synchronize()
            f = feas.cpu().numpy()
            if poison == "dt":
                assert not f[[0, 1, 2, 3, 4, 7]].any()
            else:
                assert not f.any()
    solver.set_option("force_generic_kernel", 0)


def test_cuda_reproduces_committed_goldens(solver, demo_corridor):
    """CUDA path against the committed golden vectors (tests/golden/corridor_continuous_expected.json)."""
    import json
    import os
    exp = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "corridor_continuous_expected.json")))
    fx = demo_corridor
    sig = np.array(exp["sigmas"], np.uint8)
    for dt, fe, ce in zip(exp["dts"], exp["feasible"], exp["cost"]):
        f, c, co, _ = solver.solve_batch(fx["N"], fx["x0"], fx["xf"], fx["lim"], fx["polys"], np.full(len(sig), dt), sig, True, True)
        assert f.tolist() == fe
        for k, v in enumerate(ce):
            if v is not None:
                assert abs(c[k] - v) <= REL * max(1.0, v)
        key = "%g" % dt
        if key in exp["best_coeffs"]:
            b = exp["best_coeffs"][key]
            assert np.abs(co[b["sigma_index"]] - np.array(b["coeffs"])).max() <= 1e-6
    e = exp["gen_new_traj"]
    dti = capi.dt_initial(fx["x0"], fx["xf"], fx["lim"], fx["N"])
    g = solver.gen_new_traj(fx["N"], fx["x0"], fx["xf"], fx["lim"], fx["polys"], np.arange(1.0, 11.0) * max(dti, 0.02), sig, True)
    assert g["solved"] == e["solved"] and g["dt_index"] + 1 == e["trials"] and abs(g["cost"] - e["cost"]) <= REL * e["cost"]


def test_device_side_fill_x_matches_host(solver, oracle, demo_corridor):
    """fq_gen_new_traj_sampled (fillX chained on the device) == fq_gen_new_traj + host fq_fill_x == oracle fillX."""
    fx = demo_corridor
    cases = [(fx["N"], fx["x0"], fx["xf"], fx["lim"], fx["polys"], True)]
    for seed in range(3):
        pb = cr.make_corridor(1300 + seed, 3, 6, force_final=bool(seed % 2))
        cases.append((6, pb["x0"], pb["xf"], pb["lim"], pb["polys"], bool(seed % 2)))
    DC = 0.01
    n = 0
    for N, x0, xf, lim, polys, ff in cases:
        sig = cr.monotone_sigmas(N, len(polys))
        dts = np.arange(1.0, 11.0) * max(capi.dt_initial(x0, xf, lim, N), 2 * DC)
        a = solver.gen_new_traj(N, x0, xf, lim, polys, dts, sig, ff)
        b = solver.gen_new_traj_sampled(N, x0, xf, lim, polys, dts, sig, DC, ff)
        assert a["solved"] == b["solved"] and a["dt_index"] == b["dt_index"] and a["cost"] == b["cost"]
        if a["solved"]:
            dt = dts[a["dt_index"]]
            Xh = capi.fill_x(N, a["coeffs"], dt, DC)
            Xo = oracle.fill_x(N, a["coeffs"], dt, DC)
            assert b["X"].shape == Xh.shape == Xo.shape
            assert np.allclose(b["X"], Xh, rtol=1e-12, atol=1e-12) and np.allclose(b["X"], Xo, rtol=1e-12, atol=1e-12)
            assert np.all(b["X"][-1, 3:] == 0)
            n += 1
    assert n >= 2


def test_huge_polytopes_fall_back_to_generic_kernel(solver, oracle):
    """Polytopes with hundreds of faces exceed the specialised kernel's per-warp row list in shared memory: the launch
    falls back to the size-generic kernel and still agrees with the oracle."""
    rng = np.random.default_rng(77)
    pb = cr.make_corridor(61, 3, 10)
    fat = []
    for (A, b), (v0, v1) in zip(pb["polys"], zip(pb["verts"][:-1], pb["verts"][1:])):
        mid = 0.5 * (v0 + v1)
        n = rng.normal(size=(700 - len(b), 3))
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        fat.append((np.vstack([A, n]), np.concatenate([b, n @ mid + rng.uniform(2.5, 4.0, len(n))])))
    sig = cr.monotone_sigmas(10, 3)[::3]
    dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], 10)
    dts = np.repeat(np.array([1.5, 2.5, 4.0]) * dti, len(sig))
    sigs = np.tile(sig, (3, 1))
    fg, cg, cog, _ = solver.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], fat, dts, sigs, True, True)
    fo, co_, coo = oracle.solve_batch(10, pb["x0"], pb["xf"], pb["lim"], fat, dts, sigs, True, True, threads=8)
    _compare(fg, cg, cog, fo, co_, coo, "700-face polytopes")


def test_exact_miqp_branch_and_bound_on_gpu(solver, oracle):
    """fq_gen_new_traj_exact (GPU branch-and-bound over all P^N assignments) against the oracle's branch-and-bound:
    per time allocation (incl. the known cases where the best non-decreasing assignment is NOT optimal) and as a sweep."""
    # (seed, N, P, force_final, factor): the three non-monotone optima found by the round-1 study + ordinary cases
    cases = [(5007, 10, 3, True, 5.0), (5007, 6, 3, True, 5.0), (5055, 10, 4, False, 5.0)]
    cases += [(5000 + s, N, P, ff, f) for s in range(6) for (N, P, ff) in ((10, 3, True), (10, 4, False), (6, 3, False)) for f in (2.0, 3.0)]
    n_nonmono = 0
    for seed, N, P, ff, f in cases:
        pb = cr.make_corridor(seed, P, N, "uav", ff)
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        dt = f * max(dti, 0.02)
        g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [dt], ff)
        rc, c, co, sg, nodes = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], ff)
        assert g["exact"], (seed, N, P)
        assert g["solved"] == (rc == 1), (seed, N, P, f)
        if rc == 1:
            assert abs(g["cost"] - c) <= REL * max(1.0, c), (seed, N, P, f, g["cost"], c)
            assert np.abs(g["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max())
            if np.any(np.diff(g["sigma"].astype(int)) < 0):
                n_nonmono += 1
            # the returned assignment really attains the cost
            r2, c2, _, _ = oracle.solve_fixed(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], g["sigma"], ff)
            assert r2 == 1 and abs(c2 - c) <= 1e-9 * max(1.0, c)
    assert n_nonmono >= 2          # the study's cases are reproduced: the exact optimum is not monotone there
    # sweeps (first feasible factor wins) on synthetic and forest corridors
    for seed in range(8):
        for kind in ("synthetic", "forest"):
            try:
                pb = cr.make_corridor(7000 + seed, 3, 10) if kind == "synthetic" else cr.make_forest_corridor(7100 + seed, 3, 10, True)
            except RuntimeError:
                continue
            dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], 10)
            dts = np.arange(1.0, 11.0) * max(dti, 0.02)
            g = solver.gen_new_traj_exact(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, True)
            o = oracle.gen_new_traj(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], 0.01, 1.0, 10.0, 1.0, None, True)
            assert g["exact"] and g["solved"] == o["solved"]
            if o["solved"]:
                assert g["dt_index"] + 1 == o["trials"] and abs(g["cost"] - o["cost"]) <= REL * max(1.0, o["cost"])


@pytest.mark.parametrize("N", [4, 5, 8, 11, 13, 14, 16])
@pytest.mark.parametrize("ff", [True, False])
def test_exact_miqp_branch_and_bound_across_shapes(solver, oracle, N, ff):
    """The branch-and-bound level kernel (fqb::launch_level<N, WHOLE>) on the lane-layout boundaries, whole and safe mode,
    against the oracle's branch-and-bound: single time allocations (solve_miqp) and sweeps (gen_new_traj over all
    assignments).  Two or three polytopes keep the trees small enough that the node pool cannot overflow: exact = 1."""
    P = 3 if N <= 11 else 2
    n_solved = n_unsolved = 0
    for seed in range(3):
        pb = cr.make_corridor(63000 + 31 * N + seed, P, N, "uav", ff)
        base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        for f in ((1.0, 2.0, 4.0) if ff else (0.3, 0.6, 2.0)):
            g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [f * base], ff)
            rc, c, co, _, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], f * base, pb["polys"], ff)
            what = (N, ff, seed, f)
            assert g["exact"], what
            assert g["solved"] == (rc == 1), what
            if rc == 1:
                n_solved += 1
                assert abs(g["cost"] - c) <= REL * max(1.0, c), what
                assert np.abs(g["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max()), what
                r2, c2, _, _ = oracle.solve_fixed(N, pb["x0"], pb["xf"], pb["lim"], f * base, pb["polys"], g["sigma"], ff)
                assert r2 == 1 and abs(c2 - c) <= 1e-9 * max(1.0, c), what
            else:
                n_unsolved += 1
        f0 = 1.0 if ff else 0.3
        facs = [f0]
        while facs[-1] + f0 <= 10.0 * f0:                        # the oracle's factor loop, with its rounding
            facs.append(facs[-1] + f0)
        facs = np.array(facs)
        g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], facs * base, ff)
        o = oracle.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], 0.01, f0, 10.0 * f0, f0, None, ff)
        assert g["exact"] and g["solved"] == o["solved"], (N, ff, seed)
        if o["solved"]:
            assert g["dt_index"] + 1 == o["trials"] and abs(g["cost"] - o["cost"]) <= REL * max(1.0, o["cost"]), (N, ff, seed)
    assert n_solved >= 2 and n_unsolved >= 1, (n_solved, n_unsolved)


def test_full_host_pipeline_then_gpu_solve(solver, oracle):
    """BASELINE config 4's chain with the product's own host code at every step: voxelised random forest ->
    fq_jps3d_plan_world -> fq_ellipsoid_decomp -> exact whole sweep on the GPU; checked against the numpy decomposition
    oracle and the solver oracle (branch-and-bound over all assignments) on the same JPS path."""
    from oracle import decomp_oracle as do
    n = 0
    for seed in range(500, 510):
        try:
            pb = cr.make_jps_forest_corridor(seed, 3, 10)
        except RuntimeError:
            continue
        polys_o = do.cvx_ellipsoid_decomp(pb["verts"], pb["obs"], (2.0, 2.0, 1.0), 0.42, 0.0)
        for (A1, b1), (A2, b2) in zip(pb["polys"], polys_o):
            assert A1.shape == A2.shape
            r1 = np.hstack([A1, b1[:, None]]); r2 = np.hstack([A2, b2[:, None]])
            r1 = r1[np.lexsort(np.round(r1, 7).T[::-1])]; r2 = r2[np.lexsort(np.round(r2, 7).T[::-1])]
            assert np.abs(r1 - r2).max() <= 1e-9
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], 10)
        dts = np.arange(1.0, 11.0) * max(dti, 0.02)
        g = solver.gen_new_traj_exact(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, True)
        o = oracle.gen_new_traj(10, pb["x0"], pb["xf"], pb["lim"], pb["polys"], 0.01, 1.0, 10.0, 1.0, None, True)
        assert g["exact"] and g["solved"] == o["solved"]
        if o["solved"]:
            assert g["dt_index"] + 1 == o["trials"] and abs(g["cost"] - o["cost"]) <= REL * max(1.0, o["cost"])
            # the solved trajectory stays clear of the (un-inflated) obstacle cells by the drone radius along its knots
            X = capi.fill_x(10, g["coeffs"], dts[g["dt_index"]], 0.01)[::10, :3]
            d = np.linalg.norm(pb["obs"][None, :, :] - X[:, None, :], axis=2).min()
            assert d > 0.3
            n += 1
    assert n >= 5


def test_wrong_polytope_size_hint_is_refused_not_overrun(solver):
    """The device-pointer entry trusts the caller's "max_faces_per_polytope" hint to size the per-warp row list; a hint
    that is too small must make the affected candidates "not solved" (iters = -2), never write past the list."""
    import torch
    pb = cr.make_corridor(41, 3, 10)
    sig = cr.monotone_sigmas(10, 3)[:16]
    P, fo, Ab = capi.pack_polys(pb["polys"])
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d = dict(x0=t(pb["x0"]), xf=t(pb["xf"]), lim=t(pb["lim"]), po=t(np.array([0, P], np.int32)), fo=t(fo), Ab=t(Ab),
             co=t(np.array([0, 16], np.int32)), dt=t(np.full(16, 0.6)), sg=t(sig))
    res = {}
    for hint in (2, int(np.diff(fo).max())):
        solver.set_option("max_faces_per_polytope", hint)
        feas = torch.ones(16, dtype=torch.uint8, device=dev)
        cost = torch.zeros(16, dtype=torch.float64, device=dev)
        iters = torch.zeros(16, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()        # torch's fills run on its own stream, the library on the context's (found by racecheck's timing)
        solver.solve_multi_dev(10, True, 1, d["x0"].data_ptr(), d["xf"].data_ptr(), d["lim"].data_ptr(), d["po"].data_ptr(),
                               d["fo"].data_ptr(), d["Ab"].data_ptr(), d["co"].data_ptr(), 16, int(fo[-1]), d["dt"].data_ptr(),
                               d["sg"].data_ptr(), feas.data_ptr(), cost.data_ptr(), 0, iters.data_ptr())
        torch.cuda.synchronize()
        res[hint] = (feas.cpu().numpy(), iters.cpu().numpy())
    solver.set_option("max_faces_per_polytope", 0)
    assert not res[2][0].any() and (res[2][1] == -2).all()
    assert res[int(np.diff(fo).max())][0].any()
    # the other hint, max_faces_per_prob (sizes the staged copy of the problem's rows), too small: the rows are not staged
    # at all and every candidate of the problem is "not solved" with iters = -2 (ADVICE round 1), for both kernels
    for generic in (0, 1):
        solver.set_option("force_generic_kernel", generic)
        feas = torch.ones(16, dtype=torch.uint8, device=dev)
        cost = torch.zeros(16, dtype=torch.float64, device=dev)
        iters = torch.zeros(16, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()        # torch's fills run on its own stream, the library on the context's (found by racecheck's timing)
        solver.solve_multi_dev(10, True, 1, d["x0"].data_ptr(), d["xf"].data_ptr(), d["lim"].data_ptr(), d["po"].data_ptr(),
                               d["fo"].data_ptr(), d["Ab"].data_ptr(), d["co"].data_ptr(), 16, int(fo[-1]) - 3, d["dt"].data_ptr(),
                               d["sg"].data_ptr(), feas.data_ptr(), cost.data_ptr(), 0, iters.data_ptr())
        torch.cuda.synchronize()
        assert not feas.cpu().numpy().any() and (iters.cpu().numpy() == -2).all() and np.isinf(cost.cpu().numpy()).all()
    solver.set_option("force_generic_kernel", 0)


@pytest.mark.gpu
def test_full_active_set_is_handled(solver, oracle):
    """N = 15, free final position: 39 unknowns, and many infeasible candidates are only refuted once the active set holds
    39 rows.  With a full active set every further row is dependent by definition; the solver must say so whatever
    rounding leaves in the projection (round 2: a corridor of this family made the active set grow past its storage --
    found by tools/stress_shapes.py under compute-sanitizer, fixed by the q >= NW guard).  Same corridors as that run."""
    N, ff, P = 15, False, 8
    rng = np.random.default_rng(N * 1000 + P * 10 + int(ff))
    mono = cr.sample_monotone_sigmas(N, P, 256, rng)
    for c in range(4):
        pb = cr.make_corridor(50000 + 97 * N + c, P, N, "uav", ff)
        dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
        sig = np.vstack([mono[rng.choice(len(mono), 40, replace=False)], rng.integers(0, P, size=(24, N)).astype(np.uint8)])
        dts = np.repeat(np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0]) * max(dti, 2 * pb["DC"]), len(sig))
        sigs = np.tile(sig, (6, 1))
        fo, co, _ = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, False, threads=8)
        for generic in (0, 1):
            solver.set_option("force_generic_kernel", generic)
            fg, cg, _, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, False, True)
            assert np.array_equal(fg, fo)
            assert (it >= 0).all()                              # no iteration-cap / numeric give-ups either
            ok = fo.astype(bool)
            assert (np.abs(cg[ok] - co[ok]) / np.abs(co[ok])).max() < REL
    solver.set_option("force_generic_kernel", 0)
