"""The product's CUDA kernel SOURCE, executed without a GPU: faster_b200/csrc/fq_kernels_t.cuh (fq_solve_kernel_t: persistent CTAs,
claim counters, row staging, item lists, the warp-per-candidate dual active-set iteration) is compiled for the host and run under
a lock-step emulation of one thread block (tests/cpp/simt_emu/: every CUDA thread is a fibre, warp collectives and block barriers
are rendezvous points) and compared with the CPU restatement.  This checks the kernel's LOGIC in a container that has no GPU
and is what the `-m gpu` parity tests then confirm on the hardware.  It is test
infrastructure, not a CPU path of the product (the library still refuses to work without a GPU) and ~10^4 times too slow to be one."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def _emu():
    """The harness (built under tests/cpp/_build, rebuilt when a source is newer)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    out = os.path.join(ROOT, "tests", "cpp", "_build", "libkernel_emu.so")
    srcs = [os.path.join(ROOT, "tests", "cpp", "kernel_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
            os.path.join(ROOT, "faster_b200", "csrc", "fq_kernels_t.cuh"), os.path.join(ROOT, "faster_b200", "csrc", "fq_kernels.cuh")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w",
                               "-I", os.path.join(ROOT, "tests", "cpp"), "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"),
                               "-I", os.path.join(ROOT, "faster_b200", "csrc"), "-I", os.path.join(ROOT, "include"), srcs[0], "-o", out])
    L = C.CDLL(out)
    L.emu_solve_multi.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int] + \
                                 [C.c_void_p] * 3 + [C.c_double] + [C.c_void_p] * 4
    L.emu_set_sweep.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_set_sweep.restype = None
    _LIB = L
    return L


def solve_multi(L, N, ff, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dts, sigmas, row_tol=1e-8, max_faces=None, max_poly_faces=None):
    """fq_solve_multi's layout through ONE emulated CTA of the product kernel -> (feasible, cost, coeffs, iters)."""
    TZ, T0, FT = [np.ascontiguousarray(t, np.float64) for t in capi.plan_tables(N, ff)]
    c = lambda a, t: np.ascontiguousarray(a, t)
    x0, xf, lim, Ab, dts = c(x0, np.float64), c(xf, np.float64), c(lim, np.float64), c(Ab, np.float64), c(dts, np.float64)
    poly_ofs, face_ofs, cand_ofs, sig = c(poly_ofs, np.int32), c(face_ofs, np.int32), c(cand_ofs, np.int32), c(sigmas, np.uint8)
    n_prob, n = len(cand_ofs) - 1, int(cand_ofs[-1])
    if max_faces is None:
        max_faces = int(max(face_ofs[poly_ofs[j + 1]] - face_ofs[poly_ofs[j]] for j in range(n_prob)))
    if max_poly_faces is None:
        max_poly_faces = int(np.diff(face_ofs).max()) if len(face_ofs) > 1 else 0
    feas, cost, co, it = np.zeros(n, np.uint8), np.zeros(n), np.zeros((n, N, 12)), np.zeros(n, np.int32)
    rc = L.emu_solve_multi(N, int(bool(ff)), TZ.ctypes.data, T0.ctypes.data, FT.ctypes.data, n_prob, x0.ctypes.data, xf.ctypes.data,
                           lim.ctypes.data, poly_ofs.ctypes.data, face_ofs.ctypes.data, Ab.ctypes.data, max_faces, max_poly_faces,
                           cand_ofs.ctypes.data, dts.ctypes.data, sig.ctypes.data, float(row_tol), feas.ctypes.data, cost.ctypes.data,
                           co.ctypes.data, it.ctypes.data)
    assert rc == 0, rc
    return feas, cost, co, it


def _batch(oracle, N, P, ff, profile, seeds, n_sig, factors, rng, change=None):
    """change(pb) -> corridor, if given, modifies each corridor (final state, probe rows) before it is packed."""
    x0, xf, lim, po_, fo, rows, co_, dts, sigs = [], [], [], [0], [0], [], [0], [], []
    for seed in seeds:
        pb = cr.make_corridor(seed, P, N, profile, ff)
        if change is not None:
            pb = change(pb)
        allm = cr.monotone_sigmas(N, P) if P <= 4 else cr.sample_monotone_sigmas(N, P, 200, rng)
        sig = np.vstack([allm[rng.choice(len(allm), min(n_sig - 2, len(allm)), replace=False)], rng.integers(0, P, (2, N)).astype(np.uint8)])
        base = max(oracle.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        x0.append(pb["x0"]); xf.append(pb["xf"]); lim.append(pb["lim"])
        for A, b in pb["polys"]:
            rows.append(np.hstack([A, np.asarray(b)[:, None]])); fo.append(fo[-1] + len(b))
        po_.append(po_[-1] + P)
        dts.append(np.repeat(np.asarray(factors) * base, len(sig))); sigs.append(np.tile(sig, (len(factors), 1)))
        co_.append(co_[-1] + len(dts[-1]))
    return (np.array(x0), np.array(xf), np.array(lim), np.array(po_), np.array(fo), np.vstack(rows), np.array(co_), np.concatenate(dts),
            np.vstack(sigs))


def _check(oracle, N, ff, b, got, tol=1e-9):
    out = oracle.solve_multi_port(N, ff, *b, threads=4, want_coeffs=True)      # the CPU restatement, per problem
    f, c, cc = out[0], out[1], out[2]
    assert np.array_equal(got[0], f), "flags differ at %s" % np.flatnonzero(got[0] != f)[:8]
    ok = f.astype(bool)
    assert ok.any() and (~ok).any()
    assert (np.abs(got[1][ok] - c[ok]) / np.maximum(1e-12, np.abs(c[ok]))).max() <= tol
    assert np.isinf(got[1][~ok]).all()
    assert np.abs(got[2][ok] - cc[ok].reshape(-1, N, 12)).max() <= 1e-7
    return int(ok.sum())


def test_demo_corridor_sweep_through_the_emulated_kernel(oracle, demo_corridor):
    """__graft_entry__.smoke()'s batch (the reference demo's corridor, 4 time allocations x 66 assignments) without a GPU."""
    fx = demo_corridor
    N = fx["N"]
    sig = cr.monotone_sigmas(N, 3)
    dts, sigs = np.repeat(np.array([0.6, 0.8, 1.0, 1.5]), len(sig)), np.tile(sig, (4, 1))
    fo = np.concatenate([[0], np.cumsum([len(b) for _, b in fx["polys"]])])
    Ab = np.vstack([np.hstack([A, np.asarray(b)[:, None]]) for A, b in fx["polys"]])
    got = solve_multi(_emu(), N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, len(dts)], dts, sigs)
    f, c, co = oracle.solve_batch(N, fx["x0"], fx["xf"], fx["lim"], fx["polys"], dts, sigs, True, True, threads=4)
    assert np.array_equal(got[0], f) and f.sum() == 61
    ok = f.astype(bool)
    assert (np.abs(got[1][ok] - c[ok]) / np.abs(c[ok])).max() < 1e-9 and np.abs(got[2][ok] - co[ok]).max() < 1e-7
    assert (got[3][ok] >= 0).all() and (got[3] != 0).all()


@pytest.mark.parametrize("name,N,P,ff,profile", [("cfg2", 10, 3, True, "uav"), ("cfg3", 10, 4, False, "uav"), ("cfg5", 15, 8, True, "ground"),
                                                  ("yaml", 6, 3, True, "uav"), ("small-safe", 4, 2, False, "uav"),
                                                  ("whole-5", 5, 2, True, "uav"), ("safe-11", 11, 3, False, "uav"),
                                                  ("safe-12", 12, 3, False, "uav"), ("whole-13", 13, 3, True, "uav"),
                                                  ("safe-13", 13, 4, False, "ground"), ("whole-14", 14, 4, True, "uav"),
                                                  ("safe-16", 16, 8, False, "uav"), ("whole-moving", 10, 3, True, "uav"),
                                                  ("safe-moving", 10, 3, False, "uav")])
def test_emulated_kernel_matches_the_cpu_restatement(oracle, name, N, P, ff, profile):
    """Several corridors per launch (warps adopt problems and claim candidates dynamically, as on the GPU), monotone and
    arbitrary assignments, whole and safe mode, one and two slots per lane (N = 15: 36 unknowns).  The added shapes sit on
    the lane-layout boundaries: the last one-slot shapes (whole 13, safe 12: 30 unknowns) and the first two-slot ones (whole
    14, safe 13: 33), N = 5 (one Y row per lane) and N = 11 (the first with three), and the largest safe shape.  The
    "moving" batches end in a moving final state (nonzero velocity and acceleration)."""
    from shape_cases import moving_final_state
    rng = np.random.default_rng(len(name) + N)
    b = _batch(oracle, N, P, ff, profile, [9100 + 7 * N + k for k in range(3)], 10, [0.3, 0.6, 1.0, 1.5, 2.0, 3.0, 5.0], rng,
               moving_final_state if name.endswith("moving") else None)
    got = solve_multi(_emu(), N, ff, *b)
    n_ok = _check(oracle, N, ff, b, got)
    assert n_ok >= 10
    assert (got[3] >= 0).all()


@pytest.mark.parametrize("ff,kind", [(True, "velocity"), (True, "x0_face"), (True, "xf_face"), (False, "x0_face")])
def test_emulated_kernel_honours_the_row_tolerance(oracle, ff, kind):
    """Corridors with one input-fixed row violated by 3e-7 (tests/shape_cases.py's probes) at row tolerance 1e-9 and 1e-3
    against the restatement and the tuned CPU port at the same tolerance: every probed candidate is infeasible at 1e-9,
    some are feasible at 1e-3, and the kernel never gives up."""
    from shape_cases import probe
    N, P = 10, 3
    rng = np.random.default_rng(17)
    seeds = [s for s in range(71000, 71100) if np.abs(cr.make_corridor(s, P, N, "uav", ff)["x0"][3:6]).max() >= 0.6][:2]
    b = _batch(oracle, N, P, ff, "uav", seeds, 10, [1.0, 2.0, 3.0, 5.0, 8.0], rng, lambda pb: probe(pb, kind))
    n_feas = {}
    try:
        for tol in (1e-9, 1e-3):
            oracle.set_row_tol(tol)
            oracle.port_lib().fqc_set_row_tol(tol)
            got = solve_multi(_emu(), N, ff, *b, row_tol=tol)
            assert (got[3] >= 0).all(), tol
            fo, _ = oracle.solve_multi(N, ff, *b, threads=4)
            assert np.array_equal(got[0], fo), tol
            f = got[0].astype(bool)
            if f.any() and (~f).any():
                _check(oracle, N, ff, b, got)
            n_feas[tol] = int(got[0].sum())
    finally:
        oracle.set_row_tol(1e-8)
        oracle.port_lib().fqc_set_row_tol(1e-8)
    assert n_feas[1e-9] == 0 and n_feas[1e-3] > 0, n_feas


def _prove_both(N, ff, b, i, answers, row_tol=1e-8):
    """Candidate i of a _batch: every answer (cost, coeffs) proved optimal on the literal model; their cost gap must stay
    below 2 row_tol times the larger multiplier sum (a point that violates rows by up to row_tol is at most that much cheaper)."""
    from oracle import model_fullspace as mf, proofs
    x0, xf, lim, po_, fo, Ab, co_, dts, sigs = b
    j = int(np.searchsorted(co_, i, side="right")) - 1
    polys = [(Ab[fo[p]:fo[p + 1], :3], Ab[fo[p]:fo[p + 1], 3]) for p in range(po_[j], po_[j + 1])]
    model = mf.build(N, x0[j], xf[j], lim[j], dts[i], polys, sigs[i], ff)
    lam = [proofs.assert_optimal(model, z, c, feas_tol=row_tol + 1e-7, active_tol=1e-9)["lam_sum"] for c, z in answers]
    assert abs(answers[0][0] - answers[1][0]) <= 2 * row_tol * max(lam) + 1e-12 * answers[1][0], (i, answers[0][0], answers[1][0])


@pytest.mark.parametrize("fam", ["fan", "dup", "slab", "near_parallel_1e-7", "near_parallel_1e-9", "near_parallel_1e-12", "x0_vertex"])
@pytest.mark.parametrize("N,ff,P", [(6, True, 3), (10, True, 3), (10, False, 3), (13, False, 4)])
def test_emulated_kernel_on_degenerate_corridors(oracle, fam, N, ff, P):
    """tests/degenerate_cases.py's families through the emulated kernel against the tuned CPU port: faces fanned through
    vertices and edges near the path, every face duplicated, the zero-width slab on the ground profile, copies rotated by
    1e-7, 1e-9 (the dependency cut-off) and 1e-12 rad about a line inside the polytope, x0 on a vertex.  Identical flags and
    no give-ups; fan and dup must also give the original corridor's answer.
    Near a near-parallel pair's crossing line both rows hold within the row tolerance on a wedge row_tol / theta wide (0.1 m
    at 1e-7, 10 m at 1e-9), so which row of the pair ends up active, and where, depends on the order the rows are picked in:
    the kernel and the port differ there by up to 2e-8 in cost.  A candidate beyond the 1e-9 cost or 1e-7 coefficient bar must
    then have both answers proved optimal, with a cost gap below the tolerance times the multipliers."""
    import degenerate_cases as dc
    change = {"fan": lambda pb: dc.fan(pb, 2), "dup": dc.dup, "slab": dc.slab, "x0_vertex": lambda pb: dc.on_boundary(pb, "x0", 3),
              "near_parallel_1e-7": lambda pb: dc.near_parallel(pb, 1e-7), "near_parallel_1e-9": lambda pb: dc.near_parallel(pb, 1e-9),
              "near_parallel_1e-12": lambda pb: dc.near_parallel(pb, 1e-12)}[fam]
    profile = "ground" if fam == "slab" else "uav"
    seeds, facs = [9300 + N + k for k in range(2)], [0.3, 0.6, 1.0, 2.0, 5.0]
    b = _batch(oracle, N, P, ff, profile, seeds, 8, facs, np.random.default_rng(N), change)
    got = solve_multi(_emu(), N, ff, *b)
    assert (got[3] >= 0).all()
    if not fam.startswith("near_parallel"):
        _check(oracle, N, ff, b, got)
    else:
        f, c, cc = oracle.solve_multi_port(N, ff, *b, threads=4, want_coeffs=True)
        assert np.array_equal(got[0], f) and f.any() and not f.all()
        ok = np.flatnonzero(f)
        rel = np.abs(got[1][ok] - c[ok]) / np.abs(c[ok])
        err = np.abs(got[2][ok] - cc[ok]).max(axis=(1, 2))
        for i in ok[(rel > 1e-9) | (err > 1e-7)]:
            _prove_both(N, ff, b, i, [(got[1][i], got[2][i]), (c[i], cc[i])])
    if fam in ("fan", "dup"):
        b0 = _batch(oracle, N, P, ff, profile, seeds, 8, facs, np.random.default_rng(N))
        got0 = solve_multi(_emu(), N, ff, *b0)
        ok = got0[0].astype(bool)
        assert np.array_equal(got[0], got0[0]) and (np.abs(got[1][ok] - got0[1][ok]) / got0[1][ok]).max() <= 1e-9
        assert np.abs(got[2][ok] - got0[2][ok]).max() <= 1e-7


def test_emulated_kernel_at_its_shared_memory_limit(oracle):
    """N = 10 whole with one polytope of ~950 faces: the largest problem the specialised kernel takes within an H100's 227 KB
    of shared memory (tests/capacity_cases.py), its rows tangent to a capsule around the path so that they bind, the original
    faces last (staged rows up to ~950, item lists of ~9500 entries).  Against the restatement."""
    import capacity_cases as cc
    N, ff, P = 10, True, 3
    pb = cr.make_corridor(86000, P, N, "uav", ff)
    base = [len(b) for _, b in pb["polys"]]
    n = cc.limit("spec", N, ff, "dominant", base)
    assert not cc.fits("spec", N, ff, cc.split_counts(n + 1, "dominant", base))
    pb = cc.with_faces(pb, n, "dominant", seed=1)
    counts = [len(b) for _, b in pb["polys"]]
    assert sum(counts) == n and max(counts) >= 900
    rng = np.random.default_rng(3)
    sig = np.vstack([cr.monotone_sigmas(N, P)[[0, 10, 30, 45, 65]], rng.integers(0, P, (1, N)).astype(np.uint8)])
    facs = [1.0, 2.0, 4.0]
    base_dt = max(oracle.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
    dts, sigs = np.repeat(np.array(facs) * base_dt, len(sig)), np.tile(sig, (len(facs), 1))
    Ab = np.vstack([np.hstack([A, np.asarray(b)[:, None]]) for A, b in pb["polys"]])
    fo = np.concatenate([[0], np.cumsum(counts)])
    b = ([pb["x0"]], [pb["xf"]], [pb["lim"]], [0, P], fo, Ab, [0, len(dts)], dts, sigs)
    got = solve_multi(_emu(), N, ff, *b)
    assert (got[3] >= 0).all()
    f, c, cc_ = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=4)
    assert np.array_equal(got[0], f) and f.any() and not f.all()
    ok = f.astype(bool)
    assert (np.abs(got[1][ok] - c[ok]) / c[ok]).max() <= 1e-9 and np.abs(got[2][ok] - cc_[ok]).max() <= 1e-7


def test_guards_of_the_kernel(oracle, demo_corridor):
    """What the kernel must refuse by itself because the device-pointer entry cannot validate it on the host: non-finite or
    non-positive inputs (candidate reported not solved, iters = -1), a row list that does not fit the caller's size hint
    (iters = -2) -- never an out-of-bounds access (the emulation runs under the host's address-space rules)."""
    fx = demo_corridor
    N = fx["N"]
    sig = cr.monotone_sigmas(N, 3)[:6]
    fo = np.concatenate([[0], np.cumsum([len(b) for _, b in fx["polys"]])])
    Ab = np.vstack([np.hstack([A, np.asarray(b)[:, None]]) for A, b in fx["polys"]])
    dts = np.array([0.8, np.nan, -1.0, 0.0, 1.0, np.inf])
    got = solve_multi(_emu(), N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, 6], dts, sig)
    assert list(got[3][[1, 2, 3, 5]]) == [-1, -1, -1, -1] and not got[0][[1, 2, 3, 5]].any() and np.isinf(got[1][[1, 2, 3, 5]]).all()
    assert got[3][0] > 0 and got[3][4] > 0
    x0 = np.array(fx["x0"], float)
    x0[4] = np.inf
    got = solve_multi(_emu(), N, True, [x0], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, 2], [0.8, 1.0], sig[:2])
    assert not got[0].any() and (got[3] == -1).all()
    # a size hint smaller than the problem's rows: the staging area is never overrun, the candidates are marked
    got = solve_multi(_emu(), N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, 2], [0.8, 1.0], sig[:2], max_faces=int(fo[-1]) - 3)
    assert not got[0].any() and (got[3] == -2).all()
    # a per-polytope hint that makes the item list too short for this assignment
    got = solve_multi(_emu(), N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, 2], [0.8, 1.0], sig[:2], max_poly_faces=2)
    assert not got[0].any() and (got[3] == -2).all()


def test_sweep_selection_and_early_exit_inside_the_kernel(oracle, demo_corridor):
    """The drop-in class's sweep (fq_gen_new_traj): candidates dt-major, the warp that finishes the LAST candidate selects
    genNewTraj's winner inside the kernel -- first time allocation with a feasible assignment, then minimum cost, then lowest
    index (solverGurobi.cpp:445-472) -- and writes the record a host-mapped buffer receives on the GPU.  With the early exit
    (first feasible factor wins) candidates beyond the winning time allocation are skipped (iters = -3) and the winner, its cost
    and its coefficients are the same."""
    fx = demo_corridor
    N = fx["N"]
    sig = cr.monotone_sigmas(N, 3)
    facs = np.array([0.3, 0.5, 0.6, 0.8, 1.0, 1.5, 2.0])
    dts, sigs = np.repeat(facs, len(sig)), np.tile(sig, (len(facs), 1))
    fo = np.concatenate([[0], np.cumsum([len(b) for _, b in fx["polys"]])])
    Ab = np.vstack([np.hstack([A, np.asarray(b)[:, None]]) for A, b in fx["polys"]])
    f, c, co = oracle.solve_batch(N, fx["x0"], fx["xf"], fx["lim"], fx["polys"], dts, sigs, True, True, threads=4)
    F = f.reshape(len(facs), len(sig)).astype(bool)
    dt_win = int(np.flatnonzero(F.any(axis=1))[0])
    cw = np.where(F[dt_win], c.reshape(len(facs), -1)[dt_win], np.inf)
    sig_win = int(np.argmin(cw))
    assert 0 < dt_win < len(facs) - 1                             # infeasible factors before the winner, feasible ones after it
    L = _emu()
    rec = {}
    for ee in (0, 1):
        idx, win = np.full(2, -7, np.int32), np.zeros(1 + 12 * N)
        L.emu_set_sweep(ee, len(sig), idx.ctypes.data, win.ctypes.data)
        got = solve_multi(L, N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, len(dts)], dts, sigs)
        assert list(idx) == [dt_win, sig_win], (ee, idx)
        k = dt_win * len(sig) + sig_win
        assert abs(win[0] - c[k]) <= 1e-9 * c[k] and np.abs(win[1:] - co[k].reshape(-1)).max() <= 1e-7
        upto = (dt_win + 1) * len(sig)
        assert np.array_equal(got[0][:upto], f[:upto])            # everything at or below the winning time allocation is solved
        rec[ee] = (win.copy(), got)
    assert rec[0][0].tobytes() == rec[1][0].tobytes()             # same winner record, bit for bit
    full, early = rec[0][1], rec[1][1]
    assert np.array_equal(full[0], f) and (full[3] != -3).all()
    skipped = early[3] == -3
    assert skipped.any() and not skipped[:upto].any() and not early[0][skipped].any()
    # no feasible candidate at all: the record says so
    idx, win = np.full(2, -7, np.int32), np.zeros(1 + 12 * N)
    L.emu_set_sweep(0, len(sig), idx.ctypes.data, win.ctypes.data)
    n2 = 2 * len(sig)
    got = solve_multi(L, N, True, [fx["x0"]], [fx["xf"]], [fx["lim"]], [0, 3], fo, Ab, [0, n2], dts[:n2] * 0.2, sigs[:n2])
    assert not got[0].any() and list(idx) == [-1, -1] and np.isinf(win[0])


# ---- the chained replan: every kernel of fq_replan_pairs_dev's submission (faster_b200/csrc/fq_pair_capi.cu:93-141) under emulation
_PAIR = None
RESULT_DT = np.dtype([("whole_dt_index", np.int32), ("whole_sigma_index", np.int32), ("safe_dt_index", np.int32), ("safe_sigma_index", np.int32),
                      ("whole_cost", np.float64), ("safe_cost", np.float64), ("whole_dt", np.float64), ("safe_dt", np.float64),
                      ("whole_dt_base", np.float64), ("safe_dt_base", np.float64), ("n_samples_whole", np.int32), ("k_safe", np.int32),
                      ("R", np.float64, (9,))])


def _pair_lib():
    global _PAIR
    if _PAIR is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_emu.so")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
                os.path.join(ROOT, "faster_b200", "csrc", "fq_pair.cuh"), os.path.join(ROOT, "faster_b200", "csrc", "fq_dtinit.h")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", os.path.join(ROOT, "faster_b200", "csrc"),
                                   "-I", os.path.join(ROOT, "include"), srcs[0], "-o", out])
        _PAIR = C.CDLL(out)
        for name in ("emu_dtbase", "emu_expand_grid", "emu_select_multi", "emu_pair_mid", "emu_pair_final"):
            getattr(_PAIR, name).restype = None
    return _PAIR


def _p(a):
    return C.c_void_p(a.ctypes.data)


def emulated_replan_pairs(w):
    """fq_replan_pairs_dev's submission, kernel by kernel, through the emulation: dt base -> grid -> whole sweep -> selection ->
    winners' coefficients -> R -> dt base (safe) -> grid -> safe sweep -> selection -> result records."""
    P, Nw, Ns, DC = w["n_prob"], w["N_whole"], w["N_safe"], w["DC"]
    K, L = _pair_lib(), _emu()
    c = lambda a, t: np.ascontiguousarray(a, t)
    x0, xfw, xfs, lim = c(w["x0"], np.float64), c(w["xf_whole"], np.float64), c(w["xf_safe"], np.float64), c(w["lim"], np.float64)
    out = {}
    st = {}
    for kind, N, ff, xs, xf in (("whole", Nw, True, x0, xfw), ("safe", Ns, False, None, xfs)):
        fac, sg = c(w["factors_" + kind], np.float64), c(w["sigmas_" + kind], np.uint8)
        nf, ns = len(fac), len(sg)
        n = P * nf * ns
        if kind == "safe":
            xs = st["x0_safe"]
        base = np.zeros(P)
        K.emu_dtbase(P, N, C.c_double(DC), _p(xs), _p(xf), _p(lim), _p(base))
        dt, sig, co = np.zeros(n), np.zeros((n, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_expand_grid(P, N, nf, ns, _p(fac), _p(sg), _p(base), _p(dt), _p(sig), _p(co))
        feas, cost, _, _ = solve_multi(L, N, ff, np.where(np.isfinite(xs), xs, np.nan), xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind],
                                       w["Ab_" + kind], co, dt, sig, max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        wi, wc, wdt, ws, wo = np.zeros(P, np.int32), np.zeros(P), np.zeros(P), np.zeros((P, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_select_multi(P, N, ns, _p(co), _p(dt), _p(sig), _p(feas), _p(cost), _p(wi), _p(wc), _p(wdt), _p(ws), _p(wo))
        # winners' coefficients: one candidate per corridor through the same solve kernel (losers: dt = NaN -> not solved)
        _, _, coeffs, _ = solve_multi(L, N, ff, np.where(np.isfinite(xs), xs, np.nan), xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind],
                                      w["Ab_" + kind], wo, wdt, ws, max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        st[kind] = dict(base=base, wi=wi, wc=wc, wdt=wdt, ns=ns)
        out["feasible_" + kind], out["cost_" + kind], out["coeffs_" + kind] = feas, cost, coeffs
        if kind == "whole":
            x0s, nsamp, ksafe = np.zeros((P, 9)), np.zeros(P, np.int32), np.zeros(P, np.int32)
            K.emu_pair_mid(P, N, C.c_double(DC), C.c_double(w["r_fraction"]), _p(c(coeffs, np.float64)), _p(wdt), _p(wi), _p(x0s), _p(nsamp), _p(ksafe))
            st["x0_safe"], st["nsamp"], st["ksafe"] = x0s, nsamp, ksafe
    res = np.zeros(P, RESULT_DT)
    assert RESULT_DT.itemsize == 144
    a, b = st["whole"], st["safe"]
    K.emu_pair_final(P, a["ns"], b["ns"], _p(a["wi"]), _p(b["wi"]), _p(st["nsamp"]), _p(st["ksafe"]), _p(a["wc"]), _p(b["wc"]), _p(a["wdt"]),
                     _p(b["wdt"]), _p(a["base"]), _p(b["base"]), _p(st["x0_safe"]), _p(res))
    out["results"] = res
    return out


def test_chained_replan_through_the_emulated_kernels(oracle):
    """The bench's hot path end to end without a GPU: corridors of the committed config-4 forest fixture through every kernel of
    the chain, against the CPU chain (oracle/fq_cpu_port.c's fqc_replan_pairs): the same time-allocation bases bit for bit, the
    same flags for all 2 x 1024 candidates per corridor, the same winners, R to rounding, costs to 1e-9."""
    import bench
    w = bench.load_cfg4(0, 3)
    got = emulated_replan_pairs(w)
    ref = oracle.replan_pairs_port(w, threads=4)
    r, q = got["results"], ref["results"]
    assert np.array_equal(r["whole_dt_base"], q["whole_dt_base"]) and np.array_equal(r["safe_dt_base"], q["safe_dt_base"])
    for k in ("whole", "safe"):
        assert np.array_equal(got["feasible_" + k], ref["feasible_" + k]), k
        ok = ref["feasible_" + k].astype(bool)
        assert (np.abs(got["cost_" + k][ok] - ref["cost_" + k][ok]) / np.abs(ref["cost_" + k][ok])).max() <= 1e-9
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(r[f], q[f]), f
    assert (r["whole_dt_index"] >= 0).all() and (r["safe_dt_index"] >= 0).any()
    assert np.abs(r["R"] - q["R"]).max() <= 1e-9 and np.allclose(r["whole_cost"], q["whole_cost"], rtol=1e-9) and \
        np.allclose(r["safe_cost"], q["safe_cost"], rtol=1e-9, equal_nan=True)
    assert np.abs(got["coeffs_whole"] - ref["coeffs_whole"]).max() <= 1e-7
