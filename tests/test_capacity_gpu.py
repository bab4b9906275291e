"""The solver at its size limits (tests/capacity_cases.py): where the library decides by SIZE which kernel runs, whether a
branch-and-bound answer is exact, or whether a problem is refused.

  * the size-specialised kernel up to its shared-memory limit, the size-generic one from one face beyond it -- for the
    batch solve, the sweep (whose selection runs inside the specialised kernel and as a separate launch after the generic
    one) and the chained replan;
  * the size-generic kernel up to its own limit, FQ_E_ARG one face beyond it;
  * the branch-and-bound up to 2047 faces (an item's 11-bit face field) and up to its shared-memory limit, exact = 0 beyond
    either, and when its node pool overflows;
  * FQ_MAX_POLY = 32 polytopes, and the refusal of 33.
Which kernel ran is read from the profiler, matched by exact name, so a drift between the limits mirrored in
capacity_cases.limit and the code fails here instead of quietly testing the wrong side.  Answers are compared with the CPU
restatement (oracle/fq_oracle.c) at the bar of tests/test_parity_gpu.py, and a sample is proved on the literal model."""
import math
import re

import numpy as np
import pytest

import capacity_cases as cc
from faster_b200 import capi, corridor as cr
from test_parity_gpu import REL, _compare

pytestmark = pytest.mark.gpu

FACTORS = np.array([1.0, 2.0, 3.0, 5.0])
SPEC, GENERIC, SELECT, BNB = "fq_solve_kernel_t", "fq_solve_kernel", "fq_select_kernel", "fq_bnb_level_kernel"
TOO_LARGE = "problem too large for shared memory"


def _kernel_name(name):
    """'void fqt::fq_solve_kernel_t<10, true>(FqKernelArgs, int*)' -> 'fq_solve_kernel_t'."""
    s = name.replace("(anonymous namespace)::", "")
    if s.startswith("void "):
        s = s[5:]
    return re.split(r"[<(]", s)[0].split("::")[-1].strip()


def kernels(fn, sessions=5):
    """-> (fn(), set of the names of the library's kernels it launched), recorded by the profiler's CUDA activity.  fn runs
    between two marker kernels, and only kernels that started between the markers count: a record the profiler delivers
    late, into a later session, is not attributed to the wrong call.  A session without both markers, or without a kernel
    of the library between them, is repeated (fn only reads its inputs); if none has one, the test fails."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    for _ in range(sessions):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
            out = fn()
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
        evs = [(e.time_range.start, _kernel_name(e.name)) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        marks = sorted(t for t, n in evs if n == "spin_kernel")
        if len(marks) >= 2:
            fq = {n for t, n in evs if n.startswith("fq_") and marks[-2] < t < marks[-1]}
            if fq:
                return out, fq
    raise AssertionError("the profiler recorded no kernel of the library in %d sessions" % sessions)


@pytest.fixture(scope="module")
def report():
    lines = []
    yield lines
    print("\n" + "\n".join(lines))


def candidates(pb, N, P, n_mono=4, n_arb=2, seed=0):
    rng = np.random.default_rng(seed)
    mono = cr.monotone_sigmas(N, P) if math.comb(N + P - 1, N) <= 5000 else cr.sample_monotone_sigmas(N, P, 64, rng)
    sig = np.vstack([mono[rng.choice(len(mono), min(n_mono, len(mono)), replace=False)],
                     rng.integers(0, P, (n_arb, N)).astype(np.uint8)])
    base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 2 * pb["DC"])
    return FACTORS * base, np.repeat(FACTORS * base, len(sig)), np.tile(sig, (len(FACTORS), 1)), sig


def solve(solver, N, pb, dts, sigs, ff, generic=False, profiled=True):
    """fq_solve_batch (default kernel choice, or force_generic_kernel) -> ((feasible, cost, coeffs), kernel names or None)."""
    solver.set_option("force_generic_kernel", int(generic))
    call = lambda: solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
    try:
        (f, c, co, it), names = kernels(call) if profiled else (call(), None)
    finally:
        solver.set_option("force_generic_kernel", 0)
    assert (it >= 0).all(), "iteration-cap or numeric give-ups at %s" % np.flatnonzero(it < 0)[:8]
    return (f, c, co), names


def restated_sweep(f, c, n_dt, n_sig):
    """genNewTraj's selection over a dt-major candidate list: first dt with a feasible assignment, then minimum cost."""
    F, Cc = f.reshape(n_dt, n_sig).astype(bool), c.reshape(n_dt, n_sig)
    rows = np.flatnonzero(F.any(axis=1))
    if not len(rows):
        return -1, -1
    d = int(rows[0])
    return d, int(np.argmin(np.where(F[d], Cc[d], np.inf)))


def check_sweep(g, f, c, co, n_dt, n_sig, what):
    d, s = restated_sweep(f, c, n_dt, n_sig)
    assert g["dt_index"] == d and g["solved"] == (d >= 0), (what, g["dt_index"], d)
    if d < 0:
        return
    k = d * n_sig + s
    kg = d * n_sig + g["sigma_index"]
    assert g["sigma_index"] == s or (f[kg] and abs(c[kg] - c[k]) <= REL * c[k]), (what, g["sigma_index"], s)   # or an exact tie
    assert abs(g["cost"] - c[k]) <= REL * c[k], what
    assert np.abs(g["coeffs"] - co[kg]).max() <= 1e-6 * max(1.0, np.abs(co[kg]).max()), what


# ---------------------------------------------------------------------------------------------------------------------
# 1. the specialised kernel's limit and the fall-back to the generic one
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("split", ["dominant", "even"])
@pytest.mark.parametrize("N,ff", [(4, True), (4, False), (10, True), (10, False), (16, True), (16, False)])
def test_specialised_limit_and_fallback(solver, oracle, report, N, ff, split):
    """Three polytopes with faces tangent to a capsule around the path, at the specialised kernel's limit and one face past
    it: fq_solve_batch with the default kernel and with force_generic_kernel, and fq_gen_new_traj (its winner selected in
    the specialised kernel's tail at the limit, by fq_select_kernel past it), against the restatement."""
    for k in range(8):                       # the first corridor of the series that has feasible candidates at the limit
        pb0 = cr.make_corridor(81000 + 31 * N + int(ff) + 1000 * k, 3, N, "uav", ff)
        base = [len(b) for _, b in pb0["polys"]]
        n_lim = cc.limit("spec", N, ff, split, base)
        pb = cc.with_faces(pb0, n_lim, split, seed=N)
        _, dts, sigs, _ = candidates(pb, N, 3, seed=N)
        if oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, threads=8)[0].any():
            break
    assert cc.fits("generic", N, ff, cc.split_counts(n_lim + 1, split, base))
    seen = {}
    for past in (False, True):
        n = n_lim + int(past)
        pb = cc.with_faces(pb0, n, split, seed=N)
        assert sum(len(b) for _, b in pb["polys"]) == n
        dt_list, dts, sigs, sig = candidates(pb, N, 3, seed=N)
        fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
        what = (N, ff, split, n)
        (fg, cg, cog), names = solve(solver, N, pb, dts, sigs, ff)
        assert names == ({GENERIC} if past else {SPEC}), (what, names)
        _compare(fg, cg, cog, fo, co_, coo, "default kernel %s" % (what,))
        (fg, cg, cog), names = solve(solver, N, pb, dts, sigs, ff, generic=True)
        assert names == {GENERIC}, (what, names)
        _compare(fg, cg, cog, fo, co_, coo, "generic kernel %s" % (what,))
        g, names = kernels(lambda: solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dt_list, sig, ff))
        assert names == ({GENERIC, SELECT} if past else {SPEC}), (what, names)
        check_sweep(g, fo, co_, coo, len(dt_list), len(sig), what)
        seen[past] = int(fo.sum())
        if N == 10 and not past:
            from test_degenerate_gpu import prove
            ok, bad = np.flatnonzero(fo)[:2], np.flatnonzero(~fo.astype(bool))[:2]
            prove(solver, N, pb, dts, sigs, ff, list(ok) + list(bad), fo, co_, coo)
    assert seen[False] > 0 and seen[True] > 0, seen           # both sides have feasible candidates and
    report.append("specialised limit N=%d %s %s: %d faces (largest polytope %d); generic from %d" % (
        N, "whole" if ff else "safe", split, n_lim, max(cc.split_counts(n_lim, split, base)), n_lim + 1))


# ---------------------------------------------------------------------------------------------------------------------
# 2. faces that never bind change nothing, wherever they are staged
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_faces", [500, 1200, 2000])
@pytest.mark.parametrize("N,ff", [(4, True), (10, True), (10, False), (16, False)])
def test_loose_padding_changes_nothing(solver, report, N, ff, n_faces):
    """The shape families of tests/shape_cases.py padded with provably slack faces to 500, 1200 and 2000 rows, the original
    (binding) rows last -- at 1200 and 2000 they sit above staged index 1023, at 2000 up to 1999.  Flags identical to the
    unpadded corridor's and costs within 1e-12, under the same kernel: with the default choice and with force_generic_kernel.
    Where the padded corridor no longer fits the specialised kernel, the unpadded one is run through the generic kernel.
    Which kernel that is follows from capacity_cases.limit, which test_specialised_limit_and_fallback checks with the
    profiler at every shape."""
    from shape_cases import shape_batches
    n_bits = n_cmp = n_spec = n_feas = 0
    for P, profile, c, pb, dts, sigs in shape_batches(N, ff, 1, n_mono=10, n_arb=6):
        pad = cc.pad_loose(pb, n_faces, binding_last=True, seed=P)
        counts = [len(b) for _, b in pad["polys"]]
        spec = cc.fits("spec", N, ff, counts)
        n_spec += spec
        for generic in (False, True):
            (f1, c1, co1), _ = solve(solver, N, pad, dts, sigs, ff, generic, profiled=False)
            (f0, c0, co0), _ = solve(solver, N, pb, dts, sigs, ff, generic or not spec, profiled=False)
            what = (N, ff, P, n_faces, generic)
            assert np.array_equal(f1, f0), (what, np.flatnonzero(f1 != f0)[:8])
            ok = f0.astype(bool)
            n_feas += int(ok.sum())
            assert (np.abs(c1[ok] - c0[ok]) / c0[ok]).max() <= 1e-12, what
            assert np.abs(co1[ok] - co0[ok]).max() <= 1e-9 * max(1.0, np.abs(co0[ok]).max()), what
            n_cmp += 1
            n_bits += c1.tobytes() == c0.tobytes() and co1.tobytes() == co0.tobytes()
    assert n_feas > 0
    if n_faces == 1200 and N <= 10:
        assert n_spec > 0            # the specialised kernel saw binding rows above index 1023
    report.append("loose padding N=%d %s to %d faces: %d/%d comparisons bit-identical (%d families on the specialised kernel)" % (
        N, "whole" if ff else "safe", n_faces, n_bits, n_cmp, n_spec))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the generic kernel's limit and the refusal beyond it
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,ff", [(10, True), (16, False)])
def test_generic_limit_and_refusal(solver, oracle, report, N, ff):
    pb0 = cr.make_corridor(82000 + N, 3, N, "uav", ff)
    base = [len(b) for _, b in pb0["polys"]]
    n_lim = cc.limit("generic", N, ff, "even", base)
    pb = cc.with_faces(pb0, n_lim, "even", seed=N)
    dt_list, dts, sigs, sig = candidates(pb, N, 3, n_mono=3, n_arb=1, seed=N)
    fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
    (fg, cg, cog), names = solve(solver, N, pb, dts, sigs, ff)
    assert names == {GENERIC}, names
    _compare(fg, cg, cog, fo, co_, coo, "generic limit")
    assert fo.any()
    big = cc.with_faces(pb0, n_lim + 1, "even", seed=N)
    with pytest.raises(capi.FqError, match=TOO_LARGE):
        solver.solve_batch(N, big["x0"], big["xf"], big["lim"], big["polys"], dts, sigs, ff)
    with pytest.raises(capi.FqError, match=TOO_LARGE):
        solver.gen_new_traj(N, big["x0"], big["xf"], big["lim"], big["polys"], dt_list, sig, ff)
    small = cr.make_corridor(82100 + N, 3, 10, "uav", True)
    whole, safe = (big, cr.make_corridor(82200, 4, 10, "uav", False)) if ff else (small, big)
    w = capi.make_pair_workload([whole], [safe], [1.0, 2.0, 4.0], cr.monotone_sigmas(whole["N"], 3)[:8], [1.0, 2.0, 4.0],
                                cr.monotone_sigmas(safe["N"], len(safe["polys"]))[:8], DC=0.01, r_fraction=0.3)
    with pytest.raises(capi.FqError, match=TOO_LARGE):
        solver.replan_pairs(w)
    # the context still works
    dl, d2, s2, _ = candidates(small, 10, 3, seed=1)
    f, c, co, _ = solver.solve_batch(10, small["x0"], small["xf"], small["lim"], small["polys"], d2, s2, True, True)
    _compare(f, c, co, *oracle.solve_batch(10, small["x0"], small["xf"], small["lim"], small["polys"], d2, s2, True, True, threads=8),
             "after the refusals")
    report.append("generic limit N=%d %s: %d faces solved, %d refused" % (N, "whole" if ff else "safe", n_lim, n_lim + 1))


# ---------------------------------------------------------------------------------------------------------------------
# 4. the branch-and-bound at its face cap and at its shared-memory limit
# ---------------------------------------------------------------------------------------------------------------------
def exact(solver, N, pb, dts, ff):
    return kernels(lambda: solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, ff))


def monotone_sweep(solver, N, pb, dts, ff):
    mono = capi.monotone_sigmas(N, len(pb["polys"]))
    g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, mono, ff)
    return g, mono


def assert_is_monotone_optimum(solver, N, pb, dts, ff, e, what):
    """exact = 0: the answer is the non-decreasing optimum of fq_gen_new_traj over fq_monotone_sigmas, bit for bit."""
    g, mono = monotone_sweep(solver, N, pb, dts, ff)
    assert not e["exact"], what
    assert e["solved"] == g["solved"] and e["dt_index"] == g["dt_index"], what
    if g["solved"]:
        assert np.array_equal(e["sigma"], mono[g["sigma_index"]]), what
        assert e["cost"] == g["cost"] and e["coeffs"].tobytes() == g["coeffs"].tobytes(), what


@pytest.mark.parametrize("seed,N,P,ff", [(5007, 10, 3, True), (5055, 10, 4, False)])
def test_branch_and_bound_at_its_face_cap(solver, oracle, report, seed, N, P, ff):
    """Corridors whose exact optimum is not non-decreasing, padded with slack faces (binding rows last): at 2047 faces the
    tree runs and finds it (exact = 1); at 2048 the 16-bit item list cannot name the rows and the answer is the
    non-decreasing optimum (exact = 0), whose cost is strictly higher."""
    pb = cr.make_corridor(seed, P, N, "uav", ff)
    dt = 5.0 * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
    g0 = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [dt], ff)
    rc, c, co, sg, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], ff)
    assert g0["exact"] and g0["solved"] and rc == 1 and np.any(np.diff(g0["sigma"].astype(int)) < 0)
    pad = cc.pad_loose(pb, cc.ITEM_FACE_CAP, binding_last=True, seed=seed)
    assert cc.fits("bnb", N, ff, [len(b) for _, b in pad["polys"]])
    e, names = exact(solver, N, pad, [dt], ff)
    assert BNB in names, names
    assert e["exact"] and e["solved"] and e["dt_index"] == 0, e
    assert abs(e["cost"] - g0["cost"]) <= 1e-12 * g0["cost"] and abs(e["cost"] - c) <= REL * c
    # the assignment: g0's, or one that ties with it exactly (here the first and last segments' polytopes can be swapped
    # without changing the optimum, and which of the tied leaves the tree keeps depends on the order warps finish in)
    r2, c2, _, _ = oracle.solve_fixed(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], e["sigma"], ff)
    assert r2 == 1 and abs(c2 - c) <= 1e-9 * c, (e["sigma"], g0["sigma"])
    assert np.any(np.diff(e["sigma"].astype(int)) < 0)
    pad2 = cc.pad_loose(pb, cc.ITEM_FACE_CAP + 1, binding_last=True, seed=seed)
    e2, names = exact(solver, N, pad2, [dt], ff)
    assert BNB not in names, names
    assert_is_monotone_optimum(solver, N, pad2, [dt], ff, e2, (seed, "2048 faces"))
    assert e2["solved"] and e2["cost"] > e["cost"], (e2["cost"], e["cost"])
    report.append("branch-and-bound seed %d: exact at %d faces (cost %.9g), non-decreasing optimum at %d (cost %.9g)" % (
        seed, cc.ITEM_FACE_CAP, e["cost"], cc.ITEM_FACE_CAP + 1, e2["cost"]))


def test_branch_and_bound_at_its_shared_memory_limit(solver, oracle, report):
    """N = 16 safe, two polytopes, one of which holds almost every (slack) face: at the level kernel's shared-memory limit
    the tree runs (exact = 1, the oracle's branch-and-bound optimum); one face more and the launch is refused, which the
    library reports as exact = 0 with the non-decreasing optimum."""
    N, ff, P = 16, False, 2
    pb = cr.make_corridor(63000 + 31 * N, P, N, "uav", ff)
    dt = 2.0 * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
    base = [len(b) for _, b in pb["polys"]]
    n_lim = cc.limit("bnb", N, ff, "dominant", base)
    assert n_lim < cc.ITEM_FACE_CAP
    rc, c, co, _, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], ff)
    assert rc == 1
    pad = cc.pad_loose(pb, n_lim, binding_last=True, seed=1, split="dominant")
    e, names = exact(solver, N, pad, [dt], ff)
    assert BNB in names and e["exact"] and e["solved"], (names, e["exact"])
    assert abs(e["cost"] - c) <= REL * c and np.abs(e["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max())
    pad2 = cc.pad_loose(pb, n_lim + 1, binding_last=True, seed=1, split="dominant")
    e2, names = exact(solver, N, pad2, [dt], ff)
    assert BNB not in names, names
    assert_is_monotone_optimum(solver, N, pad2, [dt], ff, e2, "bnb shared-memory limit + 1")
    report.append("branch-and-bound N=16 safe, one polytope of %d: exact at %d faces, exact = 0 at %d" % (
        max(cc.split_counts(n_lim, "dominant", base)), n_lim, n_lim + 1))


# ---------------------------------------------------------------------------------------------------------------------
# 5. the tree cut: node-pool overflow
# ---------------------------------------------------------------------------------------------------------------------
# (seed, whole, factor, copies): the first and the last two overflow the pool, the others do not
TREE_CASES = [(5007, True, 5.0, 3), (5007, True, 5.0, 2), (5034, False, 3.0, 2), (5021, False, 5.0, 2), (5021, False, 5.0, 3)]


def test_tree_cut_falls_back_to_the_monotone_optimum(solver, report):
    """Every polytope of a three-polytope corridor repeated two or three times: equal subtrees multiply the nodes that
    survive the bound until a level has more than the pool's 65536 children.  exact = 0 must then be the corridor's
    non-decreasing optimum bit for bit, exact = 1 the unduplicated corridor's exact answer."""
    N, P = 10, 3
    n_cut = 0
    for seed, ff, f, copies in TREE_CASES:
        pb = cr.make_corridor(seed, P, N, "uav", ff)
        dt = f * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        g0 = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [dt], ff)
        assert g0["exact"]
        dup = cc.duplicate_polytopes(pb, copies)
        if math.comb(N + len(dup["polys"]) - 1, N) > (1 << 20):
            continue
        e = solver.gen_new_traj_exact(N, dup["x0"], dup["xf"], dup["lim"], dup["polys"], [dt], ff)
        what = (seed, ff, f, copies, e["nodes"])
        if e["exact"]:
            assert e["solved"] == g0["solved"] and e["dt_index"] == g0["dt_index"], what
            if g0["solved"]:
                assert abs(e["cost"] - g0["cost"]) <= REL * g0["cost"], what
        else:
            n_cut += 1
            assert_is_monotone_optimum(solver, N, dup, [dt], ff, e, what)
        report.append("tree cut: seed %d %s factor %.1f x%d copies: exact = %d after %d nodes" % (
            seed, "whole" if ff else "safe", f, copies, e["exact"], e["nodes"]))
    assert n_cut >= 1, "no case overflowed the node pool"
    pb = cr.make_corridor(5007, 16, N, "uav", True)
    with pytest.raises(capi.FqError, match="assignment list too long"):
        solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [1.0], True)


# ---------------------------------------------------------------------------------------------------------------------
# 6. FQ_MAX_POLY polytopes
# ---------------------------------------------------------------------------------------------------------------------
def many_polytopes(seed, N, ff, P):
    """P polytopes over a three-segment path: polytope j is the base polytope of segment floor(3 j / P) with two capsule
    tangent faces of its own, so that neighbouring polytopes overlap and non-decreasing assignments can be feasible."""
    pb = cr.make_corridor(seed, 3, N, "uav", ff)
    polys = []
    rng = np.random.default_rng(seed)
    for j in range(P):
        s = 3 * j // P
        A, b = pb["polys"][s]
        n = cc._unit(rng, 2)
        bb = np.maximum(n @ pb["verts"][s], n @ pb["verts"][s + 1]) + rng.uniform(0.3, 0.6, 2)
        polys.append((np.vstack([n, A]), np.concatenate([bb, b])))
    return dict(pb, polys=polys, P=P)


@pytest.mark.parametrize("N,ff", [(10, True), (10, False), (16, True), (16, False)])
def test_thirty_two_polytopes(solver, oracle, N, ff):
    P = cc.MAX_POLY
    pb = many_polytopes(84000 + N + int(ff), N, ff, P)
    rng = np.random.default_rng(N)
    mono = cr.sample_monotone_sigmas(N, P, 24, rng)
    arb = rng.integers(0, P, (8, N)).astype(np.uint8)
    arb[0, -1] = P - 1
    sig = np.vstack([mono, arb])
    assert (sig == P - 1).any()
    base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
    dt_list = FACTORS * base
    dts, sigs = np.repeat(dt_list, len(sig)), np.tile(sig, (len(FACTORS), 1))
    fo, co_, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
    assert fo.any() and not fo.all()
    for generic in (False, True):
        (fg, cg, cog), names = solve(solver, N, pb, dts, sigs, ff, generic)
        assert names == {GENERIC if generic else SPEC}
        _compare(fg, cg, cog, fo, co_, coo, "P = 32, generic = %d" % generic)
    g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dt_list, sig, ff)
    check_sweep(g, fo, co_, coo, len(dt_list), len(sig), "P = 32 sweep")
    if ff:
        from oracle import pair_oracle
        from test_pair_gpu import _check_against_oracle
        safe = cr.make_corridor(84000 + N + int(ff), 3, N, "uav", False)     # the whole corridor's base polytopes
        ss = cr.monotone_sigmas(N, 3)[::4]
        w = capi.make_pair_workload([pb, pb], [safe, safe], FACTORS, sig, FACTORS, ss, DC=0.01, r_fraction=0.3)
        r = solver.replan_pairs(w)
        o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["results"]["whole_dt_base"], dt_base_safe=r["results"]["safe_dt_base"])
        _check_against_oracle(r, o, 2)
    # one polytope more is refused by every entry point
    pb33 = dict(pb, polys=pb["polys"] + [pb["polys"][-1]])
    for call in (lambda: solver.solve_batch(N, pb33["x0"], pb33["xf"], pb33["lim"], pb33["polys"], dts[:2], sigs[:2], ff),
                 lambda: solver.gen_new_traj(N, pb33["x0"], pb33["xf"], pb33["lim"], pb33["polys"], dt_list, sig, ff),
                 lambda: solver.gen_new_traj_exact(N, pb33["x0"], pb33["xf"], pb33["lim"], pb33["polys"], dt_list, ff)):
        with pytest.raises(capi.FqError, match="error -1:"):
            call()
    P33, fo33, Ab33 = capi.pack_polys(pb33["polys"])
    with pytest.raises(capi.FqError, match="error -1:.*polytope count out of range"):
        solver.solve_multi(N, ff, pb["x0"][None].copy(), pb["xf"][None].copy(), pb["lim"][None].copy(), np.array([0, 33], np.int32),
                           fo33, Ab33, np.array([0, 2], np.int32), dts[:2].copy(), np.ascontiguousarray(sigs[:2]))
    w33 = capi.make_pair_workload([pb33], [cr.make_corridor(1, 3, N, "uav", False)], FACTORS, sig, FACTORS, cr.monotone_sigmas(N, 3)[:4])
    with pytest.raises(capi.FqError, match="error -1:.*polytope count out of range"):
        solver.replan_pairs(w33)


# ---------------------------------------------------------------------------------------------------------------------
# 7. a batch with one problem past the specialised limit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slices", [1, 4])
def test_mixed_batch_with_one_oversized_problem(solver, oracle, slices):
    """fq_solve_multi: ten ordinary corridors and one a face past the specialised limit, large enough for the sliced copy
    path.  Every problem equals its own fq_solve_batch and the restatement."""
    N, ff = 10, True
    probs, cand = [], []
    for j in range(11):
        pb = cr.make_corridor(84000 + j, 3, N, "uav", ff)
        if j == 5:
            base = [len(b) for _, b in pb["polys"]]
            pb = cc.with_faces(pb, cc.limit("spec", N, ff, "even", base) + 1, "even", seed=j)
            n_sig = 8
        else:
            n_sig = 800
        rng = np.random.default_rng(j)
        sig = np.vstack([cr.monotone_sigmas(N, 3)[rng.choice(66, 40)], rng.integers(0, 3, (n_sig - 40, N)).astype(np.uint8)]) \
            if n_sig > 66 else cr.monotone_sigmas(N, 3)[rng.choice(66, n_sig, replace=False)]
        base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
        probs.append(pb)
        cand.append((np.repeat(FACTORS * base, len(sig)), np.tile(sig, (len(FACTORS), 1))))
    x0 = np.array([pb["x0"] for pb in probs]); xf = np.array([pb["xf"] for pb in probs]); lim = np.array([pb["lim"] for pb in probs])
    po_, fo, rows = [0], [0], []
    for pb in probs:
        for A, b in pb["polys"]:
            rows.append(np.hstack([A, b[:, None]])); fo.append(fo[-1] + len(b))
        po_.append(po_[-1] + len(pb["polys"]))
    co_ = np.concatenate([[0], np.cumsum([len(d) for d, _ in cand])]).astype(np.int32)
    Ab = np.ascontiguousarray(np.vstack(rows))
    dts = np.concatenate([d for d, _ in cand]); sigs = np.ascontiguousarray(np.vstack([s for _, s in cand]))
    po_, fo = np.array(po_, np.int32), np.array(fo, np.int32)
    assert 8 * len(dts) + sigs.size > 512 * 1024                    # the sliced (throughput) copy path
    solver.set_option("throughput_slices", slices)
    try:
        f, c, co, it = solver.solve_multi(N, ff, x0, xf, lim, po_, fo, Ab, co_, dts, sigs, want_coeffs=True, want_iters=True)
    finally:
        solver.set_option("throughput_slices", 0)
    assert (it >= 0).all()
    fr, cr_ = oracle.solve_multi(N, ff, x0, xf, lim, po_, fo, Ab, co_, dts, sigs, threads=8)
    _compare(f, c, None, fr, cr_, None, "mixed batch, %d slices" % slices)
    for j, pb in enumerate(probs):
        sl = slice(co_[j], co_[j + 1])
        f1, c1, co1, _ = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts[sl], sigs[sl], ff, True)
        _compare(f[sl], c[sl], co[sl], f1, c1, co1, "problem %d vs its own solve" % j)


# ---------------------------------------------------------------------------------------------------------------------
# 8. the chained replan across the fall-back
# ---------------------------------------------------------------------------------------------------------------------
def test_chained_replan_with_safe_corridors_past_the_specialised_limit(solver):
    """fq_replan_pairs where every safe corridor is past the specialised limit: the safe sweep and the winners'
    coefficient pass both run on the generic kernel; against the CPU chain."""
    from oracle import pair_oracle
    from test_pair_gpu import _check_against_oracle
    N = 10
    whole = [cr.make_corridor(85000 + j, 3, N, "uav", True) for j in range(4)]
    safe = []
    for j in range(4):
        s = cr.make_corridor(85000 + j, 4, N, "uav", False)
        base = [len(b) for _, b in s["polys"]]
        safe.append(cc.with_faces(s, cc.limit("spec", N, False, "even", base) + 1 + j, "even", seed=j, radius=0.5))
    sw, ss = cr.monotone_sigmas(N, 3)[::6], cr.monotone_sigmas(N, 4)[::30]
    w = capi.make_pair_workload(whole, safe, np.arange(1.0, 7.0), sw, np.arange(1.0, 7.0), ss, DC=0.01, r_fraction=0.3)
    (r, names) = kernels(lambda: solver.replan_pairs(w))
    assert SPEC in names and GENERIC in names, names
    o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["results"]["whole_dt_base"], dt_base_safe=r["results"]["safe_dt_base"])
    _check_against_oracle(r, o, 4)
    assert (o["safe_dt_index"] >= 0).any()
