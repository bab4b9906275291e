"""Degenerate corridors (tests/degenerate_cases.py) on every solve path: several rows tight at one point, linearly dependent
normals, ties in the row ranking and the ratio test -- where a dual active-set method goes wrong.

The CPU restatement (oracle/fq_oracle.c) is the same algorithm family with the same dependency threshold, so agreement with
it proves less here than elsewhere.  Two checks that do not share the algorithm carry the weight:
  * metamorphic relations: fan, dup, dup_scaled, symmetry and vertical_slab provably leave the problem unchanged, so the
    flags, costs and coefficients must be those of the untransformed corridor on the same path;
  * proofs on the literal model (oracle/proofs.py): KKT multipliers for "solved", the Farkas certificate of
    fq_solve_batch_cert for "not solved".
The other families (slab, near_parallel, touching, states on the boundary) have no known answer: identical flags to the
restatement, costs within REL, and proofs.  Where the rows leave a band only the row tolerance wide (TOLERANCE_BAND) two
correct solvers may stop at different points inside it -- the slab lets z wander by 1e-8 at every control point, which is
1e-5 in a cubic coefficient at dt = 0.1 s: there a candidate beyond the bars must have both answers proved, and their cost gap
must stay below row_tol times the multipliers."""
import numpy as np
import pytest

import degenerate_cases as dc
from faster_b200 import capi, corridor as cr
from test_parity_gpu import REL, _compare
from test_row_tolerance_gpu import Tol

pytestmark = pytest.mark.gpu

FACTORS = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
# lane-layout boundary shapes: (N, force_final, polytopes, profile)
SHAPES = [(4, True, 2, "uav"), (5, True, 2, "uav"), (10, True, 3, "uav"), (13, True, 3, "uav"), (14, True, 4, "uav"),
          (16, True, 4, "uav"), (4, False, 2, "uav"), (12, False, 3, "uav"), (13, False, 4, "uav"), (16, False, 4, "uav"),
          (15, True, 8, "ground")]
PROOF_SHAPES = [(10, True, 3, "uav"), (10, False, 3, "uav"), (15, True, 8, "ground")]

FAMILY_A = {
    "fan1": lambda pb: dc.fan(pb, 1), "fan2": lambda pb: dc.fan(pb, 2), "fan8": lambda pb: dc.fan(pb, 8, n_vert=2),
    "dup": dc.dup, "dup_scaled": dc.dup_scaled, "vertical_slab": dc.slab,   # vertical_slab: the original is dc.vertical(pb)
}
FAMILY_B = {
    "slab": dc.slab,
    "near_parallel_1e-12": lambda pb: dc.near_parallel(pb, 1e-12), "near_parallel_1e-9": lambda pb: dc.near_parallel(pb, 1e-9),
    "near_parallel_1e-7": lambda pb: dc.near_parallel(pb, 1e-7), "near_parallel_1e-5": lambda pb: dc.near_parallel(pb, 1e-5),
    "touching_0": lambda pb: dc.touching(pb, 0.0), "touching_1e-9": lambda pb: dc.touching(pb, 1e-9),
    "touching_1e-6": lambda pb: dc.touching(pb, 1e-6),
    "x0_face": lambda pb: dc.on_boundary(pb, "x0", 1), "x0_edge": lambda pb: dc.on_boundary(pb, "x0", 2),
    "x0_vertex": lambda pb: dc.on_boundary(pb, "x0", 3), "xf_vertex": lambda pb: dc.on_boundary(pb, "xf", 3),
    "v0_at_limit": lambda pb: dc.at_limit(pb, "v"), "a0_at_limit": lambda pb: dc.at_limit(pb, "a"),
}
# families whose rows leave a band only the row tolerance wide: the zero-width slab, copies at most 1e-7 rad apart (the
# rows hold within the tolerance on a wedge row_tol / theta wide) and polytopes that touch in a slab of 0 or 1e-9
TOLERANCE_BAND = ("slab", "near_parallel_1e-12", "near_parallel_1e-9", "near_parallel_1e-7", "touching_0", "touching_1e-9")


def _ground_only(fam):
    return fam in ("vertical_slab", "slab")


def corridor(fam, N, P, ff, profile, c):
    """(original, transformed) corridor number c of a family at this shape; None when the family does not apply."""
    if _ground_only(fam):
        profile = "ground"
    if fam == "xf_vertex" and not ff:
        return None
    pb = cr.make_corridor(52000 + 31 * N + c, P, N, profile, ff)
    if fam == "a0_at_limit" and not np.abs(pb["x0"][6:9]).max() > 0:
        return None
    if fam == "vertical_slab":
        pb = dc.vertical(pb)
    f = FAMILY_A.get(fam) or FAMILY_B[fam]
    out = f(pb)
    assert dc.specialised_fits(N, ff, out["polys"]), (fam, N)
    return pb, out


def candidates(pb, N, P, n_mono=24, n_arb=8):
    """dt-major FACTORS x assignments; the time allocations come from the ORIGINAL corridor (a transform must not move them)."""
    rng = np.random.default_rng(N * 100 + P)
    mono = cr.monotone_sigmas(N, P) if P <= 4 else cr.sample_monotone_sigmas(N, P, 200, rng)
    sig = np.vstack([mono[rng.choice(len(mono), min(n_mono, len(mono)), replace=False)], rng.integers(0, P, (n_arb, N)).astype(np.uint8)])
    base = max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 2 * pb["DC"])
    return FACTORS * base, np.repeat(FACTORS * base, len(sig)), np.tile(sig, (len(FACTORS), 1))


def run(solver, N, pb, dts, sigs, ff, generic):
    solver.set_option("force_generic_kernel", generic)
    try:
        f, c, co, it = solver.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, True)
    finally:
        solver.set_option("force_generic_kernel", 0)
    assert (it >= 0).all(), "iteration-cap or numeric give-ups at %s" % np.flatnonzero(it < 0)[:8]
    return f, c, co


def prove(solver, N, pb, dts, sigs, ff, idx, f, c, co, row_tol=1e-8):
    """Proves the flags of candidates idx: KKT multipliers for "solved", the certifying kernel's Farkas certificate for "not
    solved".  -> list of proof dicts of the solved ones.  Near-parallel copies (pb["near_parallel"]) cross the face inside
    the polytope, so a tight row's twin has a slack of up to theta times a few metres; the multipliers are then fitted on
    rows within 1e-9 (relative) of tight only, or the fit may load the twin and report its slack as a gap."""
    from oracle import model_fullspace as mf, proofs
    idx = list(idx)
    cert = solver.solve_batch_cert(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff)[2] if not f[idx].all() else None
    out = []
    for i in idx:
        model = mf.build(N, pb["x0"], pb["xf"], pb["lim"], dts[i], pb["polys"], sigs[i], ff)
        if f[i]:
            # a point may violate rows by up to row_tol, and a violated row with multiplier lam adds lam * row_tol to the gap
            r = proofs.assert_optimal(model, co[i], c[i], feas_tol=row_tol + 1e-7, gap_tol=np.inf,
                                      active_tol=1e-9 if pb.get("near_parallel") else 1e-7)
            assert r["gap"] <= 1e-7 + row_tol * r["lam_sum"] / max(1.0, r["cost"]), r
            out.append(r)
            out[-1]["model"] = model
        else:
            proofs.assert_infeasible(model, N, pb["polys"], sigs[i], cert[i], gap_max=-row_tol * 0.99)
    return out


def _margin(solver, N, ff, pb, dts, sigs):
    P, fo, Ab = capi.pack_polys(pb["polys"])
    return cr.margin_flags(solver, N, ff, pb["x0"][None], pb["xf"][None], pb["lim"][None], np.array([0, P], np.int32),
                           fo.astype(np.int32), Ab, np.array([0, len(dts)], np.int32), dts, sigs, eps=1e-6)[1]


def _same_answer(solver, N, ff, pb2, dts, sigs, got, ref, what, allow_margin, unperm=None):
    """got (transformed corridor) against ref (original corridor, same path): identical flags, costs within REL,
    coefficients within 1e-6.  allow_margin: a candidate within 1e-6 of the boundary may change its flag if the new flag
    is proved."""
    fg, cg, cog = got
    fr, cr_, cor = ref
    if unperm is not None:
        cog = dc.unpermute_coeffs(cog, *unperm)
    diff = np.flatnonzero(fg != fr)
    if len(diff) and allow_margin:
        near = _margin(solver, N, ff, pb2, dts, sigs)
        assert near[diff].all(), "%s: flags changed away from the boundary at %s" % (what, diff[~near[diff]][:8])
        prove(solver, N, pb2, dts, sigs, ff, diff, fg, cg, got[2])
        keep = np.ones(len(fg), bool)
        keep[diff] = False
        fg, cg, cog, fr, cr_, cor = fg[keep], cg[keep], cog[keep], fr[keep], cr_[keep], cor[keep]
    _compare(fg, cg, cog, fr, cr_, cor, what)


@pytest.mark.parametrize("fam", list(FAMILY_A))
@pytest.mark.parametrize("N,ff,P,profile", SHAPES)
def test_unchanging_transforms_change_nothing(solver, oracle, fam, N, ff, P, profile):
    """Both kernels: flags, costs and coefficients of the transformed corridor equal those of the original on the same path,
    and the restatement's on the transformed corridor."""
    for c in range(2):
        pb, pb2 = corridor(fam, N, P, ff, profile, c)
        _, dts, sigs = candidates(pb, N, P)
        if fam == "vertical_slab":                # the optimum without the pair already has z = h
            fo, _, coo = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
            z = coo[fo.astype(bool)][:, :, 2::3]
            assert fo.any() and np.abs(z[:, :, :3]).max() < 1e-12 and np.abs(z[:, :, 3] - pb2["slab_h"]).max() < 1e-12
        fo2, co2, coo2 = oracle.solve_batch(N, pb2["x0"], pb2["xf"], pb2["lim"], pb2["polys"], dts, sigs, ff, True, threads=8)
        for generic in (0, 1):
            what = "%s N=%d ff=%d corridor %d generic=%d" % (fam, N, ff, c, generic)
            ref = run(solver, N, pb, dts, sigs, ff, generic)
            got = run(solver, N, pb2, dts, sigs, ff, generic)
            _same_answer(solver, N, ff, pb2, dts, sigs, got, ref, what, fam == "dup_scaled")
            _compare(*got, fo2, co2, coo2, what + " vs restatement")


@pytest.mark.parametrize("N,ff,P,profile", SHAPES)
def test_axis_symmetries_change_nothing(solver, oracle, N, ff, P, profile):
    """The 48 signed axis permutations at whole and safe N = 10, eight of them at every other shape; coefficients are
    compared after undoing the permutation."""
    perms = dc.SIGNED_PERMUTATIONS if N == 10 else dc.SIGNED_PERMUTATIONS[N % 6::6]
    pb = cr.make_corridor(52000 + 31 * N, P, N, profile, ff)
    _, dts, sigs = candidates(pb, N, P, n_mono=12, n_arb=4)
    ref = {g: run(solver, N, pb, dts, sigs, ff, g) for g in (0, 1)}
    for perm, signs in perms:
        pb2 = dc.symmetry(pb, perm, signs)
        fo2, co2, coo2 = oracle.solve_batch(N, pb2["x0"], pb2["xf"], pb2["lim"], pb2["polys"], dts, sigs, ff, True, threads=8)
        for generic in (0, 1):
            what = "N=%d ff=%d perm %s signs %s generic=%d" % (N, ff, perm, signs, generic)
            got = run(solver, N, pb2, dts, sigs, ff, generic)
            _same_answer(solver, N, ff, pb2, dts, sigs, got, ref[generic], what, True, unperm=(perm, signs))
            _compare(*got, fo2, co2, coo2, what + " vs restatement")


def _cost_bar(solver, N, ff, pb, dts, sigs, fam, got, ref, what, row_tol=1e-8):
    """Identical flags, costs within REL, coefficients within 1e-6.  Where rows leave a band that is only the row tolerance
    wide (TOLERANCE_BAND), two correct solvers may stop at different points inside it: a candidate beyond those bars must
    have both answers proved and a cost gap below 2 row_tol times the larger multiplier sum (a point that violates rows by
    up to row_tol is at most that much cheaper).  -> the number of such candidates."""
    if fam not in TOLERANCE_BAND:
        _compare(*got, *ref, what)
        return 0
    fg, cg, cog = got
    fo, co_, coo = ref
    assert np.array_equal(fg, fo), "%s: flags differ at %s" % (what, np.flatnonzero(fg != fo)[:8])
    assert np.isinf(cg[fo == 0]).all()
    ok = np.flatnonzero(fo)
    rel = np.abs(cg[ok] - co_[ok]) / np.abs(co_[ok])
    err = np.abs(cog[ok] - coo[ok]).max(axis=(1, 2)) / np.maximum(1.0, np.abs(coo[ok]).max(axis=(1, 2)))
    over = ok[(rel > REL) | (err > 1e-6)]
    for i in over:
        pg = prove(solver, N, pb, dts, sigs, ff, [i], fg, cg, cog, row_tol)[0]
        po = prove(solver, N, pb, dts, sigs, ff, [i], fo, co_, coo, row_tol)[0]
        assert abs(cg[i] - co_[i]) <= 2 * row_tol * max(pg["lam_sum"], po["lam_sum"]) + 1e-12 * co_[i], (what, i, cg[i], co_[i])
    return len(over)


@pytest.mark.parametrize("fam", list(FAMILY_B))
@pytest.mark.parametrize("N,ff,P,profile", SHAPES)
def test_degenerate_corridors_match_the_restatement(solver, oracle, fam, N, ff, P, profile):
    """Both kernels against the restatement on the transformed corridor: identical flags, costs within REL (or the
    tolerance-derived bar near the cut-off), no give-ups."""
    for c in range(2):
        pbs = corridor(fam, N, P, ff, profile, c)
        if pbs is None:
            continue
        pb = pbs[1]
        _, dts, sigs = candidates(pb, N, P)
        ref = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
        for generic in (0, 1):
            _cost_bar(solver, N, ff, pb, dts, sigs, fam, run(solver, N, pb, dts, sigs, ff, generic), ref,
                      "%s N=%d ff=%d corridor %d generic=%d" % (fam, N, ff, c, generic))


def dependent_tight_rows(proof):
    """Whether the rows tight at a proved optimum (equalities and active inequalities) are linearly dependent, numerically
    at the solver's own cut-off: the rows are normalised and a singular value below 1e-8 counts as zero (two unit rows 1e-9
    rad apart have one of 7e-10)."""
    Q, Aeq, beq, Ain, bin_ = proof["model"]
    M = np.vstack([Aeq, Ain[proof["active"]]])
    if M.shape[0] > M.shape[1]:
        return True
    M = M / np.linalg.norm(M, axis=1, keepdims=True)
    return bool(np.linalg.svd(M, compute_uv=False).min() <= 1e-8)


def _proof_sample(f):
    return np.concatenate([np.flatnonzero(f)[::max(1, int(f.sum()) // 10)][:10], np.flatnonzero(f == 0)[:6]])


# families whose transform makes tight rows dependent where the original corridor had none: the proof sample of each must
# hold more optima with dependent tight rows than the same sample of the untransformed corridors
ADDS_DEPENDENCE = ("fan1", "fan2", "dup", "dup_scaled", "vertical_slab", "slab", "near_parallel_1e-12", "near_parallel_1e-9",
                   "touching_0", "touching_1e-9", "x0_face", "x0_edge", "x0_vertex", "xf_vertex", "v0_at_limit", "a0_at_limit")


@pytest.mark.parametrize("fam", list(FAMILY_A) + ["symmetry"] + list(FAMILY_B))
def test_flags_of_degenerate_corridors_are_proved(solver, fam):
    """A bounded sample of every family at whole N = 10, safe N = 10 and N = 15 (8 polytopes, ground profile): "solved" carries
    KKT multipliers, "not solved" a Farkas certificate, the certifying kernel gives the same flags.  The families of
    ADDS_DEPENDENCE must also hold more optima with dependent tight rows than the same sample of the original corridors (which
    have some already: the ground face and the bbox floor of the ground profile, the final rows of the safe mode)."""
    proved = refuted = dependent = dependent0 = 0
    for N, ff, P, profile in PROOF_SHAPES:
        if fam == "symmetry":
            pb0 = cr.make_corridor(52000 + 31 * N, P, N, profile, ff)
            pbs = (pb0, dc.symmetry(pb0, *dc.SIGNED_PERMUTATIONS[29]))
        else:
            pbs = corridor(fam, N, P, ff, profile, 0)
        if pbs is None:
            continue
        _, dts, sigs = candidates(pbs[0], N, P, n_mono=12, n_arb=4)
        for k, pb in enumerate(pbs):
            f, c, co = run(solver, N, pb, dts, sigs, ff, 0)
            fc = solver.solve_batch_cert(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff)[0]
            assert np.array_equal(f, fc), fam
            idx = _proof_sample(f)
            n_dep = sum(dependent_tight_rows(r) for r in prove(solver, N, pb, dts, sigs, ff, idx, f, c, co))
            if k == 0:
                dependent0 += n_dep
                continue
            dependent += n_dep
            proved += int(f[idx].sum())
            refuted += int((f[idx] == 0).sum())
    assert proved >= 10 and refuted >= 4, (fam, proved, refuted)
    if fam in ADDS_DEPENDENCE:
        assert dependent > dependent0, (fam, dependent, dependent0)
    print("%s: %d optima proved (%d with dependent tight rows, %d in the original corridors), %d infeasible flags proved" % (
        fam, proved, dependent, dependent0, refuted))


@pytest.mark.parametrize("fam", ["fan2", "dup", "dup_scaled", "vertical_slab", "slab", "near_parallel_1e-9", "near_parallel_1e-5",
                                 "touching_0", "x0_vertex", "xf_vertex", "v0_at_limit"])
@pytest.mark.parametrize("N,ff,P,profile", PROOF_SHAPES)
def test_sweep_on_degenerate_corridors(solver, oracle, fam, N, ff, P, profile):
    """fq_gen_new_traj (selection inside the kernel): genNewTraj's winner over the restatement's flags; for the families
    that change nothing also the winner of the original corridor."""
    from test_row_tolerance_gpu import _first_feasible_min_cost
    for c in range(2):
        pbs = corridor(fam, N, P, ff, profile, c)
        if pbs is None:
            continue
        dt_list, dts, sigs = candidates(pbs[0], N, P)
        sig = sigs[:len(sigs) // len(FACTORS)]
        for pb in pbs if fam in FAMILY_A else pbs[1:]:
            fo, co_, _ = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, False, threads=8)
            g = solver.gen_new_traj(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dt_list, sig, ff)
            d, s = _first_feasible_min_cost(fo, co_, len(FACTORS), len(sig))
            assert g["dt_index"] == d and g["solved"] == (d >= 0), (fam, c, g["dt_index"], d)
            if d >= 0:
                assert abs(g["cost"] - co_[d * len(sig) + s]) <= REL * co_[d * len(sig) + s], fam
                assert g["sigma_index"] == s or abs(co_[d * len(sig) + g["sigma_index"]] - co_[d * len(sig) + s]) <= REL * co_[d * len(sig) + s]


@pytest.mark.parametrize("fam", ["fan2", "dup", "dup_scaled", "slab", "near_parallel_1e-9", "touching_0", "x0_vertex"])
@pytest.mark.parametrize("N", [6, 10])
def test_exact_sweep_on_degenerate_corridors(solver, oracle, fam, N):
    """fq_gen_new_traj_exact (branch-and-bound from each parent's factorisation, so a degenerate active set is carried from
    node to node) against the restatement's branch-and-bound over all assignments."""
    solved = 0
    for seed, ff in ((5007, True), (5055, False)):
        pb = cr.make_corridor(seed, 3, N, "ground" if _ground_only(fam) else "uav", ff)
        pb = (FAMILY_A.get(fam) or FAMILY_B[fam])(pb)
        for f in (2.0, 5.0):
            dt = f * max(capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02)
            g = solver.gen_new_traj_exact(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], [dt], ff)
            rc, c, co, _, _ = oracle.solve_miqp(N, pb["x0"], pb["xf"], pb["lim"], dt, pb["polys"], ff)
            assert g["exact"] and g["solved"] == (rc == 1), (fam, seed, f)
            if rc == 1:
                solved += 1
                assert abs(g["cost"] - c) <= REL * max(1.0, c), (fam, seed, g["cost"], c)
                assert np.abs(g["coeffs"] - co).max() <= 1e-6 * max(1.0, np.abs(co).max()), (fam, seed)
    assert solved >= 1, fam


@pytest.mark.parametrize("fam", ["dup", "slab"])
def test_chained_replan_on_degenerate_corridors(solver, oracle, fam):
    """fq_replan_pairs with the transform on the whole and the safe corridors, against the CPU chain (oracle/pair_oracle.py)."""
    from oracle import pair_oracle
    from test_pair_gpu import _check_against_oracle
    n, profile = 6, ("ground" if fam == "slab" else "uav")
    f = FAMILY_A.get(fam) or FAMILY_B[fam]
    whole = [f(cr.make_corridor(73000 + k, 3, 10, profile, True)) for k in range(n)]
    safe = [f(dict(cr.make_corridor(73000 + k, 4, 10, profile, False))) for k in range(n)]
    fw = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
    w = capi.make_pair_workload(whole, safe, fw, cr.monotone_sigmas(10, 3)[::3], fw, cr.monotone_sigmas(10, 4)[::12], DC=0.01,
                                r_fraction=0.3)
    g = solver.replan_pairs(w)
    r = g["results"]
    o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    _check_against_oracle(g, o, n)


@pytest.mark.parametrize("tol", [1, 1000])
@pytest.mark.parametrize("fam", ["fan2", "dup_scaled", "slab", "near_parallel_1e-9", "near_parallel_1e-7", "touching_1e-9", "x0_vertex"])
def test_degenerate_corridors_at_other_row_tolerances(solver, oracle, fam, tol):
    """Row tolerance 1e-9 and 1e-6, whole and safe N = 10, both kernels against the restatement at the same tolerance."""
    with Tol(solver, oracle, tol):
        for N, ff, P, profile in PROOF_SHAPES[:2]:
            pb = corridor(fam, N, P, ff, profile, 0)[1]
            _, dts, sigs = candidates(pb, N, P)
            ref = oracle.solve_batch(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, sigs, ff, True, threads=8)
            for generic in (0, 1):
                _cost_bar(solver, N, ff, pb, dts, sigs, fam, run(solver, N, pb, dts, sigs, ff, generic), ref,
                          "%s N=%d ff=%d generic=%d tol=%de-9" % (fam, N, ff, generic, tol), row_tol=1e-9 * tol)
