"""The corridor families every compiled solver shape is checked on: N = 4..16 in whole and safe mode, 2, 3, 4 and
min(8, N) polytopes, UAV and ground-robot limits, non-decreasing assignments plus a third arbitrary ones, and time
allocations from tight (mostly infeasible) to loose.  Shared by tests/test_parity_gpu.py and tools/stress_shapes.py.
Also the two variations other tests apply to corridors: a moving final state, and a probe row violated by a known DELTA."""
import math

import numpy as np

from faster_b200 import capi, corridor as cr

DELTA = 3e-7        # a row violation above the default row tolerance 1e-8 and below Gurobi's 1e-6
SHAPES = [(N, ff) for N in range(4, 17) for ff in (True, False)]
FACTORS = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])


def families(N):
    """(number of polytopes, limits profile) of the corridors run at N."""
    return ((2, "uav"), (3, "uav"), (4, "ground"), (min(8, N), "uav"))


def moving_final_state(pb, speed=0.6, accel=(0.3, -0.2, 0.1)):
    """A copy of corridor `pb` whose final state moves: velocity `speed` along the last segment, acceleration `accel`."""
    xf = np.array(pb["xf"], float)
    d = pb["verts"][-1] - pb["verts"][-2]
    xf[3:6] = speed * d / np.linalg.norm(d)
    xf[6:9] = accel
    return dict(pb, xf=xf)


def shape_batches(N, ff, n_corr, n_mono=40, n_arb=24, final_state=None):
    """Yields (P, profile, corridor index, corridor dict, dts, sigmas): dt-major batches of FACTORS x (n_mono
    non-decreasing + n_arb arbitrary assignments) on n_corr corridors of every family.  final_state(pb) -> corridor, if
    given, replaces each corridor's final state (e.g. moving_final_state) before the time allocations are derived."""
    for P, profile in families(N):
        rng = np.random.default_rng(N * 1000 + P * 10 + int(ff))
        mono = cr.monotone_sigmas(N, P) if math.comb(N + P - 1, P - 1) <= 5000 else cr.sample_monotone_sigmas(N, P, 256, rng)
        for c in range(n_corr):
            pb = cr.make_corridor(50000 + 97 * N + c, P, N, profile, ff)
            if final_state is not None:
                pb = final_state(pb)
            dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
            sig = np.vstack([mono[rng.choice(len(mono), min(n_mono, len(mono)), replace=False)],
                             rng.integers(0, P, size=(n_arb, N)).astype(np.uint8)])
            dts = np.repeat(FACTORS * max(dti, 2 * pb["DC"]), len(sig))
            yield P, profile, c, pb, dts, np.tile(sig, (len(FACTORS), 1))


def probe(pb, kind):
    """A copy of corridor `pb` with one input-fixed row violated by DELTA."""
    pb = dict(pb, x0=pb["x0"].copy(), lim=pb["lim"].copy(), polys=[(A.copy(), b.copy()) for A, b in pb["polys"]])
    x0 = pb["x0"]
    if kind == "velocity":
        pb["lim"][0] = np.abs(x0[3:6]).max() - DELTA
    elif kind == "x0_face":                                  # every polytope that holds x0 (segments overlap)
        for A, b in pb["polys"]:
            if (A @ x0[:3] - b).max() <= 0:
                f = int(np.argmin(A @ x0[3:6]))
                b[f] = A[f] @ x0[:3] - DELTA
    else:
        assert kind == "xf_face" and pb["force_final"]
        xf, d = pb["xf"][:3], pb["verts"][-1] - pb["verts"][-2]
        for A, b in pb["polys"]:                             # every polytope that holds xf
            if (A @ xf - b).max() <= 0:
                f = int(np.argmax(A @ d))
                b[f] = A[f] @ xf - DELTA
    return pb
