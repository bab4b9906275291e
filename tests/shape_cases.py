"""The corridor families every compiled solver shape is checked on: N = 4..16 in whole and safe mode, 2, 3, 4 and
min(8, N) polytopes, UAV and ground-robot limits, non-decreasing assignments plus a third arbitrary ones, and time
allocations from tight (mostly infeasible) to loose.  Shared by tests/test_parity_gpu.py and tools/stress_shapes.py."""
import math

import numpy as np

from faster_b200 import capi, corridor as cr

SHAPES = [(N, ff) for N in range(4, 17) for ff in (True, False)]
FACTORS = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])


def families(N):
    """(number of polytopes, limits profile) of the corridors run at N."""
    return ((2, "uav"), (3, "uav"), (4, "ground"), (min(8, N), "uav"))


def shape_batches(N, ff, n_corr, n_mono=40, n_arb=24):
    """Yields (P, profile, corridor index, corridor dict, dts, sigmas): dt-major batches of FACTORS x (n_mono
    non-decreasing + n_arb arbitrary assignments) on n_corr corridors of every family."""
    for P, profile in families(N):
        rng = np.random.default_rng(N * 1000 + P * 10 + int(ff))
        mono = cr.monotone_sigmas(N, P) if math.comb(N + P - 1, P - 1) <= 5000 else cr.sample_monotone_sigmas(N, P, 256, rng)
        for c in range(n_corr):
            pb = cr.make_corridor(50000 + 97 * N + c, P, N, profile, ff)
            dti = capi.dt_initial(pb["x0"], pb["xf"], pb["lim"], N)
            sig = np.vstack([mono[rng.choice(len(mono), min(n_mono, len(mono)), replace=False)],
                             rng.integers(0, P, size=(n_arb, N)).astype(np.uint8)])
            dts = np.repeat(FACTORS * max(dti, 2 * pb["DC"]), len(sig))
            yield P, profile, c, pb, dts, np.tile(sig, (len(FACTORS), 1))
