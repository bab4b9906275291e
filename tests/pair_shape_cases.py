"""The (N_whole, N_safe) pairs the chained replan is checked at, and the corridor batches run there.

fq_replan_pairs* take N_whole in 3..16 and N_safe in 2..16 independently (the reference reads them as two parameters,
faster_ros.cpp:24-25).  The pairs: the diagonal N = 4..16, the kernel switches (N_whole = 3 and N_safe = 2 or 3 solve with the
size-generic kernel; at N_safe = 2 the safe sweep has no unknowns; N < 4 has no branch-and-bound tree), the longest sample
runs (N = 16) and unequal pairs in both orders.  Every corridor keeps P <= N - 2 polytopes (faster_ros.cpp:75-83 asks for
N > max_poly + 2), and P varies from corridor to corridor, so that per-corridor assignment lists differ in length.
Shared by tests/test_pair_shapes_gpu.py and tests/test_pair_shapes_cpu.py."""
import numpy as np

from faster_b200 import capi, corridor as cr

DIAGONAL = [(N, N) for N in range(4, 17)]
OFF_DIAGONAL = [(3, 2), (3, 3), (3, 16), (16, 2), (16, 3), (4, 16), (16, 4), (6, 10), (10, 6), (5, 12), (12, 5), (7, 4)]
PAIRS = DIAGONAL + OFF_DIAGONAL
FACTORS = np.array([1.0, 1.5, 2.0, 3.0, 5.0, 8.0])
CAP_WHOLE, CAP_SAFE = 3, 4                      # max_poly_whole / max_poly_safe of faster.yaml


def pair_id(p):
    return "%dx%d" % p


def max_poly(N, cap):
    """The most polytopes a corridor of N intervals gets here: min(cap, N - 2), at least 0."""
    return max(0, min(cap, N - 2))


def poly_counts(N, n, cap, shift=0):
    """Polytope counts of n corridors: max_poly(N, cap), one fewer, ... down to 0 and round again (shifted by `shift`)."""
    top = max_poly(N, cap)
    return [top - (j + shift) % (top + 1) for j in range(n)]


def corridors(Nw, Ns, n, seed0, uniform=False):
    """n (whole, safe) corridor pairs: corridor.make_corridor with one seed per pair, N_whole and force_final for the whole
    corridor, N_safe without force_final for the safe one (its x0 is replaced by R on the device).  uniform: every corridor
    gets the largest count, as a shared assignment list needs."""
    pw = [max_poly(Nw, CAP_WHOLE)] * n if uniform else poly_counts(Nw, n, CAP_WHOLE)
    ps = [max_poly(Ns, CAP_SAFE)] * n if uniform else poly_counts(Ns, n, CAP_SAFE, shift=1)
    seeds = [seed0 + 101 * Nw + 7 * Ns + j for j in range(n)]
    return [_corridor(s, p, Nw, True) for s, p in zip(seeds, pw)], [_corridor(s, p, Ns, False) for s, p in zip(seeds, ps)]


def _corridor(seed, P, N, force_final):
    """make_corridor; P = 0 keeps the one-segment corridor's states and drops its polytope (no corridor rows)."""
    pb = cr.make_corridor(seed, max(P, 1), N, "uav", force_final)
    if P == 0:
        pb["polys"], pb["P"] = [], 0
    return pb


def shared_list(N, P, n_sig=16):
    """A subsample of at most n_sig non-decreasing assignments of N intervals to P polytopes (one row of 0s for P <= 1)."""
    if P <= 1:
        return np.zeros((1, N), np.uint8)
    s = cr.monotone_sigmas(N, P)
    return s[np.unique(np.linspace(0, len(s) - 1, n_sig).round().astype(int))]


def shared_workload(Nw, Ns, n=4, seed0=60000, factors=FACTORS, r_fraction=0.6):
    """fq_replan_pairs' workload: uniform polytope counts and one subsampled list per sweep."""
    whole, safe = corridors(Nw, Ns, n, seed0, uniform=True)
    sw, ss = shared_list(Nw, whole[0]["P"]), shared_list(Ns, safe[0]["P"])
    return capi.make_pair_workload(whole, safe, factors, sw, factors, ss, DC=0.01, r_fraction=r_fraction)


def mixed_workload(Nw, Ns, n=5, seed0=61000, factors=FACTORS, r_fraction=0.6):
    """The per-corridor entries' workload (_assign, _window, _exact): mixed polytope counts, no shared lists."""
    whole, safe = corridors(Nw, Ns, n, seed0)
    return capi.make_pair_workload(whole, safe, factors, np.zeros((0, Nw), np.uint8), factors, np.zeros((0, Ns), np.uint8), DC=0.01,
                                   r_fraction=r_fraction)


def mixed_windows(n, seed):
    """Different windows per corridor, inc 1 (whole) and 0.5 (safe); every window holds 2 to 5 factors."""
    rng = np.random.default_rng(seed)
    iw = rng.choice([1.0, 1.5, 2.0, 3.0], n)
    is_ = rng.choice([1.0, 1.5, 2.5], n)
    return dict(init_whole=iw, final_whole=iw + rng.integers(1, 5, n), init_safe=is_, final_safe=is_ + rng.choice([0.5, 1.0, 2.0], n))


INC = (1.0, 0.5)
