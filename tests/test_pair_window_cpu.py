"""Per-corridor time-allocation windows of the chained replan (fq_replan_pairs_window*) without a GPU: fq_pair_window_factors
against genNewTraj's loop restated in Python and against the reference's own compiled loop, the next-window rule against
faster.cpp:582-588, the product's kernel SOURCE (faster_b200/csrc/fq_pair.cuh) under the block emulation of tests/cpp/simt_emu/,
the whole _window_dev submission replayed through the emulated kernels against the CPU chain, and the ctypes struct layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi

import pair_assign_oracle as pao
import pair_window_oracle as pwo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_window_emu.so")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_window_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h")] + \
               [os.path.join(ROOT, "faster_b200", "csrc", f) for f in ("fq_pair.cuh", "fq_assign.h", "fq_window.h", "fq_kernels.cuh")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", os.path.join(ROOT, "faster_b200", "csrc"),
                                   "-I", os.path.join(ROOT, "include"), srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_window_factors.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
        L.emu_window_offsets.argtypes = [C.c_int] * 4 + [C.c_longlong, C.c_int, C.c_longlong] + [C.c_void_p] * 3
        L.emu_expand_window.argtypes = [C.c_int] * 3 + [C.c_longlong] + [C.c_void_p] * 7
        L.emu_pair_window.argtypes = [C.c_int] * 3 + [C.c_void_p] * 12
        L.emu_host_factors.argtypes = [C.c_double] * 3 + [C.c_void_p, C.c_int]
        L.emu_host_next_window.argtypes = [C.c_int] + [C.c_double] * 5 + [C.c_void_p]
        for f in ("emu_window_factors", "emu_window_offsets", "emu_expand_window", "emu_pair_final_window", "emu_pair_window",
                  "emu_host_next_window"):
            getattr(L, f).restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data)


def lib_factors(fi, ff, inc):
    n = capi.lib().fq_pair_window_factors(float(fi), float(ff), float(inc), None, 0)
    if n < 0:
        return None
    out = np.zeros(n)
    assert capi.lib().fq_pair_window_factors(float(fi), float(ff), float(inc), out.ctypes.data, n) == n
    return out


def _bits_equal(a, b):
    return (a is None and b is None) or (a is not None and b is not None and a.tobytes() == b.tobytes())


WINDOWS = [(fi, fi + span, inc) for inc in (0.1, 0.3, 1 / 3, 1.0, 2.5) for fi in (1.0, 2.0, 1.3, 2.75, 17.0)
           for span in (-0.5, 0.0, 0.7, 3.0, 9.0, 20.0)]


def test_factor_lists_equal_the_loop(built_lib):
    """Sequential accumulation, bit for bit, over increments 0.1 .. 2.5, integer and fractional starts, empty and one-element
    windows; never fi + k inc."""
    for fi, ff, inc in WINDOWS:
        want = pwo.factors(fi, ff, inc)
        assert _bits_equal(lib_factors(fi, ff, inc), want), (fi, ff, inc)
    assert len(lib_factors(2.0, 1.0, 1.0)) == 0 and list(lib_factors(2.0, 2.0, 1.0)) == [2.0]
    f = lib_factors(1.0, 2.0, 0.1)
    assert len(f) == 10 and f[-1] != 1.9 and f[3] != 1.0 + 3 * 0.1      # accumulated, not multiplied
    assert len(pwo.factors(1.0, 1.0 + 10 * 0.1, 0.1)) == 10             # 1 + 10 * 0.1 = 2.0, the loop's 11th value is 2.0000000000000004
    exact = pwo.factors(1.0, 10.0, 1 / 3)[-1]                          # ff exactly on an accumulated value is visited
    assert lib_factors(1.0, exact, 1 / 3)[-1] == exact and len(lib_factors(1.0, exact, 1 / 3)) == len(pwo.factors(1.0, exact, 1 / 3))
    # partial copies: cap < |F| writes the first cap factors and still returns |F|
    out = np.full(4, -1.0)
    assert capi.lib().fq_pair_window_factors(1.0, 10.0, 1.0, out.ctypes.data, 3) == 10 and list(out) == [1.0, 2.0, 3.0, -1.0]


def test_refusals(built_lib):
    E = -1
    L = capi.lib()
    for fi, ff, inc in ((np.nan, 2.0, 1.0), (1.0, np.nan, 1.0), (1.0, 2.0, np.nan), (np.inf, 2.0, 1.0), (1.0, np.inf, 1.0),
                        (1.0, 2.0, np.inf), (1.0, 2.0, 0.0), (1.0, 2.0, -1.0), (0.0, 2.0, 1.0), (-1.0, 2.0, 1.0),
                        (1.0, 4097.0, 1.0), (1.0, 1.0 + 4096 * 0.25, 0.25), (1e17, 1e17 + 1e3, 1.0)):
        assert L.fq_pair_window_factors(fi, ff, inc, None, 0) == E, (fi, ff, inc)
        assert pwo.factors(fi, ff, inc) is None
    assert len(lib_factors(1.0, 4096.0, 1.0)) == 4096                     # the cap itself is allowed
    assert len(lib_factors(1e17, 1e17 - 1e3, 1.0)) == 0                   # empty: the loop never runs, nothing stalls


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libsolver_ref.so")),
                    reason="oracle/_ref/libsolver_ref.so is not built (needs the reference tree)")
def test_pinned_to_the_reference_loop(built_lib):
    """The reference's own genNewTraj (compiled solverGurobi.cpp; a corridor without polytopes, so optimize() is one QP per
    factor): with a solver that always fails, trials_ = |F|; with one that first succeeds at call k, factor_that_worked_ =
    F[k - 1] bit for bit."""
    from oracle import solver_ref as sr
    pb = dict(x0=np.zeros(9), xf=np.r_[2.0, 1.0, 0.5, np.zeros(6)], lim=np.array([2.0, 3.0, 4.0]))
    for fi, ff, inc in ((1.0, 10.0, 1.0), (1.0, 2.0, 0.1), (1.3, 4.0, 1 / 3), (2.75, 20.0, 2.5), (3.0, 2.0, 1.0)):
        F = lib_factors(fi, ff, inc)
        r = sr.gen_new_traj(6, pb["x0"], pb["xf"], pb["lim"], [], 0.01, fi, ff, inc, lambda *a: (False, None, 0.0))
        assert not r["solved"] and r["trials"] == len(F), (fi, ff, inc)
        for k in sorted({1, 2, len(F)} & set(range(1, len(F) + 1))):
            calls = [0]

            def qp(q, Aeq, beq, Ain, bin_, k=k):
                calls[0] += 1
                return (calls[0] >= k, np.zeros(len(q)), 1.0)
            r = sr.gen_new_traj(6, pb["x0"], pb["xf"], pb["lim"], [], 0.01, fi, ff, inc, qp)
            assert r["solved"] and r["trials"] == k and np.float64(r["factor"]).tobytes() == F[k - 1].tobytes(), (fi, ff, inc, k)


def test_next_window_rule(built_lib):
    """faster.cpp:582-588 restated: clamp to 1.0, fractional f*, unchanged unless both sweeps won."""
    L = _lib()
    out = np.zeros(2)
    cases = [(1, 3.0, 20.0, 20.0, 1.0, 10.0), (1, 25.0, 20.0, 20.0, 1.0, 10.0), (1, 2.7, 0.5, 0.25, 1.0, 10.0),
             (1, 1.0000000000000002, 1e-16, 3.0, 1.0, 10.0), (1, 21.3, 20.0, 20.0, 1.0, 10.0), (0, 5.0, 20.0, 20.0, 3.5, 7.25),
             (0, np.nan, 20.0, 20.0, 4.0, 2.0)]
    for both, f, g, gp, fi, ff in cases:
        L.emu_host_next_window(both, f, g, gp, fi, ff, _p(out))
        want = np.array(pwo.next_window(bool(both), f, g, gp, fi, ff))
        assert out.tobytes() == want.tobytes(), (both, f, g, gp)
    L.emu_host_next_window(1, 3.0, 20.0, 20.0, 1.0, 10.0, _p(out))
    assert list(out) == [1.0, 23.0]
    L.emu_host_next_window(1, 21.3, 20.0, 20.0, 1.0, 10.0, _p(out))
    assert out[0] == 21.3 - 20.0 and out[0] > 1.0


def test_emulated_window_factors_equal_the_host(built_lib):
    L = _lib()
    n, mf = len(WINDOWS), 128
    init = np.array([w[0] for w in WINDOWS] + [np.nan, 1.0, 1e17])
    fin = np.array([w[1] for w in WINDOWS] + [2.0, 200.0, 1e17 + 1e3])
    for inc in (0.1, 1 / 3, 1.0):
        fac, cnt = np.full((len(init), mf), -7.0), np.zeros(len(init), np.int32)
        L.emu_window_factors(len(init), mf, _p(init), _p(fin), inc, _p(fac), _p(cnt))
        for j in range(len(init)):
            want = pwo.factors(init[j], fin[j], inc)
            assert cnt[j] == (-1 if want is None else len(want)), j
            if want is not None:
                k = min(len(want), mf)
                assert fac[j, :k].tobytes() == want[:k].tobytes() and (fac[j, k:] == -7.0).all()
    assert n > 100


def offsets(poly_ofs, N, nf, max_fac, cap, all_limit=0, max_poly=32, block=64):
    po, nf = np.ascontiguousarray(poly_ofs, np.int32), np.ascontiguousarray(nf, np.int32)
    co = np.full(len(po), -7, np.int32)
    _lib().emu_window_offsets(block, len(po) - 1, N, max_fac, all_limit, max_poly, cap, _p(po), _p(nf), _p(co))
    return co


@pytest.mark.parametrize("block", [1, 32, 1024])
def test_emulated_offsets_and_the_capacity_rule(built_lib, block):
    rng = np.random.default_rng(block)
    P = rng.integers(0, 5, 90)
    po = np.concatenate([[0], np.cumsum(P)]).astype(np.int32)
    nf = rng.integers(0, 12, 90).astype(np.int32)
    for N, lim in ((10, 0), (6, 4096)):
        want = capi.window_offsets(po, N, nf, lim)
        tot = int(want[-1])
        assert np.array_equal(offsets(po, N, nf, 11, tot, lim, block=block), want)
        assert np.array_equal(offsets(po, N, nf, 40, tot + 999, lim, block=block), want)        # a capacity above the total
        assert not offsets(po, N, nf, 11, tot - 1, lim, block=block).any()                       # total over the capacity
        assert not offsets(po, N, nf, 10, tot, lim, block=block).any()                           # a corridor over max_fac
        bad = nf.copy()
        bad[37] = -1                                                                             # a refused window
        assert not offsets(po, N, bad, 11, tot, lim, block=block).any()


def test_emulated_expansion_from_the_factor_rows(built_lib):
    """dt = F_j[f] * base bit for bit (FQ_MUL), sigma = the corridor's own list, empty windows expand nothing."""
    L = _lib()
    P = np.array([0, 3, 1, 2, 4, 3])
    po = np.concatenate([[0], np.cumsum(P)]).astype(np.int32)
    wins = [(1.0, 3.0, 0.1), (2.0, 1.0, 0.1), (1.3, 2.0, 0.1), (1.0, 1.0, 0.1), (4.2, 5.1, 0.1), (1.0, 2.2, 0.1)]
    F = [pwo.factors(*x) for x in wins]
    mf = max(len(f) for f in F)
    rows = np.zeros((len(P), mf))
    for j, f in enumerate(F):
        rows[j, :len(f)] = f
    nf = np.array([len(f) for f in F], np.int32)
    base = np.array([0.31, 0.5, 0.7, 0.123456789, 1.1, 0.9])
    for N, lim in ((6, 4096), (10, 0)):
        co = offsets(po, N, nf, mf, 1 << 20, lim)
        n = int(co[-1])
        dt, sig = np.full(n, np.nan), np.full((n, N), 0xee, np.uint8)
        L.emu_expand_window(len(P), N, mf, lim, _p(rows), _p(nf), _p(base), _p(po), _p(co), _p(dt), _p(sig))
        for j in range(len(P)):
            lst = pao.assign_list(N, int(P[j]), lim)
            assert co[j + 1] - co[j] == len(F[j]) * len(lst)
            if not len(F[j]):
                continue
            got = sig[co[j]:co[j + 1]].reshape(len(F[j]), len(lst), N)
            assert all(np.array_equal(got[f], lst) for f in range(len(F[j])))
            assert dt[co[j]:co[j + 1]].tobytes() == np.repeat(F[j] * base[j], len(lst)).tobytes()


def _final_and_window(co_w, co_s, nf_w, nf_s, fac_w, fac_s, wi_w, wi_s, windows, gammas, Nw=4, Ns=3):
    """The record kernel with per-corridor counts, then the window kernel with its next windows written over `windows`."""
    L = _lib()
    n = len(nf_w)
    c = lambda a, t: np.ascontiguousarray(a, t)
    co_w, co_s, nf_w, nf_s, wi_w, wi_s = (c(x, np.int32) for x in (co_w, co_s, nf_w, nf_s, wi_w, wi_s))
    fac_w, fac_s = c(fac_w, np.float64), c(fac_s, np.float64)
    z = np.zeros(n)
    res = np.zeros(n, capi.PAIR_RESULT_DTYPE)
    L.emu_pair_final_window(n, Nw, Ns, _p(co_w), _p(co_s), _p(nf_w), _p(nf_s), _p(wi_w), _p(wi_s), _p(np.zeros(n, np.int32)),
                            _p(np.zeros(n, np.int32)), _p(z), _p(z), _p(z), _p(z), _p(z), _p(z), _p(np.zeros((n, 9))),
                            _p(np.zeros((n, Nw), np.uint8)), _p(np.zeros((n, Ns), np.uint8)), _p(res))
    factor, trials = np.zeros(2 * n), np.zeros(2 * n, np.int32)
    g = c(gammas, np.float64)
    L.emu_pair_window(n, fac_w.shape[1], fac_s.shape[1], _p(res), _p(co_w), _p(co_s), _p(nf_w), _p(nf_s), _p(fac_w), _p(fac_s),
                      _p(windows), _p(g), _p(factor), _p(trials), _p(windows))
    return res, factor, trials


def test_emulated_records_split_by_own_counts(built_lib):
    """Winner indices split by |F_j| x |L_j| per corridor, |F_j| = 0 included; factor, trials and next windows against the
    restatement, with the next windows written over the input windows (aliased)."""
    # corridors: lists of 2, 3, 1, 4 assignments; factor counts 3, 0, 2, 1
    L_ = np.array([2, 3, 1, 4])
    nf_w = np.array([3, 0, 2, 1])
    nf_s = np.array([2, 2, 0, 2])       # [1.2, 1.4] by 0.1: 1.2, 1.3 (the third sum is 1.4000000000000001)
    co_w = np.concatenate([[0], np.cumsum(L_ * nf_w)])
    co_s = np.concatenate([[0], np.cumsum(L_ * nf_s)])
    wins = dict(init_whole=np.array([1.0, 5.0, 2.5, 3.0]), final_whole=np.array([3.0, 4.0, 3.5, 3.0]),
                init_safe=np.array([1.0, 1.0, 2.0, 1.2]), final_safe=np.array([1.1, 1.1, 1.0, 1.4]))
    Fw = [pwo.factors(a, b, 1.0) for a, b in zip(wins["init_whole"], wins["final_whole"])]
    Fs = [pwo.factors(a, b, 0.1) for a, b in zip(wins["init_safe"], wins["final_safe"])]
    assert [len(f) for f in Fw] == list(nf_w) and [len(f) for f in Fs] == list(nf_s)
    rows = lambda F: np.array([np.pad(f, (0, 3 - len(f))) for f in F])
    wi_w = np.array([5, -1, 1, 3])           # corridor 0: factor index 2, assignment 1; corridor 2: factor index 1, assignment 0
    wi_s = np.array([3, -1, -1, -1])         # corridor 0: factor 1, assignment 1; corridor 3: no safe winner
    windows = np.concatenate([wins[k] for k in pwo.WINDOW_KEYS])
    gam = (2.0, 3.0, 0.5, 0.25)
    res, factor, trials = _final_and_window(co_w, co_s, nf_w, nf_s, rows(Fw), rows(Fs), wi_w, wi_s, windows, gam)
    assert list(res["whole_dt_index"]) == [2, -1, 1, 0] and list(res["whole_sigma_index"]) == [1, -1, 0, 3]
    assert list(res["safe_dt_index"]) == [1, -1, -1, -1] and list(res["safe_sigma_index"]) == [1, -1, -1, -1]
    want = pwo.window_outputs(res, wins, Fw, Fs, gam)
    n = 4
    assert factor[:n].tobytes() == want["factor_whole"].tobytes() and factor[n:].tobytes() == want["factor_safe"].tobytes()
    assert list(trials[:n]) == list(want["trials_whole"]) == [3, 0, 2, 1]
    assert list(trials[n:]) == list(want["trials_safe"]) == [2, 0, 0, 2]
    for i, k in enumerate(pwo.WINDOW_KEYS):
        assert windows[i * n:(i + 1) * n].tobytes() == want["next_" + k].tobytes(), k
    assert windows[0] == 1.0 and windows[n] == 6.0                 # corridor 0: both won at f*_w = 3: [max(1, 1), 3 + 3]
    assert windows[2 * n] == 1.0 and windows[3 * n] == 1.1 + 0.25  # safe f* = 1.1: [max(0.6, 1), 1.35]
    # an emptied sweep (every offset 0): nothing ran, every window stays
    windows2 = np.concatenate([wins[k] for k in pwo.WINDOW_KEYS])
    zeros = np.zeros(n + 1, np.int32)
    res, factor, trials = _final_and_window(zeros, zeros, nf_w, nf_s, rows(Fw), rows(Fs), -np.ones(n), -np.ones(n), windows2, gam)
    assert (res["whole_dt_index"] == -1).all() and not trials.any() and np.isnan(factor).all()
    assert windows2.tobytes() == np.concatenate([wins[k] for k in pwo.WINDOW_KEYS]).tobytes()


def test_window_dev_submission_through_the_emulated_kernels(built_lib, oracle):
    """fq_replan_pairs_window_dev's kernels in submission order on a small mixed batch (whole polytopes 3, 2, 1; safe 1, 4, 2;
    one window per corridor, corridor 1's safe window empty) against the CPU chain corridor by corridor."""
    from test_kernel_emu_cpu import solve_multi, _emu, _pair_lib
    from test_pair_assign_cpu import _mixed_workload
    w = _mixed_workload()
    P, Nw, Ns, DC, lim_ = w["n_prob"], w["N_whole"], w["N_safe"], w["DC"], 0
    K, S, A = _pair_lib(), _emu(), _lib()
    c = lambda a, t: np.ascontiguousarray(a, t)
    wins = dict(init_whole=np.array([1.0, 2.0, 1.5]), final_whole=np.array([2.0, 3.0, 2.5]),
                init_safe=np.array([1.0, 2.0, 1.0]), final_safe=np.array([1.2, 1.0, 1.1]))
    inc = {"whole": 1.0, "safe": 0.1}
    windows = np.concatenate([wins[k] for k in pwo.WINDOW_KEYS])
    x0, xfw, xfs, lim = c(w["x0"], np.float64), c(w["xf_whole"], np.float64), c(w["xf_safe"], np.float64), c(w["lim"], np.float64)
    st, out = {}, {}
    mf = 4
    for kind, N, ff, xf in (("whole", Nw, True, xfw), ("safe", Ns, False, xfs)):
        xs = x0 if kind == "whole" else st["x0_safe"]
        rows, nf = np.zeros((P, mf)), np.zeros(P, np.int32)
        A.emu_window_factors(P, mf, _p(c(wins["init_" + kind], np.float64)), _p(c(wins["final_" + kind], np.float64)), inc[kind], _p(rows), _p(nf))
        base = np.zeros(P)
        K.emu_dtbase(P, N, C.c_double(DC), _p(xs), _p(xf), _p(lim), _p(base))
        co = offsets(w["poly_ofs_" + kind], N, nf, mf, 1 << 20, lim_)
        n = int(co[-1])
        dt, sig = np.full(n, np.nan), np.zeros((n, N), np.uint8)
        A.emu_expand_window(P, N, mf, lim_, _p(rows), _p(nf), _p(base), _p(c(w["poly_ofs_" + kind], np.int32)), _p(co), _p(dt), _p(sig))
        feas, cost, _, _ = solve_multi(S, N, ff, xs, xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind], co, dt, sig,
                                       max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        wi, wc, wdt, ws, wo = np.zeros(P, np.int32), np.zeros(P), np.zeros(P), np.zeros((P, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_select_multi(P, N, 0, _p(co), _p(dt), _p(sig), _p(feas), _p(cost), _p(wi), _p(wc), _p(wdt), _p(ws), _p(wo))
        _, _, coeffs, _ = solve_multi(S, N, ff, xs, xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind], wo, wdt, ws,
                                      max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        st[kind] = dict(base=base, wi=wi, wc=wc, wdt=wdt, ws=ws, co=co, rows=rows, nf=nf)
        out["feasible_" + kind], out["cost_" + kind] = feas, cost
        if kind == "whole":
            x0s, nsamp, ksafe = np.zeros((P, 9)), np.zeros(P, np.int32), np.zeros(P, np.int32)
            K.emu_pair_mid(P, N, C.c_double(DC), C.c_double(w["r_fraction"]), _p(c(coeffs, np.float64)), _p(wdt), _p(wi), _p(x0s), _p(nsamp),
                           _p(ksafe))
            st["x0_safe"], st["nsamp"], st["ksafe"] = x0s, nsamp, ksafe
    a, b = st["whole"], st["safe"]
    res = np.zeros(P, capi.PAIR_RESULT_DTYPE)
    A.emu_pair_final_window(P, Nw, Ns, _p(a["co"]), _p(b["co"]), _p(a["nf"]), _p(b["nf"]), _p(a["wi"]), _p(b["wi"]), _p(st["nsamp"]),
                            _p(st["ksafe"]), _p(a["wc"]), _p(b["wc"]), _p(a["wdt"]), _p(b["wdt"]), _p(a["base"]), _p(b["base"]),
                            _p(st["x0_safe"]), _p(a["ws"]), _p(b["ws"]), _p(res))
    factor, trials = np.zeros(2 * P), np.zeros(2 * P, np.int32)
    gam = np.array([2.0, 2.0, 0.5, 0.5])
    A.emu_pair_window(P, mf, mf, _p(res), _p(a["co"]), _p(b["co"]), _p(a["nf"]), _p(b["nf"]), _p(a["rows"]), _p(b["rows"]), _p(windows),
                      _p(gam), _p(factor), _p(trials), _p(windows))
    o = pwo.replan_pairs_window(w, wins, lim_, inc=(1.0, 0.1), gamma=tuple(gam), threads=4, dt_base_whole=res["whole_dt_base"],
                                dt_base_safe=res["safe_dt_base"])
    for k in ("whole", "safe"):
        assert np.array_equal(st[k]["co"], o["cand_ofs_" + k]), k
        assert np.array_equal(out["feasible_" + k], o["feasible_" + k]), k
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(res[f], o[f]), f
    assert (res["whole_dt_index"] >= 0).any() and res["safe_dt_index"][1] == -1
    assert factor[:P].tobytes() == o["factor_whole"].tobytes() and factor[P:].tobytes() == o["factor_safe"].tobytes()
    assert np.array_equal(trials[:P], o["trials_whole"]) and np.array_equal(trials[P:], o["trials_safe"])
    for i, k in enumerate(pwo.WINDOW_KEYS):
        assert windows[i * P:(i + 1) * P].tobytes() == o["next_" + k].tobytes(), k


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_pair_window));\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_window, %s));\n' % f for f, _ in capi.PairWindow._fields_) +
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.PairWindow)
    assert got[1:] == [getattr(capi.PairWindow, f).offset for f, _ in capi.PairWindow._fields_]
