"""The exact chained replan (fq_replan_pairs_exact*) without a GPU: the product's tree kernels (faster_b200/csrc/fq_bnb.cuh:
roots, the generalised level kernel, certify, resolve) under the block emulation of tests/cpp/simt_emu/ on batches of N = 6
corridors, fed list winners computed on the CPU, against the CPU restatement of tests/pair_exact_oracle.py; a batch against
each corridor alone; the one-corridor strict path of fq_gen_new_traj_exact against the oracle's branch-and-bound; the
presolve of fq_presolve.h on the host against the roots kernel; the ranking of assignments and the ctypes layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_assign_oracle as pao
import pair_exact_oracle as peo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
ROW_TOL = 1e-8
FACTORS = np.array([5.0, 6.0, 7.0, 8.0])                 # from factor 5, where 5007 and 5055 have non-monotone optima


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_exact_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_exact_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_presolve_host.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p, C.c_double, C.c_void_p]
        L.emu_presolve_host.restype = None
        L.emu_roots.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_int] + \
                               [C.c_void_p] * 3
        L.emu_roots.restype = None
        L.emu_exact_stage.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_int, C.c_double,
                                     C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 7
        L.emu_strict_tree.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 6 + [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_double,
                                     C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 4
        L.emu_fallback.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 14
        L.emu_fallback.restype = None
        L.emu_rank.argtypes = [C.c_int, C.c_int, C.c_longlong, C.c_void_p]
        L.emu_rank.restype = C.c_longlong
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def batch(pbs, ff):
    """One sweep's corridors (corridor.make_* dicts, N = 6) with their monotone lists and FACTORS -> dict."""
    N = pbs[0]["N"]
    po, fo, rows = [0], [0], []
    for pb in pbs:
        for A, b in pb["polys"]:
            rows.append(np.hstack([np.asarray(A, float), np.asarray(b, float)[:, None]]))
            fo.append(fo[-1] + len(b))
        po.append(po[-1] + len(pb["polys"]))
    from oracle import pyoracle as po_
    base = np.array([max(po_.dt_initial(pb["x0"], pb["xf"], pb["lim"], N), 0.02) for pb in pbs])
    lists = [pao.assign_list(N, len(pb["polys"]), 0) for pb in pbs]
    co, dts, sig = [0], [], []
    for j, L in enumerate(lists):
        for f in FACTORS:
            dts += [f * base[j]] * len(L)
            sig.append(L)
        co.append(co[-1] + len(FACTORS) * len(L))
    return dict(N=N, ff=ff, n=len(pbs), x0=np.ascontiguousarray([pb["x0"] for pb in pbs], float),
                xf=np.ascontiguousarray([pb["xf"] for pb in pbs], float), lim=np.ascontiguousarray([pb["lim"] for pb in pbs], float),
                poly_ofs=np.asarray(po, np.int32), face_ofs=np.asarray(fo, np.int32), Ab=np.ascontiguousarray(np.vstack(rows)),
                cand_ofs=np.asarray(co, np.int32), dt=np.asarray(dts, float), sigma=np.ascontiguousarray(np.vstack(sig), np.uint8),
                lists=lists, base=base, pbs=pbs, max_faces=int(max(fo[po[j + 1]] - fo[po[j]] for j in range(len(pbs)))),
                max_poly_faces=int(np.diff(fo).max()))


def list_winners(b, oracle):
    """genNewTraj's selection over each corridor's list, solved by the CPU restatement (fq_select_multi_kernel's outputs)."""
    feas, cost = oracle.solve_multi(b["N"], b["ff"], b["x0"], b["xf"], b["lim"], b["poly_ofs"], b["face_ofs"], b["Ab"], b["cand_ofs"],
                                    b["dt"], b["sigma"], threads=4)
    n, N = b["n"], b["N"]
    wi, wc, wd, ws = np.full(n, -1, np.int32), np.full(n, np.inf), np.full(n, np.nan), np.zeros((n, N), np.uint8)
    for j in range(n):
        c0, c1 = b["cand_ofs"][j], b["cand_ofs"][j + 1]
        L = len(b["lists"][j])
        for f in range(len(FACTORS)):
            idx = np.arange(c0 + f * L, c0 + (f + 1) * L)
            ok = feas[idx].astype(bool)
            if ok.any():
                i = idx[ok][np.argmin(cost[idx][ok])]
                wi[j], wc[j], wd[j], ws[j] = i - c0, cost[i], b["dt"][i], b["sigma"][i]
                break
    return wi, wc, wd, ws


def exact_stage(b, oracle, cap=4096, cpc=2, win=None):
    L = _lib()
    TZ, T0, FT = capi.plan_tables(b["N"], b["ff"])
    wi, wc, wd, ws = [np.ascontiguousarray(x).copy() for x in (win or list_winners(b, oracle))]
    n = b["n"]
    changed, exact, nodes = np.zeros(n, np.uint8), np.zeros(n, np.int32), np.zeros(n, np.int64)
    rc = L.emu_exact_stage(b["N"], int(b["ff"]), _p(TZ), _p(T0), _p(FT), n, _p(b["x0"]), _p(b["xf"]), _p(b["lim"]), _p(b["poly_ofs"]),
                           _p(b["face_ofs"]), _p(b["Ab"]), b["max_faces"], b["max_poly_faces"], ROW_TOL, 0, _p(b["cand_ofs"]), _p(b["dt"]),
                           len(FACTORS), cap, cpc, _p(wi), _p(wc), _p(wd), _p(ws), _p(changed), _p(exact), _p(nodes))
    assert rc == 0
    return dict(win_idx=wi, win_cost=wc, win_dt=wd, win_sig=ws, changed=changed, exact=exact, nodes=nodes)


def corridors():
    """N = 6: the 5007 / 5055 seeds and a few ordinary corridors with 3 to 5 polytopes, whole and safe."""
    whole = [cr.make_corridor(5007, 3, 6, "uav", True)] + [cr.make_corridor(5100 + s, P, 6, "uav", True) for s, P in ((0, 3), (1, 4), (2, 5))]
    safe = [cr.make_corridor(5055, 4, 6, "uav", False)] + [cr.make_corridor(5200 + s, P, 6, "uav", False) for s, P in ((0, 3), (1, 4), (2, 5))]
    return whole, safe


@pytest.fixture(scope="module")
def stages(built_lib, oracle):
    whole, safe = corridors()
    out = {}
    for kind, pbs, ff in (("whole", whole, True), ("safe", safe, False)):
        b = batch(pbs, ff)
        out[kind] = (b, exact_stage(b, oracle))
    return out


@pytest.mark.parametrize("kind", ["whole", "safe"])
def test_emulated_stage_equals_the_restatement(stages, oracle, kind):
    b, got = stages[kind]
    N, ff = b["N"], b["ff"]
    for j, pb in enumerate(b["pbs"]):
        want = peo.exact_sweep(N, pb["x0"], pb["xf"], pb["lim"], pb["polys"], FACTORS * b["base"][j], ff)
        L = len(b["lists"][j])
        assert got["exact"][j] == 1, j
        d = got["win_idx"][j] // L if got["win_idx"][j] >= 0 else -1
        assert d == want["dt_index"], j
        if d < 0:
            continue
        assert abs(got["win_cost"][j] - want["cost"]) <= 1e-7 * max(1.0, want["cost"]), j
        st, c2, _, _ = oracle.solve_fixed(N, pb["x0"], pb["xf"], pb["lim"], got["win_dt"][j], pb["polys"], got["win_sig"][j], ff)
        assert st == 1 and abs(c2 - want["cost"]) <= 1e-9 * max(1.0, want["cost"]), j
        if got["changed"][j]:        # the tie rule: no assignment lexicographically below the winner within 1e-9 of it
            assert np.array_equal(got["win_sig"][j], peo.lexmin_tie(N, pb["x0"], pb["xf"], pb["lim"], got["win_dt"][j], pb["polys"], ff,
                                                                    want["cost"])), j
    if kind == "whole":
        assert got["changed"][0] == 1 and np.any(np.diff(got["win_sig"][0].astype(int)) < 0)   # 5007's non-monotone optimum


@pytest.mark.parametrize("kind", ["whole", "safe"])
def test_batch_equals_each_corridor_alone(stages, oracle, kind):
    b, got = stages[kind]
    for j, pb in enumerate(b["pbs"]):
        one = batch([pb], b["ff"])
        o = exact_stage(one, oracle, cap=4096, cpc=1)
        for k in ("win_cost", "win_dt", "win_sig", "changed", "exact"):
            assert o[k][0].tobytes() == got[k][j].tobytes(), (j, k)
        L = len(b["lists"][j])
        assert o["win_idx"][0] == got["win_idx"][j] and (o["win_idx"][0] < 0 or o["win_idx"][0] // L == got["win_idx"][j] // L)


def test_strict_tree_gives_the_exact_sweep(built_lib, oracle):
    """fq_gen_new_traj_exact's use of the level kernel (one corridor, strict pruning, one warp per child, the last improving
    leaf of the first time allocation with a finite incumbent) against the oracle's branch-and-bound sweep."""
    L = _lib()
    for pb, ff in ((cr.make_corridor(5007, 3, 6, "uav", True), True), (cr.make_corridor(5055, 4, 6, "uav", False), False),
                   (cr.make_corridor(5101, 4, 6, "uav", True), True)):
        b = batch([pb], ff)
        wi, wc, _, _ = list_winners(b, oracle)
        nl = len(b["lists"][0])
        fstar = int(wi[0] // nl) if wi[0] >= 0 else -1
        n_dt = len(FACTORS)
        dts = FACTORS * b["base"][0]
        inc = np.full(n_dt, np.inf)
        if fstar >= 0:
            inc[fstar] = wc[0]
        inc = np.ascontiguousarray(inc.view(np.uint64))
        TZ, T0, FT = capi.plan_tables(6, ff)
        leaves = np.zeros(4096, np.dtype([("dt", np.int32), ("pad", np.int32), ("cost", np.float64), ("sigma", np.uint8, 16)]))
        n_leaves, exact, nodes = C.c_int(0), C.c_int(0), C.c_longlong(0)
        assert L.emu_strict_tree(6, int(ff), _p(TZ), _p(T0), _p(FT), _p(b["x0"][0]), _p(b["xf"][0]), _p(b["lim"][0]), len(pb["polys"]),
                                 _p(b["face_ofs"]), _p(b["Ab"]), b["max_poly_faces"], ROW_TOL, n_dt, _p(dts),
                                 fstar + 1 if fstar >= 0 else n_dt, _p(inc), 4096, _p(leaves), C.addressof(n_leaves), C.addressof(exact),
                                 C.addressof(nodes)) == 0
        assert exact.value == 1
        want = peo.exact_sweep(6, pb["x0"], pb["xf"], pb["lim"], pb["polys"], dts, ff)
        got_dt, got_cost = -1, np.inf
        for d in range(fstar + 1 if fstar >= 0 else n_dt):
            c = inc[d:d + 1].view(np.float64)[0]
            if c < np.inf:
                got_dt, got_cost = d, c
                break
        assert got_dt == want["dt_index"]
        if got_dt >= 0:
            assert abs(got_cost - want["cost"]) <= 1e-7 * max(1.0, want["cost"])


def test_presolve_host_equals_the_roots_kernel(built_lib):
    """Random start states, some control points placed exactly on a face: fq_presolve.h on the host and in the emulated
    roots kernel give the same root lists."""
    L = _lib()
    rng = np.random.default_rng(3)
    n, N, nf = 24, 6, 5
    polys_all, x0s, xfs = [], [], []
    for j in range(n):
        P = int(rng.integers(2, 5))
        polys = []
        for p in range(P):
            A = rng.normal(size=(6, 3))
            A /= np.linalg.norm(A, axis=1, keepdims=True)
            c = rng.normal(scale=0.5, size=3)
            polys.append((A, A @ c + rng.uniform(0.3, 1.5, 6)))
        x0 = np.concatenate([rng.normal(scale=0.6, size=3), rng.normal(scale=1.0, size=3), rng.normal(scale=1.0, size=3)])
        xf = np.concatenate([rng.normal(scale=0.6, size=3), np.zeros(6)])
        if j % 3 == 0:          # cp0 exactly on face 0 of polytope 0, as the presolve computes the row
            A, b = polys[0]
            b = b.copy()
            b[0] = A[0, 0] * x0[0] + A[0, 1] * x0[1] + A[0, 2] * x0[2]
            polys[0] = (A, b)
        if j % 4 == 1:          # xf exactly on a face
            A, b = polys[-1]
            b = b.copy()
            b[2] = A[2, 0] * xf[0] + A[2, 1] * xf[1] + A[2, 2] * xf[2]
            polys[-1] = (A, b)
        polys_all.append(polys)
        x0s.append(x0)
        xfs.append(xf)
    counts = []
    for ff in (0, 1):
        pbs = [dict(N=N, x0=x0s[j], xf=xfs[j], lim=np.array([2.0, 3.0, 5.0]), polys=polys_all[j]) for j in range(n)]
        po, fo, rows = [0], [0], []
        for pl in polys_all:
            for A, b in pl:
                rows.append(np.hstack([A, b[:, None]]))
                fo.append(fo[-1] + len(b))
            po.append(po[-1] + len(pl))
        po, fo, Ab = np.asarray(po, np.int32), np.asarray(fo, np.int32), np.ascontiguousarray(np.vstack(rows))
        dts = rng.uniform(0.05, 1.0, (n, nf))
        cand_ofs, cand_dt = [0], []
        for j in range(n):
            Lj = len(pao.assign_list(N, len(polys_all[j]), 0))
            for f in range(nf):
                cand_dt += [dts[j, f]] * Lj
            cand_ofs.append(cand_ofs[-1] + nf * Lj)
        cand_ofs, cand_dt = np.asarray(cand_ofs, np.int32), np.asarray(cand_dt)
        roots, n_roots, status = np.zeros(n * nf, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
        X0, XF = np.ascontiguousarray(x0s), np.ascontiguousarray(xfs)
        L.emu_roots(N, ff, n, _p(X0), _p(XF), _p(po), _p(fo), _p(Ab), 2047, ROW_TOL, _p(cand_ofs), _p(cand_dt), nf, _p(roots), _p(n_roots),
                    _p(status))
        for j in range(n):
            assert status[j] == 1
            host = np.zeros(nf, np.uint8)
            L.emu_presolve_host(len(polys_all[j]), _p(np.ascontiguousarray(fo[po[j]:po[j + 1] + 1])), _p(Ab), _p(X0[j]), _p(XF[j]), ff, nf,
                                _p(np.ascontiguousarray(dts[j])), ROW_TOL, _p(host))
            assert list(roots[j * nf:j * nf + n_roots[j]]) == list(np.flatnonzero(host)), (ff, j)
            counts.append(int(host.sum()))
    assert 0 < sum(counts) < len(counts) * nf


def test_unconfirmed_tree_winner_falls_back_to_the_list_winner(built_lib):
    """The winners' coefficient solve may reject a winner the warm-started tree proved (iteration cap, or infeasible on a
    cold start).  Such a corridor gets its list winner back, exact = 0 and the second solve's coefficients; a confirmed tree
    winner, an unchanged corridor and a corridor whose list had no winner are handled as the resolve left them, except that
    the last reverts to "none" with no second solve."""
    L = _lib()
    n, N = 4, 5
    win_idx = np.array([7, 9, 11, 13], np.int32)
    win_cost = np.array([1.0, 2.0, 3.0, 4.0])
    win_dt = np.array([0.5, 0.6, 0.7, 0.8])
    win_sig = np.arange(n * N, dtype=np.uint8).reshape(n, N) % 3
    keep_idx = np.array([2, 3, 4, -1], np.int32)
    keep_cost = np.array([1.5, 2.5, 3.5, np.inf])
    keep_dt = np.array([0.55, 0.65, 0.75, np.nan])
    keep_sig = np.full((n, N), 1, np.uint8)
    changed = np.array([1, 1, 0, 1], np.uint8)           # 0: rejected tree winner; 1: confirmed; 2: list winner; 3: rejected, no list winner
    exact = np.ones(n, np.int32)
    feasible = np.array([0, 1, 0, 0], np.uint8)
    redo_dt = np.zeros(n)
    redo_coeffs = np.arange(n * N * 12, dtype=np.float64).reshape(n, N, 12) + 1000
    coeffs = np.zeros((n, N, 12))
    before = [x.copy() for x in (win_idx, win_cost, win_dt, win_sig)]
    L.emu_fallback(n, N, _p(win_idx), _p(win_cost), _p(win_dt), _p(win_sig), _p(keep_idx), _p(keep_cost), _p(keep_dt), _p(keep_sig),
                   _p(changed), _p(exact), _p(feasible), _p(redo_dt), _p(redo_coeffs), _p(coeffs))
    for j in (0, 3):
        assert win_idx[j] == keep_idx[j] and changed[j] == 0 and exact[j] == 0
        assert win_cost[j].tobytes() == keep_cost[j].tobytes() and win_dt[j].tobytes() == keep_dt[j].tobytes()
        assert np.array_equal(win_sig[j], keep_sig[j])
    assert redo_dt[0] == keep_dt[0] and np.array_equal(coeffs[0], redo_coeffs[0])
    for j in (1, 2, 3):
        assert np.isnan(redo_dt[j]) and not coeffs[j].any()
    for j in (1, 2):
        assert win_idx[j] == before[0][j] and win_cost[j] == before[1][j] and win_dt[j] == before[2][j]
        assert np.array_equal(win_sig[j], before[3][j]) and exact[j] == 1
    assert changed[1] == 1 and changed[2] == 0


def test_rank_inverts_the_lists(built_lib):
    """The records' *_sigma_index of a tree winner (fq_assign.h rank, used by fq_pair_final_kernel): the index in L_j, -1 off it."""
    L = _lib()
    for N, P, lim in ((4, 3, 0), (6, 4, 0), (5, 2, 0), (4, 3, 4096), (3, 1, 0), (10, 4, 0), (16, 3, 0)):
        lst = pao.assign_list(N, P, lim)
        for i in range(0, len(lst), max(1, len(lst) // 500)):
            s = np.ascontiguousarray(lst[i])
            assert L.emu_rank(N, P, lim, _p(s)) == i == peo.list_index(N, P, lim, s)
        rng = np.random.default_rng(N * 10 + P)
        for _ in range(200):
            s = np.ascontiguousarray(rng.integers(0, P, N).astype(np.uint8))
            want = peo.list_index(N, P, lim, s)
            assert L.emu_rank(N, P, lim, _p(s)) == want
            assert (want >= 0) == (lim > 0 or bool(np.all(np.diff(s.astype(int)) >= 0)))


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_pair_exact));\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_exact, %s));\n' % f for f, _ in capi.PairExact._fields_) +
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.PairExact)
    assert got[1:] == [getattr(capi.PairExact, f).offset for f, _ in capi.PairExact._fields_]
    assert capi.EXACT_KEYS == [f for f, _ in capi.PairExact._fields_]
