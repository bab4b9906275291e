"""Per-corridor assignment lists of the chained replan (fq_replan_pairs_assign*) without a GPU: the product's kernel SOURCE
(faster_b200/csrc/fq_pair.cuh: offsets, unranking grid expansion, result records) runs under the block emulation of
tests/cpp/simt_emu/ and is compared with enumerated lists, with fq_pair_assign_count, and -- together with the emulated solve
and selection kernels -- with the CPU chain on a small mixed batch."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi

import pair_assign_oracle as pao

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 1 << 20
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_assign_emu.so")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_assign_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
                os.path.join(ROOT, "faster_b200", "csrc", "fq_pair.cuh"), os.path.join(ROOT, "faster_b200", "csrc", "fq_assign.h"),
                os.path.join(ROOT, "faster_b200", "csrc", "fq_kernels.cuh")]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", os.path.join(ROOT, "faster_b200", "csrc"),
                                   "-I", os.path.join(ROOT, "include"), srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_list_len.restype = C.c_longlong
        L.emu_list_len.argtypes = [C.c_int, C.c_int, C.c_longlong]
        L.emu_assign_offsets.restype = None
        L.emu_assign_offsets.argtypes = [C.c_int] * 4 + [C.c_longlong, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p]
        L.emu_expand_assign.restype = None
        L.emu_expand_assign.argtypes = [C.c_int] * 3 + [C.c_longlong] + [C.c_void_p] * 6
        L.emu_pair_final_assign.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data)


def offsets(poly_ofs, N, n_fac, all_limit, max_poly=32, n_cand=None, block=64):
    po = np.ascontiguousarray(poly_ofs, np.int32)
    n = len(po) - 1
    if n_cand is None:
        n_cand = int(capi.assign_offsets(po, N, n_fac, all_limit)[-1])
    co = np.full(n + 1, -7, np.int32)
    _lib().emu_assign_offsets(block, n, N, n_fac, all_limit, max_poly, n_cand, _p(po), _p(co))
    return co


def expand(poly_ofs, N, factors, all_limit, dt_base, cand_ofs):
    po, co = np.ascontiguousarray(poly_ofs, np.int32), np.ascontiguousarray(cand_ofs, np.int32)
    fac, base = np.ascontiguousarray(factors, np.float64), np.ascontiguousarray(dt_base, np.float64)
    n = int(co[-1])
    dt, sig = np.full(n, np.nan), np.full((n, N), 0xee, np.uint8)
    _lib().emu_expand_assign(len(po) - 1, N, len(fac), all_limit, _p(fac), _p(base), _p(po), _p(co), _p(dt), _p(sig))
    return dt, sig


def _odometer(N, P):
    idx = np.arange(P ** N, dtype=np.int64)[:, None]
    return ((idx // (P ** np.arange(N - 1, -1, -1, dtype=np.int64))[None, :]) % P).astype(np.uint8)


def _expected(N, P, all_limit):
    if P == 0:
        return np.zeros((1, N), np.uint8)
    if P > 1 and P ** N <= all_limit:
        return _odometer(N, P)
    return capi.monotone_sigmas(N, P)


def _len(N, P, all_limit):
    if P == 0:
        return 1
    n = P ** N if P > 1 and P ** N <= all_limit else math.comb(N + P - 1, N)
    return n if n <= CAP else -1


def _check_one_corridor(N, P, all_limit):
    exp = _expected(N, P, all_limit)
    co = offsets([0, P], N, 1, all_limit)
    assert list(co) == [0, len(exp)], (N, P, all_limit)
    dt, sig = expand([0, P], N, [1.0], all_limit, [0.5], co)
    assert np.array_equal(sig, exp), (N, P, all_limit)
    assert (dt == 0.5).all()


@pytest.mark.parametrize("all_limit", [0, CAP])
def test_unranking_reproduces_the_enumerations(built_lib, all_limit):
    """Every N in 2..16 with P in 0..8: the device unranking equals fq_monotone_sigmas (all_limit 0) or the ALL odometer
    (segment 0 most significant) wherever P^N fits all_limit = 2^20, row for row."""
    for N in range(2, 17):
        for P in range(0, 9):
            if _len(N, P, all_limit) < 0:
                assert capi.assign_count(N, P, all_limit) < 0
                continue
            _check_one_corridor(N, P, all_limit)


def test_unranking_sampled_up_to_32_polytopes(built_lib):
    rng = np.random.default_rng(3)
    pairs = [(N, P) for N in range(2, 17) for P in range(9, 33) if _len(N, P, 0) > 0]
    assert (5, 32) in pairs and (2, 32) in pairs
    for i in rng.choice(len(pairs), 14, replace=False):
        _check_one_corridor(*pairs[i], 0)
    _check_one_corridor(5, 32, 0)                       # C(36, 5) = 376 992 assignments
    _check_one_corridor(4, 32, CAP)                     # 32^4 = 2^20 assignments, all of them


def test_assign_count_agrees(built_lib):
    L = _lib()
    for N in range(1, 17):
        for P in range(0, 33):
            for lim in (0, 1, 729, 4096, CAP, 1 << 40):
                want = _len(N, P, lim)
                got = capi.assign_count(N, P, lim)
                assert (got < 0 and want < 0) or got == want, (N, P, lim, got, want)
                assert L.emu_list_len(N, P, lim) == (want if want >= 0 else -1)
    assert capi.assign_count(6, 3, 4096) == 729 and capi.assign_count(6, 3, 0) == 28 and capi.assign_count(6, 3, 728) == 28
    for bad in ((0, 3, 0), (17, 3, 0), (6, -1, 0), (6, 33, 0), (6, 3, -1), (16, 32, 0)):
        assert capi.assign_count(*bad) < 0, bad


@pytest.mark.parametrize("block", [1, 32, 1024])
def test_offsets_of_a_mixed_batch(built_lib, block):
    """The scan over any CTA size equals the host offsets; a wrong total or a corridor above max_poly empties the sweep."""
    rng = np.random.default_rng(block)
    P = rng.integers(0, 6, 150)
    po = np.concatenate([[0], np.cumsum(P)]).astype(np.int32)
    for N, lim in ((10, 0), (6, 4096)):
        want = capi.assign_offsets(po, N, 5, lim)
        assert np.array_equal(offsets(po, N, 5, lim, block=block), want)
        assert not offsets(po, N, 5, lim, n_cand=int(want[-1]) + 1, block=block).any()
        assert not offsets(po, N, 5, lim, n_cand=int(want[-1]) - 1, block=block).any()
        assert not offsets(po, N, 5, lim, max_poly=4, block=block).any()


def test_expansion_of_a_mixed_batch(built_lib):
    """Factor-major candidates per corridor: dt = factor * base (bit-equal products), sigma = the corridor's own list."""
    P = np.array([0, 3, 1, 2, 4, 3])
    po = np.concatenate([[0], np.cumsum(P)]).astype(np.int32)
    fac = np.array([1.0, 1.25, 1.5])
    base = np.array([0.31, 0.5, 0.7, 0.123456789, 1.1, 0.9])
    for N, lim in ((6, 4096), (10, 0)):
        co = offsets(po, N, len(fac), lim)
        dt, sig = expand(po, N, fac, lim, base, co)
        for j in range(len(P)):
            lst = pao.assign_list(N, int(P[j]), lim)
            got = sig[co[j]:co[j + 1]].reshape(len(fac), len(lst), N)
            assert all(np.array_equal(got[f], lst) for f in range(len(fac)))
            assert np.array_equal(dt[co[j]:co[j + 1]], np.repeat(fac * base[j], len(lst)))
    # an emptied sweep expands nothing
    dt, sig = expand(po, 10, fac, 0, base, np.zeros(len(P) + 1, np.int32))
    assert len(dt) == 0


# ---- a mixed batch through every kernel of fq_replan_pairs_assign_dev's submission, against the CPU chain
def _mixed_workload(n_fac=2):
    """Three config-4 fixture corridors with their polytope lists trimmed to mixed counts (whole 3, 2, 1; safe 1, 4, 2)."""
    import bench
    w = bench.load_cfg4(0, 3)
    keep = dict(whole=[3, 2, 1], safe=[1, 4, 2])
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        npo, nfo, rows = [0], [0], []
        for j in range(3):
            for p in range(po[j], po[j] + keep[kind][j]):
                rows.append(Ab[fo[p]:fo[p + 1]])
                nfo.append(nfo[-1] + fo[p + 1] - fo[p])
            npo.append(npo[-1] + keep[kind][j])
        w["poly_ofs_" + kind], w["face_ofs_" + kind] = np.array(npo, np.int32), np.array(nfo, np.int32)
        w["Ab_" + kind] = np.ascontiguousarray(np.vstack(rows))
        nf = np.array(nfo)
        w["max_faces_" + kind] = int(max(nf[npo[j + 1]] - nf[npo[j]] for j in range(3)))
        w["max_poly_faces_" + kind] = int(np.diff(nf).max())
        w["factors_" + kind] = np.ascontiguousarray(w["factors_" + kind][:n_fac])
        w["sigmas_" + kind] = np.zeros((0, w["N_" + kind]), np.uint8)
    return w


def test_mixed_batch_through_the_emulated_kernels(built_lib, oracle):
    from test_kernel_emu_cpu import solve_multi, _emu, _pair_lib
    w = _mixed_workload()
    P, Nw, Ns, DC, lim_ = w["n_prob"], w["N_whole"], w["N_safe"], w["DC"], 0
    K, S, A = _pair_lib(), _emu(), _lib()
    c = lambda a, t: np.ascontiguousarray(a, t)
    x0, xfw, xfs, lim = c(w["x0"], np.float64), c(w["xf_whole"], np.float64), c(w["xf_safe"], np.float64), c(w["lim"], np.float64)
    st, out = {}, {}
    for kind, N, ff, xf in (("whole", Nw, True, xfw), ("safe", Ns, False, xfs)):
        xs = x0 if kind == "whole" else st["x0_safe"]
        fac = c(w["factors_" + kind], np.float64)
        base = np.zeros(P)
        K.emu_dtbase(P, N, C.c_double(DC), _p(xs), _p(xf), _p(lim), _p(base))
        co = offsets(w["poly_ofs_" + kind], N, len(fac), lim_)
        dt, sig = expand(w["poly_ofs_" + kind], N, fac, lim_, base, co)
        feas, cost, _, _ = solve_multi(S, N, ff, xs, xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind], co, dt, sig,
                                       max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        wi, wc, wdt, ws, wo = np.zeros(P, np.int32), np.zeros(P), np.zeros(P), np.zeros((P, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_select_multi(P, N, 0, _p(co), _p(dt), _p(sig), _p(feas), _p(cost), _p(wi), _p(wc), _p(wdt), _p(ws), _p(wo))
        _, _, coeffs, _ = solve_multi(S, N, ff, xs, xf, lim, w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind], wo, wdt, ws,
                                      max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        st[kind] = dict(base=base, wi=wi, wc=wc, wdt=wdt, ws=ws, co=co)
        out["feasible_" + kind], out["cost_" + kind], out["coeffs_" + kind] = feas, cost, coeffs
        if kind == "whole":
            x0s, nsamp, ksafe = np.zeros((P, 9)), np.zeros(P, np.int32), np.zeros(P, np.int32)
            K.emu_pair_mid(P, N, C.c_double(DC), C.c_double(w["r_fraction"]), _p(c(coeffs, np.float64)), _p(wdt), _p(wi), _p(x0s), _p(nsamp),
                           _p(ksafe))
            st["x0_safe"], st["nsamp"], st["ksafe"] = x0s, nsamp, ksafe
    res = np.zeros(P, capi.PAIR_RESULT_DTYPE)
    a, b = st["whole"], st["safe"]
    sw, ss = np.zeros((P, Nw), np.uint8), np.zeros((P, Ns), np.uint8)
    A.emu_pair_final_assign(P, len(w["factors_whole"]), len(w["factors_safe"]), Nw, Ns, _p(a["co"]), _p(b["co"]), _p(a["wi"]), _p(b["wi"]),
                            _p(st["nsamp"]), _p(st["ksafe"]), _p(a["wc"]), _p(b["wc"]), _p(a["wdt"]), _p(b["wdt"]), _p(a["base"]), _p(b["base"]),
                            _p(st["x0_safe"]), _p(a["ws"]), _p(b["ws"]), _p(sw), _p(ss), _p(res))
    o = pao.replan_pairs_assign(w, lim_, threads=4, dt_base_whole=res["whole_dt_base"], dt_base_safe=res["safe_dt_base"])
    for k in ("whole", "safe"):
        assert np.array_equal(st[k]["co"], o["cand_ofs_" + k])
        assert np.array_equal(out["feasible_" + k], o["feasible_" + k]), k
        ok = o["feasible_" + k].astype(bool)
        assert (np.abs(out["cost_" + k][ok] - o["cost_" + k][ok]) / np.abs(o["cost_" + k][ok])).max(initial=0) <= 1e-8
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(res[f], o[f]), f
    assert (res["whole_dt_index"] >= 0).any() and (res["safe_dt_index"] >= 0).any()
    for j in range(P):                                  # the winners' assignments are the list entries the indices name
        for kind, sg in (("whole", sw), ("safe", ss)):
            si = res[kind + "_sigma_index"][j]
            lst = pao.assign_list(w["N_" + kind], int(np.diff(w["poly_ofs_" + kind])[j]), lim_)
            assert np.array_equal(sg[j], lst[si] if si >= 0 else np.zeros(w["N_" + kind], np.uint8))
    ok = res["whole_dt_index"] >= 0
    assert np.abs(res["R"][ok] - o["R"][ok]).max() <= 1e-8
