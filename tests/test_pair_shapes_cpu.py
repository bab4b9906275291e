"""The chained replan with per-corridor lists (_assign) and windows (_window) at unequal N_whole and N_safe, without a GPU:
every kernel of the _dev submission (faster_b200/csrc/fq_pair.cuh and the solve kernel, under the block emulation of
tests/cpp/simt_emu/) in submission order, each launched with its sweep's N, against the CPU chain.  The harness
(tests/cpp/kernel_emu.cpp) instantiates the specialised solve kernel at some (N, mode) only: the pairs are the nearest it
has to (4, 16) and (16, 4) -- a short whole sweep before a long safe one and the reverse -- and (6, 10).  N < 4 and the
exact pairs are checked on the GPU (tests/test_pair_shapes_gpu.py), as are the refusals of N out of range, which need a
context."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi

import pair_assign_oracle as pao
import pair_shape_cases as psc
import pair_window_oracle as pwo

PAIRS = [(5, 16), (15, 4), (6, 10)]
FACTORS = psc.FACTORS[1:3]                           # two factors: most corridors win at the second (tests/pair_shape_cases.py)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def emulated_chain(w, all_limit, windows=None, inc=psc.INC, gamma=(2.0, 3.0, 0.5, 0.25)):
    """_assign_dev's (windows None) or _window_dev's kernels on the CPU -> (results, per-sweep state, flags / costs,
    window outputs or None)."""
    import test_pair_assign_cpu as tac
    import test_pair_window_cpu as twc
    from test_kernel_emu_cpu import _emu, _pair_lib, solve_multi
    P, DC = w["n_prob"], w["DC"]
    K, S, A, W = _pair_lib(), _emu(), tac._lib(), twc._lib()
    c = lambda a, t: np.ascontiguousarray(a, t)
    x0, lim = c(w["x0"], np.float64), c(w["lim"], np.float64)
    st, out = {}, {}
    for kind, N, ff, ik in (("whole", w["N_whole"], True, inc[0]), ("safe", w["N_safe"], False, inc[1])):
        xs = x0 if kind == "whole" else st["x0_safe"]
        xf, po = c(w["xf_" + kind], np.float64), c(w["poly_ofs_" + kind], np.int32)
        base = np.zeros(P)
        K.emu_dtbase(P, N, C.c_double(DC), _p(xs), _p(xf), _p(lim), _p(base))
        if windows is None:
            fac = c(w["factors_" + kind], np.float64)
            co = tac.offsets(po, N, len(fac), all_limit)
            dt, sig = tac.expand(po, N, fac, all_limit, base, co)
            rows, nf, mf = None, None, len(fac)
        else:
            mf = 8
            rows, nf = np.zeros((P, mf)), np.zeros(P, np.int32)
            W.emu_window_factors(P, mf, _p(c(windows["init_" + kind], np.float64)), _p(c(windows["final_" + kind], np.float64)), ik,
                                 _p(rows), _p(nf))
            co = twc.offsets(po, N, nf, mf, 1 << 20, all_limit)
            dt, sig = np.full(int(co[-1]), np.nan), np.zeros((int(co[-1]), N), np.uint8)
            W.emu_expand_window(P, N, mf, all_limit, _p(rows), _p(nf), _p(base), _p(po), _p(co), _p(dt), _p(sig))
        feas, cost, _, _ = solve_multi(S, N, ff, xs, xf, lim, po, w["face_ofs_" + kind], w["Ab_" + kind], co, dt, sig,
                                       max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        wi, wc, wdt, ws, wo = np.zeros(P, np.int32), np.zeros(P), np.zeros(P), np.zeros((P, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_select_multi(P, N, 0, _p(co), _p(dt), _p(sig), _p(feas), _p(cost), _p(wi), _p(wc), _p(wdt), _p(ws), _p(wo))
        _, _, coeffs, _ = solve_multi(S, N, ff, xs, xf, lim, po, w["face_ofs_" + kind], w["Ab_" + kind], wo, wdt, ws,
                                      max_faces=w["max_faces_" + kind], max_poly_faces=w["max_poly_faces_" + kind])
        st[kind] = dict(base=base, wi=wi, wc=wc, wdt=wdt, ws=ws, co=co, rows=rows, nf=nf, mf=mf)
        out["feasible_" + kind], out["cost_" + kind], out["coeffs_" + kind] = feas, cost, coeffs
        if kind == "whole":
            x0s, nsamp, ksafe = np.zeros((P, 9)), np.zeros(P, np.int32), np.zeros(P, np.int32)
            K.emu_pair_mid(P, N, C.c_double(DC), C.c_double(w["r_fraction"]), _p(c(coeffs, np.float64)), _p(wdt), _p(wi), _p(x0s),
                           _p(nsamp), _p(ksafe))
            st["x0_safe"], st["nsamp"], st["ksafe"] = x0s, nsamp, ksafe
    a, b = st["whole"], st["safe"]
    res = np.zeros(P, capi.PAIR_RESULT_DTYPE)
    tail = (_p(st["nsamp"]), _p(st["ksafe"]), _p(a["wc"]), _p(b["wc"]), _p(a["wdt"]), _p(b["wdt"]), _p(a["base"]), _p(b["base"]),
            _p(st["x0_safe"]), _p(a["ws"]), _p(b["ws"]))
    wout = None
    if windows is None:
        out["sigma_whole"], out["sigma_safe"] = np.zeros((P, w["N_whole"]), np.uint8), np.zeros((P, w["N_safe"]), np.uint8)
        A.emu_pair_final_assign(P, len(w["factors_whole"]), len(w["factors_safe"]), w["N_whole"], w["N_safe"], _p(a["co"]), _p(b["co"]),
                                _p(a["wi"]), _p(b["wi"]), *tail, _p(out["sigma_whole"]), _p(out["sigma_safe"]), _p(res))
    else:
        W.emu_pair_final_window(P, w["N_whole"], w["N_safe"], _p(a["co"]), _p(b["co"]), _p(a["nf"]), _p(b["nf"]), _p(a["wi"]), _p(b["wi"]),
                                *tail, _p(res))
        win = np.concatenate([c(windows[k], np.float64) for k in pwo.WINDOW_KEYS])
        factor, trials = np.zeros(2 * P), np.zeros(2 * P, np.int32)
        W.emu_pair_window(P, a["mf"], b["mf"], _p(res), _p(a["co"]), _p(b["co"]), _p(a["nf"]), _p(b["nf"]), _p(a["rows"]), _p(b["rows"]),
                          _p(win), _p(c(gamma, np.float64)), _p(factor), _p(trials), _p(win))
        wout = dict(factor_whole=factor[:P], factor_safe=factor[P:], trials_whole=trials[:P], trials_safe=trials[P:])
        wout.update({"next_" + k: win[i * P:(i + 1) * P] for i, k in enumerate(pwo.WINDOW_KEYS)})
    return res, st, out, wout


def _compare(res, st, out, o, w):
    for kind in ("whole", "safe"):
        assert np.array_equal(st[kind]["co"], o["cand_ofs_" + kind]), kind
        assert np.array_equal(out["feasible_" + kind], o["feasible_" + kind]), kind
        ok = o["feasible_" + kind].astype(bool)
        assert (np.abs(out["cost_" + kind][ok] - o["cost_" + kind][ok]) / np.abs(o["cost_" + kind][ok])).max(initial=0) <= 1e-8, kind
        assert out["coeffs_" + kind].shape == (w["n_prob"], w["N_" + kind], 12)
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(res[f], o[f]), f
    ok = res["whole_dt_index"] >= 0
    assert ok.any() and (res["safe_dt_index"] >= 0).any()
    assert np.array_equal(res["whole_dt"][ok], o["whole_dt"][ok])
    assert np.abs(res["R"][ok] - o["R"][ok]).max() <= 1e-8
    assert np.abs(out["coeffs_whole"][ok] - o["coeffs_whole"][ok]).max() < 1e-6


@pytest.mark.parametrize("pair", PAIRS, ids=[psc.pair_id(p) for p in PAIRS])
def test_assign_submission_through_the_emulated_kernels(built_lib, oracle, pair):
    w = psc.mixed_workload(*pair, n=3, factors=FACTORS)
    for all_limit in (0, 4096):
        res, st, out, _ = emulated_chain(w, all_limit)
        o = pao.replan_pairs_assign(w, all_limit, threads=4, dt_base_whole=res["whole_dt_base"], dt_base_safe=res["safe_dt_base"])
        _compare(res, st, out, o, w)
        for j in range(w["n_prob"]):                    # the winners' assignments are the list entries the indices name
            for kind in ("whole", "safe"):
                si = res[kind + "_sigma_index"][j]
                lst = pao.assign_list(w["N_" + kind], int(np.diff(w["poly_ofs_" + kind])[j]), all_limit)
                assert np.array_equal(out["sigma_" + kind][j], lst[si] if si >= 0 else np.zeros(w["N_" + kind], np.uint8)), (j, kind)


@pytest.mark.parametrize("pair", PAIRS, ids=[psc.pair_id(p) for p in PAIRS])
def test_window_submission_through_the_emulated_kernels(built_lib, oracle, pair):
    w = psc.mixed_workload(*pair, n=3, factors=FACTORS)
    windows = dict(init_whole=np.array([1.5, 1.0, 2.0]), final_whole=np.array([2.0, 2.0, 3.0]),
                   init_safe=np.array([1.0, 1.5, 2.0]), final_safe=np.array([2.0, 2.5, 2.0]))
    gamma = (2.0, 3.0, 0.5, 0.25)
    res, st, out, wout = emulated_chain(w, 0, windows, gamma=gamma)
    o = pwo.replan_pairs_window(w, windows, 0, inc=psc.INC, gamma=gamma, threads=4, dt_base_whole=res["whole_dt_base"],
                                dt_base_safe=res["safe_dt_base"])
    _compare(res, st, out, o, w)
    for k, v in wout.items():
        assert v.tobytes() == np.asarray(o[k], v.dtype).tobytes(), k
