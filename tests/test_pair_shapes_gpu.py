"""The chained replan at every (N_whole, N_safe) it accepts (tests/pair_shape_cases.py), against its CPU restatement: the
shared-list entry (oracle/pair_oracle.py), per-corridor lists (tests/pair_assign_oracle.py), windows
(tests/pair_window_oracle.py), the exact stage (tests/pair_exact_oracle.py) and the decomposing chain; the device-pointer
entries and group contexts at unequal N; the R-sampling kernel's edges bit for bit against the host fillX; and the
refusals of N out of range by every entry, group contexts included."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi

import pair_assign_oracle as pao
import pair_shape_cases as psc
import pair_window_oracle as pwo

pytestmark = pytest.mark.gpu
E_ARG = -1
GUARD = 512                                          # sentinel tail after a device output: nothing may be written there
UNEQUAL = [(4, 16), (16, 4)]


def _ids(pairs):
    return [psc.pair_id(p) for p in pairs]


def check_chain(g, o, w, all_limit=None):
    """The bars of the existing chain tests (tests/test_pair_gpu.py), plus the shapes of every per-corridor output and
    the winners' assignments.  all_limit None: shared lists (w's sigmas_*); otherwise per-corridor lists."""
    r, n, Nw, Ns = g["results"], w["n_prob"], w["N_whole"], w["N_safe"]
    assert np.array_equal(g["feasible_whole"], o["feasible_whole"]), "whole flags differ"
    for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(r[k], o[k]), k
    ok = o["whole_dt_index"] >= 0
    assert ok.any()
    assert np.allclose(r["whole_cost"][ok], o["whole_cost"][ok], rtol=1e-8)
    assert np.array_equal(r["whole_dt"][ok], o["whole_dt"][ok]), "whole dt not bit-equal"
    assert np.array_equal(r["whole_dt_base"], o["whole_dt_base_own"]), "device getDTInitial differs from the host's"
    assert np.abs(r["R"][ok] - o["R"][ok]).max() < 1e-8 and np.isnan(r["R"][~ok]).all()
    assert g["coeffs_whole"].shape == (n, Nw, 12) and g["coeffs_safe"].shape == (n, Ns, 12)
    assert np.abs(g["coeffs_whole"][ok] - o["coeffs_whole"][ok]).max() < 1e-6
    fok = o["feasible_whole"].astype(bool)
    assert np.allclose(g["cost_whole"][fok], o["cost_whole"][fok], rtol=1e-8)
    # the safe sweep starts from the device's R: its base is the host's getDTInitial of that R with N_safe, bit for bit
    for j in np.flatnonzero(ok):
        want = max(capi.dt_initial(r["R"][j], w["xf_safe"][j], w["lim"][j], Ns), 2 * w["DC"])
        assert r["safe_dt_base"][j] == want, j
    assert np.isnan(r["safe_dt_base"][~ok]).all()
    assert np.array_equal(g["feasible_safe"], o["feasible_safe"]), "safe flags differ"
    sok = o["safe_dt_index"] >= 0
    assert np.allclose(r["safe_cost"][sok], o["safe_cost"][sok], rtol=1e-6)
    if sok.any():
        assert np.abs(g["coeffs_safe"][sok] - o["coeffs_safe"][sok]).max() < 1e-5
    if all_limit is None:
        return
    assert g["sigma_whole"].shape == (n, Nw) and g["sigma_safe"].shape == (n, Ns)
    for j in range(n):
        for kind in ("whole", "safe"):
            si = r[kind + "_sigma_index"][j]
            lst = pao.assign_list(w["N_" + kind], int(np.diff(w["poly_ofs_" + kind])[j]), all_limit)
            assert np.array_equal(g["sigma_" + kind][j], lst[si] if si >= 0 else np.zeros(w["N_" + kind], np.uint8)), (j, kind)


@pytest.mark.parametrize("pair", psc.PAIRS, ids=_ids(psc.PAIRS))
def test_shared_lists_match_the_cpu_chain(solver, oracle, pair):
    from oracle import pair_oracle
    w = psc.shared_workload(*pair)
    g = solver.replan_pairs(w)
    r = g["results"]
    o = pair_oracle.replan_pairs(w, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    check_chain(g, o, w)


@pytest.mark.parametrize("pair", psc.PAIRS, ids=_ids(psc.PAIRS))
def test_assign_matches_the_cpu_chain(solver, oracle, pair):
    w = psc.mixed_workload(*pair)
    for all_limit in (0, 4096):
        g = solver.replan_pairs_assign(w, all_limit=all_limit)
        r = g["results"]
        o = pao.replan_pairs_assign(w, all_limit, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
        assert np.array_equal(g["cand_ofs_whole"], o["cand_ofs_whole"]) and np.array_equal(g["cand_ofs_safe"], o["cand_ofs_safe"])
        check_chain(g, o, w, all_limit)


@pytest.mark.parametrize("pair", psc.PAIRS, ids=_ids(psc.PAIRS))
def test_window_matches_the_cpu_chain(solver, oracle, pair):
    w = psc.mixed_workload(*pair)
    win = psc.mixed_windows(w["n_prob"], 17 * pair[0] + pair[1])
    gam = (2.0, 3.0, 0.5, 0.25)
    g = solver.replan_pairs_window(w, win, all_limit=0, inc=psc.INC, gamma=gam)
    r = g["results"]
    o = pwo.replan_pairs_window(w, win, 0, inc=psc.INC, gamma=gam, threads=8, dt_base_whole=r["whole_dt_base"],
                                dt_base_safe=r["safe_dt_base"])
    assert np.array_equal(g["cand_ofs_whole"], o["cand_ofs_whole"]) and np.array_equal(g["cand_ofs_safe"], o["cand_ofs_safe"])
    check_chain(g, o, w, 0)
    for k in ("factor_whole", "factor_safe", "trials_whole", "trials_safe") + tuple("next_" + k for k in pwo.WINDOW_KEYS):
        assert np.array_equal(g[k], o[k], equal_nan=k.startswith("factor")), k


@pytest.mark.parametrize("pair", psc.PAIRS, ids=_ids(psc.PAIRS))
def test_exact_matches_the_restatement(solver, oracle, pair):
    """Every corridor here keeps P <= N - 2, so below N = 4 a corridor has at most one polytope: its list is complete and no
    tree is needed (exact = 1, no nodes).  From N = 4 on, the trees run to the end (exact = 1)."""
    from test_pair_exact_gpu import compare_with_restatement
    w = psc.mixed_workload(*pair)
    ex = solver.replan_pairs_exact(w, all_limit=0)
    n = w["n_prob"]
    F = [w["factors_whole"]] * n
    compare_with_restatement(w, ex, F, [w["factors_safe"]] * n, oracle)
    assert (ex["exact_whole"] == 1).all() and (ex["exact_safe"] == 1).all()
    assert ex["sigma_whole"].shape == (n, pair[0]) and ex["sigma_safe"].shape == (n, pair[1])
    assert ex["coeffs_whole"].shape == (n, pair[0], 12) and ex["coeffs_safe"].shape == (n, pair[1], 12)
    for kind, N in zip(("whole", "safe"), pair):
        P = np.diff(w["poly_ofs_" + kind])
        tree = P >= 2
        if N < 4:
            assert not tree.any() and (ex["nodes_" + kind] == 0).all()
        if tree.any() and kind == "whole":
            assert (ex["nodes_whole"][tree] > 0).any()
        assert (ex["nodes_" + kind][~tree] == 0).all()
    # where no tree ran, a corridor is _assign's to the byte
    ref = solver.replan_pairs_assign(w, all_limit=0)
    for j in range(n):
        if ex["nodes_whole"][j] == 0 and ex["nodes_safe"][j] == 0:
            assert ex["results"][j:j + 1].tobytes() == ref["results"][j:j + 1].tobytes(), j
            for k in ("sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe"):
                assert ex[k][j].tobytes() == ref[k][j].tobytes(), (j, k)


@pytest.mark.parametrize("pair", [(3, 2), (3, 3), (3, 16), (16, 2), (16, 3)], ids=_ids([(3, 2), (3, 3), (3, 16), (16, 2), (16, 3)]))
def test_exact_below_four_keeps_the_list_winner(solver, pair):
    """Two polytopes at N < 4 (more than faster_ros.cpp allows, but accepted): the non-decreasing list is incomplete and the
    level kernel has no instance for N, so that sweep reports exact = 0 and keeps the list winner.  With N_whole = 3 the
    whole record is _assign's byte for byte, and so is the safe one wherever the whole winner stayed."""
    Nw, Ns = pair
    whole = [psc._corridor(62000 + j, 2, Nw, True) for j in range(4)]
    safe = [psc._corridor(62000 + j, 2, Ns, False) for j in range(4)]
    w = capi.make_pair_workload(whole, safe, psc.FACTORS, np.zeros((0, Nw), np.uint8), psc.FACTORS, np.zeros((0, Ns), np.uint8), DC=0.01)
    ex = solver.replan_pairs_exact(w, all_limit=0)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    assert (ex["results"]["whole_dt_index"] >= 0).any()
    for kind, N in zip(("whole", "safe"), pair):
        if N < 4:
            ran = ex["cand_ofs_" + kind][1:] > ex["cand_ofs_" + kind][:-1]
            assert (ex["exact_" + kind][ran] == 0).all() and (ex["nodes_" + kind] == 0).all(), kind
        else:
            assert (ex["exact_" + kind] == 1).all()
    for j in range(4):
        r, q = ex["results"][j], ref["results"][j]
        if Nw == 3 or (r["whole_dt_index"] == q["whole_dt_index"] and ex["sigma_whole"][j].tobytes() == ref["sigma_whole"][j].tobytes()
                       and r["whole_cost"] == q["whole_cost"]):
            assert ex["results"][j:j + 1].tobytes() == ref["results"][j:j + 1].tobytes(), j
            for k in ("sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe"):
                assert ex[k][j].tobytes() == ref[k][j].tobytes(), (j, k)


@pytest.mark.parametrize("pair", [(6, 10), (10, 6)], ids=_ids([(6, 10), (10, 6)]))
def test_decomp_with_unequal_n(solver, pair):
    """The decomposing chain with N_whole != N_safe against _assign on the corridors the host builds from the same paths
    (the safe path from the device's R), as tests/test_pair_decomp_gpu.py does at N = 10."""
    from faster_b200 import corridor as cr
    from test_pair_decomp_gpu import compare_records, host_built
    Nw, Ns = pair
    def run(ps):
        w = capi.make_decomp_workload(ps)
        w["N_whole"], w["N_safe"] = Nw, Ns
        w["factors_whole"], w["factors_safe"] = psc.FACTORS.copy(), psc.FACTORS.copy()
        return w, solver.replan_pairs_decomp(w)
    ps = [cr.forest_pair_paths(20500 + k, N=Nw) for k in range(12)]
    w, out = run(ps)
    # a corridor without a whole winner has no R, so its safe corridor is not decomposed: the host cannot build that one
    assert not out["status_whole"].any()
    skipped = out["status_safe"] != 0
    assert (out["status_safe"][skipped] == capi.DECOMP_STATUS["not_run"]).all()
    assert (out["results"]["whole_dt_index"][skipped] == -1).all() and skipped.sum() <= 4
    ps = [p for p, s in zip(ps, skipped) if not s]
    w, out = run(ps)
    n = len(ps)
    assert not out["status_safe"].any()
    assert out["sigma_whole"].shape == (n, Nw) and out["sigma_safe"].shape == (n, Ns) and out["coeffs_safe"].shape == (n, Ns, 12)
    whole, safe, same = host_built(ps, out, w)
    for d in whole:
        d["N"] = Nw
    for d in safe:
        d["N"] = Ns
    hw = capi.make_pair_workload(whole, safe, psc.FACTORS, np.zeros((0, Nw), np.uint8), psc.FACTORS, np.zeros((0, Ns), np.uint8), DC=w["DC"],
                                 r_fraction=w["r_fraction"])
    ref = solver.replan_pairs_assign(hw, want_candidates=False)
    compare_records(out, ref, same)
    assert (out["results"]["safe_dt_index"] >= 0).sum() >= 4


# ---------------------------------------------------------------------------------------------------------------------
# device-pointer entries and group contexts at unequal N
# ---------------------------------------------------------------------------------------------------------------------
def _guarded(torch, dev, count, dtype, fill):
    return torch.full((count + GUARD,), fill, dtype=dtype, device=dev)


def _host(t, count, fill):
    """Device output -> host copy of its first `count` elements; the guard tail must still hold `fill`."""
    h = t.cpu().numpy()
    assert (h[count:] == fill).all(), "written past the end"
    return h[:count]


@pytest.mark.parametrize("family", ["pairs", "assign", "window", "exact"])
@pytest.mark.parametrize("pair", UNEQUAL, ids=_ids(UNEQUAL))
def test_device_entries_equal_the_host_entries(solver, pair, family):
    """One _dev call per entry family on exactly sized device outputs with a sentinel tail: the records, the winners'
    assignments (n x N) and coefficients (n x N x 12) byte-identical to the host entry's."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    Nw, Ns = pair
    w = psc.shared_workload(Nw, Ns) if family == "pairs" else psc.mixed_workload(Nw, Ns)
    n = w["n_prob"]
    win = psc.mixed_windows(n, 3) if family in ("window", "exact") else None
    if family == "pairs":
        ref = solver.replan_pairs(w)
    elif family == "assign":
        ref = solver.replan_pairs_assign(w)
    elif family == "window":
        ref = solver.replan_pairs_window(w, win, inc=psc.INC)
    else:
        ref = solver.replan_pairs_exact(w, windows=win, inc=psc.INC)
    skip = ("sigmas_", "factors_") if win is not None else (("sigmas_",) if family != "pairs" else ())
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith(skip)}
    win_dev = {k: torch.from_numpy(np.ascontiguousarray(win[k], np.float64)).to(dev) for k in pwo.WINDOW_KEYS} if win is not None else None
    out = dict(results=torch.zeros(n * 144 + GUARD, dtype=torch.uint8, device=dev),
               coeffs_whole=_guarded(torch, dev, n * Nw * 12, torch.float64, -3.0), coeffs_safe=_guarded(torch, dev, n * Ns * 12, torch.float64, -3.0))
    lists = dict(sigma_whole=_guarded(torch, dev, n * Nw, torch.uint8, 0xCD), sigma_safe=_guarded(torch, dev, n * Ns, torch.uint8, 0xCD))
    exo = dict(exact_whole=_guarded(torch, dev, n, torch.int32, -9), exact_safe=_guarded(torch, dev, n, torch.int32, -9))
    a = capi.pair_args(w, lambda k: None if k.startswith(skip) else d[k].data_ptr(), {k: v.data_ptr() for k, v in out.items()})
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    if family == "pairs":
        solver.replan_pairs_dev(a, 0, st.cuda_stream)
    else:
        a.n_sig_whole = a.n_sig_safe = 0
        mp = (int(np.diff(w["poly_ofs_whole"]).max()), int(np.diff(w["poly_ofs_safe"]).max()))
        cap = (int(ref["cand_ofs_whole"][-1]), int(ref["cand_ofs_safe"][-1]))
        s = capi.assign_args(0, {k: v.data_ptr() for k, v in lists.items()}, mp[0], mp[1], *cap)
        wa = None
        if win is not None:
            a.n_fac_whole = a.n_fac_safe = 0
            mf = [max(len(pwo.factors(x, y, inc)) for x, y in zip(win["init_" + k], win["final_" + k])) for k, inc in zip(("whole", "safe"), psc.INC)]
            wa = capi.window_args(lambda k: win_dev[k].data_ptr(), {}, psc.INC, 20.0, *mf)
        if family == "assign":
            solver.replan_pairs_assign_dev(a, s, 0, st.cuda_stream)
        elif family == "window":
            solver.replan_pairs_window_dev(a, s, wa, 0, st.cuda_stream)
        else:
            solver.replan_pairs_exact_dev(a, s, wa, capi.exact_args({k: v.data_ptr() for k, v in exo.items()}), 0, st.cuda_stream)
    st.synchronize()
    res = np.frombuffer(_host(out["results"], n * 144, 0).tobytes(), capi.PAIR_RESULT_DTYPE)
    assert res.tobytes() == ref["results"].tobytes()
    assert (res["whole_dt_index"] >= 0).any()
    assert _host(out["coeffs_whole"], n * Nw * 12, -3.0).tobytes() == ref["coeffs_whole"].tobytes()
    assert _host(out["coeffs_safe"], n * Ns * 12, -3.0).tobytes() == ref["coeffs_safe"].tobytes()
    if family != "pairs":
        assert _host(lists["sigma_whole"], n * Nw, 0xCD).tobytes() == ref["sigma_whole"].tobytes()
        assert _host(lists["sigma_safe"], n * Ns, 0xCD).tobytes() == ref["sigma_safe"].tobytes()
    if family == "exact":
        assert _host(exo["exact_whole"], n, -9).tobytes() == ref["exact_whole"].tobytes()
        assert _host(exo["exact_safe"], n, -9).tobytes() == ref["exact_safe"].tobytes()


@pytest.mark.parametrize("n_gpus", [1, 2])
@pytest.mark.parametrize("pair", UNEQUAL, ids=_ids(UNEQUAL))
def test_group_contexts_give_the_same_records(solver, pair, n_gpus):
    import torch
    if torch.cuda.device_count() < n_gpus:
        pytest.skip("needs %d GPUs" % n_gpus)
    Nw, Ns = pair
    shared, mixed = psc.shared_workload(Nw, Ns, n=5), psc.mixed_workload(Nw, Ns, n=7)
    win = psc.mixed_windows(7, 5)
    g = capi.Solver(n_gpus=n_gpus, devices=list(range(n_gpus)))
    try:
        for got, ref, keys in ((g.replan_pairs(shared), solver.replan_pairs(shared), ()),
                               (g.replan_pairs_assign(mixed), solver.replan_pairs_assign(mixed), ("sigma_whole", "sigma_safe", "cand_ofs_whole", "cand_ofs_safe")),
                               (g.replan_pairs_window(mixed, win, inc=psc.INC), solver.replan_pairs_window(mixed, win, inc=psc.INC),
                                ("sigma_whole", "sigma_safe") + tuple(capi.WINDOW_OUT_KEYS))):
            assert got["results"].tobytes() == ref["results"].tobytes()
            for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe") + keys:
                assert got[k].tobytes() == ref[k].tobytes(), k
    finally:
        g.close()


# ---------------------------------------------------------------------------------------------------------------------
# R between the sweeps: fq_pair_mid_kernel against the host fillX, at its edges
# ---------------------------------------------------------------------------------------------------------------------
R_PAIRS = [(3, 2), (4, 16), (10, 6), (16, 3)]
R_FRACTIONS = (0.0, 0.5, 1 - 1e-12, 1.0)
R_FACTORS = np.array([0.05, 0.1, 0.3, 0.6, 1.0, 2.0, 5.0, 20.0])      # below 1: dt < 2 DC; up to 20: long runs


def _rest_states(n, seed):
    """States without polytopes: a third rest-to-rest with no displacement (feasible at every dt, so the smallest factor wins
    and N dt / DC can fall below 2), a third with millimetre steps, a third with metres and moving starts."""
    rng = np.random.default_rng(seed)
    x0, xf = np.zeros((n, 9)), np.zeros((n, 9))
    x0[:, :3] = rng.uniform(-5, 5, (n, 3))
    xf[:, :3] = x0[:, :3]
    m = n // 3
    xf[m:2 * m, :3] += rng.uniform(-1e-3, 1e-3, (m, 3))
    x0[2 * m:, 3:6] = rng.uniform(-2, 2, (n - 2 * m, 3))
    x0[2 * m:, 6:9] = rng.uniform(-1, 1, (n - 2 * m, 3))
    xf[2 * m:, :3] += rng.uniform(-4, 4, (n - 2 * m, 3))
    return x0, xf


def test_r_sampling_edges_match_the_host_fill_x(solver):
    n = 240
    floor2 = last = lag = 0
    for Nw, Ns in R_PAIRS:
        for DC in (1e-3, 0.01, 0.2):
            x0, xfw = _rest_states(n, 31 * Nw + int(1000 * DC))
            _, xfs = _rest_states(n, 7 * Ns + int(1000 * DC))
            lim = np.tile(np.array([5.0, 5.0, 8.0]), (n, 1))
            zero = np.zeros(n + 1, np.int32)
            for rf in R_FRACTIONS:
                w = dict(n_prob=n, N_whole=Nw, N_safe=Ns, DC=DC, r_fraction=rf, x0=x0, xf_whole=xfw, xf_safe=xfs, lim=lim,
                         poly_ofs_whole=zero, face_ofs_whole=np.zeros(1, np.int32), Ab_whole=np.zeros((1, 4)), poly_ofs_safe=zero,
                         face_ofs_safe=np.zeros(1, np.int32), Ab_safe=np.zeros((1, 4)), factors_whole=R_FACTORS,
                         sigmas_whole=np.zeros((1, Nw), np.uint8), factors_safe=R_FACTORS, sigmas_safe=np.zeros((1, Ns), np.uint8),
                         max_faces_whole=1, max_poly_faces_whole=0, max_faces_safe=1, max_poly_faces_safe=0)
                g = solver.replan_pairs(w, want_candidates=False)
                r = g["results"]
                ok = r["whole_dt_index"] >= 0
                assert ok.sum() > n // 2, (Nw, DC)
                assert (r["n_samples_whole"][~ok] == 0).all() and (r["k_safe"][~ok] == -1).all()
                for j in np.flatnonzero(ok):
                    X = capi.fill_x(Nw, g["coeffs_whole"][j], r["whole_dt"][j], DC)
                    k = min(len(X) - 1, int(rf * len(X)))
                    assert r["n_samples_whole"][j] == len(X) and r["k_safe"][j] == k, (Nw, DC, rf, j)
                    assert r["R"][j].tobytes() == X[k, :9].tobytes(), (Nw, DC, rf, j)
                    if k == len(X) - 1:
                        assert not r["R"][j][3:].any()                  # the last sample is at rest
                        last += 1
                    base = max(capi.dt_initial(r["R"][j], xfs[j], lim[j], Ns), 2 * DC)
                    assert r["safe_dt_base"][j] == base, (Nw, DC, rf, j)
                    floor2 += len(X) == 2
                    lag += DC > r["whole_dt"][j]
    # the edges were reached: the n = 2 floor, the last sample, and a sample period above dt (the interval index lags)
    assert floor2 >= 100 and last >= 500 and lag >= 100, (floor2, last, lag)


# ---------------------------------------------------------------------------------------------------------------------
# N out of range: every entry refuses, group contexts before they write anything
# ---------------------------------------------------------------------------------------------------------------------
BAD_N = [(2, 10), (17, 10), (10, 1), (10, 17)]


@pytest.mark.parametrize("bad", BAD_N, ids=_ids(BAD_N))
def test_every_entry_refuses_n_out_of_range(solver, bad):
    L = capi.lib()
    w = psc.mixed_workload(10, 10, n=3)
    win = {k: np.ascontiguousarray(v, np.float64) for k, v in psc.mixed_windows(3, 1).items()}
    res = np.zeros(3, capi.PAIR_RESULT_DTYPE)
    co = {k: np.full(4, -7, np.int32) for k in ("cand_ofs_whole", "cand_ofs_safe")}
    sig_list = np.zeros((1, 17), np.uint8)

    def args(shared=False, window=False):
        a = capi.pair_args(w, lambda k: None if k.startswith("sigmas_") or (window and k.startswith("factors_")) else w[k].ctypes.data,
                           {"results": res.ctypes.data})
        if shared:
            a.sigmas_whole = a.sigmas_safe = sig_list.ctypes.data
            a.n_sig_whole = a.n_sig_safe = 1
        else:
            a.n_sig_whole = a.n_sig_safe = 0
        if window:
            a.n_fac_whole = a.n_fac_safe = 0
        a.N_whole, a.N_safe = bad
        return a

    s = capi.assign_args(0, {k: v.ctypes.data for k, v in co.items()})
    sd = capi.assign_args(0, {}, 3, 4, 1 << 16, 1 << 16)
    wa = capi.window_args(lambda k: win[k].ctypes.data, {}, psc.INC, 20.0, 8, 8)
    ex = capi.exact_args({})
    B = C.byref
    calls = dict(
        pairs=lambda h: L.fq_replan_pairs(h, B(args(True))),
        pairs_async=lambda h: L.fq_replan_pairs_async(h, B(args(True))),
        pairs_dev=lambda h: L.fq_replan_pairs_dev(h, B(args(True)), None, None),
        assign=lambda h: L.fq_replan_pairs_assign(h, B(args()), B(s)),
        assign_async=lambda h: L.fq_replan_pairs_assign_async(h, B(args()), B(s)),
        assign_dev=lambda h: L.fq_replan_pairs_assign_dev(h, B(args()), B(sd), None, None),
        window=lambda h: L.fq_replan_pairs_window(h, B(args(window=True)), B(s), B(wa)),
        window_async=lambda h: L.fq_replan_pairs_window_async(h, B(args(window=True)), B(s), B(wa)),
        window_dev=lambda h: L.fq_replan_pairs_window_dev(h, B(args(window=True)), B(sd), B(wa), None, None),
        exact=lambda h: L.fq_replan_pairs_exact(h, B(args()), B(s), None, B(ex)),
        exact_dev=lambda h: L.fq_replan_pairs_exact_dev(h, B(args()), B(sd), None, B(ex), None, None))
    for name, call in calls.items():
        assert call(solver._h) == E_ARG, name
        assert (co["cand_ofs_whole"] == -7).all() and (co["cand_ofs_safe"] == -7).all(), name
    # the decomposing chain (its own argument set: no faces, no final states)
    from faster_b200 import corridor as cr
    pw = capi.make_decomp_workload([cr.forest_pair_paths(21000 + k) for k in range(3)])
    pw["factors_whole"], pw["factors_safe"] = psc.FACTORS.copy(), psc.FACTORS.copy()
    a = capi.PairArgs()
    a.n_prob, a.DC, a.r_fraction = 3, pw["DC"], pw["r_fraction"]
    a.N_whole, a.N_safe = bad
    for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
        setattr(a, k, pw[k].ctypes.data)
    a.n_fac_whole = a.n_fac_safe = len(psc.FACTORS)
    a.results = res.ctypes.data
    for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
        setattr(a, k, int(pw[k]))
    dc = capi.decomp_args(lambda k: pw[k].ctypes.data, {}, cr.UAV["bbox"], cr.UAV["drone_radius"], cr.UAV["z_ground"], 8000, 8000)
    assert L.fq_replan_pairs_decomp(solver._h, B(a), B(s), None, None, B(dc)) == E_ARG
    assert L.fq_replan_pairs_decomp_dev(solver._h, B(a), B(sd), None, None, B(dc), None, None) == E_ARG
    assert (co["cand_ofs_whole"] == -7).all()
    # group contexts: the sharded entries refuse before they write the caller's offsets
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        for name in ("pairs", "pairs_async", "assign", "assign_async", "window", "window_async", "exact"):
            assert calls[name](g._h) == E_ARG, ("group", name)
            assert (co["cand_ofs_whole"] == -7).all() and (co["cand_ofs_safe"] == -7).all(), ("group", name)
    finally:
        g.close()
    ok = psc.mixed_workload(10, 10, n=3)
    assert (solver.replan_pairs_assign(ok)["results"]["whole_dt_index"] >= 0).any()      # the context still works
