"""Chained replan with a per-corridor time-allocation window (fq_replan_pairs_window*): uniform windows unchanged from the
shared factor list, mixed windows equal to one corridor at a time, the union-window mismatch, consecutive replans carried on
the device against a host loop over the CPU chain, the device-pointer hints and the refusals, group contexts, and
fq_gen_new_traj over each corridor's own factors."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_assign_oracle as pao
import pair_window_oracle as pwo

pytestmark = pytest.mark.gpu
capi_E_ARG = -1                                      # FQ_E_ARG


def mixed_workload(n, N, seed0, zero_whole=(0,)):
    """n replans from corridor.make_forest_pair_mixed (polytope counts as Faster::replan trims them); the whole corridors
    listed in zero_whole lose their polytopes.  factors_* / sigmas_* are empty: the window entries take neither."""
    pairs = [cr.make_forest_pair_mixed(seed0 + j, N=N) for j in range(n)]
    for j in zero_whole:
        pairs[j][0]["polys"], pairs[j][0]["P"] = [], 0
    none = np.zeros((0, N), np.uint8)
    return capi.make_pair_workload([p[0] for p in pairs], [p[1] for p in pairs], np.zeros(0), none, np.zeros(0), none, DC=0.01,
                                   r_fraction=0.6)


def uniform(n, fi=1.0, ff=10.0):
    return {k: np.full(n, fi if k.startswith("init") else ff) for k in pwo.WINDOW_KEYS}


def mixed_windows(n, seed):
    """Different starts and ends per corridor; corridor 1's whole window is empty (final < init)."""
    rng = np.random.default_rng(seed)
    iw = rng.choice([1.0, 1.5, 2.0, 3.0, 4.25], n)
    is_ = rng.choice([1.0, 1.3, 2.0, 2.7], n)
    win = dict(init_whole=iw, final_whole=iw + rng.integers(2, 7, n), init_safe=is_, final_safe=is_ + rng.choice([0.5, 1.0, 1.5], n))
    win["final_whole"][1] = win["init_whole"][1] - 0.5
    return win


def one_corridor(w, j, all_limit, Fw, Fs):
    w1 = pao.with_own_lists(pao.corridor(w, j), all_limit)
    w1["factors_whole"], w1["factors_safe"] = np.ascontiguousarray(Fw), np.ascontiguousarray(Fs)
    return w1


def test_uniform_windows_equal_the_shared_factors(solver):
    """[1, 10] with inc 1 everywhere: bit for bit fq_replan_pairs_assign with factors 1..10."""
    import bench
    w = bench.load_cfg4(0, 8)
    w["factors_whole"] = w["factors_safe"] = np.arange(1.0, 11.0)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    got = solver.replan_pairs_window(w, uniform(8), all_limit=0, inc=1.0, gamma=20.0)
    assert got["results"].tobytes() == ref["results"].tobytes()
    for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe", "cand_ofs_whole",
              "cand_ofs_safe", "sigma_whole", "sigma_safe"):
        assert got[k].tobytes() == ref[k].tobytes(), k
    r = got["results"]
    assert (r["whole_dt_index"] >= 0).all()
    assert np.array_equal(got["factor_whole"], r["whole_dt_index"] + 1.0) and np.array_equal(got["trials_whole"], r["whole_dt_index"] + 1)


@pytest.mark.parametrize("N,all_limit", [(10, 0), (6, 4096)])
@pytest.mark.parametrize("early_exit", [0, 1])
def test_mixed_windows_equal_one_corridor_at_a_time(built_lib, N, all_limit, early_exit):
    w = mixed_workload(10, N, 9100 + N)
    win = mixed_windows(10, N)
    s = capi.Solver(0)
    s.set_option("sweep_early_exit", early_exit)
    inc = (1.0, 0.1)
    got = s.replan_pairs_window(w, win, all_limit=all_limit, inc=inc, gamma=(2.0, 3.0, 0.5, 0.25))
    r = got["results"]
    assert (r["whole_dt_index"] >= 0).sum() >= 5 and (r["safe_dt_index"] >= 0).any()
    for j in range(w["n_prob"]):
        Fw, Fs = pwo.factors(win["init_whole"][j], win["final_whole"][j], 1.0), pwo.factors(win["init_safe"][j], win["final_safe"][j], 0.1)
        assert np.array_equal(capi.window_factors(win["init_safe"][j], win["final_safe"][j], 0.1), Fs)
        for kind, F in (("whole", Fw), ("safe", Fs)):
            co = got["cand_ofs_" + kind]
            assert co[j + 1] - co[j] == len(F) * capi.assign_count(w["N_" + kind], int(np.diff(w["poly_ofs_" + kind])[j]), all_limit)
        if len(Fw) == 0:                                 # the empty window: no candidate, no winner, the window stays
            assert r["whole_dt_index"][j] == -1 and r["safe_dt_index"][j] == -1
            assert got["trials_whole"][j] == 0 and got["trials_safe"][j] == 0 and np.isnan(got["factor_whole"][j])
            assert got["next_init_whole"][j] == win["init_whole"][j] and got["next_final_whole"][j] == win["final_whole"][j]
            continue
        one = s.replan_pairs_assign(one_corridor(w, j, all_limit, Fw, Fs), all_limit=all_limit)
        assert r[j:j + 1].tobytes() == one["results"].tobytes(), j
        for kind, F in (("whole", Fw), ("safe", Fs)):
            co = got["cand_ofs_" + kind]
            assert np.array_equal(got["coeffs_" + kind][j], one["coeffs_" + kind][0])
            assert np.array_equal(got["sigma_" + kind][j], one["sigma_" + kind][0])
            if not early_exit:
                assert got["feasible_" + kind][co[j]:co[j + 1]].tobytes() == one["feasible_" + kind].tobytes()
                assert got["cost_" + kind][co[j]:co[j + 1]].tobytes() == one["cost_" + kind].tobytes()
            d = r[kind + "_dt_index"][j]
            f = got["factor_" + kind][j]
            assert (d < 0 and np.isnan(f)) or f.tobytes() == F[d].tobytes()
        assert got["trials_whole"][j] == (r["whole_dt_index"][j] + 1 if r["whole_dt_index"][j] >= 0 else len(Fw))
    want = pwo.window_outputs(r, win, [pwo.factors(a, b, 1.0) for a, b in zip(win["init_whole"], win["final_whole"])],
                              [pwo.factors(a, b, 0.1) for a, b in zip(win["init_safe"], win["final_safe"])], (2.0, 3.0, 0.5, 0.25))
    for k, v in want.items():
        assert np.array_equal(got[k], v, equal_nan=k.startswith("factor")), k
    s.close()


def test_union_window_picks_a_different_winner(solver, oracle):
    """A corridor whose first feasible factor lies below its own window start: the union of the windows (the only shared
    list that covers every corridor) hands it that smaller factor, its own window does not; its own winner is the CPU
    chain's over its own window."""
    w = mixed_workload(4, 10, 9300, zero_whole=())
    first = solver.replan_pairs_window(w, uniform(4), all_limit=0)["results"]
    j = int(np.flatnonzero(first["whole_dt_index"] >= 0)[0])
    f0 = float(first["whole_dt_index"][j] + 1)                        # its first feasible factor on [1, 10]
    win = uniform(4, 1.0, 6.0)
    win["init_whole"][j], win["final_whole"][j] = f0 + 1.0, f0 + 6.0
    own = solver.replan_pairs_window(w, win, all_limit=0)
    union = dict(w, factors_whole=pwo.factors(1.0, f0 + 6.0, 1.0), factors_safe=pwo.factors(1.0, 6.0, 1.0))
    shared = solver.replan_pairs_assign(union, all_limit=0)
    assert shared["results"]["whole_dt_index"][j] + 1 == f0                      # the union returns the factor below the window
    assert own["factor_whole"][j] >= f0 + 1.0 or np.isnan(own["factor_whole"][j])
    r = own["results"]
    o = pwo.replan_pairs_window(w, win, 0, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    assert np.array_equal(r["whole_dt_index"], o["whole_dt_index"]) and np.array_equal(r["whole_sigma_index"], o["whole_sigma_index"])
    assert np.array_equal(r["safe_dt_index"], o["safe_dt_index"])
    assert np.array_equal(own["factor_whole"], o["factor_whole"], equal_nan=True)
    ok = o["whole_dt_index"] >= 0
    assert np.allclose(r["whole_cost"][ok], o["whole_cost"][ok], rtol=1e-8)


def _device(w, torch, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith(("sigmas_", "factors_"))}


GUARD = 4096                                         # sentinel tail after every per-candidate output: nothing may be written there


def _dev_call(solver, w, d, win_dev, torch, dev, cap_w, cap_s, max_fac=(41, 41), max_poly=None, inc=1.0, gamma=20.0, next_dev=None):
    """One fq_replan_pairs_window_dev call on one stream; win_dev: device window arrays, next_dev: the next_* arrays (default:
    win_dev itself, i.e. aliased).  -> (host copies of everything, the device outputs)."""
    n = w["n_prob"]
    mp = max_poly or (int(np.diff(w["poly_ofs_whole"]).max()), int(np.diff(w["poly_ofs_safe"]).max()))
    out = dict(feasible_whole=torch.full((cap_w + GUARD,), 0xAB, dtype=torch.uint8, device=dev),
               cost_whole=torch.full((cap_w + GUARD,), -5.0, dtype=torch.float64, device=dev),
               feasible_safe=torch.full((cap_s + GUARD,), 0xAB, dtype=torch.uint8, device=dev),
               cost_safe=torch.full((cap_s + GUARD,), -5.0, dtype=torch.float64, device=dev),
               coeffs_whole=torch.zeros(n * w["N_whole"] * 12, dtype=torch.float64, device=dev),
               coeffs_safe=torch.zeros(n * w["N_safe"] * 12, dtype=torch.float64, device=dev),
               results=torch.zeros(n * 144, dtype=torch.uint8, device=dev))
    lists = dict(cand_ofs_whole=torch.full((n + 1,), -1, dtype=torch.int32, device=dev),
                 cand_ofs_safe=torch.full((n + 1,), -1, dtype=torch.int32, device=dev))
    wout = dict(factor_whole=torch.zeros(n, dtype=torch.float64, device=dev), factor_safe=torch.zeros(n, dtype=torch.float64, device=dev),
                trials_whole=torch.full((n,), -9, dtype=torch.int32, device=dev), trials_safe=torch.full((n,), -9, dtype=torch.int32, device=dev))
    nxt = win_dev if next_dev is None else next_dev
    a = capi.pair_args(w, lambda k: None if k.startswith(("sigmas_", "factors_")) else d[k].data_ptr(), {k: v.data_ptr() for k, v in out.items()})
    a.n_sig_whole = a.n_sig_safe = a.n_fac_whole = a.n_fac_safe = 0
    s = capi.assign_args(0, {k: v.data_ptr() for k, v in lists.items()}, mp[0], mp[1], cap_w, cap_s)
    optr = {k: v.data_ptr() for k, v in wout.items()}
    optr.update({"next_" + k: nxt[k].data_ptr() for k in pwo.WINDOW_KEYS})
    wa = capi.window_args(lambda k: win_dev[k].data_ptr(), optr, inc, gamma, max_fac[0], max_fac[1])
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    solver.replan_pairs_window_dev(a, s, wa, 0, st.cuda_stream)
    st.synchronize()
    h = {k: v.cpu().numpy() for k, v in list(out.items()) + list(lists.items()) + list(wout.items())}
    h.update({"next_" + k: nxt[k].cpu().numpy() for k in pwo.WINDOW_KEYS})
    h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
    return h


def test_consecutive_replans_carry_the_windows_on_the_device(solver, oracle):
    """Four replans of a rotating batch through fq_replan_pairs_window_dev with the window arrays aliased in and out (no
    host access between the steps) against a host loop: the CPU chain on each step's windows, then faster.cpp:582-588 in
    Python.  Corridor 0's whole window is empty, so it never has both winners and keeps its window."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    n, steps, gamma = 6, 4, (2.0, 2.0, 1.0, 1.0)
    pool = mixed_workload(n + steps, 10, 9400, zero_whole=())
    win = uniform(n, 1.0, 6.0)
    win["init_whole"][0], win["final_whole"][0] = 4.0, 3.0
    win_dev = {k: torch.from_numpy(v.copy()).to(dev) for k, v in win.items()}
    host = {k: v.copy() for k, v in win.items()}
    changed = 0
    for step in range(steps):
        w = _subset(pool, list(range(step, step + n)))      # the batch rotates: every slot meets new corridors
        d = _device(w, torch, dev)
        h = _dev_call(solver, w, d, win_dev, torch, dev, 1 << 16, 1 << 17, max_fac=(6, 6), inc=1.0, gamma=gamma)
        r = h["results"]
        o = pwo.replan_pairs_window(w, host, 0, inc=1.0, gamma=gamma, threads=8, dt_base_whole=r["whole_dt_base"],
                                    dt_base_safe=r["safe_dt_base"])
        for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index"):
            assert np.array_equal(r[k], o[k]), (step, k)
        for k in ("factor_whole", "factor_safe", "trials_whole", "trials_safe"):
            assert np.array_equal(h[k], o[k], equal_nan=k.startswith("factor")), (step, k)
        both = (r["whole_dt_index"] >= 0) & (r["safe_dt_index"] >= 0)
        assert not both[0]
        for k in pwo.WINDOW_KEYS:
            assert np.array_equal(h["next_" + k], o["next_" + k]), (step, k)
            assert np.array_equal(h["next_" + k][~both], host[k][~both]), (step, k)
            changed += int((h["next_" + k] != host[k]).sum())
            host[k] = o["next_" + k].copy()
        assert np.array_equal(h["cand_ofs_whole"], o["cand_ofs_whole"]) and np.array_equal(h["cand_ofs_safe"], o["cand_ofs_safe"])
    assert changed > 0


def _subset(w, idx):
    out = dict(w, n_prob=len(idx))
    for k in ("x0", "xf_whole", "xf_safe", "lim"):
        out[k] = np.ascontiguousarray(w[k][idx])
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        npo, nfo, rows = [0], [0], []
        for j in idx:
            for p in range(po[j], po[j + 1]):
                rows.append(Ab[fo[p]:fo[p + 1]])
                nfo.append(nfo[-1] + fo[p + 1] - fo[p])
            npo.append(npo[-1] + po[j + 1] - po[j])
        nfo, npo = np.asarray(nfo, np.int32), np.asarray(npo, np.int32)
        out["poly_ofs_" + kind], out["face_ofs_" + kind] = npo, nfo
        out["Ab_" + kind] = np.ascontiguousarray(np.vstack(rows)) if rows else np.zeros((1, 4))
        out["max_faces_" + kind] = max(int(max(nfo[npo[j + 1]] - nfo[npo[j]] for j in range(len(idx)))), 1)
        out["max_poly_faces_" + kind] = int(np.diff(nfo).max()) if len(nfo) > 1 else 0
    return out


def test_device_hints_empty_the_sweep(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    w = mixed_workload(6, 10, 9500)
    win = mixed_windows(6, 5)
    ref = solver.replan_pairs_window(w, win, all_limit=0, inc=(1.0, 0.1))
    ncw, ncs = int(ref["cand_ofs_whole"][-1]), int(ref["cand_ofs_safe"][-1])
    mfw = max(len(pwo.factors(a, b, 1.0)) for a, b in zip(win["init_whole"], win["final_whole"]))
    mfs = max(len(pwo.factors(a, b, 0.1)) for a, b in zip(win["init_safe"], win["final_safe"]))
    d = _device(w, torch, dev)

    def run(wn, cap_w, cap_s, mf):
        win_dev = {k: torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(dev) for k, v in wn.items()}
        return _dev_call(solver, w, d, win_dev, torch, dev, cap_w, cap_s, max_fac=mf, inc=(1.0, 0.1))

    h = run(win, ncw + 1000, ncs + 1000, (mfw + 3, mfs))        # capacities above the totals and a loose bound are fine
    assert h["results"].tobytes() == ref["results"].tobytes()
    for k in ("cand_ofs_whole", "cand_ofs_safe", "factor_whole", "factor_safe", "trials_whole", "trials_safe"):
        assert h[k].tobytes() == ref[k].tobytes(), k
    for k in pwo.WINDOW_KEYS:
        assert np.array_equal(h["next_" + k], ref["next_" + k]), k
    assert np.array_equal(h["feasible_whole"][:ncw], ref["feasible_whole"]) and (h["feasible_whole"][ncw:] == 0xAB).all()
    bad = {k: v.copy() for k, v in win.items()}
    bad["init_whole"][2] = np.nan
    for wn, cw, cs, mf in ((win, ncw, ncs, (mfw - 1, mfs)), (bad, ncw, ncs, (mfw, mfs)), (win, ncw - 1, ncs, (mfw, mfs))):
        h = run(wn, cw, cs, mf)
        r = h["results"]
        assert (r["whole_dt_index"] == -1).all() and (r["safe_dt_index"] == -1).all() and np.isnan(r["R"]).all()
        assert not h["cand_ofs_whole"].any() and (h["feasible_whole"] == 0xAB).all() and (h["cost_whole"] == -5.0).all()
        assert (h["trials_whole"] == 0).all() and (h["trials_safe"] == 0).all() and np.isnan(h["factor_whole"]).all()
        for k in pwo.WINDOW_KEYS:
            assert np.array_equal(h["next_" + k], wn[k], equal_nan=True), k
    h = run(win, ncw, ncs - 1, (mfw, mfs))                       # only the safe capacity is too small
    assert np.array_equal(h["results"]["whole_dt_index"], ref["results"]["whole_dt_index"])
    assert (h["results"]["safe_dt_index"] == -1).all() and (h["feasible_safe"] == 0xAB).all() and (h["trials_safe"] == 0).all()
    for k in pwo.WINDOW_KEYS:
        assert np.array_equal(h["next_" + k], win[k]), k


def test_refusals(solver):
    w = mixed_workload(3, 10, 9600, zero_whole=())
    L = capi.lib()
    res = np.zeros(3, capi.PAIR_RESULT_DTYPE)
    a = capi.pair_args(w, lambda k: None if k.startswith(("sigmas_", "factors_")) else w[k].ctypes.data, {"results": res.ctypes.data})
    a.n_sig_whole = a.n_sig_safe = a.n_fac_whole = a.n_fac_safe = 0
    s = capi.assign_args(0, {})

    def call(wn, inc=1.0, a=a, s=s, gamma=20.0):
        arrs = {k: np.ascontiguousarray(wn[k], np.float64) for k in pwo.WINDOW_KEYS}
        wa = capi.window_args(lambda k: arrs[k].ctypes.data, {}, inc, gamma)
        return L.fq_replan_pairs_window(solver._h, capi.C.byref(a), capi.C.byref(s) if s is not None else None, capi.C.byref(wa))

    ok = uniform(3)
    assert call(ok) == 0 and (res["whole_dt_index"] >= 0).any()
    for k, v in (("init_whole", np.nan), ("final_safe", np.inf), ("init_safe", 0.0), ("init_whole", -1.0), ("final_whole", 5000.0),
                 ("init_whole", 1e17)):
        bad = {kk: vv.copy() for kk, vv in ok.items()}
        bad[k][1] = v
        if v == 1e17:
            bad["final_whole"][1] = 1e17 + 1e3
        assert call(bad) == capi_E_ARG, (k, v)
    assert call(ok, inc=0.0) == capi_E_ARG and call(ok, inc=(1.0, -0.1)) == capi_E_ARG and call(ok, inc=np.nan) == capi_E_ARG
    assert call(ok, gamma=np.inf) == capi_E_ARG
    fac = np.arange(1.0, 4.0)
    withfac = capi.PairArgs.from_buffer_copy(a)
    withfac.factors_whole, withfac.n_fac_whole = fac.ctypes.data, 3
    assert call(ok, a=withfac) == capi_E_ARG
    assert call(ok, s=None) == capi_E_ARG
    assert call(ok) == 0                                            # the context keeps working
    for bad in ((1.0, np.nan, 1.0), (0.0, 2.0, 1.0), (1.0, 2.0, 0.0), (1.0, 5000.0, 1.0), (1e17, 1e17 + 1e3, 1.0)):
        assert L.fq_pair_window_factors(*bad, None, 0) == capi_E_ARG, bad
    # _dev hints out of range
    d = capi.PairArgs.from_buffer_copy(a)
    arrs = {k: np.ascontiguousarray(ok[k]) for k in pwo.WINDOW_KEYS}
    for mf in ((4097, 10), (10, -1)):
        wa = capi.window_args(lambda k: arrs[k].ctypes.data, {}, 1.0, 20.0, *mf)
        assert L.fq_replan_pairs_window_dev(solver._h, capi.C.byref(d), capi.C.byref(capi.assign_args(0, {}, 3, 4, 10, 10)),
                                            capi.C.byref(wa), None, None) == capi_E_ARG
    assert capi.has_feature("replan_pairs_window")


@pytest.mark.parametrize("n_gpus", [1, 2])
def test_group_context_shards_by_candidates(solver, n_gpus):
    import torch
    if torch.cuda.device_count() < n_gpus:
        pytest.skip("needs %d GPUs" % n_gpus)
    w = mixed_workload(9, 10, 9700)
    win = mixed_windows(9, 9)
    ref = solver.replan_pairs_window(w, win, all_limit=0, inc=(1.0, 0.1))
    both = (ref["cand_ofs_whole"] + ref["cand_ofs_safe"]).astype(np.int32)
    bounds = [capi.shard_range(w["n_prob"], both, r, n_gpus) for r in range(n_gpus)]
    assert bounds[0][0] == 0 and bounds[-1][1] == w["n_prob"]
    if n_gpus > 1:                                       # balanced by candidates, not by corridors
        share = [int(both[hi] - both[lo]) for lo, hi in bounds]
        assert max(share) - min(share) <= int(np.diff(both).max())
    g = capi.Solver(n_gpus=n_gpus, devices=list(range(n_gpus)))
    out = g.replan_pairs_window(w, win, all_limit=0, inc=(1.0, 0.1))
    assert out["results"].tobytes() == ref["results"].tobytes()
    for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe", "cand_ofs_whole",
              "cand_ofs_safe", "sigma_whole", "sigma_safe") + tuple(capi.WINDOW_OUT_KEYS):
        assert out[k].tobytes() == ref[k].tobytes(), k
    out2 = g.replan_pairs_window(w, win, all_limit=0, inc=(1.0, 0.1), deferred=True)
    g.wait()
    assert out2["results"].tobytes() == ref["results"].tobytes() and out2["next_init_whole"].tobytes() == ref["next_init_whole"].tobytes()
    g.close()


def test_whole_winner_equals_gen_new_traj_over_the_own_factors(solver):
    """N = 6, P <= 3, all_limit = 4096: each corridor's whole winner is fq_gen_new_traj's over F_j * dt_base x L_j."""
    w = mixed_workload(8, 6, 9800, zero_whole=())
    win = mixed_windows(8, 11)
    g = solver.replan_pairs_window(w, win, all_limit=4096, inc=(0.3, 1.0))
    r = g["results"]
    solved = 0
    for j in range(w["n_prob"]):
        F = pwo.factors(win["init_whole"][j], win["final_whole"][j], 0.3)
        if len(F) == 0:
            assert r["whole_dt_index"][j] == -1
            continue
        w1 = pao.corridor(w, j)
        P = int(w1["poly_ofs_whole"][1])
        polys = [(w1["Ab_whole"][w1["face_ofs_whole"][p]:w1["face_ofs_whole"][p + 1], :3],
                  w1["Ab_whole"][w1["face_ofs_whole"][p]:w1["face_ofs_whole"][p + 1], 3]) for p in range(P)]
        lst = pao.assign_list(6, P, 4096)
        ref = solver.gen_new_traj(6, w["x0"][j], w["xf_whole"][j], w["lim"][j], polys, F * r["whole_dt_base"][j], lst)
        assert ref["dt_index"] == r["whole_dt_index"][j], j
        if ref["solved"]:
            solved += 1
            assert ref["sigma_index"] == r["whole_sigma_index"][j]
            assert np.isclose(ref["cost"], r["whole_cost"][j], rtol=1e-12, atol=0)
            assert g["factor_whole"][j] == F[ref["dt_index"]]
    assert solved >= 4
