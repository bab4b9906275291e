"""Chained replan with the exact MIQP optimum of every corridor (fq_replan_pairs_exact*): unchanged winners byte-identical
to _assign / _window, the known non-decreasing misses against the CPU restatement, invariance under relabelled polytopes,
complete lists without a tree, isolation of cut and oversized corridors, consecutive device replans with carried windows,
CUDA-graph capture, determinism and the refusals."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import capacity_cases as cc
import pair_exact_oracle as peo
import pair_window_oracle as pwo

pytestmark = pytest.mark.gpu
REL = 1e-7                                            # the suite's cost tolerance against the CPU restatement
FAC = np.arange(1.0, 17.0)


def cfg4(n, start=0):
    import bench
    w = bench.load_cfg4(start, n)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    return w


def same_corridor(a, b, j, kinds=("whole", "safe")):
    """Corridor j's record, winners' assignments and coefficients are byte-identical in the two outputs."""
    if a["results"][j:j + 1].tobytes() != b["results"][j:j + 1].tobytes():
        return False
    return all(a[p + k][j].tobytes() == b[p + k][j].tobytes() for k in kinds for p in ("sigma_", "coeffs_"))


def changed_whole(ex, ref, j):
    e, r = ex["results"][j], ref["results"][j]
    return e["whole_dt_index"] != r["whole_dt_index"] or e["whole_cost"].tobytes() != r["whole_cost"].tobytes() or \
        ex["sigma_whole"][j].tobytes() != ref["sigma_whole"][j].tobytes()


def check_against_list(ex, ref, n):
    """Where the tree found nothing better, everything is the list chain's; elsewhere the exact winner is strictly better
    (an earlier factor, or a cost lower by more than 1e-9).  -> number of corridors whose whole winner changed."""
    n_changed = 0
    for kind in ("whole", "safe"):
        assert ex["cand_ofs_" + kind].tobytes() == ref["cand_ofs_" + kind].tobytes()
    assert ex["feasible_whole"].tobytes() == ref["feasible_whole"].tobytes()
    assert ex["cost_whole"].tobytes() == ref["cost_whole"].tobytes()
    for j in range(n):
        if not changed_whole(ex, ref, j):
            if same_corridor(ex, ref, j):
                continue
            # the whole winner stayed, so R did: only the safe sweep's tree can have moved
            e, r = ex["results"][j], ref["results"][j]
            assert e["safe_dt_index"] < r["safe_dt_index"] or e["safe_cost"] < r["safe_cost"] * (1 - 1e-9), j
            continue
        n_changed += 1
        e, r = ex["results"][j], ref["results"][j]
        assert ex["exact_whole"][j] == 1
        assert (r["whole_dt_index"] < 0 <= e["whole_dt_index"]) or e["whole_dt_index"] < r["whole_dt_index"] or \
            (e["whole_dt_index"] == r["whole_dt_index"] and e["whole_cost"] < r["whole_cost"] * (1 - 1e-9)), j
    return n_changed


def test_config4_unchanged_winners_equal_the_list_chain(solver, report):
    w = cfg4(48)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    ex = solver.replan_pairs_exact(w, all_limit=0)
    n = check_against_list(ex, ref, w["n_prob"])
    assert (ex["nodes_whole"] > 0).any()
    report_line = "config-4, 48 corridors, factors 1..16: %d whole winners changed, exact = 0 whole %d safe %d" % (
        n, int((ex["exact_whole"] == 0).sum()), int((ex["exact_safe"] == 0).sum()))
    report.append(report_line)
    # per-corridor windows: the same rule against fq_replan_pairs_window, window outputs included
    rng = np.random.default_rng(4)
    iw = rng.choice([1.0, 2.0, 3.0], 48)
    win = dict(init_whole=iw, final_whole=iw + 8.0, init_safe=np.ones(48), final_safe=np.full(48, 12.0))
    ref = solver.replan_pairs_window(w, win, all_limit=0)
    ex = solver.replan_pairs_exact(w, all_limit=0, windows=win)
    check_against_list(ex, ref, 48)
    for j in range(48):
        if same_corridor(ex, ref, j):
            for k in capi.WINDOW_OUT_KEYS:
                assert ex[k][j].tobytes() == ref[k][j].tobytes(), (j, k)


def mixed_batch():
    """Forest pairs with 5007 (whole, N = 10, P = 3) and 5055 (safe, N = 10, P = 4) among them.  r_fraction 0 puts R one
    sample after x0, so that the safe sweep of 5055's pair starts where its corridor was built for.  The whole factors start
    at 5, where 5007's optimum is not non-decreasing."""
    pairs = [cr.make_forest_pair_mixed(9700 + j, N=10) for j in range(4)]
    whole = [p[0] for p in pairs]
    safe = [p[1] for p in pairs]
    whole[1] = cr.make_corridor(5007, 3, 10, "uav", True)
    safe[1] = cr.make_corridor(5007, 3, 10, "uav", False)
    whole[2] = cr.make_corridor(5055, 4, 10, "uav", True)
    safe[2] = cr.make_corridor(5055, 4, 10, "uav", False)
    none = np.zeros((0, 10), np.uint8)
    return capi.make_pair_workload(whole, safe, np.arange(5.0, 11.0), none, np.arange(1.0, 11.0), none, DC=0.01, r_fraction=0.0)


def compare_with_restatement(w, ex, F_whole, F_safe, oracle):
    r = ex["results"]
    o = peo.replan_pairs_exact(w, F_whole, F_safe, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    for j, oj in enumerate(o):
        for kind in ("whole", "safe"):
            g, want = r[j], oj[kind]
            assert g[kind + "_dt_index"] == want["dt_index"], (j, kind)
            if want["dt_index"] < 0:
                continue
            assert abs(g[kind + "_cost"] - want["cost"]) <= REL * max(1.0, want["cost"]), (j, kind)
            P = int(np.diff(w["poly_ofs_" + kind])[j])
            sig = ex["sigma_" + kind][j]
            assert g[kind + "_sigma_index"] == peo.list_index(w["N_" + kind], P, 0, sig), (j, kind)
            # the returned assignment attains the optimum
            x0 = w["x0"][j] if kind == "whole" else g["R"]
            xf = w["xf_" + kind][j]
            st, c2, _, _ = oracle.solve_fixed(w["N_" + kind], x0, xf, w["lim"][j], g[kind + "_dt"], peo.polys_of(w, kind, j), sig, kind == "whole")
            assert st == 1 and abs(c2 - want["cost"]) <= 1e-9 * max(1.0, want["cost"]), (j, kind)
        if oj["whole"]["dt_index"] >= 0:
            assert np.allclose(r[j]["R"], oj["R"], rtol=0, atol=1e-9), j
    return o


def test_mixed_batch_finds_the_non_decreasing_misses(solver, oracle, report):
    w = mixed_batch()
    ex = solver.replan_pairs_exact(w, all_limit=0)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    assert (ex["exact_whole"] == 1).all() and (ex["exact_safe"] == 1).all()
    compare_with_restatement(w, ex, [w["factors_whole"]] * w["n_prob"], [w["factors_safe"]] * w["n_prob"], oracle)
    r = ex["results"]
    assert r["whole_sigma_index"][1] == -1 and r["whole_dt_index"][1] >= 0
    assert np.any(np.diff(ex["sigma_whole"][1].astype(int)) < 0)
    assert ref["results"]["whole_dt_index"][1] == r["whole_dt_index"][1]
    assert ref["results"]["whole_cost"][1] > r["whole_cost"][1] * (1 + 1e-9)
    report.append("mixed batch: 5007 whole cost %.9g exact vs %.9g non-decreasing; 5055 safe sigma index %d" % (
        r["whole_cost"][1], ref["results"]["whole_cost"][1], r["safe_sigma_index"][2]))


def permuted(w, seed):
    """Every corridor's polytopes in a random order -> (workload, per corridor and kind: perm with new p = old perm[p])."""
    rng = np.random.default_rng(seed)
    out, perms = dict(w), {"whole": [], "safe": []}
    for kind in ("whole", "safe"):
        po, fo, Ab = w["poly_ofs_" + kind], w["face_ofs_" + kind], w["Ab_" + kind]
        nfo, rows = [0], []
        for j in range(w["n_prob"]):
            P = int(po[j + 1] - po[j])
            perm = rng.permutation(P)
            perms[kind].append(perm)
            for q in perm:
                p = po[j] + q
                rows.append(Ab[fo[p]:fo[p + 1]])
                nfo.append(nfo[-1] + fo[p + 1] - fo[p])
        out["face_ofs_" + kind] = np.asarray(nfo, np.int32)
        out["Ab_" + kind] = np.ascontiguousarray(np.vstack(rows))
    return out, perms


def test_permuted_polytopes_give_the_same_optimum(solver, report):
    """Where both trees ran to the end.  With permuted polytopes the non-decreasing lists often have no feasible candidate
    at the corridor's first feasible factor, so the factors below the list's winner are searched without an incumbent and
    some trees are cut; those corridors are counted, not compared."""
    w = cfg4(32)
    wp, perms = permuted(w, 11)
    a, b = solver.replan_pairs_exact(w), solver.replan_pairs_exact(wp)
    la, lb = solver.replan_pairs_assign(w), solver.replan_pairs_assign(wp)
    assert (a["exact_whole"] == 1).all()
    ok = (a["exact_whole"] == 1) & (b["exact_whole"] == 1)
    assert ok.sum() >= 8
    ra, rb = a["results"], b["results"]
    assert np.array_equal(ra["whole_dt_index"][ok], rb["whole_dt_index"][ok])
    won = ok & (ra["whole_dt_index"] >= 0)
    assert np.allclose(ra["whole_cost"][won], rb["whole_cost"][won], rtol=1e-9, atol=0)
    relabelled = 0
    for j in np.flatnonzero(won):
        sig = perms["whole"][j][b["sigma_whole"][j]]          # the permuted winner in the original labels
        if np.array_equal(sig, a["sigma_whole"][j]):
            relabelled += 1
            continue
        # not relabelled: then the optimum is not unique -- the other labelling's winner attains it too (the tie rule's
        # lexicographic choice depends on the labels)
        polys = peo.polys_of(w, "whole", j)
        f, c, _, _ = solver.solve_batch(w["N_whole"], w["x0"][j], w["xf_whole"][j], w["lim"][j], polys, [ra["whole_dt"][j]], sig[None, :], True)
        assert f[0] and abs(c[0] - ra["whole_cost"][j]) <= 1e-9 * ra["whole_cost"][j], j
    assert relabelled >= won.sum() // 2
    moved = int((la["results"]["whole_cost"] != lb["results"]["whole_cost"]).sum() +
                (la["results"]["whole_dt_index"] != lb["results"]["whole_dt_index"]).sum())
    assert moved >= 3, "the non-decreasing lists did not notice the permutation"
    report.append("permuted config-4: %d of %d exact winners relabelled, %d trees cut, the list chain moved %d" % (
        relabelled, won.sum(), int((b["exact_whole"] == 0).sum()), moved))


def test_complete_lists_run_no_tree(solver):
    pairs = [cr.make_forest_pair_mixed(9800 + j, N=6) for j in range(8)]
    none = np.zeros((0, 6), np.uint8)
    w = capi.make_pair_workload([p[0] for p in pairs], [p[1] for p in pairs], np.arange(1.0, 11.0), none, np.arange(1.0, 11.0), none)
    assert max(np.diff(w["poly_ofs_whole"]).max(), 3) == 3
    ex = solver.replan_pairs_exact(w, all_limit=4096)
    ref = solver.replan_pairs_assign(w, all_limit=4096)
    assert (ex["nodes_whole"] == 0).all() and (ex["nodes_safe"] == 0).all()
    assert (ex["exact_whole"] == 1).all() and (ex["exact_safe"] == 1).all()
    for k in ("results", "sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe", "feasible_whole", "cost_whole", "feasible_safe", "cost_safe"):
        assert ex[k].tobytes() == ref[k].tobytes(), k


def test_cut_and_oversized_corridors_are_isolated(solver):
    """A corridor whose tree is cut (every polytope of 5007 three times at factor 5, where its optimum beats the list's, so
    3^10 copies of it tie) and one padded past the level kernel's 2047 faces get exact = 0 and the list chain's records; the
    other corridors of the batch still run their trees to the end and follow the rule of check_against_list."""
    base = cfg4(6)
    base["factors_whole"] = np.array([5.0])
    pb = cr.make_corridor(5007, 3, 10, "uav", True)
    dup = cc.duplicate_polytopes(pb, 3)
    pad = cc.pad_loose(pb, cc.ITEM_FACE_CAP + 1, binding_last=True, seed=5007)
    safe = cr.make_corridor(5007, 3, 10, "uav", False)
    extra = capi.make_pair_workload([dup, pad], [safe, safe], [5.0], np.zeros((0, 10), np.uint8), FAC, np.zeros((0, 10), np.uint8),
                                    DC=base["DC"], r_fraction=base["r_fraction"])
    w = _concat(base, extra)
    ex = solver.replan_pairs_exact(w)
    ref = solver.replan_pairs_assign(w)
    assert ex["exact_whole"][6] == 0 and ex["exact_whole"][7] == 0
    assert ex["nodes_whole"][6] > 0 and ex["nodes_whole"][7] == 0      # cut after a search; never started
    for j in (6, 7):
        assert same_corridor(ex, ref, j), j
    assert (ex["exact_whole"][:6] == 1).all() and (ex["exact_safe"][:6] == 1).all()
    check_against_list(ex, ref, 8)


def _concat(a, b):
    out = dict(a, n_prob=a["n_prob"] + b["n_prob"])
    for k in ("x0", "xf_whole", "xf_safe", "lim"):
        out[k] = np.ascontiguousarray(np.vstack([a[k], b[k]]))
    for kind in ("whole", "safe"):
        po = np.concatenate([a["poly_ofs_" + kind], b["poly_ofs_" + kind][1:] + a["poly_ofs_" + kind][-1]]).astype(np.int32)
        nfa = int(a["face_ofs_" + kind][-1])
        fo = np.concatenate([a["face_ofs_" + kind], b["face_ofs_" + kind][1:] + nfa]).astype(np.int32)
        out["poly_ofs_" + kind], out["face_ofs_" + kind] = po, fo
        out["Ab_" + kind] = np.ascontiguousarray(np.vstack([a["Ab_" + kind][:nfa], b["Ab_" + kind][:int(b["face_ofs_" + kind][-1])]]))
        out["max_faces_" + kind] = max(a["max_faces_" + kind], b["max_faces_" + kind])
        out["max_poly_faces_" + kind] = max(a["max_poly_faces_" + kind], b["max_poly_faces_" + kind])
    return out


def _dev_exact(solver, w, d, win_dev, torch, dev, cap_w, cap_s, max_fac, gamma, stream):
    """One fq_replan_pairs_exact_dev call with windows aliased in and out, enqueued on `stream` (no synchronisation)."""
    n = w["n_prob"]
    out = dict(coeffs_whole=torch.zeros(n * w["N_whole"] * 12, dtype=torch.float64, device=dev),
               coeffs_safe=torch.zeros(n * w["N_safe"] * 12, dtype=torch.float64, device=dev),
               results=torch.zeros(n * 144, dtype=torch.uint8, device=dev))
    extra = dict(sigma_whole=torch.zeros(n * w["N_whole"], dtype=torch.uint8, device=dev),
                 sigma_safe=torch.zeros(n * w["N_safe"], dtype=torch.uint8, device=dev),
                 exact_whole=torch.full((n,), -1, dtype=torch.int32, device=dev), exact_safe=torch.full((n,), -1, dtype=torch.int32, device=dev),
                 nodes_whole=torch.full((n,), -1, dtype=torch.int64, device=dev), nodes_safe=torch.full((n,), -1, dtype=torch.int64, device=dev))
    a = capi.pair_args(w, lambda k: None if k.startswith(("sigmas_", "factors_")) else d[k].data_ptr(), {k: v.data_ptr() for k, v in out.items()})
    a.n_sig_whole = a.n_sig_safe = a.n_fac_whole = a.n_fac_safe = 0
    mp = (int(np.diff(w["poly_ofs_whole"]).max()), int(np.diff(w["poly_ofs_safe"]).max()))
    s = capi.assign_args(0, {k: extra[k].data_ptr() for k in ("sigma_whole", "sigma_safe")}, mp[0], mp[1], cap_w, cap_s)
    wa = capi.window_args(lambda k: win_dev[k].data_ptr(), {"next_" + k: win_dev[k].data_ptr() for k in pwo.WINDOW_KEYS}, 1.0, gamma,
                          max_fac[0], max_fac[1])
    ex = capi.exact_args({k: extra[k].data_ptr() for k in capi.EXACT_KEYS})
    solver.replan_pairs_exact_dev(a, s, wa, ex, 0, stream.cuda_stream)
    out.update(extra)
    return out


def _host(o, w):
    h = {k: v.cpu().numpy() for k, v in o.items()}
    h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
    h["sigma_whole"] = h["sigma_whole"].reshape(w["n_prob"], -1)
    h["sigma_safe"] = h["sigma_safe"].reshape(w["n_prob"], -1)
    return h


def test_consecutive_device_replans_equal_the_restatement(solver, oracle):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    n, gamma = 4, (2.0, 2.0, 1.0, 1.0)
    w = mixed_batch()
    host = {k: np.full(n, 1.0 if k.startswith("init") else 6.0) for k in pwo.WINDOW_KEYS}
    win_dev = {k: torch.from_numpy(v.copy()).to(dev) for k, v in host.items()}
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith(("sigmas_", "factors_"))}
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    outs = [_dev_exact(solver, w, d, win_dev, torch, dev, 1 << 16, 1 << 17, (41, 41), gamma, st) for _ in range(3)]
    st.synchronize()
    # the host loop: the restatement on each step's windows, then faster.cpp:582-588
    for step, o in enumerate(outs):
        h = _host(o, w)
        r = h["results"]
        Fw = [pwo.factors(a, b, 1.0) for a, b in zip(host["init_whole"], host["final_whole"])]
        Fs = [pwo.factors(a, b, 1.0) for a, b in zip(host["init_safe"], host["final_safe"])]
        assert (h["exact_whole"] == 1).all() and (h["exact_safe"] == 1).all(), step
        compare_with_restatement(w, h, Fw, Fs, oracle)
        nxt = pwo.window_outputs(r, host, Fw, Fs, gamma)
        host = {k: nxt["next_" + k] for k in pwo.WINDOW_KEYS}
    for k in pwo.WINDOW_KEYS:
        assert np.array_equal(win_dev[k].cpu().numpy(), host[k]), k


def test_graph_capture_replays_the_records(solver):
    """No host round trip inside _exact_dev: after a warm-up call it captures into a CUDA graph, whose replay gives the
    same bytes."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    w = cfg4(16)
    n = w["n_prob"]
    win0 = {k: np.full(n, 1.0 if k.startswith("init") else 16.0) for k in pwo.WINDOW_KEYS}
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith(("sigmas_", "factors_"))}
    win_dev = {k: torch.from_numpy(v.copy()).to(dev) for k, v in win0.items()}
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    warm = _dev_exact(solver, w, d, win_dev, torch, dev, 1 << 16, 1 << 17, (16, 16), 20.0, st)
    st.synchronize()
    want = _host(warm, w)
    for k, v in win0.items():
        win_dev[k].copy_(torch.from_numpy(v))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_exact(solver, w, d, win_dev, torch, dev, 1 << 16, 1 << 17, (16, 16), 20.0, st)
    for k, v in win0.items():
        win_dev[k].copy_(torch.from_numpy(v))
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    got = _host(o, w)
    for k in ("results", "sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe", "exact_whole", "exact_safe"):
        assert got[k].tobytes() == want[k].tobytes(), k


def test_two_calls_give_the_same_bytes(solver):
    """Repeated calls, on config-4 corridors and on the tied corridors of duplicated polytopes that do not cut the tree."""
    w = cfg4(16)
    a, b = solver.replan_pairs_exact(w), solver.replan_pairs_exact(w)
    for k in ("results", "sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe", "exact_whole", "exact_safe"):
        assert a[k].tobytes() == b[k].tobytes(), k
    whole, safe = [], []
    for seed, copies in ((5007, 2), (5034, 2)):                  # the tied (uncut) cases of the duplicated corridors
        pb = cr.make_corridor(seed, 3, 10, "uav", True)
        whole.append(cc.duplicate_polytopes(pb, copies))
        sb = cr.make_corridor(seed, 3, 10, "uav", False)
        safe.append(cc.duplicate_polytopes(sb, copies))
    none = np.zeros((0, 10), np.uint8)
    t = capi.make_pair_workload(whole, safe, np.arange(1.0, 8.0), none, np.arange(1.0, 8.0), none, r_fraction=0.0)
    a, b = solver.replan_pairs_exact(t), solver.replan_pairs_exact(t)
    for k in ("results", "sigma_whole", "sigma_safe", "coeffs_whole", "coeffs_safe", "exact_whole", "exact_safe"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert (a["results"]["whole_dt_index"] >= 0).any()


def test_refusals(solver, built_lib):
    w = cfg4(4)
    L = capi.lib()
    out = dict(results=np.zeros(4, capi.PAIR_RESULT_DTYPE))
    a = capi.pair_args(w, lambda k: None if k.startswith("sigmas_") else w[k].ctypes.data, {k: v.ctypes.data for k, v in out.items()})
    a.n_sig_whole = a.n_sig_safe = 0
    s = capi.assign_args(0, {})
    e_out = np.zeros(4, np.int32)
    ex = capi.exact_args({"exact_whole": e_out.ctypes.data})
    h = solver._h
    assert L.fq_replan_pairs_exact(h, a, s, None, None) == capi_E_ARG
    assert L.fq_replan_pairs_exact(h, a, None, None, ex) == capi_E_ARG
    assert L.fq_replan_pairs_exact_dev(h, a, None, None, ex, None, None) == capi_E_ARG
    assert L.fq_replan_pairs_exact_dev(h, a, s, None, None, None, None) == capi_E_ARG
    win = {k: np.full(4, 1.0 if k.startswith("init") else 5.0) for k in pwo.WINDOW_KEYS}
    wa = capi.window_args(lambda k: win[k].ctypes.data, {})
    assert L.fq_replan_pairs_exact(h, a, s, wa, ex) == capi_E_ARG          # a window together with factors_*
    bad = capi.assign_args(-1, {})
    assert L.fq_replan_pairs_exact(h, a, bad, None, ex) == capi_E_ARG      # an _assign refusal
    assert L.fq_replan_pairs_exact(h, a, s, None, ex) == 0                 # and the context still works
    assert capi.has_feature("replan_pairs_exact")
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        assert L.fq_replan_pairs_exact(g._h, a, s, None, ex) == capi_E_ARG
        assert L.fq_replan_pairs_exact_async(g._h, a, s, None, ex) == capi_E_ARG
    finally:
        g.close()


capi_E_ARG = -1


@pytest.fixture(scope="module")
def report():
    lines = []
    yield lines
    print("\n" + "\n".join(lines))
