"""Chained replan with a per-corridor assignment list (fq_replan_pairs_assign*): uniform batches unchanged, mixed batches equal
to one corridor at a time, the CPU restatement, the drop-in class's ALL sweep, the device-pointer entry and its hints, the
refusals, and a group context."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_assign_oracle as pao

pytestmark = pytest.mark.gpu
capi_E_ARG = -1                                      # FQ_E_ARG


def mixed_workload(n, N, seed0, n_fac=6, zero_whole=(0,), r_fraction=0.6):
    """n replans from corridor.make_forest_pair_mixed (polytope counts as Faster::replan trims them); the whole corridors
    listed in zero_whole lose their polytopes (P = 0: no corridor rows)."""
    pairs = [cr.make_forest_pair_mixed(seed0 + j, N=N, r_fraction=r_fraction) for j in range(n)]
    for j in zero_whole:
        pairs[j][0]["polys"], pairs[j][0]["P"] = [], 0
    fac = np.linspace(1.0, 3.0, n_fac)
    none = np.zeros((0, N), np.uint8)
    return capi.make_pair_workload([p[0] for p in pairs], [p[1] for p in pairs], fac, none, fac, none, DC=0.01, r_fraction=r_fraction)


def _counts(w, kind):
    return np.diff(w["poly_ofs_" + kind])


def test_uniform_batch_equals_the_shared_lists(solver):
    """cfg4 corridors (3 whole, 4 safe polytopes each), all_limit = 0: bit for bit fq_replan_pairs with the full lists
    fq_monotone_sigmas(10, 3) / (10, 4)."""
    import bench
    w = bench.load_cfg4(0, 8)
    shared = dict(w, sigmas_whole=cr.monotone_sigmas(10, 3), sigmas_safe=cr.monotone_sigmas(10, 4))
    ref = solver.replan_pairs(shared)
    got = solver.replan_pairs_assign(w, all_limit=0)
    assert got["results"].tobytes() == ref["results"].tobytes()
    for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe"):
        assert got[k].tobytes() == ref[k].tobytes(), k
    nf = len(w["factors_whole"])
    assert np.array_equal(got["cand_ofs_whole"], np.arange(9) * nf * 66) and np.array_equal(got["cand_ofs_safe"], np.arange(9) * nf * 286)
    r = got["results"]
    for j in range(8):
        assert np.array_equal(got["sigma_whole"][j], shared["sigmas_whole"][r["whole_sigma_index"][j]])
        if r["safe_sigma_index"][j] >= 0:
            assert np.array_equal(got["sigma_safe"][j], shared["sigmas_safe"][r["safe_sigma_index"][j]])


@pytest.mark.parametrize("N,all_limit", [(10, 0), (10, 4096), (6, 0), (6, 4096)])
@pytest.mark.parametrize("early_exit", [0, 1])
def test_mixed_batch_equals_one_corridor_at_a_time(built_lib, N, all_limit, early_exit):
    w = mixed_workload(10, N, 8000 + N)
    pw, ps = _counts(w, "whole"), _counts(w, "safe")
    assert set(pw) >= {0, 1, 2, 3} and set(ps) >= {1, 2, 4}
    s = capi.Solver(0)
    s.set_option("sweep_early_exit", early_exit)
    got = s.replan_pairs_assign(w, all_limit=all_limit)
    r = got["results"]
    assert (r["whole_dt_index"] >= 0).sum() >= 5 and (r["safe_dt_index"] >= 0).any()
    for j in range(w["n_prob"]):
        w1 = pao.with_own_lists(pao.corridor(w, j), all_limit)
        one = s.replan_pairs(w1)
        assert r[j:j + 1].tobytes() == one["results"].tobytes(), j
        for kind in ("whole", "safe"):
            co = got["cand_ofs_" + kind]
            assert co[j + 1] - co[j] == len(w1["factors_" + kind]) * len(w1["sigmas_" + kind])
            assert np.array_equal(got["coeffs_" + kind][j], one["coeffs_" + kind][0])
            si = r[kind + "_sigma_index"][j]
            want = w1["sigmas_" + kind][si] if si >= 0 else np.zeros(w["N_" + kind], np.uint8)
            assert np.array_equal(got["sigma_" + kind][j], want)
            if not early_exit:
                assert got["feasible_" + kind][co[j]:co[j + 1]].tobytes() == one["feasible_" + kind].tobytes()
                assert got["cost_" + kind][co[j]:co[j + 1]].tobytes() == one["cost_" + kind].tobytes()
    s.close()


def test_mixed_batch_matches_the_cpu_chain(solver, oracle):
    """The same bars as test_pair_gpu.py's comparison with oracle/pair_oracle.py, corridor lists included."""
    w = mixed_workload(8, 10, 8100)
    g = solver.replan_pairs_assign(w, all_limit=0)
    r = g["results"]
    o = pao.replan_pairs_assign(w, 0, threads=8, dt_base_whole=r["whole_dt_base"], dt_base_safe=r["safe_dt_base"])
    assert np.array_equal(g["cand_ofs_whole"], o["cand_ofs_whole"]) and np.array_equal(g["cand_ofs_safe"], o["cand_ofs_safe"])
    assert np.array_equal(g["feasible_whole"], o["feasible_whole"]), "whole flags differ"
    assert np.array_equal(r["whole_dt_index"], o["whole_dt_index"]) and np.array_equal(r["whole_sigma_index"], o["whole_sigma_index"])
    ok = o["whole_dt_index"] >= 0
    assert ok.any()
    assert np.allclose(r["whole_cost"][ok], o["whole_cost"][ok], rtol=1e-8)
    assert np.array_equal(r["whole_dt"][ok], o["whole_dt"][ok])
    assert np.array_equal(r["n_samples_whole"], o["n_samples_whole"]) and np.array_equal(r["k_safe"], o["k_safe"])
    assert np.abs(r["R"][ok] - o["R"][ok]).max() < 1e-8 and np.isnan(r["R"][~ok]).all()
    assert np.abs(g["coeffs_whole"][ok] - o["coeffs_whole"][ok]).max() < 1e-6
    fok = o["feasible_whole"].astype(bool)
    assert np.allclose(g["cost_whole"][fok], o["cost_whole"][fok], rtol=1e-8)
    assert np.array_equal(g["feasible_safe"], o["feasible_safe"]), "safe flags differ"
    assert np.array_equal(r["safe_dt_index"], o["safe_dt_index"])
    sok = o["safe_dt_index"] >= 0
    assert np.allclose(r["safe_cost"][sok], o["safe_cost"][sok], rtol=1e-6)
    assert np.abs(g["coeffs_safe"][sok] - o["coeffs_safe"][sok]).max() < 1e-5
    assert np.allclose(r["safe_dt_base"][ok], o["safe_dt_base_own"][ok], rtol=1e-6)


def test_whole_winner_equals_the_drop_in_all_sweep(solver):
    """N = 6, P <= 3, all_limit = 4096: every assignment is enumerated, so the whole winner is fq_gen_new_traj's over the
    drop-in class's ALL list with the same time allocations."""
    w = mixed_workload(8, 6, 8200, zero_whole=())
    g = solver.replan_pairs_assign(w, all_limit=4096)
    r = g["results"]
    fac = w["factors_whole"]
    solved = 0
    for j in range(w["n_prob"]):
        w1 = pao.corridor(w, j)
        P = int(w1["poly_ofs_whole"][1])
        polys = [(w1["Ab_whole"][w1["face_ofs_whole"][p]:w1["face_ofs_whole"][p + 1], :3],
                  w1["Ab_whole"][w1["face_ofs_whole"][p]:w1["face_ofs_whole"][p + 1], 3]) for p in range(P)]
        lst = pao.all_assignments(6, P) if P > 1 else np.zeros((1, 6), np.uint8)
        ref = solver.gen_new_traj(6, w["x0"][j], w["xf_whole"][j], w["lim"][j], polys, fac * r["whole_dt_base"][j], lst)
        assert ref["dt_index"] == r["whole_dt_index"][j], j
        if ref["solved"]:
            solved += 1
            assert ref["sigma_index"] == r["whole_sigma_index"][j]
            assert np.array_equal(g["sigma_whole"][j], lst[ref["sigma_index"]])
            assert np.isclose(ref["cost"], r["whole_cost"][j], rtol=1e-12, atol=0)
    assert solved >= 4


def _device(w, torch, dev):
    return {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in capi.PAIR_INPUT_KEYS if not k.startswith("sigmas_")}


def test_device_pointer_entry_and_its_hints(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    w = mixed_workload(8, 10, 8300)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    n = w["n_prob"]
    ncw, ncs = int(ref["cand_ofs_whole"][-1]), int(ref["cand_ofs_safe"][-1])
    mpw, mps = int(_counts(w, "whole").max()), int(_counts(w, "safe").max())
    d = _device(w, torch, dev)
    GUARD = 4096                                     # sentinel tail after every output: nothing may be written there

    def run(hint_w, hint_s, max_poly_w=mpw):
        out = dict(feasible_whole=torch.full((hint_w + GUARD,), 0xAB, dtype=torch.uint8, device=dev),
                   cost_whole=torch.full((hint_w + GUARD,), -5.0, dtype=torch.float64, device=dev),
                   feasible_safe=torch.full((hint_s + GUARD,), 0xAB, dtype=torch.uint8, device=dev),
                   cost_safe=torch.full((hint_s + GUARD,), -5.0, dtype=torch.float64, device=dev),
                   coeffs_whole=torch.zeros(n * 10 * 12, dtype=torch.float64, device=dev),
                   coeffs_safe=torch.zeros(n * 10 * 12, dtype=torch.float64, device=dev),
                   results=torch.zeros(n * 144, dtype=torch.uint8, device=dev))
        lists = dict(cand_ofs_whole=torch.full((n + 1,), -1, dtype=torch.int32, device=dev),
                     cand_ofs_safe=torch.full((n + 1,), -1, dtype=torch.int32, device=dev),
                     sigma_whole=torch.zeros(n * 10, dtype=torch.uint8, device=dev), sigma_safe=torch.zeros(n * 10, dtype=torch.uint8, device=dev))
        a = capi.pair_args(w, lambda k: None if k.startswith("sigmas_") else d[k].data_ptr(), {k: v.data_ptr() for k, v in out.items()})
        a.n_sig_whole = a.n_sig_safe = 0
        s = capi.assign_args(0, {k: v.data_ptr() for k, v in lists.items()}, max_poly_w, mps, hint_w, hint_s)
        st = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize()
        solver.replan_pairs_assign_dev(a, s, 0, st.cuda_stream)
        st.synchronize()
        h = {k: v.cpu().numpy() for k, v in list(out.items()) + list(lists.items())}
        h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
        return h

    h = run(ncw, ncs)
    assert h["results"].tobytes() == ref["results"].tobytes()
    for k in ("feasible_whole", "cost_whole"):
        assert np.array_equal(h[k][:ncw], ref[k]) and (h[k][ncw:] == h[k][-1]).all(), k
    for k in ("feasible_safe", "cost_safe"):
        assert np.array_equal(h[k][:ncs], ref[k]), k
    for k in ("cand_ofs_whole", "cand_ofs_safe"):
        assert np.array_equal(h[k], ref[k]), k
    assert np.array_equal(h["sigma_whole"].reshape(n, 10), ref["sigma_whole"]) and np.array_equal(h["coeffs_whole"].reshape(n, 10, 12), ref["coeffs_whole"])
    # wrong hints: the sweep gets no candidates, every corridor's winner is "none", nothing is written to its outputs
    for hw, hs, mp in ((ncw + 1, ncs, mpw), (ncw - 1, ncs, mpw), (ncw, ncw, mpw - 1)):
        h = run(hw, hs, mp)
        r = h["results"]
        assert (r["whole_dt_index"] == -1).all() and (r["safe_dt_index"] == -1).all() and np.isnan(r["R"]).all()
        assert not h["cand_ofs_whole"].any() and (h["feasible_whole"] == 0xAB).all() and (h["cost_whole"] == -5.0).all()
        assert not h["sigma_whole"].any()
    h = run(ncw, ncs + 7)                                            # only the safe hint is wrong
    assert np.array_equal(h["results"]["whole_dt_index"], ref["results"]["whole_dt_index"])
    assert (h["results"]["safe_dt_index"] == -1).all() and (h["feasible_safe"] == 0xAB).all()


def test_refusals(solver):
    w = mixed_workload(3, 10, 8400, zero_whole=())
    a = capi.pair_args(w, lambda k: w[k].ctypes.data, {})
    L = capi.lib()
    res = np.zeros(3, capi.PAIR_RESULT_DTYPE)
    a.results = res.ctypes.data
    sig = np.zeros((1, 10), np.uint8)

    def call(a, s):
        return L.fq_replan_pairs_assign(solver._h, capi.C.byref(a), capi.C.byref(s))
    ok = capi.assign_args(0, {})
    a.sigmas_whole, a.sigmas_safe, a.n_sig_whole, a.n_sig_safe = None, None, 0, 0
    assert call(a, ok) == 0 and (res["whole_dt_index"] >= -1).all()
    for field, value in (("sigmas_whole", sig.ctypes.data), ("n_sig_safe", 1)):
        bad = capi.PairArgs.from_buffer_copy(a)
        setattr(bad, field, value)
        assert call(bad, ok) == capi_E_ARG
    assert call(a, capi.assign_args(-1, {})) == capi_E_ARG
    assert L.fq_replan_pairs_assign(solver._h, capi.C.byref(a), None) == capi_E_ARG
    # a corridor list longer than 2^20: 32 polytopes and N = 16 (C(47, 16) non-decreasing assignments)
    A1 = w["Ab_safe"][w["face_ofs_safe"][0]:w["face_ofs_safe"][1]]
    big = dict(w, N_safe=16, poly_ofs_safe=np.array([0, 32, 33, 34], np.int32),
               face_ofs_safe=np.arange(35, dtype=np.int32) * len(A1), Ab_safe=np.ascontiguousarray(np.tile(A1, (34, 1))))
    with pytest.raises(capi.FqError, match="2\\^20"):
        solver.replan_pairs_assign(big, all_limit=0)
    # more than 2^30 candidates in a sweep: 4^10 = 2^20 assignments per corridor (all_limit 2^20) x 1025 factors
    w4 = mixed_workload(1, 10, 8010, zero_whole=())               # (3, 4) polytopes
    assert _counts(w4, "safe")[0] == 4
    w4["factors_safe"] = np.linspace(1.0, 3.0, 1025)
    with pytest.raises(capi.FqError, match="too many candidates"):
        solver.replan_pairs_assign(w4, all_limit=1 << 20)
    # _dev hints out of range
    d = capi.pair_args(w, lambda k: None, {})
    d.n_sig_whole = d.n_sig_safe = 0
    for s in (capi.assign_args(0, {}, 33, 4, 10, 10), capi.assign_args(0, {}, 3, 4, (1 << 30) + 1, 10), capi.assign_args(0, {}, 3, -1, 10, 10)):
        assert L.fq_replan_pairs_assign_dev(solver._h, capi.C.byref(d), capi.C.byref(s), None, None) == capi_E_ARG
    assert capi.has_feature("replan_pairs_assign")


@pytest.mark.parametrize("n_gpus", [1, 2])
def test_group_context_shards_by_candidates(solver, n_gpus):
    import torch
    if torch.cuda.device_count() < n_gpus:
        pytest.skip("needs %d GPUs" % n_gpus)
    w = mixed_workload(9, 10, 8500)
    ref = solver.replan_pairs_assign(w, all_limit=0)
    both = (ref["cand_ofs_whole"] + ref["cand_ofs_safe"]).astype(np.int32)
    bounds = [capi.shard_range(w["n_prob"], both, r, n_gpus) for r in range(n_gpus)]
    assert bounds[0][0] == 0 and bounds[-1][1] == w["n_prob"]
    g = capi.Solver(n_gpus=n_gpus, devices=list(range(n_gpus)))
    out = g.replan_pairs_assign(w, all_limit=0)
    assert out["results"].tobytes() == ref["results"].tobytes()
    for k in ("feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe", "cand_ofs_whole",
              "cand_ofs_safe", "sigma_whole", "sigma_safe"):
        assert np.array_equal(out[k], ref[k]), k
    out2 = g.replan_pairs_assign(w, all_limit=0, deferred=True)
    g.wait()
    assert out2["results"].tobytes() == ref["results"].tobytes() and np.array_equal(out2["sigma_safe"], ref["sigma_safe"])
    g.close()
