"""The committed plan of the chained replan (fq_replan_pairs_plan*): every chain selection gives its family's own outputs byte
for byte and a plan byte-equal to tests/pair_plan_oracle.py (appendToPlan over fillX) applied to that call's coefficients and
records; config-4 against the CPU chain; the capacity suffix; the async entry; the _dev entry in an _hr closed loop with
CUDA-graph capture; the refusals."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_plan_oracle as ppo
from test_pair_hr_gpu import replans, workload, _dev_state, _host
from test_pair_map_gpu import assert_same, make_maps

pytestmark = pytest.mark.gpu
UAV = cr.UAV


def cfg4(n, start=0):
    import bench
    return bench.load_cfg4(start, n)


def shared(w):
    return dict(w, sigmas_whole=cr.monotone_sigmas(w["N_whole"], 3), sigmas_safe=cr.monotone_sigmas(w["N_safe"], 4))


def windows(n, seed=4):
    rng = np.random.default_rng(seed)
    return dict(init_whole=rng.integers(1, 4, n).astype(float), final_whole=rng.integers(6, 12, n).astype(float),
                init_safe=rng.integers(1, 4, n).astype(float), final_safe=rng.integers(6, 12, n).astype(float))


def split(out):
    """(the family's outputs, the plan) of a replan_pairs_plan return value."""
    return {k: v for k, v in out.items() if k not in ppo_keys}, {k: out[k] for k in ppo_keys}


ppo_keys = capi.PLAN_KEYS


def check_plan(out, w, plan):
    """The plan against the restatement on the call's own records and coefficients; whole row k_safe is R."""
    need = out.get("need_safe")
    want = ppo.plan(out["results"], out["coeffs_whole"], out["coeffs_safe"], w["N_whole"], w["N_safe"], w["DC"], need,
                    len(plan["states"]))
    assert plan["plan_ofs"].tobytes() == want[1].tobytes()
    assert plan["status"].tobytes() == want[2].tobytes()
    f = ppo.filled_rows(want[1], len(plan["states"]))
    assert plan["states"][:f].tobytes() == want[0][:f].tobytes()
    res = out["results"]
    for j in np.flatnonzero(plan["status"] == ppo.PLAN_OK):
        k = res["k_safe"][j]
        row = plan["states"][plan["plan_ofs"][j] + k]
        if need is None or need[j]:
            assert row[:9].tobytes() == res["R"][j].tobytes(), j
        else:
            assert k == res["n_samples_whole"][j] - 1 and not row[3:].any(), j
    return want


def run_both(solver, w, chain, *args, **kw):
    """The family's own call and the _plan call with the capacity a first _plan call with cap 0 reports: every non-plan
    output byte for byte, the plan against the restatement."""
    fam = solver.replan_pairs if chain == "shared" else getattr(solver, "replan_pairs_" + chain)
    ref = fam(w, *args, **kw)
    sized = solver.replan_pairs_plan(w, 0, chain, *args, **kw)
    total = int(sized["plan_ofs"][-1])
    assert total > 0 and (sized["status"] != ppo.PLAN_OK).all()
    got = solver.replan_pairs_plan(w, total, chain, *args, **kw)
    mine, plan = split(got)
    assert_same(mine, ref)
    assert plan["plan_ofs"].tobytes() == sized["plan_ofs"].tobytes()
    check_plan(got, w, plan)
    return got


_LISTS = [("shared", (), {}), ("assign", (), {}), ("window", None, {}), ("exact", (), {}), ("exact", None, {})]


@pytest.mark.parametrize("chain,args,kw", _LISTS, ids=["shared", "assign", "window", "exact", "exact_window"])
def test_list_chains(solver, chain, args, kw):
    w = cfg4(24)
    if chain == "shared":
        w = shared(w)
    if args is None:                                         # per-corridor windows
        kw = dict(windows=windows(24)) if chain == "exact" else {}
        args = () if chain == "exact" else (windows(24),)
    got = run_both(solver, w, chain, *args, **kw)
    st = got["status"]
    assert (st == ppo.PLAN_OK).sum() >= 8


@pytest.mark.parametrize("chain", ["decomp", "hr", "map"])
def test_decomposing_chains(solver, chain):
    ps = replans(32, 0)
    w = workload(ps)
    n = len(ps)
    kw = dict(last_factor_safe=np.random.default_rng(3).uniform(1.0, 8.0, n)) if chain != "decomp" else {}
    args = ()
    if chain == "map":
        maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
        args = (maps, np.arange(n))
        kw["max_local"] = max(len(p["unk"]) + len(p["obs"]) for p in ps)
    got = run_both(solver, w, chain, *args, **kw)
    if chain != "decomp":
        won = got["results"]["whole_dt_index"] >= 0
        assert (got["need_safe"][won] == 0).sum() >= 3 and (got["need_safe"][won] == 1).sum() >= 3
        assert ((got["status"] == ppo.PLAN_OK) & (got["need_safe"] == 0)).any()


def test_without_coefficients(solver):
    """coeffs_* NULL: the chain keeps the winners' coefficients itself; the plan is the one a call with them gives."""
    w = cfg4(16)
    a = solver.replan_pairs_plan(w, 1 << 16, "assign")
    b = solver.replan_pairs_plan(w, 1 << 16, "assign", want_coeffs=False, want_candidates=False)
    assert "coeffs_safe" not in b
    for k in capi.PLAN_KEYS + ["results"]:
        assert a[k].tobytes() == b[k].tobytes(), k
    ps = replans(16, 100)
    wh = workload(ps)
    a = solver.replan_pairs_plan(wh, 1 << 16, "hr")
    b = solver.replan_pairs_plan(wh, 1 << 16, "hr", want_coeffs=False)
    for k in capi.PLAN_KEYS + ["results", "need_safe"]:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_config4_against_the_cpu_chain(solver, oracle):
    from oracle import pair_oracle
    w = shared(cfg4(12))
    got = solver.replan_pairs_plan(w, 1 << 16, "shared")
    res = got["results"]
    ref = pair_oracle.replan_pairs(w, threads=4, dt_base_whole=res["whole_dt_base"], dt_base_safe=res["safe_dt_base"], fast=True)
    want = ppo.plan(ref, ref["coeffs_whole"], ref["coeffs_safe"], w["N_whole"], w["N_safe"], w["DC"])
    assert got["status"].tobytes() == want[2].tobytes() and got["plan_ofs"].tobytes() == want[1].tobytes()
    total = int(want[1][-1])
    x, y = got["states"][:total], want[0]
    assert (np.abs(x - y) <= 1e-9 * np.maximum(np.abs(y), 1.0)).all()
    assert (got["status"] == ppo.PLAN_OK).sum() >= 6


def test_capacity_suffix_and_async(solver):
    w = cfg4(24)
    full = solver.replan_pairs_plan(w, 1 << 16, "assign")
    ofs = full["plan_ofs"]
    total = int(ofs[-1])
    ok = np.flatnonzero(full["status"] == ppo.PLAN_OK)
    assert len(ok) >= 8
    for cap in (0, total, total - 1, int(ofs[ok[len(ok) // 2]]) + 3):
        got = solver.replan_pairs_plan(w, cap, "assign")
        assert got["plan_ofs"].tobytes() == ofs.tobytes(), cap
        f = ppo.filled_rows(ofs, cap)
        cut = full["status"].copy()
        cut[(cut == ppo.PLAN_OK) & (ofs[1:] > cap)] = ppo.PLAN_CAPACITY
        assert got["status"].tobytes() == cut.tobytes(), cap
        assert got["states"][:f].tobytes() == full["states"][:f].tobytes(), cap
        assert not got["states"][f:].any(), cap                     # the host rows past the filled prefix are untouched
        c = np.flatnonzero(cut == ppo.PLAN_CAPACITY)
        o = np.flatnonzero(cut == ppo.PLAN_OK)
        assert len(c) == 0 or len(o) == 0 or o.max() < c.min()
        if cap == total - 1:
            assert c.tolist() == [ok[-1]]
    d = solver.replan_pairs_plan(w, total, "assign", deferred=True)
    solver.wait()
    for k in capi.PLAN_KEYS + ["results"]:
        assert d[k].tobytes() == full[k][:len(d[k])].tobytes(), k


def _dev_plan_call(solver, w, d, win_dev, last_dev, plan_dev, torch, dev, stream):
    """One _plan_dev call of the _hr chain; windows and last_factor_safe are read and written in place."""
    n = w["n_prob"]
    out = dict(results=torch.zeros(n * 144, dtype=torch.uint8, device=dev), index_H=torch.full((n,), -7, dtype=torch.int32, device=dev),
               need_safe=torch.full((n,), 7, dtype=torch.uint8, device=dev))
    a = capi.PairArgs()
    a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, w["N_whole"], w["N_safe"], w["DC"], w["r_fraction"]
    for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe"):
        setattr(a, k, d[k].data_ptr())
    a.results = out["results"].data_ptr()
    for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
        setattr(a, k, int(w[k]))
    s = capi.assign_args(0, {}, 3, 4, 1 << 16, 1 << 16)
    wa = capi.window_args(lambda k: win_dev[k].data_ptr(), {"next_" + k: win_dev[k].data_ptr() for k in capi.WINDOW_IN_KEYS}, 1.0, 20.0,
                          64, 64)
    mo = int(np.diff(w["obs_ofs_whole"]).max())
    dc = capi.decomp_args(lambda k: d[k].data_ptr(), {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"], mo, mo)
    hr = capi.hr_args(d["unk_ofs"].data_ptr(), d["unk"].data_ptr(), dict(last_factor_safe=last_dev.data_ptr(),
                      index_H=out["index_H"].data_ptr(), need_safe=out["need_safe"].data_ptr()))
    pl = capi.plan_args(plan_dev["cap"], {k: plan_dev[k].data_ptr() for k in capi.PLAN_KEYS})
    solver.replan_pairs_plan_dev(a, s, wa, None, dc, hr, None, pl, 0, stream.cuda_stream)
    return out


def test_dev_closed_loop_captures(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = replans(24, 600)
    w = workload(ps)
    n = w["n_prob"]
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 10.0), init_safe=np.ones(n), final_safe=np.full(n, 10.0))
    d = _dev_state(w, torch, dev)
    st = torch.cuda.Stream(device=dev)
    cap = 1 << 15
    pd = dict(cap=cap, states=torch.full((cap + 4, 12), -3.0, dtype=torch.float64, device=dev),
              plan_ofs=torch.full((n + 1,), -9, dtype=torch.int64, device=dev), status=torch.full((n,), -9, dtype=torch.int32, device=dev))

    def reset():
        win = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
        return win, torch.zeros(n, dtype=torch.float64, device=dev)

    def snap(o):
        h = _host(o)
        h.update({k: pd[k].cpu().numpy() for k in capi.PLAN_KEYS})
        return h

    win, last = reset()
    torch.cuda.synchronize()
    outs = []
    for _ in range(4):
        o = _dev_plan_call(solver, w, d, win, last, pd, torch, dev, st)
        st.synchronize()
        outs.append(snap(o))
    assert (outs[0]["states"][cap:] == -3.0).all()                 # nothing past cap_states
    wins, lastf = {k: v.copy() for k, v in w0.items()}, np.zeros(n)
    for o in outs:
        ref = solver.replan_pairs_plan(w, cap, "hr", last_factor_safe=lastf, windows=wins)
        assert o["results"].tobytes() == ref["results"].tobytes() and o["need_safe"].tobytes() == ref["need_safe"].tobytes()
        assert o["plan_ofs"].tobytes() == ref["plan_ofs"].tobytes() and o["status"].tobytes() == ref["status"].tobytes()
        f = ppo.filled_rows(ref["plan_ofs"], cap)
        assert o["states"][:f].tobytes() == ref["states"][:f].tobytes()
        check_plan(ref, w, ref)
        wins = {k: ref["next_" + k].copy() for k in capi.WINDOW_IN_KEYS}
        lastf = ref["last_factor_safe"].copy()
    assert any((o["need_safe"] == 0).any() for o in outs) and any(o["need_safe"].any() for o in outs)
    # captured once, replayed from the start-up state twice: the first fresh call's bytes each time
    win, lastd = reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_plan_call(solver, w, d, win, lastd, pd, torch, dev, st)
    for _ in range(2):
        for k, v in w0.items():
            win[k].copy_(torch.from_numpy(v))
        lastd.zero_()
        pd["states"].fill_(-3.0)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        rep = snap(o)
        for k in rep:
            assert rep[k].tobytes() == outs[0][k].tobytes(), k


def test_refusals(solver, built_lib):
    L = capi.lib()
    B = C.byref
    w = cfg4(4)
    out = solver.replan_pairs_assign(w)
    s = capi.assign_args(0, {k: out[k].ctypes.data for k in ("cand_ofs_whole", "cand_ofs_safe", "sigma_whole", "sigma_safe")})
    a = capi.pair_args(w, lambda k: None if k.startswith("sigmas_") else w[k].ctypes.data, {"results": out["results"].ctypes.data})
    a.n_sig_whole = a.n_sig_safe = 0
    states, ofs, st = np.zeros((4096, 12)), np.zeros(5, np.int64), np.zeros(4, np.int32)
    good = capi.plan_args(4096, dict(states=states.ctypes.data, plan_ofs=ofs.ctypes.data, status=st.ctypes.data))

    def err(h=None):
        return L.fq_last_error(h or solver._h).decode()

    for fn in (L.fq_replan_pairs_plan, L.fq_replan_pairs_plan_async):
        assert fn(solver._h, B(a), B(s), None, None, None, None, None, B(good)) == 0
        solver.wait()
    for host in (True, False):
        def call(pl, s_=s, win=None):
            if host:
                return L.fq_replan_pairs_plan(solver._h, B(a), B(s_) if s_ is not None else None, win, None, None, None, None, pl)
            return L.fq_replan_pairs_plan_dev(solver._h, B(a), B(s_) if s_ is not None else None, win, None, None, None, None, pl,
                                              None, None)
        assert call(None) == -1 and err() == "plan is NULL"
        for k in ("states", "plan_ofs"):
            bad = capi.plan_args(4096, dict(states=states.ctypes.data, plan_ofs=ofs.ctypes.data))
            setattr(bad, k, None)
            assert call(B(bad)) == -1 and "must not be NULL" in err(), k
        bad = capi.plan_args(-1, dict(states=states.ctypes.data, plan_ofs=ofs.ctypes.data))
        assert call(B(bad)) == -1 and err() == "plan: cap_states < 0"
        wa = capi.window_args(lambda k: None, {})
        assert call(B(good), None, B(wa)) == -1 and err() == "assign is NULL"
    # the family's own refusals, with the family's text
    a.DC = 0.0
    assert L.fq_replan_pairs_assign(solver._h, B(a), B(s)) == -1
    want = err()
    assert L.fq_replan_pairs_plan(solver._h, B(a), B(s), None, None, None, None, None, B(good)) == -1 and err() == want
    a.DC = w["DC"]
    ps = replans(4, 800)
    wh = workload(ps)
    ref = solver.replan_pairs_hr(wh, delta_H=0.5)
    with pytest.raises(capi.FqError) as e1:
        solver.replan_pairs_hr(wh, delta_H=1.5)
    with pytest.raises(capi.FqError) as e2:
        solver.replan_pairs_plan(wh, 64, "hr", delta_H=1.5)
    assert str(e1.value) == str(e2.value)
    got = solver.replan_pairs_plan(wh, 1 << 14, "hr", delta_H=0.5)
    assert got["results"].tobytes() == ref["results"].tobytes()      # the context still works
    assert capi.has_feature("replan_pairs_plan")
    assert L.fq_replan_pairs_plan(None, None, None, None, None, None, None, None, None) == -1
    assert L.fq_replan_pairs_plan_dev(None, None, None, None, None, None, None, None, None, None, None) == -1
    # a one-device group context
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        for fn in (L.fq_replan_pairs_plan, L.fq_replan_pairs_plan_async):
            assert fn(g._h, B(a), B(s), None, None, None, None, None, B(good)) == -1
            assert "multi-GPU" in err(g._h)
        assert L.fq_replan_pairs_plan_dev(g._h, B(a), B(s), None, None, None, None, None, B(good), None, None) == -1
        assert L.fq_replan_pairs_assign(g._h, B(a), B(s)) == 0                 # the family itself shards
    finally:
        g.close()
