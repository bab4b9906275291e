"""Chained replan that chooses H and R from each corridor's unknown space (fq_replan_pairs_hr*), on forest corridors with seeded
unknown clouds (corridor.forest_unknown_cloud): H, R and need_safe bit-equal to tests/pair_hr_oracle.py applied to the device's
own whole winners; every safe-side output equal to _decomp run with r_fraction at the same index; the records against the CPU
chain; the no-safe-path branch and its window carry; hand-built edges; a closed loop of _hr_dev calls with CUDA-graph capture;
the refusals."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_hr_oracle as hro
import pair_window_oracle as pwo

pytestmark = pytest.mark.gpu
UAV = cr.UAV
FAC = np.arange(1.0, 11.0)
_PS = {}


def replans(n, start=0):
    key = (n, start)
    if key not in _PS:
        ps = [cr.forest_pair_paths(30000 + start + k) for k in range(n)]
        for p in ps:
            p["unk"] = cr.forest_unknown_cloud(p)
        _PS[key] = ps
    return _PS[key]


def workload(ps, r_fraction=0.6):
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    w["r_fraction"] = r_fraction
    return w


def check_restatement(ps, w, out, params=(0.42, 0.5, 1.0)):
    """index_H, need_safe, k_safe, n and R of every corridor bit-equal to the restatement on the device's whole winners."""
    res = out["results"]
    for j, p in enumerate(ps):
        if res["whole_dt_index"][j] < 0:
            assert out["index_H"][j] == -1 and res["k_safe"][j] == -1 and out["need_safe"][j] == 0 and np.isnan(res["R"][j]).all()
            continue
        h = hro.hr_of(out["coeffs_whole"][j], res["whole_dt"][j], w["N_whole"], w["DC"], p["unk"], p["lim"][1], *params)
        assert (out["need_safe"][j], out["index_H"][j], res["k_safe"][j], res["n_samples_whole"][j]) == \
            (h["need_safe"], h["index_H"], h["k_safe"], h["n"]), j
        assert res["R"][j].tobytes() == h["R"].tobytes(), j


@pytest.mark.parametrize("exact", [False, True])
def test_h_and_r_are_the_restatement_bit_for_bit(solver, exact):
    ps = replans(64)
    w = workload(ps)
    out = solver.replan_pairs_hr(w, exact=exact)
    check_restatement(ps, w, out)
    won = out["results"]["whole_dt_index"] >= 0
    assert (out["need_safe"][won] == 1).sum() >= 10 and (out["need_safe"][won] == 0).sum() >= 10


def test_only_k_changed(solver):
    """A corridor that needs a safe path: _decomp alone on it, with r_fraction putting R at the same index, gives the same
    record, corridors, statuses and E / M byte for byte."""
    ps = replans(64)
    w = workload(ps)
    out = solver.replan_pairs_hr(w)
    res = out["results"]
    need = np.flatnonzero(out["need_safe"] == 1)
    assert len(need) >= 10
    for j in need:
        w1 = workload([ps[j]], r_fraction=(res["k_safe"][j] + 0.5) / res["n_samples_whole"][j])
        d = solver.replan_pairs_decomp(w1)
        assert d["results"].tobytes() == res[j:j + 1].tobytes(), j
        for kind in ("whole", "safe"):
            fo, po = out["face_ofs_" + kind], w["poly_ofs_" + kind]
            mine = out["Ab_" + kind][fo[po[j]]:fo[po[j + 1]]]
            assert np.array_equal(np.diff(d["face_ofs_" + kind]), np.diff(fo[po[j]:po[j + 1] + 1])), (kind, j)
            assert d["Ab_" + kind][:len(mine)].tobytes() == mine.tobytes(), (kind, j)
            assert d["status_" + kind][0] == out["status_" + kind][j], (kind, j)
        assert d["E"].tobytes() == out["E"][j:j + 1].tobytes() and d["M"].tobytes() == out["M"][j:j + 1].tobytes(), j


def test_records_match_the_cpu_chain(solver):
    ps = replans(12, 200)
    w = workload(ps)
    out = solver.replan_pairs_hr(w)
    res = out["results"]
    assert 0 < out["need_safe"].sum() < len(ps)
    for j, p in enumerate(ps):
        ref = hro.replan_pair_hr(p, FAC, dt_base_whole=res["whole_dt_base"][j], dt_base_safe=res["safe_dt_base"][j])
        for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
            assert ref[k] == res[k][j], (k, j)
        assert ref["need_safe"] == out["need_safe"][j] and ref["index_H"] == out["index_H"][j], j
        for k in ("whole_cost", "safe_cost", "whole_dt", "safe_dt", "R"):
            x, y = np.atleast_1d(res[k][j]), np.atleast_1d(ref[k])
            assert np.array_equal(np.isfinite(x), np.isfinite(y)), (k, j)
            f = np.isfinite(y)
            assert np.all(np.abs(x[f] - y[f]) <= 1e-8 * np.maximum(np.abs(y[f]), 1.0)), (k, j)


def test_no_safe_path(solver):
    ps = replans(64)
    w = workload(ps)
    n = len(ps)
    rng = np.random.default_rng(4)
    wins = dict(init_whole=rng.integers(1, 4, n).astype(float), final_whole=rng.integers(6, 12, n).astype(float),
                init_safe=rng.integers(1, 4, n).astype(float), final_safe=rng.integers(6, 12, n).astype(float))
    last = rng.uniform(1.0, 8.0, n)
    out = solver.replan_pairs_hr(w, last_factor_safe=last, windows=wins, want_candidates=True)
    res = out["results"]
    won = res["whole_dt_index"] >= 0
    free = np.flatnonzero(won & (out["need_safe"] == 0))
    need = np.flatnonzero(won & (out["need_safe"] == 1))
    assert len(free) >= 10 and len(need) >= 10
    co = out["cand_ofs_safe"]
    for j in free:
        r = res[j]
        assert np.isnan(r["R"]).all() and r["k_safe"] == r["n_samples_whole"] - 1 and r["safe_dt_index"] == -1, j
        assert out["trials_safe"][j] == 0 and out["status_safe"][j] == capi.DECOMP_STATUS["not_run"], j
        assert not out["feasible_safe"][co[j]:co[j + 1]].any(), j
        assert out["last_factor_safe"][j] == last[j], j
        lo, hi = pwo.next_window(True, last[j], 20.0, 20.0, wins["init_safe"][j], wins["final_safe"][j])
        assert (out["next_init_safe"][j], out["next_final_safe"][j]) == (lo, hi), j
        fw = capi.window_factors(wins["init_whole"][j], wins["final_whole"][j], 1.0)[r["whole_dt_index"]]
        assert (out["next_init_whole"][j], out["next_final_whole"][j]) == pwo.next_window(True, fw, 20.0, 20.0, 0, 0), j
    for j in need:
        ds = res["safe_dt_index"][j]
        want = capi.window_factors(wins["init_safe"][j], wins["final_safe"][j], 1.0)[ds] if ds >= 0 else last[j]
        assert out["last_factor_safe"][j] == want, j
    # the other corridors of the mixed batch are byte for byte those of a batch without the corridors that need no safe path
    sub = [ps[j] for j in need]
    ws = workload(sub)
    sw = {k: v[need] for k, v in wins.items()}
    alone = solver.replan_pairs_hr(ws, last_factor_safe=last[need], windows=sw)
    assert alone["results"].tobytes() == res[need].tobytes()
    for k in capi.WINDOW_OUT_KEYS + ["last_factor_safe", "index_H", "need_safe"]:
        assert alone[k].tobytes() == out[k][need].tobytes(), k


def test_hand_built_edges(solver):
    """Clouds placed relative to the samples of a first run (the whole winner does not depend on the cloud)."""
    pool = [dict(p) for p in replans(12, 400)]
    for p in pool:
        p["unk"] = np.zeros((0, 3))
    first = solver.replan_pairs_hr(workload(pool), drone_radius=0.5)
    keep = np.flatnonzero(first["results"]["whole_dt_index"] >= 0)[:8]
    assert len(keep) == 8
    ps = [pool[j] for j in keep]
    res = first["results"][keep]
    assert not first["need_safe"][keep].any() and (first["index_H"][keep] == res["n_samples_whole"] - 1).all()   # empty clouds
    w = workload(ps)
    X = [capi.fill_x(w["N_whole"], first["coeffs_whole"][j].reshape(-1), first["results"]["whole_dt"][j], w["DC"]) for j in keep]
    f32 = np.float32
    q0 = [x[0, :3].astype(f32) for x in X]
    at = q0[0].copy()
    at[2] = q0[0][2] - f32(0.5)                                              # float distance exactly 0.5 from query 0
    assert f32(q0[0][2] - at[2]) == f32(0.5)
    inside = q0[1].copy()
    inside[2] = np.nextafter(q0[1][2] - f32(0.5), q0[1][2])                 # one float ulp inside
    clouds = [at[None].astype(np.float64), inside[None].astype(np.float64), X[2][:1, :3].copy(),
              X[3][5:6, :3] + [0.0, 0.0, 0.3], np.zeros((0, 3)), X[5][min(30, len(X[5]) - 1):][:1, :3].copy(),
              X[6][-1:, :3].copy(), X[7][:1, :3] + [0.0, 0.0, 0.2]]
    for p, c in zip(ps, clouds):
        p["unk"] = c
    w = workload(ps)
    for params in ((0.5, 0.5, 1.0), (0.5, 0.5, 0.5), (0.25, 0.3, 1.0)):
        out = solver.replan_pairs_hr(w, drone_radius=params[0], delta_a=params[1], delta_H=params[2])
        assert out["results"]["whole_dt"].tobytes() == res["whole_dt"].tobytes()
        check_restatement(ps, w, out, params)
        if params[0] == 0.5:
            assert out["need_safe"][1] == 1 and out["index_H"][1] == 0 and out["results"]["k_safe"][1] == 0
            assert out["need_safe"][2] == 1 and out["index_H"][2] == 0 and out["results"]["k_safe"][2] == 0
            assert out["need_safe"][4] == 0


def _dev_state(w, torch, dev):
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in
         ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "unk_ofs", "unk") + tuple(capi.DECOMP_IN_KEYS)}
    return d


def _dev_call(solver, w, d, win_dev, last_dev, torch, dev, stream, extra=None):
    """One _hr_dev call; windows and last_factor_safe are read and written in place (outputs aliasing the inputs)."""
    n = w["n_prob"]
    out = dict(results=torch.zeros(n * 144, dtype=torch.uint8, device=dev),
               index_H=torch.full((n,), -7, dtype=torch.int32, device=dev), need_safe=torch.full((n,), 7, dtype=torch.uint8, device=dev))
    dout = dict(status_whole=torch.full((n,), -1, dtype=torch.int32, device=dev), status_safe=torch.full((n,), -1, dtype=torch.int32, device=dev))
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
    dc = capi.decomp_args(lambda k: d[k].data_ptr(), {k: v.data_ptr() for k, v in dout.items()}, UAV["bbox"], UAV["drone_radius"],
                          UAV["z_ground"], mo, mo)
    hr = capi.hr_args(d["unk_ofs"].data_ptr(), d["unk"].data_ptr(), dict(last_factor_safe=last_dev.data_ptr(),
                      index_H=out["index_H"].data_ptr(), need_safe=out["need_safe"].data_ptr()))
    solver.replan_pairs_hr_dev(a, s, wa, None, dc, hr, 0, stream.cuda_stream)
    out.update(dout)
    return out


def _host(o):
    h = {k: v.cpu().numpy() for k, v in o.items()}
    h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
    return h


def test_closed_loop_on_the_device_is_deterministic_and_captures(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = replans(32, 600)
    w = workload(ps)
    n = w["n_prob"]
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 10.0), init_safe=np.ones(n), final_safe=np.full(n, 10.0))
    d = _dev_state(w, torch, dev)
    st = torch.cuda.Stream(device=dev)

    def reset():
        win = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
        return win, torch.zeros(n, dtype=torch.float64, device=dev)

    def loop():
        win, last = reset()
        torch.cuda.synchronize()
        outs = []
        for _ in range(8):
            o = _dev_call(solver, w, d, win, last, torch, dev, st)
            st.synchronize()
            h = _host(o)
            h.update({k: v.cpu().numpy() for k, v in win.items()}, last=last.cpu().numpy())
            outs.append(h)
        return outs

    outs = loop()
    # the host entry, windows and last_factor_safe carried on the host, each step's H and R against the restatement
    wins, last = {k: v.copy() for k, v in w0.items()}, np.zeros(n)
    for o in outs:
        ref = solver.replan_pairs_hr(w, last_factor_safe=last, windows=wins)
        check_restatement(ps, w, ref)
        assert o["results"].tobytes() == ref["results"].tobytes()
        assert o["index_H"].tobytes() == ref["index_H"].tobytes() and o["need_safe"].tobytes() == ref["need_safe"].tobytes()
        wins = {k: ref["next_" + k].copy() for k in capi.WINDOW_IN_KEYS}
        last = ref["last_factor_safe"].copy()
        for k in capi.WINDOW_IN_KEYS:
            assert o[k].tobytes() == wins[k].tobytes(), k
        assert o["last"].tobytes() == last.tobytes()
    assert any(o["need_safe"].any() for o in outs) and any((o["need_safe"] == 0).any() for o in outs)
    again = loop()
    for a, b in zip(outs, again):
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
    # one call captured in a CUDA graph and replayed from the start-up state gives the first call's bytes
    win, lastd = reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_call(solver, w, d, win, lastd, torch, dev, st)
    for k, v in w0.items():
        win[k].copy_(torch.from_numpy(v))
    lastd.zero_()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    rep = _host(o)
    for k in rep:
        assert rep[k].tobytes() == outs[0][k].tobytes(), k


def test_refusals(solver, built_lib):
    ps = replans(4, 800)
    w = workload(ps)
    solver.replan_pairs_hr(w)                                 # accepted as it stands
    L = capi.lib()
    last = np.zeros(4)

    def structs(host=True):
        a = capi.PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = 4, 10, 10, w["DC"], w["r_fraction"]
        for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
            setattr(a, k, w[k].ctypes.data)
        a.n_fac_whole = a.n_fac_safe = len(FAC)
        a.results = structs.res.ctypes.data
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        s = capi.assign_args(0, {}) if host else capi.assign_args(0, {}, 3, 4, 1 << 16, 1 << 16)
        dc = capi.decomp_args(lambda k: w[k].ctypes.data, {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"],
                              *((0, 0) if host else (8000, 8000)))
        hr = capi.hr_args(w["unk_ofs"].ctypes.data, w["unk"].ctypes.data, dict(last_factor_safe=last.ctypes.data))
        return a, s, dc, hr
    structs.res = np.zeros(4, capi.PAIR_RESULT_DTYPE)
    B = C.byref

    def call(mut=None, assign=True, decomp=True, hr_=True, win=None, host=True):
        a, s, dc, hr = structs(host)
        if mut:
            mut(a, dc, hr)
        args = (B(a), B(s) if assign else None, B(win) if win is not None else None, None, B(dc) if decomp else None,
                B(hr) if hr_ else None)
        return L.fq_replan_pairs_hr(solver._h, *args) if host else L.fq_replan_pairs_hr_dev(solver._h, *args, None, None)

    assert call() == 0
    for host in (True, False):
        assert call(hr_=False, host=host) == -1
        assert call(decomp=False, host=host) == -1
        assert call(assign=False, host=host) == -1
        for k, v in (("drone_radius", np.nan), ("drone_radius", -0.1), ("delta_a", 0.0), ("delta_a", np.inf), ("delta_H", 1.5),
                     ("delta_H", -0.1), ("delta_H", np.nan)):
            assert call(lambda a, dc, hr, k=k, v=v: setattr(hr, k, v), host=host) == -1, (k, v)
        wins = {k: np.ones(4) * (1.0 if k.startswith("init") else 10.0) for k in capi.WINDOW_IN_KEYS}
        wa = capi.window_args(lambda k: wins[k].ctypes.data, {}, 1.0, 20.0, *((0, 0) if host else (64, 64)))
        assert call(lambda a, dc, hr: setattr(hr, "last_factor_safe", None), win=wa, host=host) == -1
    bad = w["unk"].copy()
    bad[2, 1] = np.inf
    assert call(lambda a, dc, hr: setattr(hr, "unk", bad.ctypes.data)) == -1
    ofs = w["unk_ofs"].copy()
    ofs[2] = ofs[3] + 1
    assert call(lambda a, dc, hr: setattr(hr, "unk_ofs", ofs.ctypes.data)) == -1
    assert L.fq_replan_pairs_hr(None, None, None, None, None, None, None) == -1
    assert L.fq_replan_pairs_hr_dev(None, None, None, None, None, None, None, None, None) == -1
    assert call() == 0                                        # the context still works
    assert capi.has_feature("replan_pairs_hr")
    # exactly sized _dev outputs with sentinel tails: nothing is written past them
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    d = _dev_state(w, torch, dev)
    ih = torch.full((4 + 8,), -7, dtype=torch.int32, device=dev)
    ns = torch.full((4 + 8,), 7, dtype=torch.uint8, device=dev)
    lf = torch.full((4 + 8,), 3.25, dtype=torch.float64, device=dev)
    res = torch.zeros(4 * 144 + 64, dtype=torch.uint8, device=dev)
    res[4 * 144:] = 0xAB
    a, s, dc, _ = structs(False)
    for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
        setattr(a, k, torch.from_numpy(np.ascontiguousarray(w[k])).to(dev).data_ptr() if k.startswith("factors") else d[k].data_ptr())
    keep = [torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in ("factors_whole", "factors_safe")]
    a.factors_whole, a.factors_safe = keep[0].data_ptr(), keep[1].data_ptr()
    a.results = res.data_ptr()
    dc = capi.decomp_args(lambda k: d[k].data_ptr(), {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"], 8000, 8000)
    hr = capi.hr_args(d["unk_ofs"].data_ptr(), d["unk"].data_ptr(), dict(last_factor_safe=lf.data_ptr(), index_H=ih.data_ptr(),
                      need_safe=ns.data_ptr()))
    wins = {k: np.ones(4) * (1.0 if k.startswith("init") else 10.0) for k in capi.WINDOW_IN_KEYS}
    wd = {k: torch.from_numpy(v).to(dev) for k, v in wins.items()}
    a.factors_whole = a.factors_safe = None
    a.n_fac_whole = a.n_fac_safe = 0
    wa = capi.window_args(lambda k: wd[k].data_ptr(), {}, 1.0, 20.0, 64, 64)
    solver.replan_pairs_hr_dev(a, s, wa, None, dc, hr)
    torch.cuda.synchronize()
    assert (ih[4:] == -7).all() and (ns[4:] == 7).all() and (lf[4:] == 3.25).all() and (res[4 * 144:] == 0xAB).all()
    host = solver.replan_pairs_hr(w, last_factor_safe=np.full(4, 3.25), windows=wins)
    assert ih[:4].cpu().numpy().tobytes() == host["index_H"].tobytes() and ns[:4].cpu().numpy().tobytes() == host["need_safe"].tobytes()
    assert lf[:4].cpu().numpy().tobytes() == host["last_factor_safe"].tobytes()
    assert res[:4 * 144].cpu().numpy().tobytes() == host["results"].tobytes()
    # the host entries refuse multi-GPU group contexts
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        a, s, dc, hr = structs()
        assert L.fq_replan_pairs_hr(g._h, B(a), B(s), None, None, B(dc), B(hr)) == -1
        assert L.fq_replan_pairs_hr_async(g._h, B(a), B(s), None, None, B(dc), B(hr)) == -1
    finally:
        g.close()
