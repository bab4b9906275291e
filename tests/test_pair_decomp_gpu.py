"""Chained replan that decomposes its own corridors on the device (fq_replan_pairs_decomp*), on mixed forest corridors
(corridor.forest_pair_paths): the device's corridors against fq_ellipsoid_decomp on the same paths (the safe path from the
device's R), the records against _assign / _window / _exact run on those host-built corridors, the goal rule, isolation of
a failed corridor, consecutive device replans with carried windows, CUDA-graph capture, determinism and the refusals."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

pytestmark = pytest.mark.gpu
UAV = cr.UAV
FAC = np.arange(1.0, 11.0)
_PATHS = {}


def paths(n, start=0):
    key = (n, start)
    if key not in _PATHS:
        _PATHS[key] = [cr.forest_pair_paths(20000 + start + k) for k in range(n)]
    return _PATHS[key]


def workload(ps):
    w = capi.make_decomp_workload(ps)
    w["factors_whole"], w["factors_safe"] = FAC.copy(), FAC.copy()
    return w


def host_rows(path, obs):
    polys = capi.ellipsoid_decomp(path, obs, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"], cap_rows=8192)
    return polys, np.vstack([np.hstack([A, b[:, None]]) for A, b in polys])


def final_pos(polys, path, goal):
    A, b = polys[-1]
    return goal.copy() if not np.any(A @ goal - b > 0) else path[-1].copy()


def same_polytopes(dev, host, fo_dev, fo_host, path, obs):
    """Identical face counts, and rows within 1e-12 in order.  The one exception is a tie: the device's atan2/sin/cos (a few
    ulp off glibc's) can reverse two obstacle points whose distances to the final ellipsoid differ by at most 1e-12 on the
    host.  For such a polytope the first row that differs must be an obstacle face cut at exactly such a point: on the host,
    at that carving round, the point on the device's row is within 1e-12 of the host's pick.  The faces then still agree as a
    set (to 1e-11: what follows is cut in another order), and the bbox and ground rows (the last 7) in order to 1e-12.
    -> number of polytopes with such a tie."""
    from test_pair_decomp_cpu import host_round
    ties = 0
    assert np.array_equal(np.diff(fo_dev), np.diff(fo_host))
    for k in range(len(fo_host) - 1):
        a, b = dev[fo_dev[k]:fo_dev[k + 1]], host[fo_host[k]:fo_host[k + 1]]
        if np.abs(a - b).max() <= 1e-12:
            continue
        i = int(np.flatnonzero(np.abs(a - b).max(axis=1) > 1e-12)[0])
        assert i < len(a) - 7, (k, i)
        best, on_row, res = host_round(path[k], path[k + 1], obs, UAV["drone_radius"], i, a[i])
        assert res <= 1e-9 and abs(on_row - best) <= 1e-12, (k, i, best, on_row, res)
        ties += 1
        assert np.abs(a[-7:] - b[-7:]).max() <= 1e-12
        sa, sb = a[:-7][np.lexsort(np.round(a[:-7], 9).T[::-1])], b[:-7][np.lexsort(np.round(b[:-7], 9).T[::-1])]
        assert np.abs(sa - sb).max() <= 1e-11
    return ties


def host_built(ps, out, w):
    """The corridors the host makes from the same paths (the safe path from the device's R), checked against the device's
    rows of each corridor: -> (whole list, safe list, bit-equal flags)."""
    whole, safe, same = [], [], []
    for j, p in enumerate(ps):
        pw, rw = host_rows(p["path_whole"], p["obs"])
        sp = p["path_safe"].copy()
        sp[0] = out["results"]["R"][j][:3]
        psf, rs = host_rows(sp, p["obs"])
        E, M = final_pos(pw, p["path_whole"], p["goal"]), final_pos(psf, sp, p["goal"])
        xfw, xfs = np.zeros(9), np.zeros(9)
        xfw[:3], xfs[:3] = E, M
        whole.append(dict(N=p["N"], x0=p["x0"], xf=xfw, lim=p["lim"], polys=pw))
        safe.append(dict(N=p["N"], x0=p["x0"], xf=xfs, lim=p["lim"], polys=psf))
        ok = True
        for kind, rows, pos, path in (("whole", rw, E, p["path_whole"]), ("safe", rs, M, sp)):
            fo, po = out["face_ofs_" + kind], w["poly_ofs_" + kind]
            dev = out["Ab_" + kind][fo[po[j]]:fo[po[j + 1]]]
            polys = pw if kind == "whole" else psf
            fo_host = np.concatenate([[0], np.cumsum([len(b) for _, b in polys])])
            same_polytopes(dev, rows, fo[po[j]:po[j + 1] + 1] - fo[po[j]], fo_host, path, p["obs"])
            ok = ok and dev.tobytes() == rows.tobytes()
            assert np.array_equal(out["E" if kind == "whole" else "M"][j], pos), (kind, j)
        same.append(ok)
    return whole, safe, same


def compare_records(a, b, same):
    ra, rb = a["results"], b["results"]
    for k in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(ra[k], rb[k]), k
    for k in ("whole_cost", "safe_cost", "whole_dt", "safe_dt", "R"):
        x, y = ra[k], rb[k]
        fin = np.isfinite(y)
        assert np.array_equal(np.isfinite(x), fin), k
        assert np.all(np.abs(x[fin] - y[fin]) <= 1e-12 * np.maximum(np.abs(y[fin]), 1.0)), k
    for j, s in enumerate(same):
        if s:
            assert ra[j:j + 1].tobytes() == rb[j:j + 1].tobytes(), j


def test_corridors_and_records_match_the_host_built_chain(solver):
    ps = paths(128)
    w = workload(ps)
    out = solver.replan_pairs_decomp(w)
    assert not out["status_whole"].any() and not out["status_safe"].any()
    whole, safe, same = host_built(ps, out, w)
    hw = capi.make_pair_workload(whole, safe, FAC, np.zeros((1, 10)), FAC, np.zeros((1, 10)), DC=w["DC"], r_fraction=w["r_fraction"])
    ref = solver.replan_pairs_assign(hw, want_candidates=False)
    compare_records(out, ref, same)
    assert (out["results"]["safe_dt_index"] >= 0).sum() > 64
    assert sum(same) > 0           # most corridors differ in the last bits (atan2 / sin / cos), their records within 1e-12


@pytest.mark.parametrize("mode", ["window", "exact"])
def test_window_and_exact_modes_match(solver, mode):
    ps = paths(32, 500)
    w = workload(ps)
    rng = np.random.default_rng(1)
    wins = None
    if mode == "window":
        wins = dict(init_whole=rng.integers(1, 4, 32).astype(float), final_whole=rng.integers(6, 12, 32).astype(float),
                    init_safe=rng.integers(1, 4, 32).astype(float), final_safe=rng.integers(6, 12, 32).astype(float))
    out = solver.replan_pairs_decomp(w, windows=wins, exact=mode == "exact")
    whole, safe, same = host_built(ps, out, w)
    hw = capi.make_pair_workload(whole, safe, FAC, np.zeros((1, 10)), FAC, np.zeros((1, 10)), DC=w["DC"], r_fraction=w["r_fraction"])
    ref = solver.replan_pairs_window(hw, wins, want_candidates=False) if mode == "window" else \
        solver.replan_pairs_exact(hw, want_candidates=False)
    compare_records(out, ref, same)
    keys = capi.WINDOW_OUT_KEYS if mode == "window" else capi.EXACT_KEYS
    for k in keys:
        assert out[k].tobytes() == ref[k].tobytes(), k


def test_goal_inside_and_outside(solver):
    ps = paths(32, 1000)
    w = workload(ps)
    out = solver.replan_pairs_decomp(w)
    far = solver.replan_pairs_decomp(w, use_goal=False)
    n_in = 0
    for j, p in enumerate(ps):
        pw, _ = host_rows(p["path_whole"], p["obs"])
        inside = not np.any(pw[-1][0] @ p["goal"] - pw[-1][1] > 0)
        n_in += inside
        assert np.array_equal(out["E"][j], p["goal"] if inside else p["path_whole"][-1])
        assert np.array_equal(far["E"][j], p["path_whole"][-1])
    assert 0 < n_in < len(ps)


def test_a_failed_corridor_leaves_the_others_byte_identical(solver):
    ps = [dict(p) for p in paths(16, 2000)]
    w0 = workload(ps)
    base = solver.replan_pairs_decomp(w0)
    bad = dict(ps[5])
    bad["path_whole"] = np.vstack([bad["path_whole"][:1], bad["path_whole"]])      # a zero-length first segment
    ps[5] = bad
    w = workload(ps)
    out = solver.replan_pairs_decomp(w)
    assert out["status_whole"][5] == capi.DECOMP_STATUS["zero_segment"] and out["status_safe"][5] == capi.DECOMP_STATUS["not_run"]
    r = out["results"][5]
    assert r["whole_dt_index"] == -1 and r["safe_dt_index"] == -1 and np.isnan(out["E"][5]).all()
    for j in range(16):
        if j != 5:
            assert out["results"][j:j + 1].tobytes() == base["results"][j:j + 1].tobytes(), j
    # a polytope cap below what a corridor needs fails that corridor only
    w0["max_poly_faces_whole"] = int(np.diff(base["face_ofs_whole"]).max()) - 1
    capped = solver.replan_pairs_decomp(w0)
    failed = capped["status_whole"] != 0
    assert failed.any() and not failed.all()
    for j in np.flatnonzero(~failed):
        assert capped["results"][j:j + 1].tobytes() == base["results"][j:j + 1].tobytes(), j


def _dev_call(solver, w, d, win_dev, torch, dev, stream):
    n = w["n_prob"]
    out = dict(results=torch.zeros(n * 144, dtype=torch.uint8, device=dev),
               coeffs_whole=torch.zeros(n * w["N_whole"] * 12, dtype=torch.float64, device=dev),
               coeffs_safe=torch.zeros(n * w["N_safe"] * 12, dtype=torch.float64, device=dev))
    dout = dict(face_ofs_whole=torch.zeros(n * 3 + 1, dtype=torch.int32, device=dev), face_ofs_safe=torch.zeros(n * 4 + 1, dtype=torch.int32, device=dev),
                Ab_whole=torch.zeros(n * w["max_faces_whole"] * 4, dtype=torch.float64, device=dev),
                Ab_safe=torch.zeros(n * w["max_faces_safe"] * 4, dtype=torch.float64, device=dev),
                E=torch.zeros(n * 3, dtype=torch.float64, device=dev), M=torch.zeros(n * 3, dtype=torch.float64, device=dev),
                status_whole=torch.full((n,), -1, dtype=torch.int32, device=dev), status_safe=torch.full((n,), -1, dtype=torch.int32, device=dev))
    a = capi.PairArgs()
    a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, w["N_whole"], w["N_safe"], w["DC"], w["r_fraction"]
    for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe"):
        setattr(a, k, d[k].data_ptr())
    for k, v in out.items():
        setattr(a, k, v.data_ptr())
    for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
        setattr(a, k, int(w[k]))
    s = capi.assign_args(0, {}, 3, 4, 1 << 16, 1 << 16)
    wa = capi.window_args(lambda k: win_dev[k].data_ptr(), {"next_" + k: win_dev[k].data_ptr() for k in capi.WINDOW_IN_KEYS}, 1.0, 20.0,
                          64, 64)
    mo = int(np.diff(w["obs_ofs_whole"]).max())
    dc = capi.decomp_args(lambda k: d[k].data_ptr(), {k: v.data_ptr() for k, v in dout.items()}, UAV["bbox"], UAV["drone_radius"],
                          UAV["z_ground"], mo, mo)
    solver.replan_pairs_decomp_dev(a, s, wa, None, dc, 0, stream.cuda_stream)
    out.update(dout)
    return out


def _host(o):
    h = {k: v.cpu().numpy() for k, v in o.items()}
    h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
    return h


def test_device_entry_carries_windows_is_deterministic_and_captures(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = paths(32, 3000)
    w = workload(ps)
    w0 = dict(init_whole=np.ones(32), final_whole=np.full(32, 10.0), init_safe=np.ones(32), final_safe=np.full(32, 10.0))
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in
         ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe") + tuple(capi.DECOMP_IN_KEYS)}
    win_dev = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
    st = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize()
    outs = []
    for _ in range(3):
        o = _dev_call(solver, w, d, win_dev, torch, dev, st)
        st.synchronize()
        outs.append(_host(o))
    # the same three replans through the host entry, windows carried on the host
    wins = {k: v.copy() for k, v in w0.items()}
    for o in outs:
        ref = solver.replan_pairs_decomp(w, windows=wins)
        assert o["results"].tobytes() == ref["results"].tobytes()
        wins = {k: ref["next_" + k].copy() for k in capi.WINDOW_IN_KEYS}
    # two runs from the same windows give the same bytes, and so does a replay of a captured graph
    for k, v in w0.items():
        win_dev[k].copy_(torch.from_numpy(v))
    o = _dev_call(solver, w, d, win_dev, torch, dev, st)
    st.synchronize()
    first = _host(o)
    for k, v in w0.items():
        win_dev[k].copy_(torch.from_numpy(v))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_call(solver, w, d, win_dev, torch, dev, st)
    for k, v in w0.items():
        win_dev[k].copy_(torch.from_numpy(v))
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    replay = _host(o)
    for k in first:
        assert first[k].tobytes() == replay[k].tobytes(), k
    assert first["results"].tobytes() == outs[0]["results"].tobytes()


def test_refusals(solver, built_lib):
    ps = paths(4, 4000)
    w = workload(ps)
    solver.replan_pairs_decomp(w)                             # accepted as it stands
    L = capi.lib()

    def call(mut_a=None, mut_dc=None, assign=True):
        out = dict(results=np.zeros(4, capi.PAIR_RESULT_DTYPE))
        a = capi.PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = 4, 10, 10, w["DC"], w["r_fraction"]
        for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
            setattr(a, k, w[k].ctypes.data)
        a.n_fac_whole = a.n_fac_safe = len(FAC)
        a.results = out["results"].ctypes.data
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        s = capi.assign_args(0, {})
        dc = capi.decomp_args(lambda k: w[k].ctypes.data, {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"])
        if mut_a:
            mut_a(a)
        if mut_dc:
            mut_dc(dc)
        return L.fq_replan_pairs_decomp(solver._h, C.byref(a), C.byref(s) if assign else None, None, None, C.byref(dc))

    assert call() == 0
    dummy = np.zeros(64)
    for k in ("face_ofs_whole", "face_ofs_safe", "Ab_whole", "Ab_safe", "xf_whole", "xf_safe"):
        assert call(mut_a=lambda a, k=k: setattr(a, k, dummy.ctypes.data)) == -1, k
    assert call(mut_a=lambda a: setattr(a, "max_poly_faces_safe", 0)) == -1
    assert call(assign=False) == -1
    assert L.fq_replan_pairs_decomp(solver._h, None, None, None, None, None) == -1
    assert call(mut_dc=lambda dc: setattr(dc, "path_safe", None)) == -1
    assert call(mut_dc=lambda dc: setattr(dc, "inflate", -0.1)) == -1
    assert call(mut_dc=lambda dc: dc.bbox.__setitem__(1, 0.0)) == -1
    bad = w["obs_whole"].copy()
    bad[3, 1] = np.nan
    assert call(mut_dc=lambda dc: setattr(dc, "obs_whole", bad.ctypes.data)) == -1
    assert call(mut_dc=lambda dc: setattr(dc, "Ab_whole", dummy.ctypes.data + 8)) == -1
    # the device entry refuses before it touches a pointer, so host arrays stand in for device ones here
    def call_dev(mut_a=None, mut_dc=None, decomp=True):
        a = capi.PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = 4, 10, 10, w["DC"], w["r_fraction"]
        for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
            setattr(a, k, w[k].ctypes.data)
        a.n_fac_whole = a.n_fac_safe = len(FAC)
        a.results = dummy.ctypes.data
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        s = capi.assign_args(0, {}, 3, 4, 1 << 16, 1 << 16)
        dc = capi.decomp_args(lambda k: w[k].ctypes.data, {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"], 8000, 8000)
        if mut_a:
            mut_a(a)
        if mut_dc:
            mut_dc(dc)
        return L.fq_replan_pairs_decomp_dev(solver._h, C.byref(a), C.byref(s), None, None, C.byref(dc) if decomp else None, None, None)

    assert L.fq_replan_pairs_decomp_dev(None, None, None, None, None, None, None, None) == -1
    assert call_dev(decomp=False) == -1
    assert call_dev(mut_dc=lambda dc: setattr(dc, "max_obs_whole", -1)) == -1
    assert call_dev(mut_dc=lambda dc: setattr(dc, "max_obs_safe", -1)) == -1
    for k in ("face_ofs_whole", "face_ofs_safe", "Ab_whole", "Ab_safe", "xf_whole", "xf_safe"):
        assert call_dev(mut_a=lambda a, k=k: setattr(a, k, dummy.ctypes.data)) == -1, k
    assert call() == 0                                        # the context still works
    assert capi.has_feature("replan_pairs_decomp")
    # the host entries refuse multi-GPU group contexts (a group of one GPU is still a group)
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        out = dict(results=np.zeros(4, capi.PAIR_RESULT_DTYPE))
        a = capi.PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = 4, 10, 10, w["DC"], w["r_fraction"]
        for k in ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "factors_whole", "factors_safe"):
            setattr(a, k, w[k].ctypes.data)
        a.n_fac_whole = a.n_fac_safe = len(FAC)
        a.results = out["results"].ctypes.data
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        s = capi.assign_args(0, {})
        dc = capi.decomp_args(lambda k: w[k].ctypes.data, {}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"])
        assert L.fq_replan_pairs_decomp(g._h, C.byref(a), C.byref(s), None, None, C.byref(dc)) == -1
        assert L.fq_replan_pairs_decomp_async(g._h, C.byref(a), C.byref(s), None, None, C.byref(dc)) == -1
    finally:
        g.close()
