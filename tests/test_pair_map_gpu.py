"""Chained replan against indexed maps (fq_map_*, fq_replan_pairs_map*) on forest corridors with seeded unknown clouds: every
output byte for byte that of fq_replan_pairs_hr (or _decomp without hr) fed corridor j's map as obs_whole_j = O, obs_safe_j =
U ++ O and unk_j = U, with one map per corridor and with one map shared by corridors planned in the same forest; a mapper-sized
map; a map update between calls; a closed loop of _map_dev calls with CUDA-graph capture; the max_local cap; the refusals."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_hr_oracle as hro
from test_pair_hr_gpu import FAC, UAV, _host, replans, workload

pytestmark = pytest.mark.gpu


def _csr(clouds):
    ofs = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    return ofs, np.ascontiguousarray(np.vstack([np.reshape(c, (-1, 3)) for c in clouds] + [np.zeros((1, 3))]), np.float64)


def cloud_workload(w, occs, unks):
    """`w` with corridor j's clouds as the map chain reads them: whole O_j, safe U_j ++ O_j, unknown U_j."""
    r = dict(w)
    r["obs_ofs_whole"], r["obs_whole"] = _csr(occs)
    r["obs_ofs_safe"], r["obs_safe"] = _csr([np.vstack([np.reshape(u, (-1, 3)), np.reshape(o, (-1, 3))]) for u, o in zip(unks, occs)])
    r["unk_ofs"], r["unk"] = _csr(unks)
    return r


def same_forest(forest_seed, k, start=0):
    """k replans (corridor.forest_pair_paths dicts with "unk") in the forest of `forest_seed`, each with its own start and
    goal: the query seeds differ, the trees do not."""
    orig = cr.make_forest
    cr.make_forest = lambda seed, n_trees=60: orig(forest_seed, n_trees=n_trees)
    try:
        ps = []
        for s in range(start, start + 400):
            try:
                p = cr.forest_pair_paths(forest_seed * 1000 + s)
            except RuntimeError:
                continue
            p["unk"] = cr.forest_unknown_cloud(p)
            ps.append(p)
            if len(ps) == k:
                return ps
    finally:
        cr.make_forest = orig
    raise RuntimeError("not enough replans")


def assert_same(a, b, kinds=("whole", "safe")):
    """Every output of two chain calls byte for byte; of Ab_* only the rows face_ofs_* fills (the rest is undefined)."""
    assert sorted(a) == sorted(b)
    for k in a:
        if k.startswith("Ab_"):
            n = int(a["face_ofs_" + k[3:]][-1])
            assert a[k][:n].tobytes() == b[k][:n].tobytes(), k
        else:
            assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def make_maps(occs, unks):
    maps = []
    for o, u in zip(occs, unks):
        m = capi.Map()
        m.update(o, u)
        maps.append(m)
    return maps


@pytest.mark.parametrize("windows", [False, True])
@pytest.mark.parametrize("exact", [False, True])
def test_one_map_per_corridor_equals_hr_and_decomp(solver, windows, exact):
    ps = replans(16, 800)
    w = workload(ps)
    n = len(ps)
    occs, unks = [p["obs"] for p in ps], [p["unk"] for p in ps]
    maps = make_maps(occs, unks)
    rng = np.random.default_rng(2)
    wins = None
    if windows:
        wins = dict(init_whole=rng.integers(1, 4, n).astype(float), final_whole=rng.integers(6, 12, n).astype(float),
                    init_safe=rng.integers(1, 4, n).astype(float), final_safe=rng.integers(6, 12, n).astype(float))
    last = rng.uniform(1.0, 8.0, n)
    ref_w = cloud_workload(w, occs, unks)
    kw = dict(windows=wins, exact=exact, want_candidates=True)
    ml = max(len(u) + len(o) for u, o in zip(unks, occs))          # no segment can be above the cap: the contract holds
    got = solver.replan_pairs_map(w, maps, np.arange(n), max_local=ml, last_factor_safe=last, **kw)
    ref = solver.replan_pairs_hr(ref_w, last_factor_safe=last, **kw)
    assert_same(got, ref)
    assert 0 < got["need_safe"].sum() < n
    got = solver.replan_pairs_map(w, maps, np.arange(n), max_local=ml, hr=False, **kw)
    ref = solver.replan_pairs_decomp(ref_w, **kw)
    assert_same(got, ref)


def test_shared_map_in_one_forest_equals_hr(solver):
    ps = same_forest(7, 12)
    w = workload(ps)
    occ = ps[0]["obs"]
    assert all(np.array_equal(p["obs"], occ) for p in ps)
    unk = np.vstack([p["unk"] for p in ps[:4]])
    m = capi.Map()
    m.update(occ, unk)
    assert m.size() == (len(occ), len(unk))
    n = len(ps)
    ref_w = cloud_workload(w, [occ] * n, [unk] * n)
    for hr in (True, False):
        got = solver.replan_pairs_map(w, [m], None, max_local=1 << 15, hr=hr)
        ref = (solver.replan_pairs_hr if hr else solver.replan_pairs_decomp)(ref_w)
        assert_same(got, ref)
    # two maps shared by alternate corridors
    m2 = capi.Map()
    m2.update(occ, ps[5]["unk"])
    idx = np.arange(n) % 2
    got = solver.replan_pairs_map(w, [m, m2], idx, max_local=1 << 15)
    ref = solver.replan_pairs_hr(cloud_workload(w, [occ] * n, [[unk, ps[5]["unk"]][i] for i in idx]))
    assert_same(got, ref)


def mapper_cloud(p):
    """Every free cell of the forest grid (16 x 16 x 3 m at 0.15 m): what a mapper that has seen nothing would publish."""
    _, centres, radii = cr.make_forest(p["seed"] // 1000, n_trees=60)
    grid, origin, res = cr.voxelise_forest(centres, radii)
    free = np.argwhere(grid == 0)[:, ::-1]
    return np.ascontiguousarray((free + 0.5) * res + origin)


def test_mapper_sized_shared_map(solver):
    ps = same_forest(11, 64)
    w = workload(ps)
    occ, unk = ps[0]["obs"], mapper_cloud(ps[0])
    assert len(unk) + len(occ) >= 100000
    m = capi.Map()
    m.update(occ, unk)
    got = solver.replan_pairs_map(w, [m], None, max_local=1 << 15)     # about 300 MB of spill, whatever the map's size
    res = got["results"]
    assert (got["status_whole"] == 0).all() and (got["status_safe"] != capi.DECOMP_STATUS["cloud"]).all()
    # records against the CPU chain on a subset
    for j in range(0, 64, 16):
        p = dict(ps[j], unk=unk, obs=occ)
        ref = hro.replan_pair_hr(dict(p, obs=occ), FAC, dt_base_whole=res["whole_dt_base"][j], dt_base_safe=res["safe_dt_base"][j])
        for k in ("whole_dt_index", "whole_sigma_index", "n_samples_whole"):
            assert ref[k] == res[k][j], (k, j)
        assert ref["need_safe"] == got["need_safe"][j] and ref["index_H"] == got["index_H"][j], j
    # a few corridors byte for byte against _hr fed the same clouds
    sub = [0, 1, 2]
    ws = workload([ps[j] for j in sub])
    assert_same(solver.replan_pairs_map(ws, [m], None, max_local=1 << 15),
                solver.replan_pairs_hr(cloud_workload(ws, [occ] * 3, [unk] * 3)))


def test_update_between_calls(solver):
    ps = replans(8, 900)
    w = workload(ps)
    occ, unk = ps[0]["obs"], ps[0]["unk"]
    m = capi.Map()
    m.update(occ, unk)
    first = solver.replan_pairs_map(w, [m], None, max_local=1 << 15)
    unk2 = np.vstack([p["unk"] for p in ps])
    m.update(occ[::2], unk2)
    second = solver.replan_pairs_map(w, [m], None, max_local=1 << 15)
    assert_same(second, solver.replan_pairs_hr(cloud_workload(w, [occ[::2]] * 8, [unk2] * 8)))
    assert first["results"].tobytes() != second["results"].tobytes()
    m.update(occ, np.zeros((0, 3)))                               # an empty U: no safe path needed, the safe cloud is O
    third = solver.replan_pairs_map(w, [m], None, max_local=1 << 15)
    assert_same(third, solver.replan_pairs_hr(cloud_workload(w, [occ] * 8, [np.zeros((0, 3))] * 8)))
    assert not third["need_safe"].any()


def test_max_local_overflow_refuses_one_segment(solver):
    ps = replans(8, 900)
    w = workload(ps)
    occ = ps[0]["obs"]
    rng = np.random.default_rng(3)
    p = ps[0]["path_whole"]
    dense = p[0] + rng.uniform(-1.0, 1.0, (3000, 3)) * [1.5, 1.5, 0.8]     # thousands of points in corridor 0's first box
    dense = dense[np.linalg.norm(dense - p[0], axis=1) > 0.6]
    maps = make_maps([occ, np.vstack([occ, dense])], [np.zeros((0, 3))] * 2)
    idx = np.zeros(8, np.int32)
    idx[0] = 1
    got = solver.replan_pairs_map(w, maps, idx, max_local=1500, hr=False)
    assert got["status_whole"][0] == capi.DECOMP_STATUS["cloud"] and got["results"]["whole_dt_index"][0] == -1
    ref = solver.replan_pairs_map(w, maps, np.zeros(8, np.int32), max_local=1500, hr=False)
    assert got["results"][1:].tobytes() == ref["results"][1:].tobytes()


def _dev_call(solver, w, d, win_dev, last_dev, mp, torch, dev, stream):
    n = w["n_prob"]
    out = dict(results=torch.zeros(n * 144, dtype=torch.uint8, device=dev),
               index_H=torch.full((n,), -7, dtype=torch.int32, device=dev), need_safe=torch.full((n,), 7, dtype=torch.uint8, device=dev),
               status_whole=torch.full((n,), -1, dtype=torch.int32, device=dev), status_safe=torch.full((n,), -1, dtype=torch.int32, device=dev))
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
    dc = capi.decomp_args(lambda k: None if k.startswith("obs_") else d[k].data_ptr(),
                          {k: out[k].data_ptr() for k in ("status_whole", "status_safe")}, UAV["bbox"], UAV["drone_radius"], UAV["z_ground"])
    hr = capi.hr_args(None, None, dict(last_factor_safe=last_dev.data_ptr(), index_H=out["index_H"].data_ptr(),
                                       need_safe=out["need_safe"].data_ptr()))
    solver.replan_pairs_map_dev(a, s, wa, None, dc, hr, mp, 0, stream.cuda_stream)
    return out


def test_closed_loop_on_the_device_is_deterministic_and_captures(solver):
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = replans(16, 600)
    w = workload(ps)
    n = w["n_prob"]
    maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
    d_idx = torch.arange(n, dtype=torch.int32, device=dev)
    mp = capi.map_args(maps, d_idx.data_ptr(), max(len(p["obs"]) + len(p["unk"]) for p in ps))
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in
         ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "path_whole", "path_safe", "goal")}
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 10.0), init_safe=np.ones(n), final_safe=np.full(n, 10.0))
    st = torch.cuda.Stream(device=dev)

    def reset():
        return {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}, torch.zeros(n, dtype=torch.float64, device=dev)

    def loop():
        win, last = reset()
        torch.cuda.synchronize()
        outs = []
        for _ in range(6):
            o = _dev_call(solver, w, d, win, last, mp, torch, dev, st)
            st.synchronize()
            h = _host(o)
            h.update({k: v.cpu().numpy() for k, v in win.items()}, last=last.cpu().numpy())
            outs.append(h)
        return outs

    outs = loop()
    wins, last = {k: v.copy() for k, v in w0.items()}, np.zeros(n)
    ref_w = cloud_workload(w, [p["obs"] for p in ps], [p["unk"] for p in ps])
    for o in outs:
        ref = solver.replan_pairs_hr(ref_w, last_factor_safe=last, windows=wins)
        assert o["results"].tobytes() == ref["results"].tobytes()
        assert o["index_H"].tobytes() == ref["index_H"].tobytes() and o["need_safe"].tobytes() == ref["need_safe"].tobytes()
        wins = {k: ref["next_" + k].copy() for k in capi.WINDOW_IN_KEYS}
        last = ref["last_factor_safe"].copy()
        for k in capi.WINDOW_IN_KEYS:
            assert o[k].tobytes() == wins[k].tobytes(), k
    again = loop()
    for a, b in zip(outs, again):
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
    win, lastd = reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_call(solver, w, d, win, lastd, mp, torch, dev, st)
    for k, v in w0.items():
        win[k].copy_(torch.from_numpy(v))
    lastd.zero_()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    rep = _host(o)
    for k in rep:
        assert rep[k].tobytes() == outs[0][k].tobytes(), k


def test_a_captured_replan_reads_the_maps_last_update(solver):
    """A _map_dev call captured once and replayed after fq_map_update -- with the capacity kept, and grown -- gives what a
    fresh call on the updated maps gives, and the records of _hr on the new clouds."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = replans(16, 600)
    w = workload(ps)
    n = w["n_prob"]
    occs, unks = [p["obs"] for p in ps], [p["unk"] for p in ps]
    maps = make_maps(occs, unks)
    d_idx = torch.arange(n, dtype=torch.int32, device=dev)
    mp = capi.map_args(maps, d_idx.data_ptr(), 1 << 15)
    d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in
         ("x0", "lim", "poly_ofs_whole", "poly_ofs_safe", "path_whole", "path_safe", "goal")}
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 10.0), init_safe=np.ones(n), final_safe=np.full(n, 10.0))
    st = torch.cuda.Stream(device=dev)
    win = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
    last = torch.zeros(n, dtype=torch.float64, device=dev)

    def reset(wd, ld):
        for k, v in w0.items():
            wd[k].copy_(torch.from_numpy(v))
        ld.zero_()
        torch.cuda.synchronize()

    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        o = _dev_call(solver, w, d, win, last, mp, torch, dev, st)
    reset(win, last)
    g.replay()
    torch.cuda.synchronize()
    before = _host(o)
    grown = [np.vstack([occs[j]] + [occs[(j + k) % n] for k in range(1, 4)]) for j in range(n)]
    for name, new_occ, new_unk in (("kept", [x[::2] for x in occs], [x[::3] for x in unks]), ("grown", grown, unks)):
        if name == "grown":
            assert all(len(a) + len(b) > 1.25 * (len(c) + len(e)) + 1024 for a, b, c, e in zip(new_occ, new_unk, occs, unks))
        for m, a, b in zip(maps, new_occ, new_unk):
            m.update(a, b)
        reset(win, last)
        g.replay()
        torch.cuda.synchronize()
        replayed = _host(o)
        fw, fl = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}, torch.zeros(n, dtype=torch.float64, device=dev)
        fo = _dev_call(solver, w, d, fw, fl, mp, torch, dev, st)
        st.synchronize()
        fresh = _host(fo)
        for k in fresh:
            assert replayed[k].tobytes() == fresh[k].tobytes(), (name, k)
        ref = solver.replan_pairs_hr(cloud_workload(w, new_occ, new_unk), last_factor_safe=np.zeros(n), windows=w0)
        assert replayed["results"].tobytes() == ref["results"].tobytes(), name
        assert replayed["results"].tobytes() != before["results"].tobytes(), name


def test_map_update_dev_equals_update(solver):
    torch = pytest.importorskip("torch")
    ps = replans(8, 900)
    w = workload(ps)
    occ, unk = ps[0]["obs"], ps[0]["unk"]
    m1, m2 = capi.Map(), capi.Map()
    m1.update(occ, unk)
    do, du = torch.from_numpy(np.ascontiguousarray(occ)).cuda(), torch.from_numpy(np.ascontiguousarray(unk)).cuda()
    m2.update_dev(do.data_ptr(), len(occ), du.data_ptr(), len(unk), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert_same(solver.replan_pairs_map(w, [m2], None), solver.replan_pairs_map(w, [m1], None))


def test_refusals(solver, built_lib):
    L = capi.lib()
    ps = replans(4, 900)
    w = workload(ps)
    m = capi.Map()
    m.update(ps[0]["obs"], ps[0]["unk"])
    FqError = capi.FqError
    for bad in ([[np.nan, 0, 0]], [[np.inf, 1, 2]]):
        with pytest.raises(FqError, match="non-finite"):
            m.update(np.array(bad, float), np.zeros((0, 3)))
    err = lambda: L.fq_last_error(None).decode()  # noqa: E731
    buf = np.zeros((5, 3))
    assert L.fq_map_update(m.handle, None, -1, None, 0) == -1 and "negative" in err()
    assert L.fq_map_update_dev(m.handle, None, 0, None, -3, None) == -1 and "negative" in err()
    # more than 2^30 points in all (refused before any point is read)
    assert L.fq_map_update(m.handle, buf.ctypes.data, 1 << 30, buf.ctypes.data, 1) == -1 and "2^30" in err()
    assert L.fq_map_update_dev(m.handle, buf.ctypes.data, 1 << 29, buf.ctypes.data, (1 << 29) + 1, None) == -1 and "2^30" in err()
    # a NULL cloud with a positive count
    assert L.fq_map_update(m.handle, None, 3, None, 0) == -1 and "NULL cloud" in err()
    assert L.fq_map_update(m.handle, buf.ctypes.data, 1, None, 2) == -1 and "NULL cloud" in err()
    assert L.fq_map_update_dev(m.handle, None, 0, None, 2, None) == -1 and "NULL cloud" in err()
    # one array passed as both clouds: U's points beyond O's count are checked too
    buf[4, 2] = np.nan
    assert L.fq_map_update(m.handle, buf.ctypes.data, 1, buf.ctypes.data, 5) == -1 and "non-finite" in err()
    buf[4, 2] = 0.0
    assert L.fq_map_update(m.handle, ps[0]["obs"].ctypes.data, len(ps[0]["obs"]), ps[0]["unk"].ctypes.data, len(ps[0]["unk"])) == 0
    with pytest.raises(FqError, match="map_index out of range"):
        solver.replan_pairs_map(w, [m], np.array([0, 1, 0, 0]))
    with pytest.raises(FqError, match="map_index out of range"):
        solver.replan_pairs_map(w, [m], np.array([0, -1, 0, 0]))
    with pytest.raises(FqError, match="max_local"):
        solver.replan_pairs_map(w, [m], None, max_local=-1)
    with pytest.raises(FqError, match="no maps"):
        solver.replan_pairs_map(w, [], None)
    # clouds given as well as a map
    out, structs = solver._decomp_structs(w, 0, None, 1.0, 20.0, False, (2.0, 2.0, 1.0), 0.42, 0.0, True, False, True,
                                          dict(last_factor_safe=np.zeros(4), index_H=np.zeros(4, np.int32), need_safe=np.zeros(4, np.uint8)))
    mp = capi.map_args([m])
    hr = capi.hr_args(None, None, {k: out[k].ctypes.data for k in capi.HR_OUT_KEYS})
    assert L.fq_replan_pairs_map(solver._h, *structs, C.byref(hr), C.byref(mp)) == -1
    assert b"obs_" in L.fq_last_error(solver._h)
    out, structs = solver._decomp_structs(w, 0, None, 1.0, 20.0, False, (2.0, 2.0, 1.0), 0.42, 0.0, True, False, True,
                                          dict(last_factor_safe=np.zeros(4), index_H=np.zeros(4, np.int32), need_safe=np.zeros(4, np.uint8)),
                                          clouds=False)
    hr_unk = capi.hr_args(w["unk_ofs"].ctypes.data, w["unk"].ctypes.data, {k: out[k].ctypes.data for k in capi.HR_OUT_KEYS})
    assert L.fq_replan_pairs_map(solver._h, *structs, C.byref(hr_unk), C.byref(mp)) == -1
    assert b"unk" in L.fq_last_error(solver._h)
    assert L.fq_replan_pairs_map(solver._h, *structs, C.byref(hr), None) == -1
    nul = capi.PairMap()
    nul.table = (C.c_void_p * 1)(None)
    nul.maps, nul.n_maps = C.addressof(nul.table), 1
    assert L.fq_replan_pairs_map(solver._h, *structs, C.byref(hr), C.byref(nul)) == -1
    assert L.fq_replan_pairs_map(solver._h, *structs, C.byref(hr), C.byref(mp)) == 0
    # multi-GPU contexts: the host entries refuse them
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        for fn in (L.fq_replan_pairs_map, L.fq_replan_pairs_map_async):
            assert fn(g._h, *structs, C.byref(hr), C.byref(mp)) == -1
            assert b"multi-GPU" in L.fq_last_error(g._h)
    finally:
        g.close()
    # a map on another device than the context
    import torch
    if torch.cuda.device_count() > 1:
        other = capi.Map(device=1)
        with pytest.raises(FqError, match="another device"):
            solver.replan_pairs_map(w, [other], None)
    assert capi.has_feature("replan_pairs_map")
