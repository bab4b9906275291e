"""fq_map_paths* on the GPU: each corridor's whole and safe paths from its JPS_in against indexed maps, byte for byte those
of the host twin fq_paths_cloud over the same unknown clouds -- one map per corridor, one mapper-sized map shared by a
batch, a scene translated by 1e4 m -- and composed with the chained replan on one stream (fq_map_paths_dev ->
fq_replan_pairs_plan_dev with _map's structs), equal to the host route; a captured graph replayed after map updates."""
import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

from test_map_paths_cpu import LINE, STALL_PATH, STALL_UNK
from test_pair_hr_gpu import UAV, _host
from test_pair_map_gpu import make_maps, mapper_cloud, same_forest

pytestmark = pytest.mark.gpu
MW, MS = 3, 4


def corridors(n, start=0):
    """n forest replans: JPS_in from the product's JPS (fq_jps_in, Ra = 4 m) and the forest_pair_paths dict of the same
    query (its x0 moved to the start, its unknown cloud in "unk")."""
    out = []
    for seed in range(40000 + start, 40000 + start + n):
        fj, p = cr.forest_jps(seed), cr.forest_pair_paths(seed)
        ra = min(np.linalg.norm(fj["goal"] - fj["start"]) - 0.001, 4.0)
        p["x0"] = p["x0"].copy()
        p["x0"][:3] = fj["start"]
        p["jin"] = capi.jps_in(fj["jps"], fj["start"], fj["goal"], ra, 1.5)
        p["unk"] = cr.forest_unknown_cloud(p)
        out.append(p)
    return out


def same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes(), k


def test_one_map_per_corridor():
    ps = corridors(128)
    maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
    jins, unks = [p["jin"] for p in ps], [p["unk"] for p in ps]
    got = capi.map_paths(jins, maps, np.arange(len(ps)), max_poly_whole=MW, max_poly_safe=MS)
    same(got, capi.paths_cloud(jins, unks, max_poly_whole=MW, max_poly_safe=MS))
    assert 10 < got["crossed"].sum() < 118
    # the same scene 1e4 m away: the cell range is widened for the float rounding at that magnitude
    sh = np.array([1e4, -1e4, 1e4])
    for m, p in zip(maps, ps):
        m.update(p["obs"] + sh, p["unk"] + sh)
    jins, unks = [j + sh for j in jins], [u + sh for u in unks]
    same(capi.map_paths(jins, maps, np.arange(len(ps)), max_poly_whole=MW, max_poly_safe=MS),
         capi.paths_cloud(jins, unks, max_poly_whole=MW, max_poly_safe=MS))


def test_mapper_sized_shared_map():
    ps = same_forest(11, 64)
    occ, unk = ps[0]["obs"], mapper_cloud(ps[0])
    m = capi.Map()
    m.update(occ, unk)
    jins = [p["path_all"] for p in ps]
    got = capi.map_paths(jins, [m], max_poly_whole=MW, max_poly_safe=MS)
    same(got, capi.paths_cloud(jins, [unk] * len(ps), max_poly_whole=MW, max_poly_safe=MS))
    assert got["crossed"].all()                                     # every free cell is unknown: the crop always stops
    high = unk[unk[:, 2] > 1.6]                                     # unknown only above the corridors: the crops march
    m.update(occ, high)
    same(capi.map_paths(jins, [m], max_poly_whole=MW, max_poly_safe=MS),
         capi.paths_cloud(jins, [high] * len(ps), max_poly_whole=MW, max_poly_safe=MS))
    sh = np.array([-1e4, 1e4, 1e4])
    m.update(occ + sh, unk + sh)
    jins = [j + sh for j in jins]
    same(capi.map_paths(jins, [m], max_poly_whole=MW, max_poly_safe=MS),
         capi.paths_cloud(jins, [unk + sh] * len(ps), max_poly_whole=MW, max_poly_safe=MS))


def test_stall_and_statuses_on_the_device():
    torch = pytest.importorskip("torch")
    m = capi.Map()
    m.update(np.zeros((0, 3)), STALL_UNK)
    got = capi.map_paths([STALL_PATH, LINE], [m], drone_radius=1e-3)
    same(got, capi.paths_cloud([STALL_PATH, LINE], [STALL_UNK] * 2, drone_radius=1e-3))
    assert got["status"].tolist() == [capi.PATHS_STALL, capi.PATHS_OK]
    # what only the arrays tell is a status on the device: too few vertices, a NaN vertex, more than max_in, a bad map index
    dev = torch.device("cuda", 0)
    in_ofs = torch.tensor([0, 1, 6, 11, 16, 21], dtype=torch.int32, device=dev)
    pts = np.vstack([LINE[:1], LINE, LINE, LINE, LINE])
    pts[8, 2] = np.nan
    d_in = torch.from_numpy(pts).to(dev)
    idx = torch.tensor([0, 0, 0, 5, 0], dtype=torch.int32, device=dev)
    n = 5
    out = dict(poly_ofs_whole=torch.zeros(n + 1, dtype=torch.int32, device=dev), poly_ofs_safe=torch.zeros(n + 1, dtype=torch.int32, device=dev),
               path_whole=torch.zeros(n * 4 * 3, dtype=torch.float64, device=dev), path_safe=torch.zeros(n * 5 * 3, dtype=torch.float64, device=dev),
               status=torch.full((n,), -1, dtype=torch.int32, device=dev), crossed=torch.full((n,), 9, dtype=torch.uint8, device=dev))
    for max_in, want in ((5, [capi.PATHS_SHORT, capi.PATHS_OK, capi.PATHS_INPUT, capi.PATHS_MAP, capi.PATHS_OK]),
                         (4, [capi.PATHS_SHORT] + [capi.PATHS_INPUT] * 4)):
        s = capi.map_paths_args(n, in_ofs.data_ptr(), d_in.data_ptr(), {k: v.data_ptr() for k, v in out.items()}, maps=[m],
                                map_index=idx.data_ptr(), max_in=max_in, max_poly_whole=MW, max_poly_safe=MS, drone_radius=0.42)
        capi.map_paths_dev(s)
        torch.cuda.synchronize()
        assert out["status"].cpu().tolist() == want
        ofs = out["poly_ofs_whole"].cpu().numpy()
        bad = [j for j in range(n) if want[j] != capi.PATHS_OK]
        assert all(ofs[j + 1] == ofs[j] for j in bad) and (out["crossed"].cpu().numpy()[bad] == 0).all()
        pw = out["path_whole"].cpu().numpy().reshape(-1, 3)
        assert all(np.isnan(pw[ofs[j] + j]).all() for j in bad)


def _paths_dev(maps, d, out, max_in, stream):
    s = capi.map_paths_args(d["n"], d["in_ofs"].data_ptr(), d["in"].data_ptr(), {k: v.data_ptr() for k, v in out.items()},
                            maps=maps, map_index=d["idx"].data_ptr(), max_in=max_in, max_poly_whole=MW, max_poly_safe=MS,
                            drone_radius=UAV["drone_radius"])
    capi.map_paths_dev(s, stream)


def test_device_route_equals_host_route(solver):
    """fq_map_paths_dev -> fq_replan_pairs_plan_dev (the _map chain with windows and H/R) on one stream, without a host
    round trip, against fq_map_paths then fq_replan_pairs_plan on the host: every output."""
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = corridors(24, 1000)
    n = len(ps)
    maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
    ml = max(len(p["obs"]) + len(p["unk"]) for p in ps)
    # host route
    hp = capi.map_paths([p["jin"] for p in ps], maps, np.arange(n), max_poly_whole=MW, max_poly_safe=MS)
    for j, p in enumerate(ps):
        for k in ("whole", "safe"):
            o = hp["poly_ofs_" + k]
            p["path_" + k] = hp["path_" + k][o[j] + j:o[j + 1] + j + 1]
    w = capi.make_decomp_workload(ps)
    w0 = dict(init_whole=np.ones(n), final_whole=np.full(n, 8.0), init_safe=np.ones(n), final_safe=np.full(n, 8.0))
    ref = solver.replan_pairs_plan(w, 20000, "map", maps, np.arange(n), max_local=ml, last_factor_safe=np.zeros(n), windows=w0,
                                   want_coeffs=False)
    # device route: the paths stay on the device
    st = torch.cuda.Stream(device=dev)
    jins = [p["jin"] for p in ps]
    d = dict(n=n, in_ofs=torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in jins])]), dtype=torch.int32, device=dev),
             **{"in": torch.from_numpy(np.vstack(jins)).to(dev)}, idx=torch.arange(n, dtype=torch.int32, device=dev))
    po = dict(poly_ofs_whole=torch.zeros(n + 1, dtype=torch.int32, device=dev), poly_ofs_safe=torch.zeros(n + 1, dtype=torch.int32, device=dev),
              path_whole=torch.zeros(n * (MW + 1) * 3, dtype=torch.float64, device=dev),
              path_safe=torch.zeros(n * (MS + 1) * 3, dtype=torch.float64, device=dev))
    max_in = max(len(x) for x in jins)
    dw = {k: torch.from_numpy(np.ascontiguousarray(w[k])).to(dev) for k in ("x0", "lim", "goal")}
    win = {k: torch.from_numpy(v.copy()).to(dev) for k, v in w0.items()}
    last = torch.zeros(n, dtype=torch.float64, device=dev)
    cap = 20000
    out = dict(results=torch.zeros(n * 144, dtype=torch.uint8, device=dev),
               index_H=torch.full((n,), -7, dtype=torch.int32, device=dev), need_safe=torch.full((n,), 7, dtype=torch.uint8, device=dev),
               status_whole=torch.full((n,), -1, dtype=torch.int32, device=dev), status_safe=torch.full((n,), -1, dtype=torch.int32, device=dev),
               states=torch.zeros(cap * 12, dtype=torch.float64, device=dev), plan_ofs=torch.zeros(n + 1, dtype=torch.int64, device=dev),
               plan_status=torch.full((n,), -1, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()
    with torch.cuda.stream(st):
        _paths_dev(maps, d, po, max_in, st.cuda_stream)
        a = capi.PairArgs()
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, w["N_whole"], w["N_safe"], w["DC"], w["r_fraction"]
        a.x0, a.lim, a.results = dw["x0"].data_ptr(), dw["lim"].data_ptr(), out["results"].data_ptr()
        a.poly_ofs_whole, a.poly_ofs_safe = po["poly_ofs_whole"].data_ptr(), po["poly_ofs_safe"].data_ptr()
        for k in ("max_faces_whole", "max_poly_faces_whole", "max_faces_safe", "max_poly_faces_safe"):
            setattr(a, k, int(w[k]))
        max_fac = 8                                                 # |F| of the windows [1, 8] with inc 1
        longest = {m: max(capi.assign_count(w["N_whole"], P) for P in range(m + 1)) for m in (MW, MS)}
        s = capi.assign_args(0, {}, MW, MS, n * max_fac * longest[MW], n * max_fac * longest[MS])
        wa = capi.window_args(lambda k: win[k].data_ptr(), {"next_" + k: win[k].data_ptr() for k in capi.WINDOW_IN_KEYS}, 1.0, 20.0,
                              max_fac, max_fac)
        dc = capi.decomp_args(lambda k: None if k.startswith("obs_") else (po[k].data_ptr() if k in po else dw[k].data_ptr()),
                              {k: out[k].data_ptr() for k in ("status_whole", "status_safe")}, UAV["bbox"], UAV["drone_radius"],
                              UAV["z_ground"])
        hr = capi.hr_args(None, None, dict(last_factor_safe=last.data_ptr(), index_H=out["index_H"].data_ptr(),
                                           need_safe=out["need_safe"].data_ptr()))
        mp = capi.map_args(maps, d["idx"].data_ptr(), ml)
        pl = capi.plan_args(cap, dict(states=out["states"].data_ptr(), plan_ofs=out["plan_ofs"].data_ptr(),
                                      status=out["plan_status"].data_ptr()))
        solver.replan_pairs_plan_dev(a, s, wa, None, dc, hr, mp, pl, 0, st.cuda_stream)
    st.synchronize()
    got = _host({k: out[k] for k in ("results", "index_H", "need_safe", "status_whole", "status_safe")})
    for k in ("results", "index_H", "need_safe", "status_whole", "status_safe"):
        assert got[k].tobytes() == np.asarray(ref[k]).tobytes(), k
    for k in capi.WINDOW_IN_KEYS:
        assert win[k].cpu().numpy().tobytes() == ref["next_" + k].tobytes(), k
    assert last.cpu().numpy().tobytes() == ref["last_factor_safe"].tobytes()
    rows = int(ref["plan_ofs"][-1])
    assert out["plan_ofs"].cpu().numpy().tobytes() == ref["plan_ofs"].tobytes()
    assert out["plan_status"].cpu().numpy().tobytes() == ref["status"].tobytes()
    assert out["states"].cpu().numpy().reshape(-1, 12)[:rows].tobytes() == ref["states"][:rows].tobytes()
    for k in ("poly_ofs_whole", "poly_ofs_safe"):
        assert po[k].cpu().numpy().tobytes() == hp[k].tobytes(), k
    assert 0 < got["need_safe"].sum() < n and (ref["status"] == capi.PLAN_OK).sum() > n // 2


def test_captured_graph_reads_the_maps_last_update():
    torch = pytest.importorskip("torch")
    dev = torch.device("cuda", 0)
    ps = corridors(16, 2000)
    n = len(ps)
    maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
    jins = [p["jin"] for p in ps]
    d = dict(n=n, in_ofs=torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in jins])]), dtype=torch.int32, device=dev),
             **{"in": torch.from_numpy(np.vstack(jins)).to(dev)}, idx=torch.arange(n, dtype=torch.int32, device=dev))
    max_in = max(len(x) for x in jins)

    def outputs():
        return dict(poly_ofs_whole=torch.zeros(n + 1, dtype=torch.int32, device=dev),
                    poly_ofs_safe=torch.zeros(n + 1, dtype=torch.int32, device=dev),
                    path_whole=torch.zeros(n * (MW + 1) * 3, dtype=torch.float64, device=dev),
                    path_safe=torch.zeros(n * (MS + 1) * 3, dtype=torch.float64, device=dev),
                    status=torch.zeros(n, dtype=torch.int32, device=dev), crossed=torch.zeros(n, dtype=torch.uint8, device=dev))

    def host(o):
        return {k: v.cpu().numpy() for k, v in o.items()}

    st = torch.cuda.Stream(device=dev)
    o = outputs()
    with torch.cuda.stream(st):
        _paths_dev(maps, d, o, max_in, st.cuda_stream)             # warm-up outside the capture
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        _paths_dev(maps, d, o, max_in, st.cuda_stream)
    g.replay()
    torch.cuda.synchronize()
    before = host(o)
    rng = np.random.default_rng(5)
    new_unks = [np.vstack([p["unk"][::2], rng.uniform(-7, 7, (500, 3))]) for p in ps]
    for m, p, u in zip(maps, ps, new_unks):
        m.update(p["obs"], u)
    g.replay()
    torch.cuda.synchronize()
    replayed = host(o)
    fresh = outputs()
    with torch.cuda.stream(st):
        _paths_dev(maps, d, fresh, max_in, st.cuda_stream)
    st.synchronize()
    fresh = host(fresh)
    for k in fresh:                                                 # of path_* only the rows written
        rows = 3 * (int(fresh["poly_ofs_" + k[5:]][-1]) + n) if k.startswith("path_") else None
        assert replayed[k][:rows].tobytes() == fresh[k][:rows].tobytes(), k
    assert replayed["path_safe"].tobytes() != before["path_safe"].tobytes()
    ref = capi.paths_cloud(jins, new_unks, max_poly_whole=MW, max_poly_safe=MS)
    assert replayed["poly_ofs_safe"].tobytes() == ref["poly_ofs_safe"].tobytes()
    rows = int(ref["poly_ofs_safe"][-1]) + n
    assert replayed["path_safe"].reshape(-1, 3)[:rows].tobytes() == ref["path_safe"].tobytes()
