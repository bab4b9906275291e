"""Each planner's committed plan kept on the device (fq_queue_*, fq_replan_pairs_queue*): every chain selection through the
host entry gives fq_replan_pairs_plan's outputs byte for byte, and its rings equal collections.deque after appending
_plan's pieces (tests/plan_queue_oracle.py); the closed loop of tests/queue_loop.py -- select_dev, x0 read back, host JPS
from A, fq_jps_in, fq_map_paths_dev, _queue_dev through the _map chain with windows and H/R on indexed maps, pop_dev --
against the host route (deques, fq_map_paths, the _plan host entry, the window rule with the append's gate) in every
cycle; a CUDA graph of one cycle's device part; the refusals and the _dev duplicate-row status."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi

import plan_queue_oracle as pqo
import queue_loop as ql
from test_pair_hr_gpu import replans, workload
from test_pair_map_gpu import assert_same, make_maps
from test_pair_plan_gpu import cfg4, shared, windows

pytestmark = pytest.mark.gpu
CAP = ql.CAP


def pieces(out):
    """Each corridor's piece from a _plan return value, None where it appends nothing."""
    ofs, st = out["plan_ofs"], out["status"]
    return [out["states"][ofs[j]:ofs[j + 1]] if st[j] == capi.PLAN_OK else None for j in range(len(st))]


def host_queue_vs_plan(solver, w, chain, *args, **kw):
    """_queue (host entry) against _plan on rings of two-state plans on permuted rows with wrap-around."""
    n = w["n_prob"]
    rng = np.random.default_rng(n)
    rows = rng.permutation(n + 3)[:n].astype(np.int32)
    plans = [[rng.normal(0, 1, 12) for _ in range(2)] for _ in range(n + 3)]
    ring = pqo.to_ring(plans, CAP, heads=rng.integers(0, CAP, n + 3))
    dq = [pqo.from_ring(ring, r) for r in range(n + 3)]
    k_end = np.zeros(n, np.int32)
    k_end[::5] = -1                                          # no select: nothing appended
    ref = solver.replan_pairs_plan(w, 1 << 17, chain, *args, **kw)
    ke = k_end.copy()
    got = solver.replan_pairs_queue(w, ring, ke, chain, *args, rows=rows, G_term=w["x0"][:, :3], goal_radius=1e9, **kw)
    status = np.array([pqo.append(dq[rows[j]], int(k_end[j]), p, CAP) for j, p in enumerate(pieces(ref))], np.int32)
    want = {k: v for k, v in ref.items() if k not in capi.PLAN_KEYS}
    win = kw.get("windows", args[0] if chain == "window" else None)
    for k in capi.WINDOW_IN_KEYS:               # a failed append keeps the input window
        if "next_" + k in want:
            want["next_" + k] = np.where(status == pqo.QUEUE_OK, want["next_" + k], win[k])
    assert_same({k: v for k, v in got.items() if k not in ("queue_status", "goal_seen")}, want)
    assert (ke == -1).all()
    for j, st in enumerate(status):
        assert got["queue_status"][j] == st, j
        assert got["goal_seen"][j] == (st == pqo.QUEUE_OK), j
    for r in range(n + 3):
        assert np.array(pqo.from_ring(ring, r)).tobytes() == np.array(dq[r]).tobytes(), r
    assert (got["queue_status"] == pqo.QUEUE_OK).sum() >= n // 3
    return got


@pytest.mark.parametrize("chain", ["shared", "assign", "window", "exact"])
def test_list_chains_through_the_host_entry(solver, chain):
    w = cfg4(16)
    args, kw = (), {}
    if chain == "shared":
        w = shared(w)
    if chain == "window":
        args = (windows(16),)
    host_queue_vs_plan(solver, w, chain, *args, **kw)


@pytest.mark.parametrize("chain", ["decomp", "hr", "map"])
def test_decomposing_chains_through_the_host_entry(solver, chain):
    ps = replans(24, 0)
    w = workload(ps)
    n = len(ps)
    kw = dict(last_factor_safe=np.random.default_rng(3).uniform(1.0, 8.0, n)) if chain != "decomp" else {}
    args = ()
    if chain == "map":
        maps = make_maps([p["obs"] for p in ps], [p["unk"] for p in ps])
        args = (maps, np.arange(n))
        kw["max_local"] = max(len(p["unk"]) + len(p["obs"]) for p in ps)
    host_queue_vs_plan(solver, w, chain, *args, **kw)


def _route(solver, n, start, rows, stream):
    torch = pytest.importorskip("torch")
    pl = ql.planners(n, start)
    return pl, ql.DeviceRoute(solver, pl, rows, torch, torch.device("cuda", 0), stream), torch


def test_closed_loop_against_the_host_route(solver):
    """8 cycles of 24 forest planners on indexed maps.  Each cycle: select_dev, x0 read back, host JPS from A and fq_jps_in,
    pops (10 or more on some planners) between the select and the chain, fq_map_paths_dev and _queue_dev (the _map chain
    with windows and H/R), pops.  Every cycle against the host route: A, k_end, goals, paths, records, H/R, statuses,
    goal_seen, windows, last_factor_safe and every deque byte for byte."""
    torch = pytest.importorskip("torch")
    n = 24
    rng = np.random.default_rng(11)
    rows = rng.permutation(n + 5)[:n].astype(np.int32)
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    pl, dv, _ = _route(solver, n, 0, rows, st)
    host = ql.HostRoute(solver, pl, dv.maps)
    w0 = ql.windows0(n)
    with torch.cuda.stream(st):
        dv.reset(w0)
    host.reset(w0)
    seen, no_safe_ok = set(), False
    for cycle in range(8):
        mid = rng.choice([0, 2, pqo.DELTA_T - 1, pqo.DELTA_T, 13], n).astype(np.int32)
        after = rng.integers(0, 4, n).astype(np.int32)
        with torch.cuda.stream(st):
            dv.select()
            x0 = dv.read_x0()                                 # the one read-back: A, for JPS
            k_dev = dv.k_end.cpu().numpy()
            jins, ok = ql.jps_inputs(pl, x0)
            if cycle == 3:
                ok[0] = False                                 # the caller gates planner 0 out this cycle (e.g. GOAL_REACHED)
            dv.upload(jins, ok)
            dv.pop(mid)
            dv.replan()
            h = dv.snap()
            paths = {k: v.cpu().numpy() for k, v in dv.paths.items()}
            dv.pop(after)
            g_after = dv.goals.cpu().numpy()
        # ---- the host route, from the deques' own A
        x0h, kh = host.select()
        assert x0.tobytes() == x0h.tobytes() and k_dev.tobytes() == kh.tobytes(), cycle
        kh[~ok] = -1
        goals = host.pop(mid)
        for j in range(n):
            assert h["goals"][j, :mid[j]].tobytes() == goals[j].tobytes(), (cycle, j)
        r = host.replan(x0h, kh, jins)
        ref = r["ref"]
        for k in ("poly_ofs_whole", "poly_ofs_safe"):
            assert paths[k].tobytes() == r["paths"][k].tobytes(), (cycle, k)
        assert h["results"].tobytes() == ref["results"].tobytes(), cycle
        for k in ("index_H", "need_safe"):
            assert h[k].tobytes() == ref[k].tobytes(), (cycle, k)
        assert h["last"].tobytes() == ref["last_factor_safe"].tobytes(), cycle
        assert h["status"].tobytes() == r["status"].tobytes(), (cycle, h["status"], r["status"])
        assert h["goal_seen"].tobytes() == r["goal_seen"].tobytes(), cycle
        assert (h["k_end"] == -1).all()
        for k in capi.WINDOW_IN_KEYS:
            assert h["win_" + k].tobytes() == host.wins[k].tobytes(), (cycle, k)
        for j in range(n):
            assert np.array(dv.plan(j, h)).tobytes() == np.array(host.plans[j]).tobytes(), (cycle, j)
        goals = host.pop(after)
        for j in range(n):
            assert g_after[j, :after[j]].tobytes() == goals[j].tobytes(), (cycle, j)
        seen |= set(r["status"].tolist())
        no_safe_ok |= bool(((r["status"] == pqo.QUEUE_OK) & (ref["need_safe"] == 0)).any())
    assert {pqo.QUEUE_OK, pqo.QUEUE_NONE, pqo.QUEUE_PUBLISHED} <= seen, seen
    assert no_safe_ok


def test_graph_of_one_cycle_replays_the_first_call(solver):
    """select_dev, fq_map_paths_dev, _queue_dev and pop_dev captured once, replayed from the start-up state twice on the
    same JPS_in: the first eager cycle's bytes each time."""
    torch = pytest.importorskip("torch")
    n = 24
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    pl, dv, _ = _route(solver, n, 100, np.arange(n)[::-1].copy(), st)
    w0 = ql.windows0(n)
    jins, ok = ql.jps_inputs(pl, np.array([np.concatenate([p["start"], np.zeros(6)]) for p in pl]))

    def cycle():
        dv.select()
        dv.replan()
        dv.pop()

    with torch.cuda.stream(st):
        dv.reset(w0)
        dv.ticks.fill_(3)
        dv.upload(jins, np.ones(n, bool))
        cycle()
        first = dv.snap()
    assert (first["status"] == pqo.QUEUE_OK).sum() >= 8
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        cycle()
    for _ in range(2):
        with torch.cuda.stream(st):
            dv.reset(w0)
        st.synchronize()
        g.replay()
        torch.cuda.synchronize()
        rep = dv.snap()
        for k in first:
            assert rep[k].tobytes() == first[k].tobytes(), k


def test_refusals_and_the_device_row_status(solver, built_lib):
    torch = pytest.importorskip("torch")
    L = capi.lib()
    B = C.byref
    w = cfg4(4)
    out = solver.replan_pairs_assign(w)
    s = capi.assign_args(0, {k: out[k].ctypes.data for k in ("cand_ofs_whole", "cand_ofs_safe", "sigma_whole", "sigma_safe")})
    a = capi.pair_args(w, lambda k: None if k.startswith("sigmas_") else w[k].ctypes.data, {"results": out["results"].ctypes.data})
    a.n_sig_whole = a.n_sig_safe = 0
    ring = pqo.to_ring([pqo.reset(p) for p in w["x0"][:, :3]], 1024)
    k_end, status = np.zeros(4, np.int32), np.zeros(4, np.int32)

    def err(h=None):
        return L.fq_last_error(h or solver._h).decode()

    def pq(**kw):
        q = capi.pair_queue_args(capi.queue_args(ring), kw.get("rows"), k_end, status)
        for f, v in kw.items():
            if f in ("cap", "delta_t", "n_rows", "states"):
                setattr(q.ring, f, v)
            elif f != "rows":
                setattr(q, f, v)
        return q

    for host in (True, False):
        def call(q):
            if host:
                return L.fq_replan_pairs_queue(solver._h, B(a), B(s), None, None, None, None, None, q)
            return L.fq_replan_pairs_queue_dev(solver._h, B(a), B(s), None, None, None, None, None, q, None, None)
        assert call(None) == -1 and err() == "queue is NULL"
        for f, msg in [("cap", "queue: cap < 1"), ("delta_t", "queue: delta_t < 1"), ("n_rows", "queue: n_rows < 1")]:
            assert call(B(pq(**{f: 0}))) == -1 and err() == msg, f
        assert call(B(pq(states=None))) == -1 and "must not be NULL" in err()
        assert call(B(pq(k_end=None))) == -1 and "must not be NULL" in err()
    rows = np.array([0, 1, 1, 2], np.int32)
    assert L.fq_replan_pairs_queue(solver._h, B(a), B(s), None, None, None, None, None, B(pq(rows=rows))) == -1
    assert err() == "queue: a row named twice"
    # the family's own refusals, with the family's text
    a.DC = 0.0
    assert L.fq_replan_pairs_assign(solver._h, B(a), B(s)) == -1
    want = err()
    assert L.fq_replan_pairs_queue(solver._h, B(a), B(s), None, None, None, None, None, B(pq())) == -1 and err() == want
    a.DC = w["DC"]
    assert capi.has_feature("replan_pairs_queue")
    assert L.fq_replan_pairs_queue(None, None, None, None, None, None, None, None, None) == -1
    g = capi.Solver(n_gpus=1, devices=[0])
    try:
        assert L.fq_replan_pairs_queue(g._h, B(a), B(s), None, None, None, None, None, B(pq())) == -1 and "multi-GPU" in err(g._h)
    finally:
        g.close()
    # the _dev entry: corridors naming one row get FQ_QUEUE_ROWS and leave it untouched
    n = 8
    rows = np.arange(n, dtype=np.int32)
    rows[3] = rows[5] = 1
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    pl, dv, _ = _route(solver, n, 200, rows, st)
    with torch.cuda.stream(st):
        dv.reset(ql.windows0(n))
        dv.select()
        jins, _ = ql.jps_inputs(pl, np.array([np.concatenate([p["start"], np.zeros(6)]) for p in pl]))   # row 1 is empty
        dv.upload(jins, np.ones(n, bool))
        before = dv.snap()
        dv.replan()
        after = dv.snap()
    for j in (1, 3, 5):
        assert after["status"][j] == pqo.QUEUE_ROWS
    assert after["states"][1].tobytes() == before["states"][1].tobytes() and after["size"][1] == before["size"][1]
    assert (after["k_end"] == -1).all()
