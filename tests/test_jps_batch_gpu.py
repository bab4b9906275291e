"""Every planner's JPS search and JPS_in on the device (fq_jps_batch, fq_jps_batch_dev): both entries byte for byte against
tests/jps_batch_oracle.py on forest planners (per-planner grids and one shared grid) and on the device statuses; and the
replan loop with no host step -- select_dev, jps_batch_dev, fq_map_paths_dev, _queue_dev through the _map chain with
windows and H/R, pop_dev -- against the same device route fed by host JPS, eagerly and as a CUDA graph."""
import numpy as np
import pytest

from faster_b200 import capi

import jps_batch_oracle as jbo
import queue_loop as ql
from test_jps_batch_cpu import _x0, forest

pytestmark = pytest.mark.gpu


def _dev_batch(torch, grids, A, G, grid_index=None, pos=None, k_end=None, **kw):
    """fq_jps_batch_dev over device copies.  -> the outputs as host arrays."""
    dev = torch.device("cuda", 0)
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    n = len(G)
    max_in = kw.get("max_in", 512)
    gd = {k: T(v) for k, v in capi.jps_grids(grids).items()}
    out = dict(in_ofs=torch.full((n + 1,), -9, dtype=torch.int32, device=dev), status=torch.full((n,), -9, dtype=torch.int32, device=dev),
               **{"in": torch.full((n * max_in, 3), 7.0, dtype=torch.float64, device=dev)})
    ke = T(None if k_end is None else np.asarray(k_end, np.int32))
    gi = T(None if grid_index is None else np.asarray(grid_index, np.int32))
    ps = T(None if pos is None else np.asarray(pos, np.float64))
    dx0, dG = T(_x0(A)), T(np.asarray(G, np.float64))     # kept alive until the call has run: the struct holds addresses only
    a = capi.jps_batch_args(n, gd, dx0, dG, out, gi, ps, k_end=ke, **kw)
    st = torch.cuda.Stream(device=dev)
    capi.jps_batch_dev(a, st.cuda_stream)
    st.synchronize()
    h = {k: v.cpu().numpy() for k, v in out.items()}
    h["k_end"] = None if ke is None else ke.cpu().numpy()
    return h


def _both(torch, grids, A, G, **kw):
    want = jbo.batch(grids, _x0(A), G, **kw)
    jbo.assert_equal(capi.jps_batch(grids, _x0(A), G, **kw), want, "host entry")
    jbo.assert_equal(_dev_batch(torch, grids, A, G, **kw), want, "device entry")
    return want


def test_forest_planners_against_the_oracle(built_lib):
    torch = pytest.importorskip("torch")
    pl = forest(128)
    n = len(pl)
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    want = _both(torch, [p["grid"] for p in pl], A, G, grid_index=np.arange(n), pos=A + 0.3, k_end=np.arange(n))
    assert (want["status"] == jbo.OK).sum() >= n * 3 // 4
    want = _both(torch, [pl[0]["grid"]], A, G, k_end=np.arange(n))
    assert {jbo.OK, jbo.NO_PATH} <= set(want["status"].tolist())
    _both(torch, [p["grid"] for p in pl[:32]], A[:32], G[:32], grid_index=np.arange(32), use_jps=False)


def test_device_statuses(built_lib):
    """NODES, LONG and, on the device entry only, INPUT (NaN A, grid_index out of range, a bad grid)."""
    torch = pytest.importorskip("torch")
    pl = forest(6, 40)
    grids = [p["grid"] for p in pl]
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    want = _both(torch, grids, A, G, grid_index=np.arange(6), max_nodes=1, k_end=np.ones(6))
    assert jbo.NODES in want["status"]
    want = _both(torch, grids, A, G, grid_index=np.arange(6), max_in=3, dist_max=0.2)
    assert jbo.LONG in want["status"]
    A2 = A.copy()
    A2[1, 0] = np.nan
    kw = dict(grid_index=[0, 1, 7, -1, 4, 5], k_end=np.full(6, 3))
    want = jbo.batch(grids, _x0(A2), G, **kw)
    jbo.assert_equal(_dev_batch(torch, grids, A2, G, **kw), want)
    assert list(want["status"][1:4]) == [jbo.INPUT] * 3
    g, o, r = grids[0]
    got = _dev_batch(torch, [(g, o, r), (g, o, -r)], A[:2], G[:2], grid_index=[0, 1])
    assert list(got["status"]) == [jbo.batch([(g, o, r)], _x0(A[:1]), G[:1])["status"][0], jbo.INPUT]


class DeviceJpsRoute(ql.DeviceRoute):
    """queue_loop.DeviceRoute with JPS on the device: fq_jps_batch_dev from x0 writes JPS_in and k_end in place, so a cycle
    has no read-back."""

    def __init__(self, solver, pl, rows, torch, dev, stream, max_nodes=capi.JPS_MAX_NODES):
        super().__init__(solver, pl, rows, torch, dev, stream)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        self.gd = {k: T(v) for k, v in capi.jps_grids([(p["grid"], p["origin"], p["res"]) for p in pl]).items()}
        self.gi = T(np.arange(self.n, dtype=np.int32))
        self.jps_status = torch.zeros(self.n, dtype=torch.int32, device=dev)
        out = dict(in_ofs=self.jin["in_ofs"], status=self.jps_status, **{"in": self.jin["pts"]})
        self.ja = capi.jps_batch_args(self.n, self.gd, self.x0, self.G, out, self.gi, None, ql.RA, ql.DIST_MAX, True, max_nodes, ql.MAX_IN,
                                      self.k_end)

    def jps(self):
        capi.jps_batch_dev(self.ja, self.st.cuda_stream)

    def cycle(self):
        self.select()
        self.jps()
        self.replan()
        self.pop()


def host_jps(pl, x0):
    """The oracle's JPS_in from A = x0 on each planner's grid (ra from A, as the device route's pos = NULL).  -> (list of
    JPS_in, ok = status OK, the batch)."""
    b = jbo.batch([(p["grid"], p["origin"], p["res"]) for p in pl], x0, np.array([p["goal"] for p in pl]), grid_index=np.arange(len(pl)),
                  Ra=ql.RA, dist_max=ql.DIST_MAX, max_in=ql.MAX_IN)
    o = b["in_ofs"]
    return [b["in"][o[j]:o[j + 1]] for j in range(len(pl))], b["status"] == jbo.OK, b


def _routes(solver, n, start, torch):
    st = torch.cuda.Stream(device=torch.device("cuda", 0))
    pl = ql.planners(n, start)
    rows = np.random.default_rng(n + start).permutation(n + 5)[:n].astype(np.int32)
    dev = torch.device("cuda", 0)
    return pl, DeviceJpsRoute(solver, pl, rows, torch, dev, st), ql.DeviceRoute(solver, pl, rows, torch, dev, st), st


def test_closed_loop_without_a_host_step(solver):
    """8 cycles of 64 planners: the device-JPS loop against the same route fed by the oracle's host JPS, byte for byte
    (JPS_in, JPS statuses, plans, goals, records, statuses, windows, k_end)."""
    torch = pytest.importorskip("torch")
    n = 64
    pl, dv, ref, st = _routes(solver, n, 0, torch)
    rng = np.random.default_rng(5)
    w0 = ql.windows0(n)
    with torch.cuda.stream(st):
        dv.reset(w0)
        ref.reset(w0)
    seen = set()
    for cycle in range(8):
        ticks = rng.choice([1, 3, 9, 12], n).astype(np.int32)
        with torch.cuda.stream(st):
            dv.select()
            dv.jps()
            jin_dev = {k: v.cpu().numpy() for k, v in dv.jin.items()}
            jst = dv.jps_status.cpu().numpy()
            dv.replan()
            dv.pop(ticks)
            got = dv.snap()
            ref.select()
            jins, ok, b = host_jps(pl, ref.read_x0())
            ref.upload(jins, ok)
            ref.replan()
            ref.pop(ticks)
            want = ref.snap()
        assert jst.tobytes() == b["status"].tobytes(), cycle
        assert jin_dev["in_ofs"].tobytes() == b["in_ofs"].tobytes(), cycle
        assert jin_dev["pts"][:b["in_ofs"][-1]].tobytes() == b["in"].tobytes(), cycle
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), (cycle, k)
        seen |= set(got["status"].tolist())
    assert capi.QUEUE_OK in seen


def test_graph_of_one_whole_cycle(solver):
    """select_dev, jps_batch_dev, map_paths_dev, _queue_dev and pop_dev captured once and replayed 8 times: each replay's
    bytes equal the eager cycle's."""
    torch = pytest.importorskip("torch")
    n = 32
    pl, dv, _, st = _routes(solver, n, 100, torch)
    w0 = ql.windows0(n)
    eager = []
    with torch.cuda.stream(st):
        dv.reset(w0)
        dv.ticks.fill_(3)
        for _ in range(8):
            dv.cycle()
            eager.append(dv.snap())
        dv.reset(w0)
    st.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        dv.cycle()
    with torch.cuda.stream(st):
        dv.reset(w0)
    st.synchronize()
    for i in range(8):
        g.replay()
        torch.cuda.synchronize()
        rep = dv.snap()
        for k in eager[i]:
            assert rep[k].tobytes() == eager[i][k].tobytes(), (i, k)
