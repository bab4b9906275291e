"""The closed replan loop of a batch planner whose committed plans are kept on the device, and the same loop with the plans
in host deques: forest planners on indexed maps (one map per planner, its occupied and unknown clouds), each cycle
choosing A, running host JPS from A to G (start z clamped at 0, jps_manager.cpp:143), fq_jps_in, the device paths
(fq_map_paths_dev / fq_map_paths), the _map chain with windows and H/R, and getNextGoal publications.  A plain module
(no pytest): tests/test_pair_queue_gpu.py checks the two routes against each other and tools/queue_replan.py times them.

A planner whose JPS query fails gets k_end = -1 on both routes, so nothing is appended and its window is kept, as
Faster::replan returns before the append when solveJPS3D fails; its corridor is then the segment [A, G]."""
import numpy as np

from faster_b200 import capi, corridor as cr

import plan_queue_oracle as pqo

MW, MS = 3, 4                        # par_.max_poly_whole / _safe
RA = 4.0                             # par_.Ra
DIST_MAX = 1.5                       # createMoreVertexes' dist_max
MAX_IN = 512                         # the longest JPS_in the device route accepts (fq_map_paths_args.max_in)
CAP = 4096                           # states per ring row
GOAL_RADIUS = capi.GOAL_RADIUS
MAX_FAC = 64                         # bound on every window's factor count


def planners(n, start=0):
    """n forest planners: the inflated grid JPS plans on, the occupied cloud, the unknown cloud around the start, the goal
    G, the start and the limits (corridor.forest_pair_paths / forest_jps / forest_unknown_cloud of seeds 40000 + start ..)."""
    out = []
    for seed in range(40000 + start, 40000 + start + n):
        fj, p = cr.forest_jps(seed), cr.forest_pair_paths(seed)
        p["x0"] = p["x0"].copy()
        p["x0"][:3] = fj["start"]
        p["unk"] = cr.forest_unknown_cloud(p)
        _, centres, radii = cr.make_forest(seed)
        p["grid"], p["origin"], p["res"] = cr.voxelise_forest(centres, radii, inflation=0.47)
        p["start"], p["goal"] = fj["start"], fj["goal"]
        out.append(p)
    return out


def jps_inputs(pl, x0):
    """Every planner's JPS_in from A = x0[j] (host JPS, then fq_jps_in).  -> (list of [m, 3], ok: JPS found a path)."""
    jins, ok = [], np.zeros(len(pl), bool)
    for j, p in enumerate(pl):
        A, G = x0[j, :3], p["goal"]
        s = A.copy()
        s[2] = max(s[2], 0.0)
        try:
            path, _ = capi.jps3d_plan_world(p["grid"], p["origin"], p["res"], s, G, True)
        except capi.FqError:
            path = np.zeros((0, 3))
        ok[j] = len(path) >= 1
        ra = min(float(np.linalg.norm(G - A)) - 0.001, RA)
        jin = capi.jps_in(path if ok[j] else A[None], A, G, ra, DIST_MAX)
        assert len(jin) <= MAX_IN
        jins.append(jin)
    return jins, ok


def windows0(n):
    return dict(init_whole=np.ones(n), final_whole=np.full(n, 10.0), init_safe=np.ones(n), final_safe=np.full(n, 10.0))


class DeviceRoute:
    """The plans in device rings on rows `rows` of n + 5; every array the cycle touches is a device tensor and every struct
    is built once, so a CUDA graph can capture the device part of a cycle."""

    def __init__(self, solver, pl, rows, torch, dev, stream, max_ticks=16):
        self.solver, self.pl, self.torch, self.st = solver, pl, torch, stream
        n = self.n = len(pl)
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        Z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)  # noqa: E731
        f64, i32, u8 = torch.float64, torch.int32, torch.uint8
        self.ring = dict(states=Z((n + 5, CAP, 12), f64), head=Z(n + 5, i32), size=Z(n + 5, i32))
        self.q = capi.queue_args(self.ring)
        self.rows = T(np.asarray(rows, np.int32))
        self.k_end, self.ticks, self.max_ticks = Z(n, i32), Z(n, i32), max_ticks
        self.goals = Z((n, max_ticks, 12), f64)
        self.x0, self.lim, self.G = Z((n, 9), f64), T([p["lim"] for p in pl]), T([p["goal"] for p in pl])
        self.pos = T([p["start"] for p in pl])
        self.win = {k: Z(n, f64) for k in capi.WINDOW_IN_KEYS}
        self.last = Z(n, f64)
        self.out = dict(results=Z(n * 144, u8), index_H=Z(n, i32), need_safe=Z(n, u8), status=Z(n, i32), goal_seen=Z(n, u8))
        self.jin = dict(in_ofs=Z(n + 1, i32), pts=Z((n * MAX_IN, 3), f64))
        self.paths = dict(poly_ofs_whole=Z(n + 1, i32), poly_ofs_safe=Z(n + 1, i32), path_whole=Z(n * (MW + 1) * 3, f64),
                          path_safe=Z(n * (MS + 1) * 3, f64))
        self.maps = [capi.Map() for _ in pl]
        for m, p in zip(self.maps, pl):
            m.update(p["obs"], p["unk"])
        self.idx = T(np.arange(n, dtype=np.int32))
        self.ml = max(len(p["obs"]) + len(p["unk"]) for p in pl)
        self.pa = capi.map_paths_args(n, self.jin["in_ofs"].data_ptr(), self.jin["pts"].data_ptr(),
                                      {k: v.data_ptr() for k, v in self.paths.items()}, maps=self.maps, map_index=self.idx.data_ptr(),
                                      max_in=MAX_IN, max_poly_whole=MW, max_poly_safe=MS, drone_radius=cr.UAV["drone_radius"])
        a = self.a = capi.PairArgs()
        N = pl[0]["N"]
        a.n_prob, a.N_whole, a.N_safe, a.DC, a.r_fraction = n, N, N, float(pl[0]["DC"]), 0.6
        a.x0, a.lim, a.results = self.x0.data_ptr(), self.lim.data_ptr(), self.out["results"].data_ptr()
        a.poly_ofs_whole, a.poly_ofs_safe = self.paths["poly_ofs_whole"].data_ptr(), self.paths["poly_ofs_safe"].data_ptr()
        a.max_faces_whole = a.max_faces_safe = 400                   # make_decomp_workload's caps, as the host route's
        a.max_poly_faces_whole = a.max_poly_faces_safe = 64
        longest = {m: max(capi.assign_count(N, P) for P in range(m + 1)) for m in (MW, MS)}
        self.s = capi.assign_args(0, {}, MW, MS, n * MAX_FAC * longest[MW], n * MAX_FAC * longest[MS])
        self.wa = capi.window_args(lambda k: self.win[k].data_ptr(), {"next_" + k: self.win[k].data_ptr() for k in capi.WINDOW_IN_KEYS},
                                   1.0, 20.0, MAX_FAC, MAX_FAC)
        src = dict(path_whole=self.paths["path_whole"], path_safe=self.paths["path_safe"], goal=self.G)
        self.dc = capi.decomp_args(lambda k: src[k].data_ptr() if k in src else None, {}, cr.UAV["bbox"], cr.UAV["drone_radius"],
                                   cr.UAV["z_ground"])
        self.hr = capi.hr_args(None, None, dict(last_factor_safe=self.last.data_ptr(), index_H=self.out["index_H"].data_ptr(),
                                                need_safe=self.out["need_safe"].data_ptr()))
        self.mp = capi.map_args(self.maps, self.idx.data_ptr(), self.ml)
        self.pq = capi.pair_queue_args(self.q, self.rows, self.k_end, self.out["status"], self.out["goal_seen"], self.G, GOAL_RADIUS)

    def reset(self, w0):
        """Start-up: every row := [the start], the windows w0, last_factor_safe 0 (on the current stream)."""
        for k, v in w0.items():
            self.win[k].copy_(self.torch.from_numpy(v))
        self.last.zero_()
        for v in self.ring.values():
            v.zero_()
        capi.queue_reset_dev(self.q, self.n, self.rows, self.pos, self.st.cuda_stream)

    def select(self):
        capi.queue_select_dev(self.q, self.n, self.rows, self.x0, self.k_end, self.st.cuda_stream)

    def read_x0(self):
        """The cycle's one read-back: A of every planner."""
        return self.x0.cpu().numpy()

    def upload(self, jins, ok):
        """JPS_in onto the device; a planner whose JPS failed skips its append (k_end = -1)."""
        ofs = np.concatenate([[0], np.cumsum([len(x) for x in jins])]).astype(np.int32)
        self.jin["in_ofs"].copy_(self.torch.from_numpy(ofs))
        self.jin["pts"][:ofs[-1]].copy_(self.torch.from_numpy(np.vstack(jins)))
        if not ok.all():
            self.k_end[self.torch.from_numpy(np.flatnonzero(~ok)).to(self.k_end.device)] = -1

    def replan(self):
        """fq_map_paths_dev, then the _map chain appending to the rings."""
        capi.map_paths_dev(self.pa, self.st.cuda_stream)
        self.solver.replan_pairs_queue_dev(self.a, self.s, self.wa, None, self.dc, self.hr, self.mp, self.pq, 0, self.st.cuda_stream)

    def pop(self, ticks=None):
        if ticks is not None:
            self.ticks.copy_(self.torch.from_numpy(np.asarray(ticks, np.int32)))
        capi.queue_pop_dev(self.q, self.n, self.rows, self.ticks, self.max_ticks, self.goals, self.st.cuda_stream)

    def snap(self):
        h = {k: v.cpu().numpy() for k, v in self.out.items()}
        h["results"] = np.frombuffer(h["results"].tobytes(), capi.PAIR_RESULT_DTYPE)
        h.update({k: v.cpu().numpy() for k, v in self.ring.items()})
        h.update({"win_" + k: v.cpu().numpy() for k, v in self.win.items()})
        h.update(last=self.last.cpu().numpy(), goals=self.goals.cpu().numpy(), k_end=self.k_end.cpu().numpy(), x0=self.x0.cpu().numpy())
        return h

    def plan(self, j, h):
        """Planner j's plan, front to back, from a snap."""
        return pqo.from_ring(dict(states=h["states"], head=h["head"], size=h["size"]), int(self.rows[j]))


class HostRoute:
    """The plans in host deques: A chosen on the host, fq_map_paths and the _plan host entry (x0 uploaded, every piece
    copied back), appendToPlan on the deques, and the window update gated by it, as Faster::replan does."""

    def __init__(self, solver, pl, maps):
        self.solver, self.pl, self.maps = solver, pl, maps
        self.n = len(pl)
        self.ml = max(len(p["obs"]) + len(p["unk"]) for p in pl)

    def reset(self, w0):
        self.plans = [pqo.reset(p["start"]) for p in self.pl]
        self.wins = {k: v.copy() for k, v in w0.items()}
        self.lastf = np.zeros(self.n)

    def select(self):
        sel = [pqo.select(p) for p in self.plans]
        return np.array([s[0] for s in sel]), np.array([s[1] for s in sel], np.int32)

    def pop(self, ticks):
        return [pqo.pop(p, int(t)) for p, t in zip(self.plans, ticks)]

    def replan(self, x0, k_end, jins):
        """-> dict(ref (the _plan return value), status, goal_seen, paths (fq_map_paths's))."""
        n = self.n
        hp = capi.map_paths(jins, self.maps, np.arange(n), max_poly_whole=MW, max_poly_safe=MS)
        ps = []
        for j, p in enumerate(self.pl):
            q = dict(p, x0=x0[j])
            for k in ("whole", "safe"):
                o = hp["poly_ofs_" + k]
                q["path_" + k] = hp["path_" + k][o[j] + j:o[j + 1] + j + 1]
            ps.append(q)
        w = capi.make_decomp_workload(ps)
        ref = self.solver.replan_pairs_plan(w, 1 << 17, "map", self.maps, np.arange(n), max_local=self.ml, last_factor_safe=self.lastf,
                                            windows=self.wins, want_coeffs=False)
        ofs, pst = ref["plan_ofs"], ref["status"]
        status = np.array([pqo.append(self.plans[j], int(k_end[j]), ref["states"][ofs[j]:ofs[j + 1]] if pst[j] == capi.PLAN_OK else None,
                                      CAP) for j in range(n)], np.int32)
        ok = status == pqo.QUEUE_OK
        seen = np.array([ok[j] and pqo.goal_seen(self.plans[j], self.pl[j]["goal"], GOAL_RADIUS) for j in range(n)], np.uint8)
        self.wins = {k: np.where(ok, ref["next_" + k], self.wins[k]) for k in capi.WINDOW_IN_KEYS}
        self.lastf = ref["last_factor_safe"].copy()
        return dict(ref=ref, status=status, goal_seen=seen, paths=hp)
