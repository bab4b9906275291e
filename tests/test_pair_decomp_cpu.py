"""The device decomposition of the chained replan (fq_replan_pairs_decomp*) without a GPU: the product's kernel source
(faster_b200/csrc/fq_decomp.cuh) under the block emulation of tests/cpp/simt_emu/, bit for bit against the host's
fq_ellipsoid_decomp on forest corridors (whole and safe), random clouds, edge inputs and a cloud dense enough to spill;
the statuses of the caps and of degenerate input; the goal rule against a numpy restatement; the host golden; the ctypes
layout of fq_pair_decomp."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi

import decomp_cases as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
ST = capi.DECOMP_STATUS


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_decomp_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_decomp_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_decomp.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_int] + \
                                [C.c_void_p] * 6 + [C.c_int]
        L.emu_decomp.restype = None
        L.emu_host_round.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def emu_decomp(paths, clouds, inflate, first=None, goal=None, cap_pf=256, max_faces=2048, max_obs=None, max_poly=None,
               csr_threads=64):
    """One sweep of the device decomposition under the emulation.  paths: list of [P_j + 1, 3]; clouds: list of [m_j, 3].
    -> dict(face_ofs, Ab, xf, pos, status)."""
    n = len(paths)
    po = np.concatenate([[0], np.cumsum([len(p) - 1 for p in paths])]).astype(np.int32)
    path = np.ascontiguousarray(np.vstack(paths), np.float64)
    oo = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    obs = np.ascontiguousarray(np.vstack([np.reshape(c, (-1, 3)) for c in clouds] + [np.zeros((1, 3))]), np.float64)
    mp = int(np.diff(po).max()) if max_poly is None else max_poly
    mo = int(np.diff(oo).max()) if max_obs is None else max_obs
    face_ofs = np.zeros(n * mp + 1, np.int32)
    Ab = np.zeros((n * max_faces, 4))
    xf, pos, status = np.zeros((n, 9)), np.zeros((n, 3)), np.full(n, -1, np.int32)
    bbox = np.asarray(dc.BBOX, np.float64)
    first = None if first is None else np.ascontiguousarray(first, np.float64)
    goal = None if goal is None else np.ascontiguousarray(goal, np.float64)
    _lib().emu_decomp(n, mp, _p(po), _p(path), _p(first), _p(oo), _p(obs), mo, _p(bbox), float(inflate), dc.Z_GROUND, cap_pf, max_faces,
                      _p(goal), _p(face_ofs), _p(Ab), _p(xf), _p(pos), _p(status), csr_threads)
    return dict(poly_ofs=po, face_ofs=face_ofs[:po[-1] + 1], Ab=Ab, xf=xf, pos=pos, status=status)


def host_round(p1, p2, obs, inflate, k, row):
    """The host's carving round k of segment (p1, p2): (distance of its pick, the smallest host distance of the remaining
    points on the plane `row` -- the point that plane was cut at -- and that point's |a.p - b|), or None when the round does
    not exist."""
    c = lambda a: np.ascontiguousarray(a, np.float64)  # noqa: E731
    obs, out = c(np.reshape(obs, (-1, 3))), np.zeros(3)
    rc = _lib().emu_host_round(_p(c(p1)), _p(c(p2)), _p(obs), len(obs), _p(c(dc.BBOX)), float(inflate), int(k), _p(c(row)), _p(out))
    return None if rc else tuple(out)


def _host_rows(path, obs, inflate):
    polys = capi.ellipsoid_decomp(path, obs, dc.BBOX, inflate, dc.Z_GROUND, cap_rows=8192)
    return [np.hstack([A, b[:, None]]) for A, b in polys]


def _assert_bit_equal(out, j, host):
    po, fo = out["poly_ofs"], out["face_ofs"]
    assert out["status"][j] == 0
    for s, rows in enumerate(host):
        a, b = fo[po[j] + s], fo[po[j] + s + 1]
        assert b - a == len(rows), (j, s)
        assert out["Ab"][a:b].tobytes() == rows.tobytes(), (j, s)


def test_host_decomposition_matches_its_golden(built_lib):
    """fq_ellipsoid_decomp's output did not change by one bit when its arithmetic moved into fq_decomp.h."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "decomp_host.npz"))
    cases = dc.all_cases()
    assert list(g["names"]) == [c[0] for c in cases]
    for k, (name, path, obs, r) in enumerate(cases):
        rows = _host_rows(path, obs, r)
        fo = np.concatenate([[0], np.cumsum([len(x) for x in rows])])
        assert np.array_equal(fo, g["face_ofs"][g["case_ofs"][k]:g["case_ofs"][k + 1]]), name
        assert np.vstack(rows).tobytes() == g["Ab"][g["row_ofs"][k]:g["row_ofs"][k + 1]].tobytes(), name


@pytest.mark.parametrize("group", ["forest", "random", "edge"])
def test_kernel_is_bit_equal_to_the_host(built_lib, group):
    """Each group in one emulated launch, several corridors per batch, against fq_ellipsoid_decomp case by case."""
    cases = {"forest": dc.forest_cases(range(6)), "random": dc.random_cases(), "edge": dc.edge_cases()}[group]
    for r in sorted({c[3] for c in cases}):
        sub = [c for c in cases if c[3] == r]
        out = emu_decomp([c[1] for c in sub], [c[2] for c in sub], r)
        for j, (name, path, obs, _) in enumerate(sub):
            _assert_bit_equal(out, j, _host_rows(path, obs, r))


def test_safe_path_starts_at_first(built_lib):
    """`first` (the chain's R) replaces vertex 0: the rows are those of the host on the path with R in front."""
    cases = dc.forest_cases(range(6, 9))[1::2]             # the three safe paths
    paths = [c[1].copy() for c in cases]
    R = np.zeros((len(paths), 9))
    for j, p in enumerate(paths):
        R[j, :3] = p[0] + np.array([0.05, -0.03, 0.02])
        p[0] = [7.0, 7.0, 7.0]                        # never read
    out = emu_decomp(paths, [c[2] for c in cases], 0.42, first=R)
    for j, (name, path, obs, r) in enumerate(cases):
        real = path.copy()
        real[0] = R[j, :3]
        _assert_bit_equal(out, j, _host_rows(real, obs, r))
    # no R (the whole sweep found nothing): the corridor is not run, its neighbours are
    R[1, :3] = np.nan
    out = emu_decomp(paths, [c[2] for c in cases], 0.42, first=R)
    assert list(out["status"]) == [0, ST["not_run"], 0]
    assert np.isnan(out["xf"][1]).all() and np.isnan(out["pos"][1]).all()
    po, fo = out["poly_ofs"], out["face_ofs"]
    assert fo[po[1]] == fo[po[2]]                          # its polytopes are empty
    # a safe corridor without segments (its path is the single vertex R): at rest at R, or not run without R
    one = [paths[0], paths[1][:1], paths[2]]
    R[1, :3] = [0.5, -0.25, 1.0]
    out = emu_decomp(one, [c[2] for c in cases], 0.42, first=R)
    assert list(out["status"]) == [0, 0, 0] and np.array_equal(out["pos"][1], R[1, :3]) and not out["xf"][1, 3:].any()
    R[1, :3] = np.nan
    out = emu_decomp(one, [c[2] for c in cases], 0.42, first=R)
    assert list(out["status"]) == [0, ST["not_run"], 0] and np.isnan(out["xf"][1]).all()


def test_dense_cloud_spills_to_global_memory(built_lib):
    """More survivors than the CTA keeps in shared memory: the rest live in the global slice, still bit-equal."""
    fit = _lib().emu_fit_pts()
    rng = np.random.default_rng(5)
    path = np.array([[0.0, 0.0, 1.0], [1.5, 0.4, 1.2], [2.5, 1.5, 1.1]])
    obs = rng.uniform([-2.5, -2.5, 0.0], [5.0, 4.0, 2.2], (4 * fit, 3))
    d = np.min([np.linalg.norm(np.cross(obs - a, obs - b), axis=1) / np.linalg.norm(b - a) for a, b in zip(path[:-1], path[1:])], axis=0)
    obs = obs[d > 0.5]
    host = _host_rows(path, obs, 0.2)
    out = emu_decomp([path], [obs], 0.2)
    _assert_bit_equal(out, 0, host)
    # segment 0's oriented box (line_segment.h:57-98, half sizes 2, 2, 1) holds more points than shared memory does
    p1, p2 = path[0], path[1]
    dirv = (p2 - p1) / np.linalg.norm(p2 - p1)
    dh = np.array([dirv[1], -dirv[0], 0.0]) / np.linalg.norm(dirv[:2])
    dv = np.cross(dirv, dh)
    q = obs - p1
    inside = (np.abs(q @ dh) <= 2) & (q @ dirv >= -2) & (q @ dirv <= np.linalg.norm(p2 - p1) + 2) & (np.abs(q @ dv) <= 1)
    assert inside.sum() > fit


def test_statuses_of_caps_and_degenerate_input(built_lib):
    cases = dc.forest_cases(range(3))[::2]                 # three whole corridors
    paths, clouds = [c[1] for c in cases], [c[2] for c in cases]
    ok = emu_decomp(paths, clouds, 0.42)
    assert list(ok["status"]) == [0, 0, 0]
    pf = np.diff(ok["face_ofs"])
    po = ok["poly_ofs"]
    # a polytope cap just below corridor 1's largest polytope fails corridor 1 (and any other with such a polytope) only
    cap = int(pf[po[1]:po[2]].max()) - 1
    out = emu_decomp(paths, clouds, 0.42, cap_pf=cap)
    for j in range(3):
        over = pf[po[j]:po[j + 1]].max() > cap
        assert out["status"][j] == (ST["poly_faces"] if over else 0)
        if not over:
            assert out["Ab"][out["face_ofs"][po[j]]:out["face_ofs"][po[j + 1]]].tobytes() == \
                   ok["Ab"][ok["face_ofs"][po[j]]:ok["face_ofs"][po[j + 1]]].tobytes()
    # a corridor cap just below corridor 0's rows
    rows = [int(ok["face_ofs"][po[j + 1]] - ok["face_ofs"][po[j]]) for j in range(3)]
    out = emu_decomp(paths, clouds, 0.42, max_faces=rows[0] - 1)
    for j in range(3):
        assert out["status"][j] == (ST["corridor_faces"] if rows[j] > rows[0] - 1 else 0)
    # a cloud over max_obs
    cap = len(clouds[1]) - 1
    out = emu_decomp(paths, clouds, 0.42, max_obs=cap)
    assert list(out["status"]) == [ST["cloud"] if len(c) > cap else 0 for c in clouds] and out["status"][1] == ST["cloud"]
    # a zero-length segment
    p = paths[2].copy()
    p[1] = p[0]
    out = emu_decomp([paths[0], paths[1], p], clouds, 0.42)
    assert list(out["status"]) == [0, 0, ST["zero_segment"]]
    assert np.isnan(out["xf"][2]).all()


def test_goal_rule_matches_numpy(built_lib):
    """E / M = G when every row of the last polytope has a.G - b <= 0 (LinearConstraint::inside), else the last vertex."""
    cases = dc.forest_cases(range(8))[::2]
    paths, clouds = [c[1] for c in cases], [c[2] for c in cases]
    rng = np.random.default_rng(3)
    goal = np.array([p[-1] + (rng.normal(size=3) * 0.3 if j % 2 else rng.normal(size=3) * 4.0) for j, p in enumerate(paths)])
    out = emu_decomp(paths, clouds, 0.42, goal=goal)
    po, fo = out["poly_ofs"], out["face_ofs"]
    n_in = 0
    for j, p in enumerate(paths):
        last = out["Ab"][fo[po[j + 1] - 1]:fo[po[j + 1]]]
        inside = not np.any(last[:, :3] @ goal[j] - last[:, 3] > 0)
        n_in += inside
        want = goal[j] if inside else p[-1]
        assert np.array_equal(out["pos"][j], want) and np.array_equal(out["xf"][j, :3], want)
        assert not out["xf"][j, 3:].any()
    assert 0 < n_in < len(paths)


def test_host_round_follows_the_host(built_lib):
    """host_round (which the GPU test uses to tell ties from differences) picks, at every round, the point on the host's own
    row of that round: its best distance and the distance of the point on the row are the same point's."""
    n = 0
    for name, path, obs, r in dc.forest_cases(range(4)):
        for s, rows in enumerate(_host_rows(path, obs, r)):
            for k in range(len(rows) - 7):
                best, on_row, res = host_round(path[s], path[s + 1], obs, r, k, rows[k])
                assert best == on_row and res <= 1e-12, (name, s, k)
                n += 1
            assert host_round(path[s], path[s + 1], obs, r, len(rows) - 7, rows[0]) is None
    assert n > 50


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_pair_decomp));\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_decomp, %s));\n' % f for f, _ in capi.PairDecomp._fields_) +
                   'printf(" %d %d %d %d %d %d", FQ_DECOMP_OK, FQ_DECOMP_POLY_FACES, FQ_DECOMP_CORRIDOR_FACES, FQ_DECOMP_CLOUD,'
                   ' FQ_DECOMP_ZERO_SEGMENT, FQ_DECOMP_NOT_RUN);\n'
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    nf = len(capi.PairDecomp._fields_)
    assert got[0] == C.sizeof(capi.PairDecomp)
    assert got[1:1 + nf] == [getattr(capi.PairDecomp, f).offset for f, _ in capi.PairDecomp._fields_]
    assert got[1 + nf:] == [ST[k] for k in ("ok", "poly_faces", "corridor_faces", "cloud", "zero_segment", "not_run")]


def test_decomp_dev_submission_through_the_emulated_kernels(built_lib, oracle):
    """fq_replan_pairs_decomp_dev's kernels in submission order (run_chain with per-corridor lists) on three forest corridors,
    one of which fails its whole decomposition (a zero-length segment): decompose whole -> dt base from E -> offsets and
    expansion -> solve on the emulated CSR -> select -> winners' solve -> R -> decompose safe from R -> the safe half ->
    records.  Against the CPU chain on the corridors the host cuts from the same paths, the safe ones around the chain's R."""
    from faster_b200 import corridor as cr
    from test_kernel_emu_cpu import solve_multi, _emu, _pair_lib
    from test_pair_assign_cpu import offsets, expand, _lib as _assign_lib
    import pair_assign_oracle as pao
    ps = [cr.forest_pair_paths(9000 + s) for s in (0, 1, 2)]
    ps[1] = dict(ps[1])
    ps[1]["path_whole"] = np.vstack([ps[1]["path_whole"][:1], ps[1]["path_whole"]])     # corridor 1 fails
    P, N, DC, r_frac, lim_ = 3, 10, ps[0]["DC"], 0.6, 0
    fac = np.array([2.0, 3.0])
    cap_pf, max_faces = 64, 400
    K, S, A = _pair_lib(), _emu(), _assign_lib()
    c = lambda a, t: np.ascontiguousarray(a, t)  # noqa: E731
    x0, lim, goal = c([p["x0"] for p in ps], np.float64), c([p["lim"] for p in ps], np.float64), c([p["goal"] for p in ps], np.float64)
    st, corr = {}, {}
    for kind, ff in (("whole", True), ("safe", False)):
        xs = x0 if kind == "whole" else st["x0_safe"]
        d = emu_decomp([p["path_" + kind] for p in ps], [p["obs"] for p in ps], 0.42, first=None if kind == "whole" else xs, goal=goal,
                       cap_pf=cap_pf, max_faces=max_faces)
        corr[kind] = d
        po, fo, Ab, xf = d["poly_ofs"], d["face_ofs"], d["Ab"], c(d["xf"], np.float64)
        base = np.zeros(P)
        K.emu_dtbase(P, N, C.c_double(DC), _p(xs), _p(xf), _p(lim), _p(base))
        co = offsets(po, N, len(fac), lim_)
        dt, sig = expand(po, N, fac, lim_, base, co)
        feas, cost, _, _ = solve_multi(S, N, ff, xs, xf, lim, po, fo, Ab, co, dt, sig, max_faces=max_faces, max_poly_faces=cap_pf)
        wi, wc, wdt, ws, wo = np.zeros(P, np.int32), np.zeros(P), np.zeros(P), np.zeros((P, N), np.uint8), np.zeros(P + 1, np.int32)
        K.emu_select_multi(P, N, 0, _p(co), _p(dt), _p(sig), _p(feas), _p(cost), _p(wi), _p(wc), _p(wdt), _p(ws), _p(wo))
        _, _, coeffs, _ = solve_multi(S, N, ff, xs, xf, lim, po, fo, Ab, wo, wdt, ws, max_faces=max_faces, max_poly_faces=cap_pf)
        st[kind] = dict(base=base, wi=wi, wc=wc, wdt=wdt, ws=ws, co=co)
        if kind == "whole":
            x0s, nsamp, ksafe = np.zeros((P, 9)), np.zeros(P, np.int32), np.zeros(P, np.int32)
            K.emu_pair_mid(P, N, C.c_double(DC), C.c_double(r_frac), _p(c(coeffs, np.float64)), _p(wdt), _p(wi), _p(x0s), _p(nsamp), _p(ksafe))
            st["x0_safe"], st["nsamp"], st["ksafe"] = x0s, nsamp, ksafe
    res = np.zeros(P, capi.PAIR_RESULT_DTYPE)
    a, b = st["whole"], st["safe"]
    sw, ss = np.zeros((P, N), np.uint8), np.zeros((P, N), np.uint8)
    A.emu_pair_final_assign(P, len(fac), len(fac), N, N, _p(a["co"]), _p(b["co"]), _p(a["wi"]), _p(b["wi"]), _p(st["nsamp"]), _p(st["ksafe"]),
                            _p(a["wc"]), _p(b["wc"]), _p(a["wdt"]), _p(b["wdt"]), _p(a["base"]), _p(b["base"]), _p(st["x0_safe"]), _p(a["ws"]),
                            _p(b["ws"]), _p(sw), _p(ss), _p(res))
    # the failed corridor: no whole winner, so no R and no safe sweep; E / M NaN
    assert list(corr["whole"]["status"]) == [0, ST["zero_segment"], 0] and list(corr["safe"]["status"]) == [0, ST["not_run"], 0]
    assert res["whole_dt_index"][1] == -1 and res["safe_dt_index"][1] == -1 and np.isnan(res["R"][1]).all()
    assert np.isnan(corr["whole"]["xf"][1]).all() and np.isnan(corr["safe"]["xf"][1]).all()
    # the others against the CPU chain on the host's corridors (the safe paths from the chain's R)
    good = [0, 2]
    whole, safe = [], []
    for j in good:
        p = ps[j]
        sp = p["path_safe"].copy()
        sp[0] = st["x0_safe"][j][:3]
        for kind, path, lst in (("whole", p["path_whole"], whole), ("safe", sp, safe)):
            polys = capi.ellipsoid_decomp(path, p["obs"], dc.BBOX, 0.42, dc.Z_GROUND, cap_rows=8192)
            A_, b_ = polys[-1]
            xf = np.zeros(9)
            xf[:3] = p["goal"] if not np.any(A_ @ p["goal"] - b_ > 0) else path[-1]
            d = corr[kind]
            rows = np.vstack([np.hstack([q, r[:, None]]) for q, r in polys])
            assert d["Ab"][d["face_ofs"][d["poly_ofs"][j]]:d["face_ofs"][d["poly_ofs"][j + 1]]].tobytes() == rows.tobytes(), (kind, j)
            assert d["xf"][j].tobytes() == xf.tobytes(), (kind, j)
            lst.append(dict(N=N, x0=p["x0"], xf=xf, lim=p["lim"], polys=polys))
    w = capi.make_pair_workload(whole, safe, fac, np.zeros((0, N)), fac, np.zeros((0, N)), DC=DC, r_fraction=r_frac)
    o = pao.replan_pairs_assign(w, lim_, threads=4, dt_base_whole=res["whole_dt_base"][good], dt_base_safe=res["safe_dt_base"][good])
    r = res[good]
    for f in ("whole_dt_index", "whole_sigma_index", "safe_dt_index", "safe_sigma_index", "n_samples_whole", "k_safe"):
        assert np.array_equal(r[f], o[f]), f
    assert (r["whole_dt_index"] >= 0).all() and (r["safe_dt_index"] >= 0).all()
    assert np.abs(r["R"] - o["R"]).max() <= 1e-8
    assert (np.abs(r["safe_cost"] - o["safe_cost"]) / np.abs(o["safe_cost"])).max() <= 1e-8
