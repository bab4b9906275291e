"""H and R of the chained replan (fq_replan_pairs_hr*) without a GPU: the product's kernel source (faster_b200/csrc/fq_pair.cuh:
fq_pair_hr_kernel, fq_pair_mid_kernel with R's index, fq_pair_window_kernel with need_safe / last_factor_safe) under the block
emulation of tests/cpp/simt_emu/, bit for bit against tests/pair_hr_oracle.py on forest corridors and hand-built edges, at
several block sizes; and the kernels in submission order against the CPU chain with H and R."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import pair_hr_oracle as hro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
N, DC = 10, 0.01


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_hr_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_hr_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_pair_hr.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 10
        L.emu_pair_mid_hr.argtypes = [C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 7
        L.emu_pair_window_hr.argtypes = [C.c_int] * 3 + [C.c_void_p] * 14
        for f in (L.emu_pair_hr, L.emu_pair_mid_hr, L.emu_pair_window_hr):
            f.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def emu_hr(coeffs, dt, clouds, lim, params=(0.42, 0.5, 1.0), block=256, N_=N):
    """fq_pair_hr_kernel + fq_pair_mid_kernel on corridors with whole winners (coeffs n x N x 12, dt; NaN dt: no winner).
    -> dict(need, index_H, k_safe, n_samples, R)."""
    n = len(dt)
    co = np.ascontiguousarray(coeffs, np.float64)
    dt = np.ascontiguousarray(dt, np.float64)
    wi = np.where(np.isfinite(dt), 0, -1).astype(np.int32)
    lim = np.ascontiguousarray(lim, np.float64)
    uo = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    unk = np.ascontiguousarray(np.vstack([np.reshape(c, (-1, 3)) for c in clouds] + [np.zeros((1, 3))]), np.float64)
    pr = np.asarray(params, np.float64)
    r, need, ih = np.full(n, 77, np.int32), np.full(n, 9, np.uint8), np.full(n, 77, np.int32)
    L = _lib()
    L.emu_pair_hr(block, n, N_, DC, _p(pr), _p(co), _p(dt), _p(wi), _p(lim), _p(uo), _p(unk), _p(r), _p(need), _p(ih))
    x0s, ns, ks = np.zeros((n, 9)), np.zeros(n, np.int32), np.zeros(n, np.int32)
    L.emu_pair_mid_hr(n, N_, DC, _p(co), _p(dt), _p(wi), _p(r), _p(x0s), _p(ns), _p(ks))
    return dict(need=need, index_H=ih, k_safe=ks, n_samples=ns, R=x0s, r_index=r)


def assert_matches(out, coeffs, dt, clouds, lim, params=(0.42, 0.5, 1.0), N_=N):
    for j in range(len(dt)):
        if not np.isfinite(dt[j]):
            assert out["index_H"][j] == -1 and out["k_safe"][j] == -1 and out["need"][j] == 0 and np.isnan(out["R"][j]).all()
            continue
        h = hro.hr_of(coeffs[j], dt[j], N_, DC, clouds[j], lim[j][1], *params)
        assert (out["need"][j], out["index_H"][j], out["k_safe"][j], out["n_samples"][j]) == \
            (h["need_safe"], h["index_H"], h["k_safe"], h["n"]), j
        assert out["R"][j].tobytes() == h["R"].tobytes(), j


def _winners(ps):
    """The whole winners of forest replans through the CPU chain (host decomposition, the CPU port of the sweep)."""
    import pair_assign_oracle as pao
    from oracle import pair_oracle
    co, dt = [], []
    for p in ps:
        whole = hro.host_corridor(p["path_whole"], p["obs"], p["goal"], N, p["x0"], p["lim"])
        w = capi.make_pair_workload([whole], [whole], np.arange(1.0, 11.0), np.zeros((0, N)), np.arange(1.0, 11.0), np.zeros((0, N)), DC=DC)
        r = pair_oracle.replan_pairs(pao.with_own_lists(w, 0), threads=4, fast=True)
        co.append(r["coeffs_whole"][0])
        dt.append(r["whole_dt"][0])
    return np.array(co), np.array(dt)


_FOREST = {}


def forest(k=6):
    if k not in _FOREST:
        ps = [cr.forest_pair_paths(30000 + s) for s in range(k)]
        for p in ps:
            p["unk"] = cr.forest_unknown_cloud(p)
        co, dt = _winners(ps)
        _FOREST[k] = (ps, co, dt)
    return _FOREST[k]


@pytest.mark.parametrize("block", [32, 96, 256])
def test_kernel_is_bit_equal_to_the_restatement_on_forest_corridors(built_lib, block):
    ps, co, dt = forest()
    dt = dt.copy()
    dt[3] = np.nan                                          # a corridor without a whole winner
    clouds, lim = [p["unk"] for p in ps], np.array([p["lim"] for p in ps])
    out = emu_hr(co, dt, clouds, lim, block=block)
    assert_matches(out, co, dt, clouds, lim)
    assert 0 < out["need"].sum() < len(ps) - 1
    # and with delta_H = 0.5, a larger drone radius and a smaller delta_a
    params = (0.6, 0.2, 0.5)
    out = emu_hr(co, dt, clouds, lim, params, block=block)
    assert_matches(out, co, dt, clouds, lim, params)


def _line_coeffs(v=(4.0, 0.0, 0.0), p0=(0.0, 0.0, 1.0), dt=0.1, N_=N, accel=(0.0, 0.0, 0.0)):
    """Coefficients (N x 12, ax ay az bx by bz cx cy cz dx dy dz) of x(t) = p0 + v t + accel t^2 / 2, split at multiples of dt."""
    co = np.zeros((N_, 12))
    for t in range(N_):
        t0 = t * dt
        for ax in range(3):
            co[t, 3 + ax] = accel[ax] / 2
            co[t, 6 + ax] = v[ax] + accel[ax] * t0
            co[t, 9 + ax] = p0[ax] + v[ax] * t0 + accel[ax] * t0 * t0 / 2
    return co


def _edge_cases():
    """(name, coeffs, dt, cloud, params, what the restatement must say: (need, index_H, k_safe) or None)."""
    f32 = np.float32
    co = _line_coeffs()
    dt = 0.1
    X = capi.fill_x(N, co.reshape(-1), dt, DC)
    q = X[:, :3].astype(f32)
    cases = []
    # a point at float distance exactly 0.5 (= drone_radius) from query 0 in y, and one float ulp inside it
    on = q[0].copy()
    on[1] = q[0][1] + f32(0.5)
    assert f32(on[1] - q[0][1]) == f32(0.5)
    cases.append(("at_radius", co, dt, on[None].astype(np.float64), (0.5, 0.5, 1.0), (0, len(X) - 1, len(X) - 1)))
    inside = on.copy()
    inside[1] = np.nextafter(on[1], q[0][1])
    cases.append(("ulp_inside", co, dt, inside[None].astype(np.float64), (0.5, 0.5, 1.0), (1, 0, 0)))
    # a hit at query 0 exactly on the sample
    cases.append(("hit_at_0", co, dt, X[:1, :3].copy(), (0.42, 0.5, 1.0), (1, 0, 0)))
    # points 0.15 m beside samples 5, 15, 25: within a 0.2 m radius of those samples only, and 0.25 m from every query (the
    # trajectory moves 0.4 m between queries)
    cases.append(("off_query", co, dt, X[[5, 15, 25], :3] + [0, 0.15, 0], (0.2, 0.5, 1.0), None))
    # an empty cloud
    cases.append(("empty", co, dt, np.zeros((0, 3)), (0.42, 0.5, 1.0), (0, len(X) - 1, len(X) - 1)))
    # delta_H = 0.5: a hit at query 30 gives indexH 15
    cases.append(("delta_H_half", co, dt, X[30:31, :3] + [0, 0.1, 0], (0.3, 0.5, 0.5), (1, 15, None)))
    # n < 10: only query 0
    short = 0.008
    Xs = capi.fill_x(N, co.reshape(-1), short, DC)
    assert len(Xs) < 10
    cases.append(("n_below_10", co, short, Xs[-1:, :3] + [0, 0.1, 0], (0.42, 0.5, 1.0), (0, len(Xs) - 1, len(Xs) - 1)))
    # braking: H ahead in x, y velocity 0 (sign 0); delta_a chosen so that sample 0's braking distance equals |H - p| exactly
    # (not a hit) and one step smaller (a hit at 0)
    stop = _line_coeffs(v=(4.0, 0.0, 0.0), accel=(-6.0, 0.0, 0.0))
    Xb = capi.fill_x(N, stop.reshape(-1), dt, DC)
    hit = Xb[20:21, :3] + [0, 0.1, 0]
    d, v, a_max = Xb[20, 0] - Xb[0, 0], Xb[0, 3], 5.0
    da = v * v / (2 * a_max * d)
    for _ in range(64):
        b = np.sign(v * d) * (v * v) / (2 * da * a_max)
        if b == abs(d):
            break
        da = np.nextafter(da, np.inf if b > abs(d) else 0.0)
    assert np.sign(v * d) * (v * v) / (2 * da * a_max) == abs(d)
    assert Xb[0, 4] == 0
    cases.append(("brake_equal", stop, dt, hit, (0.15, da, 1.0), None))
    cases.append(("brake_above", stop, dt, hit, (0.15, np.nextafter(da, 0.0), 1.0), (1, 20, 0)))
    return cases


def test_edges_match_the_restatement(built_lib):
    for name, co, dt, cloud, params, want in _edge_cases():
        h = hro.hr_of(co, dt, N, DC, cloud, 5.0, *params)
        if want is not None:
            got = (h["need_safe"], h["index_H"], h["k_safe"])
            assert all(w is None or g == w for g, w in zip(got, want)), (name, got, want)
        if name == "off_query":
            assert h["need_safe"] == 0, name
        if name == "brake_equal":
            assert (h["need_safe"], h["index_H"]) == (1, 20) and h["k_safe"] != 0, name
        for block in (32, 256):
            out = emu_hr(co[None], np.array([dt]), [cloud], np.array([[5.0, 5.0, 8.0]]), params, block=block)
            assert_matches(out, co[None], np.array([dt]), [cloud], np.array([[5.0, 5.0, 8.0]]), params)


def test_window_kernel_without_a_safe_path(built_lib):
    """need_safe = 0: trials_safe 0, the safe window from last_factor_safe, last_factor_safe unchanged; need_safe = 1: the
    safe winner's factor becomes last_factor_safe; a NULL need_safe gives the old outputs."""
    import pair_window_oracle as pwo
    n, mf = 4, 10
    rec = np.zeros(n, capi.PAIR_RESULT_DTYPE)
    rec["whole_dt_index"] = [2, 3, -1, 4]
    rec["safe_dt_index"] = [-1, 1, -1, -1]
    fac = np.tile(np.arange(1.0, 11.0), (n, 1))
    ofs = np.array([0, 10, 20, 30, 40], np.int32)
    nf = np.full(n, 10, np.int32)
    wins = np.concatenate([np.ones(n), np.full(n, 10.0), np.ones(n), np.full(n, 10.0)])
    g = np.array([20.0, 20.0, 3.0, 4.0])
    need = np.array([0, 1, 0, 1], np.uint8)
    last = np.array([6.5, 6.5, 6.5, 6.5])
    factor, trials, nxt = np.zeros(2 * n), np.zeros(2 * n, np.int32), np.zeros(4 * n)
    L = _lib()
    L.emu_pair_window_hr(n, mf, mf, _p(rec), _p(ofs), _p(ofs), _p(nf), _p(nf), _p(fac), _p(fac), _p(wins), _p(g), _p(factor), _p(trials),
                         _p(nxt), _p(need), _p(last))
    assert list(trials[n:]) == [0, 2, 0, 10]
    assert list(last) == [6.5, 2.0, 6.5, 6.5]
    lo, hi = pwo.next_window(True, 6.5, 3.0, 4.0, 1.0, 10.0)
    assert (nxt[2 * n], nxt[3 * n]) == (lo, hi)                        # corridor 0: no safe path, whole won
    assert (nxt[2 * n + 2], nxt[3 * n + 2]) == (1.0, 10.0)             # corridor 2: no whole winner
    assert (nxt[2 * n + 3], nxt[3 * n + 3]) == (1.0, 10.0)             # corridor 3: the safe sweep ran and lost
    assert nxt[0] == max(3.0 - 20.0, 1.0) and nxt[n] == 23.0           # the whole window follows f*_whole
    assert nxt[3] == 1.0 and nxt[n + 3] == 10.0
    # NULL need_safe / last_factor_safe: as fq_replan_pairs_window
    f2, t2, n2 = np.zeros(2 * n), np.zeros(2 * n, np.int32), np.zeros(4 * n)
    L.emu_pair_window_hr(n, mf, mf, _p(rec), _p(ofs), _p(ofs), _p(nf), _p(nf), _p(fac), _p(fac), _p(wins), _p(g), _p(f2), _p(t2), _p(n2),
                         None, None)
    assert list(t2[n:]) == [10, 2, 0, 10] and (n2[2 * n], n2[3 * n]) == (1.0, 10.0)


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_pair_hr));\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_hr, %s));\n' % f for f, _ in capi.PairHR._fields_) + "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.PairHR)
    assert got[1:] == [getattr(capi.PairHR, f).offset for f, _ in capi.PairHR._fields_]


def test_hr_dev_submission_against_the_cpu_chain(built_lib):
    """fq_replan_pairs_hr_dev's H/R step in submission order -- whole winners -> fq_pair_hr_kernel -> fq_pair_mid_kernel -- on
    forest replans, then the safe corridors the host cuts around that R: every record field against pair_hr_oracle's CPU
    chain (which restates H and R itself)."""
    ps, co, dt = forest()
    clouds, lim = [p["unk"] for p in ps], np.array([p["lim"] for p in ps])
    out = emu_hr(co, dt, clouds, lim)
    fac = np.arange(1.0, 11.0)
    for j, p in enumerate(ps[:4]):
        ref = hro.replan_pair_hr(p, fac)
        assert ref["need_safe"] == out["need"][j] and ref["index_H"] == out["index_H"][j], j
        assert ref["k_safe"] == out["k_safe"][j] and ref["n_samples_whole"] == out["n_samples"][j], j
        assert np.array_equal(np.isnan(ref["R"]), np.isnan(out["R"][j])), j
        fin = np.isfinite(ref["R"])
        assert np.abs(ref["R"][fin] - out["R"][j][fin]).max(initial=0) <= 1e-8, j
        assert (ref["safe_dt_index"] >= 0) == bool(out["need"][j]), j           # a needed safe sweep wins on these corridors
