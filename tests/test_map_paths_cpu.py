"""fq_jps_in and fq_paths_cloud (the host twin of fq_map_paths) against tests/paths_oracle.py, the restatement of
faster.cpp:80-97, :361-384, :767-921 and utils.cpp:690-866, :1117-1124: bit for bit, on forest corridors from the
product's own JPS and on the cases each branch of the reference is about.  Also every refusal and the struct layout."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import paths_oracle as po
from faster_b200 import capi, corridor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DR = 0.42                                    # drone_radius (faster.yaml)


def same(a, b):
    """byte-equal outputs (NaN rows included)"""
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = np.ascontiguousarray(a[k]), np.ascontiguousarray(b[k], dtype=np.asarray(a[k]).dtype)
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), (k, x, y)


def cloud_vs_oracle(paths, unks, dr=DR, mw=3, ms=4):
    got = capi.paths_cloud(paths, unks, dr, mw, ms)
    same(got, po.paths(paths, unks, dr, mw, ms))
    return got


def forest_case(seed):
    fj = corridor.forest_jps(seed)
    ra = min(np.linalg.norm(fj["goal"] - fj["start"]) - 0.001, 4.0)
    return fj, ra, corridor.forest_unknown_cloud(fj)


@pytest.fixture(scope="module")
def forest(built_lib):
    return [forest_case(seed) for seed in range(200)]


def test_jps_in_forest(forest):
    for fj, ra, _ in forest:
        got = capi.jps_in(fj["jps"], fj["start"], fj["goal"], ra, 1.5)
        want = po.jps_in(fj["jps"], fj["start"], fj["goal"], ra, 1.5)
        assert got.tobytes() == want.tobytes()


def test_paths_cloud_forest(forest):
    po.hits.clear()
    paths = [capi.jps_in(fj["jps"], fj["start"], fj["goal"], ra, 1.5) for fj, ra, _ in forest]
    got = cloud_vs_oracle(paths, [u for _, _, u in forest])
    assert (got["status"] == capi.PATHS_OK).all()
    assert 20 < got["crossed"].sum() < 180, got["crossed"].sum()
    assert po.hits.get("collision", 0) > 0 and po.hits.get("no_point_outside", 0) > 0
    for mw, ms in ((1, 1), (2, 3), (4, 2), (32, 32)):
        cloud_vs_oracle(paths[:40], [u for _, _, u in forest[:40]], mw=mw, ms=ms)


LINE = np.array([[0.0, 0, 1], [1.0, 0, 1], [2.0, 0, 1], [3.0, 0, 1], [4.0, 0, 1]])


def hit_after(key, paths, unks, **kw):
    po.hits.clear()
    out = cloud_vs_oracle(paths, unks, **kw)
    assert po.hits.get(key, 0) > 0, (key, po.hits)
    return out


def test_empty_unknown_space():
    out = hit_after("empty_unknown", [LINE], [np.zeros((0, 3))])
    assert out["crossed"][0] == 0 and out["path_safe"].tolist() == LINE.tolist()


def test_collision_at_the_start():
    out = hit_after("collision_at_start", [LINE], [[[0.1, 0.1, 1.0]]])
    assert out["crossed"][0] == 1 and out["path_safe"][1].tolist() == [0.01, 0.0, 1.0]


def test_no_approach():
    out = hit_after("no_point_outside", [LINE], [[[2.0, 30.0, 1.0], [-5.0, -5.0, 0.0]]])
    assert out["crossed"][0] == 0


@pytest.mark.parametrize("x", [1.0 + DR + 0.05, 1.0 + DR + 1e-9, 3.6, 3.9])
def test_collision_along_the_path(x):
    """an unknown point just past a vertex, or on the last segment"""
    out = hit_after("collision", [LINE], [[[x, 0.3, 1.0]]])
    assert out["crossed"][0] == 1


def test_reduce_over_several_segments():
    dense = np.array([[0.1 * i, 0.0, 1.0] for i in range(40)])
    hit_after("reduce_several_segments", [dense], [[[2.5, 0.35, 1.0]]], ms=32)


def test_discriminant_fallback():
    """A and B one float apart on the sphere's surface: a = b = 0.  Through the crop (the nearest point 1 m behind the
    start) and through the clip at ra."""
    path = np.array([[0.0, 0, 0], [1.0, 0, 0], [1.0 + 1e-12, 0, 0], [5.0, 0, 0]])
    hit_after("discriminant_fallback", [path], [[[-1.0, 0.0, 0.0]]], dr=0.1)
    po.hits.clear()
    got = capi.jps_in(path, path[0], path[-1], 1.0, 1.5)
    assert got.tobytes() == po.jps_in(path, path[0], path[-1], 1.0, 1.5).tobytes()
    assert po.hits.get("discriminant_fallback", 0) > 0


@pytest.mark.parametrize("mw,ms", [(1, 1), (2, 2), (3, 4), (4, 3)])
def test_max_poly(mw, ms):
    paths = [LINE, LINE[:2], LINE[:3] + 0.5]
    unks = [[[3.5, 0.2, 1.0]], [[0.5, 9.0, 1.0]], np.zeros((0, 3))]
    out = cloud_vs_oracle(paths, unks, mw=mw, ms=ms)
    assert list(np.diff(out["poly_ofs_whole"])) == [min(len(p) - 1, mw) for p in paths]


def test_jps_in_edge_cases():
    po.hits.clear()
    for jps, s, g, ra in (([[1.0, 1, 1]], [0.0, 0, 1], [0.5, 0, -2], 3.0),            # one point: [start, goal], z >= 0
                          (LINE, LINE[0], LINE[-1], 10.0),                             # entirely inside ra
                          (LINE, LINE[0], LINE[-1], 2.5),                              # clipped
                          (LINE, LINE[0], LINE[-1], -0.5),                             # ra < 0: the first vertex is outside
                          (LINE * 7, LINE[0] * 7, LINE[-1] * 7, 20.0)):                # createMoreVertexes
        got = capi.jps_in(jps, s, g, ra, 1.5)
        assert got.tobytes() == po.jps_in(jps, s, g, ra, 1.5).tobytes()
    for k in ("one_point_path", "inside_ra", "first_outside"):
        assert po.hits.get(k, 0) > 0, k


STALL_PATH = np.array([[0.0, 0, 1], [20.0, 0, 1]])
STALL_UNK = np.stack([np.arange(0, 20, 1e-3), np.full(20000, 2e-3), np.ones(20000)], axis=1)   # beside the whole path


def test_stall():
    """unknown space 2 mm beside a 20 m path and drone_radius 1 mm: every step advances about 2 mm, so the crop stops at
    FQ_PATHS_MAX_STEPS with FQ_PATHS_STALL and NaN paths; the other corridor is unaffected"""
    out = cloud_vs_oracle([STALL_PATH, LINE], [STALL_UNK, [[2.0, 0.3, 1.0]]], dr=1e-3)
    assert out["status"].tolist() == [capi.PATHS_STALL, capi.PATHS_OK]
    assert np.isnan(out["path_safe"][0]).all() and np.isnan(out["path_whole"][0]).all()


def _args(paths, out, **kw):
    in_ofs = np.concatenate([[0], np.cumsum([len(p) for p in paths])]).astype(np.int32)
    in_ = np.ascontiguousarray(np.vstack(paths), np.float64)
    s = capi.map_paths_args(len(paths), in_ofs.ctypes.data, in_.ctypes.data, {k: v.ctypes.data for k, v in out.items()}, **kw)
    s.keep = (in_ofs, in_, out)
    return s


def _out(n=2):
    return dict(poly_ofs_whole=np.zeros(n + 1, np.int32), poly_ofs_safe=np.zeros(n + 1, np.int32), path_whole=np.zeros((n * 33, 3)),
                path_safe=np.zeros((n * 33, 3)), status=np.zeros(n, np.int32), crossed=np.zeros(n, np.uint8))


def test_refusals(built_lib):
    L = capi.lib()
    uo, u = np.array([0, 1, 1], np.int32), np.array([[5.0, 5, 5]])

    def refused(s, text, unk_ofs=uo, unk=u):
        assert L.fq_paths_cloud(C.byref(s) if s is not None else None, unk_ofs.ctypes.data if unk_ofs is not None else None,
                                unk.ctypes.data) == -1
        assert text in L.fq_last_error(None).decode(), L.fq_last_error(None)

    ok = lambda **kw: _args([LINE, LINE], _out(), **kw)  # noqa: E731
    assert L.fq_paths_cloud(C.byref(ok()), uo.ctypes.data, u.ctypes.data) == 0
    refused(None, "p is NULL")
    s = ok(); s.n_prob = 0; refused(s, "n_prob")
    s = ok(); s.in_ofs = None; refused(s, "in_ofs / in")
    s = ok(); s.path_safe = None; refused(s, "poly_ofs_* / path_*")
    for dr in (0.0, -1.0, math.nan, math.inf):
        refused(ok(drone_radius=dr), "drone_radius")
    for mw, ms in ((0, 4), (3, 33), (-1, 1)):
        refused(ok(max_poly_whole=mw, max_poly_safe=ms), "max_poly")
    bad = _args([LINE, LINE], _out()); bad.keep[0][:] = [1, 3, 10]; refused(bad, "start at 0")
    bad = _args([LINE, LINE], _out()); bad.keep[0][:] = [0, 6, 5]; refused(bad, "decreasing")
    refused(_args([LINE, LINE[:1]], _out()), "fewer than 2")
    refused(_args([LINE, np.zeros((4097, 3))], _out()), "more than FQ_PATHS_MAX_IN")
    nan = LINE.copy(); nan[2, 1] = np.nan
    refused(_args([LINE, nan], _out()), "non-finite vertex")
    refused(ok(), "unk_ofs is NULL", unk_ofs=None)
    refused(ok(), "unk_ofs decreasing", unk_ofs=np.array([0, 1, 0], np.int32))
    refused(ok(), "non-finite unknown", unk=np.array([[np.inf, 0, 0]]))
    # the map entries check the maps before any device is touched
    s = ok()
    assert L.fq_map_paths(C.byref(s)) == -1 and "no maps" in L.fq_last_error(None).decode()
    assert L.fq_map_paths_dev(C.byref(s), None) == -1 and "no maps" in L.fq_last_error(None).decode()
    s.table = (C.c_void_p * 1)(None)
    s.maps, s.n_maps = C.addressof(s.table), 1
    assert L.fq_map_paths(C.byref(s)) == -1 and "a NULL map" in L.fq_last_error(None).decode()
    # fq_jps_in
    p, st, g = LINE.copy(), LINE[0].copy(), LINE[-1].copy()
    out = np.zeros((64, 3))

    def jin_refused(text, jps=p, n=5, s=st, goal=g, ra=4.0, d=1.5, o=out, cap=64):
        rc = L.fq_jps_in(jps.ctypes.data if jps is not None else None, n, s.ctypes.data if s is not None else None,
                         goal.ctypes.data, ra, d, o.ctypes.data if o is not None else None, cap)
        assert rc == -1 and text in L.fq_last_error(None).decode(), (rc, L.fq_last_error(None))
    jin_refused("n < 1", n=0)
    jin_refused("jps, start or goal NULL", s=None)
    jin_refused("cap < 0", cap=-1)
    jin_refused("out NULL", o=None)
    jin_refused("non-finite vertex", jps=nan)
    jin_refused("non-finite start", s=np.array([0.0, np.nan, 0]))
    jin_refused("ra must be finite", ra=math.inf)
    for d in (0.0, -1.0, math.nan):
        jin_refused("dist_max", d=d)
    jin_refused("2^30", d=1e-12, jps=LINE * 1e3)
    assert L.fq_jps_in(p.ctypes.data, 5, st.ctypes.data, g.ctypes.data, 4.0, 1.5, None, 0) == 5   # count only


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_map_paths_args));\n' +
                   "".join('printf(" %%zu", offsetof(fq_map_paths_args, %s));\n' % f for f, _ in capi.MapPathsArgs._fields_) +
                   "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.MapPathsArgs)
    assert got[1:] == [getattr(capi.MapPathsArgs, f).offset for f, _ in capi.MapPathsArgs._fields_]
