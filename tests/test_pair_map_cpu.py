"""The chained replan against indexed maps (fq_replan_pairs_map*) without a GPU: a numpy restatement of the map's index
(faster_b200/csrc/fq_map.h, fq_map.cu), and the product's kernel source with a map (fq_decomp.cuh, fq_pair.cuh) under the block
emulation of tests/cpp/simt_emu/ on that index.  The decomposition is bit for bit fq_ellipsoid_decomp on the full clouds
(whole: O, safe: U ++ O), including a segment that spills and exact distance ties between points of different cells; H/R is
bit for bit tests/pair_hr_oracle.py, with points on cell faces and at drone_radius; at three cell edges.  Also the ctypes
layout of fq_pair_map."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import decomp_cases as dc
import pair_hr_oracle as hro
from test_pair_hr_cpu import DC, N, _edge_cases, forest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
ST = capi.DECOMP_STATUS
EDGES = [0.15, 0.5, 2.0]


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_map_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_map_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h")] + \
               [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_decomp_map.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 8 + [C.c_int] + [C.c_void_p] * 3 + [C.c_int] * 3 + \
                                    [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_int] + [C.c_void_p] * 6
        L.emu_pair_hr_map.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double] + [C.c_void_p] * 10 + [C.c_int] + [C.c_void_p] * 3
        for f in (L.emu_decomp_map, L.emu_pair_hr_map):
            f.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def build_index(occ, unk, edge=0.5):
    """The map's index, restated: one grid over the finite points of U ++ O (origin at their minimum, cell edge `edge`
    doubled until at most min(max(65536, 4 n), 2^26) cells), and per cloud its points sorted stably by cell, their indices,
    and every cell's first sorted point.  Non-finite points get the cell past the last one."""
    occ, unk = np.reshape(occ, (-1, 3)).astype(np.float64), np.reshape(unk, (-1, 3)).astype(np.float64)
    allp = np.vstack([unk, occ])
    fin = np.isfinite(allp).all(axis=1)
    limit = min(max(65536, 4 * len(allp)), 1 << 26)
    origin = allp[fin].min(axis=0) if fin.any() else np.zeros(3)
    ext = allp[fin].max(axis=0) - origin if fin.any() else np.zeros(3)
    cell = float(edge)
    while np.prod(np.floor(ext / cell) + 1) > limit:
        cell *= 2
    dims = (np.floor(ext / cell) + 1).astype(np.int64)
    n_cells = int(np.prod(dims))

    def cloud(pts):
        ok = np.isfinite(pts).all(axis=1)
        with np.errstate(invalid="ignore"):
            c = np.clip(np.floor((pts - origin) / cell), 0, dims - 1)
        key = np.where(ok, (c[:, 2] * dims[1] + c[:, 1]) * dims[0] + c[:, 0], n_cells).astype(np.int64)
        order = np.argsort(key, kind="stable")
        start = np.searchsorted(key[order], np.arange(n_cells + 1), side="left").astype(np.int32)
        xyz = np.ascontiguousarray(pts[order] if len(pts) else np.zeros((1, 3)))
        return xyz, np.ascontiguousarray(order.astype(np.int32) if len(pts) else np.zeros(1, np.int32)), start, len(pts)

    return dict(grid=np.array([*origin, cell]), dims=dims.astype(np.int32), unk=cloud(unk), occ=cloud(occ))


def _cloud_args(c):
    return [_p(c[0]), _p(c[1]), _p(c[2]), c[3]]


def emu_decomp_map(paths, index, safe, max_local=8192, first=None, cap_pf=256, max_faces=2048):
    """One sweep of the device decomposition against one map under the emulation (safe: U ++ O, else O)."""
    n = len(paths)
    po = np.concatenate([[0], np.cumsum([len(p) - 1 for p in paths])]).astype(np.int32)
    path = np.ascontiguousarray(np.vstack(paths), np.float64)
    mp = int(np.diff(po).max())
    face_ofs = np.zeros(n * mp + 1, np.int32)
    Ab = np.zeros((n * max_faces, 4))
    xf, pos, status = np.zeros((n, 9)), np.zeros((n, 3)), np.full(n, -1, np.int32)
    bbox = np.asarray(dc.BBOX, np.float64)
    first = None if first is None else np.ascontiguousarray(first, np.float64)
    _lib().emu_decomp_map(n, mp, _p(po), _p(path), _p(first), _p(index["grid"]), _p(index["dims"]), *_cloud_args(index["unk"]),
                          *_cloud_args(index["occ"]), int(safe), int(max_local), _p(bbox), 0.42, dc.Z_GROUND, cap_pf, max_faces, None,
                          _p(face_ofs), _p(Ab), _p(xf), _p(pos), _p(status))
    return dict(poly_ofs=po, face_ofs=face_ofs[:po[-1] + 1], Ab=Ab, status=status)


def _host_rows(path, obs):
    polys = capi.ellipsoid_decomp(path, obs, dc.BBOX, 0.42, dc.Z_GROUND, cap_rows=8192)
    return [np.hstack([A, b[:, None]]) for A, b in polys]


def _assert_bit_equal(out, j, host):
    po, fo = out["poly_ofs"], out["face_ofs"]
    assert out["status"][j] == 0
    for s, rows in enumerate(host):
        a, b = fo[po[j] + s], fo[po[j] + s + 1]
        assert b - a == len(rows), (j, s)
        assert out["Ab"][a:b].tobytes() == rows.tobytes(), (j, s)


def _forest_maps(k=3):
    ps = [cr.forest_pair_paths(30000 + s) for s in range(k)]
    return [(p, np.asarray(p["obs"], np.float64), cr.forest_unknown_cloud(p)) for p in ps]


def test_index_restatement_holds_every_point_in_its_cell(built_lib):
    rng = np.random.default_rng(1)
    occ = rng.uniform(-3, 3, (500, 3))
    unk = rng.uniform(-1, 5, (700, 3))
    unk[5] = np.nan
    for edge in EDGES:
        ix = build_index(occ, unk, edge)
        g, d = ix["grid"], ix["dims"]
        for pts, (xyz, idx, start, n) in ((unk, ix["unk"]), (occ, ix["occ"])):
            fin = np.isfinite(pts).all(axis=1)
            assert start[-1] == fin.sum() and n == len(pts)
            assert np.array_equal(xyz[:start[-1]], pts[idx[:start[-1]]])
            for c in range(int(np.prod(d))):
                seg = idx[start[c]:start[c + 1]]
                assert np.all(np.diff(seg) > 0)                        # (cell, index) order
                cz, cy, cx = c // (d[0] * d[1]), (c // d[0]) % d[1], c % d[0]
                lo = g[:3] + np.array([cx, cy, cz]) * g[3]
                inside = (pts[seg] >= lo - 1e-9) | (np.array([cx, cy, cz]) == 0)
                assert inside.all()


@pytest.mark.parametrize("edge", EDGES)
def test_decomposition_equals_the_host_on_the_full_clouds(built_lib, edge):
    """Whole against O and safe against U ++ O, bit for bit fq_ellipsoid_decomp on the whole cloud."""
    for p, occ, unk in _forest_maps():
        ix = build_index(occ, unk, edge)
        out = emu_decomp_map([p["path_whole"]], ix, safe=False)
        _assert_bit_equal(out, 0, _host_rows(p["path_whole"], occ))
        out = emu_decomp_map([p["path_safe"]], ix, safe=True)
        _assert_bit_equal(out, 0, _host_rows(p["path_safe"], np.vstack([unk, occ])))


def test_dense_segment_spills_and_max_local_caps_it(built_lib):
    fit = 1024                                                        # fqd::kFitPts
    rng = np.random.default_rng(5)
    path = np.array([[0.0, 0.0, 1.0], [1.5, 0.4, 1.2], [2.5, 1.5, 1.1]])
    obs = rng.uniform([-2.5, -2.5, 0.0], [5.0, 4.0, 2.2], (4 * fit, 3))
    d = np.min([np.linalg.norm(np.cross(obs - a, obs - b), axis=1) / np.linalg.norm(b - a) for a, b in zip(path[:-1], path[1:])], axis=0)
    obs = obs[d > 0.5]
    unk, occ = obs[::2], obs[1::2]
    host = _host_rows(path, np.vstack([unk, occ]))
    for edge in EDGES:
        ix = build_index(occ, unk, edge)
        out = emu_decomp_map([path], ix, safe=True, max_local=len(obs))
        _assert_bit_equal(out, 0, host)
    # segment 0 keeps more survivors than shared memory holds; below them the segment is refused, the other corridor not
    other = np.array([[5.5, 3.0, 1.0], [6.5, 3.5, 1.2]])                 # at the cloud's corner: few points in its box
    out = emu_decomp_map([path, other], build_index(occ, unk), safe=True, max_local=fit + 8)
    assert out["status"][0] == ST["cloud"] and out["status"][1] == 0
    _assert_bit_equal(out, 1, _host_rows(other, np.vstack([unk, occ])))


def _lattice_ties():
    """Voxel centres on both sides of an axis-aligned segment: mirror points are at exactly equal ellipsoid distances,
    so the host's "first strict minimum" decides between points of different cells."""
    path = np.array([[0.0, 0.0, 1.0], [1.2, 0.0, 1.0]])
    g = np.arange(-1.05, 2.3, 0.15)
    X, Y, Z = np.meshgrid(g, np.arange(-1.05, 1.06, 0.15), np.arange(0.25, 1.8, 0.15), indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel()], axis=1)
    keep = np.hypot(pts[:, 1], pts[:, 2] - 1.0) > 0.55
    return path, pts[keep]


def test_ties_between_cells_follow_the_cloud_index(built_lib):
    path, pts = _lattice_ties()
    fwd, rev = pts, pts[::-1].copy()
    h_fwd, h_rev = _host_rows(path, fwd), _host_rows(path, rev)
    assert any(a.tobytes() != b.tobytes() for a, b in zip(h_fwd, h_rev))   # the cloud order decides a tie
    for edge in EDGES:
        for cloud, host in ((fwd, h_fwd), (rev, h_rev)):
            half = len(cloud) // 3
            _assert_bit_equal(emu_decomp_map([path], build_index(cloud, np.zeros((0, 3)), edge), safe=False), 0, host)
            _assert_bit_equal(emu_decomp_map([path], build_index(cloud[half:], cloud[:half], edge), safe=True), 0, host)


def emu_hr_map(coeffs, dt, unk, lim, params=(0.42, 0.5, 1.0), edge=0.5, block=256, occ=None):
    n = len(dt)
    co = np.ascontiguousarray(coeffs, np.float64)
    dt = np.ascontiguousarray(dt, np.float64)
    wi = np.where(np.isfinite(dt), 0, -1).astype(np.int32)
    lim = np.ascontiguousarray(lim, np.float64)
    ix = build_index(np.zeros((0, 3)) if occ is None else occ, unk, edge)
    pr = np.asarray(params, np.float64)
    r, need, ih = np.full(n, 77, np.int32), np.full(n, 9, np.uint8), np.full(n, 77, np.int32)
    _lib().emu_pair_hr_map(block, n, N, DC, _p(pr), _p(co), _p(dt), _p(wi), _p(lim), _p(ix["grid"]), _p(ix["dims"]), *_cloud_args(ix["unk"]),
                           _p(r), _p(need), _p(ih))
    return need, ih, r


def _assert_hr(out, co, dt, unk, lim, params):
    need, ih, r = out
    h = hro.hr_of(co, dt, N, DC, unk, lim[1], *params)
    assert (need, ih) == (h["need_safe"], h["index_H"])
    assert r == (h["k_safe"] if h["need_safe"] else -1)


@pytest.mark.parametrize("edge", EDGES)
def test_h_and_r_equal_the_restatement_on_forest_corridors(built_lib, edge):
    ps, co, dt = forest()
    hits = 0
    for j, p in enumerate(ps):
        if not np.isfinite(dt[j]):
            continue
        for params in ((0.42, 0.5, 1.0), (0.6, 0.2, 0.5)):
            out = emu_hr_map(co[j:j + 1], dt[j:j + 1], p["unk"], p["lim"][None], params, edge, occ=p["obs"])
            _assert_hr([x[0] for x in out], co[j], dt[j], p["unk"], p["lim"], params)
            hits += int(out[0][0])
    assert hits > 0


@pytest.mark.parametrize("edge", EDGES)
def test_h_and_r_edges_on_cell_faces_and_at_the_radius(built_lib, edge):
    """The hand-built clouds of test_pair_hr_cpu, each with an anchor point that puts the grid's origin a whole number of
    cells below its first point, so that point lies exactly on a cell face."""
    lim = np.array([5.0, 5.0, 8.0])
    for name, co, dt, cloud, params, _ in _edge_cases():
        cloud = np.reshape(cloud, (-1, 3))
        if len(cloud):
            # the point is exactly 4 cells above the origin (0.15 m: 4 cells are not exact in double, so only nearly)
            anchor = cloud[0] - 4 * edge
            assert np.all((cloud[0] - anchor) / edge == 4.0) or edge == 0.15, name
            cloud = np.vstack([cloud, anchor[None]])
        for block in (32, 256):
            out = emu_hr_map(co[None], np.array([dt]), cloud, lim[None], params, edge, block)
            _assert_hr([x[0] for x in out], co, dt, cloud, lim, params)


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu", sizeof(fq_pair_map));\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_map, %s));\n' % f for f, _ in capi.PairMap._fields_) + "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.PairMap)
    assert got[1:] == [getattr(capi.PairMap, f).offset for f, _ in capi.PairMap._fields_]
