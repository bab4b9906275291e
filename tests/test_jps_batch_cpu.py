"""Every planner's JPS search and JPS_in on the device (fq_jps_batch*) without a GPU: the product's kernels
(faster_b200/csrc/fq_jps.cuh) under the block emulation of tests/cpp/simt_emu/, at 1, 2 and 4 warps per CTA, bit-equal to
tests/jps_batch_oracle.py (the host search, fq_jps_in and the header's statuses) on forest planners and on the edge cases;
the refusals of both entries, the bindings' array checks, and the layouts of fq_jps_grids and fq_jps_batch_args."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi, corridor as cr

import jps_batch_oracle as jbo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WARPS = [1, 2, 4]
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libjps_batch_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "jps_batch_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
                os.path.join(ROOT, "include", "faster_b200.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_jps_batch.argtypes = [C.c_int, C.c_int, C.POINTER(capi.JpsBatchArgs)]
        L.emu_jps_batch.restype = None
        _LIB = L
    return _LIB


def _x0(A):
    A = np.asarray(A, np.float64).reshape(-1, 3)
    return np.ascontiguousarray(np.hstack([A, np.zeros((len(A), 6))]))


def emu(warps, grids, A, G, grid_index=None, pos=None, k_end=None, write_block=1024, **kw):
    """Both kernels under the emulation.  -> dict(in_ofs, in, status, k_end) as capi.jps_batch."""
    x0, G = _x0(A), np.ascontiguousarray(G, np.float64).reshape(-1, 3)
    n = len(G)
    max_in = kw.get("max_in", 512)
    gd = capi.jps_grids(grids)
    gi = None if grid_index is None else np.ascontiguousarray(grid_index, np.int32)
    pos = None if pos is None else np.ascontiguousarray(pos, np.float64).reshape(n, 3)
    ke = None if k_end is None else np.array(k_end, np.int32)
    out = dict(in_ofs=np.full(n + 1, -9, np.int32), status=np.full(n, -9, np.int32), **{"in": np.full((n * max_in, 3), 7.0)})
    a = capi.jps_batch_args(n, gd, x0, G, out, gi, pos, k_end=ke, **kw)
    _lib().emu_jps_batch(warps, write_block, C.byref(a))
    out["in"] = out["in"][:out["in_ofs"][-1]]
    out["k_end"] = ke
    return out


def agree(grids, A, G, warps=WARPS, **kw):
    """The emulated kernels at every warp count against the oracle.  -> the oracle's result."""
    want = jbo.batch(grids, _x0(A), G, **kw)
    for w in warps:
        jbo.assert_equal(emu(w, grids, A, G, **kw), want, "warps=%d" % w)
    return want


_FOREST = {}


def forest(n, start=0):
    """n forest planners (corridor.forest_jps seeds 50000 + start ..): each one's inflated grid, start and goal."""
    key = (n, start)
    if key not in _FOREST:
        out = []
        for seed in range(50000 + start, 50000 + start + n):
            fj = cr.forest_jps(seed)
            _, centres, radii = cr.make_forest(seed)
            grid, origin, res = cr.voxelise_forest(centres, radii, inflation=0.47)
            out.append(dict(grid=(grid, origin, res), start=np.asarray(fj["start"], np.float64), goal=np.asarray(fj["goal"], np.float64)))
        _FOREST[key] = out
    return _FOREST[key]


@pytest.mark.parametrize("use_jps", [True, False])
def test_forest_planners_per_planner_grids(built_lib, use_jps):
    """200 forest planners (JPS; A*: the first 8), each on its own grid, at 4 warps per CTA, and the first 24 at 1 and 2;
    k_end kept where a path is found."""
    pl = forest(200)[:200 if use_jps else 8]
    n = len(pl)
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    kw = dict(grid_index=np.arange(n), use_jps=use_jps, k_end=np.arange(n), pos=A + 0.25)
    want = agree([p["grid"] for p in pl], A, G, warps=[4], **kw)
    assert (want["status"] == jbo.OK).sum() >= n * 3 // 4
    m = min(24, n)
    agree([p["grid"] for p in pl[:m]], A[:m], G[:m], warps=[1, 2], **{k: (v[:m] if k != "use_jps" else v) for k, v in kw.items()})


def test_forest_planners_one_shared_grid(built_lib):
    """32 planners on one grid, starts and goals from other seeds' queries (some land in occupied cells: NO_PATH)."""
    pl = forest(32, 300)
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    want = agree([pl[0]["grid"]], A, G, k_end=np.zeros(len(pl)))
    st = set(want["status"].tolist())
    assert jbo.OK in st and jbo.NO_PATH in st, st


def _box(val=0):
    """A 12 x 10 x 6 grid of cells `val`, origin 0, res 0.5."""
    return np.full((6, 10, 12), val, np.int8), np.zeros(3), 0.5


def test_edge_cases(built_lib):
    """One cell (one-vertex path -> [start, goal]); start / goal occupied or outside; start z < 0; a walled-in goal
    (NO_PATH, k_end -1); G inside Ra; pos NULL and not."""
    g, o, r = _box()
    g[:, :, 8] = 100                                  # a wall across x = 8 .. walls in every goal beyond it
    g[2, 3, 3] = 100
    g[1, 1, 1] = -1                                   # unknown: not free
    grids = [(g, o, r)]
    A = [[0.3, 0.3, 0.3], [1.7, 1.7, 1.2], [0.2, 0.2, -0.7], [1.2, 1.2, 1.2], [0.8, 0.8, 0.8], [-1.0, 1.0, 1.0], [1.0, 1.0, 1.0],
         [0.5, 4.0, 2.0], [1.2, 1.2, 1.2]]
    G = [[0.4, 0.4, 0.4], [3.0, 3.0, 1.0], [3.0, 0.5, 0.5], [4.5, 4.5, 0.5], [1.7, 1.7, 1.2], [2.0, 2.0, 1.0], [9.0, 1.0, 1.0],
         [1.0, 4.5, 2.0], [0.7, 0.7, 0.7]]
    pos = np.array(A) + [[0.1, -0.2, 0.05]]
    for p in (None, pos):
        for use_jps in (True, False):
            want = agree(grids, A, G, pos=p, k_end=np.arange(9) + 5, Ra=1.0, use_jps=use_jps)
            # 1 start occupied, 3 goal walled in, 4 goal occupied, 5 start outside, 6 goal outside, 8 goal unknown; 2 start
            # z < 0, raised to 0: the grid's lower face, which rounds to the cell below it (outside)
            NP = jbo.NO_PATH
            assert list(want["status"]) == [jbo.OK, NP, NP, NP, NP, NP, NP, jbo.OK, NP], want["status"]
            assert want["in_ofs"][1] == 2             # one cell: [start, goal] (within Ra)
            assert want["in"][want["in_ofs"][2], 2] == 0.0   # the NO_PATH JPS_in starts at A with z raised to 0
            assert list(want["k_end"]) == [5, -1, -1, -1, -1, -1, -1, 12, -1]


def test_caps_and_inputs(built_lib):
    """max_nodes too small (NODES), max_in too small (LONG), a NaN A and grid_index out of range (INPUT)."""
    pl = forest(6, 40)
    grids = [p["grid"] for p in pl]
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    want = agree(grids, A, G, grid_index=np.arange(6), max_nodes=1, k_end=np.ones(6))
    assert (want["status"] != jbo.OK).all() and jbo.NODES in want["status"]
    want = agree(grids, A, G, grid_index=np.arange(6), max_in=3, dist_max=0.2)
    assert (want["status"] == jbo.LONG).sum() >= 4
    A2 = A.copy()
    A2[1, 0] = np.nan
    want = agree(grids, A2, G, grid_index=[0, 1, 7, -1, 4, 5], k_end=np.full(6, 3))
    assert list(want["status"][1:4]) == [jbo.INPUT] * 3 and list(want["k_end"][1:4]) == [-1] * 3
    nodes = [capi.jps3d_nodes(p["grid"][0], jbo.to_int(p["start"], *p["grid"][1:]), jbo.to_int(p["goal"], *p["grid"][1:])) for p in pl]
    cut = sorted(nodes)[3]                           # some searches fit, some need one node more than there is
    want = agree(grids, A, G, grid_index=np.arange(6), max_nodes=cut)
    assert list(want["status"] == jbo.NODES) == [k > cut for k in nodes]
    assert (want["status"] == jbo.NODES).any() and (want["status"] == jbo.OK).any()


def test_the_write_kernel_at_any_block_size(built_lib):
    pl = forest(9, 60)
    A = np.array([p["start"] for p in pl])
    G = np.array([p["goal"] for p in pl])
    want = jbo.batch([pl[0]["grid"]], _x0(A), G)
    for wb in (1, 5, 32, 1024):
        jbo.assert_equal(emu(2, [pl[0]["grid"]], A, G, write_block=wb), want, wb)


def _args(n=2, **over):
    g, o, r = _box()
    gd = capi.jps_grids([(g, o, r)])
    keep = dict(gd=gd, x0=_x0(np.full((n, 3), 0.3)), G=np.full((n, 3), 2.0),
                out=dict(in_ofs=np.zeros(n + 1, np.int32), status=np.zeros(n, np.int32), **{"in": np.zeros((n * 512, 3))}))
    a = capi.jps_batch_args(n, gd, keep["x0"], keep["G"], keep["out"])
    for k, v in over.items():
        if k in ("cells", "cell_ofs", "dims", "origin", "res", "n_grids"):
            setattr(a.grids, k, v)
        else:
            setattr(a, k, v)
    a.keep = keep
    return a


def test_refusals(built_lib):
    L = capi.lib()
    cases = [(dict(n_prob=0), "n_prob out of range"), (dict(cells=None), "NULL grid array"), (dict(n_grids=0), "n_grids < 1"),
             (dict(x0=None), "x0 / goal"), (dict(status=None), "in_ofs / in / status"), (dict(Ra=np.inf), "Ra must be finite"),
             (dict(dist_max=0.0), "dist_max"), (dict(dist_max=np.nan), "dist_max"), (dict(max_nodes=0), "max_nodes out of range"),
             (dict(max_nodes=(1 << 26) + 1), "max_nodes out of range"), (dict(max_in=1), "max_in out of range"),
             (dict(max_in=4097), "max_in out of range")]
    for over, msg in cases:
        a = _args(**over)
        for call in (lambda: L.fq_jps_batch(C.byref(a)), lambda: L.fq_jps_batch_dev(C.byref(a), None)):
            assert call() == -1
            assert msg in L.fq_last_error(None).decode(), (over, L.fq_last_error(None))
    assert L.fq_jps_batch(None) == -1 and L.fq_jps_batch_dev(None, None) == -1
    # the host entry reads the grids and the inputs
    for mutate, msg in [(lambda k: k["gd"]["dims"].__setitem__((0, 1), 0), "dimension <= 0"),
                        (lambda k: k["gd"]["dims"].__setitem__((0, 1), 1 << 28), "more than 2^31"),
                        (lambda k: k["gd"]["res"].__setitem__(0, -0.5), "res must be finite"),
                        (lambda k: k["gd"]["origin"].__setitem__((0, 2), np.nan), "non-finite origin"),
                        (lambda k: k["gd"]["cell_ofs"].__setitem__(0, -1), "negative cell_ofs"),
                        (lambda k: k["x0"].__setitem__((1, 2), np.inf), "non-finite A, G or pos"),
                        (lambda k: k["G"].__setitem__((0, 0), np.nan), "non-finite A, G or pos")]:
        a = _args()
        mutate(a.keep)
        assert L.fq_jps_batch(C.byref(a)) == -1 and msg in L.fq_last_error(None).decode(), msg
    a = _args()
    idx = np.array([0, 1], np.int32)
    a.grid_index = idx.ctypes.data
    assert L.fq_jps_batch(C.byref(a)) == -1 and "grid_index out of range" in L.fq_last_error(None).decode()
    pos = np.array([[0.0, 0.0, np.nan], [0.0, 0.0, 0.0]])
    a = _args()
    a.pos = pos.ctypes.data
    assert L.fq_jps_batch(C.byref(a)) == -1 and "non-finite A, G or pos" in L.fq_last_error(None).decode()
    assert capi.has_feature("jps_batch")


def test_bindings_refuse_arrays_they_would_misread(built_lib):
    g, o, r = _box()
    gd = capi.jps_grids([(g, o, r)])
    x0, G = _x0(np.zeros((2, 3))), np.ones((2, 3))
    out = dict(in_ofs=np.zeros(3, np.int32), status=np.zeros(2, np.int32), **{"in": np.zeros((2 * 512, 3))})
    for k, bad in [("in_ofs", np.zeros(3, np.int64)), ("status", np.zeros(3, np.int32)), ("in", np.zeros((2 * 512, 3), np.float32))]:
        with pytest.raises(ValueError, match=k):
            capi.jps_batch_args(2, gd, x0, G, dict(out, **{k: bad}))
    with pytest.raises(ValueError, match="x0"):
        capi.jps_batch_args(2, gd, np.zeros((2, 3)), G, out)
    with pytest.raises(ValueError, match="goal"):
        capi.jps_batch_args(2, gd, x0, np.ones((2, 3))[:, ::-1], out)
    with pytest.raises(ValueError, match="grid cells"):
        capi.jps_batch_args(2, dict(gd, cells=gd["cells"].astype(np.uint8)), x0, G, out)
    with pytest.raises(ValueError, match="k_end"):
        capi.jps_batch_args(2, gd, x0, G, out, k_end=np.zeros(2, np.int64))


def test_struct_layouts_match_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    body = 'printf("%zu %zu %d %d %d %d %d", sizeof(fq_jps_grids), sizeof(fq_jps_batch_args), FQ_JPS_OK, FQ_JPS_NO_PATH, ' \
           'FQ_JPS_NODES, FQ_JPS_LONG, FQ_JPS_INPUT);\n'
    body += "".join('printf(" %%zu", offsetof(fq_jps_grids, %s));\n' % f for f, _ in capi.JpsGrids._fields_)
    body += "".join('printf(" %%zu", offsetof(fq_jps_batch_args, %s));\n' % f for f, _ in capi.JpsBatchArgs._fields_)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\nint main(void) {\n' + body + "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:2] == [C.sizeof(capi.JpsGrids), C.sizeof(capi.JpsBatchArgs)]
    assert got[2:7] == [capi.JPS_OK, capi.JPS_NO_PATH, capi.JPS_NODES, capi.JPS_LONG, capi.JPS_INPUT] == [0, 1, 2, 3, 4]
    ng = len(capi.JpsGrids._fields_)
    assert got[7:7 + ng] == [getattr(capi.JpsGrids, f).offset for f, _ in capi.JpsGrids._fields_]
    assert got[7 + ng:] == [getattr(capi.JpsBatchArgs, f).offset for f, _ in capi.JpsBatchArgs._fields_]
