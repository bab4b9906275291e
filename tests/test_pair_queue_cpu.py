"""Each planner's committed plan kept in rings (fq_queue_*, fq_replan_pairs_queue*) without a GPU: the host entries against
tests/plan_queue_oracle.py (collections.deque) on random sequences of resets, selects, pops and appends; the product's ring
kernels (faster_b200/csrc/fq_pair.cuh) under the block emulation of tests/cpp/simt_emu/, bit-equal to the host entries at
several block sizes, with the chain's append kernel appending the pieces of tests/pair_plan_oracle.py; the refusals; and
the layouts of fq_queue and fq_pair_queue."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi

import pair_plan_oracle as ppo
import plan_queue_oracle as pqo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DC = 0.01
BLOCKS = [128, 1, 7, 32]
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_queue_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_queue_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
                os.path.join(ROOT, "include", "faster_b200.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_queue.argtypes = [C.c_int] * 3 + [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p] * 7 + [C.c_int, C.c_void_p]
        L.emu_queue.restype = None
        L.emu_pair_queue.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_double] + [C.c_void_p] * 8 + [C.c_int, C.c_int] + \
                                    [C.c_void_p] * 5 + [C.c_double, C.c_void_p, C.c_void_p]
        L.emu_pair_queue.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _rows(rows):
    return None if rows is None else np.ascontiguousarray(rows, np.int32)


def copy_ring(ring):
    return {k: v.copy() for k, v in ring.items()}


def emu_op(op, block, ring, n, rows=None, delta_t=pqo.DELTA_T, pos=None, ticks=None, max_ticks=0):
    """One ring kernel under the emulation on `ring` (updated in place).  -> (x0, k_end) for select, goals for pop."""
    n_rows, cap = ring["states"].shape[:2]
    x0, k_end = np.full((n, 9), -7.0), np.full(n, -7, np.int32)
    goals = np.full((n, max_ticks, 12), np.nan)
    pos = None if pos is None else np.ascontiguousarray(pos, np.float64)
    ticks = None if ticks is None else np.ascontiguousarray(ticks, np.int32)
    _lib().emu_queue(op, block, n, _p(_rows(rows)), n_rows, cap, delta_t, _p(ring["states"]), _p(ring["head"]), _p(ring["size"]),
                     _p(pos), _p(x0), _p(k_end), _p(ticks), max_ticks, _p(goals))
    return (x0, k_end) if op == 1 else goals


def random_batch(rng, n, none_share=0.15):
    """Winners of n corridors (whole N 4, safe N 3; short pieces of 6 .. 40 states) as test_pair_plan_cpu.batch builds them;
    a share of them without a whole or a safe winner, and some without a safe path needed."""
    import test_pair_plan_cpu as tpc
    dt_w = rng.uniform(0.02, 0.07, n)
    dt_s = rng.uniform(0.02, 0.06, n)
    lost = rng.random(n) < none_share
    dt_w[lost & (rng.random(n) < 0.5)] = np.nan
    dt_s[lost] = np.nan
    nw = [len(ppo.po.fill_x(4, np.zeros((4, 12)), d, DC)) if np.isfinite(d) else 1 for d in dt_w]
    k = [int(rng.integers(0, m)) for m in nw]
    need = (rng.random(n) > 0.2).astype(np.uint8)
    return tpc.batch(4, 3, rng.normal(0, 2, (n, 4, 12)), rng.normal(0, 2, (n, 3, 12)), dt_w, dt_s, k, need)


def pieces(b):
    """Each corridor's piece (pair_plan_oracle), None where the replan appends nothing."""
    states, ofs, st = ppo.plan(b["rec"], b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, b["need"])
    return [states[ofs[j]:ofs[j + 1]] if st[j] == ppo.PLAN_OK else None for j in range(len(st))]


def emu_append(block, b, ring, rows, k_end, G=None, goal_radius=0.3):
    """fq_pair_queue_kernel under the emulation on `ring` and k_end (in place).  -> (status, goal_seen)."""
    r = b["rec"]
    n = len(r["whole_dt"])
    n_rows, cap = ring["states"].shape[:2]
    wi = np.ascontiguousarray(np.concatenate([r["whole_dt_index"], r["safe_dt_index"]]), np.int32)
    wd = np.ascontiguousarray(np.concatenate([r["whole_dt"], r["safe_dt"]]), np.float64)
    Ns = np.array([b["N_w"], b["N_s"]], np.int32)
    need = None if b["need"] is None else np.ascontiguousarray(b["need"], np.uint8)
    st, seen = np.full(n, -9, np.int32), np.full(n, 9, np.uint8)
    G = None if G is None else np.ascontiguousarray(G, np.float64)
    _lib().emu_pair_queue(block, n, _p(Ns), DC, _p(wi), _p(wd), _p(np.ascontiguousarray(r["n_samples_whole"], np.int32)),
                          _p(np.ascontiguousarray(r["k_safe"], np.int32)), _p(need), _p(b["co_w"]), _p(b["co_s"]), _p(_rows(rows)),
                          n_rows, cap, _p(ring["states"]), _p(ring["head"]), _p(ring["size"]), _p(k_end), _p(G), goal_radius,
                          _p(st), _p(seen))
    return st, seen


def assert_ring_is(ring, plans, rows):
    for j, r in enumerate(rows):
        got = pqo.from_ring(ring, r)
        assert len(got) == len(plans[j]), (j, len(got), len(plans[j]))
        assert np.array(got).tobytes() == np.array(plans[j]).tobytes(), j


def ring_ops_agree(ring, n, rows, pos=None, ticks=None, max_ticks=0):
    """The emulated select (and pop / reset when given) at every block size, bit-equal to the host entries."""
    for block in BLOCKS:
        host, emu = copy_ring(ring), copy_ring(ring)
        want = capi.queue_select(host, n, rows)
        got = emu_op(1, block, emu, n, rows)
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
        if ticks is not None:
            want = capi.queue_pop(host, ticks, rows, max_ticks)
            got = emu_op(2, block, emu, n, rows, ticks=ticks, max_ticks=max_ticks)
            assert got.tobytes() == want.tobytes()
        if pos is not None:
            capi.queue_reset(host, pos, rows)
            emu_op(0, block, emu, n, rows, pos=pos)
        for k in host:
            assert host[k].tobytes() == emu[k].tobytes(), k


@pytest.mark.parametrize("seed", range(6))
def test_random_sequences_against_the_deque(built_lib, seed):
    """Resets, selects, pops between select and append (0, 1, delta_t - 1, delta_t or more) and appends, on permuted rows of
    rings with wrap-around, against the deques; every emulated kernel at every block size against the host entries."""
    rng = np.random.default_rng(seed)
    n, n_rows, cap = 7, 9, int(rng.choice([40, 64]))
    rows = rng.permutation(n_rows)[:n].astype(np.int32)
    ring = capi.queue_new(n_rows, cap)
    pos = rng.normal(0, 3, (n, 3))
    ring_ops_agree(ring, n, rows, pos=pos)
    capi.queue_reset(ring, pos, rows)
    plans = [pqo.reset(p) for p in pos]
    assert_ring_is(ring, plans, rows)
    seen_status, seen_k0, seen_first = set(), False, False
    for cycle in range(16):
        x0, k_end = capi.queue_select(ring, n, rows)
        for j in range(n):
            wx, wk = pqo.select(plans[j])
            assert x0[j].tobytes() == wx.tobytes() and k_end[j] == wk, (cycle, j)
            seen_k0 |= wk == 0
            seen_first |= len(plans[j]) == 1
        ticks = rng.choice([0, 1, pqo.DELTA_T - 1, pqo.DELTA_T, pqo.DELTA_T + 3], n).astype(np.int32)
        ring_ops_agree(ring, n, rows, ticks=ticks, max_ticks=16)
        goals = capi.queue_pop(ring, ticks, rows, 16)
        for j in range(n):
            want = pqo.pop(plans[j], int(ticks[j]))
            assert goals[j, :ticks[j]].tobytes() == want.tobytes() and np.isnan(goals[j, ticks[j]:]).all()
        assert_ring_is(ring, plans, rows)
        b = random_batch(rng, n)
        G = rng.normal(0, 3, (n, 3))
        ps = pieces(b)
        for j in range(n):                      # half the time, a goal right at the piece's end
            if ps[j] is not None and rng.random() < 0.5:
                G[j] = ps[j][-1, :3] + 0.1
        block = BLOCKS[cycle % len(BLOCKS)]
        ke = k_end.copy()
        st, gs = emu_append(block, b, ring, rows, ke, G)
        assert (ke == -1).all()
        for j in range(n):
            want = pqo.append(plans[j], int(k_end[j]), ps[j], cap)
            assert st[j] == want, (cycle, j, st[j], want)
            assert gs[j] == (want == pqo.QUEUE_OK and pqo.goal_seen(plans[j], G[j], 0.3)), (cycle, j)
            seen_status.add(int(want))
        assert_ring_is(ring, plans, rows)
        # k_end consumed: appending again without a select changes nothing
        st2, _ = emu_append(block, b, ring, rows, ke, G)
        assert (st2 == pqo.QUEUE_NONE).all()
        assert_ring_is(ring, plans, rows)
        after = rng.integers(0, 4, n).astype(np.int32)
        capi.queue_pop(ring, after, rows, 4)
        for j in range(n):
            pqo.pop(plans[j], int(after[j]))
    assert seen_k0 and seen_first
    assert {pqo.QUEUE_OK, pqo.QUEUE_NONE, pqo.QUEUE_PUBLISHED} <= seen_status, seen_status


def _plan_of(size, rng):
    return pqo.to_ring([[rng.normal(0, 1, 12) for _ in range(size)]], 64)


def test_delta_t_pops_between_select_and_append(built_lib):
    """delta_t - 1 pops between select and append: OK; delta_t: PUBLISHED, and the row is untouched."""
    rng = np.random.default_rng(3)
    b = random_batch(rng, 1, none_share=0.0)
    b["need"] = None
    b["rec"]["safe_dt"][0] = 0.03
    b["rec"]["safe_dt_index"][0] = 0
    piece = pieces(b)[0]
    for pops, want in [(pqo.DELTA_T - 1, pqo.QUEUE_OK), (pqo.DELTA_T, pqo.QUEUE_PUBLISHED)]:
        ring = _plan_of(25, rng)
        plan = pqo.from_ring(ring, 0)
        _, k_end = capi.queue_select(ring, 1)
        assert k_end[0] == 25 - pqo.DELTA_T
        capi.queue_pop(ring, [pops])
        pqo.pop(plan, pops)
        before = copy_ring(ring)
        st, _ = emu_append(32, b, ring, None, k_end.copy())
        assert st[0] == want == pqo.append(plan, int(k_end[0]), piece, 64)
        assert_ring_is(ring, [plan], [0])
        if want != pqo.QUEUE_OK:
            assert all(before[k].tobytes() == ring[k].tobytes() for k in ring)


def test_capacity_is_decided_per_row(built_lib):
    """A row whose piece would exceed cap is CAPACITY and untouched; the other rows append as if alone."""
    rng = np.random.default_rng(5)
    b = random_batch(rng, 3, none_share=0.0)
    ps = pieces(b)
    assert all(p is not None for p in ps)
    longest = max(len(p) for p in ps)
    cap = longest + 2
    plans = [[rng.normal(0, 1, 12) for _ in range(s)] for s in (3, cap, 1)]
    ring = pqo.to_ring(plans, cap, heads=[cap - 1, 3, 0])
    k_end = np.array([0, 0, 0], np.int32)     # the full row keeps cap - 1 states
    dq = [pqo.from_ring(ring, r) for r in range(3)]
    st, _ = emu_append(7, b, ring, None, k_end)
    want = [pqo.append(dq[j], 0, ps[j], cap) for j in range(3)]
    assert list(st) == want and want[1] == pqo.QUEUE_CAPACITY and want[0] == want[2] == pqo.QUEUE_OK
    assert_ring_is(ring, dq, [0, 1, 2])


def test_duplicated_and_invalid_rows(built_lib):
    """The device append gives every corridor naming a shared, out-of-range or invalid row FQ_QUEUE_ROWS and touches no such
    row; the host entries refuse duplicates (pop, reset), rows out of range and invalid rows; the device select / pop / reset
    skip them."""
    rng = np.random.default_rng(9)
    ring = pqo.to_ring([[rng.normal(0, 1, 12) for _ in range(s)] for s in (4, 5, 6, 7)], 64)
    ring["size"][3] = 65                                        # not a ring
    b = random_batch(rng, 5, none_share=0.0)
    rows = np.array([1, 0, 1, 9, 3], np.int32)
    before = copy_ring(ring)
    k_end = np.zeros(5, np.int32)
    st, gs = emu_append(32, b, ring, rows, k_end)
    assert list(st[[0, 2, 3, 4]]) == [pqo.QUEUE_ROWS] * 4 and st[1] in (pqo.QUEUE_OK, pqo.QUEUE_NONE)
    assert (k_end == -1).all() and not gs[[0, 2, 3, 4]].any()
    for r in (1, 2, 3):
        assert ring["states"][r].tobytes() == before["states"][r].tobytes() and ring["size"][r] == before["size"][r]
    for bad, msg in [([0, 0], "named twice"), ([0, 4], "outside"), ([3], "invalid row")]:
        with pytest.raises(capi.FqError, match=msg):
            capi.queue_pop(copy_ring(before), [1] * len(bad), bad, 1)
    with pytest.raises(capi.FqError, match="named twice"):
        capi.queue_reset(copy_ring(before), np.zeros((2, 3)), [2, 2])
    x0, k = capi.queue_select(copy_ring(before), 2, [1, 1])   # select only reads: a row may be named twice
    assert x0[0].tobytes() == x0[1].tobytes() and k[0] == k[1]
    e = copy_ring(before)
    x0, k = emu_op(1, 32, e, 3, [0, 9, 3])
    assert k[0] >= 0 and list(k[1:]) == [-1, -1] and np.isnan(x0[1:]).all()
    g = emu_op(2, 32, e, 3, [2, 2, 3], ticks=[1, 1, 1], max_ticks=1)
    assert np.isnan(g).all() and all(e[k].tobytes() == before[k].tobytes() for k in e)
    emu_op(0, 32, e, 2, [2, 2], pos=np.ones((2, 3)))
    assert all(e[k].tobytes() == before[k].tobytes() for k in e)
    for field, val, msg in [("cap", 0, "cap < 1"), ("delta_t", 0, "delta_t < 1"), ("n_rows", 0, "n_rows < 1"), ("states", None, "NULL")]:
        q = capi.queue_args(before)
        setattr(q, field, val)
        rc = capi.lib().fq_queue_select(C.byref(q), 1, None, np.zeros(9).ctypes.data, np.zeros(1, np.int32).ctypes.data)
        assert rc == -1 and msg in capi.lib().fq_last_error(None).decode()


def test_struct_layouts_match_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    body = 'printf("%zu %zu %d %d %d %d %d", sizeof(fq_queue), sizeof(fq_pair_queue), FQ_QUEUE_OK, FQ_QUEUE_NONE, ' \
           'FQ_QUEUE_PUBLISHED, FQ_QUEUE_CAPACITY, FQ_QUEUE_ROWS);\n'
    body += "".join('printf(" %%zu", offsetof(fq_queue, %s));\n' % f for f, _ in capi.Queue._fields_)
    body += "".join('printf(" %%zu", offsetof(fq_pair_queue, %s));\n' % f for f, _ in capi.PairQueue._fields_)
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\nint main(void) {\n' + body + "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[:2] == [C.sizeof(capi.Queue), C.sizeof(capi.PairQueue)]
    want = [capi.QUEUE_OK, capi.QUEUE_NONE, capi.QUEUE_PUBLISHED, capi.QUEUE_CAPACITY, capi.QUEUE_ROWS]
    assert got[2:7] == want == [pqo.QUEUE_OK, pqo.QUEUE_NONE, pqo.QUEUE_PUBLISHED, pqo.QUEUE_CAPACITY, pqo.QUEUE_ROWS]
    nq = len(capi.Queue._fields_)
    assert got[7:7 + nq] == [getattr(capi.Queue, f).offset for f, _ in capi.Queue._fields_]
    assert got[7 + nq:] == [getattr(capi.PairQueue, f).offset for f, _ in capi.PairQueue._fields_]


def test_bindings_refuse_arrays_they_would_misread(built_lib):
    """The ring, k_end and goals are read and written in place by address: a wrong element type, a non-contiguous view or
    a wrong shape is refused before any call."""
    ring = capi.queue_new(3, 8)
    capi.queue_reset(ring, np.zeros((3, 3)))
    for k, bad in [("states", ring["states"].astype(np.float32)), ("head", ring["head"].astype(np.int64)),
                   ("size", np.zeros(4, np.int32)), ("states", np.zeros((3, 16, 12))[:, ::2])]:
        with pytest.raises(ValueError, match="ring " + k):
            capi.queue_select(dict(ring, **{k: bad}), 3)
    with pytest.raises(ValueError, match="goals"):
        capi.queue_pop(ring, [1, 1, 1], goals=np.zeros((3, 1, 12), np.float32))
    with pytest.raises(ValueError, match="k_end"):
        capi.pair_queue_args(capi.queue_args(ring), None, np.zeros(3, np.int64), np.zeros(3, np.int32))
    with pytest.raises(ValueError, match="status"):
        capi.pair_queue_args(capi.queue_args(ring), None, np.zeros(3, np.int32), np.zeros(2, np.int32))
