"""The committed plan of the chained replan (fq_replan_pairs_plan*) without a GPU: the product's two plan kernels
(faster_b200/csrc/fq_pair.cuh: fq_pair_plan_offsets_kernel, fq_pair_plan_sample_kernel) under the block emulation of
tests/cpp/simt_emu/, at several block sizes, bit for bit against tests/pair_plan_oracle.py (appendToPlan over the restated
fillX) on config-4 fixture winners, on hand-built edges and at every kind of capacity; the restatement against the
reference's own fillX where it is built; and the layout of fq_pair_plan."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from faster_b200 import capi

import pair_plan_oracle as ppo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_LIB = None
DC = 0.01
BLOCKS = [(1024, 128), (32, 1), (96, 7), (1, 32)]


def _lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(ROOT, "tests", "cpp", "_build", "libpair_plan_emu.so")
        csrc = os.path.join(ROOT, "faster_b200", "csrc")
        srcs = [os.path.join(ROOT, "tests", "cpp", "pair_plan_emu.cpp"), os.path.join(ROOT, "tests", "cpp", "simt_emu", "simt_emu.h"),
                os.path.join(ROOT, "include", "faster_b200.h")] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".h", ".cuh"))]
        if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "tests", "cpp"),
                                   "-I", os.path.join(ROOT, "tests", "cpp", "simt_emu"), "-I", csrc, "-I", os.path.join(ROOT, "include"),
                                   srcs[0], "-o", out])
        L = C.CDLL(out)
        L.emu_pair_plan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_double] + [C.c_void_p] * 7 + [C.c_longlong] + [C.c_void_p] * 3
        L.emu_pair_plan.restype = None
        _LIB = L
    return _LIB


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def batch(N_w, N_s, co_w, co_s, dt_w, dt_s, k, need=None):
    """The chain's intermediates for corridors with whole winners at dt_w (NaN: none) and safe winners at dt_s (NaN: none):
    n_samples and k_safe as fq_pair_mid_kernel leaves them (k: R's index; a corridor without a safe path needed gets n_w - 1).
    -> dict for emu / the oracle."""
    n = len(dt_w)
    dt_w, dt_s = np.asarray(dt_w, float), np.asarray(dt_s, float)
    ns = np.array([len(ppo.po.fill_x(N_w, co_w[j], dt_w[j], DC)) if np.isfinite(dt_w[j]) else 0 for j in range(n)], np.int32)
    ks = np.array([-1 if not np.isfinite(dt_w[j]) else (ns[j] - 1 if need is not None and not need[j] else k[j]) for j in range(n)], np.int32)
    rec = dict(whole_dt_index=np.where(np.isfinite(dt_w), 0, -1), safe_dt_index=np.where(np.isfinite(dt_s), 0, -1), whole_dt=dt_w,
               safe_dt=dt_s, k_safe=ks, n_samples_whole=ns)
    return dict(N_w=N_w, N_s=N_s, co_w=np.ascontiguousarray(co_w, float), co_s=np.ascontiguousarray(co_s, float), rec=rec,
                need=None if need is None else np.asarray(need, np.uint8))


def emu(b, cap=None, block_ofs=1024, block_rows=128, with_status=True):
    """fq_launch_pair_plan under the emulation.  -> (states (cap x 12, NaN where nothing was written), plan_ofs, status)."""
    r = b["rec"]
    n = len(r["whole_dt"])
    if cap is None:
        cap = ppo.plan(r, b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, b["need"])[1][-1]
    states = np.full((max(int(cap), 1), 12), np.nan)
    ofs, st = np.full(n + 1, -9, np.int64), np.full(n, -9, np.int32)
    wi = np.ascontiguousarray(np.concatenate([r["whole_dt_index"], r["safe_dt_index"]]), np.int32)
    wd = np.ascontiguousarray(np.concatenate([r["whole_dt"], r["safe_dt"]]), np.float64)
    Ns = np.array([b["N_w"], b["N_s"]], np.int32)
    need = None if b["need"] is None else np.ascontiguousarray(b["need"], np.uint8)
    _lib().emu_pair_plan(block_ofs, block_rows, n, _p(Ns), DC, _p(wi), _p(wd), _p(np.ascontiguousarray(r["n_samples_whole"], np.int32)),
                         _p(np.ascontiguousarray(r["k_safe"], np.int32)), _p(need), _p(b["co_w"]), _p(b["co_s"]), int(cap), _p(states),
                         _p(ofs), _p(st) if with_status else None)
    return states[:int(cap)], ofs, st


def assert_matches(b, cap=None, **kw):
    want = ppo.plan(b["rec"], b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, b["need"], cap)
    got = emu(b, cap, **kw)
    assert got[1].tobytes() == want[1].tobytes()
    assert got[2].tobytes() == want[2].tobytes()
    assert got[0].tobytes() == want[0].tobytes()
    return want


_FIX = {}


def fixture_batch():
    """Config-4 fixture corridors through the CPU chain (oracle/pair_oracle.py with the tuned port): their winners."""
    if "b" not in _FIX:
        import bench
        import pair_assign_oracle as pao
        from oracle import pair_oracle
        w = bench.load_cfg4(0, 4)
        r = pair_oracle.replan_pairs(pao.with_own_lists(w, 0), threads=4, fast=True)
        assert (r["whole_dt_index"] >= 0).all() and (r["safe_dt_index"] >= 0).sum() >= 2
        b = dict(N_w=w["N_whole"], N_s=w["N_safe"], co_w=r["coeffs_whole"], co_s=r["coeffs_safe"], rec=r, need=None)
        _FIX["b"] = b
    return _FIX["b"]


@pytest.mark.parametrize("block_ofs,block_rows", BLOCKS)
def test_fixture_winners_bit_equal_to_the_restatement(built_lib, oracle, block_ofs, block_rows):
    b = fixture_batch()
    states, ofs, st = assert_matches(b, block_ofs=block_ofs, block_rows=block_rows)
    r = b["rec"]
    for j in range(len(ofs) - 1):
        if st[j] != ppo.PLAN_OK:
            continue
        k = int(r["k_safe"][j])
        assert states[ofs[j] + k, :9].tobytes() == r["R"][j].tobytes(), j          # whole row k_safe is R
        assert (states[ofs[j + 1] - 1, 3:] == 0).all(), j                           # the last safe state is at rest


def test_restatement_is_the_reference_fill_x(oracle):
    """Where the reference's SolverGurobi is built, its own fillX gives the restatement's pieces: the same offsets and
    statuses, rows within 1e-12 (its compiled polynomial is not rounded as fq_fill_x's is; test_reference_solver_cpu.py holds
    fq_fill_x to the same bar), the last safe state at rest."""
    from oracle import solver_ref
    if not os.path.exists(solver_ref._SO):
        pytest.skip("oracle/_ref/libsolver_ref.so is not built")
    b = fixture_batch()
    r = b["rec"]
    want = ppo.plan(r, b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC)
    ref = ppo.plan(r, b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, fill_x=solver_ref.fill_x)
    assert want[1].tobytes() == ref[1].tobytes() and want[2].tobytes() == ref[2].tobytes()
    assert np.abs(want[0] - ref[0]).max() <= 1e-12 * max(1.0, np.abs(ref[0]).max())
    for j in range(len(want[2])):
        assert not ref[0][ref[1][j + 1] - 1, 3:].any(), j


def _coeffs(rng, n, N):
    return rng.normal(0.0, 2.0, (n, N, 12))


def edge_batches():
    """(name, batch) of hand-built winners; whole N 10, safe N 4 unless named otherwise."""
    rng = np.random.default_rng(7)
    nan = np.nan
    out = []
    # k_safe = 0; k_safe = n_w - 1 with a safe path; short and long pieces; no whole winner; whole won, safe lost; need_safe
    # 0 and 1 in one batch (k of a corridor without a safe path is n_w - 1 whatever is passed)
    dt_w = [0.3, 0.3, 0.02, 0.8, nan, 0.25, 0.4, 0.07, 0.55]
    dt_s = [0.2, 0.05, 0.9, 0.02, nan, nan, nan, 0.3, 0.013]
    k = [0, 299, 3, 400, 0, 10, 0, 15, 200]
    co_w, co_s = _coeffs(rng, 9, 10), _coeffs(rng, 9, 4)
    nw = [len(ppo.po.fill_x(10, co_w[1], 0.3, DC))]
    assert k[1] == nw[0] - 1
    out.append(("need_always", batch(10, 4, co_w, co_s, dt_w, dt_s, k)))
    need = [1, 1, 1, 1, 0, 1, 0, 1, 0]
    out.append(("need_mixed", batch(10, 4, co_w, co_s, dt_w, dt_s, k, need)))
    # N = 3 whole, 2 safe: dt exactly 2 DC, n = 2 (dt below DC: a knot per sample), equal N
    co_w, co_s = _coeffs(rng, 4, 3), _coeffs(rng, 4, 2)
    b = batch(3, 2, co_w, co_s, [2 * DC, 2 * DC, 0.011, 0.5], [2 * DC, 0.011, 0.004, 2 * DC], [5, 0, 1, 20])
    assert len(ppo.po.fill_x(2, co_s[1], 0.011, DC)) == 2 and len(ppo.po.fill_x(3, co_w[2], 0.011, DC)) == 3
    out.append(("small_n", b))
    co = _coeffs(rng, 3, 6)
    out.append(("equal_N", batch(6, 6, co, co[::-1], [0.1, 0.2, 0.3], [0.3, 0.2, 0.1], [0, 59, 30])))
    # a batch without any plan
    out.append(("none", batch(10, 4, _coeffs(rng, 2, 10), _coeffs(rng, 2, 4), [nan, 0.3], [nan, nan], [0, 5])))
    return out


@pytest.mark.parametrize("block_ofs,block_rows", BLOCKS)
def test_edges_bit_equal_to_the_restatement(block_ofs, block_rows):
    for name, b in edge_batches():
        states, ofs, st = assert_matches(b, block_ofs=block_ofs, block_rows=block_rows)
        r = b["rec"]
        for j in range(len(st)):
            if st[j] != ppo.PLAN_OK:
                assert ofs[j + 1] == ofs[j], (name, j)
                continue
            k, nw = int(r["k_safe"][j]), int(r["n_samples_whole"][j])
            # whole row k_safe keeps its velocity unless it is the whole trajectory's last sample
            assert (states[ofs[j] + k, 3:] == 0).all() == (k == nw - 1), (name, j)
        if name == "need_mixed":
            assert list(st) == [0, 0, 0, 0, 1, 1, 0, 0, 0]
            assert ofs[7] - ofs[6] == r["n_samples_whole"][6]                  # no safe path: the whole X_temp_
        if name == "need_always":
            assert list(st) == [0, 0, 0, 0, 1, 1, 1, 0, 0]
        if name == "none":
            assert list(st) == [1, 1] and ofs[-1] == 0


@pytest.mark.parametrize("block_ofs,block_rows", [(1024, 128), (3, 5)])
def test_capacity(block_ofs, block_rows):
    """cap_states 0, exactly the total, one row short, and mid-batch: a suffix of the succeeding corridors gets
    FQ_PLAN_CAPACITY, nothing is written for them, plan_ofs still counts every corridor."""
    b = dict(edge_batches())["need_mixed"]
    full = ppo.plan(b["rec"], b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, b["need"])
    ofs, total = full[1], int(full[1][-1])
    mid = int(ofs[3]) + 5
    for cap in (0, total, total - 1, mid, int(ofs[3])):
        states, o, st = assert_matches(b, cap, block_ofs=block_ofs, block_rows=block_rows)
        assert o.tobytes() == ofs.tobytes()
        cut = np.flatnonzero(st == ppo.PLAN_CAPACITY)
        ok = np.flatnonzero(st == ppo.PLAN_OK)
        assert len(cut) == 0 or len(ok) == 0 or ok.max() < cut.min()
        if cap == total:
            assert len(cut) == 0 and not np.isnan(states).any()
        if cap == total - 1:
            assert list(cut) == [len(st) - 1]
        f = ppo.filled_rows(ofs, cap)
        assert not np.isnan(states[:f]).any() and np.isnan(states[f:]).all()
    # without a status array the rows are the same
    s1 = emu(b, mid, block_ofs, block_rows, with_status=False)
    assert s1[0].tobytes() == ppo.plan(b["rec"], b["co_w"], b["co_s"], b["N_w"], b["N_s"], DC, b["need"], mid)[0].tobytes()


def test_struct_layout_matches_the_c_compiler(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "faster_b200.h"\n'
                   'int main(void) { printf("%zu %d %d %d", sizeof(fq_pair_plan), FQ_PLAN_OK, FQ_PLAN_NONE, FQ_PLAN_CAPACITY);\n' +
                   "".join('printf(" %%zu", offsetof(fq_pair_plan, %s));\n' % f for f, _ in capi.PairPlan._fields_) + "return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got[0] == C.sizeof(capi.PairPlan)
    assert got[1:4] == [capi.PLAN_OK, capi.PLAN_NONE, capi.PLAN_CAPACITY] == [ppo.PLAN_OK, ppo.PLAN_NONE, ppo.PLAN_CAPACITY]
    assert got[4:] == [getattr(capi.PairPlan, f).offset for f, _ in capi.PairPlan._fields_]
